"""BASELINE configs[2] at full size: query L=400 vs N (default 1M) synthetic HMMs on one GPU,
two-stage cs219 prefilter over the whole shard + Viterbi (with Hit.score, backtrace) on the survivors.
    python tools/config3_probe.py [N] [planted_homologs]
Prints wall-clock per query (host + device, PCIe included) and its breakdown."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hhsuite_b200 as hh  # noqa: E402
from hhsuite_b200 import synth, prefilter  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
    planted = int(sys.argv[2]) if len(sys.argv) > 2 else 3000
    lq = 400
    G = np.load(os.path.join(ROOT, "tests", "golden", "golden_v1.npz"))
    lib219 = G["cs219_lin"]
    qp, qtr, qss, qpav, qcols = synth.query_profile(lq, 1)
    t0 = time.perf_counter()
    base_n = min(n, 100000)
    rep = (n + base_n - 1) // base_n
    base = synth.prepared_db(base_n, seed=1000, query_cols=qcols, planted=64, fast=True)
    L = np.tile(base["L"], rep)[:n]
    ctx = hh.Context()
    # shard: the 100k base repeated (timing only depends on the length distribution)
    p_rows = L.astype(np.int64) + 2
    t_rows = L.astype(np.int64) + 1
    P = np.tile(base["p"], (rep, 1))[:int(p_rows.sum())]
    T = np.tile(base["tr"], (rep, 1))[:int(t_rows.sum())]
    p_off = np.concatenate([[0], np.cumsum(p_rows)[:-1]])
    tr_off = np.concatenate([[0], np.cumsum(t_rows)[:-1]])
    db = hh.TargetDB(ctx, L, P, T, p_off, tr_off)
    del P, T
    # cs219 shard: random states with the targets' lengths + `planted` noisy copies of the query's best states
    prof = hh.capi.build_prefilter_profile(qp, qpav, lib219, 50, 4)
    rng = np.random.default_rng(5)
    cs = synth.cs219_db(n, seed=3, lens=L)
    best = prof[:219].argmax(axis=0).astype(np.uint8)
    ids_planted = rng.choice(n, planted, replace=False)
    for t in ids_planted:
        Lt = int(L[t]); o = int(cs["off"][t])
        a = int(rng.integers(0, max(1, lq - Lt + 1))) if Lt < lq else 0
        seg = best[a:a + Lt].copy()
        noise = rng.random(len(seg)) < 0.25
        seg[noise] = rng.integers(0, 219, int(noise.sum()), dtype=np.uint8)
        cs["seq"][o:o + len(seg)] = seg
    csdb = hh.CsDB(ctx, cs["L"], cs["off"], cs["seq"])
    print(f"setup: {time.perf_counter() - t0:.1f} s for {n} targets, {int(L.sum())} columns", flush=True)

    def one_query():
        tm = {}
        t = time.perf_counter()
        pr = hh.capi.build_prefilter_profile(qp, qpav, lib219, 50, 4)
        tm["profile(host)"] = time.perf_counter() - t
        t = time.perf_counter()
        ids, det = prefilter.prefilter_db(csdb, pr, return_details=True)
        tm["prefilter(2 stages + selection)"] = time.perf_counter() - t
        t = time.perf_counter()
        ctx.set_query(qp, qtr)
        hits, paths = hh.viterbi_search(ctx, db, ids=ids)
        tm["viterbi(survivors)"] = time.perf_counter() - t
        return tm, ids, det, hits

    one_query()
    best_t = None
    for _ in range(3):
        t = time.perf_counter()
        tm, ids, det, hits = one_query()
        tot = time.perf_counter() - t
        if best_t is None or tot < best_t[0]:
            best_t = (tot, tm)
    tot, tm = best_t
    cells_v = float(lq) * float(L[ids].sum())
    print(f"config 3 (N={n}): {tot * 1e3:.1f} ms per query; stage-1 survivors {len(det['first'])}, "
          f"stage-2 survivors {len(ids)} ({len(set(ids.tolist()) & set(ids_planted.tolist()))} of {planted} planted)")
    for k, v in tm.items():
        print(f"   {k}: {v * 1e3:.2f} ms")
    print(f"   viterbi cells {cells_v / 1e9:.2f} G -> {cells_v / tm['viterbi(survivors)'] / 1e9:.1f} GCUPS wall; "
          f"prefilter {lq * float(L.sum()) / tm['prefilter(2 stages + selection)'] / 1e12:.2f} Tcells/s wall")
    print(f"   best hit score {hits['hit_score'].max():.2f}")


if __name__ == "__main__":
    main()
