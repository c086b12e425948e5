"""What staging from the database's own A3M records costs (DESIGN 4.12): a staged shard over a record source, a staged
shard over a page-locked store of the same database and the resident raw shard, alternated in one process on the
configs[2] shape (Lq = 400, ~3 000 prefilter survivors).

  stage     a cold stage call of the survivors (every one missing), record source vs store; a warm call (all resident)
  split     host scan / build (host parse + kernels) / gather of one cold record stage (the HHG_TIMING line)
  search    null model + search per query: one cold query, then a stream of 16 related queries, for all three arms

The database is --distinct synthetic alignments repeated to --n records (timing does not depend on which record an id
names); the cs219 sequences are random, so the prefilter keeps its minimum number of hits, set to the survivor count
wanted.  Times are best of --reps with the spread (max - min)."""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "nvidia-smi not available"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--distinct", type=int, default=2000)
    ap.add_argument("--survivors", type=int, default=3000)
    ap.add_argument("--lq", type=int, default=400)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import hhsuite_b200 as hh
    from hhsuite_b200 import synth

    if not torch.cuda.is_available():
        sys.exit("stage_records_probe needs an H100: there is nothing to measure without one")
    print("card:", card_state(), "(sampled before the run)")
    ctx = hh.Context(device=0)
    rng = np.random.default_rng(1)
    G = np.load(os.path.join(ROOT, "tests", "golden", "golden_v1.npz"))

    def host_ms(fn):
        ctx.sync(); t = time.perf_counter(); fn(); ctx.sync()
        return (time.perf_counter() - t) * 1e3

    def stat(xs):
        return f"{min(xs):9.3f} ms (spread {max(xs) - min(xs):.3f})"

    # ---- the database: --distinct alignments (median ~200 columns, 2..60 sequences) repeated to --n records
    Ld = synth.lengths(a.distinct, rng, median=200, lo=20, hi=1200)
    texts = [synth.a3m_text(int(L), int(rng.integers(2, 60)), 7000 + k, f"t{k}", with_ss=k % 4 == 0).encode() + b"\0"
             for k, L in enumerate(Ld)]
    reps_db = (a.n + a.distinct - 1) // a.distinct
    data = b"".join(texts)
    ln1 = np.array([len(t) for t in texts], np.int64)
    off1 = np.concatenate([[0], np.cumsum(ln1)[:-1]]).astype(np.int64)
    n = a.distinct * reps_db
    off, ln = np.tile(off1, reps_db), np.tile(ln1, reps_db)
    t = time.perf_counter()
    db = hh.TargetDB.from_a3m(ctx, data, off, ln, G["R"], G["pb"])
    load_s = time.perf_counter() - t
    L = db.Lh.copy()
    store = hh.HostStore.from_db(ctx, db, has_ss=True)
    t = time.perf_counter()
    src = hh.RecordSource.from_a3m(ctx, data, off, ln, G["R"], G["pb"], has_ss=True)
    src_ms = (time.perf_counter() - t) * 1e3
    cs = synth.cs219_db(n, 7, lens=L)
    cst = hh.CsDB(ctx, cs["L"], cs["off"], cs["seq"])
    cap_t = 3 * a.survivors
    cap_c = int(cap_t * float(L.mean()) * 1.3)
    sdb_s, sdb_r = hh.StagedDB(ctx, store, cap_t, cap_c), hh.StagedDB(ctx, src, cap_t, cap_c)
    print(f"database: {n} A3M records ({len(data) / 1e6:.1f} MB of distinct text), {int(L.sum())} columns; "
          f"resident load {load_s:.1f} s, record source created in {src_ms:.2f} ms; staged shards: {cap_t} slots, {cap_c} columns")

    # ---- cold and warm stage calls: fresh random survivors each time, the same ids for both staged arms
    cold_s, cold_r, warm_r = [], [], []
    for rep in range(a.reps + 1):                           # rep 0 warms up
        ids = rng.choice(n, a.survivors, replace=False).astype(np.int32)
        ms_s = host_ms(lambda: sdb_s.stage(ids))
        ms_r = host_ms(lambda: sdb_r.stage(ids))
        assert sdb_r.last_stats["copied"] >= a.survivors // 2 and sdb_r.last_stats.tobytes() == sdb_s.last_stats.tobytes()
        ms_w = host_ms(lambda: sdb_r.stage(ids))
        assert sdb_r.last_stats["copied"] == 0
        if rep:
            cold_s.append(ms_s); cold_r.append(ms_r); warm_r.append(ms_w)
    print(f"stage    cold, {a.survivors} survivors, store-backed:   {stat(cold_s)}")
    print(f"stage    cold, {a.survivors} survivors, record source:  {stat(cold_r)}")
    print(f"stage    warm (all resident), record source:           {stat(warm_r)}")

    # ---- where a cold record stage spends its time (HHG_TIMING line of hhg_db_stage, stderr)
    ids = rng.choice(n, a.survivors, replace=False).astype(np.int32)
    os.environ["HHG_TIMING"] = "1"
    with tempfile.TemporaryFile(mode="w+") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            total = host_ms(lambda: sdb_r.stage(ids))
        finally:
            os.dup2(saved, 2); os.close(saved)
            os.environ.pop("HHG_TIMING")
        f.seek(0)
        line = [x for x in f.read().splitlines() if "record stage" in x]
    print(f"split    one cold record stage, {total:.3f} ms in all: {line[-1].split(': ', 1)[1] if line else 'no timing line'}")
    m = re.search(r"host scan ([\d.]+) ms, build ([\d.]+) ms, gather ([\d.]+) ms", line[-1] if line else "")
    if m:
        print(f"split    shares: scan {float(m[1]) / total:.0%}, build {float(m[2]) / total:.0%}, gather {float(m[3]) / total:.0%}")

    # ---- search: one cold query, then 16 related queries (one profile, perturbed)
    lib = G["cs219_lin"]
    base = synth.query_profile(a.lq, 3)
    qs = []
    for k in range(16):
        p = base[0].copy()
        noise = rng.dirichlet(np.ones(20), a.lq).astype(np.float32)
        p[1:-1] = (1 - 0.02 * k) * p[1:-1] + 0.02 * k * noise
        qs.append((p, base[1], p[1:-1].mean(axis=0).astype(np.float32)))
    pfk = dict(min_prefilter_hits=a.survivors, maxnumdb=a.survivors)

    def resident(q):
        db.apply_null_model(q[2])
        return hh.pipeline.search(ctx, db, cst, q[0], q[1], q[2], lib, **pfk)

    def staged(sdb, q):
        return hh.pipeline.search_staged(ctx, sdb, cst, q[0], q[1], q[2], lib, **pfk)

    far = (np.arange(cap_t, dtype=np.int32) * 7 + 1) % n       # other records: the next staged search is cold
    resident(qs[0]); staged(sdb_s, qs[0]); staged(sdb_r, qs[0])
    res = {k: [] for k in ("c_res", "c_st", "c_rec", "s_res", "s_st", "s_rec")}
    hits = [0, 0]
    for rep in range(a.reps):
        res["c_res"].append(host_ms(lambda: resident(qs[0])))
        for key, sdb in (("st", sdb_s), ("rec", sdb_r)):
            sdb.stage(far)
            res["c_" + key].append(host_ms(lambda: staged(sdb, qs[0])))
        res["s_res"].append(host_ms(lambda: [resident(q) for q in qs]) / 16)
        for key, sdb in (("st", sdb_s), ("rec", sdb_r)):
            sdb.stage(far)
            hits = [0, 0]

            def stream16():
                for q in qs:
                    staged(sdb, q)
                    hits[0] += int(sdb.last_stats["hits"]); hits[1] += int(sdb.last_stats["copied"])
            res["s_" + key].append(host_ms(stream16) / 16)
    want, got = resident(qs[5]), staged(sdb_r, qs[5])
    assert want[0].tolist() == got[0].tolist() and [h.score for h in want[1]] == [h.score for h in got[1]]
    print(f"search   one cold query, resident (null model + search):     {stat(res['c_res'])}")
    print(f"search   one cold query, staged from the store:              {stat(res['c_st'])}")
    print(f"search   one cold query, staged from the records:            {stat(res['c_rec'])}")
    print(f"search   per query in a stream of 16 related, resident:      {stat(res['s_res'])}")
    print(f"search   per query in a stream of 16 related, store:         {stat(res['s_st'])}")
    print(f"search   per query in a stream of 16 related, records:       {stat(res['s_rec'])}   "
          f"({hits[0]} resident hits, {hits[1]} targets built over the 16)")
    print("card:", card_state(), "(sampled after the run)")
    sdb_r.close(); sdb_s.close(); src.close(); store.close(); cst.close(); db.close(); ctx.close()


if __name__ == "__main__":
    main()
