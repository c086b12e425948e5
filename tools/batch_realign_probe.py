"""MAC realignment of a query batch: one query at a time vs one hhg_mac_realign_batch call.

16 queries of mixed length search a raw 20 000-target shard (one hhg_viterbi_search_batch call); the <= 500 best hits of
each query are then realigned two ways, alternately in one process:
  (a) per query: hhg_db_apply_null_model, hhg_mac_query_set, hhg_mac_realign
  (b) hhg_mac_query_set_batch + one hhg_mac_realign_batch over the raw records
Each arm is timed with a host clock around calls that end in a device synchronise; after a warm-up the best of
--reps runs is reported, and the two arms' outputs are compared byte for byte.
    python tools/batch_realign_probe.py [--reps 5] [--hits 500]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hhsuite_b200 as hh  # noqa: E402
from hhsuite_b200 import synth  # noqa: E402

Q_LENS = (60, 95, 120, 150, 180, 200, 230, 260, 300, 340, 400, 480, 560, 700, 850, 1000)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hits", type=int, default=500)
    ap.add_argument("--targets", type=int, default=20000)
    args = ap.parse_args()
    rng = np.random.default_rng(3)
    qs = [synth.query_profile(L, 200 + k) for k, L in enumerate(Q_LENS)]
    nq = len(qs)
    db_h = synth.prepared_db(args.targets, seed=77, fast=True)
    t_pav = rng.dirichlet(np.ones(20) * 8, args.targets).astype(np.float32)
    q_pav = np.stack([q[3] for q in qs]).astype(np.float32)
    ctx = hh.Context()
    db = hh.TargetDB(ctx, db_h["L"], db_h["p"], db_h["tr"], db_h["p_off"], db_h["tr_off"], pav=t_pav)
    # first pass: every query against the whole shard in one batch search; keep each query's best hits
    all_ids = np.arange(args.targets, dtype=np.int32)
    hh.capi.query_set_batch(ctx, [(q[0], q[1]) for q in qs], q_pav=q_pav)
    req_q = np.repeat(np.arange(nq, dtype=np.int32), args.targets)
    hits, paths = hh.capi.viterbi_search_batch(ctx, db, req_q, np.tile(all_ids, nq), columnscore=1)
    rq, tg, vits = [], [], []
    for q in range(nq):
        h = hits[q * args.targets:(q + 1) * args.targets]
        best = np.argsort(-h["hit_score"], kind="stable")[:args.hits]
        for t in best:
            if h["nsteps"][t] == 0:
                continue
            i_s, j_s, _ = hh.expand_path(h[t], paths)
            rq.append(q); tg.append(int(t))
            vits.append((int(h["i1"][t]), int(h["i2"][t]), int(h["j1"][t]), int(h["j2"][t]), int(h["nsteps"][t]), i_s, j_s))
    rq = np.array(rq, np.int32); tg = np.array(tg, np.int32)
    cells = float(np.sum((np.array(Q_LENS)[rq] + 1.0) * (db_h["L"][tg] + 1.0)))
    qlin = [hh.capi.log2lin(q[1]) for q in qs]
    by_q = [np.nonzero(rq == q)[0] for q in range(nq)]

    def per_query():
        out_h = np.zeros(len(tg), hh.capi.MAC_HIT_DTYPE)
        out_p = [None] * len(tg)
        for q in range(nq):
            db.apply_null_model(q_pav[q], None, 1)
            hh.capi.mac_query_set(ctx, qs[q][0], qlin[q])
            m = by_q[q]
            h, p = hh.capi.mac_realign(ctx, db, tg[m], [vits[k] for k in m])
            out_h[m] = h
            for k, r in enumerate(m):
                out_p[r] = p[k]
        return out_h, out_p

    def batched():
        hh.capi.mac_query_set_batch(ctx, [(q[0], lin) for q, lin in zip(qs, qlin)], q_pav)
        return hh.capi.mac_realign_batch(ctx, db, rq, tg, vits, columnscore=1)

    arms = {"per_query": per_query, "batch": batched}
    times = {k: [] for k in arms}
    results = {}
    for name, fn in arms.items():     # warm-up
        results[name] = fn()
    for _ in range(args.reps):
        for name, fn in arms.items():
            t0 = time.perf_counter()
            fn()
            times[name].append(time.perf_counter() - t0)
    (ha, pa), (hb, pb_) = results["per_query"], results["batch"]
    fields = [f for f in hh.capi.MAC_HIT_DTYPE.names if f != "path_off"]
    same = all(ha[f].tobytes() == hb[f].tobytes() for f in fields) and all(
        a[f].tobytes() == b[f].tobytes() for a, b in zip(pa, pb_) for f in ("i", "j", "states", "P_posterior"))
    name, limit = card()
    best = {k: min(v) for k, v in times.items()}
    print(f"card: {name}, power limit {limit}")
    print(f"{nq} queries (Lq {min(Q_LENS)}..{max(Q_LENS)}), {len(tg)} hits of a raw {args.targets}-target shard, "
          f"{cells / 1e9:.2f} G cells")
    for k in arms:
        print(f"  {k:10s}: best {best[k] * 1e3:8.1f} ms of {args.reps}  (all: {', '.join(f'{t * 1e3:.1f}' for t in times[k])})")
    print(f"  outputs identical: {same}")
    print(json.dumps(dict(card=name, power_limit=limit, queries=nq, hits=len(tg), gcells=cells / 1e9,
                          per_query_ms=best["per_query"] * 1e3, batch_ms=best["batch"] * 1e3, identical=bool(same))))
    db.close(); ctx.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
