"""What column score 5 (the local amino-acid composition correction, k_local_bg; DESIGN 4.13) costs next to column score
1, alternated in one process on the synthetic database of DESIGN 4.12 (N random profiles, 112-byte records):

  apply     hhg_db_apply_null_model over the whole resident raw shard, columnscore 5 vs 1
  batch     hhg_viterbi_search_batch of 16 queries (Lq = 400, --survivors random targets each), columnscore 5 (the named
            targets divided in the shard first) vs 1 (the null model fused into the operand stream)

Device times from CUDA events on the context stream; best of --reps and the spread (max - min).  The card's name and
power limit are read in the same run."""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

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
    ap.add_argument("--n", type=int, default=300000)
    ap.add_argument("--survivors", type=int, default=3000)
    ap.add_argument("--lq", type=int, default=400)
    ap.add_argument("--queries", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import hhsuite_b200 as hh
    from hhsuite_b200 import capi, synth

    if not torch.cuda.is_available():
        sys.exit("localbg_probe needs an H100: there is nothing to measure without one")
    print("card:", card_state(), "(sampled before the run)")
    stream = torch.cuda.current_stream()
    ctx = hh.Context(device=0, stream=stream.cuda_stream)
    rng = np.random.default_rng(1)

    def dev_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream); fn(); e1.record(stream); e1.synchronize()
        return e0.elapsed_time(e1)

    L = synth.lengths(a.n, rng)
    cols = np.zeros(int(L.sum()), capi.COLREC_DTYPE)
    cols["p"] = rng.random((len(cols), 20), dtype=np.float32)
    pav = rng.dirichlet(np.ones(20), a.n).astype(np.float32)
    db = hh.TargetDB.from_packed(ctx, L, cols, pav)
    del cols
    print(f"shard: {a.n} profiles, {int(L.sum())} columns")
    pb = synth._PB.astype(np.float32)
    qs = [synth.query_profile(a.lq, 10 + k) for k in range(a.queries)]
    q_pav = np.stack([q[3] for q in qs]).astype(np.float32)
    q5 = [capi.query_local_background(ctx, q[0], pb) for q in qs]
    rq = np.repeat(np.arange(a.queries, dtype=np.int32), a.survivors)
    ids = rng.integers(0, a.n, len(rq)).astype(np.int32)

    def batch(cs):
        capi.query_set_batch(ctx, [(q5[k] if cs == 5 else qs[k][0], qs[k][1]) for k in range(a.queries)], q_pav=q_pav)
        return dev_ms(lambda: capi.viterbi_search_batch(ctx, db, rq, ids, columnscore=cs, pb=pb))

    arms = {"apply 1": lambda: dev_ms(lambda: db.apply_null_model(q_pav[0], pb, 1)),
            "apply 5": lambda: dev_ms(lambda: db.apply_null_model(None, pb, 5)),
            "batch 1": lambda: batch(1), "batch 5": lambda: batch(5)}
    for f in arms.values():           # warm-up of every shape
        f()
    t = {k: [] for k in arms}
    for _ in range(a.reps):
        for k, f in arms.items():
            t[k].append(f())
    for k, v in t.items():
        print(f"{k:8s}: best {min(v):9.3f} ms  spread {max(v) - min(v):7.3f} ms")
    print(f"batch: {a.queries} queries x {a.survivors} targets, Lq = {a.lq}, {len(np.unique(ids))} distinct targets")
    print("card:", card_state(), "(sampled after the run)")
    db.close(); ctx.close()


if __name__ == "__main__":
    main()
