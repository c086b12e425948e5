"""A/B of the forward kernel's strip heights on the headline shard, device-timed (CUDA events around k_viterbi).

usage: python tools/vit_ab.py [--rounds 10] [--lib PATH] [--long-targets 25000] [--json FILE]

Builds bench.py's headline shard (same seeds, through bench.headline_shard), then one context per variant (the
strip height is read from HHG_STRIP_ROWS when a context is created):
  lq400-R16, lq400-R12  : the headline plan, Lq = 400 against the whole 100k shard
  lq1500-R16, lq1500-R12: Lq = 1500 (bench's configs[4] query) against the shard's first --long-targets targets
Each round runs every variant once with plan.run_timed(), in turn, so slow drifts of the clock hit all variants alike.
Per variant it prints the median and the min..max spread of the forward-kernel ms and its GCUPS (query_L x sum
target_L / kernel time), next to the GPU name, power limit and the SM clock sampled over the rounds.
--lib runs another build of libhhg.so (e.g. the parent commit's) through this tree's Python bindings.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", default=None, help="libhhg.so to measure (default: this tree's build)")
    ap.add_argument("--strips", default="16,12", help="strip heights to compare")
    ap.add_argument("--long-targets", type=int, default=25000, help="targets of the Lq = 1500 variants (0: none)")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if args.lib:
        os.environ["HHG_LIB"] = os.path.abspath(args.lib)

    import torch
    import bench
    import hhsuite_b200 as hh
    from hhsuite_b200 import build as hbuild, synth

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    shard_args = types.SimpleNamespace(lq=400, targets=100000)
    qprof, db_h, _ = bench.headline_shard(shard_args, 0, 1)
    q1500 = synth.query_profile(1500, seed=2)

    variants = []   # (name, ctx, plan, cells)
    first = None
    strips = [int(s) for s in args.strips.split(",")]
    for lq, q, n in ((400, qprof, None), (1500, q1500, args.long_targets)):
        if n == 0:
            continue
        for R in strips:
            os.environ["HHG_STRIP_ROWS"] = str(R)
            ctx = hh.Context(device=0)
            ctx.set_query(q[0], q[1])
            if first is None:   # one resident shard, shared by every context on the device
                first = hh.TargetDB(ctx, db_h["L"], db_h["p"], db_h["tr"], db_h["p_off"], db_h["tr_off"])
            ids = None if n is None else np.arange(min(n, first.n), dtype=np.int32)
            plan = hh.Plan(ctx, first, ids)
            variants.append((f"lq{lq}-R{R}", ctx, plan, float(plan.cells)))
    os.environ.pop("HHG_STRIP_ROWS", None)

    for _ in range(args.warmup):
        for _, _, plan, _ in variants:
            plan.run_timed()
    sampler = bench.ClockSampler(0)
    sampler.start()
    sampler.mark_begin()
    ms = {v[0]: [] for v in variants}
    for _ in range(args.rounds):
        for name, _, plan, _ in variants:
            ms[name].append(plan.run_timed()[0])
    sampler.mark_end()
    clocks = sampler.stop()
    gpu = bench.gpu_info(dev)

    lib = os.environ.get("HHG_LIB") or hbuild.OUT
    print(f"library {lib}")
    print(f"GPU {gpu['name']}, power limit {gpu['power_limit_w']} W, SM clock median {clocks['sm_mhz']} MHz "
          f"(max {clocks['sm_max_mhz']}, {clocks['samples']} samples, reasons {clocks['reasons']}); {args.rounds} rounds")
    out = {"lib": lib, "gpu": gpu, "clocks": clocks, "rounds": args.rounds, "variants": {}}
    for name, _, plan, cells in variants:
        a = np.array(ms[name])
        med = float(np.median(a))
        g = cells / (med * 1e-3) / 1e9
        print(f"  {name:12s} k_viterbi {med:8.3f} ms  (min {a.min():.3f} .. max {a.max():.3f}, spread "
              f"{(a.max() - a.min()) / med * 100:.2f} %)  {g:7.1f} GCUPS  cells {cells:.4g}")
        out["variants"][name] = {"ms_median": med, "ms_min": float(a.min()), "ms_max": float(a.max()), "gcups": g,
                                 "cells": cells, "ms": a.tolist()}
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    for _, _, plan, _ in variants:
        plan.close()
    first.close()
    for _, ctx, _, _ in variants:
        ctx.close()


if __name__ == "__main__":
    main()
