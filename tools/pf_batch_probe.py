"""cs219 prefilter of a query batch: the per-query loop of prefilter.prefilter_db vs one prefilter.prefilter_db_batch.

configs[2] shape: Q queries against a seeded synthetic cs219 shard of --n sequences (median length 200); each query's
profile is built from a synthetic query HMM with the cs219 library, and noisy copies of its best states are planted in
the shard as bench.py does (about 3 000 per batch).  Three batches: 16 queries of Lq = 400; 16 queries of Lq = 512,
where the single-query kernel runs at the batch kernel's register width (WB = 8, 225 KB of shared memory, one CTA per
SM), so the two ungapped arms differ only in the batch kernel's work items and slab descriptors; and 16 queries of
mixed length (Lq 50..1500, where the slab packing of short queries matters).  For each batch the two arms alternate in
one process, after a warm-up; both the
whole prefilter (both stages, selection and E-value cut) and the ungapped stage alone (hhg_prefilter_ungapped_run per
query vs one hhg_prefilter_ungapped_batch_run) are timed with a host clock around calls that end in a device
synchronise, best of --reps.  The probe asserts that the two arms return identical survivor lists.
    python tools/pf_batch_probe.py [--n 300000] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hhsuite_b200 as hh  # noqa: E402
from hhsuite_b200 import synth  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=300_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    rng = np.random.default_rng(12)
    d = synth.cs219_db(args.n, 21)
    seq = d["seq"].copy()
    batches = {"16 x Lq 400": [400] * 16,
               "16 x Lq 512": [512] * 16,
               "16 mixed Lq 50..1500": sorted(int(x) for x in rng.integers(50, 1501, 16))}
    lib219 = np.load(os.path.join(ROOT, "tests", "golden", "golden_v1.npz"))["cs219_lin"]
    profs = {}
    for name, lens in batches.items():
        profs[name] = []
        for k, Lq in enumerate(lens):
            qp, _, _, qpav, _ = synth.query_profile(Lq, seed=100 + k + 50 * len(profs))
            p = hh.capi.build_prefilter_profile(qp, qpav, lib219, 50, 4)
            # noisy copies of the query's best states, as bench.py plants them, so both stages have survivors
            best = p[:219].argmax(axis=0).astype(np.uint8)
            for t in rng.choice(args.n, 3000 // len(lens), replace=False):
                Lt, o = int(d["L"][t]), int(d["off"][t])
                a = int(rng.integers(0, max(1, Lq - Lt + 1))) if Lt < Lq else 0
                seg = best[a:a + Lt].copy()
                noise = rng.random(len(seg)) < 0.25
                seg[noise] = rng.integers(0, 219, int(noise.sum()), dtype=np.uint8)
                seq[o:o + len(seg)] = seg
            profs[name].append(p)
    ctx = hh.Context()
    csdb = hh.CsDB(ctx, d["L"], d["off"], seq)
    kw = dict(min_prefilter_hits=100, maxnumdb=20000)
    report = []
    for name, ps in profs.items():
        def loop():
            return [hh.prefilter.prefilter_db(csdb, p, **kw) for p in ps]

        def batch():
            return hh.prefilter.prefilter_db_batch(csdb, ps, **kw)

        def loop_ungapped():
            for p in ps:
                csdb.run(p, 50)
            ctx.sync()

        def batch_ungapped():
            csdb.run_batch(ps, 50)
            ctx.sync()

        arms = {"loop": loop, "batch": batch, "loop_ungapped": loop_ungapped, "batch_ungapped": batch_ungapped}
        out = {k: fn() for k, fn in arms.items()}                      # warm-up
        same = len(out["loop"]) == len(out["batch"]) and all(
            a.tolist() == b.tolist() for a, b in zip(out["loop"], out["batch"]))
        assert same, f"{name}: survivor lists differ"
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                t0 = time.perf_counter()
                fn()
                times[k].append(time.perf_counter() - t0)
        best = {k: min(v) * 1e3 for k, v in times.items()}
        surv = int(sum(len(x) for x in out["batch"]))
        print(f"{name}: {args.n} sequences, {surv} survivors in all")
        for k in arms:
            print(f"  {k:15s}: best {best[k]:8.2f} ms of {args.reps}  (all: {', '.join(f'{t * 1e3:.2f}' for t in times[k])})")
        print(f"  survivor lists identical: {same}")
        report.append(dict(batch=name, lens=batches[name], survivors=surv, identical=bool(same),
                           **{f"{k}_ms": v for k, v in best.items()}))
    gpu, limits = card()
    print(f"card: {gpu}, power limit / max SM clock: {limits}")
    print(json.dumps(dict(card=gpu, power_limit_max_sm_clock=limits, n=args.n, reps=args.reps, results=report)))
    csdb.close(); ctx.close()


if __name__ == "__main__":
    main()
