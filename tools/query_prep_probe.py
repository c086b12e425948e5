"""Query preparation of one hhblits iteration, timed stage by stage next to the compiled reference (1 thread):
alignment -> HMM (hhg_msa_to_hmm), context-specific pseudocounts for the HMM and for the prefilter profile
(hhg_query_context_pseudocounts), prefilter byte profile (hhg_prefilter_build_profile).  Then the context
pseudocounts alone at L = 400 and 1 500: the score kernel's time (torch.profiler, CUDA activities) and the call's time,
with the card's name and power limit.  --engine picks the engine: crf (context_data.crf, the default) or lib
(context_data.lib, -contxt with the generative context library).
    python tools/query_prep_probe.py [--engine crf|lib]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hhsuite_b200 as hhg  # noqa: E402
from hhsuite_b200 import capi, synth  # noqa: E402
from oracle.binding import RefShim  # noqa: E402
from tests import crf_cases  # noqa: E402


def best(fn, n=5):
    ts = []
    for _ in range(n):
        t0 = time.perf_counter(); out = fn(); ts.append(time.perf_counter() - t0)
    return min(ts) * 1e3, out


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip() or "unknown card"


def context_pc_times(ctx, crf, pb, lengths=(400, 1500), calls=20):
    """(L, mean score-kernel time in ms, best call time in ms) of hhg_query_context_pseudocounts, query-HMM admixture."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    rows = []
    for L in lengths:
        f, neff_m, neff_hmm = crf_cases.mixed(np.random.default_rng([L, 3]), L)
        run = lambda: crf.pseudocounts(f, neff_m, neff_hmm, pb, capi.Admix.hhm())  # noqa: E731
        run()
        t_call, _ = best(run, calls)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                run()
        ks = [e.time_range.elapsed_us() for e in prof.events() if "k_crf_scores" in e.name or "k_lib_scores" in e.name]
        assert len(ks) == calls, f"{len(ks)} score kernels in the trace, expected {calls}"
        t_kernel = sum(ks) / len(ks) / 1e3
        rows.append((L, t_kernel, t_call))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", choices=("crf", "lib"), default="crf")
    args = ap.parse_args()
    r = RefShim(nocontxt=True, maxres=4096)
    pb, R = r.pb(), r.R()
    ctx = hhg.Context()
    if args.engine == "crf":
        crf, ref_pc = capi.Crf(ctx, r.crf_text()), lambda h, engine: r.context_pc(h["f"], h["neff_m"], h["neff_hmm"], engine=engine)
    else:
        from oracle.ctxlib_binding import LibRef
        from tests import ctxlib_cases as cc
        lr = LibRef()
        lr.set_pb(pb)                     # one background on both sides, as for the CRF
        crf = capi.ContextLibrary(ctx, lr.lib_text())
        ref_pc = lambda h, engine: lr.context_pc_lib(lr.lib_text(), cc.CSW, cc.CSB, h["f"], h["neff_m"], h["neff_hmm"],  # noqa: E731
                                                     *cc.admix_args((cc.ADMIX_HHM, cc.ADMIX_PREFILTER)[engine]))
    d = tempfile.mkdtemp()
    qa = os.path.join(ROOT, "oracle", "_ref", "data", "query.a3m")
    cases = [("synthetic L=400 N=300", synth.a3m_text(400, 300, 5, ident=0.5).encode())]
    if os.path.exists(qa):
        cases.append(("data/query.a3m L=431 N=59", open(qa, "rb").read()))
    for name, a3m in cases:
        path = os.path.join(d, "q.a3m")
        open(path, "wb").write(a3m)
        t_msa, raw = best(lambda: capi.msa_to_hmm(ctx, a3m, pb))
        t_hmm, (p, pav) = best(lambda: crf.pseudocounts(raw["f"], raw["neff_m"], raw["neff_hmm"], pb, capi.Admix.hhm()))
        t_pf, (ppf, pavpf) = best(lambda: crf.pseudocounts(raw["f"], raw["neff_m"], raw["neff_hmm"], pb, capi.Admix.prefilter()))
        t_tr, q = best(lambda: capi.query_from_a3m(ctx, a3m, R, pb))
        rt_msa, ref = best(lambda: r.msa_to_hmm(path, capL=1000, capN=2000), 3)
        rt_pc, (rp, rpav) = best(lambda: ref_pc(ref, 0), 3)
        same = np.array_equal(p.view(np.uint32), rp.view(np.uint32)) and np.array_equal(raw["f"].view(np.uint32), ref["f"].view(np.uint32))
        print(f"{name} [{args.engine}]: library  alignment->HMM {t_msa:.2f} ms | context pc (HMM) {t_hmm:.2f} ms | context pc (prefilter) {t_pf:.2f} ms"
              f" | transitions+nocontxt path {t_tr:.2f} ms || reference (OpenMP as built, {os.cpu_count()} cpus visible)"
              f" alignment->HMM {rt_msa:.2f} ms | context pc {rt_pc:.2f} ms || identical: {same}")
    for L, t_kernel, t_call in context_pc_times(ctx, crf, pb):
        print(f"context pc [{args.engine}, {crf.n_states} states, window {crf.window}] L={L}: score kernel "
              f"{t_kernel:.3f} ms, call {t_call:.2f} ms ({card()})")
    crf.close(); ctx.close()


if __name__ == "__main__":
    main()
