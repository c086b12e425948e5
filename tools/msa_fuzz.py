"""Randomised parity check of the alignment -> HMM path against the compiled reference, without a GPU: the host scanner
(hhg_a3m_parse) on random A3M / FASTA-like alignments under all three match-state rules, and the product's CUDA kernels
run by the CPU emulation (tests/emul) with random filter options and both weighting modes.
    python tools/msa_fuzz.py [seed] [n_scanner] [n_kernels]
Inputs the scanner rejects are checked to make the reference fail too (in a subprocess: it exits)."""
import ctypes as C
import math
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from hhsuite_b200 import capi, synth  # noqa: E402
from oracle.binding import RefShim  # noqa: E402
from tests.msa_cases import rand_a3m, rand_fasta  # noqa: E402


def same_scan(a, o):
    rows = o["keep"] > 0
    return (a["L"] == o["L"] and a["N_in"] == o["N_in"] and np.array_equal(a["X"][:, 1:-1], o["X"][:, 1:-1])
            and np.array_equal(a["I"][rows][:, :-1], o["I"][rows][:, :-1]) and np.array_equal(a["nres"], o["nres"])
            and np.array_equal(a["ksort"], o["ksort"]) and a["kfirst"] == o["kfirst"])


def main():
    seed = int(sys.argv[1]) if len(sys.argv) > 1 else 1
    n_scan = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    n_kern = int(sys.argv[3]) if len(sys.argv) > 3 else 40
    rng = np.random.default_rng(seed)
    r = RefShim()
    d = tempfile.mkdtemp()
    path = os.path.join(d, "x.a3m")
    one = os.path.join(d, "one.py")
    open(one, "w").write(f"import sys; sys.path.insert(0, {ROOT!r})\nfrom oracle.binding import RefShim\n"
                         "r = RefShim(); r.set_M(int(sys.argv[2]), int(sys.argv[3])); r.msa_to_hmm(sys.argv[1]); print('OK')\n")
    bad = errs = agree = 0
    for it in range(n_scan):
        for (M, Mg) in ((1, 50), (2, 50), (2, 25), (3, 50)):
            t = rand_a3m(rng) if M == 1 else rand_fasta(rng)
            open(path, "wb").write(t)
            try:
                a = capi.a3m_parse(t, capi.MsaParams.defaults(M=M, Mgaps=Mg))
            except capi.HhgError:
                errs += 1
                p = subprocess.run([sys.executable, one, path, str(M), str(Mg)], capture_output=True, text=True)
                agree += "OK" not in p.stdout
                continue
            r.set_M(M, Mg)
            if not same_scan(a, r.msa_to_hmm(path)):
                bad += 1; print("scanner MISMATCH", it, M, Mg); open(os.path.join(d, f"bad_{it}_{M}.a3m"), "wb").write(t)
    r.set_M(1, 50)
    print(f"scanner: {4 * n_scan} alignments, {bad} mismatches; {errs} rejected, the reference fails on {agree} of them")

    lib_path = os.path.join(ROOT, "tests", "emul", "libmsaemul.so")
    subprocess.check_call(["g++", "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-DHHG_EMUL", "-o",
                           lib_path, os.path.join(ROOT, "tests", "emul", "msa_emul.cpp")])
    lib = C.CDLL(lib_path)
    lib.emul_msa_to_hmm.argtypes = [C.c_char_p, C.c_longlong, C.c_void_p, C.c_float] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 7
    lg2 = np.zeros(1025, np.float32); dif = np.zeros(1025, np.float32); prev = np.float32(0)
    for i in range(1, 1025):
        lg2[i] = np.float32(math.log(1024 + i) * 1.442695041 - 10.0)
        dif[i - 1] = np.float32(float(np.float32(lg2[i] - prev)) * 1.2352E-4); prev = lg2[i]
    S = np.ascontiguousarray(r.S(), np.float32); pb = r.pb()
    kb = kr = 0
    for it in range(n_kern):
        L = int(rng.integers(5, 90)); n = int(rng.integers(2, 70))
        t = synth.a3m_text(L, n, int(rng.integers(1, 10 ** 6)), ident=float(rng.uniform(0.3, 0.97)),
                           dup_frac=float(rng.uniform(0, 0.7)), with_ss=bool(rng.random() < 0.2)).encode()
        filt = (int(rng.choice([15, 40, 60, 75, 90, 95, 100])), int(rng.choice([0, 0, 20, 50, 80])),
                int(rng.choice([0, 0, 15, 30, 50])), float(rng.choice([-20.0, -20.0, 0.0, 0.3])), int(rng.choice([0, 3, 5, 10, 100])))
        wg = int(rng.random() < 0.3)
        open(path, "wb").write(t)
        ip = np.array([65535, 32765, 20001, filt[0], filt[1], filt[2], filt[4], wg, 1, 50], np.int32)
        dims = np.zeros(4, np.int32); keep = np.zeros(200, np.int8); wgv = np.zeros(200, np.float32)
        f = np.zeros(102 * 20, np.float32); tr = np.zeros(101 * 7, np.float32); neff = np.zeros(3 * 101, np.float32); nh = np.zeros(1, np.float32)
        q = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        lib.emul_msa_to_hmm(t, len(t), q(ip), C.c_float(filt[3]), q(S), q(pb), q(lg2), q(dif), 64, q(dims), q(keep), q(wgv), q(f),
                            q(tr), q(neff), q(nh))
        if dims[3] != 0:
            continue                                   # the reference exits on this input
        o = r.msa_to_hmm(path, filt=filt, wg=wg)
        Lm, N = int(dims[0]), int(dims[1]); kr += 1
        ok = (int(dims[2]) == o["N_filtered"] and np.array_equal(keep[:N], o["keep"])
              and np.array_equal(f[:(Lm + 2) * 20].view(np.uint32), o["f"].ravel().view(np.uint32))
              and np.array_equal(tr[:(Lm + 1) * 7].view(np.uint32), o["tr"].ravel().view(np.uint32))
              and np.array_equal(neff[:Lm + 1].view(np.uint32), o["neff_m"].view(np.uint32))
              and np.float32(nh[0]).view(np.uint32) == np.float32(o["neff_hmm"]).view(np.uint32))
        if not ok:
            kb += 1; print("kernel MISMATCH", it, filt, wg); open(os.path.join(d, f"kbad_{it}.a3m"), "wb").write(t)
    print(f"emulated kernels: {kr} alignments with random filter options, {kb} mismatches (inputs kept in {d} on mismatch)")


if __name__ == "__main__":
    main()
