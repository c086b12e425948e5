"""The product's MAC kernels (hh-suite_b200/csrc/hhg_mac.cuh, unmodified source) executed on the CPU by the host
emulation in tests/emul/ (one OS thread per CUDA thread, barriers for __syncwarp, an exchange buffer for shuffles) and
compared bit for bit with the oracle.  This is how kernel changes are checked in the authoring container before GPU
minutes are spent.  Both scan modes run (HHG_MAC_BANDSCAN: band-limited scans by default, full-row scans with 0), and
smem=0 forces the global-scratch fallback on short inputs, which the GPU only takes for templates longer than 1747
columns (tests/mac_cases.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.util import ROOT, bits

EMUL_DIR = os.path.join(ROOT, "tests", "emul")
LIB = os.path.join(EMUL_DIR, "libmacemul.so")
c_f32p = C.POINTER(C.c_float); c_i32p = C.POINTER(C.c_int32); c_u8p = C.POINTER(C.c_uint8)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(EMUL_DIR, "mac_emul.cpp"), os.path.join(EMUL_DIR, "cuda_emul.h"),
            os.path.join(ROOT, "hh-suite_b200", "csrc", "hhg_mac.cuh")]
    if not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-o", LIB,
                               srcs[0]])
    L = C.CDLL(LIB)
    L.emul_mac_realign.restype = C.c_int
    L.emul_mac_realign.argtypes = [C.c_int, c_f32p, c_f32p, C.c_int, c_f32p, c_f32p, c_f32p, C.c_int, C.c_double, C.c_float,
                                   c_i32p, c_i32p, c_i32p, C.c_int, c_i32p, c_i32p, C.c_int, C.c_int, c_i32p, c_f32p,
                                   C.POINTER(C.c_double), c_i32p, c_i32p, c_u8p, c_f32p, c_f32p]
    return L


def _run(L, oracle, qp, qlin, tp, ttr, vit, excl=None, local=True, shift=-0.03, mact=0.35, smem=64 * 1024, band=1):
    Lq, Lt = qp.shape[0] - 2, tp.shape[0] - 2
    i1, i2, j1, j2, n, vi, vj = vit
    v5 = np.array([i1, i2, j1, j2, n], np.int32)
    vi = np.ascontiguousarray(np.asarray(vi)[1:n + 1], np.int32); vj = np.ascontiguousarray(np.asarray(vj)[1:n + 1], np.int32)
    ei = np.ascontiguousarray(excl[0], np.int32) if excl else np.zeros(1, np.int32)
    ej = np.ascontiguousarray(excl[1], np.int32) if excl else np.zeros(1, np.int32)
    ne = len(excl[0]) if excl else 0
    cap = Lq + Lt + 4
    res = np.zeros(6, np.int32); sp = np.zeros(1, np.float32); pf = C.c_double()
    oi = np.zeros(cap, np.int32); oj = np.zeros(cap, np.int32); os_ = np.zeros(cap, np.uint8); op = np.zeros(cap, np.float32)
    post = np.zeros((Lq + 1, Lt + 1), np.float32)
    arr = [np.ascontiguousarray(a, np.float32) for a in (qp, qlin, tp, ttr, oracle.log2lin(ttr))]
    cshift = float(np.float64(2.0) ** np.float64(np.float32(shift)))       # pow(2.0, shift), src/hhforwardalgorithm.cpp:16
    nn = L.emul_mac_realign(Lq, _p(arr[0], c_f32p), _p(arr[1], c_f32p), Lt, _p(arr[2], c_f32p), _p(arr[3], c_f32p),
                            _p(arr[4], c_f32p), 1 if local else 0, cshift, mact, _p(v5, c_i32p), _p(vi, c_i32p),
                            _p(vj, c_i32p), ne, _p(ei, c_i32p), _p(ej, c_i32p), smem, band, _p(res, c_i32p), _p(sp, c_f32p),
                            C.byref(pf), _p(oi, c_i32p), _p(oj, c_i32p), _p(os_, c_u8p), _p(op, c_f32p), _p(post, c_f32p))
    assert nn >= 0, nn
    return dict(i1=int(res[0]), i2=int(res[1]), j1=int(res[2]), j2=int(res[3]), nsteps=int(res[4]),
                matched_cols=int(res[5]), sum_of_probs=float(sp[0]), Pforward=pf.value, i=oi[:nn + 1].copy(),
                j=oj[:nn + 1].copy(), states=os_[:nn + 1].copy(), P_posterior=op[:nn + 1].copy(), post=post)


def _same(a, b):
    for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols", "Pforward"):
        assert a[f] == b[f], f
    assert bits(np.float32(a["sum_of_probs"])) == bits(np.float32(b["sum_of_probs"]))
    n = b["nsteps"]
    assert np.array_equal(a["i"][1:n + 1], b["i"][1:n + 1]) and np.array_equal(a["j"][1:n + 1], b["j"][1:n + 1])
    assert np.array_equal(a["states"][1:n + 1], b["states"][1:n + 1])
    assert np.array_equal(bits(a["P_posterior"][1:n + 1]), bits(b["P_posterior"][1:n + 1]))
    assert np.array_equal(bits(a["post"][1:, 1:]), bits(b["post"][1:, 1:]))


def _cases(oracle, seed, n_targets=5):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(seed)
    Lq = int(rng.integers(40, 130))
    qp, qtr, qss, qpav, qcols = synth.query_profile(Lq, 100 + seed)
    out = []
    for k in range(n_targets):
        Lt = int(rng.integers(1, 260)) if k else Lq
        tp, ttr, _ = synth.prepared_profile(Lt, rng, qcols if k % 3 != 2 else None, noise=0.1 + 0.08 * k)
        sc, i2, j2, bt = oracle.viterbi(qp, qtr, tp, ttr)
        n, i_s, j_s, st, mc = oracle.backtrace(bt, i2, j2)
        if n:
            out.append((qp, qtr, tp, ttr, (int(i_s[n]), i2, int(j_s[n]), j2, n, i_s, j_s)))
    return out


FULL = os.environ.get("HHG_EMUL_FULL") == "1"      # the extended sweep (minutes); the default subset keeps the suite short


@pytest.mark.parametrize("seed", [1, 2] if FULL else [1])
@pytest.mark.parametrize("band", [0, 1])
def test_emulated_kernel_equals_oracle(emul, oracle, seed, band):
    """band=1: the band-limited scans, the default; band=0: the full-row scans (HHG_MAC_BANDSCAN=0).  Shared-memory
    working set and the global-scratch fallback (smem=0), local/global mode, several mact, a second alignment."""
    configs = ((True, 0.35, 64 * 1024), (True, 0.0, 0), (False, 0.1, 64 * 1024)) if FULL else \
        ((True, 0.35, 64 * 1024), (False, 0.1, 0))
    for k, (qp, qtr, tp, ttr, vit) in enumerate(_cases(oracle, seed, 5 if FULL else 3)):
        qlin = oracle.log2lin(qtr)
        for local, mact, smem in configs:
            want = oracle.mac_realign(qp, qlin, tp, oracle.log2lin(ttr), vit, local=local, mact=mact)
            got = _run(emul, oracle, qp, qlin, tp, ttr, vit, local=local, mact=mact, smem=smem, band=band)
            _same(got, want)
            if want["nsteps"] > 1 and local:
                ex = (want["i"][1:], want["j"][1:])
                w2 = oracle.mac_realign(qp, qlin, tp, oracle.log2lin(ttr), vit, excl=[ex], local=local, mact=mact)
                g2 = _run(emul, oracle, qp, qlin, tp, ttr, vit, excl=ex, local=local, mact=mact, smem=smem, band=band)
                _same(g2, w2)


def test_emulated_kernel_on_reference_goldens(emul, oracle):
    """data/query.hhm vs synth150 and vs itself (reference goldens), both scan modes."""
    from tests.util import golden
    G = golden()
    qlin = oracle.log2lin(G["q_tr"])
    for name, tp, ttr in ((("t150", "t150_p", "t150_tr"), ("tself", "tself_p", "tself_tr")) if FULL else
                          (("t150", "t150_p", "t150_tr"),)):
        v = G[f"mac_{name}_vit"]
        vit = (int(v[0]), int(v[1]), int(v[2]), int(v[3]), int(v[4]), G[f"mac_{name}_vit_i"], G[f"mac_{name}_vit_j"])
        mact = float(G[f"mac_{name}_f"][1])
        for band in (0, 1):
            got = _run(emul, oracle, G["q_p"], qlin, G[tp], G[ttr], vit, mact=mact, smem=200 * 1024, band=band)
            assert [got[k] for k in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols")] == G[f"mac_{name}_res"].tolist()
            assert got["Pforward"] == G[f"mac_{name}_pforward"][0]
            n = got["nsteps"]
            assert np.array_equal(got["i"][1:n + 1], G[f"mac_{name}_i"][1:n + 1])
            assert np.array_equal(bits(got["P_posterior"][1:n + 1]), bits(G[f"mac_{name}_ppost"][1:n + 1]))


def test_emulated_kernel_with_excluded_regions(emul, oracle, refshim):
    """-excl / -template_excl ranges in the realignment against the compiled reference
    (PosteriorDecoder::exclude_regions / exclude_template_regions), both scan modes."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(56)
    qp, qtr, qss, qpav, qcols = synth.query_profile(70, 12)
    refshim.set_query(qp, qtr, qpav, None)
    tp, ttr, _ = synth.prepared_profile(80, rng, qcols, noise=0.2)
    sc, i2, j2, bt = refshim.viterbi([(tp, ttr, None)])[0]
    n, i_s, j_s, st, mc = refshim.backtrace(0)
    vit = (int(i_s[n]), i2, int(j_s[n]), j2, n, i_s, j_s)
    qlin = oracle.log2lin(qtr)
    emul.emul_mac_set_regions.argtypes = [C.c_int, C.c_int, c_i32p]
    try:
        for (qreg, treg) in (([(20, 30)], []), ([], [(35, 50), (70, 400)]), ([(1, 3), (40, 41)], [(10, 12)])):
            refshim.set_mac_exclstr(",".join(f"{a}-{b}" for a, b in qreg), ",".join(f"{a}-{b}" for a, b in treg))
            reg = np.array([a for a, _ in qreg] + [b for _, b in qreg] + [a for a, _ in treg] + [b for _, b in treg], np.int32)
            emul.emul_mac_set_regions(len(qreg), len(treg), _p(reg, c_i32p))
            want = refshim.mac_realign(tp, ttr, vit, local=True, mact=0.35)
            for band in (0, 1):
                got = _run(emul, oracle, qp, qlin, tp, ttr, vit, local=True, mact=0.35, band=band)
                _same(got, want)
    finally:
        refshim.set_mac_exclstr("", "")
        emul.emul_mac_set_regions(0, 0, _p(np.zeros(1, np.int32), c_i32p))
