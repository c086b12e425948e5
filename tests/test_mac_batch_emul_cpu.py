"""The product's MAC kernels (hh-suite_b200/csrc/hhg_mac.cuh, unmodified source) with a batch of queries in one launch,
executed on the CPU by the host emulation in tests/emul/ and compared bit for bit with the oracle.  Every request reads
its own query (MacArgs.req_q: length, emissions, transitions and scale factors) in the layout hhg_mac_realign_batch
builds; queries of very different lengths, Lq = 1 and 2 among them, sit side by side in the same k_mac_band and
k_mac_realign launch.  Templates are raw profiles with the null model of the request's query applied
(batch_cases.null_model), as the batch realignment does over a raw shard."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import batch_cases as bc
from tests.util import ROOT, bits

EMUL_DIR = os.path.join(ROOT, "tests", "emul")
LIB = os.path.join(EMUL_DIR, "libmacbatchemul.so")
c_f32p = C.POINTER(C.c_float); c_i32p = C.POINTER(C.c_int32); c_i64p = C.POINTER(C.c_int64); c_u8p = C.POINTER(C.c_uint8)
MAC_HIT_DTYPE = np.dtype([("i1", np.int32), ("i2", np.int32), ("j1", np.int32), ("j2", np.int32), ("nsteps", np.int32),
                          ("matched_cols", np.int32), ("sum_of_probs", np.float32), ("flags", np.int32),
                          ("pforward", np.float64), ("path_off", np.int64)])


def _p(a, t):
    return a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(EMUL_DIR, "mac_batch_emul.cpp"), os.path.join(EMUL_DIR, "cuda_emul.h"),
            os.path.join(ROOT, "hh-suite_b200", "csrc", "hhg_mac.cuh")]
    if not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-o", LIB,
                               srcs[0]])
    L = C.CDLL(LIB)
    L.emul_mac_realign_batch.restype = C.c_int
    L.emul_mac_realign_batch.argtypes = [C.c_int, c_i32p, c_f32p, c_f32p, C.c_int, c_i32p, c_i32p, c_f32p, c_f32p,
                                         c_i32p, c_i64p, c_i32p, c_i32p, C.c_int, C.c_double, C.c_float, C.c_int,
                                         C.c_int, C.c_void_p, c_i32p, c_i32p, c_u8p, c_f32p, c_f32p]
    return L


def _batch(oracle, seed):
    """Queries of lengths 1, 2, 37 and 90 with their own pav; raw templates; requests of every query against several
    templates (one template shared by all queries), each template null-modelled for the request's query."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(seed)
    qs = bc.queries((1, 2, 37, 90), 500 + seed)
    t_lens = (1, 3, 40, 95, 130, 60)
    raw = [bc.raw_profile(synth.prepared_profile(L, rng, qs[k % 4]["mix"] if k % 2 == 0 else None, noise=0.2), rng)
           for k, L in enumerate(t_lens)]
    cs = seed % 4
    pb = rng.dirichlet(np.ones(20) * 6).astype(np.float32)
    reqs = []
    for q in range(len(qs)):
        for t in ([q, 4, 5] if q < 2 else [q + 1, 4, 2, 0]):
            (p_raw, ttr, _), t_pav = raw[t]
            tp = bc.null_model(p_raw, t_pav, qs[q]["pav"], pb, cs)
            sc, i2, j2, bt = oracle.viterbi(qs[q]["p"], qs[q]["tr"], tp, ttr)
            n, i_s, j_s, st, mc = oracle.backtrace(bt, i2, j2)
            if n:
                reqs.append((q, tp, ttr, (int(i_s[n]), i2, int(j_s[n]), j2, n, i_s, j_s)))
    return qs, reqs


def _run(L, oracle, qs, reqs, local, mact, smem, band, shift=-0.03):
    qL = np.array([q["p"].shape[0] - 2 for q in qs], np.int32)
    qp = np.ascontiguousarray(np.concatenate([q["p"].reshape(-1) for q in qs]), np.float32)
    qlin = np.ascontiguousarray(np.concatenate([oracle.log2lin(q["tr"]).reshape(-1) for q in qs]), np.float32)
    rq = np.array([r[0] for r in reqs], np.int32)
    Lt = np.array([r[1].shape[0] - 2 for r in reqs], np.int32)
    tp = np.ascontiguousarray(np.concatenate([r[1].reshape(-1) for r in reqs]), np.float32)
    tlin = np.ascontiguousarray(np.concatenate([oracle.log2lin(r[2]).reshape(-1) for r in reqs]), np.float32)
    vit5 = np.array([r[3][:5] for r in reqs], np.int32)
    voff = np.concatenate([[0], np.cumsum(vit5[:, 4])]).astype(np.int64)
    vi = np.ascontiguousarray(np.concatenate([np.asarray(r[3][5])[1:r[3][4] + 1] for r in reqs]), np.int32)
    vj = np.ascontiguousarray(np.concatenate([np.asarray(r[3][6])[1:r[3][4] + 1] for r in reqs]), np.int32)
    n = len(reqs)
    Lq_r = qL[rq].astype(np.int64)
    cap = int(np.sum(Lq_r + Lt + 2)); ncell = int(np.sum((Lq_r + 1) * (Lt + 1)))
    hits = np.zeros(n, MAC_HIT_DTYPE)
    oi = np.zeros(cap, np.int32); oj = np.zeros(cap, np.int32); os_ = np.zeros(cap, np.uint8); op = np.zeros(cap, np.float32)
    post = np.zeros(ncell, np.float32)
    cshift = float(np.float64(2.0) ** np.float64(np.float32(shift)))
    assert L.emul_mac_realign_batch(len(qs), _p(qL, c_i32p), _p(qp, c_f32p), _p(qlin, c_f32p), n, _p(rq, c_i32p),
                                    _p(Lt, c_i32p), _p(tp, c_f32p), _p(tlin, c_f32p), _p(vit5, c_i32p), _p(voff, c_i64p),
                                    _p(vi, c_i32p), _p(vj, c_i32p), 1 if local else 0, cshift, mact, smem, band,
                                    hits.ctypes.data_as(C.c_void_p), _p(oi, c_i32p), _p(oj, c_i32p), _p(os_, c_u8p),
                                    _p(op, c_f32p), _p(post, c_f32p)) == 0
    out, po, pc = [], 0, 0
    for r in range(n):
        ns = int(hits["nsteps"][r]); a, b = int(Lq_r[r]), int(Lt[r])
        assert int(hits["path_off"][r]) == po
        out.append(dict(i1=int(hits["i1"][r]), i2=int(hits["i2"][r]), j1=int(hits["j1"][r]), j2=int(hits["j2"][r]),
                        nsteps=ns, matched_cols=int(hits["matched_cols"][r]), sum_of_probs=float(hits["sum_of_probs"][r]),
                        Pforward=float(hits["pforward"][r]), i=oi[po:po + ns + 1], j=oj[po:po + ns + 1],
                        states=os_[po:po + ns + 1], P_posterior=op[po:po + ns + 1],
                        post=post[pc:pc + (a + 1) * (b + 1)].reshape(a + 1, b + 1)))
        po += a + b + 2; pc += (a + 1) * (b + 1)
    return out


def _same(a, b, what):
    for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols", "Pforward"):
        assert a[f] == b[f], (what, f, a[f], b[f])
    assert bits(np.float32(a["sum_of_probs"])) == bits(np.float32(b["sum_of_probs"])), what
    n = b["nsteps"]
    for f in ("i", "j", "states"):
        assert np.array_equal(a[f][1:n + 1], b[f][1:n + 1]), (what, f)
    assert np.array_equal(bits(a["P_posterior"][1:n + 1]), bits(b["P_posterior"][1:n + 1])), (what, "P_posterior")
    assert np.array_equal(bits(a["post"][1:, 1:]), bits(b["post"][1:, 1:])), (what, "posterior matrix")


@pytest.mark.parametrize("band", [0, 1])
def test_emulated_query_batch_equals_oracle(emul, oracle, band):
    """One launch over the requests of four queries (Lq 1, 2, 37, 90): every request against the oracle's
    mac_realign of its own query, local mode with the shared-memory working set and global mode on the global scratch."""
    qs, reqs = _batch(oracle, 3)
    assert len({r[0] for r in reqs}) == 4 and len(reqs) >= 10
    for local, mact, smem in ((True, 0.35, 64 * 1024), (False, 0.1, 0)):
        got = _run(emul, oracle, qs, reqs, local, mact, smem, band)
        for k, (q, tp, ttr, vit) in enumerate(reqs):
            qq = qs[q]
            want = oracle.mac_realign(qq["p"], oracle.log2lin(qq["tr"]), tp, oracle.log2lin(ttr), vit, local=local,
                                      mact=mact)
            _same(got[k], want, (k, q, local, mact))
