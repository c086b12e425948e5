"""The product's ungapped query-batch prefilter kernel and its host-side plan (hh-suite_b200/csrc/hhg_prefilter.cuh,
unmodified source) executed on the CPU by the host emulation in tests/emul/ and compared with the oracle for every
(query, sequence).  Short queries share slabs with segment boundaries at lane 0, mid-warp and lane 31; one query fills a
slab exactly; queries of 513, 1025 and 2100 positions run in the same batch over several tile rounds, also cut into
one memory wave per long query.  Diagonals planted across the 512 / 1024 / 1536 tile boundaries of profiles whose
background decays score more than any single tile can see, so they hold only if the edge bytes are carried exactly."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.pf_batch_cases import carry_batch
from tests.util import ROOT

EMUL_DIR = os.path.join(ROOT, "tests", "emul")
LIB = os.path.join(EMUL_DIR, "libpfbatchemul.so")
c_i32p = C.POINTER(C.c_int32); c_i64p = C.POINTER(C.c_int64); c_u8p = C.POINTER(C.c_uint8)


def _p(a, t):
    return a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(EMUL_DIR, "pf_batch_emul.cpp"), os.path.join(EMUL_DIR, "cuda_emul_mw.h"),
            os.path.join(ROOT, "hh-suite_b200", "csrc", "hhg_prefilter.cuh"),
            os.path.join(ROOT, "hh-suite_b200", "csrc", "hhg_math.cuh")]
    if not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-std=c++20", "-fPIC", "-shared", "-pthread", "-o", LIB, srcs[0]])
    L = C.CDLL(LIB)
    L.emul_pf_ungapped_batch.restype = C.c_int
    L.emul_pf_ungapped_batch.argtypes = [C.c_int, c_i32p, C.POINTER(C.c_void_p), C.c_int, C.c_int, c_i32p, c_i64p, c_u8p,
                                         C.c_double, C.c_int, C.c_int, c_i32p, c_i32p, c_i32p, c_i32p]
    return L


def _run(L, profs, seqs, offset, budget, grid=2, threads=64):
    profs = [np.ascontiguousarray(p, np.uint8) for p in profs]
    Lq = np.array([p.shape[1] for p in profs], np.int32)
    ptrs = (C.c_void_p * len(profs))(*[p.ctypes.data for p in profs])
    Ls = np.array([len(s) for s in seqs], np.int32)
    off = np.concatenate([[0], np.cumsum(Ls.astype(np.int64))[:-1]]).astype(np.int64)
    seq = np.ascontiguousarray(np.concatenate(seqs), np.uint8)
    sc = np.full((len(profs), len(seqs)), -7, np.int32)
    nl, nw, ns = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32)
    assert L.emul_pf_ungapped_batch(len(profs), _p(Lq, c_i32p), ptrs, offset, len(seqs), _p(Ls, c_i32p), _p(off, c_i64p),
                                    _p(seq, c_u8p), budget, grid, threads, _p(sc, c_i32p), _p(nl, c_i32p),
                                    _p(nw, c_i32p), _p(ns, c_i32p)) == 0
    return sc, int(nl[0]), int(nw[0]), int(ns[0])


def _batch(seed):
    """Lq 336 + 160 + 5 fill one slab (segments start at lanes 0, 21 and 31), 512 fills a slab on its own, 1 takes a
    lane of a third slab; 513 / 1025 / 2100 take 2 / 3 / 5 tile rounds.  Sequences of 1..300 columns, planted
    near-perfect matches (saturating at 255 on the hot profiles), one across the 512 / 1024 tile boundaries."""
    rng = np.random.default_rng(seed)
    lens = [336, 160, 5, 512, 1, 513, 1025, 2100]
    profs = []
    for Lq in lens:
        p = rng.integers(30, 75, (220, Lq), dtype=np.uint8)
        p[219] = 49
        profs.append(p)
    best = [p[:219].argmax(axis=0).astype(np.uint8) for p in profs]
    for k in (0, 3, 7):                                               # hot diagonals: saturation at 255
        profs[k][best[k], np.arange(lens[k])] = 120
    seqs = [rng.integers(0, 220, L, dtype=np.uint8) for L in [1, 2, 31, 33, 64, 100, 257]]
    seqs += [best[0][:300], best[1].copy(), best[2].copy(), best[3][200:460], best[5][400:513], best[6][480:780],
             np.concatenate([rng.integers(0, 219, 9, dtype=np.uint8), best[7][1000:1100]])]
    return profs, seqs


@pytest.mark.parametrize("offset", [50, 0])
def test_emulated_batch_equals_oracle(emul, oracle, offset):
    profs, seqs = _batch(5 + offset)
    want = np.array([[oracle.ungapped(p, s, offset) for s in seqs] for p in profs])
    got, nl, nw, ns = _run(emul, profs, seqs, offset, 1e18)
    assert nw == 1 and nl == 5 and ns == 3 + 2 + 3 + 5           # three short slabs; one slab per long tile
    for q in range(len(profs)):
        assert got[q].tolist() == want[q].tolist(), (q, profs[q].shape[1])
    if offset == 50:
        assert want[0].max() == 255 - 50 and want[7].max() == 255 - 50


def test_emulated_batch_memory_waves(emul, oracle):
    """A budget of one long query's two edge slots: one wave per long query (2 + 3 + 5 launches), same scores."""
    profs, seqs = _batch(11)
    total = sum(len(s) for s in seqs)
    want = np.array([[oracle.ungapped(p, s, 50) for s in seqs] for p in profs])
    got, nl, nw, _ = _run(emul, profs, seqs, 50, 2.0 * total, grid=1, threads=32)
    assert nw == 3 and nl == 2 + 3 + 5
    assert np.array_equal(got, want)


def test_emulated_tile_boundary_carry(emul, oracle):
    """The edge bytes between tile rounds: diagonals across 512 / 1024 / 1536 score their full length (above anything a
    single tile can see), equal to the oracle, in one wave and with one wave per long query."""
    profs, seqs, cases = carry_batch(23)
    want = np.array([[oracle.ungapped(p, s, 50) for s in seqs] for p in profs])
    total = sum(len(s) for s in seqs)
    for budget in (1e18, 2.0 * total):
        got, nl, nw, _ = _run(emul, profs, seqs, 50, budget, grid=2, threads=32)
        assert np.array_equal(got, want), budget
        assert nw == (1 if budget > 1e17 else 3)
    crossing = 0
    for q, k, score, tile_best in cases:
        assert want[q, k] == score, (q, k)
        crossing += score > tile_best
    assert crossing == 3 + 2 + 1                                    # the boundaries of Lq 1700, 1100 and 700
