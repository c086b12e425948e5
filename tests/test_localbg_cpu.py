"""The local amino-acid composition correction kernel (hh-suite_b200/csrc/hhg_localbg.cuh, unmodified source, `-sc 5`)
executed on the CPU by the host emulation in tests/emul/ and compared bit for bit with the compiled reference's
HMM::DivideBySqrtOfLocalBackgroundFreqs: window half-widths around both branch points of the routine, the longest
profile, all-zero columns and tiny values, many segments of mixed lengths in one launch (transitions and ss copied,
records outside the segments untouched), and templates prepared by the reference under -sc 5."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.util import ROOT, bits, golden, ref_data_file

EMUL_DIR = os.path.join(ROOT, "tests", "emul")
LIB = os.path.join(EMUL_DIR, "liblocalbgemul.so")
INT_MAX = 2**31 - 1
SENTINEL = np.float32(-7.25)


@pytest.fixture(scope="module")
def lbref():
    """The compiled reference's routine (oracle/localbg_shim.cpp); skipped when oracle/_ref was not built."""
    from oracle.localbg_binding import LocalBgRef
    try:
        return LocalBgRef()
    except (FileNotFoundError, OSError) as e:
        pytest.skip(f"compiled reference not available: {e}")


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(EMUL_DIR, "localbg_emul.cpp"), os.path.join(EMUL_DIR, "cuda_emul.h"),
            os.path.join(ROOT, "hh-suite_b200", "csrc", "hhg_localbg.cuh")]
    if not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-o", LIB,
                               srcs[0]])
    L = C.CDLL(LIB)
    L.emul_local_bg.restype = None
    L.emul_local_bg.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    return L


def run_kernel(emul, profiles, pb, D, blocks=2, threads=64):
    """profiles: list of p[(L+2), 20].  Packs rows 1..L of each into 28-float records (random transition / ss words),
    runs k_local_bg with one segment per profile into an output array whose records between the segments hold a
    sentinel, and returns (divided profiles with rows 0 and L+1 copied from the input, source records, output records,
    segment table)."""
    rng = np.random.default_rng(len(profiles) + D % 1000)
    Ls = [p.shape[0] - 2 for p in profiles]
    src_off = np.concatenate([[0], np.cumsum(Ls)[:-1]]).astype(np.int64)
    dst_off = src_off + np.arange(len(Ls)) + 1          # one sentinel record before every segment
    src = rng.random((int(sum(Ls)), 28), dtype=np.float32)
    src[:, 27] = rng.integers(0, 2**32, len(src), dtype=np.uint64).astype(np.uint32).view(np.float32)
    for p, o, L in zip(profiles, src_off, Ls):
        src[o:o + L, :20] = p[1:L + 1]
    dst = np.full((int(dst_off[-1] + Ls[-1] + 1), 28), SENTINEL, np.float32)
    seg = np.stack([src_off, dst_off, np.array(Ls, np.int64)], axis=1).astype(np.int64)
    pbv = np.ascontiguousarray(pb, np.float32)
    emul.emul_local_bg(len(Ls), seg.ctypes.data, src.ctypes.data, dst.ctypes.data, pbv.ctypes.data, int(D), blocks, threads)
    out = []
    for p, o, L in zip(profiles, dst_off, Ls):
        q = p.copy()
        q[1:L + 1] = dst[o:o + L, :20]
        out.append(q)
    return out, src, dst, seg


def check_records(src, dst, seg):
    """Transitions and ss of every record copied bit for bit; every record outside the segments untouched."""
    inside = np.zeros(len(dst), bool)
    for s, d, L in seg:
        assert np.array_equal(bits(dst[d:d + L, 20:]), bits(src[s:s + L, 20:]))
        inside[d:d + L] = True
    assert np.all(bits(dst[~inside]) == bits(SENTINEL))


def profile(L, rng, kind):
    p = rng.random((L + 2, 20)).astype(np.float32)
    p /= p.sum(axis=1, keepdims=True)
    if kind == "zeros":
        p[rng.random(L + 2) < 0.3] = 0.0          # all-zero columns
    elif kind == "tiny":
        p[:, rng.random(20) < 0.4] *= np.float32(1e-30)
    return p.astype(np.float32)


def lengths_for(D):
    Ls = [L for L in (1, 2, 2 * D, 2 * D + 1, 2 * D + 2, 2 * D + 3) if 1 <= L <= 32767]
    return sorted(set(Ls + [32767]))


@pytest.mark.parametrize("D", [1, 2, 5, 40, 16383, 16384, 10**6, INT_MAX])
def test_kernel_equals_reference(emul, lbref, D):
    """Every length around both branch points (L <= 2D+1 averages the whole profile) and L = 32767, seeded, zero and
    tiny profiles, all in one launch per D."""
    rng = np.random.default_rng(D % 100003)
    pb = golden()["pb"]
    kinds = [(L, kind) for L in lengths_for(D) for kind in ("seeded", "zeros", "tiny")]
    profs = [profile(L, rng, kind) for L, kind in kinds]
    got, src, dst, seg = run_kernel(emul, profs, pb, D)
    check_records(src, dst, seg)
    for (L, kind), p, g in zip(kinds, profs, got):
        want = lbref.local_bg(p, pb, D)
        assert np.array_equal(bits(want[[0, -1]]), bits(p[[0, -1]]))
        if kind == "seeded":
            assert not np.array_equal(bits(want[1:-1]), bits(p[1:-1]))
        assert np.array_equal(bits(g), bits(want)), (D, p.shape[0] - 2)


def test_mixed_segments_one_launch(emul, lbref):
    """Many segments of random lengths, fewer warps than segments (grid-stride), a non-default background."""
    rng = np.random.default_rng(5)
    pb = rng.random(20).astype(np.float32)
    pb /= pb.sum()
    for D in (3, 40):
        profs = [profile(int(L), rng, ("seeded", "zeros", "tiny")[k % 3])
                 for k, L in enumerate(rng.integers(1, 400, 60))]
        got, src, dst, seg = run_kernel(emul, profs, pb, D, blocks=1, threads=96)
        check_records(src, dst, seg)
        for p, g in zip(profs, got):
            assert np.array_equal(bits(g), bits(lbref.local_bg(p, pb, D))), (D, p.shape[0] - 2)


def test_templates_prepared_by_reference(emul, lbref, tmp_path):
    """Templates read from synthetic HHM text and prepared by the reference under -sc 5 (PrepareTemplateHMM up to
    IncludeNullModelInHMM case 5): the kernel on the records before the null model gives the prepared emissions."""
    from hhsuite_b200 import synth
    for D in (40, 3):
        lbref.prepare_query_hhm(ref_data_file("query.hhm", tmp_path), 5, D)   # case 5 needs a divided query
        for k, L in enumerate((1, 5, 2 * D + 1, 2 * D + 2, 150, 333)):
            path = tmp_path / f"t{D}_{k}.hhm"
            path.write_text(synth.hhm_text(L, 40 + k, f"t{k}", with_ss=k % 2 == 1))
            t = lbref.prepare_template_hhm(path)
            got = run_kernel(emul, [t["p_raw"]], t["pb"], D)[0][0]      # pb: the record's NULL line
            assert not np.array_equal(bits(t["p"]), bits(t["p_raw"]))
            assert np.array_equal(bits(got), bits(t["p"])), (D, L)
