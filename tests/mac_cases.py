"""Long inputs for the MAC realignment (hhg_mac_realign / k_mac_realign), shared by the CPU tests (oracle against the
compiled reference) and the GPU tests (library against the oracle).

k_mac_realign keeps a request's working set in shared memory when it fits: 11 row buffers of doubles, the template's
linear transitions (7 floats) and one cell-off byte, for each of Lt+3 slots -- 117 bytes per template column
(`need` in k_mac_realign, hhg_mac.cuh; the small/large split in hhg_mac_realign, hhg_api.cu).  hhg_mac_realign runs
the requests that fit 64 KiB in one launch on the context's stream and all others in a second launch with a window of
up to 200 KiB on an auxiliary stream; a request that does not fit 200 KiB runs from the global row scratch inside that
second launch.  The constants below are the template lengths on either side of the two windows; the asserts fail if the
windows move and the tests drift off the boundaries."""
import numpy as np

from tests.util import bits

BYTES_PER_SLOT = 11 * 8 + 7 * 4 + 1
SMALL_WINDOW, LARGE_WINDOW = 64 * 1024, 200 * 1024
SMALL_MAX, LARGE_MIN = 557, 558          # last template length of the 64 KiB launch / first one of the large launch
WINDOW_MAX, FALLBACK_MIN = 1747, 1748    # last length inside the 200 KiB window / first one on the global scratch


def need(Lt):
    return BYTES_PER_SLOT * (Lt + 3)


assert BYTES_PER_SLOT == 117
assert need(SMALL_MAX) <= SMALL_WINDOW < need(LARGE_MIN)
assert need(WINDOW_MAX) <= LARGE_WINDOW < need(FALLBACK_MIN)

LONG_LT = 3000                           # the compiled reference is built with maxres 4096
BOUNDARY_LENGTHS = (1, SMALL_MAX, LARGE_MIN, WINDOW_MAX, FALLBACK_MIN, LONG_LT)
MODES = ((True, 0.35), (True, 0.0), (False, 0.1))   # (local, mact)
CLAMP = np.finfo(np.float64).tiny * 100             # DBL_MIN * 100: the forward/backward underflow clamp


def concat(parts):
    """One template from prepared profiles laid end to end: the columns of every part in order, background rows 0 and
    L+1 from the first and last part, and the start row of each later part as the junction's transitions."""
    p = np.concatenate([parts[0][0][:1]] + [x[0][1:-1] for x in parts] + [parts[-1][0][-1:]])
    tr = np.concatenate([x[1][:-1] for x in parts[:-1]] + [parts[-1][1]])
    return np.ascontiguousarray(p), np.ascontiguousarray(tr), None


def embedded(Lt, qcols, rng, noise=0.2):
    """Template of Lt columns: random | noisy copy of a stretch of the query | random, so that the homology sits in the
    middle of both the template and (when the stretch is shorter than the query) the query."""
    from hhsuite_b200 import synth
    if Lt < 3:
        return synth.prepared_profile(Lt, rng, qcols, noise=noise)
    Lh = max(1, min(qcols.shape[0], Lt // 2))
    La = (Lt - Lh) // 3
    Lb = Lt - Lh - La
    parts = [synth.prepared_profile(L, rng, qcols if k == 1 else None, noise=noise)
             for k, L in enumerate((La, Lh, Lb)) if L > 0]
    t = concat(parts)
    assert t[0].shape == (Lt + 2, 20) and t[1].shape == (Lt + 1, 7)
    return t


def two_copies(Lq, Lt, qcols, rng, noise=0.15):
    """Template of Lt columns holding two noisy copies of the whole query between random stretches."""
    from hhsuite_b200 import synth
    gap = Lt - 2 * Lq
    assert gap >= 3
    a = b = gap // 3
    parts = [synth.prepared_profile(L, rng, qcols if k in (1, 3) else None, noise=noise)
             for k, L in enumerate((a, Lq, b, Lq, gap - a - b))]
    return concat(parts)


def near_self(Lq, seed, noise=0.05):
    """A query with sharpened columns (synth.query_profile's columns squared and renormalised: about 1.2 bits per
    column of self-score instead of 0.6) and a low-noise copy of it as the template, Lt = Lq.  At Lq = 1500 the
    product of the forward scale factors falls below DBL_MIN*100 at about row 800."""
    from hhsuite_b200 import synth
    qp, qtr, qss, qpav, qcols = synth.query_profile(Lq, seed)
    f = qcols ** 2
    f /= f.sum(axis=1, keepdims=True)
    qp = qp.copy()
    qp[1:Lq + 1] = (0.9 * f + 0.1 * qp[0].astype(np.float64)).astype(np.float32)   # row 0 holds the background
    qpav = qp[1:Lq + 1].mean(axis=0).astype(np.float32)
    t = synth.prepared_profile(Lq, np.random.default_rng(seed + 1), f, noise=noise)
    return (qp, qtr, qss, qpav, f), t


def first_clamped_row(scale, Lq):
    """First forward row i at which the running product of the row scale factors scale[2..i-1] is below DBL_MIN*100,
    so that the forward pass's clamp branch zeroes it (hhforwardalgorithm.cpp; k_mac_realign); None if it never is."""
    prod = 1.0
    for i in range(2, Lq + 1):
        if prod < CLAMP:
            return i
        prod *= float(scale[i])
    return None


def ref_viterbi(refshim, tp, ttr):
    """Viterbi end points and path of the loaded query against one template, by the compiled reference."""
    sc, i2, j2, bt = refshim.viterbi([(tp, ttr, None)])[0]
    n, i_s, j_s, st, mc = refshim.backtrace(0)
    return None if n == 0 else (int(i_s[n]), i2, int(j_s[n]), j2, n, i_s, j_s)


def assert_same(want, got, what=()):
    """Field by field: end points, path, states, per-step posteriors, Pforward, sum_of_probs, posterior matrix bits."""
    for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols"):
        assert want[f] == got[f], (what, f, want[f], got[f])
    assert want["Pforward"] == got["Pforward"], (what, "Pforward", want["Pforward"], got["Pforward"])
    assert bits(np.float32(want["sum_of_probs"])) == bits(np.float32(got["sum_of_probs"])), (what, "sum_of_probs")
    n = want["nsteps"]
    for f in ("i", "j", "states"):
        assert np.array_equal(want[f][1:n + 1], got[f][1:n + 1]), (what, f)
    assert np.array_equal(bits(want["P_posterior"][1:n + 1]), bits(got["P_posterior"][1:n + 1])), (what, "P_posterior")
    assert np.array_equal(bits(want["post"][1:, 1:]), bits(got["post"][1:, 1:])), (what, "posterior matrix")
