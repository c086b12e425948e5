"""The tie-forcing Viterbi families (tests/vit_cases.py) really force ties: a float64 witness DP, exact on their dyadic
inputs, finds several maximal end cells and every kind of exact candidate equality, and its score and row-major
first maximum are the oracle's.  Without this a later edit to a generator could make it tie-free unnoticed."""
import numpy as np
import pytest

from tests import vit_cases as vc
from tests.util import bits


def _family(name):
    return name.rsplit("-", 1)[0]


def _witnessed():
    out = {}
    for name, q, tg, par in vc.tie_cases() + vc.global_cases():
        for t in tg:
            out.setdefault(_family(name), []).append((q, t, par, vc.witness(q, t, **par)))
    return out


@pytest.fixture(scope="module")
def witnessed():
    return _witnessed()


def test_witness_equals_oracle(oracle, witnessed):
    n = 0
    for fam, runs in witnessed.items():
        for q, t, par, w in runs:
            sc, i2, j2, _ = oracle.viterbi(q[0], q[1], t[0], t[1], want_bt=False, **par)
            assert bits(np.float32(w["score"])) == bits(sc), (fam, t[0].shape[0] - 2, w["score"], sc)
            assert w["first"] == (i2, j2), (fam, t[0].shape[0] - 2)
            n += 1
    assert n > 1000


def _any(runs, pred):
    return sum(1 for r in runs if pred(r[3]))


def test_every_tie_family_has_several_maxima_in_different_rows(witnessed):
    for fam, runs in witnessed.items():
        if fam.startswith("g-tandem"):      # global mode: one end row / column, ties come from the gap flags
            continue
        assert _any(runs, lambda w: len({c[0] for c in w["cells"]}) >= 2) >= 2, fam


@pytest.mark.parametrize("fam", ["tandem3", "tandem5", "tandem6", "tandem7"])
def test_tandem_maxima_cross_strips_and_backtrace_words(witnessed, fam):
    runs = witnessed[fam]
    assert _any(runs, lambda w: len({(i - 1) // 16 for i, _ in w["cells"]}) >= 2) >= 1
    assert _any(runs, lambda w: len({(i - 1) // 4 for i, _ in w["cells"]}) >= 2) >= 1
    for R in (8, 12):
        assert _any(runs, lambda w: len({(i - 1) // R for i, _ in w["cells"]}) >= 2) >= 1


def _later_column_earlier_row(w, R):
    """Two maxima in one R-row strip where the row-major first lies in a LATER column than another one: a strip swept
    column by column meets the wrong one first."""
    i0, j0 = w["first"]
    return any((i - 1) // R == (i0 - 1) // R and i > i0 and j < j0 for i, j in w["cells"])


@pytest.mark.parametrize("fam", ["anti3", "anti5", "anti6", "anti7"])
def test_antidiagonal_maxima_inside_one_strip(witnessed, fam):
    for R in (8, 12, 16):
        assert _any(witnessed[fam], lambda w: _later_column_earlier_row(w, R)) >= 2, R


def test_every_candidate_equality_occurs(witnessed):
    """c1 == c2 as the MM maximum above smin, smin == MM maximum (exact 0 in local mode) and a1 == a2 of all four
    gap-state flags."""
    need = {"gap": ("c1c2", "gd", "dg", "zero"), "g-gap": ("c1c2", "gd", "dg"), "tandem6": ("gd", "im", "dg", "mi"),
            "anti7": ("gd", "im", "dg", "mi"), "const-zero": ("zero",)}
    for fam, kinds in need.items():
        for k in kinds:
            assert _any(witnessed[fam], lambda w: w["ties"][k] > 0) >= 2, (fam, k)


def test_const_zero_family_ties_every_cell():
    """Si == 0: every local cell is exactly 0, so every cell is maximal and the first is (1, 1)."""
    q = vc.const(13, "q", level=1)
    t = vc.const(31, "t", level=1)
    w = vc.witness(q, t, shift=-1.0)
    assert w["score"] == 0.0 and len(w["cells"]) == 13 * 31 and w["first"] == (1, 1)


def test_dyadic_inputs_are_exact():
    """Every emission dot product of a tie family is a power of two (log2f4 exact), every transition dyadic."""
    for name, q, tg, par in vc.tie_cases():
        for t in tg[:4]:
            d = q[0][1:-1].astype(np.float64) @ t[0][1:-1].astype(np.float64).T
            m, _ = np.frexp(d[d > 0])
            assert np.all(m == 0.5), name
            for tr in (q[1], t[1]):
                assert np.all(tr * 4 == np.round(tr * 4)), name
