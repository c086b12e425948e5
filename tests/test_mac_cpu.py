"""CPU tests of the MAC-realignment oracle (PosteriorDecoder::realign restated in oracle/hh_oracle.c) against the
reference: committed goldens, and the compiled reference on fresh cases when it is present."""
import numpy as np
import pytest

from tests import mac_cases as mc
from tests.util import bits, golden


def _vit(G, name):
    v = G[f"mac_{name}_vit"]
    return (int(v[0]), int(v[1]), int(v[2]), int(v[3]), int(v[4]), G[f"mac_{name}_vit_i"], G[f"mac_{name}_vit_j"])


@pytest.mark.parametrize("name,tp,ttr", [("t150", "t150_p", "t150_tr"), ("tself", "tself_p", "tself_tr")])
def test_oracle_mac_equals_reference_goldens(oracle, name, tp, ttr):
    import hashlib
    G = golden()
    qlin = oracle.log2lin(G["q_tr"])
    # interior rows of the reference's linear query transitions (boundary rows are reset by the decoder)
    assert np.array_equal(bits(qlin[1:-1]), bits(G["mac_q_tr_lin"][1:-1]))
    m = oracle.mac_realign(G["q_p"], qlin, G[tp], oracle.log2lin(G[ttr]), _vit(G, name), mact=float(G[f"mac_{name}_f"][1]))
    assert [m[k] for k in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols")] == G[f"mac_{name}_res"].tolist()
    assert m["Pforward"] == G[f"mac_{name}_pforward"][0]
    assert bits(np.float32(m["sum_of_probs"])) == bits(G[f"mac_{name}_f"][0])
    assert np.array_equal(m["i"][1:], G[f"mac_{name}_i"][1:]) and np.array_equal(m["j"][1:], G[f"mac_{name}_j"][1:])
    assert np.array_equal(m["states"][1:], G[f"mac_{name}_states"][1:])
    assert np.array_equal(bits(m["P_posterior"]), bits(G[f"mac_{name}_ppost"]))
    sha = np.frombuffer(hashlib.sha256(np.ascontiguousarray(m["post"][1:, 1:]).tobytes()).digest(), np.uint8)
    assert np.array_equal(sha, G[f"mac_{name}_post_sha"])
    if name == "tself":
        m2 = oracle.mac_realign(G["q_p"], qlin, G[tp], oracle.log2lin(G[ttr]), _vit(G, name), mact=0.35,
                                excl=[(m["i"][1:], m["j"][1:])])
        assert [m2[k] for k in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols")] == G["mac_tself2_res"].tolist()
        assert m2["Pforward"] == G["mac_tself2_pforward"][0]
        assert np.array_equal(m2["i"][1:], G["mac_tself2_i"][1:]) and np.array_equal(bits(m2["P_posterior"]), bits(G["mac_tself2_ppost"]))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_oracle_mac_equals_compiled_reference(oracle, refshim, seed):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(seed)
    Lq = int(rng.integers(40, 160))
    qp, qtr, qss, qpav, qcols = synth.query_profile(Lq, 10 + seed)
    refshim.set_query(qp, qtr, qpav, None)
    qlin = oracle.log2lin(qtr)
    for k in range(4):
        Lt = int(rng.integers(20, 220))
        tp, ttr, _ = synth.prepared_profile(Lt, rng, qcols if k != 3 else None, noise=0.15 + 0.1 * k)
        res = refshim.viterbi([(tp, ttr, None)])
        sc, i2, j2, bt = res[0]
        n, i_s, j_s, st, mc = refshim.backtrace(0)
        if n == 0:
            continue
        vit = (int(i_s[n]), i2, int(j_s[n]), j2, n, i_s, j_s)
        for local, mact in ((True, 0.35), (True, 0.0), (False, 0.1)):
            ref = refshim.mac_realign(tp, ttr, vit, local=local, mact=mact)
            mine = oracle.mac_realign(qp, qlin, tp, oracle.log2lin(ttr), vit, local=local, mact=mact)
            for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols", "Pforward"):
                assert ref[f] == mine[f], (seed, k, local, mact, f)
            assert np.array_equal(ref["i"][1:], mine["i"][1:]) and np.array_equal(ref["j"][1:], mine["j"][1:])
            assert np.array_equal(ref["states"][1:], mine["states"][1:])
            assert np.array_equal(bits(ref["P_posterior"]), bits(mine["P_posterior"]))
            assert np.array_equal(bits(ref["post"][1:, 1:]), bits(mine["post"][1:, 1:]))
            # a second alignment with the first one masked out
            if ref["nsteps"] > 0:
                ex = [(ref["i"][1:], ref["j"][1:])]
                r2 = refshim.mac_realign(tp, ttr, vit, excl=ex, local=local, mact=mact)
                m2 = oracle.mac_realign(qp, qlin, tp, oracle.log2lin(ttr), vit, excl=ex, local=local, mact=mact)
                assert r2["Pforward"] == m2["Pforward"] and np.array_equal(r2["i"][1:], m2["i"][1:])
                assert np.array_equal(bits(r2["post"][1:, 1:]), bits(m2["post"][1:, 1:]))


# Lq -> template lengths: every query length crossed with some of the launch-boundary lengths (tests/mac_cases.py), so
# that every boundary length and every query length appears at least once.
LONG_CASES = {1: (1, mc.LARGE_MIN, mc.FALLBACK_MIN), 2: (1, mc.SMALL_MAX, mc.LONG_LT),
              700: (mc.SMALL_MAX, mc.LARGE_MIN, mc.WINDOW_MAX, mc.FALLBACK_MIN), 1500: (1, mc.WINDOW_MAX, mc.LONG_LT)}


def _oracle_mac(oracle, qp, qtr, t, vit, **kw):
    return oracle.mac_realign(qp, oracle.log2lin(qtr), t[0], oracle.log2lin(t[1]), vit, **kw)


@pytest.mark.parametrize("Lq", sorted(LONG_CASES))
def test_oracle_mac_equals_compiled_reference_long(oracle, refshim, Lq):
    """Queries of 1, 2, 700 and 1500 columns against templates at the shared-memory window boundaries and beyond, with
    the homology in the middle of the template; every mode, then a second alignment with the first one excluded."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(1000 + Lq)
    qp, qtr, qss, qpav, qcols = synth.query_profile(Lq, 40 + Lq)
    refshim.set_query(qp, qtr, qpav, None)
    for Lt in LONG_CASES[Lq]:
        t = mc.embedded(Lt, qcols, rng, noise=0.2)
        vit = mc.ref_viterbi(refshim, t[0], t[1])
        assert vit is not None, (Lq, Lt)
        for local, mact in mc.MODES:
            what = (Lq, Lt, local, mact)
            ref = refshim.mac_realign(t[0], t[1], vit, local=local, mact=mact)
            mc.assert_same(ref, _oracle_mac(oracle, qp, qtr, t, vit, local=local, mact=mact), what)
            if ref["nsteps"] > 0:
                ex = [(ref["i"][1:], ref["j"][1:])]
                r2 = refshim.mac_realign(t[0], t[1], vit, excl=ex, local=local, mact=mact)
                mc.assert_same(r2, _oracle_mac(oracle, qp, qtr, t, vit, excl=ex, local=local, mact=mact), what + ("excl",))


def test_oracle_mac_underflow_clamp_equals_compiled_reference(oracle, refshim):
    """A near-self hit of 1500 columns accumulates enough forward mass that the product of the row scale factors falls
    below DBL_MIN*100, so the forward and backward clamp branches run; the oracle still matches bit for bit."""
    Lq = 1500
    (qp, qtr, qss, qpav, qcols), t = mc.near_self(Lq, 78)
    refshim.set_query(qp, qtr, qpav, None)
    vit = mc.ref_viterbi(refshim, t[0], t[1])
    assert vit[4] > Lq // 2
    fw = refshim.mac_forward_only(t[0], t[1], vit)
    row = mc.first_clamped_row(fw["scale"], Lq)
    assert row is not None and row < 2 * Lq // 3, row
    assert fw["Pforward"] == refshim.mac_realign(t[0], t[1], vit, want_post=False)["Pforward"]
    for local, mact in mc.MODES:
        ref = refshim.mac_realign(t[0], t[1], vit, local=local, mact=mact)
        mc.assert_same(ref, _oracle_mac(oracle, qp, qtr, t, vit, local=local, mact=mact), (local, mact))


def test_host_log2lin_equals_oracle(oracle):
    from hhsuite_b200 import capi
    x = np.concatenate([np.random.default_rng(3).normal(-3, 4, 20000), [0.0, -1.0, -60000.0, -0.5, 1.0]]).astype(np.float32)
    assert np.array_equal(bits(capi.log2lin(x)), bits(oracle.log2lin(x)))
