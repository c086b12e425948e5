"""GPU parity of the MAC realignment (hhg_mac_realign, SURVEY 8f-3) through the C-ABI: posterior matrix, Pforward, MAC
path and per-step posteriors must be bit-identical to the reference (goldens; compiled reference when shipped) and to
the oracle's restatement, for local/global mode, several mact thresholds and alternative alignments."""
import functools

import numpy as np
import pytest

from tests import mac_cases as mc
from tests.util import bits, golden

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[0, 1], ids=["fullscan", "bandscan"], autouse=True)
def band_scan(request, monkeypatch):
    """Every MAC test runs with both scan modes of k_mac_realign: full-row scans and the band-limited scans
    (HHG_MAC_BANDSCAN, read per call by hhg_mac_realign); results must be bit-identical either way."""
    monkeypatch.setenv("HHG_MAC_BANDSCAN", str(request.param))
    return request.param


def _check(gpu_hit, gpu_path, want):
    for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols"):
        assert int(gpu_hit[f]) == want[f], f
    assert float(gpu_hit["pforward"]) == want["Pforward"]
    assert bits(gpu_hit["sum_of_probs"]) == bits(np.float32(want["sum_of_probs"]))
    n = want["nsteps"]
    assert np.array_equal(gpu_path["i"][1:n + 1], want["i"][1:n + 1]) and np.array_equal(gpu_path["j"][1:n + 1], want["j"][1:n + 1])
    assert np.array_equal(gpu_path["states"][1:n + 1], want["states"][1:n + 1])
    assert np.array_equal(bits(gpu_path["P_posterior"][1:n + 1]), bits(want["P_posterior"][1:n + 1]))


def test_mac_goldens_config1(hhg, gpu_ctx):
    """data/query.hhm vs synth150 (mact 0) and vs itself (mact 0.35) + the second alignment of the self hit."""
    G = golden()
    gpu_ctx.set_query(G["q_p"], G["q_tr"])
    db = hhg.TargetDB.from_profiles(gpu_ctx, [(G["t150_p"], G["t150_tr"], None), (G["tself_p"], G["tself_tr"], None)])
    hhg.capi.mac_query_set(gpu_ctx, G["q_p"], hhg.capi.log2lin(G["q_tr"]))
    for t, name in ((0, "t150"), (1, "tself")):
        v = G[f"mac_{name}_vit"]
        vit = (int(v[0]), int(v[1]), int(v[2]), int(v[3]), int(v[4]), G[f"mac_{name}_vit_i"], G[f"mac_{name}_vit_j"])
        mact = float(G[f"mac_{name}_f"][1])
        hits, paths = hhg.capi.mac_realign(gpu_ctx, db, [t], [vit], mact=mact)
        want = dict(zip(("i1", "i2", "j1", "j2", "nsteps", "matched_cols"), G[f"mac_{name}_res"].tolist()))
        want.update(Pforward=G[f"mac_{name}_pforward"][0], sum_of_probs=G[f"mac_{name}_f"][0], i=G[f"mac_{name}_i"],
                    j=G[f"mac_{name}_j"], states=G[f"mac_{name}_states"], P_posterior=G[f"mac_{name}_ppost"])
        _check(hits[0], paths[0], want)
        import hashlib
        post = hhg.capi.mac_debug_posterior(gpu_ctx, 0, int(db.Lh[t]))
        sha = np.frombuffer(hashlib.sha256(np.ascontiguousarray(post[1:, 1:]).tobytes()).digest(), np.uint8)
        assert np.array_equal(sha, G[f"mac_{name}_post_sha"])
        if name == "tself":
            ex = [(G["mac_tself_i"][1:], G["mac_tself_j"][1:])]
            h2, p2 = hhg.capi.mac_realign(gpu_ctx, db, [t], [vit], excl=ex, mact=mact)
            assert [int(h2[f][0]) for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols")] == G["mac_tself2_res"].tolist()
            assert float(h2["pforward"][0]) == G["mac_tself2_pforward"][0]
            n2 = int(h2["nsteps"][0])
            assert np.array_equal(p2[0]["i"][1:], G["mac_tself2_i"][1:n2 + 1])
            assert np.array_equal(bits(p2[0]["P_posterior"][1:]), bits(G["mac_tself2_ppost"][1:n2 + 1]))
    db.close()


@pytest.mark.parametrize("local,mact", [(True, 0.35), (True, 0.0), (False, 0.1)])
def test_mac_batch_equals_oracle(hhg, gpu_ctx, oracle, local, mact):
    """A batch of hits of one query (related, unrelated, short, long, L=1 templates): Viterbi on the GPU, MAC on the
    GPU, every hit against the oracle fed with the same Viterbi path; full posterior matrices compared."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(101)
    Lq = 137
    qp, qtr, qss, qpav, qcols = synth.query_profile(Lq, 23)
    lens = [137, 60, 300, 25, 1, 200, 90, 33, 410, 150]
    tg = [synth.prepared_profile(L, rng, qcols if k % 3 != 2 else None, noise=0.1 + 0.05 * k) for k, L in enumerate(lens)]
    gpu_ctx.set_query(qp, qtr)
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    hits, paths = hhg.viterbi_search(gpu_ctx, db)
    vits, ids = [], []
    for t in range(len(tg)):
        ns = int(hits["nsteps"][t])
        if ns == 0:
            continue
        i_s, j_s, st = hhg.expand_path(hits[t], paths)
        vits.append((int(hits["i1"][t]), int(hits["i2"][t]), int(hits["j1"][t]), int(hits["j2"][t]), ns, i_s, j_s))
        ids.append(t)
    assert len(ids) >= 7
    qlin = oracle.log2lin(qtr)
    hhg.capi.mac_query_set(gpu_ctx, qp, hhg.capi.log2lin(qtr))
    mh, mp = hhg.capi.mac_realign(gpu_ctx, db, ids, vits, local=local, mact=mact)
    nonempty = 0
    for r, t in enumerate(ids):
        want = oracle.mac_realign(qp, qlin, tg[t][0], oracle.log2lin(tg[t][1]), vits[r], local=local, mact=mact)
        _check(mh[r], mp[r], want)
        post = hhg.capi.mac_debug_posterior(gpu_ctx, r, lens[t])
        assert np.array_equal(bits(post[1:, 1:]), bits(want["post"][1:, 1:])), (t, "posterior matrix")
        nonempty += want["nsteps"] > 0
    assert nonempty >= 3
    db.close()


def test_mac_alternative_alignments_loop(hhg, gpu_ctx, oracle):
    """mac.realign (mirror of PosteriorDecoderRunner::executeComputation): the Viterbi runner's alternative alignments
    of each template are realigned in irep order, each round excluding the MAC alignments found before."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(7)
    Lq = 100
    qp, qtr, qss, qpav, qcols = synth.query_profile(Lq, 31)
    tg = []
    for k in range(5):
        a = synth.prepared_profile(Lq, rng, qcols, noise=0.15)
        b = synth.prepared_profile(Lq, rng, qcols, noise=0.2)
        if k % 2 == 0:   # two copies of the query in one template -> a genuine second alignment
            tg.append((np.ascontiguousarray(np.concatenate([a[0][:-1], b[0][1:]])),
                       np.ascontiguousarray(np.concatenate([a[1][:-1], b[1]])), None))
        else:
            tg.append(a)
    gpu_ctx.set_query(qp, qtr)
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    vhits = hhg.runner.ViterbiRunner(gpu_ctx, db, altali=3, smin=20.0).alignment()
    assert max(h.irep for h in vhits) >= 2
    got = hhg.mac.realign(gpu_ctx, db, qp, qtr, vhits, mact=0.35)
    vhits = [h for h in vhits if h.nsteps > 0]
    assert set(got) == {(h.target, h.irep) for h in vhits}
    qlin = oracle.log2lin(qtr)
    by_t = {}
    for h in sorted(vhits, key=lambda h: (h.target, h.irep)):
        by_t.setdefault(h.target, []).append(h)
    for t, hs in by_t.items():
        alt_i, alt_j = [], []
        for h in hs:
            ex = [(np.array(alt_i, np.int32), np.array(alt_j, np.int32))] if alt_i else ()
            want = oracle.mac_realign(qp, qlin, tg[t][0], oracle.log2lin(tg[t][1]),
                                      (h.i1, h.i2, h.j1, h.j2, h.nsteps, h.i, h.j), excl=ex, mact=0.35)
            m = got[(t, h.irep)]
            assert (m.i1, m.i2, m.j1, m.j2, m.nsteps, m.matched_cols) == tuple(want[f] for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols"))
            assert m.pforward == want["Pforward"]
            n = want["nsteps"]
            assert np.array_equal(m.i[1:], want["i"][1:n + 1]) and np.array_equal(bits(m.P_posterior[1:]), bits(want["P_posterior"][1:n + 1]))
            if n:
                alt_i += want["i"][1:n + 1].tolist(); alt_j += want["j"][1:n + 1].tolist()
            else:
                alt_i.append(want["i2"]); alt_j.append(want["j2"])
    db.close()


def test_mac_against_compiled_reference(hhg, gpu_ctx, refshim):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(55)
    Lq = 96
    qp, qtr, qss, qpav, qcols = synth.query_profile(Lq, 11)
    refshim.set_query(qp, qtr, qpav, None)
    tg = [synth.prepared_profile(L, rng, qcols if k != 3 else None, noise=0.15 + 0.1 * k) for k, L in enumerate([122, 111, 30, 25, 200])]
    gpu_ctx.set_query(qp, qtr)
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    hhg.capi.mac_query_set(gpu_ctx, qp, hhg.capi.log2lin(qtr))
    for t, (tp, ttr, _) in enumerate(tg):
        sc, i2, j2, bt = refshim.viterbi([(tp, ttr, None)])[0]
        n, i_s, j_s, st, mc = refshim.backtrace(0)
        if n == 0:
            continue
        vit = (int(i_s[n]), i2, int(j_s[n]), j2, n, i_s, j_s)
        for local, mact in ((True, 0.35), (False, 0.1)):
            ref = refshim.mac_realign(tp, ttr, vit, local=local, mact=mact)
            mh, mp = hhg.capi.mac_realign(gpu_ctx, db, [t], [vit], local=local, mact=mact)
            _check(mh[0], mp[0], ref)
            post = hhg.capi.mac_debug_posterior(gpu_ctx, 0, tp.shape[0] - 2)
            assert np.array_equal(bits(post[1:, 1:]), bits(ref["post"][1:, 1:]))
    db.close()


def test_mac_with_excluded_regions(hhg, gpu_ctx, refshim):
    """-excl / -template_excl in the realignment (PosteriorDecoder::exclude_regions / exclude_template_regions,
    src/hhposteriordecoder.cpp:120-152): the context's regions switch off whole query rows / template columns."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(56)
    Lq = 120
    qp, qtr, qss, qpav, qcols = synth.query_profile(Lq, 12)
    refshim.set_query(qp, qtr, qpav, None)
    tg = [synth.prepared_profile(L, rng, qcols, noise=0.2) for L in (130, 118)]
    gpu_ctx.set_query(qp, qtr)
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    hhg.capi.mac_query_set(gpu_ctx, qp, hhg.capi.log2lin(qtr))
    try:
        for (qreg, treg) in (([(30, 45)], []), ([], [(50, 70), (100, 400)]), ([(1, 5), (60, 62)], [(10, 12)])):
            refshim.set_mac_exclstr(",".join(f"{a}-{b}" for a, b in qreg), ",".join(f"{a}-{b}" for a, b in treg))
            gpu_ctx.set_excluded_regions(qreg, treg)
            for t, (tp, ttr, _) in enumerate(tg):
                sc, i2, j2, bt = refshim.viterbi([(tp, ttr, None)])[0]
                n, i_s, j_s, st, mc = refshim.backtrace(0)
                vit = (int(i_s[n]), i2, int(j_s[n]), j2, n, i_s, j_s)
                ref = refshim.mac_realign(tp, ttr, vit, local=True, mact=0.35)
                mh, mp = hhg.capi.mac_realign(gpu_ctx, db, [t], [vit], local=True, mact=0.35)
                _check(mh[0], mp[0], ref)
                post = hhg.capi.mac_debug_posterior(gpu_ctx, 0, tp.shape[0] - 2)
                assert np.array_equal(bits(post[1:, 1:]), bits(ref["post"][1:, 1:]))
    finally:
        refshim.set_mac_exclstr("", "")
        gpu_ctx.set_excluded_regions([], [])
    db.close()


def test_mac_error_paths(hhg, gpu_ctx):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(1)
    qp, qtr, qss, qpav, qcols = synth.query_profile(50, 3)
    tg = [synth.prepared_profile(40, rng, qcols, noise=0.2)]
    gpu_ctx.set_query(qp, qtr)
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    hhg.capi.mac_query_set(gpu_ctx, qp, hhg.capi.log2lin(qtr))
    ok = (1, 5, 1, 5, 5, np.arange(6), np.arange(6))
    hhg.capi.mac_realign(gpu_ctx, db, [0], [ok])
    with pytest.raises(hhg.HhgError, match="out of range"):
        hhg.capi.mac_realign(gpu_ctx, db, [7], [ok])
    with pytest.raises(hhg.HhgError, match="end points|leaves the matrix"):
        hhg.capi.mac_realign(gpu_ctx, db, [0], [(1, 5, 1, 45, 5, np.arange(6), np.arange(6))])
    with pytest.raises(hhg.HhgError, match="leaves the matrix"):
        hhg.capi.mac_realign(gpu_ctx, db, [0], [(1, 5, 1, 5, 5, np.arange(6), np.arange(6) + 40)])
    db.close()


# --------------------------------------------------------------------------- long queries and templates
# hhg_mac_realign runs a request in one of three places chosen from its template length (tests/mac_cases.py): the 64 KiB
# shared-memory launch on the context's stream, the 200 KiB launch on the auxiliary stream (requests mapped through
# req_map), or the global row scratch inside that second launch.  The tests below put requests on both sides of each
# boundary, in one call and in single-class calls, and compare every request with the oracle.
def _oracle_mac(oracle, q, t, vit, local, mact, excl=()):
    return oracle.mac_realign(q[0], oracle.log2lin(q[1]), t[0], oracle.log2lin(t[1]), vit, excl=excl, local=local,
                              mact=mact)


def _gpu_vits(hhg, ctx, db):
    """{target: Viterbi (i1, i2, j1, j2, nsteps, i_steps, j_steps)} of every target with a non-empty path."""
    hits, paths = hhg.viterbi_search(ctx, db)
    out = {}
    for t in range(db.n):
        ns = int(hits["nsteps"][t])
        if ns:
            i_s, j_s, _ = hhg.expand_path(hits[t], paths)
            out[t] = (int(hits["i1"][t]), int(hits["i2"][t]), int(hits["j1"][t]), int(hits["j2"][t]), ns, i_s, j_s)
    return out


def _mac_checked(hhg, ctx, db, oracle, q, tg, ids, vits, local, mact):
    """One hhg_mac_realign call over `ids`; every request (hit fields, path, per-step posteriors, posterior matrix)
    against the oracle, all mismatching requests reported together.  Returns the number of kernel launches the call
    made."""
    before = ctx.launches
    mh, mp = hhg.capi.mac_realign(ctx, db, ids, [vits[t] for t in ids], local=local, mact=mact)
    launches = ctx.launches - before
    bad = []
    for r, t in enumerate(ids):
        Lt = tg[t][0].shape[0] - 2
        got = {f: int(mh[f][r]) for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols")}
        got.update(Pforward=float(mh["pforward"][r]), sum_of_probs=mh["sum_of_probs"][r], i=mp[r]["i"], j=mp[r]["j"],
                   states=mp[r]["states"], P_posterior=mp[r]["P_posterior"], post=hhg.capi.mac_debug_posterior(ctx, r, Lt))
        try:
            mc.assert_same(_oracle_mac(oracle, q, tg[t], vits[t], local, mact), got, (r, t, Lt, local, mact))
        except AssertionError as e:
            bad.append(e.args[0] if e.args else (r, t, Lt))
    assert not bad, bad
    return launches


def _is_large(Lt):
    return mc.need(Lt) > mc.SMALL_WINDOW


@functools.lru_cache(maxsize=None)
def _long_case():
    """Lq = 1200 against a homolog at every boundary length and one unrelated template, in an order where small and
    large requests interleave."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(2024)
    q = synth.query_profile(1200, 61)
    tg = [mc.embedded(L, q[4], rng) for L in mc.BOUNDARY_LENGTHS] + [synth.prepared_profile(800, rng)]
    order = [2, 0, 5, 3, 1, 6, 4]       # 558, 1, 3000, 1747, 557, 800 (unrelated), 1748
    return q, [tg[k] for k in order]


@pytest.mark.parametrize("local,mact", mc.MODES)
def test_mac_long_mixed_call(hhg, gpu_ctx, oracle, local, mact):
    """One call holding requests of all three kinds: two launches on two streams, the large one reading its requests
    through req_map.  The small-only and large-only calls of the same requests make one launch fewer."""
    q, tg = _long_case()
    gpu_ctx.set_query(q[0], q[1])
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    vits = _gpu_vits(hhg, gpu_ctx, db)
    ids = sorted(vits)
    assert len(ids) == len(tg)
    large = [_is_large(tg[t][0].shape[0] - 2) for t in ids]
    assert any(large) and not all(large) and large != sorted(large)    # req_map is not the identity
    hhg.capi.mac_query_set(gpu_ctx, q[0], hhg.capi.log2lin(q[1]))
    mixed = _mac_checked(hhg, gpu_ctx, db, oracle, q, tg, ids, vits, local, mact)
    small_only = _mac_checked(hhg, gpu_ctx, db, oracle, q, tg, [t for t, b in zip(ids, large) if not b], vits, local, mact)
    large_only = _mac_checked(hhg, gpu_ctx, db, oracle, q, tg, [t for t, b in zip(ids, large) if b], vits, local, mact)
    assert mixed == small_only + 1 and large_only == small_only, (mixed, small_only, large_only)
    db.close()


@pytest.mark.parametrize("lens,local,mact", [((mc.LARGE_MIN, mc.WINDOW_MAX), True, 0.35),
                                             ((mc.FALLBACK_MIN, mc.LONG_LT), False, 0.1),
                                             ((mc.WINDOW_MAX, mc.FALLBACK_MIN, mc.LARGE_MIN, mc.LONG_LT), True, 0.0)],
                         ids=["window", "fallback", "window+fallback"])
def test_mac_long_single_class(hhg, gpu_ctx, oracle, lens, local, mact):
    """Calls with no small request: only requests inside the 200 KiB window, only global-scratch requests, and one
    large launch holding both."""
    q, tg = _long_case()
    gpu_ctx.set_query(q[0], q[1])
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    vits = _gpu_vits(hhg, gpu_ctx, db)
    by_len = {tg[t][0].shape[0] - 2: t for t in vits}
    ids = [by_len[L] for L in lens]
    hhg.capi.mac_query_set(gpu_ctx, q[0], hhg.capi.log2lin(q[1]))
    _mac_checked(hhg, gpu_ctx, db, oracle, q, tg, ids, vits, local, mact)
    db.close()


def test_mac_underflow_clamp_against_compiled_reference(hhg, gpu_ctx, refshim):
    """The near-self Lq = 1500 hit whose forward scale product falls below DBL_MIN*100 (both clamp branches run), in
    the 200 KiB window, against the compiled reference."""
    Lq = 1500
    (qp, qtr, qss, qpav, qcols), t = mc.near_self(Lq, 78)
    refshim.set_query(qp, qtr, qpav, None)
    vit = mc.ref_viterbi(refshim, t[0], t[1])
    assert mc.first_clamped_row(refshim.mac_forward_only(t[0], t[1], vit)["scale"], Lq) < Lq
    gpu_ctx.set_query(qp, qtr)
    db = hhg.TargetDB.from_profiles(gpu_ctx, [t])
    hhg.capi.mac_query_set(gpu_ctx, qp, hhg.capi.log2lin(qtr))
    for local, mact in mc.MODES:
        ref = refshim.mac_realign(t[0], t[1], vit, local=local, mact=mact)
        mh, mp = hhg.capi.mac_realign(gpu_ctx, db, [0], [vit], local=local, mact=mact)
        _check(mh[0], mp[0], ref)
        post = hhg.capi.mac_debug_posterior(gpu_ctx, 0, Lq)
        assert np.array_equal(bits(post[1:, 1:]), bits(ref["post"][1:, 1:])), (local, mact)
    db.close()


@pytest.mark.parametrize("Lq", [1, 2])
def test_mac_query_of_one_or_two_columns(hhg, gpu_ctx, oracle, Lq):
    """Lq = 1 skips the forward row loop and the backward row loop; Lq = 2 runs each once.  Short templates, a
    window-sized one and a global-scratch one, in one call."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(300 + Lq)
    q = synth.query_profile(Lq, 90 + Lq)
    tg = [mc.embedded(L, q[4], rng) for L in (1, 2, 60, 600, mc.FALLBACK_MIN + 52)]
    gpu_ctx.set_query(q[0], q[1])
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    vits = _gpu_vits(hhg, gpu_ctx, db)
    assert sorted(vits) == list(range(len(tg)))
    hhg.capi.mac_query_set(gpu_ctx, q[0], hhg.capi.log2lin(q[1]))
    for local, mact in mc.MODES:
        _mac_checked(hhg, gpu_ctx, db, oracle, q, tg, sorted(vits), vits, local, mact)
    db.close()


def test_mac_alternative_alignments_fallback(hhg, gpu_ctx, oracle):
    """mac.realign's exclusion rounds on templates with two copies of the query: one longer than the 200 KiB window
    (global scratch), one inside it."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(17)
    Lq = 300
    q = synth.query_profile(Lq, 33)
    qp, qtr = q[0], q[1]
    tg = [mc.two_copies(Lq, mc.FALLBACK_MIN + 152, q[4], rng), mc.two_copies(Lq, 1000, q[4], rng)]
    gpu_ctx.set_query(qp, qtr)
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    vhits = hhg.runner.ViterbiRunner(gpu_ctx, db, altali=3, smin=20.0).alignment()
    vhits = [h for h in vhits if h.nsteps > 0]
    for t in range(len(tg)):
        assert max(h.irep for h in vhits if h.target == t) >= 2, t
    got = hhg.mac.realign(gpu_ctx, db, qp, qtr, vhits, mact=0.35)
    assert set(got) == {(h.target, h.irep) for h in vhits}
    by_t = {}
    for h in sorted(vhits, key=lambda h: (h.target, h.irep)):
        by_t.setdefault(h.target, []).append(h)
    for t, hs in by_t.items():
        alt_i, alt_j = [], []
        for h in hs:
            ex = [(np.array(alt_i, np.int32), np.array(alt_j, np.int32))] if alt_i else ()
            want = _oracle_mac(oracle, q, tg[t], (h.i1, h.i2, h.j1, h.j2, h.nsteps, h.i, h.j), True, 0.35, ex)
            m = got[(t, h.irep)]
            assert (m.i1, m.i2, m.j1, m.j2, m.nsteps, m.matched_cols) == tuple(want[f] for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols"))
            assert m.pforward == want["Pforward"]
            n = want["nsteps"]
            assert np.array_equal(m.i[1:], want["i"][1:n + 1]) and np.array_equal(m.j[1:], want["j"][1:n + 1])
            assert np.array_equal(bits(m.P_posterior[1:]), bits(want["P_posterior"][1:n + 1]))
            if n:
                alt_i += want["i"][1:n + 1].tolist(); alt_j += want["j"][1:n + 1].tolist()
            else:
                alt_i.append(want["i2"]); alt_j.append(want["j2"])
    db.close()


def test_mac_short_call_after_long_call(hhg, gpu_ctx, oracle):
    """Scratch reuse on one context: a long call (global-scratch requests) leaves larger, dirty buffers behind; a short
    call that follows, and its posterior matrices, still equal the oracle."""
    from hhsuite_b200 import synth
    q, tg = _long_case()
    gpu_ctx.set_query(q[0], q[1])
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    vits = _gpu_vits(hhg, gpu_ctx, db)
    hhg.capi.mac_query_set(gpu_ctx, q[0], hhg.capi.log2lin(q[1]))
    hhg.capi.mac_realign(gpu_ctx, db, sorted(vits), [vits[t] for t in sorted(vits)], mact=0.0)
    db.close()
    rng = np.random.default_rng(5)
    qs = synth.query_profile(90, 8)
    ts = [synth.prepared_profile(L, rng, qs[4] if k != 1 else None, noise=0.2) for k, L in enumerate((90, 40, 130, 1))]
    gpu_ctx.set_query(qs[0], qs[1])
    db = hhg.TargetDB.from_profiles(gpu_ctx, ts)
    vs = _gpu_vits(hhg, gpu_ctx, db)
    hhg.capi.mac_query_set(gpu_ctx, qs[0], hhg.capi.log2lin(qs[1]))
    _mac_checked(hhg, gpu_ctx, db, oracle, qs, ts, sorted(vs), vs, True, 0.35)
    db.close()
