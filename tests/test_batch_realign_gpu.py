"""Query batches past the first Viterbi pass: path exclusions in hhg_viterbi_search_batch (the alternative alignments of
runner.BatchViterbiRunner) and the query-batch MAC realignment (hhg_mac_query_set_batch + hhg_mac_realign_batch,
mac.realign_batch).  Every result is compared, request by request and bit for bit, with the single-query calls
(hhg_db_apply_null_model + hhg_query_set / hhg_mac_query_set + hhg_viterbi_search / hhg_mac_realign for each query), and
samples with the C oracle and the compiled reference: end points, nsteps, matched_cols, sum_of_probs, Pforward, paths,
per-step posteriors and, after single-wave calls, the posterior matrices."""
import ctypes as C

import numpy as np
import pytest

from tests import batch_cases as bc
from tests import mac_cases as mc
from tests.test_kernel_variants_gpu import env_ctx
from tests.util import bits

pytestmark = pytest.mark.gpu

MAC_FIELDS = ("i1", "i2", "j1", "j2", "nsteps", "matched_cols", "flags")
VIT_FIELDS = ("target", "irep", "lastrep", "i1", "i2", "j1", "j2", "nsteps", "matched_cols")


# ------------------------------------------------------------------------------------------------ helpers
def _raw_db(hhg, ctx, targets, seed):
    """targets as a raw shard (emissions before the null model + pav); returns (db, raw targets, t_pav)."""
    rng = np.random.default_rng(seed)
    raw, pav = zip(*[bc.raw_profile(t, rng) for t in targets])
    L = np.array([t[0].shape[0] - 2 for t in targets], np.int32)
    p_off = np.concatenate([[0], np.cumsum(L.astype(np.int64) + 2)[:-1]])
    tr_off = np.concatenate([[0], np.cumsum(L.astype(np.int64) + 1)[:-1]])
    ss = None if any(r[2] is None for r in raw) else np.concatenate([r[2] for r in raw])
    db = hhg.TargetDB(ctx, L, np.concatenate([r[0] for r in raw]), np.concatenate([r[1] for r in raw]), p_off, tr_off,
                      ss, pav=np.stack(pav))
    return db, list(raw), np.stack(pav)


def _vit(hhg, hit, paths):
    i_s, j_s, _ = hhg.expand_path(hit, paths)
    return (int(hit["i1"]), int(hit["i2"]), int(hit["j1"]), int(hit["j2"]), int(hit["nsteps"]), i_s, j_s)


def _viterbi_requests(hhg, ctx, db, qs, q_pav, req_q, ids, cs, pb):
    """First-pass Viterbi hits of a query batch over a raw shard; the requests with an alignment, as MAC inputs."""
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"]) for q in qs], q_pav=q_pav)
    hits, paths = hhg.capi.viterbi_search_batch(ctx, db, req_q, ids, columnscore=cs, pb=pb)
    keep = np.nonzero(hits["nsteps"] > 0)[0]
    return (np.ascontiguousarray(req_q[keep]), np.ascontiguousarray(ids[keep]),
            [_vit(hhg, hits[k], paths) for k in keep])


def _posterior(hhg, ctx, r, Lq, Lt):
    out = np.zeros((Lq + 1, Lt + 1), np.float32)
    hhg.capi._ck(ctx.L.hhg_mac_debug_posterior(ctx.h, r, out.ctypes.data_as(C.POINTER(C.c_float))))
    return out


def _mac_batch(hhg, ctx, db, qs, q_pav, rq, ids, vits, cs, pb, local, mact, excl=None, posts=True):
    hhg.capi.mac_query_set_batch(ctx, [(q["p"], hhg.capi.log2lin(q["tr"])) for q in qs], q_pav)
    h, p = hhg.capi.mac_realign_batch(ctx, db, rq, ids, vits, excl, cs, pb, local=local, mact=mact)
    post = [_posterior(hhg, ctx, r, qs[rq[r]]["p"].shape[0] - 2, int(db.Lh[ids[r]])) for r in range(len(ids))] \
        if posts else None
    return h, p, post


def _mac_per_query(hhg, ctx, db, qs, q_pav, rq, ids, vits, cs, pb, local, mact, excl=None, posts=True):
    """The same requests with the single-query calls on the raw shard: hhg_db_apply_null_model, hhg_mac_query_set and
    hhg_mac_realign for each query."""
    n = len(ids)
    H = np.zeros(n, hhg.capi.MAC_HIT_DTYPE)
    P, POST = [None] * n, [None] * n
    for q in np.unique(rq):
        db.apply_null_model(q_pav[q], pb, cs)
        m = np.nonzero(rq == q)[0]
        hhg.capi.mac_query_set(ctx, qs[q]["p"], hhg.capi.log2lin(qs[q]["tr"]))
        h, p = hhg.capi.mac_realign(ctx, db, ids[m], [vits[k] for k in m],
                                    [excl[k] for k in m] if excl is not None else None, local=local, mact=mact)
        H[m] = h
        for k, r in enumerate(m):
            P[r] = p[k]
            if posts:
                POST[r] = _posterior(hhg, ctx, k, qs[q]["p"].shape[0] - 2, int(db.Lh[ids[r]]))
    return H, P, POST


def _same_mac(a, b, what=()):
    """Two MAC results (hits, paths, posteriors) request by request, every value on its bits."""
    ha, pa, qa = a
    hb, pb_, qb = b
    assert len(ha) == len(hb)
    for r in range(len(ha)):
        for f in MAC_FIELDS:
            assert ha[f][r] == hb[f][r], (what, r, f, ha[f][r], hb[f][r])
        assert bits(ha["sum_of_probs"][r]) == bits(hb["sum_of_probs"][r]), (what, r, "sum_of_probs")
        assert ha["pforward"][r].view(np.uint64) == hb["pforward"][r].view(np.uint64), (what, r, "pforward")
        n = int(ha["nsteps"][r])
        for f in ("i", "j", "states"):
            assert np.array_equal(pa[r][f][1:n + 1], pb_[r][f][1:n + 1]), (what, r, f)
        assert np.array_equal(bits(pa[r]["P_posterior"][1:n + 1]), bits(pb_[r]["P_posterior"][1:n + 1])), (what, r)
        if qa is not None and qb is not None:
            assert np.array_equal(bits(qa[r][1:, 1:]), bits(qb[r][1:, 1:])), (what, r, "posterior matrix")


def _check_oracle(hit, path, post, want, what=()):
    for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols"):
        assert int(hit[f]) == want[f], (what, f)
    assert float(hit["pforward"]) == want["Pforward"], what
    assert bits(hit["sum_of_probs"]) == bits(np.float32(want["sum_of_probs"])), what
    n = want["nsteps"]
    for f in ("i", "j", "states"):
        assert np.array_equal(path[f][1:n + 1], want[f][1:n + 1]), (what, f)
    assert np.array_equal(bits(path["P_posterior"][1:n + 1]), bits(want["P_posterior"][1:n + 1])), what
    if post is not None:
        assert np.array_equal(bits(post[1:, 1:]), bits(want["post"][1:, 1:])), (what, "posterior matrix")


def _excl_mask(Lq, Lt, steps):
    """Viterbi::ExcludeAlignment (src/hhviterbi.cpp:61-77): the +-40 cross around every given step."""
    m = np.zeros((Lq + 1, Lt + 1), np.uint8)
    for i, j in zip(*steps):
        m[max(i - 40, 1):min(i + 40, Lq) + 1, j] = 1
        m[i, max(j - 40, 1):min(j + 40, Lt) + 1] = 1
    return m


@pytest.fixture(scope="module")
def survivors(hhg):
    """The survivors batch of batch_cases on a raw shard, a distinct q_pav per query (module-wide context)."""
    b = bc.make_batch("survivors")
    ctx = hhg.Context()
    db, raw, t_pav = _raw_db(hhg, ctx, b["targets"], 17)
    rng = np.random.default_rng(5)
    pb = rng.dirichlet(np.ones(20) * 6).astype(np.float32)
    q_pav = np.stack([q["pav"] for q in b["queries"]]).astype(np.float32)
    assert len({bits(v).tobytes() for v in q_pav}) == len(q_pav)
    yield dict(b=b, ctx=ctx, db=db, raw=raw, t_pav=t_pav, pb=pb, q_pav=q_pav)
    db.close(); ctx.close()


# ------------------------------------------------------------------------------------------------ batch == per query
@pytest.mark.parametrize("cs,local,mact", [(1, True, 0.35), (1, True, 0.0), (1, False, 0.35), (1, False, 0.0),
                                           (0, True, 0.35), (2, False, 0.0), (3, True, 0.0)])
def test_batch_equals_per_query(hhg, oracle, survivors, cs, local, mact):
    """hhg_mac_realign_batch over a raw shard == apply_null_model(q) + hhg_mac_query_set(q) + hhg_mac_realign for every
    query, request for request, posterior matrices included; a sample == the oracle on numpy-null-modelled templates."""
    S = survivors
    b, ctx, db = S["b"], S["ctx"], S["db"]
    qs = b["queries"]
    rq, ids, vits = _viterbi_requests(hhg, ctx, db, qs, S["q_pav"], b["req_q"], b["ids"], cs, S["pb"])
    assert len(np.unique(rq)) >= 15 and len(ids) >= 300
    got = _mac_batch(hhg, ctx, db, qs, S["q_pav"], rq, ids, vits, cs, S["pb"], local, mact)
    want = _mac_per_query(hhg, ctx, db, qs, S["q_pav"], rq, ids, vits, cs, S["pb"], local, mact)
    _same_mac(got, want, (cs, local, mact))
    assert int(np.sum(got[0]["nsteps"] > 0)) >= (5 if mact else 50)
    # oracle sample: the smallest request of a few queries (Lq 1, 2 and longer ones among them)
    Lq = b["q_lens"][rq]; cells = (Lq + 1) * (b["t_lens"][ids] + 1)
    for q in sorted(set(rq.tolist()))[::4][:5]:
        m = np.nonzero(rq == q)[0]
        r = int(m[np.argmin(cells[m])])
        t = int(ids[r])
        tp = bc.null_model(S["raw"][t][0], S["t_pav"][t], S["q_pav"][q], S["pb"], cs)
        w = oracle.mac_realign(qs[q]["p"], oracle.log2lin(qs[q]["tr"]), tp, oracle.log2lin(S["raw"][t][1]), vits[r],
                               local=local, mact=mact)
        _check_oracle(got[0][r], got[1][r], got[2][r], w, (q, t))


def test_raw_shard_state_does_not_matter(hhg, survivors):
    """The batch reads the raw records: a shard last prepared for another query and columnscore (or never) gives the
    same bits."""
    S = survivors
    b, ctx, db = S["b"], S["ctx"], S["db"]
    qs = b["queries"]
    rq, ids, vits = _viterbi_requests(hhg, ctx, db, qs, S["q_pav"], b["req_q"], b["ids"], 1, S["pb"])
    sel = np.nonzero(np.isin(rq, [4, 9, 13]))[0]
    rq, ids, vits = rq[sel], ids[sel], [vits[k] for k in sel]
    first = _mac_batch(hhg, ctx, db, qs, S["q_pav"], rq, ids, vits, 1, S["pb"], True, 0.35)
    for other, cs in ((S["q_pav"][0], 3), (S["pb"], 0), (S["q_pav"][13], 1)):
        db.apply_null_model(other, S["pb"], cs)
        _same_mac(_mac_batch(hhg, ctx, db, qs, S["q_pav"], rq, ids, vits, 1, S["pb"], True, 0.35), first, cs)


# ------------------------------------------------------------------------------------------------ alternative alignments
def _same_hits(a, b, what=()):
    assert len(a) == len(b), (what, len(a), len(b))
    for k, (x, y) in enumerate(zip(a, b)):
        for f in VIT_FIELDS:
            assert getattr(x, f) == getattr(y, f), (what, k, f)
        for f in ("score", "score_ss", "vit_score"):
            assert bits(np.float32(getattr(x, f))) == bits(np.float32(getattr(y, f))), (what, k, f)
        for f in ("i", "j", "states"):
            assert np.array_equal(getattr(x, f), getattr(y, f)), (what, k, f)


@pytest.mark.parametrize("regions", [False, True], ids=["plain", "excl_regions"])
def test_alternative_alignments_and_realignment(hhg, oracle, survivors, regions):
    """runner.BatchViterbiRunner (altali 4) == runner.ViterbiRunner per query on the shard prepared for that query, every
    hit of every pass, with and without -excl / -template_excl; pass-2 hits of a sample == the oracle's Viterbi with the
    ExcludeAlignment mask; then mac.realign_batch == mac.realign per query on those hits."""
    S = survivors
    b, ctx, db, pb = S["b"], S["ctx"], S["db"], S["pb"]
    qs, cs = b["queries"], 1
    reg = ([(3, 5), (60, 70)], [(2, 2), (31, 33), (500, 520)]) if regions else ((), ())
    ctx.set_excluded_regions(*reg)
    try:
        hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"]) for q in qs], q_pav=S["q_pav"])
        got = hhg.runner.BatchViterbiRunner(ctx, db, altali=4, smin=20.0, columnscore=cs, pb=pb).alignment(
            b["req_q"], b["ids"])
        assert max(h.irep for hq in got for h in hq) >= 2
        want = []
        for q, qq in enumerate(qs):
            ctx.set_query(qq["p"], qq["tr"])
            db.apply_null_model(S["q_pav"][q], pb, cs)
            ids_q = b["ids"][b["req_q"] == q]
            want.append(hhg.runner.ViterbiRunner(ctx, db, altali=4, smin=20.0).alignment(ids_q) if len(ids_q) else [])
            _same_hits(got[q], want[q], q)
        # pass 2 against the oracle: every earlier path of the (query, target) pair masked
        checked = 0
        for q, hq in enumerate(got):
            for h in hq:
                if h.irep != 2 or checked >= 6:
                    continue
                prev = [x for x in hq if x.target == h.target and x.irep == 1 and x.score > 20.0]
                Lq, Lt = qs[q]["p"].shape[0] - 2, int(b["t_lens"][h.target])
                mask = np.zeros((Lq + 1, Lt + 1), np.uint8)
                for x in prev:
                    mask |= _excl_mask(Lq, Lt, (x.i[1:x.nsteps], x.j[1:x.nsteps]))
                if regions:
                    mask |= bc.region_mask(Lq, Lt, *reg)
                tp = bc.null_model(S["raw"][h.target][0], S["t_pav"][h.target], S["q_pav"][q], pb, cs)
                sc, i2, j2, bt = oracle.viterbi(qs[q]["p"], qs[q]["tr"], tp, S["raw"][h.target][1], celloff=mask)
                n, i_s, j_s, st, mcols = oracle.backtrace(bt, i2, j2)
                assert bits(np.float32(sc)) == bits(np.float32(h.vit_score)) and (i2, j2, n) == (h.i2, h.j2, h.nsteps)
                assert np.array_equal(i_s[1:n + 1], h.i[1:]) and np.array_equal(j_s[1:n + 1], h.j[1:])
                checked += 1
        assert checked >= min(2, sum(h.irep == 2 for hq in got for h in hq)) >= 1
        # end to end: MAC realignment of every hit of every query
        queries = [(q["p"], q["tr"]) for q in qs]
        mb = hhg.mac.realign_batch(ctx, db, queries, got, q_pav=S["q_pav"], columnscore=cs, pb=pb, mact=0.35)
        for q, qq in enumerate(qs):
            if not want[q]:
                assert mb[q] == {}
                continue
            db.apply_null_model(S["q_pav"][q], pb, cs)
            ms = hhg.mac.realign(ctx, db, qq["p"], qq["tr"], want[q], mact=0.35)
            assert set(mb[q]) == set(ms), q
            for key, m in ms.items():
                g = mb[q][key]
                for f in MAC_FIELDS[:-1]:
                    assert getattr(g, f) == getattr(m, f), (q, key, f)
                assert g.pforward == m.pforward and bits(np.float32(g.sum_of_probs)) == bits(np.float32(m.sum_of_probs))
                for f in ("i", "j", "states"):
                    assert np.array_equal(getattr(g, f), getattr(m, f)), (q, key, f)
                assert np.array_equal(bits(g.P_posterior), bits(m.P_posterior)), (q, key)
        assert any(m.irep >= 2 for mq in mb for m in mq.values())    # a round that excluded earlier MAC paths
    finally:
        ctx.set_excluded_regions()


def test_batch_search_refuses_exclusions_outside_the_request(hhg, survivors):
    """Excluded steps are checked against the request's own query length, not the first query's."""
    S = survivors
    b, ctx, db = S["b"], S["ctx"], S["db"]
    qs = b["queries"]
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"]) for q in qs], q_pav=S["q_pav"])
    q_short, q_long = 1, len(qs) - 1              # Lq 2 and 1500
    rq = np.array([q_long, q_short], np.int32); ids = np.array([5, 5], np.int32)
    ok = [(np.array([100], np.int32), np.array([1], np.int32)), (np.array([2], np.int32), np.array([1], np.int32))]
    hhg.capi.viterbi_search_batch(ctx, db, rq, ids, 1, S["pb"], exclusions=ok)
    bad = [ok[0], (np.array([3], np.int32), np.array([1], np.int32))]
    with pytest.raises(hhg.capi.HhgError, match="request 1"):
        hhg.capi.viterbi_search_batch(ctx, db, rq, ids, 1, S["pb"], exclusions=bad)


# ------------------------------------------------------------------------------------------------ compiled reference
def test_batch_against_compiled_reference(hhg, refshim):
    """A few hits of two queries in one batch call == refshim.mac_realign (prepared shard)."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(57)
    qa = synth.query_profile(96, 11); qb = synth.query_profile(41, 12)
    tg = [synth.prepared_profile(L, rng, (qa if k < 3 else qb)[4], noise=0.15 + 0.05 * k)
          for k, L in enumerate([122, 111, 30, 60, 45])]
    ctx = hhg.Context()
    db = hhg.TargetDB.from_profiles(ctx, tg)
    rq, ids, vits, wants = [], [], [], []
    for q, qq in enumerate((qa, qb)):
        refshim.set_query(qq[0], qq[1], qq[3], None)
        for t in (range(3) if q == 0 else range(1, 5)):
            sc, i2, j2, bt = refshim.viterbi([(tg[t][0], tg[t][1], None)])[0]
            n, i_s, j_s, st, mcols = refshim.backtrace(0)
            if n == 0:
                continue
            v = (int(i_s[n]), i2, int(j_s[n]), j2, n, i_s, j_s)
            rq.append(q); ids.append(t); vits.append(v)
            wants.append(refshim.mac_realign(tg[t][0], tg[t][1], v, local=True, mact=0.35))
    assert set(rq) == {0, 1} and len(ids) >= 5
    qs = [dict(p=qa[0], tr=qa[1]), dict(p=qb[0], tr=qb[1])]
    h, p, post = _mac_batch(hhg, ctx, db, qs, None, np.array(rq, np.int32), np.array(ids, np.int32), vits, 1, None,
                            True, 0.35)
    for r, w in enumerate(wants):
        _check_oracle(h[r], p[r], post[r], w, r)
    db.close(); ctx.close()


# ------------------------------------------------------------------------------------------------ shapes
def test_template_size_classes_and_shared_targets(hhg, oracle):
    """One call mixes templates on both sides of the 64 KiB and 200 KiB shared-memory windows and on the global scratch
    with queries of lengths 3 .. 1200; the same target is hit by every query and one (query, target) pair twice."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(91)
    qs = bc.queries((3, 57, 400, 1200), 71)
    tg = [mc.embedded(L, qs[k % 4]["mix"], rng) for k, L in enumerate(mc.BOUNDARY_LENGTHS)]
    tg.append(synth.prepared_profile(150, rng, qs[1]["mix"], noise=0.2))
    shared = len(tg) - 1
    ctx = hhg.Context()
    db, raw, t_pav = _raw_db(hhg, ctx, tg, 23)
    q_pav = np.stack([q["pav"] for q in qs])
    req_q = [q for q in range(4) for _ in range(len(tg))] + [1]
    ids = [t for _ in range(4) for t in range(len(tg))] + [shared]
    rq, ids, vits = _viterbi_requests(hhg, ctx, db, qs, q_pav, np.array(req_q, np.int32), np.array(ids, np.int32), 2,
                                      None)
    assert np.sum(ids == shared) >= 5 and np.sum((ids == shared) & (rq == 1)) == 2
    assert {mc.SMALL_MAX, mc.LARGE_MIN, mc.FALLBACK_MIN, mc.LONG_LT} <= set(db.Lh[ids].tolist())
    for local, mact in ((True, 0.35), (False, 0.0)):
        got = _mac_batch(hhg, ctx, db, qs, q_pav, rq, ids, vits, 2, None, local, mact)
        want = _mac_per_query(hhg, ctx, db, qs, q_pav, rq, ids, vits, 2, None, local, mact)
        _same_mac(got, want, (local, mact))
    # the oracle on the shared target for every query
    for r in np.nonzero(ids == shared)[0]:
        q = int(rq[r])
        tp = bc.null_model(raw[shared][0], t_pav[shared], q_pav[q], None, 2)
        w = oracle.mac_realign(qs[q]["p"], oracle.log2lin(qs[q]["tr"]), tp, oracle.log2lin(raw[shared][1]), vits[r],
                               local=False, mact=0.0)
        _check_oracle(got[0][r], got[1][r], got[2][r], w, r)
    db.close(); ctx.close()


# ------------------------------------------------------------------------------------------------ memory waves
def _scratch_bytes(Lq, Lt):
    """Scratch of one request of hhg_mac_realign_batch over a raw shard: posterior, cell-off and backtrace bytes per
    cell, the global row buffers, the scale factors and the template's records."""
    return 6 * (Lq + 1) * (Lt + 1) + 8 * (11 * (Lt + 3) + (Lt + 3 + 7) // 8 + 1) + 8 * (Lq + 3) + 112 * Lt


def _wave_cut(Lq, Lt, budget):
    """hhg_mac_realign_batch's memory waves: list of [first, end) request ranges."""
    waves, cur, start = [], 0, 0
    for r, (a, b) in enumerate(zip(Lq, Lt)):
        nb = _scratch_bytes(int(a), int(b))
        if r and cur and cur + nb > budget:
            waves.append((start, r)); start, cur = r, 0
        cur += nb
    waves.append((start, len(Lq)))
    return waves


def test_memory_waves(hhg, gpu_ctx):
    """A small HHG_MAX_BT_GB cuts the batch into >= 4 memory waves, one of them a single request over the budget; the
    results equal the one-wave run byte for byte and the posteriors are refused after the multi-wave call."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(44)
    qs = bc.queries((1500, 300, 60, 2), 81)
    tg = [synth.prepared_profile(L, rng, qs[k % 4]["mix"] if k % 2 == 0 else None, noise=0.25)
          for k, L in enumerate([2500] + [int(x) for x in rng.integers(20, 600, 40)])]
    q_pav = np.stack([q["pav"] for q in qs])
    req_q = np.array([0] + [int(x) for x in rng.integers(0, 4, 160)], np.int32)
    ids = np.array([0] + [int(x) for x in rng.integers(0, len(tg), 160)], np.int32)
    gb = "0.004"
    with env_ctx(hhg, HHG_MAX_BT_GB=gb) as small:
        db1, _, _ = _raw_db(hhg, gpu_ctx, tg, 3)
        db2, _, _ = _raw_db(hhg, small, tg, 3)
        rq, ids_k, vits = _viterbi_requests(hhg, gpu_ctx, db1, qs, q_pav, req_q, ids, 1, None)
        one = _mac_batch(hhg, gpu_ctx, db1, qs, q_pav, rq, ids_k, vits, 1, None, True, 0.35, posts=False)
        Lq = np.array([qs[q]["p"].shape[0] - 2 for q in rq], np.int64); Lt = db1.Lh[ids_k].astype(np.int64)
        waves = _wave_cut(Lq, Lt, bc.bt_budget(gb))
        assert len(waves) >= 4
        assert any(e - a == 1 and _scratch_bytes(int(Lq[a]), int(Lt[a])) > bc.bt_budget(gb) for a, e in waves)
        hhg.capi.mac_query_set_batch(small, [(q["p"], hhg.capi.log2lin(q["tr"])) for q in qs], q_pav)
        n0 = small.launches
        h, p = hhg.capi.mac_realign_batch(small, db2, rq, ids_k, vits, None, 1, None, local=True, mact=0.35)
        expect = 1                                         # the transitions of the distinct targets
        for a, e in waves:
            big = [int(Lt[r]) > mc.SMALL_MAX for r in range(a, e)]
            expect += 2 + (2 if any(big) and not all(big) else 1)   # records + band, then one or two realign launches
        assert small.launches - n0 == expect
        assert h.tobytes() == one[0].tobytes()
        for r in range(len(ids_k)):
            for f in ("i", "j", "states", "P_posterior"):
                assert p[r][f].tobytes() == one[1][r][f].tobytes(), (r, f)
        with pytest.raises(hhg.capi.HhgError, match="memory waves"):
            _posterior(hhg, small, 0, int(Lq[0]), int(Lt[0]))
        db1.close(); db2.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_leave_the_context_usable(hhg):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(12)
    qs = bc.queries((30, 80), 33)
    tg = [synth.prepared_profile(L, rng, qs[k % 2]["mix"], noise=0.2) for k, L in enumerate((90, 40, 120))]
    ctx = hhg.Context()
    db, _, _ = _raw_db(hhg, ctx, tg, 4)
    q_pav = np.stack([q["pav"] for q in qs])
    Err = hhg.capi.HhgError
    # before any hhg_mac_query_set_batch
    ctx.mac_batch_Lq = np.array([30, 80], np.int32)
    rq, ids, vits = _viterbi_requests(hhg, ctx, db, qs, q_pav, np.array([0, 1, 1, 0], np.int32),
                                      np.array([0, 1, 2, 2], np.int32), 1, None)
    assert len(ids) == 4
    with pytest.raises(Err, match="hhg_mac_query_set_batch first"):
        hhg.capi.mac_realign_batch(ctx, db, rq, ids, vits)
    queries = [(q["p"], hhg.capi.log2lin(q["tr"])) for q in qs]
    hhg.capi.mac_query_set_batch(ctx, queries, q_pav)
    good = hhg.capi.mac_realign_batch(ctx, db, rq, ids, vits)
    with pytest.raises(Err, match="query index 2 out of range"):
        hhg.capi.mac_realign_batch(ctx, db, np.array([0, 1, 2, 0], np.int32), ids, vits)
    # a request of the 30-row query with the end points / steps of an 80-row alignment
    r80 = int(np.nonzero((rq == 1) & (np.array([v[1] for v in vits]) > 30))[0][0])
    with pytest.raises(Err, match="outside 1..30 x"):
        hhg.capi.mac_realign_batch(ctx, db, np.array([0], np.int32), ids[r80:r80 + 1], vits[r80:r80 + 1])
    v = list(vits[r80]); v[0], v[1] = 1, 30                  # end points inside, steps outside the short query
    with pytest.raises(Err, match="path leaves the matrix 1..30"):
        hhg.capi.mac_realign_batch(ctx, db, np.array([0], np.int32), ids[r80:r80 + 1], [tuple(v)])
    with pytest.raises(Err, match="columnscore 0 needs pb"):
        hhg.capi.mac_realign_batch(ctx, db, rq, ids, vits, columnscore=0)
    hhg.capi.mac_query_set_batch(ctx, queries)               # no q_pav
    with pytest.raises(Err, match="needs q_pav"):
        hhg.capi.mac_realign_batch(ctx, db, rq, ids, vits)
    # still correct afterwards
    hhg.capi.mac_query_set_batch(ctx, queries, q_pav)
    again = hhg.capi.mac_realign_batch(ctx, db, rq, ids, vits)
    assert again[0].tobytes() == good[0].tobytes()
    for a, b in zip(again[1], good[1]):
        for f in ("i", "j", "states", "P_posterior"):
            assert a[f].tobytes() == b[f].tobytes()
    db.close(); ctx.close()
