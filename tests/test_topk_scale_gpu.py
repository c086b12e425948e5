"""The device top-K selection (hhg_plan_topk, hhg_plan_topk_by_key, hhg_plan_topk_paths) at scale and at the
radix-select edges, against the plain reference order of tests/topk_cases.py.

Plans repeat a shard of seven tiny targets (L 1-3, query L 16), so n reaches 2 000 001 requests cheaply and the
scores tie massively: by score the global ids decide.  By key, every named case of topk_cases runs at several n.
n straddles 256 (one block of k_topk_keys / k_topk_emit) and 132 SMs x 4 x 256 = 135 168 keys, above which
k_topk_hist's grid-stride loop runs on an H100 SXM; K runs over 1, 255-257, n-1, n, n+1 and 3n.

Every call must return the reference order's first min(K, n) requests: their global ids, their hit records bit for
bit (plan.fetch without paths, so path_off is the plan's own), keys equal to the restated device key and strictly
increasing, owner 0, and 18 launches (19 when K > n pads the block).  Bad input is refused with the context usable."""
import types

import numpy as np
import pytest

from tests import topk_cases as tc
from tests.test_kernel_variants_gpu import env_ctx

pytestmark = pytest.mark.gpu

LQ = 16
TINY = (1, 2, 3, 1, 2, 3, 2)
N_BIG = 2_000_001
N_LIST = (1, 2, 255, 256, 257, 135_167, 135_169, N_BIG)
NAMED_N = (257, 1000, 135_169, N_BIG)


def _ks(n):
    return sorted({K for K in (1, 255, 256, 257, n - 1, n, n + 1, 3 * n) if K >= 1})


class Bed:
    """One context, the tiny shard and one run plan per n whose ids repeat its targets."""

    def __init__(self, hhg):
        from hhsuite_b200 import synth
        self.hhg = hhg
        self.ctx = hhg.Context()
        rng = np.random.default_rng(31)
        self.query = synth.query_profile(LQ, 8)[:2]
        self.ctx.set_query(*self.query)
        self.targets = [synth.prepared_profile(L, rng, None, noise=0.3) for L in TINY]
        self.db = hhg.TargetDB.from_profiles(self.ctx, self.targets)
        self.plans = {}

    @staticmethod
    def ids(n):
        return np.random.default_rng(n).integers(0, len(TINY), n).astype(np.int32)

    def plan(self, n):
        if n not in self.plans:
            p = self.hhg.Plan(self.ctx, self.db, self.ids(n))
            p.run()
            self.plans[n] = (p, p.fetch(want_paths=False)[0])
        return self.plans[n]

    def close(self):
        for p, _ in self.plans.values():
            p.close()
        self.db.close()
        self.ctx.close()


@pytest.fixture(scope="module")
def bed(hhg):
    b = Bed(hhg)
    yield b
    b.close()


def _call(ctx, fn):
    n0 = ctx.launches
    rec = fn()
    return rec, ctx.launches - n0


def _check(rec, launched, hits, gids, order, keys, K, tag):
    n = len(hits)
    m = min(K, n)
    assert launched == 18 + (K > n), (tag, launched)
    assert len(rec) == m, (tag, len(rec))
    sel = order[:m]
    assert np.array_equal(rec["target"], gids[sel]), tag
    assert np.array_equal(np.ascontiguousarray(rec["hit"]).view(np.uint8), hits[sel].view(np.uint8)), tag
    assert np.array_equal(rec["key"], keys[sel]), tag
    assert np.all(rec["key"][1:] > rec["key"][:-1]), tag
    assert np.all(rec["owner"] == 0), tag


def _by_key(hhg, ctx, plan, K, key, gids=None, id_base=0):
    return hhg.capi.plan_topk_by_key(ctx, plan.h, None, K, key, id_base=id_base, global_ids=gids)


# ------------------------------------------------------------------------------------------------ 1. scale
@pytest.mark.parametrize("n", N_LIST)
def test_by_score_and_hit_score_at_scale(bed, n):
    """Both score fields x four id forms (scattered global ids, id_base, id_base ending at INT32_MAX, scattered ids
    just below INT32_MAX) x every K; at 2 000 001 requests each (field, id form) takes one K."""
    plan, hits = bed.plan(n)
    rng = np.random.default_rng(n + 7)
    forms = [("scattered", tc.scattered_ids(n, rng), 0), ("id_base", None, 1_000_003),
             ("id_base_to_max", None, tc.INT32_MAX - n + 1),
             ("scattered_near_max", tc.scattered_ids(n, rng, lo=tc.INT32_MAX - 4 * n + 1), 0)]
    combos = [(f, flag, form) for f, flag in (("score", False), ("hit_score", True)) for form in forms]
    for ci, (field, flag, (name, gids, base)) in enumerate(combos):
        ks = _ks(n) if n < N_BIG else [K for i, K in enumerate(_ks(n)) if i % len(combos) == ci]
        g = gids if gids is not None else (base + np.arange(n)).astype(np.int32)
        order = tc.reference_order(hits[field], g, by="score")
        keys = tc.device_keys(hits[field], g, by="score")
        for K in ks:
            rec, launched = _call(bed.ctx, lambda: plan.topk(K, by_hit_score=flag, id_base=base, global_ids=gids))
            _check(rec, launched, hits, g, order, keys, K, (n, field, name, K))


@pytest.mark.parametrize("n", NAMED_N)
@pytest.mark.parametrize("name", list(tc.CASES))
def test_named_keys(hhg, bed, name, n):
    """hhg_plan_topk_by_key on every named key distribution, at the case's own Ks and at 256 / 257."""
    plan, hits = bed.plan(n)
    c = tc.case(name, n)
    order = tc.reference_order(c["key"], c["gids"])
    keys = tc.device_keys(c["key"], c["gids"])
    for K in sorted(set(c["ks"]) | {256, 257}):
        rec, launched = _call(bed.ctx, lambda: _by_key(hhg, bed.ctx, plan, K, c["key"], c["gids"]))
        _check(rec, launched, hits, c["gids"], order, keys, K, (name, n, K))


# ------------------------------------------------------------------------------------------------ 2. one plan, reused
def test_reuse_on_one_plan(hhg):
    """K growing then shrinking, by key between two by-score calls, a re-run after set_query with another query,
    hhg_ctx_last_plan after hhg_viterbi_search and a world-1 communicator against comm = NULL."""
    from hhsuite_b200 import synth
    b = Bed(hhg)                       # a context of its own: the query changes below
    try:
        ctx, n = b.ctx, 3000
        plan, hits = b.plan(n)
        rng = np.random.default_rng(5)
        gids = tc.scattered_ids(n, rng)
        order = tc.reference_order(hits["score"], gids, by="score")
        keys = tc.device_keys(hits["score"], gids, by="score")
        seen = {}
        for K in (1, 10, 300, 2999, 3000, 5000, 9000, 5000, 700, 300, 2, 1):
            rec, launched = _call(ctx, lambda: plan.topk(K, global_ids=gids))
            _check(rec, launched, hits, gids, order, keys, K, ("grow/shrink", K))
            assert rec.tobytes() == seen.setdefault(K, rec.tobytes()), K

        c = tc.case("mixed", n)
        rec, launched = _call(ctx, lambda: _by_key(hhg, ctx, plan, 700, c["key"], c["gids"]))
        _check(rec, launched, hits, c["gids"], tc.reference_order(c["key"], c["gids"]),
               tc.device_keys(c["key"], c["gids"]), 700, "by key")
        assert plan.topk(300, global_ids=gids).tobytes() == seen[300]

        ctx.set_query(*synth.query_profile(LQ, 99)[:2])
        plan.run()
        hits2 = plan.fetch(want_paths=False)[0]
        assert not np.array_equal(hits2["hit_score"], hits["hit_score"])
        rec, launched = _call(ctx, lambda: plan.topk(500, by_hit_score=True, global_ids=gids))
        _check(rec, launched, hits2, gids, tc.reference_order(hits2["hit_score"], gids, by="score"),
               tc.device_keys(hits2["hit_score"], gids, by="score"), 500, "after set_query")

        ids3 = Bed.ids(4001)
        hits3, _ = hhg.viterbi_search(ctx, b.db, ids=ids3, want_paths=False)
        last = ctx.L.hhg_ctx_last_plan(ctx.h)
        g3 = tc.scattered_ids(len(ids3), rng)
        for K in (1, 257, 4001, 4002):
            rec, launched = _call(ctx, lambda: hhg.capi.plan_topk(ctx, last, None, K, True, 0, g3))
            _check(rec, launched, hits3, g3, tc.reference_order(hits3["hit_score"], g3, by="score"),
                   tc.device_keys(hits3["hit_score"], g3, by="score"), K, ("last plan", K))

        comm = hhg.Comm(ctx)
        try:
            for K in (1, 256, 3000, 3001):
                a = plan.topk(K, comm=comm, global_ids=gids)
                assert a.tobytes() == plan.topk(K, global_ids=gids).tobytes(), K
                a = hhg.capi.plan_topk_by_key(ctx, plan.h, comm, K, c["key"], global_ids=c["gids"])
                assert a.tobytes() == _by_key(hhg, ctx, plan, K, c["key"], c["gids"]).tobytes(), K
                assert np.array_equal(plan.topk_paths(a, comm=comm), plan.topk_paths(a)), K
        finally:
            comm.close()
    finally:
        b.close()


def test_multi_wave_plan(hhg, bed):
    """A plan that ran in >= 5 memory waves (HHG_MAX_BT_GB) gives the single-wave plan's hits, top-K list and path
    rows."""
    n = 4000
    plan1, hits1 = bed.plan(n)
    with env_ctx(hhg, HHG_MAX_BT_GB="0.00002") as ctx:
        ctx.set_query(*bed.query)
        db = hhg.TargetDB.from_profiles(ctx, bed.targets)
        plan = hhg.Plan(ctx, db, Bed.ids(n))
        n0 = ctx.launches
        plan.run()
        waves = (ctx.launches - n0 - 1) // 2          # operand stream + (forward + backtrace) per wave
        assert waves >= 5, waves
        hits = plan.fetch(want_paths=False)[0]
        assert np.array_equal(hits.view(np.uint8), hits1.view(np.uint8))
        gids = tc.scattered_ids(n, np.random.default_rng(9))
        order = tc.reference_order(hits["hit_score"], gids, by="score")
        keys = tc.device_keys(hits["hit_score"], gids, by="score")
        for K in (1, 256, n, 3 * n):
            rec, launched = _call(ctx, lambda: plan.topk(K, by_hit_score=True, global_ids=gids))
            _check(rec, launched, hits, gids, order, keys, K, ("waves", K))
            assert rec.tobytes() == plan1.topk(K, by_hit_score=True, global_ids=gids).tobytes()
        rows = plan.topk_paths(rec)
        assert np.array_equal(rows, plan1.topk_paths(rec))
        assert np.array_equal(rows, _expected_rows(plan, gids, rec, rows.shape[1]))
        plan.close()
        db.close()


# ------------------------------------------------------------------------------------------------ 3. path rows
def _expected_rows(plan, gids, recs, width):
    """Row r = the first min(nsteps, width) path states of recs[r]'s request (from plan.fetch), zero padded."""
    hc, paths = plan.fetch()
    by_gid = np.argsort(gids)
    req = by_gid[np.searchsorted(gids[by_gid], recs["target"])]
    rows = np.zeros((len(recs), width), np.uint8)
    for r, k in enumerate(req):
        w = min(int(hc["nsteps"][k]), width)
        rows[r, :w] = paths[hc["path_off"][k]:hc["path_off"][k] + w]
    return rows


@pytest.fixture(scope="module")
def listbed(hhg):
    """50 000 requests over 300 targets (L 20-259, query L 120): duplicated targets give equal hits, equal statistics
    and so ties in score_aass; file names 'db/t<global id>' put the global ids in file-name order."""
    from hhsuite_b200 import synth
    ctx = hhg.Context()
    rng = np.random.default_rng(5)
    qp, qtr, _, _, qcols = synth.query_profile(120, 12)
    tg = [synth.prepared_profile(int(L), rng, qcols if k % 5 == 0 else None, noise=0.3)
          for k, L in enumerate(rng.integers(20, 260, 300))]
    ctx.set_query(qp, qtr)
    db = hhg.TargetDB.from_profiles(ctx, tg)
    ids = rng.integers(0, len(tg), 50_000).astype(np.int32)
    plan = hhg.Plan(ctx, db, ids)
    plan.run()
    hits = plan.fetch(want_paths=False)[0]
    Lt = np.array([t[0].shape[0] - 2 for t in tg], np.int32)[ids]
    neff = rng.uniform(1, 12, len(tg)).astype(np.float32)[ids]
    stats = hhg.capi.hitlist_pvalues(hits["hit_score"], hits["score_ss"], Lt, neff, 120, 5.5, len(ids))
    gids = rng.permutation(len(ids)).astype(np.int32)
    files = [f"db/t{g:06d}" for g in gids]
    yield types.SimpleNamespace(ctx=ctx, plan=plan, hits=hits, Lt=Lt, neff=neff, stats=stats, gids=gids, files=files)
    plan.close()
    db.close()
    ctx.close()


def test_topk_paths_rows(listbed):
    """Records in list, reversed and shuffled order and a subset; width = max nsteps, far wider (zero padding) and
    narrower (today's behaviour: the first width states); no records (nothing launched)."""
    b = listbed
    plan, ctx = b.plan, b.ctx
    rec = plan.topk(3000, by_hit_score=True, global_ids=b.gids)
    maxns = int(rec["hit"]["nsteps"].max())
    perm = np.random.default_rng(3).permutation(len(rec))
    narrow = maxns // 2
    assert (rec["hit"]["nsteps"] > narrow).sum() > 100
    for tag, recs in (("list", rec), ("reversed", rec[::-1]), ("shuffled", rec[perm]), ("subset", rec[5::7])):
        for width in (maxns, 4 * maxns + 3, narrow):
            n0 = ctx.launches
            rows = plan.topk_paths(recs, width=width)
            assert ctx.launches - n0 == 1
            assert np.array_equal(rows, _expected_rows(plan, b.gids, recs, width)), (tag, width)
    n0 = ctx.launches
    assert plan.topk_paths(rec[:0]).shape == (0, 1)
    assert ctx.launches == n0


# ------------------------------------------------------------------------------------------------ 4. reference order
def test_topk_by_score_aass_is_the_hitlist_order_at_scale(hhg, listbed):
    """By score_aass (hhg_hitlist_pvalues) with global ids in file-name order, the device list is hhg_hitlist_order."""
    b = listbed
    n = len(b.gids)
    key = b.stats["score_aass"]
    assert len(np.unique(key)) < n // 10                 # duplicated targets: massive ties, the ids decide
    order = hhg.capi.hitlist_order(b.stats, b.files)
    keys = tc.device_keys(key, b.gids)
    for K in (1, 1000, n, n + 1):
        rec, launched = _call(b.ctx, lambda: _by_key(hhg, b.ctx, b.plan, K, key, b.gids))
        _check(rec, launched, b.hits, b.gids, order, keys, K, ("score_aass", K))


def test_hitlist_order_at_scale_is_the_compiled_references(hhg, listbed, refshim):
    """The same list from the compiled reference's HitList::CalculatePvalues + SortList."""
    b = listbed
    ref = refshim.hitlist_stats(b.hits["hit_score"], b.hits["score_ss"], b.Lt, b.neff, 120, 5.5, len(b.gids),
                                files=b.files)
    assert np.array_equal(np.asarray(ref["score_aass"], np.float32).view(np.uint32), b.stats["score_aass"].view(np.uint32))
    rec = _by_key(hhg, b.ctx, b.plan, len(b.gids), b.stats["score_aass"], b.gids)
    assert np.array_equal(rec["target"], b.gids[ref["order"]])


# ------------------------------------------------------------------------------------------------ 5. refusals
def _refused(bed, plan, match, fn, launched):
    """fn raises HHG_EINVAL naming `match` after `launched` launches; the same plan then answers correctly."""
    ctx = bed.ctx
    n0 = ctx.launches
    with pytest.raises(bed.hhg.HhgError, match=match):
        fn()
    assert ctx.launches - n0 == launched
    hits = plan.fetch(want_paths=False)[0]
    g = np.arange(len(hits), dtype=np.int32)[::-1].copy()
    rec, l2 = _call(ctx, lambda: plan.topk(100, global_ids=g))
    _check(rec, l2, hits, g, tc.reference_order(hits["score"], g, by="score"), tc.device_keys(hits["score"], g, by="score"),
           100, ("after refusal", match))


def test_negative_global_id_is_refused(hhg, bed):
    n = 1000
    plan, hits = bed.plan(n)
    key = tc.case("mixed", n)["key"]
    for bad in (-1, -5, -tc.INT32_MAX - 1):
        gids = tc.scattered_ids(n, np.random.default_rng(1))
        gids[123] = bad
        _refused(bed, plan, "negative", lambda: plan.topk(10, global_ids=gids), 0)
        _refused(bed, plan, "negative", lambda: _by_key(hhg, bed.ctx, plan, n, key, gids), 0)


def test_id_base_outside_int32_is_refused(hhg, bed):
    n = 1000
    plan, hits = bed.plan(n)
    for base in (tc.INT32_MAX - n + 2, tc.INT32_MAX, -1, -tc.INT32_MAX - 1):
        _refused(bed, plan, "INT32_MAX", lambda: plan.topk(10, id_base=base), 0)
    base = tc.INT32_MAX - n + 1                          # the last id is INT32_MAX itself: accepted
    g = (base + np.arange(n)).astype(np.int32)
    rec, launched = _call(bed.ctx, lambda: plan.topk(n, id_base=base))
    _check(rec, launched, hits, g, tc.reference_order(hits["score"], g, by="score"),
           tc.device_keys(hits["score"], g, by="score"), n, "id_base to INT32_MAX")


def test_duplicate_global_ids_are_refused(hhg, bed):
    """Two requests with one global id: tied at the K-th key (more than K emitted), both inside the list with equal or
    different values."""
    n = 1000
    plan, hits = bed.plan(n)
    rng = np.random.default_rng(2)
    gids = tc.scattered_ids(n, rng)
    flat = np.full(n, 0.5, np.float32)                   # equal keys: the list is the id order
    a, b = int(np.argsort(gids)[400]), int(np.argsort(gids)[700])
    dup = gids.copy()
    dup[b] = dup[a]
    r = int(np.searchsorted(np.sort(dup), dup[a]))       # the pair holds list positions r and r + 1
    _refused(bed, plan, "not unique", lambda: _by_key(hhg, bed.ctx, plan, r + 1, flat, dup), 18)
    _refused(bed, plan, "not unique", lambda: _by_key(hhg, bed.ctx, plan, n, flat, dup), 18)
    _refused(bed, plan, "not unique", lambda: _by_key(hhg, bed.ctx, plan, n + 5, flat, dup), 19)
    key = np.arange(n, dtype=np.float32)                 # different values, both inside the list
    _refused(bed, plan, "not unique", lambda: _by_key(hhg, bed.ctx, plan, max(a, b) + 1, key, dup), 18)
    _refused(bed, plan, "not unique", lambda: plan.topk(n, global_ids=dup), 18)


def test_nan_key_is_refused(hhg, bed):
    n = 1000
    plan, hits = bed.plan(n)
    c = tc.case("mixed", n)
    for nan in (np.float32(np.nan), np.uint32(0xFFC00000).view(np.float32), np.uint32(0x7F800001).view(np.float32)):
        key = c["key"].copy()
        key[77] = nan
        _refused(bed, plan, "NaN", lambda: _by_key(hhg, bed.ctx, plan, 10, key, c["gids"]), 0)
