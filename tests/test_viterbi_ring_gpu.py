"""k_viterbi's target operands come through a per-lane cp.async ring in shared memory (two column slots per warp, the
next column in flight while the current one computes).  Strip heights 12 and 16 must give byte-identical hits and
paths on a bench-like shard, and both the oracle's bits; the ring's edges -- the copy of the column after a job's last
one, items and runs that follow each other on the same warps -- must not leak into any result."""
import numpy as np
import pytest

from tests.test_kernel_variants_gpu import env_ctx
from tests.test_viterbi_gpu import _check_against_oracle
from tests.test_viterbi_ties_gpu import _check_hits_against_oracle, _region_mask
from tests.util import bits, golden

pytestmark = pytest.mark.gpu

LQS = (1, 11, 12, 13, 400, 1500)
MODES = ("local", "global", "ss", "celloff")


@pytest.fixture(scope="module")
def shard():
    """~5000 targets with bench's length distribution, plus the longest lengths (1600 .. 2000) and a 1-column
    target; the first few are planted homologs of the Lq = 400 query."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(2024)
    lens = np.concatenate([[1, 2000, 1999, 1600, 1777, 2000], synth.lengths(4994, rng)]).astype(np.int32)
    q400 = synth.query_profile(400, seed=1)
    db = synth.prepared_db(len(lens), seed=77, query_cols=q400[4], planted=24, lens=lens, fast=True)
    return db


@pytest.fixture(scope="module")
def ctxs(hhg, shard):
    """One context (and resident shard) per strip height."""
    out = {}
    with env_ctx(hhg, HHG_STRIP_ROWS=16) as c16, env_ctx(hhg, HHG_STRIP_ROWS=12) as c12:
        for R, ctx in ((16, c16), (12, c12)):
            db = hhg.TargetDB(ctx, shard["L"], shard["p"], shard["tr"], shard["p_off"], shard["tr_off"],
                              ss=shard["ss"])
            out[R] = (ctx, db)
        yield out
        for ctx, db in out.values():
            db.close()


def _regions(Lq):
    qr = [(Lq // 3 + 1, Lq // 3 + 2)] if Lq >= 3 else []
    return qr, [(5, 9), (100, 104), (1600, 1650)]


def _run(hhg, ctx, db, q, mode, S33):
    """(hits, paths, plan) of one whole-shard search; cell-off mode goes through hhg_viterbi_search, which applies
    the context's excluded regions (plan None)."""
    qp, qtr, qss = q[0], q[1], q[2]
    if mode == "ss":
        ctx.set_query(qp, qtr, qss, S33, use_ss=True)
    elif mode == "global":
        ctx.set_query(qp, qtr, local=False, egq=0.3, egt=0.1)
    else:
        ctx.set_query(qp, qtr)
    if mode == "celloff":
        ctx.set_excluded_regions(*_regions(qp.shape[0] - 2))
        hits, paths = hhg.viterbi_search(ctx, db)
        ctx.set_excluded_regions()
        return hits, paths, None
    plan = hhg.Plan(ctx, db)
    plan.run()
    hits, paths = plan.fetch()
    return hits, paths, plan


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("Lq", LQS)
def test_strip_heights_12_and_16_agree_and_match_oracle(hhg, oracle, shard, ctxs, Lq, mode):
    from hhsuite_b200 import synth
    G = golden()
    q = synth.query_profile(Lq, seed=1 if Lq == 400 else 100 + Lq)
    res = {R: _run(hhg, ctx, db, q, mode, G["S33"]) for R, (ctx, db) in ctxs.items()}
    h16, p16, plan16 = res[16]
    h12, p12, plan12 = res[12]
    # every hit field (score bits, end and start cells, path length, Hit.score, score_ss) and every path byte
    assert np.array_equal(h16.view(np.uint8), h12.view(np.uint8))
    assert np.array_equal(p16, p12)
    # a sample against the oracle: the 1-column target, the longest ones, planted homologs and random targets
    rng = np.random.default_rng(Lq)
    sample = [0, 1, 2, 3, 6, 7] + rng.choice(np.arange(8, len(shard["L"])), 4, replace=False).tolist()
    okw = dict(local=mode != "global", egq=0.3 if mode == "global" else 0.0, egt=0.1 if mode == "global" else 0.0,
               shift=-0.03, ssw=0.11)
    if mode == "ss":
        okw.update(q_ss=q[2], S33=G["S33"])
    for t in sample:
        L = int(shard["L"][t])
        o, r = int(shard["p_off"][t]), int(shard["tr_off"][t])
        tp, ttr, tss = shard["p"][o:o + L + 2], shard["tr"][r:r + L + 1], shard["ss"][o:o + L + 2]
        kw = dict(okw, t_ss=tss) if mode == "ss" else dict(okw)
        if mode == "celloff":
            kw["celloff"] = _region_mask(Lq, L, *_regions(Lq))
        sc, i2, j2, bt = oracle.viterbi(q[0], q[1], tp, ttr, **kw)
        h = h12[t]
        assert bits(h["score"]) == bits(sc), (t, L, h["score"], sc)
        assert (h["i2"], h["j2"]) == (i2, j2), (t, L)
        n, i_s, j_s, st, mc = oracle.backtrace(bt, i2, j2)
        assert (h["nsteps"], h["matched_cols"], h["i1"], h["j1"]) == (n, mc, i_s[n], j_s[n]), (t, L)
        assert np.array_equal(p12[h["path_off"]:h["path_off"] + n], st[1:]), (t, L)
        if plan12 is not None and (L <= 300 or t < 2):
            for plan in (plan12, plan16):
                assert np.array_equal(plan.debug_bt(t)[1:, 1:], bt[1:, 1:]), (t, L)
    if plan12 is not None:
        plan12.close(); plan16.close()


def _targets(lens, seed):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(seed)
    qcols = synth.query_profile(37, seed=5)[4]
    return [synth.prepared_profile(int(L), rng, qcols if k % 4 == 0 else None, noise=0.3) for k, L in enumerate(lens)]


EDGES = {
    # jobs are length-sorted, longest first: the last job is the 1-column target alone
    "last_job_one_column": [300] * 31 + [250, 1],
    # every job as long as the longest: the last job's last column is the stream's last column
    "last_job_longest": [2000] * 40,
    "single_job": [1, 2000, 17, 640, 1],
    "single_target": [1],
}


@pytest.mark.parametrize("R", [16, 12, 8])
@pytest.mark.parametrize("edge", list(EDGES))
def test_ring_edges_match_oracle(hhg, oracle, R, edge):
    from hhsuite_b200 import synth
    q = synth.query_profile(37, seed=5)[:3]
    with env_ctx(hhg, HHG_STRIP_ROWS=R) as ctx:
        _check_against_oracle(hhg, ctx, oracle, q, _targets(EDGES[edge], 3))


@pytest.mark.parametrize("R", [16, 12, 8])
def test_ring_across_memory_waves(hhg, oracle, R):
    """A backtrace cap of ~20 KB splits the plan into one memory wave per job or so: every wave is its own launch
    whose last job ends in the middle of the operand stream."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(9)
    q = synth.query_profile(29, seed=6)[:3]
    lens = [1, 2, 700] + rng.integers(3, 400, 130).tolist()
    tg = _targets(lens, 4)
    with env_ctx(hhg, HHG_STRIP_ROWS=R, HHG_MAX_BT_GB=0.00002) as ctx:
        ctx.set_query(q[0], q[1])
        db = hhg.TargetDB.from_profiles(ctx, tg)
        hits, paths = hhg.viterbi_search(ctx, db)
        _check_hits_against_oracle(oracle, q, tg, hits, paths, [None] * len(tg), {})
        db.close()


@pytest.mark.parametrize("R", [16, 12, 8])
def test_back_to_back_plans_on_one_context(hhg, oracle, R):
    """Two different plans (different queries, different shards) alternate on one context: each run must give the
    same bytes as that plan's first run, which the oracle checks -- nothing may survive in the ring from the other
    plan's items or runs."""
    from hhsuite_b200 import synth
    qa = synth.query_profile(53, seed=8)[:3]
    qb = synth.query_profile(16, seed=9)[:3]
    ta = _targets([1999, 64, 1, 33, 400, 2, 700] * 6, 10)
    tb = _targets([1, 5, 1200, 80] * 11, 11)
    with env_ctx(hhg, HHG_STRIP_ROWS=R) as ctx:
        _check_against_oracle(hhg, ctx, oracle, qa, ta)
        _check_against_oracle(hhg, ctx, oracle, qb, tb)
        first = {}
        for it in range(3):
            for name, q, tg in (("a", qa, ta), ("b", qb, tb)):
                ctx.set_query(q[0], q[1])
                db = hhg.TargetDB.from_profiles(ctx, tg)
                plan = hhg.Plan(ctx, db)
                plan.run()
                hits, paths = plan.fetch()
                cur = (hits.view(np.uint8).copy(), paths.copy())
                if it == 0:
                    first[name] = cur
                else:
                    assert np.array_equal(cur[0], first[name][0]) and np.array_equal(cur[1], first[name][1]), (name, it)
                plan.close(); db.close()
        # the first run of each plan against the oracle (score bits and end cells)
        for name, q, tg in (("a", qa, ta), ("b", qb, tb)):
            h = first[name][0].view(hhg.capi.HIT_DTYPE)
            for k, (tp, ttr, _) in enumerate(tg):
                sc, i2, j2, _bt = oracle.viterbi(q[0], q[1], tp, ttr)
                assert bits(h[k]["score"]) == bits(sc) and (h[k]["i2"], h[k]["j2"]) == (i2, j2), (name, k)
