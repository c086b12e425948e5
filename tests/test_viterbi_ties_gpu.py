"""k_viterbi / k_backtrace on inputs where ties are certain (tests/vit_cases.py): dyadic profiles on which many DP
candidates and many end cells are bit-equal, plus degenerate values.  Every result must be the oracle's bit for bit
(the oracle is pinned to the compiled reference on the same families by tests/test_oracle_vs_ref.py): the five-way
MM maximum, the gap-state flags, the row-order rule of the running maximum inside a strip, the strip merge, the
padded columns of a job and the global-mode end cells all decide something here."""
import numpy as np
import pytest

from tests import vit_cases as vc
from tests.test_kernel_variants_gpu import CONFIGS, env_ctx
from tests.test_viterbi_gpu import _check_against_oracle
from tests.util import bits, golden, rasterize_exclusion

pytestmark = pytest.mark.gpu

CFG_IDS = [",".join(f"{k[4:]}={v}" for k, v in c.items()) for c in CONFIGS]


def _oracle_kw(par):
    return dict(local=par.get("local", True), egq=par.get("egq", 0.0), egt=par.get("egt", 0.0),
                shift=par.get("shift", -0.03))


def _check_hits_against_oracle(oracle, q, tg, hits, paths, masks, par):
    """Score bits, end cells, start cells, nsteps, matched_cols and the state string of every hit (no bt access)."""
    for k, (tp, ttr, tss) in enumerate(tg):
        sc, i2, j2, bt = oracle.viterbi(q[0], q[1], tp, ttr, celloff=masks[k], **_oracle_kw(par))
        h = hits[k]
        where = (k, tp.shape[0] - 2)
        assert bits(h["score"]) == bits(sc), (where, h["score"], sc)
        assert (h["i2"], h["j2"]) == (i2, j2), where
        n, i_s, j_s, st, mc = oracle.backtrace(bt, i2, j2)
        assert (h["nsteps"], h["matched_cols"], h["i1"], h["j1"]) == (n, mc, i_s[n], j_s[n]), where
        assert np.array_equal(paths[h["path_off"]:h["path_off"] + n], st[1:]), where


def _regions_through_ties(q, tg, par):
    """-excl / -template_excl ranges through the first maximal row and column of a mid-length target."""
    Lq = q[0].shape[0] - 2
    try:
        i, j = vc.witness(q, tg[4], **par)["first"]
    except AssertionError:
        i, j = (Lq + 1) // 2, 16
    i, j = max(i, 1), max(j, 1)
    return [(i, i), (min(i + 5, Lq), min(i + 6, Lq))], [(j, j + 1), (40, 41)]


def _region_mask(Lq, Lt, q_ranges, t_ranges):
    m = np.zeros((Lq + 1, Lt + 1), np.uint8)
    for a, b in q_ranges:
        m[a:min(b, Lq) + 1, 1:] = 1
    for a, b in t_ranges:
        if a <= Lt:
            m[1:, a:min(b, Lt) + 1] = 1
    return m


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_tie_families_match_oracle(hhg, oracle, cfg):
    """Every family, every strip height / group size: plain, SS (local families) and global mode, with every
    backtrace byte compared."""
    G = golden()
    with env_ctx(hhg, **cfg) as ctx:
        for name, q, tg, par in vc.all_cases():
            _check_against_oracle(hhg, ctx, oracle, q, tg, **par)
            if par.get("local", True):
                _check_against_oracle(hhg, ctx, oracle, q, tg, S33=G["S33"], use_ss=True, **par)
                _check_against_oracle(hhg, ctx, oracle, vc.with_mixed_ss(q), [vc.with_mixed_ss(t) for t in tg],
                                      S33=G["S33"], use_ss=True, **par)


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_tie_families_excluded_regions_and_alternative_alignment(hhg, oracle, cfg):
    """Cell-off instantiations: excluded query rows / template columns through the tied maxima, then an
    alternative-alignment pass that also excludes each target's first path."""
    with env_ctx(hhg, **cfg) as ctx:
        for name, q, tg, par in vc.tie_cases() + vc.degen_cases():
            if not par.get("local", True):
                continue
            Lq = q[0].shape[0] - 2
            ctx.set_query(q[0], q[1], **par)
            db = hhg.TargetDB.from_profiles(ctx, tg)
            h0, p0 = hhg.viterbi_search(ctx, db)
            excl, path_masks = [], []
            for k, (tp, ttr, tss) in enumerate(tg):
                gi, gj, gs = hhg.expand_path(h0[k], p0)
                n = int(h0[k]["nsteps"])
                excl.append((gi[1:n], gj[1:n]) if n > 1 else None)
                path_masks.append(rasterize_exclusion(Lq, tp.shape[0] - 2, gi, gj, n))
            h1, p1 = hhg.viterbi_search(ctx, db, exclusions=excl)
            _check_hits_against_oracle(oracle, q, tg, h1, p1, path_masks, par)
            qr, tr = _regions_through_ties(q, tg, par)
            ctx.set_excluded_regions(qr, tr)
            region_masks = [_region_mask(Lq, t[0].shape[0] - 2, qr, tr) for t in tg]
            h2, p2 = hhg.viterbi_search(ctx, db)
            _check_hits_against_oracle(oracle, q, tg, h2, p2, region_masks, par)
            h3, p3 = hhg.viterbi_search(ctx, db, exclusions=excl)
            _check_hits_against_oracle(oracle, q, tg, h3, p3, [a | b for a, b in zip(region_masks, path_masks)], par)
            ctx.set_excluded_regions()
            db.close()


def test_tie_families_hit_score_vs_compiled_reference(hhg, gpu_ctx, refshim):
    """Hit.score and Hit.score_ss (Viterbi::ScoreForBacktrace over the tied paths) against the compiled reference."""
    S33 = refshim.S33()
    for name, q, tg, par in vc.all_cases():
        local = par.get("local", True)
        refshim.set_query(q[0], q[1], q[0][1:-1].mean(axis=0), q[2])
        for use_ss in ((False, True) if local else (False,)):
            gpu_ctx.set_query(q[0], q[1], q[2], S33, use_ss=use_ss, **par)
            db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
            hits, _ = hhg.viterbi_search(gpu_ctx, db)
            step = refshim.V if local else 1
            for b in range(0, len(tg), step):
                res = refshim.viterbi(tg[b:b + step], use_ss=use_ss, **par)
                for k in range(len(res)):
                    h = hits[b + k]
                    assert bits(h["score"]) == bits(res[k][0]), (name, b + k)
                    hs, hss = refshim.hit_score(k)
                    assert bits(h["hit_score"]) == bits(hs), (name, use_ss, b + k, h["hit_score"], hs)
                    assert bits(h["score_ss"]) == bits(hss), (name, use_ss, b + k)
            db.close()


def _batch_inputs():
    queries = [vc.const(1, "q"), vc.tandem(17, "q", k=5), vc.gap(13, "q"), vc.tandem(49, "q", k=3, reverse=True),
               vc.const(4, "q", level=1), vc.degen(16, "q", "zero"), vc.tandem(2, "q", k=7)]
    tg = (vc._targets(vc.const) + vc._targets(vc.tandem, k=5) + vc._targets(vc.gap) +
          vc._targets(vc.tandem, k=3, reverse=True) + [vc.degen(L, "t", "zero") for L in vc.LT])
    return queries, tg


@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[3], dict(HHG_STRIP_ROWS=8, HHG_MAX_BT_GB=0.00002)],
                         ids=["R16", "R12", "R8-waves"])
def test_query_batch_on_tie_families(hhg, oracle, cfg):
    """Several tie-family queries (Lq = 1 .. 49) in one hhg_query_set_batch plan, in local, SS, global and cell-off
    (excluded regions) mode; every request checked directly against the oracle.  R8-waves caps the backtrace memory
    so the plan runs in several memory waves."""
    G = golden()
    queries, tg = _batch_inputs()
    rng = np.random.default_rng(7)
    req_q = np.repeat(np.arange(len(queries), dtype=np.int32), len(tg))
    ids = np.tile(np.arange(len(tg), dtype=np.int32), len(queries))
    perm = rng.permutation(len(ids))
    req_q, ids = req_q[perm], ids[perm]
    variants = [dict(shift=-0.5), dict(shift=-0.5, use_ss=True), dict(local=False, shift=-0.5, egq=0.5, egt=0.25),
                dict(shift=-0.5, regions=([(1, 1), (9, 12)], [(2, 3), (31, 33)]))]
    with env_ctx(hhg, **cfg) as ctx:
        db = hhg.TargetDB.from_profiles(ctx, tg)
        for v in variants:
            par = dict(v)
            regions = par.pop("regions", None)
            use_ss = par.pop("use_ss", False)
            hhg.capi.query_set_batch(ctx, queries, S33=G["S33"], use_ss=use_ss, **par)
            if regions:
                ctx.set_excluded_regions(*regions)
            hb, pb_ = hhg.capi.viterbi_search_batch(ctx, db, req_q, ids)
            if regions:
                ctx.set_excluded_regions()
            for r in range(len(ids)):
                q = queries[req_q[r]]
                tp, ttr, tss = tg[ids[r]]
                Lq, Lt = q[0].shape[0] - 2, tp.shape[0] - 2
                okw = _oracle_kw(par)
                if use_ss:
                    okw.update(q_ss=q[2], t_ss=tss, S33=G["S33"])
                mask = _region_mask(Lq, Lt, *regions) if regions else None
                sc, i2, j2, bt = oracle.viterbi(q[0], q[1], tp, ttr, celloff=mask, **okw)
                h = hb[r]
                where = (v, int(req_q[r]), int(ids[r]))
                assert bits(h["score"]) == bits(sc) and (h["i2"], h["j2"]) == (i2, j2), where
                n, i_s, j_s, st, mc = oracle.backtrace(bt, i2, j2)
                assert (h["nsteps"], h["matched_cols"], h["i1"], h["j1"]) == (n, mc, i_s[n], j_s[n]), where
                assert np.array_equal(pb_[h["path_off"]:h["path_off"] + n], st[1:]), where
        db.close()


def test_topk_on_negative_global_scores(hhg, gpu_ctx):
    """plan.topk by score and by hit_score on a shard of tie-family targets aligned in global mode: every score is
    negative (a range of the order-preserving float key no other test reaches) and many records share a score, so
    the global id decides."""
    q = vc.gap(17, "q")
    tg = [vc.const(L, "t", level=1) for L in vc.LT] + [vc.gap(L, "t") for L in vc.LT] + \
         [vc.tandem(L, "t", k=5) for L in vc.LT]
    tg = tg * 12                                                      # 360 targets, every one 12 times
    gpu_ctx.set_query(q[0], q[1], local=False, shift=-4.0, egq=0.5, egt=0.25)
    db = hhg.TargetDB.from_profiles(gpu_ctx, tg)
    plan = hhg.Plan(gpu_ctx, db)
    plan.run()
    hits, _ = plan.fetch(want_paths=False)
    assert np.all(hits["score"] < 0)
    assert len(np.unique(hits["score"])) < len(tg) // 4
    n = len(tg)
    gids = (np.arange(n, dtype=np.int32) * 7919) % 100003           # ids not in target order
    for field, flag in (("score", False), ("hit_score", True)):
        for K in (1, 12, 37, 200, n):
            rec = plan.topk(K, by_hit_score=flag, global_ids=gids)
            exp = np.lexsort((gids, -hits[field].astype(np.float64)))[:K]
            assert np.array_equal(rec["target"], gids[exp]), (field, K)
            assert np.array_equal(rec["hit"][field].view(np.uint32), hits[field][exp].view(np.uint32)), (field, K)
        rec = plan.topk(50, by_hit_score=flag, id_base=3)
        assert np.array_equal(rec["target"], 3 + np.lexsort((np.arange(n), -hits[field].astype(np.float64)))[:50])
    plan.close(); db.close()
