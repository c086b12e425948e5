"""Query-batch Viterbi searches (hhg_query_set_batch + hhg_viterbi_search_batch) at database scale and at the length
limits.  Every request is checked against the C oracle: score bits, end and start cells, nsteps, matched_cols and the
path states; on single-wave plans the backtrace bytes of a sample of requests too.  Hit.score and Hit.score_ss are
checked against the compiled reference where it takes the lengths (<= 4094), else against single-query calls.

The batches come from tests/batch_cases.py: a "scan" batch whose automatic strip height is 16 and a "survivors" batch
whose automatic strip height is 8, 20+ queries of lengths at the padding and strip edges, 0 .. 430 requests each."""
import numpy as np
import pytest

from tests import batch_cases as bc
from tests.test_kernel_variants_gpu import env_ctx
from tests.util import bits, golden

pytestmark = pytest.mark.gpu

FIELDS = ("i2", "j2", "i1", "j1", "nsteps", "matched_cols")
PLAIN = dict()
REGIONS = ([(3, 5), (60, 70), (1200, 1210)], [(2, 2), (31, 33), (500, 520)])   # some rows lie past short queries


@pytest.fixture(scope="module")
def batches():
    return {k: bc.make_batch(k) for k in ("scan", "survivors")}


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ helpers
def _oracle_kw(mode):
    return dict(local=mode.get("local", True), egq=mode.get("egq", 0.0), egt=mode.get("egt", 0.0),
                shift=mode.get("shift", -0.03))


def _expect(oracle, q, t, mode, keep_bt=False):
    """The oracle's result for one (query, target) pair; q = (p, tr, ss), t = (p, tr, ss)."""
    okw = _oracle_kw(mode)
    if mode.get("use_ss"):
        okw.update(q_ss=q[2], t_ss=t[2], S33=golden()["S33"])
    Lq, Lt = q[0].shape[0] - 2, t[0].shape[0] - 2
    mask = bc.region_mask(Lq, Lt, *mode["regions"]) if mode.get("regions") else None
    sc, i2, j2, bt = oracle.viterbi(q[0], q[1], t[0], t[1], celloff=mask, **okw)
    n, i_s, j_s, st, mc = oracle.backtrace(bt, i2, j2)
    return dict(score=np.float32(sc), i2=i2, j2=j2, i1=int(i_s[n]), j1=int(j_s[n]), nsteps=n, matched_cols=mc,
                states=st[1:].copy(), bt=bt if keep_bt else None)


_CACHE = {}


def _expected(oracle, b, mode, name, targets=None, keep=()):
    """Oracle results of every request of batch b in `mode` (cached per batch and mode name; duplicate pairs are
    computed once).  targets: the profiles the oracle aligns with (default b's); keep: requests whose bt is kept."""
    key = (b["kind"], name)
    if key not in _CACHE:
        tg = b["targets"] if targets is None else targets
        memo, out = {}, []
        for r, (q, t) in enumerate(zip(b["req_q"].tolist(), b["ids"].tolist())):
            if (q, t) not in memo or r in keep:
                qq = b["queries"][q]
                memo[(q, t)] = _expect(oracle, (qq["p"], qq["tr"], qq["ss"]), tg[t], mode, keep_bt=r in keep)
            out.append(memo[(q, t)])
        _CACHE[key] = out
    return _CACHE[key]


def _check(hits, paths, exp, req_q, ids, where):
    """Every request against its expectation; a failure names the request, its query and target and the field."""
    assert len(hits) == len(exp)
    for r, e in enumerate(exp):
        h = hits[r]
        tag = (where, f"request {r}", f"query {int(req_q[r])}", f"target {int(ids[r])}")
        assert bits(h["score"]) == bits(e["score"]), (tag, "score", float(h["score"]), float(e["score"]))
        for f in FIELDS:
            assert int(h[f]) == e[f], (tag, f, int(h[f]), e[f])
        o = int(h["path_off"])
        assert np.array_equal(paths[o:o + e["nsteps"]], e["states"]), (tag, "path states")


def _sample(b, k=2):
    """The first k requests of every query (for backtrace-byte checks)."""
    out = []
    for q in range(len(b["q_lens"])):
        out += np.nonzero(b["req_q"] == q)[0][:k].tolist()
    return out


def _check_bt(hhg, ctx, b, exp, sample, where):
    """Backtrace bytes of the sampled requests of the context's last plan (single wave)."""
    import ctypes as C
    L = ctx.L
    plan = L.hhg_ctx_last_plan(ctx.h)
    for r in sample:
        Lq, Lt = int(b["q_lens"][b["req_q"][r]]), int(b["t_lens"][b["ids"][r]])
        bt = np.zeros((Lq + 1, Lt + 1), np.uint8)
        hhg.capi._ck(L.hhg_plan_debug_bt(ctx.h, plan, r, bt.ctypes.data_as(C.POINTER(C.c_uint8))))
        ref = exp[r]["bt"]
        assert np.array_equal(bt[1:, 1:], ref[1:, 1:]), (where, f"request {r}", "bt bytes",
                                                        int((bt[1:, 1:] != ref[1:, 1:]).sum()))


def _qset(hhg, ctx, b, queries=None, q_pav=None, **mode):
    qs = b["queries"] if queries is None else queries
    par = {k: v for k, v in mode.items() if k in ("local", "egq", "egt", "shift")}
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"], q["ss"]) for q in qs], S33=golden()["S33"], q_pav=q_pav,
                             use_ss=mode.get("use_ss", False), **par)


def _search(hhg, ctx, db, b, mode, **kw):
    if mode.get("regions"):
        ctx.set_excluded_regions(*mode["regions"])
    try:
        return hhg.capi.viterbi_search_batch(ctx, db, b["req_q"], b["ids"], **kw)
    finally:
        if mode.get("regions"):
            ctx.set_excluded_regions()


def _plan_stats(ctx):
    return ctx.L.hhg_plan_padded_cells(ctx.L.hhg_ctx_last_plan(ctx.h))


# ------------------------------------------------------------------------------------------------ 1. strip heights
@pytest.mark.parametrize("kind", ["scan", "survivors"])
def test_mixed_batch_every_strip_height(hhg, oracle, batches, sm_count, kind):
    """The batch with R chosen by the plan and forced to 8, 12 and 16; which R ran is read off the padded cells."""
    b = batches[kind]
    sample = _sample(b)
    exp = _expected(oracle, b, PLAIN, "plain", keep=set(sample))
    lq, lt = bc.request_lengths(b)
    auto = bc.strip_rows(b["q_lens"], b["req_q"], sm_count)
    assert auto == (16 if kind == "scan" else 8)
    for forced in (None, 8, 12, 16):
        env = {} if forced is None else dict(HHG_STRIP_ROWS=forced)
        with env_ctx(hhg, **env) as ctx:
            db = hhg.TargetDB.from_profiles(ctx, b["targets"])
            _qset(hhg, ctx, b)
            hits, paths = _search(hhg, ctx, db, b, PLAIN)
            R = forced or auto
            assert _plan_stats(ctx) == bc.padded_cells(bc.plan_jobs(b["q_lens"], b["req_q"], lt, R), R), (kind, R)
            _check(hits, paths, exp, b["req_q"], b["ids"], (kind, R))
            _check_bt(hhg, ctx, b, exp, sample, (kind, R))
            db.close()


# ------------------------------------------------------------------------------------------------ 2. modes
MODES = dict(glob=dict(local=False, egq=0.3, egt=0.1), ss=dict(use_ss=True), regions=dict(regions=REGIONS),
             ss_regions=dict(use_ss=True, regions=REGIONS))


@pytest.mark.parametrize("name", list(MODES))
def test_survivors_batch_modes(hhg, oracle, batches, name):
    """Global mode (egq, egt != 0), the SS term, excluded regions (some query ranges past the end of the short
    queries) and both, at the automatic strip height and at R = 16."""
    b = batches["survivors"]
    mode = MODES[name]
    exp = _expected(oracle, b, mode, name)
    for env in ({}, dict(HHG_STRIP_ROWS=16)):
        with env_ctx(hhg, **env) as ctx:
            db = hhg.TargetDB.from_profiles(ctx, b["targets"])
            _qset(hhg, ctx, b, **mode)
            hits, paths = _search(hhg, ctx, db, b, mode)
            _check(hits, paths, exp, b["req_q"], b["ids"], (name, env))
            db.close()


@pytest.mark.parametrize("use_ss", [False, True])
def test_survivors_batch_hit_score_vs_compiled_reference(hhg, gpu_ctx, batches, refshim, use_ss):
    """Hit.score and Hit.score_ss of every request against Viterbi::ScoreForBacktrace of the compiled reference."""
    b = batches["survivors"]
    db = hhg.TargetDB.from_profiles(gpu_ctx, b["targets"])
    _qset(hhg, gpu_ctx, b, use_ss=use_ss)
    hits, _ = _search(hhg, gpu_ctx, db, b, PLAIN)
    for q, qq in enumerate(b["queries"]):
        reqs = np.nonzero(b["req_q"] == q)[0]
        if not len(reqs):
            continue
        refshim.set_query(qq["p"], qq["tr"], qq["pav"], qq["ss"])
        for c in range(0, len(reqs), refshim.V):
            chunk = reqs[c:c + refshim.V]
            res = refshim.viterbi([b["targets"][b["ids"][r]] for r in chunk], use_ss=use_ss)
            for k, r in enumerate(chunk):
                h = hits[r]
                assert bits(h["score"]) == bits(res[k][0]), (f"request {r}", "score")
                hs, hss = refshim.hit_score(k)
                assert bits(h["hit_score"]) == bits(hs), (f"request {r}", "hit_score", float(h["hit_score"]), hs)
                assert bits(h["score_ss"]) == bits(hss), (f"request {r}", "score_ss")
    db.close()


# ------------------------------------------------------------------------------------------------ 3. raw shard
def _raw_shard(hhg, ctx, b, seed):
    """b's targets as a raw shard (emissions before the null model + pav); returns (db, raw targets, t_pav)."""
    rng = np.random.default_rng(seed)
    raw, pav = zip(*[bc.raw_profile(t, rng) for t in b["targets"]])
    L = b["t_lens"]
    p_off = np.concatenate([[0], np.cumsum(L.astype(np.int64) + 2)[:-1]])
    tr_off = np.concatenate([[0], np.cumsum(L.astype(np.int64) + 1)[:-1]])
    db = hhg.TargetDB(ctx, L, np.concatenate([r[0] for r in raw]), np.concatenate([r[1] for r in raw]), p_off, tr_off,
                      np.concatenate([r[2] for r in raw]), pav=np.stack(pav))
    return db, list(raw), np.stack(pav)


def _expected_raw(oracle, b, raw, t_pav, q_pav, pb, cs, mode, queries=None):
    """Oracle results of every request on the numpy-null-modelled target of its query (not cached)."""
    qs = b["queries"] if queries is None else queries
    memo, out = {}, []
    for q, t in zip(b["req_q"].tolist(), b["ids"].tolist()):
        if (q, t) not in memo:
            tp = bc.null_model(raw[t][0], t_pav[t], q_pav[q], pb, cs)
            qq = qs[q]
            memo[(q, t)] = _expect(oracle, (qq["p"], qq["tr"], qq["ss"]), (tp, raw[t][1], raw[t][2]), mode)
        out.append(memo[(q, t)])
    return out


def _survivors_subset(b, max_lq):
    """b restricted to the requests of queries with Lq <= max_lq (same queries, same shard)."""
    keep = b["q_lens"][b["req_q"]] <= max_lq
    return dict(b, kind=b["kind"] + f"<={max_lq}", req_q=b["req_q"][keep], ids=b["ids"][keep])


@pytest.mark.parametrize("columnscore", [0, 1, 2, 3])
def test_raw_shard_fused_null_model(hhg, oracle, gpu_ctx, batches, columnscore):
    """The null model applied per (query, target) inside k_interleave_cols and k_backtrace, with a distinct q_pav per
    query: plain, and with SS and excluded regions on top."""
    b = _survivors_subset(batches["survivors"], 400)
    rng = np.random.default_rng(40 + columnscore)
    db, raw, t_pav = _raw_shard(hhg, gpu_ctx, b, 41)
    q_pav = np.stack([q["pav"] for q in b["queries"]])
    pb = rng.dirichlet(np.ones(20) * 5).astype(np.float32)
    for name, mode in (("plain", PLAIN), ("ss_regions", MODES["ss_regions"])):
        _qset(hhg, gpu_ctx, b, q_pav=q_pav, **mode)
        hits, paths = _search(hhg, gpu_ctx, db, b, mode, columnscore=columnscore, pb=pb)
        exp = _expected_raw(oracle, b, raw, t_pav, q_pav, pb, columnscore, mode)
        _check(hits, paths, exp, b["req_q"], b["ids"], (f"cs{columnscore}", name))
    db.close()


# ------------------------------------------------------------------------------------------------ 4. memory waves
def test_scan_batch_memory_waves(hhg, oracle, batches, sm_count):
    """HHG_MAX_BT_GB cuts the scan batch into >= 5 memory waves, with a wave boundary inside one query's jobs and a
    job larger than the budget; the launches show the waves ran, and the results are the single-wave run's bytes."""
    b = batches["scan"]
    exp = _expected(oracle, b, PLAIN, "plain")
    lq, lt = bc.request_lengths(b)
    R = bc.strip_rows(b["q_lens"], b["req_q"], sm_count)
    jobs = bc.plan_jobs(b["q_lens"], b["req_q"], lt, R)
    waves = bc.wave_sizes(jobs, R, bc.bt_budget(bc.SCAN_WAVE_GB))
    assert len(waves) >= 5
    runs = []
    for env in ({}, dict(HHG_MAX_BT_GB=bc.SCAN_WAVE_GB)):
        with env_ctx(hhg, **env) as ctx:
            db = hhg.TargetDB.from_profiles(ctx, b["targets"])
            _qset(hhg, ctx, b)
            n0 = ctx.launches
            hits, paths = _search(hhg, ctx, db, b, PLAIN)
            # operand stream + (forward + backtrace) per wave + path gather
            assert ctx.launches - n0 == 2 + 2 * (len(waves) if env else 1), (env, ctx.launches - n0, waves)
            _check(hits, paths, exp, b["req_q"], b["ids"], ("waves", env))
            runs.append((hits.tobytes(), paths.tobytes()))
            db.close()
    assert runs[0] == runs[1]


# ------------------------------------------------------------------------------------------------ 5. one context
def test_long_lived_context_sequence(hhg, oracle, batches):
    """A seeded sequence of calls on one context and one raw shard: batch calls that change only pb (columnscore 0),
    a new query batch of the same geometry, columnscore switches, SS and regions toggled, a single-query search after
    hhg_db_apply_null_model and a Plan run.  Every result must be the oracle's for the state the call was made in."""
    b = _survivors_subset(batches["survivors"], 211)
    rng = np.random.default_rng(77)
    other = bc.queries(b["q_lens"], 9001)              # same lengths, other profiles and pav
    pbs = [rng.dirichlet(np.ones(20) * 5).astype(np.float32) for _ in range(2)]
    with env_ctx(hhg) as ctx:
        db, raw, t_pav = _raw_shard(hhg, ctx, b, 78)
        sets = {"A": b["queries"], "B": other}
        steps = [("A", 0, 0, PLAIN), ("A", 0, 1, PLAIN), ("A", 0, 0, PLAIN), ("B", 1, 0, PLAIN), ("B", 3, 0, PLAIN),
                 ("B", 0, 1, MODES["ss_regions"]), ("B", 0, 0, MODES["ss_regions"]), ("B", 2, 1, PLAIN),
                 ("single",), ("plan",), ("A", 0, 1, MODES["regions"]), ("A", 0, 0, MODES["regions"]),
                 ("A", 1, 1, MODES["ss"])]
        current = None
        for n, st in enumerate(steps):
            if st[0] in ("single", "plan"):
                q0 = sets["A"][16]                     # Lq = 211
                ctx.set_query(q0["p"], q0["tr"])
                current = None
                db.apply_null_model(q0["pav"], pbs[1], 0)
                ids = b["ids"][:40]
                if st[0] == "single":
                    hits, paths = hhg.viterbi_search(ctx, db, ids=ids)
                else:
                    plan = hhg.Plan(ctx, db, ids)
                    plan.run()
                    hits, paths = plan.fetch()
                    plan.close()
                one = dict(b, req_q=np.zeros(len(ids), np.int32), ids=ids)
                exp = _expected_raw(oracle, one, raw, t_pav, q0["pav"][None, :], pbs[1], 0, PLAIN, queries=[q0])
                _check(hits, paths, exp, one["req_q"], ids, (n, st[0]))
                continue
            name, cs, k, mode = st
            qs = sets[name]
            q_pav = np.stack([q["pav"] for q in qs])
            if current != (name, mode.get("use_ss", False)):
                _qset(hhg, ctx, b, queries=qs, q_pav=q_pav, **mode)
                current = (name, mode.get("use_ss", False))
            hits, paths = _search(hhg, ctx, db, b, mode, columnscore=cs, pb=pbs[k])
            exp = _expected_raw(oracle, b, raw, t_pav, q_pav, pbs[k], cs, mode, queries=qs)
            _check(hits, paths, exp, b["req_q"], b["ids"], (f"step {n}", name, f"columnscore {cs}", f"pb {k}"))
        db.close()


# ------------------------------------------------------------------------------------------------ 6. length limits
GLOBAL_FREE_ENDS = dict(local=False, egq=0.0, egt=0.0)   # no end-gap costs: the planted diagonal's end stays the best
def _pair(oracle, q, t, mode, keep_bt=False):
    return _expect(oracle, (q["p"], q["tr"], q["ss"]), t, mode, keep_bt=keep_bt)


def _single_batch(queries, targets, req_q, ids):
    q_lens = np.array([q["p"].shape[0] - 2 for q in queries], np.int32)
    t_lens = np.array([t[0].shape[0] - 2 for t in targets], np.int32)
    return dict(kind="limits", queries=queries, targets=targets, req_q=np.asarray(req_q, np.int32),
                ids=np.asarray(ids, np.int32), q_lens=q_lens, t_lens=t_lens)


def _single_query_hit_scores(hhg, q, targets, ids, mode):
    """Hit.score / Hit.score_ss of single-query calls on a fresh context (no reference at these lengths)."""
    with env_ctx(hhg) as ctx:
        db = hhg.TargetDB.from_profiles(ctx, targets)
        ctx.set_query(q["p"], q["tr"], **{k: v for k, v in mode.items() if k in ("local", "egq", "egt", "shift")})
        hits, _ = hhg.viterbi_search(ctx, db, ids=np.asarray(ids, np.int32), want_paths=False)
        db.close()
    return hits


@pytest.fixture(scope="module")
def longest_query():
    rng = np.random.default_rng(32767)
    q = bc.queries([bc.MAX_LEN], 5)[0]
    short = [synth_target(L, rng) for L in (1, 2, 33)]
    planted = bc.plant_tail(synth_target(200, rng), q["mix"][-200:])    # best cell at (32767, 200)
    return q, short + [planted]


def synth_target(L, rng, base=None):
    from hhsuite_b200 import synth
    return synth.prepared_profile(int(L), rng, base, noise=0.3)


@pytest.mark.parametrize("mode_name", ["local", "glob"])
def test_longest_query_every_strip_height(hhg, oracle, longest_query, mode_name):
    """Lq = 32 767 against 1..200-column targets: 4 096 strips at R = 8 (the 12-bit strip field of the hand-off tag is
    full), 2 731 at R = 12, 2 048 at R = 16; the planted target puts the best cell in row 32 767."""
    q, tg = longest_query
    mode = PLAIN if mode_name == "local" else GLOBAL_FREE_ENDS
    b = _single_batch([q], tg, [0, 0, 0, 0, 0], [0, 1, 2, 3, 3])
    exp = [_pair(oracle, q, tg[t], mode, keep_bt=(mode_name == "local" and t == 3)) for t in b["ids"]]
    assert exp[3]["i2"] == bc.MAX_LEN and exp[3]["j2"] == 200
    single = _single_query_hit_scores(hhg, q, tg, b["ids"], mode)
    for R in (8, 12, 16):
        with env_ctx(hhg, HHG_STRIP_ROWS=R) as ctx:
            db = hhg.TargetDB.from_profiles(ctx, tg)
            _qset(hhg, ctx, b, **mode)
            hits, paths = _search(hhg, ctx, db, b, mode)
            _check(hits, paths, exp, b["req_q"], b["ids"], (mode_name, R))
            for f in ("hit_score", "score_ss"):
                assert np.array_equal(bits(hits[f]), bits(single[f])), (mode_name, R, f)
            if mode_name == "local" and R == 8:
                _check_bt(hhg, ctx, b, exp, [3], (mode_name, R))
            db.close()


@pytest.mark.parametrize("mode_name", ["local", "glob"])
def test_longest_targets_and_6000_pair(hhg, oracle, mode_name):
    """Targets of 32 767 columns against short queries (the planted one puts the best cell in column 32 767) and one
    6 000 x 6 000 pair, in one batch."""
    rng = np.random.default_rng(6000)
    qs = bc.queries([1, 17, 300, 6000], 61)
    t_long = synth_target(bc.MAX_LEN, rng)
    tg = [t_long, bc.plant_tail(t_long, qs[2]["mix"]), synth_target(6000, rng, qs[3]["mix"])]
    mode = PLAIN if mode_name == "local" else GLOBAL_FREE_ENDS
    b = _single_batch(qs, tg, [0, 1, 2, 2, 3], [0, 0, 1, 0, 2])
    exp = [_pair(oracle, qs[q], tg[t], mode) for q, t in zip(b["req_q"], b["ids"])]
    assert exp[2]["j2"] == bc.MAX_LEN
    with env_ctx(hhg) as ctx:
        db = hhg.TargetDB.from_profiles(ctx, tg)
        _qset(hhg, ctx, b, **mode)
        hits, paths = _search(hhg, ctx, db, b, mode)
        _check(hits, paths, exp, b["req_q"], b["ids"], mode_name)
        db.close()
    for q in range(len(qs)):
        m = np.nonzero(b["req_q"] == q)[0]
        single = _single_query_hit_scores(hhg, qs[q], tg, b["ids"][m], mode)
        for f in ("hit_score", "score_ss"):
            assert np.array_equal(bits(hits[f][m]), bits(single[f])), (mode_name, q, f)


def test_longest_query_grouped_with_short_ones(hhg, oracle, longest_query):
    """Lq = 32 767 in one batch with Lq = 1, 8, 9 and 17 at R = 8: one group of jobs mixes 1-strip and 4 096-strip
    jobs."""
    q, tg = longest_query
    shorts = bc.queries([1, 8, 9, 17], 71)
    qs = [shorts[0], q, shorts[1], shorts[2], shorts[3]]
    req_q, ids = [], []
    for k in range(len(qs)):
        for t in range(len(tg)):
            req_q.append(k); ids.append(t)
    b = _single_batch(qs, tg, req_q, ids)
    exp = [_pair(oracle, qs[k], tg[t], PLAIN) for k, t in zip(req_q, ids)]
    with env_ctx(hhg, HHG_STRIP_ROWS=8, HHG_GROUP_JOBS=16) as ctx:
        db = hhg.TargetDB.from_profiles(ctx, tg)
        _qset(hhg, ctx, b)
        hits, paths = _search(hhg, ctx, db, b, PLAIN)
        _check(hits, paths, exp, b["req_q"], b["ids"], "grouped")
        db.close()


def test_plan_too_large_is_refused_and_the_context_recovers(hhg, oracle, longest_query):
    """65 600 requests of Lq = 32 767 need more than 2^31 - 1 path bytes: refused with "plan too large" before any
    launch, again when repeated (the failed plan must not be reused), and the context still searches correctly."""
    q, tg = longest_query
    n = 65600
    assert n * (bc.MAX_LEN + 1 + 2) > bc.PATH_LIMIT
    b = _single_batch([q], tg, np.zeros(n, np.int32), np.zeros(n, np.int32))
    with env_ctx(hhg) as ctx:
        db = hhg.TargetDB.from_profiles(ctx, tg)
        _qset(hhg, ctx, b)
        n0 = ctx.launches
        for _ in range(2):
            with pytest.raises(hhg.HhgError, match="plan too large"):
                hhg.capi.viterbi_search_batch(ctx, db, b["req_q"], b["ids"], want_paths=False)
        assert ctx.launches == n0
        with pytest.raises(hhg.HhgError, match="last build failed"):
            hhg.capi._ck(ctx.L.hhg_plan_run(ctx.h, ctx.L.hhg_ctx_last_plan(ctx.h)))
        small = _single_batch([q], tg, [0, 0], [3, 1])
        hits, paths = _search(hhg, ctx, db, small, PLAIN)
        _check(hits, paths, [_pair(oracle, q, tg[t], PLAIN) for t in (3, 1)], small["req_q"], small["ids"], "after")
        db.close()
