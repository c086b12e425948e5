"""Databases larger than device memory: the host-resident store (hhg_dbstore_*), the staged shard over it
(hhg_db_create_staged / hhg_db_stage, kernel k_stage_gather) and pipeline.search_staged / search_batch_staged.  A staged
shard must be indistinguishable from a resident raw shard of the same targets: every comparison here is `==` on bytes or
on the bits of a field -- records, lengths and pav after the gather; hits, paths and posteriors of every search entry
point; survivors and Hit fields of the whole pipeline -- plus eviction, plan invalidation, refusals and launch counts."""
import dataclasses

import numpy as np
import pytest

from hhsuite_b200 import synth
from tests import batch_cases as bc
from tests.test_batch_realign_gpu import _raw_db, _vit
from tests.test_hhm_db_gpu import _pack, _pp
from tests.util import bits, golden

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ helpers
def _random_store(hhg, ctx, lens, seed, has_ss):
    """A store of random records (any bit pattern that is a finite float) with the given lengths."""
    rng = np.random.default_rng(seed)
    L = np.asarray(lens, np.int32)
    cols = np.zeros(int(L.sum()), hhg.capi.COLREC_DTYPE)
    cols["p"] = rng.random((len(cols), 20), np.float32)
    for f in ("m2m", "m2d", "d2m", "d2d", "i2m", "i2i", "m2i"):
        cols[f] = -rng.random(len(cols), np.float32)
    cols["ss"] = rng.integers(0, 44, len(cols)) if has_ss else 0
    pav = rng.random((len(L), 20), np.float32)
    st = hhg.HostStore(ctx, len(L), int(L.sum()), has_ss)
    st.append_packed(L, cols, pav)
    return st, L, cols, pav, np.concatenate([[0], np.cumsum(L.astype(np.int64))])


def _check_resident(sdb, ids, local, L, cols, pav, off):
    g, first = sdb.lookup(local)
    assert g.tolist() == list(ids)
    spav = sdb.read_pav()
    for t, s, f in zip(ids, local, first):
        assert sdb.Lh[s] == L[t]
        assert sdb.read_cols(0, int(f), int(L[t])).tobytes() == cols[off[t]:off[t + 1]].tobytes(), t
        assert spav[s].tobytes() == pav[t].tobytes(), t


def _same_hits(a, b, what=()):
    (ha, pa), (hb, pb_) = a, b
    assert len(ha) == len(hb)
    for f in ha.dtype.names:
        if f != "path_off":
            assert np.array_equal(ha[f].view(np.uint32), hb[f].view(np.uint32)), (what, f)
    for x, y in zip(ha, hb):
        n = int(x["nsteps"])
        assert np.array_equal(pa[x["path_off"]:x["path_off"] + n], pb_[y["path_off"]:y["path_off"] + n]), what


def _same_runner_hits(a, b, what=()):
    assert len(a) == len(b), what
    for x, y in zip(a, b):
        for f in dataclasses.fields(x):
            u, v = getattr(x, f.name), getattr(y, f.name)
            if isinstance(u, np.ndarray):
                assert np.array_equal(u, v), (what, f.name)
            elif isinstance(u, float):
                assert bits(u) == bits(v), (what, f.name)
            else:
                assert u == v, (what, f.name, u, v)


@pytest.fixture(scope="module")
def world(hhg):
    """The survivors batch of batch_cases as a resident raw shard, a store made from it and the batch's queries."""
    b = bc.make_batch("survivors")
    ctx = hhg.Context()
    db, raw, t_pav = _raw_db(hhg, ctx, b["targets"], 17)
    store = hhg.HostStore.from_db(ctx, db, has_ss=True)
    rng = np.random.default_rng(5)
    q_pav = np.stack([q["pav"] for q in b["queries"]])
    pb = rng.dirichlet(np.ones(20) * 6).astype(np.float32)
    yield dict(b=b, ctx=ctx, db=db, raw=raw, t_pav=t_pav, store=store, q_pav=q_pav, pb=pb,
               L=b["t_lens"], n=len(b["targets"]))
    store.close(); db.close(); ctx.close()


# ------------------------------------------------------------------------------------------------ 1. gather parity
@pytest.mark.parametrize("has_ss", [False, True])
def test_gather_parity(hhg, gpu_ctx, has_ss):
    """Lengths 1 .. 3000 (every run-length edge of the gather: 1, 31, 32, 33, 64, 65 records and long targets of many
    runs); scrambled subsets with duplicates, then requests that mix resident and missing targets."""
    lens = [1, 2, 31, 32, 33, 63, 64, 65, 3000, 2999] + list(range(1, 3001, 13))
    st, L, cols, pav, off = _random_store(hhg, gpu_ctx, lens, 3 + has_ss, has_ss)
    sdb = hhg.StagedDB(gpu_ctx, st, len(L), int(L.sum()))
    rng = np.random.default_rng(11)
    seen = set()
    for rnd in range(4):
        ids = rng.choice(len(L), 90, replace=False)
        ids = np.concatenate([ids, ids[:7], ids[3:5]])
        ids = ids[rng.permutation(len(ids))]
        slots = np.nonzero(sdb.Lh)[0]
        was = dict(zip(sdb.to_global(slots).tolist(), slots.tolist()))
        local = sdb.stage(ids)
        uniq = set(ids.tolist())
        assert sdb.last_stats["hits"] == len(uniq & seen) and sdb.last_stats["copied"] == len(uniq - seen)
        assert sdb.last_stats["bytes"] == sum(int(L[t]) * 112 + 92 for t in uniq - seen)
        assert all(was[int(t)] == s for t, s in zip(ids, local) if int(t) in was)      # residents keep their local id
        assert len({(int(t), int(s)) for t, s in zip(ids, local)}) == len(uniq)         # duplicates share a slot
        seen |= uniq
        _check_resident(sdb, ids, local, L, cols, pav, off)
    everything = sorted(seen)
    _check_resident(sdb, everything, sdb.stage(everything), L, cols, pav, off)          # earlier rounds are intact
    assert sdb.last_stats["copied"] == 0
    sdb.close(); st.close()


def test_store_appended_in_chunks(hhg, gpu_ctx):
    """Chunks of 1, 7 and 61 targets, from host arrays and from device shards of the HHM and A3M loaders."""
    G = golden()
    texts = [synth.hhm_text(int(L), 700 + k, f"h{k}", with_ss=True).encode()
             for k, L in enumerate(np.random.default_rng(1).integers(1, 300, 70))]
    a3ms = [synth.a3m_text(int(L), 12, 800 + k, f"a{k}", with_ss=True).encode()
            for k, L in enumerate(np.random.default_rng(2).integers(5, 120, 70))]
    loaders = [lambda t: hhg.TargetDB.from_hhm(gpu_ctx, *_pack(t), G["R"], _pp(G)),
               lambda t: hhg.TargetDB.from_a3m(gpu_ctx, *_pack(t), G["R"], G["pb"])]
    for recs, load in zip((texts, a3ms), loaders):
        whole = load(recs)
        L, cols, pav = whole.Lh.copy(), whole.read_cols(0), whole.read_pav()
        off = np.concatenate([[0], np.cumsum(L.astype(np.int64))])
        one = hhg.HostStore.from_db(gpu_ctx, whole, has_ss=True)
        whole.close()
        stores = [one]
        for from_device in (False, True):
            st = hhg.HostStore(gpu_ctx, len(L), int(L.sum()), True)
            k = 0
            for size in (1, 7, 61, 1):
                if from_device:
                    part = load(recs[k:k + size])
                    st.append_db(part)
                    part.close()
                else:
                    st.append_packed(L[k:k + size], cols[off[k]:off[k + size]], pav[k:k + size])
                k += size
            assert k == len(L) == st.n and st.columns == off[-1] and st.Lh.tolist() == L.tolist()
            stores.append(st)
        for st in stores:
            sdb = hhg.StagedDB(gpu_ctx, st, len(L), int(L.sum()))
            ids = np.random.default_rng(3).permutation(len(L))
            _check_resident(sdb, ids, sdb.stage(ids), L, cols, pav, off)
            sdb.close(); st.close()


# ------------------------------------------------------------------------------------------------ 2. search parity
def test_single_query_search_parity(hhg, world, oracle, monkeypatch):
    """hhg_viterbi_search after hhg_db_apply_null_model: all hit fields and paths, strip heights 8 and 16, local and
    global, with the ss term, with excluded regions, and a second pass with path exclusions; a sample against the C
    oracle."""
    b, db, store, L = world["b"], world["db"], world["store"], world["L"]
    G = golden()
    rng = np.random.default_rng(21)
    ids = rng.permutation(world["n"])[:90].astype(np.int32)
    packed = (db.Lh, db.read_cols(0), db.read_pav(), True)
    cases = ((11, {}, 1, None, None), (16, dict(local=False, egq=0.5, egt=0.25), 0, None, "16"),
             (14, dict(use_ss=True), 2, None, "8"), (17, {}, 3, ([(5, 9)], [(3, 12)]), None))
    for qi, par, cs, regions, forced in cases:
        q = b["queries"][qi]
        if forced:
            monkeypatch.setenv("HHG_STRIP_ROWS", forced)
        else:
            monkeypatch.delenv("HHG_STRIP_ROWS", raising=False)
        ctx = hhg.Context()                                      # the strip height is read when a context is made
        rdb = hhg.TargetDB.from_packed(ctx, *packed)
        sdb = hhg.StagedDB(ctx, store, 100, int(L[ids].sum()) + 50)
        sdb.stage(ids[rng.permutation(len(ids))])                # staged in another order than requested
        local = sdb.stage(ids)
        assert sdb.last_stats["copied"] == 0
        res = []
        for shard, tids in ((rdb, ids), (sdb, local)):
            shard.apply_null_model(q["pav"], world["pb"], cs)
            ctx.set_query(q["p"], q["tr"], q["ss"], G["S33"], **par)
            if regions:
                ctx.set_excluded_regions(*regions)
            first = hhg.viterbi_search(ctx, shard, tids)
            excl = []
            for h in first[0]:
                gi, gj, _ = hhg.expand_path(h, first[1])
                excl.append((gi[1:int(h["nsteps"])], gj[1:int(h["nsteps"])]))
            res.append((first, hhg.viterbi_search(ctx, shard, tids, exclusions=excl)))
        _same_hits(res[1][0], res[0][0], (qi, "first"))
        _same_hits(res[1][1], res[0][1], (qi, "excluded"))
        if not par and not regions:
            for k in (0, 7, 33):
                t = world["raw"][ids[k]]
                tp = bc.null_model(t[0], world["t_pav"][ids[k]], q["pav"], world["pb"], cs)
                sc, i2, j2, _ = oracle.viterbi(q["p"], q["tr"], tp, t[1])
                h = res[1][0][0][k]
                assert bits(sc) == bits(h["score"]) and (i2, j2) == (h["i2"], h["j2"])
        sdb.close(); rdb.close(); ctx.close()


@pytest.mark.parametrize("cs", [0, 1, 2, 3])
def test_batch_search_parity(hhg, world, cs):
    """hhg_viterbi_search_batch with the fused null model, BatchViterbiRunner's alternative alignments and
    hhg_mac_realign_batch (fields, paths, P_posterior) over the staged shard == over the resident one."""
    b, ctx, db, store = world["b"], world["ctx"], world["db"], world["store"]
    qs = b["queries"]
    sdb = hhg.StagedDB(ctx, store, world["n"], int(world["L"].sum()))
    local = sdb.stage(b["ids"])
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"]) for q in qs], q_pav=world["q_pav"])
    want = hhg.capi.viterbi_search_batch(ctx, db, b["req_q"], b["ids"], columnscore=cs, pb=world["pb"])
    got = hhg.capi.viterbi_search_batch(ctx, sdb, b["req_q"], local, columnscore=cs, pb=world["pb"])
    _same_hits(got, want, cs)
    if cs in (0, 1):
        rw = hhg.runner.BatchViterbiRunner(ctx, db, altali=3, columnscore=cs, pb=world["pb"]).alignment(b["req_q"], b["ids"])
        rg = hhg.runner.BatchViterbiRunner(ctx, sdb, altali=3, columnscore=cs, pb=world["pb"]).alignment(b["req_q"], local)
        for q in range(len(qs)):
            _same_runner_hits(hhg.pipeline.to_global_hits(sdb, rg[q]), rw[q], (cs, q))
        keep = np.nonzero(want[0]["nsteps"] > 0)[0][:120]
        vits = [_vit(hhg, want[0][k], want[1]) for k in keep]
        hhg.capi.mac_query_set_batch(ctx, [(q["p"], hhg.capi.log2lin(q["tr"])) for q in qs], world["q_pav"])
        out = [hhg.capi.mac_realign_batch(ctx, shard, b["req_q"][keep], tids[keep], vits, None, cs, world["pb"])
               for shard, tids in ((db, b["ids"]), (sdb, local))]
        (hw, pw), (hg, pg) = out
        assert hw.tobytes() == hg.tobytes()
        for r in range(len(keep)):
            n = int(hw["nsteps"][r])
            for f in ("i", "j", "states"):
                assert np.array_equal(pw[r][f][1:n + 1], pg[r][f][1:n + 1]), (r, f)
            assert np.array_equal(bits(pw[r]["P_posterior"][1:n + 1]), bits(pg[r]["P_posterior"][1:n + 1])), r
    sdb.close()


# ------------------------------------------------------------------------------------------------ 3. eviction
def test_eviction_rounds(hhg, world):
    """Eight requests whose union is more than twice the staged shard: every round's batch search equals the resident
    shard's, the call's own targets all stay, residents keep their local ids and the statistics add up."""
    b, ctx, db, store, L = world["b"], world["ctx"], world["db"], world["store"], world["L"]
    qs = b["queries"]
    rng = np.random.default_rng(31)
    slots = 48
    sdb = hhg.StagedDB(ctx, store, slots, 30000)
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"]) for q in qs], q_pav=world["q_pav"])
    model, evicting, copied_total = {}, 0, 0
    short = np.nonzero(L <= 600)[0]
    for rnd in range(8):
        back = prev[:12] if rnd else short[:0]                    # related requests: part of the last one comes back
        ids = np.concatenate([back, rng.choice(np.setdiff1d(short, back), 40 - len(back), replace=False)]).astype(np.int32)
        prev = ids
        local = sdb.stage(ids)
        st = sdb.last_stats
        hit = [t for t in ids.tolist() if t in model]
        assert all(model[t] == s for t, s in zip(ids.tolist(), local.tolist()) if t in model)
        assert (st["hits"], st["copied"]) == (len(hit), 40 - len(hit))
        assert sdb.to_global(local).tolist() == ids.tolist()      # nothing the call names was evicted by it
        now = {int(g): int(s) for s, g in enumerate(sdb.to_global(np.arange(slots))) if g >= 0}
        assert st["evicted"] == len(set(model) - set(now)) and len(now) == len(model) + st["copied"] - st["evicted"]
        evicting += st["evicted"] > 0
        copied_total += st["copied"]
        model = now
        rq = rng.integers(0, len(qs), 40).astype(np.int32)
        want = hhg.capi.viterbi_search_batch(ctx, db, rq, ids, columnscore=1)
        got = hhg.capi.viterbi_search_batch(ctx, sdb, rq, local, columnscore=1)
        _same_hits(got, want, rnd)
    assert evicting >= 3 and copied_total > 2 * slots
    sdb.close()


# ------------------------------------------------------------------------------------------------ 4. plan invalidation
def test_plan_invalidation(hhg, world):
    """A's slots are given to B: the identical request returns B's results, a plan made over A refuses to run, the
    single-query path wants its null model again; staging B once more costs no launch and no operand-stream rebuild."""
    b, ctx, db, store, L = world["b"], world["ctx"], world["db"], world["store"], world["L"]
    q = b["queries"][12]
    order = np.argsort(L, kind="stable")
    A, B = order[40:60].astype(np.int32), order[60:80].astype(np.int32)
    sdb = hhg.StagedDB(ctx, store, 20, int(L[B].sum()))
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"])], q_pav=q["pav"][None])
    rq = np.zeros(20, np.int32)
    la = sdb.stage(A)
    _same_hits(hhg.capi.viterbi_search_batch(ctx, sdb, rq, la), hhg.capi.viterbi_search_batch(ctx, db, rq, A), "A")
    sdb.apply_null_model(q["pav"])
    plan_a = hhg.Plan(ctx, sdb, la)
    plan_a.run()
    sdb.stage(B)
    assert sdb.last_stats["evicted"] == 20 and sdb.last_stats["copied"] == 20
    now = sdb.to_global(la)                                       # the same slots, other targets
    assert sorted(now.tolist()) == sorted(B.tolist())
    _same_hits(hhg.capi.viterbi_search_batch(ctx, sdb, rq, la), hhg.capi.viterbi_search_batch(ctx, db, rq, now), "B in A's slots")
    with pytest.raises(hhg.HhgError, match="staged anew"):
        plan_a.run()
    plan_a.close()
    ctx.set_query(q["p"], q["tr"])
    with pytest.raises(hhg.HhgError, match="hhg_db_apply_null_model"):
        hhg.viterbi_search(ctx, sdb, la)
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"])], q_pav=q["pav"][None])
    want = hhg.capi.viterbi_search_batch(ctx, db, rq, now)
    _same_hits(hhg.capi.viterbi_search_batch(ctx, sdb, rq, la), want, "B")
    n0 = ctx.launches
    hhg.capi.viterbi_search_batch(ctx, sdb, rq, la)
    per_search = ctx.launches - n0                       # a repeated request: no operand-stream rebuild
    n0 = ctx.launches
    assert sdb.stage(now).tolist() == la.tolist() and sdb.last_stats["copied"] == 0
    assert ctx.launches == n0                            # no gather launch
    _same_hits(hhg.capi.viterbi_search_batch(ctx, sdb, rq, la), want, "B again")
    assert ctx.launches - n0 == per_search               # and no rebuild after it
    sdb.close()


# ------------------------------------------------------------------------------------------------ 5. refusals
def test_refusals(hhg, world):
    b, ctx, db, store, L = world["b"], world["ctx"], world["db"], world["store"], world["L"]
    q = b["queries"][12]
    order = np.argsort(L, kind="stable")
    keep = order[10:18].astype(np.int32)
    cap = int(L[keep].sum())
    sdb = hhg.StagedDB(ctx, store, 8, cap)
    local = sdb.stage(keep)
    for _ in range(2):
        with pytest.raises(hhg.HhgError, match=f"needs 9 slots and {cap + int(L[order[18]])} columns"):
            sdb.stage(order[10:19].astype(np.int32))
        big = order[-3:].astype(np.int32)
        with pytest.raises(hhg.HhgError, match=f"needs 3 slots and {int(L[big].sum())} columns"):
            sdb.stage(big)
    for bad in (world["n"], -1):
        with pytest.raises(hhg.HhgError, match="outside the store"):
            sdb.stage(np.array([keep[0], bad], np.int32))
    with pytest.raises(hhg.HhgError, match="not made by hhg_db_create_staged"):
        hhg.StagedDB.stage(db, keep)
    other = hhg.HostStore(ctx, 4, 400, has_ss=False)
    with pytest.raises(hhg.HhgError, match="has_ss"):
        other.append_db(db)
    with pytest.raises(hhg.HhgError, match="raw and not staged"):
        other.append_db(sdb)
    with pytest.raises(hhg.HhgError, match="created for 4 / 400"):
        other.append_packed(np.array([300, 200], np.int32), np.zeros(500, hhg.capi.COLREC_DTYPE), np.zeros((2, 20), np.float32))
    assert other.n == 0
    other.close()
    with pytest.raises(hhg.HhgError, match="still use the store"):
        store.close()
    ctx.set_query(q["p"], q["tr"])
    small = hhg.StagedDB(ctx, store, 4, 100)
    with pytest.raises(hhg.HhgError, match="is empty"):
        hhg.viterbi_search(ctx, small, np.array([0], np.int32))
    small.close()
    # the residents are untouched and the context still searches
    assert sdb.stage(keep).tolist() == local.tolist() and sdb.last_stats["copied"] == 0
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"])], q_pav=q["pav"][None])
    rq = np.zeros(8, np.int32)
    _same_hits(hhg.capi.viterbi_search_batch(ctx, sdb, rq, local), hhg.capi.viterbi_search_batch(ctx, db, rq, keep))
    sdb.close()


# ------------------------------------------------------------------------------------------------ 6. launch count
def test_one_launch_whatever_n(hhg, gpu_ctx):
    st, L, cols, pav, off = _random_store(hhg, gpu_ctx, np.random.default_rng(4).integers(1, 80, 10010), 9, False)
    sdb = hhg.StagedDB(gpu_ctx, st, 10010, int(L.sum()))
    n0 = gpu_ctx.launches
    sdb.stage(np.arange(10))
    few = gpu_ctx.launches - n0
    n0 = gpu_ctx.launches
    local = sdb.stage(np.arange(10, 10010))
    assert gpu_ctx.launches - n0 == few == 1 and sdb.last_stats["copied"] == 10000
    pick = np.random.default_rng(5).integers(10, 10010, 200)
    _check_resident(sdb, pick, local[pick - 10], L, cols, pav, off)
    sdb.close(); st.close()


# ------------------------------------------------------------------------------------------------ 7. end to end
def test_pipeline_end_to_end(hhg):
    """20 000 synthetic profiles with their cs219 shard, the staged shard a quarter of the database: search_staged and
    search_batch_staged (16 queries, Lq 60 .. 1000) == search on the resident raw shard, survivors and every Hit field
    of every pass, with global target ids."""
    lib = golden()["cs219_lin"]
    bg = synth._PB.astype(np.float32)
    rng = np.random.default_rng(77)
    n = 20000
    q_lens = [60, 97, 128, 150, 200, 211, 256, 300, 333, 400, 450, 512, 640, 777, 900, 1000]
    qs = [synth.query_profile(L, 300 + k) for k, L in enumerate(q_lens)]
    lens = synth.lengths(n, rng, median=120, sigma=0.5, lo=20, hi=600)
    tg = [synth.prepared_profile(int(L), rng, qs[k % 16][4] if k % 40 < 16 else None, noise=0.35) for k, L in enumerate(lens)]
    ctx = hhg.Context()
    raw = [((t[0] * bg[None, :]).astype(np.float32), t[1], None) for t in tg]
    t_pav = np.stack([r[0][1:-1].mean(axis=0) for r in raw]).astype(np.float32)
    L = np.asarray(lens, np.int32)
    db = hhg.TargetDB(ctx, L, np.concatenate([r[0] for r in raw]), np.concatenate([r[1] for r in raw]),
                      np.concatenate([[0], np.cumsum(L.astype(np.int64) + 2)[:-1]]),
                      np.concatenate([[0], np.cumsum(L.astype(np.int64) + 1)[:-1]]), pav=t_pav)
    cs_t = [hhg.pipeline.translate_cs219(r[0][1:-1], bg, lib) for r in raw]
    cst = hhg.CsDB(ctx, L, np.concatenate([[0], np.cumsum(L)[:-1]]).astype(np.int64), np.concatenate(cs_t))
    store = hhg.HostStore.from_db(ctx, db)
    sdb = hhg.StagedDB(ctx, store, n // 4, int(L.sum()) // 4)
    pfk = dict(min_prefilter_hits=100, maxnumdb=150)
    want = []
    for q in qs:
        db.apply_null_model(q[3])
        want.append(hhg.pipeline.search(ctx, db, cst, q[0], q[1], q[3], lib, altali=2, **pfk))
    assert all(len(w[0]) >= 100 for w in want)
    for k, q in enumerate(qs):
        ids, hits = hhg.pipeline.search_staged(ctx, sdb, cst, q[0], q[1], q[3], lib, altali=2, **pfk)
        assert ids.tolist() == want[k][0].tolist()
        _same_runner_hits(hits, want[k][1], ("single", k))
    got = hhg.pipeline.search_batch_staged(ctx, sdb, cst, [(q[0], q[1], q[3]) for q in qs], lib, altali=2, **pfk)
    for k, (ids, hits) in enumerate(got):
        assert ids.tolist() == want[k][0].tolist()
        _same_runner_hits(hits, want[k][1], ("batch", k))
    sdb.close(); store.close(); cst.close(); db.close(); ctx.close()
