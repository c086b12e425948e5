"""Query-batch cs219 prefilter on the GPU: hhg_prefilter_ungapped_batch_run / _select_batch / _sw_batch,
prefilter.prefilter_db_batch and pipeline.search_batch, each equal element by element to the single-query calls made
one query at a time (which are themselves checked against the oracle and the compiled reference), and to the oracle
where it is cheap enough.  Integer work: the bar is exact equality."""
import ctypes as C

import numpy as np
import pytest

from tests.pf_batch_cases import carry_batch
from tests.util import golden

pytestmark = pytest.mark.gpu
HHG_EINVAL = -1


def _db(hhg, ctx, seqs):
    L = np.array([len(s) for s in seqs], np.int32)
    off = np.concatenate([[0], np.cumsum(L.astype(np.int64))[:-1]])
    return hhg.CsDB(ctx, L, off, np.concatenate(seqs).astype(np.uint8))


def _profile(rng, Lq):
    p = rng.integers(30, 75, (220, Lq), dtype=np.uint8)          # offset 50 +- noise like real profiles
    p[219] = 49
    return p


def _homologs(rng, best, n):
    out = []
    for _ in range(n):
        cut = int(rng.integers(1, max(2, len(best) - 1)))
        ins = rng.integers(0, 219, int(rng.integers(1, 12)), dtype=np.uint8)
        out.append(np.concatenate([best[:cut], ins, best[cut + int(rng.integers(0, 8)):]]))
    return out


BATCH_LQ = [1, 31, 64, 65, 100, 130, 257, 400, 431, 512, 513, 1025, 1500, 2100, 400]   # 400 twice: a repeated query


def test_ungapped_batch_equals_oracle_and_single(hhg, gpu_ctx, oracle):
    """Every register packing of the slabs (segments of 1..32 lanes), 2..5 tile rounds, a repeated query; sequences of
    1 to over 3000 columns with planted saturating diagonals, some across the 512 / 1024 / 1536 tile boundaries."""
    rng = np.random.default_rng(17)
    profs = [_profile(rng, Lq) for Lq in BATCH_LQ]
    best = [p[:219].argmax(axis=0).astype(np.uint8) for p in profs]
    for k in (7, 12, 13):
        profs[k][best[k], np.arange(BATCH_LQ[k])] = 120                # forces saturation
    profs[-1] = profs[7].copy()
    seqs = [rng.integers(0, 220, L, dtype=np.uint8) for L in [1, 2, 31, 32, 33, 200, 777, 3100] +
            list(rng.integers(5, 400, 90))]
    seqs += [best[7].copy(), best[9].copy(), best[10].copy(), best[11][400:700], best[13][1000:1600],
             best[12][1400:1500], np.concatenate([rng.integers(0, 219, 17, dtype=np.uint8), best[13][:1100]])]
    db = _db(hhg, gpu_ctx, seqs)
    got = db.ungapped_batch(profs, 50)
    assert got.shape == (len(profs), len(seqs))
    for q, p in enumerate(profs):
        want = [oracle.ungapped(p, s, 50) for s in seqs]
        assert got[q].tolist() == want, (q, BATCH_LQ[q])
        assert db.ungapped(p, 50).tolist() == want
    assert got[7].max() == 255 - 50 and got[13].max() == 255 - 50
    assert np.array_equal(got[7], got[-1])
    db.close()


def test_ungapped_batch_tile_boundary_carry(hhg, gpu_ctx, oracle, monkeypatch):
    """Profiles whose background decays, with diagonals across the 512 / 1024 / 1536 tile boundaries that score more
    than any single tile can see: they reach their full length only through the edge bytes between tile rounds.
    One wave, then one wave per long query; equal to the oracle and to the single-query kernel."""
    profs, seqs, cases = carry_batch(31)
    want = np.array([[oracle.ungapped(p, s, 50) for s in seqs] for p in profs])
    for q, k, score, _ in cases:
        assert want[q, k] == score, (q, k)
    assert sum(score > tile_best for _, _, score, tile_best in cases) == 6
    db = _db(hhg, gpu_ctx, seqs)
    l0 = gpu_ctx.launches
    assert np.array_equal(db.ungapped_batch(profs, 50), want)
    assert gpu_ctx.launches - l0 == 4                                # ceil(1700 / 512) tile rounds
    for q, p in enumerate(profs):
        assert db.ungapped(p, 50).tolist() == want[q].tolist(), q
    db.close()
    total = sum(len(s) for s in seqs)
    budget = len(profs) * len(seqs) * 8 + 3 * total                   # score rows + one long query's edge slots
    monkeypatch.setenv("HHG_MAX_BT_GB", repr(budget / 1e9))
    ctx = hhg.Context()
    db = _db(hhg, ctx, seqs)
    l0 = ctx.launches
    assert np.array_equal(db.ungapped_batch(profs, 50), want)
    assert ctx.launches - l0 == 4 + 3 + 2                            # one wave per long query
    db.close(); ctx.close()


def test_ungapped_batch_offsets_and_extreme_profiles(hhg, gpu_ctx, oracle):
    rng = np.random.default_rng(99)
    seqs = [rng.integers(0, 220, L, dtype=np.uint8) for L in [1, 40, 333, 900]]
    for offset in (0, 1, 50, 255):
        profs = [rng.choice(np.array([0, 1, 49, 50, 51, 128, 254, 255], np.uint8), (220, Lq)) for Lq in (70, 600, 17)]
        seqs2 = seqs + [p[:219].argmax(axis=0).astype(np.uint8) for p in profs]
        db = _db(hhg, gpu_ctx, seqs2)
        got = db.ungapped_batch(profs, offset)
        for q, p in enumerate(profs):
            assert got[q].tolist() == [oracle.ungapped(p, s, offset) for s in seqs2], (q, offset)
        db.close()


def test_batch_vs_compiled_reference(hhg, gpu_ctx, refshim, tmp_path):
    """Two profiles from the reference's own stripe_query_profile (QL 300 and 1100) in one batch: ungapped scores equal
    its ungapped_sse_score and gapped scores its swStripedByte, for every sequence, the queries' own best-state
    sequences (long diagonals across the 1100 query's tile boundaries) included."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(2)
    seqs = [rng.integers(0, 219, L, dtype=np.uint8) for L in rng.integers(1, 600, 64)]
    files, profs = [], []
    for QL in (300, 1100):
        f = tmp_path / f"q{QL}.hhm"
        f.write_text(synth.hhm_text(QL, 12, f"q{QL}"))
        q = refshim.load_query_hhm(str(f))
        qc, W = refshim.stripe_query_profile(50, 4)
        pos = np.arange(q["L"])
        prof = np.stack([qc[k * W * 32 + (pos % W) * 32 + pos // W] for k in range(220)])
        files.append(f); profs.append(prof)
        best = prof[:219].argmax(axis=0).astype(np.uint8)
        seqs += [best, best[400:800].copy(), np.concatenate([rng.integers(0, 219, 30, dtype=np.uint8), best[200:]])]
    ref_u, ref_s = [], []
    for f in files:                                                   # the reference scores with its loaded query
        refshim.load_query_hhm(str(f))
        qc, _ = refshim.stripe_query_profile(50, 4)
        ref_u.append([refshim.ungapped(qc, s, 50) for s in seqs])
        ref_s.append([refshim.sw_byte(qc, s, 24, 4, 50) for s in seqs])
    db = _db(hhg, gpu_ctx, seqs)
    got = db.ungapped_batch(profs, 50)
    assert got[0].tolist() == ref_u[0] and got[1].tolist() == ref_u[1]
    n = len(seqs)
    rq = np.repeat(np.array([0, 1], np.int32), n)
    ids = np.tile(np.arange(n, dtype=np.int32), 2)
    sw = db.sw_batch(profs, rq, ids, 24, 4, 50)
    assert sw[:n].tolist() == ref_s[0] and sw[n:].tolist() == ref_s[1]
    db.close()


def _selection_case(rng, case, best):
    if case == "many_above":
        return [rng.integers(0, 219, L, dtype=np.uint8) for L in rng.integers(30, 400, 3000)] + _homologs(rng, best, 150), 100
    if case == "few_above_ties":
        base = [rng.integers(0, 219, 120, dtype=np.uint8) for _ in range(8)]
        return [base[int(rng.integers(0, 8))] for _ in range(2500)] + _homologs(rng, best, 7), 300
    if case == "tiny_db":
        return [rng.integers(0, 219, L, dtype=np.uint8) for L in rng.integers(30, 200, 37)], 100
    return [rng.integers(0, 219, 150, dtype=np.uint8)] * 1000, 64


@pytest.mark.parametrize("case", ["many_above", "few_above_ties", "tiny_db", "all_tied"])
def test_select_batch_equals_single(hhg, gpu_ctx, oracle, case):
    """The regimes of the single-query selection (more survivors than min_hits; a cut inside a tie class; a shard
    smaller than min_hits; all tied) for every query of a batch: the golden profile, a shorter and a longer one."""
    G = golden()
    rng = np.random.default_rng({"many_above": 1, "few_above_ties": 2, "tiny_db": 3, "all_tied": 4}[case])
    prof = G["pf_prof"]
    profs = [prof, prof[:, :90].copy(), np.tile(prof, (1, 3))[:, :700].copy()]
    seqs, min_hits = _selection_case(rng, case, prof[:219].argmax(axis=0).astype(np.uint8))
    perm = rng.permutation(len(seqs))
    seqs = [seqs[i] for i in perm]
    db = _db(hhg, gpu_ctx, seqs)
    Lq = [p.shape[1] for p in profs]
    db.run_batch(profs, 50)
    got = db.select_batch(Lq, 4, 10, min_hits)
    for q, p in enumerate(profs):
        db.run(p, 50)
        ids, sc = db.select(Lq[q], 4, 10, min_hits)
        assert got[q][0].tolist() == ids.tolist() and got[q][1].tolist() == sc.tolist(), q
    # the first query against the oracle's scores and the reference's rule
    corr = [oracle.lib.hho_ungapped_corrected(oracle.ungapped(prof, s, 50), Lq[0], len(s), 4) for s in seqs] \
        if case != "all_tied" else [oracle.lib.hho_ungapped_corrected(oracle.ungapped(prof, seqs[0], 50), Lq[0],
                                                                      len(seqs[0]), 4)] * len(seqs)
    order = sorted(range(len(seqs)), key=lambda k: (corr[k], k), reverse=True)
    want = []
    for k in order:
        if len(want) >= min_hits and corr[k] <= 10:
            break
        want.append(k)
    assert got[0][0].tolist() == want
    db.close()


def test_select_batch_capacity_refusal(hhg, gpu_ctx):
    rng = np.random.default_rng(8)
    seqs = [rng.integers(0, 219, L, dtype=np.uint8) for L in rng.integers(30, 300, 500)]
    profs = [_profile(rng, 120), _profile(rng, 700)]
    db = _db(hhg, gpu_ctx, seqs)
    db.run_batch(profs, 50)
    full = db.select_batch([120, 700], 4, 10, 40)
    need = sum(len(f[0]) for f in full)
    ids = np.zeros(need, np.int32); sc = np.zeros(need, np.int32); off = np.zeros(3, np.int32)
    Lq = np.array([120, 700], np.int32)
    rc = gpu_ctx.L.hhg_prefilter_select_batch(gpu_ctx.h, db.h, 2, Lq.ctypes.data_as(C.POINTER(C.c_int32)), 4, 10, 40,
                                              ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                              sc.ctypes.data_as(C.POINTER(C.c_int32)), need - 1,
                                              off.ctypes.data_as(C.POINTER(C.c_int32)))
    assert rc == HHG_EINVAL
    assert off[2] == need                                           # the capacity the call needed
    again = db.select_batch([120, 700], 4, 10, 40, cap=need)        # the context still works
    assert all(np.array_equal(a[0], b[0]) for a, b in zip(again, full))
    db.close()


def test_sw_batch_equals_oracle_and_single(hhg, gpu_ctx, oracle):
    """Queries of Lq 20, 928, 929 and 1500 (profiles in shared memory and in L2) in one launch; interleaved request
    order, one query with no requests, repeated (query, id) pairs."""
    G = golden()
    rng = np.random.default_rng(41)
    big = np.tile(G["pf_prof"], (1, 4))
    profs = [G["pf_prof"][:, :20].copy(), big[:, :928].copy(), _profile(rng, 50), big[:, 1:930].copy(),
             big[:, 3:1503].copy()]
    seqs = [rng.integers(0, 219, L, dtype=np.uint8) for L in [1, 2, 33, 500] + list(rng.integers(5, 300, 40))]
    for p in profs[1:]:
        seqs += _homologs(rng, p[:219].argmax(axis=0).astype(np.uint8), 4)
    db = _db(hhg, gpu_ctx, seqs)
    rq, ids = [], []
    for _ in range(3):
        for q in (0, 1, 3, 4):                                       # query 2 has no requests
            for i in rng.permutation(len(seqs))[:25]:
                rq.append(q); ids.append(int(i))
    rq += [1, 1, 4]; ids += [ids[1], ids[1], ids[3]]
    rq = np.array(rq, np.int32); ids = np.array(ids, np.int32)
    o = rng.permutation(len(rq)); rq, ids = rq[o], ids[o]
    got = db.sw_batch(profs, rq, ids, 24, 4, 50)
    for q in (0, 1, 3, 4):
        sel = np.nonzero(rq == q)[0]
        assert got[sel].tolist() == db.sw(profs[q], ids=ids[sel], gap_open=24, gap_extend=4, bias=50).tolist(), q
    for k in rng.permutation(len(rq))[:60]:
        assert got[k] == oracle.sw_byte(profs[rq[k]], seqs[ids[k]], 24, 4, 50), k
    assert db.sw_batch(profs, [], []).tolist() == []
    db.close()


def _scale_setup(hhg, ctx, nseq=200_000, nq=24, seed=5):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(seed)
    d = synth.cs219_db(nseq, seed)
    seq = d["seq"].copy()
    lens = [int(x) for x in rng.integers(50, 1500, nq)]
    lens[:3] = [400, 513, 1500]
    profs = [_profile(rng, Lq) for Lq in lens]
    for p in profs:                                                  # planted homologs of every query
        best = p[:219].argmax(axis=0).astype(np.uint8)
        for t in rng.integers(0, nseq, 30):
            m = min(int(d["L"][t]), len(best))
            seq[d["off"][t]:d["off"][t] + m] = best[:m]
    return hhg.CsDB(ctx, d["L"], d["off"], seq), profs


def test_prefilter_db_batch_at_scale(hhg, gpu_ctx):
    csdb, profs = _scale_setup(hhg, gpu_ctx)
    kw = dict(min_prefilter_hits=100, maxnumdb=2000)
    want = [hhg.prefilter.prefilter_db(csdb, p, **kw) for p in profs]
    l0 = gpu_ctx.launches
    got = hhg.prefilter.prefilter_db_batch(csdb, profs, **kw)
    launches = gpu_ctx.launches - l0
    assert len(got) == len(want)
    for q in range(len(profs)):
        assert got[q].tolist() == want[q].tolist(), q
    assert sum(len(w) for w in want) >= 24 * 30
    # per stage, launches do not grow with the number of queries: ceil(1500/512) tile rounds + 2 (selection) + 1 (sw)
    assert launches == 3 + 2 + 1
    l0 = gpu_ctx.launches
    two = hhg.prefilter.prefilter_db_batch(csdb, profs[1:3], **kw)
    assert gpu_ctx.launches - l0 == launches
    assert [x.tolist() for x in two] == [x.tolist() for x in want[1:3]]
    csdb.close()


def test_prefilter_db_batch_memory_waves(hhg, monkeypatch):
    """A budget of one long query's edge slots per wave: the same survivors, and the waves show in the launch count."""
    monkeypatch.setenv("HHG_MAX_BT_GB", "0.1")
    ctx = hhg.Context()
    csdb, profs = _scale_setup(hhg, ctx, nseq=200_000, nq=12, seed=9)
    csdb_total = int(np.sum(csdb.Lh))
    assert 2 * csdb_total <= 0.1e9 < 4 * csdb_total                   # one long query per wave
    kw = dict(min_prefilter_hits=50, maxnumdb=1000)
    want = [hhg.prefilter.prefilter_db(csdb, p, **kw) for p in profs]
    l0 = ctx.launches
    got = hhg.prefilter.prefilter_db_batch(csdb, profs, **kw)
    launches = ctx.launches - l0
    assert [g.tolist() for g in got] == [w.tolist() for w in want]
    n_long = sum(p.shape[1] > 512 for p in profs)
    assert n_long >= 3
    tiles = sum((p.shape[1] + 511) // 512 for p in profs if p.shape[1] > 512)
    assert launches == tiles + 2 + 1
    csdb.close(); ctx.close()


def test_prefilter_db_batch_score_budget(hhg, monkeypatch):
    """A budget that holds the score rows of 3 queries: run_batch refuses 7 before any launch, and prefilter_db_batch
    runs them in groups of 3 with the same survivors as the per-query calls."""
    rng = np.random.default_rng(21)
    seqs = [rng.integers(0, 219, L, dtype=np.uint8) for L in rng.integers(20, 400, 20000)]
    monkeypatch.setenv("HHG_MAX_BT_GB", repr(3.5 * 8 * len(seqs) / 1e9))
    ctx = hhg.Context()
    db = _db(hhg, ctx, seqs)
    assert db.max_batch() == 3
    profs = [_profile(rng, Lq) for Lq in (60, 300, 700, 90, 1200, 45, 512)]
    l0 = ctx.launches
    with pytest.raises(hhg.capi.HhgError):
        db.run_batch(profs, 50)
    assert ctx.launches == l0
    kw = dict(min_prefilter_hits=30, maxnumdb=300)
    want = [hhg.prefilter.prefilter_db(db, p, **kw) for p in profs]
    got = hhg.prefilter.prefilter_db_batch(db, profs, **kw)
    assert [g.tolist() for g in got] == [w.tolist() for w in want]
    db.close(); ctx.close()


def test_search_batch_equals_search(hhg, gpu_ctx):
    """pipeline.search_batch == pipeline.search per query: survivors and every Hit field of every pass."""
    from hhsuite_b200 import synth
    G = golden()
    lib = G["cs219_lin"]
    n = 3000
    qs = [synth.query_profile(L, s) for L, s in ((300, 5), (120, 6), (700, 7))]
    db_h = synth.prepared_db(n, seed=8, query_cols=qs[0][4], planted=25, fast=True, hi=600)
    prof_list = [(db_h["p"][db_h["p_off"][t]:db_h["p_off"][t] + int(db_h["L"][t]) + 2],
                  db_h["tr"][db_h["tr_off"][t]:db_h["tr_off"][t] + int(db_h["L"][t]) + 1], None) for t in range(n)]
    db = hhg.TargetDB.from_profiles(gpu_ctx, prof_list)
    bg = synth._PB.astype(np.float32)
    seqs = [hhg.pipeline.translate_cs219(p[1:-1] * bg[None, :], bg, lib) for (p, tr, ss) in prof_list]
    csdb = _db(hhg, gpu_ctx, seqs)
    kw = dict(min_prefilter_hits=40, maxnumdb=300)
    want = [hhg.pipeline.search(gpu_ctx, db, csdb, q[0], q[1], q[3], lib, **kw) for q in qs]
    got = hhg.pipeline.search_batch(gpu_ctx, db, csdb, [(q[0], q[1], q[3]) for q in qs], lib, **kw)
    assert len(got) == 3
    for (ids_b, hits_b), (ids_s, hits_s) in zip(got, want):
        assert ids_b.tolist() == ids_s.tolist()
        assert len(hits_b) == len(hits_s) and len(hits_s) >= len(ids_s)
        for a, b in zip(hits_b, hits_s):
            for f in ("target", "irep", "lastrep", "score", "score_ss", "vit_score", "i1", "i2", "j1", "j2", "nsteps",
                      "matched_cols"):
                assert getattr(a, f) == getattr(b, f), f
            for f in ("i", "j", "states"):
                assert np.array_equal(getattr(a, f), getattr(b, f)), f
    db.close(); csdb.close()


def test_bad_input_refused_before_launch(hhg, gpu_ctx):
    rng = np.random.default_rng(3)
    seqs = [rng.integers(0, 219, 50, dtype=np.uint8) for _ in range(20)]
    db = _db(hhg, gpu_ctx, seqs)
    L = gpu_ctx.L
    i32 = lambda a: np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int32))   # noqa: E731
    p = _profile(rng, 60)
    ptrs = (C.c_void_p * 2)(p.ctypes.data, p.ctypes.data)
    nullp = (C.c_void_p * 2)(p.ctypes.data, None)
    Lq, Lbad = np.array([60, 60], np.int32), np.array([60, 0], np.int32)
    out = np.zeros(100, np.int32); off = np.zeros(3, np.int32)
    l0 = gpu_ctx.launches
    h, c = gpu_ctx.h, db.h
    bad = [
        L.hhg_prefilter_ungapped_batch_run(h, c, 0, i32(Lq), ptrs, 50),
        L.hhg_prefilter_ungapped_batch_run(h, c, 2, i32(Lbad), ptrs, 50),
        L.hhg_prefilter_ungapped_batch_run(h, c, 2, i32(Lq), nullp, 50),
        L.hhg_prefilter_ungapped_batch_run(h, c, 2, i32(Lq), ptrs, -1),
        L.hhg_prefilter_ungapped_batch_run(h, c, 2, i32(Lq), ptrs, 256),
        L.hhg_prefilter_ungapped_batch_fetch(h, c, i32(out)),          # no batch run on this shard yet
        L.hhg_prefilter_select_batch(h, c, 2, i32(Lq), 4, 10, 5, i32(out), i32(out), 100, i32(off)),
        L.hhg_prefilter_sw_batch(h, c, 2, i32(Lq), ptrs, 1, i32([2]), i32([0]), 24, 4, 50, i32(out)),
        L.hhg_prefilter_sw_batch(h, c, 2, i32(Lq), ptrs, 1, i32([-1]), i32([0]), 24, 4, 50, i32(out)),
        L.hhg_prefilter_sw_batch(h, c, 2, i32(Lq), ptrs, 1, i32([0]), i32([20]), 24, 4, 50, i32(out)),
        L.hhg_prefilter_sw_batch(h, c, 2, i32(Lq), ptrs, 1, i32([0]), i32([-1]), 24, 4, 50, i32(out)),
        L.hhg_prefilter_sw_batch(h, c, 2, i32(Lbad), ptrs, 1, i32([0]), i32([0]), 24, 4, 50, i32(out)),
        L.hhg_prefilter_sw_batch(h, c, 2, i32(Lq), nullp, 1, i32([0]), i32([0]), 24, 4, 50, i32(out)),
        L.hhg_prefilter_sw_batch(h, c, 0, i32(Lq), ptrs, 1, i32([0]), i32([0]), 24, 4, 50, i32(out)),
        L.hhg_prefilter_sw_batch(h, c, 1, i32([9700]), ptrs, 1, i32([0]), i32([0]), 24, 4, 50, i32(out)),   # too long
    ]
    assert all(rc == HHG_EINVAL for rc in bad), bad
    assert gpu_ctx.launches == l0
    db.run_batch([p, p], 50)
    l1 = gpu_ctx.launches
    assert L.hhg_prefilter_select_batch(h, c, 1, i32(Lq), 4, 10, 5, i32(out), i32(out), 100, i32(off)) == HHG_EINVAL   # nq != run
    assert L.hhg_prefilter_select_batch(h, c, 2, i32(Lbad), 4, 10, 5, i32(out), i32(out), 100, i32(off)) == HHG_EINVAL
    assert gpu_ctx.launches == l1
    assert np.array_equal(db.fetch_batch(2)[0], db.ungapped(p, 50))
    db.close()
