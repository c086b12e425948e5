"""Column score 5 (-sc 5 / -scwin D: the local amino-acid composition correction, k_local_bg) on the device: shards of
every loader prepared by hhg_db_apply_null_model against the compiled reference, the query helper against
PrepareQueryHMM, the drop-in check under -sc 5, the batch Viterbi search and the batch MAC realignment over resident,
store-backed and record-sourced shards against the single-query calls, a seeded sequence of mode, window and background
switches on one context, the staged pipelines, and the inputs that are refused."""
import os
import subprocess

import numpy as np
import pytest

from tests import batch_cases as bc
from tests.test_batch_realign_gpu import _mac_batch, _mac_per_query, _raw_db, _same_hits, _same_mac, _viterbi_requests
from tests.util import bits, golden, ref_data_file

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "oracle", "_ref", "hh_dropin_check_localbg")   # the drop-in check with --sc / --scwin
QUERY = os.path.join(ROOT, "oracle", "_ref", "data", "query.hhm")


def _full(cols, L):
    """Emissions of L records as a profile [(L+2), 20] with zero rows 0 and L+1 (what the reference routine reads)."""
    p = np.zeros((L + 2, 20), np.float32)
    p[1:L + 1] = cols["p"]
    return p


def _words(cols):
    return np.ascontiguousarray(cols).view(np.uint32).reshape(-1, 28)


def _records(hhg, db):
    off = np.concatenate([[0], np.cumsum(db.Lh.astype(np.int64))])
    return off, db.read_cols(0), db.read_cols(1)


def _check_shard(lbref, db, pb, D):
    """read_cols(1) == the reference's routine on read_cols(0), target by target; transitions and ss unchanged."""
    off, raw, prep = _records(None, db)
    assert prep.tobytes() != raw.tobytes()
    for t, L in enumerate(db.Lh):
        a, b = raw[off[t]:off[t + 1]], prep[off[t]:off[t + 1]]
        want = lbref.local_bg(_full(a, int(L)), pb, D)[1:L + 1]
        assert np.array_equal(bits(b["p"]), bits(want)), (t, int(L))
        assert np.array_equal(_words(b)[:, 20:], _words(a)[:, 20:]), t


@pytest.fixture(scope="module")
def lbref():
    """The compiled reference's local composition correction (oracle/localbg_shim.cpp)."""
    from oracle.localbg_binding import LocalBgRef
    try:
        return LocalBgRef()
    except (FileNotFoundError, OSError) as e:
        pytest.skip(f"compiled reference not available: {e}")


# ------------------------------------------------------------------------------------------------ shards and queries
def test_apply_null_model_on_hhm_shard_equals_reference(hhg, gpu_ctx, lbref, tmp_path):
    """Templates read from HHM text by hhg_db_create_hhm and divided by apply_null_model(5) == the reference's
    PrepareTemplateHMM under -sc 5 / -scwin D (HMM::Read ... IncludeNullModelInHMM case 5), bit for bit."""
    from hhsuite_b200 import synth
    lens = [1, 7, 81, 82, 83, 150, 431, 60]
    texts = [synth.hhm_text(L, 700 + k, f"h{k}", with_ss=k % 2 == 0).encode() for k, L in enumerate(lens)]
    data = b"".join(t + b"\0" for t in texts)
    ln = np.array([len(t) + 1 for t in texts], np.int64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.int64)
    db = hhg.TargetDB.from_hhm(gpu_ctx, data, off, ln, lbref.R(), None)
    try:
        for D in (40, 3):
            lbref.prepare_query_hhm(ref_data_file("query.hhm", tmp_path), 5, D)
            want = []
            for k, t in enumerate(texts):
                path = tmp_path / f"h{k}.hhm"
                path.write_bytes(t)
                want.append(lbref.prepare_template_hhm(path))
            pb = want[0]["pb"]                 # the records' NULL line, which HMM::Read made the background
            assert all(np.array_equal(bits(w["pb"]), bits(pb)) for w in want)
            gpu_ctx.set_scwin(D)
            db.apply_null_model(None, pb, 5)
            o, raw, prep = _records(hhg, db)
            for k, L in enumerate(db.Lh):
                assert np.array_equal(bits(prep["p"][o[k]:o[k + 1]]), bits(want[k]["p"][1:L + 1])), (D, k)
            assert np.array_equal(prep["ss"], raw["ss"]) and np.array_equal(prep["m2m"], raw["m2m"])
    finally:
        gpu_ctx.set_scwin(40)
        db.close()


def test_apply_null_model_on_a3m_and_packed_shards(hhg, gpu_ctx, lbref):
    from hhsuite_b200 import synth
    G = golden()
    a3ms = [synth.a3m_text(int(L), 12, 300 + k, f"a{k}", with_ss=k % 2 == 0).encode()
            for k, L in enumerate([5, 40, 41, 83, 160, 220])]
    text = b"".join(a + b"\0" for a in a3ms)
    ln = np.array([len(a) + 1 for a in a3ms], np.int64)
    offs = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.int64)
    adb = hhg.TargetDB.from_a3m(gpu_ctx, text, offs, ln, G["R"], G["pb"])
    rng = np.random.default_rng(3)
    L = rng.integers(1, 300, 25).astype(np.int32)
    L[:3] = [1, 2, 32767]
    cols = np.zeros(int(L.sum()), hhg.capi.COLREC_DTYPE)
    cols["p"] = rng.dirichlet(np.ones(20), len(cols)).astype(np.float32)
    cols["m2m"] = rng.random(len(cols)); cols["ss"] = rng.integers(0, 100, len(cols))
    pdb = hhg.TargetDB.from_packed(gpu_ctx, L, cols, rng.random((len(L), 20)).astype(np.float32))
    try:
        for D, pb in ((40, G["pb"]), (2, rng.dirichlet(np.ones(20)).astype(np.float32))):
            gpu_ctx.set_scwin(D)
            for db in (adb, pdb):
                db.apply_null_model(None, pb, 5)
                _check_shard(lbref, db, pb, D)
    finally:
        gpu_ctx.set_scwin(40)
        adb.close(); pdb.close()


def test_query_local_background_equals_prepare_query(hhg, gpu_ctx, lbref, tmp_path):
    """PrepareQueryHMM under -sc 5 for data/query.hhm (D = 40 and 3), and the reference's routine for a query shorter
    than the window and for the longest query."""
    path = ref_data_file("query.hhm", tmp_path)
    plain, pb = lbref.prepare_query_hhm(path, 1, 40)
    try:
        for D in (40, 3):
            want = lbref.prepare_query_hhm(path, 5, D)[0]
            gpu_ctx.set_scwin(D)
            got = hhg.capi.query_local_background(gpu_ctx, plain, pb)
            assert np.array_equal(bits(got), bits(want)), D
            assert np.array_equal(bits(got[[0, -1]]), bits(plain[[0, -1]]))
        rng = np.random.default_rng(11)
        for L, D in ((5, 40), (81, 40), (32767, 40), (32767, 16383), (300, 1)):
            p = rng.dirichlet(np.ones(20), L + 2).astype(np.float32)
            gpu_ctx.set_scwin(D)
            got = hhg.capi.query_local_background(gpu_ctx, p, pb)
            assert np.array_equal(bits(got), bits(lbref.local_bg(p, pb, D))), (L, D)
    finally:
        gpu_ctx.set_scwin(40)


# ------------------------------------------------------------------------------------------------ drop-in check
def _run(args):
    r = subprocess.run([BIN] + args, capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:], r.stderr[-2000:])
    return r


@pytest.mark.skipif(not os.path.exists(BIN), reason="oracle/_ref/hh_dropin_check_localbg not built/shipped")
@pytest.mark.parametrize("scwin", [40, 3])
def test_dropin_check_with_local_composition_correction(tmp_path, scwin):
    """hh_dropin_check_localbg --sc 5 --scwin D: the reference's own PrepareQueryHMM / PrepareTemplateHMM under -sc 5
    and its runner vs the adapter (hhg_set_scwin + hhg_db_apply_null_model(5)), HHM and A3M templates, with the MAC
    realignment, every Hit and every MAC alignment identical.  (The adapter realigns A3M templates from the shard the
    Viterbi stage read, with global sequence weights, where the reference rereads them with position-specific ones, so
    --mac is checked on HHM templates.)"""
    from hhsuite_b200 import synth
    sc = ["--sc", "5", "--scwin", str(scwin)]
    hhm = []
    for k, L in enumerate([150, 60, 431, 33, 200, 7, 97]):
        f = tmp_path / f"t{k}.hhm"
        f.write_text(synth.hhm_text(L, 100 + k, f"t{k}", with_ss=k % 3 == 0))
        hhm.append(str(f))
    a3m = []
    for k, (L, n) in enumerate([(150, 40), (60, 5), (300, 120), (33, 0), (97, 60)]):
        f = tmp_path / f"a{k}.a3m"
        f.write_text(synth.a3m_text(L, n, 400 + k, f"a{k}", with_ss=k % 2 == 0))
        a3m.append(str(f))
    for args in ([QUERY, QUERY] + hhm, ["--mac", QUERY, QUERY] + hhm, ["--hhm-loader", QUERY, QUERY] + hhm,
                 ["--hhm-loader", QUERY] + a3m):
        r = _run(sc + args)
        assert f"column score 5, half window {scwin}" in r.stdout, r.stdout + r.stderr
        assert r.returncode == 0 and "all hits identical" in r.stdout, r.stdout + r.stderr
        if "--mac" in args:
            assert "all MAC alignments identical" in r.stdout, r.stdout


@pytest.mark.skipif(not os.path.exists(BIN), reason="oracle/_ref/hh_dropin_check_localbg not built/shipped")
def test_dropin_check_early_stopping_with_local_composition_correction(tmp_path):
    """--hhblits 2100 under -sc 5: the first chunk of 2000 ends the round on both sides."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(9)
    files = []
    for k in range(2100):
        f = tmp_path / f"e{k}.hhm"
        f.write_text(synth.hhm_text(int(rng.integers(30, 70)), 9000 + k, f"e{k}"))
        files.append(str(f))
    r = _run(["--sc", "5", "--hhblits", "2100", "--real-lengths", QUERY] + files)
    assert "column score 5, half window 40" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0 and "all hits identical" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert "early stop after 2000 of 2100" in r.stdout


# ------------------------------------------------------------------------------------------------ batch mode
@pytest.fixture(scope="module")
def batch5(hhg):
    b = bc.make_batch("survivors")
    ctx = hhg.Context()
    db, raw, t_pav = _raw_db(hhg, ctx, b["targets"], 23)
    rng = np.random.default_rng(8)
    pb = rng.dirichlet(np.ones(20) * 6).astype(np.float32)
    q_pav = np.stack([q["pav"] for q in b["queries"]]).astype(np.float32)
    qs = [dict(q, p=hhg.capi.query_local_background(ctx, q["p"], pb)) for q in b["queries"]]
    yield dict(b=b, ctx=ctx, db=db, raw=raw, pb=pb, q_pav=q_pav, qs=qs)
    db.close(); ctx.close()


def _single(hhg, ctx, db, qs, rq, ids, pb, altali=1):
    """apply_null_model(5) + hhg_query_set + runner.ViterbiRunner per query, hits in request order per query."""
    db.apply_null_model(None, pb, 5)
    out = [[] for _ in qs]
    for q in np.unique(rq):
        ctx.set_query(qs[q]["p"], qs[q]["tr"])
        out[q] = hhg.runner.ViterbiRunner(ctx, db, altali=altali).alignment(ids[rq == q])
    return out


def _batch(hhg, ctx, db, qs, rq, ids, pb, altali=1, q_pav=None):
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"]) for q in qs], q_pav=q_pav)
    return hhg.runner.BatchViterbiRunner(ctx, db, altali=altali, columnscore=5, pb=pb).alignment(rq, ids)


def test_batch_search_equals_single_query(hhg, batch5):
    """viterbi_search_batch(5) and BatchViterbiRunner (alternative alignments) over a raw shard == apply(5) plus the
    single-query runner per query: hits, paths, Hit.score bit for bit.  The batch leaves the shard unprepared."""
    S = batch5
    b, ctx, db, pb, qs = S["b"], S["ctx"], S["db"], S["pb"], S["qs"]
    rq, ids = b["req_q"], b["ids"]
    for altali in (1, 3):
        got = _batch(hhg, ctx, db, qs, rq, ids, pb, altali)
        with pytest.raises(hhg.capi.HhgError):
            hhg.capi.viterbi_search(ctx, db, ids[:4])
        want = _single(hhg, ctx, db, qs, rq, ids, pb, altali)
        for q in range(len(qs)):
            _same_hits(got[q], want[q], (altali, q))
        assert sum(len(x) for x in got) >= len(ids)


def test_batch_over_staged_shards_equals_resident(hhg, batch5):
    """The same batch over a store-backed staged shard equals the resident raw shard; A3M records staged from their
    text (record-sourced) equal the resident shard of the same records."""
    from hhsuite_b200 import synth
    S = batch5
    b, ctx, db, pb, qs = S["b"], S["ctx"], S["db"], S["pb"], S["qs"]
    rq, ids = b["req_q"], b["ids"]
    want = _batch(hhg, ctx, db, qs, rq, ids, pb, 2)
    store = hhg.HostStore.from_db(ctx, db, has_ss=all(r[2] is not None for r in S["raw"]))
    u = np.unique(ids)
    sdb = hhg.StagedDB(ctx, store, len(u) + 5, int(db.Lh[u].sum()) + 100)
    local = sdb.stage(ids)
    got = _batch(hhg, ctx, sdb, qs, rq, local, pb, 2)
    for q in range(len(qs)):
        _same_hits(hhg.pipeline.to_global_hits(sdb, got[q]), want[q], q)
    sdb.close(); store.close()
    # record-sourced
    G = golden()
    rng = np.random.default_rng(4)
    a3ms = [synth.a3m_text(int(L), 10, 1900 + k, f"r{k}", with_ss=k % 2 == 0).encode()
            for k, L in enumerate(rng.integers(5, 160, 24))]
    text = b"".join(a + b"\0" for a in a3ms)
    ln = np.array([len(a) + 1 for a in a3ms], np.int64)
    offs = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.int64)
    adb = hhg.TargetDB.from_a3m(ctx, text, offs, ln, G["R"], G["pb"])
    src = hhg.RecordSource.from_a3m(ctx, text, offs, ln, G["R"], G["pb"], has_ss=True)
    rsdb = hhg.StagedDB(ctx, src, 20, int(adb.Lh.sum()))
    aq = [hhg.capi.query_from_a3m(ctx, a3ms[k], G["R"], G["pb"]) for k in (3, 11)]
    aqs = [dict(p=hhg.capi.query_local_background(ctx, q["p"], pb), tr=q["tr"]) for q in aq]
    rq2 = np.array([0, 1] * 9, np.int32)
    ids2 = np.array([7, 3, 21, 11, 0, 23, 16, 5, 3, 11, 2, 9, 12, 1, 18, 4, 7, 6], np.int32)
    local2 = rsdb.stage(ids2)
    hhg.capi.query_set_batch(ctx, [(q["p"], q["tr"]) for q in aqs])
    (h1, p1), (h2, p2) = (hhg.capi.viterbi_search_batch(ctx, d, rq2, x, columnscore=5, pb=pb)
                          for d, x in ((adb, ids2), (rsdb, local2)))
    assert h1.tobytes() == h2.tobytes() and p1.tobytes() == p2.tobytes()
    rsdb.close(); src.close(); adb.close()


def test_mac_batch_equals_per_query(hhg, batch5):
    """mac_realign_batch(5) == apply_null_model(5) + mac_query_set + mac_realign per query, posteriors included."""
    S = batch5
    b, ctx, db, pb, qs = S["b"], S["ctx"], S["db"], S["pb"], S["qs"]
    rq, ids, vits = _viterbi_requests(hhg, ctx, db, qs, None, b["req_q"], b["ids"], 5, pb)
    assert len(ids) >= 100
    got = _mac_batch(hhg, ctx, db, qs, None, rq, ids, vits, 5, pb, True, 0.35)
    want = _mac_per_query(hhg, ctx, db, qs, S["q_pav"], rq, ids, vits, 5, pb, True, 0.35)
    _same_mac(got, want, 5)
    assert int(np.sum(got[0]["nsteps"] > 0)) >= 5


# ------------------------------------------------------------------------------------------------ state and refusals
def _small_case(hhg, seed):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(seed)
    qs = [synth.query_profile(int(L), seed + k) for k, L in enumerate((60, 97, 33))]
    tg = [synth.prepared_profile(int(L), rng, qs[k % 3][4] if k % 2 else None, noise=0.3)
          for k, L in enumerate(rng.integers(5, 250, 40))]
    raw = [bc.raw_profile(t, rng) for t in tg]
    return qs, raw


def _db_of(hhg, ctx, raw):
    L = np.array([r[0][0].shape[0] - 2 for r in raw], np.int32)
    return hhg.TargetDB(ctx, L, np.concatenate([r[0][0] for r in raw]), np.concatenate([r[0][1] for r in raw]),
                        np.concatenate([[0], np.cumsum(L.astype(np.int64) + 2)[:-1]]),
                        np.concatenate([[0], np.cumsum(L.astype(np.int64) + 1)[:-1]]), pav=np.stack([r[1] for r in raw]))


def _step(hhg, ctx, db, qs, q_pav, kind, cs, D, pb, ids):
    """One call of the sequence: 'single' (apply + single-query search of query 0) or 'batch' (all queries)."""
    ctx.set_scwin(D)
    qp = [hhg.capi.query_local_background(ctx, q[0], pb) if cs == 5 else q[0] for q in qs]
    if kind == "single":
        db.apply_null_model(q_pav[0], pb, cs)
        ctx.set_query(qp[0], qs[0][1])
        h, p = hhg.capi.viterbi_search(ctx, db, ids)
        return h.tobytes() + p.tobytes() + db.read_cols(1).tobytes() + qp[0].tobytes()
    hhg.capi.query_set_batch(ctx, [(p, q[1]) for p, q in zip(qp, qs)], q_pav=q_pav)
    rq = np.arange(len(ids), dtype=np.int32) % len(qs)
    h, p = hhg.capi.viterbi_search_batch(ctx, db, rq, ids, columnscore=cs, pb=pb)
    return h.tobytes() + p.tobytes()


def test_switching_modes_windows_and_backgrounds(hhg):
    """1 -> 5 -> 1 -> 5 on one context and one shard, D and pb changing, single and batch calls interleaved: every
    result equals the same call on a fresh context and shard.  After a batch under 5, a single-query search without a
    new apply_null_model is refused."""
    qs, raw = _small_case(hhg, 31)
    q_pav = np.stack([q[3] for q in qs]).astype(np.float32)
    rng = np.random.default_rng(2)
    pbs = [rng.dirichlet(np.ones(20) * 5).astype(np.float32) for _ in range(3)]
    ids = rng.integers(0, len(raw), 30).astype(np.int32)
    seq = [("single", 1, 40, pbs[0]), ("batch", 5, 40, pbs[0]), ("single", 5, 3, pbs[1]), ("batch", 1, 3, pbs[1]),
           ("batch", 5, 7, pbs[2]), ("single", 1, 7, pbs[2]), ("batch", 5, 7, pbs[0]), ("single", 5, 40, pbs[2]),
           ("batch", 5, 1, pbs[2]), ("batch", 5, 1, pbs[1])]
    ctx = hhg.Context()
    db = _db_of(hhg, ctx, raw)
    try:
        for k, (kind, cs, D, pb) in enumerate(seq):
            got = _step(hhg, ctx, db, qs, q_pav, kind, cs, D, pb, np.roll(ids, k))
            fctx = hhg.Context()
            fdb = _db_of(hhg, fctx, raw)
            want = _step(hhg, fctx, fdb, qs, q_pav, kind, cs, D, pb, np.roll(ids, k))
            fdb.close(); fctx.close()
            assert got == want, (k, kind, cs, D)
            if kind == "batch" and cs == 5:
                ctx.set_query(qs[0][0], qs[0][1])
                with pytest.raises(hhg.capi.HhgError, match="apply_null_model"):
                    hhg.capi.viterbi_search(ctx, db, ids)
    finally:
        db.close(); ctx.close()


def test_staged_pipelines_equal_resident_search(hhg):
    """pipeline.search_staged / search_batch_staged with columnscore 5 (undivided q_p in, divided for the Viterbi
    stage, prefilter on the undivided one) == pipeline.search over the resident raw shard after apply(5), given the
    divided q_p and the undivided q_prefilter_p."""
    from hhsuite_b200 import synth
    qs, raw = _small_case(hhg, 41)
    ctx = hhg.Context()
    rdb = _db_of(hhg, ctx, raw)
    lib = golden()["cs219_lin"]
    bg = synth._PB.astype(np.float32)
    cs_t = [hhg.pipeline.translate_cs219(r[0][0][1:-1], bg, lib) for r in raw]
    Lt = np.array([len(x) for x in cs_t], np.int32)
    cst = hhg.CsDB(ctx, Lt, np.concatenate([[0], np.cumsum(Lt)[:-1]]).astype(np.int64), np.concatenate(cs_t))
    store = hhg.HostStore.from_db(ctx, rdb)
    sdb = hhg.StagedDB(ctx, store, 40, int(rdb.Lh.sum()))
    pb = np.random.default_rng(6).dirichlet(np.ones(20) * 5).astype(np.float32)
    pfk = dict(min_prefilter_hits=12, maxnumdb=30)
    try:
        ctx.set_scwin(9)
        want = []
        for q_p, q_tr, _, q_pav, _ in qs:
            rdb.apply_null_model(None, pb, 5)
            want.append(hhg.pipeline.search(ctx, rdb, cst, hhg.capi.query_local_background(ctx, q_p, pb), q_tr, q_pav,
                                            lib, q_prefilter_p=q_p, altali=2, **pfk))
        for (q_p, q_tr, _, q_pav, _), w in zip(qs, want):
            got = hhg.pipeline.search_staged(ctx, sdb, cst, q_p, q_tr, q_pav, lib, altali=2, columnscore=5, pb=pb, **pfk)
            assert got[0].tolist() == w[0].tolist() and len(w[1]) > 0
            _same_hits(got[1], w[1])
        got = hhg.pipeline.search_batch_staged(ctx, sdb, cst, [(q[0], q[1], q[3]) for q in qs], lib, altali=2,
                                               columnscore=5, pb=pb, **pfk)
        for (ids, hits), w in zip(got, want):
            assert ids.tolist() == w[0].tolist()
            _same_hits(hits, w[1])
    finally:
        sdb.close(); store.close(); cst.close(); rdb.close(); ctx.close()


def test_refused_inputs_change_nothing(hhg):
    """scwin <= 0, column score 5 without pb, column score 4 and query lengths outside [1, 32767] are HHG_EINVAL and
    leave the context and the shard as they were."""
    qs, raw = _small_case(hhg, 51)
    ctx = hhg.Context()
    db = _db_of(hhg, ctx, raw)
    pb = np.random.default_rng(1).dirichlet(np.ones(20) * 5).astype(np.float32)
    try:
        ctx.set_scwin(6)
        db.apply_null_model(None, pb, 5)
        before = db.read_cols(1).tobytes()
        q = hhg.capi.query_local_background(ctx, qs[0][0], pb)
        for D in (0, -1, -(2**31)):
            with pytest.raises(hhg.capi.HhgError):
                ctx.set_scwin(D)
        with pytest.raises(hhg.capi.HhgError):
            db.apply_null_model(qs[0][3], None, 5)
        for cs in (4, 6, -1):
            with pytest.raises(hhg.capi.HhgError):
                db.apply_null_model(qs[0][3], pb, cs)
        hhg.capi.query_set_batch(ctx, [(q, qs[0][1])], q_pav=qs[0][3][None])
        ids = np.arange(5, dtype=np.int32)
        rq = np.zeros(5, np.int32)
        for cs, p in ((5, None), (4, pb)):
            with pytest.raises(hhg.capi.HhgError):
                hhg.capi.viterbi_search_batch(ctx, db, rq, ids, columnscore=cs, pb=p)
        vits = [(1, 1, 1, 1, 1, np.array([0, 1]), np.array([0, 1]))]
        hhg.capi.mac_query_set_batch(ctx, [(q, hhg.capi.log2lin(qs[0][1]))])
        for cs, p in ((5, None), (4, pb)):
            with pytest.raises(hhg.capi.HhgError):
                hhg.capi.mac_realign_batch(ctx, db, [0], [0], vits, None, cs, p)
        for L in (0, 32768):
            p = np.zeros((L + 2, 20), np.float32)
            with pytest.raises(hhg.capi.HhgError):
                hhg.capi.query_local_background(ctx, p, pb)
        # nothing changed: the shard is still prepared (a single search runs) with the same bits, D is still 6
        assert db.read_cols(1).tobytes() == before
        ctx.set_query(q, qs[0][1])
        hhg.capi.viterbi_search(ctx, db, ids)
        assert hhg.capi.query_local_background(ctx, qs[0][0], pb).tobytes() == q.tobytes()
    finally:
        db.close(); ctx.close()
