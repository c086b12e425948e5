"""Staged shards whose source is the database's own HHM, A3M or compressed-A3M records (hhg_recsrc_*,
hhg_db_create_staged_records, hhg_db_stage building the survivors from their records, hhg_db_staged_neff).  A
record-sourced shard must be indistinguishable from the resident shard of the same records and from a store-backed
staged shard fed the same ids: records, pav and Neff byte for byte; local ids, statistics and evictions; hits, paths
and realigned paths of the pipeline; and the refusals leave the shard and the context usable."""
import dataclasses

import numpy as np
import pytest

from hhsuite_b200 import synth
from tests import msa_cases
from tests.test_hhm_db_gpu import _pack, _pp
from tests.test_staged_db_gpu import _same_hits, _same_runner_hits
from tests.util import bits, golden

pytestmark = pytest.mark.gpu


def _a3m_records(n, seed, lo=5, hi=150):
    rng = np.random.default_rng(seed)
    return [synth.a3m_text(int(L), int(rng.integers(2, 14)), seed * 1000 + k, f"a{k}", with_ss=k % 3 == 0).encode()
            for k, L in enumerate(rng.integers(lo, hi, n))]


def _a2m(text):
    """An alignment whose rows all have the same number of columns (inserts dropped): what -M 2 / -M first read."""
    return b"\n".join(ln if ln[:1] in (b">", b"#") else bytes(c for c in ln if not (97 <= c <= 122 or c == 46))
                      for ln in text.split(b"\n"))


def _hhm_records(n, seed):
    rng = np.random.default_rng(seed)
    return [synth.hhm_text(int(L), seed * 1000 + k, f"h{k}", with_ss=k % 2 == 0).encode()
            for k, L in enumerate(rng.integers(1, 300, n))]


def _S():
    return np.random.default_rng(8).normal(0, 1.5, (20, 20)).astype(np.float32)


def _expect_same(sdb, local, ids, resident, has_ss):
    """Every staged target equals the resident shard's record of the same id (ss bytes zeroed without has_ss)."""
    cols, pav, L = resident.read_cols(0), resident.read_pav(), resident.Lh
    off = np.concatenate([[0], np.cumsum(L.astype(np.int64))])
    spav = sdb.read_pav()
    g, _ = sdb.lookup(local)
    assert g.tolist() == [int(t) for t in ids]
    for t, s in zip(ids, local):
        want = cols[off[t]:off[t + 1]].copy()
        if not has_ss:
            want["ss"] = 0
        assert sdb.Lh[s] == L[t]
        assert sdb.read_target(int(s)).tobytes() == want.tobytes(), t
        assert spav[s].tobytes() == pav[t].tobytes(), t


# ------------------------------------------------------------------------------------------------ 1. records
A3M_CASES = [  # (pcm, pcc, M, wg, qsc, has_ss)
    (0, 1.0, 1, 0, -20.0, True), (1, 1.0, 1, 0, -20.0, False), (2, 1.0, 1, 0, -20.0, True), (3, 1.0, 1, 1, -20.0, True),
    (2, 0.6, 1, 0, -20.0, True), (2, 1.0, 2, 0, -20.0, True), (2, 1.0, 3, 1, -20.0, False), (2, 1.0, 1, 0, 0.0, True),
]


@pytest.mark.parametrize("case", A3M_CASES)
def test_a3m_records(hhg, gpu_ctx, case):
    pcm, pcc, M, wg, qsc, has_ss = case
    G = golden()
    pp = _pp(G)
    pp.pcm, pp.pcc = pcm, pcc
    mp = hhg.capi.MsaParams.defaults(M=M, wg=wg, qsc=qsc)
    S = _S() if qsc > -10 else None
    recs = _a3m_records(60, 3 + pcm)
    if M != 1:
        recs = [_a2m(r) for r in recs]
    data, off, ln = _pack(recs)
    resident = hhg.TargetDB.from_a3m(gpu_ctx, data, off, ln, G["R"], G["pb"], S=S, params=pp, mp=mp)
    src = hhg.RecordSource.from_a3m(gpu_ctx, data, off, ln, G["R"], G["pb"], S=S, params=pp, mp=mp, has_ss=has_ss)
    assert src.n == 60
    sdb = hhg.StagedDB(gpu_ctx, src, 60, int(resident.Lh.sum()))
    ids = np.random.default_rng(1).permutation(60)[:45]
    local = sdb.stage(np.concatenate([ids, ids[:5]]))[:45]
    _expect_same(sdb, local, ids, resident, has_ss)
    want = [hhg.capi.msa_to_hmm(gpu_ctx, recs[t], G["pb"], S=S, mp=mp)["neff_hmm"] for t in ids]
    assert bits(sdb.neff(local)).tolist() == bits(np.array(want, np.float32)).tolist()
    with pytest.raises(hhg.HhgError, match="still use the record source"):
        src.close()
    sdb.close(); src.close(); resident.close()


@pytest.mark.parametrize("pcm,pcc,has_ss", [(0, 1.0, True), (1, 1.0, True), (2, 1.0, False), (3, 1.0, True), (2, 0.6, True)])
def test_hhm_records(hhg, gpu_ctx, pcm, pcc, has_ss):
    G = golden()
    pp = _pp(G)
    pp.pcm, pp.pcc = pcm, pcc
    recs = _hhm_records(50, 11 + pcm)
    data, off, ln = _pack(recs)
    resident = hhg.TargetDB.from_hhm(gpu_ctx, data, off, ln, G["R"], pp)
    src = hhg.RecordSource.from_hhm(gpu_ctx, data, off, ln, G["R"], pp, has_ss=has_ss)
    sdb = hhg.StagedDB(gpu_ctx, src, 50, int(resident.Lh.sum()))
    ids = np.random.default_rng(2).permutation(50)
    local = sdb.stage(ids)
    _expect_same(sdb, local, ids, resident, has_ss)
    want = np.array([hhg.capi.hhm_parse(recs[t])["neff_hmm"] for t in ids], np.float32)
    assert bits(sdb.neff(local)).tolist() == bits(want).tolist()
    sdb.close(); src.close(); resident.close()


def test_ca3m_records(hhg, gpu_ctx, tmp_path):
    from hhsuite_b200 import ffindex
    G = golden()
    rng = np.random.default_rng(4)
    alis = [(f"c{k}", synth.a3m_text(int(L), 8, 500 + k, f"c{k}")) for k, L in enumerate(rng.integers(5, 120, 40))]
    prefix = msa_cases.ca3m_database(tmp_path, alis)
    sq = ffindex.FFIndex(prefix + "_sequence.ffdata")
    ca = ffindex.FFIndex(prefix + "_ca3m.ffdata")
    seqs = hhg.capi.SeqDb.make(bytes(sq.data), sq.offsets, sq.lengths)
    data = bytes(ca.data)
    resident = hhg.TargetDB.from_ca3m(gpu_ctx, data, ca.offsets, ca.lengths, seqs, G["R"], G["pb"])
    src = hhg.RecordSource.from_ca3m(gpu_ctx, data, ca.offsets, ca.lengths, seqs, G["R"], G["pb"], has_ss=True)
    sdb = hhg.StagedDB(gpu_ctx, src, 40, int(resident.Lh.sum()))
    ids = rng.permutation(40)
    local = sdb.stage(ids)
    _expect_same(sdb, local, ids, resident, True)
    want = [hhg.capi.ca3m_to_hmm(gpu_ctx, bytes(ca.record(int(t))), seqs, G["pb"])["neff_hmm"] for t in ids]
    assert bits(sdb.neff(local)).tolist() == bits(np.array(want, np.float32)).tolist()
    sdb.close(); src.close(); resident.close()


# ------------------------------------------------------------------------------------------------ 2. churn
def test_churn_against_store(hhg, gpu_ctx, monkeypatch):
    """Requests over a shard far smaller than the database, with evictions and one forced re-layout: after every call
    each staged target equals the resident record, and local ids / statistics equal a store-backed shard's.  Groups
    of 7 records make every call build in several groups."""
    monkeypatch.setenv("HHG_MSA_CHUNK_RECORDS", "7")
    G = golden()
    recs = _a3m_records(160, 21, lo=20, hi=120)
    data, off, ln = _pack(recs)
    resident = hhg.TargetDB.from_a3m(gpu_ctx, data, off, ln, G["R"], G["pb"])
    L = resident.Lh.copy()
    store = hhg.HostStore.from_db(gpu_ctx, resident, has_ss=True)
    src = hhg.RecordSource.from_a3m(gpu_ctx, data, off, ln, G["R"], G["pb"], has_ss=True)
    # the re-layout: ten targets fill the arena, the even ones are named again, then the even ones and one target
    # longer than any odd run but no longer than the odd runs together
    order = np.argsort(L, kind="stable")
    ten = order[40:50]
    odd = ten[1::2]
    big = next(int(t) for t in order[::-1] if L[odd].max() < L[t] <= L[odd].sum() and t not in ten)
    cols = int(L[ten].sum())
    seq = [ten, ten[0::2], np.append(ten[0::2], big)]
    rng = np.random.default_rng(9)
    for _ in range(8):
        ids = rng.choice(160, 12, replace=False)
        keep = np.cumsum(L[ids]) <= cols
        seq.append(np.concatenate([ids[keep], ids[keep][:2]]))
    shards = [hhg.StagedDB(gpu_ctx, x, 12, cols) for x in (store, src)]
    evicted = 0
    for k, ids in enumerate(seq):
        ids = np.asarray(ids, np.int32)
        locs = [s.stage(ids) for s in shards]
        assert locs[0].tolist() == locs[1].tolist(), k
        assert shards[0].last_stats.tobytes() == shards[1].last_stats.tobytes(), k
        if k == 2:
            assert shards[1].last_stats["copied"] == 6                # the re-layout copied all of the request's targets
        evicted += int(shards[1].last_stats["evicted"])
        _expect_same(shards[1], locs[1], ids, resident, True)
        assert np.array_equal(shards[0].Lh, shards[1].Lh)
    assert evicted > 12
    assert shards[0].lookup(np.arange(12))[0].tolist() == shards[1].lookup(np.arange(12))[0].tolist()
    for s in shards:
        s.close()
    src.close(); store.close(); resident.close()


def test_forced_relayout_rebuilds(hhg, gpu_ctx):
    """The request's own residents fragment the arena: all of them are built again from their records, bit-identical."""
    G = golden()
    recs = _a3m_records(80, 23, lo=20, hi=120)
    data, off, ln = _pack(recs)
    resident = hhg.TargetDB.from_a3m(gpu_ctx, data, off, ln, G["R"], G["pb"])
    L = resident.Lh
    order = np.argsort(L, kind="stable")
    ten = order[20:30]
    odd = ten[1::2]
    big = next(int(t) for t in order[::-1] if L[odd].max() < L[t] <= L[odd].sum() and t not in ten)
    src = hhg.RecordSource.from_a3m(gpu_ctx, data, off, ln, G["R"], G["pb"], has_ss=True)
    sdb = hhg.StagedDB(gpu_ctx, src, 16, int(L[ten].sum()))
    sdb.stage(ten)
    sdb.stage(ten[0::2])
    ids = np.append(ten[0::2], big).astype(np.int32)
    local = sdb.stage(ids)
    st = sdb.last_stats
    assert (st["hits"], st["copied"], st["evicted"]) == (0, 6, 5)
    _expect_same(sdb, local, ids, resident, True)
    assert bits(sdb.neff(local)).tolist() == bits(np.array(
        [hhg.capi.msa_to_hmm(gpu_ctx, recs[t], G["pb"])["neff_hmm"] for t in ids], np.float32)).tolist()
    sdb.close(); src.close(); resident.close()


# ------------------------------------------------------------------------------------------------ 3. searches
def test_searches(hhg):
    """search_staged, search_batch_staged and mac.realign over a record source == over a store-backed shard == over
    the resident shard: survivors, every Hit field and path, and every realigned path."""
    G = golden()
    lib = G["cs219_lin"]
    bg = synth._PB.astype(np.float32)
    ctx = hhg.Context()
    recs = _a3m_records(600, 31, lo=20, hi=200)
    data, off, ln = _pack(recs)
    resident = hhg.TargetDB.from_a3m(ctx, data, off, ln, G["R"], G["pb"])
    L = resident.Lh.copy()
    cols = resident.read_cols(0)
    offs = np.concatenate([[0], np.cumsum(L.astype(np.int64))])
    cs = np.concatenate([hhg.pipeline.translate_cs219(cols["p"][offs[t]:offs[t + 1]], bg, lib) for t in range(len(L))])
    cst = hhg.CsDB(ctx, L, offs[:-1].astype(np.int64), cs)
    store = hhg.HostStore.from_db(ctx, resident, has_ss=True)
    src = hhg.RecordSource.from_a3m(ctx, data, off, ln, G["R"], G["pb"], has_ss=True)
    staged = [hhg.StagedDB(ctx, x, 600, int(L.sum())) for x in (store, src)]
    qs = []
    for t in (3, 50, 222, 404):
        q = hhg.capi.query_from_a3m(ctx, recs[t], G["R"], G["pb"])
        qs.append((q["p"], q["tr"], q["pav"]))
    pfk = dict(min_prefilter_hits=100, maxnumdb=150)
    for k, q in enumerate(qs):
        resident.apply_null_model(q[2])
        want = hhg.pipeline.search(ctx, resident, cst, *q, lib, altali=2, **pfk)
        mac_want = hhg.mac.realign(ctx, resident, q[0], q[1], want[1])
        for sdb in staged:
            ids, hits = hhg.pipeline.search_staged(ctx, sdb, cst, *q, lib, altali=2, **pfk)
            assert ids.tolist() == want[0].tolist()
            _same_runner_hits(hits, want[1], ("single", k))
            local = dict(zip(ids.tolist(), sdb.stage(ids).tolist()))
            assert sdb.last_stats["copied"] == 0
            lh = [dataclasses.replace(h, target=local[h.target]) for h in hits]
            got = hhg.mac.to_global(sdb, hhg.mac.realign(ctx, sdb, q[0], q[1], lh))
            assert sorted(got) == sorted(mac_want)
            for key, m in mac_want.items():
                g = got[key]
                for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols"):
                    assert getattr(g, f) == getattr(m, f), (k, key, f)
                assert bits(g.sum_of_probs) == bits(m.sum_of_probs)
                for f in ("i", "j", "states"):
                    assert np.array_equal(getattr(g, f), getattr(m, f)), (k, key, f)
    outs = [hhg.pipeline.search_batch_staged(ctx, sdb, cst, qs, lib, altali=2, **pfk) for sdb in staged]
    for k in range(len(qs)):
        assert outs[0][k][0].tolist() == outs[1][k][0].tolist()
        _same_runner_hits(outs[1][k][1], outs[0][k][1], ("batch", k))
    # the neff of the staged survivors is what a caller needs for E-values
    ids = outs[1][0][0]
    nf = staged[1].neff(staged[1].stage(ids))
    assert bits(nf).tolist() == bits(np.array([hhg.capi.msa_to_hmm(ctx, recs[t], G["pb"])["neff_hmm"] for t in ids],
                                              np.float32)).tolist()
    with pytest.raises(hhg.HhgError, match="store of packed records"):
        staged[0].neff(staged[0].stage(ids[:1]))
    # index alignment: a cs219 shard of another size is refused up front, a length mismatch after staging
    small = hhg.CsDB(ctx, L[:-1], offs[:-2].astype(np.int64), cs[:offs[-2]])
    with pytest.raises(ValueError, match="index-aligned"):
        hhg.pipeline.search_staged(ctx, staged[1], small, *qs[0], lib, **pfk)
    L2 = L.copy(); L2[[3, 50, 222, 404]] += 1
    o2 = np.concatenate([[0], np.cumsum(L2.astype(np.int64))])
    wrong = hhg.CsDB(ctx, L2, o2[:-1].astype(np.int64),
                     np.concatenate([np.append(cs[offs[t]:offs[t + 1]], cs[offs[t]:offs[t] + 1]) if L2[t] != L[t]
                                     else cs[offs[t]:offs[t + 1]] for t in range(len(L))]))
    with pytest.raises(ValueError, match="index-aligned"):
        hhg.pipeline.search_staged(ctx, staged[1], wrong, *qs[0], lib, **pfk)
    for s in staged:
        s.close()
    for x in (src, store, cst, small, wrong, resident):
        x.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ 4. refusals
def test_refusals(hhg, gpu_ctx):
    G = golden()
    recs = _a3m_records(30, 41)
    recs[12] = b">only a header line\n"
    recs[20] = synth.a3m_text(32768, 2, 7, "long").encode()
    data, off, ln = _pack(recs)
    mp = hhg.capi.MsaParams.defaults(maxres=40000, maxcol=40000)     # the parser takes 32 768 columns
    good = [t for t in range(30) if t not in (12, 20)]
    resident = hhg.TargetDB.from_a3m(gpu_ctx, *_pack([recs[t] for t in good]), G["R"], G["pb"], mp=mp)
    src = hhg.RecordSource.from_a3m(gpu_ctx, data, off, ln, G["R"], G["pb"], mp=mp, has_ss=True)
    Lg = dict(zip(good, resident.Lh.tolist()))
    first = good[:6]
    cap = sum(Lg[t] for t in first)
    sdb = hhg.StagedDB(gpu_ctx, src, 6, cap)
    local = sdb.stage(first)
    before = (sdb.Lh.copy(), sdb.lookup(np.arange(6))[0].tolist())

    def unchanged():
        assert np.array_equal(sdb.Lh, before[0]) and sdb.lookup(np.arange(6))[0].tolist() == before[1]

    n0 = gpu_ctx.launches
    for ids, msg in (([first[0], good[7], 12, good[8]], "record 12: "), ([good[7], 20], "record 20: length 32768"),
                     ([first[1], 30], "target id 30 outside the record source"),
                     ([first[1], -1], "target id -1 outside the record source"),
                     (good[:7], f"needs 7 slots and {cap + Lg[good[6]]} columns")):
        with pytest.raises(hhg.HhgError, match=msg):
            sdb.stage(np.array(ids, np.int32))
        unchanged()
    assert gpu_ctx.launches == n0
    # the next stage and search are correct
    ids = np.array(good[4:10], np.int32)
    local = sdb.stage(ids)
    pos = {t: k for k, t in enumerate(good)}
    q = hhg.capi.query_from_a3m(gpu_ctx, recs[good[5]], G["R"], G["pb"])
    hhg.capi.query_set_batch(gpu_ctx, [(q["p"], q["tr"])], q_pav=q["pav"][None])
    rq = np.zeros(6, np.int32)
    _same_hits(hhg.capi.viterbi_search_batch(gpu_ctx, sdb, rq, local),
               hhg.capi.viterbi_search_batch(gpu_ctx, resident, rq, np.array([pos[t] for t in ids], np.int32)))
    with pytest.raises(hhg.HhgError, match="still use the record source"):
        src.close()
    with pytest.raises(hhg.HhgError, match="out of range"):
        sdb.neff([6])
    empty = hhg.StagedDB(gpu_ctx, src, 2, 100)
    with pytest.raises(hhg.HhgError, match="is empty"):
        empty.neff([0])
    empty.close(); sdb.close(); src.close(); resident.close()
