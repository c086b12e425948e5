"""GPU tests of the alignment -> HMM path (hhg_msa_to_hmm / hhg_db_create_a3m: SURVEY 8a row a10, 8f-1): filter,
sequence weights, emission frequencies, transitions and Neff must equal, bit for bit, what the compiled reference's
Alignment::Read / Compress / Filter / FrequenciesAndTransitions produce on the same host (the position-specific
weights go through the host's RCPPS, see include/hhg.h)."""
import numpy as np
import pytest

from tests import msa_cases
from tests.util import bits

pytestmark = pytest.mark.gpu


def _cmp(got, ref, tag):
    assert (got["L"], got["N_in"], got["N_filtered"]) == (ref["L"], ref["N_in"], ref["N_filtered"]), tag
    assert np.array_equal(got["keep"], ref["keep"]), (tag, "rows kept by the filter")
    if ref["N_filtered"] > 1:
        assert np.array_equal(bits(got["wg"]), bits(ref["wg"])), (tag, "global weights")
    for key in ("f", "tr", "neff_m", "neff_i", "neff_d"):
        a, b = bits(got[key]), bits(ref[key])
        assert np.array_equal(a, b), (tag, key, np.argwhere(a != b)[:4].tolist())
    assert bits(np.float32(got["neff_hmm"])) == bits(np.float32(ref["neff_hmm"])), (tag, got["neff_hmm"], ref["neff_hmm"])
    L = ref["L"]
    want_ss = ref["ss_pred"].astype(np.int32) * 11 + ref["ss_conf"]
    assert np.array_equal(got["ss"][1:L + 1], want_ss[1:L + 1]), (tag, "ss")


def test_hmm_equals_compiled_reference(hhg, gpu_ctx, refshim, tmp_path):
    pb = refshim.pb()
    for k, t in enumerate(msa_cases.texts()):
        path = tmp_path / f"m{k}.a3m"
        path.write_bytes(t)
        ref = refshim.msa_to_hmm(str(path))
        got = hhg.capi.msa_to_hmm(gpu_ctx, t, pb)
        _cmp(got, ref, f"case {k}")


@pytest.mark.parametrize("filt", [(90, 50, 0, -20.0, 0), (70, 0, 30, -20.0, 0), (90, 0, 0, 0.2, 0), (90, 0, 0, -20.0, 8),
                                  (100, 0, 0, -20.0, 0), (50, 30, 20, 0.0, 20), (15, 0, 0, -20.0, 5)])
def test_filter_options(hhg, gpu_ctx, refshim, tmp_path, filt):
    """-id / -cov / -qid / -qsc / -diff of the database filter (max_seqid, coverage, qid, qsc, Ndiff)."""
    pb, S = refshim.pb(), refshim.S()
    mp = hhg.capi.MsaParams.defaults(max_seqid=filt[0], coverage=filt[1], qid=filt[2], qsc=filt[3], Ndiff=filt[4])
    for k, t in enumerate(msa_cases.texts()):
        if k in (5, 8):
            continue
        path = tmp_path / f"m{k}.a3m"
        path.write_bytes(t)
        ref = refshim.msa_to_hmm(str(path), filt=filt)
        got = hhg.capi.msa_to_hmm(gpu_ctx, t, pb, S=S, mp=mp)
        _cmp(got, ref, f"case {k} filter {filt}")


def test_global_weights(hhg, gpu_ctx, refshim, tmp_path):
    """par.wg = 1 (-wg): no sub-alignments, Neff from the column entropies and the weight of the rows present."""
    pb = refshim.pb()
    mp = hhg.capi.MsaParams.defaults(wg=1)
    for k, t in enumerate(msa_cases.texts()):
        path = tmp_path / f"m{k}.a3m"
        path.write_bytes(t)
        ref = refshim.msa_to_hmm(str(path), wg=1)
        got = hhg.capi.msa_to_hmm(gpu_ctx, t, pb, mp=mp)
        _cmp(got, ref, f"case {k} wg=1")


def test_fixed_match_state_rule_cases(hhg, gpu_ctx, refshim, tmp_path):
    """msa_cases.MRULE_CASES: alignments read with -M <percent> / -M first that once differed from the reference."""
    pb, S = refshim.pb(), refshim.S()
    try:
        for k, (t, M, Mg, filt) in enumerate(msa_cases.MRULE_CASES):
            path = tmp_path / f"c{k}.fas"
            path.write_bytes(t)
            refshim.set_M(M, Mg)
            for wg in (0, 1):
                mp = hhg.capi.MsaParams.defaults(M=M, Mgaps=Mg, max_seqid=filt[0], coverage=filt[1], qid=filt[2], qsc=filt[3],
                                                 Ndiff=filt[4], wg=wg)
                _cmp(hhg.capi.msa_to_hmm(gpu_ctx, t, pb, S=S, mp=mp), refshim.msa_to_hmm(str(path), filt=filt, wg=wg),
                     f"case {k} wg={wg}")
    finally:
        refshim.set_M(1, 50)


def test_reciprocal_table_is_the_hosts(hhg, gpu_ctx, refshim):
    """1-sequence sub-alignments put 1/(1*1) = RCPPS(1) into every weight: check the library saw the same value the
    reference build gets from simdf32_rcp on this host."""
    r = refshim.rcp_table(64)
    assert np.isinf(r[0]) and abs(r[1] - 1.0) < 1e-3


def _pack(texts):
    data = b"".join(t + b"\0" for t in texts)
    ln = np.array([len(t) + 1 for t in texts], np.int64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.int64)
    return data, off, ln


@pytest.mark.parametrize("pc", [(2, 1.0, 1.5, 1.0), (2, 0.9, 4.0, 0.7), (3, 1.0, 10.0, 0.5), (0, 1.0, 1.5, 1.0)])
def test_shard_from_a3m_equals_reference_prepared(hhg, gpu_ctx, refshim, tmp_path, pc, monkeypatch):
    """hhg_db_create_a3m: column records and pav == the reference's alignment branch + PrepareTemplateHMM steps.
    The second and fourth parameter set load the records in chunks of three (the loader's multi-chunk path)."""
    from tests.test_hhm_db_gpu import _expected_records
    if pc[0] in (0, 3) or pc[1] != 1.0:
        monkeypatch.setenv("HHG_MSA_CHUNK_RECORDS", "3")
    texts = msa_cases.texts()
    data, off, ln = _pack(texts)
    pp = refshim.prep_params()
    params = hhg.capi.PrepParams(pp.gapb, pp.gapd, pp.gape, pp.gapf, pp.gapg, pp.gaph, pp.gapi, pc[0], pc[1], pc[2], pc[3])
    refshim.set_pc(*pc)
    try:
        db = hhg.TargetDB.from_a3m(gpu_ctx, data, off, ln, refshim.R(), refshim.pb(), params=params)
        cols, pav = db.read_cols(0), db.read_pav()
        pos = 0
        for k, t in enumerate(texts):
            path = tmp_path / f"m{k}.a3m"
            path.write_bytes(t)
            ref = refshim.msa_to_hmm(str(path), prep=True)
            L = ref["L"]
            assert db.Lh[k] == L
            ss = (ref["ss_pred"].astype(np.int32) * 11 + ref["ss_conf"]).astype(np.uint8)
            want = _expected_records(ref["p"], ref["tr_prep"], ss, True)
            got = cols[pos:pos + L]
            assert got.tobytes() == want.tobytes(), (k, pc)
            assert np.array_equal(bits(pav[k]), bits(ref["pav"])), (k, pc)
            pos += L
        db.close()
    finally:
        refshim.set_pc(2, 1.0, 1.5, 1.0)


def test_search_over_a3m_shard(hhg, gpu_ctx, refshim, tmp_path):
    """A shard built from alignments is searchable like any other: hits equal those over a shard made from the
    reference's own prepared arrays of the same alignments."""
    from tests.util import golden
    G = golden()
    texts = msa_cases.texts()[:6]
    data, off, ln = _pack(texts)
    db = hhg.TargetDB.from_a3m(gpu_ctx, data, off, ln, refshim.R(), refshim.pb())
    gpu_ctx.set_query(G["q_p"], G["q_tr"])
    db.apply_null_model(q_pav=G["q_pav"], pb=refshim.pb(), columnscore=1)
    h1, p1 = hhg.viterbi_search(gpu_ctx, db)
    profs = []
    for k, t in enumerate(texts):
        path = tmp_path / f"m{k}.a3m"
        path.write_bytes(t)
        ref = refshim.msa_to_hmm(str(path), prep=True)
        pnul = (0.5 * (G["q_pav"].astype(np.float32) + ref["pav"])).astype(np.float32)
        p = ref["p"].copy()
        p[1:ref["L"] + 1] = (p[1:ref["L"] + 1] / pnul).astype(np.float32)
        profs.append((p, ref["tr_prep"], None))
    db2 = hhg.TargetDB.from_profiles(gpu_ctx, profs)
    h2, p2 = hhg.viterbi_search(gpu_ctx, db2)
    assert np.array_equal(bits(h1["score"]), bits(h2["score"])) and np.array_equal(h1["nsteps"], h2["nsteps"])
    assert np.array_equal(p1, p2)
    db.close(); db2.close()


def test_query_from_alignment(hhg, gpu_ctx, refshim, tmp_path):
    """hhg_query_from_a3m: the query alignment of hhblits -> the arrays hhg_query_set takes, equal to the reference's
    Read / Compress / Filter / FrequenciesAndTransitions + the nocontxt pseudocount steps; then usable as a query."""
    qa = msa_cases.texts()[-1]
    path = tmp_path / "q.a3m"
    path.write_bytes(qa)
    ref = refshim.msa_to_hmm(str(path), prep=True)
    q = hhg.capi.query_from_a3m(gpu_ctx, qa, refshim.R(), refshim.pb())
    L = ref["L"]
    assert q["L"] == L
    assert np.array_equal(bits(q["p"][1:L + 1]), bits(ref["p"][1:L + 1]))
    assert np.array_equal(bits(q["tr"]), bits(ref["tr_prep"])) and np.array_equal(bits(q["pav"]), bits(ref["pav"]))
    assert np.array_equal(bits(q["p"][0]), bits(ref["pav"])) and bits(np.float32(q["neff"])) == bits(np.float32(ref["neff_hmm"]))
    gpu_ctx.set_query(q["p"], q["tr"])
    texts = msa_cases.texts()[:4]
    data, off, ln = _pack(texts)
    db = hhg.TargetDB.from_a3m(gpu_ctx, data, off, ln, refshim.R(), refshim.pb())
    db.apply_null_model(q_pav=q["pav"], pb=refshim.pb(), columnscore=1)
    hits, _ = hhg.viterbi_search(gpu_ctx, db)
    assert len(hits) == 4 and np.all(np.isfinite(hits["score"]))
    db.close()


def test_compressed_alignment_database(hhg, gpu_ctx, refshim, tmp_path):
    """hhg_ca3m_to_hmm / hhg_db_create_ca3m (`_ca3m` + `_sequence` ffindex files, what UniClust ships) against the
    compiled reference's Alignment::ReadCompressed branch of getTemplateHMM."""
    from hhsuite_b200 import ffindex
    from tests.test_hhm_db_gpu import _expected_records
    prefix = msa_cases.ca3m_database(tmp_path)
    sq = ffindex.FFIndex(prefix + "_sequence.ffdata")
    ca = ffindex.FFIndex(prefix + "_ca3m.ffdata")
    seqs = hhg.capi.SeqDb.make(bytes(sq.data), sq.offsets, sq.lengths)
    pb = refshim.pb()
    refs = []
    for k, name in enumerate(ca.names):
        ref = refshim.ca3m_to_hmm(prefix, name, prep=True)
        got = hhg.capi.ca3m_to_hmm(gpu_ctx, bytes(ca.record(k)), seqs, pb)
        _cmp(got, ref, name)
        refs.append(ref)
    db = hhg.TargetDB.from_ca3m(gpu_ctx, bytes(ca.data), ca.offsets, ca.lengths, seqs, refshim.R(), pb)
    cols, pav = db.read_cols(0), db.read_pav()
    pos = 0
    for k, ref in enumerate(refs):
        L = ref["L"]
        want = _expected_records(ref["p"], ref["tr_prep"], np.zeros(L + 2, np.uint8), True)
        assert cols[pos:pos + L].tobytes() == want.tobytes(), k
        assert np.array_equal(bits(pav[k]), bits(ref["pav"])), k
        pos += L
    db.close(); sq.close(); ca.close()


@pytest.mark.parametrize("wg", [0, 1])
def test_large_alignment(hhg, gpu_ctx, refshim, tmp_path, wg):
    """2 500 sequences x 250 columns: many filter passes of the position-dependent schedule, sub-alignment counts
    beyond one byte, long ordered sums."""
    from hhsuite_b200 import synth
    t = synth.a3m_text(250, 2500, 31, ident=0.55, dup_frac=0.2).encode()
    path = tmp_path / "big.a3m"
    path.write_bytes(t)
    ref = refshim.msa_to_hmm(str(path), wg=wg, capL=300, capN=2600)
    got = hhg.capi.msa_to_hmm(gpu_ctx, t, refshim.pb(), mp=hhg.capi.MsaParams.defaults(wg=wg))
    assert ref["N_filtered"] > 100
    _cmp(got, ref, f"large wg={wg}")
