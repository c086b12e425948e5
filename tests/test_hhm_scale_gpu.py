"""GPU tests of the HHM loaders on the record families of tests/hhm_cases.py: the resident shard (hhg_db_create_hhm),
the record-sourced staged shard (hhg_recsrc_create_hhm + hhg_db_stage) and the query (hhg_query_from_hhm) against the
compiled reference bit for bit -- every pseudocount mode, gapb 1 and 0, the whole integer domain of the format, a shard
of more than one 2 000 000-column chunk, records longer than the reference reads (against the oracle), and the
reference's own Viterbi on the family files."""
import os
import subprocess

import numpy as np
import pytest

from tests import hhm_cases as H
from tests.test_hhm_cases_cpu import DEFAULT_PC, PC_IDS, PC_MODES, RefSettings, oracle_params, ref_hhm, ref_record  # noqa: F401
from tests.util import ROOT, bits, golden, ref_data_file

pytestmark = pytest.mark.gpu

NEFF_ZERO = ("no_neff", "neff_zero")


def _pack(texts):
    data = b"".join(t + b"\0" for t in texts)
    ln = np.array([len(t) + 1 for t in texts], np.int64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.int64)
    return data, off, ln


def _pp(pc=DEFAULT_PC, gapb=1.0):
    from hhsuite_b200.capi import PrepParams
    pp = PrepParams.defaults()
    pp.gapb = gapb
    pp.pcm, pp.pca, pp.pcb, pp.pcc = pc
    return pp


def _ss_bytes(text, ref, L):
    """What the loaders write for a record in a shard with secondary structure: the reference's ss_pred / ss_conf where
    HMM::Read sets them, 0 elsewhere, and 0 throughout for a record without ss_pred."""
    from hhsuite_b200 import capi
    out = np.zeros(L, np.uint8)
    if not capi.hhm_scan(text)[1]:
        return out
    npred, nconf = H.ss_defined(text)
    npred, nconf = min(npred, L), min(nconf, L)
    out[:npred] = ref["ss_pred"][1:npred + 1] * 11
    out[:nconf] += ref["ss_conf"][1:nconf + 1]
    return out


def _expected(ref, ss):
    from hhsuite_b200.capi import COLREC_DTYPE
    L, p, tr = ref["L"], ref["p_raw"], ref["tr"]
    r = np.zeros(L, COLREC_DTYPE)
    r["p"] = p[1:L + 1]
    r["m2m"], r["m2d"], r["d2m"], r["d2d"], r["i2m"] = tr[:L, 0], tr[:L, 2], tr[:L, 5], tr[:L, 6], tr[:L, 3]
    r["i2i"], r["m2i"] = tr[1:L + 1, 4], tr[1:L + 1, 1]
    r["ss"] = ss
    return r


def _family_texts(written):
    out = [t for f in H.FAMILIES for (_, _, t) in H.family(f, n=8)]
    out += [H.values(s, L, null=True) for s, L in [(3, 5), (4, 9)]]
    out += [H.variant(50 + k, 23 + k, {v}) for k, v in enumerate(H.VARIANTS)]
    out += [t for k, t in H.NAMED_CASES.items() if k not in NEFF_ZERO]
    return out + [t for _, t in written]


@pytest.fixture(scope="module")
def written(ref_hhm, tmp_path_factory):
    d = tmp_path_factory.mktemp("written")
    return [(f"written{s}{'-pc' if pc else ''}", H.written(ref_hhm, s, L, d, add_pc=pc))
            for s, L in [(0, 40), (1, 75), (2, 12), (3, 160)] for pc in (False, True)]


def _check_shard(hhg, ctx, ref_hhm, texts, pc, gapb, tmp_path):
    data, off, ln = _pack(texts)
    db = hhg.TargetDB.from_hhm(ctx, data, off, ln, ref_hhm.R(), _pp(pc, gapb))
    cols, pav = db.read_cols(0), db.read_pav()
    pos = 0
    with RefSettings(ref_hhm, pc, gapb):
        for k, t in enumerate(texts):
            ref = ref_record(ref_hhm, t, tmp_path / "t.hhm")
            L = ref["L"]
            assert db.Lh[k] == L, k
            want = _expected(ref, _ss_bytes(t, ref, L))
            assert cols[pos:pos + L].tobytes() == want.tobytes(), (k, pc, gapb)
            assert np.array_equal(bits(pav[k]), bits(ref["pav"])), (k, pc, gapb)
            pos += L
    db.close()


@pytest.mark.parametrize("pc", PC_MODES, ids=PC_IDS)
def test_resident_loader_equals_compiled_reference(hhg, gpu_ctx, ref_hhm, written, tmp_path, pc):
    """Every family in one shard (records with and without ss_pred mixed), gapb 1 and 0: every ColRec byte, every pav
    bit, the ss bytes where the reference sets them."""
    ref_hhm.load_query_hhm(ref_data_file("query.hhm", tmp_path))
    texts = _family_texts(written)
    assert any(hhg.capi.hhm_scan(t)[1] for t in texts) and not all(hhg.capi.hhm_scan(t)[1] for t in texts)
    for gapb in (1.0, 0.0):
        _check_shard(hhg, gpu_ctx, ref_hhm, texts, pc, gapb, tmp_path)


@pytest.mark.parametrize("pc,gapb", [((0, 1.0, 1.5, 1.0), 0.0), (DEFAULT_PC, 1.0)], ids=["pcm0-gapb0", "defaults"])
def test_sweep_equals_compiled_reference(hhg, gpu_ctx, ref_hhm, tmp_path, pc, gapb):
    """Every integer 0..99999 and '*' as emission, transition and Neff: with pcm 0 and gapb 0 the values reach the
    records unmixed (fpow2 and the integer -> float conversions on the device over their whole domain)."""
    ref_hhm.load_query_hhm(ref_data_file("query.hhm", tmp_path))
    _check_shard(hhg, gpu_ctx, ref_hhm, H.sweep_records(), pc, gapb, tmp_path)


def test_query_from_hhm_equals_compiled_reference(hhg, gpu_ctx, ref_hhm, written, tmp_path):
    """hhg_query_from_hhm on every family record = HMM::Read + PrepareQueryHMM (nocontxt): p with rows 0 and L+1, the
    transition rows 0..L, pav, ss where the reference sets it, Neff_HMM."""
    with RefSettings(ref_hhm):
        for k, t in enumerate(_family_texts(written)):
            path = tmp_path / "q.hhm"
            path.write_bytes(t)
            ref = ref_hhm.load_query_hhm(str(path))
            got = hhg.capi.query_from_hhm(gpu_ctx, t + b"\0", ref_hhm.R())
            L = got["L"]
            assert L == ref["L"], k
            assert np.array_equal(bits(got["p"]), bits(ref["p"])), k
            assert np.array_equal(bits(got["tr"]), bits(ref["tr"])), k
            assert np.array_equal(bits(got["pav"]), bits(ref["pav"])), k
            assert bits(got["neff"]) == bits(ref["neff"]), k
            if got["has_ss"]:
                assert np.array_equal(got["ss"][1:L + 1], _ss_bytes(t, ref, L)), k


def test_long_records_equal_oracle(hhg, gpu_ctx, oracle):
    """Records of 4 095..32 767 columns, longer than the compiled reference reads, against the oracle (whose agreement
    with the reference the shorter records establish)."""
    G = golden()
    texts = [H.hhmake(900 + k, L) for k, L in enumerate([4095, 9001, 32767])] + [H.values(7, 4099)]
    data, off, ln = _pack(texts)
    db = hhg.TargetDB.from_hhm(gpu_ctx, data, off, ln, G["R"], _pp())
    cols, pav = db.read_cols(0), db.read_pav()
    pos = 0
    for k, t in enumerate(texts):
        rec = oracle.hhm_parse(t, maxL=int(db.Lh[k]) + 2)
        out = oracle.hhm_prepare(rec, oracle.null_to_pb(rec["null"]), G["R"], oracle_params(DEFAULT_PC, 1.0))
        L = out["L"]
        r = {"L": L, "p_raw": out["p"], "tr": out["tr"]}
        ss = out["ss"][1:L + 1] if rec["has_ss"] else np.zeros(L, np.uint8)
        assert cols[pos:pos + L].tobytes() == _expected(r, ss).tobytes(), k
        assert np.array_equal(bits(pav[k]), bits(out["pav"])), k
        pos += L
    db.close()


def _chunked_database(seed=5):
    """About 2.1 M columns from ~150 unique hhmake / values records repeated; one record ends exactly at the first
    2 000 000-column chunk boundary, with runs of L = 1 records on both sides.  Returns (texts, unique texts)."""
    rng = np.random.default_rng(seed)
    uniq = [H.hhmake(5000 + k, int(rng.integers(2, 300))) for k in range(140)]
    uniq += [H.values(s, L) for s, L in enumerate(H.VALUE_LENGTHS)]
    ones = [H.hhmake(6000 + k, 1) for k in range(4)]
    lens = {t: hhg_len(t) for t in uniq + ones}
    order, cum = [], 0
    while cum + 4000 < 2_000_000:
        t = uniq[int(rng.integers(0, len(uniq)))]
        order.append(t); cum += lens[t]
    for k in range(25):
        order.append(ones[k % 4]); cum += 1
    filler = H.hhmake(7000, 2_000_000 - cum)
    order.append(filler); cum += hhg_len(filler)
    assert cum == 2_000_000
    for k in range(30):
        order.append(ones[(k + 1) % 4])
    while cum < 2_100_000:
        t = uniq[int(rng.integers(0, len(uniq)))]
        order.append(t); cum += lens[t]
    return order, uniq + ones + [filler]


def hhg_len(t):
    from hhsuite_b200 import capi
    return capi.hhm_scan(t)[0]


def test_multi_chunk_shard_and_staged_records(hhg, gpu_ctx, ref_hhm, tmp_path):
    """A shard of more than one chunk: every copy of a record equals its first occurrence, the unique records equal the
    reference, and a record-sourced staged shard over the same text (3 000 random ids in two calls) equals the resident
    shard in records, pav and Neff."""
    texts, uniq = _chunked_database()
    data, off, ln = _pack(texts)
    R = ref_hhm.R()
    db = hhg.TargetDB.from_hhm(gpu_ctx, data, off, ln, R, _pp())
    assert int(db.Lh.sum()) > 2_000_000
    cols, pav = db.read_cols(0), db.read_pav()
    coff = np.concatenate([[0], np.cumsum(db.Lh.astype(np.int64))])
    first = {}
    for k, t in enumerate(texts):
        blob = cols[coff[k]:coff[k + 1]].tobytes() + pav[k].tobytes()
        assert first.setdefault(t, blob) == blob, k
    any_ss = any(hhg.capi.hhm_scan(t)[1] for t in texts)
    neff = {}
    ref_hhm.load_query_hhm(ref_data_file("query.hhm", tmp_path))
    with RefSettings(ref_hhm):
        for t in uniq:
            ref = ref_record(ref_hhm, t, tmp_path / "u.hhm")
            L = ref["L"]
            want = _expected(ref, _ss_bytes(t, ref, L) if any_ss else np.zeros(L, np.uint8))
            assert first[t][:L * want.itemsize] == want.tobytes()
            assert first[t][L * want.itemsize:] == ref["pav"].tobytes()
            neff[t] = np.float32(ref["neff_hmm"])
    src = hhg.RecordSource.from_hhm(gpu_ctx, data, off, ln, R, _pp(), has_ss=any_ss)
    rng = np.random.default_rng(11)
    ids = rng.integers(0, len(texts), 3000).astype(np.int32)
    sdb = hhg.StagedDB(gpu_ctx, src, 3000, int(db.Lh[ids].sum()))
    for part in (ids[:1500], ids[1500:]):
        local = sdb.stage(part)
        spav, sneff = sdb.read_pav(), sdb.neff(local)
        for g, s, ne in zip(part, local, sneff):
            assert sdb.read_target(int(s)).tobytes() == cols[coff[g]:coff[g + 1]].tobytes(), g
            assert spav[s].tobytes() == pav[g].tobytes() and bits(ne) == bits(neff[texts[g]]), g
    sdb.close(); src.close(); db.close()


@pytest.mark.parametrize("case", NEFF_ZERO)
def test_loaders_refuse_neff_hmm_zero(hhg, gpu_ctx, case):
    """A record without NEFF / NAA (or with NEFF 0) would get pav NaN: the resident, staged and query loaders refuse it
    by name."""
    G = golden()
    good, bad = H.hhmake(1, 30), H.NAMED_CASES[case]
    data, off, ln = _pack([good, bad])
    with pytest.raises(hhg.HhgError, match="record 1: Neff_HMM is 0"):
        hhg.TargetDB.from_hhm(gpu_ctx, data, off, ln, G["R"], _pp())
    src = hhg.RecordSource.from_hhm(gpu_ctx, data, off, ln, G["R"], _pp())
    sdb = hhg.StagedDB(gpu_ctx, src, 4, 200)
    assert len(sdb.stage([0])) == 1
    with pytest.raises(hhg.HhgError, match="record 1: Neff_HMM is 0"):
        sdb.stage([1])
    sdb.close(); src.close()
    with pytest.raises(hhg.HhgError, match="Neff_HMM is 0"):
        hhg.capi.query_from_hhm(gpu_ctx, bad + b"\0", G["R"])


def test_dropin_on_family_files(written, tmp_path):
    """The reference's own ViterbiRunner reading the family files itself against the GPU adapter whose templates
    hhg_db_create_hhm loaded from the same files: hits on profiles with '*' emissions, Neff 0 columns and PCT."""
    binp = os.path.join(ROOT, "oracle", "_ref", "hh_dropin_check")
    if not os.path.exists(binp):
        pytest.skip("oracle/_ref/hh_dropin_check not built")
    qpath = ref_data_file("query.hhm", tmp_path)

    def run(query, texts, tag):
        files = []
        for k, t in enumerate(texts):
            f = tmp_path / f"{tag}{k}.hhm"
            f.write_bytes(t)
            files.append(str(f))
        r = subprocess.run([binp, "--hhm-loader", query] + files, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and "all hits identical" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]

    plain = [H.hhmake(300 + k, L) for k, L in enumerate([150, 60, 7, 230, 33, 98])]
    plain += [H.values(s, L) for s, L in [(0, 1), (2, 3), (5, 17), (6, 63)]]
    plain += [t for _, t in written]
    run(qpath, plain, "p")
    # the SS set: ss_pred with ss_conf (without it the reference's confidences are uninitialised memory) and, as in the
    # existing SS drop-in sets, no ss_dssp row
    ss = [t for t in (H.hhmake(400 + k, 40 + 7 * k) for k in range(80))
          if b">ss_pred" in t and b">ss_conf" in t and b">ss_dssp" not in t][:8]
    assert len(ss) >= 4
    q = tmp_path / "qss.hhm"
    q.write_bytes(ss[0])
    run(str(q), ss, "s")
