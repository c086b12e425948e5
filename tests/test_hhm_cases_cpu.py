"""CPU tests of the HHM reader on the record families of tests/hhm_cases.py: the families really contain their features,
the oracle's restatement of HMM::Read + PrepareTemplateHMM equals the compiled reference on them (every pseudocount
mode, gapb 1 and 0), and the product's host tokeniser equals the oracle.  The named cases pin the divergences found."""
import numpy as np
import pytest

from tests import hhm_cases as H
from tests.util import bits, ref_data_file

PC_MODES = [(0, 1.0, 1.5, 1.0), (1, 0.35, 1.5, 1.0), (2, 1.0, 1.5, 1.0), (3, 1.0, 12.0, 0.3), (2, 1.0, 1.5, 0.6),
            (2, 0.9, 2.0, 1.7)]
PC_IDS = ["pcm0", "pcm1", "pcm2", "pcm3", "pcm2-pcc0.6", "pcm2-pcc1.7"]
DEFAULT_PC = (2, 1.0, 1.5, 1.0)


def generated():
    """(name, text) of every generated family record, the sweep records and the named cases."""
    out = [(f"{fam}{s}", t) for fam in H.FAMILIES for (s, L, t) in H.family(fam, n=8)]
    out += [(f"values-null{s}", H.values(s, L, null=True)) for s, L in [(3, 5), (4, 9)]]
    out += [(f"variant-{v}", H.variant(50 + k, 23 + k, {v})) for k, v in enumerate(H.VARIANTS)]
    out += [(f"sweep{k}", t) for k, t in enumerate(H.sweep_records())]
    out += [(f"named-{k}", t) for k, t in H.NAMED_CASES.items()]
    return out


@pytest.fixture(scope="session")
def ref_hhm(refshim):
    """The compiled reference with the shim's HHM entry points (write_hhm, read_hhm_header, set_gap, set_pb); a shim
    built by an older recipe lacks them and these comparisons skip, like every comparison without oracle/_ref."""
    if not refshim.provides(*refshim.HHM_FAMILY_ENTRY_POINTS):
        pytest.skip("oracle/_ref was built without the HHM entry points of oracle/ref_shim.cpp; rebuild it")
    return refshim


@pytest.fixture(scope="module")
def written_records(ref_hhm, tmp_path_factory):
    d = tmp_path_factory.mktemp("written")
    return [(f"written{s}{'-pc' if pc else ''}", H.written(ref_hhm, s, L, d, add_pc=pc))
            for s, L in [(0, 40), (1, 75), (2, 12), (3, 160)] for pc in (False, True)]


class RefSettings:
    """Pseudocount / gap settings and the background pb of the compiled reference, put back on exit."""

    def __init__(self, ref_hhm, pc=DEFAULT_PC, gapb=1.0):
        self.r, self.pc, self.gapb = ref_hhm, pc, gapb

    def __enter__(self):
        self.pb = self.r.pb()
        self.r.set_pc(*self.pc)
        self.r.set_gap(gapb=self.gapb)
        return self

    def __exit__(self, *exc):
        self.r.set_pc(*DEFAULT_PC)
        self.r.set_gap()
        self.r.set_pb(self.pb)


def ref_record(ref_hhm, text, path):
    """The compiled reference on one record file: p_raw, tr, pav, Neff_HMM, has_pc and ss (0 where undefined)."""
    with open(path, "wb") as fh:
        fh.write(text)
    ref = ref_hhm.prepare_template_hhm_raw(str(path))
    _, ref["neff_hmm"], ref["has_pc"] = ref_hhm.read_hhm_header(str(path))
    full = ref_hhm.prepare_template_hhm(str(path))
    ref["ss_pred"], ref["ss_conf"] = full["ss_pred"], full["ss_conf"]
    return ref


def same_ss(got, ref, text):
    """ss bytes (pred * 11 + conf) of columns 1..L equal the reference's ss_pred / ss_conf where it sets them
    (hhm_cases.ss_defined); ref: dict with ss_pred / ss_conf of rows 0..L+1."""
    npred, nconf = H.ss_defined(text)
    got = np.asarray(got)
    return (np.array_equal(got[:npred] // 11, ref["ss_pred"][1:npred + 1]) and
            np.array_equal(got[:nconf] % 11, ref["ss_conf"][1:nconf + 1]))


def oracle_params(pc, gapb):
    from oracle.binding import PrepParams
    return PrepParams(gapb, 0.15, 1.0, 0.6, 0.6, 0.6, 0.6, *pc)


# ------------------------------------------------------------------------------------------------ family self-check
def _lines(t):
    return t.replace(b"\r\n", b"\n").split(b"\n")


def _emission_tokens(t):
    toks = []
    lines = _lines(t)
    k = next(i for i, l in enumerate(lines) if l.startswith(b"HMM "))
    for l in lines[k + 3:]:
        if l[:1].isalpha() or l[:1] in (b"-",):
            toks += l.split()[2:22]
    return toks


def test_families_contain_their_features():
    fam = {f: [t for (_, _, t) in H.family(f, n=8)] for f in H.FAMILIES}
    mk = fam["hhmake"]
    em = [tok for t in mk for tok in _emission_tokens(t)]
    assert em.count(b"*") > len(em) // 4
    assert any(b"\t0\t" + b"\t".join([b"*"] * 5) in t or b" 0\t*" in t for t in mk)           # one-hot columns
    assert any(b" " + b"\t".join([b"*"] * 20) + b"\t" in t for t in mk)                          # all-'*' columns
    assert all(b"\n       0\t*\t*\t0\t*\t0\t*\t" in t for t in mk)                                # hhmake's start row
    assert sum(t.count(b"\t0\t*\t0\t*\t") for t in mk) > 20                                       # Neff_I = 0 with '*'
    for key in (b">ss_dssp", b">sa_dssp", b">ss_pred", b">ss_conf", b">Consensus", b"COM   ", b"DATE  ", b"FILT  "):
        assert any(key in t for t in mk), key
    assert any(max(len(l) for l in _lines(t)[:40] if not l.startswith(b"COM")) == 100 for t in mk)   # wrapped at 100
    var = {v: H.variant(1, 30, {v}) for v in H.VARIANTS}
    assert b"\nNAA   " in var["naa"] and b"\nNEFF " in var["neff_one_space"] and b"\nNEFF  " not in var["neff_one_space"]
    assert b"\nEVD " in var["evd_desc"] and b"\nDESC " in var["evd_desc"]
    assert var["crlf"].count(b"\r\n") > 60 and b" \t \n" in var["trailing_blanks"]
    assert b"\n\n" not in var["no_gap_lines"].split(b"\nHMM ")[1]
    assert b"\t-" in var["negative_ints"] and var["no_final_newline"].endswith(b"//")
    assert b"\0" in var["nul_garbage"] and b"SEQ\n#" in var["empty_seq"]
    assert var["conf_before_pred"].index(b">ss_conf") < var["conf_before_pred"].index(b">ss_pred")
    assert var["second_pred"].count(b">ss_pred") == 2
    assert b">ss_pred" in var["pred_only"] and b">ss_conf" not in var["pred_only"]
    assert b">ss_conf" in var["conf_only"] and b">ss_pred" not in var["conf_only"]
    odd = var["ss_odd_letters"].split(b">ss_pred\n")[1].split(b">")[0]
    assert all(c in odd for c in b"h~ISTGB.Q")
    vals = fam["values"]
    assert sum(t.count(b"PCT   true") for t in vals) >= 3 and sorted({int(t.split(b"LENG  ")[1].split()[0]) % 4 for t in vals}) == [0, 1, 2, 3]
    assert {1, 2, 3} <= {int(t.split(b"LENG  ")[1].split()[0]) for t in [H.values(s, L) for s, L in enumerate(H.VALUE_LENGTHS)]}
    assert b"NULL   " in H.values(3, 5, null=True) and b"\t*\t" in H.values(3, 5, null=True).split(b"NULL")[1].split(b"\n")[0] + b"\t"
    sw = H.sweep_records()
    assert max(int(t.split(b"LENG  ")[1].split()[0]) for t in sw) <= H.MAXREF
    em = {tok for t in sw for tok in _emission_tokens(t)}
    assert len(em) == 100001                                        # 0..99999 and '*'
    rows = [l.split() for t in sw for l in _lines(t) if l.startswith(b"       ") and not l.strip().startswith(b"M->M")]
    assert len({tok for r in rows for tok in r}) == 100001


# ------------------------------------------------------------------------------------------ oracle vs the reference
@pytest.mark.parametrize("gapb", [1.0, 0.0], ids=["gapb1", "gapb0"])
@pytest.mark.parametrize("pc", PC_MODES, ids=PC_IDS)
def test_oracle_equals_compiled_reference(oracle, ref_hhm, written_records, tmp_path, pc, gapb):
    ref_hhm.load_query_hhm(ref_data_file("query.hhm", tmp_path))
    R = ref_hhm.R()
    recs = generated() + written_records
    if not (pc == DEFAULT_PC and gapb == 1.0):
        recs = [r for r in recs if not r[0].startswith("sweep")]   # the sweep runs with two settings below
    with RefSettings(ref_hhm, pc, gapb):
        for name, t in recs:
            ref = ref_record(ref_hhm, t, tmp_path / "t.hhm")
            rec = oracle.hhm_parse(t, maxL=ref["L"] + 2)
            out = oracle.hhm_prepare(rec, oracle.null_to_pb(rec["null"]), R, oracle_params(pc, gapb))
            L = out["L"]
            assert L == ref["L"], name
            assert np.array_equal(bits(out["p"][1:L + 1]), bits(ref["p_raw"][1:L + 1])), name
            assert np.array_equal(bits(out["tr"]), bits(ref["tr"])), name
            assert np.array_equal(bits(out["pav"]), bits(ref["pav"])), name
            assert bits(rec["neff_hmm"]) == bits(ref["neff_hmm"]) and rec["has_pc"] == ref["has_pc"], name
            assert same_ss(out["ss"][1:L + 1], ref, t), name


@pytest.mark.parametrize("pc,gapb", [((0, 1.0, 1.5, 1.0), 0.0)], ids=["pcm0-gapb0"])
def test_oracle_equals_compiled_reference_on_the_sweep(oracle, ref_hhm, tmp_path, pc, gapb):
    """Unmixed: p = fpow2(-x/1000) and tr = -x/1000 for every integer the file format can hold."""
    ref_hhm.load_query_hhm(ref_data_file("query.hhm", tmp_path))
    with RefSettings(ref_hhm, pc, gapb):
        for k, t in enumerate(H.sweep_records()):
            ref = ref_record(ref_hhm, t, tmp_path / "s.hhm")
            rec = oracle.hhm_parse(t, maxL=ref["L"] + 2)
            out = oracle.hhm_prepare(rec, oracle.null_to_pb(rec["null"]), ref_hhm.R(), oracle_params(pc, gapb))
            L = out["L"]
            assert np.array_equal(bits(out["p"][1:L + 1]), bits(ref["p_raw"][1:L + 1])), k
            assert np.array_equal(bits(out["tr"]), bits(ref["tr"])) and np.array_equal(bits(out["pav"]), bits(ref["pav"])), k


# ------------------------------------------------------------------------------------------ tokeniser vs the oracle
def _tokeniser_equals_oracle(oracle, name, t):
    from hhsuite_b200 import capi
    b = oracle.hhm_parse(t, maxL=capi.hhm_scan(t)[0] + 2)
    if b["neff_hmm"] == 0:
        with pytest.raises(capi.HhgError, match="Neff_HMM is 0"):
            capi.hhm_parse(t)
        return
    a = capi.hhm_parse(t)
    L = a["L"]
    assert L == b["L"] and a["has_ss"] == b["has_ss"] and a["has_pc"] == b["has_pc"], name
    assert bits(a["neff_hmm"]) == bits(b["neff_hmm"]), name
    assert np.array_equal(a["f"], b["f"][1:L + 1]) and np.array_equal(a["tr"], b["tr"]), name
    nb = b["neff"].copy()
    nb[1:, 0] = np.where(nb[1:, 0] == 0, 1000, nb[1:, 0])
    assert np.array_equal(a["neff"], nb) and np.array_equal(a["null"], b["null"]), name
    assert np.array_equal(a["ss"], b["ss"][1:L + 1] if b["has_ss"] else np.zeros(L, np.uint8)), name


def test_product_tokeniser_equals_oracle_on_every_family(oracle):
    for name, t in generated():
        _tokeniser_equals_oracle(oracle, name, t)


def test_product_tokeniser_equals_oracle_on_written_records(oracle, written_records):
    assert any(b"PCT   true" in t for _, t in written_records) and any(b">ss_pred" in t for _, t in written_records)
    for name, t in written_records:
        _tokeniser_equals_oracle(oracle, name, t)


# ------------------------------------------------------------------------------------------------------ named cases
def test_named_naa_line_sets_neff_hmm(oracle):
    from hhsuite_b200 import capi
    t = H.NAMED_CASES["naa_line"]
    assert capi.hhm_parse(t)["neff_hmm"] == np.float32(4.7)
    assert oracle.hhm_parse(t)["neff_hmm"] == np.float32(4.7)


@pytest.mark.parametrize("case", ["no_neff", "neff_zero"])
def test_named_neff_hmm_zero_is_refused(case):
    from hhsuite_b200 import capi
    with pytest.raises(capi.HhgError, match="Neff_HMM is 0"):
        capi.hhm_parse(H.NAMED_CASES[case])


def test_named_neff_line_without_number_keeps_value(oracle):
    from hhsuite_b200 import capi
    t = H.NAMED_CASES["neff_then_empty_neff"]
    assert capi.hhm_parse(t)["neff_hmm"] == np.float32(6.2) == oracle.hhm_parse(t)["neff_hmm"]


def test_named_secondary_structure_rows():
    """ss_conf alone: no secondary structure; ss_pred alone: confidence 0 (the reference leaves it unset)."""
    from hhsuite_b200 import capi
    a = capi.hhm_parse(H.NAMED_CASES["conf_only"])
    assert not a["has_ss"] and not a["ss"].any()
    b = capi.hhm_parse(H.NAMED_CASES["pred_only"])
    assert b["has_ss"] and np.array_equal(b["ss"] % 11, np.zeros(20)) and np.array_equal(b["ss"][:3] // 11, [1, 2, 3])


def test_named_cases_against_compiled_reference(ref_hhm, tmp_path):
    """Neff_HMM of the NAA record is the reference's; without NEFF/NAA the reference's pav is NaN (what the loaders
    refuse); ss_conf alone gives the reference no ss_pred."""
    from hhsuite_b200 import capi
    ref_hhm.load_query_hhm(ref_data_file("query.hhm", tmp_path))
    with RefSettings(ref_hhm):
        ref = ref_record(ref_hhm, H.NAMED_CASES["naa_line"], tmp_path / "n.hhm")
        assert bits(ref["neff_hmm"]) == bits(capi.hhm_parse(H.NAMED_CASES["naa_line"])["neff_hmm"])
        for case in ("no_neff", "neff_zero"):
            ref = ref_record(ref_hhm, H.NAMED_CASES[case], tmp_path / "z.hhm")
            assert ref["neff_hmm"] == 0 and np.isnan(ref["pav"]).all()
        ref = ref_record(ref_hhm, H.NAMED_CASES["conf_only"], tmp_path / "c.hhm")
        assert not ref["ss_pred"].any()
