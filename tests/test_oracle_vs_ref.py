"""CPU tests (authoring container, where oracle/_ref is built): the C restatement against the
UNMODIFIED compiled reference on fresh seeded inputs -- this is what pins the oracle."""
import numpy as np
import pytest

from tests.util import bits, ref_data_file


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_restatement_equals_reference_kernel(oracle, refshim, seed):
    from hhsuite_b200 import synth
    rng = np.random.default_rng(seed)
    qp, qtr, qss, qpav, qcols = synth.query_profile(int(rng.integers(40, 200)), seed)
    refshim.set_query(qp, qtr, qpav, qss)
    S33 = refshim.S33()
    tg = [synth.prepared_profile(int(L), rng, qcols if k % 2 else None, noise=0.3)
          for k, L in enumerate(rng.integers(1, 250, refshim.V))]
    co = [(rng.random((qp.shape[0] - 1, t[0].shape[0] - 1)) < 0.1).astype(np.uint8) for t in tg]
    for kw_ref, kw_or in ((dict(), dict()), (dict(use_ss=True), dict(ss=True)), (dict(celloff=co), dict(co=True)),
                          (dict(celloff=co, use_ss=True), dict(co=True, ss=True))):
        res = refshim.viterbi(tg, **kw_ref)
        for k, (tp, ttr, tss) in enumerate(tg):
            okw = {}
            if kw_or.get("ss"):
                okw.update(q_ss=qss, t_ss=tss, S33=S33)
            if kw_or.get("co"):
                okw.update(celloff=co[k])
            sc, i2, j2, bt = oracle.viterbi(qp, qtr, tp, ttr, **okw)
            rs, ri, rj, rbt = res[k]
            assert bits(sc) == bits(rs) and (i2, j2) == (ri, rj)
            assert np.array_equal(bt[1:, 1:], rbt[1:, 1:])
            n1 = refshim.backtrace(k)
            n2 = oracle.backtrace(bt, i2, j2)
            assert n1[0] == n2[0] and n1[4] == n2[4]
            for a, b in zip(n1[1:4], n2[1:4]):
                assert np.array_equal(a[1:], b[1:])


def test_synthetic_hhm_text_roundtrip_through_reference_reader(refshim, tmp_path):
    """The synthetic HHM text is accepted by HMM::Read and PrepareTemplateHMM gives finite DP inputs."""
    from hhsuite_b200 import synth
    refshim.load_query_hhm(ref_data_file("query.hhm", tmp_path))
    f = tmp_path / "s.hhm"
    f.write_text(synth.hhm_text(77, 5, "s77", with_ss=True))
    t = refshim.prepare_template_hhm(str(f))
    assert t["L"] == 77 and np.isfinite(t["p"]).all() and (t["p"][1:78] > 0).all()
    assert t["ss"][1:78].min() >= 11          # ss_pred/ss_conf were read


# ---- tie-forcing and degenerate families (tests/vit_cases.py): every tie rule of the oracle against the reference
def _celloff_through_ties(q, t, par):
    """A cell-off mask that cuts through the tied maxima: a +-2 cross around the first maximal end cell (when the
    input is dyadic) plus a sparse lattice."""
    from tests import vit_cases as vc
    Lq, Lt = q[0].shape[0] - 2, t[0].shape[0] - 2
    m = np.zeros((Lq + 1, Lt + 1), np.uint8)
    ii, jj = np.meshgrid(np.arange(Lq + 1), np.arange(Lt + 1), indexing="ij")
    m[((3 * ii + jj) % 11 == 0) & (ii > 0) & (jj > 0)] = 1
    try:
        i, j = vc.witness(q, t, **par)["first"]
    except AssertionError:          # not dyadic
        i, j = (Lq + 1) // 2, (Lt + 1) // 2
    if i > 0 and j > 0:
        m[max(i - 2, 1):i + 3, j] = 1
        m[i, max(j - 2, 1):j + 3] = 1
    return m


def _compare_case(oracle, refshim, q, tg, par, use_ss=False, co=None):
    local = par.get("local", True)
    S33 = refshim.S33() if use_ss else None
    refshim.set_query(q[0], q[1], q[0][1:-1].mean(axis=0) if q[0].shape[0] > 2 else None, q[2])
    # one target per call in global mode (the library's semantics) and with cell-off masks: in a batch the reference
    # also scans the padding columns up to the longest target, and those win when a mask switches off every real cell
    step = refshim.V if local and co is None else 1
    for b in range(0, len(tg), step):
        chunk = tg[b:b + step]
        res = refshim.viterbi(chunk, use_ss=use_ss, celloff=None if co is None else co[b:b + step], **par)
        for k, (tp, ttr, tss) in enumerate(chunk):
            okw = dict(par)
            if use_ss:
                okw.update(q_ss=q[2], t_ss=tss, S33=S33)
            if co is not None:
                okw.update(celloff=co[b + k])
            sc, i2, j2, bt = oracle.viterbi(q[0], q[1], tp, ttr, **okw)
            rs, ri, rj, rbt = res[k]
            where = (b + k, tp.shape[0] - 2)
            assert bits(sc) == bits(rs) and (i2, j2) == (ri, rj), (where, sc, rs, (i2, j2), (ri, rj))
            assert np.array_equal(bt[1:, 1:], rbt[1:, 1:]), (where, int((bt[1:, 1:] != rbt[1:, 1:]).sum()))
            n1 = refshim.backtrace(k)
            n2 = oracle.backtrace(bt, i2, j2)
            assert n1[0] == n2[0] and n1[4] == n2[4], where
            for a, c in zip(n1[1:4], n2[1:4]):
                assert np.array_equal(a[1:], c[1:]), where


def _family_ids(cases):
    return [c[0] for c in cases]


def _all_cases():
    from tests import vit_cases as vc
    return vc.all_cases()


@pytest.mark.parametrize("case", _all_cases(), ids=_family_ids(_all_cases()))
def test_tie_families_oracle_equals_reference(oracle, refshim, case):
    """Score bits, (i2, j2), every backtrace byte, the path, nsteps and matched_cols of the oracle equal the compiled
    reference's on the tie and degenerate families: plain, SS with a constant and a varying ss string, and cell-off
    masks that cut through the tied cells."""
    from tests import vit_cases as vc
    name, q, tg, par = case
    _compare_case(oracle, refshim, q, tg, par)
    _compare_case(oracle, refshim, q, tg, par, use_ss=True)
    _compare_case(oracle, refshim, vc.with_mixed_ss(q), [vc.with_mixed_ss(t) for t in tg], par, use_ss=True)
    _compare_case(oracle, refshim, q, tg, par, co=[_celloff_through_ties(q, t, par) for t in tg])
