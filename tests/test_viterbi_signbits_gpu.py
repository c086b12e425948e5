"""k_viterbi's backtrace flags on the inputs where a sign-bit test could differ from the reference's '>' compare.

The kernel takes each gap-state flag (GD, IM, DG, MI) from the sign bit of a2 - a1 rather than from a1 > a2.  The two
agree unless a2 - a1 is -0 with a1 == a2, which needs a DP value of -0; the kernel keeps those out by starting from
+0 where -i·egq or -j·egt is -0.  These cases put zeros of both signs where they could leak in, and exact ties and
-FLT_MAX / -inf values where the difference is 0, NaN or overflows:
  * transitions whose zero entries carry random signs, with egq = egt = 0 (the initial MM row and column are -0);
  * dyadic families where a1 == a2 in whole regions, at 0 and away from it (Si == 0 everywhere in 'zero');
  * global mode, whose boundary states and smin are -FLT_MAX, with '*' and -FLT_MAX transitions and gap costs that
    push the first column to -inf.
Every case runs at strip heights 8, 12 and 16, in local and global mode, with and without the ss term, and with and
without cell-off bits (excluded regions).  Without cell-off bits every backtrace byte is compared with the C oracle's;
with them the scores, end cells and paths are."""
import numpy as np
import pytest

from tests import vit_cases as vc
from tests.test_kernel_variants_gpu import env_ctx
from tests.test_viterbi_gpu import _check_against_oracle
from tests.util import bits, golden

HEIGHTS = (8, 12, 16)
LQS = (5, 13, 17, 48)
BIG = 2.0 ** 126        # -i·egq is -inf from row 2 on


def _signed_zeros(prof, seed):
    """The profile with every zero transition given a random sign (both signs in every profile)."""
    p, tr, ss = prof
    tr = tr.copy()
    zero = tr == 0.0
    neg = np.random.default_rng(seed).random(tr.shape) < 0.5
    tr[zero & neg] = np.float32(-0.0)
    tr[zero & ~neg] = np.float32(0.0)
    return p, tr, ss


def _zero_tr(prof):
    p, tr, ss = prof
    return p, np.zeros_like(tr), ss


def _family(name, Lq):
    """(query, targets, local-mode parameters) of one family; every zero transition has a random sign."""
    if name == "zero":       # Si == 0 and all transitions zero: every DP value of the local matrix is 0
        q, tg, par = vc.const(Lq, "q", level=1), vc._targets(vc.const, level=1), dict(shift=-1.0)
        q, tg = _zero_tr(q), [_zero_tr(t) for t in tg]
    elif name == "gap":      # a1 == a2 for the gap states and c1 == c2 in whole regions
        q, tg, par = vc.gap(Lq, "q"), vc._targets(vc.gap), dict(shift=-0.5)
    elif name == "tandem":
        q, tg, par = vc.tandem(Lq, "q", k=5), vc._targets(vc.tandem, k=5), dict(shift=-0.5)
    elif name == "negtr":    # '*' and -FLT_MAX transitions
        q, tg, par = vc.degen(Lq, "q", "negtr"), [vc.degen(L, "t", "negtr") for L in vc.LT], dict(shift=-0.03)
    else:
        raise ValueError(name)
    q = _signed_zeros(q, Lq)
    tg = [_signed_zeros(t, 1000 * Lq + k) for k, t in enumerate(tg)]
    return q, tg, par


FAMILIES = ("zero", "gap", "tandem", "negtr")


def _cases(local):
    for name in FAMILIES:
        for Lq in LQS:
            q, tg, par = _family(name, Lq)
            if local:
                yield q, tg, dict(par, egq=0.0, egt=0.0)
            else:
                yield q, tg, dict(par, local=False, egq=0.0, egt=0.0)
                yield q, tg, dict(par, local=False, egq=BIG, egt=BIG)


def _oracle_kw(par, q, t, S33):
    kw = dict(local=par.get("local", True), egq=par["egq"], egt=par["egt"], shift=par["shift"])
    if S33 is not None:
        kw.update(q_ss=q[2], t_ss=t[2], S33=S33)
    return kw


def _region_mask(Lq, Lt, q_ranges, t_ranges):
    m = np.zeros((Lq + 1, Lt + 1), np.uint8)
    for a, b in q_ranges:
        m[a:min(b, Lq) + 1, 1:] = 1
    for a, b in t_ranges:
        if a <= Lt:
            m[1:, a:min(b, Lt) + 1] = 1
    return m


def _check_celloff(hhg, ctx, oracle, q, tg, par, S33):
    """Excluded query rows and template columns (cell-off instantiations): scores, end cells and paths."""
    Lq = q[0].shape[0] - 2
    qr, tr = [(Lq // 2 + 1, Lq // 2 + 1)], [(2, 3), (33, 33)]
    ctx.set_query(q[0], q[1], q[2], S33, use_ss=S33 is not None, **par)
    db = hhg.TargetDB.from_profiles(ctx, tg)
    ctx.set_excluded_regions(qr, tr)
    try:
        hits, paths = hhg.viterbi_search(ctx, db)
    finally:
        ctx.set_excluded_regions()
    for k, t in enumerate(tg):
        mask = _region_mask(Lq, t[0].shape[0] - 2, qr, tr)
        sc, i2, j2, bt = oracle.viterbi(q[0], q[1], t[0], t[1], celloff=mask, **_oracle_kw(par, q, t, S33))
        h = hits[k]
        where = (k, t[0].shape[0] - 2)
        assert bits(h["score"]) == bits(sc), (where, h["score"], sc)
        assert (h["i2"], h["j2"]) == (i2, j2), where
        n, i_s, j_s, st, mc = oracle.backtrace(bt, i2, j2)
        assert (h["nsteps"], h["matched_cols"], h["i1"], h["j1"]) == (n, mc, i_s[n], j_s[n]), where
        assert np.array_equal(paths[h["path_off"]:h["path_off"] + n], st[1:]), where
    db.close()


def test_cases_have_signed_zeros_and_ties():
    """The inputs really hold zeros of both signs, and the dyadic families really tie (float64 witness)."""
    for name in FAMILIES:
        for Lq in LQS:
            q, tg, _ = _family(name, Lq)
            trs = np.concatenate([q[1].ravel()] + [t[1].ravel() for t in tg])
            z = trs[trs == 0.0]
            assert np.signbit(z).any() and (~np.signbit(z)).any(), (name, Lq)
    for name in ("zero", "gap"):
        q, tg, par = _family(name, 17)
        ties = vc.witness(q, tg[4], **par)["ties"]
        assert ties["gd"] > 0 and ties["dg"] > 0, (name, ties)


@pytest.mark.gpu
@pytest.mark.parametrize("R", HEIGHTS)
@pytest.mark.parametrize("local", [True, False], ids=["local", "global"])
@pytest.mark.parametrize("ss", [False, True], ids=["plain", "ss"])
def test_signed_zeros_ties_and_neg_boundaries_match_oracle(hhg, oracle, R, local, ss):
    S33 = golden()["S33"] if ss else None
    with env_ctx(hhg, HHG_STRIP_ROWS=R) as ctx:
        for q, tg, par in _cases(local):
            if ss:
                q, tg = vc.with_mixed_ss(q), [vc.with_mixed_ss(t) for t in tg]
                _check_against_oracle(hhg, ctx, oracle, q, tg, S33=S33, use_ss=True, **par)
            else:
                _check_against_oracle(hhg, ctx, oracle, q, tg, **par)
            _check_celloff(hhg, ctx, oracle, q, tg, par, S33)
