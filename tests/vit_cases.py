"""Tie-forcing and degenerate Viterbi inputs (test helpers, not product code).

Random float profiles almost never make two DP candidates bit-equal, so they cannot tell whether a kernel breaks ties
the way the reference does.  The generators here build *dyadic* profiles instead: every query row is one-hot (or two
halves) and every target column holds powers of two, so the 20-term dot product is an exact power of two, log2f4 of it
is an exact integer, and with dyadic transitions, shift, egq and egt every finite DP value is exact.  Ties are then
there by construction.  Profiles come in the shapes of synth.prepared_profile / synth.query_profile: (p[(L+2),20],
tr[(L+1),7], ss[L+2]), tr in the reference order M2M, M2I, M2D, I2M, I2I, D2M, D2D.

Families
  const     identical query rows against identical target columns: MM depends only on the path
  tandem    a block of k letters repeated in query and target (k in 3, 5, 6, 7): equal diagonals every k rows
  anti      the target block reversed: equal isolated matches on the anti-diagonals i + j = 1 (mod k)
  gap       transitions for which MM+m2d == GD+d2d, MM+m2i+m2m == IM+i2i+m2m, ... and c1 == c2 hold exactly
  degen     all-zero emission rows/columns (log2f4's e = -127 path), denormal products, -FLT_MAX and '*' transitions

witness() is a float64 restatement of the DP for dyadic inputs: it returns the score, the set of maximal end cells
and how often each kind of tie occurred, so a test can assert that a family really produces ties.
"""
from __future__ import annotations

import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)
NEG_STAR = np.float32(-99999.0 / 1000.0)   # what the HHM reader stores for a '*' transition (synth.NEG)

LQ = (1, 2, 3, 4, 5, 8, 12, 13, 16, 17, 48, 49)
LT = (1, 2, 3, 4, 31, 32, 33, 40, 64, 65)     # > 32 too, so one 32-lane job holds targets of unequal length

# transition rows, order M2M, M2I, M2D, I2M, I2I, D2M, D2D
TR_DIAG = (0.0, -2.0, -2.0, -1.0, -1.0, -1.0, -1.0)    # free diagonal, costly gaps
TR_TIE = (-1.0, -0.5, -0.5, -0.5, 0.0, -0.5, 0.0)      # open + extend == stay in MM: gap flags and c1 == c2 tie

QBG = np.float32(0.0625)   # query rows 0 and L+1 (never read by the DP)


def _ss(L, mixed):
    ss = np.zeros(L + 2, np.uint8)
    k = np.arange(L)
    ss[1:L + 1] = (1 + k % 3) * 11 + (1 + (k * 7) % 10) if mixed else 2 * 11 + 5
    return ss


def _profile(rows, tr_row, role, mixed_ss=False):
    L = len(rows)
    p = np.full((L + 2, 20), QBG if role == "q" else np.float32(1.0), np.float32)
    if L:
        p[1:L + 1] = rows
    tr = np.tile(np.asarray(tr_row, np.float32), (L + 1, 1))
    return p, tr, _ss(L, mixed_ss)


def _letters_rows(letters, role, hi, lo):
    """Query: one-hot 1.0 at the letter.  Target: 2**hi at the letter, 2**lo elsewhere (lo None: 0)."""
    rows = np.zeros((len(letters), 20), np.float32)
    for r, a in enumerate(letters):
        if role == "q":
            rows[r, a] = 1.0
        else:
            rows[r, :] = 0.0 if lo is None else 2.0 ** lo
            rows[r, a] = 2.0 ** hi
    return rows


def const(L, role, level=3, tr=TR_DIAG, mixed_ss=False):
    """Every query row 0.5 at letters 0 and 1, every target column 2**level at letters 0 and 1 (0.25 elsewhere):
    the dot product is 2**level in every cell (two terms)."""
    rows = np.zeros((L, 20), np.float32)
    if role == "q":
        rows[:, 0] = rows[:, 1] = 0.5
    else:
        rows[:, :] = 0.25
        rows[:, 0] = rows[:, 1] = 2.0 ** level
    return _profile(rows, tr, role, mixed_ss)


def tandem(L, role, k=5, reverse=False, hi=3, lo=-2, tr=TR_DIAG, mixed_ss=False):
    """Letters (p-1) mod k; with reverse the target uses (-p) mod k, so matches lie on i + j = 1 (mod k)."""
    pos = np.arange(1, L + 1)
    letters = ((-pos) % k) if (reverse and role == "t") else ((pos - 1) % k)
    return _profile(_letters_rows(letters, role, hi, lo), tr, role, mixed_ss)


def gap(L, role, mixed_ss=False):
    """const at level 3 with TR_TIE: with shift -0.5 the diagonal gains 0.5 per step, so c1 > 0 and the gap
    candidates equal it in whole regions."""
    return const(L, role, level=3, tr=TR_TIE, mixed_ss=mixed_ss)


def degen(L, role, kind):
    """Non-dyadic edge values.  kind: 'zero' (every third row/column all-zero, the rest const), 'denormal'
    (2**-70 x 2**-70 products), 'negtr' (-FLT_MAX and '*' transitions in alternate rows)."""
    p, tr, ss = const(L, role, level=2, tr=TR_DIAG)
    if kind == "zero":
        p[1 + (np.arange(L) % 3 == (0 if role == "q" else 1)).nonzero()[0]] = 0.0
    elif kind == "denormal":
        rows = np.zeros((L, 20), np.float32)
        rows[:, 0] = np.float32(2.0 ** -70)
        rows[:, 1 + np.arange(L) % 19] = np.float32(2.0 ** -68) if role == "t" else np.float32(2.0 ** -73)
        p[1:L + 1] = rows
    elif kind == "negtr":
        tr[1::2, 1] = -FLT_MAX          # M2I
        tr[::2, 2] = NEG_STAR           # M2D
        tr[::3, 5] = NEG_STAR           # D2M
        tr[1::3, 0] = -FLT_MAX          # M2M
    else:
        raise ValueError(kind)
    return p, tr, ss


# ------------------------------------------------------------------------------------------------- the case table
def with_mixed_ss(prof):
    """The same profile with varying ss_pred / ss_conf values instead of a constant one."""
    p, tr, _ = prof
    return p, tr, _ss(p.shape[0] - 2, True)


def _targets(fn, lts=LT, **kw):
    return [fn(L, "t", **kw) for L in lts]


def tie_cases():
    """(name, query, targets, par) of the dyadic tie families.  par: local, shift, egq, egt (all dyadic)."""
    out = []
    for Lq in LQ:
        out.append((f"const-grow-{Lq}", const(Lq, "q"), _targets(const), dict(shift=-0.5)))
        out.append((f"gap-{Lq}", gap(Lq, "q"), _targets(gap), dict(shift=-0.5)))
        for k in (3, 5, 6, 7):
            if Lq >= k or Lq in (1, 2):
                out.append((f"tandem{k}-{Lq}", tandem(Lq, "q", k=k), _targets(tandem, k=k), dict(shift=-0.5)))
                out.append((f"anti{k}-{Lq}", tandem(Lq, "q", k=k, reverse=True),
                            _targets(tandem, k=k, reverse=True), dict(shift=-0.5)))
    for Lq in (1, 5, 13, 17, 49):
        # Si == 0 everywhere: local MM is exactly 0 = smin in every cell; Si < 0: every cell restarts
        out.append((f"const-zero-{Lq}", const(Lq, "q", level=1), _targets(const, level=1), dict(shift=-1.0)))
        out.append((f"const-neg-{Lq}", const(Lq, "q", level=0), _targets(const, level=0), dict(shift=-0.5)))
    return out


def global_cases():
    """Global-mode variants (dyadic egq / egt; the library's one-target semantics: end cells i == Lq or j == Lt)."""
    out = []
    for Lq in (1, 4, 5, 13, 17, 48):
        out.append((f"g-const-{Lq}", const(Lq, "q", level=1), _targets(const, level=1),
                    dict(local=False, shift=-1.0, egq=0.0, egt=0.0)))
        out.append((f"g-gap-{Lq}", gap(Lq, "q"), _targets(gap), dict(local=False, shift=-0.5, egq=0.0, egt=0.0)))
        out.append((f"g-tandem5-{Lq}", tandem(Lq, "q", k=5), _targets(tandem, k=5),
                    dict(local=False, shift=-0.5, egq=1.0, egt=0.5)))
        out.append((f"g-anti3-{Lq}", tandem(Lq, "q", k=3, reverse=True), _targets(tandem, k=3, reverse=True),
                    dict(local=False, shift=-0.5, egq=0.25, egt=0.25)))
    return out


def degen_cases():
    """Degenerate values (not dyadic, no witness), local and global with large egq / egt."""
    out = []
    for Lq in (1, 4, 13, 17, 49):
        for kind in ("zero", "denormal", "negtr"):
            q = degen(Lq, "q", kind)
            tg = [degen(L, "t", kind) for L in LT]
            out.append((f"d-{kind}-{Lq}", q, tg, dict(shift=-0.03)))
            out.append((f"d-{kind}-glob-{Lq}", q, tg, dict(local=False, shift=-0.03, egq=1024.0, egt=2.0 ** 100)))
    return out


def all_cases():
    return tie_cases() + global_cases() + degen_cases()


# ------------------------------------------------------------------------------------------------------ witness
def _log2_exact(x):
    if x == 0.0:
        return -127.0
    m, e = np.frexp(x)
    assert m == 0.5, f"witness needs power-of-two dot products, got {x!r}"
    return float(e - 1)


def witness(q, t, local=True, shift=-0.5, egq=0.0, egt=0.0):
    """Float64 DP of Viterbi::AlignWithOutCellOff on dyadic inputs (exact there); values <= -1e30 stand for the
    reference's -FLT_MAX-saturated ones and are -inf here.  Returns dict(score, cells (maximal end cells in row-major
    order), first, ties: counts of cells where c1 == c2 is the MM maximum above smin, smin == MM maximum, and each gap
    flag's a1 == a2)."""
    qp, qtr = np.asarray(q[0], np.float64), np.asarray(q[1], np.float64)
    tp, ttr = np.asarray(t[0], np.float64), np.asarray(t[1], np.float64)
    Lq, Lt = qp.shape[0] - 2, tp.shape[0] - 2
    ninf = -np.inf

    def cl(v):
        return v if v > -1e30 else ninf

    smin = 0.0 if local else ninf
    M = np.full((Lq + 1, Lt + 1), ninf); GD = M.copy(); IM = M.copy(); DG = M.copy(); MI = M.copy()
    M[0, :] = -np.arange(Lt + 1) * egt
    M[:, 0] = -np.arange(Lq + 1) * egq
    S = np.zeros((Lq + 1, Lt + 1))
    for i in range(1, Lq + 1):
        for j in range(1, Lt + 1):
            S[i, j] = _log2_exact(float(np.dot(qp[i], tp[j])))
    ties = dict(c1c2=0, zero=0, gd=0, im=0, dg=0, mi=0)
    M2M, M2I, M2D, I2M, I2I, D2M, D2D = range(7)
    for i in range(1, Lq + 1):
        a, b = qtr[i - 1], qtr[i]
        for j in range(1, Lt + 1):
            c, d = ttr[j - 1], ttr[j]
            cand = [smin, cl(cl(M[i - 1, j - 1] + a[M2M]) + c[M2M]), cl(cl(GD[i - 1, j - 1] + a[M2M]) + c[D2M]),
                    cl(cl(IM[i - 1, j - 1] + a[I2M]) + c[M2M]), cl(cl(DG[i - 1, j - 1] + a[D2M]) + c[M2M]),
                    cl(cl(MI[i - 1, j - 1] + a[M2M]) + c[I2M])]
            mx = max(cand)
            if mx > ninf:
                if cand[1] == cand[2] == mx and mx > smin:
                    ties["c1c2"] += 1
                if local and cand[0] == mx:
                    ties["zero"] += 1
            M[i, j] = cl(mx + cl(S[i, j] + shift)) if mx > ninf else ninf
            pairs = dict(gd=(cl(M[i, j - 1] + c[M2D]), cl(GD[i, j - 1] + c[D2D])),
                         im=(cl(cl(M[i, j - 1] + b[M2I]) + c[M2M]), cl(cl(IM[i, j - 1] + b[I2I]) + c[M2M])),
                         dg=(cl(M[i - 1, j] + a[M2D]), cl(DG[i - 1, j] + a[D2D])),
                         mi=(cl(cl(M[i - 1, j] + a[M2M]) + d[M2I]), cl(cl(MI[i - 1, j] + a[M2M]) + d[I2I])))
            for key, (x, y) in pairs.items():
                if x == y and x > ninf:
                    ties[key] += 1
            GD[i, j], IM[i, j], DG[i, j], MI[i, j] = (max(v) for v in pairs.values())
    end = np.zeros_like(M, bool)
    if local:
        end[1:, 1:] = True
    else:
        end[Lq, 1:] = True
        end[1:, Lt] = True
    vals = np.where(end, M, ninf)
    score = vals.max()
    cells = [tuple(int(x) for x in c) for c in np.argwhere((vals == score) & end)] if score > ninf else []
    return dict(score=score, cells=cells, first=cells[0] if cells else (0, 0), ties=ties, MM=M)
