"""The strip's running maximum in k_viterbi: each column's record is the first row that reaches the column's maximum,
taken when it beats the strip's best or ties it at a smaller row.  These cases plant the maxima where that rule
decides: exact ties inside a column, between columns, across strip boundaries, at the first and last column, in the
padded columns of a short lane, in the last strip of a query that is not a multiple of the strip height, and in
global mode.  Every case is checked against the C oracle at strip heights 8, 12 and 16 and between them; a bench-like
shard is checked byte for byte against the records the kernel produced before the column argmax replaced the
per-row loop."""
import hashlib

import numpy as np
import pytest

from tests import vit_cases as vc
from tests.test_kernel_variants_gpu import env_ctx
from tests.test_viterbi_gpu import _check_against_oracle

pytestmark = pytest.mark.gpu

HEIGHTS = (8, 12, 16)
HI, LO = 3, -2          # with shift -0.5: +2.5 for a planted match, -2.5 elsewhere
PAR = dict(shift=-0.5)
HIT_FIELDS = ("score", "i2", "j2", "i1", "j1", "nsteps", "matched_cols", "hit_score", "score_ss")


def planted(Lq, targets):
    """Query and targets of dyadic match blocks.  targets: [(Lt, [(letter, n, i_end, j_end), ...])]: query rows
    i_end-n+1 .. i_end hold the letter, and target columns j_end-n+1 .. j_end score it high, so the block's diagonal
    ending at (i_end, j_end) is worth 2.5 n.  Query rows outside every block hold letter 0, which no column scores."""
    qlet = np.zeros(Lq, np.int64)
    for _, runs in targets:
        for a, n, i, _ in runs:
            assert a > 0 and np.all(qlet[i - n:i] * (qlet[i - n:i] != a) == 0), "query rows planted twice"
            qlet[i - n:i] = a
    q = vc._profile(vc._letters_rows(qlet, "q", HI, LO), vc.TR_DIAG, "q")
    tg = []
    for Lt, runs in targets:
        rows = np.full((Lt, 20), np.float32(2.0 ** LO), np.float32)
        for a, n, _, j in runs:
            rows[j - n:j, a] = np.float32(2.0 ** HI)
        tg.append(vc._profile(rows, vc.TR_DIAG, "t"))
    return q, tg


# name: (Lq, [(Lt, runs)], the maximal end cells of each target in row-major order (None: not asserted), par)
CASES = {
    # two rows of one column reach the same maximum: the smaller row wins
    "column-tie": (48, [(40, [(1, 2, 5, 20), (2, 2, 12, 20)])], [[(5, 20), (12, 20)]], PAR),
    # the same maximum in a later column at a smaller row wins; at a larger row it loses
    "later-column-smaller-row": (48, [(40, [(1, 2, 5, 30), (2, 2, 12, 20)]),
                                      (40, [(1, 2, 5, 20), (2, 2, 12, 30)])],
                                 [[(5, 30), (12, 20)], [(5, 20), (12, 30)]], PAR),
    # rows 16 and 18 lie in different strips at R = 8 and 16 (the strip merge decides) and in one at R = 12
    "strip-boundary": (48, [(64, [(3, 2, 16, 40), (4, 2, 18, 20)]), (64, [(3, 2, 16, 20), (4, 2, 18, 40)])],
                       [[(16, 40), (18, 20)], [(16, 20), (18, 40)]], PAR),
    # the maximum in the first column, and in the last column (a tie there with a later row)
    "first-and-last-column": (48, [(33, [(5, 1, 9, 1)]), (33, [(6, 3, 30, 33), (7, 3, 40, 33)])],
                              [[(9, 1)], [(30, 33), (40, 33)]], PAR),
    # a block that ends in the short lane's last column while its query rows go on: the padded columns 31 .. 64
    # repeat column 30, would extend the diagonals past 40 and must not count
    "padded-columns": (48, [(30, [(8, 16, 25, 30), (8, 10, 35, 30)]), (64, [(9, 3, 45, 60)])],
                       [[(i, 30) for i in range(25, 36)], [(45, 60)]], PAR),
}


def _cases():
    for Lq in (401, 407, 1500):
        # the maximum in row Lq of the last strip (padded at every height for 401 and 407; 1500 = 125 x 12), a tie
        # with a smaller row in a later column, and a single match a few rows above Lq
        CASES[f"last-strip-{Lq}"] = (
            Lq, [(50, [(10, 3, Lq, 20)]), (50, [(10, 3, Lq, 20), (11, 3, Lq - 20, 40)]),
                 (50, [(12, 1, Lq - 5, 45)])],
            [[(Lq, 20)], [(Lq - 20, 40), (Lq, 20)], [(Lq - 5, 45)]], PAR)
    # global mode: only row Lq and column Lt count, so the blocks end there; a tie between them, and one alone
    CASES["global"] = (48, [(40, [(13, 4, 48, 4), (14, 4, 4, 40)]), (40, [(13, 4, 48, 4)])],
                       [[(4, 40), (48, 4)], [(48, 4)]], dict(local=False, shift=-0.5, egq=0.0, egt=0.0))
    return CASES


@pytest.fixture(scope="module")
def cases():
    out = {}
    for name, (Lq, targets, cells, par) in _cases().items():
        q, tg = planted(Lq, targets)
        for t, want in zip(tg, cells):
            if want is not None:
                got = vc.witness(q, t, **par)["cells"]
                assert got == want, (name, got, want)
        out[name] = (q, tg, par)
    return out


def _records(plan):
    hits, paths = plan.fetch()
    return {f: hits[f].copy() for f in HIT_FIELDS}, [paths[h["path_off"]:h["path_off"] + h["nsteps"]].copy()
                                                     for h in hits]


@pytest.mark.parametrize("name", list(_cases()))
def test_planted_maxima_match_oracle_at_every_height(hhg, oracle, cases, name):
    q, tg, par = cases[name]
    seen = []
    for R in HEIGHTS:
        with env_ctx(hhg, HHG_STRIP_ROWS=R) as ctx:
            hits = _check_against_oracle(hhg, ctx, oracle, q, tg, **par)
        seen.append({f: hits[f].tobytes() for f in HIT_FIELDS})
    for R, s in zip(HEIGHTS[1:], seen[1:]):
        for f in HIT_FIELDS:
            assert s[f] == seen[0][f], (name, R, f)


# ----------------------------------------------------------------------------------------- bench-like shard
SHARD_N = 3000
SHARD_ORACLE_SAMPLE = 12
# sha256 of the hit records (HIT_FIELDS, in target order) and of the concatenated alignment paths of the shard below,
# as the per-row running-maximum loop computed them (every strip height gives the same records)
SHARD_DIGEST = "653714a33f80ae0f0b77b64b55268802a06ba37a1ed26be26912b34d645d7917"


def bench_like_shard():
    """Lq = 400 against SHARD_N seeded targets drawn like bench.py's headline shard (lognormal lengths, median 200,
    planted query columns)."""
    from hhsuite_b200 import synth
    q = synth.query_profile(400, seed=1)
    lens = synth.lengths(SHARD_N, np.random.default_rng(4242))
    db = synth.prepared_db(SHARD_N, seed=4243, query_cols=q[4], planted=64, lens=lens, fast=True)
    return q, db


def shard_digest(hits, paths):
    h = hashlib.sha256()
    for f in HIT_FIELDS:
        h.update(np.ascontiguousarray(hits[f]).tobytes())
    for p in paths:
        h.update(p.tobytes())
    return h.hexdigest()


def run_shard(hhg, ctx, q, db_h):
    ctx.set_query(q[0], q[1])
    db = hhg.TargetDB(ctx, db_h["L"], db_h["p"], db_h["tr"], db_h["p_off"], db_h["tr_off"])
    plan = hhg.Plan(ctx, db)
    plan.run()
    rec = _records(plan)
    plan.close()
    db.close()
    return rec


def test_bench_like_shard_matches_previous_records(hhg, oracle):
    q, db_h = bench_like_shard()
    for R in HEIGHTS:
        with env_ctx(hhg, HHG_STRIP_ROWS=R) as ctx:
            hits, paths = run_shard(hhg, ctx, q, db_h)
        assert shard_digest(hits, paths) == SHARD_DIGEST, R
    pick = np.random.default_rng(11).choice(SHARD_N, SHARD_ORACLE_SAMPLE, replace=False)
    for t in pick:
        o, L = int(db_h["p_off"][t]), int(db_h["L"][t])
        to = int(db_h["tr_off"][t])
        sc, i2, j2, bt = oracle.viterbi(q[0], q[1], db_h["p"][o:o + L + 2], db_h["tr"][to:to + L + 1],
                                        local=True, egq=0.0, egt=0.0, shift=-0.03)
        assert hits["score"][t].view(np.uint32) == np.float32(sc).view(np.uint32), t
        assert (hits["i2"][t], hits["j2"][t]) == (i2, j2), t
