"""Seeded query batches for the query-batch Viterbi tests (test helpers, not product code; import without a GPU).

hhg_viterbi_search_batch is the only entry point whose plan mixes queries: jobs of different Lq, first query row and
strip count share one work-item table, one group of jobs and one memory wave.  The builders here choose lengths where
that geometry changes (the 48-row query padding, strip edges at R = 8 / 12 / 16, the 32-lane job edge) and restate the
host rules the plan follows, so a test knows which strip height, how many padded cells and which memory waves the
library must produce:

  strip_rows    plan_strip_rows: R = 16 once the batch has >= 4 * SMs * 8 work items of 16-row strips, else R = 8
  plan_jobs     plan_build's jobs: per query, requests stably sorted by target length (longest first), cut into 32s
  wave_sizes    plan_build's memory waves: a new wave starts when the next job's backtrace words would overflow
                the budget (a job larger than the budget gets a wave of its own)
  null_model    HMM::IncludeNullModelInHMM: template emissions divided by pb, 0.5 (q.pav + t.pav), t.pav or q.pav in
                float32 (numpy float32 division is correctly rounded, so this is bit-exact)

Two scales: make_batch("scan") is big enough that the automatic strip height is 16 (a whole-shard search),
make_batch("survivors") small enough that it is 8 (the prefilter's survivors).
"""
from __future__ import annotations

import numpy as np

from hhsuite_b200 import synth

# query lengths at the 48-row padding and at strip edges of R = 8, 12 and 16
QUERY_LENGTHS = (1, 2, 7, 8, 9, 11, 12, 13, 16, 17, 47, 48, 49, 95, 96, 97, 211, 400, 1000, 1500)
TARGET_EDGES = (1, 2, 31, 32, 33)     # around one 32-lane job
COUNT_EDGES = (0, 1, 32, 33)          # requests per query: none, one, one full job, one job and one lane
MAX_LEN = 32767                       # longest query / target hhg_query_set and hhg_db_create take
PATH_LIMIT = 2 ** 31 - 1              # a plan refuses requests whose sum of (Lq + Lt + 2) exceeds this
H100_SMS = 132                        # H100 SXM5
SCAN_WAVE_GB = "0.015"                # HHG_MAX_BT_GB that cuts the scan batch (R = 16) into >= 5 memory waves


# ------------------------------------------------------------------------------------------------ plan geometry
def items16(q_lens, req_query):
    """Work items a plan would have at R = 16: per query ceil(requests / 32) jobs of ceil(Lq / 16) strips."""
    cnt = np.bincount(np.asarray(req_query, np.int64), minlength=len(q_lens))
    return int(sum((int(c) + 31) // 32 * ((int(L) + 15) // 16) for c, L in zip(cnt, q_lens)))


def strip_rows(q_lens, req_query, sm_count, forced=None):
    """The strip height a plan picks (plan_strip_rows); forced = HHG_STRIP_ROWS."""
    if forced:
        return int(forced)
    return 16 if items16(q_lens, req_query) >= 4 * sm_count * 8 else 8


def plan_jobs(q_lens, req_query, t_lens, R):
    """[(query, Lmax, nstrips)] in plan order: requests sorted by (query, target length descending), stable."""
    rq = np.asarray(req_query, np.int64); tl = np.asarray(t_lens, np.int64)
    order = sorted(range(len(rq)), key=lambda k: (rq[k], -tl[k]))
    out = []
    first = 0
    while first < len(order):
        q = int(rq[order[first]])
        cnt = 0
        while first + cnt < len(order) and cnt < 32 and rq[order[first + cnt]] == q:
            cnt += 1
        out.append((q, int(tl[order[first]]), (int(q_lens[q]) + R - 1) // R))
        first += cnt
    return out


def padded_cells(jobs, R):
    """hhg_plan_padded_cells: sum over jobs of nstrips * R * Lmax * 32."""
    return float(sum(ns * R * Lmax * 32 for _, Lmax, ns in jobs))


def job_bt_bytes(job, R):
    """Backtrace words of one job (one 32-bit word per 4 rows, Lmax + 1 columns, 32 lanes), in bytes."""
    _, Lmax, ns = job
    return (ns * R // 4) * (Lmax + 1) * 32 * 4


def bt_budget(gb: str):
    """The byte budget a context derives from HHG_MAX_BT_GB=gb (when below 45 % of free device memory)."""
    return int(float(gb) * 1e9)


def wave_sizes(jobs, R, budget):
    """Jobs per memory wave."""
    sizes, cur, in_wave = [], 0, 0
    for job in jobs:
        b = job_bt_bytes(job, R)
        if in_wave and cur + b > budget:
            sizes.append(in_wave)
            cur, in_wave = 0, 0
        cur += b
        in_wave += 1
    sizes.append(in_wave)
    return sizes


# ------------------------------------------------------------------------------------------------ null model
def null_model(p_raw, t_pav, q_pav, pb, columnscore):
    """HMM::IncludeNullModelInHMM on every row 0..L+1 of a template profile (columnscores 0..3)."""
    p_raw = np.asarray(p_raw, np.float32)
    t_pav = np.asarray(t_pav, np.float32); q_pav = np.asarray(q_pav, np.float32)
    pn = {0: np.asarray(pb, np.float32), 1: np.float32(0.5) * (q_pav + t_pav), 2: t_pav, 3: q_pav}[columnscore]
    return (p_raw / pn[None, :]).astype(np.float32)


def raw_profile(prepared, rng):
    """A raw template (emissions before the null model) and its pav from a prepared synth profile: the prepared
    ratios times a background, so the null model brings them back to the same scale."""
    p, tr, ss = prepared
    bg = rng.dirichlet(np.ones(20) * 8).astype(np.float32)
    p_raw = (p * bg[None, :]).astype(np.float32)
    L = p.shape[0] - 2
    pav = (p_raw[1:L + 1].mean(axis=0) if L else bg).astype(np.float32)
    return (p_raw, tr, ss), pav


def region_mask(Lq, Lt, q_ranges, t_ranges):
    """Cell-off mask of -excl / -template_excl ranges (1-based, inclusive; ranges past the end are cut)."""
    m = np.zeros((Lq + 1, Lt + 1), np.uint8)
    for a, b in q_ranges:
        m[a:min(b, Lq) + 1, 1:] = 1
    for a, b in t_ranges:
        if a <= Lt:
            m[1:, a:min(b, Lt) + 1] = 1
    return m


# ------------------------------------------------------------------------------------------------ builders
def queries(lengths, seed):
    """Prepared synth queries: list of dict(p, tr, ss, pav, mix)."""
    out = []
    for k, L in enumerate(lengths):
        p, tr, ss, pav, mix = synth.query_profile(int(L), seed + 31 * k)
        out.append(dict(p=p, tr=tr, ss=ss, pav=pav, mix=mix))
    return out


def plant_tail(target, q_mix):
    """Overwrite the target's last len(q_mix) columns with a prepared copy of the query columns q_mix (pass the
    query's last columns), so the best alignment ends in the last row of the query and the last column of the target."""
    p, tr, ss = target
    n = q_mix.shape[0]
    L = p.shape[0] - 2
    p = p.copy()
    # four times the prepared ratio: every step of the planted diagonal gains about two bits, so the best cell is the
    # last one of the diagonal
    p[L - n + 1:L + 1] = (4.0 * (0.85 * q_mix + 0.15 * synth._PB[None, :]) / synth._PB[None, :]).astype(np.float32)
    return p, tr, ss


def _target_lengths(rng, n, hi):
    """Edges first, then log-normal lengths around 200 clipped to [1, hi], a few long ones up to hi."""
    lens = list(TARGET_EDGES)
    lens += [int(x) for x in np.clip(np.round(np.exp(rng.normal(np.log(200), 0.7, n - len(lens) - 4))), 1, hi)]
    lens += [hi, hi - 1, int(rng.integers(hi // 2, hi)), 64]
    return lens


def make_batch(kind, seed=1):
    """dict(queries, targets, req_q, ids, q_lens, t_lens).

    scan:      QUERY_LENGTHS plus three more long queries; the long queries (Lq >= 400) have several hundred
               requests each against short targets (1..48 columns), the others up to 200 requests against targets of
               up to 3000 columns: >= 4 * 132 * 8 work items of 16 rows, so the automatic strip height is 16.
    survivors: QUERY_LENGTHS with 0..60 requests each: the automatic strip height is 8.
    Both: COUNT_EDGES requests for the first four queries, planted homologs, duplicate (query, target) pairs and
    requests of all queries interleaved at random."""
    rng = np.random.default_rng(seed)
    scan = kind == "scan"
    q_lens = QUERY_LENGTHS + ((1500, 1000, 400) if scan else ())
    qs = queries(q_lens, 100 * seed + (7 if scan else 3))
    lens = _target_lengths(rng, 400 if scan else 160, 3000)
    short = [int(x) for x in rng.integers(1, 49, 120)] + list(TARGET_EDGES) if scan else []
    tg = []
    for k, L in enumerate(lens + short):
        base = qs[k % len(qs)]["mix"] if k % 3 == 0 else None
        tg.append(synth.prepared_profile(int(L), rng, base, noise=0.3))
    n_long = len(lens)
    short_ids = np.arange(n_long, len(tg))
    req_q, ids = [], []
    for q, L in enumerate(q_lens):
        if q < len(COUNT_EDGES):
            cnt = COUNT_EDGES[q]
        elif scan and L >= 400:
            cnt = int(rng.integers(380, 430))
        else:
            cnt = int(rng.integers(2, 200 if scan else 60))
        pool = short_ids if (scan and L >= 400) else np.arange(n_long)
        sel = rng.choice(pool, cnt, replace=True)
        if cnt >= 4:
            sel[1] = sel[0]                      # an exact duplicate (query, target) pair
        req_q += [q] * cnt
        ids += [int(x) for x in sel]
    perm = rng.permutation(len(ids))
    req_q = np.asarray(req_q, np.int32)[perm]; ids = np.asarray(ids, np.int32)[perm]
    t_lens = np.array([t[0].shape[0] - 2 for t in tg], np.int32)
    return dict(kind=kind, queries=qs, targets=tg, req_q=req_q, ids=ids, q_lens=np.asarray(q_lens, np.int32),
                t_lens=t_lens)


def request_lengths(batch):
    """(Lq, Lt) of every request."""
    return batch["q_lens"][batch["req_q"]], batch["t_lens"][batch["ids"]]
