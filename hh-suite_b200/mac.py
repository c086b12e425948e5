"""Host-side mirror of PosteriorDecoderRunner::executeComputation (src/hhposteriordecoderrunner.cpp:45-125) on top
of the C-ABI: hits are grouped per template and ordered by irep; round k realigns the k-th hit of every template in one
hhg_mac_realign call, excluding the MAC alignments found for that template in the earlier rounds (alt_i / alt_j,
:104-108)."""
from __future__ import annotations

import numpy as np

from . import capi


class MacResult:
    __slots__ = ("target", "irep", "i1", "i2", "j1", "j2", "nsteps", "matched_cols", "sum_of_probs", "pforward",
                 "i", "j", "states", "P_posterior")

    def __repr__(self):
        return (f"MacResult(target={self.target}, irep={self.irep}, {self.i1}-{self.i2}/{self.j1}-{self.j2}, "
                f"nsteps={self.nsteps}, sum_of_probs={self.sum_of_probs:.3f})")


def realign(ctx: capi.Context, db: capi.TargetDB, q_p, q_tr, hits, local=True, shift=-0.03, mact=0.35):
    """hits: objects with .target, .irep, .i1, .i2, .j1, .j2, .nsteps, .i, .j (runner.Hit of the Viterbi stage;
    step arrays 1-based).  q_tr: the query's log2 transitions as used by Viterbi; they are put into linear space the
    way the reference does (HMM::Log2LinTransitionProbs).  Returns {(target, irep): MacResult}."""
    capi.mac_query_set(ctx, q_p, capi.log2lin(q_tr))
    by_target: dict[int, list] = {}
    for h in hits:
        if h.nsteps > 0:                      # a hit without a Viterbi alignment has no band to realign in
            by_target.setdefault(int(h.target), []).append(h)
    for v in by_target.values():
        v.sort(key=lambda h: h.irep)
    out = {}
    alt: dict[int, tuple[list, list]] = {t: ([], []) for t in by_target}
    rnd = 0
    while True:
        batch = [v[rnd] for v in by_target.values() if len(v) > rnd]
        if not batch:
            break
        targets = [int(h.target) for h in batch]
        vits = [(h.i1, h.i2, h.j1, h.j2, h.nsteps, h.i, h.j) for h in batch]
        excl = [(np.array(alt[t][0], np.int32), np.array(alt[t][1], np.int32)) for t in targets] if rnd else None
        mh, paths = capi.mac_realign(ctx, db, targets, vits, excl, local=local, shift=shift, mact=mact)
        for r, h in enumerate(batch):
            m = MacResult()
            m.target, m.irep = int(h.target), int(h.irep)
            for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols"):
                setattr(m, f, int(mh[f][r]))
            m.sum_of_probs = float(mh["sum_of_probs"][r]); m.pforward = float(mh["pforward"][r])
            m.i, m.j, m.states, m.P_posterior = paths[r]["i"], paths[r]["j"], paths[r]["states"], paths[r]["P_posterior"]
            out[(m.target, m.irep)] = m
            # hit.alt_i / alt_j collect every (i, j) the backtrace visited, including the step-0 entry of an empty path
            if m.nsteps:
                alt[m.target][0].extend(m.i[1:].tolist()); alt[m.target][1].extend(m.j[1:].tolist())
            else:
                alt[m.target][0].append(int(m.i[0]) if len(m.i) else m.i2); alt[m.target][1].append(int(m.j[0]) if len(m.j) else m.j2)
        rnd += 1
    return out


def realign_batch(ctx: capi.Context, db: capi.TargetDB, queries, hits, q_pav=None, columnscore=1, pb=None, local=True,
                  shift=-0.03, mact=0.35):
    """realign for every query of a batch at once.  queries: list of (q_p, q_tr) as realign takes them; hits[q]: the
    Viterbi hits of query q (e.g. runner.BatchViterbiRunner.alignment); q_pav [nq, 20], columnscore and pb: the null
    model of a raw shard (hhg_mac_realign_batch).  Round k realigns the k-th hit (in irep order) of every (query, target)
    pair of all queries in one call, excluding the MAC alignments found for that pair before.  Returns one
    {(target, irep): MacResult} per query."""
    capi.mac_query_set_batch(ctx, [(q[0], capi.log2lin(q[1])) for q in queries], q_pav)
    by_pair: dict[tuple[int, int], list] = {}
    for q, hq in enumerate(hits):
        for h in hq:
            if h.nsteps > 0:                  # a hit without a Viterbi alignment has no band to realign in
                by_pair.setdefault((q, int(h.target)), []).append(h)
    for v in by_pair.values():
        v.sort(key=lambda h: h.irep)
    out = [{} for _ in queries]
    alt: dict[tuple[int, int], tuple[list, list]] = {p: ([], []) for p in by_pair}
    rnd = 0
    while True:
        pairs = [p for p, v in by_pair.items() if len(v) > rnd]
        if not pairs:
            break
        batch = [by_pair[p][rnd] for p in pairs]
        vits = [(h.i1, h.i2, h.j1, h.j2, h.nsteps, h.i, h.j) for h in batch]
        excl = [(np.array(alt[p][0], np.int32), np.array(alt[p][1], np.int32)) for p in pairs] if rnd else None
        mh, paths = capi.mac_realign_batch(ctx, db, [q for q, _ in pairs], [t for _, t in pairs], vits, excl,
                                           columnscore, pb, local=local, shift=shift, mact=mact)
        for r, ((q, t), h) in enumerate(zip(pairs, batch)):
            m = MacResult()
            m.target, m.irep = t, int(h.irep)
            for f in ("i1", "i2", "j1", "j2", "nsteps", "matched_cols"):
                setattr(m, f, int(mh[f][r]))
            m.sum_of_probs = float(mh["sum_of_probs"][r]); m.pforward = float(mh["pforward"][r])
            m.i, m.j, m.states, m.P_posterior = paths[r]["i"], paths[r]["j"], paths[r]["states"], paths[r]["P_posterior"]
            out[q][(m.target, m.irep)] = m
            # hit.alt_i / alt_j collect every (i, j) the backtrace visited, including the step-0 entry of an empty path
            if m.nsteps:
                alt[(q, t)][0].extend(m.i[1:].tolist()); alt[(q, t)][1].extend(m.j[1:].tolist())
            else:
                alt[(q, t)][0].append(int(m.i[0]) if len(m.i) else m.i2); alt[(q, t)][1].append(int(m.j[0]) if len(m.j) else m.j2)
        rnd += 1
    return out


def to_global(db: capi.StagedDB, results: dict) -> dict:
    """The results of realign / one query's results of realign_batch over a staged shard (hits with LOCAL targets, all
    still resident), re-keyed and relabelled with the store's global ids.  Call before the next db.stage()."""
    g = db.to_global([t for t, _ in results])
    out = {}
    for (_, irep), t, m in zip(results, g, results.values()):
        m.target = int(t)
        out[(int(t), irep)] = m
    return out
