"""Host-side mirror of the reference's ViterbiRunner (src/hhviterbirunner.{h,cpp}) on top of the C-ABI.

``ViterbiRunner.alignment`` reproduces the control flow of ViterbiRunner::alignment
(src/hhviterbirunner.cpp:75-210) for the part that lives on the hot path:

  * pass 0 aligns every requested target; pass k>0 ("alternative alignments", par.altali, default 4)
    re-aligns only the targets whose previous hit scored above par.smin (default 20), with ALL of that
    target's earlier paths masked by the +-40 cross of Viterbi::ExcludeAlignment
    (merge_thread_results :249-271, exclude_alignments :273-289);
  * every (target, pass) yields one hit with irep = pass+1 (:257) and lastrep = (score <= smin) (:36);
  * hit.score is Hit.score (ScoreForBacktrace), computed on the device.

Two reference behaviours make results depend on the ORDER and BATCHING of the target list; both are mirrored:

  * the hhblits early-stopping filter (:109-111, 178-188, 213-247): the first pass walks the list in chunks of 2000
    and stops after a chunk whose hits sum to less than chunk_size * filter_thresh in 1/(1+Eval)
    (``early_stopping=dict(filter_thresh=0.01, dbsize=..., prefilter=True, q_neff=..., t_neff=...)``);
  * the ss mode is the consensus over the 8 lanes of a batch (:14-22), batches being cut from the chunk after a
    sort by HHEntry::sequence_length (``ss=dict(q_pred=..., t_pred=..., seqlen=...)``).  The reference sorts with
    std::sort (unstable); this mirror uses a stable sort, which is the same whenever the lengths of a chunk are
    distinct -- the C++ adapter (oracle/ref_gpu_adapter.cpp) calls std::sort itself and is exact in all cases."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from . import capi


@dataclass
class Hit:
    target: int          # index into the shard (the reference carries an HHEntry*)
    irep: int            # 1-based index of the alternative alignment (Hit::irep)
    lastrep: int         # 1 if score <= smin (Hit::lastrep)
    score: float         # Hit.score (with correlation term)
    score_ss: float
    vit_score: float     # raw Viterbi score (ViterbiResult::score)
    i1: int
    i2: int
    j1: int
    j2: int
    nsteps: int
    matched_cols: int
    i: np.ndarray = field(repr=False, default=None)       # i_steps[1..nsteps]
    j: np.ndarray = field(repr=False, default=None)
    states: np.ndarray = field(repr=False, default=None)


class ViterbiRunner:
    def __init__(self, ctx: capi.Context, db: capi.TargetDB, altali: int = 4, smin: float = 20.0, ssm: int = 2,
                 early_stopping: dict | None = None, ss: dict | None = None):
        self.ctx, self.db = ctx, db
        self.altali, self.smin, self.ssm = altali, smin, ssm
        self.early_stopping, self.ss = early_stopping, ss
        self.early_stopped_at = -1

    def _ss_groups(self, chunk):
        """Split a chunk into (targets aligned without, with) the ss term: length sort, batches of 8, consensus."""
        if self.ss is None:
            return [chunk, chunk[:0]]
        seqlen = np.asarray(self.ss["seqlen"])
        order = chunk[np.argsort(-seqlen[chunk], kind="stable")]
        t_pred = np.asarray(self.ss["t_pred"], bool)
        use = np.zeros(len(order), bool)
        for b in range(0, len(order), 8):
            use[b:b + 8] = bool(self.ss["q_pred"]) and self.ssm == 2 and bool(t_pred[order[b:b + 8]].all())
        return [order[~use], order[use]]

    def alignment(self, ids=None) -> list[Hit]:
        ids = np.arange(self.db.n, dtype=np.int32) if ids is None else np.ascontiguousarray(ids, np.int32)
        todo = ids
        excl: dict[int, list[tuple[np.ndarray, np.ndarray]]] = {}
        out: list[Hit] = []
        es = self.early_stopping
        for rep in range(self.altali):
            if len(todo) == 0:
                break
            block = 2000 if (rep == 0 and es) else max(len(todo), 1)
            nxt = []
            for start in range(0, len(todo), block):
                chunk = todo[start:start + block]
                first = len(out)
                for g, grp in enumerate(self._ss_groups(chunk)):
                    if len(grp) == 0:
                        continue
                    if self.ss is not None:
                        capi._ck(self.ctx.L.hhg_set_use_ss(self.ctx.h, g))
                    self._align_group(grp, rep, excl, out, nxt)
                if rep == 0 and es:
                    new = out[first:]
                    s = capi.early_stop_sum([h.score for h in new], self.db.Lh[[h.target for h in new]],
                                            np.asarray(es["t_neff"], np.float32)[[h.target for h in new]], self.ctx.Lq,
                                            es["q_neff"], es.get("prefilter", True), es["dbsize"])
                    if s < len(chunk) * es.get("filter_thresh", 0.01):
                        self.early_stopped_at = start + len(chunk)
                        break
            todo = np.array(nxt, np.int32)
        return out

    def _align_group(self, todo, rep, excl, out, nxt):
        exclusions = None
        if rep > 0:
            exclusions = []
            for t in todo:
                ii = np.concatenate([e[0] for e in excl[int(t)]])
                jj = np.concatenate([e[1] for e in excl[int(t)]])
                exclusions.append((ii, jj))
        hits, paths = capi.viterbi_search(self.ctx, self.db, ids=todo, exclusions=exclusions)
        for k, t in enumerate(todo):
            h = hits[k]
            gi, gj, gs = capi.expand_path(h, paths)
            n = int(h["nsteps"])
            out.append(Hit(int(t), rep + 1, 1 if h["hit_score"] <= self.smin else 0, float(h["hit_score"]),
                           float(h["score_ss"]), float(h["score"]), int(h["i1"]), int(h["i2"]), int(h["j1"]),
                           int(h["j2"]), n, int(h["matched_cols"]), gi, gj, gs))
            if h["hit_score"] > self.smin:
                nxt.append(int(t))
                # ExcludeAlignment masks steps 1 <= step < nsteps (src/hhviterbi.cpp:66)
                excl.setdefault(int(t), []).append((gi[1:n].copy(), gj[1:n].copy()))


class BatchViterbiRunner:
    """ViterbiRunner.alignment for every query of a batch at once (hhblits_omp runs one ViterbiRunner per query,
    src/hhblits_omp.cpp:119-160): pass 0 aligns every request, pass k > 0 realigns the (query, target) requests whose
    previous hit scored above smin with all earlier paths of that pair masked -- one hhg_viterbi_search_batch call per
    pass for all queries.  The queries are those of the last capi.query_set_batch; over a raw shard the null model is
    applied per query (columnscore / pb as in capi.viterbi_search_batch).  No early stopping and no per-batch ss
    consensus: split the requests by hhg_set_use_ss beforehand if the ss term is wanted for some of them."""

    def __init__(self, ctx: capi.Context, db: capi.TargetDB, altali: int = 4, smin: float = 20.0, columnscore: int = 1,
                 pb=None):
        self.ctx, self.db = ctx, db
        self.altali, self.smin = altali, smin
        self.columnscore, self.pb = columnscore, pb

    def alignment(self, req_query, ids) -> list[list[Hit]]:
        """Request k aligns query req_query[k] with target ids[k].  Returns one list of Hits per query of the batch,
        in the order ViterbiRunner.alignment(ids of that query) returns them."""
        rq = np.ascontiguousarray(req_query, np.int32); ids = np.ascontiguousarray(ids, np.int32)
        out: list[list[Hit]] = [[] for _ in range(len(self.ctx.batch_Lq))]
        excl: dict[tuple[int, int], list[tuple[np.ndarray, np.ndarray]]] = {}
        todo = list(zip(rq.tolist(), ids.tolist()))
        for rep in range(self.altali):
            if not todo:
                break
            exclusions = None
            if rep > 0:
                exclusions = [(np.concatenate([e[0] for e in excl[p]]), np.concatenate([e[1] for e in excl[p]]))
                              for p in todo]
            hits, paths = capi.viterbi_search_batch(self.ctx, self.db, [q for q, _ in todo], [t for _, t in todo],
                                                    self.columnscore, self.pb, exclusions=exclusions)
            nxt = []
            for k, (q, t) in enumerate(todo):
                h = hits[k]
                gi, gj, gs = capi.expand_path(h, paths)
                n = int(h["nsteps"])
                out[q].append(Hit(t, rep + 1, 1 if h["hit_score"] <= self.smin else 0, float(h["hit_score"]),
                                  float(h["score_ss"]), float(h["score"]), int(h["i1"]), int(h["i2"]), int(h["j1"]),
                                  int(h["j2"]), n, int(h["matched_cols"]), gi, gj, gs))
                if h["hit_score"] > self.smin:
                    nxt.append((q, t))
                    # ExcludeAlignment masks steps 1 <= step < nsteps (src/hhviterbi.cpp:66)
                    excl.setdefault((q, t), []).append((gi[1:n].copy(), gj[1:n].copy()))
            todo = nxt
        return out
