"""Host-side mirror of Prefilter::prefilter_db (src/hhprefilter.cpp:430-606) on top of the C-ABI: both
scoring stages run on the GPU (ungapped DPX kernel over the whole cs219 shard, lane-exact gapped byte SW
over the survivors); the selection logic between and after them is the reference's, restated:

  stage 1: score = raw - (int)(bit_factor*(flog2(Lq)+flog2(Lt)))  (:477); sort descending by (score, n)
           (comparePair + reverse, :489-490); keep entries while count < min_prefilter_hits or
           score > smax_thresh (:494-506)
  stage 2: evalue = N*Lq*Lt*fpow2(-score/bit_factor) (integer division, :529); keep evalue < coarse
           threshold (:530); sort ascending by ((int)evalue, n) (:545: comparePair takes std::pair<int,int>, so the
           double E-value is truncated to int by the implicit conversion); keep while count < min_prefilter_hits or
           evalue <= evalue_thresh (:547-558); cap at maxnumdb (:590)

Returned: sequence ids in the reference's output order.  Name de-duplication and the old/new split by
``previous_hits`` (:561-588) operate on ffindex entry names and stay in the reference host code."""
from __future__ import annotations

import numpy as np

from . import capi


def prefilter_db(csdb: capi.CsDB, prof: np.ndarray, gap_open=20, gap_extend=4, score_offset=50, bit_factor=4,
                 evalue_thresh=1000.0, evalue_coarse_thresh=100000.0, smax_thresh=10, min_prefilter_hits=100,
                 maxnumdb=20000, return_details=False, device_select=True):
    """device_select=True (default): the stage-1 list is chosen on the GPU (hhg_prefilter_select: histogram +
    compaction), only survivors cross PCIe.  False: all N raw scores are fetched and sorted on the host (the
    formulation closest to the reference's loop; kept as the cross-check of the device path)."""
    L = capi.load()
    Lq = prof.shape[1]
    n = csdb.n
    lens = csdb.Lh
    import ctypes as C
    lens32 = np.ascontiguousarray(lens, np.int32)
    raw = corr = None
    if device_select:
        csdb.run(prof, score_offset)
        first, first_scores = csdb.select(Lq, bit_factor, smax_thresh, min_prefilter_hits)
    else:
        raw = csdb.ungapped(prof, score_offset)
        corr32 = np.zeros(n, np.int32)
        raw32 = np.ascontiguousarray(raw, np.int32)
        capi._ck(L.hhg_prefilter_corrected_scores(n, capi._p(raw32, capi.c_i32p), capi._p(lens32, capi.c_i32p), Lq,
                                                 bit_factor, capi._p(corr32, capi.c_i32p)))
        corr = corr32.astype(np.int64)
        order = np.lexsort((np.arange(n), corr))[::-1]          # descending (score, n)
        # keep while count < min_prefilter_hits or score > smax_thresh: first position (>= min hits) whose
        # score is <= smax_thresh ends the list
        stop = np.nonzero(corr[order[min_prefilter_hits:]] <= smax_thresh)[0]
        ncut = min_prefilter_hits + int(stop[0]) if len(stop) else n
        first = order[:min(ncut, n)].astype(np.int32)
        first_scores = corr32[first]
    sw = csdb.sw(prof, ids=first, gap_open=gap_open + gap_extend, gap_extend=gap_extend, bias=score_offset) \
        if len(first) else np.zeros(0, np.int32)
    ids, ev = _stage2(csdb, Lq, first, sw, bit_factor, evalue_thresh, evalue_coarse_thresh, min_prefilter_hits, maxnumdb)
    if return_details:
        return ids, dict(raw=raw, corrected=corr, first=first, first_scores=first_scores, sw=sw, evalue=ev)
    return ids


def _stage2(csdb, Lq, first, sw, bit_factor, evalue_thresh, evalue_coarse_thresh, min_prefilter_hits, maxnumdb):
    """E-values of the stage-2 scores and the final cut (:529-590) on the host: (ids, evalues)."""
    import ctypes as C
    L = capi.load()
    ev = np.zeros(len(first), np.float64)
    if len(first):
        sw32 = np.ascontiguousarray(sw, np.int32)
        fl = np.ascontiguousarray(np.asarray(csdb.Lh, np.int32)[first])
        capi._ck(L.hhg_prefilter_evalues(len(first), capi._p(sw32, capi.c_i32p), capi._p(fl, capi.c_i32p), csdb.n, Lq,
                                        bit_factor, ev.ctypes.data_as(C.POINTER(C.c_double))))
    # coarse cut (:530), sort ascending by ((int)evalue, index) (:545), keep rule (:547-558), maxnumdb (:590) -- vectorised
    keep = np.nonzero(ev < evalue_coarse_thresh)[0]
    order = keep[np.lexsort((first[keep], ev[keep].astype(np.int64)))]
    tail = np.nonzero(ev[order[min_prefilter_hits:]] > evalue_thresh)[0]
    ncut = min_prefilter_hits + int(tail[0]) if len(tail) else len(order)
    out = order[:min(ncut, maxnumdb)]
    return (first[out] if len(out) else np.zeros(0, np.int32)), ev


def prefilter_db_batch(csdb: capi.CsDB, profs, gap_open=20, gap_extend=4, score_offset=50, bit_factor=4,
                       evalue_thresh=1000.0, evalue_coarse_thresh=100000.0, smax_thresh=10, min_prefilter_hits=100,
                       maxnumdb=20000) -> list[np.ndarray]:
    """prefilter_db for many queries against one shard (hhblits_omp): one ungapped batch run, one stage-1 selection
    and one stage-2 launch for all queries, then each query's E-values and final cut on the host.  Returns one id
    array per profile, equal to [prefilter_db(csdb, p, ...) for p in profs].  A batch whose score rows exceed the
    context's memory budget (HHG_MAX_BT_GB) runs in consecutive groups of csdb.max_batch() queries."""
    profs = [np.ascontiguousarray(p, np.uint8) for p in profs]
    kw = dict(gap_open=gap_open, gap_extend=gap_extend, score_offset=score_offset, bit_factor=bit_factor,
              evalue_thresh=evalue_thresh, evalue_coarse_thresh=evalue_coarse_thresh, smax_thresh=smax_thresh,
              min_prefilter_hits=min_prefilter_hits, maxnumdb=maxnumdb)
    group = csdb.max_batch()
    if len(profs) > group:
        return [ids for g in range(0, len(profs), group) for ids in prefilter_db_batch(csdb, profs[g:g + group], **kw)]
    Lq = [p.shape[1] for p in profs]
    csdb.run_batch(profs, score_offset)
    firsts = [f for f, _ in csdb.select_batch(Lq, bit_factor, smax_thresh, min_prefilter_hits)]
    rq = np.concatenate([np.full(len(f), q, np.int32) for q, f in enumerate(firsts)])
    sw = csdb.sw_batch(profs, rq, np.concatenate(firsts), gap_open=gap_open + gap_extend, gap_extend=gap_extend,
                       bias=score_offset)
    bounds = np.concatenate([[0], np.cumsum([len(f) for f in firsts])])
    return [_stage2(csdb, Lq[q], firsts[q], sw[bounds[q]:bounds[q + 1]], bit_factor, evalue_thresh,
                    evalue_coarse_thresh, min_prefilter_hits, maxnumdb)[0] for q in range(len(profs))]
