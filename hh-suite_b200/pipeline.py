"""One HHblits-style search iteration on the hot path (src/hhblits.cpp:1118-1221): two-stage cs219
prefilter over the whole shard, then Viterbi (with alternative alignments) on the survivors.
Everything between the stages is the reference's selection logic (prefilter.py, runner.py)."""
from __future__ import annotations

import dataclasses

import numpy as np

from . import capi, prefilter, runner


def search(ctx: capi.Context, db: capi.TargetDB, csdb: capi.CsDB, q_p, q_tr, q_pav, lib219, q_prefilter_p=None,
           altali=4, smin=20.0, cs_names=None, db_names=None, **pf_kwargs):
    """q_p/q_tr: prepared query (Viterbi); q_prefilter_p: HMM::p of the prefilter-pseudocount copy of the query
    (q_tmp, src/hhblits.cpp:1149-1163; defaults to q_p).  Returns (survivor ids in the TARGET shard, list of runner.Hit).
    Under column score 5 (db prepared by apply_null_model(pb=pb, columnscore=5)) pass q_p divided by
    capi.query_local_background and the undivided p as q_prefilter_p: the prefilter never sees the division.

    The prefilter's survivors are entries of the cs219 index; the reference carries them to the Viterbi stage BY NAME
    (src/hhprefilter.cpp:561-590, then a lookup in the hhm/a3m index), because the two indices of a real database
    need not list the same entries in the same order.  Pass both name lists (cs_names[k] = name of cs219 sequence k,
    db_names[t] = name of target t) to map by name; without them the two shards must be index-aligned, which is
    checked as far as it can be (same number of entries, same lengths)."""
    prof = capi.build_prefilter_profile(q_p if q_prefilter_p is None else q_prefilter_p, q_pav, lib219,
                                        pf_kwargs.get("score_offset", 50), pf_kwargs.get("bit_factor", 4))
    ids = _to_targets(prefilter.prefilter_db(csdb, prof, **pf_kwargs), db, csdb, cs_names, db_names)
    ctx.set_query(q_p, q_tr)
    hits = runner.ViterbiRunner(ctx, db, altali=altali, smin=smin).alignment(ids) if len(ids) else []
    return ids, hits


def search_batch(ctx: capi.Context, db: capi.TargetDB, csdb: capi.CsDB, queries, lib219, altali=4, smin=20.0,
                 cs_names=None, db_names=None, **pf_kwargs):
    """search() for many queries against one database (hhblits_omp): queries = list of (q_p, q_tr, q_pav) or
    (q_p, q_tr, q_pav, q_prefilter_p).  The prefilter of all queries runs as one batch
    (prefilter.prefilter_db_batch), the survivors are mapped to the target shard as in search(), and the Viterbi
    stage aligns every query with its own survivors through capi.query_set_batch and runner.BatchViterbiRunner.
    Returns one (survivor ids in the TARGET shard, list of runner.Hit) pair per query.

    BatchViterbiRunner has no early stopping and no per-8-lane ss consensus, unlike runner.ViterbiRunner; search()
    uses neither, so the results equal [search(ctx, db, csdb, *q, lib219, ...) for q in queries] for the settings the
    two runners share.  The batch replaces the context's query (capi.query_set_batch)."""
    so, bf = pf_kwargs.get("score_offset", 50), pf_kwargs.get("bit_factor", 4)
    profs = [capi.build_prefilter_profile(q[0] if len(q) < 4 or q[3] is None else q[3], q[2], lib219, so, bf)
             for q in queries]
    ids = [_to_targets(x, db, csdb, cs_names, db_names) for x in prefilter.prefilter_db_batch(csdb, profs, **pf_kwargs)]
    capi.query_set_batch(ctx, [(q[0], q[1]) for q in queries])
    rq = np.concatenate([np.full(len(x), q, np.int32) for q, x in enumerate(ids)])
    hits = runner.BatchViterbiRunner(ctx, db, altali=altali, smin=smin).alignment(rq, np.concatenate(ids)) \
        if len(rq) else [[] for _ in queries]
    return list(zip(ids, hits))


def search_staged(ctx: capi.Context, db: capi.StagedDB, csdb: capi.CsDB, q_p, q_tr, q_pav, lib219, q_prefilter_p=None,
                  altali=4, smin=20.0, cs_names=None, db_names=None, columnscore=1, pb=None, **pf_kwargs):
    """search() over a database whose profiles stay in host memory (db.store: a HostStore, or a RecordSource whose
    survivors are built from their records as they are staged): the prefilter's survivors are staged into db (one
    hhg_db_stage call), the query's null model is applied to the staged records (columnscore / pb as in
    TargetDB.apply_null_model) and the same runner aligns them.  Returns what search() returns over a resident raw shard
    of the whole database after apply_null_model(q_pav, pb, columnscore): survivor ids and Hit.target are GLOBAL ids.
    The survivors of one query must fit db (HhgError otherwise, with the sizes needed).  With columnscore 5, q_p is the
    undivided query: the prefilter profile is built from it and the Viterbi stage aligns its local composition
    correction (capi.query_local_background with the context's half window), as hhblits does."""
    prof = capi.build_prefilter_profile(q_p if q_prefilter_p is None else q_prefilter_p, q_pav, lib219,
                                        pf_kwargs.get("score_offset", 50), pf_kwargs.get("bit_factor", 4))
    if columnscore == 5:
        q_p = capi.query_local_background(ctx, q_p, pb)
    ids = _to_targets(prefilter.prefilter_db(csdb, prof, **pf_kwargs), db.store, csdb, cs_names, db_names)
    if not len(ids):
        return ids, []
    local = db.stage(ids)
    _check_staged(db, csdb, ids, local, cs_names, db_names)
    db.apply_null_model(q_pav, pb, columnscore)
    ctx.set_query(q_p, q_tr)
    hits = runner.ViterbiRunner(ctx, db, altali=altali, smin=smin).alignment(local)
    return ids, to_global_hits(db, hits)


def search_batch_staged(ctx: capi.Context, db: capi.StagedDB, csdb: capi.CsDB, queries, lib219, altali=4, smin=20.0,
                        cs_names=None, db_names=None, columnscore=1, pb=None, **pf_kwargs):
    """search_batch() over a database whose profiles stay in host memory: the union of all queries' survivors is staged
    in one call, then the batch runner aligns every query with its own survivors, the null model of each query fused
    into the search (so q_pav of every query is used: pass (q_p, q_tr, q_pav[, q_prefilter_p]) as for search_batch).
    Returns what search_batch() returns over a resident raw shard of the whole database, with GLOBAL ids.  The union
    must fit db.  With columnscore 5 each q_p is undivided, as in search_staged."""
    so, bf = pf_kwargs.get("score_offset", 50), pf_kwargs.get("bit_factor", 4)
    profs = [capi.build_prefilter_profile(q[0] if len(q) < 4 or q[3] is None else q[3], q[2], lib219, so, bf)
             for q in queries]
    if columnscore == 5:
        queries = [(capi.query_local_background(ctx, q[0], pb),) + tuple(q[1:]) for q in queries]
    ids = [_to_targets(x, db.store, csdb, cs_names, db_names)
           for x in prefilter.prefilter_db_batch(csdb, profs, **pf_kwargs)]
    rq = np.concatenate([np.full(len(x), q, np.int32) for q, x in enumerate(ids)])
    if not len(rq):
        return [(x, []) for x in ids]
    local = db.stage(np.concatenate(ids))
    _check_staged(db, csdb, np.concatenate(ids), local, cs_names, db_names)
    capi.query_set_batch(ctx, [(q[0], q[1]) for q in queries], q_pav=np.stack([q[2] for q in queries]))
    hits = runner.BatchViterbiRunner(ctx, db, altali=altali, smin=smin, columnscore=columnscore, pb=pb).alignment(rq, local)
    return [(x, to_global_hits(db, h)) for x, h in zip(ids, hits)]


def to_global_hits(db: capi.StagedDB, hits):
    """Hits of a search over a staged shard with Hit.target translated from local to global ids (new objects; use
    before the next stage() call, and give mac.realign the LOCAL hits)."""
    if not hits:
        return []
    g = db.to_global([h.target for h in hits])
    return [dataclasses.replace(h, target=int(t)) for h, t in zip(hits, g)]


def _to_targets(ids, db, csdb, cs_names, db_names):
    """Prefilter survivors (cs219 index) -> target shard index, by name when the name lists are given."""
    if cs_names is not None or db_names is not None:
        if cs_names is None or db_names is None:
            raise ValueError("pass both cs_names and db_names, or neither")
        where = {nm: t for t, nm in enumerate(db_names)}
        missing = [cs_names[k] for k in ids if cs_names[k] not in where]
        if missing:
            raise KeyError(f"{len(missing)} prefilter hits have no entry in the profile shard, e.g. {missing[0]!r}")
        return np.array([where[cs_names[k]] for k in ids], np.int32)
    # a record source knows the lengths only of what it has scanned: the count here, each survivor's length once staged
    if csdb.n != db.n or (not isinstance(db, capi.RecordSource) and not np.array_equal(np.asarray(csdb.Lh), np.asarray(db.Lh))):
        raise ValueError(_NOT_ALIGNED)
    return ids


_NOT_ALIGNED = ("cs219 shard and profile shard are not index-aligned (different sizes or lengths): "
                "pass cs_names / db_names so the survivors are mapped by name like the reference does")


def _check_staged(db: capi.StagedDB, csdb, ids, local, cs_names, db_names):
    """The length check of _to_targets for survivors staged from a record source: staged length == cs219 length."""
    if cs_names is None and db_names is None and isinstance(db.store, capi.RecordSource) and \
            not np.array_equal(np.asarray(db.Lh)[local], np.asarray(csdb.Lh)[ids]):
        raise ValueError(_NOT_ALIGNED)


def translate_cs219(p_cols: np.ndarray, pav_like: np.ndarray, lib219: np.ndarray) -> np.ndarray:
    """Nearest column state for synthetic data: argmax_k sum_a p[a] * lib[k][a] / bg[a] (the same score
    the prefilter profile is built from).  A stand-in for the reference's cstranslate on synthetic shards."""
    w = (lib219 / pav_like[None, :]).astype(np.float32)        # [219, 20]
    return np.argmax(p_cols.astype(np.float32) @ w.T, axis=1).astype(np.uint8)
