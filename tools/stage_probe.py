"""What a host-resident database costs (DESIGN 4.12): a resident raw shard and a staged shard over a page-locked store,
alternated in one process on the configs[2] shape (N synthetic profiles, Lq = 400, ~3 000 prefilter survivors).

  gather    k_stage_gather alone: device time (events on the context stream, which waits for the gather) and GB/s of
            cold stage calls of 3 000 and 20 000 targets for several grid sizes, next to one cudaMemcpyAsync of as many
            contiguous page-locked bytes; host time of a stage call that finds everything resident
  search    null model + search per query, resident vs staged: cold cache, then a stream of 16 related queries
  batch     the 16 queries as one batch, resident vs staged
  memory    device and page-locked host memory each arm holds

Records are random (timing does not depend on their values); the cs219 sequences are random too, so the prefilter keeps
its minimum number of hits, set to the survivor count wanted.  Times are best of --reps and the spread (max - min)."""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "nvidia-smi not available"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=300000)
    ap.add_argument("--survivors", type=int, default=3000)
    ap.add_argument("--lq", type=int, default=400)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import hhsuite_b200 as hh
    from hhsuite_b200 import capi, prefilter, runner, synth

    if not torch.cuda.is_available():
        sys.exit("stage_probe needs an H100: there is nothing to measure without one")
    print("card:", card_state(), "(sampled before the run)")
    stream = torch.cuda.current_stream()
    ctx = hh.Context(device=0, stream=stream.cuda_stream)
    rng = np.random.default_rng(1)

    def dev_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream); fn(); e1.record(stream); e1.synchronize()
        return e0.elapsed_time(e1)

    def host_ms(fn):
        ctx.sync(); t = time.perf_counter(); fn(); ctx.sync()
        return (time.perf_counter() - t) * 1e3

    def stat(xs):
        return f"{min(xs):9.3f} ms (spread {max(xs) - min(xs):.3f})"

    # ---- the database: a chunk of 20 000 random targets repeated; store, resident shard, cs219 shard
    chunk_n = 20000
    reps_db = (a.n + chunk_n - 1) // chunk_n
    Lc = synth.lengths(chunk_n, rng, median=200)
    cols = np.zeros(int(Lc.sum()), capi.COLREC_DTYPE)
    cols["p"] = rng.random((len(cols), 20), np.float32) * 0.1 + 0.001
    for f in ("m2m", "m2d", "d2m", "d2d", "i2m", "i2i", "m2i"):
        cols[f] = -rng.random(len(cols), np.float32) * 3
    pav = np.full((chunk_n, 20), 0.05, np.float32)
    n = chunk_n * reps_db
    L = np.tile(Lc, reps_db)
    free0 = torch.cuda.mem_get_info()[0]
    store = hh.HostStore(ctx, n, int(L.sum()))
    for _ in range(reps_db):
        store.append_packed(Lc, cols, pav)
    free1 = torch.cuda.mem_get_info()[0]
    db = hh.TargetDB.from_packed(ctx, L, np.tile(cols, reps_db), np.tile(pav, (reps_db, 1)))
    free2 = torch.cuda.mem_get_info()[0]
    cs = synth.cs219_db(n, 7, lens=L)
    cst = hh.CsDB(ctx, cs["L"], cs["off"], cs["seq"])
    cap_t = 25000
    cap_c = int(cap_t * float(L.mean()) * 1.3)
    sdb = hh.StagedDB(ctx, store, cap_t, cap_c)
    free3 = torch.cuda.mem_get_info()[0] + cs["seq"].nbytes
    print(f"database: {n} targets, {int(L.sum())} columns; staged shard: {cap_t} slots, {cap_c} columns")
    print(f"memory   resident arm: {(free1 - free2) / 1e9:.2f} GB device, 0 page-locked host")
    print(f"memory   staged arm:   {(free0 - free1 + free2 - free3) / 1e9:.2f} GB device, "
          f"{(int(L.sum()) * 112 + n * 80) / 1e9:.2f} GB page-locked host")

    # ---- gather alone
    block = 0
    for count in (a.survivors, 20000):
        nbytes = None
        pinned = torch.empty(int(count * float(L.mean()) * 112 * 1.2), dtype=torch.uint8).pin_memory()
        dst = torch.empty_like(pinned, device="cuda")
        res: dict[str, list] = {}
        for rep in range(a.reps + 1):                       # rep 0 warms up
            for ctas in (8, 16, 32, 64, 132):
                os.environ["HHG_STAGE_CTAS"] = str(ctas)
                ids = (rng.choice(40000, count, replace=False) + 40000 * (block % (n // 40000))).astype(np.int32)
                block += 1
                ms = dev_ms(lambda: sdb.stage(ids))
                assert sdb.last_stats["copied"] >= count * 0.8, sdb.last_stats
                nbytes = int(sdb.last_stats["bytes"])
                if rep:
                    res.setdefault(f"gather {ctas:3d} CTAs", []).append((ms, nbytes))
                ms = dev_ms(lambda: dst[:nbytes].copy_(pinned[:nbytes], non_blocking=True))
                if rep:
                    res.setdefault("cudaMemcpyAsync", []).append((ms, nbytes))
        os.environ.pop("HHG_STAGE_CTAS")
        for k, v in res.items():
            best = min(v)
            print(f"gather   {count:6d} targets  {k:16s} {stat([x[0] for x in v])}  best {best[1] / best[0] / 1e6:6.2f} GB/s "
                  f"({best[1] / 1e6:.1f} MB)")
    ids = rng.choice(n, a.survivors, replace=False).astype(np.int32)
    sdb.stage(ids)
    print(f"gather   warm call, {a.survivors} resident targets (host): {stat([host_ms(lambda: sdb.stage(ids)) for _ in range(a.reps)])}")

    # ---- search: 16 related queries (one profile, perturbed), survivors = the prefilter's minimum
    lib = np.load(os.path.join(ROOT, "tests", "golden", "golden_v1.npz"))["cs219_lin"]
    base = synth.query_profile(a.lq, 3)
    qs = []
    for k in range(16):
        p = base[0].copy()
        noise = rng.dirichlet(np.ones(20), a.lq).astype(np.float32)
        p[1:-1] = (1 - 0.02 * k) * p[1:-1] + 0.02 * k * noise
        qs.append((p, base[1], p[1:-1].mean(axis=0).astype(np.float32)))
    pfk = dict(min_prefilter_hits=a.survivors, maxnumdb=a.survivors)

    def resident(q):
        db.apply_null_model(q[2])
        return hh.pipeline.search(ctx, db, cst, q[0], q[1], q[2], lib, **pfk)

    def staged(q):
        return hh.pipeline.search_staged(ctx, sdb, cst, q[0], q[1], q[2], lib, **pfk)

    def resident_batch():
        profs = [capi.build_prefilter_profile(q[0], q[2], lib, 50, 4) for q in qs]
        ids = prefilter.prefilter_db_batch(cst, profs, **pfk)
        capi.query_set_batch(ctx, [(q[0], q[1]) for q in qs], q_pav=np.stack([q[2] for q in qs]))
        rq = np.concatenate([np.full(len(x), k, np.int32) for k, x in enumerate(ids)])
        return ids, runner.BatchViterbiRunner(ctx, db, altali=4).alignment(rq, np.concatenate(ids))

    resident(qs[0]); staged(qs[0])                          # warm-up of every kernel and plan size
    t_nm = [host_ms(lambda: db.apply_null_model(qs[0][2])) for _ in range(a.reps)]
    cold_r, cold_s, st_r, st_s, b_r, b_s = [], [], [], [], [], []
    far = np.arange(cap_t, dtype=np.int32) + n - cap_t
    for rep in range(a.reps):
        cold_r.append(host_ms(lambda: resident(qs[0])))
        sdb.stage(far)                                      # push every survivor out: the next staged search is cold
        cold_s.append(host_ms(lambda: staged(qs[0])))
        st_r.append(host_ms(lambda: [resident(q) for q in qs]) / 16)
        sdb.stage(far)
        hits = [0, 0]

        def stream16():
            for q in qs:
                staged(q)
                hits[0] += int(sdb.last_stats["hits"]); hits[1] += int(sdb.last_stats["copied"])
        st_s.append(host_ms(stream16) / 16)
        b_r.append(host_ms(resident_batch))
        sdb.stage(far)
        b_s.append(host_ms(lambda: hh.pipeline.search_batch_staged(ctx, sdb, cst, qs, lib, **pfk)))
        union = int(sdb.last_stats["hits"] + sdb.last_stats["copied"])
    want, got = resident(qs[5]), staged(qs[5])
    assert want[0].tolist() == got[0].tolist() and [h.score for h in want[1]] == [h.score for h in got[1]]
    print(f"search   resident, null model over the whole shard alone:   {stat(t_nm)}")
    print(f"search   one query, resident (null model + search):         {stat(cold_r)}")
    print(f"search   one query, staged, cold cache:                      {stat(cold_s)}")
    print(f"search   per query in a stream of 16 related, resident:      {stat(st_r)}")
    print(f"search   per query in a stream of 16 related, staged:        {stat(st_s)}   "
          f"({hits[0]} resident hits, {hits[1]} targets copied over the 16)")
    print(f"batch    16 queries, resident (fused null model):            {stat(b_r)}")
    print(f"batch    16 queries, staged, cold cache ({union} distinct survivors): {stat(b_s)}")
    print("card:", card_state(), "(sampled after the run)")
    sdb.close(); store.close(); cst.close(); db.close(); ctx.close()


if __name__ == "__main__":
    main()
