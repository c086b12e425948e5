"""A record-sourced staged shard drives the unmodified StageCache (hh-suite_b200/csrc/hhg_stage_cache.h) with a length
table that only knows the records some request has named so far (hhg_db_stage scans a request's missing records before
it places them), and with the records' text offsets as source offsets.  Placement must not depend on either: local ids,
arena runs, evictions, freed slots and statistics equal those of a store-backed cache fed the same id sequence."""
import ctypes as C

import numpy as np
import pytest

from tests.test_staged_cache_cpu import Cache, c_i32p, c_i64p, emul  # noqa: F401  (emul: the fixture)


class RecordCache(Cache):
    """A cache whose length table fills in per request, the way a record source's does."""

    def __init__(self, lib, slots, cols, lens, text_off):
        super().__init__(lib, slots, cols, lens)
        self.true_L = self.L.copy()
        self.L = np.zeros_like(self.true_L)
        self.src = np.ascontiguousarray(text_off, np.int64)

    def request(self, ids):
        ids = np.asarray(ids, np.int32)
        known = ids[(ids >= 0) & (ids < len(self.L))]
        self.L[known] = self.true_L[known]
        return super().request(ids)


@pytest.mark.parametrize("slots,cols,seed", [(40, 100000, 1), (60, 4000, 3), (16, 1200, 4)])
def test_same_placement_as_store(emul, slots, cols, seed):  # noqa: F811
    rng = np.random.default_rng(seed)
    lens = np.clip(np.round(np.exp(rng.normal(np.log(60), 0.9, 500))), 1, cols // 4).astype(np.int32)
    text_off = np.cumsum(rng.integers(100, 5000, len(lens))).astype(np.int64)
    store, recs = Cache(emul, slots, cols, lens), RecordCache(emul, slots, cols, lens, text_off)
    evicting = 0
    for k in range(200):
        want = int(rng.integers(1, slots + 1))
        base = int(rng.integers(0, len(lens) - 50))
        pool = np.concatenate([rng.integers(base, base + 50, want), rng.integers(0, len(lens), want)])
        ids = []
        for g in rng.permutation(pool):
            u = set(ids) | {int(g)}
            if len(u) <= slots and sum(int(lens[x]) for x in u) <= cols:
                ids.append(int(g))
        ids = rng.permutation(ids + ids[:3])
        a = store.request(ids)
        b = recs.request(ids)
        assert a[0] == b[0] == 0
        assert a[1].tolist() == b[1].tolist(), k                       # local ids
        assert a[2][:, 1:].tolist() == b[2][:, 1:].tolist(), k         # dst, len, slot, global of every copy
        assert b[2][:, 0].tolist() == text_off[b[2][:, 4]].tolist()    # the source is the record's own offset
        assert a[3].tolist() == b[3].tolist() and a[4].tolist() == b[4].tolist(), k   # freed slots, statistics
        assert store.state() == recs.state()
        evicting += a[4][3] > 0
    assert evicting >= 20
    # refusals: the sizes come from the lengths of the request's own (now known) records
    big = np.argsort(lens)[-slots - 1:].astype(np.int32)
    a, b = store.request(big), recs.request(big)
    assert a[0] == b[0] == -2 and a[4][:3].tolist() == b[4][:3].tolist()
    assert store.state() == recs.state()
    store.close(); recs.close()
