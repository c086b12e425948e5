"""The slot / arena / eviction bookkeeping of a staged shard (hh-suite_b200/csrc/hhg_stage_cache.h, unmodified source,
compiled without a device through tests/emul/stage_cache_emul.cpp) against a dictionary model: random request sequences
with duplicates over caches that are short of slots, short of columns or both.  After every request: each named target is
resident at the local id returned, residents named before keep their local id, arena runs never overlap or leave the
arena, exactly the missing targets are copied (all of the request's after a re-layout), nothing the request names is
evicted, the least recently staged go first, and the statistics add up.  Requests that cannot fit are refused with the
sizes they need and change nothing; a request that fits always succeeds, also when its own residents fragment the arena."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.util import ROOT

EMUL_DIR = os.path.join(ROOT, "tests", "emul")
LIB = os.path.join(EMUL_DIR, "libstagecacheemul.so")
c_i32p = C.POINTER(C.c_int32); c_i64p = C.POINTER(C.c_int64)


@pytest.fixture(scope="module")
def emul():
    srcs = [os.path.join(EMUL_DIR, "stage_cache_emul.cpp"),
            os.path.join(ROOT, "hh-suite_b200", "csrc", "hhg_stage_cache.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", LIB, srcs[0]])
    L = C.CDLL(LIB)
    L.sc_create.restype = C.c_void_p
    L.sc_create.argtypes = [C.c_int, C.c_longlong]
    L.sc_destroy.argtypes = [C.c_void_p]
    L.sc_request.argtypes = [C.c_void_p, C.c_int, c_i32p, C.c_int, c_i32p, c_i64p, c_i32p, c_i64p, c_i32p, c_i64p]
    L.sc_slot.argtypes = [C.c_void_p, C.c_int, c_i64p]
    L.sc_resident.argtypes = [C.c_void_p]
    return L


class Cache:
    """The emulated cache next to its model: resident {global: (slot, off, len)} and the request that last named it."""

    def __init__(self, lib, slots, cols, lens):
        self.lib, self.slots, self.cols = lib, slots, cols
        self.L = np.ascontiguousarray(lens, np.int32)
        self.src = np.concatenate([[0], np.cumsum(self.L.astype(np.int64))[:-1]]).astype(np.int64)
        self.h = C.c_void_p(lib.sc_create(slots, cols))
        self.res: dict[int, tuple[int, int, int]] = {}
        self.used: dict[int, int] = {}
        self.clock = 0

    def close(self):
        self.lib.sc_destroy(self.h)

    def state(self):
        out = np.zeros(3, np.int64)
        got = {}
        for s in range(self.slots):
            self.lib.sc_slot(self.h, s, out.ctypes.data_as(c_i64p))
            if out[0] >= 0:
                got[int(out[0])] = (s, int(out[1]), int(out[2]))
        return got

    def request(self, ids):
        ids = np.ascontiguousarray(ids, np.int32)
        local = np.full(len(ids), -1, np.int32)
        items = np.zeros((max(len(ids), 1), 5), np.int64)
        freed = np.zeros(self.slots, np.int32)
        out = np.zeros(6, np.int64)
        rc = self.lib.sc_request(self.h, len(ids), ids.ctypes.data_as(c_i32p), len(self.L), self.L.ctypes.data_as(c_i32p),
                                 self.src.ctypes.data_as(c_i64p), local.ctypes.data_as(c_i32p),
                                 items.ctypes.data_as(c_i64p), freed.ctypes.data_as(c_i32p), out.ctypes.data_as(c_i64p))
        return rc, local, items[:out[4]] if rc == 0 else None, freed[:out[5]] if rc == 0 else None, out

    def checked_request(self, ids):
        """One request that fits, checked against the model; returns (items, stats)."""
        uniq = list(dict.fromkeys(int(g) for g in ids))
        before = dict(self.res)
        rc, local, items, freed, out = self.request(ids)
        assert rc == 0, (rc, out[:3])
        hits, copied, nbytes, evicted = (int(x) for x in out[:4])
        now = self.state()
        assert self.lib.sc_resident(self.h) == len(now)
        # every named target is resident where the call says, with its own length
        for g, s in zip(ids, local):
            assert now[int(g)][0] == s and now[int(g)][2] == self.L[g]
        # runs lie inside the arena and do not overlap; slots are distinct
        runs = sorted((off, ln) for _, off, ln in now.values())
        assert all(off >= 0 and off + ln <= self.cols for off, ln in runs)
        assert all(a[0] + a[1] <= b[0] for a, b in zip(runs, runs[1:]))
        assert len({s for s, _, _ in now.values()}) == len(now) <= self.slots
        # residents keep their local id; one that was named before and is named again keeps its run too unless the
        # request was laid out again (then every target of the request is copied)
        missing = [g for g in uniq if g not in before]
        relaid = copied > len(missing)
        for g, (s, off, ln) in before.items():
            if g in now:
                assert now[g][0] == s
                if not relaid:
                    assert now[g][1] == off
        copied_ids = [int(x) for x in items[:, 4]]
        if relaid:
            assert sorted(copied_ids) == sorted(uniq) and set(now) == set(uniq)
        else:
            assert sorted(copied_ids) == sorted(missing)
        for src, dst, ln, slot, g in items:
            assert (src, ln) == (self.src[g], self.L[g]) and now[int(g)] == (slot, dst, ln)
        # statistics
        gone = [g for g in before if g not in now]
        assert not set(gone) & set(uniq)
        assert (hits, copied, evicted) == (len(uniq) - copied, len(items), len(gone))
        assert nbytes == sum(int(self.L[g]) * 112 + 92 for g in copied_ids)
        # least recently staged first: everything evicted was named no later than anything that stays and is not named
        stay = [self.used[g] for g in now if g not in uniq]
        if gone and stay:
            assert max(self.used[g] for g in gone) <= min(stay)
        # freed = slots that held an evicted target and hold nothing now
        assert sorted(freed.tolist()) == sorted(s for g, (s, _, _) in before.items() if g in gone
                                                and s not in {v[0] for v in now.values()})
        self.clock += 1
        for g in gone:
            del self.used[g]
        for g in uniq:
            self.used[g] = self.clock
        self.res = now
        return items, (hits, copied, nbytes, evicted)


@pytest.mark.parametrize("slots,cols,seed", [(40, 100000, 1), (400, 3000, 2), (60, 4000, 3), (16, 1200, 4)])
def test_random_requests_against_model(emul, slots, cols, seed):
    """Short of slots (1), of columns (2), of both (3), and a small cache whose requests nearly fill it (4)."""
    rng = np.random.default_rng(seed)
    lens = np.clip(np.round(np.exp(rng.normal(np.log(60), 0.9, 500))), 1, cols // 4).astype(np.int32)
    c = Cache(emul, slots, cols, lens)
    evicting = 0
    for _ in range(300):
        want = int(rng.integers(1, slots + 1))
        # related requests: half of the ids come from a window that drifts over the store
        base = int(rng.integers(0, len(lens) - 50))
        pool = np.concatenate([rng.integers(base, base + 50, want), rng.integers(0, len(lens), want)])
        ids = []
        for g in rng.permutation(pool):
            u = set(ids) | {int(g)}
            if len(u) <= slots and sum(int(lens[x]) for x in u) <= cols:
                ids.append(int(g))
        ids += ids[:3]                                   # duplicates
        items, (hits, copied, _, evicted) = c.checked_request(rng.permutation(ids))
        evicting += evicted > 0
    assert evicting >= 30
    c.close()


def test_fragmented_by_own_residents(emul):
    """Residents of the request itself at both ends of every gap: a long target fits only after a new layout."""
    lens = np.array([10] * 10 + [50], np.int32)
    c = Cache(emul, 16, 100, lens)
    c.checked_request(np.arange(10))                     # arena full: 10 runs of 10
    c.checked_request([0, 2, 4, 6, 8])                   # touch the even ones
    items, (hits, copied, _, evicted) = c.checked_request([0, 2, 4, 6, 8, 10])   # 50 free columns, in runs of 10
    assert evicted == 5 and copied == 6 and hits == 0
    assert sorted(items[:, 1].tolist()) == [0, 10, 20, 30, 40, 50]
    items, (hits, copied, _, evicted) = c.checked_request([10, 0])
    assert (hits, copied, evicted) == (2, 0, 0) and len(items) == 0
    c.close()


def test_refusals_change_nothing(emul):
    lens = np.array([30, 30, 30, 30, 5, 5, 5], np.int32)
    c = Cache(emul, 4, 100, lens)
    c.checked_request([0, 4])
    before = c.state()
    for ids, want in (([0, 1, 2, 3], (-2, 4, 120)), ([4, 5, 6, 0, 1, 4], (-2, 5, 75)), ([0, 7], (-1, 1)), ([-1], (-1, 0))):
        rc, _, _, _, out = c.request(ids)
        assert rc == want[0]
        if rc == -2:
            assert (int(out[1]), int(out[2])) == want[1:]
        else:
            assert int(out[0]) == want[1]
        assert c.state() == before
    c.checked_request([1, 2, 5])                         # still usable: evicts 0 or 4 as needed
    c.checked_request([])
    c.close()
