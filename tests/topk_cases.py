"""Key distributions and a plain reference for the device top-K selection (hhg_plan_topk / hhg_plan_topk_by_key,
csrc/hhg_topk.cuh).

  reference_order   the list order hhg_plan_topk promises: value as float64 (score descending or caller key ascending),
                    ties by int32 global id ascending; np.lexsort, so -0.0 == +0.0
  device_keys       numpy restatement of k_topk_keys: key = (orderable(value) << 32) | global id, with ~orderable for
                    scores; fold_zero=False is the key without the -0.0 -> +0.0 fold
  radix_select      numpy restatement of the 8 k_topk_hist / k_topk_scan passes; returns the K-th key and, per pass,
                    the bucket the scan picked and how many buckets were not empty.  Used to prove that each named
                    case reaches the edge it claims, not as the expected result

Named cases (case(name, n, seed)) are caller keys for hhg_plan_topk_by_key with scattered global ids:

  all_equal     one value, ids 0x5A000000 + k: the ids alone decide and share their high byte(s), so passes 7..3 see
                one bucket; K = 1 takes bucket 0 at pass 0
  adjacent      1.0 and its next 255 floats (nextafter chain), repeated: passes 7..5 see one bucket and the K-th key
                is decided in the lowest mantissa byte at pass 4
  pos_inf       a quarter finite, the rest +inf, FLT_MAX and floats >= 2^127: the K-th key in bucket 255 at pass 7
  neg_inf       a third -inf and -FLT_MAX, the rest finite: the K-th key in bucket 0 at pass 7
  mixed         random draws from +-inf, +-FLT_MAX, +-FLT_MIN, denormals, +-0.0 and a few normal values (many ties)
  signed_zero   -0.0 and +0.0 at random with a few denormals: the order of the zeros is the ids' order, which the key
                without the fold gets wrong
  id_bytes      three values; ids whose low byte is 0x00 or 0xFF: the K-th key in bucket 0 or bucket 255 at pass 0
  near_max      one value, ids INT32_MAX - k: K = n takes bucket 255 at passes 2, 1 and 0

Each case lists Ks worth selecting and claims (K, pass, kind, bucket): kind "bucket" = the scan picks that bucket,
"single" = one bucket is not empty, "split" = more than one is."""
import numpy as np

INT32_MAX = 2 ** 31 - 1
FLT_MAX = np.float32(np.finfo(np.float32).max)
FLT_MIN = np.float32(np.finfo(np.float32).tiny)
FLT_TRUE_MIN = np.float32(np.finfo(np.float32).smallest_subnormal)


# ------------------------------------------------------------------------------------------------ reference
def reference_order(value, gids, by="key"):
    """Request indices in list order: by "key" ascending, by "score" descending, ties by global id ascending."""
    v = np.asarray(value, np.float32).astype(np.float64)
    return np.lexsort((np.asarray(gids, np.int64), v if by == "key" else -v))


# ------------------------------------------------------------------------------------------------ restatement
def orderable(value):
    """orderable_f32: float32 -> uint32, monotone increasing."""
    u = np.asarray(value, np.float32).view(np.uint32)
    return u ^ np.where(u >> np.uint32(31), np.uint32(0xFFFFFFFF), np.uint32(0x80000000)).astype(np.uint32)


def device_keys(value, gids, by="key", fold_zero=True):
    v = np.array(value, np.float32)
    if fold_zero:
        v[v == 0] = np.float32(0.0)
    o = orderable(v)
    hi = (o if by == "key" else ~o).astype(np.uint64)
    return (hi << np.uint64(32)) | np.asarray(gids, np.int64).astype(np.uint32).astype(np.uint64)


def radix_select(keys, K):
    """(K-th smallest key, trace): trace[i] = dict(p, bucket, buckets) for the passes p = 7 .. 0 in order."""
    keys = np.asarray(keys, np.uint64)
    krem, prefix, trace = min(K, len(keys)), 0, []
    for p in range(7, -1, -1):
        m = keys if p == 7 else keys[(keys >> np.uint64((p + 1) * 8)) == np.uint64(prefix)]
        h = np.bincount(((m >> np.uint64(p * 8)) & np.uint64(255)).astype(np.int64), minlength=256)
        cum, d = 0, 0
        while d < 255 and cum + h[d] < krem:      # k_topk_scan: the loop falls through at bucket 255
            cum += int(h[d])
            d += 1
        trace.append(dict(p=p, bucket=d, buckets=int(np.count_nonzero(h))))
        prefix = (prefix << 8) | d
        krem -= cum
    return prefix, trace


def select_order(keys, K):
    """Request indices the restatement emits for K, in key order (k_topk_emit: every key <= the K-th)."""
    kth, _ = radix_select(keys, K)
    idx = np.nonzero(keys <= np.uint64(kth))[0]
    return idx[np.argsort(keys[idx], kind="stable")]


# ------------------------------------------------------------------------------------------------ named cases
def scattered_ids(n, rng, lo=0, hi=INT32_MAX):
    """n distinct ids in [lo, hi], in random order."""
    span = hi - lo + 1
    if span <= 4 * n:
        return (lo + rng.permutation(span)[:n]).astype(np.int32)
    ids = np.unique(rng.integers(lo, hi, int(n * 1.1) + 16, endpoint=True))
    while len(ids) < n:
        ids = np.unique(np.concatenate([ids, rng.integers(lo, hi, n, endpoint=True)]))
    return rng.permutation(ids)[:n].astype(np.int32)


def _f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def _all_equal(n, rng):
    gids = rng.permutation(0x5A000000 + np.arange(n)).astype(np.int32)
    single = [7, 6, 5, 4, 3] + ([2] if n <= 1 << 16 else [])
    claims = [(1, 0, "bucket", 0)] + [(1, p, "single", None) for p in single]
    return np.full(n, 1.5, np.float32), gids, [1, 2, n // 2, n - 1, n, n + 1], claims


def _adjacent(n, rng):
    key = rng.permutation(_f32(0x3F800000 + np.arange(n) % 256))
    K = max(1, n // 2)
    claims = [(K, p, "single", None) for p in (7, 6, 5)] + ([(K, 4, "split", None)] if n > 1 else [])
    return key, scattered_ids(n, rng), [1, n // 3, K, n - 1, n], claims


def _pos_inf(n, rng):
    c = n // 4
    huge = _f32(rng.integers(0x7F000000, 0x7F7FFFFF, n - c, endpoint=True))
    huge[::3] = np.inf
    huge[1::3] = FLT_MAX
    key = np.concatenate([rng.normal(0, 100, c).astype(np.float32), huge])
    return rng.permutation(key), scattered_ids(n, rng), [1, c, c + 1, n - 1, n], [(c + 1, 7, "bucket", 255), (n, 7, "bucket", 255)]


def _neg_inf(n, rng):
    c = max(1, n // 3)
    low = np.where(np.arange(c) % 2 == 0, -np.inf, -FLT_MAX).astype(np.float32)
    key = np.concatenate([low, rng.normal(0, 100, n - c).astype(np.float32)])
    return rng.permutation(key), scattered_ids(n, rng), [1, c, c + 1, n], [(1, 7, "bucket", 0), (c, 7, "bucket", 0)]


_SPECIAL = np.array([np.inf, -np.inf, FLT_MAX, -FLT_MAX, FLT_MIN, -FLT_MIN, FLT_TRUE_MIN, -FLT_TRUE_MIN,
                     _f32(0x007FFFFF), -_f32(0x007FFFFF), 0.0, -0.0, 1.0, -1.0, 3.25, -7.5], np.float32)


def _mixed(n, rng):
    return rng.choice(_SPECIAL, n), scattered_ids(n, rng), [1, n // 7, n // 2, n - 1, n], []


def _signed_zero(n, rng):
    key = np.where(rng.random(n) < 0.5, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
    key[rng.random(n) < 0.05] = FLT_TRUE_MIN
    key[rng.random(n) < 0.05] = -FLT_TRUE_MIN
    return key, scattered_ids(n, rng), [1, 2, n // 2, n - 1, n], []


def _id_bytes(n, rng):
    k = np.arange(n)
    gids = (0x01000000 + (k // 2) * 256 + np.where(k % 2, 255, 0)).astype(np.int32)
    key = rng.choice(np.array([-2.5, 0.75, 9.0], np.float32), n)
    perm = rng.permutation(n)
    key, gids = key[perm], gids[perm]
    low = gids[reference_order(key, gids)] & 255
    claims = []
    for b in (0, 255):
        at = np.nonzero(low == b)[0]
        if len(at):
            claims.append((int(at[len(at) // 2]) + 1, 0, "bucket", b))
    return key, gids, [1, 2, n // 2, n] + [c[0] for c in claims], claims


def _near_max(n, rng):
    gids = rng.permutation(INT32_MAX - np.arange(n)).astype(np.int32)
    return np.full(n, -3.0, np.float32), gids, [1, n - 1, n], [(n, p, "bucket", 255) for p in (2, 1, 0)]


CASES = dict(all_equal=_all_equal, adjacent=_adjacent, pos_inf=_pos_inf, neg_inf=_neg_inf, mixed=_mixed,
             signed_zero=_signed_zero, id_bytes=_id_bytes, near_max=_near_max)


def case(name, n, seed=0):
    """dict(name, n, key float32[n], gids int32[n], ks, claims) for hhg_plan_topk_by_key."""
    rng = np.random.default_rng([seed, n, list(CASES).index(name)])
    key, gids, ks, claims = CASES[name](n, rng)
    ks = sorted({int(K) for K in ks if K >= 1})
    return dict(name=name, n=n, key=np.ascontiguousarray(key, np.float32), gids=np.ascontiguousarray(gids, np.int32),
                ks=ks, claims=claims)
