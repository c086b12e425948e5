"""The top-K key distributions of tests/topk_cases.py: the numpy restatement of the device selection (keys, 8 radix
passes, compaction) gives the reference order on every case, and each case reaches the radix-select edge it claims.
The key without the -0.0 -> +0.0 fold orders signed zeros differently from the reference."""
import numpy as np
import pytest

from tests import topk_cases as tc

NS = (1, 2, 255, 256, 257, 1000, 135169)


def _cases():
    return [(name, n) for name in tc.CASES for n in NS if not (name == "signed_zero" and n < 8)]


@pytest.mark.parametrize("name,n", _cases(), ids=lambda v: str(v))
def test_restatement_is_the_reference_order(name, n):
    c = tc.case(name, n)
    keys = tc.device_keys(c["key"], c["gids"])
    order = tc.reference_order(c["key"], c["gids"])
    assert len(np.unique(c["gids"])) == n
    assert np.all(keys[order][1:] > keys[order][:-1])          # unique keys, increasing along the list
    for K in c["ks"]:
        got = tc.select_order(keys, K)
        assert np.array_equal(got, order[:K]), (name, n, K)


@pytest.mark.parametrize("name,n", _cases(), ids=lambda v: str(v))
def test_each_case_reaches_its_edge(name, n):
    c = tc.case(name, n)
    keys = tc.device_keys(c["key"], c["gids"])
    for K, p, kind, b in c["claims"]:
        _, trace = tc.radix_select(keys, K)
        t = trace[7 - p]
        assert t["p"] == p
        if kind == "bucket":
            assert t["bucket"] == b, (name, n, K, t)
        elif kind == "single":
            assert t["buckets"] == 1, (name, n, K, t)
        else:
            assert t["buckets"] > 1, (name, n, K, t)


def test_every_named_edge_is_claimed():
    """Over the cases at n = 1000: bucket 255 and bucket 0 at pass 7, both at pass 0, single-bucket passes 7..2, a
    split at pass 4 and the scan's fall-through at bucket 255 on three consecutive passes."""
    seen = set()
    for name in tc.CASES:
        for K, p, kind, b in tc.case(name, 1000)["claims"]:
            seen.add((p, kind, b))
    for edge in [(7, "bucket", 255), (7, "bucket", 0), (0, "bucket", 0), (0, "bucket", 255), (4, "split", None),
                 (2, "bucket", 255), (1, "bucket", 255)] + [(p, "single", None) for p in range(7, 1, -1)]:
        assert edge in seen, edge


def test_mixed_case_holds_every_special_value():
    c = tc.case("mixed", 1000)
    bits = set(c["key"].view(np.uint32).tolist())
    assert bits >= set(tc._SPECIAL.view(np.uint32).tolist())


@pytest.mark.parametrize("name,n", [("signed_zero", 1000), ("signed_zero", 135169), ("mixed", 1000)])
def test_key_without_the_zero_fold_breaks_the_reference_order(name, n):
    """-0.0 and +0.0 map to different raw keys, so without the fold the ids no longer decide between them."""
    c = tc.case(name, n)
    order = tc.reference_order(c["key"], c["gids"])
    raw = tc.device_keys(c["key"], c["gids"], fold_zero=False)
    assert not np.array_equal(tc.select_order(raw, n), order)
    assert np.array_equal(tc.select_order(tc.device_keys(c["key"], c["gids"]), n), order)
    z = c["key"] == 0
    assert np.signbit(c["key"][z]).any() and not np.signbit(c["key"][z]).all()


def test_reference_treats_signed_zeros_as_equal():
    key = np.array([0.0, -0.0, 0.0, -0.0], np.float32)
    assert np.array_equal(tc.reference_order(key, [3, 2, 1, 0]), [3, 2, 1, 0])
    assert np.array_equal(tc.reference_order(key, [3, 2, 1, 0], by="score"), [3, 2, 1, 0])


def test_score_keys_descend():
    """By score the key is ~orderable: higher scores first, -inf last, ties by id."""
    s = np.array([1.0, -np.inf, 7.0, 1.0, np.inf, -0.0, 0.0], np.float32)
    g = np.array([9, 1, 2, 3, 4, 6, 5], np.int32)
    keys = tc.device_keys(s, g, by="score")
    order = tc.reference_order(s, g, by="score")
    assert np.array_equal(order, [4, 2, 3, 0, 6, 5, 1])
    assert np.array_equal(np.argsort(keys, kind="stable"), order)
