"""The RangePartitioner model (tests/range_model.py) on its own, without a GPU: both of getPartition's branches agree
with each other and with "the number of bounds strictly below the key" on strictly increasing bounds, hand-made cases
pin ties, nulls, floats and DESC strings, and determineBounds yields strictly increasing bounds, at most
partitions - 1 of them."""
import struct

import numpy as np
import pytest

import range_model as rg

F64 = lambda x: struct.pack("<d", x)  # noqa: E731


def rows_of(keys, vals, seed=0):
    rng = np.random.default_rng(seed)
    return [rg.make_row(rng, keys, [v]) for v in vals]


def ids(keys, bound_vals, key_vals):
    """(getPartition, lower bound) of each key value over bounds made from bound_vals, through projected bound rows"""
    bounds = [rg.project(r, keys) for r in rows_of(keys, bound_vals, 1)]
    bk = [rg.key_of(b, rg.bound_keys(keys)) for b in bounds]
    cmp = rg.comparator(keys)
    ks = [rg.key_of(r, keys) for r in rows_of(keys, key_vals, 2)]
    got = [rg.get_partition(k, bk, cmp) for k in ks]
    assert got == [rg.lower_bound(k, bk, cmp) for k in ks]
    return got


@pytest.mark.parametrize("n_bounds", [1, 2, 5, 128, 129, 300])
def test_both_branches_agree_on_strictly_increasing_bounds(n_bounds):
    rng = np.random.default_rng(n_bounds)
    keys = rg.layout([rg.STRING, rg.KEY_INT32, rg.KEY_FLOAT64], [rg.DESC, rg.NULLS_LAST, 0])
    rows = rg.rand_rows(rng, 3000, keys)
    bounds = rg.draw_bounds(rng, rows, keys, n_bounds + 1)
    cmp = rg.comparator(keys)
    bk = [rg.key_of(b, rg.bound_keys(keys)) for b in bounds]
    assert all(cmp(a, b) < 0 for a, b in zip(bk, bk[1:]))
    for r in rows[:600]:
        k = rg.key_of(r, keys)
        want = rg.lower_bound(k, bk, cmp)
        assert rg.scan_partition(k, bk, cmp) == rg.search_partition(k, bk, cmp) == want
    for b in bk:  # a key equal to bound p goes to partition p
        assert rg.scan_partition(b, bk, cmp) == rg.search_partition(b, bk, cmp) == bk.index(b)


def test_keys_equal_below_and_above_the_bounds():
    keys = rg.layout([rg.KEY_INT32])
    assert ids(keys, [10, 20, 30], [-2**31, 5, 10, 11, 20, 29, 30, 31, 2**31 - 1]) == [0, 0, 0, 1, 1, 2, 2, 3, 3]
    keys = rg.layout([rg.KEY_INT32], [rg.DESC])
    assert ids(keys, [30, 20, 10], [40, 30, 25, 20, 10, 9]) == [0, 0, 1, 1, 2, 3]


def test_null_bounds_first_and_last():
    keys = rg.layout([rg.KEY_INT64])  # ASC NULLS FIRST: null below every value
    assert ids(keys, [None, 5], [None, -2**63, 5, 6]) == [0, 1, 1, 2]
    keys = rg.layout([rg.KEY_INT64], [rg.NULLS_LAST])
    assert ids(keys, [5, None], [None, 5, 6, 2**63 - 1]) == [1, 0, 1, 1]
    keys = rg.layout([rg.KEY_INT64], [rg.DESC | rg.NULLS_LAST])
    assert ids(keys, [5, None], [None, 7, 5, 4]) == [1, 0, 0, 1]


def test_negative_zero_and_nan():
    keys = rg.layout([rg.KEY_FLOAT64])
    nan2 = struct.pack("<Q", 0x7FF0000000000001)  # another NaN payload: equal to the canonical NaN
    got = ids(keys, [F64(-0.0), F64(float("nan"))],
              [F64(0.0), F64(-0.0), F64(-1e-300), F64(float("inf")), nan2, F64(float("-inf"))])
    assert got == [0, 0, 0, 1, 1, 0]
    keys = rg.layout([rg.KEY_FLOAT32], [rg.DESC])  # DESC: NaN first
    f = lambda x: struct.pack("<f", x)  # noqa: E731
    assert ids(keys, [f(float("nan")), f(0.0)], [f(float("nan")), f(float("inf")), f(-0.0), f(-1.0)]) == [0, 1, 1, 2]


def test_desc_strings_that_are_prefixes_of_each_other():
    keys = rg.layout([rg.STRING], [rg.DESC])  # DESC: an extension before its prefix
    assert ids(keys, [b"abc", b"ab"], [b"abcd", b"abc", b"ab\x00", b"ab", b"a", b"", None]) == [0, 0, 1, 1, 2, 2, 0]
    keys = rg.layout([rg.STRING], [rg.DESC | rg.NULLS_LAST])
    assert ids(keys, [b"abc", b""], [b"abc", b"", None, b"b" * 30]) == [0, 1, 2, 0]


@pytest.mark.parametrize("partitions", [1, 2, 3, 17, 200])
def test_determine_bounds_is_strictly_increasing_and_short_enough(partitions):
    rng = np.random.default_rng(partitions)
    keys = rg.layout([rg.KEY_INT8, rg.STRING], [0, rg.DESC])
    rows = rg.rand_rows(rng, 1500, keys, null_frac=0.3)  # few distinct keys: duplicates are skipped
    cmp = rg.comparator(keys)
    cands = [(rg.key_of(r, keys), float(rng.integers(1, 4))) for r in rows]
    b = rg.determine_bounds(cands, partitions, cmp)
    assert len(b) <= partitions - 1
    assert all(cmp(cands[i][0], cands[j][0]) < 0 for i, j in zip(b, b[1:]))
    # a bound and the key it was drawn from are the same key
    bounds = [rg.project(rows[i], keys) for i in b]
    assert [rg.key_of(x, rg.bound_keys(keys)) for x in bounds] == [cands[i][0] for i in b]
