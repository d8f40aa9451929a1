"""The central-moment model (tests/moments_model.py): hand-worked buffers, the two shortcuts it must not take, and that
its buffers, evaluated as Spark's stddev_* / var_* evaluate them, compute numpy's variance."""
import math
import struct

import numpy as np
import pytest

import hash_model as hm
import moments_model as mm
import partial_agg_model as pm


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def test_a_single_row_is_one_x_zero():
    for x in (3.0, -2.5, 1e-300, 123456789.0):
        assert mm.fold([x]) == (1.0, x, 0.0)


def test_negative_zero():
    n, avg, m2 = mm.fold([-0.0])
    assert (n, bits(avg), bits(m2)) == (1.0, bits(0.0), bits(0.0))  # 0.0 + (-0.0 / 1.0) is +0.0
    n, avg, m2 = mm.fold([-0.0, -0.0])
    assert n == 2.0 and bits(avg) == bits(0.0) and m2 == 0.0


def test_nan_and_infinities():
    n, avg, m2 = mm.fold([1.0, float("nan"), 2.0])
    assert n == 3.0 and math.isnan(avg) and math.isnan(m2)
    n, avg, m2 = mm.fold([float("inf")])
    assert n == 1.0 and avg == float("inf") and math.isnan(m2)  # inf * (inf - inf)
    n, avg, m2 = mm.fold([1.0, -float("inf")])
    assert avg == -float("inf") and math.isnan(m2)


def test_overflow():
    n, avg, m2 = mm.fold([1e300, -1e300, 1e300])
    assert n == 3.0 and math.isinf(m2)


def test_nulls_are_skipped_and_an_all_null_group_is_zero():
    assert mm.fold([None, 1.0, None, 3.0]) == mm.fold([1.0, 3.0])
    assert mm.fold([None, None]) == (0.0, 0.0, 0.0)
    assert mm.merge_all([(0.0, 0.0, 0.0), (0.0, 0.0, 0.0)]) == (0.0, 0.0, 0.0)  # newN == 0: deltaN 0, no 0 / 0


def test_the_cast_of_longs_above_two_to_the_53_rounds():
    big = (1 << 53) + 1
    assert mm.to_double(big, pm.VAL_INT64) == float(1 << 53)
    assert mm.fold([mm.to_double(big, pm.VAL_INT64)])[1] == 9007199254740992.0
    assert mm.to_double((1 << 62) + 3, pm.VAL_INT64) == float(1 << 62)


def test_float32_inputs_widen_exactly_in_the_model_rows():
    x = float(np.float32(0.1))
    row = hm.make_row(["long", "float"], [1, x])
    keys = hm.keys_of(["long", "float"], [0])
    (p,) = mm.partial_rows([row, row], keys, [(mm.VARIANCE, pm.VAL_FLOAT32, 16, 1)])
    n, avg, m2 = struct.unpack("<3d", p[16:40])
    assert (n, avg, m2) == mm.fold([x, x]) and avg == x


# fixed vectors on which each shortcut gives other bits
def test_a_merge_that_starts_from_the_first_buffer_differs():
    a, k = 0.1, 11.0
    assert (a / k) * k != a
    assert mm.merge_all([(k, a, 0.0)])[1] == (a / k) * k  # from (0, 0, 0): avg' = 0 + (a / k) * k
    rng = np.random.default_rng(1)
    differ = sum(mm.merge_all([(float(k), float(a), 0.0)])[1] != float(a)
                 for a, k in zip(rng.normal(size=10000) * 100, rng.integers(1, 1000, 10000)))
    assert 500 < differ < 2000, differ


def test_the_update_chain_is_not_a_merge_of_one_row_buffers():
    xs = [1.0, 2.0, 4.0]
    assert mm.fold(xs) != mm.merge_all([(1.0, x, 0.0) for x in xs])
    rng = np.random.default_rng(2)
    differ = 0
    for _ in range(2000):
        g = [float(v) for v in rng.integers(-100, 100, 50)]
        differ += mm.fold(g) != mm.merge_all([(1.0, x, 0.0) for x in g])
    assert differ > 100, differ


@pytest.mark.parametrize("splits", [1, 2, 7, 40])
def test_buffers_compute_numpys_variance(splits):
    rng = np.random.default_rng(splits)
    for size in (2, 3, 50, 1000):
        data = rng.normal(loc=5.0, scale=3.0, size=size)
        parts = np.array_split(data, min(splits, size))
        buf = mm.merge_all([mm.fold([float(x) for x in p]) for p in parts])
        for fn, ref in (("var_pop", np.var(data)), ("var_samp", np.var(data, ddof=1)),
                        ("stddev_pop", np.std(data)), ("stddev_samp", np.std(data, ddof=1))):
            assert math.isclose(mm.evaluate(buf, fn), ref, rel_tol=1e-12), (fn, size)
    assert mm.evaluate((1.0, 2.0, 0.0), "var_samp") is None and mm.evaluate((0.0, 0.0, 0.0), "var_pop") is None


def test_partial_rows_and_the_reduce_model_agree_with_the_whole_dataset():
    """maps' partial rows merged by the reduce model: n and avg / m2 within rounding of the whole dataset's"""
    rng = np.random.default_rng(3)
    types = ["int", "int", "double"]
    keys = hm.keys_of(types, [0])
    rows = [hm.make_row(types, [int(rng.integers(0, 5)), None if rng.random() < 0.1 else int(rng.integers(-50, 50)),
                                float(rng.normal())]) for _ in range(3000)]
    aggs = [(mm.VARIANCE, pm.VAL_INT32, 16, 1), (pm.COUNT, pm.VAL_NONE, 0, -1), (mm.VARIANCE, pm.VAL_FLOAT64, 24, 2)]
    maps = [rows[m::4] for m in range(4)]
    partials = [p for m in maps for p in mm.partial_rows(m, keys, aggs)]
    import rows_model as rm
    merged, n_rec, n_groups = mm.model_aggregate([rm.stream(partials)], pm.output_keys(keys), mm.merge_aggs(keys, aggs))
    assert n_rec == len(partials) and n_groups == 5
    whole = mm.partial_rows(rows, keys, aggs)
    at = 0
    for w in whole:
        sz = int.from_bytes(merged[at:at + 4], "big")
        got = merged[at + 4:at + 4 + sz]
        at += 4 + sz
        assert got[:16] == w[:16]  # the null word and the key
        for off in (16, 48):
            g, r = struct.unpack("<3d", got[off:off + 24]), struct.unpack("<3d", w[off:off + 24])
            assert g[0] == r[0]
            assert math.isclose(g[1], r[1], rel_tol=1e-12, abs_tol=1e-12)
            assert math.isclose(g[2], r[2], rel_tol=1e-10)
        assert got[40:48] == w[40:48]  # the count
    assert mm.merge_aggs(keys, aggs) == [(mm.AGG_VARIANCE, 16, -1), (pm.SUM_I64, 40, 4), (mm.AGG_VARIANCE, 48, -1)]
