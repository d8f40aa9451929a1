"""tests/window_frame_model.py pinned without a GPU: hand-worked frames of each Spark frame class, RANGE bounds in
every direction and null order, empty frames, a lone -0.0 sum, first-of-equal MIN and IGNORE_NULLS nth_value; on
random inputs the loop frames equal the closed-form sets, and the new frames at their unbounded ends equal the older
running and partition frames."""
import functools
import struct

import numpy as np
import pytest

from rows_model import stream
from test_gpu_sort_rows_order import DESC, NULLS_LAST, comparator
from window_agg_model import (COUNT, FRAME_PARTITION, FRAME_RANGE, FRAME_ROWS, MIN, SUM, VAL_FLOAT64, VAL_INT64,
                              model_window_aggregate)
from window_frame_model import (UNBOUNDED_FOLLOWING as UF, UNBOUNDED_PRECEDING as UP, Bounds, closed_form, frames,
                                model_window_frame)
from window_offset_model import IGNORE_NULLS, NTH_VALUE, model_window_offset

ROWS, RANGE = 4, 5
KEY_INT64, KEY_INT32, KEY_INT8 = 2, 1, 6


def rows_frames(N, lo, hi):
    return frames(N, ROWS, lo, hi, Bounds([(0,)] * N, [(KEY_INT64, 0, 8, -1)]))


def range_frames(vals, lo, hi, flags=0, kt=KEY_INT64):
    col = (kt | flags, 0, 8, 0)
    return frames(len(vals), RANGE, lo, hi, Bounds([(v,) for v in vals], [col]))


def test_each_frame_class_on_rows():
    assert rows_frames(4, UP, UF) == [[0, 1, 2, 3]] * 4  # Unbounded
    assert rows_frames(4, UP, 0) == [[0], [0, 1], [0, 1, 2], [0, 1, 2, 3]]  # UnboundedPreceding
    assert rows_frames(4, 1, UF) == [[1, 2, 3], [2, 3], [3], []]  # UnboundedFollowing
    assert rows_frames(5, -1, 1) == [[0, 1], [0, 1, 2], [1, 2, 3], [2, 3, 4], [3, 4]]  # Sliding


def test_preceding_only_following_only_and_empty_frames():
    assert rows_frames(5, -3, -2) == [[], [], [0], [0, 1], [1, 2]]
    assert rows_frames(5, 2, 3) == [[2, 3], [3, 4], [4], [], []]
    assert rows_frames(3, UP, -1) == [[], [0], [0, 1]]
    assert rows_frames(3, 5, 9) == [[], [], []]


def test_range_bounds_in_every_direction_and_null_order_with_ties_and_null_keys():
    # sorted ascending nulls first: None, None, 1, 2, 2, 5
    v = [None, None, 1, 2, 2, 5]
    assert range_frames(v, -1, 0) == [[0, 1], [0, 1], [2], [2, 3, 4], [2, 3, 4], [5]]
    assert range_frames(v, 0, 3) == [[0, 1], [0, 1], [2, 3, 4], [3, 4, 5], [3, 4, 5], [5]]
    # ascending nulls last: 1, 2, 2, 5, None
    v = [1, 2, 2, 5, None]
    assert range_frames(v, -1, 1, NULLS_LAST) == [[0, 1, 2], [0, 1, 2], [0, 1, 2], [3], [4]]
    # descending nulls first: None, 5, 2, 2, 1 (1 PRECEDING is v + 1)
    v = [None, 5, 2, 2, 1]
    assert range_frames(v, -1, 0, DESC) == [[0], [1], [2, 3], [2, 3], [2, 3, 4]]
    assert range_frames(v, -3, UF, DESC) == [[0, 1, 2, 3, 4], [1, 2, 3, 4], [1, 2, 3, 4], [1, 2, 3, 4], [2, 3, 4]]
    # descending nulls last: 5, 2, 2, 1, None
    v = [5, 2, 2, 1, None]
    assert range_frames(v, 0, 1, DESC | NULLS_LAST) == [[0], [1, 2, 3], [1, 2, 3], [3], [4]]
    assert range_frames(v, UP, -2, DESC | NULLS_LAST) == [[], [0], [0], [0], [0, 1, 2, 3, 4]]  # null: through its peers


def test_range_bound_that_wraps_is_reported():
    b = Bounds([(1,), (127,)], [(KEY_INT8, 0, 1, -1)])
    frames(2, RANGE, 0, 1, b)
    assert b.unsupported


class T:
    """rows: field 0 a partition key, 1 the order key (long, nullable), 2 a double value, 3 a long value"""
    nf, kinds = 4, [0, 0, 0, 0]
    keys = [(KEY_INT64, 8, 8, -1), (KEY_INT64, 16, 8, 1)]

    @staticmethod
    def row(p, o, d=None, x=None):
        bits = (o is None) << 1 | (d is None) << 2 | (x is None) << 3
        r = bits.to_bytes(8, "little") + (p % 2**64).to_bytes(8, "little") + ((o or 0) % 2**64).to_bytes(8, "little")
        r += struct.pack("<d", d) if d is not None else bytes(8)
        return r + (((x or 0) % 2**64).to_bytes(8, "little"))


def out_slots(out, nf, n_fns):
    """the value slots of every output row -> [[8 bytes, ...]], with the value null bits"""
    res, p = [], 0
    while p < len(out):
        size = int.from_bytes(out[p:p + 4], "big")
        row = out[p + 4:p + 4 + size]
        w = (nf + n_fns + 63) // 64
        bits = int.from_bytes(row[:8], "little")
        base = 8 * (w + nf)
        res.append([None if bits >> (nf + j) & 1 else row[base + 8 * j:base + 8 * j + 8] for j in range(n_fns)])
        p += 4 + size
    return res


def run_model(rows, fns):
    out, n, m, unsupported = model_window_frame([stream(rows)], T.keys, 1, T.nf, T.kinds, fns)
    assert not unsupported
    return out_slots(out, T.nf, len(fns))


def dbl(b):
    return None if b is None else struct.unpack("<d", b)[0]


def test_a_lone_negative_zero_sums_to_positive_zero():
    got = run_model([T.row(0, 1, -0.0)], [(SUM, 0, ROWS, VAL_FLOAT64, 24, 2, 0, 0, -1, 1)])
    assert got[0][0] == struct.pack("<d", 0.0)


def test_min_keeps_the_first_of_equal_values_with_its_bits():
    rows = [T.row(0, 1, -0.0), T.row(0, 2, 0.0), T.row(0, 3, -0.0)]
    got = run_model(rows, [(MIN, 0, ROWS, VAL_FLOAT64, 24, 2, 0, 0, -1, 1)])
    assert [g[0] for g in got] == [struct.pack("<d", -0.0), struct.pack("<d", -0.0), struct.pack("<d", 0.0)]


def test_sliding_sums_counts_and_empty_frames():
    rows = [T.row(0, i, float(i), i) for i in range(1, 6)]
    got = run_model(rows, [(SUM, 0, ROWS, VAL_INT64, 32, 3, 0, 0, -2, -1), (COUNT, 0, ROWS, VAL_INT64, 32, 3, 0, 0, 2,
                                                                             3),
                           (SUM, 0, ROWS, VAL_FLOAT64, 24, 2, 0, 0, 0, UF)])
    sums = [None if g[0] is None else int.from_bytes(g[0], "little", signed=True) for g in got]
    assert sums == [None, 1, 3, 5, 7]
    assert [int.from_bytes(g[1], "little") for g in got] == [2, 2, 1, 0, 0]
    assert [dbl(g[2]) for g in got] == [15.0, 14.0, 12.0, 9.0, 5.0]


def test_ignore_nulls_nth_value():
    rows = [T.row(0, i, None if i % 2 else float(i), i) for i in range(6)]  # doubles 0, -, 2, -, 4, -
    got = run_model(rows, [(NTH_VALUE, 2, ROWS, VAL_FLOAT64, 24, 2, IGNORE_NULLS, 0, -1, 3),
                           (NTH_VALUE, 2, ROWS, VAL_FLOAT64, 24, 2, 0, 0, -1, 3)])
    assert [dbl(g[0]) for g in got] == [2.0, 2.0, 4.0, 4.0, None, None]
    assert [dbl(g[1]) for g in got] == [None, None, 2.0, None, 4.0, None]


@pytest.mark.parametrize("seed", range(6))
def test_loop_frames_equal_the_closed_form(seed):
    rng = np.random.default_rng(seed)
    for _ in range(30):
        N = int(rng.integers(1, 25))
        flags = [0, DESC, NULLS_LAST, DESC | NULLS_LAST][int(rng.integers(4))]
        col = [(KEY_INT64 | flags, 0, 8, 0)]
        vals = [None if rng.random() < 0.15 else int(rng.integers(-5, 6)) for _ in range(N)]
        cmp = comparator(col)
        ok = sorted([(v,) for v in vals], key=functools.cmp_to_key(cmp))
        for kind in (ROWS, RANGE):
            cand = [UP, -4, -1, 0, 2, 5, UF]
            lo, hi = sorted([cand[int(rng.integers(0, 6))], cand[int(rng.integers(1, 7))]])
            b = Bounds(ok, col)
            got = frames(N, kind, lo, hi, b)
            assert not b.unsupported
            assert got == [closed_form(ok, col, kind, lo, hi, i, N) for i in range(N)], (kind, lo, hi, ok)


@pytest.mark.parametrize("seed", range(3))
def test_unbounded_bounds_equal_the_older_frames(seed):
    rng = np.random.default_rng(100 + seed)
    rows = [T.row(int(rng.integers(3)), None if rng.random() < 0.1 else int(rng.integers(6)),
                  None if rng.random() < 0.2 else float(rng.normal()), int(rng.integers(-9, 9)))
            for _ in range(120)]
    for (fr, lo, hi), old in (((ROWS, UP, 0), FRAME_ROWS), ((RANGE, UP, 0), FRAME_RANGE),
                              ((ROWS, UP, UF), FRAME_PARTITION), ((RANGE, UP, UF), FRAME_PARTITION)):
        new = [(f, 0, fr, vt, off, nb, 0, 0, lo, hi) for f, vt, off, nb in
               ((SUM, VAL_FLOAT64, 24, 2), (MIN, VAL_FLOAT64, 24, 2), (COUNT, VAL_INT64, 32, 3))]
        new.append((NTH_VALUE, 2, fr, VAL_FLOAT64, 24, 2, IGNORE_NULLS, 0, lo, hi))
        older = [f[:2] + (old,) + f[3:8] for f in new]
        a = model_window_frame([stream(rows)], T.keys, 1, T.nf, T.kinds, new)
        assert a[0] == model_window_offset([stream(rows)], T.keys, 1, T.nf, T.kinds, older)[0]
        agg = [(f[0], old, *f[3:6]) for f in new[:3]]
        assert model_window_frame([stream(rows)], T.keys, 1, T.nf, T.kinds, new[:3])[0] == \
            model_window_aggregate([stream(rows)], T.keys, 1, T.nf, T.kinds, agg)[0]


def test_rows_offset_past_the_int_range_is_reported():
    rows = [T.row(0, i, 1.0, i) for i in range(3)]
    fns = [(SUM, 0, ROWS, VAL_INT64, 32, 3, 0, 0, 0, 2**31 - 1)]
    assert model_window_frame([stream(rows)], T.keys, 1, T.nf, T.kinds, fns)[3]
    assert not model_window_frame([stream(rows[:1])], T.keys, 1, T.nf, T.kinds, fns)[3]
