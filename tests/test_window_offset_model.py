"""tests/window_offset_model.py against hand-worked partitions: LAG / LEAD at the partition's edges with and without a
default, IGNORE_NULLS whose k-th non-null input lies past the partition, an all-null partition, NTH_VALUE past its
frame, LAST over a RANGE frame with peers, and the value row's var regions in function order.  With no offset function
the model's bytes are window_agg_model's."""
import numpy as np

from join_model import DECIMAL_WIDE, FIXED, VAR, words
from test_gpu_window_agg_rows import Table, table
from window_agg_model import (AVG, COUNT, FRAME_PARTITION, FRAME_RANGE, FRAME_ROWS, MAX, SUM, VAL_INT64, VAL_NONE,
                              dec, model_window_aggregate)
from window_model import RANK, ROW_NUMBER
from window_offset_model import (FIRST, HAS_DEFAULT, IGNORE_NULLS, LAG, LAST, LEAD, NTH_VALUE, VAL_BYTES,
                                 model_window_offset, offset_values, read_input, value_row)


def b(v):
    return v.to_bytes(8, "little")


X = [b(1), b(2), None, b(4)]
END = [1, 2, 3, 4]  # every row its own peer group


def test_lag_and_lead_at_the_partition_edges():
    assert offset_values(LAG, 1, 0, 0, 0, X, END) == [None, b(1), b(2), None]
    assert offset_values(LAG, 1, 0, HAS_DEFAULT, 9, X, END) == [b(9), b(1), b(2), None]  # a null input is not defaulted
    assert offset_values(LEAD, 2, 0, 0, 0, X, END) == [None, b(4), None, None]
    assert offset_values(LEAD, 2, 0, HAS_DEFAULT, 7, X, END) == [None, b(4), b(7), b(7)]
    assert offset_values(LEAD, 4, 0, HAS_DEFAULT, 7, X, END) == [b(7)] * 4
    assert offset_values(LAG, 2**31 - 1, 0, 0, 0, X, END) == [None] * 4


def test_ignore_nulls_past_the_partition():
    xs = [b(1), None, b(2), None, None]
    end = [1, 2, 3, 4, 5]
    # the 2nd non-null after row 0 would lie past the partition: the default
    assert offset_values(LEAD, 2, 0, IGNORE_NULLS | HAS_DEFAULT, 5, xs, end) == [b(5)] * 5
    assert offset_values(LEAD, 1, 0, IGNORE_NULLS, 0, xs, end) == [b(2), b(2), None, None, None]
    assert offset_values(LAG, 2, 0, IGNORE_NULLS, 0, xs, end) == [None, None, None, b(1), b(1)]
    assert offset_values(LAG, 1, 0, IGNORE_NULLS, 0, xs, end) == [None, b(1), b(1), b(2), b(2)]


def test_an_all_null_partition():
    xs = [None] * 3
    end = [1, 2, 3]
    for fn, arg, frame in ((FIRST, 0, FRAME_ROWS), (LAST, 0, FRAME_PARTITION), (NTH_VALUE, 1, FRAME_RANGE)):
        for flags in (0, IGNORE_NULLS):
            assert offset_values(fn, arg, frame, flags, 0, xs, end) == [None] * 3
    assert offset_values(LAG, 1, 0, IGNORE_NULLS | HAS_DEFAULT, 3, xs, end) == [b(3)] * 3
    assert offset_values(LEAD, 1, 0, HAS_DEFAULT, 3, xs, end) == [None, None, b(3)]


def test_nth_value_past_its_frame():
    assert offset_values(NTH_VALUE, 3, FRAME_ROWS, 0, 0, X, END) == [None, None, None, None]  # the 3rd input is null
    assert offset_values(NTH_VALUE, 2, FRAME_ROWS, 0, 0, X, END) == [None, b(2), b(2), b(2)]
    assert offset_values(NTH_VALUE, 3, FRAME_ROWS, IGNORE_NULLS, 0, X, END) == [None, None, None, b(4)]
    assert offset_values(NTH_VALUE, 5, FRAME_PARTITION, 0, 0, X, END) == [None] * 4
    assert offset_values(FIRST, 0, FRAME_ROWS, 0, 0, [None, b(1)], [1, 2]) == [None, None]
    assert offset_values(FIRST, 0, FRAME_ROWS, IGNORE_NULLS, 0, [None, b(1)], [1, 2]) == [None, b(1)]


def test_last_over_a_range_frame_with_peers():
    xs = [b(1), b(2), None, b(3)]
    end = [2, 2, 4, 4]  # two peer groups of two
    assert offset_values(LAST, 0, FRAME_RANGE, 0, 0, xs, end) == [b(2), b(2), b(3), b(3)]
    assert offset_values(LAST, 0, FRAME_ROWS, 0, 0, xs, end) == [b(1), b(2), None, b(3)]
    assert offset_values(LAST, 0, FRAME_ROWS, IGNORE_NULLS, 0, xs, end) == [b(1), b(2), b(2), b(3)]
    xs = [b(1), None, b(2), None]
    assert offset_values(LAST, 0, FRAME_RANGE, 0, 0, xs, end) == [None, None, None, None]
    assert offset_values(LAST, 0, FRAME_RANGE, IGNORE_NULLS, 0, xs, end) == [b(1), b(1), b(2), b(2)]
    assert offset_values(FIRST, 0, FRAME_RANGE, IGNORE_NULLS, 0, [None, None, b(5), None], end) == \
        [None, None, b(5), b(5)]


def test_var_regions_follow_function_order():
    """a string, a wide decimal aggregate, an empty string, a null string and a null wide decimal offset value"""
    fns = [(LEAD, 1, 0, VAL_BYTES, 8, -1, 0, 0), (MAX, 0, 1, dec(38, 2), 16, -1, 0, 0),
           (LAG, 1, 0, VAL_BYTES, 8, -1, 0, 0), (LAG, 1, 0, VAL_BYTES, 8, -1, 0, 0),
           (FIRST, 0, 1, dec(20, 0), 24, -1, 0, 0), (ROW_NUMBER, 0, 0, VAL_NONE, 0, -1, 0, 0)]
    row, kinds = value_row([b"hello", -300, b"", None, None, 3], fns)
    assert kinds == [VAR, DECIMAL_WIDE, VAR, VAR, DECIMAL_WIDE, FIXED]
    fixed = 8 * (words(6) + 6)
    slot = [int.from_bytes(row[8 + 8 * f:16 + 8 * f], "little") for f in range(6)]
    assert int.from_bytes(row[:8], "little") == 0b11000  # the null string and the null decimal
    assert slot[0] == (fixed << 32) | 5 and row[fixed:fixed + 8] == b"hello\0\0\0"
    assert slot[1] == ((fixed + 8) << 32) | 2 and row[fixed + 8:fixed + 24] == (-300).to_bytes(2, "big", signed=True) \
        + bytes(14)
    assert slot[2] == (fixed + 24) << 32  # an empty string: its offset, no bytes
    assert slot[3] == 0
    assert slot[4] == (fixed + 24) << 32 and row[fixed + 24:fixed + 40] == bytes(16)
    assert slot[5] == 3 and len(row) == fixed + 40


def test_read_input_masks_fixed_values_to_their_width():
    t = Table([dec(8, 2)])
    r = bytearray(t.row([0, 0, 0, 0], [(None, -1)]))
    s = t.slot(t.first + 1)
    r[s:s + 8] = (2**64 - 1).to_bytes(8, "little")
    assert read_input(bytes(r), 3, s, -1) == b(0xFFFFFFFF)  # an int: 4 bytes
    assert read_input(bytes(r), 1, s, -1) == b(0xFF)
    assert read_input(bytes(r), VAL_INT64, s, t.first) is None


def test_without_offset_functions_the_model_is_the_aggregate_model():
    rng = np.random.default_rng(5)
    t = Table()
    rows = table(rng, t, 400)
    plain = [b"".join(len(r).to_bytes(4, "big") + r for r in rows)]
    fns = [ROW_NUMBER, (SUM, FRAME_ROWS, *t.value(3)), RANK, (AVG, FRAME_RANGE, *t.value(8)),
           (MAX, FRAME_PARTITION, *t.value(10)), (COUNT, FRAME_RANGE, VAL_NONE, 0, -1), (SUM, FRAME_ROWS, *t.value(9))]
    assert model_window_offset(plain, t.keys(1), 1, t.nf, t.kinds, fns) == \
        model_window_aggregate(plain, t.keys(1), 1, t.nf, t.kinds, fns)
