"""tests/window_agg_model.py against hand-worked partitions and Spark's decimal division, without a GPU."""
import decimal
import struct

import pytest

from join_model import KEY_INT64
from window_agg_model import (AVG, COUNT, FRAME_PARTITION, FRAME_RANGE, FRAME_ROWS, MAX, MIN, SUM, VAL_DECIMAL,
                              VAL_FLOAT32, VAL_FLOAT64, VAL_INT8, VAL_INT64, VAL_NONE, avg_decimal, dec,
                              model_window_aggregate, value_row, fn_list)
from window_model import RANK

NAN_A, NAN_B = 0x7FF8000000000001, 0xFFF0000000000002  # two NaN payloads, the second negative


def row2(part, order, x, x_null=False):
    """an UnsafeRow of 3 fields: partition key, order key, an 8-byte value (int or raw bytes); x_null sets field 2's
    null bit"""
    bits = 4 if x_null else 0
    xb = bytes(8) if x_null else x if isinstance(x, bytes) else (x % 2**64).to_bytes(8, "little")
    return bits.to_bytes(8, "little") + part.to_bytes(8, "little", signed=True) + \
        order.to_bytes(8, "little", signed=True) + xb


KEYS = [(KEY_INT64, 8, 8, -1), (KEY_INT64, 16, 8, -1)]


def values_of(rows, fns, npk=1):
    """run the model and read back each output row's value slots and null bits, in output order"""
    stream, n, m = model_window_aggregate([b"".join(len(r).to_bytes(4, "big") + r for r in rows)], KEYS, npk, 3,
                                          [0, 0, 0], fns)
    out, p = [], 0
    while p < len(stream):
        size = int.from_bytes(stream[p:p + 4], "big")
        r = stream[p + 4:p + 4 + size]
        bits = int.from_bytes(r[:8], "little")
        slots = [r[8 * (1 + 3 + j):8 * (1 + 3 + j) + 8] for j in range(len(fns))]
        out.append([None if (bits >> (3 + j)) & 1 else s for j, s in enumerate(slots)])
        p += 4 + size
    return out


def as_long(b):
    return None if b is None else int.from_bytes(b, "little", signed=True)


def as_double(b):
    return None if b is None else struct.unpack("<d", b)[0]


def test_rows_and_range_running_sums_with_peer_ties():
    # partition 0: order keys 1, 2, 2, 3 with x 10, 20, 30, 40; partition 1: one row
    rows = [row2(0, 1, 10), row2(0, 2, 20), row2(0, 2, 30), row2(0, 3, 40), row2(1, 5, 7)]
    fns = [(SUM, FRAME_ROWS, VAL_INT64, 24, 2), (SUM, FRAME_RANGE, VAL_INT64, 24, 2),
           (SUM, FRAME_PARTITION, VAL_INT64, 24, 2), (COUNT, FRAME_RANGE, VAL_NONE, 0, -1), RANK]
    got = [[as_long(s) for s in v[:4]] for v in values_of(rows, fns)]
    assert got == [[10, 10, 100, 1], [30, 60, 100, 3], [60, 60, 100, 3], [100, 100, 100, 4], [7, 7, 7, 1]]


def test_all_null_frames_are_null_and_count_is_zero():
    rows = [row2(0, 1, 0, True), row2(0, 2, 5), row2(0, 3, 0, True)]
    fns = [(SUM, FRAME_ROWS, VAL_INT64, 24, 2), (MIN, FRAME_ROWS, VAL_INT64, 24, 2),
           (AVG, FRAME_ROWS, VAL_INT64, 24, 2), (COUNT, FRAME_ROWS, VAL_INT64, 24, 2)]
    got = values_of(rows, fns)
    assert [as_long(v[0]) for v in got] == [None, 5, 5]
    assert [as_long(v[1]) for v in got] == [None, 5, 5]
    assert [as_double(v[2]) for v in got] == [None, 5.0, 5.0]
    assert [as_long(v[3]) for v in got] == [0, 1, 1]


def test_a_lone_negative_zero_sums_to_positive_zero():
    rows = [row2(0, 1, struct.pack("<d", -0.0))]
    got = values_of(rows, [(SUM, FRAME_ROWS, VAL_FLOAT64, 24, 2), (MIN, FRAME_ROWS, VAL_FLOAT64, 24, 2)])
    assert got[0][0] == struct.pack("<d", 0.0) and got[0][1] == struct.pack("<d", -0.0)


def test_min_max_keep_the_first_of_equal_values_with_their_bits():
    xs = [struct.pack("<d", 0.0), struct.pack("<d", -0.0), NAN_A.to_bytes(8, "little"), NAN_B.to_bytes(8, "little"),
          struct.pack("<d", -1.0)]
    rows = [row2(0, k, x) for k, x in enumerate(xs)]
    fns = [(MIN, FRAME_ROWS, VAL_FLOAT64, 24, 2), (MAX, FRAME_ROWS, VAL_FLOAT64, 24, 2)]
    got = values_of(rows, fns)
    assert [v[0] for v in got] == [xs[0], xs[0], xs[0], xs[0], xs[4]]  # -0.0 equals 0.0: the first stays
    assert [v[1] for v in got] == [xs[0], xs[0], xs[2], xs[2], xs[2]]  # NaN is the largest; the first NaN stays


def test_float32_and_int8_results_are_written_as_unsafe_row_writer_writes_them():
    # row 1: 2.5f in the low 4 bytes (low byte 0x00), junk above; row 2: 0xFD, a tiny positive float and -3 as a byte
    rows = [row2(0, 1, struct.pack("<f", 2.5) + b"\xff" * 4), row2(0, 2, 0xFD)]
    got = values_of(rows, [(MIN, FRAME_PARTITION, VAL_FLOAT32, 24, 2), (MAX, FRAME_PARTITION, VAL_FLOAT32, 24, 2),
                           (MIN, FRAME_PARTITION, VAL_INT8, 24, 2), (MAX, FRAME_PARTITION, VAL_INT8, 24, 2)])
    assert got[0] == [bytes([0xFD]) + bytes(7), struct.pack("<f", 2.5) + bytes(4), bytes([0xFD]) + bytes(7), bytes(8)]


def test_double_sum_is_the_sequential_sum_not_a_reassociated_one():
    xs = [1e16, 1.0, -1e16, 1.0]
    rows = [row2(0, k, struct.pack("<d", x)) for k, x in enumerate(xs)]
    got = [as_double(v[0]) for v in values_of(rows, [(SUM, FRAME_ROWS, VAL_FLOAT64, 24, 2)])]
    assert got == [1e16, 1e16, 0.0, 1.0]  # 1e16 + 1.0 rounds back to 1e16
    assert (1e16 + -1e16) + (1.0 + 1.0) == 2.0  # a reassociated sum differs


def test_decimal_sum_result_type_and_wide_bytes():
    # decimal(17, 2) sum is decimal(27, 2): a wide result of BigInteger bytes after the input's var bytes
    rows = [row2(0, 1, 10**17 - 1), row2(0, 2, 10**17 - 1), row2(0, 3, 0, True)]
    fns = [(SUM, FRAME_ROWS, dec(17, 2), 24, 2), (MIN, FRAME_ROWS, dec(17, 2), 24, 2)]
    stream, _, _ = model_window_aggregate([b"".join(len(r).to_bytes(4, "big") + r for r in rows)], KEYS, 1, 3,
                                          [0, 0, 0], fns)
    size = int.from_bytes(stream[:4], "big")
    r = stream[4:4 + size]
    slot = int.from_bytes(r[8 * 4:8 * 5], "little")
    o, n = slot >> 32, slot & 0xFFFFFFFF
    assert o == 8 * (1 + 3 + 2) and len(r) == o + 16
    assert int.from_bytes(r[o:o + n], "big", signed=True) == 10**17 - 1
    assert int.from_bytes(r[8 * 5:8 * 6], "little", signed=True) == 10**17 - 1  # MIN keeps decimal(17, 2): a long


def test_value_row_of_a_null_wide_decimal_keeps_its_16_zero_bytes():
    fns = fn_list([(SUM, FRAME_ROWS, dec(20, 0), 16, 2), (COUNT, FRAME_ROWS, VAL_NONE, 0, -1)])
    row, kinds = value_row([None, 3], fns)
    assert kinds == [2, 0]
    assert int.from_bytes(row[:8], "little") == 1
    assert int.from_bytes(row[8:16], "little") == (8 * 3) << 32 and row[24:] == bytes(16)


def _spark_avg(S, c, s):
    """Spark's decimal average: Decimal./ to 38 significant digits (HALF_UP), then rounded HALF_UP to scale s + 4;
    worked at 60 digits so the first division is exact before its rounding"""
    ctx = decimal.Context(prec=60, rounding=decimal.ROUND_HALF_UP)
    q = ctx.divide(decimal.Decimal(S).scaleb(-s, context=ctx), decimal.Decimal(c))
    q38 = decimal.Context(prec=38, rounding=decimal.ROUND_HALF_UP).plus(q)
    return int(q38.quantize(decimal.Decimal(1).scaleb(-(s + 4)), rounding=decimal.ROUND_HALF_UP, context=ctx)
               .scaleb(s + 4, context=ctx))


@pytest.mark.parametrize("s", [0, 2, 10, 24])
def test_decimal_average_single_rounding_equals_sparks_two_at_p24(s):
    top = 10**24 - 1
    counts = [1, 2, 3, 7, 2**31 - 1, 2**31 - 2, 99991, 4, 8, 16, 10**4, 3 * 10**4]
    for c in counts:
        for S in (top * c, -top * c, top * c - 1, -(top * c - 1), c // 2, -(c // 2), 1, -1, 0, top, -top,
                  # exact half-points at scale + 4: S 10^4 / c = k + 1/2
                  (2 * 12345 + 1) * c // 2 // 10**4 if c % 2 == 0 else 0):
            assert avg_decimal(S, c) == _spark_avg(S, c, s), (S, c, s)


def test_decimal_average_half_points_round_away_from_zero():
    # S / c = 0.00005 at scale 0 -> 10^-4 units: 0.5 -> 1; negative -> -1
    assert avg_decimal(1, 2 * 10**4) == 1 and avg_decimal(-1, 2 * 10**4) == -1
    assert _spark_avg(1, 2 * 10**4, 0) == 1 and _spark_avg(-1, 2 * 10**4, 0) == -1
    # 5 / 8 = 0.625 exactly, in 10^-4 units 6250
    assert avg_decimal(5, 8) == 6250 == _spark_avg(5, 8, 0)
    assert avg_decimal(-3, 16 * 10**4) == -_spark_avg(3, 16 * 10**4, 0) == -avg_decimal(3, 16 * 10**4)


def test_no_order_column_with_whole_partition_frames():
    rows = [row2(1, 9, 4), row2(0, 8, 1), row2(1, 7, 6), row2(0, 6, 2)]
    stream, n, m = model_window_aggregate([b"".join(len(r).to_bytes(4, "big") + r for r in rows)], KEYS[:1], 1, 3,
                                          [0, 0, 0], [(AVG, FRAME_PARTITION, VAL_INT64, 24, 2)])
    assert (n, m) == (4, 4)
    got, p = [], 0
    while p < len(stream):
        size = int.from_bytes(stream[p:p + 4], "big")
        got.append(struct.unpack("<d", stream[p + 4 + 32:p + 4 + 40])[0])
        p += 4 + size
    assert got == [1.5, 1.5, 5.0, 5.0]


def test_constants_are_numbered_after_ntile():
    from window_model import NTILE
    assert SUM == NTILE + 1 and AVG == SUM + 4 and VAL_DECIMAL == 7 and dec(38, 38) >> 16 == 38
    assert VAL_INT8 == 1 and VAL_FLOAT32 == 5 and VAL_FLOAT64 == 6
