"""The window model (tests/window_model.py) against hand-worked partitions, NTile's recurrence against the header's
closed form, and limits with ties at the boundary.  No GPU."""
import struct

import pytest

from join_model import FIXED, VAR
from rows_model import stream
from window_model import CUME_DIST, DENSE_RANK, NTILE, PERCENT_RANK, RANK, ROW_NUMBER, model_window, ntile_recurrence, \
    partition_values

INT64 = 2
DESC, NULLS_LAST = 1 << 8, 1 << 9


def test_hand_worked_partition():
    v = [1, 1, 2, 3, 3, 3]
    assert partition_values(v, ROW_NUMBER) == [1, 2, 3, 4, 5, 6]
    assert partition_values(v, RANK) == [1, 1, 3, 4, 4, 4]
    assert partition_values(v, DENSE_RANK) == [1, 1, 2, 3, 3, 3]
    assert partition_values(v, PERCENT_RANK) == [0.0, 0.0, 0.4, 0.6, 0.6, 0.6]
    assert partition_values(v, CUME_DIST) == [1 / 3, 1 / 3, 1 / 2, 1.0, 1.0, 1.0]
    assert partition_values(v, NTILE, 4) == [1, 1, 2, 2, 3, 4]


def test_single_row_and_all_peers():
    assert partition_values([7], PERCENT_RANK) == [0.0]
    assert partition_values([7], CUME_DIST) == [1.0]
    assert partition_values([5] * 4, RANK) == [1] * 4
    assert partition_values([5] * 4, DENSE_RANK) == [1] * 4
    assert partition_values([5] * 4, CUME_DIST) == [1.0] * 4
    assert partition_values([5] * 4, ROW_NUMBER) == [1, 2, 3, 4]
    assert partition_values([1, 2, 3], NTILE, 5) == [1, 2, 3]


def closed_form(i, N, k):
    """the header's NTILE: the first N % k buckets hold N / k + 1 rows, the rest N / k"""
    q, r = divmod(N, k)
    big = r * (q + 1)
    return i // (q + 1) + 1 if i < big else r + (i - big) // q + 1


def test_ntile_recurrence_is_the_closed_form():
    for N in range(1, 201):
        for k in range(1, 221):
            assert ntile_recurrence(N, k) == [closed_form(i, N, k) for i in range(N)], (N, k)


def _row(part, order):
    """two INT64 fields [partition, order], one null word (nothing null)"""
    return bytes(8) + struct.pack("<qq", part, order)


KEYS = [(INT64, 8, 8, -1), (INT64 | DESC, 16, 8, -1)]


def _values(out):
    rows, p = [], 0
    while p < len(out):
        s = int.from_bytes(out[p:p + 4], "big")
        r = out[p + 4:p + 4 + s]
        rows.append((struct.unpack("<qq", r[8:24]), [int.from_bytes(r[24 + 8 * f:28 + 8 * f], "little")
                                                      for f in range((len(r) - 24) // 8)]))
        p += 4 + s
    return rows


def test_limits_keep_ties_at_the_boundary():
    # partition 1 in DESC order: 9, 8, 8, 8, 5; partition 2: 4, 4
    rows = [_row(1, 8), _row(2, 4), _row(1, 9), _row(1, 5), _row(1, 8), _row(2, 4), _row(1, 8)]
    plain = [stream(rows[:3]), stream(rows[3:])]
    fns = [ROW_NUMBER, RANK, DENSE_RANK]
    out, n, m = model_window(plain, KEYS, 1, 2, [FIXED, FIXED], fns, (RANK, 2))
    got = _values(out)
    assert (n, m) == (7, 6)
    assert got == [((1, 9), [1, 1, 1]), ((1, 8), [2, 2, 2]), ((1, 8), [3, 2, 2]), ((1, 8), [4, 2, 2]),
                   ((2, 4), [1, 1, 1]), ((2, 4), [2, 1, 1])]
    assert [g[0] for g in _values(model_window(plain, KEYS, 1, 2, [FIXED, FIXED], fns, (DENSE_RANK, 2))[0])] == \
        [(1, 9), (1, 8), (1, 8), (1, 8), (2, 4), (2, 4)]
    assert [g[0] for g in _values(model_window(plain, KEYS, 1, 2, [FIXED, FIXED], fns, (DENSE_RANK, 3))[0])] == \
        [(1, 9), (1, 8), (1, 8), (1, 8), (1, 5), (2, 4), (2, 4)]
    assert [g[0] for g in _values(model_window(plain, KEYS, 1, 2, [FIXED, FIXED], fns, (ROW_NUMBER, 1))[0])] == \
        [(1, 9), (2, 4)]
    assert model_window(plain, KEYS, 1, 2, [FIXED, FIXED], fns, (RANK, 100))[2] == 7


def test_output_row_layout():
    """63 input fields and two functions: the null bitset grows to two words, a VAR field's offset moves past it"""
    nf, fns = 63, [ROW_NUMBER, PERCENT_RANK]
    kinds = [FIXED] * nf
    kinds[5] = VAR
    var = b"abcdefgh"
    fixed = 8 * (1 + nf)
    row = bytearray(fixed) + var
    row[0:8] = (1 << 62 | 1 << 3).to_bytes(8, "little")  # null bits 3 and 62
    row[8 + 8 * 5:16 + 8 * 5] = (fixed << 32 | len(var)).to_bytes(8, "little")
    row[8 + 8 * 1:16 + 8 * 1] = (42).to_bytes(8, "little")
    out, n, m = model_window([stream([bytes(row)])], [(INT64, 16, 8, -1)], 0, nf, kinds, fns)
    assert (n, m) == (1, 1)
    r = out[4:]
    assert int.from_bytes(out[:4], "big") == len(r) == 8 * (2 + nf + 2) + len(var)
    assert int.from_bytes(r[0:8], "little") == 1 << 62 | 1 << 3 and r[8:16] == bytes(8)
    slot = int.from_bytes(r[16 + 8 * 5:24 + 8 * 5], "little")
    assert slot >> 32 == fixed + 8 * (2 - 1 + 2) and slot & 0xFFFFFFFF == len(var)
    assert r[16 + 8 * nf:24 + 8 * nf] == (1).to_bytes(8, "little")
    assert r[24 + 8 * nf:32 + 8 * nf] == struct.pack("<d", 0.0)
    assert r[32 + 8 * nf:] == var


@pytest.mark.parametrize("flags", [0, DESC, NULLS_LAST])
def test_null_order_keys_are_peers(flags):
    keys = [(INT64 | flags, 16, 8, 1)]
    null = (1 << 1).to_bytes(8, "little") + bytes(16)
    rows = [_row(0, 3), null, _row(0, 1), null]
    out, _, _ = model_window([stream(rows)], keys, 0, 2, [FIXED, FIXED], [RANK])
    ranks = [v[1][0] for v in _values(out)]
    assert ranks == ([1, 1, 3, 4] if not flags & NULLS_LAST else [1, 2, 3, 3])
