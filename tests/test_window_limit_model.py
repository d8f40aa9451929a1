"""The partial-limit model (tests/window_limit_model.py) against hand-worked boundary ties, and the property that makes
the map-side limit safe: a reducer's window with the final limit over the maps' partially limited rows equals its
window over the unlimited rows.  No GPU."""
import struct

import numpy as np
import pytest

from hash_model import ids_scalar
from join_model import FIXED, VAR
from rows_model import STRING, stream
from test_gpu_sort_rows_order import DESC, KEY_FLOAT64, KLEN, NULLS_LAST
from window_limit_model import partial_limit
from window_model import DENSE_RANK, RANK, ROW_NUMBER, model_window

INT64 = 2
KEYS = [(INT64, 8, 8, -1), (INT64 | DESC, 16, 8, -1)]


def _row(part, order, tag=0):
    """three INT64 fields [partition, order, tag], one null word (nothing null)"""
    return bytes(8) + struct.pack("<qqq", part, order, tag)


def _triples(rows):
    return [struct.unpack("<qqq", r[8:32]) for r in rows]


# partition 1 in DESC order: 9, 8, 8, 8, 5 (the 8s in input order: tags 1, 4, 6); partition 2: 4, 4
ROWS = [_row(1, 8, 1), _row(2, 4, 2), _row(1, 9, 3), _row(1, 5, 4), _row(1, 8, 5), _row(2, 4, 6), _row(1, 8, 7)]


def test_rank_keeps_every_tie_at_the_boundary():
    assert _triples(partial_limit(ROWS, KEYS, 1, RANK, 2)) == [(1, 9, 3), (1, 8, 1), (1, 8, 5), (1, 8, 7), (2, 4, 2),
                                                               (2, 4, 6)]
    assert _triples(partial_limit(ROWS, KEYS, 1, RANK, 1)) == [(1, 9, 3), (2, 4, 2), (2, 4, 6)]
    assert _triples(partial_limit(ROWS, KEYS, 1, RANK, 4)) == [(1, 9, 3), (1, 8, 1), (1, 8, 5), (1, 8, 7), (2, 4, 2),
                                                               (2, 4, 6)]
    assert len(partial_limit(ROWS, KEYS, 1, RANK, 5)) == 7


def test_dense_rank_counts_peer_groups():
    assert _triples(partial_limit(ROWS, KEYS, 1, DENSE_RANK, 1)) == [(1, 9, 3), (2, 4, 2), (2, 4, 6)]
    assert len(partial_limit(ROWS, KEYS, 1, DENSE_RANK, 2)) == 6
    assert len(partial_limit(ROWS, KEYS, 1, DENSE_RANK, 3)) == 7


def test_row_number_cuts_ties_in_input_order():
    assert _triples(partial_limit(ROWS, KEYS, 1, ROW_NUMBER, 2)) == [(1, 9, 3), (1, 8, 1), (2, 4, 2), (2, 4, 6)]
    assert _triples(partial_limit(ROWS, KEYS, 1, ROW_NUMBER, 3)) == [(1, 9, 3), (1, 8, 1), (1, 8, 5), (2, 4, 2),
                                                                     (2, 4, 6)]


def test_no_partition_columns_is_one_partition():
    assert _triples(partial_limit(ROWS, KEYS[1:], 0, RANK, 2)) == [(1, 9, 3), (1, 8, 1), (1, 8, 5), (1, 8, 7)]
    assert _triples(partial_limit(ROWS, KEYS[1:], 0, ROW_NUMBER, 3)) == [(1, 9, 3), (1, 8, 1), (1, 8, 5)]
    assert _triples(partial_limit(ROWS, KEYS[1:], 0, DENSE_RANK, 3)) == [(1, 9, 3), (1, 8, 1), (1, 8, 5), (1, 8, 7),
                                                                         (1, 5, 4)]
    assert partial_limit([], KEYS[1:], 0, RANK, 1) == []


# ---------------------------------------------------------------------------------------------------------------
# the property: maps limited on their own, then shuffled, then limited and windowed by the reducer
# ---------------------------------------------------------------------------------------------------------------
ZEROS_NANS = [0.0, -0.0, float("nan"), struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000123))[0], 1.5, -1.5]


def _random_row(rng, strings):
    """fields: 0 a string or double partition column, 1 a nullable long order column, 2 a double order column, 3 a
    tag (the row's input position, so equal keys stay distinguishable); strings and nulls as UnsafeRowWriter writes"""
    bits = 0
    fixed = bytearray(8 + 8 * 4)
    var = b""
    if strings:
        if rng.random() < 0.1:
            bits |= 1
        else:
            s = b"cat-" * int(rng.integers(0, 6)) + bytes([65 + int(rng.integers(4))])
            fixed[8:16] = ((40 << 32) | len(s)).to_bytes(8, "little")
            var = s + bytes(-len(s) % 8)
    else:
        fixed[8:16] = struct.pack("<d", ZEROS_NANS[int(rng.integers(len(ZEROS_NANS)))])
    if rng.random() < 0.15:
        bits |= 2
    else:
        fixed[16:24] = struct.pack("<q", int(rng.integers(0, 6)))
    fixed[24:32] = struct.pack("<d", ZEROS_NANS[int(rng.integers(len(ZEROS_NANS)))])
    fixed[0:8] = bits.to_bytes(8, "little")
    return bytes(fixed) + var


@pytest.mark.parametrize("limit", [1, 2, 5])
@pytest.mark.parametrize("fn", [ROW_NUMBER, RANK, DENSE_RANK])
@pytest.mark.parametrize("strings", [True, False])
def test_partial_limits_leave_every_reducer_unchanged(fn, limit, strings):
    rng = np.random.default_rng(7 + 3 * fn + 11 * limit + strings)
    pk = (STRING if strings else KEY_FLOAT64, 8, 8, 0 if strings else -1)
    keys = [pk, (INT64 | DESC | NULLS_LAST, 16, 8, 1), (KEY_FLOAT64, 24, KLEN[KEY_FLOAT64], -1)]
    n_fields, kinds = 4, [VAR if strings else FIXED, FIXED, FIXED, FIXED]
    M, R = 4, 3
    rows = []
    for i in range(600):
        r = bytearray(_random_row(rng, strings))
        r[32:40] = struct.pack("<q", i)
        rows.append(bytes(r))
    maps = [rows[m::M] for m in range(M)]
    for red in range(R):
        # the reducer's blocks in map order, each holding that map's rows of the reducer in the map's output order
        limited = []
        unlimited = []
        for part in maps:
            kept = partial_limit(part, keys, 1, fn, limit)
            limited.append(stream([r for r, p in zip(kept, ids_scalar(kept, keys[:1], R)) if p == red]))
            unlimited.append(stream([r for r, p in zip(part, ids_scalar(part, keys[:1], R)) if p == red]))
        want = model_window(unlimited, keys, 1, n_fields, kinds, [fn], (fn, limit))
        got = model_window(limited, keys, 1, n_fields, kinds, [fn], (fn, limit))
        assert got[0] == want[0] and got[2] == want[2]
        assert got[1] <= want[1]


@pytest.mark.parametrize("fn", [ROW_NUMBER, RANK, DENSE_RANK])
def test_partial_limits_leave_a_single_partition_unchanged(fn):
    rng = np.random.default_rng(40 + fn)
    keys = [(INT64 | DESC | NULLS_LAST, 16, 8, 1), (KEY_FLOAT64, 24, 8, -1)]
    rows = [_random_row(rng, False) for _ in range(400)]
    maps = [rows[m::3] for m in range(3)]
    want = model_window([stream(p) for p in maps], keys, 0, 4, [FIXED] * 4, [fn], (fn, 7))
    got = model_window([stream(partial_limit(p, keys, 0, fn, 7)) for p in maps], keys, 0, 4, [FIXED] * 4, [fn],
                       (fn, 7))
    assert got[0] == want[0] and got[2] == want[2]
