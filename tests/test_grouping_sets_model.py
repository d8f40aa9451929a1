"""The grouping-sets model (tests/grouping_sets_model.py) pinned without a GPU: Spark's spark_grouping_id for ROLLUP,
CUBE and explicit GROUPING SETS, hand-worked Expand rows and partial rows, and partial rows of several maps merged by the
reduce-side model equal to a plain GROUP BY of each set over the whole dataset."""
import numpy as np

import decimal_model as dm
import grouping_sets_model as gm
import hash_model as hm
import partial_agg_model as pm
import rows_model as rm
from test_gpu_sort_rows_order import col_value

T = ["int", "long", "string", "int", "long", "decimal"]  # a, b, c, then the inputs: int, long, decimal(25, 0)


def agg(fn, vt, field):
    return (fn, vt, 8 + 8 * field, field)


def keys3():
    return hm.keys_of(T, [0, 1, 2])


def decode(prow, keys, aggs):
    """a partial row -> (grouping values, gid, buffer values as the model's state_values gives them)"""
    xkeys = pm.output_keys(gm.projected_keys(keys))
    nk = len(keys)
    vals = tuple(col_value(prow, k) for k in xkeys[:nk])
    g = int.from_bytes(prow[8 + 8 * nk:16 + 8 * nk], "little")
    out = []
    for b, (op, kind) in enumerate(pm.buffers(aggs)):
        f = nk + 1 + b
        if (int.from_bytes(prow[:8], "little") >> f) & 1:
            out.append(None)
            continue
        slot = prow[8 + 8 * f:16 + 8 * f]
        if pm.wide_op(op):
            s = int.from_bytes(slot, "little")
            out.append(int.from_bytes(prow[s >> 32:(s >> 32) + (s & 0xFFFFFFFF)], "big", signed=True))
        elif kind in ("int", "bool"):
            out.append(int.from_bytes(slot[:4], "little", signed=True))
        else:
            out.append(int.from_bytes(slot, "little", signed=True))
    return vals, g, out


def test_spark_grouping_ids():
    assert [gm.gid(m, 3) for m in gm.rollup(3)] == [0, 1, 3, 7]
    assert gm.rollup(3) == [0b111, 0b011, 0b001, 0]
    assert [gm.gid(m, 2) for m in gm.cube(2)] == [0, 1, 2, 3]
    assert gm.cube(2) == [0b11, 0b01, 0b10, 0]  # (a, b), (a), (b), ()
    assert [gm.gid(m, 2) for m in (0b01, 0b11, 0)] == [1, 0, 3]  # GROUPING SETS ((a), (a, b), ())
    assert len(set(gm.cube(4))) == 16 and sorted(gm.gid(m, 4) for m in gm.cube(4)) == list(range(16))


def test_expand_rows_are_row_major_with_masked_keys_and_unmasked_inputs():
    rows = [hm.make_row(T, [1, 10, b"x", 5, 50, 10**20]), hm.make_row(T, [2, None, b"yy", None, 7, None])]
    keys = keys3()
    aggs = [agg(pm.SUM, pm.VAL_INT32, 3), agg(pm.MAX, pm.VAL_INT64, 4), agg(pm.SUM, pm.val_decimal(25, 0), 5),
            (pm.COUNT, pm.VAL_NONE, 0, -1)]
    xrows, xkeys, xaggs = gm.expand(rows, keys, aggs, gm.rollup(3))
    assert len(xrows) == 8
    assert xaggs == [(pm.SUM, pm.VAL_INT32, 40, 4), (pm.MAX, pm.VAL_INT64, 48, 5),
                     (pm.SUM, pm.val_decimal(25, 0), 56, 6), (pm.COUNT, pm.VAL_NONE, 0, -1)]
    got = [(tuple(col_value(x, k) for k in xkeys), [pm.read_value(x, *a[1:]) for a in xaggs[:3]]) for x in xrows]
    assert got == [((1, 10, b"x", 0), [5, 50, 10**20]), ((1, 10, None, 1), [5, 50, 10**20]),
                   ((1, None, None, 3), [5, 50, 10**20]), ((None, None, None, 7), [5, 50, 10**20]),
                   ((2, None, b"yy", 0), [None, 7, None]), ((2, None, None, 1), [None, 7, None]),
                   ((2, None, None, 3), [None, 7, None]), ((None, None, None, 7), [None, 7, None])]


def test_rollup_partial_rows_hand_worked():
    data = [(1, 10, b"x", 5), (1, 10, b"y", 7), (1, 20, b"x", 1), (2, 10, b"x", 2)]
    rows = [hm.make_row(T, [a, b, c, v, v, v]) for a, b, c, v in data]
    aggs = [agg(pm.SUM, pm.VAL_INT32, 3), (pm.COUNT, pm.VAL_NONE, 0, -1)]
    got = [decode(p, keys3(), aggs) for p in gm.partial_rows(rows, keys3(), aggs, gm.rollup(3))]
    # the composite-key order: grouping columns nulls first, then gid
    assert got == [((None, None, None), 7, [15, 4]),
                   ((1, None, None), 3, [13, 3]), ((1, 10, None), 1, [12, 2]),
                   ((1, 10, b"x"), 0, [5, 1]), ((1, 10, b"y"), 0, [7, 1]),
                   ((1, 20, None), 1, [1, 1]), ((1, 20, b"x"), 0, [1, 1]),
                   ((2, None, None), 3, [2, 1]), ((2, 10, None), 1, [2, 1]), ((2, 10, b"x"), 0, [2, 1])]


def test_cube_and_explicit_sets_hand_worked():
    data = [(1, 10, 5), (1, 20, 7), (2, 10, None)]
    rows = [hm.make_row(T, [a, b, b"s", v, 0, 0]) for a, b, v in data]
    keys = hm.keys_of(T, [0, 1])
    aggs = [agg(pm.SUM, pm.VAL_INT32, 3), agg(pm.COUNT, pm.VAL_INT32, 3)]
    got = [decode(p, keys, aggs) for p in gm.partial_rows(rows, keys, aggs, gm.cube(2))]
    assert got == [((None, None), 3, [12, 2]), ((None, 10), 2, [5, 1]), ((None, 20), 2, [7, 1]),
                   ((1, None), 1, [12, 2]), ((1, 10), 0, [5, 1]), ((1, 20), 0, [7, 1]),
                   ((2, None), 1, [None, 0]), ((2, 10), 0, [None, 0])]
    # GROUPING SETS ((a), (a, b), ()): the grand total and a null key of its own set stay apart by gid
    rows.append(hm.make_row(T, [None, None, b"s", 1, 0, 0]))
    got = [decode(p, keys, aggs) for p in gm.partial_rows(rows, keys, aggs, [0b01, 0b11, 0])]
    assert got == [((None, None), 0, [1, 1]), ((None, None), 1, [1, 1]), ((None, None), 3, [13, 3]),
                   ((1, None), 1, [12, 2]), ((1, 10), 0, [5, 1]), ((1, 20), 0, [7, 1]),
                   ((2, None), 1, [None, 0]), ((2, 10), 0, [None, 0])]


def merged_rows(partials, keys, aggs):
    xkeys = gm.projected_keys(keys)
    buf, _, _ = dm.model_aggregate_decimal([rm.stream(partials)], pm.output_keys(xkeys), pm.merge_aggs(xkeys, aggs))
    out, at = [], 0
    while at < len(buf):
        sz = int.from_bytes(buf[at:at + 4], "big")
        out.append(bytes(buf[at + 4:at + 4 + sz]))
        at += 4 + sz
    return out


def test_several_maps_merged_equal_a_group_by_of_each_set():
    rng = np.random.default_rng(2)
    n = 600
    rows = [hm.make_row(T, [None if rng.random() < 0.1 else int(rng.integers(0, 4)),
                            None if rng.random() < 0.1 else int(rng.integers(0, 3)),
                            None if rng.random() < 0.1 else bytes(b"k%d" % rng.integers(0, 3)),
                            None if rng.random() < 0.2 else int(rng.integers(-99, 99)),
                            int(rng.integers(-10**12, 10**12)),
                            None if rng.random() < 0.2 else int(rng.integers(-10**18, 10**18)) * 1000])
            for _ in range(n)]
    keys = keys3()
    aggs = [agg(pm.SUM, pm.VAL_INT32, 3), agg(pm.AVG, pm.val_decimal(25, 0), 5), agg(pm.MIN, pm.VAL_INT64, 4),
            agg(pm.MAX, pm.val_decimal(25, 0), 5), (pm.COUNT, pm.VAL_NONE, 0, -1), agg(pm.COUNT, pm.VAL_INT32, 3),
            agg(pm.SUM, pm.val_decimal(25, 0), 5)]
    for masks in (gm.rollup(3), gm.cube(3), [0b001, 0b011, 0], [0b111]):
        maps = [rows[m::3] for m in range(3)]
        partials = [p for m in maps for p in gm.partial_rows(m, keys, aggs, masks)]
        want = gm.group_by_each_set(rows, keys, aggs, masks)
        got = {}
        for r in merged_rows(partials, keys, aggs):
            vals, g, bufs = decode(r, keys, aggs)
            got[vals + (g,)] = bufs
        assert got == want
