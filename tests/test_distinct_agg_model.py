"""The distinct aggregation model (tests/distinct_agg_model.py) on hand-worked reducers, the equivalence of PartialMerge
and the update fold for the simple buffers, and maps -> model -> final merge against numpy's distinct counts and sums.
No GPU."""
import struct

import numpy as np

import decimal_model as dm
import distinct_agg_model as da
import hash_model as hm
import moments_model as mm
import partial_agg_model as pm
import rows_model as rm

SUM, COUNT, AVG, MIN, MAX, VAR = pm.SUM, pm.COUNT, pm.AVG, pm.MIN, pm.MAX, mm.VARIANCE
INT, LONG = hm.FIELD["int"][0], hm.FIELD["long"][0]


def maps_of(types, nk, f, maps):
    """maps of input rows [G.., X.., values..] -> their map-side partial rows (keys G ++ X, f over the values)"""
    keys = hm.keys_of(types, list(range(nk)))
    aggs = [(fn, vt, keys[0][1] + 8 * (nk + j), nk + j) for fn, vt, j in f]
    return [rm.stream(mm.partial_rows([hm.make_row(types, r) for r in rows], keys, aggs)) for rows in maps]


def fields(row, n):
    return [None if rm.is_null(row, k) else row[8 + 8 * k:16 + 8 * k] for k in range(n)]


def long_at(row, k):
    return int.from_bytes(row[8 + 8 * k:16 + 8 * k], "little", signed=True)


def test_null_x_is_not_counted():
    types = ["int", "int", "long"]
    streams = maps_of(types, 2, [(SUM, pm.VAL_INT64, 0)],
                      [[[1, 5, 10], [1, None, 20], [1, 5, 1]], [[1, 7, 2], [1, None, 3]]])
    out, counts = da.reducer(streams, 1, [(INT, 4), (INT, 4)], [(SUM, pm.VAL_INT64)],
                             [(COUNT, pm.VAL_INT32, 1), (SUM, pm.VAL_INT32, 1)])
    assert counts == [4, 3, 1]
    (row,) = out
    assert [long_at(row, k) for k in (1, 2, 3)] == [36, 2, 12]  # sum(v), count(DISTINCT x), sum(DISTINCT x)


def test_count_distinct_of_two_columns_skips_a_null_side():
    types = ["int", "int", "int", "long"]
    streams = maps_of(types, 3, [(COUNT, pm.VAL_NONE, 0)],
                      [[[1, 1, 1, 0], [1, 1, None, 0], [1, None, 2, 0], [1, 2, 2, 0], [1, 1, 1, 0]]])
    out, counts = da.reducer(streams, 1, [(INT, 4)] * 3, [(COUNT, pm.VAL_NONE)], [(COUNT, pm.VAL_NONE, da.ALL)])
    assert counts == [4, 4, 1]  # the map merged its two (1, 1, 1) rows
    assert [long_at(out[0], k) for k in (1, 2)] == [5, 2]  # count(*), count(DISTINCT a, b)


def dec_partial_rows(rows):
    """map-side partial rows [G int, X int, sum decimal(38), isEmpty] written directly by pm.emit"""
    keys = hm.keys_of(["int", "int"], [0, 1])
    bufs = pm.buffers([(SUM, pm.val_decimal(28, 0), 0, -1)])
    return [pm.emit(hm.make_row(["int", "int"], [g, x]), keys, bufs, [v, int(e)]) for g, x, v, e in rows]


def test_decimal_overflow_in_one_gx_group_nulls_its_g_group():
    big = 9 * 10**37
    streams = [rm.stream(dec_partial_rows(rows)) for rows in (
        [[1, 1, big, False], [1, 2, 5, False], [2, 1, 7, False]], [[1, 1, big, False], [2, 2, 0, True]])]
    out, counts = da.reducer(streams, 1, [(INT, 4), (INT, 4)], [(SUM, pm.val_decimal(28, 0))],
                             [(COUNT, pm.VAL_INT32, 1)])
    assert counts == [5, 4, 2]
    one, two = out
    assert rm.is_null(one, 1) and not rm.is_null(two, 1)
    assert dm.dec_value(two, 16, dm.sum_decimal(38)) == 7 and long_at(two, 2) == 0  # sum 7, isEmpty false
    assert long_at(one, 3) == 2 and long_at(two, 3) == 2


def test_global_aggregate_without_rows_writes_the_initial_buffers():
    out, counts = da.reducer([], 0, [(LONG, 8)],
                             [(SUM, pm.VAL_INT64), (COUNT, pm.VAL_NONE), (AVG, pm.VAL_FLOAT64),
                              (SUM, pm.val_decimal(5, 0)), (MIN, pm.VAL_INT64), (VAR, pm.VAL_INT32)],
                             [(COUNT, pm.VAL_INT64, 0)])
    assert counts == [0, 0, 1]
    (row,) = out
    got = fields(row, 11)
    assert got[0] is None and got[6] is None  # Sum(long), Min
    assert all(got[k] == bytes(8) for k in (1, 2, 3, 4, 7, 8, 9, 10))  # count, avg [0.0, 0], decimal sum 0, (0, 0, 0)
    assert got[5] == (1).to_bytes(8, "little")  # isEmpty
    assert long_at(row, 10) == 0


def test_partial_merge_equals_the_update_fold_for_the_simple_buffers():
    """coalesce(coalesce(l, 0) + r, l) (Sum long / double) and Least / Greatest (Min / Max) over partial buffers give
    the bits pm.update gives when the buffers are its inputs"""
    rng = np.random.default_rng(1)
    vals = [None, -0.0, 0.0, float("nan"), 1.5, -2.5, 1e300, -1e300, 3.0]
    for _ in range(200):
        bufs = [vals[int(rng.integers(len(vals)))] for _ in range(int(rng.integers(1, 8)))]
        ints = [None if b is None or b != b else int(b) % 1000 - 500 for b in bufs]
        for fn, vt, xs, op in ((SUM, pm.VAL_FLOAT64, bufs, pm.SUM_F64), (SUM, pm.VAL_INT64, ints, pm.SUM_I64),
                               (MIN, pm.VAL_FLOAT64, bufs, pm.MIN_F64), (MAX, pm.VAL_FLOAT64, bufs, pm.MAX_F64),
                               (MIN, pm.VAL_INT64, ints, pm.MIN_I64), (MAX, pm.VAL_INT32, ints, pm.MAX_I32)):
            types = ["double" if vt == pm.VAL_FLOAT64 else "long" if vt == pm.VAL_INT64 else "int"]
            rows = [hm.make_row(types, [x]) for x in xs]
            st = pm.new_state([(fn, vt, 8, 0)])
            for r in rows:
                pm.update(st, [(fn, vt, 8, 0)], r)
            (upd,) = pm.state_values(st, [(fn, vt, 8, 0)])
            present = [bytes(r[8:16]) for r in rows if not rm.is_null(r, 0)]
            merged = rm.merge(op, present) if present else None
            if upd is None or merged is None:
                assert upd is None and merged is None
            elif vt == pm.VAL_FLOAT64:
                assert struct.pack("<d", upd) == merged or (upd != upd and struct.unpack("<d", merged)[0] != 0)
            else:
                assert upd == int.from_bytes(merged[:8 if vt == pm.VAL_INT64 else 4], "little", signed=True)


def final_rows(out_blocks, n_group_keys, aggs, distinct):
    """the Final merge by G of the reducers' output rows (decimal_model / moments_model's aggregated read)"""
    keys = da.input_keys([(INT, 4)] * n_group_keys)
    plain = [rm.stream(rows) for rows in out_blocks]
    merged, _, _ = mm.model_aggregate(plain, keys, da.final_aggs(n_group_keys, aggs, distinct))
    return [merged[o + 4:o + n] for o, n in rm.parse(merged)]


def test_maps_model_and_final_merge_equal_numpy():
    """over several map splits and reducers: count(DISTINCT x), sum(DISTINCT x) and avg(DISTINCT d) per g, beside
    sum(v), exact for integers and decimals and within rounding for doubles"""
    rng = np.random.default_rng(7)
    types = ["int", "int", "long", "long"]
    data = [(int(rng.integers(0, 6)), None if rng.random() < 0.05 else int(rng.integers(0, 40)),
             int(rng.integers(-1000, 1000)), int(rng.integers(-10**6, 10**6))) for _ in range(3000)]
    aggs = [(SUM, pm.VAL_INT64), (SUM, pm.val_decimal(10, 2))]
    distinct = [(COUNT, pm.VAL_INT32, 1), (SUM, pm.VAL_INT32, 1), (AVG, pm.VAL_INT32, 1)]
    for n_maps, n_red in ((1, 1), (3, 2), (5, 4)):
        maps = [[list(r) for r in data[m::n_maps]] for m in range(n_maps)]
        partial = maps_of(types, 2, [(SUM, pm.VAL_INT64, 0), (SUM, pm.val_decimal(10, 2), 1)], maps)
        # each reducer takes the (G, X) groups of its hash bucket; here by x modulo the reducers
        per_red = [[] for _ in range(n_red)]
        for s in partial:
            for o, n in rm.parse(s):
                row = s[o + 4:o + n]
                x = None if rm.is_null(row, 1) else long_at(row, 1) & 0xFFFFFFFF
                per_red[(x or 0) % n_red].append(row)
        outs = [da.reducer([rm.stream(rows)], 1, [(INT, 4), (INT, 4)], aggs, distinct)[0] for rows in per_red]
        got = {}
        for row in final_rows(outs, 1, aggs, distinct):
            g = int.from_bytes(row[8:12], "little", signed=True)
            avg_sum, avg_n = struct.unpack("<d", row[56:64])[0], long_at(row, 7)
            got[g] = (long_at(row, 1), dm.dec_value(row, 24, dm.sum_decimal(20)), long_at(row, 4), long_at(row, 5),
                      avg_sum / avg_n)
        for g in range(6):
            xs = sorted({x for gg, x, _, _ in data if gg == g and x is not None})
            assert got[g][:4] == (sum(v for gg, _, v, _ in data if gg == g), sum(d for gg, _, _, d in data if gg == g),
                                  len(xs), sum(xs))
            assert np.isclose(got[g][4], np.mean(xs), rtol=1e-12)
