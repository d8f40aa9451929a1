"""The partial-aggregation model (tests/partial_agg_model.py) pinned without a GPU: hand-worked rows for every rule of
b2s_aggregate_partition_compress_rows_hash_*, the staged-merge equivalence the device relies on (each buffer is the
reduce side's merge op over staged inputs), and partial rows of several maps merged by the reduce-side model equal to
the whole dataset's."""
import struct

import numpy as np

import decimal_model as dm
import hash_model as hm
import partial_agg_model as pm
import rows_model as rm

NK = 1


def row(types, vals):
    return hm.make_row(types, vals)


def fields(prow, n):
    """a partial row's n slots and its null word"""
    return [prow[8 + 8 * f:16 + 8 * f] for f in range(n)], int.from_bytes(prow[:8], "little")


def f64bits(b):
    return int.from_bytes(b, "little")


def agg(fn, vt, field, nullable=True):
    return (fn, vt, 8 + 8 * field, field if nullable else -1)


def one_group(types, vals_list, aggs, keys=None):
    keys = keys or hm.keys_of(types, [0])
    out = pm.partial_rows([row(types, v) for v in vals_list], keys, aggs)
    assert len(out) == 1
    return out[0]


def test_double_sums_and_min_max_keep_signed_zeros_and_nan_bits():
    t = ["int", "double"]
    r = one_group(t, [[1, -0.0]], [agg(pm.SUM, pm.VAL_FLOAT64, 1), agg(pm.MIN, pm.VAL_FLOAT64, 1)])
    s, _ = fields(r, 3)
    assert f64bits(s[1]) == 0 and f64bits(s[2]) == 1 << 63  # a lone -0.0 sums to +0.0; MIN keeps it
    r = one_group(t, [[1, 0.0], [1, -0.0]], [agg(pm.MIN, pm.VAL_FLOAT64, 1), agg(pm.MAX, pm.VAL_FLOAT64, 1)])
    s, _ = fields(r, 3)
    assert f64bits(s[1]) == 0 and f64bits(s[2]) == 0  # equal: the first stays
    nan_a, nan_b = 0x7FF8000000000001, 0xFFF8000000000002
    r = one_group(t, [[1, 1.0], [1, ("bits", nan_a)], [1, ("bits", nan_b)], [1, float("inf")]],
                  [agg(pm.MAX, pm.VAL_FLOAT64, 1), agg(pm.MIN, pm.VAL_FLOAT64, 1)])
    s, _ = fields(r, 3)
    assert f64bits(s[1]) == nan_a and struct.unpack("<d", s[2])[0] == 1.0


def test_avg_with_nulls_and_count_star():
    t = ["int", "int"]
    r = one_group(t, [[1, None], [1, 2], [1, None], [1, 4]],
                  [agg(pm.AVG, pm.VAL_INT32, 1), (pm.COUNT, pm.VAL_NONE, 0, -1), agg(pm.COUNT, pm.VAL_INT32, 1)])
    s, nulls = fields(r, 5)
    assert struct.unpack("<d", s[1])[0] == 6.0 and int.from_bytes(s[2], "little") == 2
    assert int.from_bytes(s[3], "little") == 4 and int.from_bytes(s[4], "little") == 2 and nulls == 0
    r = one_group(t, [[1, None]], [agg(pm.AVG, pm.VAL_INT32, 1), agg(pm.SUM, pm.VAL_INT32, 1)])
    s, nulls = fields(r, 4)
    assert f64bits(s[1]) == 0 and int.from_bytes(s[2], "little") == 0 and nulls == 1 << 3  # AVG never null; SUM null


def test_is_empty_with_a_nullable_and_a_non_nullable_input():
    t = ["int", "long"]
    a = agg(pm.SUM, pm.val_decimal(8, 2), 1)
    r = one_group(t, [[1, None], [1, None]], [a])
    s, nulls = fields(r, 3)
    assert int.from_bytes(s[1], "little") == 0 and int.from_bytes(s[2], "little") == 1 and nulls == 0
    r = one_group(t, [[1, 5], [1, None]], [a])
    s, _ = fields(r, 3)
    assert int.from_bytes(s[1], "little") == 5 and int.from_bytes(s[2], "little") == 0
    r = one_group(t, [[1, 0]], [agg(pm.SUM, pm.val_decimal(8, 2), 1, nullable=False)])
    s, _ = fields(r, 3)
    assert int.from_bytes(s[2], "little") == 0


def test_decimal_28_sum_buffer_is_wide_and_exact_and_decimal_27_avg_counts():
    t = ["int", "decimal"]
    big = 10**28 - 1
    r = one_group(t, [[1, big]] * 4 + [[1, -1]], [agg(pm.SUM, pm.val_decimal(28, 0), 1),
                                                   agg(pm.AVG, pm.val_decimal(27, 0), 1)])
    s, nulls = fields(r, 5)
    so = int.from_bytes(s[1], "little")
    assert (so & 0xFFFFFFFF) == len(hm.decimal_bytes(4 * big - 1))
    assert int.from_bytes(r[so >> 32:(so >> 32) + (so & 0xFFFFFFFF)], "big", signed=True) == 4 * big - 1
    assert nulls == 0 and int.from_bytes(s[4], "little") == 5


def test_key_normalization_null_group_and_padding():
    t = ["double", "int"]
    rows = [row(t, [v, 1]) for v in (0.0, -0.0, ("bits", 0x7FF8000000000001), ("bits", 0xFFF0000000000005), None)]
    out = pm.partial_rows(rows, hm.keys_of(t, [0]), [(pm.COUNT, pm.VAL_NONE, 0, -1)])
    assert len(out) == 3
    assert int.from_bytes(out[0][:8], "little") == 1  # the null key sorts first
    assert f64bits(out[1][8:16]) == 0 and f64bits(out[2][8:16]) == 0x7FF8000000000000
    assert [int.from_bytes(o[16:24], "little") for o in out] == [1, 2, 2]
    t = ["string", "decimal", "int"]
    rows = [row(t, [b"abc", 5, 1]), row(t, [None, None, 2])]
    out = pm.partial_rows(rows, hm.keys_of(t, [0, 1]), [])
    null_row, r = out
    assert len(null_row) == 8 + 16 + 16 and null_row[:8] == bytes([3]) + bytes(7)
    assert int.from_bytes(null_row[8:16], "little") == 0 and int.from_bytes(null_row[16:24], "little") == 24 << 32
    assert len(r) == 8 + 16 + 8 + 16 and r[24:32] == b"abc" + bytes(5) and r[32:48] == b"\x05" + bytes(15)
    assert int.from_bytes(r[8:16], "little") == (24 << 32 | 3) and int.from_bytes(r[16:24], "little") == (32 << 32 | 1)


# ---- the staged-merge equivalence ----
TYPES = ["string", "int", "byte", "short", "int", "long", "float", "double", "long", "decimal"]
VT = [None, None, pm.VAL_INT8, pm.VAL_INT16, pm.VAL_INT32, pm.VAL_INT64, pm.VAL_FLOAT32, pm.VAL_FLOAT64,
      pm.val_decimal(7, 2), pm.val_decimal(25, 3)]
KEYS = hm.keys_of(TYPES, [0, 1])


def rand_rows(rng, n, nkeys):
    pool = [(bytes(rng.integers(97, 100, int(rng.integers(0, 12)), dtype=np.uint8)) if rng.random() > 0.1 else None,
             int(rng.integers(0, 3)) if rng.random() > 0.1 else None) for _ in range(nkeys)]
    rows = []
    for _ in range(n):
        k = pool[int(rng.integers(nkeys))]
        vals = list(k)
        for t in TYPES[2:]:
            if rng.random() < 0.25:
                vals.append(None)
            elif t in ("float", "double"):
                vals.append([0.0, -0.0, float(np.float32(rng.normal() * 100))][int(rng.integers(3))])
            elif t == "decimal":
                vals.append(int(rng.integers(-10**18, 10**18)) * 10**6)
            else:
                bits = {"byte": 8, "short": 16, "int": 32, "long": 64}[t]
                vals.append(int(rng.integers(-(1 << (bits - 1)), (1 << (bits - 1)) - 1, dtype=np.int64)))
        vals[8] = None if vals[8] is None else vals[8] % 10**7
        rows.append(row(TYPES, vals))
    return rows


def all_pairs():
    f = lambda fn, j: (fn, VT[j], 8 + 8 * j, j)  # noqa: E731
    return [f(pm.SUM, 2), f(pm.SUM, 5), f(pm.SUM, 6), f(pm.SUM, 8), f(pm.SUM, 9), (pm.COUNT, pm.VAL_NONE, 0, -1),
            f(pm.COUNT, 7), f(pm.AVG, 3), f(pm.AVG, 8), f(pm.MIN, 4), f(pm.MAX, 7), f(pm.MIN, 8), f(pm.MAX, 9)]


def staged(r, aggs):
    """the device's staged inputs of one row, in buffer order (None: a null, skipped by the merge)"""
    out = []
    for fn, vt, off, nf in aggs:
        v = pm.read_value(r, vt, off, nf)
        dec = vt & 0xFF == pm.VAL_DECIMAL
        if fn == pm.SUM:
            out += [0 if v is None else v, int(v is None)] if dec else [v]
        elif fn == pm.COUNT:
            out.append(int(v is not None))
        elif fn == pm.AVG:
            out += [(0 if v is None else v) if dec else (0.0 if v is None else float(v)), int(v is not None)]
        else:
            out.append(v)
    return out


def merged(partials, keys, aggs):
    """the reduce side's aggregation model over partial rows -> its rows (no size prefix)"""
    buf, _, _ = dm.model_aggregate_decimal([rm.stream(partials)], pm.output_keys(keys), pm.merge_aggs(keys, aggs))
    return [r[4:] for r in _records(buf)]


def _records(buf):
    out, at = [], 0
    while at < len(buf):
        sz = int.from_bytes(buf[at:at + 4], "big")
        out.append(buf[at:at + 4 + sz])
        at += 4 + sz
    return out


def test_staged_inputs_merged_by_the_reduce_ops_are_the_update_expressions():
    rng = np.random.default_rng(1)
    rows = rand_rows(rng, 600, 25)
    aggs = all_pairs()
    bufs = pm.buffers(aggs)
    staged_rows = [pm.emit(r, KEYS, bufs, staged(r, aggs)) for r in rows]
    assert sorted(merged(staged_rows, KEYS, aggs)) == sorted(pm.partial_rows(rows, KEYS, aggs))


def test_maps_merged_by_the_reducer_equal_the_whole_dataset():
    rng = np.random.default_rng(2)
    rows = rand_rows(rng, 900, 30)
    exact = [a for a in all_pairs() if not (a[0] in (pm.SUM, pm.AVG) and a[1] in (pm.VAL_FLOAT32, pm.VAL_INT16))]
    maps = [rows[m::3] for m in range(3)]
    partials = [p for m in maps for p in pm.partial_rows(m, KEYS, exact)]
    assert sorted(merged(partials, KEYS, exact)) == sorted(pm.partial_rows(rows, KEYS, exact))
    # a double sum: each map's partial sum added in map order
    dsum = [(pm.SUM, pm.VAL_FLOAT64, 8 + 8 * 7, 7)]
    def key(p):  # everything but the sum's slot and null bit
        return (int.from_bytes(p[:8], "little") & ~4, bytes(p[8:24]), bytes(p[32:]))

    per_map = [{key(p): p for p in pm.partial_rows(m, KEYS, dsum)} for m in maps]
    got = merged([p for m in maps for p in pm.partial_rows(m, KEYS, dsum)], KEYS, dsum)
    assert len(got) == len({key(g) for g in got})
    for g in got:
        s, any_ = 0.0, False
        for pmap in per_map:
            p = pmap.get(key(g))
            if p is not None and not (int.from_bytes(p[:8], "little") >> 2) & 1:
                s += struct.unpack("<d", p[24:32])[0]
                any_ = True
        assert any_ == (not (int.from_bytes(g[:8], "little") >> 2) & 1)
        if any_:
            assert g[24:32] == struct.pack("<d", s)
