"""Aggregate windows over a reducer's UnsafeRows on the GPU (b2s_decompress_window_aggregate_rows_keys_*): every output
byte is compared with tests/window_agg_model.py, with the input and output record counts and status[]."""
import struct

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from join_model import DECIMAL_WIDE, FIXED
from rows_model import CODECS, KEY_INT32, KEY_INT64, blocks_of, build_blocks, mirror, run, stream, write_maps
from test_gpu_sort_rows_order import DESC, NULLS_LAST
from window_agg_model import (AVG, COUNT, FRAME_PARTITION, FRAME_RANGE, FRAME_ROWS, MAX, MIN, SUM, VAL_FLOAT32,
                              VAL_FLOAT64, VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64, VAL_NONE, dec,
                              model_window_aggregate)
from window_model import CUME_DIST, DENSE_RANK, NTILE, PERCENT_RANK, RANK, ROW_NUMBER, model_window

pytestmark = pytest.mark.gpu

NAME = "decompress_window_aggregate_rows_keys"
FRAMES = [FRAME_PARTITION, FRAME_ROWS, FRAME_RANGE]
F64_EDGES = [0.0, -0.0, 1.5, -2.25, 1e300, -1e-300, float("inf"), float("-inf")]
NAN64 = [0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000123]
NAN32 = [0x7FC00000, 0x7F800001, 0xFFC00123]


# ---------------------------------------------------------------------------------------------------------------
# rows: n_fields 8-byte slots after the null words; the first 3 fields partition-key candidates, field 3 the order key,
# then value fields, each twice (with a null bit, and never null); DECIMAL_WIDE values' 16 bytes after the fixed region
# ---------------------------------------------------------------------------------------------------------------
VALUE_TYPES = [VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64, VAL_FLOAT32, VAL_FLOAT64, dec(8, 2), dec(17, 2), dec(24, 3),
               dec(28, 0), dec(38, 5)]


def wide(vt):
    return vt & 0xFF == 7 and (vt >> 8) & 0xFF > 18


class Table:
    def __init__(self, value_types=VALUE_TYPES, pad=0):
        """fields: 0..2 partition keys (long, int, long), 3 the order key (long), pad filler fields, then each value
        type nullable and non-null"""
        self.vts = value_types
        self.first = 4 + pad
        self.nf = self.first + 2 * len(value_types)
        self.bw = (self.nf + 63) // 64
        self.kinds = [FIXED] * self.nf
        for k, vt in enumerate(value_types):
            if wide(vt):
                self.kinds[self.first + 2 * k] = self.kinds[self.first + 2 * k + 1] = DECIMAL_WIDE

    def slot(self, f):
        return 8 * (self.bw + f)

    def keys(self, npk, order_flags=0):
        part = [(KEY_INT64, self.slot(0), 8, 0), (KEY_INT32, self.slot(1), 4, 1), (KEY_INT64, self.slot(2), 8, -1)]
        return part[:npk] + [(KEY_INT64 | order_flags, self.slot(3), 8, 3)]

    def value(self, k, nullable=True):
        """(val_type, val_off, val_null_field) of value type k"""
        f = self.first + 2 * k + (0 if nullable else 1)
        return self.vts[k], self.slot(f), f if nullable else -1

    def row(self, keys, vals):
        """keys: 4 ints or None; vals[k]: (nullable field value, non-null value), each an int (ints, decimals) or raw
        bytes (floats); None: null"""
        fixed = 8 * (self.bw + self.nf)
        r = bytearray(fixed)
        bits = 0
        var = bytearray()
        for f, v in enumerate(keys):
            if v is None:
                bits |= 1 << f
            else:
                r[self.slot(f):self.slot(f) + 8] = (v % 2**64).to_bytes(8, "little")
        for k, pair in enumerate(vals):
            for j, v in enumerate(pair):
                f = self.first + 2 * k + j
                s = self.slot(f)
                if v is None:
                    bits |= 1 << f
                elif wide(self.vts[k]):
                    n = (v if v >= 0 else ~v).bit_length() // 8 + 1
                    b = v.to_bytes(n, "big", signed=True)
                    r[s:s + 8] = (((fixed + len(var)) << 32) | n).to_bytes(8, "little")
                    var += b + bytes(16 - n)
                elif isinstance(v, bytes):
                    r[s:s + len(v)] = v
                else:
                    w = {VAL_INT8: 1, VAL_INT16: 2, VAL_INT32: 4}.get(self.vts[k], 8)
                    r[s:s + w] = (v % 2**(8 * w)).to_bytes(w, "little")
        r[:8 * self.bw] = bits.to_bytes(8 * self.bw, "little")
        return bytes(r + var)


def rand_value(rng, vt):
    k = vt & 0xFF
    if k in (VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64):
        bits = {VAL_INT8: 8, VAL_INT16: 16, VAL_INT32: 32, VAL_INT64: 64}[k]
        return int(rng.integers(-2**(bits - 1), 2**(bits - 1), dtype=np.int64)) if rng.random() < 0.3 else \
            int(rng.integers(-100, 100))
    if k == VAL_FLOAT64:
        u = rng.random()
        if u < 0.1:
            return NAN64[int(rng.integers(3))].to_bytes(8, "little")
        if u < 0.3:
            return struct.pack("<d", F64_EDGES[int(rng.integers(len(F64_EDGES)))])
        return struct.pack("<d", float(rng.normal()) * 10.0 ** int(rng.integers(-5, 20)))
    if k == VAL_FLOAT32:
        u = rng.random()
        if u < 0.1:
            return NAN32[int(rng.integers(3))].to_bytes(4, "little")
        if u < 0.3:
            return struct.pack("<f", [0.0, -0.0, 1.5, float("inf"), -3.0][int(rng.integers(5))])
        return struct.pack("<f", float(rng.normal()) * 1000)
    p = (vt >> 8) & 0xFF
    top = 10**p - 1
    u = rng.random()
    if u < 0.2:
        return top if rng.random() < 0.5 else -top
    return int(rng.integers(-10**min(p, 18) + 1, 10**min(p, 18))) * (10**(p - 18) if p > 18 else 1) + \
        int(rng.integers(0, 1000))  # never outside (-10^p, 10^p): the last 3 digits are below the step


def clamp(v, vt):
    p = (vt >> 8) & 0xFF
    return max(-(10**p - 1), min(10**p - 1, v)) if vt & 0xFF == 7 else v


def table(rng, t, n, domains=(3, 2, 2), order_domain=6, null_frac=0.15, key_nulls=True):
    rows = []
    for _ in range(n):
        keys = [int(rng.integers(d)) - d // 2 if not (key_nulls and rng.random() < 0.05) else None for d in domains]
        keys[2] = keys[2] if keys[2] is not None else 0  # field 2 has no null bit
        keys.append(int(rng.integers(order_domain)) if rng.random() > 0.05 else None)
        vals = [(None if rng.random() < null_frac else clamp(rand_value(rng, vt), vt), clamp(rand_value(rng, vt), vt))
                for vt in t.vts]
        rows.append(t.row(keys, vals))
    return rows


def takes(fn, vt):
    k = vt & 0xFF
    if k == VAL_NONE:
        return fn == COUNT
    if k == 7:
        p = (vt >> 8) & 0xFF
        return p <= {SUM: 28, AVG: 24}.get(fn, 38)
    return True


def all_aggregates(t, nullable=True):
    out = []
    for fn in (SUM, COUNT, MIN, MAX, AVG):
        for frame in FRAMES:
            if fn == COUNT:
                out.append((COUNT, frame, VAL_NONE, 0, -1))
            for k, vt in enumerate(t.vts):
                if takes(fn, vt):
                    v, off, nb = t.value(k, nullable)
                    out.append((fn, frame, v, off, nb))
    return out


def call(capi, plain, t, keys, npk, fns, codec=1, level=0, alg=0, dev=False, cap=None):
    blocks = build_blocks(capi, codec, level, alg, plain)
    want, n, m = model_window_aggregate(plain, keys, npk, t.nf, t.kinds, fns)
    got, r = run(capi, NAME, codec, alg, blocks, (keys, npk, t.nf, t.kinds, fns), len(want) if cap is None else cap,
                 dev)
    return got, r, (want, n, m)


def check(capi, plain, t, keys, npk, fns, **kw):
    got, r, (want, n, m) = call(capi, plain, t, keys, npk, fns, **kw)
    assert (r["status"] == 0).all(), r["status"]
    assert (r["n_records"], r["n_out_records"], r["total"]) == (n, m, len(want))
    if got != want:
        at = next(i for i in range(min(len(got), len(want))) if got[i] != want[i]) if got[:len(want)] != want else 0
        raise AssertionError("first differing byte %d of %d" % (at, len(want)))
    return r


# ---------------------------------------------------------------------------------------------------------------
# 1. every function x frame x value type, nullable and not, with 0, 1 and 3 partition columns
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("npk", [0, 1, 3])
def test_every_function_frame_and_type(capi, npk, nullable):
    rng = np.random.default_rng(100 + npk + 10 * nullable)
    t = Table()
    rows = table(rng, t, 1500, order_domain=5)
    plain = blocks_of(rows, [600, 0, 900])
    fns = all_aggregates(t, nullable)
    for at in range(0, len(fns), 16):
        check(capi, plain, t, t.keys(npk, DESC if npk == 1 else 0), npk, fns[at:at + 16])


@pytest.mark.parametrize("alg", [0, 3])
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_every_codec_and_checksum(capi, name, codec, level, alg):
    rng = np.random.default_rng(200 + codec * 4 + level + alg)
    t = Table()
    rows = table(rng, t, 2000)
    fns = [(SUM, FRAME_RANGE, *t.value(5)), (AVG, FRAME_PARTITION, *t.value(8)), (MIN, FRAME_ROWS, *t.value(10)),
           (MAX, FRAME_RANGE, *t.value(4)), (COUNT, FRAME_ROWS, *t.value(3)), (SUM, FRAME_ROWS, *t.value(7, False)),
           RANK, (AVG, FRAME_RANGE, *t.value(2))]
    check(capi, blocks_of(rows, [700, 0, 1300]), t, t.keys(1), 1, fns, codec=codec, level=level, alg=alg)


# ---------------------------------------------------------------------------------------------------------------
# 2. ranking and aggregates together, 16 functions, value null bits in a new word, no ORDER BY
# ---------------------------------------------------------------------------------------------------------------
def test_ranking_and_aggregates_in_one_call_and_16_functions(capi):
    rng = np.random.default_rng(300)
    t = Table()
    rows = table(rng, t, 2500)
    fns = [ROW_NUMBER, (SUM, FRAME_ROWS, *t.value(3)), RANK, (AVG, FRAME_RANGE, *t.value(5)), DENSE_RANK,
           (NTILE, 3), (MIN, FRAME_PARTITION, *t.value(9)), PERCENT_RANK, (MAX, FRAME_ROWS, *t.value(10)), CUME_DIST,
           (COUNT, FRAME_RANGE, VAL_NONE, 0, -1), (SUM, FRAME_PARTITION, *t.value(9)),
           (AVG, FRAME_ROWS, *t.value(8, False)), (SUM, FRAME_RANGE, *t.value(6)), (MIN, FRAME_RANGE, *t.value(4)),
           (MAX, FRAME_PARTITION, *t.value(0))]
    assert len(fns) == 16
    check(capi, blocks_of(rows, [1000, 1500]), t, t.keys(1, DESC | NULLS_LAST), 1, fns)


@pytest.mark.parametrize("nf", [58, 62, 64, 70])
def test_value_null_bits_cross_into_a_new_word(capi, nf):
    """8 values after n_fields 58, 62, 64 and 70: value null bits on both sides of bit 64, or all past it"""
    rng = np.random.default_rng(310 + nf)
    t = Table([VAL_INT64, VAL_FLOAT64, dec(17, 2), dec(24, 3), dec(38, 5), VAL_INT8, VAL_FLOAT32, dec(8, 2),
               VAL_INT32, VAL_INT16, dec(20, 1)], pad=nf - 26)
    assert t.nf == nf
    rows = table(rng, t, 800, null_frac=0.4)
    fns = [(SUM, FRAME_ROWS, *t.value(2)), (MIN, FRAME_ROWS, *t.value(4)), (AVG, FRAME_RANGE, *t.value(3)),
           (MAX, FRAME_PARTITION, *t.value(1)), (SUM, FRAME_RANGE, *t.value(0)), (COUNT, FRAME_ROWS, *t.value(3)),
           (SUM, FRAME_ROWS, *t.value(10)), (AVG, FRAME_ROWS, *t.value(7))]
    check(capi, blocks_of(rows, [300, 500]), t, t.keys(1), 1, fns)


def test_no_order_column_with_whole_partition_frames(capi):
    """q98: sum(itemrevenue) over (partition by i_class), and q47's avg over several partition columns"""
    rng = np.random.default_rng(320)
    t = Table()
    rows = table(rng, t, 3000)
    for npk in (1, 3):
        keys = t.keys(npk)[:npk]
        check(capi, blocks_of(rows, [3000]), t, keys, npk,
              [(SUM, FRAME_PARTITION, *t.value(7)), (AVG, FRAME_PARTITION, *t.value(7)),
               (COUNT, FRAME_PARTITION, VAL_NONE, 0, -1)])


# ---------------------------------------------------------------------------------------------------------------
# 3. decimals: compact -> compact, compact -> wide, wide -> wide; runs of +-(10^p - 1) for the 128-bit carries
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [1, 8, 9, 17, 18, 19, 24, 28])
def test_decimal_sums_and_averages_at_the_extremes(capi, p):
    rng = np.random.default_rng(400 + p)
    vts = [dec(p, min(p, 2)), dec(min(p, 24), 0)]
    t = Table(vts + [dec(38, 0)])
    top = [10**((vt >> 8) & 0xFF) - 1 for vt in t.vts]
    rows = []
    for i in range(3000):
        run_sign = 1 if (i // 400) % 3 != 1 else -1  # long runs of one sign, then the other
        vals = [(top[k] * run_sign if rng.random() < 0.8 else None, -top[k] * run_sign if rng.random() < 0.5 else
                 top[k] * run_sign) for k in range(len(t.vts))]
        rows.append(t.row([i % 3, 0, 0, i], vals))
    fns = []
    for fr in FRAMES:
        for k in range(2):
            for nullable in (True, False):
                fns += [(SUM, fr, *t.value(k, nullable))]
                if ((t.vts[k] >> 8) & 0xFF) <= 24:
                    fns += [(AVG, fr, *t.value(k, nullable))]
        fns += [(MIN, fr, *t.value(2)), (MAX, fr, *t.value(2, False))]
    for at in range(0, len(fns), 16):
        check(capi, blocks_of(rows, [1000, 2000]), t, t.keys(1), 1, fns[at:at + 16])


# ---------------------------------------------------------------------------------------------------------------
# 4. partition sizes: one reducer-wide partition (the serial double sum across many warp rounds), many tiny ones
# ---------------------------------------------------------------------------------------------------------------
def test_one_partition_of_200k_rows(capi):
    rng = np.random.default_rng(500)
    t = Table([VAL_FLOAT64, VAL_INT64, dec(17, 2)])
    n = 200_000
    order = rng.integers(0, 50_000, n)
    x = rng.normal(size=n) * 10.0 ** rng.integers(-3, 12, n)
    rows = [t.row([0, 0, 0, int(o)], [(struct.pack("<d", float(v)) if i % 7 else None, struct.pack("<d", float(v))),
                                      (int(o) * 1_000_003, int(o)), (int(o) * 101 - 77, int(o))])
            for i, (o, v) in enumerate(zip(order.tolist(), x.tolist()))]
    fns = [(SUM, FRAME_ROWS, *t.value(0)), (SUM, FRAME_RANGE, *t.value(0, False)), (AVG, FRAME_ROWS, *t.value(1)),
           (AVG, FRAME_PARTITION, *t.value(0)), (SUM, FRAME_ROWS, *t.value(2)), (MIN, FRAME_ROWS, *t.value(0)),
           (MAX, FRAME_RANGE, *t.value(1)), (COUNT, FRAME_ROWS, *t.value(0))]
    check(capi, blocks_of(rows, [80_000, 120_000]), t, t.keys(0), 0, fns)


def test_50k_partitions_of_1_to_4_rows(capi):
    rng = np.random.default_rng(501)
    t = Table([VAL_FLOAT64, dec(24, 3), VAL_INT32])
    rows = []
    for p in range(50_000):
        for k in range(int(rng.integers(1, 5))):
            rows.append(t.row([p, 0, 0, int(rng.integers(3))],
                              [(clamp(rand_value(rng, vt), vt) if rng.random() < 0.8 else None,
                                clamp(rand_value(rng, vt), vt))
                               for vt in t.vts]))
    order = rng.permutation(len(rows))
    rows = [rows[i] for i in order]
    fns = [(SUM, FRAME_ROWS, *t.value(0)), (AVG, FRAME_RANGE, *t.value(1)), (SUM, FRAME_PARTITION, *t.value(2)),
           (MIN, FRAME_ROWS, *t.value(0)), (AVG, FRAME_ROWS, *t.value(2, False)), ROW_NUMBER]
    check(capi, blocks_of(rows, [len(rows) // 2, len(rows) - len(rows) // 2]), t, t.keys(1), 1, fns)


# ---------------------------------------------------------------------------------------------------------------
# 5. the _dev form, the size retry, bad input, bad arguments, and the ranking-only call
# ---------------------------------------------------------------------------------------------------------------
def test_dev_matches_packed(capi):
    rng = np.random.default_rng(600)
    t = Table()
    plain = blocks_of(table(rng, t, 2000), [1000, 1000])
    fns = all_aggregates(t)[:16]
    a = check(capi, plain, t, t.keys(1), 1, fns, codec=3, level=1, alg=3)
    b = check(capi, plain, t, t.keys(1), 1, fns, codec=3, level=1, alg=3, dev=True)
    assert (a["n_records"], a["n_out_records"], a["total"]) == (b["n_records"], b["n_out_records"], b["total"])


def test_dst_too_small_reports_the_exact_size(capi):
    import ctypes as C
    rng = np.random.default_rng(601)
    t = Table()
    plain = blocks_of(table(rng, t, 500), [500])
    fns = [(SUM, FRAME_ROWS, *t.value(9)), (AVG, FRAME_RANGE, *t.value(8))]
    want, n, m = model_window_aggregate(plain, t.keys(1), 1, t.nf, t.kinds, fns)
    arena, off, ln, sb, sl, sc = build_blocks(capi, 1, 0, 0, plain)
    a = capi._window_aggregate_arrays(t.keys(1), 1, t.nf, t.kinds, fns)
    dst = np.zeros(len(want) - 1, np.uint8)
    counts = [C.c_uint64(0) for _ in range(3)]
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = capi.load().b2s_decompress_window_aggregate_rows_keys_packed(
        1, 0, 1, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None, *map(capi._arg, a),
        dst.ctypes.data, dst.size, *map(C.byref, counts), st.ctypes.data, bad.ctypes.data)
    assert rc == capi.E_DST_TOO_SMALL and counts[0].value == len(want)
    got, r = run(capi, NAME, 1, 0, (arena, off, ln, sb, sl, sc), (t.keys(1), 1, t.nf, t.kinds, fns), counts[0].value)
    assert got == want and (r["n_records"], r["n_out_records"]) == (n, m)


@pytest.mark.parametrize("size", [0, 17])
def test_corrupt_wide_decimal_input_fails_its_block(capi, size):
    rng = np.random.default_rng(602)
    t = Table([dec(24, 3)])
    rows = table(rng, t, 200, null_frac=0.0)
    bad = bytearray(rows[150])
    s = t.slot(t.first + 1)  # the never-null copy
    slot = int.from_bytes(bad[s:s + 8], "little")
    bad[s:s + 8] = (((slot >> 32) << 32) | size).to_bytes(8, "little")
    plain = [stream(rows[:100]), stream(rows[100:150] + [bytes(bad)] + rows[151:])]
    fns = [(COUNT, FRAME_ROWS, *t.value(0, False))]
    got, r = run(capi, NAME, 1, 3, build_blocks(capi, 1, 0, 3, plain), (t.keys(1), 1, t.nf, t.kinds, fns), 1 << 16)
    assert list(r["status"]) == [0, capi.E_CORRUPT]
    assert (r["n_records"], r["n_out_records"], r["total"]) == (0, 0, 0) and got == b""
    assert b"block 1" in capi.load().b2s_last_error()
    # past its row: a 16-byte value whose offset runs off the end
    bad[s:s + 8] = ((len(bad) - 8) << 32 | 16).to_bytes(8, "little")
    plain = [stream(rows[:100]), stream(rows[100:150] + [bytes(bad)] + rows[151:])]
    got, r = run(capi, NAME, 1, 3, build_blocks(capi, 1, 0, 3, plain), (t.keys(1), 1, t.nf, t.kinds, fns), 1 << 16)
    assert list(r["status"]) == [0, capi.E_CORRUPT] and got == b""


def test_bad_checksum_reports_bad_slice(capi):
    rng = np.random.default_rng(603)
    t = Table([VAL_INT64])
    rows = table(rng, t, 200)
    arena, off, ln, sb, sl, sc = build_blocks(capi, 2, 0, 3, [stream(rows[:100]), stream(rows[100:])])
    sc = sc.copy()
    sc[1] ^= 1
    got, r = run(capi, NAME, 2, 3, (arena, off, ln, sb, sl, sc),
                 (t.keys(1), 1, t.nf, t.kinds, [(SUM, FRAME_ROWS, *t.value(0))]), 1 << 16)
    assert list(r["status"]) == [0, capi.E_CHECKSUM]
    assert (r["n_records"], r["n_out_records"], r["total"]) == (0, 0, 0)


def test_order_column_rules(capi):
    rng = np.random.default_rng(604)
    t = Table([VAL_INT64])
    blocks = build_blocks(capi, 1, 0, 0, [stream(table(rng, t, 20))])
    keys = t.keys(1)[:1]
    for fns in ([(SUM, FRAME_ROWS, *t.value(0))], [(SUM, FRAME_PARTITION, *t.value(0)), RANK],
                [(SUM, FRAME_PARTITION, *t.value(0)), (COUNT, FRAME_RANGE, VAL_NONE, 0, -1)]):
        with pytest.raises(capi.B2SError) as e:
            run(capi, NAME, 1, 0, blocks, (keys, 1, t.nf, t.kinds, fns), 1 << 14)
        assert e.value.code == capi.E_ARG
    with pytest.raises(capi.B2SError) as e:  # more partition columns than key columns
        run(capi, NAME, 1, 0, blocks, (keys, 2, t.nf, t.kinds, [(SUM, FRAME_PARTITION, *t.value(0))]), 1 << 14)
    assert e.value.code == capi.E_ARG


@pytest.mark.parametrize("npk", [0, 1])
def test_ranking_only_is_byte_identical_to_the_ranking_call(capi, npk):
    rng = np.random.default_rng(605 + npk)
    t = Table([dec(24, 3), VAL_INT64])
    plain = blocks_of(table(rng, t, 3000), [1000, 2000])
    blocks = build_blocks(capi, 2, 0, 3, plain)
    fns = [ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK, CUME_DIST, (NTILE, 7)]
    keys = t.keys(npk, DESC)
    a, ra = run(capi, NAME, 2, 3, blocks, (keys, npk, t.nf, t.kinds, fns), 1 << 22)
    b, rb = run(capi, "decompress_window_rows_keys", 2, 3, blocks, (keys, npk, t.nf, t.kinds, fns, None), 1 << 22)
    assert a == b and (ra["n_records"], ra["n_out_records"], ra["total"]) == (rb["n_records"], rb["n_out_records"],
                                                                              rb["total"])
    assert a == model_window(plain, keys, npk, t.nf, t.kinds, fns)[0]


def test_empty_input(capi):
    t = Table([VAL_INT64])
    r = check(capi, [b"", b""], t, t.keys(1), 1, [(SUM, FRAME_ROWS, *t.value(0))])
    assert (r["n_records"], r["n_out_records"], r["total"]) == (0, 0, 0)


# ---------------------------------------------------------------------------------------------------------------
# 6. the host mirror
# ---------------------------------------------------------------------------------------------------------------
def test_host_mirror_reads_window_aggregate_rows(capi, tmp_path):
    host = pkg.host
    d = mirror(tmp_path, "lz4")
    M, R = 3, 2
    rng = np.random.default_rng(700)
    t = Table([VAL_FLOAT64, dec(17, 2), dec(24, 3)])
    maps = []
    for m in range(M):
        rows = table(rng, t, 300)
        maps.append((rows, rng.integers(0, R, len(rows))))
    write_maps(host, d, maps, R)
    fns = [(SUM, FRAME_RANGE, *t.value(0)), (AVG, FRAME_PARTITION, *t.value(1)), (MAX, FRAME_ROWS, *t.value(2)),
           RANK]
    for red in range(R):
        plain = [stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps]
        reader = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        got = reader.readWindowAggregateRows(t.keys(1), 1, t.nf, t.kinds, fns)
        reader.close()
        assert got == model_window_aggregate(plain, t.keys(1), 1, t.nf, t.kinds, fns)
