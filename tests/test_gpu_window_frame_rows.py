"""Sliding-frame windows over a reducer's UnsafeRows on the GPU (b2s_decompress_window_frame_rows_keys_*): every output
byte is compared with tests/window_frame_model.py, with the input and output record counts and status[]."""
import struct

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from rows_model import CODECS, KEY_INT32, KEY_INT64, blocks_of, build_blocks, mirror, parse, run, stream, write_maps
from test_gpu_sort_rows_order import DESC, KEY_INT8, KEY_INT16, NULLS_LAST
from test_gpu_window_offset_rows import OTable, rand_any, table
from window_agg_model import (AVG, COUNT, FRAME_PARTITION, FRAME_RANGE, FRAME_ROWS, MAX, MIN, SUM, VAL_FLOAT32,
                              VAL_FLOAT64, VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64, VAL_NONE, dec)
from window_frame_model import UNBOUNDED_FOLLOWING as UF, UNBOUNDED_PRECEDING as UP, model_window_frame
from window_model import DENSE_RANK, NTILE, RANK, ROW_NUMBER
from window_offset_model import FIRST, IGNORE_NULLS, LAG, LAST, LEAD, NTH_VALUE, VAL_BYTES

pytestmark = pytest.mark.gpu

NAME = "decompress_window_frame_rows_keys"
ROWS, RANGE = 4, 5
ROWS_FRAMES = [(-3, 0), (-1, 1), (0, 2), (2, 5), (-5, -2), (UP, 2), (UP, -1), (-2, UF), (1, UF), (0, UF)]
AGG_TYPES = [VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64, VAL_FLOAT32, VAL_FLOAT64, dec(8, 2), dec(17, 2), dec(24, 3),
             dec(28, 0), dec(38, 5)]


def agg(t, fn, k, frame, lo, hi, nullable=True):
    return (fn, 0, frame, *t.value(k, nullable), 0, 0, lo, hi)


def off(t, fn, k, arg, frame, lo, hi, nullable=True, flags=0):
    return (fn, arg, frame, *t.value(k, nullable), flags, 0, lo, hi)


def check(capi, plain, t, keys, npk, fns, codec=1, level=0, alg=0, dev=False):
    blocks = build_blocks(capi, codec, level, alg, plain)
    want, n, m, unsupported = model_window_frame(plain, keys, npk, t.nf, t.kinds, fns)
    assert not unsupported
    got, r = run(capi, NAME, codec, alg, blocks, (keys, npk, t.nf, t.kinds, fns), len(want), dev)
    assert (r["status"] == 0).all(), r["status"]
    assert (r["n_records"], r["n_out_records"], r["total"]) == (n, m, len(want))
    if got != want:
        at = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        row = next(k for k, (o, ln) in enumerate(parse(want)) if o + ln > at)
        o = parse(want)[row][0]
        raise AssertionError("first differing byte %d of %d (output row %d, byte %d): want %s got %s" % (
            at, len(want), row, at - o, want[o:o + 400].hex(), got[o:o + 400].hex()))
    return r


def run_all(capi, plain, t, keys, npk, fns, **kw):
    for at in range(0, len(fns), 16):
        check(capi, plain, t, keys, npk, fns[at:at + 16], **kw)


# ---------------------------------------------------------------------------------------------------------------
# 1. every aggregate x value type x ROWS frame, nullable and not, 0 / 1 / 3 partition columns
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("npk", [0, 1, 3])
def test_every_aggregate_type_and_rows_frame(capi, npk, nullable):
    rng = np.random.default_rng(3000 + npk + 10 * nullable)
    t = OTable(AGG_TYPES)
    plain = blocks_of(table(rng, t, 400, order_domain=40), [150, 0, 250])
    fns = []
    for k, vt in enumerate(AGG_TYPES):
        for fn in (SUM, COUNT, MIN, MAX, AVG):
            if vt & 0xFF == 7 and ((fn == SUM and (vt >> 8) & 0xFF > 28) or (fn == AVG and (vt >> 8) & 0xFF > 24)):
                continue
            for lo, hi in ROWS_FRAMES:
                fns.append(agg(t, fn, k, ROWS, lo, hi, nullable))
    fns.append((COUNT, 0, ROWS, VAL_NONE, 0, -1, 0, 0, -2, 3))
    run_all(capi, plain, t, t.keys(npk, DESC if npk == 1 else 0), npk, fns)


# ---------------------------------------------------------------------------------------------------------------
# 2. RANGE frames over byte / short / int / long order columns, every direction and null order, ties and null keys
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, DESC, NULLS_LAST, DESC | NULLS_LAST])
@pytest.mark.parametrize("ktype,width", [(KEY_INT8, 1), (KEY_INT16, 2), (KEY_INT32, 4), (KEY_INT64, 8)])
def test_range_frames_over_every_integral_order_column(capi, ktype, width, flags):
    rng = np.random.default_rng(3100 + ktype * 8 + flags // 256)
    t = OTable([VAL_INT64, VAL_FLOAT64, dec(24, 3), VAL_BYTES])
    rows = table(rng, t, 600, order_domain=60)  # order values 0..59, and every bound, fit a byte
    keys = t.keys(1)
    keys[-1] = (ktype | flags, t.slot(3), width, 3)
    fns = []
    for lo, hi in [(-3, 0), (-5, 5), (0, 4), (2, 9), (-7, -1), (UP, 3), (-2, UF), (0, 0), (0, UF), (UP, 0)]:
        fns += [agg(t, SUM, 0, RANGE, lo, hi), agg(t, SUM, 1, RANGE, lo, hi), agg(t, MIN, 2, RANGE, lo, hi),
                agg(t, MAX, 1, RANGE, lo, hi), agg(t, AVG, 2, RANGE, lo, hi), agg(t, COUNT, 1, RANGE, lo, hi),
                off(t, LAST, 3, 0, RANGE, lo, hi, True, IGNORE_NULLS), off(t, NTH_VALUE, 0, 2, RANGE, lo, hi)]
    run_all(capi, blocks_of(rows, [250, 350]), t, keys, 1, fns)


def test_range_current_row_with_a_multi_column_order_key(capi):
    rng = np.random.default_rng(3150)
    t = OTable([VAL_INT64, VAL_FLOAT64, VAL_BYTES])
    rows = table(rng, t, 1200, order_domain=4)
    keys = t.keys(1)[:1] + [(KEY_INT64 | DESC, t.slot(2), 8, -1), (KEY_INT64 | NULLS_LAST, t.slot(3), 8, 3)]
    fns = []
    for lo, hi in [(0, 0), (UP, 0), (0, UF)]:
        fns += [agg(t, SUM, 0, RANGE, lo, hi), agg(t, MIN, 1, RANGE, lo, hi), agg(t, AVG, 1, RANGE, lo, hi),
                off(t, FIRST, 2, 0, RANGE, lo, hi, True, IGNORE_NULLS), off(t, LAST, 0, 0, RANGE, lo, hi)]
    run_all(capi, blocks_of(rows, [1200]), t, keys, 1, fns)


# ---------------------------------------------------------------------------------------------------------------
# 3. FIRST / LAST / NTH_VALUE on strings and wide decimals, mixed with ranking, LAG / LEAD and the older frames
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, IGNORE_NULLS])
def test_offset_functions_over_sliding_frames(capi, flags):
    rng = np.random.default_rng(3200 + flags)
    t = OTable([VAL_BYTES, dec(38, 5), VAL_INT32])
    rows = table(rng, t, 1500, order_domain=30, null_frac=0.4)
    fns = []
    for k in range(3):
        for fr, lo, hi in [(ROWS, -3, 0), (ROWS, 2, 5), (ROWS, -5, -2), (ROWS, 1, UF), (ROWS, UP, -1), (RANGE, -4, 2),
                           (RANGE, 0, UF)]:
            fns += [off(t, FIRST, k, 0, fr, lo, hi, True, flags), off(t, LAST, k, 0, fr, lo, hi, True, flags),
                    off(t, NTH_VALUE, k, 2, fr, lo, hi, True, flags)]
    run_all(capi, blocks_of(rows, [700, 800]), t, t.keys(1), 1, fns)


def test_every_family_in_one_call(capi):
    rng = np.random.default_rng(3250)
    t = OTable([VAL_INT64, VAL_FLOAT64, dec(24, 3), dec(38, 5), VAL_BYTES])
    rows = table(rng, t, 2000, order_domain=50)
    fns = [ROW_NUMBER, (LAG, 1, 0, *t.value(4), 0, 0), agg(t, SUM, 2, ROWS, -6, 0), (SUM, FRAME_ROWS, *t.value(0)),
           RANK, off(t, LAST, 4, 0, RANGE, -3, 3, True, IGNORE_NULLS), (NTILE, 3), agg(t, AVG, 1, RANGE, -29, 0),
           (LEAD, 2, 0, *t.value(3), 0, 0), agg(t, MAX, 3, ROWS, -50, 50), (AVG, FRAME_RANGE, *t.value(2)),
           off(t, NTH_VALUE, 3, 2, ROWS, 0, UF), (MIN, FRAME_PARTITION, *t.value(1)), DENSE_RANK,
           agg(t, COUNT, 0, ROWS, 1, UF), (FIRST, 0, FRAME_RANGE, *t.value(4), 0, 0)]
    assert len(fns) == 16
    check(capi, blocks_of(rows, [900, 1100]), t, t.keys(1, DESC | NULLS_LAST), 1, fns)


# ---------------------------------------------------------------------------------------------------------------
# 4. the old frames through the new bounds: byte-identical to the offset call
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("npk", [0, 1])
def test_unbounded_bounds_equal_the_older_frames(capi, npk):
    rng = np.random.default_rng(3300 + npk)
    t = OTable([VAL_INT64, VAL_FLOAT64, dec(24, 3), dec(38, 5), VAL_BYTES, VAL_FLOAT32])
    plain = blocks_of(table(rng, t, 2500, order_domain=20), [1000, 1500])
    blocks = build_blocks(capi, 2, 0, 3, plain)
    keys = t.keys(npk, DESC)
    for (fr, lo, hi), old in [((ROWS, UP, 0), FRAME_ROWS), ((RANGE, UP, 0), FRAME_RANGE),
                              ((ROWS, UP, UF), FRAME_PARTITION)]:
        new_fns, old_fns = [], []
        for fn, k in [(SUM, 0), (SUM, 1), (MIN, 2), (MAX, 3), (AVG, 1), (AVG, 2), (COUNT, 0), (SUM, 5), (MIN, 5),
                      (FIRST, 4), (LAST, 3), (NTH_VALUE, 1)]:
            arg, fl = (2, IGNORE_NULLS) if fn == NTH_VALUE else (0, IGNORE_NULLS if fn == LAST else 0)
            new_fns.append((fn, arg, fr, *t.value(k), fl, 0, lo, hi))
            old_fns.append((fn, arg, old, *t.value(k), fl, 0))
        a, ra = run(capi, NAME, 2, 3, blocks, (keys, npk, t.nf, t.kinds, new_fns), 1 << 23)
        b, rb = run(capi, "decompress_window_offset_rows_keys", 2, 3, blocks, (keys, npk, t.nf, t.kinds, old_fns),
                    1 << 23)
        assert a == b and (ra["n_out_records"], ra["total"]) == (rb["n_out_records"], rb["total"])
        assert a == model_window_frame(plain, keys, npk, t.nf, t.kinds, new_fns)[0]


# ---------------------------------------------------------------------------------------------------------------
# 5. edge cases: one-row partitions, frames wider than every partition, NaN / inf, wrapping sums
# ---------------------------------------------------------------------------------------------------------------
def test_one_row_partitions_and_frames_wider_than_any_partition(capi):
    rng = np.random.default_rng(3400)
    t = OTable([VAL_INT64, VAL_FLOAT64, VAL_BYTES])
    rows = [t.row([p, 0, 0, int(rng.integers(5))], [(rand_any(rng, vt) if rng.random() < 0.8 else None,
                                                     rand_any(rng, vt)) for vt in t.vts])
            for p in range(3000) for _ in range(1 + (p % 3 == 0) * int(rng.integers(0, 4)))]
    fns = [agg(t, SUM, 0, ROWS, -1000, 1000), agg(t, AVG, 1, ROWS, -1000, -1), agg(t, MIN, 1, ROWS, 1, 1000),
           agg(t, COUNT, 2 - 2, ROWS, -1, 1), off(t, LAST, 2, 0, ROWS, -1000, 1000, True, IGNORE_NULLS),
           agg(t, MAX, 0, RANGE, -100, 100), agg(t, SUM, 1, RANGE, 1, 1000), off(t, FIRST, 2, 0, RANGE, -1, UF)]
    check(capi, blocks_of(rows, [len(rows)]), t, t.keys(1), 1, fns)


def test_nan_infinities_and_wrapping_long_sums(capi):
    rng = np.random.default_rng(3450)
    t = OTable([VAL_FLOAT64, VAL_FLOAT32, VAL_INT64])
    edges = [float("nan"), float("inf"), float("-inf"), 0.0, -0.0, 1e308, -1e308, 1.5]
    edges32 = [float("nan"), float("inf"), float("-inf"), 0.0, -0.0, 3e38, -3e38, 1.5]
    rows = []
    for i in range(800):
        d = edges[int(rng.integers(len(edges)))]
        f = edges32[int(rng.integers(len(edges32)))]
        big = int(rng.choice([2**63 - 1, -2**63, 2**62, -5]))
        rows.append(t.row([i % 3, 0, 0, int(rng.integers(30))],
                          [(struct.pack("<d", d) if rng.random() < 0.9 else None, struct.pack("<d", d)),
                           (struct.pack("<f", f) if rng.random() < 0.9 else None, struct.pack("<f", f)),
                           (big if rng.random() < 0.9 else None, big)]))
    fns = []
    for lo, hi in [(-3, 0), (-2, 2), (1, UF), (0, UF)]:
        fns += [agg(t, SUM, 0, ROWS, lo, hi), agg(t, MIN, 0, ROWS, lo, hi), agg(t, MAX, 1, ROWS, lo, hi),
                agg(t, SUM, 2, ROWS, lo, hi)]
    fns += [agg(t, AVG, 2, RANGE, -5, 5), agg(t, MAX, 0, RANGE, -2, 0), agg(t, MIN, 1, RANGE, 0, 3)]
    run_all(capi, blocks_of(rows, [300, 500]), t, t.keys(1), 1, fns)


# ---------------------------------------------------------------------------------------------------------------
# 6. B2S_E_UNSUPPORTED with nothing written
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["int32 bound wraps", "int8 bound wraps", "2147483647 FOLLOWING"])
def test_wrapping_bounds_are_unsupported_and_write_nothing(capi, case):
    t = OTable([VAL_INT64])
    keys = t.keys(1)
    if case == "int32 bound wraps":
        vals = [5, 2**31 - 3, 7]
        keys[-1] = (KEY_INT32, t.slot(3), 4, 3)
        fns = [agg(t, SUM, 0, RANGE, 0, 5)]  # 5 FOLLOWING: v + 5
    elif case == "int8 bound wraps":
        vals = [1, 3, 127]
        keys[-1] = (KEY_INT8 | DESC, t.slot(3), 1, 3)
        fns = [agg(t, SUM, 0, RANGE, -1, 0)]  # descending, 1 PRECEDING: v + 1, which wraps at 127
    else:
        vals = [1, 2, 3]
        fns = [agg(t, SUM, 0, ROWS, 0, 2**31 - 1)]
    rows = [t.row([0, 0, 0, v], [(i, i)]) for i, v in enumerate(vals)]
    plain = [stream(rows)]
    assert model_window_frame(plain, keys, 1, t.nf, t.kinds, fns)[3]
    blocks = build_blocks(capi, 1, 0, 0, plain)
    dst = np.zeros(1 << 12, np.uint8)
    with pytest.raises(capi.B2SError) as e:
        getattr(capi, NAME + "_packed")(1, blocks[0], blocks[1], blocks[2], dst, keys, 1, t.nf, t.kinds, fns)
    assert e.value.code == capi.E_UNSUPPORTED
    assert not dst.any()
    # one row fewer is still inside Spark's arithmetic for the ROWS case
    if case == "2147483647 FOLLOWING":
        check(capi, [stream(rows[:1])], t, keys, 1, fns)


# ---------------------------------------------------------------------------------------------------------------
# 7. every codec, the _dev form, multi-block reducers, the host mirror
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_every_codec(capi, name, codec, level):
    rng = np.random.default_rng(3600 + codec * 4 + level)
    t = OTable([VAL_INT64, VAL_BYTES, dec(38, 5), VAL_FLOAT64])
    rows = table(rng, t, 1500, order_domain=25)
    fns = [agg(t, SUM, 3, ROWS, -6, 0), agg(t, MIN, 0, ROWS, -2, 2), off(t, LAST, 1, 0, RANGE, -2, 0, True,
                                                                        IGNORE_NULLS),
           agg(t, AVG, 3, RANGE, -3, 3), agg(t, MAX, 2, RANGE, -3, 3), off(t, NTH_VALUE, 2, 2, ROWS, 1, UF), RANK]
    check(capi, blocks_of(rows, [600, 0, 300, 600]), t, t.keys(1), 1, fns, codec=codec, level=level,
          alg=3 if codec else 0)


def test_dev_matches_packed(capi):
    rng = np.random.default_rng(3700)
    t = OTable([VAL_INT64, VAL_BYTES, dec(38, 5), VAL_FLOAT64])
    plain = blocks_of(table(rng, t, 1500, order_domain=25), [700, 800])
    fns = [agg(t, SUM, 3, ROWS, -6, 0), agg(t, MAX, 2, ROWS, -50, 50), off(t, FIRST, 1, 0, RANGE, -4, 0),
           agg(t, COUNT, 0, RANGE, 0, UF), agg(t, SUM, 3, ROWS, 0, UF)]
    a = check(capi, plain, t, t.keys(1), 1, fns, codec=3, level=1, alg=3)
    b = check(capi, plain, t, t.keys(1), 1, fns, codec=3, level=1, alg=3, dev=True)
    assert (a["n_records"], a["n_out_records"], a["total"]) == (b["n_records"], b["n_out_records"], b["total"])


def test_host_mirror_reads_window_frame_rows(capi, tmp_path):
    host = pkg.host
    d = mirror(tmp_path, "lz4")
    M, R = 3, 2
    rng = np.random.default_rng(3800)
    t = OTable([VAL_INT64, VAL_BYTES, dec(38, 5)])
    maps = []
    for m in range(M):
        rows = table(rng, t, 300, order_domain=20)
        maps.append((rows, rng.integers(0, R, len(rows))))
    write_maps(host, d, maps, R)
    fns = [agg(t, SUM, 0, ROWS, -2, 1), off(t, LAST, 1, 0, RANGE, -3, 0, True, IGNORE_NULLS),
           agg(t, MAX, 2, ROWS, 1, UF), RANK, (SUM, FRAME_RANGE, *t.value(0))]
    for red in range(R):
        plain = [stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps]
        reader = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        got = reader.readWindowFrameRows(t.keys(1), 1, t.nf, t.kinds, fns)
        reader.close()
        want = model_window_frame(plain, t.keys(1), 1, t.nf, t.kinds, fns)
        assert got == want[:3]


# ---------------------------------------------------------------------------------------------------------------
# 8. scale: one partition of about 1 M rows, a 64-wide double moving sum and a RANGE search, against numpy
# ---------------------------------------------------------------------------------------------------------------
def test_one_partition_of_a_million_rows(capi):
    rng = np.random.default_rng(3900)
    n = 1 << 20
    t = OTable([VAL_FLOAT64])
    x = rng.normal(size=n) * 10.0 ** rng.integers(-3, 6, n)
    order = np.sort(rng.integers(0, n // 4, n))  # ties; the rows arrive sorted, so the sort keeps this order
    fixed = 8 * (t.bw + t.nf)
    recs = np.zeros((n, fixed), np.uint8)
    recs[:, t.slot(3):t.slot(3) + 8] = order.astype("<i8").view(np.uint8).reshape(n, 8)
    for f in (t.first, t.first + 1):
        recs[:, t.slot(f):t.slot(f) + 8] = x.astype("<f8").view(np.uint8).reshape(n, 8)
    framed = np.zeros((n, 4 + fixed), np.uint8)
    framed[:, :4] = np.frombuffer(fixed.to_bytes(4, "big"), np.uint8)
    framed[:, 4:] = recs
    plain = [framed.tobytes()]
    fns = [agg(t, SUM, 0, ROWS, -63, 0, False), agg(t, COUNT, 0, RANGE, -100, 100, False)]
    out, r = run(capi, NAME, 0, 0, build_blocks(capi, 0, 0, 0, plain), (t.keys(0), 0, t.nf, t.kinds, fns),
                 n * (4 + fixed + 16) + 64)
    assert (r["n_records"], r["n_out_records"]) == (n, n)
    # numpy path of the model: the same add order ((0.0 + x_s) + ...) over [max(0, i - 63), i]
    want_sum = np.zeros(n)
    for d in range(63, -1, -1):
        sh = np.concatenate([np.zeros(d), x[:n - d]]) if d else x
        valid = np.arange(n) >= d
        want_sum = np.where(valid, want_sum + sh, want_sum)
    lo = np.searchsorted(order, order - 100, "left")
    hi = np.searchsorted(order, order + 100, "right")
    rows_out = np.frombuffer(out, np.uint8).reshape(n, -1)
    ow = (t.nf + 2 + 63) // 64
    base = 4 + 8 * (ow + t.nf)
    got_sum = rows_out[:, base:base + 8].copy().view("<f8").ravel()
    got_cnt = rows_out[:, base + 8:base + 16].copy().view("<i8").ravel()
    assert np.array_equal(got_sum.view(np.uint64), want_sum.view(np.uint64))
    assert np.array_equal(got_cnt, hi - lo)
