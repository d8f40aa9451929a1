"""Offset windows over a reducer's UnsafeRows on the GPU (b2s_decompress_window_offset_rows_keys_*): every output byte
is compared with tests/window_offset_model.py, with the input and output record counts and status[]."""
import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from join_model import VAR
from rows_model import CODECS, blocks_of, build_blocks, mirror, run, stream, write_maps
from test_gpu_sort_rows_order import DESC, NULLS_LAST
from test_gpu_window_agg_rows import Table, clamp, rand_value
from window_agg_model import (AVG, COUNT, FRAME_PARTITION, FRAME_RANGE, FRAME_ROWS, MAX, MIN, SUM, VAL_FLOAT32,
                              VAL_FLOAT64, VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64, VAL_NONE, dec)
from window_model import CUME_DIST, DENSE_RANK, NTILE, PERCENT_RANK, RANK, ROW_NUMBER
from window_offset_model import (FIRST, HAS_DEFAULT, IGNORE_NULLS, LAG, LAST, LEAD, NTH_VALUE, VAL_BYTES,
                                 model_window_offset)

pytestmark = pytest.mark.gpu

NAME = "decompress_window_offset_rows_keys"
AGG_NAME = "decompress_window_aggregate_rows_keys"
FRAMES = [FRAME_PARTITION, FRAME_ROWS, FRAME_RANGE]
FIXED_TYPES = [VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64, VAL_FLOAT32, VAL_FLOAT64, dec(8, 2), dec(17, 2), dec(18, 0)]
VALUE_TYPES = FIXED_TYPES + [dec(19, 1), dec(28, 3), dec(38, 5), VAL_BYTES]
WIDTH = {VAL_INT8: 1, VAL_INT16: 2, VAL_INT32: 4, VAL_FLOAT32: 4}


def wide(vt):
    return vt & 0xFF == 7 and (vt >> 8) & 0xFF > 18


class OTable(Table):
    """Table with string / binary (VAL_BYTES, VAR) value fields: their bytes after the fixed region, padded to 8"""

    def __init__(self, value_types=VALUE_TYPES, pad=0):
        super().__init__(value_types, pad)
        for k, vt in enumerate(value_types):
            if vt == VAL_BYTES:
                self.kinds[self.first + 2 * k] = self.kinds[self.first + 2 * k + 1] = VAR

    def row(self, keys, vals):
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
            vt = self.vts[k]
            for j, v in enumerate(pair):
                f = self.first + 2 * k + j
                s = self.slot(f)
                if v is None:
                    bits |= 1 << f
                elif vt == VAL_BYTES:
                    r[s:s + 8] = (((fixed + len(var)) << 32) | len(v)).to_bytes(8, "little")
                    var += v + bytes(-len(v) % 8)
                elif wide(vt):
                    n = (v if v >= 0 else ~v).bit_length() // 8 + 1
                    r[s:s + 8] = (((fixed + len(var)) << 32) | n).to_bytes(8, "little")
                    var += v.to_bytes(n, "big", signed=True) + bytes(16 - n)
                elif isinstance(v, bytes):
                    r[s:s + len(v)] = v
                else:
                    w = WIDTH.get(vt, 8)
                    r[s:s + w] = (v % 2**(8 * w)).to_bytes(w, "little")
        r[:8 * self.bw] = bits.to_bytes(8 * self.bw, "little")
        return bytes(r + var)


def rand_any(rng, vt):
    if vt == VAL_BYTES:
        n = [0, 7, 8, 9, int(rng.integers(0, 41))][int(rng.integers(5))]
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    return clamp(rand_value(rng, vt), vt)


def table(rng, t, n, domains=(3, 2, 2), order_domain=6, null_frac=0.3):
    rows = []
    for _ in range(n):
        keys = [int(rng.integers(d)) - d // 2 if rng.random() > 0.05 else None for d in domains]
        keys[2] = keys[2] if keys[2] is not None else 0  # field 2 has no null bit
        keys.append(int(rng.integers(order_domain)) if rng.random() > 0.05 else None)
        rows.append(t.row(keys, [(None if rng.random() < null_frac else rand_any(rng, vt), rand_any(rng, vt))
                                 for vt in t.vts]))
    return rows


def off_fn(t, fn, k, arg=0, frame=0, nullable=True, flags=0, default=0):
    return (fn, arg, frame, *t.value(k, nullable), flags, default)


def all_offsets(t, nullable, flags):
    out = []
    for k in range(len(t.vts)):
        for arg in (1, 2):
            out += [off_fn(t, LAG, k, arg, 0, nullable, flags), off_fn(t, LEAD, k, arg, 0, nullable, flags)]
        for fr in FRAMES:
            out += [off_fn(t, FIRST, k, 0, fr, nullable, flags), off_fn(t, LAST, k, 0, fr, nullable, flags),
                    off_fn(t, NTH_VALUE, k, 2, fr, nullable, flags)]
    return out


def check(capi, plain, t, keys, npk, fns, codec=1, level=0, alg=0, dev=False):
    blocks = build_blocks(capi, codec, level, alg, plain)
    want, n, m = model_window_offset(plain, keys, npk, t.nf, t.kinds, fns)
    got, r = run(capi, NAME, codec, alg, blocks, (keys, npk, t.nf, t.kinds, fns), len(want), dev)
    assert (r["status"] == 0).all(), r["status"]
    assert (r["n_records"], r["n_out_records"], r["total"]) == (n, m, len(want))
    if got != want:
        at = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        raise AssertionError("first differing byte %d of %d" % (at, len(want)))
    return r


# ---------------------------------------------------------------------------------------------------------------
# 1. every offset function x frame x value type, nullable and not, with and without IGNORE_NULLS, 0 / 1 / 3 partition
# columns
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, IGNORE_NULLS])
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("npk", [0, 1, 3])
def test_every_function_frame_and_type(capi, npk, nullable, flags):
    rng = np.random.default_rng(1000 + npk + 10 * nullable + 100 * flags)
    t = OTable()
    rows = table(rng, t, 1200, order_domain=5)
    plain = blocks_of(rows, [500, 0, 700])
    fns = all_offsets(t, nullable, flags)
    for at in range(0, len(fns), 16):
        check(capi, plain, t, t.keys(npk, DESC if npk == 1 else 0), npk, fns[at:at + 16])


def test_strings_of_every_length_and_one_of_100_kib(capi):
    rng = np.random.default_rng(1100)
    t = OTable([VAL_BYTES, VAL_INT64])
    lens = [0, 7, 8, 9, 1, 15, 16, 17, 100 << 10] + [int(x) for x in rng.integers(0, 60, 300)]
    rows = []
    for i, n in enumerate(lens):
        s = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        rows.append(t.row([i % 4, 0, 0, i], [(s if i % 5 else None, s), (i, i)]))
    fns = [off_fn(t, f, 0, a, fr, nl, fl) for f, a, fr in ((LAG, 1, 0), (LEAD, 1, 0), (LEAD, 3, 0), (FIRST, 0, 2),
                                                           (LAST, 0, 3), (NTH_VALUE, 2, 1))
           for nl, fl in ((True, 0), (True, IGNORE_NULLS), (False, 0))][:16]
    check(capi, blocks_of(rows, [100, len(rows) - 100]), t, t.keys(1), 1, fns)


# ---------------------------------------------------------------------------------------------------------------
# 2. defaults and offsets
# ---------------------------------------------------------------------------------------------------------------
def test_defaults_of_every_fixed_type(capi):
    rng = np.random.default_rng(1200)
    t = OTable(FIXED_TYPES)
    rows = table(rng, t, 900)
    fns = []
    for k, vt in enumerate(FIXED_TYPES):
        w = WIDTH.get(vt, 8)
        d = int(rng.integers(0, 2**63, dtype=np.uint64)) * 2 % 2**(8 * w) | 1
        fns += [off_fn(t, LAG, k, 1, 0, True, HAS_DEFAULT, d), off_fn(t, LEAD, k, 2, 0, True,
                                                                        HAS_DEFAULT | IGNORE_NULLS, d)]
    for at in range(0, len(fns), 16):
        check(capi, blocks_of(rows, [900]), t, t.keys(1), 1, fns[at:at + 16])


@pytest.mark.parametrize("k", [1, 2, 10_000, 2**31 - 1])
def test_offsets(capi, k):
    rng = np.random.default_rng(1300)
    t = OTable([VAL_INT64, VAL_BYTES, dec(38, 5)])
    rows = table(rng, t, 800)
    fns = [off_fn(t, f, x, k, 0, nl, fl, d) for f in (LAG, LEAD) for x in range(3) for nl, fl, d in (
        (True, 0, 0), (True, IGNORE_NULLS, 0), (False, HAS_DEFAULT if x == 0 else 0, 77 if x == 0 else 0))]
    fns += [off_fn(t, NTH_VALUE, 0, k, FRAME_ROWS, True, IGNORE_NULLS)]
    for at in range(0, len(fns), 16):
        check(capi, blocks_of(rows, [300, 500]), t, t.keys(1), 1, fns[at:at + 16])


# ---------------------------------------------------------------------------------------------------------------
# 3. ranking, aggregate and offset functions in one call; value null bits in a new word
# ---------------------------------------------------------------------------------------------------------------
def test_16_functions_of_all_three_families(capi):
    rng = np.random.default_rng(1400)
    t = OTable([VAL_INT64, VAL_FLOAT64, dec(24, 3), dec(38, 5), VAL_BYTES, VAL_INT32])
    rows = table(rng, t, 2500)
    fns = [ROW_NUMBER, off_fn(t, LAG, 4, 1), (SUM, FRAME_ROWS, *t.value(2)), off_fn(t, LEAD, 3, 2), RANK,
           (AVG, FRAME_RANGE, *t.value(2)), off_fn(t, LAST, 4, 0, FRAME_ROWS, True, IGNORE_NULLS), (NTILE, 3),
           off_fn(t, FIRST, 1, 0, FRAME_RANGE), (MAX, FRAME_PARTITION, *t.value(3)), PERCENT_RANK,
           off_fn(t, NTH_VALUE, 4, 2, FRAME_PARTITION, False), (COUNT, FRAME_RANGE, VAL_NONE, 0, -1),
           off_fn(t, LAG, 5, 1, 0, True, HAS_DEFAULT, 5), CUME_DIST, DENSE_RANK]
    assert len(fns) == 16
    check(capi, blocks_of(rows, [1000, 1500]), t, t.keys(1, DESC | NULLS_LAST), 1, fns)


@pytest.mark.parametrize("nf", [58, 62, 64, 70])
def test_value_null_bits_cross_into_a_new_word(capi, nf):
    rng = np.random.default_rng(1500 + nf)
    t = OTable([VAL_INT64, VAL_BYTES, dec(38, 5), VAL_FLOAT32, VAL_INT8, dec(17, 2), VAL_INT16, dec(20, 1), VAL_INT32,
                VAL_FLOAT64, VAL_BYTES], pad=nf - 26)
    assert t.nf == nf
    rows = table(rng, t, 600, null_frac=0.5)
    fns = [off_fn(t, LAG, 0, 1), off_fn(t, LEAD, 1, 1), off_fn(t, FIRST, 2, 0, FRAME_ROWS, True, IGNORE_NULLS),
           off_fn(t, LAST, 3, 0, FRAME_RANGE), off_fn(t, NTH_VALUE, 4, 2, FRAME_PARTITION),
           off_fn(t, LAG, 10, 2, 0, True, IGNORE_NULLS), (SUM, FRAME_ROWS, *t.value(5)), off_fn(t, LEAD, 7, 1)]
    check(capi, blocks_of(rows, [300, 300]), t, t.keys(1), 1, fns)


def test_first_last_nth_without_an_order_column(capi):
    rng = np.random.default_rng(1550)
    t = OTable([VAL_INT64, VAL_BYTES])
    rows = table(rng, t, 1500)
    for npk in (1, 3):
        check(capi, blocks_of(rows, [1500]), t, t.keys(npk)[:npk], npk,
              [off_fn(t, FIRST, 1, 0, FRAME_PARTITION), off_fn(t, LAST, 0, 0, FRAME_PARTITION, True, IGNORE_NULLS),
               off_fn(t, NTH_VALUE, 1, 3, FRAME_PARTITION, True, IGNORE_NULLS)])


@pytest.mark.parametrize("alg", [0, 3])
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_every_codec_and_checksum(capi, name, codec, level, alg):
    rng = np.random.default_rng(1600 + codec * 4 + level + alg)
    t = OTable([VAL_INT64, VAL_BYTES, dec(38, 5), VAL_FLOAT64])
    rows = table(rng, t, 1500)
    fns = [off_fn(t, LAG, 0, 1), off_fn(t, LEAD, 1, 1, 0, True, IGNORE_NULLS), off_fn(t, LAST, 2, 0, FRAME_ROWS),
           off_fn(t, NTH_VALUE, 3, 2, FRAME_RANGE, True, IGNORE_NULLS), RANK]
    check(capi, blocks_of(rows, [600, 0, 900]), t, t.keys(1), 1, fns, codec=codec, level=level, alg=alg)


# ---------------------------------------------------------------------------------------------------------------
# 4. partition shapes: one reducer-wide partition of 99 % nulls, many tiny partitions
# ---------------------------------------------------------------------------------------------------------------
def test_one_partition_of_200k_rows_with_99_percent_nulls(capi):
    rng = np.random.default_rng(1700)
    t = OTable([VAL_INT64, VAL_BYTES])
    n = 200_000
    order = rng.integers(0, 50_000, n).tolist()
    present = (rng.random(n) < 0.01).tolist()
    rows = [t.row([0, 0, 0, o], [(i if p else None, i), (b"s%d" % i if p else None, b"")])
            for i, (o, p) in enumerate(zip(order, present))]
    fns = [off_fn(t, LAG, 0, 1, 0, True, IGNORE_NULLS), off_fn(t, LEAD, 0, 3, 0, True, IGNORE_NULLS),
           off_fn(t, LAST, 1, 0, FRAME_ROWS, True, IGNORE_NULLS), off_fn(t, FIRST, 0, 0, FRAME_RANGE, True,
                                                                          IGNORE_NULLS),
           off_fn(t, NTH_VALUE, 1, 5, FRAME_ROWS, True, IGNORE_NULLS), off_fn(t, LAG, 0, 1)]
    check(capi, blocks_of(rows, [80_000, 120_000]), t, t.keys(0), 0, fns)


def test_50k_partitions_of_1_to_4_rows(capi):
    rng = np.random.default_rng(1701)
    t = OTable([VAL_INT64, VAL_BYTES, dec(24, 3)])
    rows = []
    for p in range(50_000):
        for _ in range(int(rng.integers(1, 5))):
            rows.append(t.row([p, 0, 0, int(rng.integers(3))],
                              [(rand_any(rng, vt) if rng.random() < 0.7 else None, rand_any(rng, vt))
                               for vt in t.vts]))
    rows = [rows[i] for i in rng.permutation(len(rows))]
    fns = [off_fn(t, LAG, 0, 1, 0, True, IGNORE_NULLS), off_fn(t, LEAD, 1, 1), off_fn(t, LAST, 1, 0, FRAME_ROWS, True,
                                                                                      IGNORE_NULLS),
           off_fn(t, NTH_VALUE, 2, 2, FRAME_PARTITION), off_fn(t, FIRST, 2, 0, FRAME_RANGE, True, IGNORE_NULLS),
           ROW_NUMBER]
    check(capi, blocks_of(rows, [len(rows) // 2, len(rows) - len(rows) // 2]), t, t.keys(1), 1, fns)


# ---------------------------------------------------------------------------------------------------------------
# 5. a corrupt string slot, the _dev form, the size retry, empty input, ranking and aggregate-only calls
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["past the row", "in the fixed region"])
def test_corrupt_string_slot_fails_its_block(capi, where):
    rng = np.random.default_rng(1800)
    t = OTable([VAL_BYTES])
    rows = table(rng, t, 200, null_frac=0.0)
    bad = bytearray(rows[150])
    s = t.slot(t.first + 1)  # the never-null copy
    fixed = 8 * (t.bw + t.nf)
    bad[s:s + 8] = ((len(bad) - 4) << 32 | 8 if where == "past the row" else (fixed - 8) << 32 | 4).to_bytes(8, "little")
    plain = [stream(rows[:100]), stream(rows[100:150] + [bytes(bad)] + rows[151:])]
    # an offset no output row reaches: every input is still checked
    fns = [off_fn(t, LAG, 0, 2**31 - 1, 0, False)]
    got, r = run(capi, NAME, 1, 3, build_blocks(capi, 1, 0, 3, plain), (t.keys(1), 1, t.nf, t.kinds, fns), 1 << 16)
    assert list(r["status"]) == [0, capi.E_CORRUPT]
    assert (r["n_records"], r["n_out_records"], r["total"]) == (0, 0, 0) and got == b""
    assert b"block 1" in capi.load().b2s_last_error()


def test_lag_and_lead_need_an_order_column(capi):
    rng = np.random.default_rng(1850)
    t = OTable([VAL_INT64])
    blocks = build_blocks(capi, 1, 0, 0, [stream(table(rng, t, 20))])
    keys = t.keys(1)[:1]
    for fns in ([off_fn(t, LAG, 0, 1)], [off_fn(t, FIRST, 0, 0, FRAME_PARTITION), off_fn(t, LEAD, 0, 1)],
                [off_fn(t, LAST, 0, 0, FRAME_ROWS)]):
        with pytest.raises(capi.B2SError) as e:
            run(capi, NAME, 1, 0, blocks, (keys, 1, t.nf, t.kinds, fns), 1 << 14)
        assert e.value.code == capi.E_ARG


def test_dev_matches_packed(capi):
    rng = np.random.default_rng(1900)
    t = OTable()
    plain = blocks_of(table(rng, t, 1500), [700, 800])
    fns = all_offsets(t, True, IGNORE_NULLS)[-16:]
    a = check(capi, plain, t, t.keys(1), 1, fns, codec=3, level=1, alg=3)
    b = check(capi, plain, t, t.keys(1), 1, fns, codec=3, level=1, alg=3, dev=True)
    assert (a["n_records"], a["n_out_records"], a["total"]) == (b["n_records"], b["n_out_records"], b["total"])


def test_dst_too_small_reports_the_exact_size(capi):
    import ctypes as C
    rng = np.random.default_rng(1901)
    t = OTable([VAL_BYTES, dec(38, 5)])
    plain = blocks_of(table(rng, t, 500), [500])
    fns = [off_fn(t, LEAD, 0, 1), off_fn(t, LAG, 1, 1, 0, True, IGNORE_NULLS)]
    want, n, m = model_window_offset(plain, t.keys(1), 1, t.nf, t.kinds, fns)
    arena, off, ln, sb, sl, sc = build_blocks(capi, 1, 0, 0, plain)
    a = capi._window_offset_arrays(t.keys(1), 1, t.nf, t.kinds, fns)
    dst = np.zeros(len(want) - 1, np.uint8)
    counts = [C.c_uint64(0) for _ in range(3)]
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = capi.load().b2s_decompress_window_offset_rows_keys_packed(
        1, 0, 1, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None, *map(capi._arg, a),
        dst.ctypes.data, dst.size, *map(C.byref, counts), st.ctypes.data, bad.ctypes.data)
    assert rc == capi.E_DST_TOO_SMALL and counts[0].value == len(want)
    got, r = run(capi, NAME, 1, 0, (arena, off, ln, sb, sl, sc), (t.keys(1), 1, t.nf, t.kinds, fns), counts[0].value)
    assert got == want and (r["n_records"], r["n_out_records"]) == (n, m)


def test_empty_input(capi):
    t = OTable([VAL_BYTES])
    r = check(capi, [b"", b""], t, t.keys(1), 1, [off_fn(t, LAG, 0, 1)])
    assert (r["n_records"], r["n_out_records"], r["total"]) == (0, 0, 0)


@pytest.mark.parametrize("npk", [0, 1])
def test_ranking_and_aggregate_only_are_byte_identical_to_the_aggregate_call(capi, npk):
    rng = np.random.default_rng(1950 + npk)
    t = OTable([dec(24, 3), VAL_INT64, VAL_FLOAT64, dec(38, 2)])
    plain = blocks_of(table(rng, t, 3000), [1000, 2000])
    blocks = build_blocks(capi, 2, 0, 3, plain)
    fns = [ROW_NUMBER, (SUM, FRAME_ROWS, *t.value(0)), RANK, (MAX, FRAME_RANGE, *t.value(3)), (NTILE, 7),
           (AVG, FRAME_PARTITION, *t.value(2)), (MIN, FRAME_ROWS, *t.value(3, False)), (COUNT, FRAME_RANGE, VAL_NONE, 0,
                                                                                        -1)]
    keys = t.keys(npk, DESC)
    a, ra = run(capi, NAME, 2, 3, blocks, (keys, npk, t.nf, t.kinds, fns), 1 << 22)
    b, rb = run(capi, AGG_NAME, 2, 3, blocks, (keys, npk, t.nf, t.kinds, fns), 1 << 22)
    assert a == b and (ra["n_records"], ra["n_out_records"], ra["total"]) == (rb["n_records"], rb["n_out_records"],
                                                                              rb["total"])
    assert a == model_window_offset(plain, keys, npk, t.nf, t.kinds, fns)[0]


# ---------------------------------------------------------------------------------------------------------------
# 6. the host mirror
# ---------------------------------------------------------------------------------------------------------------
def test_host_mirror_reads_window_offset_rows(capi, tmp_path):
    host = pkg.host
    d = mirror(tmp_path, "lz4")
    M, R = 3, 2
    rng = np.random.default_rng(2000)
    t = OTable([VAL_INT64, VAL_BYTES, dec(38, 5)])
    maps = []
    for m in range(M):
        rows = table(rng, t, 300)
        maps.append((rows, rng.integers(0, R, len(rows))))
    write_maps(host, d, maps, R)
    fns = [off_fn(t, LAG, 0, 1, 0, True, HAS_DEFAULT, 9), off_fn(t, LAST, 1, 0, FRAME_ROWS, True, IGNORE_NULLS),
           off_fn(t, LEAD, 2, 2), RANK, (SUM, FRAME_RANGE, *t.value(0))]
    for red in range(R):
        plain = [stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps]
        reader = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        got = reader.readWindowOffsetRows(t.keys(1), 1, t.nf, t.kinds, fns)
        reader.close()
        assert got == model_window_offset(plain, t.keys(1), 1, t.nf, t.kinds, fns)
