"""Row sort and row aggregation by a composite key (b2s_decompress_sort_rows_keys_* / b2s_decompress_aggregate_rows_keys_*):
up to 16 key columns compared left to right, each an unsigned byte string, a signed int32 / int64 or a variable-length
string (an UnsafeRow (offset << 32) | size slot), nulls first per column.  The model sorts the records stably by a tuple
of (not-null flag, value) per column, with strings as Python bytes (whose order is exactly unsigned lexicographic with a
proper prefix first), and groups equal tuples; every output must equal it byte for byte."""
import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from rows_model import CHECKSUMS, CODECS, KEY_BYTES, KEY_INT32, KEY_INT64, MAX_I64, MIN_I32, MIN_I64, STRING, SUM_I64, \
    blocks_of, build_blocks, mirror, model_aggregate, model_sort, run, stream, write_maps

pytestmark = pytest.mark.gpu

P, CHUNK = 20, 16  # the first pass's key bytes and a refinement round's


# ---------------------------------------------------------------------------------------------------------------
# rows: one null word, then a 16-byte area per key column, then 8-byte aggregate slots, then the strings
# ---------------------------------------------------------------------------------------------------------------
KLEN = {KEY_INT32: 4, KEY_INT64: 8, STRING: 8}


def layout(types, nullable=True, byte_len=10):
    """-> key columns [(type, off, len, null field)]; column c at 8 + 16 c, null bit c + 1 (bit 0 stays unused)"""
    return [(t, 8 + 16 * c, KLEN.get(t, byte_len), c + 1 if nullable else -1) for c, t in enumerate(types)]


def agg_layout(keys, ops):
    base = 8 + 16 * len(keys)
    return [(op, base + 8 * a, 20 + a) for a, op in enumerate(ops)]


def make_row(rng, keys, vals, aggs=(), agg_vals=(), agg_nulls=(), tail=0):
    """vals[c]: int / bytes, or None for null; strings go after the fixed region, 8-byte aligned"""
    fixed = 8 + 16 * len(keys) + 8 * len(aggs)
    r = bytearray(rng.integers(0, 256, fixed, dtype=np.uint8).tobytes())
    word = int(rng.integers(0, 2**63)) & ~((1 << 40) - 2)  # bits 1..39 (key and aggregate null bits) clear
    var = bytearray()
    for (kt, ko, kl, nf), v in zip(keys, vals):
        if v is None:
            word |= 1 << nf
            continue
        if kt == STRING:
            o = fixed + len(var)
            var += v + bytes(-len(v) % 8)
            r[ko:ko + 8] = ((o << 32) | len(v)).to_bytes(8, "little")
        elif kt == KEY_BYTES:
            r[ko:ko + kl] = v
        else:
            r[ko:ko + kl] = int(v).to_bytes(kl, "little", signed=True)
    for (op, off, anf), v, null in zip(aggs, agg_vals, agg_nulls):
        r[off:off + 8] = (int(v) % 2**64).to_bytes(8, "little")
        if null and anf >= 0:
            word |= 1 << anf
    r[0:8] = word.to_bytes(8, "little")
    return bytes(r + var + rng.integers(0, 256, tail, dtype=np.uint8).tobytes())


PREFIXES = [b"", b"ab", b"category#", b"\x00\x00\x00", b"\xff" * 12, b"Books/Fiction/" * 3]


def rand_value(rng, kt, n_choices=5, byte_len=10):
    if kt == STRING:
        pre = PREFIXES[int(rng.integers(len(PREFIXES)))]
        return pre + rng.integers(0, 256, int(rng.integers(0, 12)), dtype=np.uint8).tobytes()[: int(rng.integers(0, 12))]
    if kt == KEY_BYTES:
        return bytes(int(rng.integers(0, n_choices)) for _ in range(byte_len))
    if kt == KEY_INT32:
        return int(rng.choice([-2**31, 2**31 - 1, -1, 0, 1, int(rng.integers(-5, 5))]))
    return int(rng.choice([-2**63, 2**63 - 1, -1, 0, 1, int(rng.integers(-5, 5))]))


def rand_rows(rng, n, keys, null_frac=0.15, aggs=(), tail=True):
    rows = []
    for _ in range(n):
        vals = [None if (c[3] >= 0 and rng.random() < null_frac) else rand_value(rng, c[0], byte_len=c[2])
                for c in keys]
        av = [int(x) for x in rng.integers(-1000, 1000, len(aggs))]
        an = [rng.random() < 0.2 for _ in aggs]
        rows.append(make_row(rng, keys, vals, aggs, [v & (2**64 - 1) for v in av], an,
                             int(rng.integers(0, 20)) if tail else 0))
    return rows


def check_sort(capi, plain, keys, codec=1, level=0, alg=0, dev=False, blocks=None):
    blocks = blocks or build_blocks(capi, codec, level, alg, plain)
    total = sum(len(b) for b in plain)
    got, r = run(capi, "decompress_sort_rows_keys", codec, alg, blocks, (keys,), total, dev)
    assert (r["status"] == 0).all(), r["status"]
    want, n = model_sort(plain, keys)
    assert (r["total"], r["n_records"]) == (total, n)
    assert got == want
    return got


def check_agg(capi, plain, keys, aggs, codec=1, level=0, alg=0, dev=False, blocks=None):
    blocks = blocks or build_blocks(capi, codec, level, alg, plain)
    total = sum(len(b) for b in plain)
    got, r = run(capi, "decompress_aggregate_rows_keys", codec, alg, blocks, (keys, aggs), total, dev)
    assert (r["status"] == 0).all(), r["status"]
    want, n, g = model_aggregate(plain, keys, aggs)
    assert (r["n_records"], r["n_groups"], r["total"]) == (n, g, len(want))
    assert got == want
    return got, r


MIXED = [STRING, KEY_INT32, STRING, KEY_INT64, KEY_BYTES]


# ---------------------------------------------------------------------------------------------------------------
# 1. every codec x checksum, packed and _dev; 1, 2, 5 and 16 columns
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", CHECKSUMS)
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_sorts_and_aggregates_like_the_model(capi, name, codec, level, alg):
    rng = np.random.default_rng(codec * 10 + alg)
    keys = layout(MIXED)
    aggs = agg_layout(keys, [SUM_I64, MIN_I64])
    rows = rand_rows(rng, 3000, keys, aggs=aggs)
    plain = blocks_of(rows, [1000, 0, 1200, 800])
    blocks = build_blocks(capi, codec, level, alg, plain)
    dev = alg % 2 == 1
    check_sort(capi, plain, keys, codec, level, alg, dev, blocks)
    check_agg(capi, plain, keys, aggs, codec, level, alg, not dev, blocks)


@pytest.mark.parametrize("types", [
    [STRING], [KEY_INT64, STRING], [STRING, STRING], MIXED,
    [STRING, KEY_INT32, KEY_BYTES, KEY_INT64] * 4,
    [KEY_INT32] * 16, [KEY_INT64, KEY_INT64], [KEY_INT32] * 5])
@pytest.mark.parametrize("nullable", [False, True])
def test_column_counts_and_types(capi, types, nullable):
    rng = np.random.default_rng(len(types) * 2 + nullable)
    keys = layout(types, nullable)
    aggs = agg_layout(keys, [SUM_I64, MAX_I64])
    rows = rand_rows(rng, 2500, keys, aggs=aggs)
    plain = blocks_of(rows, [900, 1600])
    check_sort(capi, plain, keys, dev=nullable)
    check_agg(capi, plain, keys, aggs, dev=not nullable)


# ---------------------------------------------------------------------------------------------------------------
# 2. string lengths around the first pass, the chunks and the 8-byte groups; 0x00 / 0xFF; long strings
# ---------------------------------------------------------------------------------------------------------------
BOUNDARY_LENS = sorted({0, 1, 2, 7, 8, 9, 15, 16, 17, P - 1, P, P + 1, 2 * P - 1, 2 * P, 2 * P + 1, 23, 24, 25, 31, 32,
                        33, 39, 40, 41, 63, 64, 65, 71, 72, 73})


@pytest.mark.parametrize("fill", [b"\x00", b"\xff", b"a"])
def test_strings_equal_up_to_and_across_chunk_boundaries(capi, fill):
    rng = np.random.default_rng(fill[0])
    keys = layout([STRING, KEY_INT32])
    rows = []
    for ln in BOUNDARY_LENS:
        for tail in (b"", b"\x00", b"\x01", b"\xff", b"\x00\x00"):
            for k2 in (3, -3):
                rows.append(make_row(rng, keys, [fill * ln + tail, k2]))
                rows.append(make_row(rng, keys, [fill * ln + tail, k2]))
    rng.shuffle(rows)
    plain = blocks_of(rows, [len(rows) // 2, len(rows) - len(rows) // 2])
    check_sort(capi, plain, keys)
    check_agg(capi, plain, keys, [], dev=True)


def test_four_kib_strings(capi):
    rng = np.random.default_rng(4)
    keys = layout([STRING, STRING])
    base = rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()
    rows = []
    for i in range(300):
        a = base[: 4096 - int(rng.integers(0, 3))]
        if rng.random() < 0.5:
            p = int(rng.integers(0, len(a)))
            a = a[:p] + bytes([int(rng.integers(0, 256))]) + a[p + 1:]
        rows.append(make_row(rng, keys, [a, base[: int(rng.integers(0, 4097))]]))
    check_sort(capi, blocks_of(rows, [150, 150]), keys)
    check_agg(capi, blocks_of(rows, [300]), keys, [])


def test_hundred_thousand_rows_sharing_a_200_byte_prefix(capi):
    rng = np.random.default_rng(200)
    keys = layout([STRING, KEY_INT64], nullable=False)
    aggs = agg_layout(keys, [SUM_I64])
    prefix = rng.integers(0, 256, 200, dtype=np.uint8).tobytes()
    rows = []
    for i in range(100_000):
        s = prefix + rng.integers(0, 4, int(rng.integers(0, 4)), dtype=np.uint8).tobytes()
        rows.append(make_row(rng, keys, [s, int(rng.integers(0, 3))], aggs, [i], [False]))
    plain = blocks_of(rows, [25_000] * 4)
    check_sort(capi, plain, keys, codec=2)
    check_agg(capi, plain, keys, aggs, codec=2, dev=True)


# ---------------------------------------------------------------------------------------------------------------
# 3. nulls, prefixes, one group, all distinct, stability
# ---------------------------------------------------------------------------------------------------------------
def test_null_and_empty_strings_are_different_keys(capi):
    rng = np.random.default_rng(5)
    keys = layout([STRING, KEY_INT32])
    aggs = agg_layout(keys, [SUM_I64])
    rows = [make_row(rng, keys, [v, k], aggs, [i], [False])
            for i, (v, k) in enumerate([(None, 1), (b"", 1), (None, 1), (b"", 1), (b"\x00", 1), (None, None),
                                        (b"", None), (b"", 0)] * 20)]
    check_sort(capi, blocks_of(rows, [len(rows)]), keys)
    got, r = check_agg(capi, blocks_of(rows, [len(rows)]), keys, aggs)
    assert r["n_groups"] == 6


@pytest.mark.parametrize("order", ["string_first", "int_first"])
def test_prefix_strings_order_before_their_extensions(capi, order):
    """("ab", 7) against ("abc", 0): a string that is a proper prefix of another sorts first whatever follows it"""
    rng = np.random.default_rng(6)
    types = [STRING, KEY_INT32] if order == "string_first" else [KEY_INT32, STRING]
    keys = layout(types)
    pairs = [(b"ab", 7), (b"abc", 0), (b"ab", -2**31), (b"abc", 2**31 - 1), (b"a", 5), (b"", 9), (b"ab\x00", 1),
             (b"abcdefgh", 1), (b"abcdefghi", 0), (b"abcdefg", 2), (b"abcdefgh\x00", 0)]
    rows = []
    for s, k in pairs * 5:
        vals = [s, k] if order == "string_first" else [k, s]
        rows.append(make_row(rng, keys, vals))
    rng.shuffle(rows)
    check_sort(capi, blocks_of(rows, [len(rows)]), keys)
    check_agg(capi, blocks_of(rows, [len(rows)]), keys, [], dev=True)


def test_all_keys_equal_make_one_group(capi):
    rng = np.random.default_rng(7)
    keys = layout([STRING, KEY_INT64, STRING])
    aggs = agg_layout(keys, [SUM_I64, MAX_I64])
    rows = [make_row(rng, keys, [b"same string value, longer than a chunk", -5, b"x" * 33], aggs, [i, -i],
                     [False, i % 3 == 0]) for i in range(5000)]
    plain = blocks_of(rows, [2000, 3000])
    assert check_sort(capi, plain, keys) == b"".join(plain)  # stable: input order
    _, r = check_agg(capi, plain, keys, aggs)
    assert r["n_groups"] == 1


def test_all_keys_distinct(capi):
    rng = np.random.default_rng(8)
    keys = layout([STRING, KEY_INT32])
    rows = [make_row(rng, keys, [b"key-%09d" % int(x), 0]) for x in rng.permutation(20000)]
    plain = blocks_of(rows, [10000, 10000])
    check_sort(capi, plain, keys)
    _, r = check_agg(capi, plain, keys, [])
    assert r["n_groups"] == 20000


def test_shared_slot_and_null_word_between_columns(capi):
    """two columns may read the same slot and null bit (e.g. a key repeated in the grouping)"""
    rng = np.random.default_rng(9)
    keys = layout([STRING, KEY_INT32])
    keys = keys + [keys[0], (KEY_INT32, keys[1][1], 4, keys[0][3])]
    rows = rand_rows(rng, 2000, keys[:2])
    check_sort(capi, blocks_of(rows, [2000]), keys)
    check_agg(capi, blocks_of(rows, [2000]), keys, [])


# ---------------------------------------------------------------------------------------------------------------
# 4. one fixed-width column: byte for byte the single-key calls
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kt,kl", [(KEY_BYTES, 1), (KEY_BYTES, 10), (KEY_BYTES, 16), (KEY_INT32, 4), (KEY_INT64, 8)])
@pytest.mark.parametrize("nf", [-1, 1])
def test_one_column_is_the_single_key_call(capi, kt, kl, nf):
    rng = np.random.default_rng(kl * 3 + nf)
    keys = [(kt, 8, kl, nf)]
    aggs = [(SUM_I64, 24, 5), (MIN_I32, 32, -1)]
    rows = rand_rows(rng, 4000, [(kt, 8, kl, nf)], aggs=aggs)
    plain = blocks_of(rows, [1500, 2500])
    blocks = build_blocks(capi, 1, 0, 3, plain)
    arena, off, ln, sb, sl, sc = blocks
    total = sum(len(b) for b in plain)
    want = np.zeros(total, np.uint8)
    r1 = capi.decompress_sort_rows_packed(1, arena, off, ln, want, kt, 8, kl, nf, 3, sb, sl, sc)
    got, r2 = run(capi, "decompress_sort_rows_keys", 1, 3, blocks, (keys,), total)
    assert got == want.tobytes() and r1["n_records"] == r2["n_records"] == 4000
    want = np.zeros(total, np.uint8)
    a1 = capi.decompress_aggregate_rows_packed(1, arena, off, ln, want, kt, 8, kl, nf, aggs, 3, sb, sl, sc)
    got, a2 = run(capi, "decompress_aggregate_rows_keys", 1, 3, blocks, (keys, aggs), total)
    assert got == want[: a1["total"]].tobytes()
    assert (a1["n_records"], a1["n_groups"], a1["total"]) == (a2["n_records"], a2["n_groups"], a2["total"])


# ---------------------------------------------------------------------------------------------------------------
# 5. corrupt input, short destination, argument errors
# ---------------------------------------------------------------------------------------------------------------
def test_string_past_its_row_fails_the_block(capi):
    rng = np.random.default_rng(10)
    keys = layout([KEY_INT32, STRING])
    good = rand_rows(rng, 400, keys)
    bad_row = bytearray(make_row(rng, keys, [1, b"abcdef"]))
    so = keys[1][1]
    bad_row[so:so + 8] = ((len(bad_row) - 3 << 32) | 4).to_bytes(8, "little")  # 4 bytes from 3 before the end
    blocks_rows = [good[:200], good[200:300] + [bytes(bad_row)] + good[300:]]
    plain = [b"".join(len(r).to_bytes(4, "big") + r for r in b) for b in blocks_rows]
    at = sum(4 + len(r) for r in good[200:300])
    for aggregate in (False, True):
        blocks = build_blocks(capi, 2, 0, 0, plain)
        total = sum(len(b) for b in plain)
        got, r = (run(capi, "decompress_aggregate_rows_keys", 2, 0, blocks, (keys, []), total) if aggregate
                  else run(capi, "decompress_sort_rows_keys", 2, 0, blocks, (keys,), total))
        assert list(r["status"]) == [0, capi.E_CORRUPT]
        assert r["n_records"] == 0 and got == b""
        err = capi.load().b2s_last_error().decode()
        assert "block 1" in err and "byte %d" % at in err and "string" in err, err


def test_null_string_with_a_bad_slot_is_fine(capi):
    rng = np.random.default_rng(11)
    keys = layout([STRING])
    rows = [bytearray(make_row(rng, keys, [None])) for _ in range(10)]
    for r in rows:
        r[8:16] = (2**63 + 12345).to_bytes(8, "little")  # never read: the string is null
    rows = [bytes(r) for r in rows]
    check_sort(capi, blocks_of(rows, [10]), keys)


def test_bad_checksum_in_one_block(capi):
    rng = np.random.default_rng(12)
    keys = layout([STRING, KEY_INT64])
    rows = rand_rows(rng, 600, keys)
    plain = blocks_of(rows, [200, 200, 200])
    arena, off, ln, sb, sl, sc = build_blocks(capi, 1, 0, 3, plain)
    sc = sc.copy()
    sc[1] ^= 1
    blocks = (arena, off, ln, sb, sl, sc)
    total = sum(len(b) for b in plain)
    for aggregate in (False, True):
        got, r = (run(capi, "decompress_aggregate_rows_keys", 1, 3, blocks, (keys, []), total) if aggregate
                  else run(capi, "decompress_sort_rows_keys", 1, 3, blocks, (keys,), total))
        assert list(r["status"]) == [0, capi.E_CHECKSUM, 0] and r["n_records"] == 0


def test_short_destination_reports_the_bytes_needed(capi):
    rng = np.random.default_rng(13)
    keys = layout([STRING, KEY_INT32])
    rows = rand_rows(rng, 500, keys)
    plain = blocks_of(rows, [500])
    blocks = build_blocks(capi, 0, 0, 0, plain)
    total = sum(len(b) for b in plain)
    with pytest.raises(capi.B2SError) as e:
        run(capi, "decompress_sort_rows_keys", 0, 0, blocks, (keys,), total - 1)
    assert e.value.code == capi.E_DST_TOO_SMALL
    want, _, _ = model_aggregate(plain, keys, [])
    with pytest.raises(capi.B2SError) as e:
        run(capi, "decompress_aggregate_rows_keys", 0, 0, blocks, (keys, []), len(want) - 1)
    assert e.value.code == capi.E_DST_TOO_SMALL
    assert str(len(want)) in capi.load().b2s_last_error().decode()


@pytest.mark.parametrize("keys,aggs", [
    ([], []),
    ([(KEY_INT32, 8, 4, -1)] * 17, []),
    ([(4, 8, 8, -1)], []),
    ([(STRING, 8, 4, -1)], []),
    ([(KEY_INT32, 8, 8, -1)], []),
    ([(KEY_INT64, 8, 4, -1)], []),
    ([(KEY_BYTES, 8, 0, -1)], []),
    ([(KEY_BYTES, 8, 17, -1)], []),
    ([(STRING, 8, 8, -2)], []),
    ([(KEY_INT32, 8, 4, -1), (STRING, 24, 8, 1)], [(SUM_I64, 28, -1)]),  # overlaps the string slot
    ([(KEY_INT32, 8, 4, -1), (STRING, 24, 8, 1)], [(SUM_I64, 0, -1)]),   # overlaps a key's null word
    ([(STRING, 8, 8, 70)], [(SUM_I64, 8 * 1 + 0, -1), (SUM_I64, 16, -1)]),  # second null word / the slot
    ([(KEY_INT32, 8, 4, -1)], [(9, 24, -1)]),
])
def test_bad_arguments(capi, keys, aggs):
    rng = np.random.default_rng(14)
    rows = [make_row(rng, layout([KEY_INT32]), [1]) + bytes(64)]
    plain = blocks_of(rows, [1])
    blocks = build_blocks(capi, 0, 0, 0, plain)
    for aggregate in ([True] if aggs else [False, True]):
        with pytest.raises(capi.B2SError) as e:
            if aggregate:
                run(capi, "decompress_aggregate_rows_keys", 0, 0, blocks, (keys, aggs), 4096)
            else:
                run(capi, "decompress_sort_rows_keys", 0, 0, blocks, (keys,), 4096)
        assert e.value.code == capi.E_ARG


def test_null_key_arrays(capi):
    import ctypes as C
    L = capi.load()
    src = np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    t = np.array([KEY_INT32], np.uint32)
    total, nrec, ngrp = C.c_uint64(7), C.c_uint64(7), C.c_uint64(7)
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = L.b2s_decompress_sort_rows_keys_packed(0, 0, 1, src.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None,
                                                None, 1, t.ctypes.data, None, t.ctypes.data, None, src.ctypes.data,
                                                src.size, C.byref(total), C.byref(nrec), st.ctypes.data,
                                                bad.ctypes.data)
    assert rc == capi.E_ARG and total.value == 0 and nrec.value == 0
    rc = L.b2s_decompress_aggregate_rows_keys_packed(0, 0, 1, src.ctypes.data, off.ctypes.data, ln.ctypes.data, None,
                                                     None, None, 1, None, None, None, None, 0, None, None, None,
                                                     src.ctypes.data, src.size, C.byref(total), C.byref(nrec),
                                                     C.byref(ngrp), st.ctypes.data, bad.ctypes.data)
    assert rc == capi.E_ARG and ngrp.value == 0


def test_single_key_calls_still_reject_the_string_type(capi):
    rng = np.random.default_rng(15)
    rows = [make_row(rng, layout([STRING]), [b"abc"])]
    arena, off, ln, sb, sl, sc = build_blocks(capi, 0, 0, 0, blocks_of(rows, [1]))
    dst = np.zeros(4096, np.uint8)
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_sort_rows_packed(0, arena, off, ln, dst, STRING, 8, 8, 1)
    assert e.value.code == capi.E_ARG
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_aggregate_rows_packed(0, arena, off, ln, dst, STRING, 8, 8, 1, [])
    assert e.value.code == capi.E_ARG


# ---------------------------------------------------------------------------------------------------------------
# 6. the host mirror: readSortedRowsKeys / readAggregatedRowsKeys over the serialized writer's files
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_reads_rows_by_a_composite_key(capi, tmp_path, codec):
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R, per_map = 3, 2, 1500
    keys = layout([STRING, KEY_INT32, STRING])
    aggs = agg_layout(keys, [SUM_I64, MIN_I32])
    maps = []
    for m in range(M):
        rng = np.random.default_rng(90 + m)
        maps.append((rand_rows(rng, per_map, keys, aggs=aggs), rng.integers(0, R, per_map)))
    write_maps(host, d, maps, R)
    for red in range(R):
        plain = [stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps]
        rd = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        data, n = rd.readSortedRowsKeys(keys)
        want, wn = model_sort(plain, keys)
        assert n == wn and data == want
        blocks = build_blocks(capi, 0, 0, 0, plain)
        assert data == run(capi, "decompress_sort_rows_keys", 0, 0, blocks, (keys,), sum(len(b) for b in plain))[0]
        data, n, g = rd.readAggregatedRowsKeys(keys, aggs)
        rd.close()
        want, wn, wg = model_aggregate(plain, keys, aggs)
        assert (n, g) == (wn, wg) and data == want
    d.close()
