"""b2s_decompress_join_rows_keys_* on the GPU: every output byte for byte equal to the model (join_model.py) of Spark's
sort-merge join and UnsafeRowJoiner, over every join type, codec and layout the header names, its failures, a
hash-partitioned join end to end, and the host mirror's joined read of two shuffles."""
import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from hash_model import keys_of, make_row, records_of
from join_model import DECIMAL_WIDE, FIXED, INNER, LEFT_ANTI, LEFT_OUTER, LEFT_SEMI, VAR, model_join
from rows_model import blocks_of, build_blocks, mirror, stream

pytestmark = pytest.mark.gpu

JOINS = [INNER, LEFT_OUTER, LEFT_SEMI, LEFT_ANTI]
CODECS = [("none", 0, 0), ("lz4", 1, 0), ("snappy", 2, 0), ("zstd", 3, 1)]
KIND = {"string": VAR, "decimal": DECIMAL_WIDE}


def kinds(types):
    return [KIND.get(t, FIXED) for t in types]


def row(types, vals):
    """make_row, with a null Decimal(p > 18) written as UnsafeRowWriter writes it: 16 zero bytes, slot offset << 32"""
    r = bytearray(make_row(types, vals))
    bitset = 8 * ((len(types) + 63) // 64)
    for i, (t, v) in enumerate(zip(types, vals)):
        if t == "decimal" and v is None:
            r[bitset + 8 * i:bitset + 8 * i + 8] = (len(r) << 32).to_bytes(8, "little")
            r += bytes(16)
    return bytes(r)


def rand_val(rng, t, key_range=None):
    if key_range is not None and t in ("long", "int"):
        return int(rng.integers(0, key_range))
    if t == "string":
        return bytes(rng.integers(97, 100, int(rng.integers(0, 30)), dtype=np.uint8))
    if t == "decimal":
        return int(rng.integers(-10**17, 10**17)) * 10**int(rng.integers(0, 3))
    if t in ("double", "float"):
        return float(rng.normal())
    if t == "bool":
        return bool(rng.integers(2))
    return int(rng.integers(-1000, 1000))


def table(rng, types, n, key_fields=(), key_range=50, null_rate=0.1):
    rows = []
    for _ in range(n):
        vals = [None if rng.random() < null_rate else rand_val(rng, t, key_range if f in key_fields else None)
                for f, t in enumerate(types)]
        rows.append(row(types, vals))
    return rows


def split(rng, rows, parts):
    """rows cut into parts blocks (some empty)"""
    cuts = sorted(int(c) for c in rng.integers(0, len(rows) + 1, parts - 1))
    bounds = [0] + cuts + [len(rows)]
    return blocks_of(rows, [bounds[k + 1] - bounds[k] for k in range(parts)])


def call(capi, jt, left, right, lkeys, rkeys, lt, rt, codec=("lz4", 1, 0), alg=3, dev=False, cap=None, kinds_=True):
    """the join of the left and right blocks on the GPU -> (output bytes, result dict)"""
    _, c, level = codec
    arena, off, ln, sb, sl, sc = build_blocks(capi, c, level, alg, list(left) + list(right))
    lk, rk = (kinds(lt), kinds(rt)) if kinds_ else (None, None)
    args = (lkeys, rkeys, len(lt), len(rt), lk, rk, alg, sb, sl, sc)
    if cap is None:
        cap = len(model_join(jt, left, right, lkeys, rkeys, len(lt), len(rt), kinds(lt), kinds(rt))[0])
    if not dev:
        dst = np.zeros(max(cap, 1), np.uint8)
        r = capi.decompress_join_rows_keys_packed(jt, c, arena, off, ln, len(left), dst[:cap], *args)
        return dst[:r["total"]].tobytes(), r
    d_src, d_dst = capi.dev_alloc(max(arena.size, 1)), capi.dev_alloc(max(cap, 1))
    try:
        capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        r = capi.decompress_join_rows_keys_dev(jt, c, d_src, off, ln, len(left), d_dst, cap, *args)
        out = np.zeros(max(r["total"], 1), np.uint8)
        if r["total"]:
            capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        return out[:r["total"]].tobytes(), r
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)


def check(capi, jt, left, right, lkeys, rkeys, lt, rt, **kw):
    want, nl, nr, nout = model_join(jt, left, right, lkeys, rkeys, len(lt), len(rt), kinds(lt), kinds(rt))
    got, r = call(capi, jt, left, right, lkeys, rkeys, lt, rt, kinds_=jt in (INNER, LEFT_OUTER), **kw)
    assert (r["n_left_records"], r["n_right_records"], r["n_out_records"]) == (nl, nr, nout)
    assert (r["status"] == 0).all()
    assert got == want
    return got, r


# the join shape of the exchange tests: a nullable long key, sides of different schemas and key positions
LT = ["long", "string", "int", "decimal", "double"]
RT = ["string", "decimal", "long", "bool"]
LKEY, RKEY = keys_of(LT, [0]), keys_of(RT, [2])


@pytest.mark.parametrize("jt", JOINS)
@pytest.mark.parametrize("codec", CODECS, ids=[c[0] for c in CODECS])
@pytest.mark.parametrize("alg", [0, 3])
def test_join_types_codecs_and_checksums_like_the_model(capi, jt, codec, alg):
    rng = np.random.default_rng(jt * 10 + codec[1] + alg)
    left = split(rng, table(rng, LT, 700, (0,)), 4)
    right = split(rng, table(rng, RT, 500, (2,)), 3)
    check(capi, jt, left, right, LKEY, RKEY, LT, RT, codec=codec, alg=alg)


@pytest.mark.parametrize("jt", JOINS)
def test_string_int_key_with_shared_prefixes_refines(capi, jt):
    rng = np.random.default_rng(7)
    lt, rt = ["string", "int", "long"], ["long", "string", "int", "string"]
    prefix = b"p" * 45

    def t(types, kf, n):
        out = []
        for _ in range(n):
            vals = [rand_val(rng, x) for x in types]
            vals[kf[0]] = None if rng.random() < 0.05 else prefix + bytes([97 + int(rng.integers(3))]) * int(
                rng.integers(1, 3))
            vals[kf[1]] = int(rng.integers(0, 3))
            out.append(row(types, vals))
        return out

    check(capi, jt, split(rng, t(lt, (0, 1), 400), 3), split(rng, t(rt, (1, 2), 300), 2),
          keys_of(lt, [0, 1]), keys_of(rt, [1, 2]), lt, rt)


@pytest.mark.parametrize("jt", JOINS)
def test_float_zeros_and_nans_decimal_and_boolean_keys(capi, jt):
    rng = np.random.default_rng(11)
    specials = [0.0, -0.0, ("bits", 0x7FF8000000000000), ("bits", 0x7FF0000000000001), ("bits", 0xFFF8000000000123),
                1.5, float("inf")]
    lt, rt = ["double", "decimal", "bool", "string"], ["bool", "string", "decimal", "double"]

    def t(types, fd, fdec, fb, n):
        out = []
        for _ in range(n):
            vals = [rand_val(rng, x) for x in types]
            vals[fd] = specials[int(rng.integers(len(specials)))]
            vals[fdec] = None if rng.random() < 0.05 else int(rng.integers(-2, 2)) * 10**30
            vals[fb] = bool(rng.integers(2))
            out.append(row(types, vals))
        return out

    left, right = split(rng, t(lt, 0, 1, 2, 300), 2), split(rng, t(rt, 3, 2, 0, 200), 2)
    check(capi, jt, left, right, keys_of(lt, [0, 1, 2]), keys_of(rt, [3, 2, 0]), lt, rt)


@pytest.mark.parametrize("jt", JOINS)
def test_seventy_fields_cross_a_bitset_word(capi, jt):
    """40 + 30 fields: one null-bit word per input, two in the output, so the right bits and the offsets move"""
    rng = np.random.default_rng(13)
    lt = (["long", "string", "int", "decimal", "double"] * 8)[:40]
    rt = (["decimal", "string", "long"] * 10)[:30]
    left = split(rng, table(rng, lt, 300, (0,), key_range=40, null_rate=0.2), 3)
    right = split(rng, table(rng, rt, 250, (5,), key_range=40, null_rate=0.2), 3)
    check(capi, jt, left, right, keys_of(lt, [0]), keys_of(rt, [5]), lt, rt)


def test_nullability_differs_between_the_sides(capi):
    """a key nullable on the left only still matches equal right keys"""
    rng = np.random.default_rng(17)
    left = split(rng, table(rng, LT, 300, (0,)), 2)
    right = split(rng, table(rng, RT, 200, (2,), null_rate=0), 2)
    for jt in JOINS:
        check(capi, jt, left, right, keys_of(LT, [0]), keys_of(RT, [2], nullable=False), LT, RT)


@pytest.mark.parametrize("jt", JOINS)
@pytest.mark.parametrize("kt", ["long", "int"])
def test_not_null_left_key_with_a_nullable_right_key(capi, jt, kt):
    """the left key NOT NULL, the right one nullable (a NOT NULL dimension key on the left): the key is one byte wider
    than the left columns alone, on every step"""
    rng = np.random.default_rng(59)
    lt, rt = [kt, "string", "double"], ["bool", kt, "string"]
    left = split(rng, table(rng, lt, 600, (0,), null_rate=0), 3)
    right = split(rng, table(rng, rt, 400, (1,), null_rate=0.15), 3)
    check(capi, jt, left, right, keys_of(lt, [0], nullable=False), keys_of(rt, [1]), lt, rt)


@pytest.mark.parametrize("jt", JOINS)
def test_twenty_byte_left_key_that_a_nullable_right_column_widens(capi, jt):
    """(long, long, int) NOT NULL on the left encodes to exactly 20 bytes, the first pass's width; a nullable right
    column makes it 21, so the keys refine, and keys that differ only in the int's low byte must not match"""
    rng = np.random.default_rng(61)
    lt, rt = ["long", "long", "int", "string"], ["string", "int", "long", "long"]

    def t(types, fields, n, null_rate):
        out = []
        for _ in range(n):
            vals = [rand_val(rng, x) for x in types]
            vals[fields[0]], vals[fields[1]] = 7, -3
            vals[fields[2]] = 0x100 + int(rng.integers(0, 4))
            if rng.random() < null_rate:
                vals[fields[2]] = None
            out.append(row(types, vals))
        return out

    left = split(rng, t(lt, (0, 1, 2), 300, 0), 2)
    right = split(rng, t(rt, (2, 3, 1), 200, 0.1), 2)
    check(capi, jt, left, right, keys_of(lt, [0, 1, 2], nullable=False),
          [keys_of(rt, [2], nullable=False)[0], keys_of(rt, [3], nullable=False)[0], keys_of(rt, [1])[0]], lt, rt)


@pytest.mark.parametrize("jt", JOINS)
def test_empty_sides_blocks_and_all_null_keys(capi, jt):
    rng = np.random.default_rng(19)
    left, right = split(rng, table(rng, LT, 200, (0,)), 3), split(rng, table(rng, RT, 150, (2,)), 3)
    check(capi, jt, [], right, LKEY, RKEY, LT, RT)
    check(capi, jt, left, [], LKEY, RKEY, LT, RT)
    check(capi, jt, [b""] + left + [b""], [b"", b""] + right, LKEY, RKEY, LT, RT)
    nulls = [row(RT, [b"x", 1, None, True]) for _ in range(50)]
    check(capi, jt, left, [blocks_of(nulls, [50])[0]], LKEY, RKEY, LT, RT)
    nulls = [row(LT, [None, b"y", 2, None, 1.0]) for _ in range(50)]
    check(capi, jt, [blocks_of(nulls, [50])[0]], right, LKEY, RKEY, LT, RT)


def test_hot_key_many_to_many(capi):
    """1000 x 1000 rows on one key: a million joined rows from one group, beside a few ordinary keys"""
    lt, rt = ["long", "long"], ["long", "int"]
    left = [row(lt, [7, i]) for i in range(1000)] + [row(lt, [k, -k]) for k in range(100, 110)]
    right = [row(rt, [7, i]) for i in range(1000)] + [row(rt, [k, k]) for k in range(105, 120)]
    check(capi, INNER, blocks_of(left, [600, 410]), blocks_of(right, [1015]), keys_of(lt, [0]), keys_of(rt, [0]), lt,
          rt)


@pytest.mark.parametrize("jt", JOINS)
def test_dev_equals_packed(capi, jt):
    rng = np.random.default_rng(23)
    left, right = split(rng, table(rng, LT, 400, (0,)), 3), split(rng, table(rng, RT, 300, (2,)), 2)
    packed, _ = check(capi, jt, left, right, LKEY, RKEY, LT, RT)
    dev, _ = check(capi, jt, left, right, LKEY, RKEY, LT, RT, dev=True)
    assert dev == packed
    t = capi.last_timing()
    assert t["dominant_launches"] > 0 and t["kernel_ms"] >= t["top_kernel_ms"] >= t["dominant_ms"] >= 0


# ---------------------------------------------------------------------------------------------------------------
# failures
# ---------------------------------------------------------------------------------------------------------------
def _bad(capi, left, right, lkeys=LKEY, rkeys=RKEY, alg=0):
    got, r = call(capi, INNER, left, right, lkeys, rkeys, LT, RT, alg=alg, cap=1 << 20)
    assert got == b"" and r["n_out_records"] == r["n_left_records"] == r["n_right_records"] == 0
    return r


@pytest.mark.parametrize("side", [0, 1])
def test_a_corrupt_or_short_row_fails_its_block(capi, side):
    rng = np.random.default_rng(29)
    left, right = split(rng, table(rng, LT, 100, (0,)), 2), split(rng, table(rng, RT, 100, (2,)), 2)
    blocks = [list(left), list(right)]
    good = blocks[side][1]
    blocks[side][1] = good + (1000).to_bytes(4, "big") + b"\0" * 8  # runs past the block end
    r = _bad(capi, *blocks)
    bad_block = len(left) * side + 1
    assert r["status"][bad_block] == capi.E_CORRUPT
    msg = capi.load().b2s_last_error().decode()
    assert ("block %d" % bad_block) in msg and ("byte %d" % len(good)) in msg
    blocks[side][1] = good + (8).to_bytes(4, "big") + b"\0" * 8  # a row shorter than its side's fixed region
    r = _bad(capi, *blocks)
    assert r["status"][bad_block] == capi.E_CORRUPT
    msg = capi.load().b2s_last_error().decode()
    assert ("block %d" % bad_block) in msg and ("byte %d" % len(good)) in msg and "fixed region" in msg


def test_checksum_mismatch_sets_bad_slice(capi):
    rng = np.random.default_rng(31)
    left, right = split(rng, table(rng, LT, 100, (0,)), 2), split(rng, table(rng, RT, 100, (2,)), 2)
    arena, off, ln, sb, sl, sc = build_blocks(capi, 1, 0, 3, left + right)
    sc = sc.copy()
    sc[2] ^= 1
    dst = np.zeros(1 << 20, np.uint8)
    r = capi.decompress_join_rows_keys_packed(INNER, 1, arena, off, ln, 2, dst, LKEY, RKEY, len(LT), len(RT),
                                              kinds(LT), kinds(RT), 3, sb, sl, sc)
    assert r["status"][2] == capi.E_CHECKSUM and r["bad_slice"][2] == 0
    assert r["n_out_records"] == 0 and r["total"] == 0


def test_dst_too_small_gives_the_bytes_needed(capi):
    rng = np.random.default_rng(37)
    left, right = split(rng, table(rng, LT, 300, (0,)), 2), split(rng, table(rng, RT, 200, (2,)), 2)
    want = model_join(INNER, left, right, LKEY, RKEY, len(LT), len(RT), kinds(LT), kinds(RT))[0]
    arena, off, ln, sb, sl, sc = build_blocks(capi, 1, 0, 0, left + right)
    dst = np.zeros(len(want), np.uint8)
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_join_rows_keys_packed(INNER, 1, arena, off, ln, 2, dst[:len(want) - 1], LKEY, RKEY, len(LT),
                                              len(RT), kinds(LT), kinds(RT))
    assert e.value.code == capi.E_DST_TOO_SMALL
    got, _ = call(capi, INNER, left, right, LKEY, RKEY, LT, RT, alg=0, cap=len(want))
    assert got == want


BAD_ARGS = {
    "join type": dict(jt=4),
    "n_left past n": dict(n_left=5),
    "order flag": dict(lkeys=[(2 | 256, 8, 8, 0)]),
    "key type": dict(lkeys=[(4, 8, 8, 0)], rkeys=[(4, 40, 8, 2)]),
    "left slot past the fields": dict(lkeys=[(2, 8 * 6, 8, 0)]),
    "right slot in the bitset": dict(rkeys=[(2, 0, 8, 2)]),
    "null bit past the fields": dict(rkeys=[(2, 32, 8, 4)]),
    "no fields": dict(nl=0),
    "too many fields": dict(nr=65537),
    "no kinds": dict(lk=None),
    "unknown kind": dict(rk=[0, 1, 3, 0]),
}


@pytest.mark.parametrize("case", list(BAD_ARGS))
def test_bad_arguments(capi, case):
    a = dict(jt=INNER, n_left=1, lkeys=LKEY, rkeys=RKEY, nl=len(LT), nr=len(RT), lk=kinds(LT), rk=kinds(RT))
    a.update(BAD_ARGS[case])
    rng = np.random.default_rng(41)
    left, right = split(rng, table(rng, LT, 20, (0,)), 1), split(rng, table(rng, RT, 20, (2,)), 1)
    arena, off, ln, _, _, _ = build_blocks(capi, 0, 0, 0, left + right)
    dst = np.zeros(1 << 16, np.uint8)
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_join_rows_keys_packed(a["jt"], 0, arena, off, ln, a["n_left"], dst, a["lkeys"], a["rkeys"],
                                              a["nl"], a["nr"], a["lk"], a["rk"])
    assert e.value.code == capi.E_ARG


def test_semi_and_anti_take_no_kinds(capi):
    rng = np.random.default_rng(43)
    left, right = split(rng, table(rng, LT, 100, (0,)), 2), split(rng, table(rng, RT, 100, (2,)), 2)
    for jt in (LEFT_SEMI, LEFT_ANTI):
        check(capi, jt, left, right, LKEY, RKEY, LT, RT)


# ---------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------
def _records(blocks):
    out = []
    for b in blocks:
        p = 0
        while p < len(b):
            s = int.from_bytes(b[p:p + 4], "big")
            out.append(bytes(b[p:p + 4 + s]))
            p += 4 + s
    return out


@pytest.mark.parametrize("jt", JOINS)
def test_hash_partitioned_tables_join_per_reducer(capi, jt):
    """two tables of different layouts hash-partitioned on the same key columns, each reducer joined on the GPU: the
    union of the reducers' outputs is the join of the whole tables"""
    rng = np.random.default_rng(47 + jt)
    lt, rt = ["string", "long", "int", "decimal"], ["int", "double", "long", "string"]
    lkeys, rkeys = keys_of(lt, [1, 2]), keys_of(rt, [2, 0])
    R, maps = 7, 3
    side_rows = [table(rng, lt, 900, (1, 2), key_range=6), table(rng, rt, 600, (2, 0), key_range=6)]
    side_keys = [lkeys, rkeys]
    per_reducer = [[[] for _ in range(R)], [[] for _ in range(R)]]  # side -> reducer -> [(block, checksum)]
    for s in range(2):
        for m in range(maps):
            rows = side_rows[s][m::maps]
            records, rec_len = records_of(rows)
            dst = np.zeros(2 * records.size + 4096 * R, np.uint8)
            r = capi.partition_compress_rows_hash_packed(1, records, rec_len, side_keys[s], R, dst, checksum_alg=3)
            for p in range(R):
                if r["dst_len"][p]:
                    o = int(r["dst_off"][p])
                    per_reducer[s][p].append((dst[o:o + int(r["dst_len"][p])].tobytes(), int(r["checksums"][p])))
    got = []
    nlk, nrk = kinds(lt), kinds(rt)
    for p in range(R):
        blocks = per_reducer[0][p] + per_reducer[1][p]
        data = [b for b, _ in blocks]
        if not data:
            continue
        lens = np.array([len(b) for b in data], np.uint64)
        off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        arena = np.frombuffer(b"".join(data), np.uint8)
        dst = np.zeros(1 << 22, np.uint8)
        r = capi.decompress_join_rows_keys_packed(jt, 1, arena, off, lens, len(per_reducer[0][p]), dst, lkeys, rkeys,
                                                  len(lt), len(rt), nlk, nrk, 3,
                                                  np.arange(len(data) + 1, dtype=np.uint32), lens,
                                                  np.array([c for _, c in blocks], np.uint64))
        assert (r["status"] == 0).all()
        got += _records([dst[:r["total"]].tobytes()])
    want = model_join(jt, blocks_of(side_rows[0], [900]), blocks_of(side_rows[1], [600]), lkeys, rkeys, len(lt),
                      len(rt), nlk, nrk)[0]
    assert sorted(got) == sorted(_records([want]))


# ---------------------------------------------------------------------------------------------------------------
# the host mirror
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_joins_two_shuffles_per_reducer(capi, tmp_path, codec):
    """two shuffles written by the mirror's serialized writer, each reducer's partitions of both joined in one read"""
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R = 3, 3
    rng = np.random.default_rng(53)
    sides = [(LT, LKEY, 400), (RT, RKEY, 300)]
    written = []
    for shuffle, (types, keys, n) in enumerate(sides):
        maps = []
        for m in range(M):
            rows = table(rng, types, n, (keys[0][1] // 8 - 1,))
            ids = rng.integers(0, R, n)
            w = host.S3SerializedShuffleWriter(d, shuffle, m, R)
            for r, p in zip(rows, ids):
                w.insertRecord(int(p), len(r).to_bytes(4, "big") + r)
            w.commit()
            w.close()
            maps.append((rows, ids))
        written.append(maps)
    for jt in JOINS:
        for red in range(R):
            plain = [[stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps] for maps in written]
            left = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
            right = host.S3ShuffleReader(d, 1, list(range(M)), red, red + 1)
            got = left.readJoinedRows(right, jt, LKEY, RKEY, len(LT), len(RT), kinds(LT), kinds(RT))
            left.close()
            right.close()
            want = model_join(jt, plain[0], plain[1], LKEY, RKEY, len(LT), len(RT), kinds(LT), kinds(RT))
            assert got == want
    d.close()
