"""Row sort and row aggregation by a composite key in any Spark sort order (b2s_decompress_sort_rows_keys_* /
b2s_decompress_aggregate_rows_keys_*): the order flags KEY_DESCENDING / KEY_NULLS_LAST per column, and the column types
INT16, INT8, FLOAT32, FLOAT64 and DECIMAL_KEY (a Decimal(p > 18)'s big-endian bytes behind a slot).

The model does not restate the GPU's byte encoding.  It compares records column by column with a comparator: the null
ordering first, then the value, reversed for DESC; floats in Spark SQL's order (rows_model.dkey: -0.0 == 0.0, NaN above
everything), decimals as signed integers, strings as Python bytes.  It sorts stably and groups the records that compare
equal; every output must equal it byte for byte."""
import functools
import struct

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from rows_model import CHECKSUMS, CODECS, KEY_BYTES, KEY_INT32, KEY_INT64, MIN_I64, STRING, SUM_I64, blocks_of, \
    build_blocks, dkey, is_null, merge, mirror, parse, run, stream, write_maps

pytestmark = pytest.mark.gpu

KEY_INT16, KEY_INT8, KEY_FLOAT32, KEY_FLOAT64, DECIMAL = 5, 6, 7, 8, 9
DESC, NULLS_LAST = 1 << 8, 1 << 9
FLAGS = [0, DESC, NULLS_LAST, DESC | NULLS_LAST]
KLEN = {KEY_INT8: 1, KEY_INT16: 2, KEY_INT32: 4, KEY_INT64: 8, KEY_FLOAT32: 4, KEY_FLOAT64: 8, STRING: 8, DECIMAL: 8}


# ---------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------
def col_value(row, col):
    """one key column of a row -> None (null) or a value whose Python order and equality are the column's ascending
    order and equality"""
    kt, ko, kl, nf = col
    t = kt & 0xFF
    if nf >= 0 and is_null(row, nf):
        return None
    if t in (STRING, DECIMAL):
        slot = int.from_bytes(row[ko:ko + 8], "little")
        b = bytes(row[slot >> 32:(slot >> 32) + (slot & 0xFFFFFFFF)])
        return b if t == STRING else int.from_bytes(b, "big", signed=True)
    k = bytes(row[ko:ko + kl])
    if t == KEY_BYTES:
        return k
    if t == KEY_FLOAT64:
        return dkey(k)
    if t == KEY_FLOAT32:  # widening to double keeps the value, the sign of a zero and NaN-ness
        return dkey(struct.pack("<d", struct.unpack("<f", k)[0]))
    return int.from_bytes(k, "little", signed=True)


def comparator(keys):
    def cmp(a, b):
        for (kt, _, _, _), x, y in zip(keys, a, b):
            if x is None or y is None:
                if x is None and y is None:
                    continue
                c = -1 if x is None else 1
                return -c if kt & NULLS_LAST else c
            if x != y:
                c = -1 if x < y else 1
                return -c if kt & DESC else c
        return 0
    return cmp


def model(plain, keys):
    """-> (decoded bytes, records [(offset, length)], the sorted record indices split into groups)"""
    buf = b"".join(plain)
    recs = parse(buf)
    kv = [tuple(col_value(buf[o + 4:o + ln], c) for c in keys) for o, ln in recs]
    cmp = comparator(keys)
    order = sorted(range(len(recs)), key=functools.cmp_to_key(lambda i, j: cmp(kv[i], kv[j])))  # stable
    groups = []
    for i in order:
        if groups and cmp(kv[groups[-1][0]], kv[i]) == 0:
            groups[-1].append(i)
        else:
            groups.append([i])
    return buf, recs, groups


def model_sort(plain, keys):
    buf, recs, groups = model(plain, keys)
    return b"".join(buf[recs[i][0]:recs[i][0] + recs[i][1]] for g in groups for i in g), len(recs)


def model_aggregate(plain, keys, aggs):
    """each group's first record with every aggregate (op, off, null field) merged over the group in stable order"""
    buf, recs, groups = model(plain, keys)
    out = []
    for g in groups:
        o, ln = recs[g[0]]
        rec = bytearray(buf[o:o + ln])
        row = memoryview(rec)[4:]
        nulls = []
        for op, off, anf in aggs:
            vals = [bytes(buf[recs[i][0] + 4 + off:recs[i][0] + 12 + off]) for i in g
                    if not is_null(buf[recs[i][0] + 4:recs[i][0] + recs[i][1]], anf)]
            row[off:off + 8] = merge(op, vals) if vals else bytes(8)
            nulls.append((anf, not vals))
        for anf, null in nulls:
            if anf >= 0:
                w = 8 * (anf >> 6)
                v = int.from_bytes(row[w:w + 8], "little")
                v = v | (1 << (anf & 63)) if null else v & ~(1 << (anf & 63))
                row[w:w + 8] = v.to_bytes(8, "little")
        out.append(bytes(rec))
    return b"".join(out), len(recs), len(out)


# ---------------------------------------------------------------------------------------------------------------
# rows: one null word, a 16-byte area per key column, 8-byte aggregate slots, then strings and decimals
# ---------------------------------------------------------------------------------------------------------------
def layout(types, flags=None, nullable=True, byte_len=10):
    """-> key columns [(type | flags, off, len, null field)]; column c at 8 + 16 c, null bit c + 1"""
    flags = flags or [0] * len(types)
    return [(t | f, 8 + 16 * c, KLEN.get(t, byte_len), c + 1 if nullable else -1)
            for c, (t, f) in enumerate(zip(types, flags))]


def agg_layout(keys, ops):
    base = 8 + 16 * len(keys)
    return [(op, base + 8 * a, 20 + a) for a, op in enumerate(ops)]


def dec_bytes(v, size=None):
    """BigInteger.toByteArray: the shortest big-endian two's complement (or size bytes, sign-extended)"""
    n = (v if v >= 0 else ~v).bit_length() // 8 + 1
    return v.to_bytes(size or n, "big", signed=True)


def make_row(rng, keys, vals, aggs=(), agg_vals=(), agg_nulls=(), tail=0):
    """vals[c]: None for null; an int (ints), raw little-endian bytes (floats, KEY_BYTES), bytes (strings) or an int
    or (int, size) (decimals); strings and decimals go after the fixed region, 8-byte aligned"""
    fixed = 8 + 16 * len(keys) + 8 * len(aggs)
    r = bytearray(rng.integers(0, 256, fixed, dtype=np.uint8).tobytes())
    word = int(rng.integers(0, 2**63)) & ~((1 << 40) - 2)  # bits 1..39 (key and aggregate null bits) clear
    var = bytearray()
    for (kt, ko, kl, nf), v in zip(keys, vals):
        t = kt & 0xFF
        if v is None:
            word |= 1 << nf
            continue
        if t in (STRING, DECIMAL):
            b = v if t == STRING else dec_bytes(*v) if isinstance(v, tuple) else dec_bytes(v)
            o = fixed + len(var)
            var += b + bytes(-len(b) % 8)
            r[ko:ko + 8] = ((o << 32) | len(b)).to_bytes(8, "little")
        elif isinstance(v, bytes):
            r[ko:ko + kl] = v
        else:
            r[ko:ko + kl] = int(v).to_bytes(kl, "little", signed=True)
    for (op, off, anf), v, null in zip(aggs, agg_vals, agg_nulls):
        r[off:off + 8] = (int(v) % 2**64).to_bytes(8, "little")
        if null and anf >= 0:
            word |= 1 << anf
    r[0:8] = word.to_bytes(8, "little")
    return bytes(r + var + rng.integers(0, 256, tail, dtype=np.uint8).tobytes())


F32 = [0x7F800000, 0xFF800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF,
       0x3FC00000, 0xBFC00000, 0x3F800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FFFFFFF]
F64 = [0x7FF0000000000000, 0xFFF0000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 0, 1 << 63, 1, (1 << 63) | 1,
       0x000FFFFFFFFFFFFF, 0x3FF8000000000000, 0xBFF8000000000000, 0x3FF0000000000000, 0x7FF8000000000000,
       0xFFF8000000000000, 0x7FF0000000000001, 0xFFF0000000000001, 0x7FFFFFFFFFFFFFFF]
DEC_EDGES = [10**38 - 1, -(10**38 - 1), -1, 0, 1, 127, 128, -128, -129, 255, 256, 2**63, -2**63, 2**64 - 1, 2**119,
             -2**127, 2**127 - 1] + [(1 << (8 * s - 1)) - 1 for s in range(1, 17)] + [-(1 << (8 * s - 1))
                                                                                       for s in range(1, 17)]
EDGES = {
    KEY_INT8: [-128, 127, -1, 0, 1],
    KEY_INT16: [-32768, 32767, -1, 0, 1, 255, 256, -256],
    KEY_INT32: [-2**31, 2**31 - 1, -1, 0, 1],
    KEY_INT64: [-2**63, 2**63 - 1, -1, 0, 1],
    KEY_FLOAT32: [x.to_bytes(4, "little") for x in F32],
    KEY_FLOAT64: [x.to_bytes(8, "little") for x in F64],
    DECIMAL: DEC_EDGES + [(0, 16), (-1, 16), (5, 9), (-5, 3)],  # padded, as a size the shortest form would not take
}
PREFIXES = [b"", b"ab", b"category#", b"\x00\x00\x00", b"\xff" * 12, b"Books/Fiction/" * 3]


def rand_value(rng, kt, byte_len=10):
    t = kt & 0xFF
    if t == STRING:
        pre = PREFIXES[int(rng.integers(len(PREFIXES)))]
        return pre + rng.integers(0, 256, int(rng.integers(0, 12)), dtype=np.uint8).tobytes()
    if t == KEY_BYTES:
        return bytes(int(rng.integers(0, 3)) for _ in range(byte_len))
    if t == DECIMAL and rng.random() < 0.5:
        return int(rng.integers(-3, 3)) * 10**int(rng.integers(0, 37))
    e = EDGES[t]
    return e[int(rng.integers(len(e)))]


def rand_rows(rng, n, keys, null_frac=0.15, aggs=()):
    rows = []
    for _ in range(n):
        vals = [None if (c[3] >= 0 and rng.random() < null_frac) else rand_value(rng, c[0], c[2]) for c in keys]
        av = [int(x) for x in rng.integers(-1000, 1000, len(aggs))]
        an = [rng.random() < 0.2 for _ in aggs]
        rows.append(make_row(rng, keys, vals, aggs, av, an, int(rng.integers(0, 20))))
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


BOOL = (KEY_BYTES, 1)
ALL = [STRING, KEY_INT16, KEY_FLOAT64, DECIMAL, KEY_INT8, KEY_FLOAT32, BOOL, KEY_INT32, KEY_INT64, KEY_BYTES]


def mixed_layout(rng):
    types = [t[0] if isinstance(t, tuple) else t for t in ALL]
    keys = layout(types, [FLAGS[int(rng.integers(4))] for _ in types])
    keys[ALL.index(BOOL)] = keys[ALL.index(BOOL)][:2] + (1,) + keys[ALL.index(BOOL)][3:]
    return keys


def bool_rows(rng, keys, rows):
    """BooleanType: KEY_BYTES of length 1 holding 0 / 1"""
    c = ALL.index(BOOL)
    ko = keys[c][1]
    out = []
    for r in rows:
        r = bytearray(r)
        r[ko] = int(rng.integers(0, 2))
        out.append(bytes(r))
    return out


# ---------------------------------------------------------------------------------------------------------------
# 1. every codec x checksum, packed and _dev: every type, random flags per column
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", CHECKSUMS)
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_every_type_and_flag_like_the_model(capi, name, codec, level, alg):
    rng = np.random.default_rng(100 + codec * 10 + alg)
    keys = mixed_layout(rng)
    aggs = agg_layout(keys, [SUM_I64, MIN_I64])
    rows = bool_rows(rng, keys, rand_rows(rng, 2500, keys, aggs=aggs))
    plain = blocks_of(rows, [800, 0, 1000, 700])
    blocks = build_blocks(capi, codec, level, alg, plain)
    dev = alg % 2 == 1
    check_sort(capi, plain, keys, codec, level, alg, dev, blocks)
    check_agg(capi, plain, keys, aggs, codec, level, alg, not dev, blocks)


def test_every_type_with_few_distinct_values_groups_like_the_model(capi):
    """the leading columns take few values, so the later ones decide inside long ties"""
    rng = np.random.default_rng(101)
    types = [KEY_INT8, KEY_FLOAT32, DECIMAL, KEY_INT16, KEY_FLOAT64, STRING]
    keys = layout(types, [DESC, NULLS_LAST, DESC | NULLS_LAST, DESC, 0, DESC])
    rows = []
    for _ in range(3000):
        vals = [None if rng.random() < 0.2 else v for v in (
            int(rng.integers(-1, 2)), [b"\0\0\0\0", b"\0\0\0\x80", b"\0\0\xc0\x7f"][int(rng.integers(3))],
            [(0, 1), (0, 16), (-1, 1), (-1, 16)][int(rng.integers(4))], int(rng.integers(-2, 2)),
            F64[int(rng.integers(len(F64)))].to_bytes(8, "little"), [b"", b"a", b"ab"][int(rng.integers(3))])]
        rows.append(make_row(rng, keys, vals))
    plain = blocks_of(rows, [1500, 1500])
    check_sort(capi, plain, keys, dev=True)
    check_agg(capi, plain, keys, [])


# ---------------------------------------------------------------------------------------------------------------
# 2. each new type alone, every direction x null ordering, on its edge values
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("kt", [KEY_INT16, KEY_INT8, KEY_FLOAT32, KEY_FLOAT64, DECIMAL])
def test_each_type_alone_on_its_edge_values(capi, kt, flags):
    rng = np.random.default_rng(kt * 4 + flags // 256)
    keys = layout([kt], [flags])
    aggs = agg_layout(keys, [SUM_I64])
    vals = (EDGES[kt] + [None]) * 6
    rows = [make_row(rng, keys, [v], aggs, [i], [False], int(rng.integers(0, 9))) for i, v in enumerate(vals)]
    rng.shuffle(rows)
    plain = blocks_of(rows, [len(rows) // 3, len(rows) - len(rows) // 3])
    check_sort(capi, plain, keys)
    _, r = check_agg(capi, plain, keys, aggs, dev=True)
    if kt in (KEY_FLOAT32, KEY_FLOAT64):  # -0.0 with 0.0, every NaN one group; the rest distinct; the nulls
        assert r["n_groups"] == len(EDGES[kt]) - 1 - 4 + 1
    # the same key without a null bit: NULLS_LAST changes nothing
    keys = [keys[0][:3] + (-1,)]
    rows = [make_row(rng, keys, [v]) for v in EDGES[kt] * 3]
    rng.shuffle(rows)
    check_sort(capi, blocks_of(rows, [len(rows)]), keys, dev=True)


# ---------------------------------------------------------------------------------------------------------------
# 3. DESC strings: prefixes after their extensions, empty against null, differences past the first pass
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [DESC, DESC | NULLS_LAST])
@pytest.mark.parametrize("lead", [None, KEY_INT64, DECIMAL])
def test_desc_strings_with_shared_prefixes(capi, flags, lead):
    rng = np.random.default_rng(7 + flags // 256 + (lead or 0))
    types = ([lead] if lead else []) + [STRING, KEY_INT32]
    keys = layout(types, ([DESC] if lead else []) + [flags, 0])
    aggs = agg_layout(keys, [SUM_I64])
    long = b"Books/Fiction/Classics#"  # 23 bytes: a difference in its last bytes lies past the first pass
    strs = [None, b"", b"a", b"ab", b"abc", b"ab\x00", b"abcdefgh", b"abcdefghi", b"\xff", b"\xff\xff", long,
            long + b"\x00", long[:-1], long[:-1] + b"$", long + b"A" * 9, long + b"A" * 8]
    rows = []
    for i in range(6 * len(strs)):
        s = strs[i % len(strs)]
        vals = ([[3, 7][i % 2] if lead != DECIMAL else [3, 7][i % 2] * 10**30] if lead else []) + [s, i % 3 - 1]
        rows.append(make_row(rng, keys, vals, aggs, [i], [False]))
    rng.shuffle(rows)
    plain = blocks_of(rows, [len(rows) // 2, len(rows) - len(rows) // 2])
    got = check_sort(capi, plain, keys)
    check_agg(capi, plain, keys, aggs, dev=True)
    if not lead:  # "abc" before "ab" before "a" before "" (before null unless NULLS_LAST)
        firsts = []
        for o, ln in parse(got):
            s = col_value(got[o + 4:o + ln], keys[0])
            if s in (b"", b"a", b"ab", b"abc") and s not in firsts:
                firsts.append(s)
        assert firsts == [b"abc", b"ab", b"a", b""]


# ---------------------------------------------------------------------------------------------------------------
# 4. without a model: every column flipped (direction and null ordering) gives the groups in reverse, each stable
# ---------------------------------------------------------------------------------------------------------------
def runs(data, heads):
    """data's records cut before every record of heads (in order)"""
    recs = [data[o:o + ln] for o, ln in parse(data)]
    out, h = [], 0
    for r in recs:
        if h < len(heads) and r == heads[h]:
            out.append([])
            h += 1
        out[-1].append(r)
    assert h == len(heads)
    return out


def test_flipping_every_column_reverses_the_groups(capi):
    rng = np.random.default_rng(44)
    keys = mixed_layout(rng)
    rows = bool_rows(rng, keys, rand_rows(rng, 3000, keys, null_frac=0.3))
    rows = [r + i.to_bytes(4, "little") for i, r in enumerate(rows)]  # every record distinct
    plain = blocks_of(rows, [1000, 2000])
    blocks = build_blocks(capi, 3, 1, 3, plain)
    total = sum(len(b) for b in plain)
    flipped = [(k[0] ^ DESC ^ NULLS_LAST,) + k[1:] for k in keys]
    outs = []
    for ks in (keys, flipped):
        data, _ = run(capi, "decompress_sort_rows_keys", 3, 3, blocks, (ks,), total)
        heads, r = run(capi, "decompress_aggregate_rows_keys", 3, 3, blocks, (ks, []), total)
        outs.append(runs(data, [heads[o:o + ln] for o, ln in parse(heads)]))
    assert len(outs[0]) > 100
    assert outs[1] == outs[0][::-1]


# ---------------------------------------------------------------------------------------------------------------
# 5. aggregation on FLOAT64 keys: 0.0 / -0.0 and all NaNs merge, the first record's exact bits stay
# ---------------------------------------------------------------------------------------------------------------
def test_float64_keys_merge_zeros_and_nans(capi):
    rng = np.random.default_rng(55)
    keys = layout([KEY_FLOAT64])
    aggs = agg_layout(keys, [SUM_I64])
    zeros = [x.to_bytes(8, "little") for x in (1 << 63, 0)]
    nans = [x.to_bytes(8, "little") for x in (0xFFF0000000000001, 0x7FF8000000000000, 0x7FF0000000000001,
                                              0xFFFFFFFFFFFFFFFF, 0x7FF00000DEADBEEF)]
    vals = [zeros[i % 2] if i % 3 == 0 else nans[i % 5] if i % 3 == 1 else struct.pack("<d", 1.5)
            for i in range(600)]
    rows = [make_row(rng, keys, [v], aggs, [1], [False]) for v in vals]
    plain = blocks_of(rows, [200, 400])
    got, r = check_agg(capi, plain, keys, aggs)
    assert r["n_groups"] == 3
    out = [got[o:o + ln] for o, ln in parse(got)]
    assert [o[4 + 8:4 + 16] for o in out] == [zeros[0], struct.pack("<d", 1.5), nans[1]]  # first in stable order
    assert [int.from_bytes(o[4 + 24:4 + 32], "little") for o in out] == [200, 200, 200]
    got, r = check_agg(capi, plain, [(KEY_FLOAT64 | DESC,) + keys[0][1:]], aggs, dev=True)
    assert [o[4 + 8:4 + 16] for o in (got[a:a + b] for a, b in parse(got))] == [nans[1], struct.pack("<d", 1.5),
                                                                                   zeros[0]]


# ---------------------------------------------------------------------------------------------------------------
# 6. TPC-DS q67's window sort: (i_category ASC NULLS FIRST, sumsales decimal(28,2) DESC NULLS LAST) over many maps
# ---------------------------------------------------------------------------------------------------------------
def test_q67_window_key_over_many_maps(capi):
    rng = np.random.default_rng(67)
    keys = [(STRING, 8, 8, 1), (DECIMAL | DESC | NULLS_LAST, 24, 8, 2)]
    cats = [b"Books", b"Children", b"Electronics", b"Home", b"Jewelry", b"Men", b"Music", b"Shoes", b"Sports",
            b"Women", None]
    rows = []
    for _ in range(8000):
        cat = cats[int(rng.integers(len(cats)))]
        sales = None if rng.random() < 0.05 else int(rng.integers(-10**6, 10**12)) * [1, 1, 10**9][int(rng.integers(3))]
        if sales is not None and rng.random() < 0.02:
            sales = [10**27 - 1, -(10**27 - 1), 0][int(rng.integers(3))]
        rows.append(make_row(rng, [(STRING, 8, 8, 1), (DECIMAL, 24, 8, 2)], [cat, sales], tail=int(rng.integers(0, 40))))
    plain = blocks_of(rows, [int(x) for x in np.diff(np.linspace(0, 8000, 41).astype(int))])
    check_sort(capi, plain, keys, codec=2, alg=3)
    check_agg(capi, plain, keys, [], codec=2, alg=3, dev=True)


# ---------------------------------------------------------------------------------------------------------------
# 7. corrupt decimal slots; a null decimal's slot is never read
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", ["size0", "size17", "past_row"])
@pytest.mark.parametrize("types", [[DECIMAL], [KEY_INT64, DECIMAL]], ids=["fits_first_pass", "refines"])
def test_bad_decimal_slot_fails_the_block(capi, bad, types):
    rng = np.random.default_rng(70)
    keys = layout(types, [DESC] * len(types))
    good = rand_rows(rng, 300, keys)
    vals = [3] * (len(types) - 1) + [12345]
    bad_row = bytearray(make_row(rng, keys, vals))
    so = keys[-1][1]
    slot = int.from_bytes(bad_row[so:so + 8], "little")
    slot = {"size0": slot & ~0xFFFFFFFF, "size17": (slot & ~0xFFFFFFFF) | 17,
            "past_row": ((len(bad_row) - 3) << 32) | 4}[bad]
    bad_row[so:so + 8] = slot.to_bytes(8, "little")
    blocks_rows = [good[:100], good[100:180] + [bytes(bad_row)] + good[180:]]
    plain = [stream(b) for b in blocks_rows]
    at = sum(4 + len(r) for r in good[100:180])
    total = sum(len(b) for b in plain)
    blocks = build_blocks(capi, 1, 0, 2, plain)
    for aggregate in (False, True):
        got, r = (run(capi, "decompress_aggregate_rows_keys", 1, 2, blocks, (keys, []), total, aggregate) if aggregate
                  else run(capi, "decompress_sort_rows_keys", 1, 2, blocks, (keys,), total))
        assert list(r["status"]) == [0, capi.E_CORRUPT]
        assert r["n_records"] == 0 and got == b""
        err = capi.load().b2s_last_error().decode()
        assert "block 1" in err and "byte %d" % at in err and "decimal" in err, err


def test_null_decimal_with_a_garbage_slot_is_fine(capi):
    rng = np.random.default_rng(71)
    keys = layout([DECIMAL], [NULLS_LAST])
    rows = [bytearray(make_row(rng, keys, [None])) for _ in range(10)]
    for r in rows:
        r[8:16] = (2**63 + 12345).to_bytes(8, "little")  # never read: the decimal is null
    rows = [bytes(r) for r in rows] + [make_row(rng, keys, [v]) for v in (5, -5, 0)]
    check_sort(capi, blocks_of(rows, [13]), keys)
    check_agg(capi, blocks_of(rows, [13]), keys, [])


# ---------------------------------------------------------------------------------------------------------------
# 8. argument errors
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keys,aggs", [
    ([(KEY_INT32 | (1 << 10), 8, 4, -1)], []),
    ([(KEY_INT32 | (1 << 31), 8, 4, -1)], []),
    ([(STRING | DESC | (1 << 12), 8, 8, 1)], []),
    ([(KEY_INT16, 8, 4, -1)], []),
    ([(KEY_INT8, 8, 2, -1)], []),
    ([(KEY_FLOAT32, 8, 8, -1)], []),
    ([(KEY_FLOAT64, 8, 4, -1)], []),
    ([(DECIMAL, 8, 16, -1)], []),
    ([(DECIMAL | DESC, 8, 4, -1)], []),
    ([(10, 8, 8, -1)], []),
    ([(KEY_INT32, 8, 4, -1), (DECIMAL, 24, 8, 1)], [(SUM_I64, 28, -1)]),  # overlaps the decimal slot
])
def test_bad_arguments(capi, keys, aggs):
    rng = np.random.default_rng(80)
    rows = [make_row(rng, layout([KEY_INT32]), [1]) + bytes(64)]
    blocks = build_blocks(capi, 0, 0, 0, blocks_of(rows, [1]))
    for aggregate in ([True] if aggs else [False, True]):
        with pytest.raises(capi.B2SError) as e:
            if aggregate:
                run(capi, "decompress_aggregate_rows_keys", 0, 0, blocks, (keys, aggs), 4096)
            else:
                run(capi, "decompress_sort_rows_keys", 0, 0, blocks, (keys,), 4096)
        assert e.value.code == capi.E_ARG


@pytest.mark.parametrize("kt,kl", [(KEY_INT32 | DESC, 4), (KEY_INT64 | NULLS_LAST, 8), (KEY_INT16, 2), (KEY_INT8, 1),
                                   (KEY_FLOAT32, 4), (KEY_FLOAT64, 8), (DECIMAL, 8)])
def test_single_key_calls_reject_flags_and_new_types(capi, kt, kl):
    rng = np.random.default_rng(81)
    rows = [make_row(rng, layout([KEY_INT64]), [1])]
    arena, off, ln, sb, sl, sc = build_blocks(capi, 0, 0, 0, blocks_of(rows, [1]))
    dst = np.zeros(4096, np.uint8)
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_sort_rows_packed(0, arena, off, ln, dst, kt, 8, kl, 1)
    assert e.value.code == capi.E_ARG
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_aggregate_rows_packed(0, arena, off, ln, dst, kt, 8, kl, 1, [])
    assert e.value.code == capi.E_ARG


def test_flagged_one_column_key_equals_the_unflagged_sort_reversed_by_groups(capi):
    """an unflagged one-column call still gives the single-key call's bytes; DESC NULLS LAST gives its groups
    reversed"""
    rng = np.random.default_rng(82)
    keys = [(KEY_INT32, 8, 4, 1)]
    rows = [make_row(rng, keys, [None if i % 7 == 0 else int(rng.integers(-20, 20))]) + i.to_bytes(4, "little")
            for i in range(2000)]
    plain = blocks_of(rows, [2000])
    blocks = build_blocks(capi, 1, 0, 3, plain)
    arena, off, ln, sb, sl, sc = blocks
    total = sum(len(b) for b in plain)
    want = np.zeros(total, np.uint8)
    capi.decompress_sort_rows_packed(1, arena, off, ln, want, KEY_INT32, 8, 4, 1, 3, sb, sl, sc)
    got, _ = run(capi, "decompress_sort_rows_keys", 1, 3, blocks, (keys,), total)
    assert got == want.tobytes()
    check_sort(capi, plain, [(KEY_INT32 | DESC | NULLS_LAST, 8, 4, 1)], blocks=blocks, alg=3)


# ---------------------------------------------------------------------------------------------------------------
# 9. the host mirror: readSortedRowsKeys / readAggregatedRowsKeys with flagged keys over the serialized writer's files
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_reads_rows_in_any_order(capi, tmp_path, codec):
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R, per_map = 3, 2, 1200
    keys = layout([STRING, DECIMAL, KEY_FLOAT64, KEY_INT16], [0, DESC | NULLS_LAST, DESC, NULLS_LAST])
    aggs = agg_layout(keys, [SUM_I64, MIN_I64])
    maps = []
    for m in range(M):
        rng = np.random.default_rng(190 + m)
        maps.append((rand_rows(rng, per_map, keys, aggs=aggs), rng.integers(0, R, per_map)))
    write_maps(host, d, maps, R)
    for red in range(R):
        plain = [stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps]
        rd = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        data, n = rd.readSortedRowsKeys(keys)
        want, wn = model_sort(plain, keys)
        assert n == wn and data == want
        data, n, g = rd.readAggregatedRowsKeys(keys, aggs)
        rd.close()
        want, wn, wg = model_aggregate(plain, keys, aggs)
        assert (n, g) == (wn, wg) and data == want
    d.close()
