"""Ranking windows over a reducer's UnsafeRows on the GPU (b2s_decompress_window_rows_keys_*): every output byte is
compared with tests/window_model.py, with the input and output record counts and status[]."""
import struct

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from join_model import DECIMAL_WIDE, FIXED, VAR
from rows_model import CODECS, KEY_INT32, KEY_INT64, STRING, blocks_of, build_blocks, mirror, run, stream
from test_gpu_sort_rows_order import DEC_EDGES, DECIMAL, DESC, F32, F64, KEY_FLOAT32, KEY_FLOAT64, KLEN, NULLS_LAST, \
    dec_bytes
from window_model import CUME_DIST, DENSE_RANK, NTILE, PERCENT_RANK, RANK, ROW_NUMBER, model_window

pytestmark = pytest.mark.gpu

ALL6 = [ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK, CUME_DIST, (NTILE, 3)]
KIND_OF = {STRING: VAR, DECIMAL: DECIMAL_WIDE}


# ---------------------------------------------------------------------------------------------------------------
# rows: n_fields 8-byte fields after ceil(n_fields / 64) null words; key column c in field fields[c], its null bit that
# field's ordinal; strings, decimals and the other VAR / DECIMAL_WIDE fields' bytes after the fixed region
# ---------------------------------------------------------------------------------------------------------------
class Schema:
    def __init__(self, n_fields, cols, extra_kinds=None):
        """cols: [(type | flags, field, nullable)]; extra_kinds: {field: VAR or DECIMAL_WIDE} of non-key fields"""
        self.nf, self.bw = n_fields, (n_fields + 63) // 64
        self.cols = cols
        self.kinds = [FIXED] * n_fields
        for t, f, _ in cols:
            self.kinds[f] = KIND_OF.get(t & 0xFF, FIXED)
        for f, k in (extra_kinds or {}).items():
            if f not in [c[1] for c in cols]:
                self.kinds[f] = k
        self.keys = [(t, 8 * (self.bw + f), KLEN[t & 0xFF], f if nullable else -1) for t, f, nullable in cols]

    def row(self, rng, vals):
        """vals[c]: None (null), an int, raw little-endian float bytes, bytes (strings) or an int (decimals)"""
        fixed = 8 * (self.bw + self.nf)
        r = bytearray(rng.integers(0, 256, fixed, dtype=np.uint8).tobytes())
        bits = int(rng.integers(0, 2**62)) if self.nf > 1 else 0
        var = bytearray()
        by_field = {f: (t, v) for (t, f, _), v in zip(self.cols, vals)}
        for f in range(self.nf):
            bits &= ~(1 << f)
            t, v = by_field.get(f, (None, b"x" * int(rng.integers(0, 20)) if self.kinds[f] == VAR else
                                    int(rng.integers(-10**15, 10**15)) * 10**12 if self.kinds[f] == DECIMAL_WIDE else 0))
            s = 8 * (self.bw + f)
            if v is None or (t is None and self.kinds[f] != FIXED and rng.random() < 0.1):
                bits |= 1 << f
                r[s:s + 8] = bytes(8)  # UnsafeRowWriter.setNullAt
                continue
            if t is None and self.kinds[f] == FIXED:
                continue
            tt = (t or 0) & 0xFF
            if self.kinds[f] == VAR or tt == STRING:
                b = bytes(v)
            elif self.kinds[f] == DECIMAL_WIDE:
                b = dec_bytes(v)
            else:
                r[s:s + KLEN[tt]] = v if isinstance(v, bytes) else int(v).to_bytes(KLEN[tt], "little", signed=True)
                continue
            o = fixed + len(var)
            var += b + bytes(-len(b) % 8 if self.kinds[f] == VAR else 16 - len(b))
            r[s:s + 8] = ((o << 32) | len(b)).to_bytes(8, "little")
        words = bits & ((1 << self.nf) - 1) | (int(rng.integers(0, 2**62)) << self.nf if self.nf % 64 else 0)
        r[0:8 * self.bw] = (words % (1 << (64 * self.bw))).to_bytes(8 * self.bw, "little")
        return bytes(r + var)


def small_value(rng, t, domain):
    t &= 0xFF
    if t == STRING:
        return b"category#" * int(rng.integers(0, 2)) + bytes([65 + int(rng.integers(domain))])
    if t == KEY_FLOAT64:
        return struct.pack("<d", float(rng.integers(domain)) - domain / 2)
    if t == KEY_FLOAT32:
        return struct.pack("<f", float(rng.integers(domain)) - domain / 2)
    if t == DECIMAL:
        return (int(rng.integers(domain)) - domain // 2) * 10**20
    return int(rng.integers(domain)) - domain // 2


def table(rng, schema, n, domain=5, null_frac=0.1, value=small_value):
    rows = []
    for _ in range(n):
        vals = [None if nullable and rng.random() < null_frac else value(rng, t, domain) for t, _, nullable in
                schema.cols]
        rows.append(schema.row(rng, vals))
    return rows


def call(capi, plain, schema, npk, fns, limit=None, codec=1, level=0, alg=0, dev=False, cap=None):
    blocks = build_blocks(capi, codec, level, alg, plain)
    want, n, m = model_window(plain, schema.keys, npk, schema.nf, schema.kinds, fns, limit)
    got, r = run(capi, "decompress_window_rows_keys", codec, alg, blocks,
                 (schema.keys, npk, schema.nf, schema.kinds, fns, limit), len(want) if cap is None else cap, dev)
    return got, r, (want, n, m)


def check(capi, plain, schema, npk, fns, limit=None, **kw):
    got, r, (want, n, m) = call(capi, plain, schema, npk, fns, limit, **kw)
    assert (r["status"] == 0).all(), r["status"]
    assert (r["n_records"], r["n_out_records"], r["total"]) == (n, m, len(want))
    assert got == want
    return r


# ---------------------------------------------------------------------------------------------------------------
# 1. every codec x {no checksum, CRC32C}; each function alone with 0, 1 and 3 partition columns
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", [0, 3])
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_every_codec_and_checksum(capi, name, codec, level, alg):
    rng = np.random.default_rng(10 + codec * 4 + level + alg)
    s = Schema(6, [(STRING, 0, True), (KEY_INT64 | DESC, 2, True), (KEY_INT32, 4, False)])
    rows = table(rng, s, 3000, domain=6)
    check(capi, blocks_of(rows, [1000, 0, 1200, 800]), s, 1, ALL6, codec=codec, level=level, alg=alg)


@pytest.mark.parametrize("npk", [0, 1, 3])
@pytest.mark.parametrize("fn", [ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK, CUME_DIST, (NTILE, 1), (NTILE, 4),
                                (NTILE, 1000)])
def test_each_function_alone(capi, fn, npk):
    rng = np.random.default_rng(20 + npk)
    s = Schema(5, [(KEY_INT32, 0, True), (STRING, 1, True), (KEY_INT64, 2, False), (KEY_INT64 | NULLS_LAST, 3, True)])
    rows = table(rng, s, 2000, domain=4)
    check(capi, blocks_of(rows, [700, 1300]), s, npk, [fn])


def test_all_six_and_repeats_in_one_call(capi):
    rng = np.random.default_rng(29)
    s = Schema(4, [(KEY_INT32, 1, True), (KEY_INT64 | DESC | NULLS_LAST, 3, True)])
    rows = table(rng, s, 2500, domain=7)
    check(capi, blocks_of(rows, [2500]), s, 1, ALL6 + [(NTILE, 7), RANK, (NTILE, 1)])


# ---------------------------------------------------------------------------------------------------------------
# 2. key shapes: long shared string prefixes, order flags, nulls, floats, decimals
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("npk", [1, 3])
def test_string_partition_keys_sharing_30_byte_prefixes(capi, npk):
    """partitions that differ only past the first 20 encoded bytes: heads found by comparing further windows"""
    rng = np.random.default_rng(31 + npk)
    pre = b"Books/Fiction/Classics/Longer"  # 29 bytes, then the byte that differs
    assert len(pre) + 1 == 30

    def value(rng, t, domain):
        if t & 0xFF == STRING:
            return pre + bytes([65 + int(rng.integers(3))]) + (b"tail" if rng.random() < 0.5 else b"")
        return small_value(rng, t, domain)

    cols = [(STRING, 0, True), (STRING, 1, False), (KEY_INT32, 2, True), (KEY_INT64 | DESC, 3, True)]
    s = Schema(4, cols[:npk] + cols[3:] if npk == 1 else cols)
    rows = table(rng, s, 2000, domain=3, value=value)
    check(capi, blocks_of(rows, [900, 1100]), s, npk, ALL6)


@pytest.mark.parametrize("flags", [DESC, NULLS_LAST, DESC | NULLS_LAST])
def test_desc_and_nulls_last_order_columns_with_null_peers(capi, flags):
    rng = np.random.default_rng(40 + flags)
    s = Schema(3, [(KEY_INT32, 0, False), (KEY_INT64 | flags, 1, True), (STRING | flags, 2, True)])
    rows = table(rng, s, 2000, domain=3, null_frac=0.3)
    check(capi, blocks_of(rows, [2000]), s, 1, ALL6)


def test_null_partition_keys_are_one_partition(capi):
    rng = np.random.default_rng(45)
    s = Schema(3, [(STRING, 0, True), (KEY_INT64, 1, True), (KEY_INT32, 2, True)])
    rows = table(rng, s, 1500, domain=3, null_frac=0.5)
    check(capi, blocks_of(rows, [1500]), s, 2, ALL6)
    rows = table(rng, s, 300, domain=3, null_frac=1.0)  # every key null: one partition of peers
    check(capi, blocks_of(rows, [300]), s, 2, ALL6)


@pytest.mark.parametrize("part", [KEY_FLOAT64, KEY_FLOAT32])
def test_float_zeros_and_nans_in_both_roles(capi, part):
    rng = np.random.default_rng(50 + part)
    F = {KEY_FLOAT64: [x.to_bytes(8, "little") for x in F64], KEY_FLOAT32: [x.to_bytes(4, "little") for x in F32]}

    def value(rng, t, domain):
        e = F[t & 0xFF]
        return e[int(rng.integers(len(e)))]

    s = Schema(2, [(part, 0, True), ((KEY_FLOAT32 if part == KEY_FLOAT64 else KEY_FLOAT64) | DESC, 1, True)])
    rows = table(rng, s, 2000, value=value)
    check(capi, blocks_of(rows, [2000]), s, 1, ALL6)


def test_decimal_keys(capi):
    rng = np.random.default_rng(55)

    def value(rng, t, domain):
        if t & 0xFF == DECIMAL:
            return DEC_EDGES[int(rng.integers(8))] if rng.random() < 0.5 else int(rng.integers(-3, 3)) * 10**25
        return small_value(rng, t, domain)

    s = Schema(3, [(DECIMAL, 0, True), (DECIMAL | DESC | NULLS_LAST, 1, True), (KEY_INT32, 2, True)])
    rows = table(rng, s, 2000, value=value)
    check(capi, blocks_of(rows, [1000, 1000]), s, 1, ALL6)


# ---------------------------------------------------------------------------------------------------------------
# 3. output layout: the bitset grows or not, VAR and DECIMAL_WIDE offsets move
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nf,fns", [(63, [RANK]), (63, [RANK, CUME_DIST]), (64, [ROW_NUMBER]), (70, ALL6)])
def test_wide_child_schemas(capi, nf, fns):
    rng = np.random.default_rng(60 + nf + len(fns))
    extra = {f: VAR for f in range(5, nf, 9)}
    extra.update({f: DECIMAL_WIDE for f in range(7, nf, 11)})
    s = Schema(nf, [(STRING, 1, True), (KEY_INT64 | DESC, nf - 1, True)], extra)
    rows = table(rng, s, 800, domain=5)
    check(capi, blocks_of(rows, [300, 500]), s, 1, fns)


# ---------------------------------------------------------------------------------------------------------------
# 4. limits
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("limit", [1, 2, 5, 1000])
@pytest.mark.parametrize("limit_fn", [ROW_NUMBER, RANK, DENSE_RANK])
def test_limits_with_ties_on_the_limit(capi, limit_fn, limit):
    rng = np.random.default_rng(70 + limit_fn * 10 + limit)
    s = Schema(3, [(STRING, 0, True), (KEY_INT64 | DESC, 1, True), (KEY_INT32, 2, True)])
    rows = table(rng, s, 3000, domain=4)
    r = check(capi, blocks_of(rows, [1500, 1500]), s, 1, [ROW_NUMBER, RANK, DENSE_RANK], (limit_fn, limit))
    if limit == 1000:
        assert r["n_out_records"] == 3000


def test_limit_one_keeps_the_latest_row_per_key(capi):
    """row_number() over (partition by id order by ts desc) = 1"""
    rng = np.random.default_rng(75)
    s = Schema(3, [(KEY_INT64, 0, False), (KEY_INT64 | DESC, 1, False)])
    rows = table(rng, s, 4000, domain=1000)
    r = check(capi, blocks_of(rows, [2000, 2000]), s, 1, [ROW_NUMBER], (ROW_NUMBER, 1))
    assert r["n_out_records"] < 4000


# ---------------------------------------------------------------------------------------------------------------
# 5. partition sizes and empty input
# ---------------------------------------------------------------------------------------------------------------
def test_every_record_its_own_partition(capi):
    rng = np.random.default_rng(80)
    s = Schema(2, [(KEY_INT64, 0, False), (KEY_INT32, 1, True)])
    rows = [s.row(rng, [i, int(rng.integers(5))]) for i in rng.permutation(3000)]
    check(capi, blocks_of(rows, [3000]), s, 1, ALL6)


def test_one_partition_of_500k_rows(capi):
    rng = np.random.default_rng(81)
    s = Schema(1, [(KEY_INT64 | DESC, 0, False)])
    vals = rng.integers(0, 100000, 500000)
    rows = [bytes(8) + struct.pack("<q", v) for v in vals.tolist()]
    check(capi, blocks_of(rows, [200000, 300000]), s, 0, [ROW_NUMBER, RANK, DENSE_RANK, CUME_DIST, (NTILE, 7)])


def test_empty_blocks_and_empty_input(capi):
    rng = np.random.default_rng(82)
    s = Schema(2, [(KEY_INT32, 0, True), (KEY_INT64, 1, True)])
    rows = table(rng, s, 50)
    check(capi, [b"", stream(rows[:20]), b"", stream(rows[20:]), b""], s, 1, ALL6)
    r = check(capi, [b"", b""], s, 1, ALL6)
    assert (r["n_records"], r["n_out_records"], r["total"]) == (0, 0, 0)
    dst = np.zeros(16, np.uint8)
    r = capi.decompress_window_rows_keys_packed(0, np.zeros(1, np.uint8), np.zeros(0, np.uint64),
                                                np.zeros(0, np.uint64), dst, s.keys, 1, s.nf, s.kinds, [RANK])
    assert (r["n_records"], r["n_out_records"], r["total"]) == (0, 0, 0)


# ---------------------------------------------------------------------------------------------------------------
# 6. the _dev form, the size retry, bad input and bad arguments
# ---------------------------------------------------------------------------------------------------------------
def test_dev_matches_packed(capi):
    rng = np.random.default_rng(90)
    s = Schema(4, [(STRING, 0, True), (KEY_INT64 | DESC, 1, True)], {3: VAR})
    rows = table(rng, s, 2000)
    plain = blocks_of(rows, [1000, 1000])
    a = check(capi, plain, s, 1, ALL6, codec=3, level=1, alg=3)
    b = check(capi, plain, s, 1, ALL6, codec=3, level=1, alg=3, dev=True)
    assert (a["n_records"], a["n_out_records"], a["total"]) == (b["n_records"], b["n_out_records"], b["total"])
    check(capi, plain, s, 1, [RANK], (RANK, 2), dev=True)


def test_dst_too_small_then_exact_retry(capi):
    rng = np.random.default_rng(91)
    s = Schema(2, [(KEY_INT32, 0, True), (KEY_INT64, 1, True)])
    plain = blocks_of(table(rng, s, 500), [500])
    blocks = build_blocks(capi, 1, 0, 0, plain)
    want, n, m = model_window(plain, s.keys, 1, s.nf, s.kinds, ALL6)
    args = (s.keys, 1, s.nf, s.kinds, ALL6, None)
    with pytest.raises(capi.B2SError) as e:
        run(capi, "decompress_window_rows_keys", 1, 0, blocks, args, len(want) - 1)
    assert e.value.code == capi.E_DST_TOO_SMALL
    dst = np.zeros(len(want) - 1, np.uint8)
    arena, off, ln, sb, sl, sc = blocks
    L = capi.load()
    # the raw call leaves the exact size in *dst_total
    import ctypes as C
    a = capi._window_arrays(*args)
    counts = [C.c_uint64(0) for _ in range(3)]
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = L.b2s_decompress_window_rows_keys_packed(1, 0, 1, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, None,
                                                  None, None, *map(capi._arg, a), dst.ctypes.data, dst.size,
                                                  *map(C.byref, counts), st.ctypes.data, bad.ctypes.data)
    assert rc == capi.E_DST_TOO_SMALL and counts[0].value == len(want)
    got, r = run(capi, "decompress_window_rows_keys", 1, 0, blocks, args, counts[0].value)
    assert got == want and (r["n_records"], r["n_out_records"]) == (n, m)


def test_corrupt_short_row_and_bad_checksum(capi):
    rng = np.random.default_rng(92)
    s = Schema(3, [(KEY_INT32, 0, True), (KEY_INT64, 1, True)])
    rows = table(rng, s, 200)
    good = stream(rows[:100])
    short = stream(rows[100:150] + [bytes(24)] + rows[150:])  # holds its keys, not the 32-byte fixed region
    torn = stream(rows[100:])[:-3]  # the last record runs past the block end
    for bad_block in (short, torn):
        plain = [good, bad_block]
        blocks = build_blocks(capi, 1, 0, 3, plain)
        got, r = run(capi, "decompress_window_rows_keys", 1, 3, blocks, (s.keys, 1, s.nf, s.kinds, ALL6, None), 1 << 16)
        assert list(r["status"]) == [0, capi.E_CORRUPT]
        assert (r["n_records"], r["n_out_records"], r["total"]) == (0, 0, 0) and got == b""
        assert b"block 1" in capi.load().b2s_last_error()
    plain = [good, stream(rows[100:])]
    arena, off, ln, sb, sl, sc = build_blocks(capi, 2, 0, 3, plain)
    sc = sc.copy()
    sc[0] ^= 1
    got, r = run(capi, "decompress_window_rows_keys", 2, 3, (arena, off, ln, sb, sl, sc),
                 (s.keys, 1, s.nf, s.kinds, ALL6, None), 1 << 16)
    assert list(r["status"]) == [capi.E_CHECKSUM, 0] and r["n_out_records"] == 0 and r["n_records"] == 0


S = Schema(3, [(KEY_INT32, 0, True), (KEY_INT64 | DESC, 1, True)])
K = S.keys


@pytest.mark.parametrize("keys,npk,nf,kinds,fns,limit", [
    (K, 2, 3, S.kinds, [RANK], None),                                   # no order column
    (K, 16, 3, S.kinds, [RANK], None),                                  # n_partition_keys above 15
    ([K[1], K[0]], 1, 3, S.kinds, [RANK], None),                        # a flag on a partition column
    ([(KEY_INT32, 7, 4, 0), K[1]], 1, 3, S.kinds, [RANK], None),        # a key slot inside the null words
    ([K[0], (KEY_INT64, 32, 8, 1)], 1, 3, S.kinds, [RANK], None),       # a key slot past the last field
    ([K[0], (KEY_INT64, 16, 8, 3)], 1, 3, S.kinds, [RANK], None),       # a null bit not below n_fields
    (K, 1, 0, [], [RANK], None),                                        # n_fields 0
    (K, 1, 65537, [0] * 65537, [RANK], None),                           # n_fields above 65536
    (K, 1, 3, None, [RANK], None),                                      # no field kinds
    (K, 1, 3, [0, 3, 0], [RANK], None),                                 # an unknown field kind
    (K, 1, 3, S.kinds, [], None),                                       # no function
    (K, 1, 3, S.kinds, [RANK] * 17, None),                              # 17 functions
    (K, 1, 3, S.kinds, [6], None),                                      # an unknown function
    (K, 1, 3, S.kinds, [(NTILE, 0)], None),                             # NTILE of 0 buckets
    (K, 1, 3, S.kinds, [(RANK, 2)], None),                              # an argument to RANK
    (K, 1, 3, S.kinds, [RANK], (RANK, 0)),                              # a limit below 1
    (K, 1, 3, S.kinds, [RANK], (PERCENT_RANK, 3)),                      # a limit by PERCENT_RANK
    (K, 1, 3, S.kinds, [RANK, CUME_DIST], (RANK, 3)),                   # a limit with CUME_DIST
    (K, 1, 3, S.kinds, [RANK, (NTILE, 2)], (ROW_NUMBER, 3)),            # a limit with NTILE
    (K, 1, 3, S.kinds, [RANK], (0xFFFFFFFF, 5)),                        # no limit with a limit value
    ([(KEY_INT32, 8, 2, 0), K[1]], 1, 3, S.kinds, [RANK], None),        # a key_len the type does not take
    ([K[0]] * 17, 1, 3, S.kinds, [RANK], None),                         # 17 key columns
])
def test_bad_arguments(capi, keys, npk, nf, kinds, fns, limit):
    rng = np.random.default_rng(93)
    plain = [stream(table(rng, S, 10))]
    with pytest.raises(capi.B2SError) as e:
        run(capi, "decompress_window_rows_keys", 1, 0, build_blocks(capi, 1, 0, 0, plain),
            (keys, npk, nf, kinds, fns, limit), 1 << 14)
    assert e.value.code == capi.E_ARG


def test_null_count_pointer_is_an_argument_error(capi):
    import ctypes as C
    L = capi.load()
    a = capi._window_arrays(K, 1, 3, S.kinds, [RANK], None)
    dst = np.zeros(64, np.uint8)
    total, out = C.c_uint64(0), C.c_uint64(0)
    rc = L.b2s_decompress_window_rows_keys_packed(0, 0, 0, None, None, None, None, None, None, *map(capi._arg, a),
                                                  dst.ctypes.data, dst.size, C.byref(total), None, C.byref(out), None,
                                                  None)
    assert rc == capi.E_ARG


# ---------------------------------------------------------------------------------------------------------------
# 7. the host mirror, and q67 end to end
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_reads_window_rows(capi, tmp_path, codec):
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R = 3, 2
    rng = np.random.default_rng(95)
    s = Schema(4, [(STRING, 0, True), (KEY_INT64 | DESC, 1, True)], {2: VAR})
    maps = []
    for m in range(M):
        rows = table(rng, s, 300)
        ids = rng.integers(0, R, len(rows))
        w = host.S3SerializedShuffleWriter(d, 0, m, R)
        for r, p in zip(rows, ids):
            w.insertRecord(int(p), len(r).to_bytes(4, "big") + r)
        w.commit()
        w.close()
        maps.append((rows, ids))
    for red in range(R):
        plain = [stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps]
        for fns, limit in ((ALL6, None), ([RANK, ROW_NUMBER], (RANK, 2))):
            reader = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
            got = reader.readWindowRows(s.keys, 1, s.nf, s.kinds, fns, limit)
            reader.close()
            assert got == model_window(plain, s.keys, 1, s.nf, s.kinds, fns, limit)


def _records(blobs):
    out = []
    for b in blobs:
        p = 0
        while p < len(b):
            sz = int.from_bytes(b[p:p + 4], "big")
            out.append(bytes(b[p:p + 4 + sz]))
            p += 4 + sz
    return out


def test_q67_rank_100_end_to_end(capi):
    """q67's window input hash-partitioned by i_category on the GPU; each reducer's rank() over (partition by
    i_category order by sumsales desc) <= 100 on the GPU: the reducers' outputs together are the model's over all rows"""
    rng = np.random.default_rng(99)
    cats = [b"Books", b"Children", b"Electronics", b"Home", b"Jewelry", b"Men", b"Music", b"Shoes", b"Sports",
            b"Women"]

    def value(rng, t, domain):
        if t & 0xFF == STRING:
            return cats[int(rng.integers(len(cats)))]
        return int(rng.integers(-2000, 200000)) * 10**2  # sumsales, decimal(28,2)

    # i_category, i_class, i_brand, i_product_name, d_year, d_qoy, d_moy, s_store_id, sumsales
    s = Schema(9, [(STRING, 0, True), (DECIMAL | DESC | NULLS_LAST, 8, True)], {1: VAR, 2: VAR, 3: VAR, 7: VAR})
    rows = table(rng, s, 12000, null_frac=0.02, value=value)
    R, maps = 4, 5
    per_reducer = [[] for _ in range(R)]
    for m in range(maps):
        part = rows[m::maps]
        records = np.frombuffer(stream(part), np.uint8).copy()
        rec_len = np.array([4 + len(r) for r in part], np.uint32)
        dst = np.zeros(2 * records.size + 4096 * R, np.uint8)
        r = capi.partition_compress_rows_hash_packed(2, records, rec_len, s.keys[:1], R, dst, checksum_alg=3)
        for p in range(R):
            if r["dst_len"][p]:
                o = int(r["dst_off"][p])
                per_reducer[p].append((dst[o:o + int(r["dst_len"][p])].tobytes(), int(r["checksums"][p])))
    got = []
    for p in range(R):
        data = [b for b, _ in per_reducer[p]]
        if not data:
            continue
        lens = np.array([len(b) for b in data], np.uint64)
        off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        dst = np.zeros(1 << 22, np.uint8)
        r = capi.decompress_window_rows_keys_packed(2, np.frombuffer(b"".join(data), np.uint8), off, lens, dst, s.keys,
                                                    1, s.nf, s.kinds, [RANK], (RANK, 100), 3,
                                                    np.arange(len(data) + 1, dtype=np.uint32), lens,
                                                    np.array([c for _, c in per_reducer[p]], np.uint64))
        assert (r["status"] == 0).all()
        got += _records([dst[:r["total"]].tobytes()])
    want = model_window(blocks_of(rows, [len(rows)]), s.keys, 1, s.nf, s.kinds, [RANK], (RANK, 100))
    assert want[2] < len(rows) // 5
    assert sorted(got) == sorted(_records([want[0]]))
