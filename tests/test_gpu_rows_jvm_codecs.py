"""The reduce-side row calls over shuffle blocks the map side's JVM writes, and over batch-fetched blocks of several
partition streams.

Every other row test compresses its blocks with our own GPU compressor, one stream and one checksum slice per block.
In production a reducer reads what lz4-java's LZ4BlockOutputStream (liblz4's LZ4_compress_default), xerial's
SnappyOutputStream (the snappy library) and zstd-jni's ZstdOutputStream (libzstd, streaming, flushed) wrote, and under
AQE's coalesced reads one fetched block holds several reduce partitions' streams back to back, one checksum slice
each.  Here each partition stream is compressed on the CPU by such a writer (or by the oracle's restated writers, which
need no library), a block is the concatenation of its partitions' streams, and every row family (sort, aggregate, join,
window, exchange read) must be byte for byte its model, byte for byte what it makes of the GPU compressor's blocks, and
must name the right block and slice when a stream or its checksum is bad.

The writers' own streams are checked on the CPU first (unmarked tests): each decodes back to its input with the
reference decoder, so a writer bug never shows up as a GPU failure."""
import ctypes as C
import functools

import numpy as np
import pytest

import hash_model as hm
import zstd_ref
from decimal_model import model_aggregate_decimal, sum_decimal
from join_model import INNER, LEFT_ANTI, LEFT_OUTER
from oracle import oracle
from outer_join_model import FULL_OUTER, RIGHT_OUTER, model_join
from rows_model import MAX_F64, MIN_I64, SUM_I64, build_blocks, model_aggregate, model_sort, run, stream
from test_gpu_exchange_rows import cache, q67_rows, store  # noqa: F401  (cache: the exchange fixture)
from test_gpu_join_rows import LKEY, LT, RKEY, RT, kinds, table as join_table
from test_gpu_sort_rows_order import DESC, NULLS_LAST, model_sort as order_model_sort
from test_gpu_window_agg_rows import Table, table as window_agg_table
from test_gpu_window_rows import Schema, table as window_table
from window_agg_model import FRAME_PARTITION, FRAME_RANGE, FRAME_ROWS, MIN, SUM, VAL_FLOAT64, dec, \
    model_window_aggregate
from window_model import DENSE_RANK, RANK, ROW_NUMBER, model_window

LZ4, SNAPPY, ZSTD = 1, 2, 3
E_CORRUPT, E_CHECKSUM = -1, -2
GPU_LEVEL = {LZ4: 0, SNAPPY: 0, ZSTD: 1}  # the level build_blocks compresses at, per codec


# ---------------------------------------------------------------------------------------------------------------
# 1. foreign writers: one partition stream in, one compressed stream out, in the JVM codec's wire format
# ---------------------------------------------------------------------------------------------------------------
_LIBLZ4 = []


def liblz4():
    if not _LIBLZ4:
        try:
            L = C.CDLL("liblz4.so.1")
        except OSError:
            pytest.skip("liblz4.so.1 is not installed")
        L.LZ4_compressBound.restype = C.c_int
        L.LZ4_compressBound.argtypes = [C.c_int]
        L.LZ4_compress_default.restype = C.c_int
        L.LZ4_compress_default.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
        _LIBLZ4.append(L)
    return _LIBLZ4[0]


def lz4block_liblz4(data, block_size):
    """LZ4BlockOutputStream over liblz4: per block_size chunk, magic | token (method | level) | compressed length |
    original length | XXH32(seed 0x9747b28c) & 0x0FFFFFFF | payload (raw when it does not shrink), then the end mark"""
    L = liblz4()
    level = max(0, (block_size - 1).bit_length() - 10)
    out = []
    for o in range(0, len(data), block_size):
        chunk = data[o:o + block_size]
        cap = L.LZ4_compressBound(len(chunk))
        buf = C.create_string_buffer(cap)
        n = L.LZ4_compress_default(chunk, buf, len(chunk), cap)
        assert n > 0
        method, payload = (0x20, buf.raw[:n]) if n < len(chunk) else (0x10, chunk)
        chk = oracle.xxh32(chunk) & 0x0FFFFFFF
        out.append(b"LZ4Block" + bytes([method | level]) + len(payload).to_bytes(4, "little")
                   + len(chunk).to_bytes(4, "little") + chk.to_bytes(4, "little") + payload)
    return b"".join(out) + b"LZ4Block" + bytes([0x10 | level]) + bytes(12)


def xerial_pyarrow(data, block_size=32768):
    """SnappyOutputStream over the snappy library (pyarrow's): the xerial header, then [length BE][raw snappy] chunks"""
    try:
        import pyarrow as pa
    except ImportError:
        pytest.skip("pyarrow is not installed")
    if not pa.Codec.is_available("snappy"):
        pytest.skip("pyarrow has no snappy codec")
    codec = pa.Codec("snappy")
    out = [bytes([0x82]) + b"SNAPPY\x00" + (1).to_bytes(4, "big") + (1).to_bytes(4, "big")]
    for o in range(0, len(data), block_size):
        c = codec.compress(data[o:o + block_size]).to_pybytes()
        out.append(len(c).to_bytes(4, "big") + c)
    return b"".join(out)


def libzstd():
    try:
        return zstd_ref.lib()
    except OSError:
        pytest.skip("libzstd.so.1 is not installed")


def zstd_two_frames(data):
    libzstd()
    h = len(data) // 3
    return zstd_ref.compress(data[:h], 1) + zstd_ref.compress_stream(data[h:], 3, flush_every=2)


def zstd_stream(level, flush_every):
    def w(data):
        libzstd()
        return zstd_ref.compress_stream(data, level, flush_every=flush_every)
    return w


def zstd_oneshot(data):
    libzstd()
    return zstd_ref.compress(data, 3)


# name -> (codec, writer, reference decoder); the oracle writers need no library and always run
WRITERS = {
    "lz4-liblz4-32k": (LZ4, lambda d: lz4block_liblz4(d, 32768), oracle.lz4block_decompress),
    "lz4-liblz4-64k": (LZ4, lambda d: lz4block_liblz4(d, 65536), oracle.lz4block_decompress),
    "lz4-oracle-32k": (LZ4, lambda d: oracle.lz4block_compress(d, 32768, compressor=0), oracle.lz4block_decompress),
    "lz4-oracle-64k": (LZ4, lambda d: oracle.lz4block_compress(d, 65536, compressor=0), oracle.lz4block_decompress),
    "snappy-pyarrow": (SNAPPY, xerial_pyarrow, oracle.xerial_decompress),
    "snappy-oracle": (SNAPPY, lambda d: oracle.xerial_compress(d, 32768, compressor=0), oracle.xerial_decompress),
    "zstd-stream-l1": (ZSTD, zstd_stream(1, 2), zstd_ref.decompress),
    "zstd-stream-l2": (ZSTD, zstd_stream(2, 3), zstd_ref.decompress),
    "zstd-stream-l3": (ZSTD, zstd_stream(3, 1), zstd_ref.decompress),
    "zstd-oneshot": (ZSTD, zstd_oneshot, zstd_ref.decompress),
    "zstd-two-frames": (ZSTD, zstd_two_frames, zstd_ref.decompress),
}
NAMES = list(WRITERS)


def partner(name):
    """another writer of the same codec: a join's right side is written by it"""
    same = [n for n in NAMES if WRITERS[n][0] == WRITERS[name][0]]
    return same[(same.index(name) + 1) % len(same)]


def pack(streams, alg):
    """blocks of compressed streams [[bytes, ...], ...] -> build_blocks' (arena, off, len, slice_base, slice_len,
    slice_checksum): a block is its streams back to back, every stream one slice with its own checksum"""
    flat = [s for blk in streams for s in blk]
    arena = np.frombuffer(b"".join(flat) + b"\x00", np.uint8).copy()
    lens = [sum(len(s) for s in blk) for blk in streams]
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64) if lens else np.zeros(0, np.uint64)
    sb = np.concatenate([[0], np.cumsum([len(blk) for blk in streams])]).astype(np.uint32)
    ck = [oracle.checksum(alg, s) if alg else 0 for s in flat]
    return (arena, off, np.array(lens, np.uint64), sb, np.array([len(s) for s in flat], np.uint64),
            np.array(ck, np.uint64))


def compress_parts(parts_per_block, writer):
    """each partition of each block through writer (a name, or one name per block); a partition of None is one the
    map side wrote no bytes for: a zero-length slice"""
    names = writer if isinstance(writer, list) else [writer] * len(parts_per_block)
    return [[b"" if p is None else WRITERS[w][1](p) for p in blk] for blk, w in zip(parts_per_block, names)]


def jvm_blocks(codec, parts_per_block, alg, writer):
    """the plain partition streams, grouped into blocks, written by a foreign writer of codec -> the 6-tuple of
    build_blocks"""
    names = writer if isinstance(writer, list) else [writer]
    assert all(WRITERS[w][0] == codec for w in names)
    return pack(compress_parts(parts_per_block, writer), alg)


def gpu_blocks(capi, codec, parts_per_block, alg):
    """the same partitions and block shape, each stream written by the GPU compressor"""
    out = []
    for blk in parts_per_block:
        live = [p for p in blk if p is not None]
        comp, _, st = capi.compress_batch(codec, live, 0, level=GPU_LEVEL[codec]) if live else ([], [], [])
        assert st == [0] * len(live)
        it = iter(comp)
        out.append([b"" if p is None else next(it) for p in blk])
    return pack(out, alg)


def plain_of(parts_per_block):
    """each block's decoded bytes"""
    return [b"".join(p or b"" for p in blk) for blk in parts_per_block]


# ---------------------------------------------------------------------------------------------------------------
# the reducer's input: four blocks of 1, 3 and 4 partition streams
# ---------------------------------------------------------------------------------------------------------------
BIG = 110_000  # a record's tail: 40 KB of random bytes, then zeros, so it crosses several 32 KiB codec blocks


def with_big_record(rng, rows, i):
    rows = list(rows)
    rows[i] = rows[i] + rng.integers(0, 256, 40_000, dtype=np.uint8).tobytes() + bytes(BIG - 40_000)
    return rows


def shape(rows):
    """block 0: a stream, the codec's empty stream, a partition with no bytes, a stream; block 1: three streams, the
    middle one holding a record longer than three codec blocks; block 2: one partition with no bytes (an empty block);
    block 3: one stream"""
    n = len(rows)
    cut = [0] + [int(n * f) for f in (0.08, 0.23, 0.41, 0.68, 0.78)] + [n]
    s = [stream(rows[cut[k]:cut[k + 1]]) for k in range(6)]
    return [[s[0], b"", None, s[1]], [s[2], s[3], s[4]], [None], [s[5]]]


def shaped(rng, rows):
    n = len(rows)
    return shape(with_big_record(rng, rows, (int(n * 0.41) + int(n * 0.68)) // 2))


MIDDLE_BLOCK = 1  # the three-stream block


# ---------------------------------------------------------------------------------------------------------------
# the families: their inputs, calls and models
# ---------------------------------------------------------------------------------------------------------------
SORT_TYPES = ["string", "decimal", "long", "long", "long", "long", "double", "long"]
PREFIXES = [b"", b"ab", b"category#", b"\x00\x00", b"\xff" * 9, b"Books/Fiction/" * 3]


def slot(f):
    return 8 + 8 * f  # SORT_TYPES fit one null word


SORT_KEYS = hm.keys_of(SORT_TYPES, [0, 1, 2])
SORT_KEYS[1] = (SORT_KEYS[1][0] | DESC | NULLS_LAST,) + SORT_KEYS[1][1:]  # the decimal DESC NULLS LAST
SINGLE_KEY = hm.keys_of(SORT_TYPES, [2])[0]
AGG_KEYS = hm.keys_of(SORT_TYPES, [0, 2])
AGGS = [(SUM_I64, slot(3), 3), (SUM_I64, slot(4), -1), (MIN_I64, slot(5), 5), (MAX_F64, slot(6), 6),
        (sum_decimal(17), slot(7), 7)]  # sum, count (a non-null 1 per row), min, max over doubles, decimal(17) sum


def sort_rows(rng, n):
    rows = []
    for _ in range(n):
        def maybe(v, p=0.05):
            return None if rng.random() < p else v
        s = PREFIXES[int(rng.integers(len(PREFIXES)))] + bytes(rng.integers(97, 100, int(rng.integers(0, 3)),
                                                                         dtype=np.uint8))
        d = int(rng.integers(-3, 4)) * 10**int(rng.choice([0, 5, 18, 30, 37]))
        k = int(rng.choice([-2**63, 2**63 - 1, -1, 0, 1, int(rng.integers(-3, 4))]))
        dbl = hm.SPECIAL_F64[int(rng.integers(len(hm.SPECIAL_F64)))] if rng.random() < 0.4 else float(rng.normal())
        rows.append(hm.make_row(SORT_TYPES, [maybe(s), maybe(d), maybe(k), maybe(int(rng.integers(-10**6, 10**6)), 0.1),
                                             1, maybe(int(rng.integers(-2**63, 2**63 - 1, dtype=np.int64))),
                                             maybe(dbl, 0.1), maybe(int(rng.integers(-10**12, 10**12)))]))
    return rows


@functools.lru_cache(None)
def family_input(family):
    """-> the partitions per block (a join: left blocks, then right blocks) and, for a join, the number of left blocks"""
    rng = np.random.default_rng({"sort": 1, "aggregate": 2, "join": 3, "window": 4}[family])
    if family in ("sort", "aggregate"):
        return shaped(rng, sort_rows(rng, 3000)), 0
    if family == "join":
        left = shaped(rng, join_table(rng, LT, 1500, (0,), key_range=300))
        right = shape(join_table(rng, RT, 1000, (2,), key_range=300))
        return left + right, len(left)
    rows = window_table(rng, WINDOW_SCHEMA, 2000, domain=6)
    agg_rows = window_agg_table(rng, WINDOW_AGG_TABLE, 2000, order_domain=6)
    return (shaped(rng, rows), shaped(rng, agg_rows)), 0


WINDOW_SCHEMA = Schema(6, [(3, 0, True), (2, 2, True), (1 | DESC, 4, False)])  # PARTITION BY string, long; int DESC
WINDOW_FNS, WINDOW_LIMIT = [RANK, ROW_NUMBER, DENSE_RANK], (RANK, 30)
WINDOW_AGG_TABLE = Table(value_types=[VAL_FLOAT64, dec(17, 2)])


def window_agg_fns():
    t = WINDOW_AGG_TABLE
    f, d = t.value(0), t.value(1)
    return [(SUM, FRAME_ROWS) + f, (SUM, FRAME_PARTITION) + d, (MIN, FRAME_RANGE) + f]


JOINS = [INNER, LEFT_OUTER, LEFT_ANTI, RIGHT_OUTER, FULL_OUTER]


def once(f):
    return functools.lru_cache(None)(f)


@functools.lru_cache(None)
def calls(family):
    """the family's calls: [(label, run(capi, codec, alg, blocks, dev) -> (output, result), the model -> (output,
    counts), the result's count names, whether a _dev run follows the packed one)]; each model is evaluated once"""
    parts, n_left = family_input(family)
    if family == "sort":
        plain = plain_of(parts)
        total = sum(map(len, plain))
        return [
            ("sort_rows", lambda c, codec, alg, b, dev: run(c, "decompress_sort_rows", codec, alg, b, SINGLE_KEY, total,
                                                            dev),
             once(lambda: _n(model_sort(plain, [SINGLE_KEY]), total)), ("n_records", "total"), False),
            ("sort_rows_keys", lambda c, codec, alg, b, dev: run(c, "decompress_sort_rows_keys", codec, alg, b,
                                                                 (SORT_KEYS,), total, dev),
             once(lambda: _n(order_model_sort(plain, SORT_KEYS), total)), ("n_records", "total"), True)]
    if family == "aggregate":
        plain = plain_of(parts)
        total = sum(map(len, plain))

        @once
        def agg_model():
            want, n, g = model_aggregate_decimal(plain, AGG_KEYS, AGGS)
            return want, (n, g, len(want))
        return [("aggregate_rows_keys", lambda c, codec, alg, b, dev: run(c, "decompress_aggregate_rows_keys", codec,
                                                                          alg, b, (AGG_KEYS, AGGS), total, dev),
                 agg_model, ("n_records", "n_groups", "total"), False)]
    if family == "join":
        left, right = plain_of(parts[:n_left]), plain_of(parts[n_left:])
        out = []
        for jt in JOINS:
            @once
            def join_model(jt=jt):
                want, nl, nr, nout = model_join(jt, left, right, LKEY, RKEY, len(LT), len(RT), kinds(LT), kinds(RT))
                return want, (nl, nr, nout, len(want))

            def join_call(c, codec, alg, b, dev, jt=jt):
                arena, off, ln, sb, sl, sc = b
                cap = len(join_model()[0])
                dst = np.zeros(max(cap, 1), np.uint8)
                lk, rk = (None, None) if jt == LEFT_ANTI else (kinds(LT), kinds(RT))
                r = c.decompress_join_rows_keys_packed(jt, codec, arena, off, ln, n_left, dst[:cap], LKEY, RKEY,
                                                       len(LT), len(RT), lk, rk, alg, sb, sl, sc)
                return dst[:r["total"]].tobytes(), r
            out.append(("join_rows_keys[%d]" % jt, join_call, join_model,
                        ("n_left_records", "n_right_records", "n_out_records", "total"), False))
        return out
    rank_parts, agg_parts = parts
    s, t = WINDOW_SCHEMA, WINDOW_AGG_TABLE
    rank_plain, agg_plain = plain_of(rank_parts), plain_of(agg_parts)

    @once
    def rank_model():
        want, n, m = model_window(rank_plain, s.keys, 2, s.nf, s.kinds, WINDOW_FNS, WINDOW_LIMIT)
        return want, (n, m, len(want))

    @once
    def agg_model():
        want, n, m = model_window_aggregate(agg_plain, t.keys(1), 1, t.nf, t.kinds, window_agg_fns())
        return want, (n, m, len(want))
    names = ("n_records", "n_out_records", "total")
    return [("window_rows_keys", lambda c, codec, alg, b, dev: run(
                c, "decompress_window_rows_keys", codec, alg, b, (s.keys, 2, s.nf, s.kinds, WINDOW_FNS, WINDOW_LIMIT),
                len(rank_model()[0]), dev), rank_model, names, False),
            ("window_aggregate_rows_keys", lambda c, codec, alg, b, dev: run(
                c, "decompress_window_aggregate_rows_keys", codec, alg, b,
                (t.keys(1), 1, t.nf, t.kinds, window_agg_fns()), len(agg_model()[0]), dev), agg_model, names, True)]


def _n(model_out, total):
    want, n = model_out
    return want, (n, total)


def family_parts(family, label):
    """the partitions per block a call of the family reads"""
    parts, _ = family_input(family)
    if family == "window":
        return parts[0] if label == "window_rows_keys" else parts[1]
    return parts


def family_writers(family, name, parts):
    """the writer of each block: a join's right side is written by another writer of the codec"""
    if family != "join":
        return name
    n_left = family_input(family)[1]
    return [name] * n_left + [partner(name)] * (len(parts) - n_left)


def counts(r, names):
    return tuple(int(r[k]) for k in names)


def ok(r):
    assert (r["status"] == 0).all(), list(r["status"])


# ---------------------------------------------------------------------------------------------------------------
# 1. CPU self-checks of the writers
# ---------------------------------------------------------------------------------------------------------------
EDGE_INPUTS = [b"", b"a", b"abcdefghijklm", bytes(100_000), np.random.default_rng(0).integers(0, 256, 70_000,
                                                                                               dtype=np.uint8).tobytes(),
               (np.arange(9000, dtype=np.uint32) * 7).tobytes()[:33_000]]


@pytest.mark.parametrize("name", NAMES)
def test_writer_streams_decode_back_with_the_reference_decoder(name):
    codec, write, decode = WRITERS[name]
    for family in ("sort", "join", "window"):
        parts = family_input(family)[0]
        for blk in (parts if family != "window" else parts[0] + parts[1]):
            for p in blk:
                if p is not None:
                    assert decode(write(p)) == p, (family, len(p))
    for x in EDGE_INPUTS:
        assert decode(write(x)) == x, len(x)


@pytest.mark.parametrize("alg", [1, 3])
@pytest.mark.parametrize("name", NAMES)
def test_multi_stream_blocks_are_their_streams_and_slices(name, alg):
    """a block decodes (as the JVM reads a batch block, stream after stream) to its partitions back to back, and each
    slice is one stream with the checksum of its bytes"""
    codec, write, decode = WRITERS[name]
    parts, _ = family_input("sort")
    arena, off, ln, sb, sl, sc = jvm_blocks(codec, parts, alg, name)
    assert list(sb) == [0, 4, 7, 8, 9] and sl[sb[2]] == 0 and ln[2] == 0  # 4, 3, 1 and 1 slices; an empty block
    assert sl[1] > 0 and sl[2] == 0  # the codec's empty stream, then a partition with no bytes
    for b, blk in enumerate(parts):
        data = arena[int(off[b]):int(off[b] + ln[b])].tobytes()
        assert int(sl[sb[b]:sb[b + 1]].sum()) == len(data)
        assert decode(data) == b"".join(p or b"" for p in blk)  # block 2 has no bytes: an empty stream
        at = 0
        for k in range(sb[b], sb[b + 1]):
            piece = data[at:at + int(sl[k])]
            assert int(sc[k]) == oracle.checksum(alg, piece)
            at += int(sl[k])
    big = parts[MIDDLE_BLOCK][1]
    assert max(len(r) for r in _records(big)) > 3 * 32768  # the record crossing codec blocks is there


def _records(buf):
    out, p = [], 0
    while p < len(buf):
        s = int.from_bytes(buf[p:p + 4], "big")
        out.append(buf[p + 4:p + 4 + s])
        p += 4 + s
    return out


# Zstandard frames parsed on the CPU (RFC 8878): which block types, literal section types and sequence table modes the
# libzstd streams of these inputs use: frames with and without a content size, many blocks per frame, raw and RLE
# blocks, raw literals inside compressed blocks, 1- and 4-stream Huffman literals, predefined and FSE tables.
def zstd_forms(data):
    forms = set()
    p = 0
    while p < len(data):
        magic = int.from_bytes(data[p:p + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            p += 8 + int.from_bytes(data[p + 4:p + 8], "little")
            forms.add("skippable frame")
            continue
        assert magic == 0xFD2FB528
        fhd = data[p + 4]
        single = (fhd >> 5) & 1
        fcs = [1 if single else 0, 2, 4, 8][fhd >> 6]
        forms.add("content size" if fcs else "no content size")
        if (fhd >> 2) & 1:
            forms.add("content checksum")
        p += 5 + (0 if single else 1) + [0, 1, 2, 4][fhd & 3] + fcs
        nblocks = 0
        while True:
            h = int.from_bytes(data[p:p + 3], "little")
            last, btype, size = h & 1, (h >> 1) & 3, h >> 3
            p += 3
            nblocks += 1
            forms.add(["raw block", "RLE block", "compressed block"][btype])
            if btype == 2:
                forms |= compressed_block_forms(data[p:p + size])
            p += 1 if btype == 1 else size
            if last:
                break
        if nblocks > 1:
            forms.add("several blocks in a frame")
        p += 4 if (fhd >> 2) & 1 else 0
    return forms


def compressed_block_forms(b):
    forms = set()
    b0 = b[0]
    lt, sf = b0 & 3, (b0 >> 2) & 3
    forms.add(["raw literals", "RLE literals", "Huffman literals", "treeless literals"][lt])
    if lt < 2:
        hs = [1, 2, 1, 3][sf]
        regen = b0 >> 3 if sf in (0, 2) else (b0 >> 4) + (b[1] << 4) + ((b[2] << 12) if sf == 3 else 0)
        p = hs + (regen if lt == 0 else 1)
    else:
        forms.add("1-stream literals" if sf == 0 else "4-stream literals")
        hs = [3, 3, 4, 5][sf]
        h = int.from_bytes(b[:hs], "little")
        comp = {3: (h >> 14) & 0x3FF, 4: (h >> 18) & 0x3FFF, 5: (h >> 22) & 0x3FFFF}[hs]
        p = hs + comp
    n0 = b[p]
    if n0 == 0:
        forms.add("no sequences")
        return forms
    p += 1 if n0 < 128 else 2 if n0 < 255 else 3
    m = b[p]
    for name, mode in (("LL", m >> 6), ("OF", (m >> 4) & 3), ("ML", (m >> 2) & 3)):
        forms.add("%s %s" % (name, ["predefined", "RLE", "FSE", "repeat"][mode]))
    return forms


def test_zstd_writers_reach_forms_beyond_the_gpu_encoders():
    libzstd()
    forms = set()
    for name in NAMES:
        if WRITERS[name][0] != ZSTD:
            continue
        for family in ("sort", "join", "window"):
            parts = family_input(family)[0]
            for blk in (parts if family != "window" else parts[0] + parts[1]):
                for p in blk:
                    if p is not None:
                        forms |= zstd_forms(WRITERS[name][1](p))
    print("zstd forms of the libzstd writers:", sorted(forms))
    assert {"no content size", "content size", "several blocks in a frame", "raw block", "RLE block",
            "compressed block", "raw literals", "Huffman literals", "4-stream literals", "LL FSE", "LL predefined",
            "OF FSE", "ML FSE", "ML predefined"} <= forms, sorted(forms)


# ---------------------------------------------------------------------------------------------------------------
# 2. every family over foreign blocks, byte for byte its model
# ---------------------------------------------------------------------------------------------------------------
FAMILIES = ["sort", "aggregate", "join", "window"]


@pytest.mark.gpu
@pytest.mark.parametrize("alg", [1, 3], ids=["adler32", "crc32c"])
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("family", FAMILIES)
def test_family_over_foreign_blocks_like_the_model(capi, family, name, alg):
    codec = WRITERS[name][0]
    for label, call, model, names, dev in calls(family):
        parts = family_parts(family, label)
        blocks = jvm_blocks(codec, parts, alg, family_writers(family, name, parts))
        want, want_counts = model()
        got, r = call(capi, codec, alg, blocks, False)
        ok(r)
        assert counts(r, names) == want_counts, label
        assert got == want, label
        if dev:
            got, r = call(capi, codec, alg, blocks, True)
            ok(r)
            assert counts(r, names) == want_counts and got == want, label + " _dev"


# ---------------------------------------------------------------------------------------------------------------
# 3. the writer does not matter: the GPU compressor's blocks and every foreign writer's give the same bytes
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("family", FAMILIES)
def test_outputs_do_not_depend_on_the_writer(capi, family, name):
    codec, alg = WRITERS[name][0], 3
    for label, call, _, names, _ in calls(family):
        parts = family_parts(family, label)
        outs = []
        for blocks in (jvm_blocks(codec, parts, alg, family_writers(family, name, parts)),
                       gpu_blocks(capi, codec, parts, alg),
                       build_blocks(capi, codec, GPU_LEVEL[codec], alg, plain_of(parts))):
            got, r = call(capi, codec, alg, blocks, False)
            ok(r)
            outs.append((got, counts(r, names)))
        assert outs[0] == outs[1] == outs[2], label


# ---------------------------------------------------------------------------------------------------------------
# 2-3. the exchange reads: cached ranges (the GPU row partitioner's) and foreign fetched blocks in one call
# ---------------------------------------------------------------------------------------------------------------
def exchange_call(capi, name, lead, codec, alg, src, args, cap):
    arena, off, ln, sb, sl, sc = src
    dst = np.zeros(max(cap, 1), np.uint8)
    r = getattr(capi, "exchange_read_" + name + "_packed")(*lead, codec, arena, off, ln, dst, *args, alg, sb, sl, sc)
    return dst[:r["total"]].tobytes() if "aggregate" in name or r["n_records"] else b"", r


@pytest.mark.gpu
@pytest.mark.parametrize("alg", [1, 3], ids=["adler32", "crc32c"])
@pytest.mark.parametrize("name", NAMES)
def test_exchange_reads_mix_cached_ranges_with_foreign_blocks(cache, name, alg):
    codec = WRITERS[name][0]
    shuffle = 40 + NAMES.index(name) * 2 + (alg == 3)
    _, keys, aggs = q67_rows(np.random.default_rng(0), 1)
    M, R, s, e = 4, 3, 0, 2
    parts = []
    for m in range(M):
        rows = q67_rows(np.random.default_rng(60 + m), 1200)[0]
        if m == 2:
            rows = with_big_record(np.random.default_rng(m), rows, 5)
        written = store(cache, "hash", shuffle, m, rows, keys, R, codec, GPU_LEVEL[codec], alg, compare=False)
        assert written["cached"] == 1
        plain = store(cache, "hash", shuffle, m, rows, keys, R, 0, 0, 0, cached=False)
        parts.append([None if not plain["dst_len"][p] else
                      plain["data"][int(plain["dst_off"][p]):int(plain["dst_off"][p] + plain["dst_len"][p])].tobytes()
                      for p in range(s, e)])
    src = jvm_blocks(codec, parts, alg, name)
    plain = plain_of(parts)
    cap = sum(map(len, plain)) + 4096
    ids = list(range(M))
    want_sort = model_sort(plain, keys)
    want_agg = model_aggregate(plain, keys, aggs)
    for mask in ([0] * M, [1, 0, 1, 0], [0, 1, 0, 1]):
        lead = (shuffle, s, e, ids, mask)
        got, r = exchange_call(cache, "sort_rows_keys", lead, codec, alg, src, (keys,), cap)
        ok(r)
        assert (got, r["n_records"], r["total"]) == (want_sort[0], want_sort[1], len(want_sort[0])), mask
        got, r = exchange_call(cache, "aggregate_rows_keys", lead, codec, alg, src, (keys, aggs), cap)
        ok(r)
        assert (got, r["n_records"], r["n_groups"], r["total"]) == (want_agg[0], want_agg[1], want_agg[2],
                                                                     len(want_agg[0])), mask
    # the same read over the GPU writer's fetched blocks of the same partitions gives the same bytes
    gpu_src = gpu_blocks(cache, codec, parts, alg)
    for which, args in (("sort_rows_keys", (keys,)), ("aggregate_rows_keys", (keys, aggs))):
        lead = (shuffle, s, e, ids, [1, 0, 1, 0])
        a = exchange_call(cache, which, lead, codec, alg, src, args, cap)
        b = exchange_call(cache, which, lead, codec, alg, gpu_src, args, cap)
        assert a[0] == b[0] and a[1]["n_records"] == b[1]["n_records"] and a[1]["total"] == b[1]["total"]


@pytest.mark.gpu
@pytest.mark.parametrize("codec", [LZ4, SNAPPY, ZSTD], ids=["lz4", "snappy", "zstd"])
def test_block_of_no_bytes_is_an_empty_stream(capi, codec):
    """a fetched block of a partition the map side wrote no bytes for decodes to nothing, as the JVM's readers take
    an empty input, for every codec, in the plain decode and in a row call beside other blocks"""
    s = stream([bytes(range(40))])
    write = WRITERS[{LZ4: "lz4-oracle-32k", SNAPPY: "snappy-oracle", ZSTD: "zstd-oneshot"}[codec]][1]
    blocks = pack([[b""], [write(s)], [b""]], 3)
    dst = np.zeros(4096, np.uint8)
    d = capi.decompress_packed(codec, blocks[0], blocks[1], blocks[2], dst, 3, *blocks[3:])
    assert list(d["status"]) == [0, 0, 0] and list(d["dst_len"]) == [0, len(s), 0]
    got, r = run(capi, "decompress_sort_rows", codec, 3, blocks, (1, 0, 4, -1), len(s))
    ok(r)
    assert (got, r["n_records"], r["total"]) == (s, 1, len(s))


# ---------------------------------------------------------------------------------------------------------------
# 4. per-slice verdicts on multi-slice foreign blocks
# ---------------------------------------------------------------------------------------------------------------
VERDICT_CASES = [("lz4-liblz4-32k", "sort"), ("lz4-oracle-64k", "window"), ("snappy-oracle", "aggregate"),
                 ("snappy-pyarrow", "join"), ("zstd-stream-l1", "join"), ("zstd-two-frames", "sort"),
                 ("zstd-stream-l3", "window"), ("zstd-oneshot", "aggregate")]


def nothing_written(r, names, got):
    assert all(int(r[k]) == 0 for k in names) and got == b"", counts(r, names)


@pytest.mark.gpu
@pytest.mark.parametrize("name,family", VERDICT_CASES, ids=["%s-%s" % c for c in VERDICT_CASES])
def test_bad_middle_slice_is_named(capi, name, family):
    """a byte flipped in the middle stream of a three-stream block: B2S_E_CHECKSUM for that block with bad_slice 1 (the
    slice's index within its block); the other blocks B2S_OK and nothing written"""
    codec, alg = WRITERS[name][0], 3
    label, call, _, names, _ = calls(family)[0]
    parts = family_parts(family, label)
    arena, off, ln, sb, sl, sc = jvm_blocks(codec, parts, alg, family_writers(family, name, parts))
    b = MIDDLE_BLOCK
    first = int(sb[b])
    assert int(sb[b + 1]) - first == 3
    arena = arena.copy()
    arena[int(off[b] + sl[first] + sl[first + 1] // 2)] ^= 0x5A
    got, r = call(capi, codec, alg, (arena, off, ln, sb, sl, sc), False)
    want = [0] * len(ln)
    want[b] = E_CHECKSUM
    assert list(r["status"]) == want and r["bad_slice"][b] == 1
    nothing_written(r, names, got)


@pytest.mark.gpu
@pytest.mark.parametrize("name,family", VERDICT_CASES, ids=["%s-%s" % c for c in VERDICT_CASES])
def test_truncated_middle_stream_fails_its_block(capi, name, family):
    """the middle stream one byte short, its checksum recomputed so that it verifies: B2S_E_CORRUPT for that block,
    named by b2s_last_error(), and nothing written"""
    codec, alg = WRITERS[name][0], 3
    label, call, _, names, _ = calls(family)[0]
    parts = family_parts(family, label)
    streams = compress_parts(parts, family_writers(family, name, parts))
    b = MIDDLE_BLOCK
    streams[b][1] = streams[b][1][:-1]
    assert WRITERS[name][2] is not None
    with pytest.raises(IOError):  # the reference reader rejects the stream too
        WRITERS[name][2](streams[b][1])
    blocks = pack(streams, alg)
    got, r = call(capi, codec, alg, blocks, False)
    want = [0] * len(blocks[1])
    want[b] = E_CORRUPT
    assert list(r["status"]) == want
    err = capi.load().b2s_last_error()
    assert (b"block %d" % b) in err, err
    nothing_written(r, names, got)
    # the plain decode of the same blocks gives the same verdict
    dst = np.zeros(sum(map(len, plain_of(parts))) + 4096, np.uint8)
    d = capi.decompress_packed(codec, blocks[0], blocks[1], blocks[2], dst, alg, *blocks[3:])
    assert list(d["status"]) == want


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
def test_zstd_content_checksum_is_not_verified(capi, family):
    """libzstd writes a Content_Checksum when asked (zstd-jni's setChecksum), and rejects a frame whose checksum is
    wrong.  The GPU decoder skips it, as the header states, so the frame's blocks decode as they are: the row call
    agrees with the plain decode of the same blocks, and both accept a wrong checksum"""
    libzstd()
    label, call, model, names, _ = calls(family)[0]
    parts = [list(blk) for blk in family_parts(family, label)]
    b = MIDDLE_BLOCK
    streams = [[b"" if p is None else zstd_ref.compress_stream(p, 1, flush_every=2) for p in blk] for blk in parts]
    good = zstd_ref.compress_stream_params(parts[b][1], [(zstd_ref.P_LEVEL, 1), (zstd_ref.P_CHECKSUM, 1)],
                                           flush_every=1)
    assert "content checksum" in zstd_forms(good) and zstd_ref.decompress(good) == parts[b][1]
    bad = good[:-1] + bytes([good[-1] ^ 0x01])
    with pytest.raises(IOError):
        zstd_ref.decompress(bad)
    want, want_counts = model()
    plain = plain_of(parts)
    for frame in (good, bad):
        streams[b][1] = frame
        blocks = pack(streams, 3)
        got, r = call(capi, ZSTD, 3, blocks, False)
        dst = np.zeros(sum(map(len, plain)) + 4096, np.uint8)
        d = capi.decompress_packed(ZSTD, blocks[0], blocks[1], blocks[2], dst, 3, *blocks[3:])
        assert list(r["status"]) == list(d["status"]) == [0] * len(blocks[1])
        assert dst[int(d["dst_off"][b]):int(d["dst_off"][b] + d["dst_len"][b])].tobytes() == plain[b]
        assert counts(r, names) == want_counts and got == want
