"""Shared helpers for the sort-family tests (b2s_decompress_sort_* / *_sort_rows_* / *_aggregate_rows_* and their
composite-key forms): block building, a Python model of the row sort and the row aggregation, one runner for the
packed and _dev calls, and the host-mirror set-up.

The model parses the decoded UnsafeRowSerializer streams ([int32 big-endian size][row]), sorts the records stably by a
tuple of (not-null flag, value) per key column, with strings as Python bytes (whose order is exactly unsigned
lexicographic with a proper prefix first), and groups equal tuples.  A single-key call is the one-column case."""
import math
import struct
import uuid

import numpy as np

import spark_s3_shuffle_b200 as pkg

CODECS = [("none", 0, 0), ("lz4", 1, 0), ("snappy", 2, 0), ("zstd1", 3, 1), ("zstd3", 3, 3)]
CHECKSUMS = [0, 1, 2, 3]  # none, ADLER32, CRC32, CRC32C
KEY_BYTES, KEY_INT32, KEY_INT64 = 0, 1, 2
STRING = 3
SUM_I64, SUM_F64, MIN_I32, MAX_I32, MIN_I64, MAX_I64, MIN_F64, MAX_F64 = range(8)


# ---------------------------------------------------------------------------------------------------------------
# streams and blocks
# ---------------------------------------------------------------------------------------------------------------
def stream(rows):
    """UnsafeRowSerializer framing of the rows"""
    return b"".join(len(r).to_bytes(4, "big") + bytes(r) for r in rows)


def parse(buf):
    """decoded stream -> [(offset, record length)]"""
    out, p = [], 0
    while p < len(buf):
        s = int.from_bytes(buf[p:p + 4], "big")
        out.append((p, 4 + s))
        p += 4 + s
    assert p == len(buf)
    return out


def blocks_of(rows, sizes):
    out, at = [], 0
    for s in sizes:
        out.append(stream(rows[at:at + s]))
        at += s
    assert at == len(rows)
    return out


def build_blocks(capi, codec, level, alg, plain):
    """one compressed stream per block, one slice per block -> (arena, off, len, slice_base, slice_len, slice_ck)"""
    n = len(plain)
    lens = np.array([len(b) for b in plain], dtype=np.uint64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64) if n else np.zeros(0, np.uint64)
    src = np.frombuffer(b"".join(plain), np.uint8) if lens.sum() else np.zeros(1, np.uint8)
    if codec == 0:
        arena, off, ln = src, offs, lens
    else:
        bound = sum(capi.compress_bound(codec, 0, int(l)) for l in lens) + 64
        dst = np.zeros(bound, np.uint8)
        r = capi.compress_packed(codec, src, offs, lens, dst, 0, 0, level)
        assert (r["status"] == 0).all()
        arena, off, ln = dst[: max(r["total"], 1)], r["dst_off"], r["dst_len"]
    ck = capi.checksum_packed(alg, arena, off, ln) if alg and n else np.zeros(n, np.uint64)
    return arena, off, ln, np.arange(n + 1, dtype=np.uint32), np.array(ln, dtype=np.uint64), ck


# ---------------------------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------------------------
def is_null(row, f):
    return f >= 0 and (int.from_bytes(row[8 * (f >> 6):8 * (f >> 6) + 8], "little") >> (f & 63)) & 1


def f64(b):
    return struct.unpack("<d", b)[0]


def dkey(b):
    """Spark SQL's double order: -0.0 == 0.0, NaN == NaN above everything"""
    x = f64(b)
    if math.isnan(x):
        return (1, 0.0)
    return (0, x + 0.0)


def merge(op, vals):
    """vals: the non-null 8-byte slots of a group in stable order -> the result slot"""
    if op == SUM_I64:
        return (sum(int.from_bytes(v, "little") for v in vals) % 2**64).to_bytes(8, "little")
    if op == SUM_F64:
        s = 0.0
        for v in vals:
            s = s + f64(v)
        return struct.pack("<d", s)
    if op in (MIN_I32, MAX_I32):
        key = [int.from_bytes(v[:4], "little", signed=True) for v in vals]
    elif op in (MIN_I64, MAX_I64):
        key = [int.from_bytes(v, "little", signed=True) for v in vals]
    else:
        key = [dkey(v) for v in vals]
    best = 0
    for k in range(1, len(vals)):
        if (key[k] > key[best]) if op in (MAX_I32, MAX_I64, MAX_F64) else (key[k] < key[best]):
            best = k
    return vals[best][:4] + bytes(4) if op in (MIN_I32, MAX_I32) else vals[best]


def col_value(row, col):
    """one key column (type, offset, length, null field) of a row -> (not-null flag, value)"""
    kt, ko, kl, nf = col
    if nf >= 0 and is_null(row, nf):
        return (0, b"" if kt in (KEY_BYTES, STRING) else 0)
    if kt == STRING:
        slot = int.from_bytes(row[ko:ko + 8], "little")
        o, s = slot >> 32, slot & 0xFFFFFFFF
        return (1, bytes(row[o:o + s]))
    k = bytes(row[ko:ko + kl])
    return (1, k if kt == KEY_BYTES else int.from_bytes(k, "little", signed=True))


def model_keys(plain, keys):
    buf = b"".join(plain)
    recs = parse(buf)
    kv = [tuple(col_value(buf[o + 4:o + ln], c) for c in keys) for o, ln in recs]
    order = sorted(range(len(recs)), key=lambda i: kv[i])  # stable
    return buf, recs, kv, order


def model_sort(plain, keys):
    """-> (the records of the decoded blocks in key order, number of records)"""
    buf, recs, _, order = model_keys(plain, keys)
    return b"".join(buf[recs[i][0]:recs[i][0] + recs[i][1]] for i in order), len(recs)


def model_aggregate(plain, keys, aggs):
    """the first record of each group in key order, every aggregate (op, off, null field) merged over the group in
    that order -> (rows, number of records, number of groups)"""
    buf, recs, kv, order = model_keys(plain, keys)
    out, j = [], 0
    while j < len(order):
        e = j
        while e < len(order) and kv[order[e]] == kv[order[j]]:
            e += 1
        o, ln = recs[order[j]]
        rec = bytearray(buf[o:o + ln])
        row = memoryview(rec)[4:]
        nulls = []
        for op, off, anf in aggs:
            vals = []
            for i in order[j:e]:
                r = buf[recs[i][0] + 4:recs[i][0] + recs[i][1]]
                if not is_null(r, anf):
                    vals.append(bytes(r[off:off + 8]))
            row[off:off + 8] = merge(op, vals) if vals else bytes(8)
            nulls.append((anf, not vals))
        for anf, null in nulls:
            if anf >= 0:
                w = 8 * (anf >> 6)
                v = int.from_bytes(row[w:w + 8], "little")
                v = v | (1 << (anf & 63)) if null else v & ~(1 << (anf & 63))
                row[w:w + 8] = v.to_bytes(8, "little")
        out.append(bytes(rec))
        j = e
    return b"".join(out), len(recs), len(out)


# ---------------------------------------------------------------------------------------------------------------
# the calls
# ---------------------------------------------------------------------------------------------------------------
def run(capi, name, codec, alg, blocks, args, cap, dev=False):
    """capi.<name>_packed, or <name>_dev from and into device memory, over blocks with the family's own arguments
    args, into a cap-byte output -> (output bytes, result dict).  A sort that reads no records outputs b""."""
    arena, off, ln, sb, sl, sc = blocks
    whole = "aggregate" in name
    if not dev:
        dst = np.zeros(max(cap, 1), np.uint8)
        r = getattr(capi, name + "_packed")(codec, arena, off, ln, dst[:cap], *args, alg, sb, sl, sc)
        return dst[: r["total"]].tobytes() if whole or r["n_records"] else b"", r
    d_src = capi.dev_alloc(max(arena.size, 1))
    d_dst = capi.dev_alloc(max(cap, 1))
    try:
        capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        r = getattr(capi, name + "_dev")(codec, d_src, off, ln, d_dst, cap, *args, alg, sb, sl, sc)
        out = np.zeros(max(r["total"], 1), np.uint8)
        if (whole or r["n_records"]) and r["total"]:
            capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        return out[: r["total"]].tobytes() if whole or r["n_records"] else b"", r
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)


# ---------------------------------------------------------------------------------------------------------------
# the host mirror
# ---------------------------------------------------------------------------------------------------------------
def mirror(tmp_path, codec, **extra):
    """a dispatcher over file:// storage under tmp_path: CRC32C checksums, LZ4 unless codec is "none", then extra"""
    conf = {
        "spark.app.id": "app-" + uuid.uuid4().hex[:12],
        "spark.shuffle.s3.rootDir": "file://" + str(tmp_path) + "/spark-s3-shuffle",
        "spark.shuffle.checksum.enabled": True,
        "spark.shuffle.checksum.algorithm": "CRC32C",
        "spark.io.compression.codec": "lz4",
        "spark.shuffle.compress": codec != "none",
    }
    conf.update(extra)
    return pkg.host.S3ShuffleDispatcher(conf)


def write_maps(host, d, maps, R):
    """maps[m] = (rows, reduce ids): map m's rows through the serialized writer, each framed as UnsafeRowSerializer's"""
    for m, (rows, ids) in enumerate(maps):
        w = host.S3SerializedShuffleWriter(d, 0, m, R)
        for row, p in zip(rows, ids):
            w.insertRecord(int(p), len(row).to_bytes(4, "big") + row)
        w.commit()
        w.close()
