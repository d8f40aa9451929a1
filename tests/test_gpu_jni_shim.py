"""Every native of jni/b200shuffle_jni.c that reaches the device, run through the stand-in JNIEnv (tests/jni_shim.py)
in both critical-region modes and compared with the same call through capi: the return code, every output array, the
destination bytes [0, total) and b2s_last_error() must be identical, and the env must record no violation.  Each
family is also compared once with its Python model, so an error shared by the two marshallings cannot hide."""
import os
import re
import subprocess
import sys
import threading
import zlib

import numpy as np
import pytest

import hash_model as hm
import range_model as rg
import jni_shim
import spark_s3_shuffle_b200 as pkg
from join_model import model_join
from rows_model import blocks_of, build_blocks, model_aggregate, model_sort
from test_gpu_exchange_rows import decimal_rows, join_rows, q67_rows, sources, store, window_rows
from test_gpu_join_rows import kinds
from window_model import model_window

pytestmark = pytest.mark.gpu

c = pkg.capi
MODES = jni_shim.MODES
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def shim(capi):
    s = jni_shim.load()
    # the shim is bound to the library instance capi initialised
    n = s.call("deviceCount").rc
    assert n == capi.load().b2s_device_count() and n != c.E_NOT_INIT and n >= 1
    return s


def jcall(shim, mode, name, **kw):
    return shim.call(name, mode=mode, **kw)


def capi_call(fn, *a, **k):
    """-> (rc, result dict or None, b2s_last_error) of a capi helper"""
    try:
        r = fn(*a, **k)
        return 0, r, c.load().b2s_last_error()
    except c.B2SError as e:
        return e.code, None, c.load().b2s_last_error()


def i64(a):
    return None if a is None else np.ascontiguousarray(a).astype(np.uint64).view(np.int64)


def i32(a):
    return None if a is None else np.ascontiguousarray(a).astype(np.int64).astype(np.int32)


def same(r, rc, ref, err, pairs, dst_j=None, dst_c=None, total=None):
    """the JNI result r equals capi's (rc, ref, err): pairs = [(JNI array, index or slice, capi key)]"""
    assert r.rc == rc, (r.rc, rc)
    assert c.load().b2s_last_error() == err
    if rc != 0 or ref is None:
        return
    for arr, sl, key in pairs:
        got = r.arrays[arr][sl]
        want = np.asarray(ref[key])
        assert (got.astype(np.int64) == want.astype(np.uint64).view(np.int64) if want.dtype == np.uint64 else
                got == want).all(), key
    if dst_j is not None:
        assert bytes(dst_j[:total]) == bytes(dst_c[:total])


# ---------------------------------------------------------------------------------------------------------------
# write side
# ---------------------------------------------------------------------------------------------------------------
def parts_of(rng, n):
    parts = [rng.integers(0, 8, int(rng.integers(0, 5000)), dtype=np.uint8).tobytes() for _ in range(n)]
    src = np.frombuffer(b"".join(parts) or b"\0", np.uint8).copy()
    ln = np.array([len(p) for p in parts], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    return parts, src, off, ln


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("codec", [1, 2, 3])
@pytest.mark.parametrize("alg", [0, 1, 2, 3])
def test_compress_packed(shim, oracle, mode, codec, alg):
    parts, src, off, ln = parts_of(np.random.default_rng(codec * 4 + alg), 9)
    cap = sum(c.compress_bound(codec, 0, int(x)) for x in ln) + 64
    dj, dc = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    n = len(parts)
    r = jcall(shim, mode, "compressPacked", codec=codec, level=1 if codec == 3 else 0, blockSize=0, alg=alg, n=n,
              src=src.ctypes.data, off=i64(off), len=i64(ln), dst=dj.ctypes.data, dstCap=cap,
              dstOff=np.zeros(n, np.int64), dstLen=np.zeros(n, np.int64), meta=np.zeros(1, np.int64),
              checksums=np.zeros(n, np.int64), status=np.zeros(n, np.int32))
    err = c.load().b2s_last_error()
    rc, ref, cerr = capi_call(c.compress_packed, codec, src, off, ln, dc, 0, alg, 1 if codec == 3 else 0)
    assert err == cerr
    same(r, rc, ref, cerr, [("dstOff", slice(None), "dst_off"), ("dstLen", slice(None), "dst_len"),
                            ("checksums", slice(None), "checksums"), ("status", slice(None), "status")],
         dj, dc, ref["total"])
    assert r.arrays["meta"][0] == ref["total"]
    if codec == 1 and alg == 3:  # the model: the oracle decodes every stream, and CRC32C is over the stream
        for i, p in enumerate(parts):
            s = bytes(dj[r.arrays["dstOff"][i]:r.arrays["dstOff"][i] + r.arrays["dstLen"][i]])
            assert oracle.lz4block_decompress(s) == p and r.arrays["checksums"][i] == oracle.crc32c(s)


def part_out(R, checksums=True):
    return dict(dstOff=np.zeros(R, np.int64), dstLen=np.zeros(R, np.int64), meta=np.zeros(1, np.int64),
                checksums=np.zeros(R, np.int64) if checksums else None, status=np.zeros(R, np.int32))


PART_PAIRS = [("dstOff", slice(None), "dst_off"), ("dstLen", slice(None), "dst_len"),
              ("checksums", slice(None), "checksums"), ("status", slice(None), "status")]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cached", [False, True])
def test_partition_compress_packed(shim, capi, mode, cached):
    rng = np.random.default_rng(3)
    recs = [rng.integers(0, 4, int(rng.integers(1, 200)), dtype=np.uint8).tobytes() for _ in range(500)]
    buf = np.frombuffer(b"".join(recs), np.uint8).copy()
    rl = np.array([len(x) for x in recs], np.uint32)
    R = 7
    rp = rng.integers(0, R, len(recs)).astype(np.uint32)
    cap = c.partition_compress_bound(1, 0, R, buf.size) + 64
    dj, dc = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    common = dict(codec=1, level=0, blockSize=0, alg=3, numPartitions=R, nRecords=len(recs), records=buf.ctypes.data,
                  recBytes=buf.size, recLen=rl.ctypes.data, recPart=rp.ctypes.data, dst=dj.ctypes.data, dstCap=cap,
                  **part_out(R))
    if cached:
        capi.exchange_set_budget(1 << 30)
        r = jcall(shim, mode, "partitionCompressCachedPacked", shuffleId=40, mapId=1, cached=np.zeros(1, np.int32),
                  **common)
        capi.exchange_remove(40, -1)
        rc, ref, err = capi_call(c.partition_compress_cached_packed, 40, 1, 1, buf, rl, rp, R, dc, 0, 3)
        capi.exchange_remove(40, -1)
        assert r.arrays["cached"][0] == ref["cached"] == 1
    else:
        r = jcall(shim, mode, "partitionCompressPacked", **common)
        rc, ref, err = capi_call(c.partition_compress_packed, 1, buf, rl, rp, R, dc, 0, 3)
    same(r, rc, ref, err, PART_PAIRS, dj, dc, ref["total"])
    assert r.arrays["meta"][0] == ref["total"]


def key_kw(keys):
    n, kt, ko, kl, kn = c._key_arrays(keys)
    return dict(nKeys=n, keyType=i32(kt), keyOff=i32(ko), keyLen=i32(kl), keyNullField=i32(kn))


def bounds_kw(bounds):
    nb, bb, bbytes, bl = c._bound_arrays(bounds)
    return dict(nBounds=nb, bounds=bb.ctypes.data, boundBytes=bbytes, boundLen=i32(bl)[:nb]), bb


ROW_KINDS = ["hash", "range", "round_robin"]
NATIVE = {"hash": "partitionCompressRowsHash", "range": "partitionCompressRowsRange",
          "round_robin": "partitionCompressRowsRoundRobin"}


def row_writer(shim, mode, kind, rows, keys, R, cached, cap=None, shuffle=41, map_id=2):
    """one map task through the JNI row writer and through capi -> (JNI result, capi rc, capi result, its error, dst
    pair)"""
    buf, rl = hm.records_of(rows)
    if cap is None:
        cap = c.partition_compress_bound(2, 0, R, buf.size) + 64
    dj, dc = np.zeros(max(cap, 1), np.uint8), np.zeros(max(cap, 1), np.uint8)
    kw = dict(codec=2, level=0, blockSize=0, alg=3, nRecords=len(rows), records=buf.ctypes.data, recBytes=buf.size,
              recLen=rl.ctypes.data, dst=dj.ctypes.data, dstCap=cap)
    keep = None
    if kind == "hash":
        kw.update(numPartitions=R, **key_kw(keys))
        args = (buf, rl, keys, R)
    elif kind == "range":
        bounds = ([rg.framed(b) for b in rg.draw_bounds(np.random.default_rng(7), rows, keys, R, sample=500)]
                  if R > 1 else [])
        bkw, keep = bounds_kw(bounds)
        kw.update(**key_kw(keys), **bkw)
        args = (buf, rl, keys, bounds)
    else:
        kw.update(numPartitions=R, startPosition=R - 1, sortRows=1)
        args = (buf, rl, R, R - 1, 1)
    f = "partition_compress_rows_" + kind
    kw.update(part_out(R))
    if cached:
        kw["cached"] = np.zeros(1, np.int32)
        r = jcall(shim, mode, NATIVE[kind] + "CachedPacked", shuffleId=shuffle, mapId=map_id, **kw)
        c.exchange_remove(shuffle, map_id)
        rc, ref, err = capi_call(getattr(c, f + "_cached_packed"), shuffle, map_id, 2, *args, dc[:cap], 0, 3)
        c.exchange_remove(shuffle, map_id)
        if ref is not None:
            assert r.arrays["cached"][0] == ref["cached"]
    else:
        r = jcall(shim, mode, NATIVE[kind] + "Packed", **kw)
        rc, ref, err = capi_call(getattr(c, f + "_packed"), 2, *args, dc[:cap], 0, 3)
    del keep
    return r, rc, ref, err, dj, dc


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ROW_KINDS)
@pytest.mark.parametrize("cached", [False, True])
@pytest.mark.parametrize("R", [1, 65537])
def test_partition_compress_rows(shim, capi, mode, kind, cached, R):
    rows, keys = join_rows(np.random.default_rng(5), 300)
    capi.exchange_set_budget(1 << 30)
    if kind == "range" and R > 1:
        R = 5  # nBounds = R - 1 bound rows drawn from the input
    r, rc, ref, err, dj, dc = row_writer(shim, mode, kind, rows, keys, R, cached)
    same(r, rc, ref, err, PART_PAIRS, dj, dc, ref["total"])
    assert rc == 0 and r.arrays["meta"][0] == ref["total"]
    if cached:
        assert r.arrays["cached"][0] == 1


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ROW_KINDS)
def test_partition_compress_rows_dst_too_small(shim, capi, mode, kind):
    rows, keys = join_rows(np.random.default_rng(6), 200)
    r, rc, ref, err, dj, dc = row_writer(shim, mode, kind, rows, keys, 3, False, cap=64)
    assert r.rc == rc == c.E_DST_TOO_SMALL and c.load().b2s_last_error() == err
    # the shim still reports the arena bytes needed, and which partitions did not fit
    assert r.arrays["meta"][0] > 64 and (r.arrays["status"] == c.E_DST_TOO_SMALL).any()


@pytest.mark.parametrize("mode", MODES)
def test_partition_compress_range_no_bounds(shim, capi, mode):
    rows, keys = join_rows(np.random.default_rng(8), 100)
    buf, rl = hm.records_of(rows)
    cap = c.partition_compress_bound(2, 0, 1, buf.size) + 64
    dj, dc = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    r = jcall(shim, mode, "partitionCompressRowsRangePacked", codec=2, level=0, blockSize=0, alg=3,
              nRecords=len(rows), records=buf.ctypes.data, recBytes=buf.size, recLen=rl.ctypes.data, **key_kw(keys),
              nBounds=0, bounds=0, boundBytes=0, boundLen=None, dst=dj.ctypes.data, dstCap=cap, **part_out(1))
    rc, ref, err = capi_call(c.partition_compress_rows_range_packed, 2, buf, rl, keys, [], dc, 0, 3)
    same(r, rc, ref, err, PART_PAIRS, dj, dc, ref["total"])


# ---------------------------------------------------------------------------------------------------------------
# read side
# ---------------------------------------------------------------------------------------------------------------
def compressed(n, seed=0, codec=1):
    if n == 0:
        return [], np.zeros(1, np.uint8), np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.uint64)
    parts, src, off, ln = parts_of(np.random.default_rng(seed), n)
    cap = sum(c.compress_bound(codec, 0, int(x)) for x in ln) + 64
    dst = np.zeros(cap, np.uint8)
    r = c.compress_packed(codec, src, off, ln, dst, 0, 3)
    return parts, dst, r["dst_off"], r["dst_len"], r["checksums"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 600])
def test_decompressed_size_packed(shim, mode, n):
    parts, arena, off, ln, _ = compressed(n, seed=n)
    r = jcall(shim, mode, "decompressedSizePacked", codec=1, n=n, src=arena.ctypes.data, off=i64(off), len=i64(ln),
              outLen=np.zeros(n, np.int64), status=np.zeros(n, np.int32))
    assert r.rc == 0
    sizes, st = c.decompressed_size_batch(1, [arena[o:o + l] for o, l in zip(off, ln)])
    assert list(r.arrays["outLen"]) == sizes == [len(p) for p in parts]  # the model: the plain sizes
    assert list(r.arrays["status"]) == st == [0] * n


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("alg", [1, 2, 3])
def test_checksum_packed(shim, mode, alg):
    parts, arena, off, ln, _ = compressed(40, seed=alg)
    r = jcall(shim, mode, "checksumPacked", alg=alg, n=len(off), base=arena.ctypes.data, off=i64(off), len=i64(ln),
              out=np.zeros(len(off), np.int64))
    assert r.rc == 0
    assert (r.arrays["out"].view(np.uint64) == c.checksum_packed(alg, arena, off, ln)).all()
    if alg == 2:  # the model
        assert list(r.arrays["out"]) == [zlib.crc32(bytes(arena[o:o + l])) for o, l in zip(off, ln)]


def batch_blocks(seed=1):
    """blocks of several slices each (ShuffleBlockBatchId): block i is the streams of partitions GROUPS[i] back to back
    -> (plain per block, arena, off, len, sliceBase, sliceLen, sliceChecksum)"""
    groups = [[0, 1], [2], [3, 4, 5], [6]]
    parts, arena, soff, sln, sck = compressed(7, seed=seed)
    blocks = [b"".join(bytes(arena[soff[p]:soff[p] + sln[p]]) for p in g) for g in groups]
    src = np.frombuffer(b"".join(blocks), np.uint8).copy()
    ln = np.array([len(b) for b in blocks], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    sb = np.array(np.cumsum([0] + [len(g) for g in groups]), np.uint32)
    plain = [b"".join(parts[p] for p in g) for g in groups]
    return plain, src, off, ln, sb, np.array(sln, np.uint64), np.array(sck, np.uint64)


def decompress_both(shim, mode, src, off, ln, sb, sl, sc, cap, alg=3):
    n = len(off)
    dj, dc = np.zeros(max(cap, 1), np.uint8), np.zeros(max(cap, 1), np.uint8)
    r = jcall(shim, mode, "decompressPacked", codec=1, alg=alg, n=n, src=src.ctypes.data, off=i64(off), len=i64(ln),
              sliceBase=i32(sb), sliceLen=i64(sl), sliceChecksum=i64(sc), dst=dj.ctypes.data, dstCap=cap,
              dstOff=np.zeros(n, np.int64), dstLen=np.zeros(n, np.int64), meta=np.zeros(1, np.int64),
              status=np.zeros(n, np.int32), badSlice=np.zeros(n, np.int32))
    rc, ref, err = capi_call(c.decompress_packed, 1, src, off, ln, dc[:cap], alg, sb, sl, sc)
    pairs = [("dstOff", slice(None), "dst_off"), ("dstLen", slice(None), "dst_len"), ("status", slice(None), "status"),
             ("badSlice", slice(None), "bad_slice")]
    same(r, rc, ref, err, pairs, dj, dc, ref["total"] if ref else 0)
    return r, ref, dj


@pytest.mark.parametrize("mode", MODES)
def test_decompress_packed(shim, mode):
    plain, src, off, ln, sb, sl, sc = batch_blocks()
    r, ref, dj = decompress_both(shim, mode, src, off, ln, sb, sl, sc, sum(len(p) for p in plain))
    assert r.rc == 0 and list(r.arrays["status"]) == [0] * len(plain)
    for i, p in enumerate(plain):  # the model: the plain bytes of each block
        assert bytes(dj[r.arrays["dstOff"][i]:r.arrays["dstOff"][i] + r.arrays["dstLen"][i]]) == p


@pytest.mark.parametrize("mode", MODES)
def test_decompress_packed_errors(shim, mode):
    plain, src, off, ln, sb, sl, sc = batch_blocks(seed=2)
    total = sum(len(p) for p in plain)
    bad = sc.copy()
    bad[4] ^= 1  # block 2's second slice
    r, _, _ = decompress_both(shim, mode, src, off, ln, sb, sl, bad, total)
    assert r.arrays["status"][2] == c.E_CHECKSUM and r.arrays["badSlice"][2] == 1
    corrupt = src.copy()
    corrupt[int(off[1]):int(off[1] + ln[1])] = 0xFF
    r, _, _ = decompress_both(shim, mode, corrupt, off, ln, sb, sl, sc, total, alg=0)
    assert r.arrays["status"][1] == c.E_CORRUPT
    r, _, _ = decompress_both(shim, mode, src, off, ln, sb, sl, sc, 16)
    assert r.rc == c.E_DST_TOO_SMALL or (r.arrays["status"] == c.E_DST_TOO_SMALL).any()


# ---------------------------------------------------------------------------------------------------------------
# row calls
# ---------------------------------------------------------------------------------------------------------------
def block_kw(blocks, alg, n=None):
    arena, off, ln, sb, sl, sc = blocks
    n = len(off) if n is None else n
    return dict(alg=alg, n=n, src=arena.ctypes.data, off=i64(off), len=i64(ln),
                sliceBase=i32(sb) if alg else None, sliceLen=i64(sl) if alg else None,
                sliceChecksum=i64(sc) if alg else None, status=np.zeros(n, np.int32), badSlice=np.zeros(n, np.int32))


SORT_PAIRS = [("status", slice(None), "status"), ("badSlice", slice(None), "bad_slice")]
META = {2: ("total", "n_records"), 3: ("total", "n_records", "n_groups")}


def rows_both(shim, mode, native, capi_name, codec, alg, blocks, jargs, cargs, n_meta, cap):
    """native over blocks through JNI (its own arguments jargs) and capi_name through capi (cargs) -> (JNI result, capi
    result, JNI output bytes)"""
    arena, off, ln, sb, sl, sc = blocks
    dj, dc = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    r = jcall(shim, mode, native, codec=codec, dst=dj.ctypes.data, dstCap=cap, meta=np.zeros(n_meta, np.int64),
              **block_kw(blocks, alg), **jargs)
    rc, ref, err = capi_call(getattr(c, capi_name), codec, arena, off, ln, dc, *cargs, alg, sb, sl, sc)
    same(r, rc, ref, err, SORT_PAIRS, dj, dc, ref["total"] if ref else 0)
    if ref is not None:
        names = META.get(n_meta) or (("total", "n_left_records", "n_right_records", "n_out_records") if n_meta == 4
                                     else ("total", "n_records", "n_out_records"))
        names = ("total", "n_records", "n_out_records") if "window" in capi_name else names
        assert list(r.arrays["meta"]) == [ref[k] for k in names]
    return r, ref, dj[: r.arrays["meta"][0]].tobytes()


def row_blocks(rows, alg, codec=2, sizes=None):
    sizes = sizes or [len(rows) // 3, len(rows) // 3, len(rows) - 2 * (len(rows) // 3)]
    plain = blocks_of(rows, sizes)
    return plain, build_blocks(c, codec, 0, alg, plain)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("alg", [0, 3])
def test_sort_and_aggregate_rows(shim, capi, mode, alg):
    rng = np.random.default_rng(11)
    rows, keys, aggs = q67_rows(rng, 400)
    plain, blocks = row_blocks(rows, alg)
    cap = sum(len(p) for p in plain) + 64
    r, _, out = rows_both(shim, mode, "decompressSortRowsKeysPacked", "decompress_sort_rows_keys_packed", 2, alg,
                          blocks, key_kw(keys), (keys,), 2, cap)
    assert out == model_sort(plain, keys)[0]  # the model
    n, op, ao, an = c._agg_arrays(aggs)
    agg_kw = dict(nAggs=n, aggOp=i32(op), aggOff=i32(ao), aggNullField=i32(an))
    r, _, out = rows_both(shim, mode, "decompressAggregateRowsKeysPacked", "decompress_aggregate_rows_keys_packed", 2,
                          alg, blocks, {**key_kw(keys), **agg_kw}, (keys, aggs), 3, cap)
    assert out == model_aggregate(plain, keys, aggs)[0]
    # the one-key forms, by the INT32 column 2 (null bit 2)
    k1 = keys[2]
    one = dict(keyType=k1[0], keyOff=k1[1], keyLen=k1[2], nullField=k1[3])
    rows_both(shim, mode, "decompressSortRowsPacked", "decompress_sort_rows_packed", 2, alg, blocks, one,
              (k1[0], k1[1], k1[2], k1[3]), 2, cap)
    rows_both(shim, mode, "decompressAggregateRowsPacked", "decompress_aggregate_rows_packed", 2, alg, blocks,
              {**one, **agg_kw}, (k1[0], k1[1], k1[2], k1[3], aggs), 3, cap)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("alg", [0, 3])
def test_aggregate_rows_decimal(shim, capi, mode, alg):
    rows, keys, aggs = decimal_rows(np.random.default_rng(12), 300)
    plain, blocks = row_blocks(rows, alg)
    n, op, ao, an = c._agg_arrays(aggs)
    assert op[0] >> 8 == 28  # a decimal sum with its precision bits
    rows_both(shim, mode, "decompressAggregateRowsKeysPacked", "decompress_aggregate_rows_keys_packed", 2, alg, blocks,
              {**key_kw(keys), "nAggs": n, "aggOp": i32(op), "aggOff": i32(ao), "aggNullField": i32(an)},
              (keys, aggs), 3, sum(len(p) for p in plain) + 64)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("alg", [0, 3])
def test_sort_fixed_records(shim, capi, mode, alg):
    rng = np.random.default_rng(13)
    plain = [rng.integers(0, 256, 16 * k, dtype=np.uint8).tobytes() for k in (50, 0, 77)]
    blocks = build_blocks(c, 1, 0, alg, plain)
    _, _, out = rows_both(shim, mode, "decompressSortPacked", "decompress_sort_packed", 1, alg, blocks,
                          dict(recordBytes=16, keyOff=2, keyLen=5), (16, 2, 5), 2, 16 * 127 + 64)
    recs = [b"".join(plain)[i:i + 16] for i in range(0, 16 * 127, 16)]
    assert out == b"".join(sorted(recs, key=lambda x: x[2:7]))


JOINS = [c.JOIN_INNER, c.JOIN_LEFT_OUTER, c.JOIN_LEFT_SEMI, c.JOIN_LEFT_ANTI, c.JOIN_RIGHT_OUTER, c.JOIN_FULL_OUTER]


def join_both(shim, mode, jt, alg, seed=14):
    rng = np.random.default_rng(seed)
    left, keys = join_rows(rng, 200)
    right, _ = join_rows(rng, 150)
    plain = blocks_of(left, [100, 100]) + blocks_of(right, [150])
    blocks = build_blocks(c, 3, 1, alg, plain)
    semi = jt in (c.JOIN_LEFT_SEMI, c.JOIN_LEFT_ANTI)
    kd = None if semi else kinds(["long", "int", "string"])
    n, kt, kl, lo, ln, ro, rn, lk, rk = c._join_arrays(keys, keys, kd, kd)
    cap = 1 << 20
    arena, off, length, sb, sl, sc = blocks
    dj, dc = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    r = jcall(shim, mode, "decompressJoinRowsKeysPacked", joinType=jt, codec=3, nLeft=2, dst=dj.ctypes.data,
              dstCap=cap, meta=np.zeros(4, np.int64), nKeys=n, keyType=i32(kt), keyLen=i32(kl), leftKeyOff=i32(lo),
              leftKeyNullField=i32(ln), rightKeyOff=i32(ro), rightKeyNullField=i32(rn), nLeftFields=3,
              leftFieldKind=None if lk is None else lk.view(np.int8), nRightFields=3,
              rightFieldKind=None if rk is None else rk.view(np.int8), **block_kw(blocks, alg))
    rc, ref, err = capi_call(c.decompress_join_rows_keys_packed, jt, 3, arena, off, length, 2, dc, keys, keys, 3, 3,
                             kd, kd, alg, sb, sl, sc)
    same(r, rc, ref, err, SORT_PAIRS, dj, dc, ref["total"] if ref else 0)
    assert rc == 0
    assert list(r.arrays["meta"]) == [ref[k] for k in ("total", "n_left_records", "n_right_records", "n_out_records")]
    return r, dj[: r.arrays["meta"][0]].tobytes(), plain, keys, kd


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("jt", JOINS)
@pytest.mark.parametrize("alg", [0, 3])
def test_join_rows(shim, capi, mode, jt, alg):
    r, out, plain, keys, kd = join_both(shim, mode, jt, alg)
    if jt in (c.JOIN_INNER, c.JOIN_LEFT_SEMI):  # the model
        assert out == model_join(jt, plain[:2], plain[2:], keys, keys, 3, 3, kd, kd)[0]


WIN_TYPES = ["int", "string", "decimal", "long"]


def window_both(shim, mode, native, alg, fns, limit=None, seed=15):
    rows, keys = window_rows(np.random.default_rng(seed), 300)
    plain, blocks = row_blocks(rows, alg)
    kd = kinds(WIN_TYPES)
    cap = 1 << 20
    arena, off, ln, sb, sl, sc = blocks
    dj, dc = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    if native == "decompressWindowRowsKeysPacked":
        npk, n, kt, ko, kl, kn, nf, kk, nfn, fn, arg, limit_fn, lim = c._window_arrays(keys, 0, 4, kd, fns, limit)
        extra = dict(limitFn=int(np.int32(np.uint32(limit_fn))), limit=lim)
        cargs = (keys, 0, 4, kd, fns, limit)
        capi_fn = c.decompress_window_rows_keys_packed
    else:
        offset = native == "decompressWindowOffsetRowsKeysPacked"
        a = c._window_aggregate_arrays(keys, 0, 4, kd, fns, offset)
        npk, n, kt, ko, kl, kn, nf, kk, nfn, fn, arg, fr, vt, vo, vn = a[:15]
        extra = dict(fnFrame=i32(fr), valType=i32(vt), valOff=i32(vo), valNullField=i32(vn))
        if offset:
            extra.update(fnFlags=i32(a[15]), fnDefault=i64(a[16]))
        cargs = (keys, 0, 4, kd, fns)
        capi_fn = (c.decompress_window_offset_rows_keys_packed if offset else
                   c.decompress_window_aggregate_rows_keys_packed)
    r = jcall(shim, mode, native, codec=2, dst=dj.ctypes.data, dstCap=cap, meta=np.zeros(3, np.int64),
              nPartitionKeys=npk, nKeys=n, keyType=i32(kt), keyOff=i32(ko), keyLen=i32(kl), keyNullField=i32(kn),
              nFields=nf, fieldKind=kk.view(np.int8), nFns=nfn, fn=i32(fn), fnArg=i32(arg), **extra,
              **block_kw(blocks, alg))
    rc, ref, err = capi_call(capi_fn, 2, arena, off, ln, dc, *cargs, alg, sb, sl, sc)
    same(r, rc, ref, err, SORT_PAIRS, dj, dc, ref["total"] if ref else 0)
    assert rc == 0
    assert list(r.arrays["meta"]) == [ref[k] for k in ("total", "n_records", "n_out_records")]
    return r, dj[: r.arrays["meta"][0]].tobytes(), plain, keys, kd


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("alg", [0, 3])
@pytest.mark.parametrize("limit", [None, (c.WINDOW_RANK, 5)])
def test_window_rows(shim, capi, mode, alg, limit):
    # a limit takes only the three limit functions
    fns = ([c.WINDOW_ROW_NUMBER, c.WINDOW_DENSE_RANK, (c.WINDOW_NTILE, 3)] if limit is None else
           [c.WINDOW_ROW_NUMBER, c.WINDOW_RANK, c.WINDOW_DENSE_RANK])
    r, out, plain, keys, kd = window_both(shim, mode, "decompressWindowRowsKeysPacked", alg, fns, limit)
    assert out == model_window(plain, keys, 0, 4, kd, fns, limit)[0]  # the model


def slot(f):
    return 8 + 8 * f


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("alg", [0, 3])
def test_window_aggregate_rows(shim, capi, mode, alg):
    fns = [(c.WINDOW_SUM, c.WINDOW_FRAME_ROWS_RUNNING, c.WINDOW_VAL_INT64, slot(3), -1),
           (c.WINDOW_MAX, c.WINDOW_FRAME_PARTITION, c.window_val_decimal(28, 2), slot(2), 2),
           c.WINDOW_RANK]
    window_both(shim, mode, "decompressWindowAggregateRowsKeysPacked", alg, fns)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("alg", [0, 3])
def test_window_offset_rows(shim, capi, mode, alg):
    fns = [(c.WINDOW_LAG, 2, 0, c.WINDOW_VAL_INT64, slot(3), -1, c.WINDOW_HAS_DEFAULT, (1 << 63) | 5),
           (c.WINDOW_FIRST, 0, c.WINDOW_FRAME_PARTITION, c.WINDOW_VAL_INT32, slot(0), 0, c.WINDOW_IGNORE_NULLS, 0),
           (c.WINDOW_SUM, c.WINDOW_FRAME_RANGE_RUNNING, c.WINDOW_VAL_INT64, slot(3), 3)]
    window_both(shim, mode, "decompressWindowOffsetRowsKeysPacked", alg, fns)


# ---------------------------------------------------------------------------------------------------------------
# exchange cache
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_exchange_cache(shim, capi, mode):
    S = 43
    assert jcall(shim, mode, "exchangeSetBudget", dev=0, bytes=1 << 30).rc == 0
    rng = np.random.default_rng(16)
    rows, keys, aggs = q67_rows(rng, 600)
    maps = [rows[:300], rows[300:]]
    R = 4
    # map 0 cached through the JNI hash writer; map 1 written uncached and fetched
    r, rc, ref, err, dj, _ = row_writer(shim, mode, "hash", maps[0], keys, R, True, shuffle=S + 100, map_id=0)
    assert rc == 0 and r.arrays["cached"][0] == 1
    buf, rl = hm.records_of(maps[0])
    kw = dict(codec=2, level=0, blockSize=0, alg=3, numPartitions=R, nRecords=len(maps[0]), records=buf.ctypes.data,
              recBytes=buf.size, recLen=rl.ctypes.data, **key_kw(keys), dst=dj.ctypes.data, dstCap=dj.size,
              cached=np.zeros(1, np.int32), **part_out(R))
    r0 = jcall(shim, mode, "partitionCompressRowsHashCachedPacked", shuffleId=S, mapId=0, **kw)
    assert r0.rc == 0 and r0.arrays["cached"][0] == 1
    data0 = dj[: r0.arrays["meta"][0]].copy()
    m1 = store(capi, "hash", S, 1, maps[1], keys, R, cached=False)
    ids = np.array([0, 1], np.int64)
    lk = jcall(shim, mode, "exchangeLookup", shuffleId=S, startReduce=1, endReduce=3, n=2, mapIds=ids,
               len=np.zeros(2, np.int64))
    hits, lens = capi.exchange_lookup(S, 1, 3, ids)
    assert lk.rc == hits == 1 and (lk.arrays["len"].view(np.uint64) == lens).all() and lens[1] == c.NOT_RESIDENT
    dj, dc = np.zeros(1 << 20, np.uint8), np.zeros(1 << 20, np.uint8)
    rd = jcall(shim, mode, "exchangeReadPacked", shuffleId=S, startReduce=1, endReduce=3, n=1, mapIds=ids[:1],
               dst=dj.ctypes.data, dstCap=dj.size, dstOff=np.zeros(1, np.int64), dstLen=np.zeros(1, np.int64),
               meta=np.zeros(1, np.int64), status=np.zeros(1, np.int32))
    rc, ref, err = capi_call(capi.exchange_read_packed, S, 1, 3, ids[:1], dc)
    same(rd, rc, ref, err, [("dstOff", slice(None), "dst_off"), ("dstLen", slice(None), "dst_len"),
                            ("status", slice(None), "status")], dj, dc, ref["total"])
    # the sources of reducer [1, 3): map 0 from the cache, map 1 fetched
    m0 = dict(dst_off=r0.arrays["dstOff"].view(np.uint64), dst_len=r0.arrays["dstLen"].view(np.uint64),
              checksums=r0.arrays["checksums"].view(np.uint64), data=data0)
    blocks = sources([m0, m1], 1, 3)
    src, off, ln, sb, sl, sc = blocks
    cached = np.array([1, 0], np.int32)
    ex = dict(shuffleId=S, startReduce=1, endReduce=3, mapIds=ids, cached=cached, codec=2)
    cap = 1 << 20
    for native, capi_fn, jargs, cargs, n_meta in (
            ("exchangeReadSortRowsKeysPacked", capi.exchange_read_sort_rows_keys_packed, key_kw(keys), (keys,), 2),
            ("exchangeReadAggregateRowsKeysPacked", capi.exchange_read_aggregate_rows_keys_packed,
             {**key_kw(keys), "nAggs": len(aggs), "aggOp": i32([a[0] for a in aggs]),
              "aggOff": i32([a[1] for a in aggs]), "aggNullField": i32([a[2] for a in aggs])}, (keys, aggs), 3)):
        dj, dc = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
        r = jcall(shim, mode, native, **ex, dst=dj.ctypes.data, dstCap=cap, meta=np.zeros(n_meta, np.int64),
                  **jargs, **block_kw(blocks, 3))
        rc, ref, err = capi_call(capi_fn, S, 1, 3, ids, cached, 2, src, off, ln, dc, *cargs, 3, sb, sl, sc)
        same(r, rc, ref, err, SORT_PAIRS, dj, dc, ref["total"])
        assert rc == 0 and r.arrays["meta"][1] == ref["n_records"] > 0
        if native == "exchangeReadSortRowsKeysPacked":  # the model: the plain sort over every map's fetched blocks
            fetched = np.zeros(cap, np.uint8)
            q = capi.decompress_sort_rows_keys_packed(2, src, off, ln, fetched, keys, 3, sb, sl, sc)
            assert dj[: r.arrays["meta"][0]].tobytes() == fetched[: q["total"]].tobytes()
    # the fixed-record exchange read over the same shuffle: a cached map of the serialized writer
    recs = np.random.default_rng(17).integers(0, 256, 16 * 200, dtype=np.uint8)
    rl16 = np.full(200, 16, np.uint32)
    rp = (np.arange(200) % R).astype(np.uint32)
    d2 = np.zeros(c.partition_compress_bound(1, 0, R, recs.size) + 64, np.uint8)
    w = jcall(shim, mode, "partitionCompressCachedPacked", shuffleId=S + 1, mapId=5, codec=1, level=0, blockSize=0,
              alg=3, numPartitions=R, nRecords=200, records=recs.ctypes.data, recBytes=recs.size,
              recLen=rl16.ctypes.data, recPart=rp.ctypes.data, dst=d2.ctypes.data, dstCap=d2.size,
              cached=np.zeros(1, np.int32), **part_out(R))
    assert w.rc == 0 and w.arrays["cached"][0] == 1
    one = np.array([5], np.int64)
    hit = np.array([1], np.int32)
    empty = (np.zeros(1, np.uint8), np.zeros(1, np.uint64), np.zeros(1, np.uint64), np.array([0, 0], np.uint32),
             np.zeros(1, np.uint64), np.zeros(1, np.uint64))
    dj, dc = np.zeros(16 * 200, np.uint8), np.zeros(16 * 200, np.uint8)
    r = jcall(shim, mode, "exchangeReadSortPacked", shuffleId=S + 1, startReduce=0, endReduce=R, mapIds=one,
              cached=hit, codec=1, recordBytes=16, keyOff=0, keyLen=10, dst=dj.ctypes.data, dstCap=dj.size,
              meta=np.zeros(2, np.int64), **block_kw(empty, 3))
    rc, ref, err = capi_call(capi.exchange_read_sort_packed, S + 1, 0, R, one, hit, 1, *empty[:3], dc, 16, 0, 10, 3,
                             *empty[3:])
    same(r, rc, ref, err, SORT_PAIRS, dj, dc, ref["total"])
    recs16 = [recs[i:i + 16].tobytes() for i in range(0, recs.size, 16)]
    assert dj.tobytes() == b"".join(sorted(recs16, key=lambda x: x[:10]))  # the model
    # removal: the next read of the entry is B2S_E_NOT_CACHED
    for s, m in ((S, 0), (S + 1, 5), (S + 100, 0)):
        assert jcall(shim, mode, "exchangeRemove", shuffleId=s, mapId=m).rc >= 0
    r = jcall(shim, mode, "exchangeReadPacked", shuffleId=S, startReduce=1, endReduce=3, n=1, mapIds=ids[:1],
              dst=dj.ctypes.data, dstCap=dj.size, dstOff=np.zeros(1, np.int64), dstLen=np.zeros(1, np.int64),
              meta=np.zeros(1, np.int64), status=np.zeros(1, np.int32))
    assert r.rc == c.E_NOT_CACHED or r.arrays["status"][0] == c.E_NOT_CACHED
    jcall(shim, mode, "exchangeSetBudget", dev=0, bytes=0)


# ---------------------------------------------------------------------------------------------------------------
# lastTiming, short outputs, concurrency, lifecycle
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_last_timing(shim, capi, mode):
    test_checksum_packed(shim, mode, 3)
    r = jcall(shim, mode, "lastTiming", out8=np.zeros(8, np.int64))
    t = capi.last_timing()  # the same thread: the checksum call's timing
    want = [int(t[k] * 1000.0) for k in ("total_ms", "h2d_ms", "d2h_ms", "kernel_ms")] + [
        t[k] for k in ("h2d_bytes", "d2h_bytes", "src_bytes", "dst_bytes")]
    assert r.rc == 0 and list(r.arrays["out8"]) == want and want[6] > 0


@pytest.mark.parametrize("mode", MODES)
def test_short_output_arrays(shim, capi, mode):
    """a short output is B2S_E_ARG with the guards intact (the env checks them), and nothing written"""
    parts, src, off, ln = parts_of(np.random.default_rng(18), 5)
    dst = np.zeros(1 << 16, np.uint8)
    for short in ("dstOff", "dstLen", "checksums", "status", "meta"):
        outs = dict(dstOff=np.full(5, 7, np.int64), dstLen=np.full(5, 7, np.int64), meta=np.full(1, 7, np.int64),
                    checksums=np.full(5, 7, np.int64), status=np.full(5, 7, np.int32))
        outs[short] = outs[short][:-1]
        r = jcall(shim, mode, "compressPacked", codec=1, level=0, blockSize=0, alg=3, n=5, src=src.ctypes.data,
                  off=i64(off), len=i64(ln), dst=dst.ctypes.data, dstCap=dst.size, **outs)
        assert r.rc == c.E_ARG and all((r.arrays[k] == 7).all() for k in outs), short
    rows, keys = join_rows(np.random.default_rng(19), 50)
    plain, blocks = row_blocks(rows, 3)
    kw = block_kw(blocks, 3)
    kw["status"] = kw["status"][:-1]
    r = jcall(shim, mode, "decompressSortRowsKeysPacked", codec=2, dst=dst.ctypes.data, dstCap=dst.size,
              meta=np.zeros(2, np.int64), **key_kw(keys), **kw)
    assert r.rc == c.E_ARG


def test_concurrent_envs(shim, capi):
    """four threads, each with its own env, run the join and window natives at once; each output equals the same call
    run alone"""
    alone = {}
    for k in range(4):
        alone[("join", k)] = join_both(shim, MODES[k % 2], JOINS[k], 3, seed=20 + k)[1]
        alone[("window", k)] = window_both(shim, MODES[k % 2], "decompressWindowRowsKeysPacked", 3,
                                           [c.WINDOW_RANK, (c.WINDOW_NTILE, 4)], seed=30 + k)[1]
    got, errors = {}, []

    def worker(k):
        try:
            for _ in range(3):
                got[("join", k)] = join_both(shim, MODES[k % 2], JOINS[k], 3, seed=20 + k)[1]
                got[("window", k)] = window_both(shim, MODES[k % 2], "decompressWindowRowsKeysPacked", 3,
                                                 [c.WINDOW_RANK, (c.WINDOW_NTILE, 4)], seed=30 + k)[1]
        except BaseException as e:  # noqa: BLE001 - reported below
            errors.append(e)

    ts = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    assert got == alone


WORKER = r"""
import sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import jni_shim
import spark_s3_shuffle_b200 as pkg
c = pkg.capi
c.load()
s = jni_shim.load()
for mode in jni_shim.MODES:
    assert s.call("init", mode=mode, gpuMask=1, pinnedBytesPerGpu=0, streamsPerGpu=0).rc == 0
    assert s.call("deviceCount", mode=mode).rc == 1
    assert s.call("setThreadDevice", mode=mode, dev=0).rc == 0
    assert s.call("bindThreadToDevice", mode=mode, dev=0).rc == 0
    a = s.call("hostAlloc", mode=mode, bytes=1 << 20).rc
    assert a
    buf = s.call("wrap", mode=mode, addr=a, bytes=1 << 20).obj
    assert (buf.address, buf.capacity) == (a, 1 << 20)
    assert s.call("addressOf", mode=mode, directBuffer=buf).rc == a
    plain = np.frombuffer(b"shuffle " * 4000, np.uint8)
    arena = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_uint8 * (1 << 20)).from_address(a))
    arena[:plain.size] = plain
    dst = np.zeros(c.compress_bound(1, 0, plain.size) + 64, np.uint8)
    assert s.call("hostRegister", mode=mode, addr=dst.ctypes.data, bytes=dst.size).rc == 0
    r = s.call("compressPacked", mode=mode, codec=1, level=0, blockSize=0, alg=3, n=1, src=a,
               off=np.zeros(1, np.int64), len=np.array([plain.size], np.int64), dst=dst.ctypes.data, dstCap=dst.size,
               dstOff=np.zeros(1, np.int64), dstLen=np.zeros(1, np.int64), meta=np.zeros(1, np.int64),
               checksums=np.zeros(1, np.int64), status=np.zeros(1, np.int32))
    assert r.rc == 0 and r.arrays["status"][0] == 0 and 0 < r.arrays["meta"][0] < plain.size
    assert s.call("hostUnregister", mode=mode, addr=dst.ctypes.data).rc == 0
    s.call("hostFree", mode=mode, addr=a)
    s.call("shutdown", mode=mode)
    assert s.call("deviceCount", mode=mode).rc == c.E_NOT_INIT
print("lifecycle ok")
"""


LIFECYCLE = ("init", "setThreadDevice", "bindThreadToDevice", "hostAlloc", "wrap", "addressOf", "hostRegister",
             "hostUnregister", "hostFree", "shutdown")


def test_lifecycle_in_a_worker(shim):
    """init, device placement, pinned memory and shutdown through JNI, in a process of their own: shutdown would end
    this session's library"""
    p = subprocess.run([sys.executable, "-c", WORKER, ROOT], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "lifecycle ok" in p.stdout, p.stdout + p.stderr


def test_strings_and_sizes(shim, capi):
    for mode in MODES:
        for code in range(-9, 1):
            assert jcall(shim, mode, "strerror", code=code).string == capi.load().b2s_strerror(code).decode()
        assert jcall(shim, mode, "lastError").string == capi.load().b2s_last_error().decode()
        assert jcall(shim, mode, "compressBound", codec=1, blockSize=0, n=12345).rc == c.compress_bound(1, 0, 12345)


def test_every_native_is_called():
    """every native of the Scala object is called by a test of this file"""
    src = open(os.path.abspath(__file__)).read()
    natives = set(jni_shim.scala_natives())
    called = (set(re.findall(r'"(\w+)"', src)) & natives) | set(LIFECYCLE)
    called |= {NATIVE[k] + form for k in ROW_KINDS for form in ("Packed", "CachedPacked")}
    assert called == natives, natives - called
