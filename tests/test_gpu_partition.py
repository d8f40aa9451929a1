"""Partition + compress in one call (b2s_partition_compress_*): serialized records plus one reduce id per record in,
the .data arena, partition lengths and checksums out.  The model is a numpy stable argsort by partition id followed by
concatenation; the compressed arena must be byte for byte what b2s_compress_packed makes of the model's non-empty
partitions, and every partition must decode, with an independent decoder, back to the model's bytes."""
import ctypes as C
import threading

import numpy as np
import pytest

import zstd_ref
from conftest import corpus

pytestmark = pytest.mark.gpu

REC = 104  # a Kryo-serialized TeraGen record: 2-byte header, 10-byte key, row id and filler (what terasort shuffles)

CODECS = [("lz4", 1, 0), ("snappy", 2, 0), ("zstd1", 3, 1), ("zstd3", 3, 3)]
CHECKSUMS = [0, 1, 2, 3]  # none, ADLER32, CRC32, CRC32C


# ---------------------------------------------------------------------------------------------------------------
# model and helpers
# ---------------------------------------------------------------------------------------------------------------
def terasort(oracle, n_records, seed=0):
    return np.frombuffer(oracle.gen_terasort(seed * 1000, n_records).tobytes(), dtype=np.uint8)


def key_range_ids(records, num_partitions):
    """TeraSort's range partitioner: the first two key bytes (after the 2-byte record header), scaled to [0, R)"""
    k = records.reshape(-1, REC)[:, 2:4].astype(np.uint64)
    return (((k[:, 0] << 8) | k[:, 1]) * num_partitions >> 16).astype(np.uint32)


def model_partitions(records, rec_len, rec_part, num_partitions):
    """-> list of num_partitions bytes objects: each partition's records in input order"""
    rec_len = np.asarray(rec_len, dtype=np.uint64)
    rec_part = np.asarray(rec_part, dtype=np.uint32)
    order = np.argsort(rec_part, kind="stable")
    starts = np.concatenate([[0], np.cumsum(rec_len)[:-1]]).astype(np.uint64) if rec_len.size else rec_len
    buf = np.asarray(records, dtype=np.uint8)
    if rec_len.size and np.all(rec_len == rec_len[0]) and rec_len[0] > 0:
        body = buf.reshape(-1, int(rec_len[0]))[order].ravel()
    else:
        body = np.concatenate([buf[int(starts[i]):int(starts[i] + rec_len[i])] for i in order] or [buf[:0]])
    counts = np.bincount(rec_part, weights=rec_len.astype(np.float64), minlength=num_partitions).astype(np.uint64)
    bounds = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    return [body[int(bounds[p]):int(bounds[p + 1])].tobytes() for p in range(num_partitions)]


def expected(capi, codec, alg, level, parts, block_size=0):
    """what b2s_compress_packed makes of the non-empty partitions, laid out per partition as the new call reports it"""
    R = len(parts)
    ne = [p for p in range(R) if len(parts[p])]
    empty_ck = 1 if alg == capi.CHECKSUM_ADLER32 else 0
    if codec == capi.CODEC_NONE:
        arena = b"".join(parts)
        lens = np.array([len(x) for x in parts], dtype=np.uint64)
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        cks = [capi.checksum_packed(alg, np.frombuffer(arena, np.uint8) if arena else np.zeros(1, np.uint8), offs,
                                    lens)] if alg else None
        return arena, offs, lens, (cks[0] if alg else np.zeros(R, np.uint64))
    src = np.frombuffer(b"".join(parts[p] for p in ne), dtype=np.uint8)
    offs = np.concatenate([[0], np.cumsum([len(parts[p]) for p in ne])[:-1]]).astype(np.uint64) if ne else []
    bound = sum(capi.compress_bound(codec, block_size, len(parts[p])) for p in ne) + 64
    dst = np.zeros(bound, dtype=np.uint8)
    r = capi.compress_packed(codec, src, offs, [len(parts[p]) for p in ne], dst, block_size, alg, level) if ne else None
    off = np.zeros(R, np.uint64)
    ln = np.zeros(R, np.uint64)
    ck = np.full(R, empty_ck if alg else 0, np.uint64)
    at = 0
    k = 0
    for p in range(R):
        if k < len(ne) and ne[k] == p:
            assert r["status"][k] == 0
            off[p], ln[p], ck[p] = r["dst_off"][k], r["dst_len"][k], r["checksums"][k] if alg else 0
            at = int(off[p] + ln[p])
            k += 1
        else:
            off[p] = at
    return (dst[: r["total"]].tobytes() if r else b""), off, ln, ck


def run_packed(capi, codec, records, rec_len, rec_part, R, alg=0, level=0, block_size=0, dst_cap=None):
    rec_bytes = int(np.sum(np.asarray(rec_len, dtype=np.uint64)))
    cap = capi.partition_compress_bound(codec, block_size, R, rec_bytes) if dst_cap is None else dst_cap
    dst = np.zeros(max(cap, 1), dtype=np.uint8)[:cap]
    r = capi.partition_compress_packed(codec, records, rec_len, rec_part, R, dst, block_size, alg, level)
    return dst[: r["total"]].tobytes(), r


def check_against_model(capi, codec, alg, level, records, rec_len, rec_part, R, block_size=0):
    parts = model_partitions(records, rec_len, rec_part, R)
    arena, r = run_packed(capi, codec, records, rec_len, rec_part, R, alg, level, block_size)
    want_arena, off, ln, ck = expected(capi, codec, alg, level, parts, block_size)
    assert (r["status"] == 0).all()
    assert np.array_equal(r["dst_len"], ln)
    assert np.array_equal(r["dst_off"], off)
    assert np.array_equal(r["checksums"], ck)
    assert r["total"] == len(want_arena) and arena == want_arena
    assert r["total"] <= capi.partition_compress_bound(codec, block_size, R, int(np.sum(rec_len, dtype=np.uint64)))
    return parts, arena, r


def decode_lz4_liblz4(stream):
    L = C.CDLL("liblz4.so.1")
    ip, out = 0, bytearray()
    while True:
        assert stream[ip:ip + 8] == b"LZ4Block"
        method = stream[ip + 8] & 0xF0
        clen = int.from_bytes(stream[ip + 9:ip + 13], "little")
        olen = int.from_bytes(stream[ip + 13:ip + 17], "little")
        ip += 21
        if olen == 0:
            break
        if method == 0x10:  # stored RAW
            out += stream[ip:ip + clen]
        else:
            buf = C.create_string_buffer(olen)
            assert L.LZ4_decompress_safe(stream[ip:ip + clen], buf, clen, olen) == olen
            out += buf.raw
        ip += clen
    assert ip == len(stream)
    return bytes(out)


def decode_independently(oracle, codec, stream):
    if codec == 1:
        return decode_lz4_liblz4(stream)
    if codec == 2:
        return oracle.xerial_decompress(stream)
    return zstd_ref.decompress(stream)


# ---------------------------------------------------------------------------------------------------------------
# 1. equivalence with b2s_compress_packed over the partitioned records, every codec x checksum
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", CHECKSUMS)
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_equals_compress_packed_over_the_model_partitions(capi, oracle, name, codec, level, alg):
    R = 200
    records = terasort(oracle, 40000, seed=3)  # ~4 MiB, ~20 KiB per partition
    ids = key_range_ids(records, R)
    ids[ids == 7] = 8  # a few empty partitions
    lens = np.full(ids.size, REC, np.uint32)
    parts, arena, r = check_against_model(capi, codec, alg, level, records, lens, ids, R)
    assert (r["dst_len"][7] == 0) and r["checksums"][7] == (1 if alg == 1 else 0)
    for p in (0, 8, 123, 199):
        o, n = int(r["dst_off"][p]), int(r["dst_len"][p])
        assert n > 0
        assert decode_independently(oracle, codec, arena[o:o + n]) == parts[p]


@pytest.mark.parametrize("name,codec,level", CODECS)
def test_dev_equals_packed(capi, oracle, name, codec, level):
    R = 2000
    records = terasort(oracle, 30000, seed=4)
    ids = key_range_ids(records, R)
    lens = np.full(ids.size, REC, np.uint32)
    arena, r = run_packed(capi, codec, records, lens, ids, R, capi.CHECKSUM_CRC32C, level)
    cap = capi.partition_compress_bound(codec, 0, R, records.size)
    d_rec, d_len, d_part, d_dst = (capi.dev_alloc(records.size), capi.dev_alloc(lens.nbytes), capi.dev_alloc(ids.nbytes),
                                   capi.dev_alloc(cap))
    try:
        capi.dev_memcpy(d_rec, records.ctypes.data, records.size, 1)
        capi.dev_memcpy(d_len, lens.ctypes.data, lens.nbytes, 1)
        capi.dev_memcpy(d_part, ids.ctypes.data, ids.nbytes, 1)
        rd = capi.partition_compress_dev(codec, d_rec, records.size, d_len, d_part, ids.size, R, d_dst, cap,
                                         checksum_alg=capi.CHECKSUM_CRC32C, level=level)
        out = np.zeros(max(rd["total"], 1), np.uint8)
        capi.dev_memcpy(out.ctypes.data, d_dst, rd["total"], 2)
    finally:
        for p in (d_rec, d_len, d_part, d_dst):
            capi.dev_free(p)
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert np.array_equal(rd[k], r[k]), k
    assert rd["total"] == r["total"] and out[: rd["total"]].tobytes() == arena


# ---------------------------------------------------------------------------------------------------------------
# 2. codec NONE: exactly the partitioned records
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", CHECKSUMS)
def test_codec_none_is_the_partitioned_records(capi, oracle, alg):
    R = 2000
    records = terasort(oracle, 50000, seed=5)
    ids = key_range_ids(records, R)
    lens = np.full(ids.size, REC, np.uint32)
    parts = model_partitions(records, lens, ids, R)
    arena, r = run_packed(capi, capi.CODEC_NONE, records, lens, ids, R, alg)
    assert arena == b"".join(parts)
    want = [len(x) for x in parts]
    assert list(r["dst_len"]) == want and list(r["dst_off"]) == list(np.concatenate([[0], np.cumsum(want)[:-1]]))
    _, off, ln, ck = expected(capi, capi.CODEC_NONE, alg, 0, parts)
    assert np.array_equal(r["checksums"], ck)


# ---------------------------------------------------------------------------------------------------------------
# 3. shapes
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 2, 200, 2000, 65536])
@pytest.mark.parametrize("spread", ["uniform", "one", "descending", "each_once"])
def test_partition_counts_and_spreads(capi, oracle, R, spread):
    n = max(R, 6000) if spread == "each_once" else 6000
    records = terasort(oracle, n, seed=6)
    rng = np.random.default_rng(R)
    if spread == "uniform":
        ids = rng.integers(0, R, n).astype(np.uint32)
    elif spread == "one":
        ids = np.full(n, R // 2, np.uint32)
    elif spread == "descending":
        ids = np.sort(rng.integers(0, R, n).astype(np.uint32))[::-1].copy()
    else:
        ids = rng.permutation(np.resize(np.arange(R, dtype=np.uint32), n)).astype(np.uint32)
    lens = np.full(n, REC, np.uint32)
    check_against_model(capi, capi.CODEC_LZ4BLOCK, capi.CHECKSUM_CRC32C, 0, records, lens, ids, R)
    parts = model_partitions(records, lens, ids, R)
    arena, _ = run_packed(capi, capi.CODEC_NONE, records, lens, ids, R)
    assert arena == b"".join(parts)


def test_2_pow_24_partitions(capi, oracle):
    R = 1 << 24
    records = terasort(oracle, 3000, seed=7)
    rng = np.random.default_rng(1)
    ids = rng.integers(0, R, 3000).astype(np.uint32)
    ids[:3] = [0, R - 1, R - 1]
    lens = np.full(3000, REC, np.uint32)
    check_against_model(capi, capi.CODEC_ZSTD, capi.CHECKSUM_ADLER32, 1, records, lens, ids, R)
    parts = model_partitions(records, lens, ids, R)
    arena, r = run_packed(capi, capi.CODEC_NONE, records, lens, ids, R, capi.CHECKSUM_CRC32)
    assert arena == b"".join(parts) and int(r["dst_len"][R - 1]) == 2 * REC


@pytest.mark.parametrize("name,codec,level", CODECS)
def test_record_lengths_zero_one_and_100k(capi, oracle, name, codec, level):
    rng = np.random.default_rng(11)
    lens = rng.choice([0, 1, 2, 15, 16, 17, 104, 255, 256, 257, 1000, 100 * 1024], size=900,
                      p=[.1, .1, .05, .05, .05, .05, .3, .05, .05, .05, .1, .05]).astype(np.uint32)
    kinds = ["terasort", "text", "random", "runs"]
    records = np.frombuffer(b"".join(corpus(oracle, kinds[i % 4], int(lens.sum()) // 4 + 1, seed=i) for i in range(4)),
                            np.uint8)[: int(lens.sum())].copy()
    R = 37
    ids = rng.integers(0, R, lens.size).astype(np.uint32)
    ids[lens == 0] = 5  # partition 5 holds zero-length records only besides whatever else lands there
    parts, arena, r = check_against_model(capi, codec, capi.CHECKSUM_CRC32C, level, records, lens, ids, R)
    for p in range(R):
        o, n = int(r["dst_off"][p]), int(r["dst_len"][p])
        if n:
            assert decode_independently(oracle, codec, arena[o:o + n]) == parts[p]
    na, _ = run_packed(capi, capi.CODEC_NONE, records, lens, ids, R)
    assert na == b"".join(parts)


def test_only_zero_length_records_and_no_records(capi):
    for codec in (0, 1, 2, 3):
        for n in (0, 50):
            r = capi.partition_compress_packed(codec, np.zeros(0, np.uint8), np.zeros(n, np.uint32),
                                               np.arange(n, dtype=np.uint32) % 7, 7, np.zeros(16, np.uint8),
                                               checksum_alg=capi.CHECKSUM_ADLER32)
            assert r["total"] == 0 and not r["dst_len"].any() and not r["dst_off"].any()
            assert (r["checksums"] == 1).all() and not r["status"].any()


def test_above_1_gib_runs_several_compress_chunks(capi, oracle):
    """> 1 GiB of records: the compress pipeline works through more than B2S_LZ4_CHUNK_BLOCKS codec blocks"""
    n = (1 << 30) // REC + 500000
    records = capi.HostBuffer(n * REC)
    records.array[:] = terasort(oracle, n, seed=12)
    R = 200
    ids = key_range_ids(records.array, R)
    lens = np.full(n, REC, np.uint32)
    cap = capi.partition_compress_bound(capi.CODEC_LZ4BLOCK, 0, R, n * REC)
    dst = capi.HostBuffer(cap)
    try:
        r = capi.partition_compress_packed(capi.CODEC_LZ4BLOCK, records.array, lens, ids, R, dst.array,
                                           checksum_alg=capi.CHECKSUM_CRC32C)
        assert (r["status"] == 0).all()
        order = np.argsort(ids, kind="stable")
        body = records.array.reshape(-1, REC)[order].ravel()
        counts = np.bincount(ids, minlength=R).astype(np.uint64) * REC
        offs = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint64)
        want = np.zeros(capi.partition_compress_bound(capi.CODEC_LZ4BLOCK, 0, R, n * REC), np.uint8)
        w = capi.compress_packed(capi.CODEC_LZ4BLOCK, body, offs, counts, want, 0, capi.CHECKSUM_CRC32C)
        assert r["total"] == w["total"]
        assert np.array_equal(r["dst_len"], w["dst_len"]) and np.array_equal(r["checksums"], w["checksums"])
        assert np.array_equal(dst.array[: r["total"]], want[: w["total"]])
        o, ln = int(r["dst_off"][R // 2]), int(r["dst_len"][R // 2])
        part = body[int(offs[R // 2]):int(offs[R // 2] + counts[R // 2])].tobytes()
        assert decode_lz4_liblz4(dst.array[o:o + ln].tobytes()) == part
    finally:
        records.free()
        dst.free()


# ---------------------------------------------------------------------------------------------------------------
# 5. errors and the bound
# ---------------------------------------------------------------------------------------------------------------
def test_bad_partition_id_and_wrong_rec_bytes_are_arg_errors(capi, oracle):
    L = capi.load()
    records = terasort(oracle, 1000, seed=13)
    ids = key_range_ids(records, 16)
    lens = np.full(1000, REC, np.uint32)
    bad = ids.copy()
    bad[417] = 16
    bad[600] = 99
    with pytest.raises(capi.B2SError) as e:
        run_packed(capi, capi.CODEC_LZ4BLOCK, records, lens, bad, 16)
    assert e.value.code == capi.E_ARG and "record 417" in str(e.value)
    dst = np.zeros(capi.partition_compress_bound(1, 0, 16, records.size), np.uint8)
    off, ln, ck = (np.zeros(16, np.uint64) for _ in range(3))
    st = np.zeros(16, np.int32)
    total = C.c_uint64(7)
    padded = np.concatenate([records, np.zeros(1, np.uint8)])  # rec_bytes one too large still names readable memory
    for rec_bytes, what in ((records.size - 1, "record 999"), (records.size + 1, "rec_bytes")):
        rc = L.b2s_partition_compress_packed(1, 0, 0, 3, 16, 1000, padded.ctypes.data, rec_bytes, lens.ctypes.data,
                                             ids.ctypes.data, dst.ctypes.data, dst.size, off.ctypes.data,
                                             ln.ctypes.data, C.addressof(total), ck.ctypes.data, st.ctypes.data)
        assert rc == capi.E_ARG and what in L.b2s_last_error().decode()
        assert total.value == 0 and not ln.any()
    for R in (0, (1 << 24) + 1):
        with pytest.raises(capi.B2SError) as e:
            run_packed(capi, capi.CODEC_LZ4BLOCK, records, lens, ids, R)
        assert e.value.code == capi.E_ARG


def test_short_dst_cap(capi, oracle):
    records = terasort(oracle, 5000, seed=14)
    ids = key_range_ids(records, 50)
    lens = np.full(5000, REC, np.uint32)
    for codec in (0, 1, 2, 3):
        full, r = run_packed(capi, codec, records, lens, ids, 50)
        with pytest.raises(capi.B2SError) as e:
            run_packed(capi, codec, records, lens, ids, 50, dst_cap=r["total"] - 1)
        assert e.value.code == capi.E_DST_TOO_SMALL


@pytest.mark.parametrize("name,codec,level", CODECS)
def test_bound_holds_on_adversarial_spreads(capi, oracle, name, codec, level):
    R = 4096
    # every partition one byte (incompressible, most per-stream overhead), then one huge random partition
    one = np.frombuffer(corpus(oracle, "random", R, seed=15), np.uint8).copy()
    _, r = run_packed(capi, codec, one, np.ones(R, np.uint32), np.arange(R, dtype=np.uint32)[::-1].copy(), R,
                      level=level)
    assert r["total"] <= capi.partition_compress_bound(codec, 0, R, R)
    big = np.frombuffer(corpus(oracle, "random", 3 << 20, seed=16), np.uint8).copy()
    lens = np.full(3 << 10, 1024, np.uint32)
    _, r = run_packed(capi, codec, big, lens, np.full(lens.size, R - 1, np.uint32), R, level=level)
    assert r["total"] <= capi.partition_compress_bound(codec, 0, R, big.size)
    assert r["total"] > big.size  # stored raw: the bound is what it has to be


# ---------------------------------------------------------------------------------------------------------------
# 6. lanes: a partition-compress call beside a decompress call
# ---------------------------------------------------------------------------------------------------------------
def test_partition_compress_beside_decompress(capi, oracle):
    R = 200
    records = terasort(oracle, 200000, seed=17)
    ids = key_range_ids(records, R)
    lens = np.full(ids.size, REC, np.uint32)
    want_arena, want = run_packed(capi, capi.CODEC_LZ4BLOCK, records, lens, ids, R, capi.CHECKSUM_CRC32C)
    parts = [corpus(oracle, "terasort", 300000 + 1000 * i, seed=60 + i) for i in range(16)]
    streams = [oracle.lz4block_compress(p, 32768, compressor=1) for p in parts]
    errors = []

    def writer():
        try:
            for _ in range(5):
                arena, r = run_packed(capi, capi.CODEC_LZ4BLOCK, records, lens, ids, R, capi.CHECKSUM_CRC32C)
                assert arena == want_arena and np.array_equal(r["checksums"], want["checksums"])
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    def reader():
        try:
            src = np.frombuffer(b"".join(streams), np.uint8)
            off = np.concatenate([[0], np.cumsum([len(s) for s in streams])[:-1]])
            for _ in range(5):
                dst = np.zeros(sum(map(len, parts)), np.uint8)
                r = capi.decompress_packed(capi.CODEC_LZ4BLOCK, src, off, [len(s) for s in streams], dst)
                assert (r["status"] == 0).all() and dst.tobytes() == b"".join(parts)
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    ths = [threading.Thread(target=writer), threading.Thread(target=reader)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errors, errors
