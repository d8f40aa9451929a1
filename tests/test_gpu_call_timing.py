"""b2s_last_timing belongs to the call that fills it: a call never reports a step, a dominant launch or a time that an
earlier call on the same pipeline slot recorded, whether that call failed, stopped early or skipped a step.  And the
times of each kind of call keep the nesting their definitions give them."""
import numpy as np
import pytest

from conftest import corpus
from rows_model import KEY_INT64, SUM_I64, blocks_of, build_blocks, stream

pytestmark = pytest.mark.gpu

COUNTERS = ("h2d_bytes", "d2h_bytes", "src_bytes", "dst_bytes", "kernel_launches", "dominant_launches")
TIMES = ("kernel_ms", "top_kernel_ms", "dominant_ms", "h2d_ms", "d2h_ms")


def lz4_blocks(capi, oracle, n=4):
    plain = [corpus(oracle, "terasort", 60000 + 7000 * i, seed=i) for i in range(n)]
    return plain, build_blocks(capi, capi.CODEC_LZ4BLOCK, 0, capi.CHECKSUM_CRC32C, plain)


def rows(n, seed=1):
    """[int32 big-endian size][16-byte row: an int64 key, an int64 value]"""
    rng = np.random.default_rng(seed)
    keys, vals = rng.integers(0, 300, n), rng.integers(-1000, 1000, n)
    return [int(k).to_bytes(8, "little", signed=True) + int(v).to_bytes(8, "little", signed=True)
            for k, v in zip(keys, vals)]


def decompress_dev(capi, blocks, cap):
    arena, off, ln, sb, sl, sc = blocks
    d_src, d_dst = capi.dev_alloc(arena.size), capi.dev_alloc(cap)
    try:
        capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        r = capi.decompress_dev(capi.CODEC_LZ4BLOCK, d_src, off, ln, d_dst, cap, capi.CHECKSUM_CRC32C, sb, sl, sc)
        assert (r["status"] == 0).all()
        return capi.last_timing()
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)


def test_a_failed_call_leaves_no_dominant_launch_to_the_next(capi, oracle):
    plain, blocks = lz4_blocks(capi, oracle)
    cap = sum(map(len, plain))
    first = decompress_dev(capi, blocks, cap)
    assert first["dominant_launches"] == 1
    # an aggregation whose output does not fit: it decodes (one LZ4 decode launch), groups, then fails
    agg = build_blocks(capi, capi.CODEC_LZ4BLOCK, 0, capi.CHECKSUM_CRC32C, blocks_of(rows(4000), [2500, 1500]))
    arena, off, ln, sb, sl, sc = agg
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_aggregate_rows_packed(capi.CODEC_LZ4BLOCK, arena, off, ln, np.zeros(16, np.uint8), KEY_INT64,
                                              0, 8, -1, [(SUM_I64, 8, -1)], capi.CHECKSUM_CRC32C, sb, sl, sc)
    assert e.value.code == capi.E_DST_TOO_SMALL
    again = decompress_dev(capi, blocks, cap)
    assert (again["dominant_launches"], again["kernel_launches"]) == (first["dominant_launches"],
                                                                      first["kernel_launches"])
    assert again["dominant_ms"] <= again["top_kernel_ms"]


def close(a, b):
    """a time of a clean call after a clean call, and the same after a failed or short call: the same within the
    noise of a shared card"""
    return (a == 0) == (b == 0) and b <= 4 * a + 0.5 and a <= 4 * b + 0.5


def after(capi, clean, other, reps=3):
    """clean() after clean(), and clean() after other(), alternated; the counters must be equal, the times close"""
    clean()
    base, got = [], []
    for _ in range(reps):
        clean()
        base.append(capi.last_timing())
        other()
        clean()
        got.append(capi.last_timing())
    for a, b in zip(base, got):
        assert {k: a[k] for k in COUNTERS} == {k: b[k] for k in COUNTERS}
    for k in TIMES:
        x, y = min(a[k] for a in base), min(b[k] for b in got)
        assert close(x, y), (k, x, y)


def test_a_sort_after_a_failed_checksum(capi, oracle):
    recs = [oracle.gen_terasort(1000 * i, 600 + 40 * i).tobytes() for i in range(3)]
    arena, off, ln, sb, sl, sc = build_blocks(capi, capi.CODEC_LZ4BLOCK, 0, capi.CHECKSUM_CRC32C, recs)
    dst = np.zeros(sum(map(len, recs)), np.uint8)
    bad = sc.copy()
    bad[1] ^= 1

    def sort(sums):
        return capi.decompress_sort_packed(capi.CODEC_LZ4BLOCK, arena, off, ln, dst, 100, 0, 10,
                                           capi.CHECKSUM_CRC32C, sb, sl, sums)

    def failed():
        r = sort(bad)
        assert r["n_records"] == 0 and r["status"][1] == capi.E_CHECKSUM

    after(capi, lambda: sort(sc), failed)


def test_a_row_sort_after_a_malformed_block(capi):
    good = blocks_of(rows(3000, seed=2), [1000, 1200, 800])
    broken = list(good)
    broken[1] = good[1][:-3]  # its last record runs past the block end
    dst = np.zeros(sum(map(len, good)), np.uint8)
    good, broken = (build_blocks(capi, capi.CODEC_LZ4BLOCK, 0, capi.CHECKSUM_CRC32C, p) for p in (good, broken))

    def sort(blocks):
        arena, off, ln, sb, sl, sc = blocks
        return capi.decompress_sort_rows_packed(capi.CODEC_LZ4BLOCK, arena, off, ln, dst, KEY_INT64, 0, 8, -1,
                                                capi.CHECKSUM_CRC32C, sb, sl, sc)

    def failed():
        r = sort(broken)
        assert r["n_records"] == 0 and r["status"][1] == capi.E_CORRUPT

    after(capi, lambda: sort(good), failed)


def partition_records(oracle, n=3000, R=7, seed=5):
    rng = np.random.default_rng(seed)
    rec_len = rng.integers(1, 200, n).astype(np.uint32)
    rec_part = rng.integers(0, R, n).astype(np.uint32)
    return np.frombuffer(corpus(oracle, "text", int(rec_len.sum()), seed=seed), np.uint8).copy(), rec_len, rec_part


@pytest.mark.parametrize("codec", ["LZ4BLOCK", "NONE"])
def test_a_partition_after_one_with_no_records(capi, oracle, codec):
    c = getattr(capi, "CODEC_" + codec)
    records, rec_len, rec_part = partition_records(oracle)
    R = 7
    dst = np.zeros(capi.partition_compress_bound(c, 0, R, records.size), np.uint8)

    def empty():
        r = capi.partition_compress_packed(c, np.zeros(0, np.uint8), np.zeros(0, np.uint32), np.zeros(0, np.uint32), R,
                                           dst, 0, capi.CHECKSUM_CRC32C)
        assert r["total"] == 0 and (r["status"] == 0).all()
        t = capi.last_timing()
        # no codec step ran; the kernel region ends where the call stopped
        assert t["top_kernel_ms"] <= t["kernel_ms"] and t["dominant_launches"] == 0

    after(capi, lambda: capi.partition_compress_packed(c, records, rec_len, rec_part, R, dst, 0, capi.CHECKSUM_CRC32C),
          empty)


# ---------------------------------------------------------------------------------------------------------------
# the nesting of each family's times (include/b200shuffle.h): dominant_ms within top_kernel_ms where the dominant
# step is part of the top step, top_kernel_ms within kernel_ms, copy times where the call copies
# ---------------------------------------------------------------------------------------------------------------
EPS = 1e-3


def relations(t, dev, nested=True, download_timed=True):
    assert 0 <= t["dominant_ms"] <= t["kernel_ms"] + EPS and 0 <= t["top_kernel_ms"] <= t["kernel_ms"] + EPS, t
    if nested:
        assert t["dominant_ms"] <= t["top_kernel_ms"] + EPS, t
    assert (t["dominant_ms"] > 0) == (t["dominant_launches"] > 0), t
    if dev:
        assert t["h2d_ms"] == 0 and t["d2h_ms"] == 0, t
    else:
        assert (t["h2d_ms"] > 0) == (t["h2d_bytes"] > 0), t
        if download_timed:
            assert (t["d2h_ms"] > 0) == (t["d2h_bytes"] > 0), t


def test_codec_call_relations(capi, oracle):
    plain, blocks = lz4_blocks(capi, oracle)
    arena, off, ln, sb, sl, sc = blocks
    cap = sum(map(len, plain))
    relations(decompress_dev(capi, blocks, cap), dev=True)
    capi.decompress_packed(capi.CODEC_LZ4BLOCK, arena, off, ln, np.zeros(cap, np.uint8), capi.CHECKSUM_CRC32C, sb,
                           sl, sc)
    relations(capi.last_timing(), dev=False)
    src = np.frombuffer(b"".join(plain), np.uint8)
    soff = np.concatenate([[0], np.cumsum([len(p) for p in plain])[:-1]]).astype(np.uint64)
    slen = np.array([len(p) for p in plain], np.uint64)
    capi.compress_packed(capi.CODEC_LZ4BLOCK, src, soff, slen, np.zeros(2 * cap, np.uint8), 0, capi.CHECKSUM_CRC32C)
    relations(capi.last_timing(), dev=False)
    capi.checksum_packed(capi.CHECKSUM_CRC32C, src, soff, slen)
    t = capi.last_timing()
    relations(t, dev=False, download_timed=False)  # a checksum call times its uploads only
    assert t["dominant_launches"] == 0 and t["d2h_ms"] == 0
    d_src, d_dst = capi.dev_alloc(src.size), capi.dev_alloc(2 * cap)
    try:
        capi.dev_memcpy(d_src, src.ctypes.data, src.size, 1)
        capi.compress_dev(capi.CODEC_LZ4BLOCK, d_src, soff, slen, d_dst, 2 * cap, 0, capi.CHECKSUM_CRC32C)
        relations(capi.last_timing(), dev=True)
        capi.checksum_dev(capi.CHECKSUM_CRC32C, d_src, soff, slen)
        relations(capi.last_timing(), dev=True)
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)


@pytest.mark.parametrize("codec", ["LZ4BLOCK", "NONE"])
def test_partition_relations(capi, oracle, codec):
    c = getattr(capi, "CODEC_" + codec)
    records, rec_len, rec_part = partition_records(oracle, seed=8)
    dst = np.zeros(capi.partition_compress_bound(c, 0, 7, records.size), np.uint8)
    capi.partition_compress_packed(c, records, rec_len, rec_part, 7, dst, 0, capi.CHECKSUM_CRC32C)
    relations(capi.last_timing(), dev=False)
    d = [capi.dev_alloc(max(a.nbytes, 1)) for a in (records, rec_len, rec_part, dst)]
    try:
        for p, a in zip(d, (records, rec_len, rec_part)):
            capi.dev_memcpy(p, a.ctypes.data, a.nbytes, 1)
        capi.partition_compress_dev(c, d[0], records.size, d[1], d[2], rec_len.size, 7, d[3], dst.size, 0,
                                    capi.CHECKSUM_NONE)
        relations(capi.last_timing(), dev=True)
    finally:
        for p in d:
            capi.dev_free(p)
    # a hash partition: the dominant step is the hash, in front of the codec step
    body = rows(2000, seed=3)
    recs = np.frombuffer(stream(body), np.uint8)
    capi.partition_compress_rows_hash_packed(c, recs, np.full(len(body), 4 + 16, np.uint32), [(KEY_INT64, 0, 8, -1)],
                                             7, np.zeros(capi.partition_compress_bound(c, 0, 7, recs.size), np.uint8))
    t = capi.last_timing()
    relations(t, dev=False, nested=c == capi.CODEC_NONE)
    assert t["dominant_launches"] == 1


def test_sort_relations(capi):
    plain = blocks_of(rows(4000, seed=4), [2000, 2000])
    arena, off, ln, sb, sl, sc = build_blocks(capi, capi.CODEC_LZ4BLOCK, 0, capi.CHECKSUM_CRC32C, plain)
    dst = np.zeros(sum(map(len, plain)), np.uint8)
    capi.decompress_sort_rows_packed(capi.CODEC_LZ4BLOCK, arena, off, ln, dst, KEY_INT64, 0, 8, -1,
                                     capi.CHECKSUM_CRC32C, sb, sl, sc)
    relations(capi.last_timing(), dev=False)
    capi.decompress_aggregate_rows_packed(capi.CODEC_LZ4BLOCK, arena, off, ln, dst, KEY_INT64, 0, 8, -1,
                                          [(SUM_I64, 8, -1)], capi.CHECKSUM_CRC32C, sb, sl, sc)
    relations(capi.last_timing(), dev=False)
    # fixed-size records: the decoder's launch comes before the sort step, so it is not nested in it
    recs = [bytes(range(100)) * 300, bytes(range(100, 200)) * 200]
    arena, off, ln, sb, sl, sc = build_blocks(capi, capi.CODEC_LZ4BLOCK, 0, capi.CHECKSUM_CRC32C, recs)
    capi.decompress_sort_packed(capi.CODEC_LZ4BLOCK, arena, off, ln, np.zeros(50000, np.uint8), 100, 0, 10,
                                capi.CHECKSUM_CRC32C, sb, sl, sc)
    relations(capi.last_timing(), dev=False, nested=False)
