"""b2s_last_timing of the host-pointer entry points: the byte counters follow from each call's inputs and outputs, and
the launch counters are the same for two identical calls.  bench.py and the split tools read these fields."""
import numpy as np
import pytest

from conftest import corpus

pytestmark = pytest.mark.gpu


def staged_bytes(ptrs, lens):
    """the bytes a host-pointer call uploads for one chunk: runs contiguous in host memory go up as one copy, every
    other run starts at the next 16-byte boundary plus its host pointer's phase"""
    cur, end = 0, None
    for p, n in zip(ptrs, lens):
        if n == 0:
            continue
        if p != end:
            cur = (cur + 15) // 16 * 16 + (p & 15)
        cur += n
        end = p + n
    return cur


def blocks(oracle, n=5, seed=3):
    sizes = [70000 + 9001 * i for i in range(n)]
    sizes[2] = 0  # an empty stream among them
    return [np.frombuffer(corpus(oracle, "terasort", s, seed=seed + i), dtype=np.uint8).copy() for i, s in
            enumerate(sizes)]


def twice(capi, call):
    """runs call twice; -> (result of the second run, its timing), after checking the launch counts repeat"""
    call()
    first = capi.last_timing()
    out = call()
    t = capi.last_timing()
    assert t["kernel_launches"] == first["kernel_launches"] > 0
    assert t["dominant_launches"] == first["dominant_launches"]
    return out, t


def packed(arrs):
    base = np.concatenate(arrs) if arrs else np.zeros(0, np.uint8)
    lens = np.array([a.size for a in arrs], dtype=np.uint64)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    return base, off, lens


def test_checksum_calls(capi, oracle):
    arrs = blocks(oracle)
    lens = [a.size for a in arrs]
    _, t = twice(capi, lambda: capi.checksum_batch(capi.CHECKSUM_CRC32C, arrs))
    up = staged_bytes([a.ctypes.data for a in arrs], lens)
    assert (t["h2d_bytes"], t["d2h_bytes"], t["src_bytes"], t["dst_bytes"]) == (up, 8 * len(arrs), up, 0)
    assert t["dominant_launches"] == 0
    base, off, ln = packed(arrs)
    _, t = twice(capi, lambda: capi.checksum_packed(capi.CHECKSUM_CRC32C, base, off, ln))
    up = staged_bytes([base.ctypes.data + int(o) for o in off], lens)
    assert up >= sum(lens)
    assert (t["h2d_bytes"], t["d2h_bytes"], t["src_bytes"], t["dst_bytes"]) == (up, 8 * len(arrs), up, 0)
    assert t["dominant_launches"] == 0


def test_compress_calls(capi, oracle):
    arrs = blocks(oracle)
    lens = [a.size for a in arrs]
    base, off, ln = packed(arrs)
    dst = np.zeros(sum(capi.compress_bound(capi.CODEC_LZ4BLOCK, 0, n) for n in lens), dtype=np.uint8)
    r, t = twice(capi, lambda: capi.compress_packed(capi.CODEC_LZ4BLOCK, base, off, ln, dst, 32768,
                                                    capi.CHECKSUM_CRC32C))
    assert list(r["status"]) == [0] * len(arrs)
    up = staged_bytes([base.ctypes.data + int(o) for o in off], lens)
    assert (t["h2d_bytes"], t["d2h_bytes"], t["src_bytes"], t["dst_bytes"]) == (up, r["total"], up, r["total"])
    assert t["dominant_launches"] > 0

    caps = [capi.compress_bound(capi.CODEC_LZ4BLOCK, 0, n) for n in lens]
    caps[1] = 10  # too small: that stream is not copied back
    (streams, _, st), t = twice(capi, lambda: capi.compress_batch(capi.CODEC_LZ4BLOCK, arrs, 32768, dst_caps=caps))
    assert st[1] == capi.E_DST_TOO_SMALL and [s for i, s in enumerate(st) if i != 1] == [0] * (len(arrs) - 1)
    up = staged_bytes([a.ctypes.data for a in arrs], lens)
    ok = sum(len(s) for s in streams if s is not None)
    full, _, _ = capi.compress_batch(capi.CODEC_LZ4BLOCK, arrs, 32768)
    assert (t["h2d_bytes"], t["d2h_bytes"], t["src_bytes"]) == (up, ok, up)
    assert t["dst_bytes"] == sum(len(s) for s in full)
    assert t["dominant_launches"] > 0


def test_decompress_calls(capi, oracle):
    parts = [a.tobytes() for a in blocks(oracle)]
    streams = [np.frombuffer(oracle.lz4block_compress(p), dtype=np.uint8).copy() for p in parts]
    lens = [s.size for s in streams]
    base, off, ln = packed(streams)
    sums = [oracle.crc32c(s.tobytes()) for s in streams]
    dst = np.zeros(sum(map(len, parts)), dtype=np.uint8)
    r, t = twice(capi, lambda: capi.decompress_packed(capi.CODEC_LZ4BLOCK, base, off, ln, dst, capi.CHECKSUM_CRC32C,
                                                      list(range(len(streams) + 1)), lens, sums))
    assert list(r["status"]) == [0] * len(streams) and r["total"] == dst.size
    up = staged_bytes([base.ctypes.data + int(o) for o in off], lens)
    assert (t["h2d_bytes"], t["d2h_bytes"], t["src_bytes"], t["dst_bytes"]) == (up, r["total"], up, r["total"])
    assert t["dominant_launches"] > 0

    caps = [len(p) for p in parts]
    caps[3] = 100  # too small: that stream is not copied back
    (out, st, _), t = twice(capi, lambda: capi.decompress_batch(capi.CODEC_LZ4BLOCK, streams, dst_caps=caps))
    assert st[3] == capi.E_DST_TOO_SMALL and out[0] == parts[0]
    up = staged_bytes([s.ctypes.data for s in streams], lens)
    ok = sum(len(p) for p, s in zip(parts, st) if s == 0)
    assert (t["h2d_bytes"], t["d2h_bytes"], t["src_bytes"], t["dst_bytes"]) == (up, ok, up, sum(map(len, parts)))
    assert t["dominant_launches"] > 0


def _records(oracle, n=3000, R=7, seed=5):
    rng = np.random.default_rng(seed)
    rec_len = rng.integers(1, 200, n).astype(np.uint32)
    rec_part = rng.integers(0, R, n).astype(np.uint32)
    records = np.frombuffer(corpus(oracle, "text", int(rec_len.sum()), seed=seed), dtype=np.uint8).copy()
    return records, rec_len, rec_part, R


@pytest.mark.parametrize("codec", ["LZ4BLOCK", "NONE"])
def test_partition_compress_packed(capi, oracle, codec):
    c = getattr(capi, "CODEC_" + codec)
    records, rec_len, rec_part, R = _records(oracle)
    dst = np.zeros(capi.partition_compress_bound(c, 0, R, records.size), dtype=np.uint8)
    r, t = twice(capi, lambda: capi.partition_compress_packed(c, records, rec_len, rec_part, R, dst, 0,
                                                              capi.CHECKSUM_CRC32C))
    assert list(r["status"]) == [0] * R
    assert (t["h2d_bytes"], t["d2h_bytes"]) == (records.size + 8 * rec_len.size, r["total"])
    assert (t["src_bytes"], t["dst_bytes"]) == (records.size, r["total"])
    assert (t["dominant_launches"] > 0) == (c == capi.CODEC_LZ4BLOCK)


def test_sort_calls(capi, oracle):
    rb = 100
    parts = [oracle.gen_terasort(1000 * i, 900 + 50 * i).tobytes() for i in range(3)]
    streams = [oracle.lz4block_compress(p) for p in parts]
    base, off, ln = packed([np.frombuffer(s, dtype=np.uint8) for s in streams])
    sums = [oracle.crc32c(s) for s in streams]
    sb = list(range(len(streams) + 1))
    dst = np.zeros(sum(map(len, parts)), dtype=np.uint8)
    r, t = twice(capi, lambda: capi.decompress_sort_packed(capi.CODEC_LZ4BLOCK, base, off, ln, dst, rb, 0, 10,
                                                           capi.CHECKSUM_CRC32C, sb, ln, sums))
    assert r["n_records"] == dst.size // rb
    assert (t["h2d_bytes"], t["d2h_bytes"]) == (base.size, r["total"])
    assert (t["src_bytes"], t["dst_bytes"]) == (base.size, r["total"])
    # a failed checksum: nothing is sorted, nothing comes back
    bad = list(sums)
    bad[1] ^= 1
    r, t = twice(capi, lambda: capi.decompress_sort_packed(capi.CODEC_LZ4BLOCK, base, off, ln, dst, rb, 0, 10,
                                                           capi.CHECKSUM_CRC32C, sb, ln, bad))
    assert r["n_records"] == 0 and r["status"][1] == capi.E_CHECKSUM
    assert (t["h2d_bytes"], t["d2h_bytes"], t["src_bytes"]) == (base.size, 0, base.size)

    # rows: [int32 big-endian size][16-byte row, an int64 key first]
    rng = np.random.default_rng(9)
    rows = []
    for k in range(3):
        keys = rng.integers(-(1 << 40), 1 << 40, 700 + 40 * k)
        rows.append(b"".join((16).to_bytes(4, "big") + int(v).to_bytes(8, "little", signed=True) + bytes(8)
                             for v in keys))
    streams = [oracle.lz4block_compress(p) for p in rows]
    base, off, ln = packed([np.frombuffer(s, dtype=np.uint8) for s in streams])
    dst = np.zeros(sum(map(len, rows)), dtype=np.uint8)
    r, t = twice(capi, lambda: capi.decompress_sort_rows_packed(capi.CODEC_LZ4BLOCK, base, off, ln, dst,
                                                                capi.KEY_INT64, 0, 8))
    assert list(r["status"]) == [0] * 3 and r["n_records"] == sum(len(p) // 20 for p in rows)
    assert (t["h2d_bytes"], t["d2h_bytes"]) == (base.size, r["total"])
    assert (t["src_bytes"], t["dst_bytes"]) == (base.size, r["total"])
    assert t["dominant_launches"] > 0  # the row framing


def test_exchange_read_packed(capi, oracle):
    records, rec_len, rec_part, R = _records(oracle, seed=11)
    capi.exchange_set_budget(64 << 20)
    try:
        dst = np.zeros(capi.partition_compress_bound(capi.CODEC_LZ4BLOCK, 0, R, records.size), dtype=np.uint8)
        r = capi.partition_compress_cached_packed(71, 0, capi.CODEC_LZ4BLOCK, records, rec_len, rec_part, R, dst)
        assert r["cached"] == 1
        out = np.zeros(records.size, dtype=np.uint8)
        r, t = twice(capi, lambda: capi.exchange_read_packed(71, 2, 5, [0, 1], out))
        assert list(r["status"]) == [0, capi.E_NOT_CACHED] and r["total"] > 0
        assert (t["h2d_bytes"], t["d2h_bytes"], t["src_bytes"], t["dst_bytes"]) == (0, r["total"], r["total"],
                                                                                     r["total"])
        assert t["dominant_launches"] == 0
    finally:
        capi.exchange_remove(71)
        capi.exchange_set_budget(0)
