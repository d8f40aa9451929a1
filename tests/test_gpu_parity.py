"""GPU parity: the CUDA path (called through the C ABI) against the CPU oracle, bit-exact.

Mirrors what the reference's own tests exercise end to end (test/S3ShuffleManagerTest.scala runs every job with the
default lz4 codec + ADLER32 checksums, asserting on results) but at the codec boundary the reference never pins:
  (i)   cpu_decode(gpu_encode(x)) == x  and  gpu_decode(cpu_encode(x)) == x
  (ii)  gpu-encoded streams satisfy the restated JVM reader's validity rules (oracle decoder = LZ4BlockInputStream)
  (iii) checksums equal the oracle's (zlib-pinned) values
  (iv)  the GPU compressor's bytes equal its executable CPU specification (orc_lz4_compress_block_tile)
"""
import ctypes as C

import numpy as np
import pytest

from conftest import KINDS, corpus

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 3, 4, 5, 12, 13, 15, 16, 17, 63, 64, 255, 511, 512, 513, 4095, 4096, 32767, 32768, 32769, 65536,
         100000, 655360]


# ------------------------------------------------------------------ checksums (K1)
@pytest.mark.parametrize("alg_name", ["ADLER32", "CRC32", "CRC32C"])
def test_checksum_matches_oracle_all_sizes(capi, oracle, alg_name):
    alg = capi.CHECKSUM_BY_NAME[alg_name]
    data = corpus(oracle, "random", 700000, seed=3)
    blocks = [data[:n] for n in SIZES] + [data[7:7 + 33333], data[1:2], data[13:13 + 512]]
    got = capi.checksum_batch(alg, blocks)
    want = [oracle.checksum(alg, b) for b in blocks]
    assert got == want


def test_checksum_known_answers(capi):
    v = capi.checksum_batch(capi.CHECKSUM_CRC32, [b"123456789"])[0]
    assert v == 0xCBF43926
    assert capi.checksum_batch(capi.CHECKSUM_CRC32C, [b"123456789"])[0] == 0xE3069283
    assert capi.checksum_batch(capi.CHECKSUM_ADLER32, [b"123456789"])[0] == 0x091E01DE
    assert capi.checksum_batch(capi.CHECKSUM_ADLER32, [b""])[0] == 1
    assert capi.checksum_batch(capi.CHECKSUM_CRC32, [b""])[0] == 0


@pytest.mark.parametrize("alg_name", ["ADLER32", "CRC32", "CRC32C"])
def test_checksum_packed_unaligned_slices_and_large(capi, oracle, alg_name):
    """Slices at every 16-byte phase, zero-length slices in between, one slice spanning many work items."""
    alg = capi.CHECKSUM_BY_NAME[alg_name]
    rng = np.random.default_rng(11)
    base = np.frombuffer(corpus(oracle, "random", 6 << 20, seed=5), dtype=np.uint8)
    off, ln = [], []
    pos = 0
    for k in range(64):
        pos += int(rng.integers(0, 40))
        l = int(rng.integers(0, 3000)) if k % 5 else 0
        off.append(pos)
        ln.append(l)
        pos += l
    off.append(pos + 3)
    ln.append(base.size - pos - 3)  # ~6 MiB slice
    got = capi.checksum_packed(alg, base, off, ln)
    want = [oracle.checksum(alg, base[o:o + l]) for o, l in zip(off, ln)]
    assert [int(x) for x in got] == want


def test_unsupported_checksum_algorithm_is_rejected(capi):
    """helper/S3ShuffleHelper.scala:100-101 throws UnsupportedOperationException for unknown algorithms."""
    with pytest.raises(capi.B2SError) as e:
        capi.checksum_batch(7, [b"abc"])
    assert e.value.code == capi.E_UNSUPPORTED


# ------------------------------------------------------------------ LZ4Block write side (K2 + K3 + framing)
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_encode_cpu_decode_roundtrip(capi, oracle, kind):
    data = corpus(oracle, kind, 700000, seed=1)
    blocks = [data[:n] for n in SIZES]
    comp, cks, st = capi.compress_batch(capi.CODEC_LZ4BLOCK, blocks, 32768, capi.CHECKSUM_CRC32C)
    assert st == [0] * len(blocks)
    for b, c, k in zip(blocks, comp, cks):
        assert oracle.lz4block_decompress(c) == b          # restated LZ4BlockInputStream accepts and round-trips
        assert k == oracle.crc32c(c)                        # checksum is over the *compressed* stream
        assert len(c) <= capi.compress_bound(capi.CODEC_LZ4BLOCK, 32768, len(b))


def test_empty_stream_is_the_21_byte_end_mark(capi):
    comp, cks, st = capi.compress_batch(capi.CODEC_LZ4BLOCK, [b""], 32768, capi.CHECKSUM_ADLER32)
    assert st == [0]
    assert comp[0].hex() == "4c5a34426c6f636b15" + "00" * 12
    import zlib
    assert cks[0] == zlib.adler32(comp[0])


@pytest.mark.parametrize("kind", ["terasort", "text", "runs", "zeros", "random"])
def test_gpu_compressor_equals_its_cpu_specification(capi, oracle, kind):
    """Byte-for-byte: LZ4Block streams from the kernel == streams built from orc_lz4_compress_block_tile (W=16, hlog 12)."""
    data = corpus(oracle, kind, 300000, seed=2)
    blocks = [data, data[:32768], data[5:5 + 40000], data[:100]]
    comp, _, st = capi.compress_batch(capi.CODEC_LZ4BLOCK, blocks, 32768)
    assert st == [0] * len(blocks)
    for b, c in zip(blocks, comp):
        assert c == oracle.lz4block_compress(b, 32768, compressor=1)


def test_liblz4_decodes_gpu_blocks(capi, oracle):
    """The very routine lz4-java's JNI decompressor calls (LZ4_decompress_fast) must consume exactly compressedLen."""
    try:
        L = C.CDLL("liblz4.so.1")
    except OSError:
        pytest.skip("liblz4 not installed")
    data = corpus(oracle, "terasort", 32768 * 3, seed=9)
    comp, _, st = capi.compress_batch(capi.CODEC_LZ4BLOCK, [data], 32768)
    s = comp[0]
    ip = 0
    out = b""
    while True:
        assert s[ip:ip + 8] == b"LZ4Block"
        tok = s[ip + 8]
        clen = int.from_bytes(s[ip + 9:ip + 13], "little")
        olen = int.from_bytes(s[ip + 13:ip + 17], "little")
        ip += 21
        if olen == 0:
            break
        assert tok == 0x25, "terasort blocks must be stored with the LZ4 method at level 5 (32 KiB)"
        buf = C.create_string_buffer(olen)
        used = L.LZ4_decompress_fast(s[ip:ip + clen], buf, olen)
        assert used == clen
        out += buf.raw
        ip += clen
    assert out == data and ip == len(s)


def test_incompressible_blocks_are_stored_raw(capi, oracle):
    data = corpus(oracle, "random", 70000, seed=4)
    comp, _, st = capi.compress_batch(capi.CODEC_LZ4BLOCK, [data], 32768)
    s = comp[0]
    assert s[8] == 0x15 and int.from_bytes(s[9:13], "little") == 32768 == int.from_bytes(s[13:17], "little")
    assert len(s) == 70000 + 4 * 21
    assert oracle.lz4block_decompress(s) == data


@pytest.mark.parametrize("bs", [64, 1000, 4096, 65536])
def test_block_size_sweep(capi, oracle, bs):
    data = corpus(oracle, "text", 200000, seed=6)
    comp, _, st = capi.compress_batch(capi.CODEC_LZ4BLOCK, [data, data[:bs], data[:bs + 1]], bs)
    assert st == [0, 0, 0]
    for b, c in zip([data, data[:bs], data[:bs + 1]], comp):
        assert oracle.lz4block_decompress(c) == b


def test_compress_packed_layout_is_the_data_object(capi, oracle):
    """Packed output = concatenated partition streams in index order; dst_len is the partitionLengths array."""
    parts = [corpus(oracle, k, n, seed=7) for k, n in
             [("terasort", 70000), ("zeros", 0), ("text", 33000), ("random", 10), ("runs", 131072)]]
    src = np.frombuffer(b"".join(parts), dtype=np.uint8)
    ln = [len(p) for p in parts]
    off = np.concatenate([[0], np.cumsum(ln)[:-1]])
    dst = np.zeros(sum(capi.compress_bound(1, 32768, l) for l in ln), dtype=np.uint8)
    r = capi.compress_packed(capi.CODEC_LZ4BLOCK, src, off, ln, dst, 32768, capi.CHECKSUM_ADLER32)
    assert list(r["status"]) == [0] * 5
    assert list(r["dst_off"]) == list(np.concatenate([[0], np.cumsum(r["dst_len"])[:-1]]))
    assert r["total"] == int(np.sum(r["dst_len"]))
    for i, p in enumerate(parts):
        s = dst[int(r["dst_off"][i]):int(r["dst_off"][i] + r["dst_len"][i])].tobytes()
        assert oracle.lz4block_decompress(s) == p
        assert int(r["checksums"][i]) == oracle.adler32(s)
    # concatenation of all partition streams decodes as one stream too (ShuffleBlockBatchId / Unsafe fast merge)
    assert oracle.lz4block_decompress(dst[: r["total"]].tobytes()) == b"".join(parts)


def test_compress_dst_too_small(capi, oracle):
    data = corpus(oracle, "random", 50000, seed=8)
    comp, _, st = capi.compress_batch(capi.CODEC_LZ4BLOCK, [data, b"abc"], 32768, dst_caps=[1000, 100])
    assert st[0] == capi.E_DST_TOO_SMALL and comp[0] is None
    assert st[1] == 0 and oracle.lz4block_decompress(comp[1]) == b"abc"


# ------------------------------------------------------------------ LZ4Block read side (framing + K4 + K2 + K1)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("compressor", [0, 1])
def test_cpu_encode_gpu_decode_roundtrip(capi, oracle, kind, compressor):
    data = corpus(oracle, kind, 700000, seed=10)
    blocks = [data[:n] for n in SIZES]
    comp = [oracle.lz4block_compress(b, 32768, compressor=compressor) for b in blocks]
    sizes, st = capi.decompressed_size_batch(capi.CODEC_LZ4BLOCK, comp)
    assert st == [0] * len(blocks) and sizes == [len(b) for b in blocks]
    out, st, _ = capi.decompress_batch(capi.CODEC_LZ4BLOCK, comp)
    assert st == [0] * len(blocks)
    assert out == blocks


def test_gpu_decodes_liblz4_streams(capi, oracle):
    """Streams whose blocks were produced by liblz4's LZ4_compress_default (what lz4-java's JNI compressor emits)."""
    try:
        L = C.CDLL("liblz4.so.1")
    except OSError:
        pytest.skip("liblz4 not installed")
    blocks = [corpus(oracle, k, 250000, seed=12) for k in KINDS]
    comp = []
    for b in blocks:
        s = b""
        for o in range(0, len(b), 32768):
            chunk = b[o:o + 32768]
            cap = L.LZ4_compressBound(len(chunk))
            buf = C.create_string_buffer(cap)
            c = L.LZ4_compress_default(chunk, buf, len(chunk), cap)
            method, payload = (0x20, buf.raw[:c]) if c < len(chunk) else (0x10, chunk)
            chk = oracle.xxh32(chunk) & 0x0FFFFFFF
            s += (b"LZ4Block" + bytes([method | 5]) + len(payload).to_bytes(4, "little")
                  + len(chunk).to_bytes(4, "little") + chk.to_bytes(4, "little") + payload)
        s += b"LZ4Block" + bytes([0x15]) + bytes(12)
        assert oracle.lz4block_decompress(s) == b
        comp.append(s)
    out, st, _ = capi.decompress_batch(capi.CODEC_LZ4BLOCK, comp)
    assert st == [0] * len(blocks) and out == blocks


def test_concatenated_streams_decode(capi, oracle):
    """LZ4BlockInputStream(stopOnEmptyBlock=false): after an end mark the next stream continues (batch blocks)."""
    a, b = corpus(oracle, "terasort", 50000, 1), corpus(oracle, "text", 70000, 2)
    s = oracle.lz4block_compress(a) + oracle.lz4block_compress(b"") + oracle.lz4block_compress(b)
    out, st, _ = capi.decompress_batch(capi.CODEC_LZ4BLOCK, [s])
    assert st == [0] and out[0] == a + b


def test_checksum_verified_before_decode_per_slice(capi, oracle):
    """storage/S3ChecksumValidationStream.scala:63-86: each partition slice of a (batch) block is verified over the
    compressed bytes; a mismatch is reported for that block with the slice index, other blocks are unaffected."""
    parts = [corpus(oracle, "terasort", n, seed=20 + i) for i, n in enumerate([40000, 0, 70000, 1000])]
    streams = [oracle.lz4block_compress(p) for p in parts]
    alg = capi.CHECKSUM_ADLER32
    sums = [oracle.adler32(s) for s in streams]
    batch_block = b"".join(streams)                     # ShuffleBlockBatchId covering 4 reduce partitions
    single = streams[2]                                 # ShuffleBlockId
    good = [[(len(s), c) for s, c in zip(streams, sums)], [(len(single), sums[2])]]
    out, st, bad = capi.decompress_batch(capi.CODEC_LZ4BLOCK, [batch_block, single], alg, good)
    assert st == [0, 0] and out[0] == b"".join(parts) and out[1] == parts[2]
    wrong = [[(len(s), c) for s, c in zip(streams, sums)], [(len(single), sums[2])]]
    wrong[0][2] = (len(streams[2]), sums[2] ^ 1)
    out, st, bad = capi.decompress_batch(capi.CODEC_LZ4BLOCK, [batch_block, single], alg, wrong,
                                         dst_caps=[sum(map(len, parts)), len(parts[2])])
    assert st == [capi.E_CHECKSUM, 0] and bad[0] == 2 and out[0] is None and out[1] == parts[2]
    # a flipped payload bit is caught by the checksum before the codec ever sees it
    flipped = bytearray(single)
    flipped[len(flipped) // 2] ^= 0x10
    out, st, bad = capi.decompress_batch(capi.CODEC_LZ4BLOCK, [bytes(flipped)], alg, [[(len(single), sums[2])]],
                                         dst_caps=[len(parts[2])])
    assert st == [capi.E_CHECKSUM] and bad == [0]


def test_corrupt_streams_are_reported_like_the_jvm_reader(capi, oracle):
    """Everything LZ4BlockInputStream rejects with IOException("Stream is corrupted") maps to B2S_E_CORRUPT; the
    oracle (restated reader) must reject exactly the same inputs."""
    data = corpus(oracle, "terasort", 100000, seed=30)
    good = oracle.lz4block_compress(data)
    cases = {}
    m = bytearray(good); m[0] ^= 1; cases["bad magic"] = bytes(m)
    m = bytearray(good); m[8] = 0x35; cases["unknown method"] = bytes(m)
    m = bytearray(good); m[13:17] = (40000).to_bytes(4, "little"); cases["originalLen > 1<<level"] = bytes(m)
    m = bytearray(good); m[17] ^= 0x01; cases["xxh32 mismatch"] = bytes(m)
    m = bytearray(good); m[21 + 100] ^= 0xFF; cases["payload bit flips"] = bytes(m)
    cases["truncated payload"] = good[: len(good) // 2]
    cases["truncated header"] = good[:10]
    m = bytearray(good); m[9:13] = (int.from_bytes(good[9:13], "little") - 1).to_bytes(4, "little")
    cases["compressedLen too short"] = bytes(m)
    m = bytearray(good); m[-1] = 1; cases["end mark with checksum"] = bytes(m)
    names = list(cases)
    blobs = [cases[k] for k in names] + [good]
    for k in names:
        with pytest.raises(IOError):
            oracle.lz4block_decompress(cases[k])
    out, st, _ = capi.decompress_batch(capi.CODEC_LZ4BLOCK, blobs, dst_caps=[len(data) + 70000] * len(blobs))
    for k, s in zip(names, st[:-1]):
        assert s == capi.E_CORRUPT, k
    assert st[-1] == 0 and out[-1] == data


def test_decompress_dst_too_small(capi, oracle):
    data = corpus(oracle, "text", 90000, seed=31)
    s = oracle.lz4block_compress(data)
    out, st, _ = capi.decompress_batch(capi.CODEC_LZ4BLOCK, [s, s], dst_caps=[1000, 90000])
    assert st == [capi.E_DST_TOO_SMALL, 0] and out[1] == data


# ------------------------------------------------------------------ many blocks, multiple chunks, device API
def test_many_small_blocks_config3_shape(capi, oracle):
    """Config-3 shape: thousands of ~64 KiB shuffle blocks in one call (~197 MB: many streams in one host chunk; the
    pipelines over several chunks and slots are tested in test_gpu_chunk_pipelines.py)."""
    n, per = 3000, 65520
    raw = oracle.gen_terasort(0, n * per // 104 + 1).tobytes()
    blocks = [raw[i * per:(i + 1) * per] for i in range(n)]
    comp, cks, st = capi.compress_batch(capi.CODEC_LZ4BLOCK, blocks, 32768, capi.CHECKSUM_CRC32C)
    assert st == [0] * n
    for i in range(0, n, 97):
        assert oracle.lz4block_decompress(comp[i]) == blocks[i] and cks[i] == oracle.crc32c(comp[i])
    slices = [[(len(c), k)] for c, k in zip(comp, cks)]
    out, st, _ = capi.decompress_batch(capi.CODEC_LZ4BLOCK, comp, capi.CHECKSUM_CRC32C, slices,
                                       dst_caps=[per] * n)
    assert st == [0] * n and out == blocks


def test_full_size_roundtrip_properties_device_resident(capi, oracle):
    """BASELINE config-2 shape at 1 GiB through the device API: decode(encode(x)) == x checked on the device with a
    checksum of checksums (CRC32C per shuffle block of the input vs of the round-tripped output)."""
    per = 655200  # 6300 records
    n = 1600
    total = n * per
    d_src = capi.dev_alloc(total)
    d_cmp = capi.dev_alloc(int(total * 1.01) + 4096 * n)
    d_out = capi.dev_alloc(total)
    try:
        capi.gen_terasort_dev(d_src, 0, total // 104)
        off = np.arange(n, dtype=np.uint64) * per
        ln = np.full(n, per, dtype=np.uint64)
        want = capi.checksum_dev(capi.CHECKSUM_CRC32C, d_src, off, ln)
        # spot-check the generator + checksum against the oracle on the first block
        first = oracle.gen_terasort(0, per // 104).tobytes()
        assert int(want[0]) == oracle.crc32c(first)
        w = capi.compress_dev(capi.CODEC_LZ4BLOCK, d_src, off, ln, d_cmp, int(total * 1.01) + 4096 * n, 32768,
                              capi.CHECKSUM_CRC32C)
        assert not w["status"].any()
        ratio = w["total"] / total
        assert 0.3 < ratio < 0.7
        sb = np.arange(n + 1, dtype=np.uint32)
        r = capi.decompress_dev(capi.CODEC_LZ4BLOCK, d_cmp, w["dst_off"], w["dst_len"], d_out, total,
                                capi.CHECKSUM_CRC32C, sb, w["dst_len"], w["checksums"])
        assert not r["status"].any() and r["total"] == total
        assert (r["dst_len"] == ln).all() and (r["dst_off"] == off).all()
        got = capi.checksum_dev(capi.CHECKSUM_CRC32C, d_out, off, ln)
        assert (got == want).all()
        # first compressed stream equals the CPU specification of the kernel
        host = np.empty(int(w["dst_len"][0]), dtype=np.uint8)
        capi.dev_memcpy(host.ctypes.data, d_cmp + int(w["dst_off"][0]), host.size, 2)
        assert host.tobytes() == oracle.lz4block_compress(first, 32768, compressor=1)
    finally:
        for p in (d_src, d_cmp, d_out):
            capi.dev_free(p)
