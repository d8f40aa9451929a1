"""CPU oracle pinned against golden vectors and the native libraries the reference's JVM dependencies wrap (no GPU).

The reference's tests hold no vectors at the codec boundary (SURVEY.md §8c); tests/golden/vectors.json was generated
from liblz4 / zlib / xxhash / snappy (tests/golden/make_golden.py) and is the pin for the oracle — and, through the
gpu-marked tests, for the CUDA path.
"""
import ctypes as C
import json
import os
import zlib

import numpy as np
import pytest

from conftest import KINDS, corpus

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "vectors.json")))
SIZES = [0, 1, 4, 5, 12, 13, 14, 64, 1000, 32767, 32768, 32769, 65536, 100000]


def test_known_answers(oracle):
    k = GOLDEN["kat"]
    assert oracle.crc32(b"123456789") == k["crc32_123456789"]
    assert oracle.crc32c(b"123456789") == k["crc32c_123456789"]
    assert oracle.adler32(b"123456789") == k["adler32_123456789"]
    assert oracle.crc32c(bytes(32)) == k["crc32c_32_zero_bytes"]
    assert oracle.crc32c(b"\xff" * 32) == k["crc32c_32_ff_bytes"]
    assert oracle.crc32c(bytes(range(32))) == k["crc32c_32_incrementing"]
    assert oracle.crc32c(bytes(range(31, -1, -1))) == k["crc32c_32_decrementing"]
    assert oracle.xxh32(b"abc") == k["xxh32_abc_seed9747b28c"]
    assert oracle.xxh32(b"", seed=0) == k["xxh32_empty_seed0"]
    assert oracle.lz4block_compress(b"").hex() == k["lz4block_empty_stream_hex"]
    assert oracle.index_bytes([3, 0, 5]).hex() == k["index_for_lengths_3_0_5_hex"]
    assert oracle.xerial_compress(b"")[:16].hex() == k["xerial_header_hex"]
    assert oracle.adler32(b"") == 1 and oracle.crc32(b"") == 0 and oracle.crc32c(b"") == 0


@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_golden_streams_decode_and_checksum(oracle, name):
    """liblz4-produced LZ4Block streams / snappy-produced xerial streams decode through the restated JVM readers and
    reproduce the zlib / xxhash values recorded when the vectors were made."""
    c = GOLDEN["cases"][name]
    stream = bytes.fromhex(c["lz4block_stream_hex"])
    data = oracle.lz4block_decompress(stream)
    assert len(data) == c["input_len"] == oracle.lz4block_decompressed_size(stream)
    if c["input_hex"] is not None:
        assert data.hex() == c["input_hex"]
    assert oracle.crc32(data) == c["crc32"] and oracle.adler32(data) == c["adler32"]
    assert oracle.xxh32(data) == c["xxh32_seed9747b28c"]
    assert oracle.crc32(stream) == c["lz4block_stream_crc32"]
    assert oracle.adler32(stream) == c["lz4block_stream_adler32"]
    assert oracle.xerial_decompress(bytes.fromhex(c["xerial_stream_hex"])) == data
    # and our own encoders produce streams the same readers accept
    for comp in (0, 1):
        assert oracle.lz4block_decompress(oracle.lz4block_compress(data, 32768, comp)) == data
    assert oracle.xerial_decompress(oracle.xerial_compress(data)) == data


@pytest.mark.parametrize("kind", KINDS)
def test_checksums_match_zlib(oracle, kind):
    data = corpus(oracle, kind, 200000, seed=1)
    for n in SIZES:
        x = data[:n]
        assert oracle.crc32(x) == zlib.crc32(x)
        assert oracle.adler32(x) == zlib.adler32(x)


def test_xxh32_matches_xxhash(oracle):
    xxhash = pytest.importorskip("xxhash")
    data = corpus(oracle, "random", 100000, seed=2)
    for n in SIZES + [15, 16, 17, 31, 33]:
        assert oracle.xxh32(data[:n]) == xxhash.xxh32(data[:n], seed=0x9747B28C).intdigest()


def _liblz4():
    try:
        return C.CDLL("liblz4.so.1")
    except OSError:
        pytest.skip("liblz4.so.1 not present")


@pytest.mark.parametrize("kind", KINDS)
def test_lz4_block_cross_checks_with_liblz4(oracle, kind):
    """restated compressor -> LZ4_decompress_fast (what lz4-java's JNI reader calls) and
    LZ4_compress_default (what its writer calls) -> restated decompressor; both directions exact."""
    L = _liblz4()
    data = corpus(oracle, kind, 70000, seed=3)
    for n in [13, 100, 4096, 32768, 65536]:
        x = data[:n]
        for win in (False, True):
            c = oracle.lz4_compress_block(x, win=win)
            out = C.create_string_buffer(n)
            assert L.LZ4_decompress_fast(c, out, n) == len(c) and out.raw == x
        cap = L.LZ4_compressBound(n)
        buf = C.create_string_buffer(cap)
        cl = L.LZ4_compress_default(x, buf, n, cap)
        y, used = oracle.lz4_decompress_block(buf.raw[:cl], n)
        assert y == x and used == cl


def test_window_model_ratio_is_close_to_liblz4(oracle):
    """The GPU compressor's specification must not give up ratio against the reference's compressor."""
    L = _liblz4()
    for kind, slack in (("terasort", 1.01), ("text", 1.06), ("runs", 1.10), ("period", 1.6)):
        x = corpus(oracle, kind, 32768, seed=4)
        cap = L.LZ4_compressBound(len(x))
        buf = C.create_string_buffer(cap)
        ref = L.LZ4_compress_default(x, buf, len(x), cap)
        ours = len(oracle.lz4_compress_block(x, win=True))
        assert ours <= ref * slack + 16, (kind, ours, ref)


def test_lz4_decoder_enforces_end_of_block_rules(oracle):
    """LZ4_decompress_fast rejects blocks whose last match starts < 12 bytes or ends < 5 bytes before the end."""
    good = oracle.lz4_compress_block(bytes(64))
    y, used = oracle.lz4_decompress_block(good, 64)
    assert y == bytes(64) and used == len(good)
    # one literal 'a' then a match of 19 covering up to the very end (no last literals)
    bad = bytes([0x1F, ord("a"), 0x01, 0x00, 0x00])
    y, used = oracle.lz4_decompress_block(bad, 20)
    assert y is None
    # offset 0 and offset beyond the output are corrupt
    assert oracle.lz4_decompress_block(bytes([0x10, 1, 0, 0]) + bytes(20), 40)[0] is None
    assert oracle.lz4_decompress_block(bytes([0x10, 1, 9, 0]) + bytes(20), 40)[0] is None


def test_lz4_decoder_bounds_long_length_runs(oracle):
    """A literal or match length extended by 9 MiB of 0xFF bytes would pass 2^31: the block is rejected, not decoded
    with a wrapped length (a codec block claiming 32 MiB, lz4-java's largest)."""
    run = b"\xff" * (9 << 20) + b"\x00"
    lit = bytes(range(64))
    olen = 32 << 20
    payloads = [b"\xf0" + run + lit,  # literal length of the first sequence
                bytes([0x40]) + b"abcd" + b"\x01\x00" + bytes([0x0F]) + b"\x01\x00" + run + bytes([0xF0, 49]) + lit]
    for payload in payloads:
        assert oracle.lz4_decompress_block(payload, olen)[0] is None
        frame = (b"LZ4Block" + bytes([0x2F]) + len(payload).to_bytes(4, "little") + olen.to_bytes(4, "little")
                 + (oracle.xxh32(b"") & 0x0FFFFFFF).to_bytes(4, "little") + payload)
        with pytest.raises(IOError):
            oracle.lz4block_decompress(frame + b"LZ4Block" + bytes([0x15]) + bytes(12))


def test_lz4block_reader_rejections(oracle):
    data = corpus(oracle, "terasort", 50000, seed=5)
    good = oracle.lz4block_compress(data)
    assert oracle.lz4block_decompress(good) == data
    assert oracle.lz4block_decompress(good + good) == data + data      # concatenation (stopOnEmptyBlock=false)
    for mutate in (lambda m: m.__setitem__(0, m[0] ^ 1), lambda m: m.__setitem__(8, 0x35),
                   lambda m: m.__setitem__(17, m[17] ^ 1), lambda m: m.__setitem__(200, m[200] ^ 0xFF),
                   lambda m: m.__setitem__(len(m) - 1, 1)):
        m = bytearray(good)
        mutate(m)
        with pytest.raises(IOError):
            oracle.lz4block_decompress(bytes(m))
    with pytest.raises(IOError):
        oracle.lz4block_decompress(good[:-30])


def test_snappy_cross_checks_with_pyarrow(oracle):
    pa = pytest.importorskip("pyarrow")
    codec = pa.Codec("snappy")
    for kind in KINDS:
        data = corpus(oracle, kind, 150000, seed=6)
        for n in [1, 20, 1000, 70000, 150000]:
            x = data[:n]
            assert codec.decompress(oracle.snappy_compress_raw(x), decompressed_size=n).to_pybytes() == x
            assert oracle.snappy_uncompress_raw(codec.compress(x).to_pybytes()) == x
            assert oracle.xerial_decompress(oracle.xerial_compress(x)) == x
    s = oracle.xerial_compress(b"hello world" * 100)
    assert oracle.xerial_decompress(s + s) == b"hello world" * 200       # header re-occurrence = concatenation


def test_index_and_checksum_file_formats(oracle):
    """helper/S3ShuffleHelper.scala:44-59,105-121"""
    lengths = [3, 0, 5, 1 << 33]
    idx = oracle.index_bytes(lengths)
    assert len(idx) == 8 * (len(lengths) + 1)
    assert list(oracle.read_be64(idx)) == [0, 3, 3, 8, 8 + (1 << 33)]
    cs = oracle.be64_bytes([0xCBF43926, 1])
    assert cs.hex() == "00000000cbf43926" "0000000000000001"
    with pytest.raises(ValueError):
        oracle.read_be64(idx[:-1])                                      # "Unexpected file length" (:112-114)


def test_validate_slices_follows_the_reference_stream(oracle):
    """storage/S3ChecksumValidationStream.scala:63-86 over a batch block [start, end) with an empty partition inside."""
    parts = [b"alpha" * 100, b"", b"gamma" * 50, b"d"]
    lengths = [len(p) for p in parts]
    cumulative = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    for alg, fn in ((oracle.ADLER32, zlib.adler32), (oracle.CRC32, zlib.crc32)):
        ref = np.array([fn(p) for p in parts], dtype=np.int64)
        assert oracle.validate_slices(alg, b"".join(parts), cumulative, ref, 0, 4) == -1
        assert oracle.validate_slices(alg, b"".join(parts[1:3]), cumulative, ref, 1, 3) == -1
        bad = ref.copy()
        bad[2] ^= 1
        assert oracle.validate_slices(alg, b"".join(parts), cumulative, bad, 0, 4) == 2
        bad = ref.copy()
        bad[1] = 7   # the empty partition's stored checksum must equal the empty-input checksum too (:80-82)
        assert oracle.validate_slices(alg, b"".join(parts), cumulative, bad, 0, 4) == 1


def test_terasort_generator_layout(oracle):
    r = oracle.gen_terasort(0x1234, 3).tobytes()
    assert len(r) == 312
    rec = r[:104]
    assert rec[:2] == b"\x01\x0b" and rec[12:16] == b"\x01\x5b\x00\x11" and rec[48:52] == b"\x88\x99\xaa\xbb"
    assert rec[16:48] == b"0" * 28 + b"1234" and rec[100:] == b"\xcc\xdd\xee\xff"
    assert all(rec[52 + 4 * k: 56 + 4 * k] == rec[52 + 4 * k: 53 + 4 * k] * 4 for k in range(12))
    assert oracle.gen_terasort(0x1235, 1).tobytes() == r[104:208]        # counter-based: any range reproduces


def test_cpu_baseline_driver_roundtrips(oracle):
    data = oracle.gen_terasort(0, 40 * 630)
    for use in (True, False):
        r = oracle.baseline_run(data, 65520, threads=4, use_liblz4=use)
        assert r["rc"] == 0 and r["errors"] == 0 and 0.3 < r["compressed_bytes"] / r["bytes"] < 0.7


def test_cpu_baseline_driver_other_codecs(oracle):
    """bench.py --codec snappy|zstd: the driver verifies every block it decodes (errors == 0 means bit-exact round
    trips), zstd runs through libzstd.so.1"""
    data = oracle.gen_terasort(7, 30 * 630)
    for codec, lo, hi in (("lz4", 0.3, 0.7), ("snappy", 0.25, 0.7), ("zstd", 0.15, 0.5)):
        r = oracle.baseline_run_codec(codec, data, 65520, threads=3)
        assert r["rc"] == 0 and r["errors"] == 0 and lo < r["compressed_bytes"] / r["bytes"] < hi, (codec, r)


def test_snappy_window_model_is_valid_snappy(oracle):
    """The CPU model of the GPU Snappy compressor (orc_snappy_compress_raw_win via xerial_compress(compressor=1))
    emits streams that the restated reader AND the real snappy library (pyarrow) decode."""
    pa = pytest.importorskip("pyarrow")
    codec = pa.Codec("snappy")
    for kind in KINDS:
        for n in (0, 1, 12, 13, 64, 1000, 32768, 32769, 100000):
            x = corpus(oracle, kind, n, seed=n % 7)
            s = oracle.xerial_compress(x, 32768, compressor=1)
            assert oracle.xerial_decompress(s) == x
            ip = 16
            out = b""
            while ip < len(s):
                clen = int.from_bytes(s[ip:ip + 4], "big")
                chunk = s[ip + 4:ip + 4 + clen]
                ulen = min(32768, n - len(out))
                out += codec.decompress(chunk, decompressed_size=ulen).to_pybytes()
                ip += 4 + clen
            assert out == x
