"""The warp-per-block LZ4 decoder (lz4_decode_warp_kernel): token boundaries found in 128-byte windows, length
extensions, decoy literal bytes, match forms, every corruption rule, RAW blocks and empty streams.

The streams are LZ4Block (lz4-java framing) assembled sequence by sequence, so that token starts, offsets and
extension bytes land at known window positions.  Every good stream is checked against the oracle's decoder first, then
decoded on the GPU through the C ABI; every corrupt one must be rejected by the oracle and by the GPU, without
disturbing the bytes of the streams around it.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import corpus

pytestmark = pytest.mark.gpu

END_MARK = b"LZ4Block" + bytes([0x15]) + bytes(12)
WIN = 128  # compressed bytes per window of the decoder


# ------------------------------------------------------------------ stream assembly
def ext(n):
    """the LZ4 length-extension bytes of a 4-bit field that is saturated (n = length - 15 >= 0)"""
    out = bytearray()
    while n >= 255:
        out.append(255)
        n -= 255
    out.append(n)
    return bytes(out)


def enc_seq(lit, off, ml):
    """one sequence: literals, then a match (off, ml >= 4); -> encoded bytes"""
    ll = len(lit)
    e = bytearray([(min(ll, 15) << 4) | min(ml - 4, 15)])
    if ll >= 15:
        e += ext(ll - 15)
    e += lit + off.to_bytes(2, "little")
    if ml - 4 >= 15:
        e += ext(ml - 4 - 15)
    return bytes(e)


def enc_last(lit):
    e = bytearray([min(len(lit), 15) << 4])
    if len(lit) >= 15:
        e += ext(len(lit) - 15)
    return bytes(e + lit)


def block(seqs, tail):
    """raw LZ4 block from [(literals, offset, match length)] and the final literals; -> (payload, decoded bytes)"""
    out, enc = bytearray(), bytearray()
    for lit, off, ml in seqs:
        assert ml >= 4 and 1 <= off <= len(out) + len(lit)
        enc += enc_seq(lit, off, ml)
        out += lit
        for _ in range(ml):  # byte by byte: overlapping matches repeat what they have just written
            out.append(out[-off])
    enc += enc_last(tail)
    out += tail
    return bytes(enc), bytes(out)


def frame(oracle, payload, olen, data=None):
    """one LZ4Block codec block: compressed payload (None = stored RAW of data) claiming olen decoded bytes"""
    data = data if data is not None else b""
    level = max(0, (max(olen, 1) - 1).bit_length() - 10)
    method, body = (0x20, payload) if payload is not None else (0x10, data)
    chk = oracle.xxh32(data) & 0x0FFFFFFF
    return (b"LZ4Block" + bytes([method | level]) + len(body).to_bytes(4, "little") + olen.to_bytes(4, "little")
            + chk.to_bytes(4, "little") + body)


def stream(oracle, blocks):
    """[(payload, decoded bytes)] -> LZ4Block stream (payload None = stored RAW)"""
    return b"".join(frame(oracle, p, len(d), d) for p, d in blocks) + END_MARK


def oracle_stream(oracle, data, block_size):
    """data compressed block by block by the oracle's LZ4 compressor (stored RAW where it does not shrink)"""
    s = b""
    for i in range(0, len(data), block_size):
        piece = data[i:i + block_size]
        c = oracle.lz4_compress_block(piece, cap=len(piece) - 1) if len(piece) > 1 else None
        s += frame(oracle, c, len(piece), piece)
    return s + END_MARK


def liblz4_stream(oracle, data, block_size=65536):
    """data compressed by liblz4's LZ4_compress_default, in LZ4Block framing"""
    L = C.CDLL("liblz4.so.1")
    L.LZ4_compress_default.restype = C.c_int
    s = b""
    for i in range(0, len(data), block_size):
        piece = data[i:i + block_size]
        cap = len(piece) + len(piece) // 255 + 64
        out = C.create_string_buffer(cap)
        n = L.LZ4_compress_default(C.c_char_p(piece), out, len(piece), cap)
        assert n > 0
        s += frame(oracle, out.raw[:n], len(piece), piece)
    return s + END_MARK


# ------------------------------------------------------------------ decoding
def decode(capi, streams, dev=False):
    """-> (decoded bytes or None per stream, status, the whole destination arena, decompress result)"""
    ln = np.array([len(s) for s in streams], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    src = np.frombuffer(b"".join(streams) + b"\0", np.uint8)
    cap = int(sum(max(0, capi.decompressed_size_batch(capi.CODEC_LZ4BLOCK, [s])[0][0]) for s in streams)) + 4096
    dst = np.full(cap, 0xA5, np.uint8)
    if dev:
        d_src, d_dst = capi.dev_alloc(src.size), capi.dev_alloc(cap)
        try:
            capi.dev_memcpy(d_src, src.ctypes.data, src.size, 1)
            capi.dev_memcpy(d_dst, dst.ctypes.data, cap, 1)
            r = capi.decompress_dev(capi.CODEC_LZ4BLOCK, d_src, off, ln, d_dst, cap)
            capi.dev_memcpy(dst.ctypes.data, d_dst, cap, 2)
        finally:
            capi.dev_free(d_src)
            capi.dev_free(d_dst)
    else:
        r = capi.decompress_packed(capi.CODEC_LZ4BLOCK, src, off, ln, dst)
    outs = [dst[int(o):int(o) + int(n)].tobytes() if s == 0 else None
            for o, n, s in zip(r["dst_off"], r["dst_len"], r["status"])]
    return outs, [int(s) for s in r["status"]], dst, r


def check_good(capi, oracle, streams, expected):
    for s, e in zip(streams, expected):
        assert oracle.lz4block_decompress(s) == e
    for dev in (False, True):
        outs, st, dst, r = decode(capi, streams, dev)
        assert st == [0] * len(streams)
        for i, e in enumerate(expected):
            assert outs[i] == e, (dev, i)
        assert (dst[int(r["total"]):] == 0xA5).all()  # nothing past the decoded streams


# ------------------------------------------------------------------ tests
def test_token_boundaries_at_every_window_position(capi, oracle):
    """A first sequence of 1..300 literals shifts everything after it, so each token start, offset and extension byte
    of the sequences that follow lands at every residue of the window, and across the window's end."""
    rng = np.random.default_rng(1)
    streams, expected = [], []
    for lead in range(1, 300):
        lit0 = rng.integers(0, 256, lead, dtype=np.uint8).tobytes()
        seqs = [(lit0, 1, 4)]
        for k in range(40):
            seqs.append((bytes([k]) * (k % 5), 1 + k % 7, 4 + k % 9))
        seqs.append((bytes(range(20)), 3, 40))  # both lengths extended
        seqs.append((b"q" * 15, 15, 19))  # extension bytes of value 0
        for k in range(40):
            seqs.append((b"", 1 + k % 3, 5))
        payload, data = block(seqs, b"t" * 12)
        streams.append(stream(oracle, [(payload, data)]))
        expected.append(data)
    check_good(capi, oracle, streams, expected)


@pytest.mark.parametrize("which", ["ll", "ml"])
def test_length_extension_chains(capi, oracle, which):
    """0, 1, 2 and many 0xFF extension bytes on the literal or the match length, at several window positions"""
    rng = np.random.default_rng(2)
    streams, expected = [], []
    for n in (14, 15, 16, 200, 269, 270, 271, 524, 525, 526, 1000, 5000):
        for lead in (1, 5, 60, 120, 126, 127):
            seqs = [(rng.integers(0, 256, lead, dtype=np.uint8).tobytes(), 1, 4)]
            if which == "ll":
                seqs.append((rng.integers(0, 256, n, dtype=np.uint8).tobytes(), 7, 4))
            else:
                seqs.append((b"ab", 2, n + 4))
            seqs += [(b"z", 2, 6)] * 30
            payload, data = block(seqs, b"end of block".ljust(12, b"."))
            streams.append(stream(oracle, [(payload, data)]))
            expected.append(data)
    check_good(capi, oracle, streams, expected)


def test_long_literal_runs_and_all_literal_blocks(capi, oracle):
    rng = np.random.default_rng(3)
    blocks = []
    for n in (15, 270, 32000):
        payload, data = block([(rng.integers(0, 256, n, dtype=np.uint8).tobytes(), 3, 9)] * 2, b"0123456789ab")
        blocks.append((payload, data))
    streams = [stream(oracle, [b]) for b in blocks]
    expected = [b[1] for b in blocks]
    for n in (12, 13, 100, 4000, 65000):  # a block that is one literals-only sequence (clen < 64 KiB)
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        streams.append(stream(oracle, [(enc_last(data), data)]))
        expected.append(data)
    check_good(capi, oracle, streams, expected)


def test_decoy_literal_bytes(capi, oracle):
    """literal bytes that would parse as long tokens (0xFF, 0xF0, 0x0F) if the chain were resolved wrongly"""
    streams, expected = [], []
    for pat in (b"\xff", b"\xf0", b"\x0f", b"\xff\x0f", b"\xf0\xff\xff", b"\x0f\xff\x00"):
        for n in (1, 2, 3, 7, 14, 15, 16, 40):
            lit = (pat * n)[:n]
            seqs = [(lit, 1, 4)] + [((pat * 9)[: 1 + k % 9], 1 + k % 4, 4 + k % 6) for k in range(60)]
            payload, data = block(seqs, (pat * 12)[:12] + b"\xff" * 3)
            streams.append(stream(oracle, [(payload, data)]))
            expected.append(data)
    check_good(capi, oracle, streams, expected)


def test_match_forms(capi, oracle):
    """offsets 1..16 with match lengths 4..300 (overlapping copies), a last match that ends 5 bytes before the end"""
    rng = np.random.default_rng(4)
    streams, expected = [], []
    for off in range(1, 17):
        seqs = [(rng.integers(0, 256, 16, dtype=np.uint8).tobytes(), off, 4)]
        for ml in (4, 5, 7, 8, 15, 16, 17, 18, 19, 20, 33, 64, 95, 96, 97, 128, 255, 300):
            seqs.append((rng.integers(0, 256, int(rng.integers(0, 4)), dtype=np.uint8).tobytes(), off, ml))
        payload, data = block(seqs, b"x" * 12)
        streams.append(stream(oracle, [(payload, data)]))
        expected.append(data)
        # the last match starts 12 bytes before the end and leaves exactly 5 literals
        payload, data = block([(b"abcdefgh", 8, 4), (b"", off if off <= 12 else 12, 7)], b"12345")
        streams.append(stream(oracle, [(payload, data)]))
        expected.append(data)
    check_good(capi, oracle, streams, expected)


@pytest.mark.parametrize("size", [13, 100, 1000, 4096, 32768, 65536])
def test_compressed_blocks_of_every_size(capi, oracle, size):
    """blocks of 13 bytes to 64 KiB from the oracle's compressor and from liblz4"""
    streams, expected = [], []
    # (random bytes in 64 KiB blocks would expand past 64 KiB, which is the tile decoder's case)
    for kind in ("terasort", "text", "runs", "period") + (("random",) if size < 65536 else ()):
        data = corpus(oracle, kind, size * 3 + 7, seed=size)
        streams.append(oracle_stream(oracle, data, size))
        expected.append(data)
        streams.append(liblz4_stream(oracle, data, size))
        expected.append(data)
    check_good(capi, oracle, streams, expected)


def test_raw_blocks_and_empty_streams(capi, oracle):
    rng = np.random.default_rng(5)
    data = corpus(oracle, "terasort", 100000, seed=5)
    raw = rng.integers(0, 256, 30000, dtype=np.uint8).tobytes()
    mixed = oracle.lz4block_compress(data)[: -len(END_MARK)] + frame(oracle, None, len(raw), raw) + \
        oracle.lz4block_compress(data[:777])
    streams = [mixed, END_MARK, oracle.lz4block_compress(data), END_MARK, stream(oracle, [(None, raw)] * 3)]
    expected = [data + raw + data[:777], b"", data, b"", raw * 3]
    check_good(capi, oracle, streams, expected)


# ------------------------------------------------------------------ corruption
def good_prefix(n):
    """n short sequences (token, 1 literal, 2-byte offset: 4 compressed bytes, 5 decoded bytes each)"""
    return [(bytes([65 + k % 26]), 1, 4) for k in range(n)]


def corrupt_case(rule, n):
    """a raw block that breaks `rule` right after n good sequences; -> (payload, claimed decoded length)"""
    pre, out = block(good_prefix(n), b"")[0][:-1], 5 * n  # drop the empty final token
    if rule == "token_past_end":  # the block ends where a token must start
        return pre + enc_seq(b"a", 1, 4), out + 5 + 20
    if rule == "extension_past_end":  # the literal-length extension runs off the end
        return pre + b"\xf0" + b"\xff" * 3, out + 2000
    if rule == "literals_past_output":  # ll > olen - op
        return pre + enc_last(b"L" * 20), out + 19
    if rule == "literals_past_input":  # ll > clen - ip
        return pre + bytes([0xE0]) + b"L" * 5, out + 14
    if rule == "last_short_output":  # fewer than 12 bytes left after the literals, but op != olen
        return pre + enc_last(b"L" * 13), out + 20
    if rule == "last_trailing_input":  # op == olen after the last literals, but bytes are left over
        return pre + enc_last(b"L" * 13) + b"\x00", out + 13
    if rule == "offset_past_end":  # ip + 2 > clen before the offset
        return pre + bytes([0x20]) + b"LL" + b"\x01", out + 100
    if rule == "offset_zero":
        return pre + enc_seq(b"a", 1, 4)[:2] + b"\x00\x00" + enc_last(b"T" * 12), out + 5 + 12
    if rule == "offset_past_output":  # off > op
        return pre + enc_seq(b"a", 1, 4)[:2] + (out + 2).to_bytes(2, "little") + enc_last(b"T" * 12), out + 5 + 12
    if rule == "match_past_output":  # ml > olen - op
        return pre + enc_seq(b"a", 1, 30) + enc_last(b"T" * 12), out + 1 + 20
    if rule == "match_into_last_literals":  # fewer than 5 bytes left after a match
        return pre + enc_seq(b"a", 1, 10) + enc_last(b"T" * 3), out + 1 + 10 + 3
    raise ValueError(rule)


RULES = ["token_past_end", "extension_past_end", "literals_past_output", "literals_past_input", "last_short_output",
         "last_trailing_input", "offset_past_end", "offset_zero", "offset_past_output", "match_past_output",
         "match_into_last_literals"]


@pytest.mark.parametrize("rule", RULES)
def test_one_corrupt_stream_among_good_ones(capi, oracle, rule):
    """one corrupt stream between good ones, with the bad sequence inside a batch (after 10 good ones) and at batch
    and window boundaries (after 31, 32, 33 and 64): it alone is CORRUPT and the neighbours decode intact"""
    data = corpus(oracle, "terasort", 70000, seed=6)
    good = oracle.lz4block_compress(data)
    for n in (0, 10, 31, 32, 33, 64):
        payload, olen = corrupt_case(rule, n)
        bad = frame(oracle, payload, olen) + END_MARK
        with pytest.raises(IOError):
            oracle.lz4block_decompress(bad)
        streams = [good, bad, good]
        for dev in (False, True):
            outs, st, dst, r = decode(capi, streams, dev)
            assert st == [0, capi.E_CORRUPT, 0], (rule, n, dev)
            assert outs[0] == data and outs[2] == data, (rule, n, dev)
            end = int(r["dst_off"][2]) + int(r["dst_len"][2])
            assert (dst[end:] == 0xA5).all()
