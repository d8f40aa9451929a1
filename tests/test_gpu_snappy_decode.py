"""The Snappy decoder (xerial_walk_kernel -> snappy_tokens_kernel -> snappy_copy_kernel) on every element form, the
edges of its 16-bit record fields and record workspace, batches of more than one group of chunks, every rejection rule,
and chunks whose claim it does not decode.

Streams are xerial framing (SnappyOutputStream) over raw Snappy chunks assembled element by element, so that every
literal-length encoding (the 3- and 4-byte extensions too, which no compressor in the suite writes) and every copy kind
lands where it is meant to.  Every good stream is checked against the oracle's decoder first, then decoded on the GPU
through the packed and the device call into a destination filled with 0xA5; every bad stream sits between good ones
and must be the only one that fails, with the neighbours intact and nothing written past the last stream.  A CPU test
holds each hand-assembled chunk's verdict to the real snappy library's (pyarrow), the library snappy-java wraps.
"""
import numpy as np
import pytest

from conftest import corpus

HEADER = b"\x82SNAPPY\x00" + (1).to_bytes(4, "big") + (1).to_bytes(4, "big")
RNG = np.random.default_rng(11)


def rand(n):
    return RNG.integers(0, 256, n, dtype=np.uint8).tobytes()


# ------------------------------------------------------------------ element assembly
def varint(n):
    out = bytearray()
    while n >= 0x80:
        out.append((n & 0x7F) | 0x80)
        n >>= 7
    out.append(n)
    return bytes(out)


def lit(data, ext=None):
    """a literal element; ext = number of length-extension bytes (0..4; None: the shortest form)"""
    n1 = len(data) - 1
    if ext is None:
        ext = 0 if n1 < 60 else 1 if n1 < 256 else 2 if n1 < 65536 else 3
    if ext == 0:
        assert n1 < 60
        return bytes([n1 << 2]) + data
    return bytes([(59 + ext) << 2]) + n1.to_bytes(ext, "little") + data


def copy1(off, ln):
    assert 4 <= ln <= 11 and 0 <= off < 2048
    return bytes([1 | ((ln - 4) << 2) | ((off >> 8) << 5), off & 0xFF])


def copy2(off, ln):
    assert 1 <= ln <= 64 and 0 <= off < 65536
    return bytes([2 | ((ln - 1) << 2)]) + off.to_bytes(2, "little")


def copy4(off, ln):
    assert 1 <= ln <= 64
    return bytes([3 | ((ln - 1) << 2)]) + off.to_bytes(4, "little")


def copy(off, ln):
    return copy1(off, ln) if 4 <= ln <= 11 and off < 2048 else copy2(off, ln)


class Chunk:
    """a raw Snappy chunk built element by element, with the bytes it decodes to"""

    def __init__(self):
        self.enc, self.out = bytearray(), bytearray()

    def lit(self, data, ext=None):
        self.enc += lit(data, ext)
        self.out += data
        return self

    def copy(self, off, ln, form=None):
        assert 1 <= off <= len(self.out)
        self.enc += {None: copy, 1: copy1, 2: copy2, 4: copy4}[form](off, ln)
        for _ in range(ln):  # byte by byte: an overlapping copy repeats what it has just written
            self.out.append(self.out[-off])
        return self

    def raw(self, claim=None):
        return varint(len(self.out) if claim is None else claim) + bytes(self.enc)


def xerial(raws):
    """[raw chunk | b"HEADER" (a concatenated stream's header)] -> xerial stream"""
    return HEADER + b"".join(HEADER if r == b"HEADER" else len(r).to_bytes(4, "big") + r for r in raws)


def one(chunk, claim=None):
    return xerial([chunk.raw(claim)])


# ------------------------------------------------------------------ decoding
def decode(capi, streams, dev=False):
    """-> (decoded bytes or None per stream, status, the whole destination arena, decompress result).  The
    destination holds any claim the decoder accepts (at most 64 decoded bytes per 3 compressed bytes)."""
    ln = np.array([len(s) for s in streams], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    src = np.frombuffer(b"".join(streams) + b"\0", np.uint8)
    cap = int(ln.sum()) * 22 + 4096
    dst = np.full(cap, 0xA5, np.uint8)
    if dev:
        d_src, d_dst = capi.dev_alloc(src.size), capi.dev_alloc(cap)
        try:
            capi.dev_memcpy(d_src, src.ctypes.data, src.size, 1)
            capi.dev_memcpy(d_dst, dst.ctypes.data, cap, 1)
            r = capi.decompress_dev(capi.CODEC_SNAPPY_XERIAL, d_src, off, ln, d_dst, cap)
            capi.dev_memcpy(dst.ctypes.data, d_dst, cap, 2)
        finally:
            capi.dev_free(d_src)
            capi.dev_free(d_dst)
    else:
        r = capi.decompress_packed(capi.CODEC_SNAPPY_XERIAL, src, off, ln, dst)
    outs = [dst[int(o):int(o) + int(n)].tobytes() if s == 0 else None
            for o, n, s in zip(r["dst_off"], r["dst_len"], r["status"])]
    return outs, [int(s) for s in r["status"]], dst, r


def check_good(capi, oracle, streams, expected, paths=(False, True)):
    for s, e in zip(streams, expected):
        assert oracle.xerial_decompress(s) == e
    for dev in paths:
        outs, st, dst, r = decode(capi, streams, dev)
        assert st == [0] * len(streams), dev
        for i, e in enumerate(expected):
            assert outs[i] == e, (dev, i)
        assert (dst[int(r["total"]):] == 0xA5).all()  # nothing past the decoded streams


def check_alone(capi, streams, expect, paths=(False, True)):
    """streams[i] must get status expect[i]; the good ones decode to what the oracle makes of them, and nothing is
    written past the last stream"""
    want = [oracle_or_none(s) if e == 0 else None for s, e in zip(streams, expect)]
    for dev in paths:
        outs, st, dst, r = decode(capi, streams, dev)
        assert st == expect, dev
        for i, w in enumerate(want):
            if w is not None:
                assert outs[i] == w, (dev, i)
        end = int(r["dst_off"][-1]) + int(r["dst_len"][-1])
        assert (dst[end:] == 0xA5).all(), dev


def oracle_or_none(s):
    from oracle import oracle as o
    try:
        return o.xerial_decompress(s)
    except IOError:
        return None


# ------------------------------------------------------------------ good forms
def literal_form_streams():
    """every literal length encoding: inline 1..60, and 1-, 2-, 3- and 4-byte extensions, minimal or not"""
    streams, expected = [], []
    for n in list(range(1, 61)) + [61, 62, 200, 255, 256, 257, 258, 4000, 30000]:
        for ext in range(5):
            if (ext == 0 and n > 60) or (ext == 1 and n > 256):
                continue
            c = Chunk().lit(rand(n), ext)
            c.copy(min(n, 7), 9).lit(rand(3), ext)  # a literal paired with a copy, then a trailing one
            streams.append(one(c))
            expected.append(bytes(c.out))
    return streams, expected


@pytest.mark.gpu
def test_literal_length_forms(capi, oracle):
    check_good(capi, oracle, *literal_form_streams())


def copy_form_streams():
    streams, expected = [], []
    # copy-1: all eight lengths at every offset 1..2047, one chunk per length
    raws, out = [], b""
    for ln in range(4, 12):
        c = Chunk().lit(rand(2048))
        for off in range(1, 2048):
            c.copy(off, ln, 1)
        raws.append(c.raw())
        out += bytes(c.out)
    streams.append(xerial(raws))
    expected.append(out)
    # copy-2: lengths 1..64 (1..3 included, which only copy-2 and copy-4 encode) at spread offsets
    c = Chunk().lit(rand(3000))
    for ln in range(1, 65):
        for off in (1, 2, 3, 17, 255, 256, 2047, 2048, 2999):
            c.copy(off, ln, 2)
    streams.append(one(c))
    expected.append(bytes(c.out))
    # copy-2 at offsets up to 65535: a chunk of 65536 decoded bytes whose last copies reach back to its first byte
    c = Chunk()
    for k in range(4):
        c.lit(rand(16350))  # consecutive literals
    c.copy(65400, 64, 2).copy(65464, 64, 2).copy(65528, 7, 2).copy(65535, 1, 2)
    assert len(c.out) == 65536
    streams.append(one(c))
    expected.append(bytes(c.out))
    # copy-4 at several lengths and offsets
    c = Chunk().lit(rand(5000))
    for off, ln in [(1, 1), (1, 64), (2, 3), (7, 33), (2048, 12), (4999, 64), (5000, 2), (40000, 64), (65535, 5)]:
        if off <= len(c.out):
            c.copy(off, ln, 4)
    c.copy(len(c.out), 64, 4)
    while len(c.out) < 65535:
        c.copy(min(len(c.out), 60000), min(64, 65535 - len(c.out)), 2)
    c.copy(65535, 1, 4)
    streams.append(one(c))
    expected.append(bytes(c.out))
    # overlapping copies: offsets 1..16, each copy kind, lengths across the warp's byte groups
    for form in (1, 2, 4):
        c = Chunk().lit(rand(16))
        for off in range(1, 17):
            for ln in ((4, 5, 8, 11) if form == 1 else (1, 2, 3, 4, 8, 15, 16, 17, 31, 32, 33, 63, 64)):
                c.copy(off, ln, form)
            c.lit(rand(off % 3 + 1))
        streams.append(one(c))
        expected.append(bytes(c.out))
    return streams, expected


@pytest.mark.gpu
def test_copy_forms(capi, oracle):
    check_good(capi, oracle, *copy_form_streams())


def edge_streams():
    streams, expected = [], []
    # consecutive literals of every header size, with and without a copy between them
    c = Chunk().lit(rand(3)).lit(rand(70)).lit(rand(300)).lit(rand(1)).copy(5, 20).lit(rand(2)).lit(rand(61), 4)
    streams.append(one(c))
    expected.append(bytes(c.out))
    # the largest chunk taken: 65535 compressed bytes of one-byte literals (records fill the workspace stride)
    c = Chunk()
    for _ in range(32766):
        c.lit(rand(1))
    assert len(c.raw()) == 65535
    streams.append(one(c))
    expected.append(bytes(c.out))
    # a chunk of 65536 decoded bytes made of copies
    c = Chunk().lit(rand(1))
    for _ in range(1023):
        c.copy(1, 64, 2)
    c.copy(64, 63, 2)
    assert len(c.out) == 65536
    streams.append(one(c))
    expected.append(bytes(c.out))
    # a literal of more than 65000 bytes, paired with copies
    c = Chunk().lit(rand(65100)).copy(65100, 64).copy(3, 11).copy(65000, 64)
    streams.append(one(c))
    expected.append(bytes(c.out))
    # a literal that starts past compressed position 65000, paired with a copy
    c = Chunk().lit(rand(65010))
    assert len(c.enc) + 2 > 65000  # the second literal's bytes start there (after its 2-byte header)
    c.lit(rand(100)).copy(100, 4).copy(65000, 60)
    streams.append(one(c))
    expected.append(bytes(c.out))
    # a 4-byte literal length of 0xFFFFFFFF: the snappy library's 32-bit length wraps to an empty literal, and
    # snappy-java accepts the chunk
    c = Chunk().lit(rand(20))
    c.enc += bytes([63 << 2]) + b"\xff" * 4
    c.copy(20, 30).lit(rand(5))
    c.enc += bytes([63 << 2]) + b"\xff" * 4
    streams.append(one(c))
    expected.append(bytes(c.out))
    # the stream header again mid-stream (concatenated streams), twice in a row too
    a, b = Chunk().lit(rand(40)).copy(40, 64), Chunk().lit(b"x").copy(1, 30)
    streams.append(xerial([a.raw(), b"HEADER", b.raw(), b"HEADER", b"HEADER", a.raw()]))
    expected.append(bytes(a.out) + bytes(b.out) + bytes(a.out))
    # an empty stream and a header-only stream
    streams += [b"", HEADER]
    expected += [b"", b""]
    return streams, expected


@pytest.mark.gpu
def test_record_field_and_workspace_edges(capi, oracle):
    """the largest chunk and the 16-bit record fields, with chunks around them in the same launch"""
    streams, expected = edge_streams()
    data = corpus(oracle, "text", 100000, seed=12)
    good = oracle.xerial_compress(data)
    streams = [good] + [x for s in streams for x in (s, good)]
    expected = [data] + [x for e in expected for x in (e, data)]
    check_good(capi, oracle, streams, expected)


def max_expansion_chunk():
    """the most decoded bytes per compressed byte: one literal byte, then copy-2 elements of 64 bytes"""
    c = Chunk().lit(b"m")
    for _ in range(1023):
        c.copy(1, 64, 2)
    return c


@pytest.mark.gpu
def test_max_expansion_chunk_is_within_the_claim_bound(capi, oracle):
    """A chunk of 3071 element bytes that decodes to 65473 bytes (64 per 3): the claim bound of the walk (3 * claim
    <= 64 * element bytes) takes it.  The same elements under a claim above 65536 that the bound allows are
    UNSUPPORTED (not CORRUPT), and under a claim past the bound CORRUPT."""
    c = max_expansion_chunk()
    e = len(c.enc)
    assert 3 * len(c.out) <= 64 * e < 3 * (len(c.out) + 42)
    check_good(capi, oracle, [one(c)], [bytes(c.out)])
    d = Chunk().lit(rand(200)).copy(200, 64, 2)
    for _ in range(2000):
        d.copy(64, 64, 2)
    assert 64 * len(d.enc) // 3 > 65537
    good = oracle.xerial_compress(corpus(oracle, "text", 50000, seed=13))
    for claim, want in ((65537, capi.E_UNSUPPORTED), (64 * len(d.enc) // 3, capi.E_UNSUPPORTED),
                        (64 * len(d.enc) // 3 + 1, capi.E_CORRUPT), (64 * e // 3 + 1, capi.E_CORRUPT)):
        bad = one(d if claim != 64 * e // 3 + 1 else c, claim)
        check_alone(capi, [good, bad, good], [0, want, 0])


@pytest.mark.gpu
def test_more_chunks_than_one_group(capi, oracle):
    """A batch of 70400 chunks (the decoder runs groups of 65536), with a bad stream whose chunks straddle the group
    boundary and whose bad element is in the second group: it alone is CORRUPT.  Through the device call, which keeps
    the batch in one launch sequence."""
    def small(k):
        c = Chunk().lit(bytes([k & 255, 7, k >> 8 & 255])).copy(3, 4 + k % 8).copy(1 + k % 3, 1 + k % 20, 2)
        return c
    streams, expected = [], []
    for s in range(320):  # 220 chunks a stream
        cs = [small(s * 220 + k) for k in range(220)]
        streams.append(xerial([c.raw() for c in cs]))
        expected.append(b"".join(bytes(c.out) for c in cs))
    check_good(capi, oracle, streams, expected, paths=(True,))
    at = 65536 // 220  # the stream holding chunk 65536
    cs = [small(k) for k in range(220)]
    raws = [c.raw() for c in cs]
    k_bad = 65536 - at * 220 + 3  # three chunks past the boundary
    raws[k_bad] = raws[k_bad][:1] + bytes([40 << 2]) + raws[k_bad][2:]  # a literal longer than the chunk
    bad = xerial(raws)
    with pytest.raises(IOError):
        oracle.xerial_decompress(bad)
    streams[at] = bad
    expect = [0] * len(streams)
    expect[at] = capi.E_CORRUPT
    check_alone(capi, streams, expect, paths=(True,))


# ------------------------------------------------------------------ rejection rules
def bad_chunks():
    """name -> a raw chunk (after the framing) that the format rejects"""
    base = Chunk().lit(rand(20)).copy(20, 30)
    n = len(base.out)
    pre = bytes(base.enc)
    return {
        "varint_longer_than_5": b"\x80\x80\x80\x80\x80\x01" + pre,
        "varint_above_2_32": b"\xff\xff\xff\xff\x10" + pre,
        "claim_more_than_produced": varint(n + 1) + pre,
        "claim_fewer_than_produced": varint(n - 1) + pre,
        "literal_extension_past_input": varint(n + 300) + pre + bytes([61 << 2, 0x2C]),
        "literal_4byte_extension_past_input": varint(n + 300) + pre + bytes([63 << 2, 0x2C, 1, 0]),
        "literal_past_input": varint(n + 10) + pre + bytes([9 << 2]) + b"12345",
        "literal_past_output": varint(n + 9) + pre + lit(b"0123456789"),
        "copy1_offset_past_input": varint(n + 4) + pre + bytes([1]),
        "copy2_offset_past_input": varint(n + 4) + pre + bytes([2 | (3 << 2), 1]),
        "copy4_offset_past_input": varint(n + 4) + pre + bytes([3 | (3 << 2), 1, 0, 0]),
        "copy1_offset_0": varint(n + 4) + pre + copy1(0, 4),
        "copy2_offset_0": varint(n + 4) + pre + copy2(0, 4),
        "copy4_offset_0": varint(n + 4) + pre + copy4(0, 4),
        "offset_op_plus_1": varint(n + 4) + pre + copy2(n + 1, 4),
        "copy_before_any_output": varint(4) + copy2(1, 4),
        "copy_past_output": varint(n + 3) + pre + copy2(1, 4),
        "copy4_offset_65536": varint(n + 4) + pre + copy4(65536, 4),
        "copy4_offset_2_32_minus_1": varint(n + 4) + pre + copy4(0xFFFFFFFF, 4),
        "copy1_at_end_past_output": varint(n) + pre + copy1(1, 4),
    }


def bad_streams():
    """name -> a xerial stream that breaks one framing or element rule"""
    good = Chunk().lit(rand(30)).copy(30, 40)
    g = good.raw()
    out = {
        "bad_magic": HEADER[:1] + b"S" + b"n" + HEADER[3:] + len(g).to_bytes(4, "big") + g,
        "bad_magic_tail": HEADER[:7] + b"\x01" + HEADER[8:] + len(g).to_bytes(4, "big") + g,
        "short_stream_1": HEADER[:1],
        "short_stream_15": HEADER[:15],
        "chunk_length_past_end": HEADER + (len(g) + 1).to_bytes(4, "big") + g,
        "chunk_length_0": HEADER + bytes(4),
        "chunk_length_0_after_a_chunk": xerial([g]) + bytes(4),
        "mid_header_bad_tail": xerial([g]) + HEADER[:4] + b"PAPPY\x00" + HEADER[10:] + len(g).to_bytes(4, "big") + g,
        "mid_header_truncated": xerial([g]) + HEADER[:12],
    }
    for k in (1, 2, 3):
        out["trailing_%d_bytes" % k] = xerial([g]) + bytes(k)
    for name, raw in bad_chunks().items():
        out[name] = xerial([g, raw])
    # the same offset at exactly op is valid; op + 1 reaches into the previous chunk's output in the arena
    ok = Chunk().lit(rand(8)).copy(8, 4, 2)
    out["offset_op_plus_1_after_a_chunk"] = xerial([g, varint(12) + lit(bytes(ok.out[:8])) + copy2(9, 4)])
    return out


def valid_offset_at_op():
    g = Chunk().lit(rand(30)).copy(30, 40)
    ok = Chunk().lit(rand(8)).copy(8, 4, 2)
    return xerial([g.raw(), ok.raw()]), bytes(g.out) + bytes(ok.out)


BAD = sorted(bad_streams())


@pytest.mark.gpu
@pytest.mark.parametrize("rule", BAD)
def test_one_bad_stream_among_good_ones(capi, oracle, rule):
    """the bad stream alone is CORRUPT; its neighbours (one of them with chunks of 64 KiB) decode intact"""
    bad = bad_streams()[rule]
    with pytest.raises(IOError):
        oracle.xerial_decompress(bad)
    data = [corpus(oracle, "text", 100000, seed=14), corpus(oracle, "terasort", 70000, seed=15)]
    good = [oracle.xerial_compress(data[0], 65536), oracle.xerial_compress(data[1], compressor=1)]
    check_alone(capi, [good[0], bad, good[1]], [0, capi.E_CORRUPT, 0])


@pytest.mark.gpu
def test_offset_at_exactly_op_is_valid(capi, oracle):
    s, e = valid_offset_at_op()
    check_good(capi, oracle, [s], [e])


# ------------------------------------------------------------------ chunks above 64 KiB: their stream alone
def oversized_claim_stream(oracle):
    """a three-chunk stream whose chunk varints claim 2^32 - 1 bytes each (a flipped bit in a real stream's varint
    can claim gigabytes): no element sequence of its size decodes to that"""
    s = bytearray(oracle.xerial_compress(corpus(oracle, "text", 3 * 32768, seed=16)))
    ip, out = 16, bytearray(HEADER)
    while ip < len(s):
        clen = int.from_bytes(s[ip:ip + 4], "big")
        raw = bytes(s[ip + 4:ip + 4 + clen])
        v = 0
        while raw[v] & 0x80:
            v += 1
        raw = b"\xff\xff\xff\xff\x0f" + raw[v + 1:]
        out += len(raw).to_bytes(4, "big") + raw
        ip += 4 + clen
    return bytes(out)


@pytest.mark.gpu
def test_oversized_chunk_claim_fails_its_stream_alone(capi, oracle):
    """A chunk varint claiming 2^32 - 1 bytes: the stream is CORRUPT, and the call and its other streams go on (the
    claim used to fail the whole call with UNSUPPORTED).  Plain, packed, device and size calls."""
    data = [corpus(oracle, "text", 90000, seed=17), corpus(oracle, "terasort", 50000, seed=18)]
    good = [oracle.xerial_compress(d) for d in data]
    bad = oversized_claim_stream(oracle)
    with pytest.raises(IOError):
        oracle.xerial_decompress(bad)
    streams = [good[0], bad, good[1]]
    check_alone(capi, streams, [0, capi.E_CORRUPT, 0])
    sizes, st = capi.decompressed_size_batch(capi.CODEC_SNAPPY_XERIAL, streams)
    assert st == [0, capi.E_CORRUPT, 0] and sizes[0] == len(data[0]) and sizes[2] == len(data[1])
    out, st, _ = capi.decompress_batch(capi.CODEC_SNAPPY_XERIAL, streams,
                                       dst_caps=[len(data[0]), 1 << 20, len(data[1])])
    assert st == [0, capi.E_CORRUPT, 0] and out[0] == data[0] and out[2] == data[1]


def unsupported_streams(oracle):
    """name -> a stream with one chunk of more than 64 KiB that the format allows"""
    data = corpus(oracle, "text", 300000, seed=19)
    big_lit = Chunk().lit(rand(65536))
    ones = Chunk()  # 65533 element bytes decoding to 32767: with the 3-byte varint, 65536 compressed bytes
    for _ in range(32765):
        ones.lit(rand(1))
    ones.lit(rand(2))
    return {
        "block_size_128k": (oracle.xerial_compress(data, 131072), data),  # snappy-java's blockSize above 64 KiB
        "literal_65536": (one(big_lit), bytes(big_lit.out)),
        "clen_65536": (one(ones), bytes(ones.out)),
    }


@pytest.mark.gpu
def test_chunks_above_64k_fail_their_stream_alone(capi, oracle):
    data = [corpus(oracle, "text", 90000, seed=20), corpus(oracle, "terasort", 50000, seed=21)]
    good = [oracle.xerial_compress(d) for d in data]
    for name, (s, want) in unsupported_streams(oracle).items():
        if name == "clen_65536":
            assert int.from_bytes(s[16:20], "big") == 65536
        assert oracle.xerial_decompress(s) == want, name
        streams = [good[0], s, good[1]]
        check_alone(capi, streams, [0, capi.E_UNSUPPORTED, 0])
        sizes, st = capi.decompressed_size_batch(capi.CODEC_SNAPPY_XERIAL, streams)
        assert st == [0, capi.E_UNSUPPORTED, 0], name
        out, st, _ = capi.decompress_batch(capi.CODEC_SNAPPY_XERIAL, streams)
        assert st == [0, capi.E_UNSUPPORTED, 0] and out[0] == data[0] and out[2] == data[1], name


@pytest.mark.gpu
@pytest.mark.parametrize("dev", [False, True])
def test_row_sort_with_an_oversized_claim_reports_the_block(capi, oracle, dev):
    """A row sort over [good, bad claim, good] with dst_cap sized for the good blocks returns 0 with the bad block
    CORRUPT, nothing sorted, and no DST_TOO_SMALL asking for the claim"""
    from rows_model import KEY_INT64, run, stream
    rng = np.random.default_rng(22)
    plain = [stream([rng.integers(0, 256, 40, dtype=np.uint8).tobytes() for _ in range(n)]) for n in (900, 700)]
    good = [oracle.xerial_compress(p) for p in plain]
    parts = [good[0], oversized_claim_stream(oracle), good[1]]
    ln = np.array([len(p) for p in parts], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    arena = np.frombuffer(b"".join(parts), np.uint8)
    blocks = (arena, off, ln, None, None, None)
    cap = len(plain[0]) + len(plain[1])
    _, r = run(capi, "decompress_sort_rows", capi.CODEC_SNAPPY_XERIAL, 0, blocks, (KEY_INT64, 0, 8, -1), cap, dev)
    assert list(r["status"]) == [0, capi.E_CORRUPT, 0]
    assert r["n_records"] == 0 and r["total"] == 0
    blocks = (np.frombuffer(good[0] + good[1], np.uint8), np.array([0, len(good[0])], np.uint64),
              np.array([len(g) for g in good], np.uint64), None, None, None)
    _, r = run(capi, "decompress_sort_rows", capi.CODEC_SNAPPY_XERIAL, 0, blocks, (KEY_INT64, 0, 8, -1), cap, dev)
    assert list(r["status"]) == [0, 0] and r["n_records"] == 1600 and r["total"] == cap


# ------------------------------------------------------------------ the rules against the snappy library (CPU)
def raw_chunks_with_verdicts():
    """every hand-assembled raw chunk of this file -> (raw chunk, claimed length, accepted?)"""
    out = []

    def walk(s, ok):
        ip = 16
        while ip < len(s):
            if s[ip:ip + 4] == HEADER[:4]:
                ip += 16
                continue
            clen = int.from_bytes(s[ip:ip + 4], "big")
            out.append((s[ip + 4:ip + 4 + clen], ok))
            ip += 4 + clen
    for ss, _ in (literal_form_streams(), copy_form_streams(), edge_streams()):
        for s in ss:
            walk(s, True)
    walk(valid_offset_at_op()[0], True)
    walk(one(max_expansion_chunk()), True)
    for name, raw in bad_chunks().items():
        out.append((raw, False))
    return out


def test_chunk_verdicts_match_the_snappy_library(oracle):
    """the oracle's raw decoder and pyarrow's snappy (the library snappy-java wraps) accept and reject the same
    chunks, and decode the accepted ones alike"""
    pa = pytest.importorskip("pyarrow")
    codec = pa.Codec("snappy")
    chunks = raw_chunks_with_verdicts()
    assert len(chunks) > 350
    for raw, ok in chunks:
        try:
            want = oracle.snappy_uncompress_raw(raw)
        except IOError:
            want = None
        assert (want is not None) == ok, raw[:16].hex()
        v, claim = 0, 0
        while v < 5 and v < len(raw):
            claim |= (raw[v] & 0x7F) << (7 * v)
            if not raw[v] & 0x80:
                break
            v += 1
        try:
            got = codec.decompress(raw, decompressed_size=min(claim, 1 << 20)).to_pybytes()
            got = got if claim <= 1 << 20 else None
        except (OSError, ValueError, pa.ArrowException):
            got = None
        assert got == want, raw[:16].hex()
