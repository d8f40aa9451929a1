"""The byte movement of the LZ4 / Snappy copy kernel (lz4_copy_kernel + lz_execute_matches), case by case.

Short literals and short non-overlapping matches are read as aligned 8-byte words and re-aligned in registers,
overlapping matches are copied byte by byte, long literals and matches by the whole warp.  The blocks here are
assembled sequence by sequence so that every one of those branches is hit at known offsets, lengths and alignments;
every stream is checked against the oracle's decoder first, then decoded on the GPU and compared with the input.
"""
import numpy as np
import pytest

from conftest import corpus

pytestmark = pytest.mark.gpu

END_MARK = b"LZ4Block" + bytes([0x15]) + bytes(12)
XERIAL_HEADER = bytes.fromhex("82534e41505059000000000100000001")


# ------------------------------------------------------------------ stream assembly
def lz4_sequences(seqs, tail):
    """Raw LZ4 block from [(literals, offset, match length)] and the final literals; -> (payload, decoded bytes)"""
    out, enc = bytearray(), bytearray()
    for lit, off, ml in seqs:
        assert ml >= 4 and 1 <= off <= min(len(out) + len(lit), 65535)
        ll = len(lit)
        enc.append((min(ll, 15) << 4) | min(ml - 4, 15))
        if ll >= 15:
            r = ll - 15
            while r >= 255:
                enc.append(255)
                r -= 255
            enc.append(r)
        enc += lit
        out += lit
        enc += off.to_bytes(2, "little")
        if ml - 4 >= 15:
            r = ml - 4 - 15
            while r >= 255:
                enc.append(255)
                r -= 255
            enc.append(r)
        for _ in range(ml):  # byte by byte: overlapping matches repeat what they have just written
            out.append(out[-off])
    assert len(tail) >= 12  # the last match starts >= 12 bytes before the end, the last 5 bytes are literals
    ll = len(tail)
    enc.append(min(ll, 15) << 4)
    if ll >= 15:
        r = ll - 15
        while r >= 255:
            enc.append(255)
            r -= 255
        enc.append(r)
    enc += tail
    out += tail
    return bytes(enc), bytes(out)


def lz4block(oracle, blocks):
    """LZ4Block stream (lz4-java framing) from [(payload, decoded bytes)], payload None = stored RAW;
    -> (stream, decoded bytes)"""
    s = b""
    for payload, data in blocks:
        level = max(0, (max(len(data), 1) - 1).bit_length() - 10)
        method, body = (0x20, payload) if payload is not None else (0x10, data)
        chk = oracle.xxh32(data) & 0x0FFFFFFF
        s += (b"LZ4Block" + bytes([method | level]) + len(body).to_bytes(4, "little")
              + len(data).to_bytes(4, "little") + chk.to_bytes(4, "little") + body)
    return s + END_MARK, b"".join(data for _, data in blocks)


def snappy_elements(seqs, tail):
    """Raw Snappy block from [(literals, offset, copy length)] and the final literals; -> (raw block, decoded bytes)"""
    out, enc = bytearray(), bytearray()

    def literal(b):
        n = len(b) - 1
        if n < 60:
            enc.append(n << 2)
        elif n < 256:
            enc.extend(bytes([60 << 2, n]))
        else:
            enc.extend(bytes([61 << 2]) + n.to_bytes(2, "little"))
        enc.extend(b)
        out.extend(b)

    for lit, off, ml in seqs:
        if lit:
            literal(lit)
        assert 1 <= off <= len(out)
        left = ml
        while left:
            n = min(left, 64)
            if 4 <= n <= 11 and off < 2048:  # copy with a 1-byte offset
                enc += bytes([1 | ((n - 4) << 2) | ((off >> 8) << 5), off & 0xFF])
            else:  # copy with a 2-byte offset
                enc += bytes([2 | ((n - 1) << 2)]) + off.to_bytes(2, "little")
            for _ in range(n):
                out.append(out[-off])
            left -= n
    if tail:
        literal(tail)
    pre, n = bytearray(), len(out)
    while True:
        if n < 0x80:
            pre.append(n)
            break
        pre.append((n & 0x7F) | 0x80)
        n >>= 7
    return bytes(pre) + bytes(enc), bytes(out)


def xerial(chunks):
    """-> (stream, decoded bytes)"""
    return XERIAL_HEADER + b"".join(len(c).to_bytes(4, "big") + c for c, _ in chunks), b"".join(d for _, d in chunks)


def rand_bytes(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def lz4_raw_prefix(rng, shift):
    """a stored block of 32 + shift bytes: places the next codec block's output `shift` bytes further along"""
    return (None, rand_bytes(rng, 32 + shift))


def check_lz4(capi, oracle, cases):
    """cases: [(stream, decoded bytes)]; the oracle's reader must agree with the input first, then the GPU"""
    streams, want = [s for s, _ in cases], [d for _, d in cases]
    assert [oracle.lz4block_decompress(s) for s in streams] == want
    out, st, _ = capi.decompress_batch(capi.CODEC_LZ4BLOCK, streams)
    assert st == [0] * len(streams)
    assert out == want


# ------------------------------------------------------------------ sequence sets
def offset_length_grid(rng, offs, lens, lit_lens):
    """one sequence per (offset, length): overlapping (off < ml), just not overlapping (off == ml) and disjoint"""
    seqs = [(rand_bytes(rng, 24), 1, 4)]  # a window of >= 24 bytes for the first matches to read from
    k = 0
    for off in offs:
        for ml in lens:
            seqs.append((rand_bytes(rng, lit_lens[k % len(lit_lens)]), off, ml))
            k += 1
    return seqs


@pytest.mark.parametrize("lit_cycle", [(0,), (1, 2, 3), (0, 5, 17, 7)])
def test_lz4_every_offset_1_to_20_against_lengths_4_to_40(capi, oracle, lit_cycle):
    rng = np.random.default_rng(sum(lit_cycle) + 1)
    seqs = offset_length_grid(rng, range(1, 21), range(4, 41), lit_cycle)
    streams = [lz4block(oracle, [lz4_raw_prefix(rng, shift), lz4_sequences(seqs, rand_bytes(rng, 16))])
               for shift in range(0, 16, 5)]
    check_lz4(capi, oracle, streams)


def test_lz4_sources_at_every_alignment(capi, oracle):
    """Short disjoint matches whose sources start at every position mod 32, so they straddle 8- and 32-byte
    boundaries at all eight alignments; the output lands at every alignment mod 16 through the stored prefix block."""
    rng = np.random.default_rng(7)
    streams = []
    for shift in range(16):
        seqs = [(rand_bytes(rng, 64), 1, 4)]
        for ml in range(4, 17):
            for back in range(32):  # the source starts `back` bytes further back each time
                seqs.append((rand_bytes(rng, 1 + (back + ml) % 3), ml + back, ml))
        streams.append(lz4block(oracle, [lz4_raw_prefix(rng, shift), lz4_sequences(seqs, rand_bytes(rng, 13))]))
    check_lz4(capi, oracle, streams)


def test_lz4_match_reads_an_earlier_lane_of_the_same_batch(capi, oracle):
    """Sequence i + 1 copies what sequence i's match just produced (offsets that reach only into that match's
    output), across full 32-sequence batches: the reads must see the stores of the round before."""
    rng = np.random.default_rng(8)
    seqs = [(rand_bytes(rng, 40), 1, 4)]
    for i in range(200):
        ml = 4 + i % 13
        prev_ml = seqs[-1][2]
        seqs.append((b"", prev_ml, ml) if i % 2 else (rand_bytes(rng, i % 4), prev_ml + (i % 4), ml))
    streams = [lz4block(oracle, [lz4_raw_prefix(rng, s), lz4_sequences(seqs, rand_bytes(rng, 12))]) for s in (0, 3)]
    check_lz4(capi, oracle, streams)


def test_lz4_literal_runs_short_and_long(capi, oracle):
    """Literal runs of 0..17 bytes (the per-lane path) and >= 96 bytes (the whole-warp path), at every alignment."""
    rng = np.random.default_rng(9)
    streams = []
    for shift in range(16):
        seqs = [(rand_bytes(rng, 20), 1, 4)]
        for lit in list(range(18)) * 3 + [96, 97, 100, 111, 200, 1000, 4099]:
            seqs.append((rand_bytes(rng, lit), 1 + int(rng.integers(0, 20)), 4 + int(rng.integers(0, 14))))
        streams.append(lz4block(oracle, [lz4_raw_prefix(rng, shift), lz4_sequences(seqs, rand_bytes(rng, 17))]))
    check_lz4(capi, oracle, streams)


def test_lz4_64k_codec_blocks_long_offsets_and_lengths(capi, oracle):
    """64 KiB codec blocks: offsets up to 65,535, short and long matches and literals, and compressed blocks of
    real data."""
    rng = np.random.default_rng(10)
    seqs, size = [], 0
    first = rand_bytes(rng, 20000)
    seqs.append((first, 1, 4))
    size = 20004
    while size < 65536 - 400:
        lit = rand_bytes(rng, int(rng.choice([0, 1, 3, 8, 16, 17, 100])))
        ml = int(rng.choice([4, 7, 8, 9, 15, 16, 17, 33, 96, 300]))
        off = int(rng.integers(1, min(size + len(lit), 65535) + 1))
        if size + len(lit) + ml > 65536 - 200:
            break
        seqs.append((lit, off, ml))
        size += len(lit) + ml
    payload, data = lz4_sequences(seqs, rand_bytes(rng, 65536 - size))
    assert len(data) == 65536 and len(payload) < 65536
    real = corpus(oracle, "terasort", 65536 * 3, seed=4)
    blocks = [(payload, data)] + [(oracle.lz4_compress_block(real[i:i + 65536]), real[i:i + 65536])
                                  for i in range(0, len(real), 65536)]
    streams = [lz4block(oracle, blocks), lz4block(oracle, [lz4_raw_prefix(rng, 9)] + blocks)]
    check_lz4(capi, oracle, streams)


def test_lz4_raw_blocks_between_compressed_ones(capi, oracle):
    rng = np.random.default_rng(11)
    seqs = offset_length_grid(rng, (1, 4, 8, 9, 16), range(4, 20), (0, 2))
    comp = lz4_sequences(seqs, rand_bytes(rng, 12))
    streams = []
    for shift in range(16):
        raw = (None, rand_bytes(rng, 1000 + shift))
        streams.append(lz4block(oracle, [raw, comp, (None, rand_bytes(rng, shift + 1)), comp, raw]))
    check_lz4(capi, oracle, streams)


def test_lz4_corrupt_streams_still_reported_for_the_same_block(capi, oracle):
    """The cases the JVM reader rejects, in a batch between valid streams: each is reported as corrupt, the valid
    streams beside it decode."""
    data = corpus(oracle, "terasort", 100000, seed=30)
    good = oracle.lz4block_compress(data)
    cases = []
    m = bytearray(good); m[0] ^= 1; cases.append(bytes(m))
    m = bytearray(good); m[8] = 0x35; cases.append(bytes(m))
    m = bytearray(good); m[13:17] = (40000).to_bytes(4, "little"); cases.append(bytes(m))
    m = bytearray(good); m[17] ^= 0x01; cases.append(bytes(m))
    m = bytearray(good); m[21 + 100] ^= 0xFF; cases.append(bytes(m))
    cases.append(good[: len(good) // 2])
    cases.append(good[:10])
    m = bytearray(good); m[9:13] = (int.from_bytes(good[9:13], "little") - 1).to_bytes(4, "little"); cases.append(bytes(m))
    m = bytearray(good); m[-1] = 1; cases.append(bytes(m))
    # crafted: a match reaching before the block's first byte, and an offset of 0
    rng = np.random.default_rng(12)
    lit = rand_bytes(rng, 10)
    for bad in ((lit, 11, 4), (lit, 0, 4)):
        enc = bytes([(10 << 4) | 0]) + lit + bad[1].to_bytes(2, "little") + bytes([0xC0]) + rand_bytes(rng, 12)
        cases.append(lz4block(oracle, [(enc, lit + bytes(16))])[0])
    for c in cases:
        with pytest.raises(IOError):
            oracle.lz4block_decompress(c)
    blobs = []
    for c in cases:
        blobs += [good, c]
    blobs.append(good)
    out, st, _ = capi.decompress_batch(capi.CODEC_LZ4BLOCK, blobs, dst_caps=[len(data) + 70000] * len(blobs))
    for i, s in enumerate(st):
        if i % 2:
            assert s == capi.E_CORRUPT, i
        else:
            assert s == 0 and out[i] == data, i


# ------------------------------------------------------------------ Snappy (xerial framing), same kernels
def check_snappy(capi, oracle, cases):
    streams, want = [s for s, _ in cases], [d for _, d in cases]
    assert [oracle.xerial_decompress(s) for s in streams] == want
    out, st, _ = capi.decompress_batch(capi.CODEC_SNAPPY_XERIAL, streams)
    assert st == [0] * len(streams)
    assert out == want


def snappy_prefix(rng, shift):
    d = rand_bytes(rng, 32 + shift)
    return snappy_elements([], d)


@pytest.mark.parametrize("lit_cycle", [(0,), (1, 2, 3), (0, 5, 17, 7)])
def test_snappy_every_offset_1_to_20_against_lengths_1_to_40(capi, oracle, lit_cycle):
    rng = np.random.default_rng(20 + sum(lit_cycle))
    seqs = offset_length_grid(rng, range(1, 21), range(1, 41), lit_cycle)
    streams = [xerial([snappy_prefix(rng, shift), snappy_elements(seqs, rand_bytes(rng, 3))])
               for shift in range(0, 16, 5)]
    check_snappy(capi, oracle, streams)


def test_snappy_sources_and_literals_at_every_alignment(capi, oracle):
    rng = np.random.default_rng(21)
    streams = []
    for shift in range(16):
        seqs = [(rand_bytes(rng, 64), 1, 4)]
        for ml in range(1, 17):
            for back in range(32):
                seqs.append((rand_bytes(rng, (back + ml) % 18), ml + back, ml))
        for lit in [96, 97, 130, 1000]:
            seqs.append((rand_bytes(rng, lit), 1 + int(rng.integers(0, 40)), 1 + int(rng.integers(0, 100))))
        streams.append(xerial([snappy_prefix(rng, shift), snappy_elements(seqs, rand_bytes(rng, 1))]))
    check_snappy(capi, oracle, streams)


def test_snappy_copy_chains_and_real_data(capi, oracle):
    """Copies that read the previous copy's output (whole batches of them), then chunks of real data."""
    rng = np.random.default_rng(22)
    seqs = [(rand_bytes(rng, 40), 1, 4)]
    for i in range(300):
        ml = 1 + i % 16
        prev_ml = seqs[-1][2]
        seqs.append((b"", prev_ml, ml) if i % 3 else (rand_bytes(rng, i % 5), prev_ml + (i % 5), ml))
    crafted = snappy_elements(seqs, b"")
    real = corpus(oracle, "text", 100000, seed=6)
    streams = [xerial([crafted]), (oracle.xerial_compress(real), real), xerial([snappy_prefix(rng, 7), crafted])]
    check_snappy(capi, oracle, streams)
