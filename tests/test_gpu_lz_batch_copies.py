"""The match copies of a decode batch (lz_batch.cuh), shared by the LZ4 warp decoder and the Snappy copy kernel: long
matches apart from their source at every length around the lane copy's 16 bytes and the warp copy's 96-byte switch,
overlapping matches short and long, and matches whose source lies inside the output of an earlier match of the same
batch, whose reads are moved onto that match's own source.  Each case is hand-assembled so that it lands inside one
batch, and is checked against the CPU oracle and the byte-by-byte decode of its sequences; a corrupt sequence behind
such matches must leave its stream CORRUPT and the neighbouring streams intact.
"""
import numpy as np
import pytest

import test_gpu_lz4_warp_decode as lz4
import test_gpu_snappy_decode as sn
from conftest import corpus

pytestmark = pytest.mark.gpu

RNG = np.random.default_rng(21)


def rand(n):
    return RNG.integers(0, 256, n, dtype=np.uint8).tobytes()


def lz4_streams(oracle, cases):
    """[(sequences, final literals)] -> (LZ4Block streams of one codec block each, decoded bytes)"""
    streams, expected = [], []
    for seqs, tail in cases:
        payload, data = lz4.block(seqs, tail)
        streams.append(lz4.stream(oracle, [(payload, data)]))
        expected.append(data)
    return streams, expected


def snappy_streams(cases):
    """the same sequences as xerial Snappy streams (copies of up to 64 bytes per element)"""
    streams, expected = [], []
    for seqs, tail in cases:
        ch = sn.Chunk()
        for lit, off, ml in seqs:
            if lit:
                ch.lit(lit)
            while ml > 0:
                n = min(ml, 64) if ml - min(ml, 64) == 0 or ml - min(ml, 64) >= 4 else ml - 4
                ch.copy(off, n, form=2)
                ml -= n
        if tail:
            ch.lit(tail)
        streams.append(sn.one(ch))
        expected.append(bytes(ch.out))
    return streams, expected


def check_both(capi, oracle, cases, snappy=True):
    streams, expected = lz4_streams(oracle, cases)
    lz4.check_good(capi, oracle, streams, expected)
    if snappy:
        streams, expected = snappy_streams(cases)
        sn.check_good(capi, oracle, streams, expected)


def test_long_disjoint_matches_at_every_alignment(capi, oracle):
    """every length 17..100 (up to and past the warp copy's 96-byte switch), destinations at every residue mod 16 and
    offsets ml..ml+15, so the source takes every residue relative to the destination"""
    cases = []
    for ml in range(17, 101):
        seqs = [(rand(128), 1 + ml % 7, 4)]
        for lead in range(16):
            for d in range(16):
                seqs.append((rand(lead), ml + d, ml))
        cases.append((seqs, rand(12)))
    check_both(capi, oracle, cases)


def test_longer_and_overlapping_long_matches(capi, oracle):
    cases = []
    for ml in (101, 127, 128, 129, 200, 255, 300, 1000):
        seqs = [(rand(1100), 1, 4)] + [(rand(lead), ml + lead * 3, ml) for lead in range(16)]
        cases.append((seqs, rand(12)))
    for off in range(1, 17):
        seqs = [(rand(16), off, 4)]
        for ml in list(range(17, 101)) + [128, 200, 300]:
            seqs.append((rand(ml % 3), off, ml))
        cases.append((seqs, rand(12)))
    check_both(capi, oracle, cases)


def test_short_overlapping_matches(capi, oracle):
    """every off < ml <= 16, at several destination residues"""
    cases = []
    for off in range(1, 16):
        seqs = [(rand(20), 1, 4)]
        for ml in range(max(off + 1, 4), 17):
            for lead in range(8):
                seqs.append((rand(lead), off, ml))
        cases.append((seqs, rand(12)))
    check_both(capi, oracle, cases)


def chain(depth, ml, lit=b""):
    """a record of ml random bytes, then `depth` matches each copying the one before it (lit before each)"""
    return [(rand(ml), 1, 4)] + [(lit, ml + len(lit), ml) for _ in range(depth)]


def test_match_on_match_chains(capi, oracle):
    """chains of depth 1..31 inside one batch (sources entirely inside the previous match's output, which is apart
    from its own source), with and without literals between the links, and sources that straddle a literal run, two
    matches, or an overlapping match's output, and overlapping matches whose window lies in an earlier match's output"""
    cases = []
    for depth in range(1, 32):
        for ml, lit in ((4, b""), (8, b""), (18, b""), (35, b""), (20, b"x"), (48, b""), (60, b"")):
            cases.append(([(rand(40), 3, 4)] + chain(depth, ml, lit) + [(rand(3), 7, 9)], rand(12)))
    for k in range(1, 12):
        # a source inside a part of the previous match's output only, shifted by k
        cases.append(([(rand(64), 1, 4), (b"", 40, 30), (b"", 30 - k, 20), (b"", 20 + k, 17)], rand(12)))
        # across a literal run and the match after it
        cases.append(([(rand(64), 1, 4), (b"", 40, 20), (rand(k), 30, 10), (b"", 10 + k + 5, 10 + k)], rand(12)))
        # across two matches
        cases.append(([(rand(64), 1, 4), (b"", 40, 20), (b"", 50, 20), (b"", 20 + k, 20)], rand(12)))
        # inside an overlapping match's output
        cases.append(([(rand(64), 1, 4), (b"", k, 40), (b"", 40 - k, 20), (b"", 20, 17)], rand(12)))
        # an overlapping match whose off-byte window lies inside an earlier match's output, short and long
        cases.append(([(rand(64), 1, 4), (b"", 40, 20), (b"", k, k + 4), (b"", k, 30)], rand(12)))
        cases.append(([(rand(64), 1, 4), (b"", 40, 30), (rand(2), 2 + k, 16)] + chain(3, 20) + [(b"", k, 40)], rand(12)))
        # a chain through a link that is two records back
        cases.append(([(rand(30), 1, 4), (b"", 30, 30), (b"", 60, 30), (b"", 30 + k, 25)], rand(12)))
    check_both(capi, oracle, cases)


def test_terasort_blocks(capi, oracle):
    data = corpus(oracle, "terasort", 600000, seed=12)
    lz4.check_good(capi, oracle, [oracle.lz4block_compress(data)], [data])


@pytest.mark.parametrize("n", [0, 5, 20, 31])
def test_corrupt_sequence_after_long_matches_and_chains(capi, oracle, n):
    """n long matches and chained matches, then a bad offset (past the output) in the same batch: the stream alone
    is CORRUPT, its neighbours decode intact and nothing past them is written"""
    data = corpus(oracle, "terasort", 70000, seed=13)
    good = oracle.lz4block_compress(data)
    for kind in ("long", "chain"):
        seqs = [(rand(60), 1, 4)]
        seqs += [(b"", 60, 35)] * n if kind == "long" else chain(n, 35)
        pre, out = lz4.block(seqs, b"")
        pre = pre[:-1]  # drop the empty final token
        bad_seq = lz4.enc_seq(b"a", 1, 4)[:2] + (len(out) + 2).to_bytes(2, "little") + lz4.enc_last(b"T" * 12)
        bad = lz4.frame(oracle, pre + bad_seq, len(out) + 1 + 12) + lz4.END_MARK
        with pytest.raises(IOError):
            oracle.lz4block_decompress(bad)
        for dev in (False, True):
            outs, st, dst, r = lz4.decode(capi, [good, bad, good], dev)
            assert st == [0, capi.E_CORRUPT, 0], (kind, n, dev)
            assert outs[0] == data and outs[2] == data, (kind, n, dev)
            end = int(r["dst_off"][2]) + int(r["dst_len"][2])
            assert (dst[end:] == 0xA5).all()


def test_block_ending_at_the_end_of_its_allocation(capi, oracle):
    """a stream without an end mark whose last codec block's bytes end exactly where the device allocation ends,
    its last window shorter than 128 bytes, with long matches and chains in that window"""
    for tail_seqs in range(1, 12):
        seqs = [(rand(200), 1, 4)] + [(b"", 100, 35)] * 40 + chain(tail_seqs, 35)
        payload, data = lz4.block(seqs, rand(12))
        s = lz4.frame(oracle, payload, len(data), data)
        assert oracle.lz4block_decompress(s + lz4.END_MARK) == data
        src = np.frombuffer(s, np.uint8)
        cap = len(data)
        dst = np.full(cap, 0xA5, np.uint8)
        d_src, d_dst = capi.dev_alloc(src.size), capi.dev_alloc(cap)
        try:
            capi.dev_memcpy(d_src, src.ctypes.data, src.size, 1)
            r = capi.decompress_dev(capi.CODEC_LZ4BLOCK, d_src, np.zeros(1, np.uint64),
                                    np.array([src.size], np.uint64), d_dst, cap)
            capi.dev_memcpy(dst.ctypes.data, d_dst, cap, 2)
        finally:
            capi.dev_free(d_src)
            capi.dev_free(d_dst)
        assert [int(x) for x in r["status"]] == [0]
        assert dst.tobytes() == data
