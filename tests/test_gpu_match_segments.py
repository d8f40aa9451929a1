"""GPU match finding against its CPU specification on inputs built around window boundaries.

The match kernel splits a codec block into contiguous segments of whole 32-position windows, one per warp, and starts
each warp from the hash table the sequential window walk holds at its segment's first window.  Where the segments
begin depends on the block length and on how many warps the launch gives a block, so every input here puts its
feature at every window boundary (or at many distances) rather than at one computed boundary.  Each stream is compared
byte for byte with the oracle's LZ4Block and Snappy window models and with the Zstandard model at levels 1 / 2 / 3
(hash tables of 2^11 / 2^12 / 2^13 slots).
"""
import numpy as np
import pytest

from conftest import corpus
from test_gpu_zstd import zmodel  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

CODECS = ["lz4", "snappy", "zstd1", "zstd2", "zstd3"]


def expected(oracle, zmodel, codec, p, bs):
    if codec == "lz4":
        return oracle.lz4block_compress(p, bs, compressor=1)
    if codec == "snappy":
        return oracle.xerial_compress(p, bs, compressor=1)
    return zmodel(p, bs, {"zstd1": 11, "zstd2": 12, "zstd3": 13}[codec])


def codec_args(capi, codec):
    if codec == "lz4":
        return capi.CODEC_LZ4BLOCK, 0
    if codec == "snappy":
        return capi.CODEC_SNAPPY_XERIAL, 0
    return capi.CODEC_ZSTD, int(codec[-1])


def check_batch(capi, oracle, zmodel, codec, parts, bs=32768):
    cid, level = codec_args(capi, codec)
    comp, _, st = capi.compress_batch(cid, parts, bs, level=level)
    assert st == [0] * len(parts)
    for i, (p, c) in enumerate(zip(parts, comp)):
        assert c == expected(oracle, zmodel, codec, p, bs), "stream %d (%d B) differs from the specification" % (i, len(p))


def rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def copies_across_boundaries(n, seed, length, lead):
    """random bytes; at every window boundary 32j a copy of `length` earlier bytes starting `lead` bytes before it"""
    rng = np.random.default_rng(seed)
    b = rand(n, seed)
    for j in range(4, n // 32):
        at = 32 * j - lead
        if at + length > n:
            break
        src = int(rng.integers(0, at - length)) if at > length else 0
        b[at:at + length] = b[src:src + length].copy()
    return b.tobytes()


def byte_runs_at_boundaries(n, seed, delta, parity):
    """random bytes; a byte run of 40 starting at 32j + delta for every j of the given parity"""
    rng = np.random.default_rng(seed)
    b = rand(n, seed)
    for j in range(1 + parity, n // 32, 2):
        at = 32 * j + delta
        if at + 40 > n:
            break
        b[at:at + 40] = int(rng.integers(0, 256))
    return b.tobytes()


def tokens_far_apart(n, seed, filler):
    """unique 8-byte tokens written twice, 2,000 to 24,000 bytes apart, over zeros or random filler: a token's hash
    slot is last written by its first occurrence, many windows (several segments) before the second"""
    rng = np.random.default_rng(seed)
    b = np.zeros(n, dtype=np.uint8) if filler == "zeros" else rand(n, seed + 1)
    for _ in range(60):
        d = int(rng.integers(2000, 24000))
        a = int(rng.integers(0, n - d - 8))
        t = rng.integers(0, 256, 8, dtype=np.uint8)
        b[a:a + 8] = t
        b[a + d:a + d + 8] = t
    return b.tobytes()


def boundary_corpora(n):
    parts = [copies_across_boundaries(n, s, length, lead)
             for s, (length, lead) in enumerate([(24, 8), (60, 20), (100, 1), (45, 31)])]
    per = (rand(1000, 7).tobytes() * (n // 1000 + 1))[:n]  # one match run through every window of the block
    parts += [per, per[:n - 5] + b"\x01\x02\x03\x04\x05"]
    parts += [byte_runs_at_boundaries(n, 20 + d, d, par) for d in (-3, -1, 0, 1) for par in (0, 1)]
    parts += [tokens_far_apart(n, 40, "zeros"), tokens_far_apart(n, 41, "random")]
    return parts


@pytest.mark.parametrize("codec", CODECS)
def test_matches_across_window_boundaries(capi, oracle, zmodel, codec):
    """match runs crossing every window boundary, full-window runs continuing into the next window and long matches
    measured far past it, byte runs beginning around every boundary, hash slots last written thousands of positions
    earlier"""
    check_batch(capi, oracle, zmodel, codec, boundary_corpora(32768))


@pytest.mark.parametrize("codec", CODECS)
def test_mflimit_on_window_boundaries(capi, oracle, zmodel, codec):
    """n = 32k + 12 puts mflimit = n - 12 on a window start: the last window holds one position"""
    base = bytes(copies_across_boundaries(32768 + 64, 3, 60, 20))
    ks = list(range(1, 160)) + list(range(900, 1023))
    parts = [base[:32 * k + 12 + d] for k in ks for d in (-1, 0, 1)]
    check_batch(capi, oracle, zmodel, codec, parts)


@pytest.mark.parametrize("codec", CODECS)
def test_block_lengths(capi, oracle, zmodel, codec):
    lengths = [13, 64, 300, 4096, 32752, 32768]
    parts = [corpus(oracle, kind, n, seed=i) for i, n in enumerate(lengths) for kind in ("terasort", "text", "runs")]
    bc = boundary_corpora(32768)
    parts += [bc[k][:n] for n in lengths for k in (1, 4, 7, 12)]
    check_batch(capi, oracle, zmodel, codec, parts)


@pytest.mark.parametrize("codec", ["lz4", "zstd1", "zstd2", "zstd3"])
def test_64k_blocks(capi, oracle, zmodel, codec):
    parts = [corpus(oracle, kind, 65536, seed=3) for kind in ("terasort", "text", "runs", "random")]
    parts += boundary_corpora(65536)
    parts += [parts[0][:65536 - 5], corpus(oracle, "terasort", 3 * 65536 + 777, seed=4)]
    check_batch(capi, oracle, zmodel, codec, parts, bs=65536)


@pytest.mark.parametrize("codec", CODECS)
def test_source_blocks_at_every_offset_mod_16(capi, oracle, zmodel, codec):
    """one arena, streams starting at every byte offset mod 16, some shorter than 16 bytes, the last one ending at the
    arena's end"""
    cid, level = codec_args(capi, codec)
    data = corpus(oracle, "terasort", 200000, seed=9) + bytes(boundary_corpora(32768)[1])
    lengths = [13, 20, 31, 300, 4111, 32768 + 4001] * 3
    off, ln, at = [], [], 0
    for i, n in enumerate(lengths):  # stream i starts at i mod 16
        at += (i - at) % 16
        off.append(at)
        ln.append(n)
        at += n
    assert len(data) >= at
    src = np.frombuffer(data[:at], dtype=np.uint8).copy()
    cap = sum(int(capi.compress_bound(cid, 32768, n)) for n in ln)
    dst = np.zeros(cap, dtype=np.uint8)
    r = capi.compress_packed(cid, src, off, ln, dst, 32768, level=level)
    assert not r["status"].any()
    for o, n, do, dl in zip(off, ln, r["dst_off"], r["dst_len"]):
        got = dst[int(do):int(do) + int(dl)].tobytes()
        assert got == expected(oracle, zmodel, codec, src[o:o + n].tobytes(), 32768), (o, n)
