"""GPU parity of the Zstandard decoder on frames from every libzstd strategy, not only levels 1..3: negative levels,
levels 4..22 (split blocks, Repeat_Mode tables, treeless literals, every repeat-offset form), frame options, long
distance matching with offsets of 13 MiB, and frames built from explicit sequences so that each repeat-offset form is
the first repeat code of a 32-sequence batch at warp position 0, 1, 2 and later.  Those reach device code the host
build of the core never runs (the warp's repeat-offset prefix, the per-lane and warp-wide literal copies, the
four-lane Huffman streams).  tests/test_zstd_levels.py proves on the CPU that each class of frame contains those
features; here the C ABI's output must equal the input, which libzstd also decodes to."""
import numpy as np
import pytest

import zstd_ref
from conftest import KINDS, corpus
from test_zstd_levels import long_distance_input, repeat_offset_frames, reset_stream

pytestmark = pytest.mark.gpu

LEVELS = [-5, -1, 4, 6, 9, 13, 16, 19, 22]
SIZES = [0, 1, 5000, 131072, 131073, 1 << 20]


@pytest.fixture(scope="module")
def level_frames(oracle):
    """every level x corpus x size in zstd-jni's streaming shape -> (parts, frames)"""
    parts, frames = [], []
    for li, level in enumerate(LEVELS):
        for kind in KINDS:
            for si, n in enumerate(SIZES):
                d = corpus(oracle, kind, n, seed=li * 10 + si)
                parts.append(d)
                frames.append(zstd_ref.compress_stream(d, level))
    return parts, frames


def decode_all(capi, oracle, frames):
    """decompress_batch with one CRC32C slice per stream (dst_caps from the sizes) -> (outputs, status)"""
    slices = [[(len(f), oracle.crc32c(f))] for f in frames]
    out, st, _ = capi.decompress_batch(capi.CODEC_ZSTD, frames, capi.CHECKSUM_CRC32C, slices)
    return out, st


def test_every_level_in_one_call(capi, oracle, level_frames):
    """all strategies' blocks side by side in one entropy launch; sizes from the size-only pass, then the decode"""
    parts, frames = level_frames
    sizes, st = capi.decompressed_size_batch(capi.CODEC_ZSTD, frames)
    assert st == [0] * len(frames)
    assert sizes == [len(p) for p in parts]
    out, st = decode_all(capi, oracle, frames)
    assert st == [0] * len(frames)
    bad = [i for i, (o, p) in enumerate(zip(out, parts)) if o != p]
    assert not bad, [(LEVELS[i // (len(KINDS) * len(SIZES))], KINDS[i // len(SIZES) % len(KINDS)],
                      SIZES[i % len(SIZES)]) for i in bad[:10]]


def test_frame_options(capi, oracle):
    P = zstd_ref
    text, ts = corpus(oracle, "text", 300000, 3), corpus(oracle, "terasort", 300000, 4)
    big = corpus(oracle, "text", 4 << 20, 5)
    checked = P.compress_stream_params(text, [(P.P_LEVEL, 3), (P.P_CHECKSUM, 1)])
    assert checked[4] & 0x04
    # Content_Checksum is skipped, not verified: a frame whose checksum bytes are wrong still decodes
    wrong_sum = checked[:-4] + bytes(b ^ 0xFF for b in checked[-4:])
    parts = [text, text, big, text]
    frames = [checked, wrong_sum,
              P.compress_stream_params(big, [(P.P_LEVEL, 3), (P.P_WORKERS, 2), (P.P_JOB_SIZE, 1 << 20)]),
              P.compress_stream_params(text, [(P.P_LEVEL, 3), (P.P_LITERAL_MODE, 2)])]
    for strategy in range(1, 10):
        for d in (text, ts):
            parts.append(d)
            frames.append(P.compress_stream_params(d, [(P.P_LEVEL, 3), (P.P_STRATEGY, strategy)]))
    for i, (f, d) in enumerate(zip(frames, parts)):
        if i != 1:
            assert P.decompress(f) == d
    out, st = decode_all(capi, oracle, frames)
    assert st == [0] * len(frames)
    assert [i for i, (o, p) in enumerate(zip(out, parts)) if o != p] == []


def test_long_distance_offsets_into_a_device_buffer(capi, oracle):
    """21 MiB in one frame whose matches reach 13 MiB back (window 2^27): decoded device to device, checked by a
    device CRC32C of the whole output and by host copies of windows around the repeated region"""
    d = long_distance_input(oracle)
    f = zstd_ref.compress_stream_params(d, [(zstd_ref.P_LEVEL, 3), (zstd_ref.P_WINDOW_LOG, 27), (zstd_ref.P_LDM, 1)])
    src = np.frombuffer(f, np.uint8)
    d_src, d_dst = capi.dev_alloc(len(f)), capi.dev_alloc(len(d))
    try:
        capi.dev_memcpy(d_src, src.ctypes.data, len(f), 1)
        r = capi.decompress_dev(capi.CODEC_ZSTD, d_src, [0], [len(f)], d_dst, len(d))
        assert r["status"].tolist() == [0] and r["total"] == len(d) and r["dst_len"].tolist() == [len(d)]
        assert int(capi.checksum_dev(capi.CHECKSUM_CRC32C, d_dst, [0], [len(d)])[0]) == oracle.crc32c(d)
        for at in (0, (12 << 20) - 3000, (13 << 20) - 5000, (13 << 20) + 4097, (21 << 20) - 70000):
            n = min(65536, len(d) - at)
            win = np.zeros(n, np.uint8)
            capi.dev_memcpy(win.ctypes.data, d_dst + at, n, 2)
            assert win.tobytes() == d[at:at + n], at
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)


def test_repeat_offset_forms_at_every_batch_position(capi, oracle):
    frames = repeat_offset_frames()
    out, st = decode_all(capi, oracle, [f for f, _, _ in frames])
    assert st == [0] * len(frames)
    for o, (_, src, _) in zip(out, frames):
        assert o == src


def test_repeat_offsets_reset_at_each_frame(capi, oracle):
    stream, content, _ = reset_stream()
    assert zstd_ref.decompress(stream) == content
    out, st = decode_all(capi, oracle, [stream])
    assert st == [0] and out[0] == content


def test_offset_zero_is_corrupt_between_valid_streams(capi, oracle):
    bad = zstd_ref.offset_zero_frame()
    good, content = zstd_ref.offset_six_frame()
    assert zstd_ref.decompress(good) == content
    text = corpus(oracle, "text", 70000, 9)
    frames = [zstd_ref.compress_stream(text, 19), bad, good]
    out, st, _ = capi.decompress_batch(capi.CODEC_ZSTD, frames, dst_caps=[len(text), 64, len(content)])
    assert st == [0, capi.E_CORRUPT, 0]
    assert out[0] == text and out[2] == content


def test_dictionary_id_is_unsupported_for_that_stream_only(capi, oracle):
    a, b = corpus(oracle, "text", 50000, 8), corpus(oracle, "terasort", 50000, 9)
    fa, fb = zstd_ref.compress_stream(a, 19), zstd_ref.compress_stream(b, 19)
    frames = [fa, zstd_ref.with_dictionary_id(fb), fa]
    out, st, _ = capi.decompress_batch(capi.CODEC_ZSTD, frames, dst_caps=[len(a), len(b), len(a)])
    assert st == [0, capi.E_UNSUPPORTED, 0]
    assert out[0] == a and out[2] == a


def lexsort_records(plain, rb, ko, kl):
    """the blocks back to back, records stably sorted by their unsigned key bytes"""
    recs = np.frombuffer(b"".join(plain), np.uint8).reshape(-1, rb)
    order = np.lexsort([recs[:, ko + j] for j in range(kl - 1, -1, -1)])  # the last key given is the primary one
    return recs[order].tobytes()


def test_sort_path_on_level_19_frames(capi, oracle):
    """decompress + key-sort of TeraSort blocks that libzstd wrote at level 19 (the other sort tests feed only the
    GPU's own encoder)"""
    rng = np.random.default_rng(4)
    plain = [oracle.gen_terasort(i * 100000, int(n)).tobytes() for i, n in enumerate(rng.integers(1, 5000, 24))]
    plain.append(oracle.gen_terasort(7, 10000).tobytes())
    frames = [zstd_ref.compress_stream(p, 19) for p in plain]
    arena = np.frombuffer(b"".join(frames), np.uint8)
    ln = np.array([len(f) for f in frames], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    total = sum(len(p) for p in plain)
    dst = np.zeros(total, np.uint8)
    r = capi.decompress_sort_packed(capi.CODEC_ZSTD, arena, off, ln, dst, 104, 2, 10)
    assert (r["status"] == 0).all() and r["total"] == total and r["n_records"] == total // 104
    assert dst.tobytes() == lexsort_records(plain, 104, 2, 10)
