"""The Zstandard decoder on frames that break one format rule each, and on a seeded corpus of mutated frames.

Each rule frame is built by hand (zstd_ref.hand_frame) or from a libzstd frame with one field changed.  libzstd must
reject it, and the host build of the decoder core (tests/native/zstd_core_host.cpp) too; on the GPU it sits between
two good streams, alone gets B2S_E_CORRUPT, and nothing is written past the last stream.  The mutated corpus (from
frames of levels 1, 3 and 19 and from the repeat-offset frames) is first screened on the CPU under AddressSanitizer and
UBSan, which must be clean and agree with the plain host build; the GPU then decodes it in a few batched calls and
every verdict must be the host core's, with the same bytes where both accept.
"""
import os
import subprocess

import numpy as np
import pytest

import zstd_ref
from conftest import corpus
from test_zstd_levels import repeat_offset_frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAGIC = bytes.fromhex("28b52ffd")


# ------------------------------------------------------------------ the rule frames
def raw_block(data, last=True):
    return ((len(data) << 3) | int(last)).to_bytes(3, "little") + data


def seq_block(nlit, ll_code, modes=0x54, bits=0b1010, of_code=3, ml_code=1):
    """a compressed block: nlit raw literals, then one sequence in RLE mode for all three tables (modes 0x54):
    LL code ll_code, OF code of_code, ML code 1 (4 bytes); bits is the sequence bit-stream (padding marker, then the
    offset's extra bits: 0b1010 -> offset value 10, offset 7)"""
    lits = b"ABCDEFGHIJKLMNOP"[:nlit]
    return bytes([nlit << 3]) + lits + bytes([1, modes, ll_code, of_code, ml_code]) + bits.to_bytes(1, "little")


def treeless_block():
    """treeless Huffman literals (regen 8, 2 bytes of stream), no sequences: needs a previous block's table"""
    regen, comp = 8, 2
    h = 3 | (regen << 4) | (comp << 14)
    return h.to_bytes(3, "little") + b"\x5a\xa5" + b"\x00"


def repeat_mode_block():
    """8 raw literals and one sequence with every table in Repeat_Mode: needs a previous block's tables"""
    return bytes([8 << 3]) + b"ABCDEFGH" + bytes([1, 0xFC, 0b1010])


def with_window(frame, exponent):
    """a hand_frame with Window_Descriptor 2^(10 + exponent)"""
    return frame[:5] + bytes([exponent << 3]) + frame[6:]


def rule_frames(oracle):
    """name -> a stream that breaks that rule"""
    text = corpus(oracle, "text", 200000, seed=30)
    lib19 = zstd_ref.compress_stream(text, 19)
    checked = zstd_ref.compress_stream_params(text[:50000], [(zstd_ref.P_LEVEL, 3), (zstd_ref.P_CHECKSUM, 1)])
    fcs_frame = MAGIC + bytes([0x20, 100]) + raw_block(text[:100])  # single segment, 1-byte content size
    big = bytes(131073)
    out = {
        "reserved_descriptor_bit": zstd_ref.hand_frame([(0, b"abcdef")])[:4] + b"\x08" +
                                   zstd_ref.hand_frame([(0, b"abcdef")])[5:],
        "block_type_3": zstd_ref.hand_frame([(0, b"abcdef"), (3, b"xyz")]),
        "raw_block_above_128k": with_window(zstd_ref.hand_frame([(0, big)]), 8),
        "rle_block_above_128k": with_window(MAGIC + b"\x00\x00" + ((131073 << 3) | (1 << 1) | 1).to_bytes(3, "little")
                                            + b"z", 8),
        "compressed_block_above_128k": with_window(zstd_ref.hand_frame([(2, bytes([0x0C]) + big[:131072])]), 8),
        "block_truncated": lib19[:-1],
        "block_header_truncated": zstd_ref.hand_frame([(0, b"abcdef")])[:8],
        "checksum_truncated_1": checked[:-1],
        "checksum_truncated_3": checked[:-3],
        "treeless_literals_first_block": zstd_ref.hand_frame([(2, treeless_block())]),
        "repeat_mode_first_block": zstd_ref.hand_frame([(2, repeat_mode_block())]),
        "treeless_literals_second_frame": lib19 + zstd_ref.hand_frame([(2, treeless_block())]),
        "repeat_mode_second_frame": lib19 + zstd_ref.hand_frame([(2, repeat_mode_block())]),
        "content_size_above": fcs_frame[:5] + bytes([101]) + fcs_frame[6:],
        "content_size_below": fcs_frame[:5] + bytes([99]) + fcs_frame[6:],
        "offset_before_stream": zstd_ref.hand_frame([(2, seq_block(0, 0))]),
        "offset_into_previous_frame": zstd_ref.hand_frame([(0, b"0123456789abcdef")]) +
                                      zstd_ref.hand_frame([(2, seq_block(0, 0))]),
        "offset_past_frame_output": zstd_ref.hand_frame([(2, seq_block(4, 4))]),
        "sequence_bits_left_over": zstd_ref.hand_frame([(2, seq_block(8, 8, bits=0b10100))]),
        "literal_length_past_regen": zstd_ref.hand_frame([(2, seq_block(8, 9))]),
        "reserved_mode_bits": zstd_ref.hand_frame([(2, seq_block(8, 8, modes=0x55))]),
    }
    return out


def good_streams(oracle):
    data = [corpus(oracle, "text", 90000, seed=31), corpus(oracle, "terasort", 60000, seed=32)]
    return data, [zstd_ref.compress_stream(data[0], 19), zstd_ref.compress_stream(data[1], 1, 32768, 2)]


# ------------------------------------------------------------------ host core and libzstd
@pytest.fixture(scope="module")
def screen(tmp_path_factory):
    """the plain and the sanitized host build of the screening driver -> run(frames, caps) -> (plain, sanitized)"""
    d = tmp_path_factory.mktemp("zscreen")
    src = os.path.join(ROOT, "tests", "native", "zstd_core_screen.cpp")
    plain, asan = str(d / "plain"), str(d / "asan")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", plain, src])
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", asan, src])

    def run(frames, caps):
        path = str(d / "corpus.bin")
        with open(path, "wb") as f:
            for fr, cap in zip(frames, caps):
                f.write(int(cap).to_bytes(8, "little") + len(fr).to_bytes(8, "little") + fr)
        res = []
        for exe in (plain, asan):
            p = subprocess.run([exe, path], capture_output=True, text=True,
                               env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0",
                                        UBSAN_OPTIONS="print_stacktrace=1"))
            assert p.returncode == 0 and not p.stderr, (exe, p.returncode, p.stderr[-3000:])
            res.append([tuple(line.split()) for line in p.stdout.splitlines()])
        assert len(res[0]) == len(frames)
        return res
    return run


def host_verdicts(screen, frames, caps):
    """-> per frame (decoded length or negative error, fnv of the bytes); both statements and both builds agree"""
    plain, asan = screen(frames, caps)
    assert plain == asan
    out = []
    for r, r2, h, h2 in plain:
        r, r2 = int(r), int(r2)
        assert (r < 0 and r2 < 0) or (r == r2 and h == h2), (r, r2)
        out.append((r, h))
    return out


def libzstd_rejects(frame):
    try:
        zstd_ref.decompress(frame)
    except IOError:
        return True
    return False


# The format requires the modes byte's low two bits to be zero; libzstd 1.5.5 does not check them.
LIBZSTD_TOLERATES = {"reserved_mode_bits"}


def test_rule_frames_are_rejected_by_libzstd_and_the_host_core(oracle, screen):
    """every rule frame is CORRUPT for both statements of the host core and rejected by libzstd; the hand-built
    compressed block they start from is valid as it stands"""
    rules = rule_frames(oracle)
    v = host_verdicts(screen, list(rules.values()), [300000] * len(rules))
    for (name, f), (r, _) in zip(rules.items(), v):
        assert libzstd_rejects(f) != (name in LIBZSTD_TOLERATES), name
        assert r == -1, (name, r)  # kErrCorrupt
    ok = zstd_ref.hand_frame([(2, seq_block(8, 8))])
    assert zstd_ref.decompress(ok) == b"ABCDEFGH" + b"BCDE"
    assert host_verdicts(screen, [ok], [64])[0][0] == 12


# Room for any mutated frame's output: none of the source frames has more than five blocks of at most 128 KiB, so a
# host verdict of "destination too small" (-3) never stands in for a decode the GPU, which sizes its own arena, makes.
SCREEN_CAP = 1 << 20


def mutated_corpus(oracle):
    """a fixed-seed corpus of truncated, overwritten, 0xFF-patched and shortened frames -> (frames, caps)"""
    rng = np.random.default_rng(33)
    frames, caps = [], []
    sources = []
    for kind in ("terasort", "text", "runs"):
        d = corpus(oracle, kind, 70000, seed=34)
        sources += [(zstd_ref.compress(d, 3), d), (zstd_ref.compress_stream(d, 1, 32768, 2), d),
                    (zstd_ref.compress_stream(d, 19), d)]
    sources += [(f, src) for f, src, _ in repeat_offset_frames()]
    for si, (f, d) in enumerate(sources):
        for it in range(36):
            g = bytearray(f)
            mode = it % 4
            if mode == 0:
                g = g[: int(rng.integers(0, len(g)))]
            elif mode == 1:
                i = int(rng.integers(0, len(g)))
                g[i:i + 4] = bytes(rng.integers(0, 256, 4, dtype=np.uint8))
            elif mode == 2:
                g[int(rng.integers(0, len(g)))] = 0xFF
            else:
                i = int(rng.integers(0, len(g) - 8))
                del g[i:i + int(rng.integers(1, 8))]
            frames.append(bytes(g))
            caps.append(SCREEN_CAP)
    return frames, caps


def test_mutated_corpus_is_clean_under_sanitizers(oracle, screen):
    """every mutated frame through both statements of the host core, plain and under ASan/UBSan: no report, the same
    verdicts and bytes; some are accepted and many rejected, so the corpus exercises both"""
    frames, caps = mutated_corpus(oracle)
    assert len(frames) >= 300
    v = host_verdicts(screen, frames, caps)
    assert all(r != -3 for r, _ in v)
    ok = sum(r >= 0 for r, _ in v)
    assert 10 <= ok <= len(frames) - 100, ok


# ------------------------------------------------------------------ the GPU
def gpu_decode(capi, streams, caps):
    """decompress_packed into a 0xA5-filled arena of the caps' sum -> (outputs or None, status, arena, result)"""
    ln = np.array([len(s) for s in streams], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    src = np.frombuffer(b"".join(streams) + b"\0", np.uint8)
    cap = int(sum(caps)) + 4096
    dst = np.full(cap, 0xA5, np.uint8)
    r = capi.decompress_packed(capi.CODEC_ZSTD, src, off, ln, dst)
    outs = [dst[int(o):int(o) + int(n)].tobytes() if s == 0 else None
            for o, n, s in zip(r["dst_off"], r["dst_len"], r["status"])]
    return outs, [int(s) for s in r["status"]], dst, r


RULES = ["reserved_descriptor_bit", "block_type_3", "raw_block_above_128k", "rle_block_above_128k",
         "compressed_block_above_128k", "block_truncated", "block_header_truncated", "checksum_truncated_1",
         "checksum_truncated_3", "treeless_literals_first_block", "repeat_mode_first_block",
         "treeless_literals_second_frame", "repeat_mode_second_frame", "content_size_above", "content_size_below",
         "offset_before_stream", "offset_into_previous_frame", "offset_past_frame_output", "sequence_bits_left_over",
         "literal_length_past_regen", "reserved_mode_bits"]


def test_rule_list_is_complete(oracle):
    assert sorted(RULES) == sorted(rule_frames(oracle))


@pytest.mark.gpu
@pytest.mark.parametrize("rule", RULES)
def test_one_bad_frame_among_good_ones(capi, oracle, rule):
    """[good, bad, good]: the bad stream alone is CORRUPT, as the host core says; the good ones decode intact and
    nothing is written past them.  Both neighbours are tried on the left, so an offset reaching before the bad
    stream's first byte lands in real output."""
    bad = rule_frames(oracle)[rule]
    assert libzstd_rejects(bad) != (rule in LIBZSTD_TOLERATES)
    data, good = good_streams(oracle)
    for a, b in ((0, 1), (1, 0)):
        outs, st, dst, r = gpu_decode(capi, [good[a], bad, good[b]], [len(data[a]), 300000, len(data[b])])
        assert st == [0, capi.E_CORRUPT, 0], (rule, st)
        assert outs[0] == data[a] and outs[2] == data[b]
        end = int(r["dst_off"][2]) + int(r["dst_len"][2])
        assert (dst[end:] == 0xA5).all()


@pytest.mark.gpu
def test_mutated_corpus_verdicts_match_the_host_core(capi, oracle, screen):
    """the screened corpus in batched calls of 40 frames, each frame between good streams: every verdict is the
    host core's (accepted or not), outputs match where both accept, the good streams are intact, nothing is written
    past the last stream"""
    frames, caps = mutated_corpus(oracle)
    v = host_verdicts(screen, frames, caps)
    data, good = good_streams(oracle)
    for b0 in range(0, len(frames), 40):
        streams, stream_caps, idx = [good[0]], [len(data[0])], []
        for k in range(b0, min(b0 + 40, len(frames))):
            idx.append(len(streams))
            streams += [frames[k], good[k % 2]]
            stream_caps += [caps[k], len(data[k % 2])]
        outs, st, dst, r = gpu_decode(capi, streams, stream_caps)
        for j, k in zip(idx, range(b0, b0 + len(idx))):
            hr, _ = v[k]
            assert st[j] == min(hr, 0), (k, st[j], hr)  # kErrCorrupt -1 / kErrUnsupported -4 are the B2S codes
            if hr >= 0:
                assert len(outs[j]) == hr and outs[j] == host_bytes(frames[k], caps[k]), k
            assert outs[j + 1] == data[k % 2], k
        assert outs[0] == data[0]
        end = int(r["dst_off"][-1]) + int(r["dst_len"][-1])
        assert (dst[end:] == 0xA5).all()


def host_bytes(frame, cap):
    """the host core's decoded bytes (single-pass statement, through ctypes)"""
    import ctypes as C
    lib = _host_lib()
    out = C.create_string_buffer(max(cap, 1))
    r = lib.zc_decode(frame, len(frame), out, cap)
    return out.raw[:max(r, 0)]


_LIB = []


def _host_lib():
    import ctypes as C
    import tempfile
    if not _LIB:
        out = os.path.join(tempfile.mkdtemp(prefix="zc"), "libzc.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out,
                               os.path.join(ROOT, "tests", "native", "zstd_core_host.cpp")])
        L = C.CDLL(out)
        L.zc_decode.restype = C.c_longlong
        L.zc_decode.argtypes = [C.c_char_p, C.c_ulonglong, C.c_char_p, C.c_ulonglong]
        _LIB.append(L)
    return _LIB[0]
