"""The Zstandard decoder core (zstd_core.h, zstd_par.h) compiled for the host, on frames from every libzstd strategy:
negative levels (raw literals inside compressed blocks), levels 4..22 (lazy to btultra2; from btopt up: split blocks,
Repeat_Mode tables, treeless literals, all six repeat-offset forms), long distance matching with a 128 MiB window, frame options, and
frames built from explicit sequences so that every repeat-offset form lands where the GPU's 32-sequence batches treat
it differently.  Coverage probes (zc_frame_sequences, zc_frame_blocks) prove that each class of frame really contains
what it is meant to exercise; tests/test_gpu_zstd_levels.py sends the same classes through the CUDA kernels."""
import ctypes as C
import os
import subprocess

import pytest

import zstd_ref
from conftest import KINDS, corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = [-5, -1, 4, 6, 9, 13, 16, 19, 22]


@pytest.fixture(scope="module")
def zc(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("zc") / "libzc.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "native", "zstd_core_host.cpp")])
    L = C.CDLL(out)
    L.zc_decode.restype = C.c_longlong
    L.zc_decode.argtypes = [C.c_char_p, C.c_ulonglong, C.c_char_p, C.c_ulonglong]
    L.zc_decode_par.restype = C.c_longlong
    L.zc_decode_par.argtypes = [C.c_char_p, C.c_ulonglong, C.c_char_p, C.c_ulonglong, C.c_int]
    L.zc_frame_sequences.restype = C.c_longlong
    L.zc_frame_sequences.argtypes = [C.c_char_p, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulonglong]
    L.zc_frame_blocks.restype = C.c_longlong
    L.zc_frame_blocks.argtypes = [C.c_char_p, C.c_ulonglong, C.c_void_p, C.c_ulonglong]
    return L


def decode(zc, frame, cap):
    """single-pass decode_stream and the walk -> entropy -> execute decomposition; both must agree"""
    out = C.create_string_buffer(max(cap, 1))
    r = zc.zc_decode(frame, len(frame), out, cap)
    out2 = C.create_string_buffer(max(cap, 1))
    r2 = zc.zc_decode_par(frame, len(frame), out2, cap, 0)
    assert (r < 0 and r2 < 0) or r == r2, (r, r2)
    if r >= 0:
        assert out.raw[:r] == out2.raw[:r2]
        assert zc.zc_decode_par(frame, len(frame), None, 0, 1) == r  # the size pass
    return r, out.raw[:max(r, 0)]


def check_decodes(zc, frame, data):
    assert zstd_ref.decompress(frame) == data
    r, out = decode(zc, frame, len(data))
    assert r == len(data) and out == data


def sequences(zc, frame):
    """[(literal length, match length, offset value)] of every sequence of the frame"""
    n = zc.zc_frame_sequences(frame, len(frame), None, None, None, 0)
    assert n >= 0
    a, b, c = ((C.c_uint * max(n, 1))() for _ in range(3))
    assert zc.zc_frame_sequences(frame, len(frame), a, b, c, n) == n
    return list(zip(a[:n], b[:n], c[:n]))


def blocks(zc, frame):
    """[(type, literals type, streams, modes byte, Huffman weights FSE-compressed, sequence count)] per block"""
    n = zc.zc_frame_blocks(frame, len(frame), None, 0)
    assert n >= 0
    o = (C.c_int * (6 * max(n, 1)))()
    assert zc.zc_frame_blocks(frame, len(frame), o, n) == n
    return [tuple(o[6 * i:6 * i + 6]) for i in range(n)]


def repeat_modes(bl):
    """which of LL / OF / ML some compressed block of bl takes in Repeat_Mode"""
    return {k for b in bl if b[0] == 2 and b[5] for k in range(3) if (b[3] >> (6 - 2 * k)) & 3 == 3}


def rep_forms(seqs):
    return {(v, l == 0) for l, _, v in seqs if v <= 3}


ALL_FORMS = set(zstd_ref.REP_FORMS)


@pytest.mark.parametrize("level", LEVELS)
def test_every_level_decodes_on_the_host(zc, oracle, level):
    for kind in KINDS:
        for n in (0, 1, 5000, 131072, 131073, 400000):
            d = corpus(oracle, kind, n, seed=n % 7)
            check_decodes(zc, zstd_ref.compress_stream(d, level), d)


def test_negative_levels_store_raw_literals_in_compressed_blocks(zc, oracle):
    for level in (-5, -1):
        bl, seqs = [], []
        for kind in ("text", "terasort", "ints"):
            d = corpus(oracle, kind, 300000, seed=1)
            f = zstd_ref.compress_stream(d, level)
            check_decodes(zc, f, d)
            bl += blocks(zc, f)
            seqs += sequences(zc, f)
        assert any(b[0] == 2 and b[1] == 0 and b[5] > 0 for b in bl), level
        assert all(b[1] == 0 for b in bl if b[0] == 2), level  # no Huffman literals at all
        assert seqs


def test_high_levels_write_every_repeat_form_and_table_mode(zc, oracle):
    """levels 19 and 22 over every corpus at 1 MiB: all six repeat-offset forms, treeless literals, Repeat_Mode for each
    of the three sequence tables, 1- and 4-stream Huffman literals"""
    bl, forms = [], set()
    for level in (19, 22):
        for kind in KINDS:
            d = corpus(oracle, kind, 1 << 20, seed=7)
            f = zstd_ref.compress_stream(d, level)
            check_decodes(zc, f, d)
            bl += blocks(zc, f)
            forms |= rep_forms(sequences(zc, f))
    assert forms == ALL_FORMS
    assert any(b[0] == 2 and b[1] == 3 for b in bl)                        # treeless literals
    assert repeat_modes(bl) == {0, 1, 2}
    assert {b[2] for b in bl if b[0] == 2 and b[1] >= 2} == {1, 4}          # 1- and 4-stream Huffman
    assert {b[4] for b in bl if b[0] == 2 and b[1] == 2} >= {1}             # FSE-compressed Huffman weights


def long_distance_input(oracle):
    """12 MiB random, 1 MiB text, then the first 8 MiB again: only a window of 2^27 and long distance matching find
    the repeat, 13 MiB back"""
    head = corpus(oracle, "random", 12 << 20, 1) + corpus(oracle, "text", 1 << 20, 2)
    return head + head[:8 << 20]


def test_long_distance_matching_frame(zc, oracle):
    d = long_distance_input(oracle)
    f = zstd_ref.compress_stream_params(d, [(zstd_ref.P_LEVEL, 3), (zstd_ref.P_WINDOW_LOG, 27), (zstd_ref.P_LDM, 1)])
    assert len(f) < len(d) * 0.65
    check_decodes(zc, f, d)
    assert max(v for _, _, v in sequences(zc, f)) > 1 << 23


def test_frame_options(zc, oracle):
    text, ts = corpus(oracle, "text", 300000, 3), corpus(oracle, "terasort", 300000, 4)
    P = zstd_ref
    f = P.compress_stream_params(text, [(P.P_LEVEL, 3), (P.P_CHECKSUM, 1)])
    assert f[4] & 0x04                                                      # Content_Checksum_Flag
    check_decodes(zc, f, text)
    big = corpus(oracle, "text", 4 << 20, 5)
    check_decodes(zc, P.compress_stream_params(big, [(P.P_LEVEL, 3), (P.P_WORKERS, 2), (P.P_JOB_SIZE, 1 << 20)]), big)
    f = P.compress_stream_params(text, [(P.P_LEVEL, 3), (P.P_LITERAL_MODE, 2)])
    assert {b[1] for b in blocks(zc, f) if b[0] == 2} == {0}
    check_decodes(zc, f, text)
    for strategy in range(1, 10):
        for d in (text, ts):
            check_decodes(zc, P.compress_stream_params(d, [(P.P_LEVEL, 3), (P.P_STRATEGY, strategy)]), d)


def repeat_offset_frames():
    """-> [(frame, content, expected offset values)]: the sequence plan with Huffman and with raw literals"""
    bl, expect = zstd_ref.plan_sequences(zstd_ref.repeat_offset_tokens(1), 1)
    src = zstd_ref.execute_sequences(bl, 1)
    return [(zstd_ref.compress_sequences(src, bl, 3, raw), src, expect) for raw in (False, True)]


def batch_coverage(bl, seqs):
    """(form, warp position of the batch's first repeat code: 0, 1, 2 or 3 for later) for every 32-sequence batch;
    whether a block has repeat codes as its sequences 31 and 32; the forms that open a block after a block that ended
    in a new offset"""
    found, at_31_32, block_start = set(), False, set()
    i = 0
    prev_last = None
    for b in bl:
        if b[0] != 2:
            continue
        s = seqs[i:i + b[5]]
        for j0 in range(0, len(s), 32):
            reps = [j for j in range(j0, min(j0 + 32, len(s))) if s[j][2] <= 3]
            if reps:
                j = reps[0]
                found.add(((s[j][2], s[j][0] == 0), min(j - j0, 3)))
        if len(s) > 32 and s[31][2] <= 3 and s[32][2] <= 3:
            at_31_32 = True
        if s and prev_last is not None and prev_last > 3 and s[0][2] <= 3:
            block_start.add((s[0][2], s[0][0] == 0))
        if s:
            prev_last = s[-1][2]
        i += b[5]
    assert i == len(seqs)
    return found, at_31_32, block_start


def test_repeat_offset_forms_at_every_batch_position(zc):
    frames = repeat_offset_frames()
    for f, src, expect in frames:
        check_decodes(zc, f, src)
        seqs = sequences(zc, f)
        assert [v for _, _, v in seqs] == expect      # libzstd wrote exactly the planned repeat codes
        bl = blocks(zc, f)
        assert all(b[0] == 2 for b in bl) and len(bl) > 40
        found, at_31_32, block_start = batch_coverage(bl, seqs)
        assert found == {(form, p) for form in ALL_FORMS for p in range(4)}
        assert at_31_32
        assert block_start == ALL_FORMS
        assert any(ll > 32 for ll, _, _ in seqs) and any(v > 3 and v - 3 < ml for _, ml, v in seqs)
    assert {b[1] for b in blocks(zc, frames[0][0])} >= {2, 3}               # Huffman literals, then raw ones
    assert {b[1] for b in blocks(zc, frames[1][0])} == {0}


def reset_stream():
    """two frames back to back; the second one's first sequence is offset 4 written as repeat code 2 (the initial
    repeat offsets are 1, 4, 8; the first frame ends with three other offsets) -> (stream, content, second frame)"""
    (f1, src1, _), _ = repeat_offset_frames()
    plan = [([(8, 4, 12), (3, 20, 9)], 5)]
    src2 = zstd_ref.execute_sequences(plan, 2)
    f2 = zstd_ref.compress_sequences(src2, plan, 3)
    return f1 + f2, src1 + src2, f2


def test_repeat_offsets_reset_at_each_frame(zc):
    stream, content, f2 = reset_stream()
    assert sequences(zc, f2)[0] == (8, 12, 2)
    check_decodes(zc, stream, content)


def libzstd_on_offset_zero(frame):
    """libzstd 1.5.5 notes that offset 0 means corrupt input but substitutes offset 1 and goes on; a libzstd that
    rejects the frame is fine too.  -> libzstd's bytes, or None when it rejects"""
    try:
        return zstd_ref.decompress(frame)
    except IOError:
        return None


def test_offset_zero_is_corrupt_and_rep0_minus_one_decodes(zc):
    """repeat code 3 with literal length 0 while rep0 is 1 resolves to offset 0, which no valid frame contains: the
    decoder rejects the frame instead of guessing an offset"""
    bad = zstd_ref.offset_zero_frame()
    assert libzstd_on_offset_zero(bad) in (None, b"0123456789abcdef" + b"f" * 4)
    assert decode(zc, bad, 64)[0] == -1                                     # kErrCorrupt
    assert sequences(zc, bad) == [(0, 4, 3)]
    good, content = zstd_ref.offset_six_frame()
    check_decodes(zc, good, content)
    assert sequences(zc, good) == [(8, 4, 10), (0, 4, 3)]


def test_dictionary_id_is_unsupported(zc, oracle):
    d = corpus(oracle, "text", 50000, 8)
    f = zstd_ref.with_dictionary_id(zstd_ref.compress_stream(d, 3))
    assert decode(zc, f, len(d))[0] == -4                                   # kErrUnsupported, from both statements
    assert zc.zc_decode_par(f, len(f), None, 0, 1) == -4
