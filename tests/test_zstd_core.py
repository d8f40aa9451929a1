"""The Zstandard decoder core (spark-s3-shuffle_b200/csrc/zstd_core.h — the functions the CUDA kernels call) compiled
for the host and pinned on libzstd.so.1: frames produced by the real library at levels 1..3, in the shapes zstd-jni
writes them, plus the encoder model.  Levels -5 to 22, frame options, long distance matching and every repeat-offset
form are pinned in tests/test_zstd_levels.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import zstd_ref
from conftest import KINDS, corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def zc(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("zc") / "libzc.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "native", "zstd_core_host.cpp")])
    L = C.CDLL(out)
    L.zc_decode.restype = C.c_longlong
    L.zc_decode.argtypes = [C.c_char_p, C.c_ulonglong, C.c_char_p, C.c_ulonglong]
    L.zc_size.restype = C.c_longlong
    L.zc_size.argtypes = [C.c_char_p, C.c_ulonglong]
    L.zc_decode_par.restype = C.c_longlong
    L.zc_decode_par.argtypes = [C.c_char_p, C.c_ulonglong, C.c_char_p, C.c_ulonglong, C.c_int]
    single_pass_size = L.zc_size

    def size_both(frame, n):
        """size pass of the single-pass decoder and of the block-parallel decomposition must agree"""
        a = single_pass_size(frame, n)
        b = L.zc_decode_par(frame, n, None, 0, 1)
        # the single-pass decoder also resolves repeat offsets while sizing; the decomposition leaves that to its
        # execute stage, so it may size a frame that only decoding rejects — never the other way round
        assert (a >= 0 and a == b) or (a < 0 and (b < 0 or b >= 0)), (a, b)
        assert not (b < 0 and a >= 0), (a, b)
        return a

    L.zc_size = size_both
    return L


def decode(zc, frame, cap):
    """every frame goes through BOTH statements of the decoder — decode_stream (single pass, zstd_core.h) and
    walk -> entropy -> execute (block-parallel, zstd_par.h); they must agree"""
    out = C.create_string_buffer(max(cap, 1))
    r = zc.zc_decode(frame, len(frame), out, cap)
    out2 = C.create_string_buffer(max(cap, 1))
    r2 = zc.zc_decode_par(frame, len(frame), out2, cap, 0)
    assert (r < 0 and r2 < 0) or r == r2, (r, r2)
    if r >= 0:
        assert out.raw[:r] == out2.raw[:r2]
    return r, out.raw[:max(r, 0)]


@pytest.mark.parametrize("kind", KINDS)
def test_one_shot_frames_levels_1_to_3(zc, oracle, kind):
    for n in (0, 1, 10, 100, 1000, 5000, 40000, 131072, 131073, 400000):
        d = corpus(oracle, kind, n, seed=2)
        for lvl in (1, 2, 3):
            f = zstd_ref.compress(d, lvl)
            r, out = decode(zc, f, n)
            assert r == n and out == d, (kind, n, lvl, r)
            assert zc.zc_size(f, len(f)) == n


@pytest.mark.parametrize("kind", ["terasort", "text", "runs", "ints", "random"])
def test_streaming_frames_as_zstd_jni_writes_them(zc, oracle, kind):
    """no Frame_Content_Size, window descriptor, 32 KiB writes, optional flushes (block boundaries mid-frame)"""
    for n in (0, 5, 32768, 100000, 700000):
        d = corpus(oracle, kind, n, seed=3)
        for lvl, flush in ((1, 0), (3, 0), (1, 2), (3, 5)):
            f = zstd_ref.compress_stream(d, lvl, 32768, flush)
            assert zstd_ref.decompress(f) == d
            r, out = decode(zc, f, n)
            assert r == n and out == d, (kind, n, lvl, flush, r)
            assert zc.zc_size(f, len(f)) == n


def test_concatenated_and_skippable_frames(zc, oracle):
    a, b = corpus(oracle, "text", 70000, 1), corpus(oracle, "terasort", 50000, 2)
    skip = (0x184D2A53).to_bytes(4, "little") + (5).to_bytes(4, "little") + b"hello"
    f = zstd_ref.compress_stream(a, 1) + skip + zstd_ref.compress(b, 3) + zstd_ref.compress(b"", 1)
    r, out = decode(zc, f, len(a) + len(b))
    assert r == len(a) + len(b) and out == a + b
    assert zstd_ref.decompress(f) == a + b


def test_destination_too_small_and_truncation(zc, oracle):
    d = corpus(oracle, "text", 50000, 4)
    f = zstd_ref.compress_stream(d, 3)
    assert decode(zc, f, len(d) - 1)[0] == -3
    assert zc.zc_decode_par(f, len(f), C.create_string_buffer(len(d)), len(d) - 1, 0) == -3  # same class from both
    for cut in (1, 3, 5, 9, len(f) // 2, len(f) - 1):
        assert decode(zc, f[:cut], len(d))[0] < 0


def test_bit_flips_never_crash_and_agree_with_libzstd_when_it_rejects(zc, oracle):
    rng = np.random.default_rng(5)
    d = corpus(oracle, "terasort", 60000, 6)
    f = bytearray(zstd_ref.compress_stream(d, 1))
    accepted_wrong = 0
    for _ in range(300):
        g = bytearray(f)
        i = int(rng.integers(0, len(g)))
        g[i] ^= 1 << int(rng.integers(0, 8))
        r, out = decode(zc, bytes(g), len(d) + 1024)
        try:
            ref = zstd_ref.decompress(bytes(g))
        except IOError:
            ref = None
        if r >= 0 and ref is not None:
            assert out == ref          # both accept: same bytes
        elif r >= 0 and ref is None:
            accepted_wrong += 1        # we accepted what libzstd rejects (no checksum in the frame: tolerated, counted)
    assert accepted_wrong <= 30


def test_mutated_frames_never_crash_and_both_decoders_agree(zc, oracle):
    """truncations, overwritten words, deleted bytes: the single-pass decoder and the block-parallel decomposition give
    the same verdict and the same bytes (decode() asserts it); run under ASAN/UBSAN during development
    (LD_PRELOAD=libasan.so with -fsanitize=address,undefined on tests/native/zstd_core_host.cpp: clean)"""
    rng = np.random.default_rng(9)
    for kind in ("terasort", "text", "runs"):
        d = corpus(oracle, kind, 70000, seed=4)
        for f in (zstd_ref.compress(d, 3), zstd_ref.compress_stream(d, 1, 32768, 2)):
            for it in range(60):
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
                decode(zc, bytes(g), len(d) + 64)
                zc.zc_size(bytes(g), len(g))


def test_encoder_model_frames_are_read_by_libzstd(zc, oracle):
    """zstd_enc_core.h (raw literals + FSE sequences with the block's own or the predefined tables) through the CPU model
    of the GPU encoder: libzstd and our own decoder core both reproduce the input; incompressible blocks fall back to
    Raw_Block."""
    zc.zc_compress_model.restype = C.c_longlong
    zc.zc_compress_model.argtypes = [C.c_char_p, C.c_ulonglong, C.c_uint, C.c_char_p, C.c_ulonglong]
    for kind in KINDS:
        for n in (0, 1, 12, 13, 100, 1000, 32768, 32769, 100000, 300000):
            for bs in (32768, 65536, 1000):
                d = corpus(oracle, kind, n, seed=1)
                cap = n + n // 64 + 9 + 3 * (n // bs + 2)
                buf = C.create_string_buffer(cap)
                c = zc.zc_compress_model(d, n, bs, buf, cap)
                assert 9 <= c <= cap
                f = buf.raw[:c]
                assert zstd_ref.decompress(f) == d
                r, out = decode(zc, f, n)
                assert r == n and out == d
    assert zc.zc_compress_model(b"", 0, 32768, buf, cap) == 9   # frame header + empty last block


def test_block_parallel_decoder_with_shared_table_storage(tmp_path, oracle):
    """the device build of zstd_par.h overlays the Huffman and the sequence tables (B2S_ZSTD_UNION_TABLES): same frames,
    same answers"""
    out = str(tmp_path / "libzcu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DB2S_ZSTD_UNION_TABLES", "-o", out,
                           os.path.join(ROOT, "tests", "native", "zstd_core_host.cpp")])
    L = C.CDLL(out)
    L.zc_decode_par.restype = C.c_longlong
    L.zc_decode_par.argtypes = [C.c_char_p, C.c_ulonglong, C.c_char_p, C.c_ulonglong, C.c_int]
    assert L.zc_workspace_bytes() < 7000
    for kind in ("terasort", "text", "ints", "runs"):
        for n in (0, 777, 40000, 500000):
            d = corpus(oracle, kind, n, seed=11)
            for f in (zstd_ref.compress(d, 3), zstd_ref.compress_stream(d, 1, 32768, 3), zstd_ref.compress_stream(d, 3)):
                buf = C.create_string_buffer(max(n, 1))
                assert L.zc_decode_par(f, len(f), buf, n, 0) == n and buf.raw[:n] == d
                assert L.zc_decode_par(f, len(f), None, 0, 1) == n


def test_committed_libzstd_frames(zc):
    """tests/golden/zstd_vectors.json (made by tests/golden/make_golden_zstd.py from libzstd.so.1): both decoder
    statements reproduce every input, sized and decoded"""
    import json
    import zlib
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "zstd_vectors.json")))
    n = 0
    for name, c in gold["cases"].items():
        for kind, hexframe in c["frames"].items():
            f = bytes.fromhex(hexframe)
            r, out = decode(zc, f, c["input_len"])
            assert r == c["input_len"] and zlib.crc32(out) == c["crc32"], (name, kind, r)
            assert zc.zc_size(f, len(f)) == c["input_len"]
            n += 1
    assert n == 40


def test_block_tables_normalisation_and_description_round_trip(zc):
    """normalize_counts: probabilities sum to 1 << log and every symbol that occurs keeps >= 1; write_ncount: the table
    description is read back by the decoder's fse_read_header (and, inside frames, by libzstd — the test above)"""
    import random
    rng = random.Random(5)
    zc.zc_normalize.argtypes = [C.POINTER(C.c_uint16), C.c_int, C.c_uint, C.c_int, C.POINTER(C.c_int16)]
    zc.zc_ncount_roundtrip.argtypes = [C.POINTER(C.c_int16), C.c_int, C.c_int, C.c_int, C.c_int]
    for nsym, max_sym, log, max_log in ((36, 35, 7, 9), (32, 31, 6, 8), (53, 52, 7, 9), (36, 35, 9, 9), (53, 52, 6, 9)):
        for trial in range(300):
            present = rng.sample(range(nsym), rng.randint(2, min(nsym, 1 << log)))
            cnt = [0] * nsym
            shape = trial % 4
            for s in present:
                cnt[s] = (1 if shape == 0 else rng.randint(1, 8000) if shape == 1 else
                          int(8000 * rng.random() ** 6) + 1 if shape == 2 else rng.choice((1, 1, 1, 5000)))
            while sum(cnt) > 65535:
                cnt = [(c + 1) // 2 if c else 0 for c in cnt]
            arr = (C.c_uint16 * nsym)(*cnt)
            norm = (C.c_int16 * (nsym + 1))()
            zc.zc_normalize(arr, nsym, sum(cnt), log, norm)
            got = list(norm)[:nsym]
            assert sum(got) == 1 << log, (cnt, got)
            assert all((g >= 1) == (c > 0) for g, c in zip(got, cnt)), (cnt, got)
            n = zc.zc_ncount_roundtrip(norm, nsym, log, max_sym, max_log)
            assert 0 < n <= 70, (cnt, got, n)


def test_block_tables_pay_on_the_terasort_shape(zc, oracle):
    """the reason they exist: 14 sequences per 104-byte record, whose codes cost ~12.5 bits with the predefined tables
    and ~5 with the block's own (ratio 0.43 -> 0.30); all three tables of a full block are FSE_Compressed"""
    zc.zc_compress_model.restype = C.c_longlong
    zc.zc_compress_model.argtypes = [C.c_char_p, C.c_ulonglong, C.c_uint, C.c_char_p, C.c_ulonglong]
    d = corpus(oracle, "terasort", 671112, seed=1)
    buf = C.create_string_buffer(len(d))
    c = zc.zc_compress_model(d, len(d), 32768, buf, len(d))
    assert 0 < c < 0.32 * len(d)
    f = buf.raw[:c]
    assert zstd_ref.decompress(f) == d
    # first block: 6-byte frame header, 3-byte block header, raw literals header, literals, nseq, modes
    bh = int.from_bytes(f[6:9], "little")
    assert (bh >> 1) & 3 == 2                      # Compressed_Block
    assert f[9] & 3 == 0                           # Raw_Literals
    fmt = (f[9] >> 2) & 3
    hl = 1 if fmt in (0, 2) else 2 if fmt == 1 else 3
    nlit = int.from_bytes(f[9:9 + hl], "little") >> (3 if hl == 1 else 4)
    q = 9 + hl + nlit
    assert f[q] >= 128                             # >= 128 sequences: two-byte count
    assert f[q + 2] == 0b10101000                  # LL, OF, ML all FSE_Compressed_Mode


def test_encoder_model_fuzz_mixed_streams_decode_with_libzstd(zc, oracle):
    """mixed corpora, tiny alphabets, long periodic runs, odd block sizes, all three match-table sizes: every frame the
    encoder model writes (any mix of own / predefined tables per block, Raw_Block fallback) is decoded by libzstd"""
    import random
    rng = random.Random(11)
    zc.zc_compress_model_hlog.restype = C.c_longlong
    zc.zc_compress_model_hlog.argtypes = [C.c_char_p, C.c_ulonglong, C.c_uint, C.c_char_p, C.c_ulonglong, C.c_int]
    for _ in range(120):
        parts = [corpus(oracle, rng.choice(KINDS), rng.choice([0, 5, 13, 50, 200, 1000, 5000, 40000, 70000]),
                        seed=rng.randint(0, 1000)) for _ in range(rng.randint(1, 3))]
        if rng.random() < 0.4:
            parts.append(bytes(rng.randrange(256) for _ in range(rng.randint(1, 40))) * rng.randint(1, 3000))
        if rng.random() < 0.3:
            a = bytes(rng.randrange(4) for _ in range(rng.randint(20, 3000)))
            parts.append(a + bytes(rng.randrange(256) for _ in range(rng.randint(0, 50))) + a)
        d = b"".join(parts)
        n, bs, hlog = len(d), rng.choice([1000, 4096, 20000, 32768, 65536]), rng.choice([11, 12, 13])
        cap = n + n // 64 + 9 + 3 * (n // bs + 2) + 64
        buf = C.create_string_buffer(cap)
        c = zc.zc_compress_model_hlog(d, n, bs, buf, cap, hlog)
        assert 9 <= c <= cap
        assert zstd_ref.decompress(buf.raw[:c]) == d
