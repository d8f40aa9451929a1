"""The frame window calls (b2s_decompress_window_frame_rows_keys_*) without a GPU: their constants and prototypes match
the header and the host mirror declares the read, every argument rule of the frames is B2S_E_ARG before the device is
looked at, the aggregate and offset calls still reject the new frames, and a valid call fails loudly with B2S_E_CUDA —
there is no CPU fallback — writing nothing but zeros to its outputs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from test_window_rows_abi import _has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
c_ = pkg.capi
ROWS, RANGE = c_.WINDOW_FRAME_ROWS, c_.WINDOW_FRAME_RANGE
UP, UF = c_.WINDOW_UNBOUNDED_PRECEDING, c_.WINDOW_UNBOUNDED_FOLLOWING
I64, F64, BYTES = c_.WINDOW_VAL_INT64, c_.WINDOW_VAL_FLOAT64, c_.WINDOW_VAL_BYTES


def test_window_frame_constants_and_prototypes_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    for name, v in (("B2S_WINDOW_FRAME_ROWS", ROWS), ("B2S_WINDOW_FRAME_RANGE", RANGE)):
        assert int(re.search(r"#define %s (\d+)\n" % name, hdr).group(1)) == v
    assert re.search(r"#define B2S_WINDOW_UNBOUNDED_PRECEDING INT64_MIN\n", hdr) and UP == -2**63
    assert re.search(r"#define B2S_WINDOW_UNBOUNDED_FOLLOWING INT64_MAX\n", hdr) and UF == 2**63 - 1
    assert ROWS == c_.WINDOW_FRAME_RANGE_RUNNING + 1
    protos = dict((p[0], p[2]) for p in c_.PROTOTYPES)
    for name, extra in (("b2s_decompress_window_frame_rows_keys_packed", 0),
                        ("b2s_decompress_window_frame_rows_keys_dev", 1)):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(protos[name]) == decl.count(",") + 1 == 35 + extra
        assert ("const uint64_t* fn_default, const int64_t* frame_lower, const int64_t* frame_upper"
                in " ".join(decl.split()))


def test_host_mirror_declares_the_window_frame_read():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle_host.h")).read()
    decl = re.search(r"int b2sh_reader_read_window_frame_rows\((.*?)\);", hdr, re.S).group(1)
    protos = dict((p[0], p[2]) for p in pkg.host.PROTOTYPES)
    assert len(protos["b2sh_reader_read_window_frame_rows"]) == decl.count(",") + 1 == 24
    assert hasattr(pkg.host.S3ShuffleReader, "readWindowFrameRows")


# fields: 0 a long partition key, 1 a long order key, 2 a long value, 3 a DECIMAL_WIDE value, 4 a double value,
# 5 a string, 6 an int order key, 7 a byte order key, 8 a compact decimal, 9 a double order key
KINDS = [0, 0, 0, 2, 0, 1, 0, 0, 0, 0]
NF = len(KINDS)


def _slot(f):
    return 8 + 8 * f


KEYS = [(2, _slot(0), 8, 0), (2, _slot(1), 8, 1)]


def _fr(fn, frame, lo, hi, arg=0, vt=I64, f=2, null=2, flags=0):
    return (fn, arg, frame, vt, _slot(f), null, flags, 0, lo, hi)


def _call(fns, keys=KEYS, npk=1):
    src, dst = np.zeros(64, np.uint8), np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    return c_.decompress_window_frame_rows_keys_packed(c_.CODEC_LZ4BLOCK, src, off, ln, dst, keys, npk, NF, KINDS,
                                                       fns)


def _order(kt, f, flags=0, width=8):
    return [KEYS[0], (kt | flags, _slot(f), width, f)]


BAD = [
    ("bounds on frame 2", [_fr(c_.WINDOW_SUM, 2, -1, 0)], KEYS),
    ("a lower bound on frame 1", [_fr(c_.WINDOW_MAX, 1, 0, 3)], KEYS),
    ("a bound on a ranking function", [(c_.WINDOW_RANK, 0, 0, 0, 0, -1, 0, 0, 0, 1)], KEYS),
    ("LAG with frame 4", [_fr(c_.WINDOW_LAG, ROWS, -1, 0, arg=1)], KEYS),
    ("LEAD with frame 5", [_fr(c_.WINDOW_LEAD, RANGE, 0, 0, arg=1)], KEYS),
    ("RANK with frame 4", [(c_.WINDOW_RANK, 0, ROWS, 0, 0, -1, 0, 0, 0, 0)], KEYS),
    ("frame 6", [_fr(c_.WINDOW_SUM, 6, -1, 0)], KEYS),
    ("lower above upper", [_fr(c_.WINDOW_SUM, ROWS, 2, 1)], KEYS),
    ("UNBOUNDED FOLLOWING as the lower bound", [_fr(c_.WINDOW_SUM, ROWS, UF, UF)], KEYS),
    ("UNBOUNDED PRECEDING as the upper bound", [_fr(c_.WINDOW_COUNT, RANGE, UP, UP)], KEYS),
    ("a ROWS offset below the int range", [_fr(c_.WINDOW_SUM, ROWS, -2**31 - 1, 0)], KEYS),
    ("a ROWS offset above the int range", [_fr(c_.WINDOW_MIN, ROWS, 0, 2**31)], KEYS),
    ("a RANGE offset with two order columns", [_fr(c_.WINDOW_SUM, RANGE, -1, 0)], KEYS + [(1, _slot(6), 4, 6)]),
    ("a RANGE offset over a double column", [_fr(c_.WINDOW_SUM, RANGE, -1, 0)], _order(8, 9)),
    ("a RANGE offset over a string column", [_fr(c_.WINDOW_SUM, RANGE, 0, 2)], _order(3, 5)),
    ("a RANGE offset past an int", [_fr(c_.WINDOW_SUM, RANGE, -2**31 - 1, 0)], _order(1, 6, 0, 4)),
    ("a RANGE offset past a byte", [_fr(c_.WINDOW_SUM, RANGE, 0, 128)], _order(6, 7, 0, 1)),
    ("a descending RANGE offset at a byte's minimum", [_fr(c_.WINDOW_SUM, RANGE, -128, 0)], _order(6, 7, 1 << 8, 1)),
    ("a descending RANGE offset at a short's minimum", [_fr(c_.WINDOW_SUM, RANGE, -32768, 0)], _order(5, 6, 1 << 8, 2)),
    ("a RANGE offset past a short", [_fr(c_.WINDOW_SUM, RANGE, 0, 32768)], _order(5, 6, 0, 2)),
    ("a bad frame after good ones", [_fr(c_.WINDOW_SUM, ROWS, -1, 1), _fr(c_.WINDOW_FIRST, RANGE, 0, UF),
                                     _fr(c_.WINDOW_AVG, ROWS, 1, 0)], KEYS),
]


@pytest.mark.parametrize("why,fns,keys", BAD, ids=[b[0] for b in BAD])
def test_bad_frames_are_argument_errors_before_the_device(why, fns, keys):
    with pytest.raises(c_.B2SError) as e:
        _call(fns, keys)
    assert e.value.code == c_.E_ARG, why


def test_argument_error_writes_zeros_and_a_message():
    L = c_.load()
    outs = [C.c_uint64(7) for _ in range(3)]
    dst = np.zeros(64, np.uint8)
    a = c_._window_frame_arrays(KEYS, 1, NF, KINDS, [_fr(c_.WINDOW_SUM, ROWS, 3, -3)])
    rc = L.b2s_decompress_window_frame_rows_keys_packed(0, 0, 0, None, None, None, None, None, None,
                                                        *map(c_._arg, a), dst.ctypes.data, dst.size,
                                                        *map(C.byref, outs), None, None)
    assert rc == c_.E_ARG and [o.value for o in outs] == [0, 0, 0] and not dst.any()
    assert b"lower bound" in L.b2s_last_error()
    for at in (17, 18):  # no frame_lower, no frame_upper
        b = list(c_._window_frame_arrays(KEYS, 1, NF, KINDS, [_fr(c_.WINDOW_SUM, ROWS, -1, 0)]))
        b[at] = None
        outs = [C.c_uint64(7) for _ in range(3)]
        rc = L.b2s_decompress_window_frame_rows_keys_packed(0, 0, 0, None, None, None, None, None, None,
                                                            *map(c_._arg, b), dst.ctypes.data, dst.size,
                                                            *map(C.byref, outs), None, None)
        assert rc == c_.E_ARG and [o.value for o in outs] == [0, 0, 0]


def test_the_aggregate_and_offset_calls_still_reject_the_new_frames():
    src, dst = np.zeros(64, np.uint8), np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    for frame in (ROWS, RANGE):
        with pytest.raises(c_.B2SError) as e:
            c_.decompress_window_aggregate_rows_keys_packed(c_.CODEC_LZ4BLOCK, src, off, ln, dst, KEYS, 1, NF, KINDS,
                                                            [(c_.WINDOW_SUM, frame, I64, _slot(2), 2)])
        assert e.value.code == c_.E_ARG
        with pytest.raises(c_.B2SError) as e:
            c_.decompress_window_offset_rows_keys_packed(c_.CODEC_LZ4BLOCK, src, off, ln, dst, KEYS, 1, NF, KINDS,
                                                         [(c_.WINDOW_LAST, 0, frame, I64, _slot(2), 2, 0, 0)])
        assert e.value.code == c_.E_ARG


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_window_frame_calls_return_cuda_error_without_a_device():
    L = c_.load()
    assert L.b2s_init(0, 0, 0) == c_.E_CUDA
    fns = [_fr(c_.WINDOW_SUM, ROWS, -6, 0), c_.WINDOW_RANK, (c_.WINDOW_SUM, 2, I64, _slot(2), 2),
           _fr(c_.WINDOW_MAX, RANGE, -3, 3, vt=F64, f=4, null=4), _fr(c_.WINDOW_LAST, ROWS, 1, UF, vt=BYTES, f=5,
                                                                      null=5, flags=c_.WINDOW_IGNORE_NULLS),
           _fr(c_.WINDOW_NTH_VALUE, RANGE, 0, UF, arg=2, vt=c_.window_val_decimal(20, 2), f=3, null=3),
           (c_.WINDOW_LAG, 1, 0, I64, _slot(2), 2, 0, 0)]
    with pytest.raises(c_.B2SError) as e:
        _call(fns)
    assert e.value.code == c_.E_CUDA
    for keys in (_order(1, 6, 0, 4), _order(6, 7, 1 << 9, 1)):  # an int and a byte order column take offsets
        with pytest.raises(c_.B2SError) as e:
            _call([_fr(c_.WINDOW_SUM, RANGE, -100 if keys[1][2] == 4 else -127, 127)], keys)
        assert e.value.code == c_.E_CUDA
    a = c_._window_frame_arrays(KEYS, 1, NF, KINDS, fns)
    src = np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    outs = [C.c_uint64(7) for _ in range(3)]
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = L.b2s_decompress_window_frame_rows_keys_dev(0, c_.CODEC_LZ4BLOCK, 0, 1, src.ctypes.data, off.ctypes.data,
                                                     ln.ctypes.data, None, None, None, *map(c_._arg, a), 0, 0,
                                                     *map(C.byref, outs), st.ctypes.data, bad.ctypes.data)
    assert rc == c_.E_CUDA and [o.value for o in outs] == [0, 0, 0]
    assert L.b2s_last_error()
