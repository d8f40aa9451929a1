"""The aggregate window calls (b2s_decompress_window_aggregate_rows_keys_*) without a GPU: their constants and
prototypes match the header, every argument rule of the functions is B2S_E_ARG before the device is looked at, and a
valid call fails loudly with B2S_E_CUDA — there is no CPU fallback — writing nothing but zeros to its outputs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from test_window_rows_abi import _has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_window_aggregate_constants_and_prototypes_match_the_header():
    c = pkg.capi
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    consts = {"B2S_WINDOW_SUM": c.WINDOW_SUM, "B2S_WINDOW_COUNT": c.WINDOW_COUNT, "B2S_WINDOW_MIN": c.WINDOW_MIN,
              "B2S_WINDOW_MAX": c.WINDOW_MAX, "B2S_WINDOW_AVG": c.WINDOW_AVG,
              "B2S_WINDOW_FRAME_PARTITION": c.WINDOW_FRAME_PARTITION,
              "B2S_WINDOW_FRAME_ROWS_RUNNING": c.WINDOW_FRAME_ROWS_RUNNING,
              "B2S_WINDOW_FRAME_RANGE_RUNNING": c.WINDOW_FRAME_RANGE_RUNNING,
              "B2S_WINDOW_VAL_NONE": c.WINDOW_VAL_NONE, "B2S_WINDOW_VAL_INT8": c.WINDOW_VAL_INT8,
              "B2S_WINDOW_VAL_INT16": c.WINDOW_VAL_INT16, "B2S_WINDOW_VAL_INT32": c.WINDOW_VAL_INT32,
              "B2S_WINDOW_VAL_INT64": c.WINDOW_VAL_INT64, "B2S_WINDOW_VAL_FLOAT32": c.WINDOW_VAL_FLOAT32,
              "B2S_WINDOW_VAL_FLOAT64": c.WINDOW_VAL_FLOAT64, "B2S_WINDOW_VAL_DECIMAL": c.WINDOW_VAL_DECIMAL}
    for name, v in consts.items():
        assert int(re.search(r"#define %s (\d+)\n" % name, hdr).group(1)) == v
    assert c.WINDOW_SUM == c.WINDOW_NTILE + 1  # one fn array mixes ranking and aggregate functions
    assert c.window_val_decimal(17, 2) == 7 | 17 << 8 | 2 << 16
    protos = dict((p[0], p[2]) for p in c.PROTOTYPES)
    for name, extra in (("b2s_decompress_window_aggregate_rows_keys_packed", 0),
                        ("b2s_decompress_window_aggregate_rows_keys_dev", 1)):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(protos[name]) == decl.count(",") + 1 == 31 + extra


def test_host_mirror_declares_the_window_aggregate_read():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle_host.h")).read()
    decl = re.search(r"int b2sh_reader_read_window_aggregate_rows\((.*?)\);", hdr, re.S).group(1)
    protos = dict((p[0], p[2]) for p in pkg.host.PROTOTYPES)
    assert len(protos["b2sh_reader_read_window_aggregate_rows"]) == decl.count(",") + 1 == 20


def test_jni_declares_the_window_aggregate_call():
    jni = open(os.path.join(ROOT, "jni", "b200shuffle_jni.c")).read()
    assert "J(decompressWindowAggregateRowsKeysPacked)" in jni
    assert "b2s_decompress_window_aggregate_rows_keys_packed(" in jni


# fields: 0 a long key, 1 a long order key, 2 a long value, 3 a DECIMAL_WIDE value, 4 a double value
KINDS = [0, 0, 0, 2, 0]
KEYS = [(2, 8 + 0, 8, 0), (2, 8 + 8, 8, 1)]


def _call(fns, kinds=KINDS, n_fields=5):
    c = pkg.capi
    src, dst = np.zeros(64, np.uint8), np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    return c.decompress_window_aggregate_rows_keys_packed(c.CODEC_LZ4BLOCK, src, off, ln, dst, KEYS, 1, n_fields,
                                                          kinds, fns)


def _agg(fn, frame=1, vt=None, off=24, null=2):
    c = pkg.capi
    return (fn, frame, c.WINDOW_VAL_INT64 if vt is None else vt, off, null)


def _d(p, s):
    return pkg.capi.window_val_decimal(p, s)


c_ = pkg.capi
BAD = [
    ("no function", []),
    ("17 functions", [_agg(c_.WINDOW_SUM)] * 17),
    ("an unknown function", [_agg(11)]),
    ("a ranking function with a frame", [(c_.WINDOW_RANK, 1, c_.WINDOW_VAL_NONE, 0, -1)]),
    ("a ranking function with an input", [(c_.WINDOW_RANK, 0, c_.WINDOW_VAL_INT64, 24, 2)]),
    ("NTILE of 0 buckets", [(c_.WINDOW_NTILE, 0)]),
    ("an aggregate with frame 0", [_agg(c_.WINDOW_SUM, 0)]),
    ("an unknown frame", [_agg(c_.WINDOW_MAX, 4)]),
    ("SUM of VAL_NONE", [_agg(c_.WINDOW_SUM, vt=c_.WINDOW_VAL_NONE)]),
    ("MIN of VAL_NONE", [_agg(c_.WINDOW_MIN, vt=c_.WINDOW_VAL_NONE)]),
    ("an unknown val_type", [_agg(c_.WINDOW_COUNT, vt=8)]),
    ("a precision on an int", [_agg(c_.WINDOW_SUM, vt=c_.WINDOW_VAL_INT64 | 5 << 8)]),
    ("decimal p 0", [_agg(c_.WINDOW_MIN, vt=_d(0, 0))]),
    ("decimal p 39", [_agg(c_.WINDOW_MIN, vt=_d(39, 0), off=32, null=3)]),
    ("decimal s above p", [_agg(c_.WINDOW_MIN, vt=_d(10, 11))]),
    ("decimal SUM above p 28", [_agg(c_.WINDOW_SUM, vt=_d(29, 2), off=32, null=3)]),
    ("decimal AVG above p 24", [_agg(c_.WINDOW_AVG, vt=_d(25, 2), off=32, null=3)]),
    ("a compact decimal on a DECIMAL_WIDE field", [_agg(c_.WINDOW_SUM, vt=_d(18, 2), off=32, null=3)]),
    ("a wide decimal on a FIXED field", [_agg(c_.WINDOW_SUM, vt=_d(19, 2), off=24, null=2)]),
    ("a long on a DECIMAL_WIDE field", [_agg(c_.WINDOW_MAX, off=32, null=3)]),
    ("a value slot in the null words", [_agg(c_.WINDOW_SUM, off=0)]),
    ("a value slot not on a slot boundary", [_agg(c_.WINDOW_SUM, off=28)]),
    ("a value slot past the last field", [_agg(c_.WINDOW_SUM, off=48)]),
    ("a value null bit not below n_fields", [_agg(c_.WINDOW_SUM, null=5)]),
    ("a value null bit below -1", [_agg(c_.WINDOW_SUM, null=-2)]),
    ("a bad function after a good one", [_agg(c_.WINDOW_SUM), c_.WINDOW_RANK, _agg(c_.WINDOW_AVG, 9)]),
]


@pytest.mark.parametrize("why,fns", BAD, ids=[b[0] for b in BAD])
def test_bad_functions_are_argument_errors_before_the_device(why, fns):
    with pytest.raises(pkg.capi.B2SError) as e:
        _call(fns)
    assert e.value.code == pkg.capi.E_ARG, why


def test_bad_fields_are_argument_errors_before_the_device():
    c = pkg.capi
    for kinds, nf in ((None, 5), ([0, 0, 0, 3, 0], 5), ([], 0), ([0] * 65537, 65537)):
        with pytest.raises(c.B2SError) as e:
            _call([_agg(c.WINDOW_SUM)], kinds, nf)
        assert e.value.code == c.E_ARG


def test_argument_error_writes_zeros_and_a_message():
    c = pkg.capi
    L = c.load()
    a = c._window_aggregate_arrays(KEYS, 1, 5, KINDS, [_agg(c.WINDOW_SUM, 0)])
    outs = [C.c_uint64(7) for _ in range(3)]
    dst = np.zeros(64, np.uint8)
    rc = L.b2s_decompress_window_aggregate_rows_keys_packed(0, 0, 0, None, None, None, None, None, None,
                                                            *map(c._arg, a), dst.ctypes.data, dst.size,
                                                            *map(C.byref, outs), None, None)
    assert rc == c.E_ARG and [o.value for o in outs] == [0, 0, 0]
    assert b"fn_frame" in L.b2s_last_error()
    a = list(a)
    a[11] = None  # no fn_frame array
    rc = L.b2s_decompress_window_aggregate_rows_keys_packed(0, 0, 0, None, None, None, None, None, None,
                                                            *map(c._arg, a), dst.ctypes.data, dst.size,
                                                            *map(C.byref, outs), None, None)
    assert rc == c.E_ARG


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_window_aggregate_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    fns = [_agg(c.WINDOW_SUM, 2), _agg(c.WINDOW_AVG, 3, _d(24, 2), 32, 3), c.WINDOW_RANK,
           (c.WINDOW_COUNT, 1, c.WINDOW_VAL_NONE, 0, -1), _agg(c.WINDOW_MIN, 1, c.WINDOW_VAL_FLOAT64, 40, -1)]
    with pytest.raises(c.B2SError) as e:
        _call(fns)
    assert e.value.code == c.E_CUDA
    a = c._window_aggregate_arrays(KEYS, 1, 5, KINDS, fns)
    src = np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    outs = [C.c_uint64(7) for _ in range(3)]
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = L.b2s_decompress_window_aggregate_rows_keys_dev(0, c.CODEC_LZ4BLOCK, 0, 1, src.ctypes.data, off.ctypes.data,
                                                         ln.ctypes.data, None, None, None, *map(c._arg, a), 0, 0,
                                                         *map(C.byref, outs), st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0]
    assert L.b2s_last_error()
