"""The offset window calls (b2s_decompress_window_offset_rows_keys_*) without a GPU: their constants and prototypes match
the header, the JNI shim and the host mirror, every argument rule of the functions is B2S_E_ARG before the device is
looked at, and a valid call fails loudly with B2S_E_CUDA — there is no CPU fallback — writing nothing but zeros to its
outputs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from test_window_rows_abi import _has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_window_offset_constants_and_prototypes_match_the_header():
    c = pkg.capi
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    consts = {"B2S_WINDOW_LAG": c.WINDOW_LAG, "B2S_WINDOW_LEAD": c.WINDOW_LEAD, "B2S_WINDOW_FIRST": c.WINDOW_FIRST,
              "B2S_WINDOW_LAST": c.WINDOW_LAST, "B2S_WINDOW_NTH_VALUE": c.WINDOW_NTH_VALUE,
              "B2S_WINDOW_VAL_BYTES": c.WINDOW_VAL_BYTES, "B2S_WINDOW_IGNORE_NULLS": c.WINDOW_IGNORE_NULLS,
              "B2S_WINDOW_HAS_DEFAULT": c.WINDOW_HAS_DEFAULT}
    for name, v in consts.items():
        assert int(re.search(r"#define %s (\d+)\n" % name, hdr).group(1)) == v
    assert c.WINDOW_LAG == c.WINDOW_AVG + 1  # one fn array mixes all three families
    assert c.WINDOW_VAL_BYTES == c.WINDOW_VAL_DECIMAL + 1
    protos = dict((p[0], p[2]) for p in c.PROTOTYPES)
    for name, extra in (("b2s_decompress_window_offset_rows_keys_packed", 0),
                        ("b2s_decompress_window_offset_rows_keys_dev", 1)):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(protos[name]) == decl.count(",") + 1 == 33 + extra
        assert "const uint32_t* fn_flags, const uint64_t* fn_default" in " ".join(decl.split())


def test_host_mirror_declares_the_window_offset_read():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle_host.h")).read()
    decl = re.search(r"int b2sh_reader_read_window_offset_rows\((.*?)\);", hdr, re.S).group(1)
    protos = dict((p[0], p[2]) for p in pkg.host.PROTOTYPES)
    assert len(protos["b2sh_reader_read_window_offset_rows"]) == decl.count(",") + 1 == 22
    assert hasattr(pkg.host.S3ShuffleReader, "readWindowOffsetRows")


def test_jni_declares_the_window_offset_call():
    jni = open(os.path.join(ROOT, "jni", "b200shuffle_jni.c")).read()
    assert "J(decompressWindowOffsetRowsKeysPacked)" in jni
    assert "b2s_decompress_window_offset_rows_keys_packed(" in jni


# fields: 0 a long key, 1 a long order key, 2 a long value, 3 a DECIMAL_WIDE value, 4 a double value, 5 a string,
# 6 an int, 7 a byte, 8 a compact decimal
KINDS = [0, 0, 0, 2, 0, 1, 0, 0, 0]
NF = len(KINDS)
KEYS = [(2, 8 + 0, 8, 0), (2, 8 + 8, 8, 1)]


def _slot(f):
    return 8 + 8 * f


def _call(fns, kinds=KINDS, n_fields=NF):
    c = pkg.capi
    src, dst = np.zeros(64, np.uint8), np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    return c.decompress_window_offset_rows_keys_packed(c.CODEC_LZ4BLOCK, src, off, ln, dst, KEYS, 1, n_fields, kinds,
                                                       fns)


c_ = pkg.capi
I64, BYTES, F64, I32, I8 = c_.WINDOW_VAL_INT64, c_.WINDOW_VAL_BYTES, c_.WINDOW_VAL_FLOAT64, c_.WINDOW_VAL_INT32, \
    c_.WINDOW_VAL_INT8
IGN, DEF = c_.WINDOW_IGNORE_NULLS, c_.WINDOW_HAS_DEFAULT


def _off(fn, arg=1, frame=0, vt=I64, f=2, null=2, flags=0, default=0):
    return (fn, arg, frame, vt, _slot(f), null, flags, default)


def _d(p, s):
    return pkg.capi.window_val_decimal(p, s)


BAD = [
    ("an unknown function", [_off(16)]),
    ("LAG offset 0", [_off(c_.WINDOW_LAG, 0)]),
    ("LEAD offset below 0", [_off(c_.WINDOW_LEAD, -1)]),
    ("NTH_VALUE n 0", [_off(c_.WINDOW_NTH_VALUE, 0, 1)]),
    ("FIRST with an argument", [_off(c_.WINDOW_FIRST, 1, 1)]),
    ("LAST with an argument", [_off(c_.WINDOW_LAST, 2, 2)]),
    ("LAG with a frame", [_off(c_.WINDOW_LAG, 1, 1)]),
    ("LEAD with a frame", [_off(c_.WINDOW_LEAD, 1, 3)]),
    ("FIRST with frame 0", [_off(c_.WINDOW_FIRST, 0, 0)]),
    ("NTH_VALUE with an unknown frame", [_off(c_.WINDOW_NTH_VALUE, 1, 4)]),
    ("an offset function of VAL_NONE", [_off(c_.WINDOW_LAG, vt=c_.WINDOW_VAL_NONE)]),
    ("an unknown val_type", [_off(c_.WINDOW_LAG, vt=9)]),
    ("an aggregate of VAL_BYTES", [(c_.WINDOW_MIN, 1, BYTES, _slot(5), 5)]),
    ("VAL_BYTES on a FIXED field", [_off(c_.WINDOW_LAG, vt=BYTES, f=2)]),
    ("a long on a VAR field", [_off(c_.WINDOW_LAG, f=5, null=5)]),
    ("a wide decimal on a FIXED field", [_off(c_.WINDOW_LAG, vt=_d(20, 2), f=2)]),
    ("a compact decimal on a DECIMAL_WIDE field", [_off(c_.WINDOW_LAG, vt=_d(18, 2), f=3, null=3)]),
    ("decimal p 39", [_off(c_.WINDOW_LAG, vt=_d(39, 2), f=3, null=3)]),
    ("a value slot past the last field", [_off(c_.WINDOW_LAG, f=NF)]),
    ("a value null bit not below n_fields", [_off(c_.WINDOW_LAG, null=NF)]),
    ("an unknown flag bit", [_off(c_.WINDOW_LAG, flags=4)]),
    ("flags on a ranking function", [(c_.WINDOW_RANK, 0, 0, c_.WINDOW_VAL_NONE, 0, -1, IGN, 0)]),
    ("flags on an aggregate", [(c_.WINDOW_SUM, 0, 1, I64, _slot(2), 2, IGN, 0)]),
    ("a default on FIRST", [_off(c_.WINDOW_FIRST, 0, 1, flags=DEF, default=1)]),
    ("a default on NTH_VALUE", [_off(c_.WINDOW_NTH_VALUE, 1, 1, flags=DEF)]),
    ("a default on a string", [_off(c_.WINDOW_LAG, vt=BYTES, f=5, null=5, flags=DEF)]),
    ("a default on a wide decimal", [_off(c_.WINDOW_LEAD, vt=_d(20, 2), f=3, null=3, flags=DEF)]),
    ("a default without HAS_DEFAULT", [_off(c_.WINDOW_LAG, default=5)]),
    ("default bits above an int", [_off(c_.WINDOW_LAG, vt=I32, f=6, null=6, flags=DEF, default=1 << 32)]),
    ("default bits above a byte", [_off(c_.WINDOW_LEAD, vt=I8, f=7, null=7, flags=DEF, default=0x100)]),
    ("a bad function after good ones", [_off(c_.WINDOW_LAG), c_.WINDOW_RANK, (c_.WINDOW_SUM, 1, I64, _slot(2), 2),
                                        _off(c_.WINDOW_LEAD, 0)]),
    ("17 functions", [_off(c_.WINDOW_LAG)] * 17),
    ("no function", []),
]


@pytest.mark.parametrize("why,fns", BAD, ids=[b[0] for b in BAD])
def test_bad_functions_are_argument_errors_before_the_device(why, fns):
    with pytest.raises(pkg.capi.B2SError) as e:
        _call(fns)
    assert e.value.code == pkg.capi.E_ARG, why


def test_argument_error_writes_zeros_and_a_message():
    c = pkg.capi
    L = c.load()
    a = c._window_offset_arrays(KEYS, 1, NF, KINDS, [_off(c.WINDOW_LAG, flags=DEF, vt=BYTES, f=5, null=5)])
    outs = [C.c_uint64(7) for _ in range(3)]
    dst = np.zeros(64, np.uint8)
    rc = L.b2s_decompress_window_offset_rows_keys_packed(0, 0, 0, None, None, None, None, None, None,
                                                         *map(c._arg, a), dst.ctypes.data, dst.size,
                                                         *map(C.byref, outs), None, None)
    assert rc == c.E_ARG and [o.value for o in outs] == [0, 0, 0]
    assert b"HAS_DEFAULT" in L.b2s_last_error()
    for at in (15, 16):  # no fn_flags, no fn_default
        b = list(c._window_offset_arrays(KEYS, 1, NF, KINDS, [_off(c.WINDOW_LAG)]))
        b[at] = None
        rc = L.b2s_decompress_window_offset_rows_keys_packed(0, 0, 0, None, None, None, None, None, None,
                                                             *map(c._arg, b), dst.ctypes.data, dst.size,
                                                             *map(C.byref, outs), None, None)
        assert rc == c.E_ARG and [o.value for o in outs] == [0, 0, 0]


def test_the_aggregate_call_still_rejects_the_offset_codes():
    c = pkg.capi
    src, dst = np.zeros(64, np.uint8), np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    for fns in ([(c.WINDOW_LAG, 0, I64, _slot(2), 2)], [(c.WINDOW_MIN, 1, BYTES, _slot(5), 5)]):
        with pytest.raises(c.B2SError) as e:
            c.decompress_window_aggregate_rows_keys_packed(c.CODEC_LZ4BLOCK, src, off, ln, dst, KEYS, 1, NF, KINDS,
                                                           fns)
        assert e.value.code == c.E_ARG


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_window_offset_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    fns = [_off(c.WINDOW_LAG, 1, 0, I64, 2, 2, IGN | DEF, 7), c.WINDOW_RANK, (c.WINDOW_SUM, 2, I64, _slot(2), 2),
           _off(c.WINDOW_LEAD, 3, 0, BYTES, 5, 5), _off(c.WINDOW_NTH_VALUE, 2, 1, _d(20, 2), 3, 3, IGN),
           _off(c.WINDOW_LAST, 0, 3, F64, 4, -1, IGN), _off(c.WINDOW_FIRST, 0, 2, _d(9, 2), 8, 8)]
    with pytest.raises(c.B2SError) as e:
        _call(fns)
    assert e.value.code == c.E_CUDA
    a = c._window_offset_arrays(KEYS, 1, NF, KINDS, fns)
    src = np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    outs = [C.c_uint64(7) for _ in range(3)]
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = L.b2s_decompress_window_offset_rows_keys_dev(0, c.CODEC_LZ4BLOCK, 0, 1, src.ctypes.data, off.ctypes.data,
                                                      ln.ctypes.data, None, None, None, *map(c._arg, a), 0, 0,
                                                      *map(C.byref, outs), st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0]
    assert L.b2s_last_error()
