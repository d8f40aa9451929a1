"""The sort-merge join calls (b2s_decompress_join_rows_keys_*) without a GPU: their constants and prototypes match the
header, and like every compute entry point they fail loudly with B2S_E_CUDA — there is no CPU fallback — writing
nothing but zeros to their outputs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return os.path.exists("/dev/nvidia0")


def test_join_constants_and_prototypes_match_the_header():
    c = pkg.capi
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    consts = {"B2S_JOIN_INNER": c.JOIN_INNER, "B2S_JOIN_LEFT_OUTER": c.JOIN_LEFT_OUTER,
              "B2S_JOIN_LEFT_SEMI": c.JOIN_LEFT_SEMI, "B2S_JOIN_LEFT_ANTI": c.JOIN_LEFT_ANTI,
              "B2S_FIELD_FIXED": c.FIELD_FIXED, "B2S_FIELD_VAR": c.FIELD_VAR,
              "B2S_FIELD_DECIMAL_WIDE": c.FIELD_DECIMAL_WIDE}
    for name, v in consts.items():
        assert int(re.search(r"#define %s (\d+)" % name, hdr).group(1)) == v
    protos = dict((p[0], p[2]) for p in c.PROTOTYPES)
    for name, extra in (("b2s_decompress_join_rows_keys_packed", 0), ("b2s_decompress_join_rows_keys_dev", 1)):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(protos[name]) == decl.count(",") + 1 == 30 + extra


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_join_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    src, dst = np.zeros(256, np.uint8), np.zeros(256, np.uint8)
    off, ln = np.zeros(2, np.uint64), np.full(2, 24, np.uint64)
    kt, kl = np.array([c.KEY_INT64], np.uint32), np.array([8], np.uint32)
    ko, kn = np.array([8], np.uint32), np.array([0], np.int32)
    kinds = np.array([c.FIELD_FIXED, c.FIELD_VAR], np.uint8)
    outs = [C.c_uint64(7) for _ in range(4)]
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    keys = (1, kt.ctypes.data, kl.ctypes.data, ko.ctypes.data, kn.ctypes.data, ko.ctypes.data, kn.ctypes.data,
            2, kinds.ctypes.data, 2, kinds.ctypes.data, dst.ctypes.data, dst.size)
    blocks = (src.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None)
    rc = L.b2s_decompress_join_rows_keys_packed(c.JOIN_INNER, c.CODEC_NONE, 0, 1, 2, *blocks, *keys,
                                                *map(C.byref, outs), st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0, 0]
    assert L.b2s_last_error()
    for o in outs:
        o.value = 7
    rc = L.b2s_decompress_join_rows_keys_dev(0, c.JOIN_LEFT_OUTER, c.CODEC_LZ4BLOCK, 0, 1, 2, *blocks, *keys,
                                             *map(C.byref, outs), st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0, 0]
    with pytest.raises(c.B2SError) as e:
        c.decompress_join_rows_keys_packed(c.JOIN_LEFT_SEMI, c.CODEC_LZ4BLOCK, src, off, ln, 1, dst,
                                           [(c.KEY_INT64, 8, 8, 0)], [(c.KEY_INT64, 8, 8, 0)], 2, 2)
    assert e.value.code == c.E_CUDA
