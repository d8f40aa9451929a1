"""The right and full outer join types of b2s_decompress_join_rows_keys_* without a GPU: their constants match the
header, and both entry points fail loudly with B2S_E_CUDA for them, writing nothing but zeros to their outputs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from test_join_rows_abi import _has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_outer_join_constants_match_the_header():
    c = pkg.capi
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    for name, v in (("B2S_JOIN_RIGHT_OUTER", c.JOIN_RIGHT_OUTER), ("B2S_JOIN_FULL_OUTER", c.JOIN_FULL_OUTER)):
        assert int(re.search(r"#define %s (\d+)" % name, hdr).group(1)) == v
    assert (c.JOIN_RIGHT_OUTER, c.JOIN_FULL_OUTER) == (5, 6)
    assert not re.search(r"#define B2S_JOIN_\w+ 4\b", hdr)  # 4 stays unassigned


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
@pytest.mark.parametrize("jt", [5, 6])
def test_outer_join_calls_return_cuda_error_without_a_device(jt):
    c = pkg.capi
    L = c.load()
    src, dst = np.zeros(256, np.uint8), np.zeros(256, np.uint8)
    off, ln = np.zeros(2, np.uint64), np.full(2, 24, np.uint64)
    kt, kl = np.array([c.KEY_INT64], np.uint32), np.array([8], np.uint32)
    ko, kn = np.array([8], np.uint32), np.array([0], np.int32)
    kinds = np.array([c.FIELD_FIXED, c.FIELD_DECIMAL_WIDE], np.uint8)
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    keys = (1, kt.ctypes.data, kl.ctypes.data, ko.ctypes.data, kn.ctypes.data, ko.ctypes.data, kn.ctypes.data,
            2, kinds.ctypes.data, 2, kinds.ctypes.data, dst.ctypes.data, dst.size)
    blocks = (src.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None)
    outs = [C.c_uint64(7) for _ in range(4)]
    rc = L.b2s_decompress_join_rows_keys_packed(jt, c.CODEC_NONE, 0, 1, 2, *blocks, *keys, *map(C.byref, outs),
                                                st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0, 0]
    assert L.b2s_last_error()
    outs = [C.c_uint64(7) for _ in range(4)]
    rc = L.b2s_decompress_join_rows_keys_dev(0, jt, c.CODEC_LZ4BLOCK, 0, 1, 2, *blocks, *keys, *map(C.byref, outs),
                                             st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0, 0]
    with pytest.raises(c.B2SError) as e:
        c.decompress_join_rows_keys_packed(jt, c.CODEC_LZ4BLOCK, src, off, ln, 1, dst, [(c.KEY_INT64, 8, 8, 0)],
                                           [(c.KEY_INT64, 8, 8, 0)], 2, 2, kinds, kinds)
    assert e.value.code == c.E_CUDA
