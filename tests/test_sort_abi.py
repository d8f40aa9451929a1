"""The key-sorted read calls (b2s_decompress_sort_*) without a GPU: like every compute entry point they fail loudly
with B2S_E_CUDA — there is no CPU fallback — and write nothing but zeros to their outputs."""
import ctypes as C
import os

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return os.path.exists("/dev/nvidia0")


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_sort_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    src = np.zeros(256, np.uint8)
    dst = np.zeros(256, np.uint8)
    off = np.zeros(1, np.uint64)
    ln = np.full(1, 208, np.uint64)
    total, nrec = C.c_uint64(7), C.c_uint64(7)
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = L.b2s_decompress_sort_packed(c.CODEC_NONE, 0, 1, src.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None,
                                      None, 104, 2, 10, dst.ctypes.data, dst.size, C.byref(total), C.byref(nrec),
                                      st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and total.value == 0 and nrec.value == 0
    assert L.b2s_last_error()
    rc = L.b2s_decompress_sort_dev(0, c.CODEC_LZ4BLOCK, 0, 1, src.ctypes.data, off.ctypes.data, ln.ctypes.data, None,
                                   None, None, 104, 2, 10, dst.ctypes.data, dst.size, C.byref(total), C.byref(nrec),
                                   st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA
    with pytest.raises(c.B2SError) as e:
        c.decompress_sort_packed(c.CODEC_LZ4BLOCK, src, off, ln, dst, 104, 2, 10)
    assert e.value.code == c.E_CUDA


def test_sort_prototypes_match_the_header_order():
    """the ctypes prototypes of the two calls take the header's argument count"""
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    assert len(protos["b2s_decompress_sort_packed"]) == 18
    assert len(protos["b2s_decompress_sort_dev"]) == 19
