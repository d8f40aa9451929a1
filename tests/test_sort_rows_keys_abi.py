"""The composite-key row calls (b2s_decompress_sort_rows_keys_* / b2s_decompress_aggregate_rows_keys_*) without a GPU:
like every compute entry point they fail loudly with B2S_E_CUDA — there is no CPU fallback — and write nothing but
zeros to their outputs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["b2s_decompress_sort_rows_keys_packed", "b2s_decompress_sort_rows_keys_dev",
         "b2s_decompress_aggregate_rows_keys_packed", "b2s_decompress_aggregate_rows_keys_dev"]


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return os.path.exists("/dev/nvidia0")


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_composite_key_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    src = np.zeros(256, np.uint8)
    dst = np.zeros(256, np.uint8)
    off = np.zeros(1, np.uint64)
    ln = np.full(1, 24, np.uint64)
    kt = np.array([c.STRING_KEY, c.KEY_INT32], np.uint32)
    ko = np.array([8, 16], np.uint32)
    kl = np.array([8, 4], np.uint32)
    kn = np.array([0, -1], np.int32)
    op = np.array([c.AGG_SUM_INT64], np.uint32)
    aoff = np.array([24], np.uint32)
    anf = np.array([-1], np.int32)
    total, nrec, ngrp = C.c_uint64(7), C.c_uint64(7), C.c_uint64(7)
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    keys = (2, kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data)
    tail = (dst.ctypes.data, dst.size, C.byref(total), C.byref(nrec))
    rc = L.b2s_decompress_sort_rows_keys_packed(c.CODEC_NONE, 0, 1, src.ctypes.data, off.ctypes.data, ln.ctypes.data,
                                                None, None, None, *keys, *tail, st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and total.value == 0 and nrec.value == 0
    assert L.b2s_last_error()
    total.value, nrec.value = 7, 7
    rc = L.b2s_decompress_sort_rows_keys_dev(0, c.CODEC_LZ4BLOCK, 0, 1, src.ctypes.data, off.ctypes.data,
                                             ln.ctypes.data, None, None, None, *keys, *tail, st.ctypes.data,
                                             bad.ctypes.data)
    assert rc == c.E_CUDA and total.value == 0 and nrec.value == 0
    aggs = (1, op.ctypes.data, aoff.ctypes.data, anf.ctypes.data)
    total.value, nrec.value = 7, 7
    rc = L.b2s_decompress_aggregate_rows_keys_packed(c.CODEC_NONE, 0, 1, src.ctypes.data, off.ctypes.data,
                                                     ln.ctypes.data, None, None, None, *keys, *aggs, *tail,
                                                     C.byref(ngrp), st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and total.value == 0 and nrec.value == 0 and ngrp.value == 0
    total.value, nrec.value, ngrp.value = 7, 7, 7
    rc = L.b2s_decompress_aggregate_rows_keys_dev(0, c.CODEC_SNAPPY_XERIAL, 0, 1, src.ctypes.data, off.ctypes.data,
                                                  ln.ctypes.data, None, None, None, *keys, 0, None, None, None, *tail,
                                                  C.byref(ngrp), st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and total.value == 0 and nrec.value == 0 and ngrp.value == 0
    with pytest.raises(c.B2SError) as e:
        c.decompress_sort_rows_keys_packed(c.CODEC_LZ4BLOCK, src, off, ln, dst, [(c.STRING_KEY, 8, 8, 0)])
    assert e.value.code == c.E_CUDA
    with pytest.raises(c.B2SError) as e:
        c.decompress_aggregate_rows_keys_packed(c.CODEC_LZ4BLOCK, src, off, ln, dst, [(c.KEY_INT64, 8, 8, -1)],
                                                aggs=[(c.AGG_MAX_FLOAT64, 16, 1)])
    assert e.value.code == c.E_CUDA


def test_composite_key_prototypes_match_the_header():
    """the ctypes prototypes take the header's argument counts, and the string key constant matches the header's"""
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    assert [len(protos[n]) for n in NAMES] == [20, 21, 25, 26]
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    assert int(re.search(r"#define B2S_STRING_KEY (\d+)", hdr).group(1)) == pkg.capi.STRING_KEY
    assert pkg.capi.STRING_KEY not in (pkg.capi.KEY_BYTES, pkg.capi.KEY_INT32, pkg.capi.KEY_INT64)
    for name in NAMES:
        decl = re.search(name + r"\(([^;]*)\);", hdr).group(1)
        assert decl.count(",") + 1 == len(protos[name])
