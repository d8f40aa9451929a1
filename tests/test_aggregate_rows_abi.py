"""The row aggregation calls (b2s_decompress_aggregate_rows_*) without a GPU: like every compute entry point they fail
loudly with B2S_E_CUDA — there is no CPU fallback — and write nothing but zeros to their outputs."""
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


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_aggregate_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    src = np.zeros(256, np.uint8)
    dst = np.zeros(256, np.uint8)
    off = np.zeros(1, np.uint64)
    ln = np.full(1, 24, np.uint64)
    op = np.array([c.AGG_SUM_INT64], np.uint32)
    aoff = np.array([16], np.uint32)
    anf = np.array([-1], np.int32)
    total, nrec, ngrp = C.c_uint64(7), C.c_uint64(7), C.c_uint64(7)
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = L.b2s_decompress_aggregate_rows_packed(c.CODEC_NONE, 0, 1, src.ctypes.data, off.ctypes.data, ln.ctypes.data,
                                                None, None, None, c.KEY_INT64, 8, 8, 0, 1, op.ctypes.data,
                                                aoff.ctypes.data, anf.ctypes.data, dst.ctypes.data, dst.size,
                                                C.byref(total), C.byref(nrec), C.byref(ngrp), st.ctypes.data,
                                                bad.ctypes.data)
    assert rc == c.E_CUDA and total.value == 0 and nrec.value == 0 and ngrp.value == 0
    assert L.b2s_last_error()
    total.value, nrec.value, ngrp.value = 7, 7, 7
    rc = L.b2s_decompress_aggregate_rows_dev(0, c.CODEC_LZ4BLOCK, 0, 1, src.ctypes.data, off.ctypes.data,
                                             ln.ctypes.data, None, None, None, c.KEY_INT32, 8, 4, -1, 0, None, None,
                                             None, dst.ctypes.data, dst.size, C.byref(total), C.byref(nrec),
                                             C.byref(ngrp), st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and total.value == 0 and nrec.value == 0 and ngrp.value == 0
    with pytest.raises(c.B2SError) as e:
        c.decompress_aggregate_rows_packed(c.CODEC_LZ4BLOCK, src, off, ln, dst, c.KEY_INT64, 0, 8,
                                           aggs=[(c.AGG_MAX_FLOAT64, 8, 1)])
    assert e.value.code == c.E_CUDA


def test_aggregate_prototypes_match_the_header():
    """the ctypes prototypes take the header's argument counts, and the aggregate ops match the header's"""
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    assert len(protos["b2s_decompress_aggregate_rows_packed"]) == 24
    assert len(protos["b2s_decompress_aggregate_rows_dev"]) == 25
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    ops = dict((k, int(v)) for k, v in re.findall(r"#define B2S_(AGG_\w+) (\d+)", hdr))
    names = ["AGG_SUM_INT64", "AGG_SUM_FLOAT64", "AGG_MIN_INT32", "AGG_MAX_INT32", "AGG_MIN_INT64", "AGG_MAX_INT64",
             "AGG_MIN_FLOAT64", "AGG_MAX_FLOAT64"]
    assert ops == {k: getattr(pkg.capi, k) for k in names}
    for name in ("b2s_decompress_aggregate_rows_packed", "b2s_decompress_aggregate_rows_dev"):
        decl = re.search(name + r"\(([^;]*)\);", hdr).group(1)
        assert decl.count(",") + 1 == len(protos[name])
