"""The window calls (b2s_decompress_window_rows_keys_*) without a GPU: their constants and prototypes match the header,
and like every compute entry point they fail loudly with B2S_E_CUDA — there is no CPU fallback — writing nothing but
zeros to their outputs."""
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


def test_window_constants_and_prototypes_match_the_header():
    c = pkg.capi
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    consts = {"B2S_WINDOW_ROW_NUMBER": c.WINDOW_ROW_NUMBER, "B2S_WINDOW_RANK": c.WINDOW_RANK,
              "B2S_WINDOW_DENSE_RANK": c.WINDOW_DENSE_RANK, "B2S_WINDOW_PERCENT_RANK": c.WINDOW_PERCENT_RANK,
              "B2S_WINDOW_CUME_DIST": c.WINDOW_CUME_DIST, "B2S_WINDOW_NTILE": c.WINDOW_NTILE}
    for name, v in consts.items():
        assert int(re.search(r"#define %s (\d+)\n" % name, hdr).group(1)) == v
    assert int(re.search(r"#define B2S_WINDOW_NO_LIMIT (0x[0-9a-f]+)u", hdr).group(1), 16) == c.WINDOW_NO_LIMIT
    protos = dict((p[0], p[2]) for p in c.PROTOTYPES)
    for name, extra in (("b2s_decompress_window_rows_keys_packed", 0), ("b2s_decompress_window_rows_keys_dev", 1)):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(protos[name]) == decl.count(",") + 1 == 29 + extra


def test_host_mirror_declares_the_window_read():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle_host.h")).read()
    decl = re.search(r"int b2sh_reader_read_window_rows\((.*?)\);", hdr, re.S).group(1)
    protos = dict((p[0], p[2]) for p in pkg.host.PROTOTYPES)
    assert len(protos["b2sh_reader_read_window_rows"]) == decl.count(",") + 1 == 18


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_window_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    src, dst = np.zeros(256, np.uint8), np.zeros(256, np.uint8)
    off, ln = np.zeros(2, np.uint64), np.full(2, 24, np.uint64)
    kt = np.array([c.KEY_INT64, c.KEY_INT32 | c.KEY_DESCENDING], np.uint32)
    ko, kl, kn = np.array([16, 24], np.uint32), np.array([8, 4], np.uint32), np.array([0, 1], np.int32)
    kinds = np.array([c.FIELD_FIXED, c.FIELD_FIXED, c.FIELD_VAR], np.uint8)
    fn, arg = np.array([c.WINDOW_RANK], np.uint32), np.zeros(1, np.int32)
    outs = [C.c_uint64(7) for _ in range(3)]
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    args = (1, 2, kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data, 3, kinds.ctypes.data, 1,
            fn.ctypes.data, arg.ctypes.data, c.WINDOW_RANK, 100, dst.ctypes.data, dst.size)
    blocks = (src.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None)
    rc = L.b2s_decompress_window_rows_keys_packed(c.CODEC_NONE, 0, 2, *blocks, *args, *map(C.byref, outs),
                                                  st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0]
    assert L.b2s_last_error()
    for o in outs:
        o.value = 7
    rc = L.b2s_decompress_window_rows_keys_dev(0, c.CODEC_LZ4BLOCK, 0, 2, *blocks, *args, *map(C.byref, outs),
                                               st.ctypes.data, bad.ctypes.data)
    assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0]
    with pytest.raises(c.B2SError) as e:
        c.decompress_window_rows_keys_packed(c.CODEC_LZ4BLOCK, src, off, ln, dst, [(c.KEY_INT64, 16, 8, 0)] * 2, 1, 3,
                                             kinds, [c.WINDOW_ROW_NUMBER, (c.WINDOW_NTILE, 4)])
    assert e.value.code == c.E_CUDA
