"""The exchange-cache calls (b2s_exchange_*, b2s_partition_compress_cached_packed) without a GPU: argument errors are
reported as B2S_E_ARG before any device is needed, and every well-formed call fails loudly with B2S_E_CUDA — there is no
CPU fallback."""
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


def _sort_args(L, c, **kw):
    """b2s_exchange_read_sort_packed with one fetched source and one cached one; kw overrides arguments"""
    a = dict(shuffle=0, start=0, end=1, ids=np.array([0, 1], np.int64), cached=np.array([0, 1], np.uint8),
             rb=104, ko=2, kl=10)
    a.update(kw)
    src = np.zeros(256, np.uint8)
    dst = np.zeros(512, np.uint8)
    off = np.zeros(2, np.uint64)
    ln = np.array([208, 0], np.uint64)
    total, nrec = C.c_uint64(7), C.c_uint64(7)
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    ids = a["ids"].ctypes.data if a["ids"] is not None else None
    cm = a["cached"].ctypes.data if a["cached"] is not None else None
    rc = L.b2s_exchange_read_sort_packed(a["shuffle"], a["start"], a["end"], ids, cm, c.CODEC_NONE, 0, 2,
                                         src.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None, a["rb"],
                                         a["ko"], a["kl"], dst.ctypes.data, dst.size, C.byref(total), C.byref(nrec),
                                         st.ctypes.data, bad.ctypes.data)
    return rc, total.value, nrec.value


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_exchange_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    assert L.b2s_exchange_set_budget(0, 1 << 30) == c.E_CUDA
    assert L.b2s_exchange_remove(0, -1) == c.E_CUDA
    ids = np.array([0, 1], np.int64)
    ln = np.zeros(2, np.uint64)
    assert L.b2s_exchange_lookup(0, 0, 1, 2, ids.ctypes.data, ln.ctypes.data) == c.E_CUDA
    dst = np.zeros(64, np.uint8)
    off, dl = np.zeros(2, np.uint64), np.zeros(2, np.uint64)
    total = C.c_uint64(7)
    st = np.zeros(2, np.int32)
    assert L.b2s_exchange_read_packed(0, 0, 1, 2, ids.ctypes.data, dst.ctypes.data, dst.size, off.ctypes.data,
                                      dl.ctypes.data, C.byref(total), st.ctypes.data) == c.E_CUDA
    assert total.value == 0
    rc, total, nrec = _sort_args(L, c)
    assert rc == c.E_CUDA and total == 0 and nrec == 0
    assert L.b2s_last_error()
    recs = np.zeros(208, np.uint8)
    rl, rp = np.full(2, 104, np.uint32), np.zeros(2, np.uint32)
    doff, dlen, cks = np.zeros(1, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    cached, total = C.c_int32(7), C.c_uint64(7)
    out = np.zeros(512, np.uint8)
    rc = L.b2s_partition_compress_cached_packed(0, 0, c.CODEC_LZ4BLOCK, 0, 0, 0, 1, 2, recs.ctypes.data, 208,
                                                rl.ctypes.data, rp.ctypes.data, out.ctypes.data, out.size,
                                                doff.ctypes.data, dlen.ctypes.data, C.byref(total),
                                                cks.ctypes.data, st.ctypes.data, C.byref(cached))
    assert rc == c.E_CUDA and cached.value == 0
    with pytest.raises(c.B2SError) as e:
        c.exchange_lookup(0, 0, 1, [0, 1])
    assert e.value.code == c.E_CUDA


@pytest.mark.parametrize("start,end", [(-1, 1), (3, 2), (0, (1 << 24) + 1)])
def test_reduce_range_outside_bounds_is_an_argument_error(start, end):
    c = pkg.capi
    L = c.load()
    ids = np.array([0], np.int64)
    ln = np.zeros(1, np.uint64)
    assert L.b2s_exchange_lookup(0, start, end, 1, ids.ctypes.data, ln.ctypes.data) == c.E_ARG
    dst = np.zeros(8, np.uint8)
    off, dl, st = np.zeros(1, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.int32)
    total = C.c_uint64(0)
    assert L.b2s_exchange_read_packed(0, start, end, 1, ids.ctypes.data, dst.ctypes.data, dst.size, off.ctypes.data,
                                      dl.ctypes.data, C.byref(total), st.ctypes.data) == c.E_ARG
    assert _sort_args(L, c, start=start, end=end)[0] == c.E_ARG


@pytest.mark.parametrize("rb,ko,kl", [(0, 0, 1), (104, 2, 0), (104, 2, 17), (104, 100, 10)])
def test_bad_key_or_record_size_is_an_argument_error(rb, ko, kl):
    c = pkg.capi
    assert _sort_args(c.load(), c, rb=rb, ko=ko, kl=kl)[0] == c.E_ARG


def test_null_arrays_are_argument_errors():
    c = pkg.capi
    L = c.load()
    assert _sort_args(L, c, ids=None)[0] == c.E_ARG
    assert _sort_args(L, c, cached=None)[0] == c.E_ARG
    ln = np.zeros(1, np.uint64)
    assert L.b2s_exchange_lookup(0, 0, 1, 1, None, ln.ctypes.data) == c.E_ARG
    ids = np.zeros(1, np.int64)
    assert L.b2s_exchange_lookup(0, 0, 1, 1, ids.ctypes.data, None) == c.E_ARG
    total = C.c_uint64(0)
    assert L.b2s_exchange_read_packed(0, 0, 1, 1, ids.ctypes.data, None, 0, None, None, C.byref(total),
                                      None) == c.E_ARG
    st = np.zeros(1, np.int32)
    assert L.b2s_partition_compress_cached_packed(0, 0, c.CODEC_NONE, 0, 0, 0, 1, 0, None, 0, None, None, None, 0,
                                                  None, None, None, None, st.ctypes.data, None) == c.E_ARG


def test_exchange_prototypes_match_the_header_order():
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    assert len(protos["b2s_partition_compress_cached_packed"]) == 20
    assert len(protos["b2s_exchange_read_sort_packed"]) == 23
    assert len(protos["b2s_exchange_read_sort_dev"]) == 24
    assert len(protos["b2s_exchange_read_packed"]) == 11
    assert len(protos["b2s_exchange_lookup"]) == 6
    assert pkg.capi.load().b2s_strerror(pkg.capi.E_NOT_CACHED) == b"not resident in the exchange cache"
