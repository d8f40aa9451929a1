"""The exchange cache's row calls (b2s_partition_compress_rows_*_cached_packed, b2s_exchange_read_*_rows_keys_*)
without a GPU: their prototypes, argument errors reported as B2S_E_ARG before any device is needed, and B2S_E_CUDA for
every well-formed call — there is no CPU fallback."""
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


ROW = bytes(24)  # one null-bit word and two 8-byte slots: the key and an aggregate
RECS = np.frombuffer(b"".join(len(ROW).to_bytes(4, "big") + ROW for _ in range(2)), np.uint8).copy()
RL = np.full(2, 4 + len(ROW), np.uint32)


def _keys(n=1):
    return (np.zeros(max(n, 1), np.uint32) + pkg.capi.KEY_INT64, np.full(max(n, 1), 8, np.uint32),
            np.full(max(n, 1), 8, np.uint32), np.zeros(max(n, 1), np.int32))


def _store(L, kind, cached=True):
    """one cached row store of the two records into one partition -> (rc, *cached, *dst_total)"""
    c = pkg.capi
    kt, ko, kl, kn = _keys()
    out = np.zeros(512, np.uint8)
    doff, dlen, cks = np.zeros(1, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    st = np.zeros(1, np.int32)
    total, flag = C.c_uint64(7), C.c_int32(7)
    tail = (out.ctypes.data, out.size, doff.ctypes.data, dlen.ctypes.data, C.byref(total), cks.ctypes.data,
            st.ctypes.data, C.byref(flag) if cached else None)
    rec = (2, RECS.ctypes.data, RECS.size, RL.ctypes.data)
    keys = (1, kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data)
    if kind == "hash":
        rc = L.b2s_partition_compress_rows_hash_cached_packed(0, 0, c.CODEC_LZ4BLOCK, 0, 0, 0, 1, *rec, *keys, *tail)
    elif kind == "range":
        rc = L.b2s_partition_compress_rows_range_cached_packed(0, 0, c.CODEC_LZ4BLOCK, 0, 0, 0, *rec, *keys, 0, None,
                                                               0, None, *tail)
    else:
        rc = L.b2s_partition_compress_rows_round_robin_cached_packed(0, 0, c.CODEC_LZ4BLOCK, 0, 0, 0, 1, 0, 0, *rec,
                                                                     *tail)
    return rc, flag.value, total.value


def _read(L, symbol, ids=True, cached=True, status=True, start=0, end=1, n_keys=1, groups=True):
    """one exchange row read of one fetched source (the two records, codec NONE) and one cached source"""
    c = pkg.capi
    dev = symbol.endswith("_dev")
    kt, ko, kl, kn = _keys(n_keys)
    map_ids = np.array([0, 1], np.int64)
    cm = np.array([0, 1], np.uint8)
    off, ln = np.zeros(2, np.uint64), np.array([RECS.size, 0], np.uint64)
    dst = np.zeros(512, np.uint8)
    total, nrec, ngroups = C.c_uint64(7), C.c_uint64(7), C.c_uint64(7)
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    agg = "_aggregate_" in symbol
    args = ([0] if dev else []) + [0, start, end, map_ids.ctypes.data if ids else None,
                                   cm.ctypes.data if cached else None, c.CODEC_NONE, 0, 2, RECS.ctypes.data,
                                   off.ctypes.data, ln.ctypes.data, None, None, None, n_keys, kt.ctypes.data,
                                   ko.ctypes.data, kl.ctypes.data, kn.ctypes.data]
    if agg:
        op, ao, an = np.array([c.AGG_SUM_INT64], np.uint32), np.array([16], np.uint32), np.array([-1], np.int32)
        args += [1, op.ctypes.data, ao.ctypes.data, an.ctypes.data]
    args += [dst.ctypes.data, dst.size, C.byref(total), C.byref(nrec)]
    if agg:
        args.append(C.byref(ngroups) if groups else None)
    args += [st.ctypes.data if status else None, bad.ctypes.data]
    rc = getattr(L, symbol)(*args)
    return rc, total.value, nrec.value


READS = ["b2s_exchange_read_sort_rows_keys_packed", "b2s_exchange_read_sort_rows_keys_dev",
         "b2s_exchange_read_aggregate_rows_keys_packed", "b2s_exchange_read_aggregate_rows_keys_dev"]
STORES = ["hash", "range", "round_robin"]


def test_row_exchange_prototypes_cover_the_header():
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    lens = {"b2s_partition_compress_rows_hash_cached_packed": 24, "b2s_partition_compress_rows_range_cached_packed": 27,
            "b2s_partition_compress_rows_round_robin_cached_packed": 21,
            "b2s_exchange_read_sort_rows_keys_packed": 25, "b2s_exchange_read_sort_rows_keys_dev": 26,
            "b2s_exchange_read_aggregate_rows_keys_packed": 30, "b2s_exchange_read_aggregate_rows_keys_dev": 31}
    for name, n in lens.items():
        assert len(protos[name]) == n, name
        assert name in pkg.capi.SYMBOLS
    # each cached store takes its uncached form's arguments behind (shuffle_id, map_id), and cached last
    for kind in STORES:
        plain = protos["b2s_partition_compress_rows_%s_packed" % kind]
        assert protos["b2s_partition_compress_rows_%s_cached_packed" % kind][2:-1] == plain
    # each read takes its plain form's arguments behind (shuffle_id, start_reduce, end_reduce, map_ids, cached)
    for name in READS:
        plain = protos[name.replace("exchange_read", "decompress")]
        mine = protos[name]
        if name.endswith("_dev"):
            assert mine[0] == plain[0] and mine[6:] == plain[1:]
        else:
            assert mine[5:] == plain


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_row_exchange_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    for kind in STORES:
        rc, flag, total = _store(L, kind)
        assert (rc, flag, total) == (c.E_CUDA, 0, 0), kind
    for name in READS:
        rc, total, nrec = _read(L, name)
        assert (rc, total, nrec) == (c.E_CUDA, 0, 0), name
    assert L.b2s_last_error()


@pytest.mark.parametrize("kind", STORES)
def test_null_cached_flag_is_an_argument_error(kind):
    c = pkg.capi
    rc, _, total = _store(c.load(), kind, cached=False)
    assert rc == c.E_ARG and total == 0


@pytest.mark.parametrize("name", READS)
def test_read_argument_errors(name):
    c = pkg.capi
    L = c.load()
    assert _read(L, name, ids=False)[0] == c.E_ARG
    assert _read(L, name, cached=False)[0] == c.E_ARG
    assert _read(L, name, status=False)[0] == c.E_ARG
    for start, end in ((-1, 1), (3, 2), (0, (1 << 24) + 1)):
        assert _read(L, name, start=start, end=end)[0] == c.E_ARG
    for n_keys in (0, 17):
        assert _read(L, name, n_keys=n_keys)[0] == c.E_ARG
    if "_aggregate_" in name:
        rc, total, nrec = _read(L, name, groups=False)
        assert (rc, total, nrec) == (c.E_ARG, 0, 0)
