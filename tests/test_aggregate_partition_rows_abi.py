"""The partial-aggregation write calls (b2s_aggregate_partition_compress_rows_hash_*) without a GPU: a well-formed call
fails loudly with B2S_E_CUDA and reports nothing as written; every ill-formed call is B2S_E_ARG before any device is
needed.  Also: the prototypes match the header."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["b2s_aggregate_partition_compress_rows_hash_packed", "b2s_aggregate_partition_compress_rows_hash_dev"]
SUM, COUNT, MIN, MAX, AVG = 6, 7, 8, 9, 10
NONE, I8, I16, I32, I64, F32, F64, DEC, BYTES = range(9)


def dec(p, s=0):
    return DEC | p << 8 | s << 16


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return os.path.exists("/dev/nvidia0")


AGGS = [(SUM, I64, 16, 1), (COUNT, NONE, 0, -1), (AVG, dec(10, 2), 24, 2), (MIN, F64, 32, -1)]


def _call(L, c, dev=False, R=4, n=2, keys=((1, 8, 4, 0),), aggs=AGGS, rec_len=(44, 44), records=True, groups=True,
          agg_arrays=True, rec_bytes=None):
    rec = np.zeros(128, np.uint8)
    rl = np.array(rec_len, np.uint32)
    nbytes = int(rl.sum()) if rec_bytes is None else rec_bytes
    kt = np.array([k[0] for k in keys] or [0], np.uint32)
    ko = np.array([k[1] for k in keys] or [0], np.uint32)
    kl = np.array([k[2] for k in keys] or [0], np.uint32)
    kn = np.array([k[3] for k in keys] or [0], np.int32)
    fn = np.array([a[0] for a in aggs] or [0], np.uint32)
    vt = np.array([a[1] for a in aggs] or [0], np.uint32)
    vo = np.array([a[2] for a in aggs] or [0], np.uint32)
    vn = np.array([a[3] for a in aggs] or [0], np.int32)
    doff, dlen, cks = np.zeros(R, np.uint64), np.zeros(R, np.uint64), np.zeros(R, np.uint64)
    st = np.zeros(R, np.int32)
    out = np.zeros(512, np.uint8)
    total, ng = C.c_uint64(7), C.c_uint64(9)
    a = (lambda x: x.ctypes.data) if agg_arrays else (lambda x: None)
    args = (c.CODEC_LZ4BLOCK, 0, 0, c.CHECKSUM_CRC32C, R, n, rec.ctypes.data if records else None, nbytes,
            rl.ctypes.data, len(keys), kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data, len(aggs),
            a(fn), a(vt), a(vo), a(vn), out.ctypes.data, out.size, doff.ctypes.data, dlen.ctypes.data,
            C.byref(total), cks.ctypes.data, st.ctypes.data, C.byref(ng) if groups else None)
    rc = L.b2s_aggregate_partition_compress_rows_hash_dev(0, *args) if dev else \
        L.b2s_aggregate_partition_compress_rows_hash_packed(*args)
    return rc, total.value, ng.value


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    for dev in (False, True):
        for aggs in (AGGS, ()):
            rc, total, ng = _call(L, c, dev, aggs=aggs)
            assert rc == c.E_CUDA and total == 0 and ng == 0
            assert L.b2s_last_error()
    with pytest.raises(c.B2SError) as e:
        c.aggregate_partition_compress_rows_hash_packed(c.CODEC_LZ4BLOCK, np.zeros(28, np.uint8), [28],
                                                        [(c.KEY_INT64, 8, 8, -1)], [], 200, np.zeros(64, np.uint8))
    assert e.value.code == c.E_CUDA


@pytest.mark.parametrize("kw", [
    # the hash call's rejections
    dict(R=0), dict(keys=()), dict(keys=((1, 8, 4, -1),) * 17), dict(keys=((4, 8, 8, -1),)),
    dict(keys=((0, 8, 2, -1),)), dict(keys=((1 | (1 << 8), 8, 4, -1),)), dict(keys=((1, 8, 4, -2),)),
    dict(records=False), dict(n=2**32, rec_len=(44, 44)),
    # the aggregates'
    dict(aggs=[(SUM, I64, 16, 1)] * 17), dict(agg_arrays=False), dict(groups=False),
    dict(aggs=[(5, I64, 16, 1)]), dict(aggs=[(11, I64, 16, 1)]), dict(aggs=[(SUM, 9, 16, 1)]),
    dict(aggs=[(SUM, I64 | 1 << 8, 16, 1)]), dict(aggs=[(SUM, dec(0), 16, 1)]), dict(aggs=[(SUM, dec(39), 16, 1)]),
    dict(aggs=[(SUM, DEC | 5 << 8 | 6 << 16, 16, 1)]), dict(aggs=[(SUM, NONE, 0, -1)]),
    dict(aggs=[(AVG, BYTES, 16, 1)]), dict(aggs=[(MIN, I8, 16, 1)]), dict(aggs=[(MAX, I16, 16, 1)]),
    dict(aggs=[(MIN, F32, 16, 1)]), dict(aggs=[(MAX, BYTES, 16, 1)]), dict(aggs=[(SUM, dec(29), 16, 1)]),
    dict(aggs=[(AVG, dec(28), 16, 1)]), dict(aggs=[(AVG, I64, 16, 1)] * 9), dict(aggs=[(SUM, dec(20), 16, 1)] * 9),
    dict(aggs=[(SUM, I64, 12, 1)]), dict(aggs=[(SUM, I64, 0, 1)]), dict(aggs=[(SUM, I64, 16, -2)]),
    dict(aggs=[(SUM, I64, 16, 65536)]),
    # records the lengths do not cover
    dict(n=0, rec_bytes=44), dict(n=0, rec_bytes=44, aggs=())])
def test_ill_formed_calls_are_argument_errors_before_the_device(kw):
    c = pkg.capi
    L = c.load()
    for dev in (False, True):
        rc, total, ng = _call(L, c, dev, **kw)
        assert rc == c.E_ARG and total == 0, kw


@pytest.mark.skipif(_has_gpu(), reason="GPU present: the zero-filled records would be bad records")
def test_sixteen_buffers_and_distinct_are_well_formed_without_a_device():
    c = pkg.capi
    L = c.load()
    for aggs in ([(AVG, I64, 16, 1)] * 8, [(SUM, dec(28), 16, 1)] * 8, [(AVG, dec(27), 16, 1)] * 8, [],
                 [(COUNT, BYTES, 16, 1), (MIN, dec(30), 16, -1), (MAX, dec(18), 16, 1), (MIN, I32, 16, 1)]):
        rc, _, _ = _call(L, c, aggs=aggs)
        assert rc == c.E_CUDA, (aggs, rc)


def test_prototypes_match_the_headers():
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    assert [len(protos[n]) for n in NAMES] == [27, 28]
    assert set(NAMES) <= set(pkg.capi.SYMBOLS)
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    for name in NAMES:
        decl = re.search(name + r"\(([^;]*)\);", hdr).group(1)
        assert decl.count(",") + 1 == len(protos[name])
    hp = dict((p[0], p[2]) for p in pkg.host.PROTOTYPES)
    assert "b2sh_serialized_writer_aggregate_rows" in pkg.host.SYMBOLS
    host = open(os.path.join(ROOT, "include", "b200shuffle_host.h")).read()
    decl = re.search(r"b2sh_serialized_writer_aggregate_rows\(([^;]*)\);", host).group(1)
    assert decl.count(",") + 1 == len(hp["b2sh_serialized_writer_aggregate_rows"]) == 6
