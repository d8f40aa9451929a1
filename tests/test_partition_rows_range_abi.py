"""The range-partitioning write calls (b2s_partition_compress_rows_range_*) without a GPU: like every compute entry
point they fail loudly with B2S_E_CUDA — there is no CPU fallback — and report nothing as written; an ill-formed call,
bound arrays included, is B2S_E_ARG before any device is needed.  Also: the prototypes match the header, and the JNI
and host-mirror declarations exist."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["b2s_partition_compress_rows_range_packed", "b2s_partition_compress_rows_range_dev"]
BOUND = (20).to_bytes(4, "big") + bytes(20)  # a bound row of two fields: null word, two slots


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return os.path.exists("/dev/nvidia0")


def _call(L, c, dev=False, n=2, keys=((1 | (1 << 8), 8, 4, 0), (3 | (1 << 9), 16, 8, -1)), rec_len=(28, 28),
          records=True, bounds=(BOUND, BOUND), n_bounds=None, bound_sum=None, bound_arrays=True):
    rec = np.zeros(64, np.uint8)
    rl = np.array(rec_len, np.uint32)
    kt = np.array([k[0] for k in keys] or [0], np.uint32)
    ko = np.array([k[1] for k in keys] or [0], np.uint32)
    kl = np.array([k[2] for k in keys] or [0], np.uint32)
    kn = np.array([k[3] for k in keys] or [0], np.int32)
    bb = np.frombuffer(b"".join(bounds) or b"\0", np.uint8).copy()
    bl = np.array([len(b) for b in bounds] or [0], np.uint32)
    nb = len(bounds) if n_bounds is None else n_bounds
    R = min(nb, 64) + 1
    doff, dlen, cks = np.zeros(R, np.uint64), np.zeros(R, np.uint64), np.zeros(R, np.uint64)
    st = np.zeros(R, np.int32)
    out = np.zeros(512, np.uint8)
    total = C.c_uint64(7)
    args = (c.CODEC_LZ4BLOCK, 0, 0, c.CHECKSUM_CRC32C, n, rec.ctypes.data if records else None, int(rl.sum()),
            rl.ctypes.data, len(keys), kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data, nb,
            bb.ctypes.data if bound_arrays else None, int(bl.sum()) if bound_sum is None else bound_sum,
            bl.ctypes.data if bound_arrays else None, out.ctypes.data, out.size, doff.ctypes.data, dlen.ctypes.data,
            C.byref(total), cks.ctypes.data, st.ctypes.data)
    rc = L.b2s_partition_compress_rows_range_dev(0, *args) if dev else L.b2s_partition_compress_rows_range_packed(*args)
    return rc, total.value


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_range_partition_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    for kw in (dict(), dict(bounds=()), dict(n=0, rec_len=())):
        for dev in (False, True):
            rc, total = _call(L, c, dev, **kw)
            assert rc == c.E_CUDA and total == 0
            assert L.b2s_last_error()
    with pytest.raises(c.B2SError) as e:
        c.partition_compress_rows_range_packed(c.CODEC_SNAPPY_XERIAL, np.zeros(28, np.uint8), [28],
                                               [(c.KEY_INT64 | c.KEY_DESCENDING, 8, 8, -1)], [BOUND],
                                               np.zeros(64, np.uint8))
    assert e.value.code == c.E_CUDA


@pytest.mark.parametrize("kw", [
    dict(keys=()), dict(keys=((1, 8, 4, -1),) * 17), dict(keys=((4, 8, 8, -1),)), dict(keys=((10, 8, 8, -1),)),
    dict(keys=((0, 8, 17, -1),)), dict(keys=((0, 8, 0, -1),)), dict(keys=((1, 8, 8, -1),)), dict(keys=((3, 8, 4, -1),)),
    dict(keys=((1 | (1 << 10), 8, 4, -1),)), dict(keys=((1, 8, 4, -2),)), dict(records=False),
    dict(n_bounds=1 << 24), dict(n_bounds=0xFFFFFFFF), dict(bound_arrays=False), dict(bound_sum=47),
    dict(bound_sum=0)])
def test_ill_formed_calls_are_argument_errors_before_the_device(kw):
    c = pkg.capi
    L = c.load()
    for dev in (False, True):
        rc, total = _call(L, c, dev, **kw)
        assert rc == c.E_ARG and total == 0, kw
        assert L.b2s_last_error()


def test_range_partition_prototypes_match_the_header():
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    assert [len(protos[n]) for n in NAMES] == [24, 25]
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    for name in NAMES:
        decl = re.search(name + r"\(([^;]*)\);", hdr).group(1)
        assert decl.count(",") + 1 == len(protos[name])
    host = open(os.path.join(ROOT, "include", "b200shuffle_host.h")).read()
    decl = re.search(r"b2sh_serialized_writer_range_rows\(([^;]*)\);", host).group(1)
    hp = dict((p[0], p[2]) for p in pkg.host.PROTOTYPES)
    assert decl.count(",") + 1 == len(hp["b2sh_serialized_writer_range_rows"])
    jni = open(os.path.join(ROOT, "jni", "b200shuffle_jni.c")).read()
    assert "J(partitionCompressRowsRangePacked)" in jni and "b2s_partition_compress_rows_range_packed(" in jni
