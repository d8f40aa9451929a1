"""The round-robin write calls (b2s_partition_compress_rows_round_robin_*) without a GPU: like every compute entry point
they fail loudly with B2S_E_CUDA — there is no CPU fallback — and report nothing as written; an ill-formed call is
B2S_E_ARG before any memory is read or any device is needed.  Also: the prototypes match the header, and the JNI and
host-mirror declarations exist."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["b2s_partition_compress_rows_round_robin_packed", "b2s_partition_compress_rows_round_robin_dev"]


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return os.path.exists("/dev/nvidia0")


def _call(L, c, dev=False, R=5, start=2, sort=1, n=2, rec_len=(12, 12), records=True, arrays=True):
    """records and rec_len are never read by a call that must fail before the device: n may exceed them"""
    rec = np.zeros(64, np.uint8)
    rl = np.array(rec_len or [0], np.uint32)
    Ro = max(min(R, 64), 1)
    doff, dlen, cks = np.zeros(Ro, np.uint64), np.zeros(Ro, np.uint64), np.zeros(Ro, np.uint64)
    st = np.zeros(Ro, np.int32)
    out = np.zeros(512, np.uint8)
    total = C.c_uint64(7)
    args = (c.CODEC_LZ4BLOCK, 0, 0, c.CHECKSUM_CRC32C, R, start, sort, n, rec.ctypes.data if records else None,
            int(sum(rec_len)), rl.ctypes.data if arrays else None, out.ctypes.data, out.size, doff.ctypes.data, dlen.ctypes.data, C.byref(total), cks.ctypes.data,
            st.ctypes.data)
    if dev:
        rc = L.b2s_partition_compress_rows_round_robin_dev(0, *args)
    else:
        rc = L.b2s_partition_compress_rows_round_robin_packed(*args)
    return rc, total.value


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_round_robin_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    # the last one: start + n == 2^31 - 1, Spark's last position that does not wrap, is well-formed
    for kw in (dict(), dict(sort=0), dict(R=1, start=0), dict(n=0, rec_len=()), dict(R=1 << 24, start=(1 << 24) - 1),
               dict(R=7, start=6, n=(1 << 31) - 7)):
        for dev in (False, True):
            rc, total = _call(L, c, dev, **kw)
            assert rc == c.E_CUDA and total == 0, kw
            assert L.b2s_last_error()
    with pytest.raises(c.B2SError) as e:
        c.partition_compress_rows_round_robin_packed(c.CODEC_SNAPPY_XERIAL, np.zeros(12, np.uint8), [12], 3, 0, 1,
                                                     np.zeros(64, np.uint8))
    assert e.value.code == c.E_CUDA


@pytest.mark.parametrize("kw", [
    dict(R=0, start=0), dict(R=(1 << 24) + 1, start=0), dict(start=-1), dict(start=5), dict(R=1, start=1),
    dict(sort=2), dict(sort=0xFFFFFFFF), dict(start=(1 << 24) - 1, R=1 << 24, n=(1 << 31) - (1 << 24) + 1),
    dict(start=4, n=(1 << 31) - 4), dict(R=3, start=2, n=(1 << 31) - 2, sort=0), dict(n=1 << 32), dict(records=False),
    dict(arrays=False)])
def test_ill_formed_calls_are_argument_errors_before_the_device(kw):
    c = pkg.capi
    L = c.load()
    for dev in (False, True):
        rc, total = _call(L, c, dev, **kw)
        assert rc == c.E_ARG and total == 0, (kw, rc)
        assert L.b2s_last_error()


def test_round_robin_prototypes_match_the_header():
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    assert [len(protos[n]) for n in NAMES] == [18, 19]
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    for name in NAMES:
        decl = re.search(name + r"\(([^;]*)\);", hdr).group(1)
        assert decl.count(",") + 1 == len(protos[name])
    host = open(os.path.join(ROOT, "include", "b200shuffle_host.h")).read()
    decl = re.search(r"b2sh_serialized_writer_round_robin_rows\(([^;]*)\);", host).group(1)
    hp = dict((p[0], p[2]) for p in pkg.host.PROTOTYPES)
    assert decl.count(",") + 1 == len(hp["b2sh_serialized_writer_round_robin_rows"])
    jni = open(os.path.join(ROOT, "jni", "b200shuffle_jni.c")).read()
    assert "J(partitionCompressRowsRoundRobinPacked)" in jni
    assert "b2s_partition_compress_rows_round_robin_packed(" in jni
