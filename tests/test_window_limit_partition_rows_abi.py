"""The window-limit write calls (b2s_window_limit_partition_compress_rows_hash_*) without a GPU: a well-formed call fails
loudly with B2S_E_CUDA and reports nothing as written; every ill-formed call is B2S_E_ARG with b2s_last_error set
before any device is needed.  Also: the prototypes match the headers."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["b2s_window_limit_partition_compress_rows_hash_packed", "b2s_window_limit_partition_compress_rows_hash_dev"]
ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK = 0, 1, 2, 3
STRING, DECIMAL = 3, 9
DESC, NULLS_LAST = 1 << 8, 1 << 9


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return os.path.exists("/dev/nvidia0")


# q67's window key: i_category (a string), sumsales decimal(28,2) DESC NULLS LAST
KEYS = ((STRING, 8, 8, 0), (DECIMAL | DESC | NULLS_LAST, 16, 8, 1))


def _call(L, c, dev=False, R=4, n=2, npk=1, keys=KEYS, fn=RANK, limit=100, rec_len=(44, 44), records=True,
          out_count=True, key_arrays=True, rec_bytes=None):
    rec = np.zeros(128, np.uint8)
    rl = np.array(rec_len, np.uint32)
    nbytes = int(rl.sum()) if rec_bytes is None else rec_bytes
    kt = np.array([k[0] for k in keys] or [0], np.uint32)
    ko = np.array([k[1] for k in keys] or [0], np.uint32)
    kl = np.array([k[2] for k in keys] or [0], np.uint32)
    kn = np.array([k[3] for k in keys] or [0], np.int32)
    doff, dlen, cks = np.zeros(R or 1, np.uint64), np.zeros(R or 1, np.uint64), np.zeros(R or 1, np.uint64)
    st = np.zeros(R or 1, np.int32)
    out = np.zeros(512, np.uint8)
    total, kept = C.c_uint64(7), C.c_uint64(9)
    a = (lambda x: x.ctypes.data) if key_arrays else (lambda x: None)
    args = (c.CODEC_LZ4BLOCK, 0, 0, c.CHECKSUM_CRC32C, R, n, rec.ctypes.data if records else None, nbytes,
            rl.ctypes.data, npk, len(keys), a(kt), a(ko), a(kl), a(kn), fn, limit, out.ctypes.data, out.size,
            doff.ctypes.data, dlen.ctypes.data, C.byref(total), cks.ctypes.data, st.ctypes.data,
            C.byref(kept) if out_count else None)
    rc = L.b2s_window_limit_partition_compress_rows_hash_dev(0, *args) if dev else \
        L.b2s_window_limit_partition_compress_rows_hash_packed(*args)
    return rc, total.value, kept.value, L.b2s_last_error()


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_calls_return_cuda_error_without_a_device():
    c = pkg.capi
    L = c.load()
    assert L.b2s_init(0, 0, 0) == c.E_CUDA
    for dev in (False, True):
        for fn in (ROW_NUMBER, RANK, DENSE_RANK):
            for kw in (dict(), dict(npk=0, R=1), dict(limit=1), dict(limit=2**31 - 1), dict(n=0, rec_len=()),
                       dict(keys=KEYS + tuple((1 | DESC, 24 + 8 * k, 4, -1) for k in range(14))),
                       dict(npk=15, keys=tuple((1, 8 + 8 * k, 4, -1) for k in range(15)) + ((2 | DESC, 128, 8, 2),))):
                rc, total, kept, err = _call(L, c, dev, fn=fn, **kw)
                assert rc == c.E_CUDA and total == 0 and kept == 0 and err, kw
    with pytest.raises(c.B2SError) as e:
        c.window_limit_partition_compress_rows_hash_packed(c.CODEC_LZ4BLOCK, np.zeros(28, np.uint8), [28],
                                                           [(c.KEY_INT64, 8, 8, -1), (c.KEY_INT64, 16, 8, -1)], 1,
                                                           ROW_NUMBER, 1, 200, np.zeros(64, np.uint8))
    assert e.value.code == c.E_CUDA


@pytest.mark.parametrize("kw", [
    # the window key's
    dict(npk=2), dict(npk=3), dict(npk=16, keys=((1, 8, 4, -1),) * 17), dict(keys=((1, 8, 4, -1),) * 17),
    dict(npk=0, keys=()), dict(key_arrays=False), dict(keys=((STRING | DESC, 8, 8, 0), KEYS[1])),
    dict(keys=((STRING | NULLS_LAST, 8, 8, 0), KEYS[1])), dict(keys=(KEYS[0], (4, 16, 8, -1))),
    dict(keys=(KEYS[0], (1 | (1 << 10), 16, 4, -1))), dict(keys=(KEYS[0], (1, 16, 8, -1))),
    dict(keys=(KEYS[0], (1, 16, 4, -2))),
    # the hash call's for the partition columns
    dict(keys=((0, 8, 2, -1), KEYS[1])), dict(keys=((4, 8, 8, -1), KEYS[1])), dict(R=0), dict(R=(1 << 24) + 1),
    dict(records=False), dict(n=2**32, rec_len=(44, 44)),
    # the limit's
    dict(fn=PERCENT_RANK), dict(fn=6), dict(fn=0xFFFFFFFF), dict(limit=0), dict(limit=-5), dict(npk=0, R=2),
    dict(npk=0, R=200), dict(out_count=False),
    # records the lengths do not cover, with and without partition columns
    dict(n=0, rec_bytes=44), dict(n=0, rec_bytes=44, npk=0, R=1)])
def test_ill_formed_calls_are_argument_errors_before_the_device(kw):
    c = pkg.capi
    L = c.load()
    for dev in (False, True):
        rc, total, kept, err = _call(L, c, dev, **kw)
        assert rc == c.E_ARG and total == 0 and err, kw
        assert kept == (0 if kw.get("out_count", True) else 9), kw  # *n_out_records is zeroed when there is one


def test_rejections_name_their_rule():
    c = pkg.capi
    L = c.load()
    for kw, words in ((dict(npk=2), b"ORDER BY"), (dict(keys=((STRING | DESC, 8, 8, 0), KEYS[1])), b"order flag"),
                      (dict(fn=PERCENT_RANK), b"limit_fn"), (dict(limit=0), b"limit"),
                      (dict(npk=0, R=2), b"SinglePartition"), (dict(keys=((0, 8, 2, -1), KEYS[1])), b"boolean"),
                      (dict(n=2**32), b"2^32")):
        rc, _, _, err = _call(L, c, **kw)
        assert rc == c.E_ARG and words in err, (kw, err)


def test_prototypes_match_the_headers():
    protos = dict((p[0], p[2]) for p in pkg.capi.PROTOTYPES)
    assert [len(protos[n]) for n in NAMES] == [25, 26]
    assert set(NAMES) <= set(pkg.capi.SYMBOLS)
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    for name in NAMES:
        decl = re.search(name + r"\(([^;]*)\);", hdr).group(1)
        assert decl.count(",") + 1 == len(protos[name])
        assert "uint32_t n_partition_keys, uint32_t n_keys" in " ".join(decl.split())
        assert "uint32_t limit_fn, int32_t limit" in " ".join(decl.split())
    hp = dict((p[0], p[2]) for p in pkg.host.PROTOTYPES)
    assert "b2sh_serialized_writer_window_limit" in pkg.host.SYMBOLS
    host = open(os.path.join(ROOT, "include", "b200shuffle_host.h")).read()
    decl = re.search(r"b2sh_serialized_writer_window_limit\(([^;]*)\);", host).group(1)
    assert decl.count(",") + 1 == len(hp["b2sh_serialized_writer_window_limit"]) == 9
