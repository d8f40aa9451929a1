"""B2S_KEY_NULL_SAFE and B2S_JOIN_EXISTENCE without a GPU: the constants match the header with 4 and 7 unassigned, the
map-side calls that must refuse the flag refuse it before the device while the hash call takes it, and the join calls
fail loudly with B2S_E_CUDA for null-safe keys and the existence join, writing nothing but zeros."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from test_join_rows_abi import _has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NS = 1 << 10


def test_constants_match_the_header_and_4_and_7_stay_unassigned():
    c = pkg.capi
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    assert int(re.search(r"#define B2S_JOIN_EXISTENCE (\d+)", hdr).group(1)) == c.JOIN_EXISTENCE == 8
    assert int(re.search(r"#define B2S_KEY_NULL_SAFE \(1u << (\d+)\)", hdr).group(1)) == 10
    assert c.KEY_NULL_SAFE == NS
    for v in (4, 7):
        assert not re.search(r"#define B2S_JOIN_\w+ %d\b" % v, hdr)


def _records():
    row = (8).to_bytes(8, "little") + (5).to_bytes(8, "little") + bytes(8)  # field 0 null (bit 3 unused), 2 fields
    rec = len(row).to_bytes(4, "big") + row
    return np.frombuffer(rec * 3, np.uint8).copy(), [len(rec)] * 3


KEY = (pkg.capi.KEY_INT64, 8, 8, 0)


def _refusals():
    c = pkg.capi
    recs, lens = _records()
    dst = np.zeros(4096, np.uint8)
    ns = [(KEY[0] | NS,) + KEY[1:]]
    agg = [(c.WINDOW_COUNT, c.WINDOW_VAL_NONE, 0, -1)]
    return {
        "range": lambda: c.partition_compress_rows_range_packed(c.CODEC_LZ4BLOCK, recs, lens, ns, [], dst),
        "partial aggregation": lambda: c.aggregate_partition_compress_rows_hash_packed(c.CODEC_LZ4BLOCK, recs, lens, ns,
                                                                                       agg, 4, dst),
        "grouping sets": lambda: c.aggregate_grouping_sets_partition_compress_rows_hash_packed(
            c.CODEC_LZ4BLOCK, recs, lens, ns, agg, [1], 4, dst),
        "window limit": lambda: c.window_limit_partition_compress_rows_hash_packed(
            c.CODEC_LZ4BLOCK, recs, lens, [KEY] + ns, 1, c.WINDOW_ROW_NUMBER, 1, 4, dst),
    }


@pytest.mark.parametrize("call", ["range", "partial aggregation", "grouping sets", "window limit"])
def test_map_side_calls_other_than_the_hash_call_refuse_the_flag(call):
    c = pkg.capi
    with pytest.raises(c.B2SError) as e:
        _refusals()[call]()
    assert e.value.code == c.E_ARG


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
def test_the_hash_call_takes_the_flag_and_no_other_new_bit():
    c = pkg.capi
    recs, lens = _records()
    dst = np.zeros(4096, np.uint8)
    for keys, code in (([(KEY[0] | NS,) + KEY[1:]], c.E_CUDA), ([(KEY[0] | NS, 8, 8, -1)], c.E_CUDA),
                       ([(c.KEY_BYTES | NS, 8, 1, 0)], c.E_CUDA), ([(KEY[0] | (1 << 11),) + KEY[1:]], c.E_ARG),
                       ([(KEY[0] | NS | c.KEY_DESCENDING,) + KEY[1:]], c.E_ARG),
                       ([(c.KEY_BYTES | NS, 8, 2, 0)], c.E_ARG)):
        with pytest.raises(c.B2SError) as e:
            c.partition_compress_rows_hash_packed(c.CODEC_LZ4BLOCK, recs, lens, keys, 4, dst)
        assert e.value.code == code, keys


@pytest.mark.skipif(_has_gpu(), reason="GPU present")
@pytest.mark.parametrize("jt", [2, 3, 6, 8])
def test_join_calls_return_cuda_error_without_a_device(jt):
    c = pkg.capi
    L = c.load()
    src, dst = np.zeros(256, np.uint8), np.zeros(256, np.uint8)
    off, ln = np.zeros(2, np.uint64), np.full(2, 24, np.uint64)
    kt, kl = np.array([c.KEY_INT64 | NS], np.uint32), np.array([8], np.uint32)
    ko, kn, rn = np.array([8], np.uint32), np.array([0], np.int32), np.array([-1], np.int32)
    kinds = np.array([c.FIELD_FIXED, c.FIELD_VAR], np.uint8)
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    keys = (1, kt.ctypes.data, kl.ctypes.data, ko.ctypes.data, kn.ctypes.data, ko.ctypes.data, rn.ctypes.data,
            2, kinds.ctypes.data, 2, None, dst.ctypes.data, dst.size)
    blocks = (src.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None)
    for fn, lead in ((L.b2s_decompress_join_rows_keys_packed, ()), (L.b2s_decompress_join_rows_keys_dev, (0,))):
        outs = [C.c_uint64(7) for _ in range(4)]
        rc = fn(*lead, jt, c.CODEC_LZ4BLOCK, 0, 1, 2, *blocks, *keys, *map(C.byref, outs), st.ctypes.data,
                bad.ctypes.data)
        assert rc == c.E_CUDA and [o.value for o in outs] == [0, 0, 0, 0]
        assert L.b2s_last_error()
    with pytest.raises(c.B2SError) as e:
        c.decompress_join_rows_keys_packed(jt, c.CODEC_LZ4BLOCK, src, off, ln, 1, dst, [(c.KEY_INT64 | NS, 8, 8, 0)],
                                           [(c.KEY_INT64 | NS, 8, 8, -1)], 2, 2, kinds, None)
    assert e.value.code == c.E_CUDA
