"""The central-moment aggregates without a GPU: B2S_WINDOW_VARIANCE (16) of the partial-aggregation calls and
B2S_AGG_VARIANCE (12) of the aggregated reads in the header and in capi, every new argument rule B2S_E_ARG before the
device, well-formed calls past argument checking to B2S_E_CUDA, and the window calls still rejecting 16."""
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
import test_aggregate_grouping_sets_rows_abi as gs_abi
import test_aggregate_partition_rows_abi as pa_abi
import test_window_agg_rows_abi as wa_abi
import test_window_frame_rows_abi as wf_abi
import test_window_offset_rows_abi as wo_abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
c = pkg.capi
VAR = 16
SUM, COUNT, AVG = 6, 7, 10
NONE, I8, I16, I32, I64, F32, F64, DEC, BYTES = range(9)
has_gpu = pa_abi._has_gpu()


def test_constants_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    assert "#define B2S_AGG_VARIANCE (B2S_AGG_MAX_DECIMAL + 1)" in hdr
    assert c.AGG_VARIANCE == c.AGG_MAX_DECIMAL + 1 == 12
    assert int(re.search(r"#define B2S_WINDOW_VARIANCE (\d+)", hdr).group(1)) == c.WINDOW_VARIANCE == VAR


# ---- the map side ----
def var_aggs(k, vt=I64):
    return [(VAR, vt, 16, 1)] * k


@pytest.mark.parametrize("aggs", [
    [(VAR, DEC | 10 << 8 | 2 << 16, 16, 1)], [(VAR, DEC | 30 << 8, 16, 1)], [(VAR, BYTES, 16, 1)],
    [(VAR, NONE, 0, -1)], [(VAR, I64 | 1 << 8, 16, 1)], [(VAR, I64, 12, 1)], [(VAR, I64, 16, -2)],
    [(17, I64, 16, 1)], var_aggs(17)])
def test_ill_formed_variance_inputs_are_argument_errors(aggs):
    L = c.load()
    for dev in (False, True):
        assert pa_abi._call(L, c, dev, aggs=aggs)[:2] == (c.E_ARG, 0), aggs
        assert gs_abi._call(L, c, dev, aggs=aggs)[:2] == (c.E_ARG, 0), aggs


def test_more_than_32_partial_row_fields_are_argument_errors():
    L = c.load()
    one, two, three = ((1, 8, 4, 0),), ((1, 8, 4, 0), (2, 16, 8, -1)), ((1, 8, 4, 0), (2, 16, 8, -1), (1, 24, 4, 2))
    for dev in (False, True):
        # 1 key + 11 variances = 34 fields; 3 keys + 10 variances = 33; 2 keys + 10 variances + a count = 33
        for keys, aggs in ((one, var_aggs(11)), (three, var_aggs(10)), (two, var_aggs(10) + [(COUNT, NONE, 0, -1)])):
            rc, total, _ = pa_abi._call(L, c, dev, keys=keys, aggs=aggs)
            assert (rc, total) == (c.E_ARG, 0)
            assert b"32" in L.b2s_last_error()
        # with grouping sets gid takes a field too: 2 keys + gid + 10 variances = 33
        rc, total, _, err = gs_abi._call(L, c, dev, keys=two, aggs=var_aggs(10), sets=(0b11, 0))
        assert (rc, total) == (c.E_ARG, 0) and b"32" in err


@pytest.mark.skipif(has_gpu, reason="GPU present: the zero-filled records would be bad records")
def test_well_formed_variance_calls_reach_the_device():
    L = c.load()
    q17 = [(COUNT, I32, 16, 1), (AVG, I32, 16, 1), (VAR, I32, 16, 1)] * 3  # 9 entries of the 12 (one key column)
    three = ((1, 8, 4, 0), (2, 16, 8, -1), (1, 24, 4, 2))
    for dev in (False, True):
        for vt in (I8, I16, I32, I64, F32, F64):
            assert pa_abi._call(L, c, dev, aggs=[(VAR, vt, 16, 1), (SUM, F64, 24, -1)])[0] == c.E_CUDA, vt
            assert gs_abi._call(L, c, dev, aggs=[(VAR, vt, 16, 1)])[0] == c.E_CUDA, vt
        # 2 keys + 10 variances = 32 fields; q17: 3 keys and 12 entries of 18 fields
        assert pa_abi._call(L, c, dev, keys=three[:2], aggs=var_aggs(10))[0] == c.E_CUDA
        assert pa_abi._call(L, c, dev, keys=three, aggs=q17 + q17[:3])[0] == c.E_CUDA
        # with grouping sets: 1 key + gid + 10 variances
        assert gs_abi._call(L, c, dev, keys=three[:1], aggs=var_aggs(10), sets=(1, 0))[0] == c.E_CUDA


def test_the_window_calls_still_reject_variance():
    for call, fns in ((wa_abi._call, [wa_abi._agg(VAR)]), (wo_abi._call, [wo_abi._off(VAR)]),
                      (wf_abi._call, [wf_abi._fr(VAR, 1, wf_abi.c_.WINDOW_UNBOUNDED_PRECEDING,
                                                 wf_abi.c_.WINDOW_UNBOUNDED_FOLLOWING)])):
        with pytest.raises(c.B2SError) as e:
            call(fns)
        assert e.value.code == c.E_ARG


# ---- the reduce side (its argument errors need a device: tests/test_gpu_aggregate_variance_rows.py) ----
def reads(aggs):
    """every aggregated read over one block, a nullable long key in slot 8"""
    src, dst = np.zeros(64, np.uint8), np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    key = (c.KEY_INT64, 8, 8, 0)
    yield lambda: c.decompress_aggregate_rows_packed(c.CODEC_NONE, src, off, ln, dst, *key, aggs=aggs)
    yield lambda: c.decompress_aggregate_rows_keys_packed(c.CODEC_NONE, src, off, ln, dst, [key], aggs)
    yield lambda: c.exchange_read_aggregate_rows_keys_packed(0, 0, 1, [0], [0], c.CODEC_NONE, src, off, ln, dst,
                                                             [key], aggs)


@pytest.mark.skipif(has_gpu, reason="GPU present")
def test_variance_entries_reach_the_device():
    for aggs in ([(c.AGG_VARIANCE, 16, -1)], [(c.AGG_VARIANCE, 16, -1), (c.AGG_SUM_INT64, 40, -1)],
                 [(c.agg_sum_decimal(20), 16, 1), (c.AGG_VARIANCE, 24, -1), (c.AGG_VARIANCE, 48, -1)],
                 [(c.AGG_VARIANCE, 16 + 24 * k, -1) for k in range(16)]):
        for call in reads(aggs):
            with pytest.raises(c.B2SError) as e:
                call()
            assert e.value.code == c.E_CUDA, aggs
