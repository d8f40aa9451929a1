"""b2s_decompress_aggregate_distinct_partition_compress_rows_hash_* without a GPU: the header's constant and
prototypes, every argument rule B2S_E_ARG before the device, and a well-formed call past argument checking to
B2S_E_CUDA."""
import os
import re

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
import test_aggregate_partition_rows_abi as pa_abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
c = pkg.capi
SUM, COUNT, MIN, MAX, AVG, VAR = 6, 7, 8, 9, 10, 16
NONE, I8, I16, I32, I64, F32, F64, DEC, BYTES = range(9)
KI32, KI64, KSTR, KF64, KDEC, KBYTES, KI8 = 1, 2, 3, 8, 9, 0, 6
ALL = c.DISTINCT_ALL_COLUMNS
has_gpu = pa_abi._has_gpu()


def dec(p, s=0):
    return DEC | p << 8 | s << 16


def test_constant_and_prototypes_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    assert int(re.search(r"#define B2S_DISTINCT_ALL_COLUMNS \((-?\d+)\)", hdr).group(1)) == ALL == -1
    for form in ("packed", "dev"):
        assert "b2s_decompress_aggregate_distinct_partition_compress_rows_hash_" + form + "(" in hdr
        assert hasattr(c.load(), "b2s_decompress_aggregate_distinct_partition_compress_rows_hash_" + form)


def call(ng=1, keys=((KI64, 8), (KI32, 4)), aggs=((SUM, I64),), distinct=((COUNT, I32, 1),), R=4, codec=1, alg=0,
         dev=None, dst=None, n=1, **kw):
    src = np.zeros(64, np.uint8)
    off, ln = np.zeros(n, np.uint64), np.full(n, 16, np.uint64)
    dst = np.zeros(1024, np.uint8) if dst is None else dst
    if dev is not None:
        src, dst = 1 << 20, 1 << 21  # device addresses: never touched before the checks
        kw["dst_cap"] = 1024
    with pytest.raises(c.B2SError) as e:
        c.aggregate_distinct_partition_compress_rows_hash(codec, src, off, ln, dst, ng, list(keys), list(aggs),
                                                          list(distinct), R, checksum_alg=alg, dev=dev, **kw)
    return e.value.code


BAD = [
    dict(ng=2),                                                        # no distinct column
    dict(ng=16, keys=[(KI64, 8)] * 17),                                # 17 key columns
    dict(keys=[(KI64 | 1 << 8, 8), (KI32, 4)]),                        # an order flag
    dict(keys=[(KI64, 4), (KI32, 4)]),                                 # key_len does not match its type
    dict(keys=[(KBYTES, 2), (KI32, 4)]),                               # a hashed G boolean of 2 bytes
    dict(ng=0, R=2),                                                   # no G: SinglePartition
    dict(distinct=[]),                                                 # no distinct function
    dict(distinct=[(MIN, I32, 1)]),                                    # MIN(DISTINCT) is plain MIN
    dict(distinct=[(MAX, I32, 1)]),
    dict(distinct=[(17, I32, 1)]),                                     # unknown function
    dict(distinct=[(COUNT, I32, 0)]),                                  # a G column
    dict(distinct=[(COUNT, I32, 2)]),                                  # past n_keys
    dict(distinct=[(COUNT, I64, 1)]),                                  # INT32 column read as a long
    dict(distinct=[(SUM, F64, 1)]),
    dict(distinct=[(COUNT, BYTES, 1)]),                                # bytes of an int column
    dict(keys=[(KI64, 8), (KSTR, 8)], distinct=[(SUM, BYTES, 1)]),     # a string is only counted
    dict(keys=[(KI64, 8), (KSTR, 8)], distinct=[(COUNT, I64, 1)]),
    dict(keys=[(KI64, 8), (KI64, 8)], distinct=[(SUM, dec(20), 1)]),   # a long column holds p <= 18
    dict(keys=[(KI64, 8), (KDEC, 8)], distinct=[(SUM, dec(12), 1)]),   # a decimal key column holds p > 18
    dict(keys=[(KI64, 8), (KDEC, 8)], distinct=[(SUM, dec(30), 1)]),   # decimal SUM p <= 28
    dict(keys=[(KI64, 8), (KDEC, 8)], distinct=[(AVG, dec(28), 1)]),   # decimal AVG p <= 27
    dict(keys=[(KI64, 8), (KI64, 8)], distinct=[(VAR, dec(10), 1)]),   # VARIANCE of a decimal
    dict(distinct=[(SUM, NONE, ALL)]),                                 # ALL takes COUNT only
    dict(keys=[(KI64, 8), (KI32, 4), (KI32, 4)], distinct=[(COUNT, I32, 1)]),  # several X: a function takes them all
    dict(distinct=[(COUNT, I32, ALL)]),                                # ALL takes VAL_NONE
    dict(aggs=[(MIN, I8)]),                                            # F by the map side's rules
    dict(aggs=[(SUM, dec(30))]),
    dict(aggs=[(VAR, I64)] * 11),                                      # 2 keys + 33 fields in the input
    dict(aggs=[(COUNT, NONE)] * 16),                                   # 16 + 1 buffers in the output
    dict(aggs=[(COUNT, NONE)] * 17),                                   # 17 buffers in the input
    dict(R=0),                                                         # the partition step's rules
]


@pytest.mark.parametrize("k", range(len(BAD)))
@pytest.mark.parametrize("dev", [None, 0])
def test_every_rule_is_an_argument_error_before_the_device(k, dev):
    assert call(dev=dev, **BAD[k]) == c.E_ARG, BAD[k]


def test_an_unknown_codec_is_unsupported_as_in_the_aggregated_read():
    for dev in (None, 0):
        assert call(dev=dev, codec=9) == c.E_UNSUPPORTED


def test_more_than_32_output_fields():
    # 1 G + 1 X; F 5 variances (15 fields); D 6 variances (18 fields): 1 + 33 output fields
    assert call(keys=[(KI64, 8), (KI64, 8)], aggs=[(VAR, I64)] * 5, distinct=[(VAR, I64, 1)] * 6) == c.E_ARG
    assert b"32" in c.load().b2s_last_error()


@pytest.mark.skipif(has_gpu, reason="a GPU is present: the call runs")
def test_a_well_formed_call_without_a_device_is_a_cuda_error():
    for dev in (None, 0):
        assert call(dev=dev) == c.E_CUDA
        assert call(ng=0, R=1, dev=dev, keys=[(KI32, 4)], distinct=[(COUNT, NONE, ALL), (SUM, I32, 0)]) == c.E_CUDA
        assert call(dev=dev, keys=[(KI64, 8), (KI32, 4), (KI32, 4)], distinct=[(COUNT, NONE, ALL)]) == c.E_CUDA
        # 2 keys + 27 + 3 fields fill the input's null word, 1 + 30 + 1 the output's
        assert call(dev=dev, aggs=[(VAR, I64)] * 9 + [(COUNT, NONE)] * 3) == c.E_CUDA
