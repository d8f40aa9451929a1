"""The Decimal aggregate ops of the row aggregation in the C header and in capi, without a GPU: the same values on both
sides, op 8 still unassigned, every new define parenthesised, and SUM_DECIMAL's precision in bits 8..15."""
import os
import re

import spark_s3_shuffle_b200 as pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_decimal_ops_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    ops = dict((k, int(v)) for k, v in re.findall(r"#define B2S_(AGG_\w+) \((\d+)\)", hdr))
    names = ["AGG_SUM_DECIMAL", "AGG_MIN_DECIMAL", "AGG_MAX_DECIMAL"]
    assert ops == {k: getattr(pkg.capi, k) for k in names} == {names[0]: 9, names[1]: 10, names[2]: 11}
    every = [int(v) for v in re.findall(r"#define B2S_AGG_\w+ \(?(\d+)\)?", hdr)]
    assert sorted(every) == [0, 1, 2, 3, 4, 5, 6, 7, 9, 10, 11] and 8 not in every
    assert not re.search(r"#define B2S_AGG_\w+ \d", hdr.split("B2S_AGG_MAX_FLOAT64 7")[1])


def test_sum_decimal_carries_its_precision():
    c = pkg.capi
    assert c.agg_sum_decimal(17) == 9 | (17 << 8)
    assert c.agg_sum_decimal(38) & 0xFF == c.AGG_SUM_DECIMAL and c.agg_sum_decimal(38) >> 8 == 38
