"""The composite-key calls' column types and order flags (B2S_KEY_INT16 .. B2S_DECIMAL_KEY, B2S_KEY_DESCENDING,
B2S_KEY_NULLS_LAST): the header's values equal the capi constants.  Runs without a GPU."""
import os
import re

import spark_s3_shuffle_b200 as pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_constants_equal_capi():
    hdr = open(os.path.join(ROOT, "include", "b200shuffle.h")).read()
    found = {}
    for name, value, shift in re.findall(r"#define B2S_(\w+) \((\d+)u?(?: << (\d+))?\)", hdr):
        found[name] = int(value) << int(shift or 0)
    c = pkg.capi
    want = {"KEY_INT16": c.KEY_INT16, "KEY_INT8": c.KEY_INT8, "KEY_FLOAT32": c.KEY_FLOAT32,
            "KEY_FLOAT64": c.KEY_FLOAT64, "DECIMAL_KEY": c.DECIMAL_KEY, "KEY_DESCENDING": c.KEY_DESCENDING,
            "KEY_NULLS_LAST": c.KEY_NULLS_LAST}
    assert {k: found.get(k) for k in want} == want
    # 4 stays unassigned; the flags lie above every type
    types = [c.KEY_BYTES, c.KEY_INT32, c.KEY_INT64, c.STRING_KEY, c.KEY_INT16, c.KEY_INT8, c.KEY_FLOAT32,
             c.KEY_FLOAT64, c.DECIMAL_KEY]
    assert sorted(types) == [0, 1, 2, 3, 5, 6, 7, 8, 9]
    assert c.KEY_DESCENDING & 0xFF == 0 and c.KEY_NULLS_LAST & 0xFF == 0 and c.KEY_DESCENDING != c.KEY_NULLS_LAST
