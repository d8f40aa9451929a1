#!/usr/bin/env python
"""Cost of an aggregate-window reducer on the GPU: b2s_decompress_window_aggregate_rows_keys_dev over a reducer's
shuffled blocks, against today's GPU path for the same blocks, one b2s_decompress_sort_rows_keys_dev call by the
window's key, which leaves the Window to the JVM.

Each reducer gets --rows rows in --maps Snappy blocks with CRC32C checksums.  Shapes:
  q98    : [i_class (16-byte string), i_item_desc string, itemrevenue decimal(17,2)]: sum(itemrevenue) over
           (partition by i_class), --classes classes per reducer; the whole-partition frame, no ORDER BY.
  q47    : [i_category, i_brand, s_store_name, s_company_name (16-byte strings), d_year int, sum_sales decimal(17,2)]:
           avg(sum_sales) over (partition by the five), about 2,000 partitions.
  q51    : [item_sk long, d_date long, sales decimal(17,2), name string]: sum(sales) over (partition by item_sk order by
           d_date rows between unbounded preceding and current row), about 2,000 items.
  serial : [t long, x double, tag string]: sum(x) over (order by t rows between unbounded preceding and current row),
           one reducer-wide partition: the double sum's serial fold over every row.
Every timed reducer's output is checked against the model (tests/window_agg_model.py) before it is timed.  Per
reducer, after one untimed call of each path, each path is timed once (b2s_last_timing: kernel_ms = the whole call on
the device, dominant_ms = the window step).  The packed forms of both are called once more for their device-to-host
bytes.  The card's name and power limit are read in the same run.

    python tools/window_agg_rows_bench.py [--rows 91000] [--maps 400] [--reducers 3] [--shapes q98,q47,q51,serial]

Prints one JSON document.
"""
import argparse
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from join_rows_bench import CRC32C, SNAPPY, blocks, card, rows_of, spread  # noqa: E402

INT32, INT64, STRING = 1, 2, 3
FIXED, VAR = 0, 1
SUM, AVG = 6, 10
FRAME_PARTITION, FRAME_ROWS = 1, 2
VAL_FLOAT64, VAL_DECIMAL = 6, 7


def dec(p, s):
    return VAL_DECIMAL | p << 8 | s << 16


def strings(rng, n, domain, prefix):
    return np.frombuffer(b"".join(b"%s%08d" % (prefix, c) for c in rng.integers(0, domain, n)), np.uint8).reshape(n, 16)


def cents(rng, n):
    return rng.integers(-10**6, 10**9, n).astype(np.int64).view(np.uint64)


def shape_rows(rng, shape, n, classes):
    """-> ((records, lengths), keys, n_partition_keys, kinds, fns)"""
    if shape == "q98":
        slots = np.zeros((n, 3), np.uint64)
        slots[:, 2] = cents(rng, n)
        var = {0: strings(rng, n, classes, b"Class###"), 1: 8 * rng.integers(2, 12, n)}
        return (rows_of(slots, var, rng), [(STRING, 8, 8, -1)], 1, [VAR, VAR, FIXED],
                [(SUM, FRAME_PARTITION, dec(17, 2), 8 + 16, -1)])
    if shape == "q47":
        slots = np.zeros((n, 6), np.uint64)
        slots[:, 4] = rng.integers(1999, 2002, n).astype(np.uint64)
        slots[:, 5] = cents(rng, n)
        var = {0: strings(rng, n, 10, b"Categor#"), 1: strings(rng, n, 20, b"Brand###"),
               2: strings(rng, n, 3, b"Store###"), 3: strings(rng, n, 1, b"Company#")}
        keys = [(STRING, 8, 8, -1), (STRING, 16, 8, -1), (STRING, 24, 8, -1), (STRING, 32, 8, -1), (INT32, 40, 4, -1)]
        return (rows_of(slots, var, rng), keys, 5, [VAR, VAR, VAR, VAR, FIXED, FIXED],
                [(AVG, FRAME_PARTITION, dec(17, 2), 8 + 40, -1)])
    if shape == "q51":
        slots = np.zeros((n, 4), np.uint64)
        slots[:, 0] = rng.integers(0, 2000, n).astype(np.uint64)
        slots[:, 1] = rng.integers(2450000, 2451000, n).astype(np.uint64)
        slots[:, 2] = cents(rng, n)
        return (rows_of(slots, {3: 8 * rng.integers(1, 4, n)}, rng), [(INT64, 8, 8, -1), (INT64, 16, 8, -1)], 1,
                [FIXED, FIXED, FIXED, VAR], [(SUM, FRAME_ROWS, dec(17, 2), 8 + 16, -1)])
    slots = np.zeros((n, 3), np.uint64)
    slots[:, 0] = rng.integers(0, 1 << 40, n).astype(np.uint64)
    slots[:, 1] = (rng.normal(size=n) * 1e3).view(np.uint64)
    return (rows_of(slots, {2: 8 * rng.integers(1, 3, n)}, rng), [(INT64, 8, 8, -1)], 0, [FIXED, FIXED, VAR],
            [(SUM, FRAME_ROWS, VAL_FLOAT64, 8 + 8, -1)])


def run(capi, args, shape, red, d_src, d_dst, cap):
    from window_agg_model import model_window_aggregate
    rng = np.random.default_rng(1000 * red + len(shape))
    (rec, rec_len), keys, npk, kinds, fns = shape_rows(rng, shape, args.rows, args.classes)
    nf = len(kinds)
    plain, arena, off, ln, ck = blocks(capi, rec, rec_len, args.maps, rng)
    n = off.size
    sb, sl = np.arange(n + 1, dtype=np.uint32), ln.astype(np.uint64)
    capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
    stream, _, rows = model_window_aggregate(plain, keys, npk, nf, kinds, fns)

    def window():
        r = capi.decompress_window_aggregate_rows_keys_dev(SNAPPY, d_src, off, ln, d_dst, cap, keys, npk, nf, kinds,
                                                           fns, CRC32C, sb, sl, ck)
        return r, capi.last_timing()

    def sort():
        capi.decompress_sort_rows_keys_dev(SNAPPY, d_src, off, ln, d_dst, cap, keys, CRC32C, sb, sl, ck)
        return capi.last_timing()

    r, _ = window()
    out = np.zeros(max(r["total"], 1), np.uint8)
    capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
    assert (hashlib.sha256(out[:r["total"]].tobytes()).hexdigest(), r["n_out_records"]) == \
        (hashlib.sha256(stream).hexdigest(), rows), "%s differs from the model" % shape
    _, t = window()
    sort()
    s = sort()
    host = np.zeros(int(rec_len.sum()) + len(stream) + 64, np.uint8)
    capi.decompress_window_aggregate_rows_keys_packed(SNAPPY, arena, off, ln, host, keys, npk, nf, kinds, fns, CRC32C,
                                                      sb, sl, ck)
    w_d2h = capi.last_timing()["d2h_bytes"]
    capi.decompress_sort_rows_keys_packed(SNAPPY, arena, off, ln, host, keys, CRC32C, sb, sl, ck)
    s_d2h = capi.last_timing()["d2h_bytes"]
    return {"in_rows": int(rec_len.size), "in_mb": float(rec_len.sum()) / 1e6, "window_kernel_ms": t["kernel_ms"],
            "window_step_ms": t["dominant_ms"], "sort_kernel_ms": s["kernel_ms"], "out_rows": r["n_out_records"],
            "out_mb": r["total"] / 1e6, "window_d2h_mb": w_d2h / 1e6, "sort_d2h_mb": s_d2h / 1e6}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=91000, help="rows per reducer")
    ap.add_argument("--maps", type=int, default=400)
    ap.add_argument("--reducers", type=int, default=3)
    ap.add_argument("--classes", type=int, default=20, help="q98 classes per reducer")
    ap.add_argument("--shapes", default="q98,q47,q51,serial")
    ap.add_argument("--cap-gib", type=float, default=0.5, help="device output buffer")
    args = ap.parse_args()
    import spark_s3_shuffle_b200 as pkg
    capi = pkg.capi
    capi.init(1)
    cap = int(args.cap_gib * 2**30)
    d_src, d_dst = capi.dev_alloc(1 << 30), capi.dev_alloc(cap)
    res = {"card": card(), "rows": args.rows, "maps": args.maps, "shapes": {}}
    try:
        for shape in args.shapes.split(","):
            per = [run(capi, args, shape, red, d_src, d_dst, cap) for red in range(args.reducers)]
            res["shapes"][shape] = {k: spread([p[k] for p in per]) for k in per[0]}
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
