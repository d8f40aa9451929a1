#!/usr/bin/env python
"""Cost of a sliding-frame window reducer on the GPU: b2s_decompress_window_frame_rows_keys_dev over a reducer's
shuffled blocks, against the same functions on the running frame through b2s_decompress_window_offset_rows_keys_dev,
and against today's GPU path for the same blocks, one b2s_decompress_sort_rows_keys_dev call by the window's key, which
leaves the Window to the JVM.

Each reducer gets --rows rows in --maps Snappy blocks with CRC32C checksums.  Shapes:
  ma7    : [item_sk long, d_date int, price decimal(17,2), name string]: avg(price) over (partition by item_sk order by
           d_date rows between 6 preceding and current row), about 2,000 items
  days30 : [item_sk long, d_date int (a date), x double, name string]: sum(x) over (partition by item_sk order by d_date
           range between 29 preceding and current row), about 2,000 items over 1,000 days
  minmax : [item_sk long, t long, v long, name string]: min(v), max(v) over (partition by item_sk order by t rows
           between 50 preceding and 50 following), about 2,000 items
  suffix : [item_sk long, t long, x double, name string]: sum(x) over (partition by item_sk order by t rows between
           current row and unbounded following), partitions of about 3,000 rows: a fresh fold per row, quadratic
Each shape's output is checked against the model (tests/window_frame_model.py) before it is timed: every reducer's,
but only the first reducer's for minmax and suffix, whose model is slow.  Per reducer, after one untimed call of each
path, each path is timed once (b2s_last_timing: kernel_ms = the whole call on the device, dominant_ms = the window
step).  The card's name and power limit are read in the same run.

    python tools/window_frame_rows_bench.py [--rows 91000] [--maps 400] [--reducers 3] [--shapes ma7,days30,minmax,suffix]

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

INT32, INT64 = 1, 2
FIXED, VAR = 0, 1
SUM, MIN, MAX, AVG = 6, 8, 9, 10
FRAME_ROWS_RUNNING, FRAME_RANGE_RUNNING, FRAME_ROWS, FRAME_RANGE = 2, 3, 4, 5
VAL_INT64, VAL_FLOAT64, VAL_DECIMAL = 4, 6, 7
UF = 2**63 - 1


def dec(p, s):
    return VAL_DECIMAL | p << 8 | s << 16


def shape_rows(rng, shape, n):
    """-> ((records, lengths), keys, kinds, frame fns, the running-frame fns of the offset call)"""
    slots = np.zeros((n, 4), np.uint64)
    items = 30 if shape == "suffix" else 2000
    slots[:, 0] = rng.integers(0, items, n).astype(np.uint64)
    if shape in ("ma7", "days30"):
        slots[:, 1] = rng.integers(2450000, 2451000, n).astype(np.uint64)
        keys = [(INT64, 8, 8, -1), (INT32, 16, 4, -1)]
    else:
        slots[:, 1] = rng.integers(0, 1 << 40, n).astype(np.uint64)
        keys = [(INT64, 8, 8, -1), (INT64, 16, 8, -1)]
    if shape == "ma7":
        slots[:, 2] = rng.integers(-10**6, 10**9, n).astype(np.int64).view(np.uint64)
        vt, funcs = dec(17, 2), [(AVG, FRAME_ROWS, -6, 0, FRAME_ROWS_RUNNING)]
    elif shape == "minmax":
        slots[:, 2] = rng.integers(-2**62, 2**62, n).astype(np.int64).view(np.uint64)
        vt, funcs = VAL_INT64, [(MIN, FRAME_ROWS, -50, 50, FRAME_ROWS_RUNNING),
                                (MAX, FRAME_ROWS, -50, 50, FRAME_ROWS_RUNNING)]
    else:
        slots[:, 2] = (rng.normal(size=n) * 1e3).view(np.uint64)
        vt = VAL_FLOAT64
        funcs = [(SUM, FRAME_RANGE, -29, 0, FRAME_RANGE_RUNNING)] if shape == "days30" else \
            [(SUM, FRAME_ROWS, 0, UF, FRAME_ROWS_RUNNING)]
    fns = [(fn, 0, fr, vt, 8 + 16, -1, 0, 0, lo, hi) for fn, fr, lo, hi, _ in funcs]
    running = [(fn, 0, old, vt, 8 + 16, -1, 0, 0) for fn, _, _, _, old in funcs]
    return rows_of(slots, {3: 8 * rng.integers(1, 3, n)}, rng), keys, [FIXED, FIXED, FIXED, VAR], fns, running


def run(capi, args, shape, red, d_src, d_dst, cap):
    from window_frame_model import model_window_frame
    rng = np.random.default_rng(1000 * red + len(shape))
    (rec, rec_len), keys, kinds, fns, running = shape_rows(rng, shape, args.rows)
    nf = len(kinds)
    plain, arena, off, ln, ck = blocks(capi, rec, rec_len, args.maps, rng)
    n = off.size
    sb, sl = np.arange(n + 1, dtype=np.uint32), ln.astype(np.uint64)
    capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)

    def frame():
        r = capi.decompress_window_frame_rows_keys_dev(SNAPPY, d_src, off, ln, d_dst, cap, keys, 1, nf, kinds, fns,
                                                       CRC32C, sb, sl, ck)
        return r, capi.last_timing()

    def offset():
        capi.decompress_window_offset_rows_keys_dev(SNAPPY, d_src, off, ln, d_dst, cap, keys, 1, nf, kinds, running,
                                                    CRC32C, sb, sl, ck)
        return capi.last_timing()

    def sort():
        capi.decompress_sort_rows_keys_dev(SNAPPY, d_src, off, ln, d_dst, cap, keys, CRC32C, sb, sl, ck)
        return capi.last_timing()

    r, _ = frame()
    checked = red == 0 or shape in ("ma7", "days30")
    if checked:
        stream, _, rows, unsupported = model_window_frame(plain, keys, 1, nf, kinds, fns)
        out = np.zeros(max(r["total"], 1), np.uint8)
        capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        assert not unsupported
        assert (hashlib.sha256(out[:r["total"]].tobytes()).hexdigest(), r["n_out_records"]) == \
            (hashlib.sha256(stream).hexdigest(), rows), "%s differs from the model" % shape
    _, t = frame()
    offset()
    o = offset()
    sort()
    s = sort()
    return {"in_rows": int(rec_len.size), "in_mb": float(rec_len.sum()) / 1e6, "checked": int(checked),
            "frame_kernel_ms": t["kernel_ms"], "frame_step_ms": t["dominant_ms"],
            "frame_launches": t["kernel_launches"], "running_kernel_ms": o["kernel_ms"],
            "running_step_ms": o["dominant_ms"], "sort_kernel_ms": s["kernel_ms"], "out_rows": r["n_out_records"]}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=91000, help="rows per reducer")
    ap.add_argument("--maps", type=int, default=400)
    ap.add_argument("--reducers", type=int, default=3)
    ap.add_argument("--shapes", default="ma7,days30,minmax,suffix")
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
