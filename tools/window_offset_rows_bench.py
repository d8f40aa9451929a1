#!/usr/bin/env python
"""Cost of an offset-window reducer on the GPU: b2s_decompress_window_offset_rows_keys_dev over a reducer's shuffled
blocks, against today's GPU path for the same blocks, one b2s_decompress_sort_rows_keys_dev call by the window's key,
which leaves the Window to the JVM.

Each reducer gets --rows rows in --maps Snappy blocks with CRC32C checksums.  Shapes:
  session : [user long, ts long, page string, tag string]: lag(ts) over (partition by user order by ts), about 2,000
            users.
  lead    : [id long, t long, status string of 20..60 bytes, tag]: lead(status) over (partition by id order by t), about
            2,000 ids: the string copy.
  ffill   : [sym long, ts long, price double, 30 % null, tag]: last(price, true) over (partition by sym order by ts rows
            between unbounded preceding and current row), about 2,000 symbols: the non-null index.
  nth     : [k long, t long, x long, tag]: nth_value(x, 2) over (partition by k order by t rows between unbounded
            preceding and unbounded following), about 2,000 groups.
  sparse  : [_, t long, x long, 99 % null, tag]: lag(x, 1) ignore nulls over (order by t), one reducer-wide partition.
Every timed reducer's output is checked against the model (tests/window_offset_model.py) before it is timed.  Per
reducer, after one untimed call of each path, each path is timed once (b2s_last_timing: kernel_ms = the whole call on
the device, dominant_ms = the window step).  The packed forms of both are called once more for their device-to-host
bytes.  The card's name and power limit are read in the same run.

    python tools/window_offset_rows_bench.py [--rows 91000] [--maps 400] [--reducers 3]
                                             [--shapes session,lead,ffill,nth,sparse]

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

INT64 = 2
FIXED, VAR = 0, 1
LAG, LEAD, LAST, NTH_VALUE = 11, 12, 14, 15
FRAME_PARTITION, FRAME_ROWS = 1, 2
VAL_INT64, VAL_FLOAT64, VAL_BYTES = 4, 6, 8
IGNORE_NULLS = 1


def set_nulls(rec, rec_len, field, null):
    """sets field's null bit (and zeroes its slot, as UnsafeRowWriter does) in the rows where null is true"""
    starts = np.concatenate([[0], np.cumsum(rec_len.astype(np.int64))[:-1]])[null]
    rec[starts + 4 + field // 8] |= np.uint8(1 << (field % 8))
    for b in range(8):
        rec[starts + 4 + 8 + 8 * field + b] = 0


def set_sizes(rec, rec_len, field, size):
    """a VAR field's slot size (its low 32 bits) in every row: its bytes stay padded to 8"""
    starts = np.concatenate([[0], np.cumsum(rec_len.astype(np.int64))[:-1]])
    for b in range(4):
        rec[starts + 4 + 8 + 8 * field + b] = ((size >> (8 * b)) & 0xFF).astype(np.uint8)


def shape_rows(rng, shape, n, groups):
    """-> ((records, lengths), keys, n_partition_keys, kinds, fns)"""
    keys = [(INT64, 8, 8, -1), (INT64, 16, 8, -1)]
    slots = np.zeros((n, 4), np.uint64)
    tag = {3: np.full(n, 8)}  # every shape's rows end with an 8-byte tag string
    slots[:, 0] = rng.integers(0, groups, n).astype(np.uint64)
    slots[:, 1] = rng.integers(1_600_000_000, 1_700_000_000, n).astype(np.uint64)
    if shape == "session":
        return (rows_of(slots, {2: 8 * rng.integers(2, 8, n), **tag}, rng), keys, 1, [FIXED, FIXED, VAR, VAR],
                [(LAG, 1, 0, VAL_INT64, 8 + 8, -1, 0, 0)])
    if shape == "lead":
        size = rng.integers(20, 61, n)
        rec, rec_len = rows_of(slots, {2: (size + 7) // 8 * 8, **tag}, rng)
        set_sizes(rec, rec_len, 2, size)
        return ((rec, rec_len), keys, 1, [FIXED, FIXED, VAR, VAR], [(LEAD, 1, 0, VAL_BYTES, 8 + 16, -1, 0, 0)])
    if shape == "ffill":
        slots[:, 2] = (rng.normal(size=n) * 100).view(np.uint64)
        rec, rec_len = rows_of(slots, tag, rng)
        set_nulls(rec, rec_len, 2, rng.random(n) < 0.3)
        return ((rec, rec_len), keys, 1, [FIXED] * 3 + [VAR],
                [(LAST, 0, FRAME_ROWS, VAL_FLOAT64, 8 + 16, 2, IGNORE_NULLS, 0)])
    if shape == "nth":
        slots[:, 2] = rng.integers(0, 1 << 40, n).astype(np.uint64)
        return (rows_of(slots, tag, rng), keys, 1, [FIXED] * 3 + [VAR],
                [(NTH_VALUE, 2, FRAME_PARTITION, VAL_INT64, 8 + 16, -1, 0, 0)])
    slots[:, 2] = rng.integers(0, 1 << 40, n).astype(np.uint64)
    rec, rec_len = rows_of(slots, tag, rng)
    set_nulls(rec, rec_len, 2, rng.random(n) >= 0.01)
    return ((rec, rec_len), keys[1:], 0, [FIXED] * 3 + [VAR], [(LAG, 1, 0, VAL_INT64, 8 + 16, 2, IGNORE_NULLS, 0)])


def run(capi, args, shape, red, d_src, d_dst, cap):
    from window_offset_model import model_window_offset
    rng = np.random.default_rng(1000 * red + len(shape))
    (rec, rec_len), keys, npk, kinds, fns = shape_rows(rng, shape, args.rows, args.groups)
    nf = len(kinds)
    plain, arena, off, ln, ck = blocks(capi, rec, rec_len, args.maps, rng)
    n = off.size
    sb, sl = np.arange(n + 1, dtype=np.uint32), ln.astype(np.uint64)
    capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
    stream, _, rows = model_window_offset(plain, keys, npk, nf, kinds, fns)

    def window():
        r = capi.decompress_window_offset_rows_keys_dev(SNAPPY, d_src, off, ln, d_dst, cap, keys, npk, nf, kinds, fns,
                                                        CRC32C, sb, sl, ck)
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
    capi.decompress_window_offset_rows_keys_packed(SNAPPY, arena, off, ln, host, keys, npk, nf, kinds, fns, CRC32C,
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
    ap.add_argument("--groups", type=int, default=2000, help="partitions per reducer (all shapes but sparse)")
    ap.add_argument("--shapes", default="session,lead,ffill,nth,sparse")
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
