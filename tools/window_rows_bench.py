#!/usr/bin/env python
"""Cost of a ranking-window reducer on the GPU: b2s_decompress_window_rows_keys_dev over a reducer's shuffled blocks,
against today's GPU path for the same blocks, one b2s_decompress_sort_rows_keys_dev call by the window's key, which
leaves WindowGroupLimit and Window to the JVM.

Each reducer gets --rows rows in --maps Snappy blocks with CRC32C checksums.  Shapes:
  q67     : TPC-DS q67's window input, [i_category, i_class, i_brand, i_product_name, d_year, d_qoy, d_moy, s_store_id,
            sumsales decimal(28,2)], --categories categories per reducer; rank() over (partition by i_category order by
            sumsales desc nulls last) with WindowGroupLimit rank <= 100.
  dedup   : [id long, ts long, payload string]: row_number() over (partition by id order by ts desc) = 1, one row in
            four kept.
  all6    : the q67 rows, all six functions (row_number, rank, dense_rank, percent_rank, cume_dist, ntile(4)), no limit.
Every timed reducer's output is checked against the model (tests/window_model.py) before it is timed.  Per reducer,
after one untimed call of each path, each path is timed once (b2s_last_timing: kernel_ms = the whole call on the
device, dominant_ms = the window step).  The packed forms of both are called once more for their device-to-host bytes.
The card's name and power limit are read in the same run.

    python tools/window_rows_bench.py [--rows 91000] [--maps 400] [--reducers 3] [--shapes q67,dedup,all6]

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

INT64, STRING, DECIMAL = 2, 3, 9
DESC, NULLS_LAST = 1 << 8, 1 << 9
FIXED, VAR, DECIMAL_WIDE = 0, 1, 2
ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK, CUME_DIST, NTILE = range(6)


def q67_rows(rng, n, categories):
    """9 fields: 0 i_category (16-byte string), 1..3 strings, 4..6 ints, 7 string, 8 sumsales (a 16-byte decimal)"""
    slots = np.zeros((n, 9), np.uint64)
    slots[:, 4] = rng.integers(1998, 2003, n).astype(np.uint64)
    slots[:, 5] = rng.integers(1, 5, n).astype(np.uint64)
    slots[:, 6] = rng.integers(1, 13, n).astype(np.uint64)
    cat = np.frombuffer(b"".join(b"Category%08d" % c for c in rng.integers(0, categories, n)), np.uint8).reshape(n, 16)
    cents = rng.integers(0, 10**12, n)  # sumsales * 100, big-endian two's complement in 16 bytes
    dec = np.zeros((n, 16), np.uint8)
    dec[:, 8:] = cents.astype(">i8").view(np.uint8).reshape(n, 8)
    var = {0: cat, 1: 8 * rng.integers(1, 4, n), 2: 8 * rng.integers(1, 4, n), 3: 8 * rng.integers(2, 7, n),
           7: np.full(n, 16), 8: dec}
    keys = [(STRING, 8, 8, -1), (DECIMAL | DESC | NULLS_LAST, 8 + 8 * 8, 8, -1)]
    kinds = [VAR, VAR, VAR, VAR, FIXED, FIXED, FIXED, VAR, DECIMAL_WIDE]
    return rows_of(slots, var, rng), keys, kinds


def dedup_rows(rng, n):
    slots = np.zeros((n, 3), np.uint64)
    slots[:, 0] = rng.integers(0, max(n // 4, 1), n).astype(np.uint64)
    slots[:, 1] = rng.integers(0, 1 << 40, n).astype(np.uint64)
    keys = [(INT64, 8, 8, -1), (INT64 | DESC, 16, 8, -1)]
    return rows_of(slots, {2: 8 * rng.integers(1, 5, n)}, rng), keys, [FIXED, FIXED, VAR]


SHAPES = {"q67": ([RANK], (RANK, 100)), "dedup": ([ROW_NUMBER], (ROW_NUMBER, 1)),
          "all6": ([ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK, CUME_DIST, (NTILE, 4)], None)}


def run(capi, args, shape, red, d_src, d_dst, cap):
    from window_model import model_window
    rng = np.random.default_rng(1000 * red + len(shape))
    if shape == "dedup":
        (rec, rec_len), keys, kinds = dedup_rows(rng, args.rows)
    else:
        (rec, rec_len), keys, kinds = q67_rows(rng, args.rows, args.categories)
    fns, limit = SHAPES[shape]
    nf = len(kinds)
    plain, arena, off, ln, ck = blocks(capi, rec, rec_len, args.maps, rng)
    n = off.size
    sb, sl = np.arange(n + 1, dtype=np.uint32), ln.astype(np.uint64)
    capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
    stream, _, rows = model_window(plain, keys, 1, nf, kinds, fns, limit)

    def window():
        r = capi.decompress_window_rows_keys_dev(SNAPPY, d_src, off, ln, d_dst, cap, keys, 1, nf, kinds, fns, limit,
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
    capi.decompress_window_rows_keys_packed(SNAPPY, arena, off, ln, host, keys, 1, nf, kinds, fns, limit, CRC32C, sb,
                                            sl, ck)
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
    ap.add_argument("--categories", type=int, default=1, help="q67 categories per reducer")
    ap.add_argument("--shapes", default="q67,dedup,all6")
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
