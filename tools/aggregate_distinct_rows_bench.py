"""Measure one DISTINCT group's middle stage on the GPU: b2s_decompress_aggregate_distinct_partition_compress_rows_hash_dev
per reducer, against today's path in the same run: the aggregated read by G ++ X
(b2s_decompress_aggregate_rows_keys_dev) plus b2s_partition_compress_rows_hash_dev over its rows (the JVM's stage 3
is not timed, so today's path is a lower bound).  The call's output is checked against tests/distinct_agg_model.py on a
small reducer of each shape before anything is timed.

Shapes (one reducer: M maps' partial rows for keys G ++ X, LZ4 blocks with CRC32C, in device memory):
  q16    : a global count(DISTINCT order) beside two sum(decimal(7, 2)): 1 M orders, no G, SinglePartition
  grouped: count(DISTINCT user) GROUP BY day beside count(*): 365 days x 20 k users, 1 M partial rows, R = 200
  skewed : the grouped shape with half of the partial rows on one day
Reported per shape: the call's kernel time (kernel_ms) and its stage 3 (dominant_ms), and today's path's kernel time
(read + hash call), min / median / max over --reps runs after two warm-up runs.  The card's name and power limit are
read in the same run.  One JSON line per shape."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COUNT, SUM = 7, 6
VAL_NONE, VAL_INT64 = 0, 4
KEY_INT64 = 2
AGG_SUM_I64, AGG_MIN_I32, AGG_SUM_DEC = 0, 2, 9
ALL = -1


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def dec7():
    return 7 | 7 << 8 | 2 << 16  # VAL_DECIMAL (7) | p 7 << 8 | s 2 << 16


def partial_rows(cols):
    """fixed-width partial rows, no nulls: [null word][8-byte fields...] framed as records -> (records, row length)"""
    n, w = cols[0].size, len(cols)
    rows = np.zeros((n, 4 + 8 + 8 * w), np.uint8)
    rows[:, 0:4] = np.frombuffer((8 + 8 * w).to_bytes(4, "big"), np.uint8)
    for j, c in enumerate(cols):
        rows[:, 12 + 8 * j:20 + 8 * j] = c.astype(np.int64).view(np.uint8).reshape(n, 8)
    return rows, 8 + 8 * w


def shape(name, rng, M, n):
    """-> (per-map records, n_group_keys, keys, aggs, distinct, R, the aggregated read's merge entries)"""
    if name == "q16":
        order = rng.permutation(n)
        s1, s2 = order % 1000, order % 97
        cols = [order, s1, np.zeros(n), s2, np.zeros(n)]  # [order, sum, isEmpty, sum, isEmpty]
        rows, _ = partial_rows(cols)
        keys, aggs, distinct, ng, R = [(KEY_INT64, 8)], [(SUM, dec7()), (SUM, dec7())], [(COUNT, VAL_INT64, 0)], 0, 1
        merge = [(AGG_SUM_DEC | 17 << 8, 16, 1), (AGG_MIN_I32, 24, 2), (AGG_SUM_DEC | 17 << 8, 32, 3),
                 (AGG_MIN_I32, 40, 4)]
    else:
        day = rng.integers(0, 365, n)
        if name == "skewed":
            day[: n // 2] = 7
        user = rng.integers(0, 20000, n)
        rows, _ = partial_rows([day, user, rng.integers(1, 5, n)])  # [day, user, count]
        keys, aggs, distinct, ng, R = [(KEY_INT64, 8)] * 2, [(COUNT, VAL_NONE)], [(COUNT, VAL_INT64, 1)], 1, 200
        merge = [(AGG_SUM_I64, 24, 2)]
    rng.shuffle(rows)
    maps = [rows[m::M].reshape(-1).tobytes() for m in range(M)]
    return maps, ng, keys, aggs, distinct, R, merge


def check(c, rng, name):
    """the call on a small reducer of the shape == the model's rows through the partition call"""
    import distinct_agg_model as da
    import rows_model as rm
    maps, ng, keys, aggs, distinct, R, _ = shape(name, rng, 4, 3000)
    want, counts = da.reducer(maps, ng, keys, aggs, distinct)
    import hash_model as hm
    prec, prl = hm.records_of(want)
    arena, off, ln, sb, sl, ck = rm.build_blocks(c, 1, 1, 3, maps)
    cap = c.partition_compress_bound(1, 0, R, prec.size) + 64
    got_dst, ref_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    got = c.aggregate_distinct_partition_compress_rows_hash(1, arena, off, ln, got_dst, ng, keys, aggs, distinct, R,
                                                            checksum_alg=3, slice_base=sb, slice_len=sl,
                                                            slice_checksum=ck)
    if ng:
        ref = c.partition_compress_rows_hash_packed(1, prec, prl, da.input_keys(keys)[:ng], R, ref_dst, checksum_alg=3)
    else:
        ref = c.partition_compress_packed(1, prec, prl, np.zeros(prl.size, np.uint32), 1, ref_dst, checksum_alg=3)
    assert got["counts"] == counts and got["total"] == ref["total"]
    assert np.array_equal(got_dst[:ref["total"]], ref_dst[:ref["total"]]), name


def run(c, name, M, n, reps):
    import rows_model as rm
    rng = np.random.default_rng(1)
    check(c, rng, name)
    maps, ng, keys, aggs, distinct, R, merge = shape(name, rng, M, n)
    arena, off, ln, sb, sl, ck = rm.build_blocks(c, 1, 1, 3, maps)
    slices = dict(checksum_alg=3, slice_base=sb, slice_len=sl, slice_checksum=ck)
    raw = sum(len(m) for m in maps)
    cap = c.partition_compress_bound(1, 0, R, raw) + (1 << 20)
    d_src, d_dst, d_rows = c.dev_alloc(arena.size), c.dev_alloc(cap), c.dev_alloc(raw + 64)
    row_len = 4 + int.from_bytes(maps[0][:4], "big")  # every record of a shape, merged or not, has one length
    d_len = c.dev_alloc(4 * (raw // row_len + 1))
    try:
        c.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        lens = np.full(raw // row_len + 1, row_len, np.uint32)
        c.dev_memcpy(d_len, lens.ctypes.data, lens.nbytes, 1)
        call_k, call_s3, today_k = [], [], []
        hkeys = [(KEY_INT64, 8 + 8 * k, 8, k) for k in range(max(ng, 1))]
        for _ in range(reps + 2):
            r = c.aggregate_distinct_partition_compress_rows_hash(1, d_src, off, ln, d_dst, ng, keys, aggs, distinct,
                                                                  R, dev=0, dst_cap=cap, **slices)
            t = c.last_timing()
            call_k.append(t["kernel_ms"])
            call_s3.append(t["dominant_ms"])
            a = c.decompress_aggregate_rows_keys_dev(1, d_src, off, ln, d_rows, raw + 64,
                                                     [(KEY_INT64, 8 + 8 * k, 8, k) for k in range(len(keys))], merge,
                                                     **slices)
            k_read = c.last_timing()["kernel_ms"]
            c.partition_compress_rows_hash_dev(1, d_rows, a["total"], d_len, a["n_groups"], hkeys, R, d_dst, cap,
                                               checksum_alg=3)
            today_k.append(k_read + c.last_timing()["kernel_ms"])
        return {"shape": name, "card": card(), "maps": M, "partial_rows": r["counts"][0], "gx_groups": r["counts"][1],
                "rows_written": r["counts"][2], "call_kernel_ms": spread(call_k[2:]),
                "call_stage3_ms": spread(call_s3[2:]), "today_read_plus_hash_kernel_ms": spread(today_k[2:])}
    finally:
        for p in (d_src, d_dst, d_rows, d_len):
            c.dev_free(p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="q16,grouped,skewed")
    ap.add_argument("--maps", type=int, default=64)
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import spark_s3_shuffle_b200 as pkg
    c = pkg.capi
    c.init(1)
    for name in args.shapes.split(","):
        print(json.dumps(run(c, name, args.maps, args.rows, args.reps)), flush=True)


if __name__ == "__main__":
    main()
