"""Measure the central-moment aggregates on the GPU: B2S_WINDOW_VARIANCE in the map side's partial aggregation
(b2s_aggregate_partition_compress_rows_hash_packed) and B2S_AGG_VARIANCE in the reducer's aggregated read
(b2s_decompress_aggregate_rows_keys_packed), each against the same call with a shape of ordinary buffers in its place.
Every output is checked against tests/moments_model.py before it is timed.

Map shapes (one map task, rows of [null word][long key][int a][int b][int c], inputs null in 5 %):
  q39   : 1 M rows, 100 k keys, stddev_samp(a) + avg(a)                     against avg(a) + avg(a)
  q17   : 1 M rows, 100 k keys, count, avg, stddev_samp of a, b and c       against avg in place of each stddev
  low   : 8.4 M rows, 8 keys, stddev_samp(a)                                against avg(a) (its double add chain)
Reduce shapes (partial rows [null word][long key][n][avg][m2][count] of M maps, codec NONE):
  median: 64 maps x 20 k keys (keys drawn from 20 k, so groups of ~64)      variance triple against four ops
  skewed: the same with half of all rows on one key
The map shapes report the call's kernel time (kernel_ms) and its aggregation step (dominant_ms); the reduce shapes the
call's kernel time and its aggregation step.  min / median / max over --reps runs; the card's name and power limit are
read in the same run.  One JSON line per shape."""
import argparse
import json
import os
import statistics
import struct
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

COUNT, AVG, SUM, VAR = 7, 10, 6, 16
VAL_I32, KEY_INT64 = 3, 2
AGG_SUM_I64, AGG_SUM_F64, AGG_VAR = 0, 1, 12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def map_rows(rng, n, n_keys):
    """[null word][key][a][b][c]: 40-byte rows; a, b, c ints in [1, 100), null in 5 %"""
    key = rng.integers(0, n_keys, n).astype(np.int64)
    vals = rng.integers(1, 100, (3, n)).astype(np.int32)
    nulls = rng.random((3, n)) < 0.05
    rows = np.zeros((n, 44), np.uint8)
    rows[:, 0:4] = np.frombuffer((40).to_bytes(4, "big"), np.uint8)
    word = np.zeros(n, np.uint64)
    for j in range(3):
        word |= nulls[j].astype(np.uint64) << np.uint64(2 + j)
        rows[:, 20 + 8 * j:24 + 8 * j] = np.where(nulls[j], 0, vals[j]).view(np.uint8).reshape(n, 4)
    rows[:, 4:12] = word.view(np.uint8).reshape(n, 8)
    rows[:, 12:20] = key.view(np.uint8).reshape(n, 8)
    return rows.reshape(-1), np.full(n, 44, np.uint32), (key, vals, nulls)


def check_map(c, recs, rl, keys, aggs, cols):
    """the call with codec NONE over one partition: every group's variance buffers are the update chain's"""
    import moments_model as mm
    key, vals, nulls = cols
    dst = np.zeros(c.partition_compress_bound(0, 0, 1, recs.size * 2) + 4096, np.uint8)
    got = c.aggregate_partition_compress_rows_hash_packed(0, recs, rl, keys, aggs, 1, dst)
    buf = dst[:got["total"]].tobytes()
    order = np.argsort(key, kind="stable")
    starts = np.flatnonzero(np.r_[True, np.diff(key[order]) != 0])
    bounds = list(starts) + [len(order)]
    var_fields, f = [], 1
    for fn, _, off, _ in aggs:
        if fn == VAR:
            var_fields.append((f, (off - 16) // 8))
        f += {COUNT: 1, AVG: 2, SUM: 1, VAR: 3}[fn]
    at = 0
    for g in range(len(starts)):
        sz = int.from_bytes(buf[at:at + 4], "big")
        row = buf[at + 4:at + 4 + sz]
        at += 4 + sz
        idx = order[bounds[g]:bounds[g + 1]]
        assert struct.unpack("<q", row[8:16])[0] == key[idx[0]]
        for f, j in var_fields:
            xs = [float(v) for v, nl in zip(vals[j][idx].tolist(), nulls[j][idx].tolist()) if not nl]
            assert struct.unpack("<3d", row[8 + 8 * f:32 + 8 * f]) == mm.fold(xs), (g, f)
    assert at == len(buf) and got["n_groups"] == len(starts)


def time_map(c, recs, rl, keys, aggs, reps, R=200):
    dst = np.zeros(c.partition_compress_bound(1, 0, R, recs.size * 2) + 4096, np.uint8)
    k, d = [], []
    for _ in range(reps + 2):
        c.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, R, dst, checksum_alg=3)
        t = c.last_timing()
        k.append(t["kernel_ms"])
        d.append(t["dominant_ms"])
    return {"kernel_ms": spread(k[2:]), "aggregation_ms": spread(d[2:])}


def reduce_blocks(rng, maps, n_keys, per_map, skew):
    """maps' partial rows [null word][key][n][avg][m2][count]: 48-byte rows -> (arena, off, len, keys)"""
    blocks = []
    for _ in range(maps):
        key = rng.integers(0, n_keys, per_map).astype(np.int64)
        if skew:
            key[rng.random(per_map) < 0.5] = 0
        key.sort(kind="stable")
        rows = np.zeros((per_map, 52), np.uint8)
        rows[:, 0:4] = np.frombuffer((48).to_bytes(4, "big"), np.uint8)
        rows[:, 12:20] = key.view(np.uint8).reshape(per_map, 8)
        n = rng.integers(1, 60, per_map).astype(np.float64)
        rows[:, 20:28] = n.view(np.uint8).reshape(per_map, 8)
        rows[:, 28:36] = (rng.normal(size=per_map) * 50).view(np.uint8).reshape(per_map, 8)
        rows[:, 36:44] = (np.abs(rng.normal(size=per_map)) * 1e4).view(np.uint8).reshape(per_map, 8)
        rows[:, 44:52] = n.astype(np.int64).view(np.uint8).reshape(per_map, 8)
        blocks.append(rows.reshape(-1))
    arena = np.concatenate(blocks)
    ln = np.array([b.size for b in blocks], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    return arena, off, ln, [(KEY_INT64, 8, 8, -1)]


VAR_AGGS = [(AGG_VAR, 16, -1), (AGG_SUM_I64, 40, -1)]
FOUR_OPS = [(AGG_SUM_F64, 16, -1), (AGG_SUM_F64, 24, -1), (AGG_SUM_F64, 32, -1), (AGG_SUM_I64, 40, -1)]


def check_reduce(c, rng):
    import moments_model as mm
    for skew in (False, True):
        arena, off, ln, keys = reduce_blocks(rng, 8, 2000, 4000, skew)
        plain = [arena[int(o):int(o + n)].tobytes() for o, n in zip(off, ln)]
        want = mm.model_aggregate(plain, keys, VAR_AGGS)[0]
        dst = np.zeros(arena.size + 4096, np.uint8)
        r = c.decompress_aggregate_rows_keys_packed(0, arena, off, ln, dst, keys, VAR_AGGS)
        assert dst[:r["total"]].tobytes() == want


def time_reduce(c, arena, off, ln, keys, aggs, reps):
    dst = np.zeros(arena.size + 4096, np.uint8)
    k, d = [], []
    for _ in range(reps + 2):
        c.decompress_aggregate_rows_keys_packed(0, arena, off, ln, dst, keys, aggs)
        t = c.last_timing()
        k.append(t["kernel_ms"])
        d.append(t["dominant_ms"])
    return {"kernel_ms": spread(k[2:]), "aggregation_ms": spread(d[2:])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--shapes", default="q39,q17,low,median,skewed")
    args = ap.parse_args()
    import spark_s3_shuffle_b200 as pkg
    c = pkg.capi
    c.init(1)
    gpu = card()
    rng = np.random.default_rng(0)
    keys = [(KEY_INT64, 8, 8, -1)]
    a, b, cc = [(0, VAL_I32, 16 + 8 * j, 2 + j) for j in range(3)]
    f = lambda fn, x: (fn,) + x[1:]  # noqa: E731
    for shape in args.shapes.split(","):
        out = {"shape": shape, "gpu": gpu}
        if shape in ("q39", "q17", "low"):
            n, nk = (8_400_000, 8) if shape == "low" else (1_000_000, 100_000)
            recs, rl, cols = map_rows(rng, n, nk)
            if shape == "q39":
                var, ref = [f(VAR, a), f(AVG, a)], [f(AVG, a), f(AVG, a)]
            elif shape == "q17":
                var = [f(fn, x) for x in (a, b, cc) for fn in (COUNT, AVG, VAR)]
                ref = [f(fn, x) for x in (a, b, cc) for fn in (COUNT, AVG, AVG)]
            else:
                var, ref = [f(VAR, a)], [f(AVG, a)]
            check_map(c, recs, rl, keys, var, cols)
            out.update(rows=n, keys=nk, variance=time_map(c, recs, rl, keys, var, args.reps),
                       reference=time_map(c, recs, rl, keys, ref, args.reps))
            if shape == "low":  # the chain's cost per row: the aggregation step over the rows of the largest group
                out["ns_per_row"] = round(out["variance"]["aggregation_ms"]["median"] * 1e6 / (n / nk), 2)
        else:
            if "checked" not in main.__dict__:
                check_reduce(c, rng)
                main.checked = True
            arena, off, ln, rkeys = reduce_blocks(rng, 64, 20000, 20000, shape == "skewed")
            out.update(records=64 * 20000, variance=time_reduce(c, arena, off, ln, rkeys, VAR_AGGS, args.reps),
                       four_ops=time_reduce(c, arena, off, ln, rkeys, FOUR_OPS, args.reps))
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
