"""Measure b2s_aggregate_partition_compress_rows_hash_packed (a map task's partial aggregation and hash exchange on the
GPU) against the two hash-call paths it replaces or skips: b2s_partition_compress_rows_hash_packed over the model's
partial rows (the GPU's share of today's path, where the JVM aggregates first) and over the raw rows (shuffling without
combining).  Every output is checked against the model (tests/partial_agg_model.py; vectorized with numpy for the
long-key shapes) before it is timed.

Shapes (one map task, rows of [null word][long key or string + int key][long v][double d]):
  high      : 8 M rows, 10 k long keys, decimal(7, 2) sum + count(*) + decimal(7, 2) avg
  low       : 8 M rows, 8 long keys, the same aggregates
  low_dsum  : 8 M rows, 8 long keys, the same plus a double sum (the per-group add chain)
  none      : 8 M rows, keys ~ rows / 2, the same aggregates
  composite : 1 M rows, 10 k (string, int) keys, the same aggregates (checked by the row-by-row model)
Reports min / median / max of each call's kernel time (kernel_ms) and, for the aggregating call, its aggregation step
(dominant_ms), and the .data bytes of each; the card's name and power limit read in the same run.  One JSON line per
shape."""
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

SUM, COUNT, AVG = 6, 7, 10
VAL_NONE, VAL_DEC72, VAL_F64 = 0, 7 | 7 << 8 | 2 << 16, 6
KEY_INT64, KEY_INT32, STRING = 2, 1, 3


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def long_rows(rng, n, n_keys):
    """[null word][key][v: decimal(7, 2) as a long, null in 10 %][d: double, null in 10 %]: 32-byte rows"""
    key = rng.integers(0, n_keys, n).astype(np.int64) * 7919 - 12345
    v = rng.integers(-10**7 + 1, 10**7, n).astype(np.int64)
    d = rng.normal(size=n) * 1e3
    vn, dn = rng.random(n) < 0.1, rng.random(n) < 0.1
    rows = np.zeros((n, 36), np.uint8)
    rows[:, 0:4] = np.frombuffer((32).to_bytes(4, "big"), np.uint8)
    word = vn.astype(np.uint64) << np.uint64(1) | dn.astype(np.uint64) << np.uint64(2)
    rows[:, 4:12] = word.view(np.uint8).reshape(n, 8)
    rows[:, 12:20] = key.view(np.uint8).reshape(n, 8)
    rows[:, 20:28] = np.where(vn, 0, v).view(np.uint8).reshape(n, 8)
    rows[:, 28:36] = np.where(dn, 0.0, d).view(np.uint8).reshape(n, 8)
    return rows.reshape(-1), np.full(n, 36, np.uint32), (key, v, vn, d, dn)


def long_model(cols, dsum):
    """the partial rows of the long-key shapes, vectorized: keys ascending; buffers sum(v) + isEmpty, count(*), avg(v)
    sum + count, [sum(d) in input order]"""
    key, v, vn, d, dn = cols
    order = np.argsort(key, kind="stable")
    ks = key[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    G = starts.size
    vv = np.where(vn, 0, v)[order]
    cnt_nn = np.add.reduceat((~vn[order]).astype(np.int64), starts)
    sums = np.add.reduceat(vv, starts)
    size = np.diff(np.r_[starts, ks.size])
    nb = 6 if dsum else 5
    nf = 1 + nb
    rb = 8 + 8 * nf
    out = np.zeros((G, 4 + rb), np.uint8)
    out[:, 0:4] = np.frombuffer(rb.to_bytes(4, "big"), np.uint8)
    cols_out = [ks[starts], sums, (cnt_nn == 0).astype(np.int64), size.astype(np.int64), sums, cnt_nn]
    if dsum:
        dd = np.where(dn, 0.0, d)[order]
        ds = np.empty(G)
        bounds = np.r_[starts, ks.size]
        for g in range(G):  # one add chain per group, in input order, from +0.0
            ds[g] = np.cumsum(np.r_[0.0, dd[bounds[g]:bounds[g + 1]]])[-1]
        cols_out.append(ds.view(np.int64))
    for f, c in enumerate(cols_out):
        out[:, 12 + 8 * f:20 + 8 * f] = np.ascontiguousarray(c, dtype=np.int64).view(np.uint8).reshape(G, 8)
    return out.reshape(-1), np.full(G, 4 + rb, np.uint32)


def composite_rows(rng, n, n_keys):
    import hash_model as hm
    types = ["string", "int", "long", "double"]
    pool = [(bytes(rng.integers(97, 123, int(rng.integers(4, 24)), dtype=np.uint8)), int(rng.integers(0, 1000)))
            for _ in range(n_keys)]
    picks = rng.integers(0, n_keys, n)
    rows = []
    for p in picks:
        s, i = pool[p]
        rows.append(hm.make_row(types, [s, i, int(rng.integers(-10**7 + 1, 10**7)) if rng.random() > 0.1 else None,
                                        float(rng.normal()) if rng.random() > 0.1 else None]))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=8 << 20)
    ap.add_argument("--composite-rows", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--partitions", type=int, default=200)
    ap.add_argument("--codec", type=int, default=1)
    ap.add_argument("--shapes", default="high,low,low_dsum,none,composite")
    a = ap.parse_args()
    import hash_model as hm
    import partial_agg_model as pm
    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    info = card()
    rng = np.random.default_rng(7)
    R, codec = a.partitions, a.codec
    for shape in a.shapes.split(","):
        dsum = shape == "low_dsum"
        if shape == "composite":
            rows = composite_rows(rng, a.composite_rows, 10_000)
            keys = [(STRING, 8, 8, 0), (KEY_INT32, 16, 4, 1)]
            aggs = [(SUM, VAL_DEC72, 24, 2), (COUNT, VAL_NONE, 0, -1), (AVG, VAL_DEC72, 24, 2)]
            recs, rl = hm.records_of(rows)
            prec, prl = hm.records_of(pm.partial_rows(rows, keys, aggs))
        else:
            n_keys = {"high": 10_000, "low": 8, "low_dsum": 8, "none": a.rows // 2}[shape]
            recs, rl, cols = long_rows(rng, a.rows, n_keys)
            keys = [(KEY_INT64, 8, 8, -1)]
            aggs = [(SUM, VAL_DEC72, 16, 1), (COUNT, VAL_NONE, 0, -1), (AVG, VAL_DEC72, 16, 1)]
            if dsum:
                aggs.append((SUM, VAL_F64, 24, 2))
            prec, prl = long_model(cols, dsum)
        okeys = pm.output_keys(keys)
        cap = c.partition_compress_bound(codec, 0, R, max(recs.size, prec.size)) + 64
        ref_dst, got_dst, raw_dst = (np.zeros(cap, np.uint8) for _ in range(3))
        ref = c.partition_compress_rows_hash_packed(codec, prec, prl, okeys, R, ref_dst)
        got = c.aggregate_partition_compress_rows_hash_packed(codec, recs, rl, keys, aggs, R, got_dst)
        assert got["n_groups"] == prl.size, shape
        assert got["total"] == ref["total"] and np.array_equal(got_dst[:ref["total"]], ref_dst[:ref["total"]]), shape
        for k in ("dst_off", "dst_len", "checksums", "status"):
            assert np.array_equal(got[k], ref[k]), (shape, k)
        agg_k, agg_dom, part_k, raw_k = [], [], [], []
        raw = None
        for rep in range(a.reps + 2):
            c.aggregate_partition_compress_rows_hash_packed(codec, recs, rl, keys, aggs, R, got_dst)
            t = c.last_timing()
            c.partition_compress_rows_hash_packed(codec, prec, prl, okeys, R, ref_dst)
            tp = c.last_timing()
            raw = c.partition_compress_rows_hash_packed(codec, recs, rl, keys, R, raw_dst)
            tr = c.last_timing()
            if rep >= 2:  # two warm-up rounds
                agg_k.append(t["kernel_ms"])
                agg_dom.append(t["dominant_ms"])
                part_k.append(tp["kernel_ms"])
                raw_k.append(tr["kernel_ms"])
        print(json.dumps({"shape": shape, "card": info, "rows": int(rl.size), "groups": int(prl.size),
                          "partitions": R, "codec": codec,
                          "aggregate_call_kernel_ms": spread(agg_k), "aggregation_step_ms": spread(agg_dom),
                          "hash_over_partial_rows_kernel_ms": spread(part_k), "hash_over_raw_rows_kernel_ms":
                          spread(raw_k), "data_bytes": {"aggregate_call": got["total"],
                                                        "hash_over_partial_rows": ref["total"],
                                                        "hash_over_raw_rows": raw["total"]}}), flush=True)


if __name__ == "__main__":
    main()
