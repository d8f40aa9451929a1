#!/usr/bin/env python
"""Cost of a co-located reducer's composite-key row sort and aggregation served from the exchange cache
(b2s_exchange_read_sort_rows_keys_dev / b2s_exchange_read_aggregate_rows_keys_dev), against the same read over fetched
blocks, and against the same cached read over entries without record boundaries (walked instead of marked).

Workloads, --gib GiB of rows over --maps map tasks and --partitions reducers (one .data block per map and reducer:
snappy + CRC32C, as the fetched path reads them):
  join : a sort-merge join's build side, 56-byte rows: a nullable INT64 key (5 % null), an int, a 24-byte string
  q67  : q67-like partial-aggregate rows, 96 bytes: two 24-byte strings with long shared prefixes and an int (the key;
         it refines), then a long sum and a count
Every map deals its rows round-robin (b2s_partition_compress_rows_round_robin_cached_packed, no sort), which stores the
entry with record boundaries; the same partitioned rows go through the id-taking cached store (ids (k + 1) mod R) into
a second shuffle, whose entries keep no boundaries.  Both .data arenas are byte-identical, so the three paths read the
same bytes.  Per timed reducer (--reducers of them), after one untimed call of each path, each path is timed once
(b2s_last_timing: kernel_ms = the whole call on the device, dominant_ms = framing for the sort) and the outputs must be
byte-identical.  The store's extra cost is its total_ms against the uncached round-robin call on each map.
The card's name and power limit are read in the same run.

    python tools/exchange_rows_bench.py [--gib 2] [--maps 16] [--partitions 200] [--reducers 8]

Prints one JSON document.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SNAPPY, CRC32C = 2, 3


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def framed(rows):
    """fixed-size rows (n, size) -> records with their big-endian size prefix, back to back"""
    n, size = rows.shape
    out = np.empty((n, 4 + size), np.uint8)
    out[:, :4] = np.frombuffer(size.to_bytes(4, "big"), np.uint8)
    out[:, 4:] = rows
    return out.reshape(-1), np.full(n, 4 + size, np.uint32)


def slot(off, size, n):
    return np.full(n, (off << 32) | size, "<u8").view(np.uint8).reshape(n, 8)


def join_rows(rng, n):
    rows = np.zeros((n, 56), np.uint8)
    null = rng.random(n) < 0.05
    rows[:, 0] = null
    key = np.where(null, 0, rng.integers(-(1 << 40), 1 << 40, n))
    rows[:, 8:16] = key.astype("<i8").view(np.uint8).reshape(n, 8)
    rows[:, 16:20] = rng.integers(-1000, 1000, n).astype("<i4").view(np.uint8).reshape(n, 4)
    rows[:, 24:32] = slot(32, 24, n)
    rows[:, 32:56] = rng.integers(97, 123, (n, 24), dtype=np.uint8)
    return rows


def q67_rows(rng, n, groups=20000):
    rows = np.zeros((n, 96), np.uint8)
    g = rng.integers(0, groups, n)
    a = np.frombuffer(b"Electronics and more/abc", np.uint8)
    b = np.frombuffer(b"AAAAAAAAAAAAAAAAAAAAAAAA", np.uint8)
    rows[:, 8:16] = slot(48, 24, n)
    rows[:, 16:24] = slot(72, 24, n)
    rows[:, 24:28] = (g % 7).astype("<i4").view(np.uint8).reshape(n, 4)
    rows[:, 32:40] = rng.integers(-10**9, 10**9, n).astype("<i8").view(np.uint8).reshape(n, 8)
    rows[:, 40:48] = np.ones(n, "<i8").view(np.uint8).reshape(n, 8)
    rows[:, 48:72] = a
    rows[:, 72:96] = b
    rows[:, 69:72] = (48 + np.stack([g // 100 % 10, g // 10 % 10, g % 10], 1)).astype(np.uint8)
    rows[:, 93:96] = (48 + np.stack([g // 1000 % 10, g // 10000 % 10, g % 7], 1)).astype(np.uint8)
    return rows


def timed(c, fn, *args, **kw):
    r = fn(*args, **kw)
    t = c.last_timing()
    return r, t["kernel_ms"], t["dominant_ms"], t["total_ms"]


def run_shape(c, name, make, keys, aggs, args):
    R, M = args.partitions, args.maps
    row_bytes = make(np.random.default_rng(0), 1).shape[1] + 4
    per_map = int(args.gib * (1 << 30) / row_bytes / M)
    with_b, without_b = {"join": (101, 102), "q67": (103, 104)}[name]
    datas, cks, store_ms, plain_ms = [], [], [], []
    plain_len = np.zeros((M, R), np.uint64)
    for m in range(M):
        rec, rl = framed(make(np.random.default_rng(100 + m), per_map))
        dst = np.zeros(c.partition_compress_bound(SNAPPY, 0, R, rec.size) + 64, np.uint8)
        start = m % R
        _, _, _, t_plain = timed(c, c.partition_compress_rows_round_robin_packed, SNAPPY, rec, rl, R, start, 0, dst,
                                 0, CRC32C)
        r, _, _, t_store = timed(c, c.partition_compress_rows_round_robin_cached_packed, with_b, m, SNAPPY, rec, rl, R,
                                 start, 0, dst, 0, CRC32C)
        assert r["cached"] == 1
        ids = ((start + 1 + np.arange(per_map)) % R).astype(np.uint32)
        dst2 = np.zeros_like(dst)
        q = c.partition_compress_cached_packed(without_b, m, SNAPPY, rec, rl, ids, R, dst2, 0, CRC32C)
        assert q["cached"] == 1 and q["total"] == r["total"] and bytes(dst2[: q["total"]]) == bytes(dst[: r["total"]])
        datas.append((dst[: r["total"]].copy(), r["dst_off"].copy(), r["dst_len"].copy()))
        cks.append(r["checksums"].copy())
        store_ms.append(t_store)
        plain_ms.append(t_plain)
        for p in range(R):
            plain_len[m, p] = c.exchange_lookup(with_b, p, p + 1, [m])[1][0]
    out = {"rows_per_map": per_map, "row_bytes": row_bytes,
           "store_total_ms": spread(store_ms), "uncached_total_ms": spread(plain_ms),
           "store_extra_ms_median": round(statistics.median(s - p for s, p in zip(store_ms, plain_ms)), 3)}
    reads = [("sort", "sort_rows_keys", (keys,))] + ([("aggregate", "aggregate_rows_keys", (keys, aggs))] if aggs else [])
    for label, fn, extra in reads:
        res = {k: {"kernel_ms": [], "dominant_ms": []} for k in ("fetched", "marked", "walked")}
        for red in range(min(args.reducers, R)):
            blocks = [d[int(o[red]):int(o[red] + ln[red])] for d, o, ln in datas]
            lens = np.array([b.size for b in blocks], np.uint64)
            arena = np.concatenate(blocks + [np.zeros(1, np.uint8)])
            off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
            ck = np.array([k[red] for k in cks], np.uint64)
            sb = np.arange(M + 1, dtype=np.uint32)
            cap = int(plain_len[:, red].sum()) + 4096
            d_src, d_dst = c.dev_alloc(arena.size), c.dev_alloc(cap)
            c.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
            ids = list(range(M))
            paths = {
                "fetched": lambda: getattr(c, "decompress_" + fn + "_dev")(SNAPPY, d_src, off, lens, d_dst, cap,
                                                                           *extra, CRC32C, sb, lens, ck),
                "marked": lambda: getattr(c, "exchange_read_" + fn + "_dev")(with_b, red, red + 1, ids, [1] * M,
                                                                             SNAPPY, d_src, off, lens, d_dst, cap,
                                                                             *extra, CRC32C, sb, lens, ck),
                "walked": lambda: getattr(c, "exchange_read_" + fn + "_dev")(without_b, red, red + 1, ids, [1] * M,
                                                                             SNAPPY, d_src, off, lens, d_dst, cap,
                                                                             *extra, CRC32C, sb, lens, ck),
            }
            outs = {}
            for k, f in paths.items():
                f()  # warm-up
                r, kms, dms, _ = timed(c, f)
                assert (r["status"] == 0).all(), (k, r["status"])
                buf = np.zeros(max(r["total"], 1), np.uint8)
                c.dev_memcpy(buf.ctypes.data, d_dst, r["total"], 2)
                outs[k] = (bytes(buf[: r["total"]]), r["n_records"], r.get("n_groups"))
                res[k]["kernel_ms"].append(kms)
                res[k]["dominant_ms"].append(dms)
            assert outs["fetched"] == outs["marked"] == outs["walked"], (label, red)
            c.dev_free(d_src)
            c.dev_free(d_dst)
        out[label] = {k: {m: spread(v) for m, v in d.items()} for k, d in res.items()}
        out[label]["records_per_reducer"] = int(outs["fetched"][1])
    c.exchange_remove(with_b, -1)
    c.exchange_remove(without_b, -1)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--gib", type=float, default=2.0)
    ap.add_argument("--maps", type=int, default=16)
    ap.add_argument("--partitions", type=int, default=200)
    ap.add_argument("--reducers", type=int, default=8)
    ap.add_argument("--shapes", default="join,q67")
    args = ap.parse_args()
    import spark_s3_shuffle_b200 as pkg
    c = pkg.capi
    c.init(1)
    c.exchange_set_budget(int(args.gib * 3 * (1 << 30)) + (1 << 30))
    doc = {"card": card(), "gib": args.gib, "maps": args.maps, "partitions": args.partitions}
    shapes = {"join": (join_rows, [(c.KEY_INT64, 8, 8, 0)], None),
              "q67": (q67_rows, [(c.STRING_KEY, 8, 8, 0), (c.STRING_KEY, 16, 8, 1), (c.KEY_INT32, 24, 4, 2)],
                      [(c.AGG_SUM_INT64, 32, 3), (c.AGG_SUM_INT64, 40, 4)])}
    for s in args.shapes.split(","):
        make, keys, aggs = shapes[s]
        doc[s] = run_shape(c, s, make, keys, aggs, args)
    c.exchange_set_budget(0)
    print(json.dumps(doc))


if __name__ == "__main__":
    main()
