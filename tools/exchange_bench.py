#!/usr/bin/env python
"""What a reducer saves when its map outputs are resident in the exchange cache (b2s_exchange_read_sort_*), against
fetching, verifying and decoding the same maps' blocks (b2s_decompress_sort_*).

Workload: tools/sort_bench.py's — --gib GiB of device-generated TeraSort records (gen_terasort_dev, seed 42; 104-byte
records, 10-byte key at byte 2) split into --maps map tasks, reduce ids from the key range (the first two key bytes
scaled to --partitions), LZ4 + CRC32C.  Each map task's records are copied to pinned host memory and go through
partition_compress_packed and then partition_compress_cached_packed (the store: the same outputs, and the partitioned
records kept in HBM); the difference of the two calls' times is the store's extra cost.  Every map output is resident
(the budget holds them all).  After --warmup untimed calls on reducer 0, every reducer is timed once per path:
  fetched  decompress_sort_dev over its M device-resident blocks (verify + decode + sort)
  cached   exchange_read_sort_dev over its M cached sources (gather + sort)
and the packed forms, which move the blocks from and the records to host memory:
  fetched  decompress_sort_packed (H2D of the compressed blocks, D2H of the sorted records)
  cached   exchange_read_sort_packed (D2H of the sorted records only)
Per path: min / median / max over the reducers of kernel_ms and top_kernel_ms (the sort step) and their sums, and for
the packed forms total_ms and the H2D / D2H bytes.  The sorted records of the two paths must be byte-identical for every
reducer.  The card's name and power limit are read in the same run.

    python tools/exchange_bench.py [--gib 10] [--maps 16] [--partitions 200] [--warmup 2]

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

RECORD, KEY_OFF, KEY_LEN = 104, 2, 10
SHUFFLE = 0


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3),
            "sum": round(sum(xs), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--maps", type=int, default=16)
    ap.add_argument("--partitions", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch

    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    M, R = args.maps, args.partitions
    n = int(args.gib * (1 << 30)) // RECORD
    dev = torch.device("cuda", 0)
    per = [n // M // 2 * 2] * (M - 1)
    per.append(n - sum(per))
    first = [sum(per[:m]) for m in range(M)]
    c.exchange_set_budget(n * RECORD + (1 << 30))

    # map side: each map task through the plain and the cached store, from pinned host memory
    biggest = max(per)
    h_rec = c.HostBuffer(biggest * RECORD)
    bound = c.partition_compress_bound(c.CODEC_LZ4BLOCK, 0, R, biggest * RECORD) + 64
    h_dst = c.HostBuffer(bound)
    rec_len = np.full(biggest, RECORD, np.uint32)
    data, maps, store_plain, store_cached = [], [], [], []
    for m in range(M):
        rec = torch.empty(per[m] * RECORD, dtype=torch.uint8, device=dev)
        c.gen_terasort_dev(rec.data_ptr(), first[m], per[m], 42)
        rv = rec.view(per[m], RECORD)
        key = rv[:, 2:4].to(torch.int64)
        part = (((key[:, 0] << 8) | key[:, 1]) * R >> 16).to(torch.int32).cpu().numpy().view(np.uint32)
        torch.cuda.synchronize()
        h_rec.array[: per[m] * RECORD] = rec.cpu().numpy()
        del rec, rv, key
        src = h_rec.array[: per[m] * RECORD]
        for _ in range(2 if m == 0 else 1):  # the first map's calls once untimed: they grow the library's buffers
            r = c.partition_compress_packed(c.CODEC_LZ4BLOCK, src, rec_len[: per[m]], part, R, h_dst.array, 0,
                                            c.CHECKSUM_CRC32C)
            t_plain = c.last_timing()["total_ms"]
            plain = h_dst.array[: r["total"]].copy()
            q = c.partition_compress_cached_packed(SHUFFLE, m, c.CODEC_LZ4BLOCK, src, rec_len[: per[m]], part, R,
                                                   h_dst.array, 0, c.CHECKSUM_CRC32C)
            t_cached = c.last_timing()["total_ms"]
        store_plain.append(t_plain)
        store_cached.append(t_cached)
        assert q["cached"] == 1 and not q["status"].any()
        assert np.array_equal(h_dst.array[: q["total"]], plain) and np.array_equal(q["dst_len"], r["dst_len"])
        data.append(plain)
        maps.append(q)
    torch.cuda.empty_cache()

    # the fetched path's blocks: every map's .data arena, device-resident, map m at map_base[m]
    map_base = [sum((len(d) + 255) // 256 * 256 for d in data[:m]) for m in range(M)]
    compressed = torch.empty(map_base[-1] + len(data[-1]) + 256, dtype=torch.uint8, device=dev)
    for m in range(M):
        compressed[map_base[m]:map_base[m] + len(data[m])] = torch.from_numpy(data[m]).to(dev)
    torch.cuda.synchronize()

    def blocks(red, host=False):
        off = [(0 if host else map_base[m]) + int(maps[m]["dst_off"][red]) for m in range(M)]
        ln = [int(maps[m]["dst_len"][red]) for m in range(M)]
        ck = [int(maps[m]["checksums"][red]) for m in range(M)]
        return off, ln, list(range(M + 1)), ln, ck

    cap = max(sum(int(q["dst_len"][red]) for q in maps) for red in range(R)) * 8 + (1 << 20)
    out_a = torch.empty(cap, dtype=torch.uint8, device=dev)
    out_b = torch.empty(cap, dtype=torch.uint8, device=dev)
    ids, hit = list(range(M)), [True] * M
    zeros = [0] * M
    h_src = c.HostBuffer(max(sum(int(q["dst_len"][red]) for q in maps) for red in range(R)) + 64)
    h_out_a, h_out_b = c.HostBuffer(cap), c.HostBuffer(cap)

    def dev_fetched(red):
        off, ln, sb, sl, ck = blocks(red)
        return c.decompress_sort_dev(c.CODEC_LZ4BLOCK, compressed.data_ptr(), off, ln, out_a.data_ptr(), cap, RECORD,
                                     KEY_OFF, KEY_LEN, c.CHECKSUM_CRC32C, sb, sl, ck)

    def dev_cached(red):
        return c.exchange_read_sort_dev(SHUFFLE, red, red + 1, ids, hit, c.CODEC_LZ4BLOCK, compressed.data_ptr(),
                                        zeros, zeros, out_b.data_ptr(), cap, RECORD, KEY_OFF, KEY_LEN,
                                        c.CHECKSUM_CRC32C, [0] * (M + 1), [], [])

    def packed_fetched(red):
        _, ln, sb, sl, ck = blocks(red)
        off, at = [], 0
        for m in range(M):
            lo = int(maps[m]["dst_off"][red])
            h_src.array[at:at + ln[m]] = data[m][lo:lo + ln[m]]
            off.append(at)
            at += ln[m]
        return c.decompress_sort_packed(c.CODEC_LZ4BLOCK, h_src.array, off, ln, h_out_a.array, RECORD, KEY_OFF,
                                        KEY_LEN, c.CHECKSUM_CRC32C, sb, sl, ck)

    def packed_cached(red):
        return c.exchange_read_sort_packed(SHUFFLE, red, red + 1, ids, hit, c.CODEC_LZ4BLOCK, h_src.array, zeros,
                                           zeros, h_out_b.array, RECORD, KEY_OFF, KEY_LEN, c.CHECKSUM_CRC32C,
                                           [0] * (M + 1), [], [])

    for _ in range(args.warmup):
        for f in (dev_fetched, dev_cached, packed_fetched, packed_cached):
            f(0)
    rows = {k: {"kernel_ms": [], "top_kernel_ms": [], "total_ms": [], "h2d_bytes": [], "d2h_bytes": []}
            for k in ("dev_fetched", "dev_cached", "packed_fetched", "packed_cached")}
    identical = True
    for red in range(R):
        for name, f in (("dev_fetched", dev_fetched), ("dev_cached", dev_cached), ("packed_fetched", packed_fetched),
                        ("packed_cached", packed_cached)):
            r = f(red)
            t = c.last_timing()
            assert not r["status"].any() and r["n_records"] * RECORD == r["total"], (name, red)
            for k in rows[name]:
                rows[name][k].append(t[k])
            if name == "dev_fetched":
                total = r["total"]
            else:
                identical &= r["total"] == total
        identical &= bool(torch.equal(out_a[:total], out_b[:total]))
        identical &= bool(np.array_equal(h_out_a.array[:total], h_out_b.array[:total]))
        identical &= bool(np.array_equal(h_out_a.array[:total], out_a[:total].cpu().numpy()))

    result = {
        "card": card(), "records": n, "record_bytes": n * RECORD, "maps": M, "partitions": R,
        "compressed_bytes": sum(len(d) for d in data),
        "store_ms_per_map": {"partition_compress_packed": spread(store_plain),
                             "partition_compress_cached_packed": spread(store_cached),
                             "extra": spread([b - a for a, b in zip(store_plain, store_cached)])},
        "outputs_identical": identical,
    }
    for name, cols in rows.items():
        result[name] = {"kernel_ms": spread(cols["kernel_ms"]), "top_kernel_ms": spread(cols["top_kernel_ms"])}
        if name.startswith("packed"):
            result[name].update({"total_ms": spread(cols["total_ms"]), "h2d_bytes": sum(cols["h2d_bytes"]),
                                 "d2h_bytes": sum(cols["d2h_bytes"])})
    print(json.dumps(result, indent=1))
    c.exchange_set_budget(0)
    c.shutdown()


if __name__ == "__main__":
    main()
