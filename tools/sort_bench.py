#!/usr/bin/env python
"""Cost of key-sorting a reduce task's records on the GPU (b2s_decompress_sort_dev), against decoding the same blocks.

Input: --gib GiB of device-generated TeraSort records (gen_terasort_dev, seed 42; 104-byte records, 10-byte key at
byte 2), split into --maps map tasks.  Each map task goes through partition_compress_dev (LZ4 + CRC32C) with reduce
ids from the key range (the first two key bytes scaled to --partitions), as in tools/partition_bench.py.  One GPU,
everything device-resident.  After --warmup untimed calls, every reducer's M blocks are timed two ways:
  (a) decompress_dev alone (verify + decode)
  (b) decompress_sort_dev (verify + decode + key sort)
Times are CUDA events on the library's stream (b2s_mark), per call; the sort step is (b)'s top_kernel_ms.  min /
median / max over the reducers and the sums over all reducers are printed.  The sort step's algorithmic bytes are
computed here: every record read once and written once, every key read once, and 8 B of (key word, index) pairs read
and 8 B written per radix pass (one pass per key byte); its rate is those bytes over the sort step's time and its share
of peak that rate over the 3.35 TB/s HBM3 of the H100 SXM data sheet.  TeraValidate: the concatenated outputs of (b)
over the reducers in order must have non-decreasing keys, and the record count and an order-independent digest must
equal the input's.  The card's name and power limit are read in the same run.

    python tools/sort_bench.py [--gib 10] [--maps 16] [--partitions 200] [--warmup 2]

Prints one JSON document.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RECORD, KEY_OFF, KEY_LEN = 104, 2, 10
HBM_PEAK = 3.35e12  # H100 SXM data sheet


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def digest(torch, recs):
    """order-independent digest of (n, 104) uint8 records: the wrapping sum of a per-record mix of its 13 words"""
    total = torch.zeros((), dtype=torch.int64, device=recs.device)
    k = torch.tensor([j * 0x9E3779B97F4A7C15 % (1 << 61) for j in range(1, 14)], dtype=torch.int64, device=recs.device)
    for i in range(0, recs.shape[0], 1 << 22):
        w = recs[i:i + (1 << 22)].contiguous().view(torch.int64) + k
        w = (w ^ (w >> 31)) * 0x5851F42D4C957F2D
        w = (w ^ (w >> 29)) * 0x14057B7EF767814F
        total += (w ^ (w >> 32)).sum(dim=1).sum()
    return int(total)


def key_parts(torch, recs):
    """the 10-byte keys as (first 6 bytes, last 4 bytes) big-endian int64 pairs"""
    b = recs[:, KEY_OFF:KEY_OFF + KEY_LEN].to(torch.int64)
    hi = torch.zeros(recs.shape[0], dtype=torch.int64, device=recs.device)
    for j in range(6):
        hi = (hi << 8) | b[:, j]
    lo = torch.zeros_like(hi)
    for j in range(6, 10):
        lo = (lo << 8) | b[:, j]
    return hi, lo


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
    records = torch.empty(n * RECORD, dtype=torch.uint8, device=dev)
    c.gen_terasort_dev(records.data_ptr(), 0, n, 42)
    rv = records.view(n, RECORD)
    in_digest = digest(torch, rv)

    # map side: M map tasks, partitioned + compressed by key range into one arena (map m at map_base[m])
    # an even record count per map keeps every map's records 16-byte aligned (2 x 104 = 13 x 16), and every map's
    # output starts on a 256-byte boundary, as the library's own allocations do
    per = [n // M // 2 * 2] * (M - 1)
    per.append(n - sum(per))
    first = [sum(per[:m]) for m in range(M)]
    bounds = [(c.partition_compress_bound(c.CODEC_LZ4BLOCK, 0, R, per[m] * RECORD) + 255) // 256 * 256
              for m in range(M)]
    map_base = [sum(bounds[:m]) for m in range(M)]
    compressed = torch.empty(sum(bounds), dtype=torch.uint8, device=dev)
    maps = []
    for m in range(M):
        rec = rv[first[m]:first[m] + per[m]]
        key = rec[:, 2:4].to(torch.int64)
        part = (((key[:, 0] << 8) | key[:, 1]) * R >> 16).to(torch.int32)
        rec_len = torch.full((per[m],), RECORD, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        r = c.partition_compress_dev(c.CODEC_LZ4BLOCK, rec.data_ptr(), per[m] * RECORD, rec_len.data_ptr(),
                                     part.data_ptr(), per[m], R, compressed.data_ptr() + map_base[m], bounds[m],
                                     checksum_alg=c.CHECKSUM_CRC32C)
        assert not r["status"].any()
        maps.append(r)
    del records, rv, rec, key, part, rec_len
    torch.cuda.empty_cache()

    def blocks(red):
        """reducer red's M blocks: offsets in the arena, lengths, and one checksum slice per block"""
        off = [map_base[m] + int(maps[m]["dst_off"][red]) for m in range(M)]
        ln = [int(maps[m]["dst_len"][red]) for m in range(M)]
        ck = [int(maps[m]["checksums"][red]) for m in range(M)]
        return off, ln, list(range(M + 1)), ln, ck

    out = torch.empty(n * RECORD, dtype=torch.uint8, device=dev)  # (b)'s outputs, reducer after reducer
    scratch = torch.empty(max(1, (n * RECORD) // R * 4), dtype=torch.uint8, device=dev)  # (a)'s output

    def timed(fn):
        c.mark(0)
        r = fn()
        c.mark(1)
        return r, c.marks_elapsed_ms()

    def call_a(red):
        off, ln, sb, sl, ck = blocks(red)
        return c.decompress_dev(c.CODEC_LZ4BLOCK, compressed.data_ptr(), off, ln, scratch.data_ptr(), scratch.numel(),
                                c.CHECKSUM_CRC32C, sb, sl, ck)

    def call_b(red, at):
        off, ln, sb, sl, ck = blocks(red)
        return c.decompress_sort_dev(c.CODEC_LZ4BLOCK, compressed.data_ptr(), off, ln, out.data_ptr() + at,
                                     out.numel() - at, RECORD, KEY_OFF, KEY_LEN, c.CHECKSUM_CRC32C, sb, sl, ck)

    for _ in range(args.warmup):
        call_a(0)
        call_b(0, 0)
    ta, tb, tsort, sort_bytes, recs_per = [], [], [], [], []
    at = 0
    ok = True
    for red in range(R):
        ra, t_a = timed(lambda: call_a(red))
        rb, t_b = timed(lambda: call_b(red, at))
        tsort.append(c.last_timing()["top_kernel_ms"])
        ok &= not ra["status"].any() and not rb["status"].any() and ra["total"] == rb["total"]
        ta.append(t_a)
        tb.append(t_b)
        nr = rb["n_records"]
        recs_per.append(nr)
        passes = KEY_LEN  # one 8-bit pass per key byte
        sort_bytes.append(2 * rb["total"] + nr * KEY_LEN + passes * nr * 16)
        at += rb["total"]

    ov = out[:at].view(-1, RECORD)
    hi, lo = key_parts(torch, ov)
    nondecreasing = bool(((hi[:-1] < hi[1:]) | ((hi[:-1] == hi[1:]) & (lo[:-1] <= lo[1:]))).all())
    valid = ok and nondecreasing and ov.shape[0] == n and digest(torch, ov) == in_digest

    sort_s = sum(tsort) * 1e-3
    mid = sorted(range(R), key=lambda i: recs_per[i])[R // 2]
    result = {
        "card": card(), "records": n, "record_bytes": n * RECORD, "maps": M, "partitions": R,
        "compressed_bytes": sum(int(m["dst_len"].sum()) for m in maps),
        "records_per_reducer": spread(recs_per),
        "a_decompress_ms": spread(ta), "b_decompress_sort_ms": spread(tb), "sort_step_ms": spread(tsort),
        "sum_ms": {"a_decompress": round(sum(ta), 3), "b_decompress_sort": round(sum(tb), 3),
                   "sort_step": round(sum(tsort), 3)},
        "sort_algorithmic_bytes": sum(sort_bytes),
        "sort_GBps": round(sum(sort_bytes) / sort_s / 1e9, 1),
        "sort_share_of_3.35TBps": round(sum(sort_bytes) / sort_s / HBM_PEAK, 3),
        "median_reducer": {"records": recs_per[mid], "a_decompress_ms": round(ta[mid], 3),
                           "sort_step_ms": round(tsort[mid], 3)},
        "teravalidate": valid,
    }
    print(json.dumps(result, indent=1))
    c.shutdown()


if __name__ == "__main__":
    main()
