#!/usr/bin/env python
"""Cost of row-sorting a reduce task's UnsafeRow records on the GPU (b2s_decompress_sort_rows_dev), against decoding the
same blocks.

Input: --gib GiB of device-generated, seeded UnsafeRow-shaped records in the shape of the "sql join" config: each row
is an 8-byte null bitset, five 8-byte fields (field 0: an int64 join key, negatives included, null in ~5 % of rows) and
a variable-length region of 0..64 bytes in steps of 8, so a record ([int32 big-endian size][row]) is 52..116 bytes.  The
rows are split into --maps map tasks; each goes through partition_compress_dev (--codec, default snappy, + CRC32C) with
a random reduce id per row.  One GPU, everything device-resident.  After --warmup untimed calls, every reducer's blocks
are timed two ways:
  (a) decompress_dev alone (verify + decode)
  (b) decompress_sort_rows_dev (verify + decode + framing + sort; INT64 key at row offset 8, null_field 0)
Times are CUDA events on the library's stream (b2s_mark), per call.  Framing is (b)'s dominant_ms, the sort step (b)'s
top_kernel_ms minus that.  min / median / max over the reducers and the sums over all reducers are printed.  The sort
step's algorithmic bytes are computed here: every record read once and written once, every key and null word read once,
and 8 B of (key word, index) pairs read and 8 B written per radix pass (9 passes: the null byte and 8 key bytes); its
rate is those bytes over the sort step's time, and its share of peak that rate over the 3.35 TB/s HBM3 of the H100 SXM
data sheet.  Validation, per reducer: the output is parsed independently (pointer doubling over the 4-byte-aligned
positions), the keys must be non-decreasing in signed order with nulls first, and over all reducers the record count,
the bytes, an order-independent digest of the records' fixed part and the sum of all bytes must equal the input's.  The
card's name and power limit are read in the same run.

    python tools/sort_rows_bench.py [--gib 10] [--maps 400] [--partitions 200] [--codec snappy] [--warmup 2]

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

FIXED = 52            # size prefix + null bitset + five 8-byte fields
KEY_OFF, NULL_FIELD = 8, 0  # field 0 of the row: after the one-word null bitset
HBM_PEAK = 3.35e12    # H100 SXM data sheet
MIX = [0x9E3779B97F4A7C15 % (1 << 61), 0x5851F42D4C957F2D % (1 << 61)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def gather(torch, buf, off, width):
    """(n, width) uint8: the width bytes at each offset"""
    return buf[off[:, None] + torch.arange(width, device=buf.device)]


def digest(torch, buf, off):
    """order-independent digest of the records at off: a wrapping sum of a mix of each record's first 48 bytes (size
    prefix, null bitset, the key and the next four fields; every record is at least 52 bytes long)"""
    total = 0
    for i in range(0, off.numel(), 1 << 20):
        w = gather(torch, buf, off[i:i + (1 << 20)], 48).view(torch.int64)
        w = w + torch.arange(1, 7, device=buf.device) * MIX[0]
        w = (w ^ (w >> 31)) * MIX[1]
        total = (total + int((w ^ (w >> 29)).sum())) % (1 << 64)  # torch's int64 sums wrap: compare mod 2^64
    return total


def record_starts(torch, buf):
    """every record start of a UnsafeRowSerializer stream whose records are multiples of 4 bytes long: position i (in
    4-byte units) jumps to i + size / 4 + 1; the starts are the positions reachable from 0 (pointer doubling)"""
    n4 = buf.numel() // 4
    if n4 == 0:
        return torch.zeros(0, dtype=torch.int64, device=buf.device)
    b = buf[: n4 * 4].view(n4, 4).to(torch.int64)
    size = (b[:, 0] << 24) | (b[:, 1] << 16) | (b[:, 2] << 8) | b[:, 3]
    nxt = torch.clamp(torch.arange(n4, device=buf.device) + size // 4 + 1, max=n4)
    nxt = torch.cat([nxt, torch.tensor([n4], device=buf.device)])  # n4: past the end, a fixed point
    reach = torch.zeros(n4 + 1, dtype=torch.bool, device=buf.device)
    reach[0] = True
    while True:
        before = int(reach.sum())
        reach[nxt[reach]] = True
        nxt = nxt[nxt]
        if int(reach.sum()) == before and bool((nxt == n4).all()):
            break
    return torch.nonzero(reach[:n4]).flatten() * 4


def make_map(torch, gen, n, R, dev):
    """n records of one map task: (records, rec_len u32, reduce ids u32, n_null)"""
    L = FIXED + 8 * torch.randint(0, 9, (n,), generator=gen, device=dev)
    off = torch.cumsum(L, 0) - L
    total = int(L.sum())
    buf = torch.randint(0, 256, (total,), generator=gen, device=dev, dtype=torch.uint8)
    n_null = 0
    for i in range(0, n, 1 << 22):
        o, ln = off[i:i + (1 << 22)], L[i:i + (1 << 22)]
        m = o.numel()
        s = ln - 4
        pre = torch.stack([(s >> 24) & 255, (s >> 16) & 255, (s >> 8) & 255, s & 255], 1).to(torch.uint8)
        buf[o[:, None] + torch.arange(4, device=dev)] = pre
        null = torch.rand(m, generator=gen, device=dev) < 0.05
        n_null += int(null.sum())
        buf[o[:, None] + torch.arange(4, 12, device=dev)] = null.to(torch.int64)[:, None].view(torch.uint8).view(m, 8)
        key = torch.randint(-(1 << 62), 1 << 62, (m,), generator=gen, device=dev, dtype=torch.int64)
        buf[o[:, None] + torch.arange(12, 20, device=dev)] = key[:, None].view(torch.uint8).view(m, 8)
    part = torch.randint(0, R, (n,), generator=gen, device=dev, dtype=torch.int32)
    return buf, off, L.to(torch.int32), part, n_null


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--maps", type=int, default=400)
    ap.add_argument("--partitions", type=int, default=200)
    ap.add_argument("--codec", default="snappy", choices=["none", "lz4", "snappy", "zstd"])
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()

    import torch

    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    codec = c.CODEC_NONE if args.codec == "none" else c.CODEC_BY_NAME[args.codec]
    M, R = args.maps, args.partitions
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev)
    gen.manual_seed(args.seed)
    n = int(args.gib * (1 << 30)) // (FIXED + 32)  # 84 bytes per record on average
    per = [n // M] * (M - 1) + [n - n // M * (M - 1)]

    # map side: every map task partitioned + compressed into one arena (map m at map_base[m], 256-byte aligned)
    bounds, maps, map_base = [], [], []
    in_digest, in_bytes, in_null, in_sum = 0, 0, 0, 0
    compressed = None
    for m in range(M):
        rec, off, rec_len, part, n_null = make_map(torch, gen, per[m], R, dev)
        in_digest = (in_digest + digest(torch, rec, off)) % (1 << 64)
        in_bytes += rec.numel()
        in_sum += sum(int(rec[i:i + (1 << 28)].sum(dtype=torch.int64)) for i in range(0, rec.numel(), 1 << 28))
        in_null += n_null
        bound = (c.partition_compress_bound(codec, 0, R, rec.numel()) + 255) // 256 * 256
        if compressed is None:  # one arena for every map: sized from the first map's bound, with room to spare
            cap = bound * M + bound
            compressed = torch.empty(cap, dtype=torch.uint8, device=dev)
        at = sum(bounds)
        assert at + bound <= compressed.numel()
        torch.cuda.synchronize()
        r = c.partition_compress_dev(codec, rec.data_ptr(), rec.numel(), rec_len.data_ptr(), part.data_ptr(), per[m],
                                     R, compressed.data_ptr() + at, bound, checksum_alg=c.CHECKSUM_CRC32C)
        assert not r["status"].any()
        maps.append(r)
        map_base.append(at)
        bounds.append(bound)
        del rec, off, rec_len, part
    torch.cuda.empty_cache()

    def blocks(red):
        off = [map_base[m] + int(maps[m]["dst_off"][red]) for m in range(M)]
        ln = [int(maps[m]["dst_len"][red]) for m in range(M)]
        ck = [int(maps[m]["checksums"][red]) for m in range(M)]
        return off, ln, list(range(M + 1)), ln, ck

    biggest = max(sum(int(maps[m]["dst_len"][red]) for m in range(M)) for red in range(R))
    cap = (biggest * (1 if codec == c.CODEC_NONE else 4)) + (1 << 20)
    out = torch.empty(cap + 64, dtype=torch.uint8, device=dev)
    scratch = torch.empty(cap, dtype=torch.uint8, device=dev)

    def timed(fn):
        c.mark(0)
        r = fn()
        c.mark(1)
        return r, c.marks_elapsed_ms()

    def call_a(red):
        off, ln, sb, sl, ck = blocks(red)
        return c.decompress_dev(codec, compressed.data_ptr(), off, ln, scratch.data_ptr(), scratch.numel(),
                                c.CHECKSUM_CRC32C, sb, sl, ck)

    def call_b(red):
        off, ln, sb, sl, ck = blocks(red)
        return c.decompress_sort_rows_dev(codec, compressed.data_ptr(), off, ln, out.data_ptr(), cap, c.KEY_INT64,
                                          KEY_OFF, 8, NULL_FIELD, c.CHECKSUM_CRC32C, sb, sl, ck)

    for _ in range(args.warmup):
        call_a(0)
        call_b(0)
    ta, tb, tframe, tsort, sort_bytes, recs_per = [], [], [], [], [], []
    ok, ordered = True, True
    out_digest, out_records, out_bytes, out_sum = 0, 0, 0, 0
    for red in range(R):
        ra, t_a = timed(lambda: call_a(red))
        rb, t_b = timed(lambda: call_b(red))
        t = c.last_timing()
        tframe.append(t["dominant_ms"])
        tsort.append(t["top_kernel_ms"] - t["dominant_ms"])
        ok &= not ra["status"].any() and not rb["status"].any() and ra["total"] == rb["total"]
        ta.append(t_a)
        tb.append(t_b)
        nr = rb["n_records"]
        recs_per.append(nr)
        sort_bytes.append(2 * rb["total"] + nr * 16 + 9 * nr * 16)
        # independent check of the reducer's output
        o = out[: rb["total"] + 8]
        starts = record_starts(torch, o[: rb["total"]])
        ok &= starts.numel() == nr
        w = gather(torch, o, starts, 20)
        null = w[:, 4] != 0
        key = w[:, 12:20].contiguous().view(torch.int64).flatten()
        rank = torch.where(null, torch.zeros_like(key), key)
        nn = int(null.sum())
        ordered &= bool(null[:nn].all()) and not bool(null[nn:].any()) and bool((rank[nn + 1:] >= rank[nn:-1]).all())
        out_digest = (out_digest + digest(torch, o, starts)) % (1 << 64)
        out_sum += int(o[: rb["total"]].sum(dtype=torch.int64))
        out_records += nr
        out_bytes += rb["total"]
    same = out_records == n and out_bytes == in_bytes and out_digest == in_digest and out_sum == in_sum
    valid = ok and ordered and same

    sort_s = sum(tsort) * 1e-3
    mid = sorted(range(R), key=lambda i: recs_per[i])[R // 2]
    result = {
        "card": card(), "codec": args.codec, "records": n, "record_bytes": in_bytes, "null_keys": in_null, "maps": M,
        "partitions": R, "compressed_bytes": sum(int(m["dst_len"].sum()) for m in maps),
        "records_per_reducer": spread(recs_per),
        "a_decompress_ms": spread(ta), "b_decompress_sort_rows_ms": spread(tb), "framing_ms": spread(tframe),
        "sort_step_ms": spread(tsort),
        "sum_ms": {"a_decompress": round(sum(ta), 3), "b_decompress_sort_rows": round(sum(tb), 3),
                   "framing": round(sum(tframe), 3), "sort_step": round(sum(tsort), 3),
                   "framing_plus_sort": round(sum(tframe) + sum(tsort), 3)},
        "sort_algorithmic_bytes": sum(sort_bytes),
        "sort_GBps": round(sum(sort_bytes) / sort_s / 1e9, 1),
        "sort_share_of_3.35TBps": round(sum(sort_bytes) / sort_s / HBM_PEAK, 3),
        "median_reducer": {"records": recs_per[mid], "a_decompress_ms": round(ta[mid], 3),
                           "framing_ms": round(tframe[mid], 3), "sort_step_ms": round(tsort[mid], 3)},
        "valid": bool(valid), "counts_and_digest_match": bool(ok and same),
        "keys_ordered": bool(ordered),
    }
    print(json.dumps(result, indent=1))
    c.shutdown()


if __name__ == "__main__":
    main()
