#!/usr/bin/env python
"""Cost of partitioning a map task's serialized records by reduce id on the GPU (b2s_partition_compress_dev), against
the write pass it sits in front of.

Input: --gib GiB of device-generated terasort records (gen_terasort_dev, seed 42; 104-byte records), reduce ids from
the key range (TeraSort's range partitioner: the first two key bytes, after the record's
2-byte Kryo header, scaled to R), one GPU, device-resident.
For each R in --partitions, after --warmup untimed rounds, --reps timed rounds of:
  (a) partition_compress_dev with codec NONE and no checksum: the partition step alone
  (b) partition_compress_dev with --codec and CRC32C: partition + compress in one call
  (c) compress_dev with --codec and CRC32C over the arena (a) produced: compression alone
Times are CUDA events on the library's stream (b2s_mark), per call; min / median / max over the reps are printed.
The partition step's algorithmic bytes are computed here: every record read once and written once, plus 8 B per
record (id + index) read and 8 B written per radix pass; its achieved rate is those bytes over the time of (a), and
its share of peak is that rate over the 3.35 TB/s HBM3 of the H100 SXM data sheet.  The outputs of (b) and (c) are
compared byte for byte.  The card's name and power limit are read in the same run.

    python tools/partition_bench.py [--gib 10] [--partitions 200,2000] [--codec lz4] [--reps 5] [--warmup 2]

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

RECORD = 104
HBM_PEAK = 3.35e12  # H100 SXM data sheet


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def radix_passes(R):
    bits = max(0, (R - 1).bit_length())
    return (bits + 7) // 8


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--partitions", default="200,2000")
    ap.add_argument("--codec", default="lz4", choices=["lz4", "snappy", "zstd"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch

    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    codec = c.CODEC_BY_NAME[args.codec]
    level = 3 if args.codec == "zstd" else 0
    n = int(args.gib * (1 << 30)) // RECORD
    rec_bytes = n * RECORD
    dev = torch.device("cuda", 0)
    records = torch.empty(rec_bytes, dtype=torch.uint8, device=dev)
    c.gen_terasort_dev(records.data_ptr(), 0, n, 42)
    rec_len = torch.full((n,), RECORD, dtype=torch.int32, device=dev)
    cap = c.partition_compress_bound(codec, 0, max(int(r) for r in args.partitions.split(",")), rec_bytes)
    arena = torch.empty(rec_bytes, dtype=torch.uint8, device=dev)  # (a)'s partitioned records, (c)'s input
    out_b = torch.empty(cap, dtype=torch.uint8, device=dev)
    out_c = torch.empty(cap, dtype=torch.uint8, device=dev)
    key = records.view(n, RECORD)[:, 2:4].to(torch.int64)  # the first two key bytes, after the 2-byte record header
    result = {"card": card(), "records": n, "record_bytes": rec_bytes, "codec": args.codec, "runs": []}

    def timed(fn):
        c.mark(0)
        r = fn()
        c.mark(1)
        return r, c.marks_elapsed_ms()

    for R in (int(x) for x in args.partitions.split(",")):
        part = (((key[:, 0] << 8) | key[:, 1]) * R >> 16).to(torch.int32)
        torch.cuda.synchronize()

        def step_a():
            return c.partition_compress_dev(c.CODEC_NONE, records.data_ptr(), rec_bytes, rec_len.data_ptr(),
                                            part.data_ptr(), n, R, arena.data_ptr(), rec_bytes)

        def step_b():
            return c.partition_compress_dev(codec, records.data_ptr(), rec_bytes, rec_len.data_ptr(), part.data_ptr(),
                                            n, R, out_b.data_ptr(), cap, checksum_alg=c.CHECKSUM_CRC32C, level=level)

        def step_c(a):
            ne = a["dst_len"] > 0
            return c.compress_dev(codec, arena.data_ptr(), a["dst_off"][ne], a["dst_len"][ne], out_c.data_ptr(), cap,
                                  checksum_alg=c.CHECKSUM_CRC32C, level=level)

        t = {"a": [], "b": [], "c": []}
        for k in range(args.warmup + args.reps):
            ra, ta = timed(step_a)
            rb, tb = timed(step_b)
            rc, tc = timed(lambda: step_c(ra))
            if k >= args.warmup:
                t["a"].append(ta)
                t["b"].append(tb)
                t["c"].append(tc)
        ne = ra["dst_len"] > 0
        same = (rb["total"] == rc["total"] and bool((rb["dst_len"][ne] == rc["dst_len"]).all())
                and bool((rb["checksums"][ne] == rc["checksums"]).all()) and not rb["status"].any()
                and bool(torch.equal(out_b[: rb["total"]], out_c[: rc["total"]])))
        passes = radix_passes(R)
        alg_bytes = 2 * rec_bytes + passes * n * 16
        ta_med = statistics.median(t["a"]) * 1e-3
        result["runs"].append({
            "partitions": R, "radix_passes": passes,
            "a_partition_ms": spread(t["a"]), "b_partition_compress_ms": spread(t["b"]), "c_compress_ms": spread(t["c"]),
            "partition_algorithmic_bytes": alg_bytes,
            "partition_GBps": round(alg_bytes / ta_med / 1e9, 1),
            "partition_share_of_3.35TBps": round(alg_bytes / ta_med / HBM_PEAK, 3),
            "compressed_bytes": rb["total"],
            "b_equals_c": same,
        })
    print(json.dumps(result, indent=1))
    c.shutdown()


if __name__ == "__main__":
    main()
