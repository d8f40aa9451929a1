#!/usr/bin/env python
"""Where the write pass of bench.py's flagship wave goes (config 2: 16,000 terasort shuffle blocks of 671,112 B,
LZ4Block 32 KiB + CRC32C, one GPU, device-resident), split by kernel.  The write-side mirror of decode_split.py.

The wave is built as bench.py builds it (gen_terasort_dev, seed 42); the write call (compress_dev) is then timed over
--calls calls after --warmup untimed ones.  Per call, from last_timing():
  match_ms     dominant_ms: the match launches (CUDA events around each launch, summed)
  compress_ms  top_kernel_ms: the whole compress step (match + parse + scan + emit)
  write_ms     kernel_ms: the whole write pass (compress, CRC32C over the compressed streams, stream metadata)
The card's name and power limit are read in the same run.

    python tools/compress_split.py [--calls 7] [--warmup 3] [--codec lz4|snappy|zstd] [--level N] [--blocks N]
                                   [--block-size 32768]

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

RECORD = 104
RECORDS_PER_BLOCK = 6453  # bench.py config 2: 671,112-byte shuffle blocks


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    if r.returncode != 0:
        raise SystemExit("nvidia-smi failed: %s" % r.stderr.strip())
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--codec", default="lz4", choices=["lz4", "snappy", "zstd"])
    ap.add_argument("--level", type=int, default=0, help="Zstandard level (0 = the library default)")
    ap.add_argument("--blocks", type=int, default=16000, help="shuffle blocks in the wave (bench.py config 2: 16,000)")
    ap.add_argument("--block-size", type=int, default=32768, help="codec block size (bench.py: 32 KiB)")
    args = ap.parse_args()
    if args.calls < 5:
        raise SystemExit("--calls must be >= 5")

    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    codec = {"lz4": c.CODEC_LZ4BLOCK, "snappy": c.CODEC_SNAPPY_XERIAL, "zstd": c.CODEC_ZSTD}[args.codec]
    n = args.blocks
    block_bytes = RECORDS_PER_BLOCK * RECORD
    wave_bytes = n * block_bytes
    cmp_cap = int(c.compress_bound(codec, args.block_size, block_bytes)) * n
    d_src, d_cmp = c.dev_alloc(wave_bytes), c.dev_alloc(cmp_cap)
    c.gen_terasort_dev(d_src, 0, n * RECORDS_PER_BLOCK, 42)
    off = np.arange(n, dtype=np.uint64) * block_bytes
    ln = np.full(n, block_bytes, dtype=np.uint64)

    def write_call():
        w = c.compress_dev(codec, d_src, off, ln, d_cmp, cmp_cap, args.block_size, c.CHECKSUM_CRC32C,
                           level=args.level)
        assert not w["status"].any(), "compress_dev reported errors"
        return w, c.last_timing()

    for _ in range(args.warmup):
        write_call()
    rows = []
    for _ in range(args.calls):
        w, t = write_call()
        rows.append(t)
    match = [t["dominant_ms"] for t in rows]
    comp = [t["top_kernel_ms"] for t in rows]
    write = [t["kernel_ms"] for t in rows]

    def summary(v):
        return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3),
                "calls": [round(x, 3) for x in v]}

    doc = {
        "card": card(),
        "workload": "bench.py config 2 wave: %d shuffle blocks x %d B, %s %d B blocks + CRC32C, write pass "
                    "(compress_dev)" % (n, block_bytes, args.codec, args.block_size),
        "level": args.level,
        "compressed_bytes": int(w["total"]),
        "ratio": round(int(w["total"]) / wave_bytes, 5),
        "match_launches": rows[-1]["dominant_launches"],
        "match_ms": summary(match),
        "compress_ms": summary(comp),
        "write_ms": summary(write),
        "match_share_of_write": round(statistics.median(match) / statistics.median(write), 3),
    }
    print(json.dumps(doc, indent=1))
    c.dev_free(d_src)
    c.dev_free(d_cmp)
    return 0


if __name__ == "__main__":
    sys.exit(main())
