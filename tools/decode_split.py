#!/usr/bin/env python
"""Where the read pass of bench.py's flagship wave goes (config 2: 16,000 terasort shuffle blocks of 671,112 B,
LZ4Block 32 KiB + CRC32C, one GPU, device-resident), split by kernel.

The wave is built as bench.py builds it (gen_terasort_dev, seed 42, then compress_dev); the read call
(decompress_dev) is then timed over --calls calls after --warmup untimed ones.  Per call, from last_timing():
  copy_ms    dominant_ms: the lz4_copy_kernel launches (CUDA events around each launch, summed)
  decode_ms  top_kernel_ms: token walk + copy, first token launch to last copy launch
  read_ms    kernel_ms: the whole read pass (CRC32C verify, descriptors, decode, XXH32 verify)
A child process, run first, repeats one read call with B2S_TRACE=1 and reports the per-chunk timeline: the token walk
of a chunk runs on the side stream while the previous chunk's copies run on the main one.  The card's name and power
limit are read in the same run.

    python tools/decode_split.py [--calls 7] [--warmup 3] [--codec lz4|snappy] [--blocks N] [--chunk-blocks N]

Prints one JSON document.  --chunk-blocks sets B2S_LZ4D_CHUNK_BLOCKS (codec blocks per token/copy launch pair).
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RECORD = 104
LZ4_BLOCK = 32768
RECORDS_PER_BLOCK = 6453  # bench.py config 2: 671,112-byte shuffle blocks
TRACE_ROW = re.compile(r"chunk +(\d+): A\(match\|tokens\) +([\d.]+)\.\. *([\d.]+) +B\(parse\|copy\) +([\d.]+)\.\. *"
                       r"([\d.]+) +end +([\d.]+) ms")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    if r.returncode != 0:
        raise SystemExit("nvidia-smi failed: %s" % r.stderr.strip())
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power}


def make_wave(c, codec, n):
    """-> (d_cmp, write result, d_out, wave bytes, slice base): bench.py's config-2 wave, compressed on the device"""
    block_bytes = RECORDS_PER_BLOCK * RECORD
    wave_bytes = n * block_bytes
    cmp_cap = int(c.compress_bound(codec, LZ4_BLOCK, block_bytes)) * n
    d_src, d_cmp = c.dev_alloc(wave_bytes), c.dev_alloc(cmp_cap)
    c.gen_terasort_dev(d_src, 0, n * RECORDS_PER_BLOCK, 42)
    off = np.arange(n, dtype=np.uint64) * block_bytes
    ln = np.full(n, block_bytes, dtype=np.uint64)
    w = c.compress_dev(codec, d_src, off, ln, d_cmp, cmp_cap, LZ4_BLOCK, c.CHECKSUM_CRC32C)
    assert not w["status"].any(), "compress_dev reported errors"
    c.dev_free(d_src)  # the read pass needs only the compressed wave and an output arena
    return d_cmp, w, c.dev_alloc(wave_bytes), wave_bytes, np.arange(n + 1, dtype=np.uint32)


def read_call(c, codec, wave):
    d_cmp, w, d_out, wave_bytes, sb = wave
    r = c.decompress_dev(codec, d_cmp, w["dst_off"], w["dst_len"], d_out, wave_bytes, c.CHECKSUM_CRC32C, sb,
                         w["dst_len"], w["checksums"])
    assert not r["status"].any() and r["total"] == wave_bytes, "decompress_dev failed"
    return c.last_timing()


def traced_timeline(args):
    """per-chunk timeline of one read call, from a child process run with B2S_TRACE=1"""
    env = dict(os.environ, B2S_TRACE="1")
    cmd = [sys.executable, os.path.abspath(__file__), "--trace-only", "--codec", args.codec,
           "--blocks", str(args.blocks)]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        raise SystemExit("traced run failed:\n" + p.stderr)
    timeline = []
    for line in p.stderr.split("--- read call ---", 1)[-1].splitlines():
        m = TRACE_ROW.search(line)
        if m:
            k, t0, t1, c0, c1, end = m.groups()
            timeline.append({"chunk": int(k), "tokens_ms": [float(t0), float(t1)], "copy_ms": [float(c0), float(end)]})
    return timeline


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--codec", default="lz4", choices=["lz4", "snappy"])
    ap.add_argument("--blocks", type=int, default=16000, help="shuffle blocks in the wave (bench.py config 2: 16,000)")
    ap.add_argument("--chunk-blocks", type=int, default=0, help="B2S_LZ4D_CHUNK_BLOCKS (0 = the library default)")
    ap.add_argument("--trace-only", action="store_true", help=argparse.SUPPRESS)  # the B2S_TRACE=1 child
    args = ap.parse_args()
    if args.calls < 5:
        raise SystemExit("--calls must be >= 5")
    if args.chunk_blocks:
        os.environ["B2S_LZ4D_CHUNK_BLOCKS"] = str(args.chunk_blocks)

    if not args.trace_only:  # first, while this process holds no device memory: both waves do not fit at once
        timeline = traced_timeline(args)

    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    codec = {"lz4": c.CODEC_LZ4BLOCK, "snappy": c.CODEC_SNAPPY_XERIAL}[args.codec]
    wave = make_wave(c, codec, args.blocks)
    if args.trace_only:  # one traced read call; the timeline rows go to stderr, after this marker
        read_call(c, codec, wave)
        sys.stderr.flush()
        os.write(2, b"--- read call ---\n")
        read_call(c, codec, wave)
        return 0

    for _ in range(args.warmup):
        read_call(c, codec, wave)
    rows = [read_call(c, codec, wave) for _ in range(args.calls)]
    copy = [t["dominant_ms"] for t in rows]
    decode = [t["top_kernel_ms"] for t in rows]
    read = [t["kernel_ms"] for t in rows]

    def summary(v):
        return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3),
                "calls": [round(x, 3) for x in v]}

    doc = {
        "card": card(),
        "workload": "bench.py config 2 wave: %d shuffle blocks x %d B, %s 32 KiB + CRC32C, read pass (decompress_dev)"
                    % (args.blocks, RECORDS_PER_BLOCK * RECORD, args.codec),
        "chunk_blocks": os.environ.get("B2S_LZ4D_CHUNK_BLOCKS", "default"),
        "copy_launches": rows[-1]["dominant_launches"],
        "copy_ms": summary(copy),
        "decode_ms": summary(decode),
        "read_ms": summary(read),
        "copy_share_of_decode": round(statistics.median(copy) / statistics.median(decode), 3),
        "copy_share_of_read": round(statistics.median(copy) / statistics.median(read), 3),
        "timeline_ms": timeline,
    }
    print(json.dumps(doc, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
