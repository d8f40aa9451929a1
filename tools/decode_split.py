#!/usr/bin/env python
"""Where the read pass of bench.py's flagship wave goes (config 2: 16,000 terasort shuffle blocks of 671,112 B,
LZ4Block 32 KiB + CRC32C, one GPU, device-resident), split by kernel.

The wave is built as bench.py builds it (gen_terasort_dev, seed 42, then compress_dev); the read call
(decompress_dev) is then timed over --calls calls after --warmup untimed ones.  Per call, from last_timing():
  copy_ms    dominant_ms: the decode launches (CUDA events around each launch, summed): lz4_decode_warp_kernel for
             LZ4, the snappy_copy_kernel launches for Snappy
  decode_ms  top_kernel_ms: the whole decode (Snappy: first token launch to last copy launch)
  read_ms    kernel_ms: the whole read pass (CRC32C verify, descriptors, decode, XXH32 verify)
The card's name and power limit are read in the same run.

    python tools/decode_split.py [--calls 7] [--warmup 3] [--codec lz4|snappy] [--blocks N] [--chunk-blocks N]
                                 [--block-size N] [--extra-stream-block-size N]

Prints one JSON document.  --chunk-blocks sets B2S_LZ4D_CHUNK_BLOCKS (Snappy: codec blocks per token/copy launch pair).

LZ4 codec blocks larger than the GPU compressor writes (it takes up to 64 KiB; lz4-java writes up to 32 MiB) are
compressed on the host with liblz4's LZ4_compress_default, in LZ4Block framing:
  --block-size N                the whole wave in N-byte codec blocks; a shuffle block is max(671,112 B, N) so that it
                                holds at least one codec block, and --blocks defaults to the fewest shuffle blocks that
                                make a wave of at least 1 GiB
  --extra-stream-block-size N   bench.py's wave as above, plus one more 671,112-B shuffle block in N-byte codec blocks
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RECORD = 104
LZ4_BLOCK = 32768
RECORDS_PER_BLOCK = 6453  # bench.py config 2: 671,112-byte shuffle blocks
END_MARK = b"LZ4Block" + bytes([0x15]) + bytes(12)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    if r.returncode != 0:
        raise SystemExit("nvidia-smi failed: %s" % r.stderr.strip())
    name, power = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power}


def make_wave(c, codec, n, extra_block_size=0):
    """-> the wave to read: bench.py's config-2 wave, compressed on the device (plus, with extra_block_size, one more
    shuffle block compressed on the host in codec blocks of that size)"""
    block_bytes = RECORDS_PER_BLOCK * RECORD
    wave_bytes = n * block_bytes
    extra = host_streams(c, 1, block_bytes, extra_block_size, n * RECORDS_PER_BLOCK) if extra_block_size else []
    cmp_cap = int(c.compress_bound(codec, LZ4_BLOCK, block_bytes)) * n + sum(len(e) for e in extra)
    d_src, d_cmp = c.dev_alloc(wave_bytes), c.dev_alloc(cmp_cap)
    c.gen_terasort_dev(d_src, 0, n * RECORDS_PER_BLOCK, 42)
    off = np.arange(n, dtype=np.uint64) * block_bytes
    ln = np.full(n, block_bytes, dtype=np.uint64)
    w = c.compress_dev(codec, d_src, off, ln, d_cmp, cmp_cap, LZ4_BLOCK, c.CHECKSUM_CRC32C)
    assert not w["status"].any(), "compress_dev reported errors"
    c.dev_free(d_src)  # the read pass needs only the compressed wave and an output arena
    off, ln, cks = w["dst_off"], w["dst_len"], w["checksums"]
    if extra:
        end = int(off[-1] + ln[-1])
        e = np.frombuffer(extra[0], np.uint8)
        c.dev_memcpy(d_cmp + end, e.ctypes.data, e.size, 1)
        off, ln = np.append(off, np.uint64(end)), np.append(ln, np.uint64(e.size))
        cks = np.append(cks, np.uint64(c.checksum_batch(c.CHECKSUM_CRC32C, extra)[0]))
        wave_bytes += block_bytes
    return {"d_cmp": d_cmp, "off": off, "len": ln, "checksums": cks, "d_out": c.dev_alloc(wave_bytes),
            "bytes": wave_bytes}


def host_streams(c, n, shuffle_bytes, block_size, first_record):
    """-> n LZ4Block streams of shuffle_bytes terasort bytes each (gen_terasort_dev, seed 42, from first_record on), in
    block_size-byte codec blocks compressed by liblz4's LZ4_compress_default (what lz4-java's JNI compressor calls)"""
    from oracle import oracle  # XXH32 of each codec block, for the LZ4Block headers

    n_rec = -(-n * shuffle_bytes // RECORD)
    d = c.dev_alloc(n_rec * RECORD)
    c.gen_terasort_dev(d, first_record, n_rec, 42)
    data = np.empty(n_rec * RECORD, np.uint8)
    c.dev_memcpy(data.ctypes.data, d, data.size, 2)
    c.dev_free(d)
    L = ctypes.CDLL("liblz4.so.1")
    L.LZ4_compress_default.restype = ctypes.c_int
    level = max(0, (block_size - 1).bit_length() - 10)
    buf = ctypes.create_string_buffer(block_size + block_size // 255 + 64)
    streams = []
    for i in range(n):
        s = bytearray()
        for b in range(i * shuffle_bytes, (i + 1) * shuffle_bytes, block_size):
            piece = data[b:min(b + block_size, (i + 1) * shuffle_bytes)]
            k = L.LZ4_compress_default(ctypes.c_void_p(piece.ctypes.data), buf, piece.size, len(buf))
            assert k > 0, "LZ4_compress_default failed"
            s += (b"LZ4Block" + bytes([0x20 | level]) + k.to_bytes(4, "little") + piece.size.to_bytes(4, "little")
                  + (oracle.xxh32(piece) & 0x0FFFFFFF).to_bytes(4, "little") + buf.raw[:k])
        streams.append(bytes(s + END_MARK))
    return streams


def make_host_wave(c, n, block_size):
    """-> the wave to read: n shuffle blocks of max(671,112 B, block_size), compressed on the host"""
    shuffle_bytes = max(RECORDS_PER_BLOCK * RECORD, block_size)
    streams = host_streams(c, n, shuffle_bytes, block_size, 0)
    ln = np.array([len(s) for s in streams], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    d_cmp = c.dev_alloc(int(ln.sum()))
    for o, s in zip(off, streams):
        c.dev_memcpy(d_cmp + int(o), np.frombuffer(s, np.uint8).ctypes.data, len(s), 1)
    cks = np.array(c.checksum_batch(c.CHECKSUM_CRC32C, streams), np.uint64)
    return {"d_cmp": d_cmp, "off": off, "len": ln, "checksums": cks, "d_out": c.dev_alloc(n * shuffle_bytes),
            "bytes": n * shuffle_bytes}


def read_call(c, codec, wave):
    n = wave["off"].size
    r = c.decompress_dev(codec, wave["d_cmp"], wave["off"], wave["len"], wave["d_out"], wave["bytes"],
                         c.CHECKSUM_CRC32C, np.arange(n + 1, dtype=np.uint32), wave["len"], wave["checksums"])
    bad = np.flatnonzero(r["status"])
    assert not bad.size and r["total"] == wave["bytes"], "decompress_dev failed: streams %s status %s, %d of %d bytes" % (
        bad[:8].tolist(), r["status"][bad[:8]].tolist(), r["total"], wave["bytes"])
    return c.last_timing()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--codec", default="lz4", choices=["lz4", "snappy"])
    ap.add_argument("--blocks", type=int, default=0,
                    help="shuffle blocks in the wave (default: bench.py config 2's 16,000; with --block-size, 1 GiB)")
    ap.add_argument("--chunk-blocks", type=int, default=0, help="B2S_LZ4D_CHUNK_BLOCKS (0 = the library default)")
    ap.add_argument("--block-size", type=int, default=0, help="LZ4 codec block bytes, compressed on the host")
    ap.add_argument("--extra-stream-block-size", type=int, default=0,
                    help="LZ4 codec block bytes of one more shuffle block, compressed on the host")
    args = ap.parse_args()
    if args.calls < 5:
        raise SystemExit("--calls must be >= 5")
    host_sizes = [b for b in (args.block_size, args.extra_stream_block_size) if b]
    if host_sizes and (args.codec != "lz4" or len(host_sizes) > 1):
        raise SystemExit("--block-size and --extra-stream-block-size: LZ4 only, one of the two")
    if any(b < 64 or b > 32 << 20 for b in host_sizes):
        raise SystemExit("LZ4Block codec blocks are 64 B to 32 MiB")
    shuffle_bytes = max(RECORDS_PER_BLOCK * RECORD, args.block_size)
    if not args.blocks:
        args.blocks = -(-(1 << 30) // shuffle_bytes) if args.block_size else 16000
    if args.chunk_blocks:
        os.environ["B2S_LZ4D_CHUNK_BLOCKS"] = str(args.chunk_blocks)

    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    codec = {"lz4": c.CODEC_LZ4BLOCK, "snappy": c.CODEC_SNAPPY_XERIAL}[args.codec]
    if args.block_size:
        wave = make_host_wave(c, args.blocks, args.block_size)
        workload = "%d shuffle blocks x %d B of terasort records, LZ4 %d-B codec blocks (liblz4) + CRC32C" % (
            args.blocks, shuffle_bytes, args.block_size)
    else:
        wave = make_wave(c, codec, args.blocks, args.extra_stream_block_size)
        workload = "bench.py config 2 wave: %d shuffle blocks x %d B, %s 32 KiB + CRC32C" % (
            args.blocks, RECORDS_PER_BLOCK * RECORD, args.codec)
        if args.extra_stream_block_size:
            workload += ", and one more in LZ4 %d-B codec blocks (liblz4)" % args.extra_stream_block_size

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
        "workload": workload + ", read pass (decompress_dev)",
        "chunk_blocks": os.environ.get("B2S_LZ4D_CHUNK_BLOCKS", "default"),
        "copy_launches": rows[-1]["dominant_launches"],
        "copy_ms": summary(copy),
        "decode_ms": summary(decode),
        "read_ms": summary(read),
        "copy_share_of_decode": round(statistics.median(copy) / statistics.median(decode), 3),
        "copy_share_of_read": round(statistics.median(copy) / statistics.median(read), 3),
    }
    print(json.dumps(doc, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
