"""Measure b2s_partition_compress_rows_hash_dev (Spark's HashPartitioning ids computed on the GPU, then the partition +
compress step) against b2s_partition_compress_dev over the same rows with the ids computed on the host by the Murmur3
model (tests/hash_model.py), the two alternated in one session, with byte-identical outputs checked on the device.

Shapes (one map task's output, device-resident, generated with torch):
  join : the rows of tools/sort_rows_bench.py: an 8-byte null bitset, five 8-byte fields (field 0 an int64 join key,
         null in ~5 % of rows) and a variable region of 0..64 bytes: records of 52..116 bytes; key (INT64, 8, 8, 0)
  q67  : the string composite of tools/sort_rows_keys_bench.py's q67 shape, reduced to its key columns' types: three
         strings of 4..23 bytes (one null in ~5 % of rows) and an int, plus a decimal(28) sum; key (string, string,
         string, int)
Reports per configuration the hash step alone (dominant_ms of the hashed call), each call's kernel time
(kernel_ms: partition step + codec) and wall time, and top_kernel_ms, which with codec none is the partition step
(plus, for the hashed call, the hash step); the card's name and power limit read in the same run.  Prints one JSON
line per configuration."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FIXED = 52


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def put(torch, buf, o, cols, val_u8):
    buf[o[:, None] + torch.arange(cols[0], cols[1], device=buf.device)] = val_u8


def join_rows(torch, gen, n, dev):
    """-> (records, rec_len int32, keys, starts of the rows) for the join shape"""
    L = FIXED + 8 * torch.randint(0, 9, (n,), generator=gen, device=dev)
    off = torch.cumsum(L, 0) - L
    buf = torch.randint(0, 256, (int(L.sum()),), generator=gen, device=dev, dtype=torch.uint8)
    for i in range(0, n, 1 << 22):
        o, ln = off[i:i + (1 << 22)], L[i:i + (1 << 22)]
        m = o.numel()
        s = ln - 4
        put(torch, buf, o, (0, 4), torch.stack([(s >> 24) & 255, (s >> 16) & 255, (s >> 8) & 255, s & 255],
                                               1).to(torch.uint8))
        null = (torch.rand(m, generator=gen, device=dev) < 0.05).to(torch.int64)
        put(torch, buf, o, (4, 12), null[:, None].view(torch.uint8).view(m, 8))
    return buf, L.to(torch.int32), [(2, 8, 8, 0)], off + 4


def q67_rows(torch, gen, n, dev):
    """the q67 shape: bitset, slots (3 strings, int, decimal), then the three strings and the decimal's 16 bytes"""
    lens = torch.randint(4, 24, (n, 3), generator=gen, device=dev)
    pad = (lens + 7) // 8 * 8
    row = 8 + 5 * 8 + pad.sum(1) + 16
    L = row + 4
    off = torch.cumsum(L, 0) - L
    buf = torch.randint(97, 123, (int(L.sum()),), generator=gen, device=dev, dtype=torch.uint8)
    for i in range(0, n, 1 << 22):
        o, ln = off[i:i + (1 << 22)], L[i:i + (1 << 22)]
        m = o.numel()
        s = ln - 4
        put(torch, buf, o, (0, 4), torch.stack([(s >> 24) & 255, (s >> 16) & 255, (s >> 8) & 255, s & 255],
                                               1).to(torch.uint8))
        null = (torch.rand(m, generator=gen, device=dev) < 0.05).to(torch.int64) << 1  # field 1 null
        put(torch, buf, o, (4, 12), null[:, None].view(torch.uint8).view(m, 8))
        at = torch.full((m,), 48, device=dev, dtype=torch.int64)
        for f in range(3):
            ls = lens[i:i + m, f]
            put(torch, buf, o, (12 + 8 * f, 20 + 8 * f), ((at << 32) | ls)[:, None].view(torch.uint8).view(m, 8))
            at = at + pad[i:i + m, f]
        put(torch, buf, o, (44, 52), ((at << 32) | 11)[:, None].view(torch.uint8).view(m, 8))  # decimal(28): 11 bytes
    keys = [(3, 8, 8, 0), (3, 16, 8, 1), (3, 24, 8, 2), (1, 32, 4, 3)]
    return buf, L.to(torch.int32), keys, off + 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="join", choices=["join", "q67"])
    ap.add_argument("--gib", type=float, nargs="+", default=[2.0, 10.0])
    ap.add_argument("--partitions", type=int, nargs="+", default=[200, 2000])
    ap.add_argument("--codec", nargs="+", default=["none", "snappy", "lz4"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()

    import numpy as np
    import torch

    import hash_model as hm
    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    dev = torch.device("cuda", 0)
    name = card()
    for gib in args.gib:
        gen = torch.Generator(device=dev)
        gen.manual_seed(args.seed)
        avg = FIXED + 32 if args.shape == "join" else 4 + 48 + 3 * 16 + 16
        n = int(gib * (1 << 30)) // avg
        make = join_rows if args.shape == "join" else q67_rows
        rec, rec_len, keys, starts = make(torch, gen, n, dev)
        host = rec.cpu().numpy()
        st = starts.cpu().numpy()
        for R in args.partitions:
            ids = torch.from_numpy(hm.ids_np(host, st, keys, R).view(np.int32)).to(dev)
            for codec_name in args.codec:
                codec = c.CODEC_NONE if codec_name == "none" else c.CODEC_BY_NAME[codec_name]
                cap = c.partition_compress_bound(codec, 0, R, rec.numel()) + 64
                out = {k: torch.empty(cap, dtype=torch.uint8, device=dev) for k in ("hash", "ids")}
                t = {k: [] for k in ("hash_step", "hash_kernel", "hash_total", "hash_top", "ids_kernel",
                                     "ids_total", "ids_top")}
                res = {}
                for rep in range(args.reps + 1):
                    for kind in ("ids", "hash") if rep % 2 else ("hash", "ids"):
                        if kind == "hash":
                            r = c.partition_compress_rows_hash_dev(codec, rec.data_ptr(), rec.numel(),
                                                                   rec_len.data_ptr(), n, keys, R,
                                                                   out[kind].data_ptr(), cap, checksum_alg=3)
                        else:
                            r = c.partition_compress_dev(codec, rec.data_ptr(), rec.numel(), rec_len.data_ptr(),
                                                         ids.data_ptr(), n, R, out[kind].data_ptr(), cap,
                                                         checksum_alg=3)
                        tm = c.last_timing()
                        res[kind] = r
                        if rep == 0:
                            continue  # warm-up: buffers grow
                        t[kind + "_kernel"].append(tm["kernel_ms"])
                        t[kind + "_total"].append(tm["total_ms"])
                        t[kind + "_top"].append(tm["top_kernel_ms"])
                        if kind == "hash":
                            t["hash_step"].append(tm["dominant_ms"])
                a, b = res["hash"], res["ids"]
                same = (a["total"] == b["total"] and all((a[k] == b[k]).all() for k in
                                                         ("dst_off", "dst_len", "checksums", "status")) and
                        torch.equal(out["hash"][:a["total"]], out["ids"][:b["total"]]))
                print(json.dumps({
                    "card": name, "shape": args.shape, "gib": gib, "records": n, "partitions": R,
                    "codec": codec_name, "checksum": "CRC32C", "identical": bool(same),
                    "hash_step_ms": spread(t["hash_step"]),
                    "call_kernel_ms": {"hash": spread(t["hash_kernel"]), "host_ids": spread(t["ids_kernel"])},
                    "call_total_ms": {"hash": spread(t["hash_total"]), "host_ids": spread(t["ids_total"])},
                    "top_kernel_ms": {"hash": spread(t["hash_top"]), "host_ids": spread(t["ids_top"])},
                    "hash_GBps_of_records": round(rec.numel() / (statistics.median(t["hash_step"]) * 1e6), 1),
                }), flush=True)
                del out
                torch.cuda.empty_cache()  # the library allocates its own workspace for the next codec
            del ids
        del rec, rec_len, starts, host
        torch.cuda.empty_cache()
    c.shutdown()


if __name__ == "__main__":
    main()
