"""Measure b2s_partition_compress_rows_range_dev (Spark's RangePartitioner ids computed on the GPU, then the partition +
compress step) against b2s_partition_compress_dev over the same rows with the ids computed another way, the two
alternated in one session after a warm-up, with byte-identical outputs checked on the device.

Shapes (one map task's output, device-resident, generated with torch by tools/partition_rows_hash_bench.py):
  join : int64 join key, null in ~5 % of rows, ORDER BY key ASC NULLS FIRST; the other call's ids by torch.searchsorted
         over the bounds (a null key as the lowest int64)
  q67  : three strings and an int, ORDER BY s0 ASC, s1 DESC NULLS LAST, s2 ASC, i ASC; the other call's ids by the
         Python model (tests/range_model.py), which is slow, so that call and the identity check run on the first
         --model-rows records only (reported as model_records); the range call is also timed at the full size
Bounds are RangePartitioner.determineBounds over a sample of 20 rows per partition (Spark's default sample size),
projected to the sort key's UnsafeRow.  Reports per configuration the range step (dominant_ms: bound checks + id
kernel), each call's kernel time (partition step + codec), top_kernel_ms and wall time, with the card's name and power
limit read in the same run.  One JSON line per configuration."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from partition_rows_hash_bench import FIXED, card, join_rows, q67_rows, spread  # noqa: E402

DESC, NULLS_LAST = 1 << 8, 1 << 9


def draw(rg, np, host, starts, lens, keys, R, rng):
    """determineBounds over 20 R sampled rows -> the bound rows (UnsafeProjection of the sort key, unframed)"""
    idx = rng.choice(len(starts), size=min(20 * R, len(starts)), replace=False)
    rows = [host[starts[i]:starts[i] + lens[i] - 4].tobytes() for i in idx]
    return rg.draw_bounds(rng, rows, keys, R)


def equal(torch, a, b, n):
    """a[:n] == b[:n], 1 GiB at a time (one comparison of 10 GiB would need its own 10 GiB)"""
    return all(torch.equal(a[o:min(o + (1 << 30), n)], b[o:min(o + (1 << 30), n)]) for o in range(0, n, 1 << 30))


def timed(c, kind, call, reps, t):
    for rep in range(reps + 1):
        r = call()
        tm = c.last_timing()
        if rep:  # the first is the warm-up: buffers grow
            for k in ("dominant_ms", "kernel_ms", "top_kernel_ms", "total_ms"):
                t.setdefault(kind + ":" + k, []).append(tm[k])
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="join", choices=["join", "q67"])
    ap.add_argument("--gib", type=float, nargs="+", default=[2.0, 10.0])
    ap.add_argument("--partitions", type=int, nargs="+", default=[200, 2000])
    ap.add_argument("--codec", nargs="+", default=["snappy", "lz4"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--model-rows", type=int, default=100000)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()

    import numpy as np
    import torch

    import range_model as rg
    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    dev = torch.device("cuda", 0)
    name = card()
    rng = np.random.default_rng(args.seed)
    for gib in args.gib:
        gen = torch.Generator(device=dev)
        gen.manual_seed(args.seed)
        avg = FIXED + 32 if args.shape == "join" else 4 + 48 + 3 * 16 + 16
        n = int(gib * (1 << 30)) // avg
        rec, rec_len, keys, starts = (join_rows if args.shape == "join" else q67_rows)(torch, gen, n, dev)
        if args.shape == "q67":
            keys = [(keys[0][0], 8, 8, 0), (keys[1][0] | DESC | NULLS_LAST, 16, 8, 1), (keys[2][0], 24, 8, 2),
                    (keys[3][0], 32, 4, 3)]
        host = rec.cpu().numpy()
        st = starts.cpu().numpy()
        lens = rec_len.cpu().numpy()
        for R in args.partitions:
            rows_b = draw(rg, np, host, st, lens, keys, R, rng)
            bounds = [rg.framed(b) for b in rows_b]
            m = n
            if args.shape == "join":
                kv = rec[starts[:, None] + torch.arange(8, 16, device=dev)].view(torch.int64).view(-1)
                null = (rec[starts[:, None] + torch.arange(0, 8, device=dev)].view(torch.int64).view(-1) & 1) == 1
                kv = torch.where(null, torch.iinfo(torch.int64).min, kv)
                bk = [int.from_bytes(b[12:20], "little", signed=True) if not (b[4] & 1) else -2**63 for b in bounds]
                ids = torch.searchsorted(torch.tensor(bk, dtype=torch.int64, device=dev), kv).to(torch.int32)
                del kv, null
            else:
                m = min(n, args.model_rows)
                rows = [host[st[i]:st[i] + lens[i] - 4].tobytes() for i in range(m)]
                ids = torch.from_numpy(rg.model_ids(rows, keys, rows_b).view(np.int32)).to(dev)
            sub = int(rec_len[:m].to(torch.int64).sum())
            for codec_name in args.codec:
                codec = c.CODEC_BY_NAME[codec_name]
                cap = c.partition_compress_bound(codec, 0, len(bounds) + 1, rec.numel()) + 64
                out = {k: torch.empty(cap, dtype=torch.uint8, device=dev) for k in ("range", "ids")}
                t, res = {}, {}
                for rep in range(3):  # the two calls alternated three times
                    for kind in ("ids", "range") if rep % 2 else ("range", "ids"):
                        if kind == "range":
                            res[kind] = timed(c, kind, lambda: c.partition_compress_rows_range_dev(
                                codec, rec.data_ptr(), sub, rec_len.data_ptr(), m, keys, bounds,
                                out[kind].data_ptr(), cap, checksum_alg=3), args.reps if rep == 0 else 1, t)
                        else:
                            res[kind] = timed(c, kind, lambda: c.partition_compress_dev(
                                codec, rec.data_ptr(), sub, rec_len.data_ptr(), ids.data_ptr(), m,
                                len(bounds) + 1, out[kind].data_ptr(), cap, checksum_alg=3),
                                args.reps if rep == 0 else 1, t)
                a, b = res["range"], res["ids"]
                same = (a["total"] == b["total"] and all((a[k] == b[k]).all() for k in
                                                         ("dst_off", "dst_len", "checksums", "status")) and
                        equal(torch, out["range"], out["ids"], a["total"]))
                line = {"card": name, "shape": args.shape, "gib": gib, "records": n, "model_records": m,
                        "partitions": len(bounds) + 1, "codec": codec_name, "checksum": "CRC32C",
                        "identical": bool(same), "range_step_ms": spread(t["range:dominant_ms"]),
                        "call_kernel_ms": {"range": spread(t["range:kernel_ms"]), "ids": spread(t["ids:kernel_ms"])},
                        "top_kernel_ms": {"range": spread(t["range:top_kernel_ms"]),
                                          "ids": spread(t["ids:top_kernel_ms"])},
                        "call_total_ms": {"range": spread(t["range:total_ms"]), "ids": spread(t["ids:total_ms"])}}
                if m < n:  # the range call alone at the full size
                    full = {}
                    timed(c, "full", lambda: c.partition_compress_rows_range_dev(
                        codec, rec.data_ptr(), rec.numel(), rec_len.data_ptr(), n, keys, bounds,
                        out["range"].data_ptr(), cap, checksum_alg=3), args.reps, full)
                    line["full_size_range"] = {"range_step_ms": spread(full["full:dominant_ms"]),
                                               "kernel_ms": spread(full["full:kernel_ms"]),
                                               "total_ms": spread(full["full:total_ms"])}
                print(json.dumps(line), flush=True)
                del out
                torch.cuda.empty_cache()
            del ids
        del rec, rec_len, starts, host
        torch.cuda.empty_cache()
    c.shutdown()


if __name__ == "__main__":
    main()
