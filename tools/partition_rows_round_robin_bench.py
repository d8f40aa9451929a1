"""Measure b2s_partition_compress_rows_round_robin_dev (Spark's repartition(n): the sortBeforeRepartition sort of a map
task's rows by (row hash, row bytes), then the position's ids, then the partition + compress step) against
b2s_partition_compress_dev fed the same rows already in the writer's order with their ids, the two alternated in one
session after a warm-up, with byte-identical outputs checked on the device.

The reference order is the model of tests/round_robin_model.py restated in torch on the device (Murmur3 over each
row's words, then stable LSD sorts by the row's big-endian words, its size and its signed hash), so it shares no code
with the CUDA path.  Shapes (one map task's output, device-resident):
  join : the join rows of tools/partition_rows_hash_bench.py (52..116 bytes)
  q67  : its q67 rows (three strings, an int, a decimal)
  dup  : 1000 distinct join rows, each repeated: the refinement's worst case (every record tied to the end of its row)
Reports per configuration the round-robin step (dominant_ms: checks, hash, sort with its rounds, ids) with and without
the sort, the tied records and the model's refinement rounds, each call's kernel and wall time, and the card's name and
power limit read in the same run.  Prints one JSON line per configuration."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

M32 = 0xFFFFFFFF


def murmur_words(torch, buf, starts, size):
    """hashUnsafeWords(row, 42) of every row (size a multiple of 8), int64 holding the unsigned 32-bit value"""
    h = torch.full_like(size, 42)
    for w in range(int(size.max()) // 4 if size.numel() else 0):
        sel = torch.nonzero(size > 4 * w).squeeze(1)
        p = starts[sel] + 4 * w
        k = (buf[p].long() | (buf[p + 1].long() << 8) | (buf[p + 2].long() << 16) | (buf[p + 3].long() << 24))
        k = (k * 0xCC9E2D51) & M32
        k = ((k << 15) | (k >> 17)) & M32
        k = (k * 0x1B873593) & M32
        x = h[sel] ^ k
        x = ((x << 13) | (x >> 19)) & M32
        h[sel] = (x * 5 + 0xE6546B64) & M32
    h = h ^ size
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    return h ^ (h >> 16)


def model_order(torch, buf, starts, size):
    """the writer's order: signed hash, then size, then the row's bytes (big-endian words, zero-padded); stable LSD"""
    n = size.numel()
    order = torch.arange(n, device=buf.device)
    for w in range(int(size.max()) // 4 - 1 if n else -1, -1, -1):
        s, z = starts[order], size[order]
        p = (s + 4 * w).clamp(max=buf.numel() - 4)
        word = (buf[p].long() << 24) | (buf[p + 1].long() << 16) | (buf[p + 2].long() << 8) | buf[p + 3].long()
        word = torch.where(z > 4 * w, word, torch.zeros_like(word))
        order = order[torch.sort(word, stable=True).indices]
    order = order[torch.sort(size[order], stable=True).indices]
    h = murmur_words(torch, buf, starts, size)
    hs = torch.where(h >= (1 << 31), h - (1 << 32), h)
    order = order[torch.sort(hs[order], stable=True).indices]
    return order, hs


def tie_stats(torch, buf, starts, size, order, hs):
    """records in a run of equal hash, and the refinement rounds the longest tie needs (model)"""
    a, b = order[:-1], order[1:]
    tie = (hs[a] == hs[b]) & (size[a] == size[b])
    tied = torch.zeros(order.numel(), dtype=torch.bool, device=buf.device)
    tied[:-1] |= tie
    tied[1:] |= tie
    rounds = 0
    if bool(tie.any()):
        ta, tb = a[tie], b[tie]
        lcp = size[ta].clone()  # identical rows tie to their end
        for w in range(int(size[ta].max()) // 4):
            alive = (lcp == size[ta]) & (size[ta] > 4 * w)
            if not bool(alive.any()):
                break
            i = torch.nonzero(alive).squeeze(1)
            pa, pb = starts[ta[i]] + 4 * w, starts[tb[i]] + 4 * w
            diff = torch.zeros_like(i, dtype=torch.bool)
            for q in range(4):
                diff |= buf[pa + q] != buf[pb + q]
            lcp[i[diff]] = 4 * w
        rounds = int(((8 + lcp - 4) // 16).max()) + 1
    return int(tied.sum()), rounds


def gather_rows(torch, buf, starts, size, order, dev, chunk=1 << 22):
    """the framed records in the order given, back to back, and their rec_len"""
    ln = (size[order] + 4)
    out = torch.empty(int(ln.sum()), dtype=torch.uint8, device=dev)
    dst = torch.cumsum(ln, 0) - ln
    for i in range(0, order.numel(), chunk):
        o, l, d = starts[order[i:i + chunk]] - 4, ln[i:i + chunk], dst[i:i + chunk]
        rep = torch.repeat_interleave(torch.arange(o.numel(), device=dev), l)
        within = torch.arange(rep.numel(), device=dev) - (torch.cumsum(l, 0) - l)[rep]
        out[d[0] + torch.arange(rep.numel(), device=dev)] = buf[o[rep] + within]
    return out, ln.to(torch.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", nargs="+", default=["join", "q67", "dup"], choices=["join", "q67", "dup"])
    ap.add_argument("--gib", type=float, nargs="+", default=[2.0, 10.0])
    ap.add_argument("--partitions", type=int, nargs="+", default=[200, 2000])
    ap.add_argument("--codec", nargs="+", default=["snappy", "lz4"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()

    import torch

    import partition_rows_hash_bench as hb
    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    dev = torch.device("cuda", 0)
    name = hb.card()
    for shape in args.shape:
        for gib in args.gib:
            gen = torch.Generator(device=dev)
            gen.manual_seed(args.seed)
            avg = hb.FIXED + 32 if shape != "q67" else 4 + 48 + 3 * 16 + 16
            n = int(gib * (1 << 30)) // avg
            if shape == "q67":
                rec, rec_len, _, starts = hb.q67_rows(torch, gen, n, dev)
            else:
                rec, rec_len, _, starts = hb.join_rows(torch, gen, 1000 if shape == "dup" else n, dev)
                if shape == "dup":
                    pick = torch.randint(0, 1000, (n,), generator=gen, device=dev)
                    rec, rec_len = gather_rows(torch, rec, starts, rec_len.long() - 4, pick, dev)
                    starts = torch.cumsum(rec_len.long(), 0) - rec_len.long() + 4
            size = rec_len.long() - 4
            order, hs = model_order(torch, rec, starts, size)
            tied, rounds = tie_stats(torch, rec, starts, size, order, hs)
            wrec, wlen = gather_rows(torch, rec, starts, size, order, dev)
            del order, hs
            for R in args.partitions:
                start = int(torch.randint(0, R, (1,), generator=gen, device=dev))
                ids = ((start + 1 + torch.arange(n, device=dev)) % R).to(torch.int32)
                for codec_name in args.codec:
                    codec = c.CODEC_BY_NAME[codec_name]
                    cap = c.partition_compress_bound(codec, 0, R, rec.numel()) + 64
                    out = {k: torch.empty(cap, dtype=torch.uint8, device=dev) for k in ("rr", "ids")}
                    t = {k: [] for k in ("step", "step_nosort", "rr_kernel", "rr_total", "ids_kernel", "ids_total")}
                    res = {}
                    for rep in range(args.reps + 1):
                        for kind in ("ids", "rr0", "rr") if rep % 2 else ("rr", "rr0", "ids"):
                            if kind == "ids":
                                r = c.partition_compress_dev(codec, wrec.data_ptr(), wrec.numel(), wlen.data_ptr(),
                                                             ids.data_ptr(), n, R, out["ids"].data_ptr(), cap,
                                                             checksum_alg=3)
                            else:
                                r = c.partition_compress_rows_round_robin_dev(
                                    codec, rec.data_ptr(), rec.numel(), rec_len.data_ptr(), n, R, start,
                                    1 if kind == "rr" else 0, out["rr"].data_ptr(), cap, checksum_alg=3)
                            tm = c.last_timing()
                            res[kind] = r
                            if rep == 0:
                                continue  # warm-up: buffers grow
                            if kind == "rr0":
                                t["step_nosort"].append(tm["dominant_ms"])
                                continue
                            t[kind + "_kernel"].append(tm["kernel_ms"])
                            t[kind + "_total"].append(tm["total_ms"])
                            if kind == "rr":
                                t["step"].append(tm["dominant_ms"])
                    # the unsorted call shares out["rr"]: the sorted one writes it once more for the comparison
                    res["rr"] = c.partition_compress_rows_round_robin_dev(
                        codec, rec.data_ptr(), rec.numel(), rec_len.data_ptr(), n, R, start, 1, out["rr"].data_ptr(),
                        cap, checksum_alg=3)
                    a, b = res["rr"], res["ids"]
                    same = (a["total"] == b["total"] and all((a[k] == b[k]).all() for k in
                                                             ("dst_off", "dst_len", "checksums", "status")) and
                            torch.equal(out["rr"][:a["total"]], out["ids"][:b["total"]]))
                    print(json.dumps({
                        "card": name, "shape": shape, "gib": gib, "records": n, "partitions": R, "start": start,
                        "codec": codec_name, "checksum": "CRC32C", "identical": bool(same),
                        "tied_records": tied, "refine_rounds_model": rounds,
                        "rr_step_ms": {"sort": hb.spread(t["step"]), "no_sort": hb.spread(t["step_nosort"])},
                        "call_kernel_ms": {"rr": hb.spread(t["rr_kernel"]), "presorted_ids": hb.spread(t["ids_kernel"])},
                        "call_total_ms": {"rr": hb.spread(t["rr_total"]), "presorted_ids": hb.spread(t["ids_total"])},
                    }), flush=True)
                    del out
                    torch.cuda.empty_cache()
                del ids
            del rec, rec_len, starts, size, wrec, wlen
            torch.cuda.empty_cache()
    c.shutdown()


if __name__ == "__main__":
    main()
