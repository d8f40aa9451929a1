#!/usr/bin/env python
"""Cost of merging a reduce task's partial-aggregate UnsafeRow records on the GPU (b2s_decompress_aggregate_rows_dev),
against decoding the same blocks and against row-sorting them.

Input: --gib GiB of device-generated, seeded rows in the shape of a grouped aggregation's shuffle (the map side's
partial aggregates, HashAggregateExec(Partial)): an 8-byte null bitset, an int64 grouping key (null in ~5 % of rows,
which form one large group on reducer 0 in both shapes) and four buffers: count (long, never null), sum (double), min (long) and max (double), each null in ~10 % of rows.  A
record ([int32 big-endian size][row]) is 52 bytes.  The rows are split into --maps map tasks; each goes through
partition_compress_dev (--codec, default snappy, + CRC32C) with the reduce id a hash of the key (nulls to reducer 0), so
that every key lands on one reducer, as Spark's hash partitioning does.  Two key shapes are run:
  many : --keys distinct keys (default: records / maps, so a key has about `maps` records, one per map)
  hot  : the same, with one key holding a --hot fraction of all rows (skew: one reducer gets a very large group)
After --warmup untimed calls, every reducer's blocks are timed three ways:
  (a) decompress_dev alone (verify + decode)
  (b) decompress_sort_rows_dev (verify + decode + framing + sort; the sort's full gather of every record)
  (c) decompress_aggregate_rows_dev (verify + decode + framing + keys + radix + aggregation)
Times are CUDA events on the library's stream (b2s_mark), per call; the aggregation step is (c)'s dominant_ms (from the
sorted indices to the written output, including its one readback).  min / median / max over the reducers and the sums
are printed.  The aggregation step's algorithmic bytes are computed here: per record, its sorted index (4 B), its key
words read twice (12 B each: a nullable int64 key is three words), its null word and four slots read (40 B), the dense
copies of the slots and null bits written and read back (2 x 36 B) and its head flag written, scanned and read (3 x 8 B);
per group, the head record read and written (2 x 52 B) and its slots and null word rewritten (40 B).  The rate is those
bytes over the step's time; its share of peak is that rate over the 3.35 TB/s HBM3 of the H100 SXM data sheet.
Validation: every reducer's output is read back, and over all reducers each key must appear exactly once, with the
count and min equal to a torch scatter reference exactly (the count mod 2^64), max equal exactly, the null bits as the
reference's, and the double sum within 1e-12 of the sum of the absolute inputs of its key (torch adds in another order).
The card's name and power limit are read in the same run.

--buffers decimal swaps the four buffers for Spark's Decimal ones, the shape of sum(decimal(28,2)) and
avg(decimal(28,2)) partials: [sum, isEmpty] and [sum, count], i.e. B2S_AGG_SUM_DECIMAL | 28 << 8 (out of line, never
null: no partial overflowed), MIN_INT32 (isEmpty, 1 in ~2 % of rows), SUM_DECIMAL | 28 << 8 and SUM_INT64 (the count).
A record is 84 bytes: the 52-byte layout's four slots, then each sum's 16 bytes (|v| < 10^15, written as all 16
big-endian bytes).  Its algorithmic bytes add, per record, the two 16-byte values read and their high words staged
(2 x 16 B), and per group the two 16-byte regions rewritten.  Validation: every key appears once, with both sums equal
to the exact per-key sum (torch adds the high and low 32-bit halves in int64; Python joins them), the count exact,
isEmpty the AND of the inputs and no null bit but the null key's.  Both buffer kinds report the largest reducer's
aggregation step per row (one warp merges its one large group).

    python tools/aggregate_rows_bench.py [--gib 2] [--maps 400] [--partitions 200] [--codec snappy] [--hot 0.05]
                                         [--buffers longs|decimal]

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

REC = 52              # size prefix + null bitset + key + count + sum + min + max
REC_DEC = 84          # size prefix + null bitset + key + sum, isEmpty, sum, count slots + two 16-byte decimals
P_DEC = 28
KEY_OFF = 8           # field 0 of the row: after the one-word null bitset
HBM_PEAK = 3.35e12    # H100 SXM data sheet


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def make_map(torch, gen, n, K, hot, R, dev):
    """n rows of one map task -> (records, rec_len u32, reduce ids u32, dense key index (K = null), fields)"""
    key = torch.randint(0, K, (n,), generator=gen, device=dev, dtype=torch.int64)
    if hot:
        key[torch.rand(n, generator=gen, device=dev) < hot] = 0
    knull = torch.rand(n, generator=gen, device=dev) < 0.05
    cnt = torch.randint(1, 100, (n,), generator=gen, device=dev, dtype=torch.int64)
    fsum = torch.randn(n, generator=gen, device=dev, dtype=torch.float64) * 1000.0
    fmin = torch.randint(-(1 << 40), 1 << 40, (n,), generator=gen, device=dev, dtype=torch.int64)
    fmax = torch.randn(n, generator=gen, device=dev, dtype=torch.float64)
    nulls = [torch.rand(n, generator=gen, device=dev) < 0.1 for _ in range(3)]  # sum, min, max
    bits = knull.to(torch.int64) | (nulls[0].to(torch.int64) << 2) | (nulls[1].to(torch.int64) << 3) | \
        (nulls[2].to(torch.int64) << 4)
    rec = torch.empty((n, REC), dtype=torch.uint8, device=dev)
    rec[:, :4] = torch.tensor([0, 0, 0, REC - 4], dtype=torch.uint8, device=dev)
    for k, col in enumerate([bits, key, cnt, fsum.view(torch.int64), fmin, fmax.view(torch.int64)]):
        rec[:, 4 + 8 * k:12 + 8 * k] = col[:, None].view(torch.uint8).view(n, 8)
    part = torch.where(knull, torch.zeros_like(key), (key * 2654435761) % R).to(torch.int32)
    dense = torch.where(knull, torch.full_like(key, K), key)
    return rec.flatten(), torch.full((n,), REC, dtype=torch.int32, device=dev), part, dense, \
        (cnt, fsum, fmin, fmax, nulls)


def make_map_decimal(torch, gen, n, K, hot, R, dev):
    """the --buffers decimal rows of one map task -> (records, rec_len u32, reduce ids u32, dense key index, fields)"""
    key = torch.randint(0, K, (n,), generator=gen, device=dev, dtype=torch.int64)
    if hot:
        key[torch.rand(n, generator=gen, device=dev) < hot] = 0
    knull = torch.rand(n, generator=gen, device=dev) < 0.05
    s1 = torch.randint(-10**15, 10**15, (n,), generator=gen, device=dev, dtype=torch.int64)
    s2 = torch.randint(-10**15, 10**15, (n,), generator=gen, device=dev, dtype=torch.int64)
    empty = (torch.rand(n, generator=gen, device=dev) < 0.02).to(torch.int64)
    cnt = torch.randint(1, 100, (n,), generator=gen, device=dev, dtype=torch.int64)
    row = REC_DEC - 4
    slot1 = torch.full((n,), (48 << 32) | 16, dtype=torch.int64, device=dev)
    slot2 = torch.full((n,), (64 << 32) | 16, dtype=torch.int64, device=dev)
    rec = torch.empty((n, REC_DEC), dtype=torch.uint8, device=dev)
    rec[:, :4] = torch.tensor([0, 0, 0, row], dtype=torch.uint8, device=dev)
    for k, col in enumerate([knull.to(torch.int64), key, slot1, empty, slot2, cnt]):
        rec[:, 4 + 8 * k:12 + 8 * k] = col[:, None].view(torch.uint8).view(n, 8)
    for k, v in enumerate([s1, s2]):  # 16 big-endian bytes: the sign, then the long
        o = 4 + 48 + 16 * k
        rec[:, o:o + 8] = torch.where(v < 0, 255, 0).to(torch.uint8)[:, None].expand(n, 8)
        rec[:, o + 8:o + 16] = v[:, None].view(torch.uint8).view(n, 8).flip(1)
    part = torch.where(knull, torch.zeros_like(key), (key * 2654435761) % R).to(torch.int32)
    dense = torch.where(knull, torch.full_like(key, K), key)
    return rec.flatten(), torch.full((n,), REC_DEC, dtype=torch.int32, device=dev), part, dense, (s1, s2, empty, cnt)


def run_shape(torch, c, args, codec, K, hot, dev, gen):
    if args.buffers == "decimal":
        return run_shape_decimal(torch, c, args, codec, K, hot, dev, gen)
    M, R = args.maps, args.partitions
    n = int(args.gib * (1 << 30)) // REC
    per = [n // M] * (M - 1) + [n - n // M * (M - 1)]
    G = K + 1
    ref_cnt = torch.zeros(G, dtype=torch.int64, device=dev)
    ref_sum = torch.zeros(G, dtype=torch.float64, device=dev)
    ref_abs = torch.zeros(G, dtype=torch.float64, device=dev)
    ref_min = torch.full((G,), 1 << 62, dtype=torch.int64, device=dev)
    ref_max = torch.full((G,), -float("inf"), dtype=torch.float64, device=dev)
    ref_has = torch.zeros((3, G), dtype=torch.int64, device=dev)
    ref_rows = torch.zeros(G, dtype=torch.int64, device=dev)
    maps, map_base, bounds, compressed = [], [], [], None
    for m in range(M):
        rec, rec_len, part, dense, (cnt, fsum, fmin, fmax, nulls) = make_map(torch, gen, per[m], K, hot, R, dev)
        ref_rows.index_add_(0, dense, torch.ones_like(dense))
        ref_cnt.index_add_(0, dense, cnt)
        ok = [~x for x in nulls]
        ref_sum.index_add_(0, dense[ok[0]], fsum[ok[0]])
        ref_abs.index_add_(0, dense[ok[0]], fsum[ok[0]].abs())
        ref_min.scatter_reduce_(0, dense[ok[1]], fmin[ok[1]], "amin")
        ref_max.scatter_reduce_(0, dense[ok[2]], fmax[ok[2]], "amax")
        for k in range(3):
            ref_has[k].index_add_(0, dense[ok[k]], torch.ones_like(dense[ok[k]]))
        bound = (c.partition_compress_bound(codec, 0, R, rec.numel()) + 255) // 256 * 256
        if compressed is None:
            compressed = torch.empty(bound * (M + 1), dtype=torch.uint8, device=dev)
        at = sum(bounds)
        assert at + bound <= compressed.numel()
        torch.cuda.synchronize()
        r = c.partition_compress_dev(codec, rec.data_ptr(), rec.numel(), rec_len.data_ptr(), part.data_ptr(), per[m],
                                     R, compressed.data_ptr() + at, bound, checksum_alg=c.CHECKSUM_CRC32C)
        assert not r["status"].any()
        maps.append(r)
        map_base.append(at)
        bounds.append(bound)
        del rec, rec_len, part, dense
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
    aggs = [(c.AGG_SUM_INT64, 16, -1), (c.AGG_SUM_FLOAT64, 24, 2), (c.AGG_MIN_INT64, 32, 3),
            (c.AGG_MAX_FLOAT64, 40, 4)]

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
        return c.decompress_sort_rows_dev(codec, compressed.data_ptr(), off, ln, scratch.data_ptr(), cap, c.KEY_INT64,
                                          KEY_OFF, 8, 0, c.CHECKSUM_CRC32C, sb, sl, ck)

    def call_c(red):
        off, ln, sb, sl, ck = blocks(red)
        return c.decompress_aggregate_rows_dev(codec, compressed.data_ptr(), off, ln, out.data_ptr(), cap,
                                               c.KEY_INT64, KEY_OFF, 8, 0, aggs, c.CHECKSUM_CRC32C, sb, sl, ck)

    for _ in range(args.warmup):
        call_a(0)
        call_b(0)
        call_c(0)
    ta, tb, tc, tagg, agg_bytes, recs_per, groups_per = [], [], [], [], [], [], []
    got_seen = torch.zeros(G, dtype=torch.int64, device=dev)
    got = {k: torch.zeros(G, dtype=torch.int64, device=dev) for k in ("bits", "cnt", "sum", "min", "max")}
    ok = True
    for red in range(R):
        ra, t_a = timed(lambda: call_a(red))
        rb, t_b = timed(lambda: call_b(red))
        rc, t_c = timed(lambda: call_c(red))
        t = c.last_timing()
        ok &= not ra["status"].any() and not rb["status"].any() and not rc["status"].any()
        ok &= rb["n_records"] == rc["n_records"] and rc["total"] == rc["n_groups"] * REC
        ta.append(t_a)
        tb.append(t_b)
        tc.append(t_c)
        tagg.append(t["dominant_ms"])
        nr, ng = rc["n_records"], rc["n_groups"]
        recs_per.append(nr)
        groups_per.append(ng)
        agg_bytes.append(nr * (4 + 24 + 40 + 72 + 24) + ng * (2 * REC + 40))
        o = out[: ng * REC].view(ng, REC)[:, 4:].contiguous().view(torch.int64).view(ng, 6)
        bits, key = o[:, 0], o[:, 1]
        dense = torch.where((bits & 1) != 0, torch.full_like(key, K), key)
        got_seen.index_add_(0, dense, torch.ones_like(dense))
        for k, col in zip(("bits", "cnt", "sum", "min", "max"), (bits, o[:, 2], o[:, 3], o[:, 4], o[:, 5])):
            got[k][dense] = col
    present = ref_rows > 0
    ok &= bool((got_seen == present.to(torch.int64)).all())
    # the reference's null bits and values; a null result has an all-zero slot
    want_bits = (ref_has[0] == 0).to(torch.int64) << 2 | (ref_has[1] == 0).to(torch.int64) << 3 | \
        (ref_has[2] == 0).to(torch.int64) << 4
    want_bits = want_bits | (torch.arange(G, device=dev) == K).to(torch.int64)
    ok_bits = bool(((got["bits"] & 0b11101) == want_bits)[present].all())
    ok_cnt = bool((got["cnt"] == ref_cnt)[present].all())
    ok_min = bool((got["min"] == ref_min)[present & (ref_has[1] > 0)].all()) and \
        bool((got["min"][present & (ref_has[1] == 0)] == 0).all())
    gmax = got["max"].view(torch.float64)
    ok_max = bool((gmax[present & (ref_has[2] > 0)] == ref_max[present & (ref_has[2] > 0)]).all()) and \
        bool((got["max"][present & (ref_has[2] == 0)] == 0).all())
    gsum = got["sum"].view(torch.float64)
    sel = present & (ref_has[0] > 0)
    err = (gsum[sel] - ref_sum[sel]).abs() / ref_abs[sel].clamp(min=1e-300)
    ok_sum = bool((err <= 1e-12).all()) and bool((got["sum"][present & (ref_has[0] == 0)] == 0).all())
    valid = ok and ok_bits and ok_cnt and ok_min and ok_max and ok_sum

    agg_s = sum(tagg) * 1e-3
    mid = sorted(range(R), key=lambda i: recs_per[i])[R // 2]
    big = max(range(R), key=lambda i: recs_per[i])
    return {
        "keys": K, "hot": hot, "records": n, "groups": int(present.sum()),
        "largest_group": int(ref_rows.max()), "compressed_bytes": sum(int(m["dst_len"].sum()) for m in maps),
        "records_per_reducer": spread(recs_per), "groups_per_reducer": spread(groups_per),
        "a_decompress_ms": spread(ta), "b_decompress_sort_rows_ms": spread(tb),
        "c_decompress_aggregate_rows_ms": spread(tc), "aggregation_step_ms": spread(tagg),
        "sum_ms": {"a_decompress": round(sum(ta), 3), "b_decompress_sort_rows": round(sum(tb), 3),
                   "c_decompress_aggregate_rows": round(sum(tc), 3), "aggregation_step": round(sum(tagg), 3)},
        "aggregation_algorithmic_bytes": sum(agg_bytes),
        "aggregation_GBps": round(sum(agg_bytes) / agg_s / 1e9, 1),
        "aggregation_share_of_3.35TBps": round(sum(agg_bytes) / agg_s / HBM_PEAK, 3),
        "median_reducer": {"records": recs_per[mid], "groups": groups_per[mid], "a_ms": round(ta[mid], 3),
                           "b_ms": round(tb[mid], 3), "c_ms": round(tc[mid], 3),
                           "aggregation_step_ms": round(tagg[mid], 3)},
        "largest_reducer": {"records": recs_per[big], "groups": groups_per[big], "c_ms": round(tc[big], 3),
                            "aggregation_step_ms": round(tagg[big], 3),
                            "aggregation_ns_per_row": round(tagg[big] * 1e6 / max(recs_per[big], 1), 1)},
        "valid": bool(valid),
        "checks": {"calls_and_groups": bool(ok), "null_bits": ok_bits, "count": ok_cnt, "min": ok_min, "max": ok_max,
                   "sum_within_1e-12": ok_sum, "max_sum_rel_err": float(err.max()) if err.numel() else 0.0},
    }


def stage_maps(torch, c, args, codec, M, R, per, make, dev, on_map):
    """every map's rows made by make(m) and partition-compressed into one device arena; on_map(fields, dense) feeds
    the reference -> (per-map results, their arena offsets, the arena)"""
    maps, map_base, bounds, compressed = [], [], [], None
    for m in range(M):
        rec, rec_len, part, dense, fields = make(m)
        on_map(fields, dense)
        bound = (c.partition_compress_bound(codec, 0, R, rec.numel()) + 255) // 256 * 256
        if compressed is None:
            compressed = torch.empty(bound * (M + 1), dtype=torch.uint8, device=dev)
        at = sum(bounds)
        assert at + bound <= compressed.numel()
        torch.cuda.synchronize()
        r = c.partition_compress_dev(codec, rec.data_ptr(), rec.numel(), rec_len.data_ptr(), part.data_ptr(), per[m],
                                     R, compressed.data_ptr() + at, bound, checksum_alg=c.CHECKSUM_CRC32C)
        assert not r["status"].any()
        maps.append(r)
        map_base.append(at)
        bounds.append(bound)
        del rec, rec_len, part, dense
    torch.cuda.empty_cache()
    return maps, map_base, compressed


def run_shape_decimal(torch, c, args, codec, K, hot, dev, gen):
    """run_shape with the Decimal buffers (module docstring, --buffers decimal)"""
    M, R = args.maps, args.partitions
    n = int(args.gib * (1 << 30)) // REC_DEC
    per = [n // M] * (M - 1) + [n - n // M * (M - 1)]
    G = K + 1
    halves = torch.zeros((4, G), dtype=torch.int64, device=dev)  # s1 lo, s1 hi, s2 lo, s2 hi
    ref_cnt = torch.zeros(G, dtype=torch.int64, device=dev)
    ref_empty = torch.ones(G, dtype=torch.int64, device=dev)
    ref_rows = torch.zeros(G, dtype=torch.int64, device=dev)

    def on_map(fields, dense):
        s1, s2, empty, cnt = fields
        ref_rows.index_add_(0, dense, torch.ones_like(dense))
        for k, v in enumerate((s1, s2)):
            halves[2 * k].index_add_(0, dense, v & 0xFFFFFFFF)
            halves[2 * k + 1].index_add_(0, dense, v >> 32)
        ref_cnt.index_add_(0, dense, cnt)
        ref_empty.scatter_reduce_(0, dense, empty, "amin")

    maps, map_base, compressed = stage_maps(torch, c, args, codec, M, R, per,
                                            lambda m: make_map_decimal(torch, gen, per[m], K, hot, R, dev), dev,
                                            on_map)

    def blocks(red):
        off = [map_base[m] + int(maps[m]["dst_off"][red]) for m in range(M)]
        ln = [int(maps[m]["dst_len"][red]) for m in range(M)]
        ck = [int(maps[m]["checksums"][red]) for m in range(M)]
        return off, ln, list(range(M + 1)), ln, ck

    biggest = max(sum(int(maps[m]["dst_len"][red]) for m in range(M)) for red in range(R))
    cap = (biggest * (1 if codec == c.CODEC_NONE else 4)) + (1 << 20)
    out = torch.empty(cap + 64, dtype=torch.uint8, device=dev)
    sum_op = c.agg_sum_decimal(P_DEC)
    aggs = [(sum_op, 16, 2), (c.AGG_MIN_INT32, 24, -1), (sum_op, 32, 4), (c.AGG_SUM_INT64, 40, -1)]

    def call_c(red):
        off, ln, sb, sl, ck = blocks(red)
        return c.decompress_aggregate_rows_dev(codec, compressed.data_ptr(), off, ln, out.data_ptr(), cap,
                                               c.KEY_INT64, KEY_OFF, 8, 0, aggs, c.CHECKSUM_CRC32C, sb, sl, ck)

    for _ in range(args.warmup):
        call_c(0)
    tc, tagg, agg_bytes, recs_per, groups_per = [], [], [], [], []
    got = {}  # dense key -> (bits, s1, isEmpty, s2, count)
    ok = True
    for red in range(R):
        c.mark(0)
        rc = call_c(red)
        c.mark(1)
        tc.append(c.marks_elapsed_ms())
        t = c.last_timing()
        ok &= not rc["status"].any() and rc["total"] == rc["n_groups"] * REC_DEC
        tagg.append(t["dominant_ms"])
        nr, ng = rc["n_records"], rc["n_groups"]
        recs_per.append(nr)
        groups_per.append(ng)
        agg_bytes.append(nr * (4 + 24 + 40 + 32 + 2 * 52 + 24) + ng * (2 * REC_DEC + 40 + 32))
        o = out[: ng * REC_DEC].view(ng, REC_DEC)[:, 4:].cpu().numpy()
        for row in o:
            word = int.from_bytes(row[0:8].tobytes(), "little")
            dk = K if word & 1 else int.from_bytes(row[8:16].tobytes(), "little", signed=True)
            vals = []
            for so in (16, 32):
                slot = int.from_bytes(row[so:so + 8].tobytes(), "little")
                p, ln = slot >> 32, slot & 0xFFFFFFFF
                vals.append(int.from_bytes(row[p:p + ln].tobytes(), "big", signed=True))
            ok &= dk not in got
            got[dk] = (word, vals[0], int.from_bytes(row[24:32].tobytes(), "little"), vals[1],
                       int.from_bytes(row[40:48].tobytes(), "little", signed=True))
    h, cnt = halves.cpu().tolist(), ref_cnt.cpu().tolist()
    emp, rows_ = ref_empty.cpu().tolist(), ref_rows.cpu().tolist()
    present = [g for g in range(G) if rows_[g]]
    ok_keys = sorted(got) == present
    ok_sum = ok_cnt = ok_bits = True
    for g in present:
        if g not in got:
            continue
        word, v1, e, v2, k = got[g]
        ok_sum &= v1 == h[1][g] * 2**32 + h[0][g] and v2 == h[3][g] * 2**32 + h[2][g]
        ok_cnt &= k == cnt[g] and e == emp[g]
        ok_bits &= (word & 0b10101) == (1 if g == K else 0)
    valid = ok and ok_keys and ok_sum and ok_cnt and ok_bits
    agg_s = sum(tagg) * 1e-3
    mid = sorted(range(R), key=lambda i: recs_per[i])[R // 2]
    big = max(range(R), key=lambda i: recs_per[i])
    return {
        "buffers": "decimal", "keys": K, "hot": hot, "records": n, "groups": len(present),
        "largest_group": max(rows_), "compressed_bytes": sum(int(m["dst_len"].sum()) for m in maps),
        "records_per_reducer": spread(recs_per), "groups_per_reducer": spread(groups_per),
        "c_decompress_aggregate_rows_ms": spread(tc), "aggregation_step_ms": spread(tagg),
        "sum_ms": {"c_decompress_aggregate_rows": round(sum(tc), 3), "aggregation_step": round(sum(tagg), 3)},
        "aggregation_algorithmic_bytes": sum(agg_bytes),
        "aggregation_GBps": round(sum(agg_bytes) / agg_s / 1e9, 1),
        "aggregation_share_of_3.35TBps": round(sum(agg_bytes) / agg_s / HBM_PEAK, 3),
        "median_reducer": {"records": recs_per[mid], "groups": groups_per[mid], "c_ms": round(tc[mid], 3),
                           "aggregation_step_ms": round(tagg[mid], 3)},
        "largest_reducer": {"records": recs_per[big], "groups": groups_per[big], "c_ms": round(tc[big], 3),
                            "aggregation_step_ms": round(tagg[big], 3),
                            "aggregation_ns_per_row": round(tagg[big] * 1e6 / max(recs_per[big], 1), 1)},
        "valid": bool(valid),
        "checks": {"calls_and_groups": bool(ok), "keys_once": ok_keys, "sums_exact": ok_sum,
                   "count_and_isEmpty": ok_cnt, "null_bits": ok_bits},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=2.0)
    ap.add_argument("--maps", type=int, default=400)
    ap.add_argument("--partitions", type=int, default=200)
    ap.add_argument("--codec", default="snappy", choices=["none", "lz4", "snappy", "zstd"])
    ap.add_argument("--keys", type=int, default=0, help="distinct keys (0: records / maps)")
    ap.add_argument("--hot", type=float, default=0.05)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--buffers", default="longs", choices=["longs", "decimal"],
                    help="longs: count, double sum, long min, double max; decimal: Sum / Average decimal buffers")
    args = ap.parse_args()

    import torch

    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    codec = c.CODEC_NONE if args.codec == "none" else c.CODEC_BY_NAME[args.codec]
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev)
    gen.manual_seed(args.seed)
    rec = REC if args.buffers == "longs" else REC_DEC
    K = args.keys or max(1, int(args.gib * (1 << 30)) // rec // args.maps)
    shapes = {"many": run_shape(torch, c, args, codec, K, 0.0, dev, gen),
              "hot": run_shape(torch, c, args, codec, K, args.hot, dev, gen)}
    result = {"card": card(), "buffers": args.buffers, "codec": args.codec, "maps": args.maps,
              "partitions": args.partitions, "gib": args.gib, "shapes": shapes,
              "valid": all(s["valid"] for s in shapes.values())}
    print(json.dumps(result, indent=1))
    c.shutdown()


if __name__ == "__main__":
    main()
