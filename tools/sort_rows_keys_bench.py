#!/usr/bin/env python
"""Cost of sorting and aggregating a reduce task's UnsafeRow records by a composite key on the GPU
(b2s_decompress_sort_rows_keys_dev / b2s_decompress_aggregate_rows_keys_dev), against decoding the same blocks and
against the single-key row sort.

Two workloads, each --rows seeded rows over --maps map tasks and --partitions reducers (a map's rows of one reducer are
one block: --codec, default snappy, + CRC32C), the reducer a hash of the key:
  q67  : partial-aggregate rows of a GROUP BY of eight columns, TPC-DS q67's shape: four strings of 5-50 bytes
         (i_category, i_class, i_brand, i_product_name: a few category / class prefixes shared by many values) and four
         ints, then a count and a sum buffer (longs).  --groups distinct keys, so a key has about rows / groups rows.
         --q67-decimal adds q67's real buffers to the same rows: sum(ss_sales_price * ss_quantity)'s decimal(28,2)
         [sum, isEmpty], the sum out of line (BigInteger.toByteArray of the long sum x 10^17, 1..9 bytes, in a 16-byte
         region) and isEmpty false; the aggregation is then also timed with those two buffers
         (B2S_AGG_SUM_DECIMAL | 28 << 8, MIN_INT32) and every merged sum checked against the long sum x 10^17.
  join : the build side of a sort-merge join on (string id, int): a 16-40 byte id with a shared 12-byte prefix, an int,
         and two longs (the second used for the two-INT64 comparison below).
  window: q67's window input, rank() over (partition by i_category order by sumsales desc): i_category (one of ten
         names, or null) and sumsales, a nullable decimal(28,2) (out of line, 1..16 bytes), plus a long.  The exchange
         hashes i_category, so only the reducers holding a category have rows, and only they are timed.
Strings sit in a 56-byte area per column after the fixed fields (rows are fixed-length, slots hold the real sizes).
Per reducer, after --warmup untimed calls, CUDA-event times (b2s_last_timing.kernel_ms: the whole call on the device):
  decode   : decompress_dev alone (verify + decode)
  keys     : the composite-key call; framing (its dominant_ms for the sort)
  first    : the same rows sorted by one INT32 column (resolved by the first pass: no refinement)
  agg      : q67 only, the composite-key aggregation; its aggregation step is dominant_ms
  agg_dec  : q67 with --q67-decimal, the same with the decimal [sum, isEmpty] buffers instead of the longs
  i64x2    : join only, the two-INT64 composite beside the single-INT64 row sort on the same rows
  window   : window only, the sort by (i_category ASC NULLS FIRST, sumsales DESC NULLS LAST), as the WindowExec's
             SortExec asks; asc: the same columns ASC NULLS FIRST; i64: a one-INT64 row sort of the same rows.  Every
             output is checked against a Python sort of the reducer's rows.
Refinement rounds and the records tied in each are counted by a CPU model of the key encoding (20 bytes first, then 16
per round), which also validates every output byte against a Python sort (and the aggregation's groups and sums).
The card's name and power limit are read in the same run.

    python tools/sort_rows_keys_bench.py [--rows 1000000] [--maps 400] [--partitions 200] [--codec snappy]
                                         [--q67-decimal]

Prints one JSON document.
"""
import argparse
import functools
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STRING, KEY_INT32, KEY_INT64, DECIMAL = 3, 1, 2, 9
DESC, NULLS_LAST = 1 << 8, 1 << 9
CATEGORIES = [b"Books", b"Children", b"Electronics", b"Home", b"Jewelry", b"Men", b"Music", b"Shoes", b"Sports",
              b"Women"]
SLOT = 56  # bytes of string area per string column


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3),
            "sum": round(sum(xs), 3)}


def strings(rng, n, prefixes, lo, hi):
    """n values: a prefix from the list, then random letters up to a length in [lo, hi]"""
    pre = rng.integers(0, len(prefixes), n)
    ln = rng.integers(lo, hi + 1, n)
    out = np.zeros((n, SLOT), np.uint8)
    letters = rng.integers(97, 123, (n, SLOT), dtype=np.uint8)
    for k, p in enumerate(prefixes):
        out[pre == k, :len(p)] = np.frombuffer(p, np.uint8)
    plen = np.array([len(prefixes[k]) for k in pre])
    cols = np.arange(SLOT)[None, :]
    fill = (cols >= plen[:, None]) & (cols < ln[:, None])
    out[fill] = letters[fill]
    return out, np.maximum(ln, plen)


def to_byte_array(x):
    """java.math.BigInteger.toByteArray"""
    return x.to_bytes((x if x >= 0 else ~x).bit_length() // 8 + 1, "big", signed=True)


def make_rows(rng, shape, n, groups, decimal=False):
    """-> (rows uint8 [n, L], key columns [(type, off, len, null field)], aggs, partition key, decimal aggs (q67 with
    decimal: [sum, isEmpty] after the long buffers, the sum's 16 bytes after the strings; else []))"""
    if shape == "q67":
        g = rng.integers(0, groups, n)  # the group of each row: its key values come from the group id
        grng = np.random.default_rng(7)
        cat = [b"Books", b"Electronics", b"Home", b"Sports", b"Women", b"Men", b"Music", b"Children"]
        cls = [b"fiction/", b"computers/", b"accessories/", b"outdoor/"]
        s_vals = [strings(grng, groups, cat, 5, 11), strings(grng, groups, cls, 8, 20),
                  strings(grng, groups, [b"brandbrand#", b"corpcorp#", b"importoimporto #"], 12, 30),
                  strings(grng, groups, [b"ationationought", b"eingeingpri", b"barbarese"], 20, 50)]
        i_vals = grng.integers(-2**31, 2**31, (groups, 4))
        n_str, n_int, n_agg = 4, 4, 2
    else:
        g = np.arange(n)
        s_vals = [strings(rng, n, [b"AAAAAAAABBBB"], 16, 40)]
        i_vals = np.stack([rng.integers(-100, 100, n), rng.integers(-2**62, 2**62, n), rng.integers(0, 8, n)], 1)
        n_str, n_int, n_agg = 1, 3, 0
    n_dec = 2 if shape == "q67" and decimal else 0
    fields = n_str + n_int + n_agg + n_dec
    fixed = 8 + 8 * fields
    L = fixed + SLOT * n_str + (16 if n_dec else 0)
    rows = np.zeros((n, L), np.uint8)
    keys = []
    for s in range(n_str):
        data, ln = s_vals[s]
        so = fixed + SLOT * s
        rows[:, so:so + SLOT] = data[g]
        slot = (np.uint64(so) << np.uint64(32)) | ln[g].astype(np.uint64)
        rows[:, 8 + 8 * s:16 + 8 * s] = slot.view(np.uint8).reshape(n, 8)
        keys.append((STRING, 8 + 8 * s, 8, -1))
    for k in range(n_int):
        o = 8 + 8 * (n_str + k)
        v = i_vals[g, k] if shape == "q67" else i_vals[:, k]
        if shape == "q67" or k == 0:
            rows[:, o:o + 4] = v.astype(np.int32).view(np.uint8).reshape(n, 4)
            keys.append((KEY_INT32, o, 4, -1))
        else:
            rows[:, o:o + 8] = v.astype(np.int64).view(np.uint8).reshape(n, 8)
    aggs = []
    for a in range(n_agg):
        o = 8 + 8 * (n_str + n_int + a)
        rows[:, o:o + 8] = (np.ones(n, np.int64) if a == 0 else rng.integers(-1000, 1000, n)).view(np.uint8).reshape(n, 8)
        aggs.append((0, o, -1))
    dec_aggs = []
    if n_dec:  # the long sum x 10^17 as a decimal(28,2) sum: its minimal bytes, one table row per long value
        lsum = rows[:, aggs[1][1]:aggs[1][1] + 8].copy().view(np.int64).ravel()
        table = np.zeros((2001, 16), np.uint8)
        size = np.zeros(2001, np.uint64)
        for v in range(-1000, 1001):
            b = to_byte_array(v * 10**17)
            table[v + 1000, :len(b)] = np.frombuffer(b, np.uint8)
            size[v + 1000] = len(b)
        o, region = 8 + 8 * (n_str + n_int + n_agg), fixed + SLOT * n_str
        rows[:, region:region + 16] = table[lsum + 1000]
        slot = (np.uint64(region) << np.uint64(32)) | size[lsum + 1000]
        rows[:, o:o + 8] = slot.view(np.uint8).reshape(n, 8)
        dec_aggs = [(9 | 28 << 8, o, n_str + n_int + n_agg), (2, o + 8, -1)]  # SUM_DECIMAL(28), MIN_INT32 (isEmpty 0)
    if shape == "join":  # sort key (string id, int); the two longs for the INT64 comparison
        keys = [keys[0], keys[1]]
    return rows, keys, aggs, g, dec_aggs


def window_rows(rng, n):
    """-> (rows uint8 [n, 64], category id per row (len(CATEGORIES): null), sumsales per row (None: null))
    row: null word (bit 1 i_category, bit 2 sumsales), i_category slot, sumsales slot, a long, then 16 bytes of string
    and 16 of decimal"""
    cat = rng.integers(0, len(CATEGORIES) + 1, n)
    cents = rng.integers(0, 10**9, n) * rng.choice(np.array([1, 1, 1, 10**9]), n)  # a few wider than 8 bytes
    null_sales = rng.random(n) < 0.01
    rows = np.zeros((n, 64), np.uint8)
    rows[:, 24:32] = rng.integers(-2**62, 2**62, n).view(np.uint8).reshape(n, 8)
    word = np.where(cat == len(CATEGORIES), 2, 0) | np.where(null_sales, 4, 0)
    rows[:, 0:8] = word.astype(np.uint64).view(np.uint8).reshape(n, 8)
    sales = []
    for i in range(n):
        if cat[i] < len(CATEGORIES):
            b = CATEGORIES[cat[i]]
            rows[i, 32:32 + len(b)] = np.frombuffer(b, np.uint8)
            rows[i, 8:16] = np.frombuffer(((32 << 32) | len(b)).to_bytes(8, "little"), np.uint8)
        if null_sales[i]:
            sales.append(None)
            continue
        v = int(cents[i]) * (1 if i % 7 else -1)
        b = v.to_bytes((v if v >= 0 else ~v).bit_length() // 8 + 1, "big", signed=True)  # BigInteger.toByteArray
        rows[i, 48:48 + len(b)] = np.frombuffer(b, np.uint8)
        rows[i, 16:24] = np.frombuffer(((48 << 32) | len(b)).to_bytes(8, "little"), np.uint8)
        sales.append(v)
    return rows, cat, sales


def col_value(row, c):
    kt, ko, kl, _ = c
    if kt == STRING:
        slot = int.from_bytes(row[ko:ko + 8], "little")
        return bytes(row[slot >> 32:(slot >> 32) + (slot & 0xFFFFFFFF)])
    return int.from_bytes(row[ko:ko + kl], "little", signed=True)


def encoded_len(key):
    return sum(9 * max(1, (len(v) + 7) // 8) if isinstance(v, bytes) else 4 for v in key)


def encode(key):
    out = b""
    for v in key:
        if isinstance(v, bytes):
            groups = max(1, (len(v) + 7) // 8)
            for g in range(groups):
                part = v[8 * g:8 * g + 8]
                out += part + bytes(8 - len(part)) + bytes([9 if g + 1 < groups else len(part)])
        else:
            out += ((v + 2**31) % 2**32).to_bytes(4, "big")
    return out


def rounds(enc_sorted):
    """records tied at each refinement round: runs of equal first-d bytes of 2+ records whose keys go on past d"""
    per, d = [], 20
    while True:
        tied, j, n = 0, 0, len(enc_sorted)
        while j < n:
            e = j + 1
            while e < n and enc_sorted[e][:d] == enc_sorted[j][:d]:
                e += 1
            if e - j > 1 and len(enc_sorted[j]) > d:
                tied += e - j
            j = e
        if not tied:
            return per
        per.append(tied)
        d += 16


def stage(c, codec, alg, plain):
    """one reducer's blocks (plain: one stream per map) compressed, checksummed and put on the device -> (the _dev
    calls' leading arguments, their slice keywords, decoded bytes, d_src, d_dst)"""
    lens = np.array([len(b) for b in plain], np.uint64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    src = np.frombuffer(b"".join(plain), np.uint8)
    if codec:
        dst = np.zeros(sum(c.compress_bound(codec, 0, int(x)) for x in lens) + 64, np.uint8)
        cr = c.compress_packed(codec, src, offs, lens, dst, 0, 0)
        arena, off, ln = dst[:max(cr["total"], 1)], cr["dst_off"], cr["dst_len"]
    else:
        arena, off, ln = src, offs, lens
    ck = c.checksum_packed(alg, arena, off, ln)
    sb, sl = np.arange(len(plain) + 1, dtype=np.uint32), np.array(ln, np.uint64)
    total = int(lens.sum())
    d_src, d_dst = c.dev_alloc(max(arena.size, 1)), c.dev_alloc(max(total, 1))
    c.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
    sk = dict(checksum_alg=alg, slice_base=sb, slice_len=sl, slice_checksum=ck)
    return (codec, d_src, off, ln, d_dst, total), sk, total, d_src, d_dst


def timed_call(c, warmup, f, *a, **k):
    for _ in range(warmup):
        f(*a, **k)
    res = f(*a, **k)
    return res, c.last_timing()


def window(c, args, rng, codec, alg):
    """the window shape (module docstring): per non-empty reducer the flagged sort, the ASC one and one INT64"""
    rows, cat, sales = window_rows(rng, args.rows)
    L = rows.shape[1]
    red = (cat * 2654435761 % 2**32) % args.partitions
    mp = rng.integers(0, args.maps, args.rows)
    order = np.lexsort((mp, red))
    prefix = L.to_bytes(4, "big")
    sorts = {"window": [(STRING, 8, 8, 1), (DECIMAL | DESC | NULLS_LAST, 16, 8, 2)],
             "asc": [(STRING, 8, 8, 1), (DECIMAL, 16, 8, 2)]}
    stats, ok, sizes = {k: [] for k in ("decode", "window", "asc", "i64")}, True, []
    for r in sorted(set(red.tolist())):
        idx = order[red[order] == r]
        maps_of = mp[idx]
        plain = [b"".join(prefix + rows[i].tobytes() for i in idx[maps_of == m]) for m in range(args.maps)]
        ins = [i for m in range(args.maps) for i in idx[maps_of == m]]  # block order
        a, sk, total, d_src, d_dst = stage(c, codec, alg, plain)
        _, t = timed_call(c, args.warmup, c.decompress_dev, *a, **sk)
        stats["decode"].append(t["kernel_ms"])
        got = np.zeros(max(total, 1), np.uint8)
        models = {  # Python sort keys: category ASC NULLS FIRST, then sumsales DESC NULLS LAST / ASC NULLS FIRST
            "window": lambda i: (cat[i] != len(CATEGORIES), CATEGORIES[cat[i]] if cat[i] < len(CATEGORIES) else b"",
                                 sales[i] is None, -(sales[i] or 0)),
            "asc": lambda i: (cat[i] != len(CATEGORIES), CATEGORIES[cat[i]] if cat[i] < len(CATEGORIES) else b"",
                              sales[i] is not None, sales[i] or 0),
            "i64": lambda i: int(rows[i, 24:32].view(np.int64)[0])}
        for name, model in models.items():
            if name == "i64":
                res, t = timed_call(c, args.warmup, c.decompress_sort_rows_dev, *a, KEY_INT64, 24, 8, -1, **sk)
            else:
                res, t = timed_call(c, args.warmup, c.decompress_sort_rows_keys_dev, *a, sorts[name], **sk)
            stats[name].append(t["kernel_ms"])
            c.dev_memcpy(got.ctypes.data, d_dst, total, 2)
            want = b"".join(prefix + rows[i].tobytes() for i in sorted(ins, key=model))  # stable
            ok &= got[:total].tobytes() == want and res["n_records"] == len(ins)
        sizes.append(len(ins))
        c.dev_free(d_src)
        c.dev_free(d_dst)
    return {"reducers": len(sizes), "rows_per_reducer": spread(sizes), "validated": bool(ok),
            "ms_per_reducer": {k: spread(v) for k, v in stats.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--maps", type=int, default=400)
    ap.add_argument("--partitions", type=int, default=200)
    ap.add_argument("--groups", type=int, default=50_000)
    ap.add_argument("--codec", default="snappy", choices=["none", "lz4", "snappy", "zstd"])
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--reducers", type=int, default=0, help="reducers timed (0: all)")
    ap.add_argument("--shapes", default="q67,join,window")
    ap.add_argument("--q67-decimal", action="store_true", help="also aggregate q67 with its decimal [sum, isEmpty]")
    args = ap.parse_args()
    import spark_s3_shuffle_b200 as pkg
    c = pkg.capi
    c.init()
    codec = c.CODEC_BY_NAME.get(args.codec, c.CODEC_NONE)
    alg = c.CHECKSUM_CRC32C
    out = {"card": card(), "rows": args.rows, "maps": args.maps, "partitions": args.partitions, "codec": args.codec}
    rng = np.random.default_rng(args.seed)
    timed = functools.partial(timed_call, c, args.warmup)
    for shape in [x for x in args.shapes.split(",") if x in ("q67", "join")]:
        rows, keys, aggs, g, dec_aggs = make_rows(rng, shape, args.rows, args.groups, args.q67_decimal)
        L = rows.shape[1]
        red = (g * 2654435761 % 2**32) % args.partitions
        mp = rng.integers(0, args.maps, args.rows)
        order = np.lexsort((mp, red))  # reducer, then map; stable within
        R = args.reducers or args.partitions
        stats = {k: [] for k in ("decode", "keys", "framing", "first", "agg", "agg_step", "agg_dec", "agg_dec_step",
                                 "i64x2", "i64")}
        round_counts, ok = [], True
        prefix = L.to_bytes(4, "big")  # every record's size prefix
        ik = next(k for k in keys if k[0] == KEY_INT32)
        for r in range(R):
            idx = order[red[order] == r]
            maps_of = mp[idx]
            plain = []
            for m in range(args.maps):
                sel = rows[idx[maps_of == m]]
                recs = np.concatenate([np.tile(np.frombuffer(prefix, np.uint8), (sel.shape[0], 1)), sel], 1)
                plain.append(recs.tobytes())
            a, sk, total, d_src, d_dst = stage(c, codec, alg, plain)
            _, t = timed(c.decompress_dev, *a, **sk)
            stats["decode"].append(t["kernel_ms"])
            _, t = timed(c.decompress_sort_rows_dev, *a, KEY_INT32, ik[1], 4, -1, **sk)
            stats["first"].append(t["kernel_ms"])
            res, t = timed(c.decompress_sort_rows_keys_dev, *a, keys, **sk)
            stats["keys"].append(t["kernel_ms"])
            stats["framing"].append(t["dominant_ms"])
            got = np.zeros(max(total, 1), np.uint8)
            if total:
                c.dev_memcpy(got.ctypes.data, d_dst, total, 2)
            # the model: rows of this reducer in block order, stably sorted by the key
            blk = np.frombuffer(b"".join(plain), np.uint8).reshape(-1, 4 + L)[:, 4:] if total else np.zeros((0, L))
            kv = [tuple(col_value(bytes(row), k) for k in keys) for row in blk]
            srt = sorted(range(len(kv)), key=lambda i: kv[i])
            want = b"".join(prefix + bytes(blk[i]) for i in srt)
            ok &= got[:total].tobytes() == want and res["n_records"] == len(kv)
            round_counts.append(rounds([encode(kv[i]) for i in srt]))
            if shape == "q67":
                res, t = timed(c.decompress_aggregate_rows_keys_dev, *a, keys, aggs, **sk)
                stats["agg"].append(t["kernel_ms"])
                stats["agg_step"].append(t["dominant_ms"])
                ngroups = len(set(kv))
                ok &= res["n_groups"] == ngroups
                if res["total"]:
                    c.dev_memcpy(got.ctypes.data, d_dst, res["total"], 2)
                outrows = got[:res["total"]].reshape(-1, 4 + L)[:, 4:]
                cnt = outrows[:, aggs[0][1]:aggs[0][1] + 8].copy().view(np.int64).ravel()
                ok &= int(cnt.sum()) == len(kv)
                if dec_aggs:
                    res, t = timed(c.decompress_aggregate_rows_keys_dev, *a, keys, dec_aggs, **sk)
                    stats["agg_dec"].append(t["kernel_ms"])
                    stats["agg_dec_step"].append(t["dominant_ms"])
                    ok &= res["n_groups"] == ngroups
                    if res["total"]:
                        c.dev_memcpy(got.ctypes.data, d_dst, res["total"], 2)
                    want_sum = {}
                    lo = aggs[1][1]
                    for k, row in zip(kv, blk):
                        want_sum[k] = want_sum.get(k, 0) + int(row[lo:lo + 8].view(np.int64)[0])
                    do = dec_aggs[0][1]
                    for row in got[:res["total"]].reshape(-1, 4 + L)[:, 4:]:
                        slot = int(row[do:do + 8].view(np.uint64)[0])
                        p, ln = slot >> 32, slot & 0xFFFFFFFF
                        v = int.from_bytes(row[p:p + ln].tobytes(), "big", signed=True)
                        ok &= v == want_sum.get(tuple(col_value(bytes(row), k) for k in keys)) * 10**17
            else:
                _, t = timed(c.decompress_sort_rows_dev, *a, KEY_INT64, keys[1][1] + 8, 8, -1, **sk)
                stats["i64"].append(t["kernel_ms"])
                i64x2 = [(KEY_INT64, keys[1][1] + 8, 8, -1), (KEY_INT64, keys[1][1] + 16, 8, -1)]
                _, t = timed(c.decompress_sort_rows_keys_dev, *a, i64x2, **sk)
                stats["i64x2"].append(t["kernel_ms"])
            c.dev_free(d_src)
            c.dev_free(d_dst)
        n_rounds = [len(x) for x in round_counts]
        out[shape] = {
            "reducers": R, "validated": bool(ok),
            "ms_per_reducer": {k: spread(v) for k, v in stats.items() if v},
            "refinement_rounds": spread(n_rounds),
            "tied_records_per_round_median_reducer": round_counts[sorted(range(R), key=lambda i: n_rounds[i])[R // 2]],
        }
    if "window" in args.shapes.split(","):
        out["window"] = window(c, args, rng, codec, alg)
    c.shutdown()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
