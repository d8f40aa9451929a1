#!/usr/bin/env python
"""Cost of a sort-merge-join reducer on the GPU: b2s_decompress_join_rows_keys_dev over a reducer's two shuffled sides,
against today's GPU path for the same blocks, two b2s_decompress_sort_rows_keys_dev calls (one per side), which leave
the merge and the joined rows to the JVM.

The shape is SURVEY config 4: --maps map tasks and --partitions reducers, one Snappy .data block per map and reducer
with CRC32C checksums; each timed reducer's blocks are built for that reducer alone (its share of --gib GiB of left
rows).  Workloads:
  a : fact x dimension.  Left rows of 52..116 bytes ([long key, long, int, double, string of 0..64 bytes]) with keys
      uniform over --keys; the right side is the unique-key dimension ([long key, long, string of 8..24 bytes]) of the
      reducer's share of those keys.
  b : the same with a (string, int) key: a 16-byte string made from the key and an int of key mod 7.
  c : a: plus a skewed key: 1 % of each reducer's left rows carry one hot key that 2000 right rows match (many to
      many: 2000 joined rows per hot left row).
  d : a, with partners missing on both sides: no left row carries 25 % of the dimension's keys, and 10 % of the left
      rows carry a key outside the dimension, so right and full outer joins emit null-side rows.
  e : b with both key columns null-safe (<=>, the keys of an INTERSECT or EXCEPT) and each of them null in 5 % of the
      rows on both sides, so about 10 % of the keys hold a null; run it as left_semi and left_anti.  Its two sorts
      take the same columns as plain ones (the sort calls take no null-safe flag).
--join-types (inner, left_outer, left_semi, left_anti, right_outer, full_outer, existence; default inner) are joined on
the same blocks.  Every timed reducer's output is checked against the model (tests/outer_join_model.py, and
tests/null_safe_join_model.py for workload e and the existence join) before it is timed.  Per
reducer, after one untimed call of each path, each path is timed once (b2s_last_timing: kernel_ms = the whole call on
the device, dominant_ms = the join step); the sorts' kernel_ms are summed over the two calls.  The card's name and
power limit are read in the same run.  --model-cache DIR keeps each checked output's length and SHA-256 there, so
runs over the same blocks (two builds alternated) check against the model without recomputing it.

    python tools/join_rows_bench.py [--gib 2] [--maps 400] [--partitions 200] [--reducers 3] [--workloads a,b,c]
                                    [--join-types inner]

Prints one JSON document.
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SNAPPY, CRC32C = 2, 3
INT64, INT32, STRING = 2, 1, 3
FIXED, VAR = 0, 1
JOIN_TYPES = {"inner": 0, "left_outer": 1, "left_semi": 2, "left_anti": 3, "right_outer": 5, "full_outer": 6,
              "existence": 8}
NULL_SAFE = 1 << 10


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def rows_of(slots, var, rng):
    """UnsafeRows of nf < 64 fields without nulls, framed ([int32 big-endian size][row]) in input order.  slots: (n,
    nf) uint64 slot values; var: {field: (n,) lengths (multiples of 8) or (n, L) uint8 contents} — a VAR field's slot
    is set here to its offset and size, its bytes random unless given.  -> (uint8 records, uint32 record lengths)"""
    n, nf = slots.shape
    fixed = 8 + 8 * nf
    fields = sorted(var)
    lens = np.stack([var[f] if var[f].ndim == 1 else np.full(n, var[f].shape[1]) for f in fields], 1).astype(np.int64)
    size = fixed + lens.sum(1)
    starts = np.concatenate([[0], np.cumsum(4 + size)[:-1]])
    out = np.zeros(int((4 + size).sum()), np.uint8)
    for combo in np.unique(lens, axis=0):
        sel = np.nonzero((lens == combo).all(1))[0]
        w = fixed + int(combo.sum())
        rec = np.zeros((sel.size, 4 + w), np.uint8)
        rec[:, :4] = np.frombuffer(w.to_bytes(4, "big"), np.uint8)
        s = slots[sel].copy()
        at = fixed
        for f, L in zip(fields, combo):
            s[:, f] = (np.uint64(at) << np.uint64(32)) | np.uint64(L)
            body = var[f][sel] if var[f].ndim == 2 else rng.integers(97, 123, (sel.size, int(L)), dtype=np.uint8)
            rec[:, 4 + at:4 + at + int(L)] = body
            at += int(L)
        rec[:, 12:12 + 8 * nf] = s.view(np.uint8).reshape(sel.size, 8 * nf)
        out[(starts[sel][:, None] + np.arange(4 + w)).reshape(-1)] = rec.reshape(-1)
    return out, (4 + size).astype(np.uint32)


def set_nulls(records, rec_len, fields, rate, rng):
    """sets each of fields' null bits (all in the first null word) in a share rate of the framed rows"""
    starts = np.concatenate([[0], np.cumsum(rec_len.astype(np.int64))[:-1]])
    bits = np.zeros(rec_len.size, np.uint8)
    for f in fields:
        bits |= ((rng.random(rec_len.size) < rate) << f).astype(np.uint8)
    records[starts + 4] |= bits


def key_string(keys):
    """16 bytes: "cust" and the key's 12 decimal digits"""
    digits = (keys[:, None] // 10 ** np.arange(11, -1, -1, dtype=np.int64)) % 10 + 48
    return np.concatenate([np.tile(np.frombuffer(b"cust", np.uint8), (keys.size, 1)), digits.astype(np.uint8)], 1)


def reducer_sides(rng, workload, n_left, keys, partitions, red):
    """the reducer's left and right rows -> ((records, rec_len, key columns, field kinds) per side)"""
    share = np.arange(red, keys, partitions, dtype=np.int64)  # the dimension keys that hash here
    lk = rng.choice(share, n_left)
    rk = rng.permutation(share)
    if workload == "d":  # the first quarter of rk has no left row; a tenth of the left rows no dimension row
        lk = rng.choice(rk[rk.size // 4:], n_left)
        lk[rng.random(n_left) < 0.1] += keys
    if workload == "c":
        hot = int(share[0])
        lk[rng.random(n_left) < 0.01] = hot
        rk = np.concatenate([rk, np.full(1999, hot)])
        rk = rk[rng.permutation(rk.size)]
    n_r = rk.size
    l_slots = np.zeros((n_left, 5), np.uint64)
    r_slots = np.zeros((n_r, 3), np.uint64)
    l_slots[:, 1] = rng.integers(0, 1 << 62, n_left).astype(np.uint64)
    l_slots[:, 2] = rng.integers(0, 1 << 31, n_left).astype(np.uint64)
    l_slots[:, 3] = rng.random(n_left).view(np.uint64)
    r_slots[:, 1] = rng.integers(0, 1 << 62, n_r).astype(np.uint64)
    l_var = {4: 8 * rng.integers(0, 9, n_left)}
    r_var = {2: 8 * rng.integers(1, 4, n_r)}
    if workload in "be":
        l_var[0] = key_string(lk)
        r_var[0] = key_string(rk)
        l_slots[:, 2] = (lk % 7).astype(np.uint64)
        r_slots[:, 1] = (rk % 7).astype(np.uint64)
        lkeys, rkeys = [(STRING, 8, 8, -1), (INT32, 24, 4, -1)], [(STRING, 8, 8, -1), (INT32, 16, 4, -1)]
    else:
        l_slots[:, 0] = lk.astype(np.uint64)
        r_slots[:, 0] = rk.astype(np.uint64)
        lkeys, rkeys = [(INT64, 8, 8, -1)], [(INT64, 8, 8, -1)]
    lkind = [VAR if f in l_var else FIXED for f in range(5)]
    rkind = [VAR if f in r_var else FIXED for f in range(3)]
    left, right = rows_of(l_slots, l_var, rng), rows_of(r_slots, r_var, rng)
    if workload == "e":  # the key columns are fields 0 and 2 on the left, 0 and 1 on the right
        set_nulls(*left, (0, 2), 0.05, rng)
        set_nulls(*right, (0, 1), 0.05, rng)
        lkeys = [(STRING | NULL_SAFE, 8, 8, 0), (INT32 | NULL_SAFE, 24, 4, 2)]
        rkeys = [(STRING | NULL_SAFE, 8, 8, 0), (INT32 | NULL_SAFE, 16, 4, 1)]
    return ((*left, lkeys, lkind), (*right, rkeys, rkind))


def blocks(capi, records, rec_len, maps, rng):
    """the records dealt to maps blocks (map m's rows for this reducer), Snappy-compressed with CRC32C checksums"""
    ends = np.cumsum(rec_len.astype(np.int64))
    starts = ends - rec_len
    cut = np.sort(rng.integers(0, rec_len.size + 1, maps - 1))
    bounds = np.concatenate([[0], cut, [rec_len.size]])
    plain = [records[starts[a]:starts[a]] if a == b else records[starts[a]:ends[b - 1]]
             for a, b in zip(bounds[:-1], bounds[1:])]
    lens = np.array([p.size for p in plain], np.uint64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    src = np.concatenate(plain) if lens.sum() else np.zeros(1, np.uint8)
    bound = sum(capi.compress_bound(SNAPPY, 0, int(x)) for x in lens) + 64
    dst = np.zeros(bound, np.uint8)
    r = capi.compress_packed(SNAPPY, src, offs, lens, dst, 0, 0)
    ck = capi.checksum_packed(CRC32C, dst, r["dst_off"], r["dst_len"])
    return [p.tobytes() for p in plain], dst[:r["total"]], r["dst_off"], r["dst_len"], ck


def run(capi, args, workload, red, d_src, d_dst, cap):
    import null_safe_join_model
    import outer_join_model
    rng = np.random.default_rng(1000 * red + ord(workload))
    n_left = int(args.gib * 2**30 / 84 / args.partitions)
    (lrec, llen, lkeys, lkind), (rrec, rlen, rkeys, rkind) = reducer_sides(rng, workload, n_left, args.keys,
                                                                           args.partitions, red)
    lplain, la, lo, ll, lc = blocks(capi, lrec, llen, args.maps, rng)
    rplain, ra, ro, rl, rc = blocks(capi, rrec, rlen, args.maps, rng)
    arena = np.concatenate([la, ra])
    off = np.concatenate([lo, ro + np.uint64(la.size)])
    ln = np.concatenate([ll, rl])
    ck = np.concatenate([lc, rc])
    n = off.size
    sb, sl = np.arange(n + 1, dtype=np.uint32), ln.astype(np.uint64)
    capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)

    def join(jt):
        r = capi.decompress_join_rows_keys_dev(jt, SNAPPY, d_src, off, ln, args.maps, d_dst, cap, lkeys, rkeys, 5, 3,
                                               lkind, rkind, CRC32C, sb, sl, ck)
        return r, capi.last_timing()

    def sorts():
        t = []
        for lo_, hi_, keys in ((0, args.maps, lkeys), (args.maps, n, rkeys)):
            keys = [(t & ~NULL_SAFE, o, ln_, nf) for t, o, ln_, nf in keys]  # the sort takes plain columns
            capi.decompress_sort_rows_keys_dev(SNAPPY, d_src, off[lo_:hi_], ln[lo_:hi_], d_dst, cap, keys, CRC32C,
                                               np.arange(hi_ - lo_ + 1, dtype=np.uint32), sl[lo_:hi_], ck[lo_:hi_])
            t.append(capi.last_timing()["kernel_ms"])
        return sum(t)

    res = {"in_bytes": int(llen.sum() + rlen.sum()), "left_rows": int(llen.size), "right_rows": int(rlen.size)}
    for name in args.join_types.split(","):
        jt = JOIN_TYPES[name]
        cached = args.model_cache and os.path.join(args.model_cache, "%s-%s-%d-%s.json" % (
            workload, name, red, hashlib.sha256(json.dumps([args.gib, args.maps, args.partitions, args.keys]).encode()).hexdigest()[:12]))
        if cached and os.path.exists(cached):
            want = json.load(open(cached))
        else:
            model = (null_safe_join_model if workload == "e" or name == "existence" else outer_join_model).model_join
            stream, _, _, rows = model(jt, lplain, rplain, lkeys, rkeys, 5, 3, lkind, rkind)
            want = {"bytes": len(stream), "sha256": hashlib.sha256(stream).hexdigest(), "rows": rows}
            if cached:
                os.makedirs(args.model_cache, exist_ok=True)
                json.dump(want, open(cached, "w"))
        assert want["bytes"] <= cap, "--cap-gib is below the reducer's output"
        r, _ = join(jt)
        out = np.zeros(max(r["total"], 1), np.uint8)
        capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        got = hashlib.sha256(out[:r["total"]].tobytes()).hexdigest()
        assert (got, r["n_out_records"]) == (want["sha256"], want["rows"]), "%s differs from the model" % name
        _, t = join(jt)
        res[name + "_kernel_ms"] = t["kernel_ms"]
        res[name + "_step_ms"] = t["dominant_ms"]
        res[name + "_out_rows"] = r["n_out_records"]
        res[name + "_out_mb"] = r["total"] / 1e6
    sorts()
    res["two_sorts_kernel_ms"] = sorts()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--gib", type=float, default=2.0, help="left rows over all reducers")
    ap.add_argument("--maps", type=int, default=400)
    ap.add_argument("--partitions", type=int, default=200)
    ap.add_argument("--reducers", type=int, default=3)
    ap.add_argument("--keys", type=int, default=10**7)
    ap.add_argument("--workloads", default="a,b,c")
    ap.add_argument("--join-types", default="inner", help="comma-separated: " + ", ".join(JOIN_TYPES))
    ap.add_argument("--cap-gib", type=float, default=1.0, help="device output buffer")
    ap.add_argument("--model-cache", default=None, help="a directory for the model outputs' lengths and hashes")
    args = ap.parse_args()
    import spark_s3_shuffle_b200 as pkg
    capi = pkg.capi
    capi.init(1)
    cap = int(args.cap_gib * 2**30)
    d_src, d_dst = capi.dev_alloc(1 << 30), capi.dev_alloc(cap)
    res = {"card": card(), "maps": args.maps, "partitions": args.partitions, "gib": args.gib, "workloads": {}}
    try:
        for w in args.workloads.split(","):
            per = [run(capi, args, w, red, d_src, d_dst, cap) for red in range(args.reducers)]
            res["workloads"][w] = {k: spread([p[k] for p in per]) for k in per[0]}
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
