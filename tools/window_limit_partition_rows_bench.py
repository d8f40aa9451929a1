#!/usr/bin/env python
"""Measure b2s_window_limit_partition_compress_rows_hash_packed (a map task's Sort and WindowGroupLimitExec(Partial)
and its exchange on the GPU) against the two hash-call paths around it: b2s_partition_compress_rows_hash_packed over
the model's kept rows (the GPU's share of today's path, where the JVM sorts and limits first) and over all rows
(shuffling without the partial limit).  The JVM's Sort and limit are not run here, so no speed-up over them is claimed.

Shapes (one map task of --rows rows, LZ4, CRC32C):
  q67    : tools/window_rows_bench.py's q67 rows, --categories categories; rank() over (partition by i_category order
           by sumsales desc nulls last) <= 100; R = 200
  dedup  : [id long, ts long, payload string], about 4 rows per id; row_number() over (partition by id order by ts
           desc) = 1; R = 200
  topk   : [id long, v long, payload string], 1000 ids; rank() over (partition by id order by v desc) <= 5; R = 200
  global : [v long, payload string]; rank() over (order by v desc) <= 10, no partition column (SinglePartition); R = 1
The kept rows come from a numpy form of tests/window_limit_model.py (lexsort, then each partition's limit value), which
is checked against the model itself on the shape's first --check rows.  The limiting call's outputs are checked byte
for byte against the hash call over those kept rows before anything is timed.  Each path is then timed --iters times after
--warmup calls: min / median / max of kernel_ms (the whole call on the device) and, for the limiting call, dominant_ms
(the limit step, the sort included).  The card's name and power limit are read in the same run.  One JSON document.

    python tools/window_limit_partition_rows_bench.py [--rows 1000000] [--shapes q67,dedup,topk,global]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from join_rows_bench import card, rows_of, spread  # noqa: E402
from window_rows_bench import DESC, INT64, dedup_rows, q67_rows  # noqa: E402

LZ4, CRC32C = 1, 3
ROW_NUMBER, RANK, DENSE_RANK = 0, 1, 2


def shape_rows(name, rng, n, categories):
    """-> (records, rec_len, keys, n_partition_keys, limit_fn, limit, R, partition values, order values (ascending
    in the key's order))"""
    if name == "q67":
        (rec, ln), keys, _ = q67_rows(rng, n, categories)
        cat = _field_bytes(rec, ln, 0, 16)
        dec = _field_bytes(rec, ln, 8, 16)
        pv = np.array([int(c[8:]) for c in cat.view("S16").ravel()], np.int64)
        ov = -dec[:, 8:].copy().view(">i8").ravel().astype(np.int64)  # DESC: smaller sorts first
        return rec, ln, keys, 1, RANK, 100, 200, pv, ov
    if name == "dedup":
        (rec, ln), keys, _ = dedup_rows(rng, n)
        pv, ts = _slot(rec, ln, 0), _slot(rec, ln, 1)
        return rec, ln, keys, 1, ROW_NUMBER, 1, 200, pv, -ts
    slots = np.zeros((n, 3), np.uint64)
    if name == "topk":
        slots[:, 0] = rng.integers(0, 1000, n).astype(np.uint64)
        slots[:, 1] = rng.integers(0, 2000, n).astype(np.uint64)
        rec, ln = rows_of(slots, {2: 8 * rng.integers(1, 5, n)}, rng)
        keys = [(INT64, 8, 8, -1), (INT64 | DESC, 16, 8, -1)]
        return rec, ln, keys, 1, RANK, 5, 200, slots[:, 0].astype(np.int64), -slots[:, 1].astype(np.int64)
    slots[:, 0] = rng.integers(0, 1 << 20, n).astype(np.uint64)
    rec, ln = rows_of(slots[:, :2], {1: 8 * rng.integers(1, 5, n)}, rng)
    return rec, ln, [(INT64 | DESC, 8, 8, -1)], 0, RANK, 10, 1, np.zeros(n, np.int64), -slots[:, 0].astype(np.int64)


def _starts(ln):
    return np.concatenate([[0], np.cumsum(ln.astype(np.int64))[:-1]])


def _field_bytes(rec, ln, field, width):
    """each row's var bytes of a field (rows of one null word; the slot's offset and size)"""
    st = _starts(ln) + 4
    slot = rec[(st + 8 + 8 * field)[:, None] + np.arange(8)].view("<u8").ravel()
    off = (slot >> np.uint64(32)).astype(np.int64)
    return rec[(st + off)[:, None] + np.arange(width)]


def _slot(rec, ln, field):
    st = _starts(ln) + 4
    return rec[(st + 8 + 8 * field)[:, None] + np.arange(8)].view("<i8").ravel()


def kept_numpy(pv, ov, fn, limit):
    """the model's kept positions in sorted order: a stable sort by (partition, order), then each partition's value"""
    order = np.lexsort((ov, pv))
    p, o = pv[order], ov[order]
    n = len(order)
    pstart = np.concatenate([[True], p[1:] != p[:-1]]) if n else np.zeros(0, bool)
    peer = pstart | np.concatenate([[True], o[1:] != o[:-1]]) if n else pstart
    idx = np.arange(n)
    ps = np.maximum.accumulate(np.where(pstart, idx, 0))
    if fn == ROW_NUMBER:
        v = idx - ps + 1
    elif fn == RANK:
        v = np.maximum.accumulate(np.where(peer, idx, 0)) - ps + 1
    else:
        g = np.cumsum(peer)
        v = g - g[ps] + 1
    return order[v <= limit]


def gather(rec, ln, sel):
    st = _starts(ln)
    parts = [rec[s:s + int(l)] for s, l in zip(st[sel], ln[sel])]
    return (np.concatenate(parts) if parts else np.zeros(0, np.uint8)), ln[sel].copy()


def rows_list(rec, ln, m):
    st = _starts(ln)
    return [rec[s + 4:s + int(l)].tobytes() for s, l in zip(st[:m], ln[:m])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--categories", type=int, default=10)
    ap.add_argument("--shapes", default="q67,dedup,topk,global")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--check", type=int, default=20_000)
    args = ap.parse_args()
    import spark_s3_shuffle_b200 as pkg
    from window_limit_model import partial_limit
    capi = pkg.capi
    capi.init(1)
    out = {"card": card(), "rows": args.rows, "shapes": {}}
    for name in args.shapes.split(","):
        rng = np.random.default_rng(sum(name.encode()))
        rec, ln, keys, npk, fn, limit, R, pv, ov = shape_rows(name, rng, args.rows, args.categories)
        m = min(args.check, len(ln))  # the numpy form against the model itself
        sel = kept_numpy(pv[:m], ov[:m], fn, limit)
        assert rows_list(*gather(rec[:int(ln[:m].sum())], ln[:m], sel), len(sel)) == \
            partial_limit(rows_list(rec, ln, m), keys, npk, fn, limit), name
        kept_rec, kept_ln = gather(rec, ln, kept_numpy(pv, ov, fn, limit))
        cap = capi.partition_compress_bound(LZ4, 0, R, rec.size) + 64
        dst = [np.zeros(cap, np.uint8) for _ in range(3)]

        def limited():
            return capi.window_limit_partition_compress_rows_hash_packed(LZ4, rec, ln, keys, npk, fn, limit, R, dst[0],
                                                                         checksum_alg=CRC32C)

        def hashed(records, lens, d):
            if npk:
                return capi.partition_compress_rows_hash_packed(LZ4, records, lens, keys[:npk], R, d,
                                                                checksum_alg=CRC32C)
            return capi.partition_compress_packed(LZ4, records, lens, np.zeros(lens.size, np.uint32), R, d,
                                                  checksum_alg=CRC32C)

        paths = {"window_limit": limited, "hash_kept": lambda: hashed(kept_rec, kept_ln, dst[1]),
                 "hash_all": lambda: hashed(rec, ln, dst[2])}
        a, b = limited(), paths["hash_kept"]()
        assert a["n_out_records"] == kept_ln.size and a["total"] == b["total"], name
        for k in ("dst_off", "dst_len", "checksums", "status"):
            assert (a[k] == b[k]).all(), (name, k)
        assert (dst[0][:a["total"]] == dst[1][:b["total"]]).all(), name
        res = {"R": R, "kept_rows": int(kept_ln.size), "input_bytes": int(rec.size)}
        for p, f in paths.items():
            for _ in range(args.warmup):
                f()
            kms, dms = [], []
            for _ in range(args.iters):
                r = f()
                t = capi.last_timing()
                kms.append(t["kernel_ms"])
                dms.append(t["dominant_ms"])
            res[p] = {"kernel_ms": spread(kms), "data_bytes": int(r["total"])}
            if p == "window_limit":
                res[p]["limit_step_ms"] = spread(dms)
        out["shapes"][name] = res
        print(json.dumps({name: res}), file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
