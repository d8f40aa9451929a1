"""Measure b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed (a map task's Expand over grouping sets, its
partial aggregation and hash exchange on the GPU) against:
  - b2s_aggregate_partition_compress_rows_hash_packed over the materialised Expand rows: the difference is the cost of
    expanding on the device;
  - b2s_partition_compress_rows_hash_packed over the partial rows: the GPU's share of today's path, where the JVM
    expands and aggregates first;
  - b2s_partition_compress_rows_hash_packed over the raw Expand rows (the .data bytes of shuffling without combining).
Before it is timed, every shape is checked: the new call's outputs equal the aggregating call's over the materialised
Expand rows (built with numpy, and checked against tests/grouping_sets_model.py's projection row by row on a prefix),
and on a prefix of the rows both equal the row-by-row model's partial rows through the hash call.

Shapes (one map task each, R = 200, LZ4):
  q67  : ROLLUP over 4 strings, 3 ints and a 16-byte string (9 sets), sum of a decimal(7, 2)
  q22  : ROLLUP over 4 strings (5 sets), avg of an int
  cube : CUBE over 3 ints (8 sets), count(*), sum of an int, avg of a double
Reports min / median / max of each call's kernel_ms and, for the aggregating calls, the aggregation step (dominant_ms),
and the .data bytes of each; the card's name and power limit read in the same run.  One JSON line per shape."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SUM, COUNT, AVG = 6, 7, 10
VAL_NONE, VAL_INT32, VAL_F64, VAL_DEC72 = 0, 3, 6, 7 | 7 << 8 | 2 << 16
KEY_INT32, STRING = 1, 3


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or "unknown"


def spread(xs):
    return {"min": round(min(xs), 3), "median": round(statistics.median(xs), 3), "max": round(max(xs), 3)}


def gid(mask, nk):
    return sum(1 << (nk - 1 - c) for c in range(nk) if not (mask >> c) & 1)


class Table:
    """n rows of fixed layout: key columns (("string", L, pool size) or ("int", cardinality)), then value columns
    ("int" | "long" | "double", null in 10 %); every key non-null, every string of length L"""

    def __init__(self, rng, n, key_cols, val_cols):
        self.n, self.key_cols, self.val_cols = n, key_cols, val_cols
        nf = len(key_cols) + len(val_cols)
        self.fixed = 8 + 8 * nf
        self.kvals, self.pools = [], []
        var = 0
        self.str_at = []
        for kc in key_cols:
            if kc[0] == "string":
                L, P = kc[1], kc[2]
                pool = rng.integers(97, 123, (P, L), dtype=np.uint8)
                pool[:, 0] = np.arange(P) % 26 + 65  # distinct strings
                pool[:, 1:4] = (np.arange(P)[:, None] >> np.array([0, 5, 10])) % 32 + 48
                self.pools.append(pool)
                self.str_at.append(self.fixed + var)
                var += (L + 7) // 8 * 8
            else:
                self.pools.append(None)
                self.str_at.append(None)
            self.kvals.append(rng.integers(0, kc[2] if kc[0] == "string" else kc[1], n))
        self.rowb = self.fixed + var
        self.vvals = [rng.integers(-10**6, 10**6, n) if t != "double" else rng.normal(size=n) * 1e3
                      for t in val_cols]
        self.vnull = [rng.random(n) < 0.1 for _ in val_cols]

    def records(self):
        n, nk = self.n, len(self.key_cols)
        arr = np.zeros((n, 4 + self.rowb), np.uint8)
        arr[:, 0:4] = np.frombuffer(self.rowb.to_bytes(4, "big"), np.uint8)
        word = np.zeros(n, np.uint64)
        for j, vn in enumerate(self.vnull):
            word |= vn.astype(np.uint64) << np.uint64(nk + j)
        arr[:, 4:12] = word.view(np.uint8).reshape(n, 8)
        for c, kc in enumerate(self.key_cols):
            s = 12 + 8 * c
            if kc[0] == "string":
                arr[:, s:s + 8] = np.full(n, (self.str_at[c] << 32) | kc[1], np.uint64).view(np.uint8).reshape(n, 8)
                a = 4 + self.str_at[c]
                arr[:, a:a + kc[1]] = self.pools[c][self.kvals[c]]
            else:
                arr[:, s:s + 4] = self.kvals[c].astype(np.int32).view(np.uint8).reshape(n, 4)
        for j, t in enumerate(self.val_cols):
            s = 12 + 8 * (nk + j)
            v = np.where(self.vnull[j], 0, self.vvals[j])
            arr[:, s:s + 8] = (v.astype(np.float64) if t == "double" else v.astype(np.int64)).view(np.uint8).reshape(
                n, 8)
        return arr.reshape(-1), np.full(n, 4 + self.rowb, np.uint32)

    def keys(self):
        return [(STRING if kc[0] == "string" else KEY_INT32, 8 + 8 * c, 8 if kc[0] == "string" else 4, -1)
                for c, kc in enumerate(self.key_cols)]

    def expand(self, recs, aggs, masks):
        """the materialised Expand output (grouping_sets_model.project's bytes), row-major, built per set with numpy"""
        n, nk = self.n, len(self.key_cols)
        rows = recs.reshape(n, 4 + self.rowb)[:, 4:]
        ins = [a for a in aggs if a[1] != VAL_NONE]
        nf = nk + 1 + len(ins)
        fixed = 8 + 8 * nf
        blocks = []
        for m in masks:
            var = sum((kc[1] + 7) // 8 * 8 for c, kc in enumerate(self.key_cols) if kc[0] == "string" and (m >> c) & 1)
            b = np.zeros((n, 4 + fixed + var), np.uint8)
            b[:, 0:4] = np.frombuffer((fixed + var).to_bytes(4, "big"), np.uint8)
            word = np.full(n, sum(1 << c for c in range(nk) if not (m >> c) & 1), np.uint64)
            at = fixed
            for c, kc in enumerate(self.key_cols):
                if not (m >> c) & 1:
                    continue
                s = 12 + 8 * c
                if kc[0] == "string":
                    b[:, s:s + 8] = np.full(n, (at << 32) | kc[1], np.uint64).view(np.uint8).reshape(n, 8)
                    src = self.str_at[c]
                    b[:, 4 + at:4 + at + kc[1]] = rows[:, src:src + kc[1]]
                    at += (kc[1] + 7) // 8 * 8
                else:
                    b[:, s:s + 4] = rows[:, 8 + 8 * c:12 + 8 * c]
            b[:, 12 + 8 * nk:20 + 8 * nk] = np.full(n, gid(m, nk), np.int64).view(np.uint8).reshape(n, 8)
            for i, (fn, vt, off, nfield) in enumerate(ins):
                f = nk + 1 + i
                null = self.vnull[nfield - nk]
                word |= null.astype(np.uint64) << np.uint64(f)
                if fn != COUNT:
                    b[:, 12 + 8 * f:20 + 8 * f] = rows[:, off:off + 8]
            b[:, 4:12] = word.view(np.uint8).reshape(n, 8)
            blocks.append(b)
        out = np.concatenate(blocks, axis=1)  # row-major: every set of row 0, then of row 1, ...
        return out.reshape(-1), np.tile(np.array([blk.shape[1] for blk in blocks], np.uint32), n)


SHAPES = {
    "q67": (dict(key_cols=[("string", 10, 10), ("string", 12, 100), ("string", 16, 500), ("string", 24, 2000),
                           ("int", 5), ("int", 4), ("int", 12), ("string", 16, 50)], val_cols=["long"]),
            lambda nk: [(SUM, VAL_DEC72, 8 + 8 * nk, nk)], "rollup"),
    "q22": (dict(key_cols=[("string", 24, 5000), ("string", 16, 500), ("string", 12, 100), ("string", 10, 10)],
                 val_cols=["int"]), lambda nk: [(AVG, VAL_INT32, 8 + 8 * nk, nk)], "rollup"),
    "cube": (dict(key_cols=[("int", 50), ("int", 20), ("int", 10)], val_cols=["int", "double"]),
             lambda nk: [(COUNT, VAL_NONE, 0, -1), (SUM, VAL_INT32, 8 + 8 * nk, nk),
                         (AVG, VAL_F64, 8 + 8 * (nk + 1), nk + 1)], "cube"),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--check-rows", type=int, default=3000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--partitions", type=int, default=200)
    ap.add_argument("--codec", type=int, default=1)
    ap.add_argument("--shapes", default="q67,q22,cube")
    a = ap.parse_args()
    import grouping_sets_model as gm
    import hash_model as hm
    import partial_agg_model as pm
    import spark_s3_shuffle_b200 as pkg

    c = pkg.capi
    c.init(1)
    info = card()
    R, codec = a.partitions, a.codec
    for shape in a.shapes.split(","):
        spec, aggs_of, kind = SHAPES[shape]
        nk = len(spec["key_cols"])
        masks = gm.rollup(nk) if kind == "rollup" else gm.cube(nk)
        aggs = aggs_of(nk)
        for n in (a.check_rows, a.rows):
            t = Table(np.random.default_rng(7), n, **spec)
            recs, rl = t.records()
            keys = t.keys()
            xrec, xrl = t.expand(recs, aggs, masks)
            xkeys, xaggs = gm.projected_keys(keys), gm.projected_aggs(keys, aggs)
            if n == a.check_rows:  # the numpy Expand and the outputs against the row-by-row model
                rows = [recs[4 + i * (4 + t.rowb):(i + 1) * (4 + t.rowb)].tobytes() for i in range(n)]
                xrows, _, _ = gm.expand(rows, keys, aggs, masks)
                want, _ = hm.records_of(xrows)
                assert np.array_equal(want, xrec), shape
                prec, prl = hm.records_of(pm.partial_rows(xrows, xkeys, xaggs))
                cap = c.partition_compress_bound(codec, 0, R, prec.size) + 64
                ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
                ref = c.partition_compress_rows_hash_packed(codec, prec, prl, pm.output_keys(xkeys), R, ref_dst)
                got = c.aggregate_grouping_sets_partition_compress_rows_hash_packed(codec, recs, rl, keys, aggs, masks,
                                                                                   R, got_dst)
                assert got["total"] == ref["total"] and np.array_equal(got_dst[:got["total"]],
                                                                       ref_dst[:got["total"]]), shape
                continue
        # the partial rows, as the aggregating call over the Expand rows writes them with no codec into one partition
        pcap = c.partition_compress_bound(0, 0, 1, xrec.size) + 64
        pdst = np.zeros(pcap, np.uint8)
        p = c.aggregate_partition_compress_rows_hash_packed(0, xrec, xrl, xkeys, xaggs, 1, pdst)
        prec = pdst[:p["total"]].copy()
        prl, at = [], 0
        while at < prec.size:
            sz = int.from_bytes(prec[at:at + 4].tobytes(), "big")
            prl.append(4 + sz)
            at += 4 + sz
        prl = np.array(prl, np.uint32)
        okeys = pm.output_keys(xkeys)
        cap = c.partition_compress_bound(codec, 0, R, max(xrec.size, prec.size)) + 64
        got_dst, agg_dst, ref_dst, raw_dst = (np.zeros(cap, np.uint8) for _ in range(4))
        got = c.aggregate_grouping_sets_partition_compress_rows_hash_packed(codec, recs, rl, keys, aggs, masks, R,
                                                                           got_dst)
        agg = c.aggregate_partition_compress_rows_hash_packed(codec, xrec, xrl, xkeys, xaggs, R, agg_dst)
        ref = c.partition_compress_rows_hash_packed(codec, prec, prl, okeys, R, ref_dst)
        assert got["n_groups"] == agg["n_groups"] == prl.size, shape
        for r, r_dst in ((agg, agg_dst), (ref, ref_dst)):
            assert r["total"] == got["total"] and np.array_equal(got_dst[:got["total"]], r_dst[:got["total"]]), shape
            for k in ("dst_off", "dst_len", "checksums", "status"):
                assert np.array_equal(got[k], r[k]), (shape, k)
        new_k, new_dom, agg_k, agg_dom, part_k, raw_k = [], [], [], [], [], []
        raw = None
        for rep in range(a.reps + 2):
            c.aggregate_grouping_sets_partition_compress_rows_hash_packed(codec, recs, rl, keys, aggs, masks, R,
                                                                          got_dst)
            tn = c.last_timing()
            c.aggregate_partition_compress_rows_hash_packed(codec, xrec, xrl, xkeys, xaggs, R, agg_dst)
            ta = c.last_timing()
            c.partition_compress_rows_hash_packed(codec, prec, prl, okeys, R, ref_dst)
            tp = c.last_timing()
            raw = c.partition_compress_rows_hash_packed(codec, xrec, xrl, xkeys, R, raw_dst)
            tr = c.last_timing()
            if rep >= 2:  # two warm-up rounds
                new_k.append(tn["kernel_ms"])
                new_dom.append(tn["dominant_ms"])
                agg_k.append(ta["kernel_ms"])
                agg_dom.append(ta["dominant_ms"])
                part_k.append(tp["kernel_ms"])
                raw_k.append(tr["kernel_ms"])
        print(json.dumps({"shape": shape, "card": info, "rows": int(rl.size), "sets": len(masks),
                          "input_bytes": int(recs.size), "expand_bytes": int(xrec.size), "groups": int(prl.size),
                          "partitions": R, "codec": codec,
                          "grouping_sets_call_kernel_ms": spread(new_k), "grouping_sets_aggregation_step_ms":
                          spread(new_dom), "aggregate_over_expand_rows_kernel_ms": spread(agg_k),
                          "aggregate_over_expand_rows_step_ms": spread(agg_dom),
                          "hash_over_partial_rows_kernel_ms": spread(part_k),
                          "data_bytes": {"grouping_sets_call": got["total"], "hash_over_raw_expand_rows":
                                         raw["total"]}}), flush=True)


if __name__ == "__main__":
    main()
