"""Spark's RangePartitioner over UnsafeRow sort keys, as a model for b2s_partition_compress_rows_range_*.

Keys are compared with the composite-key sort's comparator model (test_gpu_sort_rows_order: col_value, comparator),
which compares typed values column by column and does not restate the GPU's byte encoding.  On top of it:
- get_partition restates RangePartitioner.getPartition for ascending = true (every SQL sort): a linear scan while the
  key is above bound p for at most 128 bounds, Arrays.binarySearch above that (-(insertion point) - 1 mapped back);
- determine_bounds restates RangePartitioner.determineBounds (weighted candidates sorted stably, a bound at each step
  of the cumulative weight, keys not above the previous bound skipped), so tests draw bounds the way Spark does;
- project builds the bound rows Spark holds: UnsafeProjection(sort order children) of a row, key column c as field c."""
import functools

import numpy as np

from rows_model import is_null
from test_gpu_sort_rows_order import (BOOL, DECIMAL, DESC, FLAGS, KEY_FLOAT32, KEY_FLOAT64, KEY_INT8, KEY_INT16, KLEN,
                                      NULLS_LAST, col_value, comparator, layout, make_row, rand_rows, rand_value)
from rows_model import KEY_BYTES, KEY_INT32, KEY_INT64, STRING


def key_of(row, keys):
    """the typed key of a row (no size prefix)"""
    return tuple(col_value(row, c) for c in keys)


def bound_keys(keys):
    """the key columns of a bound row: field c, its null bit c when the records' column is nullable"""
    words = 8 * ((len(keys) + 63) // 64)
    return [(kt, words + 8 * c, kl, c if nf >= 0 else -1) for c, (kt, _, kl, nf) in enumerate(keys)]


def project(row, keys):
    """UnsafeProjection(sort order children) of a row: the bound row Spark's RangePartitioner holds"""
    n = len(keys)
    fixed = 8 * ((n + 63) // 64) + 8 * n
    out = bytearray(fixed)
    var = bytearray()
    for c, (kt, ko, kl, nf) in enumerate(keys):
        slot = 8 * ((n + 63) // 64) + 8 * c
        if nf >= 0 and is_null(row, nf):
            w = 8 * (c >> 6)
            out[w:w + 8] = (int.from_bytes(out[w:w + 8], "little") | 1 << (c & 63)).to_bytes(8, "little")
            continue
        if kt & 0xFF in (STRING, DECIMAL):
            s = int.from_bytes(row[ko:ko + 8], "little")
            b = bytes(row[s >> 32:(s >> 32) + (s & 0xFFFFFFFF)])
            out[slot:slot + 8] = ((fixed + len(var)) << 32 | len(b)).to_bytes(8, "little")
            var += b + bytes(-len(b) % 8)
        else:
            out[slot:slot + kl] = row[ko:ko + kl]
    return bytes(out + var)


def framed(row):
    return len(row).to_bytes(4, "big") + row


def scan_partition(k, bounds, cmp):
    """getPartition's branch for at most 128 bounds: scan while the key is above bound p"""
    p = 0
    while p < len(bounds) and cmp(k, bounds[p]) > 0:
        p += 1
    return p


def search_partition(k, bounds, cmp):
    """getPartition's branch for more than 128 bounds: java.util.Arrays.binarySearch(bounds, k, ordering)"""
    lo, hi = 0, len(bounds) - 1
    while lo <= hi:
        mid = (lo + hi) >> 1
        c = cmp(bounds[mid], k)
        if c < 0:
            lo = mid + 1
        elif c > 0:
            hi = mid - 1
        else:
            return mid
    return lo  # not found: binarySearch's -(insertion point) - 1, mapped back to the insertion point


def get_partition(k, bounds, cmp):
    """RangePartitioner.getPartition(k) over the bounds' keys, ascending"""
    return scan_partition(k, bounds, cmp) if len(bounds) <= 128 else search_partition(k, bounds, cmp)


def lower_bound(k, bounds, cmp):
    """the number of bounds strictly below k"""
    return sum(1 for b in bounds if cmp(b, k) < 0)


def determine_bounds(candidates, partitions, cmp):
    """RangePartitioner.determineBounds: candidates = [(key, weight)] -> at most partitions - 1 strictly increasing
    bound indices into candidates"""
    order = sorted(range(len(candidates)), key=functools.cmp_to_key(lambda i, j: cmp(candidates[i][0],
                                                                                      candidates[j][0])))
    step = sum(float(w) for _, w in candidates) / partitions
    cum, target, out, prev = 0.0, step, [], None
    for i in order:
        if len(out) >= partitions - 1:
            break
        key, w = candidates[i]
        cum += float(w)
        if cum >= target and (prev is None or cmp(key, prev) > 0):
            out.append(i)
            target += step
            prev = key
    return out


def draw_bounds(rng, rows, keys, partitions, sample=None):
    """bound rows as Spark draws them: determineBounds over a sample of the rows (weight 1 each), projected"""
    cmp = comparator(keys)
    idx = rng.choice(len(rows), size=min(sample or len(rows), len(rows)), replace=False) if rows else []
    cands = [(key_of(rows[i], keys), 1.0) for i in idx]
    return [project(rows[idx[j]], keys) for j in determine_bounds(cands, partitions, cmp)]


def model_ids(rows, keys, bounds):
    """every row's reduce id, by getPartition over the bound rows' keys"""
    cmp = comparator(keys)
    bk = [key_of(b, bound_keys(keys)) for b in bounds]
    return np.array([get_partition(key_of(r, keys), bk, cmp) for r in rows], dtype=np.uint32)


def records_of(rows):
    """-> (records back to back as uint8, rec_len u32)"""
    recs = [framed(r) for r in rows]
    buf = np.frombuffer(b"".join(recs) or b"\0", np.uint8)[:sum(len(r) for r in recs)].copy()
    return buf, np.array([len(r) for r in recs], np.uint32)
