"""A model of the limit step of b2s_window_limit_partition_compress_rows_hash_*, written from its header contract: Spark's
Sort(pk ++ ord, global = false) -> WindowGroupLimitExec(pk, ord, limit_fn, limit, Partial) on a map task.

The rows are sorted stably with window_model's composite-key comparator (the one the reducer's window call sorts with),
split into partitions on the partition columns, and each partition's rows are kept while their limit_fn value
(window_model.partition_values, peers compared on the order columns) is at most limit."""
import functools

from test_gpu_sort_rows_order import col_value, comparator
from window_model import partition_values


def partial_limit(rows, keys, n_partition_keys, limit_fn, limit):
    """rows: UnsafeRows (no size prefix); keys: the window key [(type | flags, off, len, null field)], the first
    n_partition_keys the partition columns -> the kept rows in sorted order"""
    kv = [tuple(col_value(r, c) for c in keys) for r in rows]
    cmp_all = comparator(keys)
    order = sorted(range(len(rows)), key=functools.cmp_to_key(lambda i, j: cmp_all(kv[i], kv[j])))  # stable
    cmp_part = comparator(keys[:n_partition_keys])
    cmp_order = comparator(keys[n_partition_keys:])
    parts = []
    for i in order:
        if parts and cmp_part(kv[parts[-1][0]][:n_partition_keys], kv[i][:n_partition_keys]) == 0:
            parts[-1].append(i)
        else:
            parts.append([i])
    out = []
    for p in parts:
        values = partition_values([kv[i][n_partition_keys:] for i in p], limit_fn, 0,
                                  lambda x, y: cmp_order(x, y) == 0)
        out += [rows[i] for i, v in zip(p, values) if v <= limit]
    return out
