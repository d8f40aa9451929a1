"""A model of b2s_decompress_window_rows_keys_*, written from its header contract: Spark's Sort -> [WindowGroupLimit] ->
Window on a reducer for the ranking functions, with each output row the input row joined with the row of values.

The records are sorted stably with the composite-key comparator of test_gpu_sort_rows_order (null ordering, then the
value, reversed for DESC; floats in Spark SQL's order, so -0.0 == 0.0 and NaN == NaN).  Two records are in one partition
when that comparator finds them equal on the partition columns, peers when it finds them equal on the order columns.
Each function is then evaluated as Spark evaluates it, row by row over a partition in sorted order:
  RowNumber   rowNumber + 1
  RankLike    rank = (order equal to the previous row's and rank != 0) ? rank : rowNumber (rank) / rank + 1 (dense)
  NTile       Spark's bucket / bucketThreshold recurrence over bucketSize = n / k and bucketsWithPadding = n % k
  PercentRank (rank - 1) / (n - 1), 0 when n == 1
  CumeDist    rowNumber / n after the whole peer group (its frame is RANGE UNBOUNDED PRECEDING .. CURRENT ROW)
and the output row is join_model.joined(row, the UnsafeRow of the values, ...), the layout the join tests trust."""
import functools
import struct

from join_model import FIXED, joined, words
from rows_model import parse
from test_gpu_sort_rows_order import col_value, comparator

ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK, CUME_DIST, NTILE = range(6)
NO_LIMIT = 0xFFFFFFFF


def fn_list(fns):
    """fns as the ctypes wrapper takes them -> [(fn, arg)]"""
    return [f if isinstance(f, tuple) else (f, 0) for f in fns]


def ntile_recurrence(N, k):
    """NTile(k) over a partition of N rows, updated row by row as Spark's NTile does -> the buckets"""
    row_number = bucket = threshold = 0
    size, padding = N // k, N % k
    out = []
    for _ in range(N):
        over = row_number >= threshold  # every update reads the old buffer
        row_number, bucket, threshold = (row_number + 1, bucket + (1 if over else 0),
                                         threshold + ((size + (1 if bucket < padding else 0)) if over else 0))
        out.append(bucket)
    return out


def partition_values(order_keys, fn, arg=0, equal=lambda a, b: a == b):
    """the values of fn over one partition whose rows, in sorted order, have the order-column values order_keys"""
    N = len(order_keys)
    if fn == NTILE:
        return ntile_recurrence(N, arg)
    # the peer group's end of each row: CumeDist's frame reaches it
    end = [0] * N
    for i in range(N - 1, -1, -1):
        end[i] = end[i + 1] if i + 1 < N and equal(order_keys[i + 1], order_keys[i]) else i + 1
    out = []
    rank = dense = 0
    row_number = 1  # RankLike's rowNumber starts at 1
    for i in range(N):
        same = i > 0 and equal(order_keys[i], order_keys[i - 1])
        rank = rank if same and rank != 0 else row_number
        dense = dense if same and dense != 0 else dense + 1
        row_number += 1
        if fn == ROW_NUMBER:
            out.append(i + 1)
        elif fn == RANK:
            out.append(rank)
        elif fn == DENSE_RANK:
            out.append(dense)
        elif fn == PERCENT_RANK:
            out.append((rank - 1) / (N - 1) if N > 1 else 0.0)
        elif fn == CUME_DIST:
            out.append(end[i] / N)
        else:
            raise ValueError(fn)
    return out


def value_row(values, fns):
    """the UnsafeRow of the functions' values: no nulls; an int as UnsafeRowWriter writes it, a double as 8 bytes"""
    slots = [struct.pack("<d", v) if f in (PERCENT_RANK, CUME_DIST) else (v & 0xFFFFFFFF).to_bytes(8, "little")
             for (f, _), v in zip(fns, values)]
    return bytes(8 * words(len(fns))) + b"".join(slots)


def model_window(plain, keys, n_partition_keys, n_fields, kinds, fns, limit=None):
    """plain: the decoded blocks; keys: the composite key [(type | flags, off, len, null field)]; limit: None or
    (limit_fn, limit) -> (the output stream's bytes, n_records, n_out_records)"""
    fns = fn_list(fns)
    buf = b"".join(plain)
    recs = parse(buf)
    rows = [buf[o + 4:o + ln] for o, ln in recs]
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
        ok = [kv[i][n_partition_keys:] for i in p]
        vals = [partition_values(ok, f, a, lambda x, y: cmp_order(x, y) == 0) for f, a in fns]
        keep = [True] * len(p)
        if limit is not None:
            lim = partition_values(ok, limit[0], 0, lambda x, y: cmp_order(x, y) == 0)
            keep = [v <= limit[1] for v in lim]
        for k, i in enumerate(p):
            if keep[k]:
                out.append(joined(rows[i], value_row([v[k] for v in vals], fns), n_fields, len(fns), kinds,
                                  [FIXED] * len(fns)))
    return b"".join(len(r).to_bytes(4, "big") + r for r in out), len(rows), len(out)
