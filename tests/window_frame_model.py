"""A model of b2s_decompress_window_frame_rows_keys_*, written from its header contract: Spark 3.5's WindowExec over
sliding ROWS and RANGE frames, mixed with ranking functions, LAG / LEAD and the older frames.

The records are sorted, partitioned and grouped into peers as window_offset_model does, with its comparator; ranking
functions, LAG / LEAD and the frames 1..3 are evaluated there.  A frame 4 / 5 function's frames come from a literal
transcription of Spark's four frame classes, driven by its two bound orderings:
  RowBoundOrdering(k)    compare(input j, output i) = j - (i + k) in Java int arithmetic
  RangeBoundOrdering     the input's order value against bound(i) under the column's sort order; bound(i) is v + k
                         ascending and v + (-k) descending in the column type's (wrapping) arithmetic, null when v is;
                         CURRENT ROW compares the whole order key
  UnboundedWindowFunctionFrame           the whole partition
  UnboundedPrecedingWindowFunctionFrame  rows added while ubound.compare(row, inputIndex, current, i) <= 0
  UnboundedFollowingWindowFunctionFrame  rows skipped while lbound.compare(row, inputIndex, current, i) < 0, then
                                         every row to the partition's end
  SlidingWindowFunctionFrame             the buffer's head dropped while lbound.compare(...) < 0, then rows added while
                                         ubound.compare(...) <= 0 (a row below the lower bound only moves inputLowIndex)
Each function's value is then its fold over the frame's rows in order (window_agg_model.fold, or First / Last /
NthValue's update), so growing frames are the running fold and every other frame a fresh fold from its first row.
The model also reports where the call returns B2S_E_UNSUPPORTED: a partition of N records with N - 1 + |k| > 2^31 - 1
for a finite ROWS offset k, or a non-null order value whose exact v +- k leaves the column's type."""
import functools
from collections import deque

from join_model import joined
from rows_model import parse
from test_gpu_sort_rows_order import DESC, col_value, comparator
from window_agg_model import COUNT, FRAME_PARTITION, FRAME_ROWS, SUM, fold, read_value
from window_model import partition_values
from window_offset_model import (FIRST, IGNORE_NULLS, LAG, LAST, read_input, offset_values, value_row)

FRAME_ROWS_SLIDING, FRAME_RANGE_SLIDING = 4, 5
UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING = -2**63, 2**63 - 1
KEY_BITS = {6: 8, 5: 16, 1: 32, 2: 64}  # B2S_KEY_INT8 / INT16 / INT32 / INT64


def jint(x):
    """Java int arithmetic: x wrapped to 32 bits"""
    return (x + 2**31) % 2**32 - 2**31


def wrap(x, bits):
    return (x + 2**(bits - 1)) % 2**bits - 2**(bits - 1)


def fn_list(fns):
    """fns as the ctypes wrapper takes them -> [(fn, arg, frame, val_type, val_off, val_null_field, flags, default,
    lower, upper)]"""
    out = []
    for f in fns:
        if isinstance(f, tuple) and len(f) == 10:
            out.append(tuple(f))
        elif isinstance(f, tuple) and len(f) == 8:
            out.append(tuple(f) + (0, 0))
        elif isinstance(f, tuple) and len(f) == 5:
            out.append((f[0], 0) + tuple(f[1:]) + (0, 0, 0, 0))
        else:
            fn, arg = f if isinstance(f, tuple) else (f, 0)
            out.append((fn, arg, 0, 0, 0, -1, 0, 0, 0, 0))
    return out


class Bounds:
    """the bound orderings of one partition: ok[i] its order keys (tuples of col_value), order_keys the key columns"""

    def __init__(self, ok, order_keys):
        self.ok = ok
        self.cmp_order = comparator(order_keys)
        self.col = order_keys[0]
        self.cmp_col = comparator(order_keys[:1])
        self.unsupported = False

    def ordering(self, kind, k):
        """compare(input row r, input index j, output row i) of the bound k (0 CURRENT ROW, else the offset) as
        Spark's createBoundOrdering builds it: ROWS reads the index, RANGE the row"""
        if kind == FRAME_ROWS_SLIDING:
            return lambda r, j, i: jint(j - jint(i + k))
        if k == 0:
            return lambda r, j, i: self.cmp_order(self.ok[r], self.ok[i])
        kt = self.col[0]
        bits = KEY_BITS[kt & 0xFF]
        d = -k if kt & DESC else k

        def bound(i):
            v = self.ok[i][0]
            if v is None:
                return None
            exact = v + d
            if wrap(exact, bits) != exact:
                self.unsupported = True
            return wrap(exact, bits)  # Add / DateAdd in the column's type
        return lambda r, j, i: self.cmp_col((self.ok[r][0],), (bound(i),))


def frames(N, kind, lo, hi, b):
    """the rows each output row of a partition of N folds over, by Spark's frame class for (lo, hi) -> [[j, ...]]"""
    out = []
    if lo == UNBOUNDED_PRECEDING and hi == UNBOUNDED_FOLLOWING:  # UnboundedWindowFunctionFrame
        return [list(range(N)) for _ in range(N)]
    if lo == UNBOUNDED_PRECEDING:  # UnboundedPrecedingWindowFunctionFrame
        ubound = b.ordering(kind, hi)
        input_index = 0
        for i in range(N):
            while input_index < N and ubound(input_index, input_index, i) <= 0:
                input_index += 1
            out.append(list(range(input_index)))
        return out
    lbound = b.ordering(kind, lo)
    if hi == UNBOUNDED_FOLLOWING:  # UnboundedFollowingWindowFunctionFrame
        input_index = 0
        for i in range(N):
            while input_index < N and lbound(input_index, input_index, i) < 0:
                input_index += 1
            out.append(list(range(input_index, N)))
        return out
    ubound = b.ordering(kind, hi)  # SlidingWindowFunctionFrame
    buf = deque()
    next_row, low, high = 0, 0, 0
    for i in range(N):
        while buf and lbound(buf[0], low, i) < 0:
            buf.popleft()
            low += 1
        while next_row < N and ubound(next_row, high, i) <= 0:
            if lbound(next_row, low, i) < 0:
                low += 1
            else:
                buf.append(next_row)
            next_row += 1
            high += 1
        out.append(list(buf))
    return out


def closed_form(ok, npk_keys_order, kind, lo, hi, i, N):
    """the frame of position i as the header states it, for the tests: ROWS clipped offsets, RANGE {j : lo <= v_j <=
    hi} in sort order -> [j, ...]"""
    if kind == FRAME_ROWS_SLIDING:
        s = 0 if lo == UNBOUNDED_PRECEDING else max(0, i + lo)
        e = N - 1 if hi == UNBOUNDED_FOLLOWING else min(N - 1, i + hi)
        return list(range(s, e + 1))
    cmp_order = comparator(npk_keys_order)
    cmp_col = comparator(npk_keys_order[:1])
    kt = npk_keys_order[0][0]

    def side(j, k, upper):
        if k in (UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING):
            return True
        if k == 0:
            c = cmp_order(ok[j], ok[i])
        else:
            v = ok[i][0]
            c = cmp_col((ok[j][0],), (None if v is None else v + (-k if kt & DESC else k),))
        return c <= 0 if upper else c >= 0
    return [j for j in range(N) if side(j, lo, False) and side(j, hi, True)]


def frame_value(fn, arg, vt, flags, xs):
    """fn's value over the inputs xs of one frame, folded in order (None: null)"""
    if fn < LAG:
        if not xs:
            return 0 if fn == COUNT else None
        return fold(fn, vt, xs)[-1]
    ign = bool(flags & IGNORE_NULLS)
    seen = [x for x in xs if not ign or x is not None]
    if fn == FIRST:
        return seen[0] if seen else None
    if fn == LAST:
        return seen[-1] if seen else None
    return seen[arg - 1] if len(seen) >= arg else None


def model_window_frame(plain, keys, n_partition_keys, n_fields, kinds, fns):
    """plain: the decoded blocks; keys: the composite key [(type | flags, off, len, null field)] -> (the output
    stream's bytes, n_records, n_out_records, unsupported).  Unsupported: the call returns B2S_E_UNSUPPORTED."""
    fns = fn_list(fns)
    buf = b"".join(plain)
    rows = [buf[o + 4:o + ln] for o, ln in parse(buf)]
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
    unsupported = False
    for p in parts:
        N = len(p)
        ok = [kv[i][n_partition_keys:] for i in p]
        end = [0] * N  # each position's peer group end
        for i in range(N - 1, -1, -1):
            end[i] = end[i + 1] if i + 1 < N and cmp_order(ok[i + 1], ok[i]) == 0 else i + 1
        vals = []
        for fn, arg, frame, vt, off, nfield, flags, default, lo, hi in fns:
            if fn < SUM:
                vals.append(partition_values(ok, fn, arg, lambda x, y: cmp_order(x, y) == 0))
                continue
            read = read_value if fn < LAG else read_input
            xs = [read(rows[i], vt, off, nfield) for i in p]
            if frame < FRAME_ROWS_SLIDING:
                if fn < LAG:
                    states = fold(fn, vt, xs)
                    last = [N - 1 if frame == FRAME_PARTITION else i if frame == FRAME_ROWS else end[i] - 1
                            for i in range(N)]
                    vals.append([states[e] for e in last])
                else:
                    vals.append(offset_values(fn, arg, frame, flags, default, xs, end))
                continue
            if frame == FRAME_ROWS_SLIDING:
                for k in (lo, hi):
                    if k not in (UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING) and N - 1 + abs(k) > 2**31 - 1:
                        unsupported = True
            if frame == FRAME_RANGE_SLIDING:
                kt = keys[n_partition_keys][0]
                for k in (lo, hi):
                    if k in (0, UNBOUNDED_PRECEDING, UNBOUNDED_FOLLOWING):
                        continue
                    d, bits = (-k if kt & DESC else k), KEY_BITS[kt & 0xFF]
                    if any(o[0] is not None and wrap(o[0] + d, bits) != o[0] + d for o in ok):
                        unsupported = True
            b = Bounds(ok, keys[n_partition_keys:])
            fr = frames(N, frame, lo, hi, b)
            unsupported |= b.unsupported
            vals.append([frame_value(fn, arg, vt, flags, [xs[j] for j in f]) for f in fr])
        for k, i in enumerate(p):
            vrow, vkinds = value_row([v[k] for v in vals], [f[:8] for f in fns])
            out.append(joined(rows[i], vrow, n_fields, len(fns), kinds, vkinds))
    if unsupported:
        return b"", len(rows), 0, True
    return b"".join(len(r).to_bytes(4, "big") + r for r in out), len(rows), len(out), False
