"""A model of b2s_decompress_window_offset_rows_keys_*, written from its header contract: Spark's WindowExec with offset
functions (lag, lead, first, last, nth_value), mixed with ranking and aggregate functions.

The records are sorted, partitioned and grouped into peers as window_model does, with its comparator; ranking and
aggregate functions are evaluated by window_agg_model.  Each offset function is evaluated row by row over its partition
in sorted order, as Spark does:
  Lag / Lead   FrameLessOffsetWindowFunctionFrame: the input k rows before / after, else the default; with ignoreNulls
               the k-th non-null input before / after, kept as the list of non-null inputs seen so far (walking forward
               for lag, backward for lead)
  First / Last / NthValue  the DeclarativeAggregate's update over the frame's rows from the partition's first, in order
               (the first value, the last value, the n-th counted value; with ignoreNulls only non-null inputs count),
               read at the frame's last row
The value row is the UnsafeRow UnsafeRowWriter would write (null bits, zeroed slots, a string's bytes padded to 8, wide
decimals' 16 bytes, all var regions in function order), joined to the input row with join_model.joined."""
import functools
import struct

from join_model import DECIMAL_WIDE, FIXED, VAR, joined, words
from rows_model import is_null, parse
from test_gpu_sort_rows_order import col_value, comparator
from window_agg_model import (FRAME_PARTITION, FRAME_ROWS, SUM, VAL_DECIMAL, VAL_FLOAT32, VAL_INT8, VAL_INT16,
                              VAL_INT32, VAL_NONE, big_bytes, dec_ps, fold, read_value, slot_bytes, wide_result)
from window_model import CUME_DIST, PERCENT_RANK, partition_values

LAG, LEAD, FIRST, LAST, NTH_VALUE = range(11, 16)
VAL_BYTES = 8
IGNORE_NULLS, HAS_DEFAULT = 1, 2
WIDTH = {VAL_INT8: 1, VAL_INT16: 2, VAL_INT32: 4, VAL_FLOAT32: 4}


def fn_list(fns):
    """fns as the ctypes wrapper takes them -> [(fn, arg, frame, val_type, val_off, val_null_field, flags, default)]"""
    out = []
    for f in fns:
        if isinstance(f, tuple) and len(f) == 8:
            out.append(tuple(f))
        elif isinstance(f, tuple) and len(f) == 5:
            out.append((f[0], 0) + tuple(f[1:]) + (0, 0))
        else:
            fn, arg = f if isinstance(f, tuple) else (f, 0)
            out.append((fn, arg, 0, VAL_NONE, 0, -1, 0, 0))
    return out


def wide_input(vt):
    return vt & 0xFF == VAL_DECIMAL and dec_ps(vt)[0] > 18


def read_input(row, vt, off, null_field):
    """an offset function's input: None (null), a string's bytes, a wide decimal's unscaled int, or a fixed-width
    value's 8 slot bytes as UnsafeRowWriter writes its type (the type's width, zeros above)"""
    if null_field >= 0 and is_null(row, null_field):
        return None
    slot = int.from_bytes(row[off:off + 8], "little")
    if vt & 0xFF == VAL_BYTES:
        return bytes(row[slot >> 32:(slot >> 32) + (slot & 0xFFFFFFFF)])
    if wide_input(vt):
        return read_value(row, vt, off, null_field)
    w = WIDTH.get(vt & 0xFF, 8)
    return (slot % 2**(8 * w)).to_bytes(8, "little")


def offset_values(fn, k, frame, flags, default, xs, end):
    """fn over one partition whose inputs, in sorted order, are xs (None: null); end[i]: i's peer group end -> values
    (None: null)"""
    N = len(xs)
    ign = bool(flags & IGNORE_NULLS)
    dflt = default.to_bytes(8, "little") if flags & HAS_DEFAULT else None
    out = [None] * N
    if fn in (LAG, LEAD):
        seen = []  # the inputs already passed (non-null ones with ignoreNulls), nearest last
        walk = range(N) if fn == LAG else range(N - 1, -1, -1)
        for i in walk:
            out[i] = seen[-k] if len(seen) >= k else dflt  # a null input there stays null
            if not ign or xs[i] is not None:
                seen.append(xs[i])
        return out
    # the aggregate's state after each row, read at the frame's last row
    states = []
    first = last = nth = None
    have_first = False
    count = 0
    for x in xs:
        if not ign or x is not None:
            if not have_first:
                first, have_first = x, True
            last = x
            count += 1
            if count == k:
                nth = x
        states.append(first if fn == FIRST else last if fn == LAST else nth)
    for i in range(N):
        e = N - 1 if frame == FRAME_PARTITION else i if frame == FRAME_ROWS else end[i] - 1
        out[i] = states[e]
    return out


def value_row(values, fns):
    """the UnsafeRow of the functions' values (None: null) -> (row, its field kinds)"""
    n = len(fns)
    fixed = 8 * (words(n) + n)
    bits, slots, var, kinds = 0, [], b"", []
    for j, ((fn, _, _, vt, _, _, _, _), v) in enumerate(zip(fns, values)):
        if fn < SUM:
            slots.append(struct.pack("<d", v) if fn in (PERCENT_RANK, CUME_DIST) else
                         (v & 0xFFFFFFFF).to_bytes(8, "little"))
            kinds.append(FIXED)
            continue
        if v is None:
            bits |= 1 << j
        bytes_val = fn >= LAG and vt & 0xFF == VAL_BYTES
        wide = wide_input(vt) if fn >= LAG else wide_result(fn, vt)
        kinds.append(VAR if bytes_val else DECIMAL_WIDE if wide else FIXED)
        if bytes_val:
            if v is None:
                slots.append(bytes(8))
            else:
                slots.append((((fixed + len(var)) << 32) | len(v)).to_bytes(8, "little"))
                var += v + bytes(-len(v) % 8)
        elif wide:
            o = fixed + len(var)
            b = b"" if v is None else big_bytes(v)
            slots.append(((o << 32) | len(b)).to_bytes(8, "little"))
            var += b.ljust(16, b"\0")
        elif v is None:
            slots.append(bytes(8))
        else:
            slots.append(v if fn >= LAG else slot_bytes(fn, vt, v))
    return bits.to_bytes(8 * words(n), "little") + b"".join(slots) + var, kinds


def model_window_offset(plain, keys, n_partition_keys, n_fields, kinds, fns):
    """plain: the decoded blocks; keys: the composite key [(type | flags, off, len, null field)] -> (the output
    stream's bytes, n_records, n_out_records)"""
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
    for p in parts:
        N = len(p)
        ok = [kv[i][n_partition_keys:] for i in p]
        end = [0] * N  # each position's peer group end
        for i in range(N - 1, -1, -1):
            end[i] = end[i + 1] if i + 1 < N and cmp_order(ok[i + 1], ok[i]) == 0 else i + 1
        vals = []
        for fn, arg, frame, vt, off, nfield, flags, default in fns:
            if fn < SUM:
                vals.append(partition_values(ok, fn, arg, lambda x, y: cmp_order(x, y) == 0))
            elif fn < LAG:
                states = fold(fn, vt, [read_value(rows[i], vt, off, nfield) for i in p])
                last = [N - 1 if frame == FRAME_PARTITION else i if frame == FRAME_ROWS else end[i] - 1
                        for i in range(N)]
                vals.append([states[e] for e in last])
            else:
                xs = [read_input(rows[i], vt, off, nfield) for i in p]
                vals.append(offset_values(fn, arg, frame, flags, default, xs, end))
        for k, i in enumerate(p):
            vrow, vkinds = value_row([v[k] for v in vals], fns)
            out.append(joined(rows[i], vrow, n_fields, len(fns), kinds, vkinds))
    return b"".join(len(r).to_bytes(4, "big") + r for r in out), len(rows), len(out)
