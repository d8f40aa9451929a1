"""A model of b2s_decompress_window_aggregate_rows_keys_*, written from its header contract: Spark's WindowExec with
aggregate functions (sum, count, min, max, avg) over whole-partition and running frames, mixed with ranking functions.

The records are sorted, partitioned and grouped into peers as window_model does, with its comparator.  Each aggregate
is then folded row by row over its partition in sorted order, as Spark's UnboundedWindowFunctionFrame and
UnboundedPrecedingWindowFunctionFrame feed AggregateProcessor: the state after position k is the fold of positions
0..k, and a record's value is the state at its frame's last position (the partition's last, itself for ROWS, its last
peer for RANGE).  Double sums are Python floats (IEEE doubles) added in order; decimals are Python ints, and the
decimal average is rounded HALF_UP with integer arithmetic.  The value row is the UnsafeRow UnsafeRowWriter would
write (null bits, zeroed slots, wide decimals' 16 bytes), joined to the input row with join_model.joined."""
import functools
import math
import struct

from join_model import DECIMAL_WIDE, FIXED, joined, words
from rows_model import is_null, parse
from test_gpu_sort_rows_order import col_value, comparator
from window_model import CUME_DIST, PERCENT_RANK, partition_values

SUM, COUNT, MIN, MAX, AVG = range(6, 11)
FRAME_PARTITION, FRAME_ROWS, FRAME_RANGE = 1, 2, 3
VAL_NONE, VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64, VAL_FLOAT32, VAL_FLOAT64, VAL_DECIMAL = range(8)
INT_BYTES = {VAL_INT8: 1, VAL_INT16: 2, VAL_INT32: 4, VAL_INT64: 8}


def dec(p, s):
    return VAL_DECIMAL | p << 8 | s << 16


def dec_ps(vt):
    return (vt >> 8) & 0xFF, vt >> 16


def fn_list(fns):
    """fns as the ctypes wrapper takes them -> [(fn, arg, frame, val_type, val_off, val_null_field)]"""
    out = []
    for f in fns:
        if isinstance(f, tuple) and len(f) == 5:
            out.append((f[0], 0) + tuple(f[1:]))
        else:
            fn, arg = f if isinstance(f, tuple) else (f, 0)
            out.append((fn, arg, 0, VAL_NONE, 0, -1))
    return out


def result_precision(fn, vt):
    p, _ = dec_ps(vt)
    return p + (10 if fn == SUM else 4 if fn == AVG else 0)


def wide_result(fn, vt):
    return vt & 0xFF == VAL_DECIMAL and fn in (SUM, AVG, MIN, MAX) and result_precision(fn, vt) > 18


def read_value(row, vt, off, null_field):
    """the input of one record: None (null), an int (ints, decimals) or (float, raw bits) for floats and doubles"""
    k = vt & 0xFF
    if k == VAL_NONE:
        return 0
    if null_field >= 0 and is_null(row, null_field):
        return None
    raw = bytes(row[off:off + 8])
    if k in INT_BYTES:
        return int.from_bytes(raw[:INT_BYTES[k]], "little", signed=True)
    if k == VAL_FLOAT32:
        return (struct.unpack("<f", raw[:4])[0], raw[:4])
    if k == VAL_FLOAT64:
        return (struct.unpack("<d", raw)[0], raw)
    p, _ = dec_ps(vt)
    if p <= 18:
        return int.from_bytes(raw, "little", signed=True)
    slot = int.from_bytes(raw, "little")
    o, n = slot >> 32, slot & 0xFFFFFFFF
    return int.from_bytes(bytes(row[o:o + n]), "big", signed=True)


def spark_less(a, b):
    """Spark SQL's a < b for (float, bits) inputs: -0.0 == 0.0, NaN above everything and equal to every NaN"""
    if math.isnan(b[0]):
        return not math.isnan(a[0])
    return a[0] < b[0]


def avg_decimal(S, c):
    """S / c in units of 10^-4 of S's unit, rounded HALF_UP (ties away from zero)"""
    q = (2 * abs(S) * 10**4 + c) // (2 * c)
    return -q if S < 0 else q


def fold(fn, vt, xs):
    """the running states of fn over the inputs xs (None: null) -> [result after position k] (None: null)"""
    k = vt & 0xFF
    floating = k in (VAL_FLOAT32, VAL_FLOAT64)
    double_fold = (fn == SUM and floating) or (fn == AVG and k != VAL_DECIMAL)
    out = []
    cnt = 0
    acc = 0.0 if double_fold else 0
    best = None
    for x in xs:
        if x is not None:
            cnt += 1
            if double_fold:
                acc = acc + (x[0] if floating else float(x))
            elif fn in (SUM, AVG):
                acc += x
            elif fn in (MIN, MAX):
                if best is None:
                    best = x
                else:
                    later_wins = (spark_less(x, best) if fn == MIN else spark_less(best, x)) if floating else \
                        (x < best if fn == MIN else best < x)
                    if later_wins:
                        best = x
        if fn == COUNT:
            out.append(cnt)
        elif cnt == 0:
            out.append(None)
        elif fn == SUM:
            out.append(acc if double_fold or k == VAL_DECIMAL else (acc + 2**63) % 2**64 - 2**63)
        elif fn == AVG:
            out.append(acc / cnt if double_fold else avg_decimal(acc, cnt))
        else:
            out.append(best)
    return out


def slot_bytes(fn, vt, v):
    """a non-null value's 8 slot bytes, as UnsafeRowWriter writes the result type"""
    k = vt & 0xFF
    if fn == COUNT:
        return v.to_bytes(8, "little")
    if fn in (SUM, AVG) and (isinstance(v, float)):
        return struct.pack("<d", v)
    if fn in (MIN, MAX) and k in (VAL_FLOAT32, VAL_FLOAT64):
        return v[1].ljust(8, b"\0")
    if fn in (MIN, MAX) and k in INT_BYTES:
        return (v % 2**(8 * INT_BYTES[k])).to_bytes(8, "little")
    return (v % 2**64).to_bytes(8, "little")  # longs and compact decimals


def big_bytes(v):
    """BigInteger.toByteArray(v)"""
    n = (v if v >= 0 else ~v).bit_length() // 8 + 1
    return v.to_bytes(n, "big", signed=True)


def value_row(values, fns):
    """the UnsafeRow of the functions' values (None: null) -> (row, its field kinds)"""
    n = len(fns)
    fixed = 8 * (words(n) + n)
    bits, slots, var, kinds = 0, [], b"", []
    for j, ((fn, _, _, vt, _, _), v) in enumerate(zip(fns, values)):
        if fn < SUM:
            slots.append(struct.pack("<d", v) if fn in (PERCENT_RANK, CUME_DIST) else
                         (v & 0xFFFFFFFF).to_bytes(8, "little"))
            kinds.append(FIXED)
            continue
        wide = wide_result(fn, vt)
        kinds.append(DECIMAL_WIDE if wide else FIXED)
        if v is None:
            bits |= 1 << j
        if wide:
            o = fixed + len(var)
            b = b"" if v is None else big_bytes(v)
            slots.append(((o << 32) | len(b)).to_bytes(8, "little"))
            var += b.ljust(16, b"\0")
        else:
            slots.append(bytes(8) if v is None else slot_bytes(fn, vt, v))
    return bits.to_bytes(8 * words(n), "little") + b"".join(slots) + var, kinds


def model_window_aggregate(plain, keys, n_partition_keys, n_fields, kinds, fns):
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
        for fn, arg, frame, vt, off, nfield in fns:
            if fn < SUM:
                vals.append(partition_values(ok, fn, arg, lambda x, y: cmp_order(x, y) == 0))
                continue
            states = fold(fn, vt, [read_value(rows[i], vt, off, nfield) for i in p])
            last = [N - 1 if frame == FRAME_PARTITION else i if frame == FRAME_ROWS else end[i] - 1 for i in range(N)]
            vals.append([states[e] for e in last])
        for k, i in enumerate(p):
            vrow, vkinds = value_row([v[k] for v in vals], fns)
            out.append(joined(rows[i], vrow, n_fields, len(fns), kinds, vkinds))
    return b"".join(len(r).to_bytes(4, "big") + r for r in out), len(rows), len(out)
