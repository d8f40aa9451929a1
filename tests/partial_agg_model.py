"""Spark's partial HashAggregateExec, row by row, as a model for b2s_aggregate_partition_compress_rows_hash_*.

A dict by the normalized key (the composite-key comparator model's typed values: test_gpu_sort_rows_order.col_value)
in first-seen order; each function's buffers updated by its DeclarativeAggregate.updateExpressions (Spark 3.5, ANSI
off) for every row in input order.  The partial rows are written as UnsafeProjection(groupingAttributes ++
aggBufferAttributes) writes them, in the key sort's order (ascending, nulls first).  It does not restate the device's
staging or folds; test_partial_agg_model.py checks that those (the reduce side's merge ops over staged inputs) equal it.
"""
import functools
import struct

from hash_model import decimal_bytes
from rows_model import KEY_BYTES, STRING, is_null
from test_gpu_sort_rows_order import DECIMAL, KEY_FLOAT32, KEY_FLOAT64, col_value, comparator

SUM, COUNT, MIN, MAX, AVG = 6, 7, 8, 9, 10
VAL_NONE, VAL_INT8, VAL_INT16, VAL_INT32, VAL_INT64, VAL_FLOAT32, VAL_FLOAT64, VAL_DECIMAL, VAL_BYTES = range(9)
# the reduce side's merge ops (B2S_AGG_*)
SUM_I64, SUM_F64, MIN_I32, MAX_I32, MIN_I64, MAX_I64, MIN_F64, MAX_F64 = range(8)
SUM_DEC, MIN_DEC, MAX_DEC = 9, 10, 11
INT_BYTES = {VAL_INT8: 1, VAL_INT16: 2, VAL_INT32: 4, VAL_INT64: 8}


def val_decimal(p, s):
    return VAL_DECIMAL | p << 8 | s << 16


def buffers(aggs):
    """aggs [(fn, val_type, off, null field)] -> the buffers in order: (merge op, kind), kind one of "long", "double",
    "int", "bool", "dec" (a decimal: its unscaled value; out of line when the op is wide)"""
    out = []
    for fn, vt, _, _ in aggs:
        kind, p = vt & 0xFF, (vt >> 8) & 0xFF
        dec, fp = kind == VAL_DECIMAL, kind in (VAL_FLOAT32, VAL_FLOAT64)
        if fn == SUM:
            out += [(SUM_DEC | (p + 10) << 8, "dec"), (MIN_I32, "bool")] if dec else \
                [(SUM_F64, "double") if fp else (SUM_I64, "long")]
        elif fn == COUNT:
            out.append((SUM_I64, "long"))
        elif fn == AVG:
            out += [(SUM_DEC | (p + 10) << 8, "dec") if dec else (SUM_F64, "double"), (SUM_I64, "long")]
        else:
            mx = fn == MAX
            if kind == VAL_INT32:
                out.append((MAX_I32 if mx else MIN_I32, "int"))
            elif kind == VAL_INT64 or (dec and p <= 18):
                out.append((MAX_I64 if mx else MIN_I64, "long" if kind == VAL_INT64 else "dec"))
            elif kind == VAL_FLOAT64:
                out.append((MAX_F64 if mx else MIN_F64, "double"))
            else:
                out.append((MAX_DEC if mx else MIN_DEC, "dec"))
    return out


def wide_op(op):
    base, p = op & 0xFF, (op >> 8) & 0xFF
    return base in (MIN_DEC, MAX_DEC) or (base == SUM_DEC and p > 18)


def read_value(row, vt, off, nf):
    """a row's input -> None (null) or its value: an int, a float (floats widened), or a decimal's unscaled int"""
    kind, p = vt & 0xFF, (vt >> 8) & 0xFF
    if kind == VAL_NONE:
        return 1
    if nf >= 0 and is_null(row, nf):
        return None
    if kind == VAL_BYTES:
        return 1
    slot = bytes(row[off:off + 8])
    if kind in INT_BYTES:
        return int.from_bytes(slot[:INT_BYTES[kind]], "little", signed=True)
    if kind == VAL_FLOAT32:
        return struct.unpack("<f", slot[:4])[0]
    if kind == VAL_FLOAT64:
        return struct.unpack("<d", slot)[0]
    if p <= 18:
        return int.from_bytes(slot, "little", signed=True)
    s = int.from_bytes(slot, "little")
    return int.from_bytes(bytes(row[s >> 32:(s >> 32) + (s & 0xFFFFFFFF)]), "big", signed=True)


def dorder(x):
    """Spark SQL's double order as a Python key: -0.0 == 0.0, every NaN equal and above +inf"""
    return (1, 0.0) if x != x else (0, x + 0.0)


def new_state(aggs):
    st = []
    for fn, vt, _, _ in aggs:
        dec = vt & 0xFF == VAL_DECIMAL
        st.append({SUM: [0, True] if dec else [None], COUNT: [0], AVG: [0 if dec else 0.0, 0]}.get(fn, [None]))
    return st


def update(st, aggs, row):
    for s, (fn, vt, off, nf) in zip(st, aggs):
        v = read_value(row, vt, off, nf)
        kind = vt & 0xFF
        dec, fp = kind == VAL_DECIMAL, kind in (VAL_FLOAT32, VAL_FLOAT64)
        if fn == COUNT:
            s[0] += v is not None
        elif fn == SUM:
            if dec:  # If(child.isNull, sum, sum + child); isEmpty && child.isNull
                if v is not None:
                    s[0] += v
                    s[1] = False
            elif v is not None:  # Add(coalesce(sum, 0), child)
                s[0] = ((0.0 if s[0] is None else s[0]) + v) if fp else ((s[0] or 0) + v)
        elif fn == AVG:  # sum + coalesce(child.cast(sumType), 0); count + (child not null)
            s[0] = s[0] + (0 if v is None else v) if dec else s[0] + (0.0 if v is None else float(v))
            s[1] += v is not None
        elif v is not None:  # Least / Greatest: the first of equal values stays
            key = dorder if fp else (lambda x: x)
            if s[0] is None or (key(v) > key(s[0]) if fn == MAX else key(v) < key(s[0])):
                s[0] = v


def state_values(st, aggs):
    """the buffers' values in order (None: null)"""
    out = []
    for s, (fn, vt, _, _) in zip(st, aggs):
        if fn == SUM and vt & 0xFF == VAL_DECIMAL:
            out += [s[0], int(s[1])]
        elif fn == AVG:
            out += [s[0], s[1]]
        else:
            out.append(s[0])
    return out


def norm_float(b, width):
    if width == 4:
        v = int.from_bytes(b, "little")
        mag = v & 0x7FFFFFFF
        return (0 if mag == 0 else 0x7FC00000 if mag > 0x7F800000 else v).to_bytes(4, "little")
    v = int.from_bytes(b, "little")
    mag = v & 0x7FFFFFFFFFFFFFFF
    return (0 if mag == 0 else 0x7FF8000000000000 if mag > 0x7FF0000000000000 else v).to_bytes(8, "little")


def emit(first, keys, bufs, values):
    """the partial row of a group: its first row's key columns, then the buffers' values"""
    nk = len(keys)
    nf = nk + len(bufs)
    assert nf <= 32
    fixed = 8 + 8 * nf
    out = bytearray(fixed)
    var = bytearray()
    nulls = 0

    def put_var(f, data, pad_to):
        out[8 + 8 * f:16 + 8 * f] = ((fixed + len(var)) << 32 | len(data)).to_bytes(8, "little")
        var.extend(data + bytes(pad_to - len(data)))

    for c, (kt, ko, kl, nf_) in enumerate(keys):
        null = nf_ >= 0 and is_null(first, nf_)
        t = kt & 0xFF
        if null:
            nulls |= 1 << c
            if t == DECIMAL:
                out[8 + 8 * c:16 + 8 * c] = ((fixed + len(var)) << 32).to_bytes(8, "little")
                var.extend(bytes(16))
            continue
        if t in (STRING, DECIMAL):
            s = int.from_bytes(first[ko:ko + 8], "little")
            b = bytes(first[s >> 32:(s >> 32) + (s & 0xFFFFFFFF)])
            if t == STRING:
                put_var(c, b, len(b) + (-len(b) % 8))
            else:
                put_var(c, decimal_bytes(int.from_bytes(b, "big", signed=True)), 16)
        elif t in (KEY_FLOAT32, KEY_FLOAT64):
            out[8 + 8 * c:8 + 8 * c + kl] = norm_float(bytes(first[ko:ko + kl]), kl)
        else:
            out[8 + 8 * c:8 + 8 * c + kl] = first[ko:ko + kl]
    for k, ((op, kind), v) in enumerate(zip(bufs, values)):
        f = nk + k
        slot = 8 + 8 * f
        if v is None:
            nulls |= 1 << f
            if wide_op(op):
                out[slot:slot + 8] = ((fixed + len(var)) << 32).to_bytes(8, "little")
                var.extend(bytes(16))
            continue
        if wide_op(op):
            put_var(f, decimal_bytes(v), 16)
        elif kind == "double":
            out[slot:slot + 8] = struct.pack("<d", v)
        elif kind in ("int", "bool"):
            out[slot:slot + 4] = int(v).to_bytes(4, "little", signed=True)
        else:
            out[slot:slot + 8] = (int(v) % 2**64).to_bytes(8, "little")
    out[0:8] = nulls.to_bytes(8, "little")
    return bytes(out + var)


def partial_rows(rows, keys, aggs):
    """rows (UnsafeRows, no size prefix) -> the partial rows in key-sort order"""
    groups = {}
    for r in rows:
        k = tuple(col_value(r, c) for c in keys)
        if k not in groups:
            groups[k] = (r, new_state(aggs))
        update(groups[k][1], aggs, r)
    cmp = comparator(keys)
    order = sorted(groups, key=functools.cmp_to_key(cmp))
    bufs = buffers(aggs)
    return [emit(groups[k][0], keys, bufs, state_values(groups[k][1], aggs)) for k in order]


def output_keys(keys):
    """the key columns at their partial-row slots"""
    return [(kt, 8 + 8 * c, kl, c if nf >= 0 else -1) for c, (kt, _, kl, nf) in enumerate(keys)]


def merge_aggs(keys, aggs):
    """the reduce side's aggregates (op, slot, null bit) over the partial rows"""
    nk = len(keys)
    return [(op, 8 + 8 * (nk + k), nk + k) for k, (op, _) in enumerate(buffers(aggs))]
