"""A Python model of the row aggregation with the Decimal ops (B2S_AGG_SUM_DECIMAL | P << 8, MIN / MAX_DECIMAL), on
Python integers, beside rows_model.model_aggregate (whose functions it reuses for grouping and for the other ops).

SUM_DECIMAL is Spark's Sum / Average decimal merge into an UnsafeRow buffer: over the group's records in stable order,
from 0, the result is null once an input is null or a running sum reaches |S_k| >= 10^P, and stays null.  Out-of-line
results (P > 18, and MIN / MAX_DECIMAL) are written as UnsafeRow.setDecimal writes them: the 16 bytes at the head row's
offset zeroed, BigInteger.toByteArray's bytes there and the slot (offset << 32) | length; null keeps offset << 32."""
from rows_model import is_null, merge, model_keys

SUM_DEC, MIN_DEC, MAX_DEC = 9, 10, 11


def sum_decimal(p):
    return SUM_DEC | (p << 8)


def wide(op):
    return (op & 0xFF) in (MIN_DEC, MAX_DEC) or ((op & 0xFF) == SUM_DEC and (op >> 8) > 18)


def to_byte_array(x):
    """java.math.BigInteger.toByteArray"""
    n = (x if x >= 0 else ~x).bit_length() // 8 + 1
    return x.to_bytes(n, "big", signed=True)


def slot(row, off):
    return int.from_bytes(row[off:off + 8], "little")


def dec_value(row, off, op):
    """a Decimal op's input: the long of a compact sum, else the out-of-line bytes"""
    s = slot(row, off)
    if not wide(op):
        return s - (1 << 64) if s >> 63 else s
    o, n = s >> 32, s & 0xFFFFFFFF
    return int.from_bytes(bytes(row[o:o + n]), "big", signed=True)


def merge_decimal(op, vals):
    """vals: the group's inputs in stable order, None for a null input -> the result, None for null"""
    if op & 0xFF == SUM_DEC:
        p, acc = op >> 8, 0
        for v in vals:
            if v is None:
                return None
            acc += v
            if abs(acc) >= 10**p:
                return None
        return acc
    vals = [v for v in vals if v is not None]
    if not vals:
        return None
    return max(vals) if op & 0xFF == MAX_DEC else min(vals)


def put_decimal(row, op, off, x):
    if not wide(op):
        row[off:off + 8] = (0 if x is None else x & (2**64 - 1)).to_bytes(8, "little")
        return
    o = slot(row, off) >> 32
    row[o:o + 16] = bytes(16)
    if x is None:
        row[off:off + 8] = (o << 32).to_bytes(8, "little")
    else:
        b = to_byte_array(x)
        row[o:o + len(b)] = b
        row[off:off + 8] = ((o << 32) | len(b)).to_bytes(8, "little")


def model_aggregate_decimal(plain, keys, aggs):
    """model_aggregate with the Decimal ops as well -> (rows, number of records, number of groups)"""
    buf, recs, kv, order = model_keys(plain, keys)
    out, j = [], 0
    while j < len(order):
        e = j
        while e < len(order) and kv[order[e]] == kv[order[j]]:
            e += 1
        o, ln = recs[order[j]]
        rec = bytearray(buf[o:o + ln])
        row = memoryview(rec)[4:]
        nulls = []
        rows = [buf[recs[i][0] + 4:recs[i][0] + recs[i][1]] for i in order[j:e]]
        for op, off, anf in aggs:
            if op & 0xFF >= SUM_DEC:
                x = merge_decimal(op, [None if is_null(r, anf) else dec_value(r, off, op) for r in rows])
                put_decimal(row, op, off, x)
                nulls.append((anf, x is None))
                continue
            vals = [bytes(r[off:off + 8]) for r in rows if not is_null(r, anf)]
            row[off:off + 8] = merge(op, vals) if vals else bytes(8)
            nulls.append((anf, not vals))
        for anf, null in nulls:
            if anf >= 0:
                w = 8 * (anf >> 6)
                v = int.from_bytes(row[w:w + 8], "little")
                v = v | (1 << (anf & 63)) if null else v & ~(1 << (anf & 63))
                row[w:w + 8] = v.to_bytes(8, "little")
        out.append(bytes(rec))
        j = e
    return b"".join(out), len(recs), len(out)
