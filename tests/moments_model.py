"""Spark's central-moment aggregates of order 2 (stddev, stddev_samp, stddev_pop, variance, var_samp, var_pop) as a model
for B2S_WINDOW_VARIANCE on the map side and B2S_AGG_VARIANCE on the reduce side.

All six are CentralMomentAgg with momentOrder = 2 (Spark 3.5, ANSI off): three DoubleType buffers [n, avg, m2], never
null, initially 0.0, over the input Cast(child, DoubleType).  Python floats are IEEE binary64 and every operation below
is one rounded-to-nearest operation, evaluated left to right, as the JVM evaluates the expressions.

    updateExpressionsDef (a null input leaves the buffers as they are):
        newN = n + 1.0; delta = x - avg; deltaN = delta / newN
        avg' = avg + deltaN; m2' = m2 + delta * (delta - deltaN); n' = newN
    mergeExpressions (left: the group's buffer, right: the input buffer):
        newN = n1 + n2; delta = avg2 - avg1; deltaN = If(newN === 0.0, 0.0, delta / newN)
        avg' = avg1 + deltaN * n2; m2' = m2a + m2b + delta * deltaN * n1 * n2; n' = newN

The update is not the merge of one-row buffers (1, x, 0), and a merge that started from a group's first buffer
instead of (0, 0, 0) would not give the same avg ((a / k) * k != a), so the map side and the reduce side each have
their own chain.  evaluateExpression (stddev_* / var_*) runs on the JVM after the final merge; it is here only to check
that the buffers compute a variance.
"""
import math
import struct

import decimal_model as dm
import partial_agg_model as pm
import rows_model as rm

VARIANCE = 16      # B2S_WINDOW_VARIANCE: the map side's function
AGG_VARIANCE = 12  # B2S_AGG_VARIANCE: the reduce side's entry over [n, avg, m2]
VAL_TYPES = (pm.VAL_INT8, pm.VAL_INT16, pm.VAL_INT32, pm.VAL_INT64, pm.VAL_FLOAT32, pm.VAL_FLOAT64)


def update(buf, x):
    """one non-null input x (a float) into buf [n, avg, m2]"""
    n, avg, m2 = buf
    new_n = n + 1.0
    delta = x - avg
    delta_n = delta / new_n
    buf[:] = [new_n, avg + delta_n, m2 + delta * (delta - delta_n)]


def merge(buf, other):
    """buf [n1, avg1, m2a] merged with other (n2, avg2, m2b)"""
    n1, avg1, m2a = buf
    n2, avg2, m2b = other
    new_n = n1 + n2
    delta = avg2 - avg1
    delta_n = 0.0 if new_n == 0.0 else delta / new_n
    buf[:] = [new_n, avg1 + delta_n * n2, (m2a + m2b) + ((delta * delta_n) * n1) * n2]


def fold(xs):
    """the update chain over inputs xs (None: null) from (0, 0, 0)"""
    buf = [0.0, 0.0, 0.0]
    for x in xs:
        if x is not None:
            update(buf, x)
    return tuple(buf)


def merge_all(bufs):
    """the merge chain over buffers in order from (0, 0, 0)"""
    buf = [0.0, 0.0, 0.0]
    for b in bufs:
        merge(buf, b)
    return tuple(buf)


def evaluate(buf, fn):
    """CentralMomentAgg.evaluateExpression (nullOnDivideByZero, the default) for fn in var_pop, var_samp, stddev_pop,
    stddev_samp -> a float or None"""
    n, _, m2 = buf
    if n == 0.0:
        return None
    if fn.endswith("samp"):
        if n == 1.0:
            return None
        v = m2 / (n - 1.0)
    else:
        v = m2 / n
    return math.sqrt(v) if fn.startswith("stddev") else v


def to_double(v, vt):
    """Cast(child, DoubleType) of pm.read_value's value: integers rounded to nearest, floats as they are (a float32 was
    widened exactly)"""
    return None if v is None else float(v)


# ---- the map side: pm's model with VARIANCE beside the other functions ----
def buffers(aggs):
    """pm.buffers with a VARIANCE's three double fields (each (AGG_VARIANCE, "double"))"""
    out = []
    for a in aggs:
        out += [(AGG_VARIANCE, "double")] * 3 if a[0] == VARIANCE else pm.buffers([a])
    return out


def partial_rows(rows, keys, aggs):
    """pm.partial_rows with VARIANCE functions: each writes its [n, avg, m2] fields"""
    import functools
    groups = {}
    for r in rows:
        k = tuple(pm.col_value(r, c) for c in keys)
        if k not in groups:
            groups[k] = (r, [[0.0, 0.0, 0.0] if a[0] == VARIANCE else pm.new_state([a])[0] for a in aggs])
        for s, a in zip(groups[k][1], aggs):
            if a[0] == VARIANCE:
                x = to_double(pm.read_value(r, a[1], a[2], a[3]), a[1])
                if x is not None:
                    update(s, x)
            else:
                pm.update([s], [a], r)
    order = sorted(groups, key=functools.cmp_to_key(pm.comparator(keys)))
    bufs = buffers(aggs)
    out = []
    for k in order:
        first, st = groups[k]
        values = []
        for s, a in zip(st, aggs):
            values += list(s) if a[0] == VARIANCE else pm.state_values([s], [a])
        out.append(pm.emit(first, keys, bufs, values))
    return out


def merge_aggs(keys, aggs):
    """the reduce side's entries over the partial rows: (AGG_VARIANCE, slot of n, -1) per VARIANCE, pm's merge ops for
    the other buffers"""
    nk, f, out = len(keys), 0, []
    for a in aggs:
        if a[0] == VARIANCE:
            out.append((AGG_VARIANCE, 8 + 8 * (nk + f), -1))
            f += 3
            continue
        for op, _ in pm.buffers([a]):
            out.append((op, 8 + 8 * (nk + f), nk + f))
            f += 1
    return out


# ---- the reduce side: the aggregated read's model with AGG_VARIANCE entries ----
def triple(row, off):
    return struct.unpack("<3d", bytes(row[off:off + 24]))


def model_aggregate(plain, keys, aggs):
    """dm.model_aggregate_decimal with AGG_VARIANCE entries (op, off, -1): each group's triples merged in stable order
    from (0, 0, 0) and written over the head row's 24 bytes -> (rows, number of records, number of groups)"""
    others = [a for a in aggs if a[0] != AGG_VARIANCE]
    out, n_rec, n_groups = dm.model_aggregate_decimal(plain, keys, others)
    var = [a for a in aggs if a[0] == AGG_VARIANCE]
    if not var:
        return out, n_rec, n_groups
    buf, recs, kv, order = rm.model_keys(plain, keys)
    patched, at, j = [], 0, 0
    while j < len(order):
        e = j
        while e < len(order) and kv[order[e]] == kv[order[j]]:
            e += 1
        sz = int.from_bytes(out[at:at + 4], "big")
        rec = bytearray(out[at:at + 4 + sz])
        at += 4 + sz
        rows = [buf[recs[i][0] + 4:recs[i][0] + recs[i][1]] for i in order[j:e]]
        for _, off, _ in var:
            m = merge_all([triple(r, off) for r in rows])
            rec[4 + off:4 + off + 24] = struct.pack("<3d", *m)
        patched.append(bytes(rec))
        j = e
    return b"".join(patched), n_rec, n_groups
