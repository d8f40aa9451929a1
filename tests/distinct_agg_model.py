"""One DISTINCT group's middle stage (AggUtils.planAggregateWithOneDistinct, Spark 3.5, ANSI off) row by row, as a
model for b2s_decompress_aggregate_distinct_partition_compress_rows_hash_*.

G are the grouping columns, X the distinct columns, F the non-distinct functions and D the distinct ones.  The map side
writes partial rows for key columns G ++ X and functions F (moments_model.partial_rows); a reducer of that exchange
runs
    stage 2: HashAggregate(G ++ X, F: PartialMerge): the aggregated read's stable sort by the composite key and its
             merges (rows_model.merge, decimal_model's merge_decimal and put_decimal, moments_model.merge_all);
    stage 3: HashAggregate(G, F: PartialMerge, D: Partial) over the merged rows in their order: per G group, F's
             buffers merged by mergeExpressions from their initial values (rows_model.merge, decimal_model's
             merge_decimal, moments_model.merge_all) and D's buffers updated by updateExpressions over the distinct
             column (partial_agg_model.update, moments_model.update),
and writes one partial row per G group as the map side writes its own (partial_agg_model.emit).  The merges and folds
are those models'; this module only orders, groups and wires them.  keys are [(key_type, key_len)], the first n_group_keys G; aggs are [(fn, val_type)];
distinct are [(fn, val_type, column or ALL)].
"""
import functools
import struct

import decimal_model as dm
import moments_model as mm
import partial_agg_model as pm
import rows_model as rm

ALL = -1  # B2S_DISTINCT_ALL_COLUMNS


def input_keys(keys):
    """the key columns at the partial rows' slots: column c at 8 + 8 c, null bit c"""
    return [(kt, 8 + 8 * c, kl, c) for c, (kt, kl) in enumerate(keys)]


def f_aggs(aggs):
    """F as the map-side models take them (no input slot: only the buffers' layout is read)"""
    return [(fn, vt, 0, -1) for fn, vt in aggs]


def merge_aggs(keys, aggs):
    """stage 2's entries: the aggregated read's merge ops over F's buffers"""
    return mm.merge_aggs(input_keys(keys), f_aggs(aggs))


def set_null(row, f, null):
    w = 8 * (f >> 6)
    v = int.from_bytes(row[w:w + 8], "little")
    row[w:w + 8] = (v | (1 << (f & 63)) if null else v & ~(1 << (f & 63))).to_bytes(8, "little")


def stage2(streams, keys, aggs):
    """the blocks' decoded streams -> (merged rows, input rows, (G, X) groups): the rows sorted stably by G ++ X in the
    composite-key order (partial_agg_model's comparator: its typed values group 0.0 with -0.0, NaN with NaN, decimals
    by value), each group's head row with F's buffers merged over the group as the aggregated read merges them"""
    buf = b"".join(streams)
    rows = [buf[o + 4:o + n] for o, n in rm.parse(buf)]
    ks = input_keys(keys)
    kv = [tuple(pm.col_value(r, c) for c in ks) for r in rows]
    cmp = pm.comparator(ks)
    order = sorted(range(len(rows)), key=functools.cmp_to_key(lambda a, b: cmp(kv[a], kv[b])))
    out, j = [], 0
    while j < len(order):
        e = j
        while e < len(order) and kv[order[e]] == kv[order[j]]:
            e += 1
        group = [rows[i] for i in order[j:e]]
        head = bytearray(group[0])
        for op, off, nf in merge_aggs(keys, aggs):
            if op == mm.AGG_VARIANCE:
                head[off:off + 24] = struct.pack("<3d", *mm.merge_all([mm.triple(r, off) for r in group]))
            elif op & 0xFF >= dm.SUM_DEC:
                x = dm.merge_decimal(op, [None if rm.is_null(r, nf) else dm.dec_value(r, off, op) for r in group])
                dm.put_decimal(memoryview(head), op, off, x)
                set_null(head, nf, x is None)
            else:
                vals = [bytes(r[off:off + 8]) for r in group if not rm.is_null(r, nf)]
                head[off:off + 8] = rm.merge(op, vals) if vals else bytes(8)
                set_null(head, nf, not vals)
        out.append(bytes(head))
        j = e
    return out, len(rows), len(out)


def _value(op, kind, slot):
    if kind == "double":
        return struct.unpack("<d", slot)[0]
    if kind in ("int", "bool"):
        return int.from_bytes(slot[:4], "little", signed=True)
    return int.from_bytes(slot, "little", signed=True)


def merge_f(rows, keys, aggs):
    """F's buffers of one G group merged from their initial values over its merged rows in order -> values"""
    values = []
    if not rows:  # no input: the initial values
        for a in f_aggs(aggs):
            values += [0.0, 0.0, 0.0] if a[0] == mm.VARIANCE else pm.state_values(pm.new_state([a]), [a])
        return values
    entries = merge_aggs(keys, aggs)
    bufs = [b for b in mm.buffers(f_aggs(aggs))]
    k = 0
    for op, off, nf in entries:
        if op == mm.AGG_VARIANCE:
            values += list(mm.merge_all([mm.triple(r, off) for r in rows]))
            k += 3
            continue
        kind = bufs[k][1]
        k += 1
        if op & 0xFF >= dm.SUM_DEC:
            values.append(dm.merge_decimal(op, [None if rm.is_null(r, nf) else dm.dec_value(r, off, op)
                                                for r in rows]))
            continue
        vals = [bytes(r[off:off + 8]) for r in rows if not rm.is_null(r, nf)]
        values.append(_value(op, kind, rm.merge(op, vals)) if vals else None)
    return values


def d_aggs(distinct):
    return [(fn, vt, 8 + 8 * col, col) for fn, vt, col in distinct]


def update_d(rows, n_group_keys, keys, distinct):
    """D's buffers of one G group updated over the distinct column of each merged row in order -> values"""
    values = []
    for fn, vt, col in distinct:
        if col == ALL:  # Count(x1, .., xn): the rows with no distinct column null
            values.append(sum(all(not rm.is_null(r, c) for c in range(n_group_keys, len(keys))) for r in rows))
            continue
        a = (fn, vt, 8 + 8 * col, col)
        if fn == mm.VARIANCE:
            values += list(mm.fold([mm.to_double(pm.read_value(r, vt, a[2], col), vt) for r in rows]))
            continue
        st = pm.new_state([a])
        for r in rows:
            pm.update(st, [a], r)
        values += pm.state_values(st, [a])
    return values


def out_buffers(aggs, distinct):
    """the output row's buffers (merge op, kind): F's, then D's"""
    out = mm.buffers(f_aggs(aggs))
    for fn, vt, col in distinct:
        out += [(pm.SUM_I64, "long")] if col == ALL else mm.buffers([(fn, vt, 0, -1)])
    return out


def stage3(merged, n_group_keys, keys, aggs, distinct):
    """the merged (G, X) rows in order -> the output partial rows, one per G group (one initial row without G and
    without rows)"""
    g_keys = input_keys(keys)[:n_group_keys]
    bufs = out_buffers(aggs, distinct)
    groups = []
    for r in merged:
        k = tuple(pm.col_value(r, c) for c in g_keys)
        if groups and groups[-1][0] == k:
            groups[-1][1].append(r)
        else:
            groups.append((k, [r]))
    if not groups and not n_group_keys:
        groups = [((), [])]
    out = []
    for _, rows in groups:
        values = merge_f(rows, keys, aggs) + update_d(rows, n_group_keys, keys, distinct)
        out.append(pm.emit(rows[0] if rows else b"", g_keys, bufs, values))
    return out


def reducer(streams, n_group_keys, keys, aggs, distinct):
    """stages 2 and 3 of one reduce task -> (output rows, [input rows, (G, X) groups, output rows])"""
    merged, n_rec, n_gx = stage2(streams, keys, aggs)
    out = stage3(merged, n_group_keys, keys, aggs, distinct)
    return out, [n_rec, n_gx, len(out)]


def final_aggs(n_group_keys, aggs, distinct):
    """the Final merge's entries (b2s_decompress_aggregate_rows_keys_*) over the output rows, keyed by G"""
    g = [(0, 0)] * n_group_keys
    fa = f_aggs(aggs) + [(pm.COUNT, pm.VAL_NONE, 0, -1) if col == ALL else (fn, vt, 0, -1)
                         for fn, vt, col in distinct]
    return mm.merge_aggs(input_keys(g), fa)
