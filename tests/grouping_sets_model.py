"""Spark's Expand for grouping sets (ROLLUP, CUBE, GROUPING SETS), row by row, as a model for
b2s_aggregate_grouping_sets_partition_compress_rows_hash_*.

Each input row is projected once per grouping set, in ExpandExec's row-major order: key column c keeps its value when
bit c of the set's mask is set and is null otherwise, gid (spark_grouping_id: the sum of 1 << (n_keys - 1 - c) over the
columns outside the set) follows the key columns, and each aggregate's input is read from the row unmasked.  The
projected rows feed partial_agg_model.partial_rows with the keys and aggregates expand() returns.
"""
import partial_agg_model as pm
from rows_model import is_null
from test_gpu_sort_rows_order import DECIMAL, col_value

STRING, KEY_INT64 = 3, 2


def gid(mask, n_keys):
    """Spark's spark_grouping_id of a set: bit n_keys - 1 - c set for every key column c outside it"""
    return sum(1 << (n_keys - 1 - c) for c in range(n_keys) if not (mask >> c) & 1)


def rollup(n):
    """ROLLUP(c0, .., c{n-1}): the masks of (c0..c{n-1}), (c0..c{n-2}), .., (), in Spark's order"""
    return [(1 << m) - 1 for m in range(n, -1, -1)]


def cube(n):
    """CUBE(c0, .., c{n-1}): every subset, in Spark's order (its gid counting up from 0)"""
    full = (1 << n) - 1
    return [full & ~sum(1 << c for c in range(n) if (g >> (n - 1 - c)) & 1) for g in range(1 << n)]


def projected_keys(keys):
    """the key columns of the projected rows: the grouping columns (each with a null bit), then gid"""
    nk = len(keys)
    return [(kt, 8 + 8 * c, kl, c) for c, (kt, _, kl, _) in enumerate(keys)] + [(KEY_INT64, 8 + 8 * nk, 8, -1)]


def projected_aggs(keys, aggs):
    """the aggregates over the projected rows: input i (of the functions that take one) at field n_keys + 1 + i"""
    out, i = [], 0
    for fn, vt, off, nf in aggs:
        if vt & 0xFF == pm.VAL_NONE:
            out.append((fn, vt, 0, -1))
            continue
        f = len(keys) + 1 + i
        out.append((fn, vt, 8 + 8 * f, f if nf >= 0 else -1))
        i += 1
    return out


def _wide(vt):
    return vt & 0xFF == pm.VAL_DECIMAL and (vt >> 8) & 0xFF > 18


def project(row, keys, aggs, mask):
    """one input row under one grouping set -> the projected UnsafeRow"""
    nk = len(keys)
    ins = [a for a in aggs if a[1] & 0xFF != pm.VAL_NONE]
    nf = nk + 1 + len(ins)
    assert nf <= 32
    fixed = 8 + 8 * nf
    out = bytearray(fixed)
    var = bytearray()
    nulls = 0

    def put_var(f, data, pad_to):
        out[8 + 8 * f:16 + 8 * f] = ((fixed + len(var)) << 32 | len(data)).to_bytes(8, "little")
        var.extend(data + bytes(pad_to - len(data)))

    def out_of_line(at):
        s = int.from_bytes(row[at:at + 8], "little")
        return bytes(row[s >> 32:(s >> 32) + (s & 0xFFFFFFFF)])

    for c, (kt, ko, kl, knf) in enumerate(keys):
        t = kt & 0xFF
        if not (mask >> c) & 1 or (knf >= 0 and is_null(row, knf)):
            nulls |= 1 << c
            if (mask >> c) & 1 and t == DECIMAL:
                put_var(c, b"", 16)
            continue
        if t == STRING:
            b = out_of_line(ko)
            put_var(c, b, len(b) + (-len(b) % 8))
        elif t == DECIMAL:
            put_var(c, out_of_line(ko), 16)
        else:
            out[8 + 8 * c:8 + 8 * c + kl] = row[ko:ko + kl]
    out[8 + 8 * nk:16 + 8 * nk] = gid(mask, nk).to_bytes(8, "little")
    for i, (fn, vt, off, anf) in enumerate(ins):
        f = nk + 1 + i
        null = anf >= 0 and is_null(row, anf)
        if null:
            nulls |= 1 << f
        reads = fn != pm.COUNT and not null
        if _wide(vt):
            put_var(f, out_of_line(off) if reads else b"", 16)
        elif reads:
            out[8 + 8 * f:16 + 8 * f] = row[off:off + 8]
    out[0:8] = nulls.to_bytes(8, "little")
    return bytes(out + var)


def expand(rows, keys, aggs, masks):
    """ExpandExec's output in row-major order (every set of row 0, then of row 1, ...) -> (projected rows, their key
    columns, their aggregates)"""
    return ([project(r, keys, aggs, m) for r in rows for m in masks], projected_keys(keys),
            projected_aggs(keys, aggs))


def partial_rows(rows, keys, aggs, masks):
    """the map side's partial rows: Expand, then HashAggregateExec(Partial) over the projected rows"""
    xrows, xkeys, xaggs = expand(rows, keys, aggs, masks)
    return pm.partial_rows(xrows, xkeys, xaggs)


def group_by_each_set(rows, keys, aggs, masks):
    """the whole dataset grouped by each set on its own, as a plain GROUP BY of the set's columns would group it ->
    {(grouping values with None outside the set, gid): buffer values}"""
    out = {}
    for m in masks:
        groups = {}
        for r in rows:
            k = tuple(col_value(r, col) if (m >> c) & 1 else None for c, col in enumerate(keys))
            if k not in groups:
                groups[k] = pm.new_state(aggs)
            pm.update(groups[k], aggs, r)
        for k, st in groups.items():
            vals = pm.state_values(st, aggs)  # a long sum wraps, as Spark's Add with ANSI off
            out[k + (gid(m, len(keys)),)] = [(v + 2**63) % 2**64 - 2**63 if v is not None and kind == "long" else v
                                             for v, (_, kind) in zip(vals, pm.buffers(aggs))]
    return out
