"""A model of b2s_decompress_join_rows_keys_*, written from its header contract: Spark's SortMergeJoinExec on a reducer
(inner, left outer, left semi, left anti) with the joined rows UnsafeRowJoiner builds.

Keys are compared as Spark compares join keys after NormalizeFloatingNumbers: per column (not-null flag, value), ints
signed, floats with -0.0 made 0.0 and every NaN one value, decimals as signed unscaled integers, strings and BYTES as
Python bytes.  A key with a null column matches nothing.  The joined row is built here from the rows' bytes with Python
integers for the null bitsets, independently of the GPU code."""
import math
import struct

from rows_model import is_null, parse

KEY_BYTES, KEY_INT32, KEY_INT64, STRING, KEY_INT16, KEY_INT8, KEY_FLOAT32, KEY_FLOAT64, DECIMAL = 0, 1, 2, 3, 5, 6, 7, 8, 9
INNER, LEFT_OUTER, LEFT_SEMI, LEFT_ANTI = 0, 1, 2, 3
FIXED, VAR, DECIMAL_WIDE = 0, 1, 2


def words(n):
    return (n + 63) // 64


def _float(b, fmt):
    x = struct.unpack(fmt, b)[0]
    return (1, 0.0) if math.isnan(x) else (0, x + 0.0)


def col_value(row, col):
    """one key column (type, offset, length, null field) of a row -> (not-null flag, normalized value)"""
    kt, ko, kl, nf = col
    if nf >= 0 and is_null(row, nf):
        return (0, None)
    raw = bytes(row[ko:ko + kl])
    if kt in (STRING, DECIMAL):
        slot = int.from_bytes(raw, "little")
        data = bytes(row[slot >> 32:(slot >> 32) + (slot & 0xFFFFFFFF)])
        return (1, data if kt == STRING else int.from_bytes(data, "big", signed=True))
    if kt == KEY_BYTES:
        return (1, raw)
    if kt == KEY_FLOAT32:
        return (1, _float(raw, "<f"))
    if kt == KEY_FLOAT64:
        return (1, _float(raw, "<d"))
    return (1, int.from_bytes(raw, "little", signed=True))


def side_records(plain_blocks):
    """the rows (without size prefixes) of a side's decoded blocks, in block order"""
    buf = b"".join(plain_blocks)
    return [buf[o + 4:o + ln] for o, ln in parse(buf)]


def sort_side(rows, keys):
    """-> [(key, row)] stably sorted by the key (ascending, nulls first)"""
    kv = [tuple(col_value(r, c) for c in keys) for r in rows]
    order = sorted(range(len(rows)), key=lambda i: [(f, 0 if v is None else v) for f, v in kv[i]])
    return [(kv[i], rows[i]) for i in order]


def joined(left, right, nl, nr, lkinds, rkinds):
    """UnsafeRowJoiner's row of left and right (None: the null right side of a left outer join)"""
    bl, br, b = words(nl), words(nr), words(nl + nr)
    var_l = bytes(left[8 * (bl + nl):])
    lbits = int.from_bytes(left[:8 * bl], "little") & ((1 << nl) - 1)
    wide = [f for f in range(nr) if rkinds[f] == DECIMAL_WIDE]
    if right is None:
        rbits = (1 << nr) - 1
        rslots = [0] * nr
        var_r = bytes(16 * len(wide))
        for k, f in enumerate(wide):
            rslots[f] = (8 * (b + nl + nr) + len(var_l) + 16 * k) << 32
    else:
        rbits = int.from_bytes(right[:8 * br], "little") & ((1 << nr) - 1)
        rslots = [int.from_bytes(right[8 * (br + f):8 * (br + f) + 8], "little") for f in range(nr)]
        var_r = bytes(right[8 * (br + nr):])
        for f in range(nr):
            if rkinds[f] != FIXED and rslots[f]:
                rslots[f] += (8 * (b - br + nl) + len(var_l)) << 32
    lslots = [int.from_bytes(left[8 * (bl + f):8 * (bl + f) + 8], "little") for f in range(nl)]
    for f in range(nl):
        if lkinds[f] != FIXED and lslots[f]:
            lslots[f] += (8 * (b - bl + nr)) << 32
    bits = (lbits | (rbits << nl)).to_bytes(8 * b, "little")
    row = bits + b"".join(s.to_bytes(8, "little") for s in lslots + rslots) + var_l + var_r
    return row


def model_join(join_type, left_plain, right_plain, left_keys, right_keys, nl, nr, lkinds=None, rkinds=None):
    """-> (the output stream's bytes, n_left_records, n_right_records, n_out_records)"""
    L = sort_side(side_records(left_plain), left_keys)
    R = sort_side(side_records(right_plain), right_keys)
    by_key = {}
    for k, r in R:
        if all(f for f, _ in k):
            by_key.setdefault(k, []).append(r)
    out = []
    for k, l in L:
        matches = by_key.get(k, []) if all(f for f, _ in k) else []
        if join_type == LEFT_SEMI:
            out += [l] if matches else []
        elif join_type == LEFT_ANTI:
            out += [] if matches else [l]
        else:
            out += [joined(l, r, nl, nr, lkinds, rkinds) for r in matches]
            if join_type == LEFT_OUTER and not matches:
                out.append(joined(l, None, nl, nr, lkinds, rkinds))
    stream = b"".join(len(r).to_bytes(4, "big") + r for r in out)
    return stream, len(L), len(R), len(out)
