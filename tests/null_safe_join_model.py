"""A model of the join call's null-safe (<=>) key columns and existence join, and of the hash call's null-safe columns,
written from the header contract beside join_model.py and outer_join_model.py (whose row builders it uses unchanged).

The Spark 3.5 facts it rests on, each next to the expression it comes from:
- ExtractEquiJoinKeys turns `l <=> r` into two key pairs, in this order:
  (Coalesce(l :: Literal.default(l.dataType) :: Nil), Coalesce(r :: Literal.default(r.dataType) :: Nil)), then
  (IsNull(l), IsNull(r)).  So a null-safe column is the pair (coalesce(v, default), isnull(v)); both sort ascending
  (SortMergeJoinExec.requiredChildOrdering over the expanded keys), and a null equals a null and sorts directly after
  the non-null default.  Only a null in a plain column makes a key unmatchable (the join's anyNull test runs over the
  expanded keys, which are never null).
- When a side's column is not nullable, the optimizer folds that side's pair to (col, false): the same pair with
  isnull false, which is what a null field of -1 means here.
- Literal.default: 0 for numeric, date and timestamp types (DefaultValue of IntegerType, LongType, ...), 0 for decimals
  (Decimal(0)), UTF8String.EMPTY_UTF8 for strings, an empty array for binary, false for booleans.
- HashPartitioning over the expanded keys is Murmur3Hash(coalesce, isnull): the coalesced value by its type's rule (a
  wide decimal of 0 as BigInteger.ZERO.toByteArray(), the one byte 0x00; the empty string as hashUnsafeBytes of no
  bytes), then the boolean as hashInt(isnull ? 1 : 0).  A null no longer leaves h unchanged.
- SortMergeJoinExec(ExistenceJoin(exists)) outputs left.output :+ exists, exists a non-nullable boolean: one row per
  left row, in the left side's key order, built by UnsafeProjection (the boolean's slot zeroed, then one byte).
- ReplaceIntersectWithSemiJoin / ReplaceExceptWithAntiJoin: INTERSECT is Distinct(LeftSemi(l, r, <=> over every
  column)), EXCEPT is Distinct(LeftAnti(l, r, <=> over every column))."""
from hash_model import SEED, col_hash, hash_bytes, hash_int, hash_long
from join_model import (DECIMAL, DECIMAL_WIDE, FIXED, INNER, KEY_BYTES, KEY_FLOAT32, KEY_FLOAT64, KEY_INT64, LEFT_ANTI,
                        LEFT_OUTER, LEFT_SEMI, STRING, VAR, col_value, side_records, words)
from outer_join_model import FULL_OUTER, RIGHT_OUTER, join_row
from rows_model import is_null

NULL_SAFE = 1 << 10
EXISTENCE = 8
ALL_JOINS = [INNER, LEFT_OUTER, LEFT_SEMI, LEFT_ANTI, RIGHT_OUTER, FULL_OUTER, EXISTENCE]
__all__ = ["NULL_SAFE", "EXISTENCE", "ALL_JOINS", "DECIMAL_WIDE", "FIXED", "VAR"]


def default_value(kt, kl):
    """Literal.default of the column's type, normalized as join_model.col_value normalizes values"""
    if kt == KEY_BYTES:
        return bytes(kl)  # boolean false
    if kt == STRING:
        return b""
    if kt in (KEY_FLOAT32, KEY_FLOAT64):
        return (0, 0.0)
    return 0  # ints, dates, timestamps, decimals


def key_element(row, col):
    """one key column's order element: a plain column (not-null flag, value), a null-safe one (coalesce(v, default),
    isnull(v)); both compare as Python tuples"""
    kt, ko, kl, nf = col
    if kt & NULL_SAFE:
        f, v = col_value(row, (kt & 0xFF, ko, kl, nf))
        return (default_value(kt & 0xFF, kl), 1) if not f else (v, 0)
    f, v = col_value(row, col)
    return (f, 0 if v is None else v)


def matchable(key, cols):
    """a key can match: none of its plain columns is null"""
    return all(c[0] & NULL_SAFE or e[0] for e, c in zip(key, cols))


def sort_side(rows, cols):
    """-> [(key, row)] stably sorted by the key"""
    keyed = [(tuple(key_element(r, c) for c in cols), r) for r in rows]
    return sorted(keyed, key=lambda kr: kr[0])


def exists_row(left, nl, lkinds, exists):
    """left.output :+ exists: b = ceil((nl + 1) / 64) null words, the left's slots, the boolean, the left's var bytes;
    each non-zero VAR / DECIMAL_WIDE slot moved by 8 (b - bl + 1)"""
    bl, b = words(nl), words(nl + 1)
    bits = int.from_bytes(left[:8 * bl], "little") & ((1 << nl) - 1)
    slots = [int.from_bytes(left[8 * (bl + f):8 * (bl + f) + 8], "little") for f in range(nl)]
    for f in range(nl):
        if lkinds[f] != FIXED and slots[f]:
            slots[f] += (8 * (b - bl + 1)) << 32
    return (bits.to_bytes(8 * b, "little") + b"".join(s.to_bytes(8, "little") for s in slots) +
            int(exists).to_bytes(8, "little") + bytes(left[8 * (bl + nl):]))


def model_join(join_type, left_plain, right_plain, left_keys, right_keys, nl, nr, lkinds=None, rkinds=None):
    """every join type, null-safe columns (key type | NULL_SAFE, the left's types for both sides) included
    -> (the output stream's bytes, n_left_records, n_right_records, n_out_records)"""
    L = sort_side(side_records(left_plain), left_keys)
    R = sort_side(side_records(right_plain), right_keys)
    runs = {}
    for s, side in enumerate((L, R)):
        for k, x in side:
            runs.setdefault(k, ([], []))[s].append(x)

    def partners(k, s):
        return runs[k][s] if matchable(k, left_keys) and k in runs else []

    def row(l, r):
        return join_row(l, r, nl, nr, lkinds, rkinds)
    out = []
    if join_type == RIGHT_OUTER:
        for k, r in R:
            out += [row(l, r) for l in partners(k, 0)] or [row(None, r)]
    elif join_type == FULL_OUTER:
        for k in sorted(runs):
            ls, rs = runs[k]
            match = matchable(k, left_keys) and ls and rs
            for l in ls:
                out += [row(l, r) for r in rs] if match else [row(l, None)]
            if not match:
                out += [row(None, r) for r in rs]
    else:
        for k, l in L:
            rs = partners(k, 1)
            if join_type == LEFT_SEMI:
                out += [l] if rs else []
            elif join_type == LEFT_ANTI:
                out += [] if rs else [l]
            elif join_type == EXISTENCE:
                out.append(exists_row(l, nl, lkinds, bool(rs)))
            else:
                out += [row(l, r) for r in rs]
                if join_type == LEFT_OUTER and not rs:
                    out.append(row(l, None))
    stream = b"".join(len(r).to_bytes(4, "big") + r for r in out)
    return stream, len(L), len(R), len(out)


def col_hash_null_safe(row, col, h):
    """one key column folded into h: a plain column as hash_model.col_hash; a null-safe one its coalesced value by its
    type's rule (the default when null), then hashInt(isnull)"""
    kt, ko, kl, nf = col
    if not kt & NULL_SAFE:
        return col_hash(row, col, h)
    base = kt & 0xFF
    null = bool(is_null(row, nf))
    if not null:
        h = col_hash(row, (base, ko, kl, -1), h)
    elif base == STRING:
        h = hash_bytes(b"", h)
    elif base == DECIMAL:
        h = hash_bytes(b"\x00", h)  # BigInteger.ZERO.toByteArray()
    elif base in (KEY_INT64, KEY_FLOAT64):
        h = hash_long(0, h)
    else:
        h = hash_int(0, h)  # false, 0, 0.0f
    return hash_int(1 if null else 0, h)


def row_hash(row, keys):
    """Murmur3Hash(expanded keys, 42) of a row (bytes without the size prefix), unsigned 32 bits"""
    h = SEED
    for col in keys:
        h = col_hash_null_safe(row, col, h)
    return h
