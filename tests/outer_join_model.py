"""A model of b2s_decompress_join_rows_keys_*'s right and full outer joins, written from its header contract, beside
join_model.py's model of the other join types (which it serves unchanged).

The null left side of a joined row is what UnsafeRowJoiner makes of the row UnsafeRowWriter writes with every field
null: every bit set, zero slots, and each DECIMAL_WIDE field's 16 zero bytes with slot offset << 32.  Joining that row
moves each wide decimal's slot to 8 (b + nL + nR) + 16 k, and the right side's offsets past its 16-byte regions, as the
contract states; so join_model.joined builds every row here."""
import join_model
from join_model import DECIMAL_WIDE, joined, side_records, sort_side, words

RIGHT_OUTER, FULL_OUTER = 5, 6


def null_row(n, kinds):
    """the UnsafeRow of n fields, all null: every bit set, zero slots, a null wide decimal's 16 zero bytes"""
    bw = words(n)
    wide = [f for f in range(n) if kinds[f] == DECIMAL_WIDE]
    slots = [0] * n
    for k, f in enumerate(wide):
        slots[f] = (8 * (bw + n) + 16 * k) << 32
    bits = ((1 << n) - 1).to_bytes(8 * bw, "little")
    return bits + b"".join(s.to_bytes(8, "little") for s in slots) + bytes(16 * len(wide))


def join_row(left, right, nl, nr, lkinds, rkinds):
    """the joined row of left and right (None: an outer join's null side; never both)"""
    return joined(null_row(nl, lkinds) if left is None else left, right, nl, nr, lkinds, rkinds)


def key_order(k):
    """the sort order of a key (ascending, nulls first; a null column compares equal to every null), as sort_side's"""
    return [(f, 0 if v is None else v) for f, v in k]


def model_join(join_type, left_plain, right_plain, left_keys, right_keys, nl, nr, lkinds=None, rkinds=None):
    """join_model.model_join for every join type -> (the output stream's bytes, n_left_records, n_right_records,
    n_out_records).  Right and full outer joins go by runs: the records of both sides whose keys are equal in the sort
    order (nulls equal to nulls); a run matches when its key has no null column and it holds records of both sides."""
    if join_type not in (RIGHT_OUTER, FULL_OUTER):
        return join_model.model_join(join_type, left_plain, right_plain, left_keys, right_keys, nl, nr, lkinds, rkinds)
    L = sort_side(side_records(left_plain), left_keys)
    R = sort_side(side_records(right_plain), right_keys)
    runs = {}
    for s, side in enumerate((L, R)):
        for k, x in side:
            runs.setdefault(k, ([], []))[s].append(x)

    def row(l, r):
        return join_row(l, r, nl, nr, lkinds, rkinds)
    out = []
    if join_type == RIGHT_OUTER:  # for each r of Rs, its run's left records in Ls order, or the null left side
        for k, r in R:
            ls = runs[k][0] if all(f for f, _ in k) else []
            out += [row(l, r) for l in ls] or [row(None, r)]
    else:
        for k in sorted(runs, key=key_order):
            ls, rs = runs[k]
            match = all(f for f, _ in k) and ls and rs
            for l in ls:
                out += [row(l, r) for r in rs] if match else [row(l, None)]
            if not match:
                out += [row(None, r) for r in rs]
    stream = b"".join(len(r).to_bytes(4, "big") + r for r in out)
    return stream, len(L), len(R), len(out)
