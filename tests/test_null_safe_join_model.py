"""The null-safe join and existence join model (null_safe_join_model.py) pinned on hand-worked cases: where a null-safe
null sorts, that the model reduces to the plain join without nulls, that existence rows are semi and anti rows with the
bit, that INTERSECT and EXCEPT come out as Python's set logic, and the two-step hash."""
import numpy as np
import pytest

import null_safe_join_model as M
from hash_model import SEED, col_hash, hash_bytes, hash_int, hash_long, keys_of, make_row, row_hash
from join_model import LEFT_ANTI, LEFT_SEMI, col_value, side_records
from outer_join_model import model_join as plain_join
from rows_model import blocks_of

NS = M.NULL_SAFE


def ns(keys):
    return [(t | NS, o, ln, nf) for t, o, ln, nf in keys]


def order(t, vals):
    rows = [make_row([t], [v]) for v in vals]
    keys = ns(keys_of([t], [0]))
    return [col_value(r, (keys[0][0] & 0xFF,) + keys[0][1:])[1] for _, r in M.sort_side(rows, keys)]


def test_a_null_sorts_directly_after_the_default():
    assert order("string", [b"a", None, b"", b"\x00"]) == [b"", None, b"\x00", b"a"]
    assert order("int", [1, None, 0, -1]) == [-1, 0, None, 1]
    assert order("long", [None, 0, -5]) == [-5, 0, None]
    assert order("bool", [True, None, False]) == [b"\x00", None, b"\x01"]
    nan = ("bits", 0x7FF8000000000000)
    got = order("double", [nan, 1.0, None, -0.0, 0.0, -1.0])
    assert got == [(0, -1.0), (0, 0.0), (0, 0.0), None, (0, 1.0), (1, 0.0)]  # -0.0 == 0.0, NaN above every value
    assert order("float", [None, -0.0]) == [(0, 0.0), None]
    assert order("decimal", [10**30, None, 0, -(10**30)]) == [-(10**30), 0, None, 10**30]


def test_null_safe_nulls_match_and_plain_nulls_do_not():
    lt = rt = ["int", "string"]
    L = [make_row(lt, [None, b"x"]), make_row(lt, [1, None]), make_row(lt, [None, None])]
    R = [make_row(rt, [None, b"x"]), make_row(rt, [1, None])]
    keys = keys_of(lt, [0, 1])
    both = ns(keys)
    mixed = [both[0], keys[1]]  # column 0 null-safe, column 1 plain
    semi = lambda k: M.model_join(LEFT_SEMI, blocks_of(L, [3]), blocks_of(R, [2]), k, k, 2, 2)  # noqa: E731
    assert semi(both)[3] == 2 and semi(mixed)[3] == 1 and semi(keys)[3] == 0


@pytest.mark.parametrize("jt", M.ALL_JOINS[:6])
def test_without_nulls_a_null_safe_join_is_the_plain_join(jt):
    rng = np.random.default_rng(jt)
    lt, rt = ["long", "string", "decimal"], ["decimal", "long", "string"]
    kinds_l, kinds_r = [0, 1, 2], [2, 0, 1]

    def rows(types, n):
        out = []
        for _ in range(n):
            v = {"long": int(rng.integers(0, 6)), "string": bytes(rng.integers(97, 99, 2, dtype=np.uint8)),
                 "decimal": int(rng.integers(-2, 2)) * 10**25}
            out.append(make_row(types, [v[t] for t in types]))
        return out
    L, R = blocks_of(rows(lt, 60), [30, 30]), blocks_of(rows(rt, 50), [50])
    lk, rk = keys_of(lt, [0, 1]), keys_of(rt, [1, 2])
    want = plain_join(jt, L, R, lk, rk, 3, 3, kinds_l, kinds_r)
    assert M.model_join(jt, L, R, ns(lk), ns(rk), 3, 3, kinds_l, kinds_r) == want
    assert M.model_join(jt, L, R, [ns(lk)[0], lk[1]], [ns(rk)[0], rk[1]], 3, 3, kinds_l, kinds_r) == want


@pytest.mark.parametrize("nl", [1, 3, 63, 64])
def test_existence_rows_are_semi_and_anti_rows_with_the_bit(nl):
    rng = np.random.default_rng(nl)
    types = ["string"] + ["long"] * (nl - 1)
    kinds = [1] + [0] * (nl - 1)

    def rows(n):
        return [make_row(types, [None if rng.random() < 0.2 else bytes([97 + int(rng.integers(4))])] +
                         [int(rng.integers(9)) for _ in range(nl - 1)]) for _ in range(n)]
    L, R = blocks_of(rows(40), [40]), blocks_of(rows(10), [10])
    k = ns(keys_of(types, [0]))
    stream, n_l, _, n_out = M.model_join(M.EXISTENCE, L, R, k, k, nl, 1, kinds)
    assert n_out == n_l == 40
    got = side_records([stream])
    kept = set(side_records([M.model_join(LEFT_SEMI, L, R, k, k, nl, 1)[0]]))
    dropped = set(side_records([M.model_join(LEFT_ANTI, L, R, k, k, nl, 1)[0]]))
    order_ = [r for _, r in M.sort_side(side_records(L), k)]
    assert [M.exists_row(r, nl, kinds, r in kept) for r in order_] == got
    assert all((r in kept) != (r in dropped) for r in order_)
    b = (nl + 64) // 64
    for r, g in zip(order_, got):
        assert int.from_bytes(g[8 * (b + nl):8 * (b + nl) + 8], "little") == (r in kept)
        assert len(g) == len(r) + 8 * (b - (nl + 63) // 64 + 1)


def test_intersect_and_except_are_set_logic_over_tuples_with_none():
    rng = np.random.default_rng(5)
    types = ["int", "string", "long"]
    pick = lambda: (None if rng.random() < 0.3 else int(rng.integers(3)),  # noqa: E731
                    None if rng.random() < 0.3 else bytes([97 + int(rng.integers(2))]),
                    None if rng.random() < 0.3 else int(rng.integers(2)))
    lv, rv = [pick() for _ in range(200)], [pick() for _ in range(150)]
    L = blocks_of([make_row(types, list(v)) for v in lv], [100, 100])
    R = blocks_of([make_row(types, list(v)) for v in rv], [150])
    k = ns(keys_of(types, [0, 1, 2]))
    plain = keys_of(types, [0, 1, 2])

    def values(stream):
        return {tuple(col_value(r, c)[1] for c in plain) for r in side_records([stream])}
    assert values(M.model_join(LEFT_SEMI, L, R, k, k, 3, 3)[0]) == set(lv) & set(rv)
    assert values(M.model_join(LEFT_ANTI, L, R, k, k, 3, 3)[0]) == set(lv) - set(rv)


def test_the_null_safe_hash_takes_two_steps():
    types = ["int", "string", "decimal", "double", "bool", "long", "float"]
    null_row = make_row(types, [None] * len(types))
    keys = keys_of(types, range(len(types)))
    h = SEED
    for step in (lambda h: hash_int(0, h), lambda h: hash_bytes(b"", h), lambda h: hash_bytes(b"\x00", h),
                 lambda h: hash_long(0, h), lambda h: hash_int(0, h), lambda h: hash_long(0, h),
                 lambda h: hash_int(0, h)):
        h = hash_int(1, step(h))
    assert M.row_hash(null_row, ns(keys)) == h
    assert row_hash(null_row, keys) == SEED  # a plain null leaves h
    full = make_row(types, [7, b"abc", 10**30, -0.0, True, -3, 2.5])
    h = SEED
    for c in keys:  # the value by hash_model's plain rule, then hashInt(false)
        h = hash_int(0, col_hash(full, c, h))
    assert M.row_hash(full, ns(keys)) == h
    # a column without a null bit is never null: its second step is hashInt(0)
    k = [(keys[0][0] | NS, keys[0][1], keys[0][2], -1)]
    assert M.row_hash(null_row, k) == hash_int(0, hash_int(0, SEED))
