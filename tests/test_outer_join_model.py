"""The model of right and full outer joins (outer_join_model.py) pinned without a GPU: their rows against a nested-loop
definition over the rows' Python values, written here independently of the model, and their order on small hand-built
cases (null keys on both sides, keys on one side only, a two-column key with one column null)."""
import numpy as np
import pytest

from hash_model import keys_of
from join_model import INNER, LEFT_OUTER
from outer_join_model import FULL_OUTER, RIGHT_OUTER, join_row, model_join
from rows_model import blocks_of
from test_gpu_join_rows import kinds, row

LT = ["long", "string", "decimal", "int"]
RT = ["decimal", "string", "long"]


def _records(stream):
    out, p = [], 0
    while p < len(stream):
        s = int.from_bytes(stream[p:p + 4], "big")
        out.append(stream[p + 4:p + 4 + s])
        p += 4 + s
    return out


def _model(jt, lrows, rrows, lkeys, rkeys, lt=LT, rt=RT):
    got = model_join(jt, blocks_of(lrows, [len(lrows)]), blocks_of(rrows, [len(rrows)]), lkeys, rkeys, len(lt),
                     len(rt), kinds(lt), kinds(rt))
    assert got[1:3] == (len(lrows), len(rrows))
    return _records(got[0])


def _tables(rng, n_left, n_right, key_range, null_rate):
    """LT and RT rows' values, the long key (left field 0, right field 2) in [0, key_range) or null"""
    def key():
        return None if rng.random() < null_rate else int(rng.integers(0, key_range))

    def s():
        return bytes(rng.integers(97, 100, int(rng.integers(0, 9)), dtype=np.uint8))

    def dec():
        return int(rng.integers(-10**17, 10**17)) * 1000
    return ([[key(), s(), dec(), int(rng.integers(-9, 9))] for _ in range(n_left)],
            [[dec(), s(), key()] for _ in range(n_right)])


@pytest.mark.parametrize("seed", range(6))
def test_outer_rows_are_the_nested_loop_definition(seed):
    rng = np.random.default_rng(seed)
    lv, rv = _tables(rng, 40 + 10 * seed, 30 + 7 * seed, key_range=8 + seed, null_rate=0.15)
    lrows, rrows = [row(LT, v) for v in lv], [row(RT, v) for v in rv]
    lkeys, rkeys = keys_of(LT, [0]), keys_of(RT, [2])

    def j(l, r):
        return join_row(None if l is None else lrows[l], None if r is None else rrows[r], len(LT), len(RT), kinds(LT),
                      kinds(RT))

    def eq(a, b):
        return a is not None and b is not None and a == b

    pairs = [(i, k) for i in range(len(lv)) for k in range(len(rv)) if eq(lv[i][0], rv[k][2])]
    left_alone = [i for i in range(len(lv)) if not any(eq(lv[i][0], r[2]) for r in rv)]
    right_alone = [k for k in range(len(rv)) if not any(eq(l[0], rv[k][2]) for l in lv)]
    inner = [j(i, k) for i, k in pairs]
    full = inner + [j(i, None) for i in left_alone] + [j(None, k) for k in right_alone]
    right_outer = inner + [j(None, k) for k in right_alone]
    assert sorted(_model(FULL_OUTER, lrows, rrows, lkeys, rkeys)) == sorted(full)
    assert sorted(_model(RIGHT_OUTER, lrows, rrows, lkeys, rkeys)) == sorted(right_outer)
    assert sorted(_model(INNER, lrows, rrows, lkeys, rkeys)) == sorted(inner)
    # a full outer join's rows with a left side are the left outer join's, in its order
    lo = _model(LEFT_OUTER, lrows, rrows, lkeys, rkeys)
    null_left = set(j(None, k) for k in range(len(rv)))
    assert [x for x in _model(FULL_OUTER, lrows, rrows, lkeys, rkeys) if x not in null_left] == lo


def _order_case(lt, rt, lvals, rvals, lkeys, rkeys):
    """-> (expect: the joined rows of (left index or None, right index or None) pairs, got: a join type's model rows)"""
    lrows, rrows = [row(lt, v) for v in lvals], [row(rt, v) for v in rvals]

    def expect(pairs):
        return [join_row(None if l is None else lrows[l], None if r is None else rrows[r], len(lt), len(rt), kinds(lt),
                       kinds(rt)) for l, r in pairs]

    def got(jt):
        return _model(jt, lrows, rrows, lkeys, rkeys, lt, rt)
    return expect, got


def test_order_with_null_keys_on_both_sides_and_keys_on_one_side_only():
    # left keys: L0 2, L1 null, L2 1, L3 2, L4 5; right keys: R0 2, R1 null, R2 3, R3 2, R4 1
    lvals = [[k, b"l%d" % i, None, i] for i, k in enumerate([2, None, 1, 2, 5])]
    rvals = [[10**19 + i, b"r%d" % i, k] for i, k in enumerate([2, None, 3, 2, 1])]
    expect, got = _order_case(LT, RT, lvals, rvals, keys_of(LT, [0]), keys_of(RT, [2]))
    # runs in key order, nulls first: null (L1 | R1), 1 (L2 | R4), 2 (L0 L3 | R0 R3), 3 (| R2), 5 (L4 |)
    assert got(FULL_OUTER) == expect([(1, None), (None, 1), (2, 4), (0, 0), (0, 3), (3, 0), (3, 3), (None, 2),
                                      (4, None)])
    # Rs order: R1, R4, R0, R3, R2, each with its left matches in Ls order
    assert got(RIGHT_OUTER) == expect([(None, 1), (2, 4), (0, 0), (3, 0), (0, 3), (3, 3), (None, 2)])


def test_order_with_a_two_column_key_one_column_null():
    lt, rt = ["long", "int", "int"], ["int", "long", "int"]
    lvals = [[1, None, 0], [1, 2, 1], [None, 2, 2]]
    rvals = [[None, 1, 0], [2, 1, 1], [2, None, 2], [3, 1, 3]]
    expect, got = _order_case(lt, rt, lvals, rvals, keys_of(lt, [0, 1]), keys_of(rt, [1, 0]))
    # keys in order: (null, 2) L2 R2, (1, null) L0 R0, (1, 2) L1 R1, (1, 3) R3; only (1, 2) matches
    assert got(FULL_OUTER) == expect([(2, None), (None, 2), (0, None), (None, 0), (1, 1), (None, 3)])
    assert got(RIGHT_OUTER) == expect([(None, 2), (None, 0), (1, 1), (None, 3)])


def test_null_left_side_layout():
    """the null left side: every left bit set, zero slots, a wide decimal's 16 zero bytes at offset << 32, and the right
    side's offsets moved by the left var bytes"""
    lt, rt = ["decimal", "string", "decimal"], ["string", "long"]
    r = row(rt, [b"abc", 4])
    out = join_row(None, r, 3, 2, kinds(lt), kinds(rt))
    assert out[:8] == (0b00111).to_bytes(8, "little")
    slots = [int.from_bytes(out[8 + 8 * f:16 + 8 * f], "little") for f in range(5)]
    fixed = 8 * (1 + 5)
    assert slots[:3] == [fixed << 32, 0, (fixed + 16) << 32]
    assert slots[3] == ((fixed + 32) << 32) | 3 and slots[4] == 4
    assert out[fixed:fixed + 32] == bytes(32) and out[fixed + 32:fixed + 35] == b"abc"
