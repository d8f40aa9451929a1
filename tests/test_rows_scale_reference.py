"""The vectorised references and generators of test_gpu_rows_scale.py against the scalar models, on small seeded inputs,
and the comparison's sensitivity: a swapped pair of equal-key rows, one flipped bit of a double sum and one row moved
across a partition must each make it fail.  These run on the CPU and are what lets the large GPU cases trust them."""
import numpy as np
import pytest

import hash_model as hm
import round_robin_model as rr
from join_model import model_join
from rows_model import model_aggregate, model_sort
from test_gpu_rows_scale import (AGGS, COMPOSITE_KEYS, D, IDX, J_REC, JOIN_KEYS, KEY, KEY_INT64, NF, ONE, REC, W_FNS, W_KEYS, W_REC,
                                 WindowRef, aggregate_ref, field, first_diff, hash_ids, is_null, join_index,
                                 joined_rows, keyed_order, make_join, make_keyed_rows, make_rows, partition_perm, round_robin_order, row_hashes,
                                 sequential_sums, sort_order)
from test_gpu_sort_rows_order import model_sort as model_sort_keys
from window_offset_model import model_window_offset

SORT_KEY = [(KEY_INT64, KEY, 8, 0)]


def plain(rec):
    return [rec.tobytes()]


@pytest.fixture(scope="module", params=[(0.5, 0.03, 300), (0.05, 0.2, 40)], ids=["giant_group", "many_nulls"])
def rows(request):
    giant, nulls, domain = request.param
    return make_rows(3000, 11, giant, nulls, domain)


def test_generated_rows(rows):
    assert rows.shape == (3000, REC)
    assert (rows[:, :4] == np.frombuffer((REC - 4).to_bytes(4, "big"), np.uint8)).all()
    assert np.array_equal(field(rows, IDX), np.arange(3000)) and (field(rows, ONE) == 1).all()
    null = is_null(rows)
    assert 0 < null.sum() < 3000 and np.array_equal(field(rows, 0) & ~1, np.zeros(3000, np.int64))
    assert not np.isnan(field(rows, D, "<f8")).any()


def test_sort_order_is_the_model(rows):
    want, n = model_sort(plain(rows), SORT_KEY)
    assert n == 3000 and rows[sort_order(rows)].tobytes() == want


@pytest.mark.parametrize("domain", [40, 1])
def test_composite_key_order_is_the_model(domain):
    """int32 DESC then a string with a 24-byte shared prefix; domain 1: the int ties on nearly every row"""
    rec = make_keyed_rows(4000, 13, nulls=0.05, domain=domain)
    length = field(rec, 16) & 0xFFFFFFFF
    assert length.min() == 25 and length.max() == 32
    want, n = model_sort_keys(plain(rec), COMPOSITE_KEYS)
    assert n == 4000 and rec[keyed_order(rec)].tobytes() == want


@pytest.mark.parametrize("long_group", [4096, 8])
def test_aggregate_is_the_model(rows, long_group):
    """both paths of the double sum: rounds only, and np.add.accumulate for every group longer than 8"""
    want, n, g = model_aggregate(plain(rows), SORT_KEY, AGGS)
    got = aggregate_ref(rows, sort_order(rows), long_group)
    assert got.shape[0] == g and got.tobytes() == want


def test_sequential_sums_are_sequential():
    """values whose sum depends on the order of the additions: pairwise or reassociated sums give other bits"""
    x = np.array([1e16, 1.0, -1e16, 1.0, 3.0, 1e-3, -0.0] * 300)
    starts, lens = np.array([0, 7, 700]), np.array([7, 693, 1400])
    for lg in (4096, 10):
        got = sequential_sums(x, starts, lens, lg)
        for g, (s, n) in enumerate(zip(starts, lens)):
            acc = 0.0
            for v in x[s:s + n]:
                acc = acc + v
            assert got[g].tobytes() == np.float64(acc).tobytes()
    assert sequential_sums(np.array([-0.0]), np.array([0]), np.array([1]))[0].tobytes() == np.float64(0.0).tobytes()


def test_window_is_the_model(rows):
    want, n, m = model_window_offset(plain(rows), W_KEYS, 1, NF, [0] * NF, W_FNS)
    ref = WindowRef(rows, sort_order(rows))
    got = np.concatenate([ref.rows(a, min(a + 700, 3000)) for a in range(0, 3000, 700)])
    assert got.shape == (3000, W_REC) and got.tobytes() == want


@pytest.mark.parametrize("join_type", [0, 1], ids=["inner", "left_outer"])
def test_join_is_the_model(join_type):
    left, right = make_join(5, hot=(40, 60), small_keys=50, unmatched=300, nulls=100)
    want, nl, nr, m = model_join(join_type, plain(left), plain(right), JOIN_KEYS, JOIN_KEYS, 2, 3, [0, 0], [0, 0, 0])
    li, ri = join_index(left, right, outer=join_type == 1)
    assert li.size == m == 40 * 60 + 50 * 6 + join_type * 400
    got = joined_rows(left, right, li, ri)
    assert got.shape[1] == J_REC and got.tobytes() == want


def test_hash_ids_are_the_model(rows):
    rs = [r[4:].tobytes() for r in rows]
    for R in (1, 7, 200):
        assert hash_ids(rows, R).tolist() == hm.ids_scalar(rs, SORT_KEY, R).tolist()


def test_row_hashes_are_the_model(rows):
    assert row_hashes(rows[:500]).tolist() == [rr.row_hash(r[4:].tobytes()) for r in rows[:500]]


def hash_collisions():
    """rows among 200k (differing in their index only) that share a row hash with another, and 300 others"""
    rec = make_rows(200_000, 12)
    h = row_hashes(rec)
    order = np.argsort(h, kind="stable")
    same = np.flatnonzero(h[order][1:] == h[order][:-1])
    pick = np.unique(np.concatenate([order[same], order[same + 1], np.arange(300)]))
    return rec[pick], same.size


def test_round_robin_order_is_the_model():
    rec, ties = hash_collisions()
    assert ties > 0  # the byte comparison of equal hashes runs
    rs = [r[4:].tobytes() for r in rec]
    assert round_robin_order(rec).tolist() == rr.sorted_order(rs, True, 200)


def test_partition_perm_is_the_model(rows):
    R = 13
    ids = hash_ids(rows, R)
    perm, counts = partition_perm(ids, R)
    assert perm.tolist() == [i for p in range(R) for i in range(3000) if ids[i] == p]
    assert counts.tolist() == [int((ids == p).sum()) for p in range(R)]
    start = 5
    order = round_robin_order(rows)
    rr_ids = np.array(rr.ids(3000, start, R), np.uint32)
    perm, _ = partition_perm(rr_ids, R)
    want = rr.sorted_order([r[4:].tobytes() for r in rows], True, R)
    assert order[perm].tolist() == [want[k] for p in range(R) for k in range(3000) if rr_ids[k] == p]


# ---------------------------------------------------------------------------------------------------------------
# sensitivity: the comparison the GPU cases use fails on each planted difference
# ---------------------------------------------------------------------------------------------------------------
def test_swapped_equal_key_rows_fail_the_sort_comparison(rows):
    order = sort_order(rows)
    want = rows[order]
    got = want.copy()
    k = field(got, KEY)
    live = ~is_null(got)
    i = int(np.flatnonzero(live[:-1] & live[1:] & (k[:-1] == k[1:]))[0])
    got[[i, i + 1]] = got[[i + 1, i]]
    assert first_diff(want, want, REC, 0) is None
    bad = first_diff(got, want, REC, 1000)
    assert bad is not None and bad.startswith("record %d " % (1000 + i))


def test_flipped_double_sum_bit_fails_the_aggregate_comparison(rows):
    want = aggregate_ref(rows, sort_order(rows))
    got = want.copy()
    g = int(np.argmax(field(want, ONE)))
    field(got, D)[g] ^= 1  # the last mantissa bit of the largest group's double sum
    bad = first_diff(got, want, REC, 0)
    assert bad is not None and bad.startswith("record %d byte %d " % (g, 4 + D))


def test_moved_row_fails_the_partition_comparison(rows):
    R = 13
    perm, counts = partition_perm(hash_ids(rows, R), R)
    want = rows[perm]
    moved = perm.copy()
    e = int(counts[0])  # the first row of partition 1 moved to the end of partition 0: same counts but one
    moved[e - 1], moved[e] = perm[e], perm[e - 1]
    assert first_diff(rows[moved], want, REC, 0) is not None
    assert first_diff(rows[perm], want, REC, 0) is None
