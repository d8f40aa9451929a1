"""b2s_decompress_join_rows_keys_* as right and full outer joins on the GPU: every output byte equal to the model
(outer_join_model.py), over every codec, checksum and layout of the join tests, hot keys, keys on one side only, failures,
cross-checks against the other join types' GPU output, a hash-partitioned join end to end and the host mirror."""
import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
import test_gpu_join_rows as T
from hash_model import keys_of
from join_model import INNER, LEFT_OUTER
from outer_join_model import FULL_OUTER, RIGHT_OUTER, model_join
from rows_model import blocks_of, build_blocks, mirror, stream
from test_gpu_join_rows import LKEY, LT, RKEY, RT, kinds, row, split, table

pytestmark = pytest.mark.gpu

OUTER = [RIGHT_OUTER, FULL_OUTER]
IDS = ["right_outer", "full_outer"]


def call(capi, jt, left, right, lkeys, rkeys, lt, rt, cap=None, **kw):
    """the join tests' call, its output buffer sized by the model of every join type"""
    if cap is None:
        cap = len(model_join(jt, left, right, lkeys, rkeys, len(lt), len(rt), kinds(lt), kinds(rt))[0])
    return T.call(capi, jt, left, right, lkeys, rkeys, lt, rt, cap=cap, **kw)


def check(capi, jt, left, right, lkeys, rkeys, lt, rt, **kw):
    want, nl, nr, nout = model_join(jt, left, right, lkeys, rkeys, len(lt), len(rt), kinds(lt), kinds(rt))
    got, r = call(capi, jt, left, right, lkeys, rkeys, lt, rt, **kw)
    assert (r["n_left_records"], r["n_right_records"], r["n_out_records"]) == (nl, nr, nout)
    assert (r["status"] == 0).all()
    assert got == want
    return got, r


@pytest.fixture
def shared(monkeypatch):
    """the join tests' bodies, run with this file's check (which passes the field kinds every outer join needs) and the
    model of every join type"""
    monkeypatch.setattr(T, "check", check)
    monkeypatch.setattr(T, "model_join", model_join)
    return T


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
@pytest.mark.parametrize("codec", T.CODECS, ids=[c[0] for c in T.CODECS])
@pytest.mark.parametrize("alg", [0, 3])
def test_codecs_and_checksums_like_the_model(shared, capi, jt, codec, alg):
    """LT has a string and a DECIMAL_WIDE field: the null left side's zero region moves the right side's offsets"""
    shared.test_join_types_codecs_and_checksums_like_the_model(capi, jt, codec, alg)


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_key_layouts_like_the_model(shared, capi, jt):
    shared.test_string_int_key_with_shared_prefixes_refines(capi, jt)
    shared.test_float_zeros_and_nans_decimal_and_boolean_keys(capi, jt)
    shared.test_seventy_fields_cross_a_bitset_word(capi, jt)


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_nullability_differs_between_the_sides(shared, capi, jt):
    rng = np.random.default_rng(17 + jt)
    left = split(rng, table(rng, LT, 300, (0,)), 2)
    right = split(rng, table(rng, RT, 200, (2,), null_rate=0), 2)
    check(capi, jt, left, right, keys_of(LT, [0]), keys_of(RT, [2], nullable=False), LT, RT)
    for kt in ("long", "int"):
        shared.test_not_null_left_key_with_a_nullable_right_key(capi, jt, kt)
    shared.test_twenty_byte_left_key_that_a_nullable_right_column_widens(capi, jt)


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_empty_sides_blocks_and_all_null_keys(shared, capi, jt):
    shared.test_empty_sides_blocks_and_all_null_keys(capi, jt)
    rng = np.random.default_rng(19)
    nulls = [row(LT, [None, b"y", 2, None, 1.0]) for _ in range(50)]
    rnulls = [row(RT, [b"x", 1, None, True]) for _ in range(40)]
    check(capi, jt, [blocks_of(nulls, [50])[0]], [blocks_of(rnulls, [40])[0]], LKEY, RKEY, LT, RT)
    check(capi, jt, [], split(rng, table(rng, RT, 50, (2,)), 2), LKEY, RKEY, LT, RT)


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_keys_on_one_side_only(capi, jt):
    """left keys even, right keys multiples of three: a third of the keys match, the rest have one side null"""
    lt, rt = ["long", "decimal", "string"], ["string", "long", "decimal"]
    left = [row(lt, [2 * (i % 40), i * 10**20, b"l%d" % i]) for i in range(300)]
    right = [row(rt, [b"r%d" % i, 3 * (i % 30), None if i % 7 == 0 else -i]) for i in range(200)]
    check(capi, jt, blocks_of(left, [120, 180]), blocks_of(right, [200]), keys_of(lt, [0]), keys_of(rt, [1]), lt, rt)


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_hot_keys(capi, jt):
    """one right row matched by 1000 left rows (a right outer join's right row drives 1000 rows), and 1000 x 1000"""
    lt, rt = ["long", "long"], ["long", "int"]
    left = [row(lt, [7, i]) for i in range(1000)] + [row(lt, [k, -k]) for k in range(100, 110)]
    right = [row(rt, [7, 1])] + [row(rt, [k, k]) for k in range(105, 120)]
    check(capi, jt, blocks_of(left, [600, 410]), blocks_of(right, [16]), keys_of(lt, [0]), keys_of(rt, [0]), lt, rt)
    right = [row(rt, [7, i]) for i in range(1000)] + right[1:]
    check(capi, jt, blocks_of(left, [600, 410]), blocks_of(right, [1015]), keys_of(lt, [0]), keys_of(rt, [0]), lt, rt)


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_dev_equals_packed(shared, capi, jt):
    shared.test_dev_equals_packed(capi, jt)


# ---------------------------------------------------------------------------------------------------------------
# failures
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jt", OUTER, ids=IDS)
@pytest.mark.parametrize("side", [0, 1])
def test_a_corrupt_or_short_row_fails_its_block(capi, jt, side):
    rng = np.random.default_rng(29)
    left, right = split(rng, table(rng, LT, 100, (0,)), 2), split(rng, table(rng, RT, 100, (2,)), 2)
    blocks = [list(left), list(right)]
    good = blocks[side][1]
    bad_block = len(left) * side + 1
    for tail, words in (((1000).to_bytes(4, "big") + b"\0" * 8, ()),  # runs past the block end
                        ((8).to_bytes(4, "big") + b"\0" * 8, ("fixed region",))):  # shorter than the fixed region
        blocks[side][1] = good + tail
        got, r = call(capi, jt, *blocks, LKEY, RKEY, LT, RT, alg=0, cap=1 << 20)
        assert got == b"" and r["n_out_records"] == r["n_left_records"] == r["n_right_records"] == 0
        assert r["status"][bad_block] == capi.E_CORRUPT
        msg = capi.load().b2s_last_error().decode()
        assert ("block %d" % bad_block) in msg and ("byte %d" % len(good)) in msg
        assert all(w in msg for w in words)


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_checksum_mismatch_sets_bad_slice(capi, jt):
    rng = np.random.default_rng(31)
    left, right = split(rng, table(rng, LT, 100, (0,)), 2), split(rng, table(rng, RT, 100, (2,)), 2)
    arena, off, ln, sb, sl, sc = build_blocks(capi, 1, 0, 3, left + right)
    sc = sc.copy()
    sc[3] ^= 1
    dst = np.zeros(1 << 20, np.uint8)
    r = capi.decompress_join_rows_keys_packed(jt, 1, arena, off, ln, 2, dst, LKEY, RKEY, len(LT), len(RT), kinds(LT),
                                              kinds(RT), 3, sb, sl, sc)
    assert r["status"][3] == capi.E_CHECKSUM and r["bad_slice"][3] == 0
    assert r["n_out_records"] == 0 and r["total"] == 0


@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_dst_too_small_gives_the_bytes_needed(capi, jt):
    rng = np.random.default_rng(37)
    left, right = split(rng, table(rng, LT, 300, (0,)), 2), split(rng, table(rng, RT, 200, (2,)), 2)
    want = model_join(jt, left, right, LKEY, RKEY, len(LT), len(RT), kinds(LT), kinds(RT))[0]
    arena, off, ln, _, _, _ = build_blocks(capi, 1, 0, 0, left + right)
    dst = np.zeros(len(want), np.uint8)
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_join_rows_keys_packed(jt, 1, arena, off, ln, 2, dst[:len(want) - 1], LKEY, RKEY, len(LT),
                                              len(RT), kinds(LT), kinds(RT))
    assert e.value.code == capi.E_DST_TOO_SMALL
    got, r = call(capi, jt, left, right, LKEY, RKEY, LT, RT, alg=0, cap=len(want))
    assert got == want and r["total"] == len(want)


@pytest.mark.parametrize("case", ["no left kinds", "no right kinds", "join type 4", "join type 7"])
@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_bad_arguments(capi, jt, case):
    lk, rk = kinds(LT), kinds(RT)
    if case == "no left kinds":
        lk = None
    elif case == "no right kinds":
        rk = None
    else:
        jt = int(case[-1])
    rng = np.random.default_rng(41)
    left, right = split(rng, table(rng, LT, 20, (0,)), 1), split(rng, table(rng, RT, 20, (2,)), 1)
    arena, off, ln, _, _, _ = build_blocks(capi, 0, 0, 0, left + right)
    dst = np.zeros(1 << 16, np.uint8)
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_join_rows_keys_packed(jt, 0, arena, off, ln, 1, dst, LKEY, RKEY, len(LT), len(RT), lk, rk)
    assert e.value.code == capi.E_ARG


# ---------------------------------------------------------------------------------------------------------------
# cross-checks between GPU calls on the same inputs
# ---------------------------------------------------------------------------------------------------------------
def _null_left(rec, nl):
    """a joined record whose left null bits are all set: the null left side (the left rows here never are all null)"""
    bits = int.from_bytes(rec[4:4 + 8 * ((nl + 63) // 64)], "little")
    return bits & ((1 << nl) - 1) == (1 << nl) - 1


@pytest.mark.parametrize("seed", [0, 1])
def test_outer_joins_agree_with_inner_and_left_outer_on_the_gpu(capi, seed):
    """right outer = inner + the null-left rows (as multisets); full outer without its null-left rows = left outer,
    in order.  Left field 2 is never null, so no left row is all null."""
    rng = np.random.default_rng(71 + seed)
    lrows = []
    for _ in range(600):
        v = [None if rng.random() < 0.2 else int(rng.integers(0, 60)), None if rng.random() < 0.5 else b"s",
             int(rng.integers(-5, 5)), None, None if rng.random() < 0.5 else 2.5]
        lrows.append(row(LT, v))
    left = split(rng, lrows, 3)
    right = split(rng, table(rng, RT, 500, (2,), key_range=80, null_rate=0.2), 3)
    out = {}
    for jt in (INNER, LEFT_OUTER, RIGHT_OUTER, FULL_OUTER):
        got, _ = call(capi, jt, left, right, LKEY, RKEY, LT, RT)
        out[jt] = T._records([got])
    null_left = [x for x in out[FULL_OUTER] if _null_left(x, len(LT))]
    assert null_left and len(null_left) == sum(_null_left(x, len(LT)) for x in out[RIGHT_OUTER])
    assert sorted(out[RIGHT_OUTER]) == sorted(out[INNER] + null_left)
    assert [x for x in out[FULL_OUTER] if not _null_left(x, len(LT))] == out[LEFT_OUTER]


# ---------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jt", OUTER, ids=IDS)
def test_hash_partitioned_tables_join_per_reducer(shared, capi, jt):
    shared.test_hash_partitioned_tables_join_per_reducer(capi, jt)


@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_joins_two_shuffles_per_reducer(capi, tmp_path, codec):
    """two shuffles written by the mirror's serialized writer, each reducer's partitions of both joined in one read;
    a hot key makes the joined rows far larger than the fetched blocks, so the mirror's first size guess (the
    blocks' bytes, four times that when compressed) is too small and it retries with the exact size"""
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R = 3, 2
    rng = np.random.default_rng(67)
    sides = [(LT, LKEY, 300), (RT, RKEY, 200)]
    written = []
    for shuffle, (types, keys, n) in enumerate(sides):
        maps = []
        for m in range(M):
            rows = table(rng, types, n, (keys[0][1] // 8 - 1,), key_range=400)
            rows += [row(LT, [5, b"hot", 1, None, 0.0]) if shuffle == 0 else row(RT, [b"hot", 1, 5, True])] * 40
            ids = rng.integers(0, R, len(rows))
            ids[n:] = 0
            w = host.S3SerializedShuffleWriter(d, shuffle, m, R)
            for r, p in zip(rows, ids):
                w.insertRecord(int(p), len(r).to_bytes(4, "big") + r)
            w.commit()
            w.close()
            maps.append((rows, ids))
        written.append(maps)
    for jt in OUTER:
        for red in range(R):
            plain = [[stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps] for maps in written]
            left = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
            right = host.S3ShuffleReader(d, 1, list(range(M)), red, red + 1)
            got = left.readJoinedRows(right, jt, LKEY, RKEY, len(LT), len(RT), kinds(LT), kinds(RT))
            left.close()
            right.close()
            want = model_join(jt, plain[0], plain[1], LKEY, RKEY, len(LT), len(RT), kinds(LT), kinds(RT))
            assert got == want
            if red == 0:  # 120 x 120 hot rows: more than four times every input byte
                assert len(want[0]) > 4 * sum(len(b) for side in plain for b in side)
    d.close()
