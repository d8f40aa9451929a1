"""Null-safe (<=>) join keys and the existence join of b2s_decompress_join_rows_keys_* on the GPU, and null-safe keys
in the hash call: every output byte for byte equal to null_safe_join_model.py, over every join type and key type, the
failures the join reports, INTERSECT and EXCEPT end to end through hash-partitioned maps, and the host mirror."""
import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from hash_model import keys_of, pmod, records_of
from null_safe_join_model import ALL_JOINS, EXISTENCE, NULL_SAFE, model_join, row_hash
from join_model import LEFT_ANTI, LEFT_SEMI, col_value, side_records
from rows_model import blocks_of, build_blocks, mirror, stream
from test_gpu_join_rows import _records, call, kinds, row, split

pytestmark = pytest.mark.gpu

CODECS = [("none", 0, 0), ("lz4", 1, 0), ("snappy", 2, 0), ("zstd", 3, 1)]
NAN = ("bits", 0x7FF8000000000000)
# each type's values around its default, so that nulls sort and match next to them
DOMAIN = {"long": [0, 1, -1], "int": [0, 2, -3], "short": [0, 1], "byte": [0, -1], "bool": [False, True],
          "string": [b"", b"a", b"\x00", b"ab"], "decimal": [0, 10**30, -1], "double": [0.0, -0.0, NAN, 1.5],
          "float": [0.0, -0.0, 2.5]}
TYPES = ["long", "int", "short", "byte", "bool", "string", "decimal", "double", "float"]


def ns(keys, which=None):
    return [(t | NULL_SAFE, o, ln, nf) if which is None or c in which else (t, o, ln, nf)
            for c, (t, o, ln, nf) in enumerate(keys)]


def gen(rng, types, n, null_rate=0.2, no_null=(), hot=None):
    out = []
    for _ in range(n):
        vals = []
        for f, t in enumerate(types):
            d = DOMAIN[t] if hot is None else DOMAIN[t][:1]
            vals.append(None if f not in no_null and rng.random() < null_rate else d[int(rng.integers(len(d)))])
        out.append(row(types, vals))
    return out


def check(capi, jt, left, right, lk, rk, lt, rt, **kw):
    want, nl, nr, nout = model_join(jt, left, right, lk, rk, len(lt), len(rt), kinds(lt), kinds(rt))
    whole = jt in (LEFT_SEMI, LEFT_ANTI)
    got, r = call(capi, jt, left, right, lk, rk, lt, rt, cap=len(want), kinds_=not whole, **kw)
    assert (r["n_left_records"], r["n_right_records"], r["n_out_records"]) == (nl, nr, nout)
    assert (r["status"] == 0).all()
    assert got == want
    return got, r


@pytest.mark.parametrize("jt", ALL_JOINS)
@pytest.mark.parametrize("t", TYPES)
def test_every_join_type_over_every_key_type(capi, jt, t):
    rng = np.random.default_rng(jt * 100 + TYPES.index(t))
    lt, rt = [t, "string", "long"], ["decimal", t]
    left, right = split(rng, gen(rng, lt, 300), 3), split(rng, gen(rng, rt, 200), 2)
    check(capi, jt, left, right, ns(keys_of(lt, [0])), ns(keys_of(rt, [1])), lt, rt)


@pytest.mark.parametrize("jt", ALL_JOINS)
def test_mixed_plain_and_null_safe_columns_and_one_sided_nullability(capi, jt):
    rng = np.random.default_rng(7 + jt)
    lt, rt = ["int", "string", "double", "decimal"], ["string", "decimal", "int", "double"]
    left, right = split(rng, gen(rng, lt, 400), 3), split(rng, gen(rng, rt, 300, no_null=(0, 3)), 2)
    lk, rk = keys_of(lt, [0, 1, 2, 3]), keys_of(rt, [2, 0, 3, 1])
    rk = [rk[0], (rk[1][0], rk[1][1], rk[1][2], -1), (rk[2][0], rk[2][1], rk[2][2], -1), rk[3]]  # never null there
    for which in ((0, 1, 2, 3), (0, 2), (1, 3), (1,)):
        check(capi, jt, left, right, ns(lk, which), ns(rk, which), lt, rt)


@pytest.mark.parametrize("jt", ALL_JOINS)
def test_all_null_keys(capi, jt):
    rng = np.random.default_rng(3)
    lt, rt = ["long", "string"], ["string", "long"]
    left, right = split(rng, gen(rng, lt, 50, null_rate=1.0), 2), split(rng, gen(rng, rt, 40, null_rate=1.0), 2)
    check(capi, jt, left, right, ns(keys_of(lt, [0, 1])), ns(keys_of(rt, [1, 0])), lt, rt)
    check(capi, jt, left, right, ns(keys_of(lt, [0, 1]), (0,)), ns(keys_of(rt, [1, 0]), (0,)), lt, rt)


@pytest.mark.parametrize("jt", ALL_JOINS)
def test_long_string_keys_refine(capi, jt):
    rng = np.random.default_rng(11 + jt)
    prefix = b"q" * 41
    lt, rt = ["string", "int", "long"], ["long", "string", "int"]

    def t(types, fs, fi, n):
        out = []
        for _ in range(n):
            vals = [DOMAIN[x][0] for x in types]
            vals[fs] = None if rng.random() < 0.2 else prefix + bytes([97 + int(rng.integers(2))])
            vals[fi] = None if rng.random() < 0.2 else int(rng.integers(2))
            out.append(row(types, vals))
        return out
    check(capi, jt, split(rng, t(lt, 0, 1, 300), 2), split(rng, t(rt, 1, 2, 200), 2),
          ns(keys_of(lt, [0, 1])), ns(keys_of(rt, [1, 2])), lt, rt)


@pytest.mark.parametrize("jt", [LEFT_SEMI, 6, EXISTENCE])
@pytest.mark.parametrize("codec", CODECS, ids=[c[0] for c in CODECS])
@pytest.mark.parametrize("alg", [0, 1, 2, 3])
def test_codecs_and_checksums(capi, jt, codec, alg):
    rng = np.random.default_rng(jt * 10 + codec[1] + alg)
    lt, rt = ["long", "string", "decimal"], ["string", "long"]
    left, right = split(rng, gen(rng, lt, 300), 3), split(rng, gen(rng, rt, 200), 2)
    check(capi, jt, left, right, ns(keys_of(lt, [0, 1])), ns(keys_of(rt, [1, 0])), lt, rt, codec=codec, alg=alg)


@pytest.mark.parametrize("jt", ALL_JOINS)
def test_dev_equals_packed(capi, jt):
    rng = np.random.default_rng(17 + jt)
    lt, rt = ["string", "long", "decimal"], ["long", "string"]
    left, right = split(rng, gen(rng, lt, 300), 2), split(rng, gen(rng, rt, 200), 2)
    lk, rk = ns(keys_of(lt, [1, 0])), ns(keys_of(rt, [0, 1]))
    a, _ = check(capi, jt, left, right, lk, rk, lt, rt)
    b, _ = check(capi, jt, left, right, lk, rk, lt, rt, dev=True)
    assert a == b


@pytest.mark.parametrize("jt", ALL_JOINS)
def test_hot_keys(capi, jt):
    rng = np.random.default_rng(19)
    lt, rt = ["long", "int"], ["int", "long"]
    left, right = split(rng, gen(rng, lt, 600, hot=True), 3), split(rng, gen(rng, rt, 300, hot=True), 2)
    check(capi, jt, left, right, ns(keys_of(lt, [0])), ns(keys_of(rt, [1])), lt, rt)


@pytest.mark.parametrize("nl", [62, 63, 64, 65])
def test_existence_rows_where_the_null_bitset_grows(capi, nl):
    rng = np.random.default_rng(nl)
    lt = ["string", "decimal"] + ["long"] * (nl - 2)
    rt = ["long", "string"]
    left, right = split(rng, gen(rng, lt, 200), 2), split(rng, gen(rng, rt, 60), 2)
    lk, rk = ns(keys_of(lt, [2, 0])), ns(keys_of(rt, [0, 1]))
    want, _ = check(capi, EXISTENCE, left, right, lk, rk, lt, rt)
    arena, off, ln, _, _, _ = build_blocks(capi, 1, 0, 0, left + right)
    dst = np.zeros(len(want), np.uint8)
    r = capi.decompress_join_rows_keys_packed(EXISTENCE, 1, arena, off, ln, len(left), dst, lk, rk, len(lt), len(rt),
                                              kinds(lt), None)  # the right side's kinds are not needed
    assert r["n_out_records"] == r["n_left_records"] == 200 and dst.tobytes() == want


def _bad(capi, jt, left, right, lk, rk, lt, rt):
    arena, off, ln, sb, sl, sc = build_blocks(capi, 1, 0, 0, list(left) + list(right))
    dst = np.zeros(1 << 20, np.uint8)
    r = capi.decompress_join_rows_keys_packed(jt, 1, arena, off, ln, len(left), dst, lk, rk, len(lt), len(rt),
                                              kinds(lt), kinds(rt))
    assert r["n_out_records"] == 0 and r["total"] == 0
    return r


@pytest.mark.parametrize("jt", [LEFT_ANTI, EXISTENCE])
@pytest.mark.parametrize("side", [0, 1])
def test_a_corrupt_or_short_row_fails_its_block(capi, jt, side):
    rng = np.random.default_rng(29)
    lt, rt = ["long", "string"], ["string", "long"]
    left, right = split(rng, gen(rng, lt, 100), 2), split(rng, gen(rng, rt, 100), 2)
    lk, rk = ns(keys_of(lt, [0, 1])), ns(keys_of(rt, [1, 0]))
    blocks = [list(left), list(right)]
    good = blocks[side][1]
    bad_block = len(left) * side + 1
    for tail in ((1000).to_bytes(4, "big") + b"\0" * 8, (8).to_bytes(4, "big") + b"\0" * 8):
        blocks[side][1] = good + tail
        r = _bad(capi, jt, *blocks, lk, rk, lt, rt)
        assert r["status"][bad_block] == capi.E_CORRUPT
        msg = capi.load().b2s_last_error().decode()
        assert ("block %d" % bad_block) in msg and ("byte %d" % len(good)) in msg


@pytest.mark.parametrize("jt", [EXISTENCE, 0])
def test_dst_too_small_gives_the_bytes_needed(capi, jt):
    rng = np.random.default_rng(37)
    lt, rt = ["long", "string"], ["string", "long"]
    left, right = split(rng, gen(rng, lt, 300), 2), split(rng, gen(rng, rt, 200), 2)
    lk, rk = ns(keys_of(lt, [0])), ns(keys_of(rt, [1]))
    want = model_join(jt, left, right, lk, rk, 2, 2, kinds(lt), kinds(rt))[0]
    arena, off, ln, _, _, _ = build_blocks(capi, 1, 0, 0, left + right)
    dst = np.zeros(len(want), np.uint8)
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_join_rows_keys_packed(jt, 1, arena, off, ln, 2, dst[:len(want) - 1], lk, rk, 2, 2, kinds(lt),
                                              kinds(rt))
    assert e.value.code == capi.E_DST_TOO_SMALL
    r = capi.decompress_join_rows_keys_packed(jt, 1, arena, off, ln, 2, dst, lk, rk, 2, 2, kinds(lt), kinds(rt))
    assert r["total"] == len(want) and dst.tobytes() == want


@pytest.mark.parametrize("case", ["no left kinds", "type 7", "type 4", "order flag", "unknown flag"])
def test_bad_arguments(capi, case):
    rng = np.random.default_rng(41)
    lt, rt = ["long", "string"], ["string", "long"]
    left, right = split(rng, gen(rng, lt, 20), 1), split(rng, gen(rng, rt, 20), 1)
    lk, rk = ns(keys_of(lt, [0])), ns(keys_of(rt, [1]))
    jt, lkinds = EXISTENCE, kinds(lt)
    if case == "no left kinds":
        lkinds = None
    elif case in ("type 7", "type 4"):
        jt = int(case[-1])
    else:
        flag = capi.KEY_DESCENDING if case == "order flag" else 1 << 11
        lk = [(lk[0][0] | flag,) + lk[0][1:]]
    arena, off, ln, _, _, _ = build_blocks(capi, 1, 0, 0, left + right)
    with pytest.raises(capi.B2SError) as e:
        capi.decompress_join_rows_keys_packed(jt, 1, arena, off, ln, 1, np.zeros(1 << 16, np.uint8), lk, rk, 2, 2,
                                              lkinds, None)
    assert e.value.code == capi.E_ARG


def test_the_other_reduce_calls_refuse_the_flag(capi):
    rng = np.random.default_rng(43)
    lt = ["long", "string"]
    arena, off, ln, _, _, _ = build_blocks(capi, 1, 0, 0, split(rng, gen(rng, lt, 20), 1))
    keys = ns(keys_of(lt, [0]))
    dst = np.zeros(1 << 16, np.uint8)
    for f in (lambda: capi.decompress_sort_rows_keys_packed(1, arena, off, ln, dst, keys),
              lambda: capi.decompress_aggregate_rows_keys_packed(1, arena, off, ln, dst, keys),
              lambda: capi.decompress_window_rows_keys_packed(1, arena, off, ln, dst, keys_of(lt, [1]) + keys, 1, 2,
                                                              kinds(lt), [capi.WINDOW_ROW_NUMBER])):
        with pytest.raises(capi.B2SError) as e:
            f()
        assert e.value.code == capi.E_ARG


# ---------------------------------------------------------------------------------------------------------------
# end to end: INTERSECT and EXCEPT through hash-partitioned maps
# ---------------------------------------------------------------------------------------------------------------
def _values(rows, keys):
    return {tuple(col_value(r, (t & 0xFF, o, ln, nf))[1] for t, o, ln, nf in keys) for r in rows}


@pytest.mark.parametrize("jt", [LEFT_SEMI, LEFT_ANTI])
def test_intersect_and_except_through_hash_partitioned_maps(capi, jt):
    """both tables hash-partitioned on every column null-safe, each reducer joined: distinct of the union is Python's
    set intersection (INTERSECT) or difference (EXCEPT) of the tables' tuples"""
    rng = np.random.default_rng(61 + jt)
    types = ["string", "long", "decimal", "double"]
    keys = ns(keys_of(types, [0, 1, 2, 3]))
    R, maps = 5, 3
    side_rows = [gen(rng, types, 700, null_rate=0.3), gen(rng, types, 500, null_rate=0.3)]
    per_reducer = [[[] for _ in range(R)], [[] for _ in range(R)]]
    for s in range(2):
        for m in range(maps):
            rows = side_rows[s][m::maps]
            records, rec_len = records_of(rows)
            dst = np.zeros(2 * records.size + 4096 * R, np.uint8)
            r = capi.partition_compress_rows_hash_packed(1, records, rec_len, keys, R, dst, checksum_alg=3)
            ids = [pmod(row_hash(x, keys), R) for x in rows]
            for p in range(R):
                o, n = int(r["dst_off"][p]), int(r["dst_len"][p])
                plain = capi.decompress_batch(1, [dst[o:o + n].tobytes()])[0][0] if n else b""
                assert plain == stream([x for x, i in zip(rows, ids) if i == p])  # the model's partition ids
                if n:
                    per_reducer[s][p].append((dst[o:o + n].tobytes(), int(r["checksums"][p])))
    got = []
    for p in range(R):
        blocks = per_reducer[0][p] + per_reducer[1][p]
        data = [b for b, _ in blocks]
        if not data:
            continue
        lens = np.array([len(b) for b in data], np.uint64)
        off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        arena = np.frombuffer(b"".join(data), np.uint8)
        dst = np.zeros(1 << 22, np.uint8)
        r = capi.decompress_join_rows_keys_packed(jt, 1, arena, off, lens, len(per_reducer[0][p]), dst, keys, keys,
                                                  len(types), len(types), None, None, 3,
                                                  np.arange(len(data) + 1, dtype=np.uint32), lens,
                                                  np.array([c for _, c in blocks], np.uint64))
        assert (r["status"] == 0).all()
        got += [x[4:] for x in _records([dst[:r["total"]].tobytes()])]
    lv, rv = _values(side_rows[0], keys), _values(side_rows[1], keys)
    assert _values(got, keys) == (lv & rv if jt == LEFT_SEMI else lv - rv)
    want = model_join(jt, blocks_of(side_rows[0], [700]), blocks_of(side_rows[1], [500]), keys, keys, 4, 4)[0]
    assert sorted(got) == sorted(side_records([want]))


def test_host_mirror_hash_writes_and_joined_reads(capi, tmp_path):
    """two shuffles hash-partitioned by the mirror's writer on null-safe keys, each reducer's partitions joined (every
    type, existence included) in one read"""
    host = pkg.host
    d = mirror(tmp_path, "lz4")
    M, R = 2, 3
    rng = np.random.default_rng(67)
    lt, rt = ["long", "string", "decimal"], ["string", "long"]
    lk, rk = ns(keys_of(lt, [0, 1])), ns(keys_of(rt, [1, 0]))
    written = []
    for shuffle, (types, keys, n) in enumerate(((lt, lk, 300), (rt, rk, 200))):
        maps = []
        for m in range(M):
            rows = gen(rng, types, n)
            w = host.S3SerializedShuffleWriter(d, shuffle, m, R)
            w.hashRows(keys)
            for x in rows:
                w.insertRecord(0, len(x).to_bytes(4, "big") + x)
            w.commit()
            w.close()
            maps.append((rows, [pmod(row_hash(x, keys), R) for x in rows]))
        written.append(maps)
    for jt in ALL_JOINS:
        for red in range(R):
            plain = [[stream([x for x, p in zip(rows, ids) if p == red]) for rows, ids in maps] for maps in written]
            left = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
            right = host.S3ShuffleReader(d, 1, list(range(M)), red, red + 1)
            got = left.readJoinedRows(right, jt, lk, rk, len(lt), len(rt), kinds(lt), kinds(rt))
            left.close()
            right.close()
            assert got == model_join(jt, plain[0], plain[1], lk, rk, len(lt), len(rt), kinds(lt), kinds(rt))
