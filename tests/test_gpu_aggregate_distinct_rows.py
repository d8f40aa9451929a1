"""One DISTINCT group's middle stage on the GPU: b2s_decompress_aggregate_distinct_partition_compress_rows_hash_* is
byte for byte b2s_partition_compress_rows_hash_packed over the model's output rows (tests/distinct_agg_model.py), or
b2s_partition_compress_packed with one partition without grouping columns.  End to end, maps by G ++ X, this call per
reducer and the final merge by G equal numpy's distinct counts and sums."""
import threading

import numpy as np
import pytest

import distinct_agg_model as da
import hash_model as hm
import moments_model as mm
import partial_agg_model as pm
import rows_model as rm
import spark_s3_shuffle_b200 as pkg
import test_distinct_agg_model as tm

pytestmark = pytest.mark.gpu

SUM, COUNT, AVG, MIN, MAX, VAR = pm.SUM, pm.COUNT, pm.AVG, pm.MIN, pm.MAX, mm.VARIANCE
ALL = da.ALL
DEC12, DEC25 = pm.val_decimal(12, 2), pm.val_decimal(25, 3)
# the map side's value columns: long, double, decimal(12, 2) as a long, decimal(25, 3), int
VALUE_TYPES = ["long", "double", "long", "decimal", "int"]


@pytest.fixture(scope="module")
def capi():
    c = pkg.capi
    c.init(1)
    return c


def value(rng, t):
    if rng.random() < 0.15:
        return None
    if t == "long":
        return int(rng.integers(-10**9, 10**9))
    if t == "int":
        return int(rng.integers(-1000, 1000))
    if t == "double":
        return float(rng.normal() * 1e3) if rng.random() < 0.9 else [-0.0, float("nan"), 0.0][int(rng.integers(3))]
    return int(rng.integers(-10**18, 10**18)) * 10**4


def key_value(rng, pool):
    return pool[int(rng.integers(len(pool)))]


def make_maps(rng, M, n, g_types, g_pool, x_types, x_pool):
    """M maps of n rows [G..., X..., values...] -> (maps, types)"""
    types = g_types + x_types + VALUE_TYPES
    maps = []
    for _ in range(M):
        rows = []
        for _ in range(n):
            g = [key_value(rng, p) for p in g_pool]
            x = [key_value(rng, p) for p in x_pool]
            rows.append(hm.make_row(types, g + x + [value(rng, t) for t in VALUE_TYPES]))
        maps.append(rows)
    return maps, types


def map_side(maps, types, nk, f):
    """the model's map-side partial rows (keys G ++ X, functions f over the value columns) of each map"""
    keys = hm.keys_of(types, list(range(nk)))
    aggs = [(fn, vt, hm.keys_of(types, [nk + j])[0][1], nk + j) if vt != pm.VAL_NONE else (fn, vt, 0, -1)
            for fn, vt, j in f]
    return [mm.partial_rows(rows, keys, aggs) for rows in maps]


def call_keys(types, nk):
    return [(k[0], k[2]) for k in hm.keys_of(types, list(range(nk)))]


def check(capi, partial_maps, ng, keys, aggs, distinct, R, codec=1, alg=3, dev=False):
    """the call over the maps' blocks == the partition call over the model's rows -> (result, model rows)"""
    streams = [rm.stream(p) for p in partial_maps]
    want, counts = da.reducer(streams, ng, keys, aggs, distinct)
    arena, off, ln, sb, sl, ck = rm.build_blocks(capi, codec, 1, alg, streams)
    prec, prl = hm.records_of(want)
    cap = capi.partition_compress_bound(codec, 0, R, prec.size) + 64
    ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    if ng:
        ref = capi.partition_compress_rows_hash_packed(codec, prec, prl, da.input_keys(keys)[:ng], R, ref_dst,
                                                       checksum_alg=alg)
    else:
        ref = capi.partition_compress_packed(codec, prec, prl, np.zeros(prl.size, np.uint32), 1, ref_dst,
                                             checksum_alg=alg)
    kw = dict(checksum_alg=alg, slice_base=sb, slice_len=sl, slice_checksum=ck)
    if dev:
        d_src, d_dst = capi.dev_alloc(max(arena.size, 1)), capi.dev_alloc(cap)
        try:
            capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
            got = capi.aggregate_distinct_partition_compress_rows_hash(codec, d_src, off, ln, d_dst, ng, keys, aggs,
                                                                       distinct, R, dev=0, dst_cap=cap, **kw)
            capi.dev_memcpy(got_dst.ctypes.data, d_dst, got["total"], 2)
        finally:
            capi.dev_free(d_src)
            capi.dev_free(d_dst)
    else:
        got = capi.aggregate_distinct_partition_compress_rows_hash(codec, arena, off, ln, got_dst, ng, keys, aggs,
                                                                   distinct, R, **kw)
    assert got["counts"] == counts
    assert got["total"] == ref["total"]
    for k, r in (("dst_off", "dst_off"), ("dst_len", "dst_len"), ("checksums", "checksums"), ("part_status", "status")):
        assert np.array_equal(got[k], ref[r]), k
    assert np.array_equal(got_dst[:ref["total"]], ref_dst[:ref["total"]])
    assert (got["status"] == 0).all()
    return got, want


@pytest.mark.parametrize("codec", [0, 1, 2, 3])
@pytest.mark.parametrize("alg", [0, 1, 2, 3])
def test_every_codec_and_checksum(capi, codec, alg):
    rng = np.random.default_rng(10 * codec + alg)
    maps, types = make_maps(rng, 3, 600, ["long"], [list(range(40)) + [None]], ["int"],
                            [list(range(-30, 30)) + [None]])
    f = [(SUM, DEC12, 2), (COUNT, pm.VAL_NONE, 0), (AVG, pm.VAL_FLOAT64, 1)]
    pmaps = map_side(maps, types, 2, f)
    check(capi, pmaps, 1, call_keys(types, 2), [(a, b) for a, b, _ in f],
          [(COUNT, pm.VAL_INT32, 1), (SUM, pm.VAL_INT32, 1)], 5, codec=codec, alg=alg, dev=(codec + alg) % 2 == 1)


# every buffer kind of F, in two calls (at most 16 buffers in the output); X is one long column
F1 = [(SUM, pm.VAL_INT64, 0), (SUM, pm.VAL_FLOAT64, 1), (SUM, DEC12, 2), (SUM, DEC25, 3), (COUNT, pm.VAL_NONE, 0),
      (AVG, pm.VAL_FLOAT64, 1), (AVG, DEC12, 2)]
D1 = [(COUNT, pm.VAL_INT64, 1), (SUM, pm.VAL_INT64, 1), (AVG, pm.VAL_INT64, 1)]
F2 = [(COUNT, pm.VAL_INT64, 0), (MIN, pm.VAL_INT32, 4), (MAX, pm.VAL_FLOAT64, 1), (MAX, DEC25, 3),
      (VAR, pm.VAL_INT64, 0)]
D2 = [(VAR, pm.VAL_INT64, 1), (COUNT, pm.VAL_NONE, ALL), (COUNT, pm.VAL_INT64, 1), (SUM, pm.VAL_INT64, 1)]


@pytest.mark.parametrize("g", ["int", "long", "string", "decimal", "double"])
def test_grouping_column_types_and_every_buffer(capi, g):
    """G of every hashed kind with nulls (NaN and -0.0 for double), X a long with nulls"""
    rng = np.random.default_rng(["int", "long", "string", "decimal", "double"].index(g))
    pools = {"int": list(range(-20, 20)), "long": [10**12 + k for k in range(30)],
             "string": [b"", b"a", b"apple", b"banana" * 5] + [b"k%03d" % k for k in range(20)],
             "decimal": [k * 10**20 - 7 for k in range(-10, 10)],
             "double": [0.0, -0.0, float("nan"), ("bits", 0x7FF8000000000123), 1.5, -2.25, float("inf")]}
    maps, types = make_maps(rng, 4, 700, [g], [pools[g] + [None]], ["long"], [list(range(25)) + [None]])
    for f, d in ((F1, D1), (F2, D2)):
        check(capi, map_side(maps, types, 2, f), 1, call_keys(types, 2), [(a, b) for a, b, _ in f], d, 7)


@pytest.mark.parametrize("x,pool,distinct", [
    ("decimal", [k * 10**19 + 3 for k in range(-6, 6)], [(SUM, DEC25, 1), (AVG, DEC25, 1), (COUNT, pm.VAL_NONE, ALL)]),
    ("double", [0.0, -0.0, float("nan"), 2.5], [(COUNT, pm.VAL_FLOAT64, 1), (SUM, pm.VAL_FLOAT64, 1),
                                                (VAR, pm.VAL_FLOAT64, 1)]),
    ("float", [0.5, -0.0, 0.0, ("bits", 0x7FC00000)], [(AVG, pm.VAL_FLOAT32, 1), (COUNT, pm.VAL_FLOAT32, 1)]),
    ("string", [b"", b"x", b"yy" * 9], [(COUNT, pm.VAL_BYTES, 1), (COUNT, pm.VAL_NONE, ALL)]),
    ("bool", [True, False], [(COUNT, pm.VAL_BYTES, 1)])])
def test_distinct_column_types(capi, x, pool, distinct):
    """D over a decimal, double (NaN, -0.0), float, string or boolean X with nulls"""
    rng = np.random.default_rng(len(x))
    maps, types = make_maps(rng, 3, 800, ["int"], [list(range(12))], [x], [pool + [None]])
    pmaps = map_side(maps, types, 2, [(COUNT, pm.VAL_NONE, 0), (VAR, pm.VAL_FLOAT64, 1)])
    check(capi, pmaps, 1, call_keys(types, 2), [(COUNT, pm.VAL_NONE), (VAR, pm.VAL_FLOAT64)], distinct, 3)


def test_count_distinct_of_several_columns(capi):
    """X = (long, string, int): count(DISTINCT a, b, c), the rows with no X null, beside F"""
    rng = np.random.default_rng(4)
    maps, types = make_maps(rng, 3, 900, ["int"], [list(range(10))], ["long", "string", "int"],
                            [list(range(6)) + [None], [b"p", b"q", None], [1, 2, None]])
    pmaps = map_side(maps, types, 4, [(SUM, pm.VAL_INT64, 0), (COUNT, pm.VAL_NONE, 0)])
    check(capi, pmaps, 1, call_keys(types, 4), [(SUM, pm.VAL_INT64), (COUNT, pm.VAL_NONE)],
          [(COUNT, pm.VAL_NONE, ALL)], 4)


def test_decimal_sum_overflow_in_one_group(capi):
    """partial rows [G, X, sum decimal(38), isEmpty]: (1, 1)'s two sums pass 10^38 when merged, so its G group's sum is
    null; G 3 holds an input that had overflowed on its map (null, not empty); G 2 is exact"""
    big = 9 * 10**37
    maps = [tm.dec_partial_rows(rows) for rows in (
        [[1, 1, big, False], [1, 2, 5, False], [2, 1, 7, False], [3, 2, 4, False]],
        [[1, 1, big, False], [2, 2, 3, False], [2, 3, 0, True]],
        [[3, 1, None, False], [3, 3, 1, False]])]
    keys = call_keys(["int", "int"], 2)
    _, want = check(capi, maps, 1, keys, [(SUM, pm.val_decimal(28, 0))], [(COUNT, pm.VAL_INT32, 1)], 2)
    nulls = [int.from_bytes(r[0:8], "little") for r in want]
    assert [bool(v & 2) for v in nulls] == [True, False, True]  # field 1: the sum


def test_group_sizes_across_every_fold(capi):
    """G groups of 1 to more than 2049 (G, X) rows: the thread, warp, chunk and chain folds"""
    rng = np.random.default_rng(5)
    types = ["long", "long"] + VALUE_TYPES
    rows = []
    for g, size in enumerate([1, 2, 31, 32, 33, 100, 2047, 2048, 2049, 5000]):
        for x in range(size):
            rows.append(hm.make_row(types, [g, x] + [value(rng, t) for t in VALUE_TYPES]))
    rng.shuffle(rows)
    maps = [rows[k::3] for k in range(3)]
    f = [(SUM, pm.VAL_FLOAT64, 1), (SUM, DEC25, 3), (AVG, DEC12, 2), (VAR, pm.VAL_INT64, 0), (MIN, DEC25, 3)]
    pmaps = map_side(maps, types, 2, f)
    check(capi, pmaps, 1, call_keys(types, 2), [(a, b) for a, b, _ in f],
          [(COUNT, pm.VAL_INT64, 1), (SUM, pm.VAL_INT64, 1), (AVG, pm.VAL_INT64, 1), (VAR, pm.VAL_INT64, 1)], 4)


def test_one_group_of_a_million_rows(capi):
    """q16's shape: a global count(DISTINCT order) beside two decimal sums over one G group of 2^20 (G, X) rows: the
    maps' partial rows [order, sum, isEmpty, sum, isEmpty] are written directly (each order once per map)"""
    n = 1 << 20
    rng = np.random.default_rng(6)
    order = rng.permutation(n)
    types = ["long", "long", "bool", "long", "bool"]
    maps = [[hm.make_row(types, [int(o), int(o % 1000), False, int(o % 97) - 48, False]) for o in order[m::4]]
            for m in range(4)]
    dec7 = pm.val_decimal(7, 2)
    got, want = check(capi, maps, 0, [(hm.FIELD["long"][0], 8)], [(SUM, dec7), (SUM, dec7)],
                      [(COUNT, pm.VAL_INT64, 0)], 1)
    assert got["counts"] == [n, n, 1]
    assert int.from_bytes(want[0][40:48], "little") == n  # the distinct count, after [sum, isEmpty] * 2


def test_empty_reducer(capi):
    """no blocks: one initial row without G; nothing in any partition with G"""
    for ng, R in ((0, 1), (1, 4)):
        keys = [(hm.FIELD["long"][0], 8)] * (ng + 1)
        aggs = [(SUM, pm.VAL_INT64), (SUM, DEC12), (COUNT, pm.VAL_NONE), (AVG, pm.VAL_FLOAT64), (AVG, DEC25),
                (MIN, pm.VAL_INT64), (VAR, pm.VAL_INT32)]
        got, want = check(capi, [], ng, keys, aggs, [(COUNT, pm.VAL_INT64, ng), (SUM, pm.VAL_INT64, ng)], R)
        assert len(want) == (0 if ng else 1)
        # blocks that hold no rows give the same
        check(capi, [[], []], ng, keys, aggs, [(COUNT, pm.VAL_INT64, ng)], R, codec=0)


def test_corrupt_block_and_short_destination(capi):
    rng = np.random.default_rng(8)
    maps, types = make_maps(rng, 3, 300, ["long"], [list(range(20))], ["int"], [list(range(50))])
    pmaps = map_side(maps, types, 2, [(COUNT, pm.VAL_NONE, 0)])
    keys = call_keys(types, 2)
    streams = [rm.stream(p) for p in pmaps]
    arena, off, ln, sb, sl, ck = rm.build_blocks(capi, 1, 1, 3, streams)
    bad = ck.copy()
    bad[1] ^= 1
    dst = np.full(1 << 16, 7, np.uint8)
    r = capi.aggregate_distinct_partition_compress_rows_hash(1, arena, off, ln, dst, 1, keys, [(COUNT, pm.VAL_NONE)],
                                                             [(COUNT, pm.VAL_INT32, 1)], 3, checksum_alg=3,
                                                             slice_base=sb, slice_len=sl, slice_checksum=bad)
    assert r["total"] == 0 and r["status"][1] != 0 and (r["status"][[0, 2]] == 0).all()
    assert (r["dst_len"] == 0).all() and r["counts"] == [0, 0, 0] and (dst == 7).all()
    full = capi.aggregate_distinct_partition_compress_rows_hash(1, arena, off, ln, dst, 1, keys, [(COUNT, pm.VAL_NONE)],
                                                                [(COUNT, pm.VAL_INT32, 1)], 3)
    with pytest.raises(capi.B2SError) as e:
        capi.aggregate_distinct_partition_compress_rows_hash(1, arena, off, ln, np.zeros(full["total"] - 1, np.uint8), 1,
                                                             keys, [(COUNT, pm.VAL_NONE)], [(COUNT, pm.VAL_INT32, 1)], 3)
    assert e.value.code == capi.E_DST_TOO_SMALL
    assert full["total"] > 0


def test_end_to_end_equals_numpy(capi):
    """maps by G ++ X on the GPU, this call per reducer, the final merge by G: count(DISTINCT x) and sum(DISTINCT x)
    per g, and sum(v) beside them, equal numpy's"""
    rng = np.random.default_rng(12)
    types = ["int", "int", "long"]
    M, R1, R2 = 4, 3, 2
    data = []
    maps = []
    for m in range(M):
        rows = []
        for _ in range(4000):
            g, x, v = int(rng.integers(0, 25)), int(rng.integers(0, 300)), int(rng.integers(-10**6, 10**6))
            x = None if rng.random() < 0.05 else x
            data.append((g, x, v))
            rows.append(hm.make_row(types, [g, x, v]))
        maps.append(rows)
    keys_in = hm.keys_of(types, [0, 1])
    f = [(SUM, pm.VAL_INT64, keys_in[1][1] + 8, 2)]
    outs = []
    for rows in maps:
        recs, rl = hm.records_of(rows)
        dst = np.zeros(capi.partition_compress_bound(1, 0, R1, recs.size) + 64, np.uint8)
        outs.append((dst, capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys_in, f, R1, dst)))
    keys = call_keys(types, 2)
    distinct = [(COUNT, pm.VAL_INT32, 1), (SUM, pm.VAL_INT32, 1)]
    stage3_out = []
    for p in range(R1):
        blocks = [d[int(g["dst_off"][p]):int(g["dst_off"][p] + g["dst_len"][p])].tobytes() for d, g in outs]
        src = np.frombuffer(b"".join(blocks), np.uint8).copy()
        off = np.cumsum([0] + [len(b) for b in blocks[:-1]]).astype(np.uint64)
        ln = np.array([len(b) for b in blocks], np.uint64)
        dst = np.zeros(1 << 20, np.uint8)
        stage3_out.append((dst, capi.aggregate_distinct_partition_compress_rows_hash(1, src, off, ln, dst, 1, keys,
                                                                                      [(SUM, pm.VAL_INT64)], distinct,
                                                                                      R2)))
    okeys = da.input_keys(keys[:1])
    merge = da.final_aggs(1, [(SUM, pm.VAL_INT64)], distinct)
    seen = {}
    for p in range(R2):
        blocks = [d[int(g["dst_off"][p]):int(g["dst_off"][p] + g["dst_len"][p])].tobytes() for d, g in stage3_out]
        blocks = [b for b in blocks if b]
        src = np.frombuffer(b"".join(blocks), np.uint8).copy()
        off = np.cumsum([0] + [len(b) for b in blocks[:-1]]).astype(np.uint64)
        ln = np.array([len(b) for b in blocks], np.uint64)
        out = np.zeros(1 << 20, np.uint8)
        res = capi.decompress_aggregate_rows_keys_packed(1, src, off, ln, out, okeys, merge)
        buf = out[:res["total"]].tobytes()
        for o, n in rm.parse(buf):
            row = buf[o + 4:o + n]
            g = int.from_bytes(row[8:12], "little", signed=True)
            seen[g] = [int.from_bytes(row[16 + 8 * k:24 + 8 * k], "little", signed=True) for k in range(3)]
    for g in range(25):
        xs = {x for gg, x, _ in data if gg == g and x is not None}
        vs = [v for gg, _, v in data if gg == g]
        assert seen[g] == [sum(vs), len(xs), sum(xs)], g


def test_q16_global_count_sums_over_reducers(capi):
    """a global count(DISTINCT order): each reducer's one row counts its own orders; their sum is the exact count (codec
    NONE, so the rows can be read back from the .data arena)"""
    rng = np.random.default_rng(16)
    types = ["long", "long"]
    orders = rng.integers(0, 5000, 30000)
    maps = [[hm.make_row(types, [int(o), 1]) for o in orders[m::3]] for m in range(3)]
    keys_in = hm.keys_of(types, [0])
    R1 = 4
    outs = []
    for rows in maps:
        recs, rl = hm.records_of(rows)
        dst = np.zeros(capi.partition_compress_bound(0, 0, R1, recs.size) + 64, np.uint8)
        outs.append((dst, capi.aggregate_partition_compress_rows_hash_packed(
            0, recs, rl, keys_in, [(SUM, pm.VAL_INT64, keys_in[0][1] + 8, 1)], R1, dst)))
    total = 0
    for p in range(R1):
        blocks = [d[int(g["dst_off"][p]):int(g["dst_off"][p] + g["dst_len"][p])].tobytes() for d, g in outs]
        src = np.frombuffer(b"".join(blocks), np.uint8).copy()
        off = np.cumsum([0] + [len(b) for b in blocks[:-1]]).astype(np.uint64)
        ln = np.array([len(b) for b in blocks], np.uint64)
        dst = np.zeros(1 << 16, np.uint8)
        r = capi.aggregate_distinct_partition_compress_rows_hash(0, src, off, ln, dst, 0, [(hm.FIELD["long"][0], 8)],
                                                                 [(SUM, pm.VAL_INT64)], [(COUNT, pm.VAL_INT64, 0)], 1)
        buf = dst[:r["total"]].tobytes()
        (o, n), = rm.parse(buf)
        total += int.from_bytes(buf[o + 4 + 16:o + 4 + 24], "little")
    assert total == len(set(orders.tolist()))


def test_beside_a_write_lane_call(capi):
    """this call (read lane) and a map-side aggregation (write lane) at once on one device, each equal to its model"""
    rng = np.random.default_rng(21)
    maps, types = make_maps(rng, 3, 3000, ["long"], [list(range(100))], ["int"], [list(range(200))])
    pmaps = map_side(maps, types, 2, [(COUNT, pm.VAL_NONE, 0)])
    keys = call_keys(types, 2)
    errors = []

    def reader():
        try:
            for _ in range(5):
                check(capi, pmaps, 1, keys, [(COUNT, pm.VAL_NONE)], [(COUNT, pm.VAL_INT32, 1)], 3)
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(e)

    def writer():
        try:
            recs, rl = hm.records_of(maps[0])
            keys_in = hm.keys_of(types, [0])
            for _ in range(5):
                dst = np.zeros(capi.partition_compress_bound(1, 0, 4, recs.size) + 64, np.uint8)
                r = capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys_in, [(COUNT, pm.VAL_NONE, 0,
                                                                                               -1)], 4, dst)
                assert r["n_groups"] == len(pm.partial_rows(maps[0], keys_in, [(COUNT, pm.VAL_NONE, 0, -1)]))
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=reader), threading.Thread(target=writer)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def _files(d, shuffle, map_id):
    out = []
    for kind in ("data", "index", "checksum"):
        path = d.getPath(kind, shuffle, map_id)
        path = path[len("file://"):] if path.startswith("file://") else path
        with open(path, "rb") as f:
            out.append(f.read())
    return out


@pytest.mark.parametrize("codec,ng", [("lz4", 1), ("none", 1), ("lz4", 0)])
def test_host_mirror_commits_the_writers_files(capi, tmp_path, codec, ng):
    """maps by G ++ X through the serialized writer's aggregateRows; per reducer, aggregateDistinctRows into a writer
    of shuffle 1 equals a writer of shuffle 2 fed the model's rows of the same blocks (hashRows by G, or one partition)"""
    host = pkg.host
    d = rm.mirror(tmp_path, codec)
    rng = np.random.default_rng(31 + ng)
    M, R1, R2 = 3, 2, 3 if ng else 1
    maps, types = make_maps(rng, M, 800, ["long"], [list(range(30)) + [None]], ["int"], [list(range(40)) + [None]])
    keys_in = hm.keys_of(types, [0, 1])
    f = [(SUM, pm.VAL_INT64, 0), (AVG, pm.VAL_FLOAT64, 1), (COUNT, pm.VAL_NONE, 0)]
    f_in = [(fn, vt, hm.keys_of(types, [2 + j])[0][1], 2 + j) if vt != pm.VAL_NONE else (fn, vt, 0, -1)
            for fn, vt, j in f]
    for m, rows in enumerate(maps):
        w = host.S3SerializedShuffleWriter(d, 0, m, R1)
        w.hashRows(keys_in)
        w.aggregateRows(f_in)
        for r in rows:
            w.insertRecord(0, len(r).to_bytes(4, "big") + r)
        w.commit()
        w.close()
    keys = call_keys(types, 2)  # without G both columns are X: count(DISTINCT g, x)
    aggs = [(a, b) for a, b, _ in f]
    distinct = [(COUNT, pm.VAL_INT32, 1), (SUM, pm.VAL_INT32, 1)] if ng else [(COUNT, pm.VAL_NONE, ALL)]
    for red in range(R1):
        reader = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        w = host.S3SerializedShuffleWriter(d, 1, red, R2)
        lengths, counts = reader.aggregateDistinctRows(w, ng, keys, aggs, distinct)
        w.close()
        # the same rows as one stream sorted stably by G ++ X (maps, then blocks, in order): the model's stage 2
        # sorts stably by that key again, so its groups and their merge orders are the call's
        plain = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        rows, _ = plain.readSortedRowsKeys(da.input_keys(keys))
        plain.close()
        reader.close()
        want, want_counts = da.reducer([rows], ng, keys, aggs, distinct)
        assert counts == want_counts
        ref = host.S3SerializedShuffleWriter(d, 2, red, R2)
        if ng:
            ref.hashRows(da.input_keys(keys)[:ng])
        for r in want:
            ref.insertRecord(0, len(r).to_bytes(4, "big") + r)
        assert np.array_equal(ref.commit(), lengths)
        ref.close()
        assert _files(d, 1, red) == _files(d, 2, red)
