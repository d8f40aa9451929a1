"""The central-moment aggregates on the GPU.  Map side: b2s_aggregate_partition_compress_rows_hash_* and the grouping
sets call with B2S_WINDOW_VARIANCE are byte for byte b2s_partition_compress_rows_hash_packed over the model's partial
rows (tests/moments_model.py).  Reduce side: every aggregated read with B2S_AGG_VARIANCE merges partial rows byte for
byte as the merge model does.  End to end: maps, then reducers, then stddev_samp, within rounding of numpy."""
import struct

import numpy as np
import pytest

import grouping_sets_model as gm
import hash_model as hm
import moments_model as mm
import partial_agg_model as pm
import rows_model as rm
import spark_s3_shuffle_b200 as pkg
import test_gpu_aggregate_partition_rows as ta
import test_gpu_exchange_rows as te

pytestmark = pytest.mark.gpu

VAR = mm.VARIANCE
NONE_CODEC = 0


@pytest.fixture(scope="module")
def capi():
    c = pkg.capi
    c.init(1)
    return c


def f_of(nk, nullable=True):
    """(fn, j): the function over value field j of ta.dataset's rows"""
    return lambda fn, j: (fn, ta.VT[j], 8 + 8 * (nk + j), nk + j if nullable else -1)


def check(capi, rows, keys, aggs, R, codec=1, alg=3, dev=False):
    """the call (packed or _dev) == the hash call over the model's partial rows -> (outputs, .data, partial rows)"""
    partial = mm.partial_rows(rows, keys, aggs)
    recs, rl = hm.records_of(rows)
    prec, prl = hm.records_of(partial)
    cap = capi.partition_compress_bound(codec, 0, R, prec.size) + 64
    ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    ref = capi.partition_compress_rows_hash_packed(codec, prec, prl, pm.output_keys(keys), R, ref_dst,
                                                   checksum_alg=alg)
    if dev:
        d_rec, d_len, d_dst = capi.dev_alloc(max(recs.size, 1)), capi.dev_alloc(max(rl.size * 4, 4)), \
            capi.dev_alloc(cap)
        try:
            capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
            capi.dev_memcpy(d_len, rl.ctypes.data, rl.size * 4, 1)
            got = capi.aggregate_partition_compress_rows_hash_dev(codec, d_rec, recs.size, d_len, rl.size, keys, aggs,
                                                                 R, d_dst, cap, checksum_alg=alg)
            capi.dev_memcpy(got_dst.ctypes.data, d_dst, got["total"], 2)
        finally:
            for p in (d_rec, d_len, d_dst):
                capi.dev_free(p)
    else:
        got = capi.aggregate_partition_compress_rows_hash_packed(codec, recs, rl, keys, aggs, R, got_dst,
                                                                 checksum_alg=alg)
    assert got["n_groups"] == len(partial)
    assert got["total"] == ref["total"]
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(got_dst[:ref["total"]], ref_dst[:ref["total"]])
    return got, got_dst, partial


def same_nan(a, b):
    """partial rows equal field by field, any NaN equal to any NaN (the JVM pins no NaN payload)"""
    assert len(a) == len(b)
    for o in range(0, len(a), 8):
        x, y = struct.unpack("<d", a[o:o + 8])[0], struct.unpack("<d", b[o:o + 8])[0]
        assert (x != x and y != y) or a[o:o + 8] == b[o:o + 8], o


def plain_rows(capi, rows, keys, aggs):
    """the call with codec NONE and one partition -> its partial rows"""
    recs, rl = hm.records_of(rows)
    dst = np.zeros(capi.partition_compress_bound(NONE_CODEC, 0, 1, recs.size * 4 + 4096) + 4096, np.uint8)
    got = capi.aggregate_partition_compress_rows_hash_packed(NONE_CODEC, recs, rl, keys, aggs, 1, dst)
    buf = dst[:got["total"]].tobytes()
    return [buf[o + 4:o + n] for o, n in rm.parse(buf)]


# ---- the map side ----
@pytest.mark.parametrize("nullable", [True, False])
def test_every_input_type_beside_the_other_buffers(capi, nullable):
    rng = np.random.default_rng(1 + nullable)
    rows, types = ta.dataset(rng, 4000, ["string", "int"], 300)
    f = f_of(2, nullable)
    # without null bits a null input reads as its zeroed slot: a decimal(12, 2) sum then, whose slot is a long
    dsum = f(pm.SUM, 7 if nullable else 8)
    aggs = [f(VAR, j) for j in (0, 1, 2, 3, 4, 5)] + [f(pm.SUM, 5), dsum, (pm.COUNT, pm.VAL_NONE, 0, -1), f(pm.AVG, 2)]
    keys = hm.keys_of(types, [0, 1])
    for dev in (False, True):
        check(capi, rows, keys, aggs, 7, dev=dev)


@pytest.mark.parametrize("codec", [0, 1, 2, 3])
def test_every_codec(capi, codec):
    rng = np.random.default_rng(10 + codec)
    rows, types = ta.dataset(rng, 3000, ["long"], 200)
    f = f_of(1)
    check(capi, rows, hm.keys_of(types, [0]), [f(VAR, 5), f(pm.AVG, 3), f(VAR, 3)], 5, codec)


def test_group_sizes_across_every_fold(capi):
    """groups of 1, 32 (a thread's), 33, 2048 and 2049 records (the warp chains), nulls among them"""
    rng = np.random.default_rng(3)
    sizes = [1, 32, 33, 2048, 2049, 5, 31]
    types = ["int", "int", "double", "long", "float"]
    rows = []
    for k, s in enumerate(sizes):
        for _ in range(s):
            big = int(rng.integers(2**53, 2**62)) * (1 if rng.random() < 0.5 else -1)
            rows.append(hm.make_row(types, [k, None if rng.random() < 0.1 else int(rng.integers(-10**9, 10**9)),
                                            None if rng.random() < 0.1 else float(rng.normal() * 1e6),
                                            big, float(np.float32(rng.normal()))]))
    order = rng.permutation(len(rows))
    rows = [rows[i] for i in order]
    keys = hm.keys_of(types, [0])
    aggs = [(VAR, pm.VAL_INT32, 16, 1), (VAR, pm.VAL_FLOAT64, 24, 2), (pm.SUM, pm.VAL_FLOAT64, 24, 2),
            (VAR, pm.VAL_INT64, 32, 3), (VAR, pm.VAL_FLOAT32, 40, 4)]
    for R in (1, 3):
        check(capi, rows, keys, aggs, R)


def test_one_group_of_over_a_million_rows(capi):
    rng = np.random.default_rng(4)
    n = 1_100_000
    kcol = np.where(rng.random(n) < 0.97, 0, rng.integers(1, 4, n))
    dv = rng.normal(size=n) * 1e3 + 5.0
    nulls = rng.random(n) < 0.05
    rowb = 8 + 8 * 2
    arr = np.zeros((n, rowb), np.uint8)
    arr[:, 0:8] = np.where(nulls, np.uint64(1) << np.uint64(1), np.uint64(0)).view(np.uint8).reshape(n, 8)
    arr[:, 8:16] = kcol.astype(np.int64).view(np.uint8).reshape(n, 8)
    arr[:, 16:24] = np.where(nulls, 0.0, dv).view(np.uint8).reshape(n, 8)
    pre = np.frombuffer(struct.pack(">i", rowb), np.uint8)
    recs = np.concatenate([np.tile(pre, (n, 1)), arr], axis=1).reshape(-1)
    rl = np.full(n, 4 + rowb, np.uint32)
    keys = [(hm.FIELD["long"][0], 8, 8, -1)]
    aggs = [(VAR, pm.VAL_FLOAT64, 16, 1), (pm.SUM, pm.VAL_FLOAT64, 16, 1)]
    dst = np.zeros(1 << 16, np.uint8)
    got = capi.aggregate_partition_compress_rows_hash_packed(NONE_CODEC, recs, rl, keys, aggs, 1, dst)
    assert got["n_groups"] == 4
    buf = dst[:got["total"]].tobytes()
    for (o, ln), k in zip(rm.parse(buf), range(4)):
        m = kcol == k
        xs = dv[m & ~nulls].tolist()
        s = 0.0
        for x in xs:
            s += x
        row = buf[o + 4:o + ln]
        assert struct.unpack("<q", row[8:16])[0] == k
        assert struct.unpack("<4d", row[16:48]) == mm.fold(xs) + (s,)


def test_special_values(capi):
    """-0.0, NaN, infinities and 1e300 inputs: the model's buffers, any NaN for any NaN"""
    rng = np.random.default_rng(5)
    types = ["int", "double"]
    specials = [0.0, -0.0, float("nan"), float("inf"), -float("inf"), 1e300, -1e300, 1.0, 2.5]
    rows = [hm.make_row(types, [int(rng.integers(0, 40)), None if rng.random() < 0.1 else
                                specials[int(rng.integers(len(specials)))]]) for _ in range(3000)]
    rows += [hm.make_row(types, [100 + k, x]) for k, x in enumerate(specials)]
    rows += [hm.make_row(types, [200, -0.0]), hm.make_row(types, [200, -0.0]), hm.make_row(types, [201, None])]
    keys = hm.keys_of(types, [0])
    aggs = [(VAR, pm.VAL_FLOAT64, 16, 1)]
    got = plain_rows(capi, rows, keys, aggs)
    want = mm.partial_rows(rows, keys, aggs)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        same_nan(g, w)
    by_key = {struct.unpack("<i", g[8:12])[0]: struct.unpack("<3d", g[16:40]) for g in got}
    assert by_key[201] == (0.0, 0.0, 0.0) and by_key[200] == (2.0, 0.0, 0.0)
    assert by_key[103][1] == float("inf") and by_key[103][2] != by_key[103][2]
    # and byte for byte where no NaN arises
    finite = [r for r in rows if not hm.is_null(r, 1) and abs(struct.unpack("<d", r[16:24])[0]) < 1e10]
    check(capi, finite, keys, aggs, 3)


def test_q17_and_q39_shapes(capi):
    rng = np.random.default_rng(6)
    # q17: count, avg and stddev_samp of three int quantities, grouped by three string columns: 12 entries, 21 fields
    types = ["string", "string", "string", "int", "int", "int"]
    pool = [(b"AAAAAAAABAAAAAAA%03d" % k, b"state%02d" % (k % 50), b"item desc %d" % (k % 7)) for k in range(400)]
    rows = [hm.make_row(types, list(pool[int(rng.integers(len(pool)))]) +
                        [None if rng.random() < 0.05 else int(rng.integers(1, 100)) for _ in range(3)])
            for _ in range(20000)]
    aggs = []
    for j in range(3):
        a = (0, pm.VAL_INT32, 8 + 8 * (3 + j), 3 + j)
        aggs += [(pm.COUNT,) + a[1:], (pm.AVG,) + a[1:], (VAR,) + a[1:]]
    aggs += [(pm.COUNT, pm.VAL_NONE, 0, -1)] * 3
    assert len(aggs) == 12 and len(mm.buffers(aggs)) + 3 <= 32
    check(capi, rows, hm.keys_of(types, [0, 1, 2]), aggs, 200)
    # q39: stddev_samp and avg of an int grouped by four columns
    types = ["int", "int", "string", "int", "int"]
    rows = [hm.make_row(types, [int(rng.integers(0, 5)), int(rng.integers(0, 30)), b"wh%d" % rng.integers(0, 5),
                                int(rng.integers(1, 13)), int(rng.integers(0, 1000))]) for _ in range(20000)]
    aggs = [(VAR, pm.VAL_INT32, 40, 4), (pm.AVG, pm.VAL_INT32, 40, 4)]
    check(capi, rows, hm.keys_of(types, [0, 1, 2, 3]), aggs, 200)


def test_a_bad_value_slot_is_named(capi):
    types = ["int", "long", "double"]
    rows = [hm.make_row(types, [k % 3, k, float(k)]) for k in range(50)]
    rows[17] = rows[17][:24]  # no double slot
    recs, rl = hm.records_of(rows)
    with pytest.raises(capi.B2SError) as e:
        capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, hm.keys_of(types, [0]),
                                                           [(VAR, pm.VAL_FLOAT64, 24, 2)], 4, np.zeros(1 << 14, np.uint8))
    assert e.value.code == capi.E_ARG and "record 17" in str(e.value)


def test_grouping_sets(capi):
    """the grouping sets call == the aggregating call over the materialised Expand rows == the model's partial rows"""
    rng = np.random.default_rng(7)
    rows, types = ta.dataset(rng, 3000, ["string", "int"], 200)
    keys = hm.keys_of(types, [0, 1])
    f = f_of(2)
    aggs = [f(VAR, 2), f(VAR, 5), f(pm.AVG, 2), f(VAR, 4), (pm.COUNT, pm.VAL_NONE, 0, -1)]
    for masks in (gm.rollup(2), gm.cube(2)):
        xrows, xkeys, xaggs = gm.expand(rows, keys, aggs, masks)
        _, agg_dst, partial = check(capi, xrows, xkeys, xaggs, 9)
        recs, rl = hm.records_of(rows)
        cap = agg_dst.size
        got_dst = np.zeros(cap, np.uint8)
        got = capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, masks, 9,
                                                                               got_dst, checksum_alg=3)
        prec, prl = hm.records_of(partial)
        ref_dst = np.zeros(cap, np.uint8)
        ref = capi.partition_compress_rows_hash_packed(1, prec, prl, pm.output_keys(xkeys), 9, ref_dst,
                                                       checksum_alg=3)
        assert got["n_groups"] == len(partial) and got["total"] == ref["total"]
        assert np.array_equal(got_dst[:got["total"]], ref_dst[:ref["total"]])


# ---- the reduce side ----
LONE = -1  # the key of one lone buffer (11, 0.1, 0), whose merge from (0, 0, 0) has avg (0.1 / 11) * 11 != 0.1


def partial_maps(rng, M, n_keys, n_per_map, big_key=None, big=0):
    """M maps' partial rows [null word, long key, (n, avg, m2), count, (n, avg, m2)] with random buffers, map 0 with
    big more rows of big_key and the LONE row"""
    types = ["long", "double", "double", "double", "long", "double", "double", "double"]
    maps = []
    for m in range(M):
        rows = []
        for i in range(n_per_map + (big if m == 0 else 0)):
            k = big_key if i >= n_per_map else int(rng.integers(0, n_keys))
            t = [float(rng.integers(0, 60)), float(rng.normal() * 100), float(abs(rng.normal()) * 1e4)]
            u = [float(rng.integers(0, 3)), float(rng.normal()), float(abs(rng.normal()))]
            rows.append(hm.make_row(types, [k] + t + [int(rng.integers(0, 60))] + u))
        if m == 0:
            rows.append(hm.make_row(types, [LONE, 11.0, 0.1, 0.0, 11, 0.0, 0.0, 0.0]))
        maps.append(rows)
    keys = hm.keys_of(types, [0])
    aggs = [(mm.AGG_VARIANCE, 16, -1), (pm.SUM_I64, 40, 4), (mm.AGG_VARIANCE, 48, -1)]
    return maps, keys, aggs


def blocks_of(maps):
    streams = [rm.stream(r) for r in maps]
    src = np.frombuffer(b"".join(streams), np.uint8).copy()
    off = np.cumsum([0] + [len(s) for s in streams[:-1]]).astype(np.uint64)
    return src, off, np.array([len(s) for s in streams], np.uint64), streams


@pytest.mark.parametrize("n_keys", [300, 30000])
def test_reduce_merges_variance_triples(capi, n_keys):
    """groups of a few records (a thread's) and of more than 16 (a warp's), one of over 6000, single-key and
    composite-key calls"""
    rng = np.random.default_rng(8 + n_keys)
    maps, keys, aggs = partial_maps(rng, 5, n_keys, 2000, big_key=7, big=6000)
    src, off, ln, streams = blocks_of(maps)
    want, n_rec, n_groups = mm.model_aggregate(streams, keys, aggs)
    dst = np.zeros(len(want) + 4096, np.uint8)
    r = capi.decompress_aggregate_rows_keys_packed(0, src, off, ln, dst, keys, aggs)
    assert (r["n_records"], r["n_groups"]) == (n_rec, n_groups) and dst[:r["total"]].tobytes() == want
    kt, ko, kl, kn = keys[0]
    dst[:] = 0
    r = capi.decompress_aggregate_rows_packed(0, src, off, ln, dst, kt, ko, kl, kn, aggs)
    assert dst[:r["total"]].tobytes() == want
    lone = {struct.unpack("<q", want[o + 12:o + 20])[0]: want[o + 4:o + n] for o, n in rm.parse(want)}[LONE]
    assert struct.unpack("<3d", lone[16:40]) == (11.0, (0.1 / 11.0) * 11.0, 0.0) and (0.1 / 11.0) * 11.0 != 0.1


def test_reduce_argument_errors(capi):
    src, dst = np.zeros(64, np.uint8), np.zeros(64, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.full(1, 24, np.uint64)
    key, late = (capi.KEY_INT64, 8, 8, 0), (capi.KEY_INT64, 48, 8, -1)
    V, S = capi.AGG_VARIANCE, capi.AGG_SUM_INT64
    for aggs, k in (([(V, 16, 1)], key), ([(V | 5 << 8, 16, -1)], key), ([(V, 32, -1)], late),
                    ([(V, 16, -1), (S, 32, -1)], key), ([(S, 24, -1), (V, 16, -1)], key),
                    ([(V, 16, -1), (V, 32, -1)], key), ([(S, 56, 192), (V, 16, -1)], late), ([(13, 16, -1)], key)):
        for call in (lambda: capi.decompress_aggregate_rows_packed(0, src, off, ln, dst, *k, aggs=aggs),
                     lambda: capi.decompress_aggregate_rows_keys_packed(0, src, off, ln, dst, [k], aggs)):
            with pytest.raises(capi.B2SError) as e:
                call()
            assert e.value.code == capi.E_ARG, aggs


@pytest.fixture
def cache(capi):
    capi.exchange_set_budget(4 << 30)
    yield capi
    capi.exchange_set_budget(0)
    for s in range(40, 44):
        capi.exchange_remove(s, -1)


def test_exchange_cached_read_equals_the_fetched_one(cache):
    rng = np.random.default_rng(9)
    maps, keys, aggs = partial_maps(rng, 3, 200, 1500, big_key=3, big=3000)
    stored = [te.store(cache, "hash", 40, m, rows, keys, 4, compare=False) for m, rows in enumerate(maps)]
    want = te.check_read(cache, 40, stored, 0, 4, "aggregate_rows_keys", (keys, aggs))
    model, _, _ = mm.model_aggregate([rm.stream(r) for r in maps], keys, aggs)
    assert want[0] == model


def test_end_to_end_stddev_samp(capi):
    """maps written by the GPU, merged by the GPU reducer, evaluated as stddev_samp / var_pop: numpy's, within
    rounding"""
    rng = np.random.default_rng(12)
    types = ["int", "int", "double"]
    keys = hm.keys_of(types, [0])
    M, R = 4, 3
    data = {k: [] for k in range(30)}
    maps = []
    for m in range(M):
        rows = []
        for _ in range(5000):
            k = int(rng.integers(0, 30))
            x = int(rng.integers(-1000, 1000))
            data[k].append(x)
            rows.append(hm.make_row(types, [k, x, float(x) / 7]))
        maps.append(rows)
    aggs = [(VAR, pm.VAL_INT32, 16, 1), (pm.AVG, pm.VAL_INT32, 16, 1), (VAR, pm.VAL_FLOAT64, 24, 2)]
    datas = []
    for rows in maps:
        recs, rl = hm.records_of(rows)
        dst = np.zeros(capi.partition_compress_bound(1, 0, R, recs.size) + 64, np.uint8)
        datas.append((dst, capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, R, dst,
                                                                              checksum_alg=3)))
    okeys, merge = pm.output_keys(keys), mm.merge_aggs(keys, aggs)
    seen = 0
    for p in range(R):
        blocks = [d[int(g["dst_off"][p]):int(g["dst_off"][p] + g["dst_len"][p])].tobytes() for d, g in datas]
        blocks = [b for b in blocks if b]
        src = np.frombuffer(b"".join(blocks), np.uint8).copy()
        off = np.cumsum([0] + [len(b) for b in blocks[:-1]]).astype(np.uint64)
        ln = np.array([len(b) for b in blocks], np.uint64)
        out = np.zeros(1 << 20, np.uint8)
        res = capi.decompress_aggregate_rows_keys_packed(1, src, off, ln, out, okeys, merge)
        buf = out[:res["total"]].tobytes()
        for o, n in rm.parse(buf):
            row = buf[o + 4:o + n]
            k = struct.unpack("<i", row[8:12])[0]
            got = mm.evaluate(struct.unpack("<3d", row[16:40]), "stddev_samp")
            assert np.isclose(got, np.std(data[k], ddof=1), rtol=1e-12)
            got = mm.evaluate(struct.unpack("<3d", row[56:80]), "var_pop")
            assert np.isclose(got, np.var(np.array(data[k], float) / 7), rtol=1e-10)
            seen += 1
    assert seen == 30
