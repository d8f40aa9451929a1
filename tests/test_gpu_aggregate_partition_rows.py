"""b2s_aggregate_partition_compress_rows_hash_*: a map task's partial aggregation on the GPU.  Every output must be byte
for byte what b2s_partition_compress_rows_hash_packed returns for the model's partial rows (tests/partial_agg_model.py)
keyed by the key columns at their output slots; end to end, the reduce side's merge over the partial rows of several
maps must equal the model of the whole dataset."""
import ctypes as C
import struct

import numpy as np
import pytest

import hash_model as hm
import partial_agg_model as pm
import spark_s3_shuffle_b200 as pkg

pytestmark = pytest.mark.gpu

CODECS = [(0, 0), (1, 0), (2, 0), (3, 1)]
# value fields after the key fields: byte, short, int, long, float, double, decimal(7, 2), decimal(25, 3),
# decimal(12, 2) (a compact input into a wide sum buffer), and a double with NaN payloads and infinities
VALUE_TYPES = ["byte", "short", "int", "long", "float", "double", "long", "decimal", "long", "double"]
VT = [pm.VAL_INT8, pm.VAL_INT16, pm.VAL_INT32, pm.VAL_INT64, pm.VAL_FLOAT32, pm.VAL_FLOAT64, pm.val_decimal(7, 2),
      pm.val_decimal(25, 3), pm.val_decimal(12, 2), pm.VAL_FLOAT64]
SPECIAL = [("bits", 0x7FF8000000000000), ("bits", 0x7FF0000000000001), ("bits", 0xFFF8000000000123),
           ("bits", 0x7FFFFFFFFFFFFFFF), float("inf"), -float("inf"), 0.0, -0.0]


@pytest.fixture(scope="module")
def capi():
    c = pkg.capi
    c.init(1)
    return c


def value(rng, t, j, finite):
    if rng.random() < 0.2:
        return None
    if j == 6:  # decimal(7, 2) as a long
        return int(rng.integers(-10**7 + 1, 10**7))
    if j == 8:  # decimal(12, 2) as a long, negative half the time
        return int(rng.integers(-10**12 + 1, 10**12))
    if j == 9 and rng.random() < 0.3:
        return SPECIAL[int(rng.integers(len(SPECIAL)))]
    if t == "decimal":
        return int(rng.integers(-10**18, 10**18)) * 10**6 + int(rng.integers(0, 10**6))
    if t in ("float", "double"):
        if not finite and rng.random() < 0.2:  # signed zeros (NaN and infinity appear as keys)
            return [0.0, -0.0][int(rng.integers(2))]
        x = float(rng.normal() * 1e3)
        return float(np.float32(x)) if t == "float" else x
    bits = {"byte": 8, "short": 16, "int": 32, "long": 64}[t]
    return int(rng.integers(-(1 << (bits - 1)), (1 << (bits - 1)) - 1, dtype=np.int64))


def dataset(rng, n, key_types, n_keys_distinct, finite=True, null_keys=True):
    """rows of [key fields..., value fields...]: keys drawn from a pool of n_keys_distinct key tuples"""
    nk = len(key_types)
    pool = [r for r in hm.random_rows(rng, 2 * n_keys_distinct + 40, types=key_types,
                                      null_rate=0.1 if null_keys else 0.0)
            if null_keys or not any(hm.is_null(r, c) for c in range(nk))][:n_keys_distinct]
    types = key_types + VALUE_TYPES
    rows = []
    picks = rng.integers(0, len(pool), n)
    for p in picks:
        base = pool[p]
        vals = [value(rng, t, j, finite) for j, t in enumerate(VALUE_TYPES)]
        rows.append(splice(base, key_types, vals))
    return rows, types


def splice(key_row, key_types, vals):
    """a row of the key row's key fields followed by value fields (rebuilt with make_row from the key row's values)"""
    nk = len(key_types)
    kvals = []
    bitset = 8 * ((nk + 63) // 64)
    for c, t in enumerate(key_types):
        if hm.is_null(key_row, c):
            kvals.append(None)
            continue
        slot = key_row[bitset + 8 * c:bitset + 8 * c + 8]
        if t in ("string", "decimal"):
            s = int.from_bytes(slot, "little")
            b = key_row[s >> 32:(s >> 32) + (s & 0xFFFFFFFF)]
            kvals.append(bytes(b) if t == "string" else int.from_bytes(b, "big", signed=True))
        elif t in ("float", "double"):
            w = 4 if t == "float" else 8
            kvals.append(("bits", int.from_bytes(slot[:w], "little")))
        elif t == "bool":
            kvals.append(bool(slot[0]))
        else:
            kvals.append(int.from_bytes(slot[:hm.FIELD[t][1]], "little", signed=True))
    return hm.make_row(key_types + VALUE_TYPES, kvals + vals)


def all_aggs(nk, with_avg_fp=True):
    """the table's (function, type) pairs over the value fields of dataset's rows (16 buffers); the NaN-bearing double
    (field 9) only through MIN / MAX, whose result keeps an input's bits"""
    slot = lambda j: 8 + 8 * (nk + j)  # noqa: E731  (one null word: nk + 8 <= 64 fields)
    f = lambda fn, j: (fn, VT[j], slot(j), nk + j)  # noqa: E731
    return [f(pm.SUM, 0), f(pm.SUM, 3), f(pm.SUM, 5), f(pm.SUM, 8), f(pm.SUM, 7), (pm.COUNT, pm.VAL_NONE, 0, -1),
            f(pm.COUNT, 4), f(pm.AVG, 6), f(pm.MIN, 2), f(pm.MAX, 3), f(pm.MIN, 9), f(pm.MAX, 9), f(pm.MAX, 7)]


def check(capi, rows, keys, aggs, R, codec=1, lvl=0, alg=3, dev=False):
    partial = pm.partial_rows(rows, keys, aggs)
    recs, rl = hm.records_of(rows)
    prec, prl = hm.records_of(partial)
    okeys = pm.output_keys(keys)
    cap = capi.partition_compress_bound(codec, 0, R, prec.size) + 64
    ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    ref = capi.partition_compress_rows_hash_packed(codec, prec, prl, okeys, R, ref_dst, checksum_alg=alg, level=lvl)
    if dev:
        d_rec = capi.dev_alloc(max(recs.size, 1))
        d_len = capi.dev_alloc(max(rl.size * 4, 4))
        d_dst = capi.dev_alloc(cap)
        try:
            if recs.size:
                capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
                capi.dev_memcpy(d_len, rl.ctypes.data, rl.size * 4, 1)
            got = capi.aggregate_partition_compress_rows_hash_dev(codec, d_rec, recs.size, d_len, rl.size, keys, aggs,
                                                                 R, d_dst, cap, checksum_alg=alg, level=lvl)
            if got["total"]:
                capi.dev_memcpy(got_dst.ctypes.data, d_dst, got["total"], 2)
        finally:
            for p in (d_rec, d_len, d_dst):
                capi.dev_free(p)
    else:
        got = capi.aggregate_partition_compress_rows_hash_packed(codec, recs, rl, keys, aggs, R, got_dst,
                                                                 checksum_alg=alg, level=lvl)
    assert got["n_groups"] == len(partial)
    assert got["total"] == ref["total"]
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(got_dst[:ref["total"]], ref_dst[:ref["total"]])
    return got, got_dst, partial


@pytest.mark.parametrize("codec,lvl", CODECS)
@pytest.mark.parametrize("alg", [0, 1, 2, 3])
def test_every_codec_and_checksum(capi, codec, lvl, alg):
    rng = np.random.default_rng(codec * 10 + alg)
    kt = ["string", "int"]
    rows, types = dataset(rng, 3000, kt, 300)
    check(capi, rows, hm.keys_of(types, [0, 1]), all_aggs(2), 7, codec, lvl, alg)


@pytest.mark.parametrize("ktype", ["bool", "byte", "short", "int", "long", "float", "double", "string", "decimal"])
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("composite", [False, True])
def test_every_key_type(capi, ktype, nullable, composite):
    rng = np.random.default_rng(len(ktype) * 1000 + ord(ktype[1]) * 4 + 2 * nullable + composite)
    kt = [ktype, "string"] if composite else [ktype]
    rows, types = dataset(rng, 2000, kt, 150, finite=False, null_keys=nullable)
    keys = hm.keys_of(types, range(len(kt)), nullable=nullable)
    for dev in (False, True):
        check(capi, rows, keys, all_aggs(len(kt), True), 13, dev=dev)


@pytest.mark.parametrize("n,distinct", [(0, 1), (1, 1), (5000, 1), (5000, 5000), (40000, 4), (20000, 20000)])
@pytest.mark.parametrize("R", [1, 2000])
def test_shapes(capi, n, distinct, R):
    rng = np.random.default_rng(n + distinct + R)
    rows, types = dataset(rng, n, ["long"], distinct) if n else ([], ["long"] + VALUE_TYPES)
    keys = hm.keys_of(types, [0])
    for aggs in (all_aggs(1), []):
        check(capi, rows, keys, aggs, R)


def test_sixteen_buffers_and_every_pair(capi):
    rng = np.random.default_rng(5)
    rows, types = dataset(rng, 4000, ["int"], 40)
    nk = 1
    slot = lambda j: 8 + 8 * (nk + j)  # noqa: E731
    f = lambda fn, j: (fn, VT[j], slot(j), nk + j)  # noqa: E731
    pairs = [f(pm.SUM, j) for j in range(9)] + [f(pm.COUNT, j) for j in range(10)] + [(pm.COUNT, pm.VAL_NONE, 0, -1)]
    pairs += [f(pm.AVG, j) for j in range(9)] + [f(pm.MIN, j) for j in (2, 3, 5, 6, 7, 8, 9)] + \
        [f(pm.MAX, j) for j in (2, 3, 5, 6, 7, 8, 9)]
    # at most 16 buffers per call: take the pairs in calls that fill them
    calls, cur = [], []
    for p in pairs:
        nb = len(pm.buffers(cur + [p]))
        if nb > 16:
            calls.append(cur)
            cur = []
        cur.append(p)
    calls.append(cur)
    assert any(len(pm.buffers(c)) == 16 for c in calls)
    for c in calls:
        check(capi, rows, hm.keys_of(types, [0]), c, 5)


def test_large_groups_over_a_million_rows(capi):
    """a few keys over 1.2 M rows: the chunked folds and the double-sum chains"""
    rng = np.random.default_rng(11)
    n, K = 1_200_000, 3
    nk = 1
    types = ["long"] + VALUE_TYPES
    keys = hm.keys_of(types, [0])
    kcol = rng.integers(0, K, n)
    lv = rng.integers(-2**40, 2**40, n)
    dv = rng.normal(size=n) * 1e3
    iv = rng.integers(-2**31, 2**31 - 1, n)
    nulls = rng.random(n) < 0.1
    # rows of the 16 fields built in bulk: null word, key, byte, short, int, long, float, double, long, decimal(unused)
    nf = len(types)
    rowb = 8 + 8 * nf
    arr = np.zeros((n, rowb), np.uint8)
    word = np.where(nulls, np.uint64(1) << np.uint64(nk + 5), np.uint64(0)) | \
        (np.uint64(1) << np.uint64(nk + 7))  # the decimal(25) field is always null
    arr[:, 0:8] = word.view(np.uint8).reshape(n, 8)
    arr[:, 8:16] = kcol.astype(np.int64).view(np.uint8).reshape(n, 8)
    arr[:, 8 + 8 * (nk + 2):8 + 8 * (nk + 2) + 4] = iv.astype(np.int32).view(np.uint8).reshape(n, 4)
    arr[:, 8 + 8 * (nk + 3):8 + 8 * (nk + 4)] = lv.astype(np.int64).view(np.uint8).reshape(n, 8)
    arr[:, 8 + 8 * (nk + 5):8 + 8 * (nk + 6)] = np.where(nulls, 0.0, dv).view(np.uint8).reshape(n, 8)
    pre = np.frombuffer(struct.pack(">i", rowb), np.uint8)
    recs = np.concatenate([np.tile(pre, (n, 1)), arr], axis=1).reshape(-1)
    rl = np.full(n, 4 + rowb, np.uint32)
    slot = lambda j: 8 + 8 * (nk + j)  # noqa: E731
    f = lambda fn, j: (fn, VT[j], slot(j), nk + j)  # noqa: E731
    aggs = [f(pm.SUM, 3), f(pm.SUM, 5), f(pm.AVG, 2), f(pm.MIN, 5), f(pm.MAX, 3), f(pm.MIN, 2), f(pm.COUNT, 5),
            f(pm.AVG, 5)]
    # the model's partial rows, folded with numpy where exact and in order for the double sums
    out = []
    for k in range(K):
        m = kcol == k
        d = dv[m & ~nulls]
        s = 0.0
        for x in d.tolist():
            s += x
        a = 0.0
        for x in np.where(nulls[m], 0.0, dv[m]).tolist():
            a += x
        ints = iv[m]
        ia = 0.0
        for x in ints.tolist():
            ia += float(x)
        dmin_i = int(np.argmin(np.where(nulls[m], np.inf, dv[m])))
        vals = [int(lv[m].sum()) % 2**64, s, ia, int(m.sum()), int(ints.min()), int(lv[m].max()),
                float(dv[m][dmin_i]), int(ints.min()), int((m & ~nulls).sum()), a, int((m & ~nulls).sum())]
        first = bytes(np.concatenate([pre, arr[np.argmax(m)]]).tobytes()[4:])
        # buffers: SUM long, SUM double, AVG int (sum, count), MIN double, MAX long, MIN int, COUNT, AVG double
        bv = [vals[0], vals[1], vals[2], vals[3], vals[6], int(lv[m].max()), vals[4], vals[8], vals[9], vals[10]]
        out.append(pm.emit(first, keys, pm.buffers(aggs), bv))
    for R in (1, 4):
        prec, prl = hm.records_of(out)
        okeys = pm.output_keys(keys)
        cap = capi.partition_compress_bound(1, 0, R, prec.size) + 64
        ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
        ref = capi.partition_compress_rows_hash_packed(1, prec, prl, okeys, R, ref_dst, checksum_alg=3)
        got = capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, R, got_dst, checksum_alg=3)
        assert got["n_groups"] == K
        for k in ("dst_off", "dst_len", "checksums", "status"):
            assert np.array_equal(got[k], ref[k]), k
        assert np.array_equal(got_dst[:ref["total"]], ref_dst[:ref["total"]])
        t = capi.last_timing()
        assert t["dominant_ms"] > 0 and t["dominant_ms"] <= t["kernel_ms"]


def test_bad_records_are_named(capi):
    rng = np.random.default_rng(3)
    rows, types = dataset(rng, 50, ["int"], 5)
    keys = hm.keys_of(types, [0])
    aggs = all_aggs(1)
    rows = list(rows)
    rows[30] = rows[30][:16]  # holds the key slot, not the value slots
    recs, rl = hm.records_of(rows)
    dst = np.zeros(1 << 16, np.uint8)
    with pytest.raises(capi.B2SError) as e:
        capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, 4, dst)
    assert e.value.code == capi.E_ARG and "record 30" in str(e.value)
    rows[12] = rows[12][:8]  # a lower record that does not hold the key slot
    recs, rl = hm.records_of(rows)
    with pytest.raises(capi.B2SError) as e:
        capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, 4, dst)
    assert "record 12" in str(e.value)


def test_bad_value_null_words_and_decimals_are_named(capi):
    rng = np.random.default_rng(31)
    types = ["int"] + ["long"] * 12 + ["decimal"]
    rows = [hm.make_row(types, [int(rng.integers(0, 5))] + [int(x) for x in rng.integers(-99, 99, 12)] +
                        [int(rng.integers(-10**18, 10**18)) * 100]) for _ in range(60)]
    keys = hm.keys_of(types, [0])
    dst = np.zeros(1 << 16, np.uint8)
    # a null bit whose word (bytes 96..104) is past record 30's row, which still holds every slot the call reads
    count_far = [(pm.COUNT, pm.VAL_INT64, 16, 64 * 12)]
    short = list(rows)
    short[30] = short[30][:96]
    recs, rl = hm.records_of(short)
    with pytest.raises(capi.B2SError) as e:
        capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, count_far, 4, dst)
    assert e.value.code == capi.E_ARG and "record 30" in str(e.value) and "null word" in str(e.value)
    # a decimal(25) input whose size is 17 (record 20) or runs past its row (record 40)
    dsum = [(pm.SUM, pm.val_decimal(25, 0), 8 + 8 * 13, 13)]
    for at, bad in ((20, lambda s: (s >> 32) << 32 | 17), (40, lambda s: s + (1 << 40))):
        broken = list(rows)
        r = bytearray(broken[at])
        slot = int.from_bytes(r[112:120], "little")
        r[112:120] = bad(slot).to_bytes(8, "little")
        broken[at] = bytes(r)
        recs, rl = hm.records_of(broken)
        with pytest.raises(capi.B2SError) as e:
            capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, dsum, 4, dst)
        assert e.value.code == capi.E_ARG and "record %d" % at in str(e.value) and "decimal" in str(e.value)
    check(capi, rows, keys, count_far[:0] + dsum, 4)  # the rows as made are well-formed


def raw_call(capi, dev, recs, rl, keys, aggs, R, cap):
    """the C call itself (not the raising wrapper), packed or on device buffers -> (rc, *dst_total, *n_groups, .data)"""
    L = capi.load()
    nk, kt, ko, kl, kn = capi._key_arrays(keys)
    na, fn, vt, vo, vn = capi._partial_agg_arrays(aggs)
    doff, dlen, cks, st = capi._partition_out(R)
    total, ng = C.c_uint64(0), C.c_uint64(0)
    dst = np.zeros(max(cap, 1), np.uint8)
    tail = (nk, kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data, na, fn.ctypes.data, vt.ctypes.data,
            vo.ctypes.data, vn.ctypes.data)
    outs = (doff.ctypes.data, dlen.ctypes.data, C.byref(total), cks.ctypes.data, st.ctypes.data, C.byref(ng))
    if not dev:
        rc = L.b2s_aggregate_partition_compress_rows_hash_packed(1, 0, 0, 3, R, rl.size, recs.ctypes.data, recs.size,
                                                                 rl.ctypes.data, *tail, dst.ctypes.data, cap, *outs)
        return rc, total.value, ng.value, dst[:min(total.value, cap)].tobytes()
    d_rec, d_len, d_dst = capi.dev_alloc(recs.size), capi.dev_alloc(rl.size * 4), capi.dev_alloc(max(cap, 1))
    try:
        capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
        capi.dev_memcpy(d_len, rl.ctypes.data, rl.size * 4, 1)
        rc = L.b2s_aggregate_partition_compress_rows_hash_dev(0, 1, 0, 0, 3, R, rl.size, d_rec, recs.size, d_len,
                                                              *tail, d_dst, cap, *outs)
        if rc == 0 and total.value:
            capi.dev_memcpy(dst.ctypes.data, d_dst, total.value, 2)
    finally:
        for q in (d_rec, d_len, d_dst):
            capi.dev_free(q)
    return rc, total.value, ng.value, dst[:min(total.value, cap)].tobytes()


@pytest.mark.parametrize("dev", [False, True])
def test_short_destination_reports_the_exact_size_then_succeeds(capi, dev):
    rng = np.random.default_rng(4)
    rows, types = dataset(rng, 3000, ["string"], 200)
    keys, aggs = hm.keys_of(types, [0]), all_aggs(1)
    recs, rl = hm.records_of(rows)
    got, got_dst, _ = check(capi, rows, keys, aggs, 9)  # the exact arena, against the model
    need = got["total"]
    rc, total, _, _ = raw_call(capi, dev, recs, rl, keys, aggs, 9, 64)
    assert rc == capi.E_DST_TOO_SMALL and total == need
    rc, total, ng, data = raw_call(capi, dev, recs, rl, keys, aggs, 9, need)
    assert rc == 0 and total == need and ng == got["n_groups"] and data == got_dst[:need].tobytes()


def test_nan_and_infinite_inputs_to_the_double_sums(capi):
    """the sum chains over NaN payloads and infinities: a NaN result wherever the model's is one (IEEE leaves which
    NaN's payload a sum carries to the hardware), every other value and every other byte of the row exact"""
    rng = np.random.default_rng(17)
    rows, types = dataset(rng, 6000, ["int"], 30)
    keys = hm.keys_of(types, [0])
    nk = 1
    f = lambda fn, j: (fn, VT[j], 8 + 8 * (nk + j), nk + j)  # noqa: E731
    aggs = [f(pm.SUM, 9), f(pm.AVG, 9), f(pm.MIN, 9), f(pm.MAX, 9), f(pm.SUM, 5)]
    partial = pm.partial_rows(rows, keys, aggs)
    assert any(struct.unpack("<d", r[16:24])[0] != struct.unpack("<d", r[16:24])[0] for r in partial)
    recs, rl = hm.records_of(rows)
    dst = np.zeros(capi.partition_compress_bound(0, 0, 1, recs.size) + 64, np.uint8)
    got = capi.aggregate_partition_compress_rows_hash_packed(0, recs, rl, keys, aggs, 1, dst)  # codec NONE, R = 1
    want, _ = hm.records_of(partial)
    data = dst[:got["total"]].tobytes()
    assert got["n_groups"] == len(partial) and len(data) == want.size
    sums = [8 + 8 * f for f in (1, 2, 6)]  # the double sums' slots (SUM, AVG's sum, the finite SUM)
    at = 0
    for r in partial:
        g = data[at + 4:at + 4 + len(r)]
        at += 4 + len(r)
        for o in range(0, len(r), 8):
            a, b = struct.unpack("<d", g[o:o + 8])[0], struct.unpack("<d", r[o:o + 8])[0]
            if o in sums and b != b:
                assert a != a, o
            else:
                assert g[o:o + 8] == r[o:o + 8], o


def test_end_to_end_with_the_reduce_merge(capi):
    """M maps, then per reducer the reduce-side aggregation over the .data slices: the whole dataset's model"""
    rng = np.random.default_rng(8)
    kt = ["string", "int"]
    nk = 2
    pool_rows, types = dataset(rng, 6000, kt, 120)
    keys = hm.keys_of(types, [0, 1])
    slot = lambda j: 8 + 8 * (nk + j)  # noqa: E731
    f = lambda fn, j: (fn, VT[j], slot(j), nk + j)  # noqa: E731
    aggs = [f(pm.SUM, 3), f(pm.SUM, 6), f(pm.SUM, 7), (pm.COUNT, pm.VAL_NONE, 0, -1), f(pm.AVG, 6), f(pm.MIN, 2),
            f(pm.MAX, 7), f(pm.MAX, 5)]
    M, R = 3, 5
    maps = [pool_rows[m::M] for m in range(M)]
    datas = []
    for rows in maps:
        recs, rl = hm.records_of(rows)
        cap = capi.partition_compress_bound(1, 0, R, recs.size * 4 + 1 << 16) + (1 << 16)
        dst = np.zeros(cap, np.uint8)
        got = capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, R, dst, checksum_alg=3)
        datas.append((dst, got))
    okeys = pm.output_keys(keys)
    merge = pm.merge_aggs(keys, aggs)
    whole = {bytes(r) for r in pm.partial_rows(pool_rows, keys, aggs)}
    # the merged rows of every reducer: partial rows of maps merged by the reduce-side aggregation
    merged = []
    for p in range(R):
        blocks = [dst[int(g["dst_off"][p]):int(g["dst_off"][p] + g["dst_len"][p])].tobytes() for dst, g in datas]
        blocks = [b for b in blocks if b]
        if not blocks:
            continue
        src = np.frombuffer(b"".join(blocks), np.uint8).copy()
        off = np.cumsum([0] + [len(b) for b in blocks[:-1]]).astype(np.uint64)
        ln = np.array([len(b) for b in blocks], np.uint64)
        out = np.zeros(1 << 22, np.uint8)
        res = capi.decompress_aggregate_rows_keys_packed(1, src, off, ln, out, okeys, merge)
        buf = out[:res["total"]].tobytes()
        at = 0
        while at < len(buf):
            sz = int.from_bytes(buf[at:at + 4], "big")
            merged.append(buf[at + 4:at + 4 + sz])
            at += 4 + sz
    # the whole dataset's partial rows equal the merged ones except the double sum, which the reducer adds per map
    assert len(merged) == len(whole)
    nb = len(pm.buffers(aggs))
    dsum = [k for k, (op, _) in enumerate(pm.buffers(aggs)) if op == pm.SUM_F64]
    assert not dsum  # integer and decimal buffers only: exact in any grouping
    assert {bytes(r) for r in merged} == whole, nb


def reduce_merge(partials, keys, aggs):
    """the reduce side's aggregation model over partial rows in the order given -> {row bytes}"""
    import decimal_model as dm
    import rows_model as rm
    buf, _, _ = dm.model_aggregate_decimal([rm.stream(partials)], pm.output_keys(keys), pm.merge_aggs(keys, aggs))
    out, at = set(), 0
    while at < len(buf):
        sz = int.from_bytes(buf[at:at + 4], "big")
        out.add(bytes(buf[at + 4:at + 4 + sz]))
        at += 4 + sz
    return out


def test_end_to_end_double_sums_add_each_maps_partial_sum_in_map_order(capi):
    """the reducer merges this call's double sums (SUM and AVG of a double and of an int) map by map: the merged rows
    equal the reduce model over the model's partial rows of every map, in map order"""
    rng = np.random.default_rng(9)
    kt = ["string", "int"]
    nk = 2
    pool_rows, types = dataset(rng, 6000, kt, 80)
    keys = hm.keys_of(types, [0, 1])
    f = lambda fn, j: (fn, VT[j], 8 + 8 * (nk + j), nk + j)  # noqa: E731
    aggs = [f(pm.SUM, 5), f(pm.AVG, 5), f(pm.AVG, 2), f(pm.SUM, 4), f(pm.SUM, 3)]
    M, R = 4, 3
    maps = [pool_rows[m::M] for m in range(M)]
    datas = []
    for rows in maps:
        recs, rl = hm.records_of(rows)
        dst = np.zeros(capi.partition_compress_bound(1, 0, R, recs.size) + 64, np.uint8)
        datas.append((dst, capi.aggregate_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, R, dst,
                                                                              checksum_alg=3)))
    okeys, merge = pm.output_keys(keys), pm.merge_aggs(keys, aggs)
    got = set()
    for p in range(R):
        blocks = [d[int(g["dst_off"][p]):int(g["dst_off"][p] + g["dst_len"][p])].tobytes() for d, g in datas]
        blocks = [b for b in blocks if b]
        src = np.frombuffer(b"".join(blocks), np.uint8).copy()
        off = np.cumsum([0] + [len(b) for b in blocks[:-1]]).astype(np.uint64)
        ln = np.array([len(b) for b in blocks], np.uint64)
        out = np.zeros(1 << 22, np.uint8)
        res = capi.decompress_aggregate_rows_keys_packed(1, src, off, ln, out, okeys, merge)
        buf, at = out[:res["total"]].tobytes(), 0
        while at < len(buf):
            sz = int.from_bytes(buf[at:at + 4], "big")
            got.add(buf[at + 4:at + 4 + sz])
            at += 4 + sz
    assert got == reduce_merge([r for m in maps for r in pm.partial_rows(m, keys, aggs)], keys, aggs)


@pytest.mark.parametrize("cache", [0, 64 << 20])
def test_host_mirror_writer_and_aggregated_read(tmp_path, cache):
    """the serialized writer's aggregateRows (after hashRows, before the first insert; the uncached call even with the
    exchange cache on) and the reader's readAggregatedRowsKeys: per reducer the merged rows of the whole dataset"""
    import rows_model as rm
    host = pkg.host
    extra = {"spark.shuffle.s3.gpu.exchangeCacheBytes": cache} if cache else {}
    d = rm.mirror(tmp_path / "agg", "lz4", **extra)
    d_ref = rm.mirror(tmp_path / "ref", "lz4")
    rng = np.random.default_rng(12)
    kt = ["string", "int"]
    nk = 2
    pool_rows, types = dataset(rng, 4000, kt, 60)
    keys = hm.keys_of(types, [0, 1])
    f = lambda fn, j: (fn, VT[j], 8 + 8 * (nk + j), nk + j)  # noqa: E731
    aggs = [f(pm.SUM, 3), f(pm.SUM, 8), f(pm.AVG, 6), (pm.COUNT, pm.VAL_NONE, 0, -1), f(pm.MIN, 2), f(pm.MAX, 7)]
    M, R = 3, 4
    maps = [pool_rows[m::M] for m in range(M)]
    for m, rows in enumerate(maps):
        w = host.S3SerializedShuffleWriter(d, 0, m, R)
        with pytest.raises(Exception):
            w.aggregateRows(aggs)  # before hashRows
        w.hashRows(keys)
        w.aggregateRows(aggs)
        for row in rows:
            w.insertRecord(0, len(row).to_bytes(4, "big") + row)
        with pytest.raises(Exception):
            w.aggregateRows(aggs)  # after the first insert
        lens = w.commit()
        w.close()
        # the files are what the hash-mode writer makes of the model's partial rows
        w = host.S3SerializedShuffleWriter(d_ref, 0, m, R)
        w.hashRows(pm.output_keys(keys))
        for r in pm.partial_rows(rows, keys, aggs):
            w.insertRecord(0, len(r).to_bytes(4, "big") + r)
        assert list(w.commit()) == list(lens)
        w.close()
        for kind in ("data", "index", "checksum"):
            assert open(d.getPath(kind, 0, m), "rb").read() == open(d_ref.getPath(kind, 0, m), "rb").read()
    whole = {bytes(r) for r in pm.partial_rows(pool_rows, keys, aggs)}
    got = set()
    for red in range(R):
        rd = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        data, n, g = rd.readAggregatedRowsKeys(pm.output_keys(keys), pm.merge_aggs(keys, aggs))
        rd.close()
        at = 0
        while at < len(data):
            sz = int.from_bytes(data[at:at + 4], "big")
            got.add(bytes(data[at + 4:at + 4 + sz]))
            at += 4 + sz
    assert got == whole  # integer and decimal buffers: exact however the maps split the rows
    d.close()
    d_ref.close()


def test_host_mirror_writer_sizes_partial_rows_larger_than_the_input(tmp_path):
    """rows of a key alone, every key distinct, three count(*)s: the partial rows outgrow the input's bound, so commit
    retries with the exact size the call reports; the files are the hash-mode writer's over the model's partial rows"""
    import rows_model as rm
    host = pkg.host
    d, d_ref = rm.mirror(tmp_path / "agg", "lz4"), rm.mirror(tmp_path / "ref", "lz4")
    rows = [hm.make_row(["long"], [k]) for k in range(20000)]
    keys = hm.keys_of(["long"], [0])
    aggs = [(pm.COUNT, pm.VAL_NONE, 0, -1)] * 3
    partial = pm.partial_rows(rows, keys, aggs)
    assert sum(4 + len(r) for r in partial) > 2 * sum(4 + len(r) for r in rows)
    for dd, rs, ks, agg in ((d, rows, keys, aggs), (d_ref, partial, pm.output_keys(keys), None)):
        w = host.S3SerializedShuffleWriter(dd, 0, 0, 3)
        w.hashRows(ks)
        if agg:
            w.aggregateRows(agg)
        for r in rs:
            w.insertRecord(0, len(r).to_bytes(4, "big") + r)
        w.commit()
        w.close()
    for kind in ("data", "index", "checksum"):
        assert open(d.getPath(kind, 0, 0), "rb").read() == open(d_ref.getPath(kind, 0, 0), "rb").read()
    d.close()
    d_ref.close()
