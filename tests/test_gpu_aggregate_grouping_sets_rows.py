"""b2s_aggregate_grouping_sets_partition_compress_rows_hash_*: a map task's Expand over grouping sets and its partial
aggregation on the GPU.  Every output must be byte for byte what b2s_aggregate_partition_compress_rows_hash_packed
returns over the model's materialised Expand rows (tests/grouping_sets_model.py), and what the hash call returns for the
model's partial rows; end to end, the reduce side's merge over several maps' partial rows must equal a plain GROUP BY
of each set over the whole dataset."""
import functools
import struct

import numpy as np
import pytest

import grouping_sets_model as gm
import hash_model as hm
import partial_agg_model as pm
import spark_s3_shuffle_b200 as pkg
import test_gpu_aggregate_partition_rows as ta
from test_grouping_sets_model import decode
from test_gpu_sort_rows_order import col_value, comparator

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    c = pkg.capi
    c.init(1)
    return c


def outputs_equal(a, b, a_dst, b_dst):
    assert a["total"] == b["total"]
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a_dst[:a["total"]], b_dst[:b["total"]])


def run(capi, codec, recs, rl, keys, aggs, masks, R, cap, alg=3, lvl=0, dev=False):
    """the new call, packed or on device buffers -> (outputs, .data arena)"""
    dst = np.zeros(cap, np.uint8)
    if not dev:
        return capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(
            codec, recs, rl, keys, aggs, masks, R, dst, checksum_alg=alg, level=lvl), dst
    d_rec, d_len, d_dst = capi.dev_alloc(max(recs.size, 1)), capi.dev_alloc(max(rl.size * 4, 4)), capi.dev_alloc(cap)
    try:
        if recs.size:
            capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
            capi.dev_memcpy(d_len, rl.ctypes.data, rl.size * 4, 1)
        got = capi.aggregate_grouping_sets_partition_compress_rows_hash_dev(
            codec, d_rec, recs.size, d_len, rl.size, keys, aggs, masks, R, d_dst, cap, checksum_alg=alg, level=lvl)
        if got["total"]:
            capi.dev_memcpy(dst.ctypes.data, d_dst, got["total"], 2)
    finally:
        for p in (d_rec, d_len, d_dst):
            capi.dev_free(p)
    return got, dst


def check(capi, rows, keys, aggs, masks, R, codec=1, lvl=0, alg=3, dev=False):
    """the new call == the partial-aggregation call over the materialised Expand rows == the hash call over the model's
    partial rows"""
    xrows, xkeys, xaggs = gm.expand(rows, keys, aggs, masks)
    partial = pm.partial_rows(xrows, xkeys, xaggs)
    recs, rl = hm.records_of(rows)
    xrec, xrl = hm.records_of(xrows)
    prec, prl = hm.records_of(partial)
    cap = capi.partition_compress_bound(codec, 0, R, prec.size) + 64
    ref_dst, agg_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    ref = capi.partition_compress_rows_hash_packed(codec, prec, prl, pm.output_keys(xkeys), R, ref_dst,
                                                   checksum_alg=alg, level=lvl)
    agg = capi.aggregate_partition_compress_rows_hash_packed(codec, xrec, xrl, xkeys, xaggs, R, agg_dst,
                                                             checksum_alg=alg, level=lvl)
    got, got_dst = run(capi, codec, recs, rl, keys, aggs, masks, R, cap, alg, lvl, dev)
    assert got["n_groups"] == agg["n_groups"] == len(partial)
    outputs_equal(got, agg, got_dst, agg_dst)
    outputs_equal(got, ref, got_dst, ref_dst)
    return got, got_dst, partial


@pytest.mark.parametrize("codec,lvl", ta.CODECS)
@pytest.mark.parametrize("alg", [0, 1, 2, 3])
def test_every_codec_and_checksum(capi, codec, lvl, alg):
    rng = np.random.default_rng(100 + codec * 10 + alg)
    rows, types = ta.dataset(rng, 1200, ["string", "int"], 150)
    check(capi, rows, hm.keys_of(types, [0, 1]), ta.all_aggs(2), gm.rollup(2), 7, codec, lvl, alg)


@pytest.mark.parametrize("ktype", ["bool", "byte", "short", "int", "long", "float", "double", "string", "decimal"])
@pytest.mark.parametrize("nullable", [True, False])
def test_every_key_type(capi, ktype, nullable):
    """CUBE over the type and a string: wide decimals, strings, and float keys with -0.0 and NaN payloads"""
    rng = np.random.default_rng(len(ktype) * 1000 + ord(ktype[1]) * 4 + 2 * nullable)
    kt = [ktype, "string"]
    rows, types = ta.dataset(rng, 700, kt, 120, finite=False, null_keys=nullable)
    keys = hm.keys_of(types, range(len(kt)), nullable=nullable)
    for dev in (False, True):
        check(capi, rows, keys, ta.all_aggs(len(kt)), gm.cube(2), 13, dev=dev)


def test_every_aggregate_pair(capi):
    rng = np.random.default_rng(5)
    rows, types = ta.dataset(rng, 1500, ["int", "long"], 40)
    nk = 2
    f = lambda fn, j: (fn, ta.VT[j], 8 + 8 * (nk + j), nk + j)  # noqa: E731
    pairs = [f(pm.SUM, j) for j in range(9)] + [f(pm.COUNT, j) for j in range(10)] + [(pm.COUNT, pm.VAL_NONE, 0, -1)]
    pairs += [f(pm.AVG, j) for j in range(9)] + [f(pm.MIN, j) for j in (2, 3, 5, 6, 7, 8, 9)] + \
        [f(pm.MAX, j) for j in (2, 3, 5, 6, 7, 8, 9)]
    calls, cur = [], []
    for p in pairs:
        if len(pm.buffers(cur + [p])) > 16:
            calls.append(cur)
            cur = []
        cur.append(p)
    calls.append(cur)
    assert any(len(pm.buffers(c)) == 16 for c in calls)
    for c in calls:
        check(capi, rows, hm.keys_of(types, [0, 1]), c, gm.rollup(2), 5)


def test_rollup_over_eight_columns(capi):
    rng = np.random.default_rng(8)
    kt = ["string", "int", "long", "string", "short", "decimal", "double", "byte"]
    rows, types = ta.dataset(rng, 900, kt, 300)
    keys = hm.keys_of(types, range(8))
    check(capi, rows, keys, ta.all_aggs(8)[:6], gm.rollup(8), 11)
    check(capi, rows, keys, ta.all_aggs(8)[:6], gm.rollup(8), 3, dev=True)


@pytest.mark.parametrize("masks", [gm.cube(4), [0b0001, 0b0011, 0b1100, 0], [0b1111], [0], [0b0110, 0b1001]],
                         ids=["cube4", "explicit_with_empty", "one_full_set", "grand_total_only", "disjoint"])
@pytest.mark.parametrize("dev", [False, True])
def test_cube_and_explicit_sets(capi, masks, dev):
    rng = np.random.default_rng(len(masks) * 7 + masks[0])
    rows, types = ta.dataset(rng, 900, ["int", "string", "decimal", "float"], 200, finite=False)
    check(capi, rows, hm.keys_of(types, range(4)), ta.all_aggs(4), masks, 9, dev=dev)


@pytest.mark.parametrize("n", [0, 1, 20000])
def test_shapes(capi, n):
    rng = np.random.default_rng(n)
    rows, types = ta.dataset(rng, n, ["long", "int"], 50) if n else ([], ["long", "int"] + ta.VALUE_TYPES)
    keys = hm.keys_of(types, [0, 1])
    for aggs in (ta.all_aggs(2), []):
        check(capi, rows, keys, aggs, gm.rollup(2) if n < 20000 else gm.cube(2), 200)


def test_bad_records_are_named_by_input_index(capi):
    rng = np.random.default_rng(3)
    rows, types = ta.dataset(rng, 50, ["int"], 5)
    keys, aggs = hm.keys_of(types, [0]), ta.all_aggs(1)
    dst = np.zeros(1 << 16, np.uint8)
    rows = list(rows)
    rows[30] = rows[30][:16]  # holds the key slot, not the value slots
    for masks in (gm.rollup(1), [0]):
        recs, rl = hm.records_of(rows)
        with pytest.raises(capi.B2SError) as e:
            capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, masks, 4, dst)
        assert e.value.code == capi.E_ARG and "record 30 " in str(e.value) and "value slot" in str(e.value)
    rows[12] = rows[12][:8]  # a lower record that does not hold the key slot
    recs, rl = hm.records_of(rows)
    with pytest.raises(capi.B2SError) as e:
        capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, gm.rollup(1), 4, dst)
    assert e.value.code == capi.E_ARG and "record 12" in str(e.value)
    # a null word past the row, and decimal(25) inputs of size 17 or running past the row
    types = ["int"] + ["long"] * 12 + ["decimal"]
    rows = [hm.make_row(types, [int(rng.integers(0, 5))] + [int(x) for x in rng.integers(-99, 99, 12)] +
                        [int(rng.integers(-10**18, 10**18)) * 100]) for _ in range(60)]
    keys = hm.keys_of(types, [0])
    short = list(rows)
    short[30] = short[30][:96]
    recs, rl = hm.records_of(short)
    with pytest.raises(capi.B2SError) as e:
        capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(
            1, recs, rl, keys, [(pm.COUNT, pm.VAL_INT64, 16, 64 * 12)], gm.rollup(1), 4, dst)
    assert e.value.code == capi.E_ARG and "record 30 " in str(e.value) and "null word" in str(e.value)
    dsum = [(pm.SUM, pm.val_decimal(25, 0), 8 + 8 * 13, 13)]
    for at, bad in ((20, lambda s: (s >> 32) << 32 | 17), (40, lambda s: s + (1 << 40))):
        broken = list(rows)
        r = bytearray(broken[at])
        slot = int.from_bytes(r[112:120], "little")
        r[112:120] = bad(slot).to_bytes(8, "little")
        broken[at] = bytes(r)
        recs, rl = hm.records_of(broken)
        with pytest.raises(capi.B2SError) as e:
            capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(1, recs, rl, keys, dsum, gm.cube(1), 4,
                                                                            dst)
        assert e.value.code == capi.E_ARG and "record %d " % at in str(e.value) and "decimal" in str(e.value)
    check(capi, rows, keys, dsum, gm.cube(1), 4)  # the rows as made are well-formed


def raw_call(capi, dev, recs, rl, keys, aggs, masks, R, cap):
    """the C call itself (not the raising wrapper) -> (rc, *dst_total, *n_groups, .data)"""
    import ctypes as C
    L = capi.load()
    nk, kt, ko, kl, kn = capi._key_arrays(keys)
    na, fn, vt, vo, vn = capi._partial_agg_arrays(aggs)
    m = np.array(masks, np.uint32)
    doff, dlen, cks, st = capi._partition_out(R)
    total, ng = C.c_uint64(0), C.c_uint64(0)
    dst = np.zeros(max(cap, 1), np.uint8)
    tail = (nk, kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data, na, fn.ctypes.data, vt.ctypes.data,
            vo.ctypes.data, vn.ctypes.data, len(masks), m.ctypes.data)
    outs = (doff.ctypes.data, dlen.ctypes.data, C.byref(total), cks.ctypes.data, st.ctypes.data, C.byref(ng))
    if not dev:
        rc = L.b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed(
            1, 0, 0, 3, R, rl.size, recs.ctypes.data, recs.size, rl.ctypes.data, *tail, dst.ctypes.data, cap, *outs)
        return rc, total.value, ng.value, dst[:min(total.value, cap)].tobytes()
    d_rec, d_len, d_dst = capi.dev_alloc(recs.size), capi.dev_alloc(rl.size * 4), capi.dev_alloc(max(cap, 1))
    try:
        capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
        capi.dev_memcpy(d_len, rl.ctypes.data, rl.size * 4, 1)
        rc = L.b2s_aggregate_grouping_sets_partition_compress_rows_hash_dev(
            0, 1, 0, 0, 3, R, rl.size, d_rec, recs.size, d_len, *tail, d_dst, cap, *outs)
        if rc == 0 and total.value:
            capi.dev_memcpy(dst.ctypes.data, d_dst, total.value, 2)
    finally:
        for q in (d_rec, d_len, d_dst):
            capi.dev_free(q)
    return rc, total.value, ng.value, dst[:min(total.value, cap)].tobytes()


@pytest.mark.parametrize("dev", [False, True])
def test_short_destination_reports_the_exact_size_then_succeeds(capi, dev):
    rng = np.random.default_rng(4)
    rows, types = ta.dataset(rng, 1500, ["string", "int"], 200)
    keys, aggs, masks = hm.keys_of(types, [0, 1]), ta.all_aggs(2), gm.cube(2)
    recs, rl = hm.records_of(rows)
    got, got_dst, _ = check(capi, rows, keys, aggs, masks, 9)
    need = got["total"]
    rc, total, _, _ = raw_call(capi, dev, recs, rl, keys, aggs, masks, 9, 64)
    assert rc == capi.E_DST_TOO_SMALL and total == need
    rc, total, ng, data = raw_call(capi, dev, recs, rl, keys, aggs, masks, 9, need)
    assert rc == 0 and total == need and ng == got["n_groups"] and data == got_dst[:need].tobytes()
    t = capi.last_timing()
    assert 0 < t["dominant_ms"] <= t["kernel_ms"]


def merged_by_reducers(capi, datas, R, keys, aggs):
    """per reducer the reduce-side aggregation (b2s_decompress_aggregate_rows_keys_packed, keyed by the grouping columns
    and gid) over every map's slice -> {(grouping values, gid): buffer values}"""
    xkeys = gm.projected_keys(keys)
    got = {}
    for p in range(R):
        blocks = [d[int(g["dst_off"][p]):int(g["dst_off"][p] + g["dst_len"][p])].tobytes() for d, g in datas]
        blocks = [b for b in blocks if b]
        if not blocks:
            continue
        src = np.frombuffer(b"".join(blocks), np.uint8).copy()
        off = np.cumsum([0] + [len(b) for b in blocks[:-1]]).astype(np.uint64)
        ln = np.array([len(b) for b in blocks], np.uint64)
        out = np.zeros(1 << 22, np.uint8)
        res = capi.decompress_aggregate_rows_keys_packed(1, src, off, ln, out, pm.output_keys(xkeys),
                                                         pm.merge_aggs(xkeys, aggs))
        add_rows(got, out[:res["total"]].tobytes(), keys, aggs)
    return got


def add_rows(got, buf, keys, aggs):
    at = 0
    while at < len(buf):
        sz = int.from_bytes(buf[at:at + 4], "big")
        vals, g, bufs = decode(buf[at + 4:at + 4 + sz], keys, aggs)
        assert vals + (g,) not in got
        got[vals + (g,)] = bufs
        at += 4 + sz


def exact_aggs(nk):
    f = lambda fn, j: (fn, ta.VT[j], 8 + 8 * (nk + j), nk + j)  # noqa: E731
    return [f(pm.SUM, 3), f(pm.SUM, 6), f(pm.SUM, 7), (pm.COUNT, pm.VAL_NONE, 0, -1), f(pm.AVG, 6), f(pm.MIN, 2),
            f(pm.MAX, 7), f(pm.COUNT, 4)]


@pytest.mark.parametrize("masks", [gm.rollup(3), gm.cube(3), [0b001, 0b011, 0]], ids=["rollup", "cube", "sets"])
def test_end_to_end_with_the_reduce_merge(capi, masks):
    """M maps, then per reducer the reduce-side aggregation over the .data slices: a GROUP BY of each set"""
    rng = np.random.default_rng(len(masks))
    kt = ["string", "int", "long"]
    pool_rows, types = ta.dataset(rng, 4000, kt, 120)
    keys, aggs = hm.keys_of(types, [0, 1, 2]), exact_aggs(3)
    M, R = 3, 5
    datas = []
    for m in range(M):
        recs, rl = hm.records_of(pool_rows[m::M])
        dst = np.zeros(capi.partition_compress_bound(1, 0, R, recs.size * len(masks)) + (1 << 16), np.uint8)
        datas.append((dst, capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(
            1, recs, rl, keys, aggs, masks, R, dst, checksum_alg=3)))
    assert merged_by_reducers(capi, datas, R, keys, aggs) == gm.group_by_each_set(pool_rows, keys, aggs, masks)


def test_host_mirror_writer_and_aggregated_read(tmp_path):
    """the serialized writer's hashRows -> aggregateRows -> groupingSets, then readAggregatedRowsKeys: the files are the
    hash-mode writer's over the model's partial rows, and the merged rows a GROUP BY of each set"""
    import rows_model as rm
    host = pkg.host
    d, d_ref = rm.mirror(tmp_path / "agg", "lz4"), rm.mirror(tmp_path / "ref", "lz4")
    rng = np.random.default_rng(12)
    kt = ["string", "int"]
    pool_rows, types = ta.dataset(rng, 3000, kt, 60)
    keys, aggs, masks = hm.keys_of(types, [0, 1]), exact_aggs(2), gm.cube(2)
    xkeys = gm.projected_keys(keys)
    M, R = 3, 4
    for m in range(M):
        rows = pool_rows[m::M]
        w = host.S3SerializedShuffleWriter(d, 0, m, R)
        w.hashRows(keys)
        with pytest.raises(Exception):
            w.groupingSets(masks)  # before aggregateRows
        w.aggregateRows(aggs)
        w.groupingSets(masks)
        for row in rows:
            w.insertRecord(0, len(row).to_bytes(4, "big") + row)
        with pytest.raises(Exception):
            w.groupingSets(masks)  # after the first insert
        lens = w.commit()
        w.close()
        w = host.S3SerializedShuffleWriter(d_ref, 0, m, R)
        w.hashRows(pm.output_keys(xkeys))
        for r in gm.partial_rows(rows, keys, aggs, masks):
            w.insertRecord(0, len(r).to_bytes(4, "big") + r)
        assert list(w.commit()) == list(lens)
        w.close()
        for kind in ("data", "index", "checksum"):
            assert open(d.getPath(kind, 0, m), "rb").read() == open(d_ref.getPath(kind, 0, m), "rb").read()
    got = {}
    for red in range(R):
        rd = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        data, _, _ = rd.readAggregatedRowsKeys(pm.output_keys(xkeys), pm.merge_aggs(xkeys, aggs))
        rd.close()
        add_rows(got, data, keys, aggs)
    assert got == gm.group_by_each_set(pool_rows, keys, aggs, masks)
    d.close()
    d_ref.close()


def test_host_mirror_writer_retries_with_the_exact_size(tmp_path):
    """CUBE over four columns of distinct keys: 16 partial rows per input row outgrow the input's bound"""
    import rows_model as rm
    host = pkg.host
    d, d_ref = rm.mirror(tmp_path / "agg", "lz4"), rm.mirror(tmp_path / "ref", "lz4")
    types = ["long"] * 4
    rows = [hm.make_row(types, [k, k + 1, k + 2, k + 3]) for k in range(3000)]
    keys, aggs, masks = hm.keys_of(types, range(4)), [(pm.COUNT, pm.VAL_NONE, 0, -1)], gm.cube(4)
    partial = gm.partial_rows(rows, keys, aggs, masks)
    assert sum(4 + len(r) for r in partial) > 4 * sum(4 + len(r) for r in rows)
    w = host.S3SerializedShuffleWriter(d, 0, 0, 3)
    w.hashRows(keys)
    w.aggregateRows(aggs)
    w.groupingSets(masks)
    for r in rows:
        w.insertRecord(0, len(r).to_bytes(4, "big") + r)
    w.commit()
    w.close()
    w = host.S3SerializedShuffleWriter(d_ref, 0, 0, 3)
    w.hashRows(pm.output_keys(gm.projected_keys(keys)))
    for r in partial:
        w.insertRecord(0, len(r).to_bytes(4, "big") + r)
    w.commit()
    w.close()
    for kind in ("data", "index", "checksum"):
        assert open(d.getPath(kind, 0, 0), "rb").read() == open(d_ref.getPath(kind, 0, 0), "rb").read()
    d.close()
    d_ref.close()


def test_projected_arena_past_four_gib(capi):
    """CUBE over five key columns that all name one 64-byte string: 32 sets, 80 string copies per input row, so 600 k
    rows (under 60 MB) project to more than 4 GiB.  The four strings and the grand total give 4 * 31 + 1 groups."""
    n, L = 600_000, 64
    strings = [bytes([65 + s]) * L for s in range(4)]
    rng = np.random.default_rng(21)
    pick = rng.integers(0, 4, n)
    v = rng.integers(-2**40, 2**40, n)
    # rows: null word, the string's slot, a long; then the string
    rowb = 8 + 16 + L
    arr = np.zeros((n, rowb), np.uint8)
    arr[:, 8:16] = np.full(n, (24 << 32) | L, np.uint64).view(np.uint8).reshape(n, 8)
    arr[:, 16:24] = v.astype(np.int64).view(np.uint8).reshape(n, 8)
    arr[:, 24:] = np.frombuffer(b"".join(strings), np.uint8).reshape(4, L)[pick]
    recs = np.concatenate([np.tile(np.frombuffer(struct.pack(">i", rowb), np.uint8), (n, 1)), arr], axis=1).reshape(-1)
    rl = np.full(n, 4 + rowb, np.uint32)
    keys = [(hm.FIELD["string"][0], 8, 8, -1)] * 5
    aggs = [(pm.SUM, pm.VAL_INT64, 16, -1), (pm.COUNT, pm.VAL_NONE, 0, -1)]
    masks = gm.cube(5)
    first = [bytes(arr[int(np.argmax(pick == s))]) for s in range(4)]
    projected = sum(int((pick == s).sum()) * (4 + len(gm.project(first[s], keys, aggs, m)))
                    for s in range(4) for m in masks)
    assert recs.size < 1 << 30 and projected > 1 << 32
    # the expected partial rows: per set and string, the sum and count of its rows
    xrows, xkeys, xaggs = gm.expand(first, keys, aggs, masks)
    bufs = pm.buffers(xaggs)
    want = {}
    for j, x in enumerate(xrows):
        s, m = divmod(j, len(masks))
        sel = pick == s if m != len(masks) - 1 else np.ones(n, bool)
        want.setdefault(bytes(pm.emit(x, xkeys, bufs, [int(v[sel].sum()) % 2**64, int(sel.sum())])), None)
    okeys = pm.output_keys(xkeys)
    cmp = comparator(okeys)
    partial = sorted(want, key=functools.cmp_to_key(lambda a, b: cmp(tuple(col_value(a, k) for k in okeys),
                                                                     tuple(col_value(b, k) for k in okeys))))
    assert len(partial) == 4 * 31 + 1
    prec, prl = hm.records_of(partial)
    R = 16
    cap = capi.partition_compress_bound(1, 0, R, prec.size) + 64
    ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    ref = capi.partition_compress_rows_hash_packed(1, prec, prl, pm.output_keys(xkeys), R, ref_dst, checksum_alg=3)
    got = capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(1, recs, rl, keys, aggs, masks, R, got_dst,
                                                                          checksum_alg=3)
    assert got["n_groups"] == len(partial)
    outputs_equal(got, ref, got_dst, ref_dst)
    # a small call after it is still exact
    rows, types = ta.dataset(np.random.default_rng(1), 300, ["int"], 20)
    check(capi, rows, hm.keys_of(types, [0]), ta.all_aggs(1), gm.rollup(1), 4)
