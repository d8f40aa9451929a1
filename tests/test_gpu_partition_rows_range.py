"""b2s_partition_compress_rows_range_*: Spark's RangePartitioner ids of serialized UnsafeRows computed on the GPU from
the sort-key columns and the partitioner's bound rows, then the partition + compress step.  Every output must be byte
for byte what b2s_partition_compress_packed returns when fed the same records and the ids of the model
(tests/range_model.py: getPartition's two branches over the comparator model); with codec NONE every partition must
hold exactly the model's rows in input order, which pins every record's id."""
import ctypes as C
import functools
import struct

import numpy as np
import pytest

import range_model as rg
import rows_model as rm
import spark_s3_shuffle_b200 as pkg

pytestmark = pytest.mark.gpu

CODECS = [("none", 0, 0), ("lz4", 1, 0), ("snappy", 2, 0), ("zstd1", 3, 1), ("zstd3", 3, 3)]
RS = [1, 2, 129, 130, 2000]  # partitions: no bound, one, both of getPartition's branches, a large exchange
ALL = [rg.STRING, rg.KEY_INT16, rg.KEY_FLOAT64, rg.DECIMAL, rg.KEY_INT8, rg.KEY_FLOAT32, rg.KEY_INT32, rg.KEY_INT64,
       rg.KEY_BYTES]


def wide_rows(rng, n):
    """(string, int, long) rows with many distinct keys: as many bounds as asked for"""
    keys = rg.layout([rg.STRING, rg.KEY_INT32, rg.KEY_INT64])
    rows = [rg.make_row(rng, keys, [None if rng.random() < 0.03 else bytes(rng.integers(97, 123, int(rng.integers(3, 30)),
                                                                                           dtype=np.uint8)),
                                    int(rng.integers(-2**31, 2**31)) if rng.random() > 0.05 else None,
                                    int(rng.integers(-2**62, 2**62))]) for _ in range(n)]
    return rows, keys


def shapes(rng, n):
    """(name, rows, keys) per key shape: one INT32, one INT64, one string, every type with random flags and nulls"""
    rows, keys = wide_rows(rng, n)
    out = [("int", rows, [keys[1]]), ("long", rows, [keys[2][:3] + (-1,)]), ("string", rows, [keys[0]])]
    k = rg.layout(ALL, [rg.FLAGS[int(rng.integers(4))] for _ in ALL], byte_len=8)
    out.append(("every", rg.rand_rows(rng, n, k), k))
    return out


_CASES = {}


def case(name, R, n=1500):
    """(records, rec_len, keys, framed bounds, model ids) of a shape at R partitions, computed once per module"""
    if (name, R, n) not in _CASES:
        rng = np.random.default_rng(R * 7 + n)
        rows, keys = {s[0]: s[1:] for s in shapes(rng, n)}[name]
        bounds = rg.draw_bounds(rng, rows, keys, R)
        recs, rl = rg.records_of(rows)
        _CASES[(name, R, n)] = (recs, rl, keys, [rg.framed(b) for b in bounds], rg.model_ids(rows, keys, bounds))
    return _CASES[(name, R, n)]


def both(capi, codec, lvl, alg, recs, rl, keys, bounds, ids):
    R = len(bounds) + 1
    cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
    ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    ref = capi.partition_compress_packed(codec, recs, rl, ids, R, ref_dst, checksum_alg=alg, level=lvl)
    got = capi.partition_compress_rows_range_packed(codec, recs, rl, keys, bounds, got_dst, checksum_alg=alg,
                                                    level=lvl)
    return ref, got, ref_dst, got_dst


def same(ref, got, ref_dst, got_dst):
    assert got["total"] == ref["total"]
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert (got[k] == ref[k]).all(), k
    assert (got_dst[:got["total"]] == ref_dst[:ref["total"]]).all()


@pytest.mark.parametrize("alg", rm.CHECKSUMS)
@pytest.mark.parametrize("codec_name,codec,lvl", CODECS)
def test_parity_with_partition_compress_of_the_model_ids(capi, codec_name, codec, lvl, alg):
    for name in ("int", "long", "string", "every"):
        for R in (1, 2, 130, 2000):
            recs, rl, keys, bounds, ids = case(name, R)
            same(*both(capi, codec, lvl, alg, recs, rl, keys, bounds, ids))
    recs, rl = rg.records_of([])
    _, _, keys, bounds, _ = case("every", 130)
    ref, got, ref_dst, got_dst = both(capi, codec, lvl, alg, recs, rl, keys, bounds, np.zeros(0, np.uint32))
    same(ref, got, ref_dst, got_dst)
    assert got["total"] == 0 and (got["dst_len"] == 0).all()


def partitions_are_the_models(capi, recs, rl, keys, bounds, ids, alg=3):
    """codec NONE: partition p of the arena is the records of id p in input order"""
    dst = np.zeros(max(recs.size, 1), np.uint8)
    got = capi.partition_compress_rows_range_packed(0, recs, rl, keys, bounds, dst, checksum_alg=alg)
    assert got["total"] == recs.size
    start = np.concatenate([[0], np.cumsum(rl.astype(np.int64))]).astype(np.int64)
    for p in np.unique(ids):
        want = b"".join(recs[start[i]:start[i + 1]].tobytes() for i in np.nonzero(ids == p)[0])
        o, ln = int(got["dst_off"][p]), int(got["dst_len"][p])
        assert dst[o:o + ln].tobytes() == want
    assert int(got["dst_len"].sum()) == recs.size
    return got


@pytest.mark.parametrize("R", RS)
def test_bound_counts_cover_both_branches(capi, R):
    for name in ("long", "string"):
        recs, rl, keys, bounds, ids = case(name, R, 3000)
        assert len(bounds) == R - 1
        partitions_are_the_models(capi, recs, rl, keys, bounds, ids)
        t = capi.last_timing()
        assert t["dominant_launches"] == 1 + min(R - 1, 2) and t["dominant_ms"] > 0


def run_dev(capi, codec, lvl, alg, recs, rl, keys, bounds):
    R = len(bounds) + 1
    cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
    d_rec, d_len, d_dst = capi.dev_alloc(max(recs.size, 1)), capi.dev_alloc(max(rl.nbytes, 4)), capi.dev_alloc(cap)
    try:
        if recs.size:
            capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
            capi.dev_memcpy(d_len, rl.ctypes.data, rl.nbytes, 1)
        r = capi.partition_compress_rows_range_dev(codec, d_rec, recs.size, d_len, rl.size, keys, bounds, d_dst, cap,
                                                   checksum_alg=alg, level=lvl)
        out = np.zeros(max(r["total"], 1), np.uint8)
        if r["total"]:
            capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        return r, out
    finally:
        for p in (d_rec, d_len, d_dst):
            capi.dev_free(p)


@pytest.mark.parametrize("codec_name,codec,lvl", CODECS)
def test_dev_equals_packed(capi, codec_name, codec, lvl):
    for name in ("int", "string", "every"):
        for R in (1, 130, 2000):
            recs, rl, keys, bounds, _ = case(name, R)
            cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
            dst = np.zeros(cap, np.uint8)
            ref = capi.partition_compress_rows_range_packed(codec, recs, rl, keys, bounds, dst, checksum_alg=3,
                                                            level=lvl)
            got, out = run_dev(capi, codec, lvl, 3, recs, rl, keys, bounds)
            same(ref, got, dst, out)
    t = capi.last_timing()
    assert t["dominant_launches"] == 3 and t["dominant_ms"] > 0 and t["h2d_ms"] == 0


def test_ties_long_prefixes_and_huge_strings(capi):
    """records equal to bounds; strings sharing 20 to 60 bytes with a bound, so the id step compares further windows;
    a few 1 MiB strings; under ASC and DESC"""
    rng = np.random.default_rng(5)
    for flags in (0, rg.DESC, rg.DESC | rg.NULLS_LAST):
        keys = rg.layout([rg.STRING, rg.KEY_INT32], [flags, rg.NULLS_LAST])
        stem = b"Books/Fiction/Classics/Europe#"  # 30 bytes: past the first window
        vals = []
        for i in range(3000):
            s = stem[:int(rng.integers(18, 31))] + bytes(rng.integers(0, 3, int(rng.integers(0, 40)), dtype=np.uint8))
            vals.append([None if i % 97 == 0 else s, None if i % 13 == 0 else int(rng.integers(0, 4))])
        for i in (7, 1500, 2999):
            vals[i] = [stem + bytes(rng.integers(0, 3, (1 << 20) + i % 5, dtype=np.uint8)), 1]
        rows = [rg.make_row(rng, keys, v) for v in vals]
        for R in (7, 200):
            bounds = rg.draw_bounds(rng, rows, keys, R, sample=800)
            recs, rl = rg.records_of(rows)
            ids = rg.model_ids(rows, keys, bounds)
            fb = [rg.framed(b) for b in bounds]
            partitions_are_the_models(capi, recs, rl, keys, fb, ids)
            same(*both(capi, 1, 0, 3, recs, rl, keys, fb, ids))
            # every bound is itself a record: equal keys go to the bound's partition
            bk = rg.bound_keys(keys)
            brows = [rg.make_row(rng, keys, [rg.col_value(b, c) for c in bk]) for b in bounds]
            brecs, brl = rg.records_of(brows)
            bids = rg.model_ids(brows, keys, bounds)
            assert list(bids) == list(range(len(bounds)))
            partitions_are_the_models(capi, brecs, brl, keys, fb, bids)


def raw_call(capi, recs, rl, keys, bounds, codec=1):
    L = capi.load()
    nk, kt, ko, kl, kn = capi._key_arrays(keys)
    nb, bb, bbytes, bl = capi._bound_arrays(bounds)
    R = nb + 1
    doff, dlen, cks = np.zeros(R, np.uint64), np.zeros(R, np.uint64), np.zeros(R, np.uint64)
    st = np.zeros(R, np.int32)
    dst = np.zeros(capi.partition_compress_bound(codec, 0, R, recs.size) + 64, np.uint8)
    total = C.c_uint64(7)
    rc = L.b2s_partition_compress_rows_range_packed(
        codec, 0, 0, 3, rl.size, recs.ctypes.data if recs.size else None, recs.size, rl.ctypes.data, nk,
        kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data, nb, bb.ctypes.data, bbytes, bl.ctypes.data,
        dst.ctypes.data, dst.size, doff.ctypes.data, dlen.ctypes.data, C.byref(total), cks.ctypes.data,
        st.ctypes.data)
    return rc, total.value, L.b2s_last_error().decode()


KEYS = rg.layout([rg.KEY_INT32, rg.STRING, rg.DECIMAL, rg.KEY_INT64])  # slots 8, 24, 40, 56; null bits 1..4


def good_rows(n=400):
    rng = np.random.default_rng(1)
    return [rg.make_row(rng, KEYS, [i, bytes(rng.integers(0, 256, i % 30, dtype=np.uint8)),
                                    int(rng.integers(-2**62, 2**62)) << (i % 40), None]) for i in range(n)]


def bad_framed(good, kind, slots, size_name="rec"):
    """a framed row the call must reject: slots = (string slot, decimal slot, last slot) of its layout"""
    s_str, s_dec, s_last = slots
    if kind == "short":
        return b"\x00\x00\x01"
    if kind == "prefix":
        return (len(good) + 1).to_bytes(4, "big") + good
    if kind == "key":
        return rg.framed(good[:s_last])  # ends before the last slot
    r = bytearray(good)
    if kind == "string":
        r[s_str:s_str + 8] = ((len(good) - 2) << 32 | 6).to_bytes(8, "little")
    elif kind == "decimal0":
        r[s_dec:s_dec + 8] = (int.from_bytes(r[s_dec:s_dec + 8], "little") & ~0xFFFFFFFF).to_bytes(8, "little")
    elif kind == "decimal17":
        r[s_dec:s_dec + 8] = ((s_last + 8) << 32 | 17).to_bytes(8, "little")
    elif kind == "decimal_past":
        r[s_dec:s_dec + 8] = ((len(good) - 1) << 32 | 2).to_bytes(8, "little")
    return rg.framed(bytes(r))


BAD = [("short", "below 4"), ("prefix", "size prefix"), ("key", "key slot"), ("string", "string key"),
       ("decimal0", "decimal key"), ("decimal17", "decimal key"), ("decimal_past", "decimal key")]


@pytest.mark.parametrize("kind,why", BAD)
def test_bad_bounds_are_rejected_naming_the_lowest(capi, kind, why):
    rows = good_rows()
    recs, rl = rg.records_of(rows)
    bounds = [rg.framed(rg.project(rows[i], KEYS)) for i in range(5, 400, 10)]  # increasing by the INT32 column
    for at in (0, 17, len(bounds) - 1):
        bb = list(bounds)
        bb[at] = bad_framed(rg.project(rows[5 + 10 * at], KEYS), kind, (16, 24, 32))
        if at + 3 < len(bb):
            bb[at + 3] = bad_framed(rg.project(rows[0], KEYS), "prefix", (16, 24, 32))
            bb[at + 5] = bb[at + 4]  # an order error after it is not named either
        rc, total, err = raw_call(capi, recs, rl, KEYS, bb)
        assert rc == capi.E_ARG and total == 0
        assert ("bound %d " % at) in err and why in err, err
        # a bad record as well: the bound is named
        r2 = list(rows)
        r2[0] = r2[0][:20]
        rc, total, err = raw_call(capi, *rg.records_of(r2), KEYS, bb)
        assert rc == capi.E_ARG and ("bound %d " % at) in err, err
    # an order error before a malformed bound is the lowest
    bb = list(bounds)
    bb[3], bb[4] = bb[4], bb[3]
    bb[9] = bad_framed(rg.project(rows[0], KEYS), kind, (16, 24, 32))
    rc, total, err = raw_call(capi, recs, rl, KEYS, bb)
    assert rc == capi.E_ARG and "bound 4 " in err and "not above" in err, err


F64 = lambda x: struct.pack("<d", x)  # noqa: E731


@pytest.mark.parametrize("keys,vals,at", [
    (rg.layout([rg.KEY_INT64]), [1, 5, 5, 9], 2),                           # equal
    (rg.layout([rg.KEY_INT64]), [1, 9, 5, 12], 2),                          # swapped
    (rg.layout([rg.KEY_INT64], [rg.DESC]), [9, 5, 6], 2),                   # ascending under DESC
    (rg.layout([rg.KEY_FLOAT64]), [F64(-5.0), F64(-0.0), F64(0.0), F64(3.0)], 2),  # equal only once normalised
    (rg.layout([rg.KEY_FLOAT64]), [F64(1.0), F64(float("nan")), struct.pack("<Q", 0xFFF0000000000001)], 2),
    (rg.layout([rg.KEY_FLOAT64]), [None, None, F64(1.0)], 1),               # two nulls
    (rg.layout([rg.STRING], [rg.DESC]), [b"b" * 40 + b"z", b"b" * 40 + b"z", b"a"], 1),  # equal past the first window
    (rg.layout([rg.STRING]), [b"b" * 40 + b"z", b"b" * 40 + b"y"], 1)])     # below past the first window
def test_bounds_not_strictly_increasing_are_rejected(capi, keys, vals, at):
    rng = np.random.default_rng(3)
    bounds = [rg.framed(rg.project(rg.make_row(rng, keys, [v]), keys)) for v in vals]
    rows = [rg.make_row(rng, keys, [vals[-1]])] * 5
    rc, total, err = raw_call(capi, *rg.records_of(rows), keys, bounds)
    assert rc == capi.E_ARG and total == 0
    assert ("bound %d is not above" % at) in err, err
    rc, total, err = raw_call(capi, *rg.records_of([]), keys, bounds)  # without records too
    assert rc == capi.E_ARG and ("bound %d is not above" % at) in err, err
    good = sorted(set(range(len(vals))) - {at})  # without the offending bound the call succeeds
    rc, _, err = raw_call(capi, *rg.records_of(rows), keys, [bounds[i] for i in good])
    assert rc == 0, err


@pytest.mark.parametrize("kind,why", [("short", "rec_len is below 4"), ("prefix", "size prefix")] + BAD[2:])
def test_bad_records_are_rejected_naming_the_lowest(capi, kind, why):
    rows = good_rows()
    recs = [rg.framed(r) for r in rows]
    bounds = [rg.framed(rg.project(rows[i], KEYS)) for i in (50, 200, 350)]
    for at in (0, 137, 399):
        rr = list(recs)
        rr[at] = bad_framed(rows[at], kind, (24, 40, 56))
        if at + 50 < len(rr):
            rr[at + 50] = bad_framed(rows[at + 50], "prefix", (24, 40, 56))
        buf = np.frombuffer(b"".join(rr), np.uint8).copy()
        rc, total, err = raw_call(capi, buf, np.array([len(r) for r in rr], np.uint32), KEYS, bounds)
        assert rc == capi.E_ARG and total == 0
        assert ("record %d " % at) in err and why in err, err


def test_dst_too_small_matches_partition_compress(capi):
    recs, rl, keys, bounds, ids = case("every", 130)
    R = len(bounds) + 1
    L = capi.load()
    nk, kt, ko, kl, kn = capi._key_arrays(keys)
    nb, bb, bbytes, bl = capi._bound_arrays(bounds)
    for codec in (0, 1):
        res = []
        for ranged in (False, True):
            doff, dlen, cks = np.zeros(R, np.uint64), np.zeros(R, np.uint64), np.zeros(R, np.uint64)
            st = np.zeros(R, np.int32)
            dst = np.zeros(recs.size // 2, np.uint8)
            total = C.c_uint64(0)
            tail = (dst.ctypes.data, dst.size, doff.ctypes.data, dlen.ctypes.data, C.byref(total), cks.ctypes.data,
                    st.ctypes.data)
            if ranged:
                rc = L.b2s_partition_compress_rows_range_packed(
                    codec, 0, 0, 3, rl.size, recs.ctypes.data, recs.size, rl.ctypes.data, nk, kt.ctypes.data,
                    ko.ctypes.data, kl.ctypes.data, kn.ctypes.data, nb, bb.ctypes.data, bbytes, bl.ctypes.data, *tail)
            else:
                rc = L.b2s_partition_compress_packed(codec, 0, 0, 3, R, rl.size, recs.ctypes.data, recs.size,
                                                     rl.ctypes.data, ids.ctypes.data, *tail)
            res.append((rc, total.value, doff.copy(), dlen.copy(), st.copy(), dst.copy()))
        assert res[0][0] == res[1][0] == capi.E_DST_TOO_SMALL
        assert res[0][1] == res[1][1]
        for a, b in zip(res[0][2:], res[1][2:]):
            assert (a == b).all()


def test_end_to_end_global_order_by(capi):
    """ORDER BY (string DESC, long NULLS LAST, double) over M maps: range-partitioned by bounds drawn from a sample
    of every map, each reducer's blocks row-sorted by the same key; reducers 0..R-1 concatenated are the stable sort of
    all rows, byte for byte"""
    rng = np.random.default_rng(11)
    keys = rg.layout([rg.STRING, rg.KEY_INT64, rg.KEY_FLOAT64], [rg.DESC, rg.NULLS_LAST, 0])
    M, R = 4, 13
    names = [b"", b"a", b"spark", b"\xff\x80x", b"shuffle-partition-0123456789", b"shuffle-partition-0123456789!"]
    maps = []
    for m in range(M):
        maps.append([rg.make_row(rng, keys, [None if rng.random() < 0.05 else names[int(rng.integers(len(names)))],
                                             None if rng.random() < 0.05 else int(rng.integers(-50, 50)),
                                             F64(float(rng.integers(-3, 3)) * 0.5)]) for _ in range(2500)])
    every = [r for rows in maps for r in rows]
    bounds = [rg.framed(b) for b in rg.draw_bounds(rng, every, keys, R, sample=2000)]
    assert len(bounds) == R - 1
    outs = []
    for rows in maps:
        recs, rl = rg.records_of(rows)
        dst = np.zeros(capi.partition_compress_bound(1, 0, R, recs.size) + 64, np.uint8)
        outs.append((dst, capi.partition_compress_rows_range_packed(1, recs, rl, keys, bounds, dst, checksum_alg=3)))
    got = b""
    for red in range(R):
        blocks = [(dst[int(r["dst_off"][red]):int(r["dst_off"][red] + r["dst_len"][red])], int(r["checksums"][red]))
                  for dst, r in outs if r["dst_len"][red]]
        if not blocks:
            continue
        src = np.concatenate([b for b, _ in blocks])
        ln = np.array([b.size for b, _ in blocks], np.uint64)
        off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
        out = np.zeros(sum(len(r) + 4 for r in every), np.uint8)
        res = capi.decompress_sort_rows_keys_packed(1, src, off, ln, out, keys, checksum_alg=3,
                                                    slice_base=np.arange(len(blocks) + 1), slice_len=ln,
                                                    slice_checksum=[c for _, c in blocks])
        got += out[:res["total"]].tobytes()
    cmp = rg.comparator(keys)
    kv = [rg.key_of(r, keys) for r in every]
    order = sorted(range(len(every)), key=functools.cmp_to_key(lambda i, j: cmp(kv[i], kv[j])))
    assert got == b"".join(rg.framed(every[i]) for i in order)


def test_host_mirror_range_mode_files_identical_and_readable(tmp_path):
    recs, rl, keys, bounds, ids = case("every", 130)
    R = len(bounds) + 1
    start = np.concatenate([[0], np.cumsum(rl.astype(np.int64))]).astype(np.int64)
    records = [recs[start[i]:start[i + 1]].tobytes() for i in range(rl.size)]
    host = pkg.host
    d_range, d_ids = rm.mirror(tmp_path / "range", "lz4"), rm.mirror(tmp_path / "ids", "lz4")
    w = host.S3SerializedShuffleWriter(d_range, 0, 0, R)
    w.rangeRows(keys, bounds)
    for r in records:
        w.insertRecord(0, r)
    lens_range = w.commit()
    w.close()
    w = host.S3SerializedShuffleWriter(d_ids, 0, 0, R)
    for r, p in zip(records, ids):
        w.insertRecord(int(p), r)
    lens_ids = w.commit()
    w.close()
    assert list(lens_range) == list(lens_ids)
    for kind in ("data", "index", "checksum"):
        assert open(d_range.getPath(kind, 0, 0), "rb").read() == open(d_ids.getPath(kind, 0, 0), "rb").read()
    for red in (0, 7, R - 1):
        rd = host.S3ShuffleReader(d_range, 0, [0], red, red + 1)
        got = b"".join(b for _, b in rd.read())
        rd.close()
        assert got == b"".join(r for r, p in zip(records, ids) if p == red)
    w = host.S3SerializedShuffleWriter(d_ids, 0, 1, R + 1)  # n_bounds + 1 must be num_partitions
    with pytest.raises(Exception):
        w.rangeRows(keys, bounds)
    w.close()
