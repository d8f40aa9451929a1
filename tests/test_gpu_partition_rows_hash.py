"""b2s_partition_compress_rows_hash_*: Spark's HashPartitioning ids of serialized UnsafeRows computed on the GPU, then
the partition + compress step.  Every output must be byte for byte what b2s_partition_compress_packed returns when fed
the same records and the ids of the Murmur3 model (tests/hash_model.py, pinned to Spark's published vectors); with
codec NONE every partition must hold exactly the model's rows in input order, which pins every record's id."""
import ctypes as C

import numpy as np
import pytest

import hash_model as hm
import rows_model as rm
import spark_s3_shuffle_b200 as pkg

pytestmark = pytest.mark.gpu

CODECS = [("lz4", 1, 0), ("snappy", 2, 0), ("zstd1", 3, 1), ("zstd3", 3, 3)]
RS = [1, 2, 7, 200, 2000, 65537]


def shapes(rng, n):
    """(rows, keys) per key shape: one INT32, one INT64, one string, and the composite of every type with nulls"""
    out = []
    ti = ["long", "int", "string"]
    rows = [hm.make_row(ti, [int(rng.integers(0, 1 << 40)), int(rng.integers(-2**31, 2**31)) if rng.random() > 0.05
                             else None, bytes(rng.integers(0, 256, int(rng.integers(0, 60)), dtype=np.uint8))])
            for _ in range(n)]
    out.append((rows, hm.keys_of(ti, [1])))
    out.append((rows, hm.keys_of(ti, [0], nullable=False)))
    out.append((rows, hm.keys_of(ti, [2])))
    out.append((hm.random_rows(rng, n), hm.keys_of(hm.COMPOSITE, range(8))))
    return out


def both(capi, codec, lvl, alg, rows, keys, R):
    recs, rl = hm.records_of(rows)
    ids = hm.record_ids_np(recs, rl, keys, R)
    cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
    ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    ref = capi.partition_compress_packed(codec, recs, rl, ids, R, ref_dst, checksum_alg=alg, level=lvl)
    got = capi.partition_compress_rows_hash_packed(codec, recs, rl, keys, R, got_dst, checksum_alg=alg, level=lvl)
    return recs, rl, ids, ref, got, ref_dst, got_dst


def same(ref, got, ref_dst, got_dst):
    assert got["total"] == ref["total"]
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert (got[k] == ref[k]).all(), k
    assert (got_dst[:got["total"]] == ref_dst[:ref["total"]]).all()


@pytest.mark.parametrize("alg", rm.CHECKSUMS)
@pytest.mark.parametrize("codec_name,codec,lvl", CODECS)
def test_parity_with_partition_compress_of_the_model_ids(capi, codec_name, codec, lvl, alg):
    rng = np.random.default_rng(codec * 10 + lvl + alg)
    for rows, keys in shapes(rng, 1500):
        for R in RS:
            _, _, _, ref, got, ref_dst, got_dst = both(capi, codec, lvl, alg, rows, keys, R)
            same(ref, got, ref_dst, got_dst)
    _, _, _, ref, got, ref_dst, got_dst = both(capi, codec, lvl, alg, [], hm.keys_of(["int"], [0]), 7)
    same(ref, got, ref_dst, got_dst)
    assert got["total"] == 0 and (got["dst_len"] == 0).all()


def partitions_are_the_models(capi, rows, keys, R, alg=3):
    """codec NONE: partition p of the arena is the records of id p in input order"""
    recs, rl = hm.records_of(rows)
    ids = hm.record_ids_np(recs, rl, keys, R)
    dst = np.zeros(max(recs.size, 1), np.uint8)
    got = capi.partition_compress_rows_hash_packed(0, recs, rl, keys, R, dst, checksum_alg=alg)
    assert got["total"] == recs.size
    start = np.concatenate([[0], np.cumsum(rl.astype(np.int64))]).astype(np.int64)
    for p in np.unique(ids):
        want = b"".join(recs[start[i]:start[i + 1]].tobytes() for i in np.nonzero(ids == p)[0])
        o, ln = int(got["dst_off"][p]), int(got["dst_len"][p])
        assert dst[o:o + ln].tobytes() == want
    assert int(got["dst_len"].sum()) == recs.size
    return recs, rl, ids, got, dst


@pytest.mark.parametrize("R", RS)
def test_codec_none_partitions_hold_the_models_rows_in_input_order(capi, R):
    rng = np.random.default_rng(R)
    for rows, keys in shapes(rng, 3000):
        partitions_are_the_models(capi, rows, keys, R)
    # the scalar model over a sample agrees with the ids the partitions imply
    rows = hm.random_rows(rng, 400)
    keys = hm.keys_of(hm.COMPOSITE, range(8))
    recs, rl, ids, _, _ = partitions_are_the_models(capi, rows, keys, R)
    assert (ids == hm.ids_scalar(rows, keys, R)).all()


def run_dev(capi, codec, lvl, alg, recs, rl, keys, R):
    cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
    d_rec, d_len, d_dst = capi.dev_alloc(max(recs.size, 1)), capi.dev_alloc(max(rl.nbytes, 4)), capi.dev_alloc(cap)
    try:
        if recs.size:
            capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
            capi.dev_memcpy(d_len, rl.ctypes.data, rl.nbytes, 1)
        r = capi.partition_compress_rows_hash_dev(codec, d_rec, recs.size, d_len, rl.size, keys, R, d_dst, cap,
                                                  checksum_alg=alg, level=lvl)
        out = np.zeros(max(r["total"], 1), np.uint8)
        if r["total"]:
            capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        return r, out
    finally:
        for p in (d_rec, d_len, d_dst):
            capi.dev_free(p)


@pytest.mark.parametrize("codec_name,codec,lvl", [("none", 0, 0)] + CODECS)
def test_dev_equals_packed(capi, codec_name, codec, lvl):
    rng = np.random.default_rng(40 + codec + lvl)
    for rows, keys in shapes(rng, 2000):
        for R in (1, 200, 65537):
            recs, rl = hm.records_of(rows)
            cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
            dst = np.zeros(cap, np.uint8)
            ref = capi.partition_compress_rows_hash_packed(codec, recs, rl, keys, R, dst, checksum_alg=3, level=lvl)
            got, out = run_dev(capi, codec, lvl, 3, recs, rl, keys, R)
            same(ref, got, dst, out)
    t = capi.last_timing()
    assert t["dominant_launches"] == 1 and t["dominant_ms"] > 0


def test_long_strings(capi):
    """strings of 0 B to 4 KiB, and a few rows holding 1 MiB strings, hashed 16 bytes per load"""
    rng = np.random.default_rng(9)
    types = ["string", "int", "string"]
    rows = []
    for i in range(3000):
        ln = int(rng.integers(0, 4097)) if i % 10 else i % 40
        s = bytes(rng.integers(0, 256, ln, dtype=np.uint8))
        rows.append(hm.make_row(types, [s, i, None if i % 7 == 0 else s[: i % 23]]))
    for i in (5, 1000, 2999):
        rows[i] = hm.make_row(types, [bytes(rng.integers(0, 256, (1 << 20) + i % 4, dtype=np.uint8)), i, b"x"])
    keys = hm.keys_of(types, [0, 1, 2])
    for R in (7, 2000):
        partitions_are_the_models(capi, rows, keys, R)
        _, _, _, ref, got, ref_dst, got_dst = both(capi, 1, 0, 3, rows, keys, R)
        same(ref, got, ref_dst, got_dst)


def raw_call(capi, recs, rl, keys, R=7, codec=1):
    L = capi.load()
    nk, kt, ko, kl, kn = capi._key_arrays(keys)
    doff, dlen, cks = np.zeros(R, np.uint64), np.zeros(R, np.uint64), np.zeros(R, np.uint64)
    st = np.zeros(R, np.int32)
    dst = np.zeros(capi.partition_compress_bound(codec, 0, R, recs.size) + 64, np.uint8)
    total = C.c_uint64(7)
    rc = L.b2s_partition_compress_rows_hash_packed(
        codec, 0, 0, 3, R, rl.size, recs.ctypes.data if recs.size else None, recs.size, rl.ctypes.data, nk,
        kt.ctypes.data, ko.ctypes.data, kl.ctypes.data, kn.ctypes.data, dst.ctypes.data, dst.size, doff.ctypes.data,
        dlen.ctypes.data, C.byref(total), cks.ctypes.data, st.ctypes.data)
    return rc, total.value, L.b2s_last_error().decode()


TYPES = ["int", "string", "decimal", "long"]
KEYS = hm.keys_of(TYPES, [0, 1, 2, 3])


def bad_record(kind):
    """one record that the call must reject, as (bytes with prefix, rec_len)"""
    good = hm.make_row(TYPES, [1, b"abcdef", 12345, 7])
    if kind == "short":
        return b"\x00\x00\x01", 3
    if kind == "prefix":
        return (len(good) + 1).to_bytes(4, "big") + good, 4 + len(good)
    if kind == "key":
        row = good[:8 + 8 * 3]  # ends before the long's slot
        return len(row).to_bytes(4, "big") + row, 4 + len(row)
    r = bytearray(good)
    if kind == "string":
        r[16:24] = ((len(good) - 2) << 32 | 6).to_bytes(8, "little")
    elif kind == "decimal0":
        r[24:32] = (int.from_bytes(r[24:32], "little") & ~0xFFFFFFFF).to_bytes(8, "little")
    elif kind == "decimal17":
        r[24:32] = ((8 + 32) << 32 | 17).to_bytes(8, "little")
    elif kind == "decimal_past":
        r[24:32] = ((len(good) - 1) << 32 | 2).to_bytes(8, "little")
    return len(r).to_bytes(4, "big") + bytes(r), 4 + len(r)


@pytest.mark.parametrize("kind,why", [("short", "rec_len is below 4"), ("prefix", "size prefix"),
                                      ("key", "key slot"), ("string", "string key"), ("decimal0", "decimal key"),
                                      ("decimal17", "decimal key"), ("decimal_past", "decimal key")])
def test_bad_records_are_rejected_naming_the_lowest(capi, kind, why):
    rng = np.random.default_rng(1)
    rows = [hm.make_row(TYPES, [int(i), bytes(rng.integers(0, 256, i % 30, dtype=np.uint8)),
                                int(rng.integers(-2**62, 2**62)) << (i % 40), None]) for i in range(400)]
    recs = [len(r).to_bytes(4, "big") + r for r in rows]
    lens = [len(r) for r in recs]
    bad, bl = bad_record(kind)
    for at in (0, 137, 399):
        rr, ll = list(recs), list(lens)
        rr[at], ll[at] = bad, bl
        if at + 50 < len(rr):
            rr[at + 50], ll[at + 50] = bad_record("prefix")
        buf = np.frombuffer(b"".join(rr), np.uint8).copy()
        rc, total, err = raw_call(capi, buf, np.array(ll, np.uint32), KEYS)
        assert rc == capi.E_ARG and total == 0
        assert ("record %d " % at) in err and why in err, err


def test_null_word_out_of_row_and_null_slots_not_read(capi):
    types = ["int", "string"]
    keys = [(hm.KEY_INT32, 8, 4, 200), (hm.STRING, 16, 8, 1)]  # null bit 200: in the 8-byte word at row offset 24
    short = hm.make_row(types, [5, None])  # 24 bytes: holds both key slots, not the null word 24..32
    row = bytearray(short + bytes(8))
    row[16:24] = (10**6 << 32 | 99).to_bytes(8, "little")  # a null string's slot is not read
    recs = [len(r).to_bytes(4, "big") + bytes(r) for r in (row, row, short)]
    buf = np.frombuffer(b"".join(recs), np.uint8).copy()
    rl = np.array([len(r) for r in recs], np.uint32)
    rc, total, err = raw_call(capi, buf, rl, keys)
    assert rc == capi.E_ARG and total == 0 and "record 2 " in err and "null word" in err
    rc, total, err = raw_call(capi, buf[: int(rl[:2].sum())], rl[:2], keys)
    assert rc == 0, err


@pytest.mark.parametrize("kw", [dict(R=0), dict(keys=[]), dict(keys=[(1, 8, 4, -1)] * 17),
                                dict(keys=[(4, 8, 8, -1)]), dict(keys=[(0, 8, 2, -1)]), dict(keys=[(1, 8, 8, -1)]),
                                dict(keys=[(1 | (1 << 8), 8, 4, -1)]), dict(keys=[(2 | (1 << 9), 8, 8, 0)]),
                                dict(keys=[(1, 8, 4, -2)]), dict(sum_off=1)])
def test_argument_errors(capi, kw):
    rows = [hm.make_row(["int"], [i]) for i in range(10)]
    recs, rl = hm.records_of(rows)
    keys = kw.get("keys", hm.keys_of(["int"], [0]))
    if "sum_off" in kw:
        rl = rl.copy()
        rl[3] += 1  # rec_len no longer sums to rec_bytes
    rc, total, err = raw_call(capi, recs, rl, keys, R=kw.get("R", 7))
    assert rc == capi.E_ARG and total == 0, err


def test_dst_too_small_matches_partition_compress(capi):
    rng = np.random.default_rng(3)
    rows = hm.random_rows(rng, 2000)
    keys = hm.keys_of(hm.COMPOSITE, range(8))
    recs, rl = hm.records_of(rows)
    ids = hm.record_ids_np(recs, rl, keys, 200)
    L = capi.load()
    for codec in (0, 1):
        res = []
        for hashed in (False, True):
            doff, dlen, cks = np.zeros(200, np.uint64), np.zeros(200, np.uint64), np.zeros(200, np.uint64)
            st = np.zeros(200, np.int32)
            dst = np.zeros(recs.size // 2, np.uint8)
            total = C.c_uint64(0)
            nk, kt, ko, kl, kn = capi._key_arrays(keys)
            tail = (dst.ctypes.data, dst.size, doff.ctypes.data, dlen.ctypes.data, C.byref(total), cks.ctypes.data,
                    st.ctypes.data)
            head = (codec, 0, 0, 3, 200, rl.size, recs.ctypes.data, recs.size, rl.ctypes.data)
            if hashed:
                rc = L.b2s_partition_compress_rows_hash_packed(*head, nk, kt.ctypes.data, ko.ctypes.data,
                                                               kl.ctypes.data, kn.ctypes.data, *tail)
            else:
                rc = L.b2s_partition_compress_packed(*head, ids.ctypes.data, *tail)
            res.append((rc, total.value, doff.copy(), dlen.copy(), st.copy(), dst.copy()))
        assert res[0][0] == res[1][0] == capi.E_DST_TOO_SMALL
        assert res[0][1] == res[1][1]
        for a, b in zip(res[0][2:], res[1][2:]):
            assert (a == b).all()


def test_end_to_end_hash_exchange_then_grouped_aggregation(capi):
    """M maps hash-partitioned by (string, long); each reducer aggregates its blocks by the same key: every key is on
    exactly one reducer, pmod(hash, R), and the merged rows equal a Python group-by"""
    rng = np.random.default_rng(11)
    types = ["string", "long", "long"]
    keys = hm.keys_of(types, [0, 1])
    M, R = 4, 13
    names = [b"", b"a", b"spark", b"\xff\x80x", b"shuffle-partition-0123456789"]
    maps, want = [], {}
    for m in range(M):
        rows = []
        for i in range(2500):
            k0 = None if rng.random() < 0.05 else names[int(rng.integers(len(names)))]
            k1 = None if rng.random() < 0.05 else int(rng.integers(-50, 50))
            v = int(rng.integers(-1000, 1000))
            rows.append(hm.make_row(types, [k0, k1, v]))
            want[(k0, k1)] = want.get((k0, k1), 0) + v
        recs, rl = hm.records_of(rows)
        dst = np.zeros(capi.partition_compress_bound(1, 0, R, recs.size) + 64, np.uint8)
        r = capi.partition_compress_rows_hash_packed(1, recs, rl, keys, R, dst, checksum_alg=3)
        maps.append((dst, r))
    seen = {}
    for red in range(R):
        blocks = [(dst[int(r["dst_off"][red]):int(r["dst_off"][red] + r["dst_len"][red])], int(r["checksums"][red]))
                  for dst, r in maps if r["dst_len"][red]]
        if not blocks:
            continue
        src = np.concatenate([b for b, _ in blocks])
        ln = np.array([b.size for b, _ in blocks], np.uint64)
        off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
        out = np.zeros(1 << 20, np.uint8)
        res = capi.decompress_aggregate_rows_keys_packed(1, src, off, ln, out, keys, aggs=[(rm.SUM_I64, 24, 2)],
                                                         checksum_alg=3, slice_base=np.arange(len(blocks) + 1),
                                                         slice_len=ln, slice_checksum=[c for _, c in blocks])
        buf = out[:res["total"]].tobytes()
        for o, n in rm.parse(buf):
            row = buf[o + 4:o + n]
            key = tuple(None if v[0] == 0 else v[1] for v in (rm.col_value(row, c) for c in
                                                               [(3, 8, 8, 0), (2, 16, 8, 1)]))
            assert key not in seen, key
            seen[key] = red
            assert hm.pmod(hm.row_hash(row, keys), R) == red
            assert int.from_bytes(row[24:32], "little", signed=True) == want[key]
    assert set(seen) == set(want)


def test_host_mirror_hash_mode_files_identical_and_readable(tmp_path):
    rng = np.random.default_rng(21)
    rows = hm.random_rows(rng, 3000)
    keys = hm.keys_of(hm.COMPOSITE, range(8))
    R = 31
    recs, rl = hm.records_of(rows)
    ids = hm.record_ids_np(recs, rl, keys, R)
    host = pkg.host
    d_hash, d_ids = rm.mirror(tmp_path / "hash", "lz4"), rm.mirror(tmp_path / "ids", "lz4")
    w = host.S3SerializedShuffleWriter(d_hash, 0, 0, R)
    w.hashRows(keys)
    for row in rows:
        w.insertRecord(0, len(row).to_bytes(4, "big") + row)
    lens_hash = w.commit()
    w.close()
    w = host.S3SerializedShuffleWriter(d_ids, 0, 0, R)
    for row, p in zip(rows, ids):
        w.insertRecord(int(p), len(row).to_bytes(4, "big") + row)
    lens_ids = w.commit()
    w.close()
    assert list(lens_hash) == list(lens_ids)
    for kind in ("data", "index", "checksum"):
        assert open(d_hash.getPath(kind, 0, 0), "rb").read() == open(d_ids.getPath(kind, 0, 0), "rb").read()
    for red in (0, 7, R - 1):
        rd = host.S3ShuffleReader(d_hash, 0, [0], red, red + 1)
        got = b"".join(b for _, b in rd.read())
        rd.close()
        assert got == b"".join(len(r).to_bytes(4, "big") + r for r, p in zip(rows, ids) if p == red)
