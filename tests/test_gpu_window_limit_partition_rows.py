"""A map task's partial window limit on the GPU (b2s_window_limit_partition_compress_rows_hash_*): every output is byte
for byte the hash call's over tests/window_limit_model.py's kept rows, and reducers fed by it compute what reducers fed
by the unlimited rows compute."""
import struct

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from join_model import VAR
from rows_model import CHECKSUMS, CODECS, KEY_INT32, KEY_INT64, STRING, mirror, stream
from test_gpu_sort_rows_order import DECIMAL, DESC, FLAGS, KEY_FLOAT32, KEY_FLOAT64, KEY_INT8, KEY_INT16, \
    NULLS_LAST
from test_gpu_window_rows import Schema, _records, table
from window_limit_model import partial_limit
from window_model import DENSE_RANK, RANK, ROW_NUMBER, model_window

pytestmark = pytest.mark.gpu

FNS = [ROW_NUMBER, RANK, DENSE_RANK]


def _framed(rows):
    return np.frombuffer(stream(rows) or b"\0", np.uint8)[:sum(4 + len(r) for r in rows)].copy(), \
        np.array([4 + len(r) for r in rows], np.uint32)


def _hash_of(capi, rows, keys, R, codec=1, level=0, alg=3, bs=0):
    """the hash call over rows (the defining contract), or the plain partition call with every id 0 (keys empty)"""
    records, rec_len = _framed(rows)
    dst = np.zeros(capi.partition_compress_bound(codec, bs, R, records.size) + 64, np.uint8)
    if keys:
        r = capi.partition_compress_rows_hash_packed(codec, records, rec_len, keys, R, dst, block_size=bs,
                                                     checksum_alg=alg, level=level)
    else:
        r = capi.partition_compress_packed(codec, records, rec_len, np.zeros(len(rows), np.uint32), R, dst,
                                           block_size=bs, checksum_alg=alg, level=level)
    return r, dst[:r["total"]].tobytes()


def check(capi, rows, keys, npk, fn, limit, R=8, codec=1, level=0, alg=3, bs=0, kept=None):
    """kept: the model's kept rows when the caller has them"""
    records, rec_len = _framed(rows)
    dst = np.zeros(capi.partition_compress_bound(codec, bs, R, records.size) + 64, np.uint8)
    got = capi.window_limit_partition_compress_rows_hash_packed(codec, records, rec_len, keys, npk, fn, limit, R, dst,
                                                                block_size=bs, checksum_alg=alg, level=level)
    kept = partial_limit(rows, keys, npk, fn, limit) if kept is None else kept
    want, want_bytes = _hash_of(capi, kept, keys[:npk], R, codec, level, alg, bs)
    assert got["n_out_records"] == len(kept)
    assert got["total"] == want["total"]
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert (got[k] == want[k]).all(), k
    assert dst[:got["total"]].tobytes() == want_bytes
    return got, kept


# ---------------------------------------------------------------------------------------------------------------
# 1. every codec and checksum; every key type as a partition and as an order column, with every order flag
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", CHECKSUMS)
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_every_codec_and_checksum(capi, name, codec, level, alg):
    rng = np.random.default_rng(1 + codec * 5 + level + 7 * alg)
    s = Schema(5, [(STRING, 0, True), (KEY_INT64 | DESC, 2, True), (KEY_INT32, 4, False)], {1: VAR})
    rows = table(rng, s, 3000, domain=7)
    check(capi, rows, s.keys, 1, RANK, 3, codec=codec, level=level, alg=alg)


@pytest.mark.parametrize("t", [STRING, KEY_INT8, KEY_INT16, KEY_INT32, KEY_INT64, KEY_FLOAT32, KEY_FLOAT64, DECIMAL])
def test_every_key_type_as_partition_and_order_column(capi, t):
    rng = np.random.default_rng(20 + t)
    for k, flags in enumerate(FLAGS):
        s = Schema(4, [(t, 0, True), (KEY_INT64 | flags, 1, True), (KEY_INT32, 2, False)])
        check(capi, table(rng, s, 1500, domain=5), s.keys, 1, FNS[k % 3], 2)
        o = Schema(4, [(KEY_INT32, 0, True), (t | flags, 1, True), (KEY_INT64, 2, False)])
        check(capi, table(rng, o, 1500, domain=5), o.keys, 1, FNS[(k + 1) % 3], 2)


# ---------------------------------------------------------------------------------------------------------------
# 2. limits: 1, inside a peer group, at or above every partition's size; shapes
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", FNS)
def test_limits_one_inside_peer_groups_and_past_every_partition(capi, fn):
    rng = np.random.default_rng(30 + fn)
    s = Schema(4, [(STRING, 0, True), (KEY_FLOAT64 | DESC | NULLS_LAST, 1, True), (KEY_INT32, 2, False)])
    rows = table(rng, s, 4000, domain=4, null_frac=0.1)
    for limit in (1, 2, 3, 5, 40):
        check(capi, rows, s.keys, 1, fn, limit)
    got, kept = check(capi, rows, s.keys, 1, fn, 2**31 - 1)
    assert len(kept) == len(rows)  # every record kept: the hash call over all rows in sorted order


def test_one_partition_of_over_a_million_rows_and_many_one_row_partitions(capi):
    rng = np.random.default_rng(40)
    n = 1_100_000
    v = rng.integers(0, 50_000, n)
    big = [struct.pack("<qqqq", 0, 7, int(x), i) for i, x in enumerate(v)]
    keys = [(KEY_INT64, 8, 8, -1), (KEY_INT64 | DESC, 16, 8, -1)]
    order = np.argsort(-v, kind="stable")  # the model's sort, in numpy: one partition, order DESC, ties in input order
    sv = v[order]
    first = np.searchsorted(-sv, -sv, side="left")  # each position's peer group start
    dense = np.cumsum(np.concatenate([[1], sv[1:] != sv[:-1]]))
    for fn, value in ((ROW_NUMBER, np.arange(1, n + 1)), (RANK, first + 1), (DENSE_RANK, dense)):
        got, kept = check(capi, big, keys, 1, fn, 100, R=16, kept=[big[i] for i in order[value <= 100]])
        assert len(kept) >= 100
    one = [struct.pack("<qqq", 0, i, i % 3) for i in rng.permutation(200_000)]
    got, kept = check(capi, one, keys, 1, RANK, 1, R=200)
    assert len(kept) == len(one)


@pytest.mark.parametrize("fn", FNS)
def test_no_partition_columns_is_single_partition(capi, fn):
    rng = np.random.default_rng(50 + fn)
    s = Schema(3, [(KEY_INT64 | DESC, 0, True), (STRING, 1, True)])
    rows = table(rng, s, 5000, domain=30)
    got, kept = check(capi, rows, s.keys, 0, fn, 10, R=1)
    assert got["dst_len"][0] > 0 and 10 <= len(kept) < len(rows)


def test_empty_input(capi):
    keys = [(KEY_INT64, 8, 8, -1), (KEY_INT64, 16, 8, -1)]
    for npk, R in ((1, 4), (0, 1)):
        got = capi.window_limit_partition_compress_rows_hash_packed(1, np.zeros(0, np.uint8), [], keys, npk, RANK, 3,
                                                                    R, np.zeros(64, np.uint8), checksum_alg=3)
        assert got["n_out_records"] == 0 and got["total"] == 0 and (got["dst_len"] == 0).all()


# ---------------------------------------------------------------------------------------------------------------
# 3. bad records, the exact size on a short destination, the _dev form
# ---------------------------------------------------------------------------------------------------------------
def test_bad_records_and_bad_key_slots_are_named(capi):
    s = Schema(3, [(STRING, 0, True), (DECIMAL | DESC, 1, True)])
    rows = table(np.random.default_rng(60), s, 50)
    # with their null words cleared: a row too short for the order column's slot, a string and a decimal past the row
    for i, bad, words in ((7, rows[7][:16], b"key slot"),
                          (12, bytes(8) + ((1 << 40) | 9).to_bytes(8, "little") + rows[12][16:], b"string"),
                          (30, bytes(8) + rows[30][8:16] + ((24 << 32) | 17).to_bytes(8, "little") + rows[30][24:], b"decimal")):
        bad_rows = list(rows)
        bad_rows[i] = bad
        records, rec_len = _framed(bad_rows)
        with pytest.raises(capi.B2SError) as e:
            capi.window_limit_partition_compress_rows_hash_packed(1, records, rec_len, s.keys, 1, RANK, 2, 4,
                                                                  np.zeros(1 << 16, np.uint8))
        assert e.value.code == capi.E_ARG
        msg = capi.load().b2s_last_error()
        assert b"record %d " % i in msg and words in msg, msg


def test_short_destination_reports_the_exact_size_then_succeeds(capi):
    rng = np.random.default_rng(70)
    s = Schema(3, [(STRING, 0, True), (KEY_INT64 | DESC, 1, True)])
    rows = table(rng, s, 3000, domain=5)
    records, rec_len = _framed(rows)
    L = capi.load()
    args = capi._key_arrays(s.keys)
    R = 4
    doff, dlen, cks = np.zeros(R, np.uint64), np.zeros(R, np.uint64), np.zeros(R, np.uint64)
    st = np.zeros(R, np.int32)
    import ctypes as C
    total, kept = C.c_uint64(0), C.c_uint64(0)
    small = np.zeros(100, np.uint8)
    rc = L.b2s_window_limit_partition_compress_rows_hash_packed(
        1, 0, 0, 3, R, len(rows), records.ctypes.data, records.size, rec_len.ctypes.data, 1, args[0],
        *[a.ctypes.data for a in args[1:]], RANK, 3, small.ctypes.data, small.size, doff.ctypes.data, dlen.ctypes.data,
        C.byref(total), cks.ctypes.data, st.ctypes.data, C.byref(kept))
    assert rc == capi.E_DST_TOO_SMALL and total.value > small.size
    dst = np.zeros(total.value, np.uint8)
    got = capi.window_limit_partition_compress_rows_hash_packed(1, records, rec_len, s.keys, 1, RANK, 3, R, dst,
                                                                checksum_alg=3)
    assert got["total"] == total.value
    want, want_bytes = _hash_of(capi, partial_limit(rows, s.keys, 1, RANK, 3), s.keys[:1], R)
    assert dst.tobytes() == want_bytes


def test_dev_matches_packed(capi):
    rng = np.random.default_rng(80)
    s = Schema(3, [(STRING, 0, True), (KEY_FLOAT32 | NULLS_LAST, 1, True)])
    rows = table(rng, s, 5000, domain=6)
    records, rec_len = _framed(rows)
    R = 6
    cap = capi.partition_compress_bound(1, 0, R, records.size) + 64
    dst = np.zeros(cap, np.uint8)
    want = capi.window_limit_partition_compress_rows_hash_packed(1, records, rec_len, s.keys, 1, DENSE_RANK, 2, R, dst,
                                                                 checksum_alg=3)
    d_rec, d_len, d_dst = capi.dev_alloc(records.size), capi.dev_alloc(rec_len.nbytes), capi.dev_alloc(cap)
    try:
        capi.dev_memcpy(d_rec, records.ctypes.data, records.size, 1)
        capi.dev_memcpy(d_len, rec_len.ctypes.data, rec_len.nbytes, 1)
        got = capi.window_limit_partition_compress_rows_hash_dev(1, d_rec, records.size, d_len, len(rows), s.keys, 1,
                                                                 DENSE_RANK, 2, R, d_dst, cap, checksum_alg=3)
        out = np.zeros(got["total"], np.uint8)
        capi.dev_memcpy(out.ctypes.data, d_dst, got["total"], 2)
    finally:
        for p in (d_rec, d_len, d_dst):
            capi.dev_free(p)
    assert got["n_out_records"] == want["n_out_records"] and got["total"] == want["total"]
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert (got[k] == want[k]).all(), k
    assert out.tobytes() == dst[:want["total"]].tobytes()


# ---------------------------------------------------------------------------------------------------------------
# 4. end to end: limited maps, then the reducers' window with the same limit; and the host mirror
# ---------------------------------------------------------------------------------------------------------------
def _reduce(capi, per_reducer, s, npk, fn, limit):
    got = []
    for blocks in per_reducer:
        data = [b for b, _ in blocks]
        if not data:
            continue
        lens = np.array([len(b) for b in data], np.uint64)
        off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        dst = np.zeros(1 << 23, np.uint8)
        r = capi.decompress_window_rows_keys_packed(1, np.frombuffer(b"".join(data), np.uint8), off, lens, dst, s.keys,
                                                    npk, s.nf, s.kinds, [fn], (fn, limit), 3,
                                                    np.arange(len(data) + 1, dtype=np.uint32), lens,
                                                    np.array([c for _, c in blocks], np.uint64))
        assert (r["status"] == 0).all()
        got.append(dst[:r["total"]].tobytes())
    return got


def _maps(capi, rows, s, npk, fn, limit, R, maps, limited):
    per_reducer = [[] for _ in range(R)]
    for m in range(maps):
        part = rows[m::maps]
        records, rec_len = _framed(part)
        dst = np.zeros(capi.partition_compress_bound(1, 0, R, records.size) + 64, np.uint8)
        if limited:
            r = capi.window_limit_partition_compress_rows_hash_packed(1, records, rec_len, s.keys, npk, fn, limit, R,
                                                                      dst, checksum_alg=3)
        else:
            r = capi.partition_compress_rows_hash_packed(1, records, rec_len, s.keys[:npk], R, dst, checksum_alg=3)
        for p in range(R):
            if r["dst_len"][p]:
                o = int(r["dst_off"][p])
                per_reducer[p].append((dst[o:o + int(r["dst_len"][p])].tobytes(), int(r["checksums"][p])))
    return per_reducer


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("shape", ["q67", "dedup"])
def test_limited_maps_leave_every_reducer_unchanged(capi, fn, shape):
    rng = np.random.default_rng(90 + fn + (shape == "dedup") * 10)
    cats = [b"Books", b"Children", b"Electronics", b"Home", b"Jewelry", b"Men", b"Music", b"Shoes", b"Sports",
            b"Women"]
    if shape == "q67":
        def value(rng, t, domain):
            if t & 0xFF == STRING:
                return cats[int(rng.integers(len(cats)))]
            return int(rng.integers(-2000, 20000)) * 10**2  # sumsales, decimal(28,2)

        s = Schema(9, [(STRING, 0, True), (DECIMAL | DESC | NULLS_LAST, 8, True)], {1: VAR, 2: VAR, 3: VAR, 7: VAR})
        rows, limit, R = table(rng, s, 12000, null_frac=0.02, value=value), 100, 4
    else:  # row_number() over (partition by id order by ts desc) = 1
        s = Schema(4, [(KEY_INT64, 0, False), (KEY_INT64 | DESC, 1, False)], {2: VAR})
        rows = table(rng, s, 12000, value=lambda rng, t, d: int(rng.integers(0, 3000)) if t == KEY_INT64 else
                     int(rng.integers(0, 5)))
        limit, R = 1, 5
    want = _reduce(capi, _maps(capi, rows, s, 1, fn, limit, R, 5, False), s, 1, fn, limit)
    got = _reduce(capi, _maps(capi, rows, s, 1, fn, limit, R, 5, True), s, 1, fn, limit)
    assert got == want
    assert sum(len(_records([g])) for g in got) < len(rows) // 2


@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_writes_limited_rows(capi, tmp_path, codec):
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R = 3, 2
    rng = np.random.default_rng(95)
    s = Schema(4, [(STRING, 0, True), (KEY_INT64 | DESC, 1, True)], {2: VAR})
    maps = []
    for m in range(M):
        rows = table(rng, s, 400)
        w = host.S3SerializedShuffleWriter(d, 0, m, R)
        w.windowLimitRows(s.keys, 1, RANK, 2)
        for r in rows:
            w.insertRecord(0, len(r).to_bytes(4, "big") + r)
        w.commit()
        w.close()
        maps.append(rows)
    for red in range(R):
        reader = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        got = reader.readWindowRows(s.keys, 1, s.nf, s.kinds, [RANK], (RANK, 2))
        reader.close()
        from hash_model import ids_scalar
        plain = [stream([r for r, p in zip(rows, ids_scalar(rows, s.keys[:1], R)) if p == red]) for rows in maps]
        want = model_window(plain, s.keys, 1, s.nf, s.kinds, [RANK], (RANK, 2))
        assert got[0] == want[0] and got[2] == want[2]
