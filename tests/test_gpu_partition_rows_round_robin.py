"""b2s_partition_compress_rows_round_robin_*: Spark's RoundRobinPartitioning of serialized UnsafeRows on the GPU (the
sortBeforeRepartition sort, then the position's ids), then the partition + compress step.  Every output must be byte
for byte what b2s_partition_compress_packed returns when fed the records in the order of the model
(tests/round_robin_model.py) with the model's ids; ties of hash and size, engineered Murmur3 collisions included, must
come out in the model's order."""
import ctypes as C

import numpy as np
import pytest

import hash_model as hm
import round_robin_model as rr
import rows_model as rm
import spark_s3_shuffle_b200 as pkg

pytestmark = pytest.mark.gpu

CODECS = [("none", 0, 0), ("lz4", 1, 0), ("snappy", 2, 0), ("zstd1", 3, 1)]
RS = [1, 2, 3, 129, 2000]
M32 = 0xFFFFFFFF


def rows_of(rng, n, dup=0.2):
    """UnsafeRows of several shapes, rows of size 0, and duplicates"""
    rows = hm.random_rows(rng, n)
    for i in range(0, n, 97):
        rows[i] = b""
    for i in rng.integers(0, n, int(n * dup)):
        rows[int(i)] = rows[int(rng.integers(0, n))]
    return rows


def starts(rng, R):
    return sorted({0, R - 1, int(rng.integers(0, R))})


def both(capi, codec, lvl, alg, recs, rl, R, start, sort):
    wr, wl, ids = rr.writer_records(recs, rl, start, R, sort)
    cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
    ref_dst, got_dst = np.zeros(cap, np.uint8), np.zeros(cap, np.uint8)
    ref = capi.partition_compress_packed(codec, wr, wl, ids, R, ref_dst, checksum_alg=alg, level=lvl)
    got = capi.partition_compress_rows_round_robin_packed(codec, recs, rl, R, start, sort, got_dst, checksum_alg=alg,
                                                          level=lvl)
    return ref, got, ref_dst, got_dst


def same(ref, got, ref_dst, got_dst):
    assert got["total"] == ref["total"]
    for k in ("dst_off", "dst_len", "checksums", "status"):
        assert (got[k] == ref[k]).all(), k
    assert (got_dst[:got["total"]] == ref_dst[:ref["total"]]).all()


def check(capi, rows, R, start, sort, codec=0, lvl=0, alg=3):
    recs, rl = hm.records_of(rows)
    same(*both(capi, codec, lvl, alg, recs, rl, R, start, sort))


@pytest.mark.parametrize("alg", rm.CHECKSUMS)
@pytest.mark.parametrize("codec_name,codec,lvl", CODECS)
def test_parity_with_partition_compress_of_the_model(capi, codec_name, codec, lvl, alg):
    rng = np.random.default_rng(codec * 10 + lvl + alg)
    rows = rows_of(rng, 1200)
    recs, rl = hm.records_of(rows)
    for R in RS:
        for start in starts(rng, R):
            for sort in (0, 1):
                same(*both(capi, codec, lvl, alg, recs, rl, R, start, sort))
    empty = hm.records_of([])
    for sort in (0, 1):
        ref, got, ref_dst, got_dst = both(capi, codec, lvl, alg, *empty, 7, 3, sort)
        same(ref, got, ref_dst, got_dst)
        assert got["total"] == 0 and (got["dst_len"] == 0).all()


def test_rows_of_size_zero_only(capi):
    for R in (1, 2, 129):
        for sort in (0, 1):
            check(capi, [b""] * 500, R, R - 1, sort)


def run_dev(capi, codec, lvl, alg, recs, rl, R, start, sort):
    cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
    d_rec, d_len, d_dst = capi.dev_alloc(max(recs.size, 1)), capi.dev_alloc(max(rl.nbytes, 4)), capi.dev_alloc(cap)
    try:
        if recs.size:
            capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
            capi.dev_memcpy(d_len, rl.ctypes.data, rl.nbytes, 1)
        r = capi.partition_compress_rows_round_robin_dev(codec, d_rec, recs.size, d_len, rl.size, R, start, sort, d_dst,
                                                         cap, checksum_alg=alg, level=lvl)
        out = np.zeros(max(r["total"], 1), np.uint8)
        if r["total"]:
            capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        return r, out
    finally:
        for p in (d_rec, d_len, d_dst):
            capi.dev_free(p)


@pytest.mark.parametrize("codec_name,codec,lvl", CODECS)
def test_dev_equals_packed(capi, codec_name, codec, lvl):
    rng = np.random.default_rng(40 + codec + lvl)
    recs, rl = hm.records_of(rows_of(rng, 3000))
    for R in (1, 200, 2000):
        for sort in (0, 1):
            start = int(rng.integers(0, R))
            cap = capi.partition_compress_bound(codec, 0, R, recs.size) + 64
            dst = np.zeros(cap, np.uint8)
            ref = capi.partition_compress_rows_round_robin_packed(codec, recs, rl, R, start, sort, dst, checksum_alg=3,
                                                                  level=lvl)
            got, out = run_dev(capi, codec, lvl, 3, recs, rl, R, start, sort)
            same(ref, got, dst, out)
    got, _ = run_dev(capi, codec, lvl, 3, *hm.records_of([]), 5, 4, 1)
    assert got["total"] == 0


# ---- engineered Murmur3 collisions: hashUnsafeWords is invertible in its last word ----
def _inv(a):
    return pow(a, -1, 1 << 32)


def _rotr(x, r):
    return ((x >> r) | (x << (32 - r))) & M32


def _fmix_inv(h):
    h ^= h >> 16
    h = (h * _inv(0xC2B2AE35)) & M32
    h ^= (h >> 13) ^ (h >> 26)
    h = (h * _inv(0x85EBCA6B)) & M32
    return h ^ (h >> 16)


def collide(prefix, target, size):
    """a row of size bytes (a multiple of 8) starting with prefix (size - 4 bytes) whose hashUnsafeWords(., 42) is
    target: the last word is solved for"""
    assert len(prefix) == size - 4 and size % 8 == 0
    h = rr.SEED
    for i in range(0, len(prefix), 4):
        h = hm._mix_h1(h, hm._mix_k1(int.from_bytes(prefix[i:i + 4], "little")))
    hm_ = _fmix_inv(target) ^ size  # the state before fmix
    k = _rotr(((hm_ - 0xE6546B64) * _inv(5)) & M32, 13) ^ h  # mix_h1(h, k) == hm_
    w = (_rotr((k * _inv(0x1B873593)) & M32, 15) * _inv(0xCC9E2D51)) & M32  # mix_k1(w) == k
    row = prefix + w.to_bytes(4, "little")
    assert rr.hash_unsafe_words(row) == target
    return row


def collisions(rng, n_groups=40):
    """groups of rows of one hash: equal size, differing in the first refinement window (row bytes 0..11), in a later
    one, or only in their last 8 bytes; and of different sizes"""
    rows = []
    for g in range(n_groups):
        size = 8 * int(rng.integers(2, 40))
        base = bytearray(rng.integers(0, 256, size - 4, dtype=np.uint8).tobytes())
        target = int(rng.integers(0, 1 << 32))
        for where in (3, 40, size - 8, None):
            p = bytearray(base)
            if where is not None and where < size - 4:
                p[where] ^= 1 << int(rng.integers(0, 8))
            rows.append(collide(bytes(p), target, size))
        rows.append(collide(bytes(rng.integers(0, 256, size + 4, dtype=np.uint8)), target, size + 8))
        rows.append(collide(bytes(rng.integers(0, 256, 4, dtype=np.uint8)), target, 8))
    return rows


def test_hash_collisions_come_out_in_the_models_order(capi):
    rng = np.random.default_rng(5)
    rows = collisions(rng) + rows_of(rng, 500)
    for _ in range(3):
        rng.shuffle(rows)
        for R in (2, 129):
            check(capi, rows, R, int(rng.integers(0, R)), 1)
    h = [rr.row_hash(r) for r in rows]
    assert len(set(h)) < len(h) - 100


def test_many_duplicate_rows(capi):
    rng = np.random.default_rng(6)
    distinct = rows_of(rng, 50, dup=0)
    rows = [distinct[int(i)] for i in rng.integers(0, len(distinct), 20000)]
    for R in (3, 2000):
        check(capi, rows, R, 1, 1, codec=1)


def test_long_rows_with_long_shared_prefixes(capi):
    """1 MiB rows whose colliding pairs agree on their first 8 KiB: hundreds of refinement rounds"""
    rng = np.random.default_rng(7)
    size = 1 << 20
    rows = []
    for g in range(3):
        shared = rng.integers(0, 256, size - 4, dtype=np.uint8)
        target = int(rng.integers(0, 1 << 32))
        for d in (8192, 8200, 8192 + 4096):
            p = shared.copy()
            p[d] ^= 0x80
            rows.append(collide(p.tobytes(), target, size))
    rows += rows_of(rng, 300)
    rng.shuffle(rows)
    check(capi, rows, 5, 4, 1, codec=1)


def test_sorted_output_is_the_same_for_every_input_order(capi):
    """the point of the sort: a retried map task, seeing its rows in another order, writes the same bytes"""
    rng = np.random.default_rng(8)
    rows = rows_of(rng, 4000) + collisions(rng, 10)
    R = 200
    outs = []
    for _ in range(4):
        rng.shuffle(rows)
        recs, rl = hm.records_of(rows)
        dst = np.zeros(capi.partition_compress_bound(2, 0, R, recs.size) + 64, np.uint8)
        r = capi.partition_compress_rows_round_robin_packed(2, recs, rl, R, 17, 1, dst, checksum_alg=3)
        outs.append((dst[:r["total"]].tobytes(), list(r["dst_len"]), list(r["checksums"])))
    assert all(o == outs[0] for o in outs[1:])


def raw_call(capi, recs, rl, R=7, start=3, sort=1, codec=1, cap=None):
    L = capi.load()
    doff, dlen, cks = np.zeros(R, np.uint64), np.zeros(R, np.uint64), np.zeros(R, np.uint64)
    st = np.zeros(R, np.int32)
    dst = np.zeros(capi.partition_compress_bound(codec, 0, R, recs.size) + 64 if cap is None else max(cap, 1), np.uint8)
    total = C.c_uint64(7)
    rc = L.b2s_partition_compress_rows_round_robin_packed(
        codec, 0, 0, 3, R, start, sort, rl.size, recs.ctypes.data if recs.size else None, recs.size, rl.ctypes.data,
        dst.ctypes.data, dst.size if cap is None else cap, doff.ctypes.data, dlen.ctypes.data, C.byref(total),
        cks.ctypes.data, st.ctypes.data)
    return rc, total.value, L.b2s_last_error().decode(), (doff, dlen, st, dst)


def bad_record(kind):
    if kind == "short":
        return b"\x00\x00\x01", 3
    if kind == "prefix":
        return (17).to_bytes(4, "big") + bytes(16), 20
    return (12).to_bytes(4, "big") + bytes(12), 16  # words: 12 bytes is not an UnsafeRow


@pytest.mark.parametrize("sort", [0, 1])
@pytest.mark.parametrize("kind,why", [("short", "rec_len is below 4"), ("prefix", "size prefix"),
                                      ("words", "not a multiple of 8")])
def test_bad_records_are_rejected_naming_the_lowest(capi, kind, why, sort):
    rng = np.random.default_rng(1)
    rows = rows_of(rng, 400)
    recs = [len(r).to_bytes(4, "big") + r for r in rows]
    lens = [len(r) for r in recs]
    bad, bl = bad_record(kind)
    for at in (0, 137, 399):
        rs, ll = list(recs), list(lens)
        rs[at], ll[at] = bad, bl
        if at + 50 < len(rs):
            rs[at + 50], ll[at + 50] = bad_record("prefix")
        buf = np.frombuffer(b"".join(rs), np.uint8).copy()
        rc, total, err, _ = raw_call(capi, buf, np.array(ll, np.uint32), sort=sort)
        assert rc == capi.E_ARG and total == 0
        assert ("record %d " % at) in err and why in err, err


@pytest.mark.parametrize("sort", [0, 1])
def test_rec_len_past_rec_bytes(capi, sort):
    rng = np.random.default_rng(2)
    recs, rl = hm.records_of(rows_of(rng, 300) + collisions(rng, 5))
    rl = rl.copy()
    rl[-1] += 64  # the last record ends past rec_bytes: it is not read, and the length sum names it
    rc, total, err, _ = raw_call(capi, recs, rl, sort=sort)
    assert rc == capi.E_ARG and total == 0 and ("record %d ends past rec_bytes" % (rl.size - 1)) in err, err
    rl[-1] -= 64
    rl[150] += 64  # inside rec_bytes, record 150 now disagrees with its size prefix
    rc, total, err, _ = raw_call(capi, recs, rl, sort=sort)
    assert rc == capi.E_ARG and total == 0 and "record 150 " in err and "size prefix" in err, err


def test_dst_too_small_matches_partition_compress(capi):
    rng = np.random.default_rng(3)
    recs, rl = hm.records_of(rows_of(rng, 2000))
    R, start = 200, 11
    wr, wl, ids = rr.writer_records(recs, rl, start, R, 1)
    L = capi.load()
    for codec in (0, 1):
        rc, total, _, got = raw_call(capi, recs, rl, R=R, start=start, sort=1, codec=codec, cap=recs.size // 2)
        doff, dlen, cks = np.zeros(R, np.uint64), np.zeros(R, np.uint64), np.zeros(R, np.uint64)
        st = np.zeros(R, np.int32)
        dst = np.zeros(recs.size // 2, np.uint8)
        t = C.c_uint64(0)
        rc2 = L.b2s_partition_compress_packed(codec, 0, 0, 3, R, wl.size, wr.ctypes.data, wr.size, wl.ctypes.data,
                                              ids.ctypes.data, dst.ctypes.data, dst.size, doff.ctypes.data,
                                              dlen.ctypes.data, C.byref(t), cks.ctypes.data, st.ctypes.data)
        assert rc == rc2 == capi.E_DST_TOO_SMALL and total == t.value
        for a, b in zip(got, (doff, dlen, st, dst)):
            assert (a[:b.size] == b).all()


def test_timing_covers_the_round_robin_step(capi):
    rng = np.random.default_rng(4)
    recs, rl = hm.records_of(rows_of(rng, 5000))
    dst = np.zeros(capi.partition_compress_bound(1, 0, 64, recs.size) + 64, np.uint8)
    capi.partition_compress_rows_round_robin_packed(1, recs, rl, 64, 5, 0, dst, checksum_alg=3)
    t = capi.last_timing()
    assert t["dominant_launches"] == 2 and t["dominant_ms"] > 0  # the checks and the ids
    capi.partition_compress_rows_round_robin_packed(1, recs, rl, 64, 5, 1, dst, checksum_alg=3)
    t2 = capi.last_timing()
    assert t2["dominant_launches"] > 2 + 4 and t2["dominant_ms"] > 0  # + hash sort, rounds


def test_end_to_end_repartition_over_several_maps(capi):
    """repartition(R) of M maps, read back per reducer by b2s_decompress_packed: every row lands once, and each
    map's partitions differ in row count by at most one"""
    rng = np.random.default_rng(11)
    M, R = 5, 13
    maps, every = [], []
    for m in range(M):
        rows = rows_of(rng, 1000 + 137 * m)
        every += rows
        recs, rl = hm.records_of(rows)
        dst = np.zeros(capi.partition_compress_bound(1, 0, R, recs.size) + 64, np.uint8)
        r = capi.partition_compress_rows_round_robin_packed(1, recs, rl, R, int(rng.integers(0, R)), 1, dst,
                                                            checksum_alg=3)
        maps.append((dst, r))
    got = []
    counts = np.zeros((M, R), np.int64)
    for red in range(R):
        for m, (dst, r) in enumerate(maps):
            if not r["dst_len"][red]:
                continue
            blk = dst[int(r["dst_off"][red]):int(r["dst_off"][red] + r["dst_len"][red])]
            out = np.zeros(1 << 22, np.uint8)
            res = capi.decompress_packed(1, blk, [0], [blk.size], out, checksum_alg=3, slice_base=[0, 1],
                                         slice_len=[blk.size], slice_checksum=[int(r["checksums"][red])])
            buf = out[:int(res["dst_len"][0])].tobytes()
            for o, n in rm.parse(buf):
                got.append(buf[o + 4:o + n])
                counts[m, red] += 1
    assert sorted(got) == sorted(every)
    assert (counts.max(axis=1) - counts.min(axis=1) <= 1).all()


def test_host_mirror_round_robin_mode_files_identical_and_readable(tmp_path):
    rng = np.random.default_rng(21)
    rows = rows_of(rng, 3000)
    R, start = 31, 9
    recs, rl = hm.records_of(rows)
    wr, wl, ids = rr.writer_records(recs, rl, start, R, 1)
    host = pkg.host
    d_rr, d_ids = rm.mirror(tmp_path / "rr", "lz4"), rm.mirror(tmp_path / "ids", "lz4")
    w = host.S3SerializedShuffleWriter(d_rr, 0, 0, R)
    w.roundRobinRows(R, start, True)
    for row in rows:
        w.insertRecord(0, len(row).to_bytes(4, "big") + row)
    lens_rr = w.commit()
    w.close()
    w = host.S3SerializedShuffleWriter(d_ids, 0, 0, R)
    off = np.concatenate([[0], np.cumsum(wl.astype(np.int64))])
    for k, p in enumerate(ids):
        w.insertRecord(int(p), wr[off[k]:off[k + 1]].tobytes())
    lens_ids = w.commit()
    w.close()
    assert list(lens_rr) == list(lens_ids)
    for kind in ("data", "index", "checksum"):
        assert open(d_rr.getPath(kind, 0, 0), "rb").read() == open(d_ids.getPath(kind, 0, 0), "rb").read()
    for red in (0, 7, R - 1):
        rd = host.S3ShuffleReader(d_rr, 0, [0], red, red + 1)
        got = b"".join(b for _, b in rd.read())
        rd.close()
        assert got == b"".join(wr[off[k]:off[k + 1]].tobytes() for k in range(len(ids)) if ids[k] == red)
