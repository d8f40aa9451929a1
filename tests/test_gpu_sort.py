"""Verify + decompress + key-sort in one call (b2s_decompress_sort_*): a reduce task's fetched blocks in, every record of
every block out, sorted by the unsigned bytes [key_off, key_off + key_len) of each fixed-size record.  The model is a
stable numpy lexsort over the key bytes of the concatenated decoded blocks followed by a gather; the sort must be
byte for byte that model.  Errors follow the decompress calls: per-block status, nothing sorted when a block fails."""
import threading

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from rows_model import CHECKSUMS, CODECS, build_blocks, mirror, run

pytestmark = pytest.mark.gpu

REC, KEY_OFF, KEY_LEN = 104, 2, 10  # a Kryo-serialized TeraSort record: 0x01 0x0B, 10-byte key, 0x01 0x5B, 90 bytes


# ---------------------------------------------------------------------------------------------------------------
# model and helpers
# ---------------------------------------------------------------------------------------------------------------
def model_sort(plain_blocks, rb, ko, kl):
    """the decoded blocks back to back, records stably sorted by their key bytes (unsigned, lexicographic)"""
    buf = np.frombuffer(b"".join(plain_blocks), np.uint8)
    if buf.size == 0:
        return b""
    recs = buf.reshape(-1, rb)
    order = np.lexsort([recs[:, ko + j] for j in range(kl - 1, -1, -1)])  # last key is the primary one
    return recs[order].tobytes()


def random_records(rng, n, rb, ko, kl, alphabet=None):
    """random records; with an alphabet the key bytes come from it (ties, and the bytes either side of 0x80)"""
    r = rng.integers(0, 256, (n, rb), dtype=np.uint8)
    if alphabet is not None:
        r[:, ko:ko + kl] = rng.choice(np.array(alphabet, dtype=np.uint8), (n, kl))
    return r


def split_blocks(recs, sizes):
    """records -> list of block plaintexts holding `sizes` records each"""
    out, at = [], 0
    for s in sizes:
        out.append(recs[at:at + s].tobytes())
        at += s
    assert at == len(recs)
    return out


def check(capi, codec, level, alg, plain, rb, ko, kl, dev=False):
    blocks = build_blocks(capi, codec, level, alg, plain)
    total = sum(len(b) for b in plain)
    got, r = run(capi, "decompress_sort", codec, alg, blocks, (rb, ko, kl), total, dev)
    assert (r["status"] == 0).all(), r["status"]
    assert r["total"] == total and r["n_records"] == total // rb
    assert got == model_sort(plain, rb, ko, kl)
    return got


def terasort_records(oracle, n, seed=0):
    return np.frombuffer(oracle.gen_terasort(seed * 1000, n).tobytes(), np.uint8).reshape(n, REC)


# ---------------------------------------------------------------------------------------------------------------
# 1. every codec x checksum, _dev against _packed
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", CHECKSUMS)
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_sorts_like_the_model(capi, oracle, name, codec, level, alg):
    recs = terasort_records(oracle, 20_000, seed=1)
    plain = split_blocks(recs, [7000, 0, 1, 4999, 8000])  # an empty block and a one-record block among them
    check(capi, codec, level, alg, plain, REC, KEY_OFF, KEY_LEN)


@pytest.mark.parametrize("name,codec,level", CODECS)
def test_dev_matches_packed(capi, oracle, name, codec, level):
    recs = terasort_records(oracle, 30_000, seed=2)
    plain = split_blocks(recs, [10_000, 10_000, 10_000])
    a = check(capi, codec, level, 3, plain, REC, KEY_OFF, KEY_LEN)
    b = check(capi, codec, level, 3, plain, REC, KEY_OFF, KEY_LEN, dev=True)
    assert a == b
    t = capi.last_timing()
    assert t["top_kernel_ms"] > 0 and t["dst_bytes"] == len(a)


def test_blocks_with_several_slices(capi, oracle):
    """a ShuffleBlockBatchId block: several concatenated partition streams, one checksum slice each"""
    recs = terasort_records(oracle, 12_000, seed=3)
    parts = split_blocks(recs, [3000, 1000, 2000, 6000])
    a_arena, a_off, a_ln, _, _, a_ck = build_blocks(capi, 1, 0, 3, parts)
    # blocks = parts (0, 1) and (2, 3): each block is the two streams back to back
    off = np.array([a_off[0], a_off[2]], np.uint64)
    ln = np.array([a_ln[0] + a_ln[1], a_ln[2] + a_ln[3]], np.uint64)
    blocks = (a_arena, off, ln, np.array([0, 2, 4], np.uint32), np.array(a_ln, np.uint64), np.array(a_ck, np.uint64))
    got, r = run(capi, "decompress_sort", 1, 3, blocks, (REC, KEY_OFF, KEY_LEN), recs.size)
    assert (r["status"] == 0).all() and got == model_sort(parts, REC, KEY_OFF, KEY_LEN)
    bad_ck = blocks[5].copy()
    bad_ck[3] ^= 1  # second slice of the second block
    got, r = run(capi, "decompress_sort", 1, 3, blocks[:5] + (bad_ck,), (REC, KEY_OFF, KEY_LEN), recs.size)
    assert list(r["status"]) == [0, capi.E_CHECKSUM] and r["bad_slice"][1] == 1 and r["n_records"] == 0


# ---------------------------------------------------------------------------------------------------------------
# 2. key shapes and record sizes
# ---------------------------------------------------------------------------------------------------------------
EDGE_BYTES = [0x00, 0x01, 0x7F, 0x80, 0xFE, 0xFF]


@pytest.mark.parametrize("where", ["start", "unaligned", "end"])
@pytest.mark.parametrize("kl", list(range(1, 17)))
def test_key_lengths_and_offsets(capi, kl, where):
    ko = {"start": 0, "unaligned": 3, "end": REC - kl}[where]
    rng = np.random.default_rng(kl * 10 + len(where))
    recs = random_records(rng, 3000, REC, ko, kl, EDGE_BYTES)
    check(capi, 1, 0, 3, split_blocks(recs, [1000, 2000]), REC, ko, kl)


@pytest.mark.parametrize("rb,ko,kl", [(1, 0, 1), (104, 2, 10), (4096, 4096 - 16, 16), (4096, 5, 7)])
def test_record_sizes(capi, rb, ko, kl):
    """1-byte records; TeraSort's; 4 KiB records, which the gather copies with a whole warp each"""
    rng = np.random.default_rng(rb + ko)
    n = {1: 100_000, 104: 20_000, 4096: 700}[rb]
    recs = random_records(rng, n, rb, ko, kl, EDGE_BYTES)
    third = n // 3
    check(capi, 1, 0, 2, split_blocks(recs, [third, third, n - 2 * third]), rb, ko, kl)
    check(capi, 0, 0, 0, split_blocks(recs, [n]), rb, ko, kl, dev=True)


def test_stable_for_equal_keys(capi):
    """two distinct keys only; each record carries its input position as a tag, which must come out ascending per key"""
    n = 50_000
    recs = np.zeros((n, REC), np.uint8)
    recs[:, KEY_OFF:KEY_OFF + KEY_LEN] = np.where(np.arange(n)[:, None] % 3 == 0, 0xFF, 0x00).astype(np.uint8)
    recs[:, 20:24] = np.arange(n, dtype="<u4").view(np.uint8).reshape(n, 4)
    got = check(capi, 3, 1, 1, split_blocks(recs, [n // 2, n - n // 2]), REC, KEY_OFF, KEY_LEN)
    out = np.frombuffer(got, np.uint8).reshape(n, REC)
    tags = out[:, 20:24].copy().view("<u4").ravel()
    lo = out[:, KEY_OFF] == 0
    assert lo[: int(lo.sum())].all()  # every 0x00 key before every 0xFF key (unsigned order)
    assert (np.diff(tags[lo].astype(np.int64)) > 0).all() and (np.diff(tags[~lo].astype(np.int64)) > 0).all()


def test_every_key_equal(capi):
    rng = np.random.default_rng(7)
    recs = random_records(rng, 10_000, REC, KEY_OFF, KEY_LEN, [0x42])
    plain = split_blocks(recs, [4000, 6000])
    assert check(capi, 2, 0, 3, plain, REC, KEY_OFF, KEY_LEN) == b"".join(plain)


def test_zero_blocks_empty_blocks_and_one_record(capi):
    for codec in (0, 1):
        r = capi.decompress_sort_packed(codec, np.zeros(1, np.uint8), [], [], np.zeros(1, np.uint8), REC, 2, 10)
        assert r["total"] == 0 and r["n_records"] == 0
        assert check(capi, codec, 0, 3, [b"", b"", b""], REC, KEY_OFF, KEY_LEN) == b""
        one = bytes(range(REC))
        assert check(capi, codec, 0, 3, [b"", one, b""], REC, KEY_OFF, KEY_LEN) == one


def test_more_than_2_pow_24_records_and_2_gib(capi):
    """16.8 M records of 136 bytes (2.3 GB decoded) in 16 LZ4 blocks: several decode chunks, 24+ bit record indices"""
    n, rb, ko, kl = (1 << 24) + 4096, 136, 4, 8
    rng = np.random.default_rng(11)
    recs = np.zeros((n, rb), np.uint8)
    recs[:, ko:ko + 6] = rng.integers(0, 4, (n, 6), dtype=np.uint8)  # ties
    recs[:, ko + 6:ko + 8] = rng.integers(0, 256, (n, 2), dtype=np.uint8)
    recs[:, 12:16] = np.arange(n, dtype="<u4").view(np.uint8).reshape(n, 4)
    sizes = [n // 16] * 15 + [n - 15 * (n // 16)]
    plain = split_blocks(recs, sizes)
    blocks = build_blocks(capi, 1, 0, 3, plain)
    del plain
    got, r = run(capi, "decompress_sort", 1, 3, blocks, (rb, ko, kl), recs.size)
    assert (r["status"] == 0).all() and r["n_records"] == n and r["total"] == recs.size
    key = recs[:, ko:ko + kl].copy().view(">u8").ravel()
    order = np.argsort(key, kind="stable")
    out = np.frombuffer(got, np.uint8).reshape(n, rb)
    assert np.array_equal(out[:, 12:16].copy().view("<u4").ravel(), order.astype(np.uint32))
    assert np.array_equal(out, recs[order])


# ---------------------------------------------------------------------------------------------------------------
# 3. errors
# ---------------------------------------------------------------------------------------------------------------
def test_bad_arguments(capi, oracle):
    blocks = build_blocks(capi, 1, 0, 0, [terasort_records(oracle, 100).tobytes()])
    for rb, ko, kl in [(REC, 2, 0), (REC, 2, 17), (REC, REC - 9, 10), (0, 0, 1), (10, 0, 11)]:
        with pytest.raises(capi.B2SError) as e:
            run(capi, "decompress_sort", 1, 0, blocks, (rb, ko, kl), 100 * REC)
        assert e.value.code == capi.E_ARG
    with pytest.raises(capi.B2SError) as e:
        run(capi, "decompress_sort", 1, 7, blocks, (REC, 2, 10), 100 * REC)
    assert e.value.code == capi.E_UNSUPPORTED


def test_bad_checksum_in_one_slice(capi, oracle):
    recs = terasort_records(oracle, 9000, seed=4)
    plain = split_blocks(recs, [3000, 3000, 3000])
    for codec in (0, 1, 2, 3):
        blocks = list(build_blocks(capi, codec, 1, 2, plain))
        blocks[5] = blocks[5].copy()
        blocks[5][1] ^= 0x10
        for dev in (False, True):
            got, r = run(capi, "decompress_sort", codec, 2, tuple(blocks), (REC, 2, 10), recs.size, dev)
            assert list(r["status"]) == [0, capi.E_CHECKSUM, 0] and r["bad_slice"][1] == 0
            assert r["n_records"] == 0 and got == b""


def test_block_that_is_not_whole_records(capi, oracle):
    recs = terasort_records(oracle, 300, seed=5).tobytes()
    plain = [recs[:100 * REC], recs[100 * REC:200 * REC - 1], recs[200 * REC - 1:]]
    for codec in (0, 1):
        blocks = build_blocks(capi, codec, 0, 3, plain)
        got, r = run(capi, "decompress_sort", codec, 3, blocks, (REC, 2, 10), len(recs))
        assert list(r["status"]) == [0, capi.E_CORRUPT, capi.E_CORRUPT] and r["n_records"] == 0 and got == b""
        assert b"block 1 " in capi.load().b2s_last_error()


def test_corrupt_stream(capi, oracle):
    recs = terasort_records(oracle, 6000, seed=6)
    plain = split_blocks(recs, [2000, 2000, 2000])
    for codec in (1, 2, 3):
        arena, off, ln, sb, sl, sc = build_blocks(capi, codec, 1, 0, plain)
        arena = arena.copy()
        arena[int(off[2]):int(off[2] + ln[2])] = 0xA5  # every byte of the third stream
        got, r = run(capi, "decompress_sort", codec, 0, (arena, off, ln, sb, sl, sc), (REC, 2, 10), recs.size)
        assert r["status"][2] == capi.E_CORRUPT and r["n_records"] == 0 and got == b""


def test_short_destination_reports_the_bytes_needed(capi, oracle):
    import ctypes as C
    recs = terasort_records(oracle, 1000, seed=8)
    arena, off, ln, sb, sl, sc = build_blocks(capi, 1, 0, 0, split_blocks(recs, [500, 500]))
    dst = np.zeros(recs.size, np.uint8)
    total, nrec = C.c_uint64(0), C.c_uint64(0)
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    rc = capi.load().b2s_decompress_sort_packed(1, 0, 2, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None,
                                                None, REC, 2, 10, dst.ctypes.data, recs.size - 1, C.byref(total),
                                                C.byref(nrec), st.ctypes.data, bad.ctypes.data)
    assert rc == capi.E_DST_TOO_SMALL and total.value == recs.size and nrec.value == 0


def test_more_records_than_u32_indices(capi):
    """2^32 one-byte records: rejected before anything is allocated for them (codec NONE, no checksum: the block bytes
    are never read)"""
    d = capi.dev_alloc(64)
    try:
        with pytest.raises(capi.B2SError) as e:
            capi.decompress_sort_dev(0, d, [0], [1 << 32], d, 64, 1, 0, 1)
        assert e.value.code == capi.E_ARG
    finally:
        capi.dev_free(d)


# ---------------------------------------------------------------------------------------------------------------
# 4. beside a concurrent compress on the write lane
# ---------------------------------------------------------------------------------------------------------------
def test_beside_a_concurrent_compress(capi, oracle):
    recs = terasort_records(oracle, 200_000, seed=9)
    plain = split_blocks(recs, [50_000] * 4)
    blocks = build_blocks(capi, 1, 0, 3, plain)
    want_sorted, _ = run(capi, "decompress_sort", 1, 3, blocks, (REC, 2, 10), recs.size)
    src = recs.ravel()
    offs = np.arange(0, src.size, 1 << 20, dtype=np.uint64)
    lens = np.minimum(np.uint64(1 << 20), np.uint64(src.size) - offs).astype(np.uint64)
    cdst = np.zeros(sum(capi.compress_bound(1, 0, int(l)) for l in lens) + 64, np.uint8)
    want_c = capi.compress_packed(1, src, offs, lens, cdst, 0, 3)
    want_bytes = cdst[: want_c["total"]].tobytes()
    out = {}

    def sorter():
        out["sort"] = [run(capi, "decompress_sort", 1, 3, blocks, (REC, 2, 10), recs.size)[0] for _ in range(3)]

    def compressor():
        res = []
        for _ in range(3):
            d = np.zeros_like(cdst)
            r = capi.compress_packed(1, src, offs, lens, d, 0, 3)
            res.append((d[: r["total"]].tobytes(), list(r["checksums"])))
        out["compress"] = res

    th = [threading.Thread(target=sorter), threading.Thread(target=compressor)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert all(s == want_sorted for s in out["sort"])
    assert all(b == want_bytes and c == list(want_c["checksums"]) for b, c in out["compress"])


# ---------------------------------------------------------------------------------------------------------------
# 5. a whole TeraSort shuffle: partition + compress by key range, then verify + decode + sort per reducer
# ---------------------------------------------------------------------------------------------------------------
def key_range_ids(recs, R):
    k = recs[:, 2:4].astype(np.uint64)
    return (((k[:, 0] << 8) | k[:, 1]) * R >> 16).astype(np.uint32)


@pytest.mark.parametrize("name,codec,level", [("lz4", 1, 0), ("zstd1", 3, 1), ("none", 0, 0)])
def test_terasort_end_to_end(capi, oracle, name, codec, level):
    M, R, per_map = 4, 16, 40_000
    maps = [terasort_records(oracle, per_map, seed=20 + m) for m in range(M)]
    outs = []
    for m in range(M):
        ids = key_range_ids(maps[m], R)
        cap = capi.partition_compress_bound(codec, 0, R, maps[m].size)
        dst = np.zeros(cap, np.uint8)
        r = capi.partition_compress_packed(codec, maps[m].ravel(), np.full(per_map, REC, np.uint32), ids, R, dst, 0,
                                           3, level)
        outs.append((dst[: r["total"]].copy(), r))
    sorted_all = []
    for red in range(R):
        blocks = [outs[m][0][int(outs[m][1]["dst_off"][red]):int(outs[m][1]["dst_off"][red] + outs[m][1]["dst_len"][red])]
                  for m in range(M)]
        lens = np.array([b.size for b in blocks], np.uint64)
        arena = np.concatenate(blocks + [np.zeros(1, np.uint8)])
        off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        ck = np.array([outs[m][1]["checksums"][red] for m in range(M)], np.uint64)
        decoded = sum(int(np.sum(key_range_ids(maps[m], R) == red)) for m in range(M)) * REC
        got, r = run(capi, "decompress_sort", codec, 3, (arena, off, lens, np.arange(M + 1, dtype=np.uint32), lens, ck),
                     (REC, 2, 10), decoded)
        assert (r["status"] == 0).all() and r["total"] == decoded
        sorted_all.append(got)
    out = np.frombuffer(b"".join(sorted_all), np.uint8).reshape(-1, REC)
    assert out.shape[0] == M * per_map
    keys = [bytes(k) for k in out[:, 2:12]]
    assert all(keys[i] <= keys[i + 1] for i in range(len(keys) - 1))  # TeraValidate: globally sorted
    assert out.tobytes() == model_sort([m.tobytes() for m in maps], REC, 2, 10)  # a permutation, stable by map order


@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_terasort_through_the_host_mirror(tmp_path, oracle, codec):
    """serialized-writer files of M maps, read back per reducer with b2sh_reader_read_sorted"""
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R, per_map = 3, 8, 5000
    maps = [terasort_records(oracle, per_map, seed=40 + m) for m in range(M)]
    for m in range(M):
        w = host.S3SerializedShuffleWriter(d, 0, m, R)
        for rec, p in zip(maps[m], key_range_ids(maps[m], R)):
            w.insertRecord(int(p), rec.tobytes())
        w.commit()
        w.close()
    got = []
    for red in range(R):
        rd = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        data, n = rd.readSorted(REC, 2, 10)
        rd.close()
        assert len(data) == n * REC
        got.append(data)
    assert b"".join(got) == model_sort([m.tobytes() for m in maps], REC, 2, 10)


@pytest.mark.parametrize("shape", ["terasort", "compressible"])
@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_blocks_larger_than_the_task_budget(tmp_path, oracle, codec, shape):
    """bsize = min(maxBufferSizeTask, block size): blocks above the 20,000-byte budget reach read_sorted as a buffered
    head plus a tail read through from the block stream, and must be staged whole.  The compressible records (zero
    payload) decode to more than 4x their compressed size, past the first output guess of read_sorted."""
    host = pkg.host
    d = mirror(tmp_path, codec, **{"spark.shuffle.s3.maxBufferSizeTask": 20_000})
    M, R, per_map = 2, 2, 4000
    maps = [terasort_records(oracle, per_map, seed=60 + m).copy() for m in range(M)]
    if shape == "compressible":
        for m in maps:
            m[:, 12:] = 0
    for m in range(M):
        w = host.S3SerializedShuffleWriter(d, 0, m, R)
        ids = key_range_ids(maps[m], R)
        ids[:5] = R - 1  # a few records keep the last reducer's blocks small
        ids[5:] = np.minimum(ids[5:], R - 2)
        for rec, p in zip(maps[m], ids):
            w.insertRecord(int(p), rec.tobytes())
        lens = w.commit()
        w.close()
        assert lens[0] > 20_000 > lens[R - 1] > 0
    for batch in (False, True):
        rd = host.S3ShuffleReader(d, 0, list(range(M)), 0, R, batch)
        data, n = rd.readSorted(REC, 2, 10)
        rd.close()
        assert n == M * per_map
        assert data == model_sort([m.tobytes() for m in maps], REC, 2, 10)
