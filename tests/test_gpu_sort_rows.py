"""Verify + decompress + row-sort in one call (b2s_decompress_sort_rows_*): a reduce task's blocks of UnsafeRowSerializer
records ([int32 big-endian size][row]) in, every record out, sorted by one typed key of the row (unsigned bytes, signed
little-endian int32 / int64), nulls first, stable.  The model parses the decoded streams in Python and sorts the
records stably by (non-null flag, key); the call must be byte for byte that model."""
import ctypes as C

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from rows_model import CHECKSUMS, CODECS, KEY_BYTES, KEY_INT32, KEY_INT64, blocks_of, build_blocks, mirror, \
    model_sort, run, stream, write_maps

pytestmark = pytest.mark.gpu

KEY_LEN = {KEY_INT32: 4, KEY_INT64: 8}
INT_EDGES = {KEY_INT32: [-2**31, 2**31 - 1, 0, -1, 1], KEY_INT64: [-2**63, 2**63 - 1, 0, -1, 1, -2**31 - 1, 2**31]}


# ---------------------------------------------------------------------------------------------------------------
# model and helpers
# ---------------------------------------------------------------------------------------------------------------
def make_rows(rng, n, kt, ko, kl, nf=-1, lens=None, keys=None, null_frac=0.0, tag_at=None):
    """n random rows of lens[i] bytes (default 56) with the key at ko and, when nf >= 0, the null bit set with
    probability null_frac.  keys: the key values (ints, or bytes); tag_at: the row's index as 4 bytes there."""
    rows = []
    for i in range(n):
        ln = int(lens[i]) if lens is not None else 56
        r = bytearray(rng.integers(0, 256, ln, dtype=np.uint8).tobytes())
        if keys is not None:
            k = keys[i]
            r[ko:ko + kl] = k if isinstance(k, (bytes, bytearray)) else int(k).to_bytes(kl, "little", signed=True)
        if nf >= 0:
            w = 8 * (nf >> 6)
            v = int.from_bytes(r[w:w + 8], "little") & ~(1 << (nf & 63))
            if rng.random() < null_frac:
                v |= 1 << (nf & 63)
            r[w:w + 8] = v.to_bytes(8, "little")
        if tag_at is not None:
            r[tag_at:tag_at + 4] = i.to_bytes(4, "little")
        rows.append(bytes(r))
    return rows


def int_keys(rng, n, kt, ties=False):
    if ties:
        return rng.integers(-3, 3, n)
    bits = 32 if kt == KEY_INT32 else 64
    k = [int(x) for x in rng.integers(-2**(bits - 1), 2**(bits - 1) - 1, n, dtype=np.int64)]
    edges = INT_EDGES[kt]
    for j in range(0, n, 7):
        k[j] = edges[(j // 7) % len(edges)]
    return k


def check(capi, codec, level, alg, plain, kt, ko, kl, nf=-1, dev=False, blocks=None):
    blocks = blocks or build_blocks(capi, codec, level, alg, plain)
    total = sum(len(b) for b in plain)
    got, r = run(capi, "decompress_sort_rows", codec, alg, blocks, (kt, ko, kl, nf), total, dev)
    assert (r["status"] == 0).all(), r["status"]
    want, n = model_sort(plain, [(kt, ko, kl, nf)])
    assert r["total"] == total and r["n_records"] == n
    assert got == want
    return got


# ---------------------------------------------------------------------------------------------------------------
# 1. every codec x checksum x key type, _dev against _packed
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kt", [KEY_BYTES, KEY_INT32, KEY_INT64])
@pytest.mark.parametrize("alg", CHECKSUMS)
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_sorts_like_the_model(capi, name, codec, level, alg, kt):
    rng = np.random.default_rng(codec * 100 + alg * 10 + kt)
    n, ko = 6000, 16  # a one-word null bitset, then the key field
    kl = KEY_LEN.get(kt, 10)
    keys = None if kt == KEY_BYTES else int_keys(rng, n, kt)
    lens = rng.integers(32, 120, n)
    rows = make_rows(rng, n, kt, ko, kl, nf=1, lens=lens, keys=keys, null_frac=0.05)
    plain = blocks_of(rows, [2500, 0, 1, 1499, 2000])  # an empty block and a one-record block among them
    a = check(capi, codec, level, alg, plain, kt, ko, kl, nf=1)
    b = check(capi, codec, level, alg, plain, kt, ko, kl, nf=1, dev=True)
    assert a == b


def test_timing_reports_the_framing_step(capi):
    rng = np.random.default_rng(5)
    rows = make_rows(rng, 50_000, KEY_INT64, 8, 8, lens=rng.integers(16, 100, 50_000))
    check(capi, 1, 0, 3, blocks_of(rows, [25_000, 25_000]), KEY_INT64, 8, 8, dev=True)
    t = capi.last_timing()
    assert t["dominant_launches"] > 0 and 0 < t["dominant_ms"] <= t["top_kernel_ms"] <= t["kernel_ms"]


# ---------------------------------------------------------------------------------------------------------------
# 2. keys, nulls and stability
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kt", [KEY_INT32, KEY_INT64])
@pytest.mark.parametrize("ties", [False, True])
def test_signed_edges_and_ties(capi, kt, ties):
    rng = np.random.default_rng(kt * 2 + ties)
    n, ko, kl = 20_000, 24, KEY_LEN[kt]
    rows = make_rows(rng, n, kt, ko, kl, keys=int_keys(rng, n, kt, ties), lens=np.full(n, 40), tag_at=36)
    got = check(capi, 1, 0, 3, blocks_of(rows, [7000, 13_000]), kt, ko, kl)
    if ties:  # equal keys keep input order: the tags of each key come out ascending
        out = [got[i:i + 44] for i in range(0, len(got), 44)]
        key = [int.from_bytes(r[4 + ko:4 + ko + kl], "little", signed=True) for r in out]
        tag = [int.from_bytes(r[40:44], "little") for r in out]
        assert key == sorted(key)
        assert all(tag[i] < tag[i + 1] for i in range(len(out) - 1) if key[i] == key[i + 1])


@pytest.mark.parametrize("nf", [0, 5, 63, 64, 70, 127])
def test_nulls_first_and_stable(capi, nf):
    """nulls before every key, in input order; a null field >= 64 reads the second bitset word"""
    rng = np.random.default_rng(nf)
    n = 10_000
    ko = 16 if nf < 64 else 24  # one or two bitset words in front of the key
    rows = make_rows(rng, n, KEY_INT64, ko, 8, nf=nf, keys=int_keys(rng, n, KEY_INT64, ties=True),
                     lens=np.full(n, 48), null_frac=0.3, tag_at=40)
    got = check(capi, 3, 1, 2, blocks_of(rows, [3000, 3000, 4000]), KEY_INT64, ko, 8, nf=nf)
    out = [got[i:i + 52] for i in range(0, len(got), 52)]
    w = 4 + 8 * (nf >> 6)
    null = [(int.from_bytes(r[w:w + 8], "little") >> (nf & 63)) & 1 for r in out]
    k = null.index(0)
    assert 0 < k and all(null[:k]) and not any(null[k:])
    tags = [int.from_bytes(r[44:48], "little") for r in out[:k]]
    assert tags == sorted(tags)


@pytest.mark.parametrize("kl,ko", [(1, 0), (3, 5), (10, 8), (16, 0), (16, 33)])
def test_byte_keys(capi, kl, ko):
    rng = np.random.default_rng(kl * 7 + ko)
    n = 8000
    keys = [bytes(rng.choice(np.array([0, 1, 0x7F, 0x80, 0xFF], np.uint8), kl)) for _ in range(n)]
    rows = make_rows(rng, n, KEY_BYTES, ko, kl, nf=2, lens=rng.integers(ko + kl, 90, n), keys=keys, null_frac=0.1)
    check(capi, 2, 0, 1, blocks_of(rows, [4000, 4000]), KEY_BYTES, ko, kl, nf=2)


# ---------------------------------------------------------------------------------------------------------------
# 3. row lengths
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,codec,level", [("none", 0, 0), ("lz4", 1, 0), ("zstd1", 3, 1)])
def test_row_lengths_across_the_gather_split(capi, name, codec, level):
    """from the shortest row that holds the key (12 bytes: key at 4) to 300 bytes, either side of the gather's 256-byte
    lane / warp split"""
    rng = np.random.default_rng(codec)
    n = 30_000
    lens = rng.integers(12, 301, n)
    lens[:289] = np.arange(12, 301)
    rows = make_rows(rng, n, KEY_INT64, 4, 8, keys=int_keys(rng, n, KEY_INT64), lens=lens)
    check(capi, codec, level, 3, blocks_of(rows, [10_000, 20_000]), KEY_INT64, 4, 8)
    check(capi, codec, level, 3, blocks_of(rows, [10_000, 20_000]), KEY_INT64, 4, 8, dev=True)


@pytest.mark.parametrize("name,codec,level", CODECS)
def test_rows_longer_than_a_window_and_a_codec_block(capi, name, codec, level):
    """a few ~100 KiB rows among short ones: longer than the framing's staging windows and a 32 KiB codec block"""
    rng = np.random.default_rng(30 + codec)
    n = 3000
    lens = rng.integers(16, 200, n)
    for j in (0, 17, 1500, 1501, n - 1):
        lens[j] = 100_000 + j
    rows = make_rows(rng, n, KEY_INT32, 8, 4, nf=0, keys=int_keys(rng, n, KEY_INT32), lens=lens, null_frac=0.05)
    check(capi, codec, level, 2, blocks_of(rows, [1501, 1499]), KEY_INT32, 8, 4, nf=0)


@pytest.mark.parametrize("name,codec,level", [("lz4", 1, 0), ("snappy", 2, 0), ("zstd3", 3, 3)])
def test_size_prefixes_straddle_codec_blocks(capi, name, codec, level):
    """rows sized so that size prefixes start 1, 2 and 3 bytes before 32 KiB codec-block boundaries"""
    rng = np.random.default_rng(40 + codec)
    rows, at = [], 0
    for b in range(1, 40):
        target = b * 32768 - (b % 3 + 1)  # where the next prefix starts
        while target - at > 400:  # the last row before the target is then 190..396 bytes
            ln = int(rng.integers(20, 200))
            rows.append(ln)
            at += 4 + ln
        rows.append(target - at - 4)
        at = target
    keys = int_keys(rng, len(rows), KEY_INT64)
    rows = make_rows(rng, len(rows), KEY_INT64, 8, 8, keys=keys, lens=np.array(rows))
    check(capi, codec, level, 3, [stream(rows)], KEY_INT64, 8, 8)


# ---------------------------------------------------------------------------------------------------------------
# 4. block shapes
# ---------------------------------------------------------------------------------------------------------------
def test_zero_blocks_empty_blocks_and_one_record(capi):
    for codec in (0, 1):
        r = capi.decompress_sort_rows_packed(codec, np.zeros(1, np.uint8), [], [], np.zeros(1, np.uint8), KEY_INT32, 0, 4)
        assert r["total"] == 0 and r["n_records"] == 0
        assert check(capi, codec, 0, 3, [b"", b"", b""], KEY_INT32, 0, 4) == b""
        one = stream([bytes(range(40))])
        assert check(capi, codec, 0, 3, [b"", one, b""], KEY_INT32, 0, 4, nf=-1) == one


def test_two_thousand_tiny_blocks(capi):
    rng = np.random.default_rng(50)
    sizes = [int(x) for x in rng.integers(0, 4, 2000)]
    rows = make_rows(rng, sum(sizes), KEY_INT64, 8, 8, nf=3, keys=int_keys(rng, sum(sizes), KEY_INT64, True),
                     lens=rng.integers(16, 40, sum(sizes)), null_frac=0.1)
    check(capi, 1, 0, 3, blocks_of(rows, sizes), KEY_INT64, 8, 8, nf=3)
    check(capi, 0, 0, 0, blocks_of(rows, sizes), KEY_INT64, 8, 8, nf=3, dev=True)


def test_one_block_of_a_million_records(capi):
    """1.2 M records in one block: the framing walks one serial chain of that length"""
    n, L = 1_200_000, 16  # row: null bitset word, int64 key
    rng = np.random.default_rng(51)
    rec = np.zeros((n, 4 + L), np.uint8)
    rec[:, :4] = np.frombuffer(L.to_bytes(4, "big"), np.uint8)
    nulls = rng.random(n) < 0.05
    rec[:, 4:12] = np.where(nulls, 1, 0).astype("<u8").view(np.uint8).reshape(n, 8)
    keys = rng.integers(-1000, 1000, n).astype("<i8")
    rec[:, 12:20] = keys.view(np.uint8).reshape(n, 8)
    for codec in (1, 0):
        blocks = build_blocks(capi, codec, 0, 3, [rec.tobytes()])
        got, r = run(capi, "decompress_sort_rows", codec, 3, blocks, (KEY_INT64, 8, 8, 0), rec.size)
        assert (r["status"] == 0).all() and r["n_records"] == n
        order = np.lexsort((np.where(nulls, 0, keys), ~nulls))  # stable: non-null flag, then key
        assert got == rec[order].tobytes()


def test_block_of_two_concatenated_streams(capi):
    """a ShuffleBlockBatchId block: two partition streams back to back, one checksum slice each"""
    rng = np.random.default_rng(52)
    rows = make_rows(rng, 8000, KEY_INT32, 8, 4, keys=int_keys(rng, 8000, KEY_INT32), lens=rng.integers(12, 80, 8000))
    parts = blocks_of(rows, [3000, 1000, 2500, 1500])
    a_arena, a_off, a_ln, _, _, a_ck = build_blocks(capi, 2, 0, 3, parts)
    off = np.array([a_off[0], a_off[2]], np.uint64)
    ln = np.array([a_ln[0] + a_ln[1], a_ln[2] + a_ln[3]], np.uint64)
    blocks = (a_arena, off, ln, np.array([0, 2, 4], np.uint32), np.array(a_ln, np.uint64), np.array(a_ck, np.uint64))
    check(capi, 2, 0, 3, parts, KEY_INT32, 8, 4, blocks=blocks)


# ---------------------------------------------------------------------------------------------------------------
# 5. errors
# ---------------------------------------------------------------------------------------------------------------
def good_rows(rng, n=500):
    return make_rows(rng, n, KEY_INT64, 8, 8, keys=int_keys(rng, n, KEY_INT64), lens=rng.integers(24, 60, n))


@pytest.mark.parametrize("rule", ["negative", "past_end", "cut_prefix", "short_for_key", "short_for_null"])
def test_each_corruption_rule_fails_its_block(capi, rule):
    rng = np.random.default_rng(60)
    good = [stream(good_rows(rng)) for _ in range(3)]
    head = stream(good_rows(rng, 10))
    bad = {
        "negative": head + (-5).to_bytes(4, "big", signed=True) + bytes(16),
        "past_end": head + (100).to_bytes(4, "big") + bytes(50),
        "cut_prefix": head + bytes(2),
        "short_for_key": head + stream([bytes(15)]),      # key at 8..16
        "short_for_null": head + stream([bytes(17)]),     # holds the key, not the third bitset word (bytes 16..24)
    }[rule]
    nf = 130 if rule == "short_for_null" else 70
    plain = [good[0], bad, good[1], good[2]]
    for codec in (0, 1, 3):
        blocks = build_blocks(capi, codec, 1, 3, plain)
        for dev in (False, True):
            got, r = run(capi, "decompress_sort_rows", codec, 3, blocks, (KEY_INT64, 8, 8, nf), sum(map(len, plain)),
                         dev)
            assert list(r["status"]) == [0, capi.E_CORRUPT, 0, 0] and r["n_records"] == 0 and got == b""
            err = capi.load().b2s_last_error()
            assert b"block 1: " in err and (b"at byte %d:" % len(head)) in err, err


def test_bad_checksum_in_one_block(capi):
    rng = np.random.default_rng(61)
    plain = [stream(good_rows(rng)) for _ in range(3)]
    for codec in (0, 1, 2, 3):
        blocks = list(build_blocks(capi, codec, 1, 2, plain))
        blocks[5] = blocks[5].copy()
        blocks[5][1] ^= 0x10
        for dev in (False, True):
            got, r = run(capi, "decompress_sort_rows", codec, 2, tuple(blocks), (KEY_INT64, 8, 8, -1),
                         sum(map(len, plain)), dev)
            assert list(r["status"]) == [0, capi.E_CHECKSUM, 0] and r["bad_slice"][1] == 0
            assert r["n_records"] == 0 and got == b""


def test_short_destination_reports_the_bytes_needed(capi):
    rng = np.random.default_rng(62)
    plain = [stream(good_rows(rng)) for _ in range(2)]
    arena, off, ln, _, _, _ = build_blocks(capi, 1, 0, 0, plain)
    need = sum(map(len, plain))
    dst = np.zeros(need, np.uint8)
    total, nrec = C.c_uint64(0), C.c_uint64(0)
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    rc = capi.load().b2s_decompress_sort_rows_packed(1, 0, 2, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, None,
                                                     None, None, KEY_INT64, 8, 8, -1, dst.ctypes.data, need - 1,
                                                     C.byref(total), C.byref(nrec), st.ctypes.data, bad.ctypes.data)
    assert rc == capi.E_DST_TOO_SMALL and total.value == need and nrec.value == 0


@pytest.mark.parametrize("kt,ko,kl,nf", [(3, 0, 4, -1), (KEY_BYTES, 0, 0, -1), (KEY_BYTES, 0, 17, -1),
                                         (KEY_INT32, 0, 8, -1), (KEY_INT32, 0, 3, -1), (KEY_INT64, 0, 4, -1),
                                         (KEY_INT64, 0, 16, -1), (KEY_INT64, 8, 8, -2)])
def test_bad_arguments(capi, kt, ko, kl, nf):
    rng = np.random.default_rng(63)
    blocks = build_blocks(capi, 1, 0, 0, [stream(good_rows(rng))])
    with pytest.raises(capi.B2SError) as e:
        run(capi, "decompress_sort_rows", 1, 0, blocks, (kt, ko, kl, nf), 1 << 16)
    assert e.value.code == capi.E_ARG


# ---------------------------------------------------------------------------------------------------------------
# 6. end to end: UnsafeRow records written by several maps, each reducer read back sorted
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,codec,level", [("snappy", 2, 0), ("lz4", 1, 0), ("none", 0, 0)])
def test_sql_exchange_end_to_end(capi, name, codec, level):
    M, R, per_map = 4, 8, 20_000
    maps = []
    for m in range(M):
        rng = np.random.default_rng(70 + m)
        rows = make_rows(rng, per_map, KEY_INT64, 8, 8, nf=0, keys=int_keys(rng, per_map, KEY_INT64, ties=True),
                         lens=8 * rng.integers(2, 15, per_map), null_frac=0.05)
        maps.append((rows, rng.integers(0, R, per_map).astype(np.uint32)))
    outs = []
    for rows, ids in maps:
        recs = np.frombuffer(stream(rows), np.uint8)
        rec_len = np.array([4 + len(r) for r in rows], np.uint32)
        dst = np.zeros(capi.partition_compress_bound(codec, 0, R, recs.size), np.uint8)
        r = capi.partition_compress_packed(codec, recs, rec_len, ids, R, dst, 0, 3, level)
        outs.append((dst[: r["total"]].copy(), r))
    for red in range(R):
        blocks = [o[int(r["dst_off"][red]):int(r["dst_off"][red] + r["dst_len"][red])] for o, r in outs]
        lens = np.array([b.size for b in blocks], np.uint64)
        arena = np.concatenate(blocks + [np.zeros(1, np.uint8)])
        off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        ck = np.array([r["checksums"][red] for _, r in outs], np.uint64)
        plain = [stream([row for row, p in zip(rows, ids) if p == red]) for rows, ids in maps]
        check(capi, codec, level, 3, plain, KEY_INT64, 8, 8, nf=0,
              blocks=(arena, off, lens, np.arange(M + 1, dtype=np.uint32), lens, ck))


# ---------------------------------------------------------------------------------------------------------------
# 7. the host mirror: b2sh_reader_read_sorted_rows over the serialized writer's files
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_reads_rows_sorted(tmp_path, codec):
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R, per_map = 3, 4, 3000
    maps = []
    for m in range(M):
        rng = np.random.default_rng(80 + m)
        rows = make_rows(rng, per_map, KEY_INT32, 8, 4, nf=0, keys=int_keys(rng, per_map, KEY_INT32, ties=True),
                         lens=rng.integers(12, 100, per_map), null_frac=0.05)
        maps.append((rows, rng.integers(0, R, per_map)))
    write_maps(host, d, maps, R)
    for red in range(R):
        rd = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        data, n = rd.readSortedRows(KEY_INT32, 8, 4, 0)
        rd.close()
        want, wn = model_sort([stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps],
                              [(KEY_INT32, 8, 4, 0)])
        assert n == wn and data == want
    d.close()


def test_host_mirror_checksum_and_malformed_errors(tmp_path):
    host = pkg.host
    d = mirror(tmp_path, "lz4")
    rng = np.random.default_rng(90)
    rows = make_rows(rng, 2000, KEY_INT64, 8, 8, keys=int_keys(rng, 2000, KEY_INT64), lens=np.full(2000, 40))
    write_maps(host, d, [(rows, np.zeros(2000, np.int64))], 2)
    # map 1: a partition whose stream is not whole rows (a row cut short by 3 bytes)
    w = host.S3SerializedShuffleWriter(d, 0, 1, 2)
    w.insertRecord(0, (40).to_bytes(4, "big") + bytes(37))
    w.commit()
    w.close()
    rd = host.S3ShuffleReader(d, 0, [1], 0, 1)
    with pytest.raises(host.IOException):
        rd.readSortedRows(KEY_INT64, 8, 8, -1)
    rd.close()
    path = d.getPath("data", 0, 0)
    raw = bytearray(open(path, "rb").read())
    raw[30] ^= 0x04
    open(path, "wb").write(raw)
    rd = host.S3ShuffleReader(d, 0, [0], 0, 1)
    with pytest.raises(host.SparkException, match=r"Invalid checksum detected for shuffle_0_0_0$"):
        rd.readSortedRows(KEY_INT64, 8, 8, -1)
    rd.close()
    d.close()
