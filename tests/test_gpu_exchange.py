"""The exchange cache (b2s_exchange_*, b2s_partition_compress_cached_packed): map outputs kept in HBM by the serialized
writer's call and read back by reducers on the same device, plain or key-sorted mixed with fetched blocks.  The models:
the cached store is byte for byte b2s_partition_compress_packed; a plain read is the stably partitioned records; a
sorted read is byte for byte b2s_decompress_sort_packed over every map's fetched blocks in source order."""
import threading

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg

pytestmark = pytest.mark.gpu

CODECS = [("none", 0, 0), ("lz4", 1, 0), ("snappy", 2, 0), ("zstd1", 3, 1), ("zstd3", 3, 3)]
LAYOUTS = [(104, 2, 10), (104, 3, 7), (64, 5, 16)]  # TeraSort; a key at an odd offset; a 16-byte key


@pytest.fixture
def cache(capi):
    """a generous budget on device 0; everything cached is released afterwards"""
    capi.exchange_set_budget(8 << 30)
    yield capi
    capi.exchange_set_budget(0)
    for s in range(64):
        capi.exchange_remove(s, -1)


def map_records(rng, n, rb, ko, kl, R):
    """n random records with keys drawn from a small alphabet (ties), range-partitioned on the first key byte"""
    recs = rng.integers(0, 256, (n, rb), dtype=np.uint8)
    recs[:, ko:ko + kl] = rng.choice(np.array([0, 1, 0x7f, 0x80, 0xff], np.uint8), (n, kl))
    recs[:, ko] = rng.integers(0, 256, n, dtype=np.uint8)
    ids = (recs[:, ko].astype(np.int64) * R) >> 8
    return recs, ids.astype(np.uint32)


def partitioned(recs, ids, R):
    """the model of the partition step: records stably sorted by reduce id, and the partition offsets"""
    order = np.argsort(ids, kind="stable")
    rb = recs.shape[1]
    start = np.concatenate([[0], np.cumsum(np.bincount(ids, minlength=R))]) * rb
    return recs[order].tobytes(), start


def store(capi, shuffle, map_id, codec, level, alg, recs, ids, R, rec_len=None, compare=True):
    flat = recs.reshape(-1)
    rl = np.full(len(ids), recs.shape[1], np.uint32) if rec_len is None else rec_len
    bound = capi.partition_compress_bound(codec, 0, R, flat.size) + 64
    dst = np.zeros(bound, np.uint8)
    r = capi.partition_compress_cached_packed(shuffle, map_id, codec, flat, rl, ids, R, dst, 0, alg, level)
    r["data"] = dst[: r["total"]].copy()
    if compare:
        ref = np.zeros(bound, np.uint8)
        q = capi.partition_compress_packed(codec, flat, rl, ids, R, ref, 0, alg, level)
        assert r["total"] == q["total"] and bytes(r["data"]) == bytes(ref[: q["total"]])
        for k in ("dst_off", "dst_len", "checksums", "status"):
            assert (r[k] == q[k]).all(), k
    return r


def fetched_blocks(r, s, e, batch):
    """the .data ranges a reducer of [s, e) fetches from one map output: one batch block, or one per reduce id;
    empty ones are skipped, as the reader does -> list of (bytes, slice lengths, slice checksums)"""
    ranges = [(s, e)] if batch else [(q, q + 1) for q in range(s, e)]
    out = []
    for a, b in ranges:
        lo, n = int(r["dst_off"][a]), int(r["dst_len"][a:b].sum())
        if n:
            out.append((bytes(r["data"][lo:lo + n]), list(r["dst_len"][a:b]), list(r["checksums"][a:b])))
    return out


def arena_of(blocks):
    """blocks -> (arena, off, len, slice_base, slice_len, slice_checksum)"""
    off, ln, sb, sl, sc = [], [], [0], [], []
    at = 0
    for b, lens, cks in blocks:
        off.append(at)
        ln.append(len(b))
        at += len(b)
        sl += lens
        sc += cks
        sb.append(len(sl))
    arena = np.frombuffer(b"".join(b for b, _, _ in blocks), np.uint8) if at else np.zeros(1, np.uint8)
    return (arena, np.array(off, np.uint64), np.array(ln, np.uint64), np.array(sb, np.uint32),
            np.array(sl, np.uint64), np.array(sc, np.uint64))


def sources(outs, hit, s, e, batch):
    """the sources of a mixed read in map order: one cached source for a hit, else the map's fetched blocks"""
    ids, cached, blocks = [], [], []
    for m, r in enumerate(outs):
        if hit[m]:
            ids.append(m)
            cached.append(True)
            blocks.append((b"", [], []))
        else:
            for b in fetched_blocks(r, s, e, batch):
                ids.append(m)
                cached.append(False)
                blocks.append(b)
    return ids, cached, blocks


def sort_reference(capi, codec, alg, outs, s, e, batch, rb, ko, kl):
    blocks = [b for r in outs for b in fetched_blocks(r, s, e, batch)]
    arena, off, ln, sb, sl, sc = arena_of(blocks)
    dst = np.zeros(rb * 200_000, np.uint8)
    q = capi.decompress_sort_packed(codec, arena, off, ln, dst, rb, ko, kl, alg, sb, sl, sc)
    assert (q["status"] == 0).all()
    return dst[: q["total"]].tobytes(), q


def read_sort(capi, shuffle, s, e, ids, cached, codec, alg, blocks, rb, ko, kl, cap, dev=False):
    arena, off, ln, sb, sl, sc = arena_of(blocks)
    if not dev:
        dst = np.zeros(max(cap, 1), np.uint8)
        r = capi.exchange_read_sort_packed(shuffle, s, e, ids, cached, codec, arena, off, ln, dst[:cap], rb, ko, kl,
                                           alg, sb, sl, sc)
        return (dst[: r["total"]].tobytes() if r["n_records"] else b""), r
    d_src = capi.dev_alloc(max(arena.size, 1))
    d_dst = capi.dev_alloc(max(cap, 1))
    try:
        capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        r = capi.exchange_read_sort_dev(shuffle, s, e, ids, cached, codec, d_src, off, ln, d_dst, cap, rb, ko, kl,
                                        alg, sb, sl, sc)
        out = np.zeros(max(r["total"], 1), np.uint8)
        if r["n_records"] and r["total"]:
            capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        return (out[: r["total"]].tobytes() if r["n_records"] else b""), r
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)


# ---------------------------------------------------------------------------------------------------------------
# store
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", [0, 1, 2, 3])
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_cached_store_is_byte_identical_and_cached(cache, name, codec, level, alg):
    rng = np.random.default_rng(codec * 10 + alg)
    R = 7
    recs, ids = map_records(rng, 3000, 104, 2, 10, R)
    r = store(cache, 1, 5, codec, level, alg, recs, ids, R)
    assert r["cached"] == 1
    want, start = partitioned(recs, ids, R)
    hits, ln = cache.exchange_lookup(1, 0, R, [5, 6])
    assert hits == 1 and ln[0] == len(want) and ln[1] == cache.NOT_RESIDENT
    out = np.zeros(len(want) + 16, np.uint8)
    q = cache.exchange_read_packed(1, 0, R, [5], out)
    assert q["status"][0] == 0 and q["total"] == len(want) and out[: len(want)].tobytes() == want


# ---------------------------------------------------------------------------------------------------------------
# plain read
# ---------------------------------------------------------------------------------------------------------------
def test_plain_read_ranges(cache, oracle):
    rng = np.random.default_rng(3)
    R = 16
    outs, models = [], []
    for m in range(3):
        recs, ids = map_records(rng, 4000 + 500 * m, 104, 2, 10, R)
        store(cache, 2, m, 1, 0, 3, recs, ids, R)
        models.append(partitioned(recs, ids, R))
    for s, e in [(0, 1), (5, 6), (15, 16), (2, 9), (0, 16), (5, 5), (16, 16)]:
        want = [mod[0][mod[1][s]:mod[1][e]] for mod in models]
        out = np.zeros(sum(len(w) for w in want) + 1, np.uint8)
        q = cache.exchange_read_packed(2, s, e, [0, 1, 9, 2], out)
        assert list(q["status"]) == [0, 0, cache.E_NOT_CACHED, 0]
        got = [out[int(o):int(o) + int(n)].tobytes() for o, n in zip(q["dst_off"], q["dst_len"])]
        assert got == [want[0], want[1], b"", want[2]]
        assert q["total"] == sum(len(w) for w in want)
        hits, ln = cache.exchange_lookup(2, s, e, [0, 1, 9, 2])
        assert hits == 3 and list(ln) == [len(want[0]), len(want[1]), cache.NOT_RESIDENT, len(want[2])]
    # the .data slices decode to the same partitions
    data = store(cache, 2, 7, 1, 0, 0, *map_records(np.random.default_rng(9), 2000, 104, 2, 10, R), R)
    part = np.zeros(data["total"] + 1, np.uint8)
    q = cache.exchange_read_packed(2, 3, 4, [7], part)
    stream = bytes(data["data"][int(data["dst_off"][3]):int(data["dst_off"][3] + data["dst_len"][3])])
    assert oracle.lz4block_decompress(stream) == part[: q["total"]].tobytes()
    with pytest.raises(cache.B2SError) as e:
        cache.exchange_read_packed(2, 0, R + 1, [0], np.zeros(1 << 20, np.uint8))
    assert e.value.code == cache.E_ARG


def test_short_destination_reports_the_bytes_needed(cache):
    import ctypes as C
    rng = np.random.default_rng(4)
    recs, ids = map_records(rng, 1000, 104, 2, 10, 2)
    store(cache, 3, 0, 0, 0, 0, recs, ids, 2)
    L = cache.load()
    mid = np.zeros(1, np.int64)
    dst = np.zeros(100, np.uint8)
    off, dl, st = np.zeros(1, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.int32)
    total = C.c_uint64(0)
    rc = L.b2s_exchange_read_packed(3, 0, 2, 1, mid.ctypes.data, dst.ctypes.data, dst.size, off.ctypes.data,
                                    dl.ctypes.data, C.byref(total), st.ctypes.data)
    assert rc == cache.E_DST_TOO_SMALL and total.value == 1000 * 104
    blocks = [(b"", [], [])]
    with pytest.raises(cache.B2SError) as e:
        read_sort(cache, 3, 0, 2, [0], [True], 0, 0, blocks, 104, 2, 10, 1000)
    assert e.value.code == cache.E_DST_TOO_SMALL and str(1000 * 104) in str(e.value)


# ---------------------------------------------------------------------------------------------------------------
# sorted read, mixed with fetched blocks
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rb,ko,kl", LAYOUTS)
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_sorted_read_matches_decompress_sort(cache, name, codec, level, rb, ko, kl):
    rng = np.random.default_rng(codec * 7 + kl)
    R, M, s, e = 4, 6, 1, 3
    outs = []
    for m in range(M):
        recs, ids = map_records(rng, 1500 + 300 * m, rb, ko, kl, R)
        outs.append(store(cache, 4, m, codec, level, 3, recs, ids, R, compare=False))
    for batch in (True, False):
        want, q = sort_reference(cache, codec, 3, outs, s, e, batch, rb, ko, kl)
        masks = [[True] * M, [False] * M] + [list(rng.integers(0, 2, M).astype(bool)) for _ in range(3)]
        for hit in masks:
            ids, cached, blocks = sources(outs, hit, s, e, batch)
            for dev in (False, True):
                got, r = read_sort(cache, 4, s, e, ids, cached, codec, 3, blocks, rb, ko, kl, len(want) + 64, dev)
                assert (r["status"] == 0).all(), r["status"]
                assert r["n_records"] == q["n_records"] and r["total"] == q["total"]
                assert got == want, (batch, hit, dev)
    t = cache.last_timing()
    assert t["kernel_ms"] >= t["top_kernel_ms"] > 0


def test_removed_source_is_not_cached_and_nothing_is_sorted(cache):
    rng = np.random.default_rng(5)
    outs = [store(cache, 5, m, 1, 0, 3, *map_records(rng, 2000, 104, 2, 10, 3), 3, compare=False) for m in range(3)]
    assert cache.exchange_remove(5, 1) == 1
    ids, cached, blocks = sources(outs, [True, True, False], 0, 3, True)
    got, r = read_sort(cache, 5, 0, 3, ids, cached, 1, 3, blocks, 104, 2, 10, 1 << 20)
    assert got == b"" and r["n_records"] == 0
    assert list(r["status"]) == [0, cache.E_NOT_CACHED, 0]


def test_fetched_block_failures_with_cached_sources(cache):
    rng = np.random.default_rng(6)
    outs = [store(cache, 6, m, 1, 0, 3, *map_records(rng, 2000, 104, 2, 10, 3), 3, compare=False) for m in range(3)]
    ids, cached, blocks = sources(outs, [True, False, True], 0, 3, False)
    k = cached.index(False) + 1  # the second fetched block of map 1
    b, lens, cks = blocks[k]
    blocks[k] = (b, lens, [cks[0] ^ 1])
    got, r = read_sort(cache, 6, 0, 3, ids, cached, 1, 3, blocks, 104, 2, 10, 1 << 20)
    assert got == b"" and r["n_records"] == 0
    assert r["status"][k] == cache.E_CHECKSUM and r["bad_slice"][k] == 0
    assert all(r["status"][i] == 0 for i in range(len(ids)) if i != k)
    corrupt = bytearray(b)
    corrupt[0:8] = b"\xff" * 8  # the LZ4Block magic
    blocks[k] = (bytes(corrupt), lens, cks)
    got, r = read_sort(cache, 6, 0, 3, ids, cached, 1, 0, blocks, 104, 2, 10, 1 << 20)
    assert got == b"" and r["status"][k] == cache.E_CORRUPT


def test_cached_range_that_is_not_whole_records_is_corrupt(cache):
    rng = np.random.default_rng(7)
    recs, ids = map_records(rng, 500, 104, 2, 10, 2)
    rl = np.full(500, 104, np.uint32)
    rl[10], rl[11] = 50, 158  # the same bytes, cut at other record boundaries
    ids[10], ids[11] = 0, 1
    store(cache, 8, 0, 0, 0, 0, recs, ids, 2, rec_len=rl, compare=False)
    got, r = read_sort(cache, 8, 0, 1, [0], [True], 0, 0, [(b"", [], [])], 104, 2, 10, 1 << 20)
    assert got == b"" and r["n_records"] == 0 and r["status"][0] == cache.E_CORRUPT


# ---------------------------------------------------------------------------------------------------------------
# budget, LRU, removal
# ---------------------------------------------------------------------------------------------------------------
def test_lru_eviction_and_budget(cache):
    rng = np.random.default_rng(8)
    R, n = 4, 5000
    size = n * 104
    cache.exchange_set_budget(3 * size + size // 2)
    maps = [map_records(rng, n, 104, 2, 10, R) for _ in range(5)]
    for m in range(3):
        assert store(cache, 9, m, 1, 0, 0, *maps[m], R, compare=False)["cached"] == 1
    cache.exchange_read_packed(9, 0, 1, [0], np.zeros(size, np.uint8))  # a read is a use: map 0 is now the newest
    for m in (3, 4):
        assert store(cache, 9, m, 1, 0, 0, *maps[m], R, compare=False)["cached"] == 1
    hits, ln = cache.exchange_lookup(9, 0, R, list(range(5)))
    assert hits == 3 and [int(x) != cache.NOT_RESIDENT for x in ln] == [True, False, False, True, True]
    # an entry larger than the budget: not cached, outputs still exact
    cache.exchange_set_budget(size // 2)
    assert cache.exchange_lookup(9, 0, R, list(range(5)))[0] == 0
    assert store(cache, 9, 5, 1, 0, 3, *maps[0], R)["cached"] == 0
    cache.exchange_set_budget(4 * size)
    assert store(cache, 9, 5, 1, 0, 3, *maps[0], R)["cached"] == 1
    cache.exchange_set_budget(0)
    assert cache.exchange_lookup(9, 0, R, [5])[0] == 0
    assert store(cache, 9, 6, 1, 0, 3, *maps[0], R)["cached"] == 0


def test_remove_one_map_and_whole_shuffles(cache):
    rng = np.random.default_rng(10)
    for s in (11, 12):
        for m in range(3):
            store(cache, s, m, 1, 0, 0, *map_records(rng, 1000, 104, 2, 10, 2), 2, compare=False)
    assert cache.exchange_remove(11, 1) == 1
    assert list(cache.exchange_lookup(11, 0, 2, [0, 1, 2])[1] != cache.NOT_RESIDENT) == [True, False, True]
    assert cache.exchange_remove(11, -1) == 2
    assert cache.exchange_lookup(11, 0, 2, [0, 1, 2])[0] == 0
    assert cache.exchange_lookup(12, 0, 2, [0, 1, 2])[0] == 3


def test_restore_replaces_the_entry(cache):
    rng = np.random.default_rng(12)
    a, b = map_records(rng, 800, 104, 2, 10, 2), map_records(rng, 900, 104, 2, 10, 2)
    store(cache, 13, 0, 1, 0, 0, *a, 2, compare=False)
    store(cache, 13, 0, 1, 0, 0, *b, 2, compare=False)
    out = np.zeros(900 * 104, np.uint8)
    q = cache.exchange_read_packed(13, 0, 2, [0], out)
    assert out[: q["total"]].tobytes() == partitioned(b[0], b[1], 2)[0]


# ---------------------------------------------------------------------------------------------------------------
# threads
# ---------------------------------------------------------------------------------------------------------------
def test_reads_beside_stores_under_a_tight_budget(cache):
    rng = np.random.default_rng(11)
    R, n, M = 3, 4000, 10
    maps = [map_records(rng, n, 104, 2, 10, R) for _ in range(M)]
    models = [partitioned(recs, ids, R)[0] for recs, ids in maps]
    cache.exchange_set_budget(3 * n * 104)
    sorted_all = {}
    done = threading.Event()
    errors = []

    def writer():
        try:
            for m in range(M):
                store(cache, 14, m, 1, 0, 0, *maps[m], R, compare=False)
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(e)
        finally:
            done.set()

    def plain_reader():
        try:
            out = np.zeros(M * n * 104, np.uint8)
            while not done.is_set():
                q = cache.exchange_read_packed(14, 0, R, list(range(M)), out)
                for m in range(M):
                    if q["status"][m] == 0:
                        o = int(q["dst_off"][m])
                        assert out[o:o + int(q["dst_len"][m])].tobytes() == models[m]
                    else:
                        assert q["status"][m] == cache.E_NOT_CACHED
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    def sorted_reader():
        try:
            while not done.is_set():
                got, r = read_sort(cache, 14, 0, R, list(range(M)), [True] * M, 0, 0, [(b"", [], [])] * M, 104, 2,
                                   10, M * n * 104)
                if r["n_records"]:
                    assert (r["status"] == 0).all()
                    sorted_all[got] = True
                else:
                    assert set(r["status"]) <= {0, cache.E_NOT_CACHED}
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=f) for f in (writer, plain_reader, sorted_reader)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


# ---------------------------------------------------------------------------------------------------------------
# memory pressure: a full cache gives way to a workspace that cannot grow otherwise (an allocation test)
# ---------------------------------------------------------------------------------------------------------------
def test_workspace_allocation_evicts_the_cache(cache, oracle):
    torch = pytest.importorskip("torch")
    free0, _ = torch.cuda.mem_get_info(0)
    n = (1 << 30) // 104
    recs = np.zeros((n, 104), np.uint8)
    ids = np.zeros(n, np.uint32)
    sort_recs = np.frombuffer(oracle.gen_terasort(0, n).tobytes(), np.uint8)
    need = 3 * sort_recs.size // 2  # below the blocks + sorted copy (+ sort workspace) of a 1 GiB codec-NONE sort
    cache.exchange_set_budget(1 << 40)
    stored = 0
    while torch.cuda.mem_get_info(0)[0] > need and stored < 200:  # until the sort cannot get its buffers
        r = store(cache, 15, stored, 0, 0, 0, recs, ids, 1, compare=False)
        if not r["cached"]:
            break
        stored += 1
    assert stored > 0
    dst = np.zeros(sort_recs.size, np.uint8)
    q = cache.decompress_sort_packed(0, sort_recs, np.zeros(1, np.uint64), np.array([sort_recs.size], np.uint64),
                                     dst, 104, 2, 10)
    assert (q["status"] == 0).all() and q["n_records"] == n
    hits, _ = cache.exchange_lookup(15, 0, 1, list(range(stored)))
    assert hits < stored
    cache.exchange_set_budget(0)
    assert cache.exchange_lookup(15, 0, 1, list(range(stored)))[0] == 0
    assert torch.cuda.mem_get_info(0)[0] > free0 - (6 << 30)  # only the library's grow-only workspaces remain


# ---------------------------------------------------------------------------------------------------------------
# host mirror: the serialized writer stores, the reader asks the cache first
# ---------------------------------------------------------------------------------------------------------------
def test_host_mirror_terasort_with_and_without_the_cache(tmp_path, cache, oracle):
    import os

    host = pkg.host
    M, R, n = 4, 6, 6000
    maps = []
    for m in range(M):
        recs = np.frombuffer(oracle.gen_terasort(m * n, n).tobytes(), np.uint8).reshape(n, 104)
        maps.append((recs, ((recs[:, 2].astype(np.int64) * R) >> 8).astype(np.int32)))
    runs = {}
    for on in (False, True):
        d = host.S3ShuffleDispatcher({
            "spark.app.id": "app-exchange",
            "spark.shuffle.s3.rootDir": "file://%s/%s" % (tmp_path, on),
            "spark.shuffle.checksum.algorithm": "CRC32C",
            "spark.io.compression.codec": "lz4",
            "spark.shuffle.s3.gpu.exchangeCacheBytes": str(1 << 30) if on else "0",
        })
        for m, (recs, ids) in enumerate(maps):
            w = host.S3SerializedShuffleWriter(d, 0, m, R)
            for j in range(n):
                w.insertRecord(int(ids[j]), recs[j])
            w.commit()
            w.close()
        files = {(m, k): open(d.getPath(k, 0, m), "rb").read() for m in range(M) for k in ("data", "index", "checksum")}
        hits = cache.exchange_lookup(0, 0, R, list(range(M)))[0]
        assert hits == (M if on else 0)
        out = []
        for s, e, batch in [(r, r + 1, False) for r in range(R)] + [(1, 4, True), (1, 4, False)]:
            rd = host.S3ShuffleReader(d, 0, list(range(M)), s, e, batch)
            data, nrec = rd.readSorted(104, 2, 10)
            assert rd.remoteBytesRead == 0 or not on
            blocks = rd.read()
            assert rd.remoteBytesRead == 0 or not on
            rd.close()
            plain = b"".join(b for _, b in sorted(blocks, key=lambda blk: blk[0]))
            per_map = {}
            for (m, _, _), b in sorted(blocks, key=lambda blk: blk[0]):
                per_map[m] = per_map.get(m, b"") + b
            out.append((data, nrec, per_map))
            assert len(plain) == len(data)
        runs[on] = (files, out)
        if on:
            d.removeShuffle(0)
            assert cache.exchange_lookup(0, 0, R, list(range(M)))[0] == 0
            assert not os.path.exists(d.getPath("data", 0, 0))
        d.close()
    assert runs[True][0] == runs[False][0]
    assert runs[True][1] == runs[False][1]
