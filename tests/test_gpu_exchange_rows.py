"""The exchange cache's row forms on the GPU: the hash, range and round-robin row writers' cached stores
(b2s_partition_compress_rows_*_cached_packed), which keep each record's offset beside the rows, and the composite-key
row sort and aggregation over cached and fetched sources (b2s_exchange_read_*_rows_keys_*), which mark a cached range's
records from those offsets instead of walking its size chain.  The models: a cached store is byte for byte its uncached
call; an exchange read is byte for byte the composite-key call over every map's fetched blocks in the same source
order."""
import numpy as np
import pytest

import hash_model as hm
import range_model as rg
import spark_s3_shuffle_b200 as pkg
from rows_model import CHECKSUMS, CODECS, MAX_I64, MIN_I32, MIN_I64, SUM_I64, mirror, parse

pytestmark = pytest.mark.gpu

c = pkg.capi
KINDS = ["hash", "range", "round_robin"]


@pytest.fixture
def cache(capi):
    """a generous budget on device 0; everything cached is released afterwards"""
    capi.exchange_set_budget(8 << 30)
    yield capi
    capi.exchange_set_budget(0)
    for s in range(64):
        capi.exchange_remove(s, -1)


# ---------------------------------------------------------------------------------------------------------------
# row shapes
# ---------------------------------------------------------------------------------------------------------------
def join_rows(rng, n):
    """a sort-merge join's rows: a nullable INT64 key (5 % null), an int and a string payload"""
    types = ["long", "int", "string"]
    rows = []
    for _ in range(n):
        k = None if rng.random() < 0.05 else int(rng.integers(-1000, 1000))
        payload = bytes(rng.integers(0, 256, int(rng.integers(0, 30)), dtype=np.uint8))
        rows.append(hm.make_row(types, [k, int(rng.integers(-9, 9)), payload]))
    return rows, hm.keys_of(types, [0])


def q67_rows(rng, n, n_keys=300):
    """q67-like rows: strings with long shared prefixes and ints, so the sort refines, then [long sum, min, max, count]"""
    types = ["string", "string", "int", "long", "long", "long", "long"]
    tuples = [(b"Electronics and more/%d" % (k % 5), b"AAAAAAAAAAAAAAAAAAAAB%02d" % (k % 13), k % 7)
              for k in range(n_keys)]
    rows = []
    for _ in range(n):
        a, b, i = tuples[int(rng.integers(0, n_keys))]
        v = int(rng.integers(-10**12, 10**12))
        rows.append(hm.make_row(types, [a, None if rng.random() < 0.03 else b, i, v, v, v, 1]))
    keys = hm.keys_of(types, [0, 1, 2])
    bitset = 8
    aggs = [(SUM_I64, bitset + 24, 3), (MIN_I64, bitset + 32, 4), (MAX_I64, bitset + 40, 5), (SUM_I64, bitset + 48, 6)]
    return rows, keys, aggs


def window_rows(rng, n):
    """a window's order: an int DESC, a string NULLS_LAST, a decimal(28, 2)"""
    types = ["int", "string", "decimal", "long"]
    rows = []
    for _ in range(n):
        s = None if rng.random() < 0.1 else b"w%d" % int(rng.integers(0, 20))
        d = None if rng.random() < 0.05 else int(rng.integers(-10**15, 10**15)) * 10**5
        rows.append(hm.make_row(types, [int(rng.integers(0, 30)), s, d, int(rng.integers(0, 1 << 40))]))
    keys = hm.keys_of(types, [0, 1, 2])
    keys[0] = (keys[0][0] | c.KEY_DESCENDING,) + keys[0][1:]
    keys[1] = (keys[1][0] | c.KEY_NULLS_LAST,) + keys[1][1:]
    return rows, keys


def decimal_rows(rng, n, n_keys=40):
    """[decimal(28, 2) sum, isEmpty] and decimal(38) min / max buffers, grouped by an INT64 key: field 0 the key, fields
    1..4 the buffers, then each out-of-line decimal's 16-byte region"""
    rows = []
    for _ in range(n):
        k = int(rng.integers(0, n_keys))
        vals = [int(rng.integers(-10**18, 10**18)) * 10**int(rng.integers(0, 9)) for _ in range(3)]
        fixed = 8 + 8 * 5
        r = bytearray(fixed + 16 * 3)
        r[8:16] = k.to_bytes(8, "little", signed=True)
        for a, v in enumerate(vals):
            o = fixed + 16 * a
            b = hm.decimal_bytes(v)
            r[o:o + len(b)] = b
            slot = 16 + 8 * (a if a == 0 else a + 1)
            r[slot:slot + 8] = ((o << 32) | len(b)).to_bytes(8, "little")
        rows.append(bytes(r))
    keys = [(c.KEY_INT64, 8, 8, 0)]
    aggs = [(c.agg_sum_decimal(28), 16, 1), (MIN_I32, 24, -1), (c.AGG_MIN_DECIMAL, 32, 3),
            (c.AGG_MAX_DECIMAL, 40, 4)]
    return rows, keys, aggs


# ---------------------------------------------------------------------------------------------------------------
# stores and sources
# ---------------------------------------------------------------------------------------------------------------
def store(capi, kind, shuffle, map_id, rows, keys, R, codec=2, level=0, alg=3, bounds=None, cached=True,
          compare=True):
    """one map task's rows through a row writer (range: over bounds, by default drawn from the rows for R
    partitions); cached: its cached form, checked byte for byte against the uncached call -> the result dict with
    "data" (the .data arena)"""
    buf, rl = hm.records_of(rows)
    bound = capi.partition_compress_bound(codec, 0, R, buf.size) + 64
    dst, ref = np.zeros(bound, np.uint8), np.zeros(bound, np.uint8)
    if kind == "hash":
        args, f = (buf, rl, keys, R), "partition_compress_rows_hash"
    elif kind == "range":
        if bounds is None:
            bounds = [rg.framed(b) for b in rg.draw_bounds(np.random.default_rng(7), rows, keys, R, sample=500)]
        args, f = (buf, rl, keys, bounds), "partition_compress_rows_range"
    else:
        args, f = (buf, rl, R, map_id % R, 1), "partition_compress_rows_round_robin"
    if not cached:
        r = getattr(capi, f + "_packed")(codec, *args, dst, 0, alg, level)
    else:
        r = getattr(capi, f + "_cached_packed")(shuffle, map_id, codec, *args, dst, 0, alg, level)
    r["data"] = dst[: r["total"]].copy()
    if cached and r["cached"]:  # each partition's bytes of records, as the cache holds them
        r["plain"] = np.array([capi.exchange_lookup(shuffle, p, p + 1, [map_id])[1][0]
                               for p in range(len(r["dst_off"]))], np.uint64)
    if cached and compare:
        q = getattr(capi, f + "_packed")(codec, *args, ref, 0, alg, level)
        assert r["total"] == q["total"] and bytes(r["data"]) == bytes(ref[: q["total"]])
        for k in ("dst_off", "dst_len", "checksums", "status"):
            assert (r[k] == q[k]).all(), k
    return r


def sources(maps, s, e):
    """every map's fetched .data range of reducer [s, e), one block each, one slice per partition, in map order ->
    (arena, off, len, slice_base, slice_len, slice_checksum)"""
    blocks, off, ln, sb, sl, sc = [], [], [], [0], [], []
    at = 0
    for r in maps:
        lo, n = int(r["dst_off"][s]), int(r["dst_len"][s:e].sum())
        blocks.append(r["data"][lo:lo + n])
        off.append(at)
        ln.append(n)
        at += n
        sl += list(r["dst_len"][s:e])
        sc += list(r["checksums"][s:e])
        sb.append(len(sl))
    arena = np.concatenate(blocks + [np.zeros(1, np.uint8)])
    return (arena, np.array(off, np.uint64), np.array(ln, np.uint64), np.array(sb, np.uint32),
            np.array(sl, np.uint64), np.array(sc, np.uint64))


def cap_of(maps, s, e):
    """room for every map's decoded records of reducer [s, e)"""
    return int(sum(int(r["plain"][s:e].sum()) for r in maps)) + 4096


def fetched(capi, name, codec, src, args, cap, dev=False):
    """the plain call over the fetched sources -> (output, result)"""
    return call(capi, "decompress_" + name, None, codec, src, args, cap, dev)


def call(capi, name, lead, codec, src, args, cap, dev=False):
    """capi.<name>_packed / _dev (lead: the exchange read's (shuffle, start, end, map_ids, cached)) -> (output, result)"""
    arena, off, ln, sb, sl, sc = src
    whole = "aggregate" in name
    lead = tuple(lead or ())
    if not dev:
        dst = np.zeros(max(cap, 1), np.uint8)
        r = getattr(capi, name + "_packed")(*lead, codec, arena, off, ln, dst, *args, 3, sb, sl, sc)
        return dst[: r["total"]].tobytes() if whole or r["n_records"] else b"", r
    d_src, d_dst = capi.dev_alloc(max(arena.size, 1)), capi.dev_alloc(max(cap, 1))
    try:
        capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        r = getattr(capi, name + "_dev")(*lead, codec, d_src, off, ln, d_dst, cap, *args, 3, sb, sl, sc)
        out = np.zeros(max(r["total"], 1), np.uint8)
        if (whole or r["n_records"]) and r["total"]:
            capi.dev_memcpy(out.ctypes.data, d_dst, r["total"], 2)
        return out[: r["total"]].tobytes() if whole or r["n_records"] else b"", r
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)


def same(a, b):
    assert a[0] == b[0]
    for k in ("n_records", "n_groups", "total"):
        if k in a[1]:
            assert a[1][k] == b[1][k], k
    assert (a[1]["status"] == b[1]["status"]).all()


# ---------------------------------------------------------------------------------------------------------------
# 1. the stores
# ---------------------------------------------------------------------------------------------------------------
_JOIN = {}


def join_data(n=600):
    if n not in _JOIN:
        _JOIN[n] = join_rows(np.random.default_rng(n), n)
    return _JOIN[n]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("R", [1, 3, 200])
@pytest.mark.parametrize("name,codec,level", CODECS)
@pytest.mark.parametrize("alg", CHECKSUMS)
def test_cached_store_equals_uncached_call(cache, kind, R, name, codec, level, alg):
    rows, keys = join_data()
    r = store(cache, kind, 1, 5, rows, keys, R, codec, level, alg)
    assert r["cached"] == 1
    R_out = len(r["dst_off"])
    plain = store(cache, kind, 1, 5, rows, keys, R, 0, 0, 0, cached=False)
    hits, ln = cache.exchange_lookup(1, 0, R_out, [5])
    assert hits == 1 and int(ln[0]) == len(plain["data"])
    for p in range(R_out):
        assert int(cache.exchange_lookup(1, p, p + 1, [5])[1][0]) == int(plain["dst_len"][p])


def test_round_robin_entry_reads_back_its_uncompressed_partitions(cache):
    rows, keys = join_data()
    R = 7
    store(cache, "round_robin", 2, 3, rows, keys, R)
    plain = store(cache, "round_robin", 2, 3, rows, keys, R, 0, 0, 0, cached=False)
    dst = np.zeros(len(plain["data"]) + 64, np.uint8)
    r = cache.exchange_read_packed(2, 0, R, [3], dst)
    assert r["total"] == len(plain["data"]) and bytes(dst[: r["total"]]) == bytes(plain["data"])
    r = cache.exchange_read_packed(2, 2, 5, [3], dst)
    lo, hi = int(plain["dst_off"][2]), int(plain["dst_off"][4] + plain["dst_len"][4])
    assert bytes(dst[: r["total"]]) == bytes(plain["data"][lo:hi])


# ---------------------------------------------------------------------------------------------------------------
# 2-4. sorted and aggregated reads over cached, fetched and mixed sources
# ---------------------------------------------------------------------------------------------------------------
def maps_of(capi, shuffle, kind, shape_rows, keys, M, R, codec=2, seed=0):
    """M map tasks' rows (shape_rows(rng)) through a cached row writer; a range writer's bounds are drawn from the first
    map's rows"""
    out, bounds = [], None
    for m in range(M):
        rows = shape_rows(np.random.default_rng(seed + m))
        if kind == "range" and bounds is None:
            bounds = [rg.framed(b) for b in rg.draw_bounds(np.random.default_rng(seed), rows, keys, R, sample=500)]
        out.append(store(capi, kind, shuffle, m, rows, keys, R, codec, bounds=bounds, compare=False))
        assert out[-1]["cached"] == 1
    return out


def check_read(capi, shuffle, maps, s, e, name, args, codec=2):
    """the exchange read with every source cached, none, alternating, and with one map evicted, each byte for byte the
    fetched call's; _dev equals _packed.  -> the fetched output"""
    M = len(maps)
    src = sources(maps, s, e)
    cap = cap_of(maps, s, e)
    want = fetched(capi, name, codec, src, args, cap)
    assert (want[1]["status"] == 0).all()
    ids = list(range(M))
    for mask in ([1] * M, [0] * M, [m % 2 for m in range(M)], [1 - m % 2 for m in range(M)]):
        lead = (shuffle, s, e, ids, mask)
        got = call(capi, "exchange_read_" + name, lead, codec, src, args, cap)
        same(got, want)
        same(call(capi, "exchange_read_" + name, lead, codec, src, args, cap, dev=True), got)
    # one map evicted: read as cached it is not resident and nothing is sorted; fetched, the output is unchanged
    assert capi.exchange_remove(shuffle, 1) == 1
    out, r = call(capi, "exchange_read_" + name, (shuffle, s, e, ids, [1] * M), codec, src, args, cap)
    assert r["status"][1] == c.E_NOT_CACHED and r["n_records"] == 0 and out == b""
    assert (np.delete(r["status"], 1) == 0).all()
    mask = [0 if m == 1 else 1 for m in range(M)]
    same(call(capi, "exchange_read_" + name, (shuffle, s, e, ids, mask), codec, src, args, cap), want)
    return want


@pytest.mark.parametrize("kind", KINDS)
def test_join_sort_reads(cache, kind):
    keys = join_data()[1]
    maps = maps_of(cache, 3, kind, lambda g: join_rows(g, 800)[0], keys, 4, 5)
    want = check_read(cache, 3, maps, 1, 4, "sort_rows_keys", (keys,))
    assert len(parse(want[0])) == want[1]["n_records"] > 0


def test_q67_sort_and_aggregate_reads(cache):
    _, keys, aggs = q67_rows(np.random.default_rng(0), 1)
    maps = maps_of(cache, 4, "hash", lambda g: q67_rows(g, 1500)[0], keys, 4, 3)
    check_read(cache, 4, maps, 0, 2, "sort_rows_keys", (keys,))
    maps = maps_of(cache, 5, "hash", lambda g: q67_rows(g, 1500)[0], keys, 4, 3)
    want = check_read(cache, 5, maps, 0, 2, "aggregate_rows_keys", (keys, aggs))
    assert 0 < want[1]["n_groups"] < want[1]["n_records"]


def test_window_order_sort_reads(cache):
    keys = window_rows(np.random.default_rng(0), 1)[1]
    hash_keys = [(k[0] & 0xFF,) + k[1:] for k in keys]
    maps = maps_of(cache, 6, "hash", lambda g: window_rows(g, 1000)[0], hash_keys, 3, 4)
    check_read(cache, 6, maps, 0, 4, "sort_rows_keys", (keys,))
    maps = maps_of(cache, 7, "range", lambda g: window_rows(g, 1000)[0], keys, 3, 4)
    check_read(cache, 7, maps, 1, 3, "sort_rows_keys", (keys,))


def test_decimal_aggregate_reads(cache):
    _, keys, aggs = decimal_rows(np.random.default_rng(0), 1)
    maps = maps_of(cache, 8, "hash", lambda g: decimal_rows(g, 1200)[0], keys, 4, 3)
    want = check_read(cache, 8, maps, 0, 3, "aggregate_rows_keys", (keys, aggs))
    assert want[1]["n_groups"] > 0


def test_one_key_exchange_read_equals_the_single_key_calls(cache):
    rows, keys = join_data()
    maps = [store(cache, "hash", 9, m, rows, keys, 3) for m in range(3)]
    src = sources(maps, 0, 3)
    cap = cap_of(maps, 0, 3)
    kt, ko, kl, kn = keys[0]
    got = call(cache, "exchange_read_sort_rows_keys", (9, 0, 3, [0, 1, 2], [1, 1, 1]), 2, src, (keys,), cap)
    same(got, fetched(cache, "sort_rows", 2, src, (kt, ko, kl, kn), cap))
    aggs = [(SUM_I64, 16, -1)]  # the int field's slot
    got = call(cache, "exchange_read_aggregate_rows_keys", (9, 0, 3, [0, 1, 2], [1, 1, 1]), 2, src, (keys, aggs), cap)
    same(got, fetched(cache, "aggregate_rows", 2, src, (kt, ko, kl, kn, aggs), cap))


def test_reads_over_empty_partitions(cache):
    """ranges holding empty partitions, at their ends and alone, and maps with nothing in the range: a partition with no
    records starts at the next non-empty one's first record, or past the last record"""
    rows, keys = join_data(300)
    R, M = 200, 3
    maps = [store(cache, "hash", 15, m, rows[m * 40:m * 40 + 120 + 60 * m], keys, R) for m in range(M)]
    # a range writer whose bounds all lie below every non-null key: partitions 1 and 2 stay empty
    bounds = [rg.framed(hm.make_row(["long"], [-10**6 - b])) for b in (3, 2, 1)]
    skew = [store(cache, "range", 16, m, rows, keys, 4, bounds=bounds) for m in range(2)]
    empty = [p for p in range(R) if all(r["dst_len"][p] == 0 for r in maps)]
    assert empty and empty[0] < R - 1
    ranges = [(0, R), (5, 37), (empty[0], empty[0] + 1), (empty[-1], R), (R - 1, R), (0, empty[0] + 1)]
    for shuffle, ms, rs in [(15, maps, ranges), (16, skew, [(0, 4), (0, 3), (1, 4), (3, 4)])]:
        for s, e in rs:
            live = [m for m in range(len(ms)) if ms[m]["dst_len"][s:e].sum()]
            cap = cap_of(ms, s, e)
            src = sources(ms, s, e)
            if live:
                want = fetched(cache, "sort_rows_keys", 2, sources([ms[m] for m in live], s, e), (keys,), cap)
            else:
                want = (b"", {"n_records": 0})
            ids = list(range(len(ms)))
            for mask in ([1] * len(ms), [0 if m in live and m % 2 == 0 else 1 for m in ids]):
                got = call(cache, "exchange_read_sort_rows_keys", (shuffle, s, e, ids, mask), 2, src, (keys,), cap)
                assert (got[1]["status"] == 0).all(), (shuffle, s, e, mask)
                assert got[0] == want[0] and got[1]["n_records"] == want[1]["n_records"], (shuffle, s, e, mask)


# ---------------------------------------------------------------------------------------------------------------
# 5. marked and walked ranges agree
# ---------------------------------------------------------------------------------------------------------------
def test_marked_and_walked_reads_agree(cache):
    rows, keys, aggs = q67_rows(np.random.default_rng(3), 2000)
    R = 5
    buf, rl = hm.records_of(rows)
    ids = hm.record_ids_np(buf, rl, keys, R)
    with_bounds = store(cache, "hash", 10, 0, rows, keys, R)
    dst = np.zeros(cache.partition_compress_bound(2, 0, R, buf.size) + 64, np.uint8)
    without = cache.partition_compress_cached_packed(11, 0, 2, buf, rl, ids, R, dst, 0, 3)
    assert without["cached"] == 1 and bytes(dst[: without["total"]]) == bytes(with_bounds["data"])
    src = sources([with_bounds], 1, 4)
    cap = cap_of([with_bounds], 1, 4)
    for name, args in (("sort_rows_keys", (keys,)), ("aggregate_rows_keys", (keys, aggs))):
        marked = call(cache, "exchange_read_" + name, (10, 1, 4, [0], [1]), 2, src, args, cap)
        walked = call(cache, "exchange_read_" + name, (11, 1, 4, [0], [1]), 2, src, args, cap)
        same(marked, walked)
        same(marked, fetched(cache, name, 2, src, args, cap))


# ---------------------------------------------------------------------------------------------------------------
# 6. verdicts of rows the map side accepts but the read's key, null word or aggregate slot rejects
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("short,name,args", [
    (8, "sort_rows_keys", ([(c.KEY_INT64, 8, 8, -1)],)),  # no room for the key slot
    (8, "sort_rows_keys", ([(c.KEY_INT64, 0, 8, 70)],)),  # no room for null word 1
    (16, "aggregate_rows_keys", ([(c.KEY_INT64, 8, 8, 0)], [(SUM_I64, 16, -1)])),  # no room for the aggregate slot
])
def test_short_rows_fail_their_source_as_the_fetched_path_names_them(cache, short, name, args):
    rng = np.random.default_rng(4)
    rows = [bytes(rng.integers(0, 256, 24, dtype=np.uint8)) for _ in range(300)]
    rows[137] = rows[137][:short]
    rows[250] = rows[250][:short]
    R = 2
    maps = [store(cache, "round_robin", 12, m, rows if m == 1 else rows[:100], None, R) for m in range(3)]
    src = sources(maps, 0, R)
    cap = cap_of(maps, 0, R)
    want = fetched(cache, name, 2, src, args, cap)
    want_err = c.load().b2s_last_error()
    assert want[1]["status"][1] == c.E_CORRUPT and want[1]["n_records"] == 0
    for mask in ([1, 1, 1], [0, 1, 0]):
        got = call(cache, "exchange_read_" + name, (12, 0, R, [0, 1, 2], mask), 2, src, args, cap)
        assert got[0] == b"" and got[1]["n_records"] == 0
        assert list(got[1]["status"]) == [0, c.E_CORRUPT, 0]
        err = c.load().b2s_last_error()
        assert err == want_err.replace(b"block 1", b"cached source 1"), (err, want_err)


# ---------------------------------------------------------------------------------------------------------------
# 7. a reducer of more than a million rows from one map
# ---------------------------------------------------------------------------------------------------------------
def test_one_map_reducer_of_a_million_rows(cache):
    n = 1 << 20
    rng = np.random.default_rng(5)
    size = 24
    keys_v = rng.integers(-(1 << 40), 1 << 40, n)
    rec = np.zeros((n, 4 + size), np.uint8)
    rec[:, :4] = np.frombuffer(size.to_bytes(4, "big"), np.uint8)
    rec[:, 4 + 8:4 + 16] = keys_v.astype("<i8").view(np.uint8).reshape(n, 8)
    rec[:, 4 + 16:] = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    buf, rl = rec.reshape(-1), np.full(n, 4 + size, np.uint32)
    keys = [(c.KEY_INT64, 8, 8, 0)]
    dst = np.zeros(cache.partition_compress_bound(2, 0, 1, buf.size) + 64, np.uint8)
    r = cache.partition_compress_rows_hash_cached_packed(13, 0, 2, buf, rl, keys, 1, dst, 0, 3)
    assert r["cached"] == 1
    r["data"] = dst[: r["total"]].copy()
    src = sources([r], 0, 1)
    out, res = call(cache, "exchange_read_sort_rows_keys", (13, 0, 1, [0], [1]), 2, src, (keys,), buf.size + 64)
    assert res["n_records"] == n and (res["status"] == 0).all()
    got = np.frombuffer(out, np.uint8).reshape(n, 4 + size)
    order = np.argsort(keys_v, kind="stable")
    assert (got == rec[order]).all()


# ---------------------------------------------------------------------------------------------------------------
# 8. the budget counts the boundaries
# ---------------------------------------------------------------------------------------------------------------
def test_boundaries_count_against_the_budget(cache):
    rows, keys = join_data()
    buf, rl = hm.records_of(rows)
    n, bytes_ = len(rows), buf.size
    need = (bytes_ + 7) // 8 * 8 + 8 * n  # the records, 8-aligned, and their offsets
    ids = hm.record_ids_np(buf, rl, keys, 1)
    dst = np.zeros(cache.partition_compress_bound(2, 0, 1, bytes_) + 64, np.uint8)
    # the records alone fit, the records and their boundaries do not: not stored; the id-taking store fits
    cache.exchange_set_budget(need - 1)
    assert store(cache, "hash", 14, 0, rows, keys, 1)["cached"] == 0
    assert cache.exchange_lookup(14, 0, 1, [0])[0] == 0
    assert cache.partition_compress_cached_packed(14, 1, 2, buf, rl, ids, 1, dst, 0, 3)["cached"] == 1
    cache.exchange_remove(14, -1)
    # exactly two row entries fit; a third evicts the least recently used, and a read counts as a use
    cache.exchange_set_budget(2 * need)
    for m in range(2):
        assert store(cache, "hash", 14, m, rows, keys, 1)["cached"] == 1
    assert cache.exchange_lookup(14, 0, 1, [0, 1])[0] == 2
    src = sources([store(cache, "hash", 14, 0, rows, keys, 1, cached=False)], 0, 1)
    call(cache, "exchange_read_sort_rows_keys", (14, 0, 1, [0], [1]), 2, src, (keys,), bytes_ + 64)
    assert store(cache, "hash", 14, 2, rows, keys, 1)["cached"] == 1
    hits, ln = cache.exchange_lookup(14, 0, 1, [0, 1, 2])
    assert hits == 2 and ln[1] == c.NOT_RESIDENT and ln[0] == ln[2] == bytes_
    # removal frees the charge: both evicted entries' room is back
    assert cache.exchange_remove(14, -1) == 2
    for m in range(2):
        assert store(cache, "hash", 14, 10 + m, rows, keys, 1)["cached"] == 1
    # a budget lowered below one row entry evicts it
    cache.exchange_set_budget(need - 1)
    assert cache.exchange_lookup(14, 0, 1, [10, 11])[0] == 0


# ---------------------------------------------------------------------------------------------------------------
# 10. the host mirror: the row writers store, the row reads ask the cache first
# ---------------------------------------------------------------------------------------------------------------
def mirror_run(tmp_path, on, shapes, R, evict=None, rounds=1):
    """shapes[s] = (shuffle, maps' rows, keys, aggs): every map through the hash row writer, then every reducer's sorted
    and aggregated reads (composite and one-key), rounds times.  evict(shuffle, stop): run beside the reads, in another
    thread per shuffle, until stop is set -> (files, outputs)"""
    import threading

    d = mirror(tmp_path / str(on), "lz4", **{"spark.shuffle.s3.gpu.exchangeCacheBytes": str(1 << 30) if on else "0"})
    files, outs = {}, []
    try:
        for shuffle, maps, keys, _ in shapes:
            for m, rows in enumerate(maps):
                w = pkg.host.S3SerializedShuffleWriter(d, shuffle, m, R)
                w.hashRows(keys)
                for row in rows:
                    w.insertRecord(0, len(row).to_bytes(4, "big") + row)
                w.commit()
                w.close()
                for k in ("data", "index", "checksum"):
                    files[(shuffle, m, k)] = open(d.getPath(k, shuffle, m), "rb").read()
            assert c.exchange_lookup(shuffle, 0, R, list(range(len(maps))))[0] == (len(maps) if on else 0)
        stop = threading.Event()
        threads = [threading.Thread(target=evict, args=(shuffle, stop)) for shuffle, _, _, _ in shapes] if evict else []
        for t in threads:
            t.start()
        try:
            for _ in range(rounds):
                for shuffle, maps, keys, aggs in shapes:
                    for s, e in [(r, r + 1) for r in range(R)] + [(0, R)]:
                        rd = pkg.host.S3ShuffleReader(d, shuffle, list(range(len(maps))), s, e)
                        outs.append(rd.readSortedRowsKeys(keys))
                        if len(keys) == 1:  # the one-key reads take a fixed-width column
                            outs.append(rd.readSortedRows(*keys[0]))
                        if aggs:
                            outs.append(rd.readAggregatedRowsKeys(keys, aggs))
                        if aggs and len(keys) == 1:
                            outs.append(rd.readAggregatedRows(*keys[0], aggs=aggs))
                        if on and not evict:
                            assert rd.remoteBytesRead == 0  # every map is resident: nothing is fetched
                        rd.close()
        finally:
            stop.set()
            for t in threads:
                t.join()
    finally:
        for shuffle, _, _, _ in shapes:
            d.removeShuffle(shuffle)
        d.close()
    return files, outs


def mirror_shapes():
    join = [join_rows(np.random.default_rng(30 + m), 700)[0] for m in range(3)]
    q67 = [q67_rows(np.random.default_rng(40 + m), 900)[0] for m in range(3)]
    _, q67_keys, aggs = q67_rows(np.random.default_rng(0), 1)
    one_key_aggs = [(SUM_I64, 32, 3), (MIN_I64, 40, 4)]
    return [(20, join, join_data()[1], None), (21, q67, [q67_keys[2]], one_key_aggs), (22, q67, q67_keys, aggs)]


def test_host_mirror_rows_with_and_without_the_cache(tmp_path, cache):
    R = 4
    off = mirror_run(tmp_path, False, mirror_shapes(), R)
    on = mirror_run(tmp_path, True, mirror_shapes(), R)
    assert on[0] == off[0]  # .data / .index / .checksum byte for byte
    assert on[1] == off[1]


def test_host_mirror_row_reads_refetch_maps_evicted_under_them(tmp_path, cache):
    """other threads keep removing maps' entries and storing them again while the reducers read: a map evicted between
    a read's lookup and its call is fetched and the call repeated, so every output is the cache-off one"""
    R, rounds = 4, 8
    shapes = mirror_shapes()
    # each map's entry as the writer stores it (the entry holds uncompressed partitioned rows, so codec NONE will do)
    entries = {shuffle: (keys, [hm.records_of(rows) for rows in maps]) for shuffle, maps, keys, _ in shapes}
    removed, errors = [], []

    def evict(shuffle, stop):
        keys, recs = entries[shuffle]
        rng = np.random.default_rng(shuffle)
        try:
            while not stop.is_set():
                m = int(rng.integers(0, len(recs)))
                removed.append(c.exchange_remove(shuffle, m))
                buf, rl = recs[m]
                dst = np.zeros(c.partition_compress_bound(0, 0, R, buf.size) + 64, np.uint8)
                c.partition_compress_rows_hash_cached_packed(shuffle, m, 0, buf, rl, keys, R, dst)
        except Exception as e:  # reported by the test, not lost in the thread
            errors.append(e)

    off = mirror_run(tmp_path, False, shapes, R)
    on = mirror_run(tmp_path, True, shapes, R, evict, rounds)
    assert not errors, errors
    assert sum(removed) > 0
    assert on[0] == off[0]
    assert on[1] == off[1] * rounds
