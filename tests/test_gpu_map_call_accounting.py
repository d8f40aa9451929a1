"""b2s_last_timing's byte counters of every map-side partition call, packed and on device memory: src_bytes is the
call's input (its records, or the DISTINCT call's blocks), dst_bytes the .data arena, h2d_bytes what a packed call
uploads (the records, 4 bytes of rec_len per record, 4 more of rec_part when the caller gives the ids, and the range
call's bound rows; the DISTINCT call's blocks) and d2h_bytes the arena it downloads.  A device call moves nothing over
PCIe.  bench.py and the split tools read these fields."""
import numpy as np
import pytest

import hash_model as hm
import partial_agg_model as pm
import range_model as rg
import rows_model as rm

pytestmark = pytest.mark.gpu

TYPES = ["long", "int", "long", "string"]
R = 5
CODECS = [0, 1]  # NONE, LZ4BLOCK


def _rows(n=2000, seed=7):
    rng = np.random.default_rng(seed)
    rows = [hm.make_row(TYPES, [int(rng.integers(0, 300)), int(rng.integers(-1000, 1000)) if rng.random() > 0.1
                                else None, int(rng.integers(0, 1 << 40)),
                                bytes(rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8))])
            for _ in range(n)]
    recs, rl = hm.records_of(rows)
    return rows, recs, rl


KEYS = hm.keys_of(TYPES, [0])
AGGS = [(pm.SUM, pm.VAL_INT64, KEYS[0][1] + 16, 2), (pm.COUNT, pm.VAL_NONE, 0, -1)]


def _calls(capi, rows, recs, rl):
    """name -> (packed call(codec, dst), device call(codec, d_rec, d_len, d_dst, cap, d_part), bytes a packed call
    uploads)"""
    n, b = rl.size, recs.size
    ids = hm.record_ids_np(recs, rl, KEYS, R)
    bounds = [rg.framed(x) for x in rg.draw_bounds(np.random.default_rng(3), rows, KEYS, R)]
    up = b + 4 * n
    return {
        "plain": (lambda c, dst: capi.partition_compress_packed(c, recs, rl, ids, R, dst),
                  lambda c, dr, dl, dd, cap, dp: capi.partition_compress_dev(c, dr, b, dl, dp, n, R, dd, cap),
                  up + 4 * n),
        "hash": (lambda c, dst: capi.partition_compress_rows_hash_packed(c, recs, rl, KEYS, R, dst),
                 lambda c, dr, dl, dd, cap, dp: capi.partition_compress_rows_hash_dev(c, dr, b, dl, n, KEYS, R, dd,
                                                                                       cap),
                 up),
        "range": (lambda c, dst: capi.partition_compress_rows_range_packed(c, recs, rl, KEYS, bounds, dst),
                  lambda c, dr, dl, dd, cap, dp: capi.partition_compress_rows_range_dev(c, dr, b, dl, n, KEYS, bounds,
                                                                                        dd, cap),
                  up + sum(len(x) for x in bounds)),
        "round_robin": (lambda c, dst: capi.partition_compress_rows_round_robin_packed(c, recs, rl, R, 2, 1, dst),
                        lambda c, dr, dl, dd, cap, dp: capi.partition_compress_rows_round_robin_dev(
                            c, dr, b, dl, n, R, 2, 1, dd, cap),
                        up),
        "aggregate": (lambda c, dst: capi.aggregate_partition_compress_rows_hash_packed(c, recs, rl, KEYS, AGGS, R,
                                                                                        dst),
                      lambda c, dr, dl, dd, cap, dp: capi.aggregate_partition_compress_rows_hash_dev(
                          c, dr, b, dl, n, KEYS, AGGS, R, dd, cap),
                      up),
        "grouping_sets": (lambda c, dst: capi.aggregate_grouping_sets_partition_compress_rows_hash_packed(
                              c, recs, rl, KEYS, AGGS, [1, 0], R, dst),
                          lambda c, dr, dl, dd, cap, dp: capi.aggregate_grouping_sets_partition_compress_rows_hash_dev(
                              c, dr, b, dl, n, KEYS, AGGS, [1, 0], R, dd, cap),
                          up),
        "window_limit": (lambda c, dst: capi.window_limit_partition_compress_rows_hash_packed(
                             c, recs, rl, hm.keys_of(TYPES, [0, 2]), 1, 1, 3, R, dst),
                         lambda c, dr, dl, dd, cap, dp: capi.window_limit_partition_compress_rows_hash_dev(
                             c, dr, b, dl, n, hm.keys_of(TYPES, [0, 2]), 1, 1, 3, R, dd, cap),
                         up),
        "window_limit_single": (lambda c, dst: capi.window_limit_partition_compress_rows_hash_packed(
                                    c, recs, rl, hm.keys_of(TYPES, [2]), 0, 1, 10, 1, dst),
                                lambda c, dr, dl, dd, cap, dp: capi.window_limit_partition_compress_rows_hash_dev(
                                    c, dr, b, dl, n, hm.keys_of(TYPES, [2]), 0, 1, 10, 1, dd, cap),
                                up),
    }


def _check(capi, r, src, up):
    t = capi.last_timing()
    assert (t["src_bytes"], t["dst_bytes"], t["h2d_bytes"], t["d2h_bytes"]) == (src, r["total"], up, r["total"])
    assert (r["status"] == 0).all()


@pytest.mark.parametrize("codec", CODECS)
@pytest.mark.parametrize("name", ["plain", "hash", "range", "round_robin", "aggregate", "grouping_sets",
                                  "window_limit", "window_limit_single"])
def test_map_calls(capi, codec, name):
    rows, recs, rl = _rows()
    packed, dev, up = _calls(capi, rows, recs, rl)[name]
    cap = capi.partition_compress_bound(codec, 0, R, 4 * recs.size) + 64  # room for grouping sets' projected rows
    dst = np.zeros(cap, np.uint8)
    r = packed(codec, dst)
    _check(capi, r, recs.size, up)
    assert r["total"] > 0
    ids = hm.record_ids_np(recs, rl, KEYS, R)
    d_rec, d_len, d_part, d_dst = (capi.dev_alloc(recs.size), capi.dev_alloc(rl.size * 4), capi.dev_alloc(rl.size * 4),
                                   capi.dev_alloc(cap))
    try:
        capi.dev_memcpy(d_rec, recs.ctypes.data, recs.size, 1)
        capi.dev_memcpy(d_len, rl.ctypes.data, rl.size * 4, 1)
        capi.dev_memcpy(d_part, ids.ctypes.data, ids.size * 4, 1)
        rd = dev(codec, d_rec, d_len, d_dst, cap, d_part)
        t = capi.last_timing()
        assert (t["src_bytes"], t["dst_bytes"], t["h2d_bytes"], t["d2h_bytes"]) == (recs.size, rd["total"], 0, 0)
        assert rd["total"] == r["total"] and (rd["status"] == 0).all()
    finally:
        for p in (d_rec, d_len, d_part, d_dst):
            capi.dev_free(p)


@pytest.mark.parametrize("codec", CODECS)
def test_cached_map_calls(capi, codec):
    rows, recs, rl = _rows(seed=9)
    ids = hm.record_ids_np(recs, rl, KEYS, R)
    bounds = [rg.framed(x) for x in rg.draw_bounds(np.random.default_rng(3), rows, KEYS, R)]
    dst = np.zeros(capi.partition_compress_bound(codec, 0, R, recs.size) + 64, np.uint8)
    up = recs.size + 4 * rl.size
    capi.exchange_set_budget(64 << 20)
    try:
        for call, h2d in ((lambda: capi.partition_compress_cached_packed(81, 0, codec, recs, rl, ids, R, dst),
                           up + 4 * rl.size),
                          (lambda: capi.partition_compress_rows_hash_cached_packed(81, 1, codec, recs, rl, KEYS, R,
                                                                                   dst), up),
                          (lambda: capi.partition_compress_rows_range_cached_packed(81, 2, codec, recs, rl, KEYS,
                                                                                    bounds, dst),
                           up + sum(len(x) for x in bounds)),
                          (lambda: capi.partition_compress_rows_round_robin_cached_packed(81, 3, codec, recs, rl, R, 0,
                                                                                          1, dst), up)):
            r = call()
            assert r["cached"] == 1
            _check(capi, r, recs.size, h2d)
    finally:
        capi.exchange_remove(81)
        capi.exchange_set_budget(0)


@pytest.mark.parametrize("codec", CODECS)
@pytest.mark.parametrize("ng", [1, 0])
def test_distinct_call(capi, codec, ng):
    """the DISTINCT call's input is its blocks of the map side's partial rows (keys G ++ X)"""
    rows, _, _ = _rows(600, seed=11)
    keys = hm.keys_of(TYPES, [0, 1][1 - ng:])  # G (the long column, when ng is 1) ++ X (the int column)
    partial = [pm.partial_rows(rows[i::3], keys, [(pm.COUNT, pm.VAL_NONE, 0, -1)]) for i in range(3)]
    streams = [rm.stream(p) for p in partial]
    arena, off, ln, sb, sl, ck = rm.build_blocks(capi, codec, 1, 3, streams)
    call_keys = [(k[0], k[2]) for k in keys]
    Rd = R if ng else 1
    dst = np.zeros(capi.partition_compress_bound(codec, 0, Rd, arena.size * 4) + 4096, np.uint8)
    kw = dict(checksum_alg=3, slice_base=sb, slice_len=sl, slice_checksum=ck)
    r = capi.aggregate_distinct_partition_compress_rows_hash(codec, arena, off, ln, dst, ng, call_keys,
                                                             [(pm.COUNT, pm.VAL_NONE)], [(pm.COUNT, pm.VAL_INT32, ng)],
                                                             Rd, **kw)
    srcb = int(ln.sum())
    t = capi.last_timing()
    assert (t["src_bytes"], t["dst_bytes"], t["h2d_bytes"], t["d2h_bytes"]) == (srcb, r["total"], srcb, r["total"])
    assert r["total"] > 0 and (r["part_status"] == 0).all() and r["counts"][2] > 0
    d_src, d_dst = capi.dev_alloc(max(arena.size, 1)), capi.dev_alloc(dst.size)
    try:
        capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        rd = capi.aggregate_distinct_partition_compress_rows_hash(codec, d_src, off, ln, d_dst, ng, call_keys,
                                                                  [(pm.COUNT, pm.VAL_NONE)],
                                                                  [(pm.COUNT, pm.VAL_INT32, ng)], Rd, dev=0,
                                                                  dst_cap=dst.size, **kw)
        t = capi.last_timing()
        assert (t["src_bytes"], t["dst_bytes"], t["h2d_bytes"], t["d2h_bytes"]) == (srcb, rd["total"], 0, 0)
        assert rd["total"] == r["total"]
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)
