"""Verify + decompress + group + merge in one call (b2s_decompress_aggregate_rows_*): a reduce task's blocks of partial
aggregate rows in, one row per key out.  The model parses the decoded streams in Python, groups the records in stable
sorted order (the row sort's order), and merges every aggregate over each group in that order — the double sum
sequentially — into a copy of the group's first record.  The call must be byte for byte that model."""
import ctypes as C
import struct

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from rows_model import CHECKSUMS, CODECS, KEY_BYTES, KEY_INT32, KEY_INT64, MAX_F64, MAX_I32, MAX_I64, MIN_F64, \
    MIN_I32, MIN_I64, SUM_F64, SUM_I64, blocks_of, build_blocks, mirror, model_aggregate, parse, run, stream, write_maps

pytestmark = pytest.mark.gpu

ALL_OPS = list(range(8))
KEY_LEN = {KEY_INT32: 4, KEY_INT64: 8, KEY_BYTES: 6}


# ---------------------------------------------------------------------------------------------------------------
# rows: nw null-bitset words, then 8-byte fields (field 0 the key), then a variable-length region
# ---------------------------------------------------------------------------------------------------------------
def field(nw, f):
    return 8 * nw + 8 * f


def agg_values(rng, op, n):
    """8-byte slots with the op's edge cases mixed into random values"""
    if op == SUM_I64:
        v = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64, endpoint=True)
        v[::5] = 2**63 - 1
        v[1::7] = -2**63
        return v.view(np.uint64)
    if op == SUM_F64:
        v = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 12, n)
        v[::9] = -0.0
        v[1::13] = 0.0
        v[2::17] = 1e300
        return v.view(np.uint64)
    if op in (MIN_I32, MAX_I32):
        lo = rng.integers(-2**31, 2**31 - 1, n, dtype=np.int64, endpoint=True)
        lo[::5] = -2**31
        lo[1::5] = 2**31 - 1
        hi = rng.integers(0, 2**32, n, dtype=np.uint64)  # garbage in the high slot bytes
        return (lo.astype(np.uint64) & np.uint64(0xFFFFFFFF)) | (hi << np.uint64(32))
    if op in (MIN_I64, MAX_I64):
        v = rng.integers(-50, 50, n).astype(np.int64)
        v[::11] = -2**63
        v[1::11] = 2**63 - 1
        return v.view(np.uint64)
    specials = np.array([0.0, -0.0, np.inf, -np.inf, 1.5, -1.5], np.float64).view(np.uint64)
    nans = np.array([0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000123, 0x7FFFFFFFFFFFFFFF], np.uint64)
    v = rng.choice(specials, n)
    pick = rng.random(n) < 0.15
    v[pick] = rng.choice(nans, int(pick.sum()))
    return v


def make_rows(rng, n, kt, keys, ops, nw=1, key_null=-1, key_null_frac=0.0, agg_null_frac=0.2, tail=True,
              agg_null_fields=None):
    """-> rows, aggs.  Field 0 is the key; aggregate a is field a + 1 with null bit agg_null_fields[a] (default a + 1,
    -1 = none)."""
    kl = KEY_LEN[kt]
    m = len(ops)
    anf = agg_null_fields if agg_null_fields is not None else [a + 1 for a in range(m)]
    aggs = [(op, field(nw, a + 1), anf[a]) for a, op in enumerate(ops)]
    vals = [agg_values(rng, op, n) for op in ops]
    fixed = field(nw, m + 1)
    tails = rng.integers(0, 40, n) if tail else np.zeros(n, np.int64)
    bits = rng.integers(0, 2**63, (n, nw), dtype=np.uint64)  # unrelated bits stay as they are
    rows = []
    for i in range(n):
        r = bytearray(rng.integers(0, 256, fixed + int(tails[i]), dtype=np.uint8).tobytes())
        words = [int(b) for b in bits[i]]
        k = keys[i]
        ko = field(nw, 0)
        r[ko:ko + kl] = k if isinstance(k, (bytes, bytearray)) else int(k).to_bytes(kl, "little", signed=True)
        for f in [key_null] + anf:
            if f >= 0:
                words[f >> 6] &= ~(1 << (f & 63))
        if key_null >= 0 and rng.random() < key_null_frac:
            words[key_null >> 6] |= 1 << (key_null & 63)
        for a in range(m):
            r[aggs[a][1]:aggs[a][1] + 8] = int(vals[a][i]).to_bytes(8, "little")
            if anf[a] >= 0 and rng.random() < agg_null_frac:
                words[anf[a] >> 6] |= 1 << (anf[a] & 63)
        for w in range(nw):
            r[8 * w:8 * w + 8] = words[w].to_bytes(8, "little")
        rows.append(bytes(r))
    return rows, aggs


def check(capi, codec, level, alg, plain, kt, ko, kl, nf, aggs, dev=False, blocks=None):
    blocks = blocks or build_blocks(capi, codec, level, alg, plain)
    total = sum(len(b) for b in plain)
    got, r = run(capi, "decompress_aggregate_rows", codec, alg, blocks, (kt, ko, kl, nf, aggs), total, dev)
    assert (r["status"] == 0).all(), r["status"]
    want, n, g = model_aggregate(plain, [(kt, ko, kl, nf)], aggs)
    assert (r["n_records"], r["n_groups"], r["total"]) == (n, g, len(want))
    assert got == want
    return got, r


# ---------------------------------------------------------------------------------------------------------------
# 1. every codec x checksum x key type, _dev against _packed
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kt", [KEY_BYTES, KEY_INT32, KEY_INT64])
@pytest.mark.parametrize("alg", CHECKSUMS)
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_aggregates_like_the_model(capi, name, codec, level, alg, kt):
    rng = np.random.default_rng(codec * 100 + alg * 10 + kt)
    n = 3000
    if kt == KEY_BYTES:
        keys = [bytes(rng.choice(np.array([0, 1, 0x80, 0xFF], np.uint8), 6)) for _ in range(n)]
    else:
        keys = rng.integers(-200, 200, n)
    rows, aggs = make_rows(rng, n, kt, keys, [SUM_I64, SUM_F64, MIN_I32, MAX_I64, MAX_F64], key_null=0,
                           key_null_frac=0.05)
    plain = blocks_of(rows, [1200, 0, 1, 799, 1000])
    a, _ = check(capi, codec, level, alg, plain, kt, 8, KEY_LEN[kt], 0, aggs)
    b, _ = check(capi, codec, level, alg, plain, kt, 8, KEY_LEN[kt], 0, aggs, dev=True)
    assert a == b


def test_timing_reports_the_aggregation_step(capi):
    rng = np.random.default_rng(5)
    n = 20_000
    rows, aggs = make_rows(rng, n, KEY_INT64, rng.integers(0, 500, n), [SUM_I64, SUM_F64], tail=False)
    check(capi, 1, 0, 3, blocks_of(rows, [10_000, 10_000]), KEY_INT64, 8, 8, -1, aggs, dev=True)
    t = capi.last_timing()
    assert t["dominant_launches"] > 0 and 0 < t["dominant_ms"] <= t["top_kernel_ms"] <= t["kernel_ms"]


# ---------------------------------------------------------------------------------------------------------------
# 2. every op with its edges, nulls
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", ALL_OPS)
@pytest.mark.parametrize("group", [3, 40, 700])
def test_each_op_small_and_large_groups(capi, op, group):
    """groups of 3 (a thread each), 40 and 700 records (a warp each), with the op's edge values and nulls"""
    rng = np.random.default_rng(op * 10 + group)
    n = 6000
    keys = rng.permutation(np.arange(n) // group)
    rows, aggs = make_rows(rng, n, KEY_INT64, keys, [op, op], agg_null_frac=0.3, agg_null_fields=[1, -1])
    check(capi, 1, 0, 3, blocks_of(rows, [2000, 4000]), KEY_INT64, 8, 8, -1, aggs)


def slot_rows(key, slots, null=None):
    """rows of one null word, an int64 key and one aggregate slot (null bit 1)"""
    out = []
    for i, s in enumerate(slots):
        nb = (1 << 1) if null and null[i] else 0
        out.append(nb.to_bytes(8, "little") + int(key).to_bytes(8, "little", signed=True) + s)
    return out


def d(x):
    return struct.pack("<d", x)


def test_op_edge_values(capi):
    nan_a, nan_b = (0x7FF8000000000001).to_bytes(8, "little"), (0xFFF0000000000002).to_bytes(8, "little")
    cases = [
        (SUM_I64, [(2**63 - 1).to_bytes(8, "little"), (5).to_bytes(8, "little")], (2**63 + 4).to_bytes(8, "little")),
        (SUM_F64, [d(-0.0)], d(0.0)),
        (SUM_F64, [d(1e16), d(1.0), d(1.0)], d((1e16 + 1.0) + 1.0)),
        (MIN_I32, [(0xDEADBEEF80000000).to_bytes(8, "little"), (0x123456787FFFFFFF).to_bytes(8, "little")],
         (0x80000000).to_bytes(8, "little")),
        (MAX_I32, [(0xDEADBEEF80000000).to_bytes(8, "little"), (0x12345678FFFFFFFF).to_bytes(8, "little")],
         (0xFFFFFFFF).to_bytes(8, "little")),
        (MIN_F64, [d(0.0), d(-0.0)], d(0.0)),
        (MIN_F64, [d(-0.0), d(0.0)], d(-0.0)),
        (MAX_F64, [d(0.0), d(-0.0)], d(0.0)),
        (MAX_F64, [d(np.inf), nan_a, nan_b], nan_a),
        (MIN_F64, [nan_b, d(np.inf)], d(np.inf)),
        (MIN_F64, [nan_b, nan_a], nan_b),
    ]
    for k, (op, slots, want) in enumerate(cases):
        rows = slot_rows(k, slots)
        got, r = check(capi, 0, 0, 0, [stream(rows)], KEY_INT64, 8, 8, -1, [(op, 16, 1)])
        assert got[4 + 16:4 + 24] == want, (k, got[20:28].hex(), want.hex())


def test_all_null_and_mixed_null_groups(capi):
    rows = slot_rows(1, [d(1.0), d(2.0)], null=[1, 1]) + slot_rows(2, [d(5.0), d(7.0)], null=[1, 0])
    for op in ALL_OPS:
        got, r = check(capi, 0, 0, 0, [stream(rows)], KEY_INT64, 8, 8, -1, [(op, 16, 1)])
        first = got[4:4 + 24]
        assert first[:8] == (2).to_bytes(8, "little") and first[16:24] == bytes(8)  # null bit set, slot zero
        assert got[32:40] == bytes(8)  # second group: null bit cleared


@pytest.mark.parametrize("nw,key_null,agg_nulls", [(1, 0, [1, 2, 3]), (2, 70, [64, 5, 127]), (2, 3, [66, 67, -1])])
def test_nullable_key_and_shared_null_words(capi, nw, key_null, agg_nulls):
    """the null-key group; aggregates whose null bits share a word with each other and with the key's, in the first
    or second bitset word"""
    rng = np.random.default_rng(nw * 100 + key_null)
    n = 5000
    rows, aggs = make_rows(rng, n, KEY_INT32, rng.integers(-20, 20, n), [SUM_I64, MIN_F64, MAX_I32], nw=nw,
                           key_null=key_null, key_null_frac=0.1, agg_null_frac=0.4, agg_null_fields=agg_nulls)
    check(capi, 3, 1, 2, blocks_of(rows, [2500, 2500]), KEY_INT32, field(nw, 0), 4, key_null, aggs)


@pytest.mark.parametrize("m", [0, 16])
def test_zero_and_sixteen_aggregates(capi, m):
    rng = np.random.default_rng(m)
    n = 4000
    ops = [ALL_OPS[a % 8] for a in range(m)]
    rows, aggs = make_rows(rng, n, KEY_INT64, rng.integers(0, 300, n), ops, nw=1,
                           agg_null_fields=[a + 1 if a < 40 else -1 for a in range(m)])
    got, r = check(capi, 2, 0, 3, blocks_of(rows, [1000, 3000]), KEY_INT64, 8, 8, -1, aggs)
    assert r["n_groups"] == len(set(x[8:16] for x in rows))


def test_groups_spanning_blocks_keep_the_first_blocks_row(capi):
    """every key in every block: the output row is the first block's (its tail bytes tag the block)"""
    rng = np.random.default_rng(7)
    plain = []
    for b in range(4):
        rows, aggs = make_rows(rng, 300, KEY_INT64, rng.permutation(300), [SUM_I64, MAX_F64])
        plain.append(stream([r + bytes([b]) * 8 for r in rows]))
    got, r = check(capi, 1, 0, 3, plain, KEY_INT64, 8, 8, -1, aggs)
    assert r["n_groups"] == 300 and all(got[o + ln - 8:o + ln] == bytes(8) for o, ln in parse(got))


def test_all_distinct_keys(capi):
    rng = np.random.default_rng(8)
    n = 20_000
    rows, aggs = make_rows(rng, n, KEY_INT64, rng.permutation(n) - 10_000, [SUM_F64, MIN_I64], tail=False)
    got, r = check(capi, 0, 0, 0, blocks_of(rows, [7000, 13_000]), KEY_INT64, 8, 8, -1, aggs)
    assert r["n_groups"] == n


def test_one_group_of_more_than_a_million_records(capi):
    """1.1 M records of one key: the double sum is the sequential sum, bit for bit"""
    n, L = 1_100_000, 48  # null word, int64 key, then sum(double), count, max(double), min(int64) at 16, 24, 32, 40
    rng = np.random.default_rng(9)
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-5, 8, n)
    nulls = rng.random(n) < 0.1
    rec = np.zeros((n, 4 + L), np.uint8)
    rec[:, :4] = np.frombuffer(L.to_bytes(4, "big"), np.uint8)
    rec[:, 4:12] = np.where(nulls, 1 << 1, 0).astype("<u8").view(np.uint8).reshape(n, 8)
    rec[:, 12:20] = np.full(n, 77, "<i8").view(np.uint8).reshape(n, 8)
    rec[:, 20:28] = x.view(np.uint8).reshape(n, 8)
    rec[:, 28:36] = np.ones(n, "<i8").view(np.uint8).reshape(n, 8)
    rec[:, 36:44] = x.view(np.uint8).reshape(n, 8)
    iv = rng.integers(-2**62, 2**62, n).astype("<i8")
    rec[:, 44:52] = iv.view(np.uint8).reshape(n, 8)
    aggs = [(SUM_F64, 16, 1), (SUM_I64, 24, -1), (MAX_F64, 32, -1), (MIN_I64, 40, -1)]
    blocks = build_blocks(capi, 1, 0, 3, [rec.tobytes()])
    got, r = run(capi, "decompress_aggregate_rows", 1, 3, blocks, (KEY_INT64, 8, 8, -1, aggs), rec.size)
    assert (r["status"] == 0).all() and r["n_records"] == n and r["n_groups"] == 1
    want = bytearray(rec[0].tobytes())
    want[4:12] = bytes(8)
    want[20:28] = np.add.accumulate(np.concatenate([[0.0], x[~nulls]]))[-1:].tobytes()
    want[28:36] = int(n).to_bytes(8, "little")
    want[36:44] = x[int(np.argmax(x))].tobytes()
    want[44:52] = iv.min().tobytes()
    assert got == bytes(want)


# ---------------------------------------------------------------------------------------------------------------
# 3. errors
# ---------------------------------------------------------------------------------------------------------------
def good_rows(rng, n=300):
    return make_rows(rng, n, KEY_INT64, rng.integers(0, 30, n), [SUM_I64], tail=False)[0]


AGG1 = [(SUM_I64, 16, 1)]


@pytest.mark.parametrize("rule", ["negative", "past_end", "cut_prefix", "short_for_key", "short_for_null",
                                  "short_for_agg", "short_for_agg_null"])
def test_each_framing_rule_fails_its_block(capi, rule):
    rng = np.random.default_rng(60)
    pad = lambda rows: [r + bytes(16) for r in rows]  # 40-byte rows: room for every slot and null word below
    good = [stream(pad(good_rows(rng))) for _ in range(3)]
    head = stream(pad(good_rows(rng, 10)))
    bad = {
        "negative": head + (-5).to_bytes(4, "big", signed=True) + bytes(16),
        "past_end": head + (100).to_bytes(4, "big") + bytes(50),
        "cut_prefix": head + bytes(2),
        "short_for_key": head + stream([bytes(15)]),
        "short_for_null": head + stream([bytes(17)]),      # holds the key, not the key's null word 16..24
        "short_for_agg": head + stream([bytes(23)]),       # not the slot 16..24
        "short_for_agg_null": head + stream([bytes(24)]),  # not aggregate null bit 200's word 24..32
    }[rule]
    nf = 130 if rule == "short_for_null" else 0
    aggs = {"short_for_null": [(SUM_I64, 24, -1)], "short_for_agg_null": [(SUM_I64, 16, 200)]}.get(rule, AGG1)
    plain = [good[0], bad, good[1], good[2]]
    why = {"short_for_agg": b"shorter than an aggregate slot", "short_for_agg_null": b"shorter than an aggregate slot"}
    for codec in (0, 1):
        blocks = build_blocks(capi, codec, 1, 3, plain)
        for dev in (False, True):
            got, r = run(capi, "decompress_aggregate_rows", codec, 3, blocks, (KEY_INT64, 8, 8, nf, aggs),
                         sum(map(len, plain)), dev)
            assert list(r["status"]) == [0, capi.E_CORRUPT, 0, 0]
            assert r["n_records"] == 0 and r["n_groups"] == 0 and r["total"] == 0 and got == b""
            err = capi.load().b2s_last_error()
            assert b"block 1: " in err and (b"at byte %d:" % len(head)) in err, err
            assert why.get(rule, b"") in err


def test_bad_checksum_in_one_block(capi):
    rng = np.random.default_rng(61)
    plain = [stream(good_rows(rng)) for _ in range(3)]
    for codec in (0, 2):
        blocks = list(build_blocks(capi, codec, 1, 2, plain))
        blocks[5] = blocks[5].copy()
        blocks[5][1] ^= 0x10
        for dev in (False, True):
            got, r = run(capi, "decompress_aggregate_rows", codec, 2, tuple(blocks), (KEY_INT64, 8, 8, -1, AGG1),
                         sum(map(len, plain)), dev)
            assert list(r["status"]) == [0, capi.E_CHECKSUM, 0] and r["bad_slice"][1] == 0
            assert r["n_groups"] == 0 and got == b""


def test_short_destination_reports_the_output_bytes(capi):
    rng = np.random.default_rng(62)
    plain = [stream(good_rows(rng)) for _ in range(2)]
    want, _, _ = model_aggregate(plain, [(KEY_INT64, 8, 8, -1)], AGG1)
    blocks = build_blocks(capi, 1, 0, 0, plain)
    for dev in (False, True):
        with pytest.raises(capi.B2SError) as e:
            run(capi, "decompress_aggregate_rows", 1, 0, blocks, (KEY_INT64, 8, 8, -1, AGG1), len(want) - 1, dev)
        assert e.value.code == capi.E_DST_TOO_SMALL
    arena, off, ln, _, _, _ = blocks
    dst = np.zeros(len(want), np.uint8)
    total, nrec, ngrp = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    st, bad = np.zeros(2, np.int32), np.zeros(2, np.int32)
    op, ao, an = np.array([SUM_I64], np.uint32), np.array([16], np.uint32), np.array([1], np.int32)
    rc = capi.load().b2s_decompress_aggregate_rows_packed(
        1, 0, 2, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None, KEY_INT64, 8, 8, -1, 1,
        op.ctypes.data, ao.ctypes.data, an.ctypes.data, dst.ctypes.data, len(want) - 1, C.byref(total), C.byref(nrec),
        C.byref(ngrp), st.ctypes.data, bad.ctypes.data)
    assert rc == capi.E_DST_TOO_SMALL and total.value == len(want) and ngrp.value == 0
    got, r = run(capi, "decompress_aggregate_rows", 1, 0, blocks, (KEY_INT64, 8, 8, -1, AGG1), len(want))
    assert got == want


@pytest.mark.parametrize("aggs,nf", [
    ([(SUM_I64, 16 + 8 * k, -1) for k in range(17)], -1),  # n_aggs > 16
    ([(8, 16, -1)], -1),                                    # unknown op
    ([(SUM_I64, 16, -2)], -1),                              # agg_null_field < -1
    ([(SUM_I64, 16, -1), (MIN_I64, 20, -1)], -1),           # slots overlap
    ([(SUM_I64, 12, -1)], -1),                              # slot overlaps the key (8..16)
    ([(SUM_I64, 0, -1)], 3),                                # slot overlaps the key's null word
    ([(SUM_I64, 16, -1), (MAX_I64, 24, 130)], -1),          # slot overlaps an aggregate's null word (16..24)
])
def test_bad_aggregate_arguments(capi, aggs, nf):
    rng = np.random.default_rng(63)
    blocks = build_blocks(capi, 1, 0, 0, [stream(good_rows(rng))])
    with pytest.raises(capi.B2SError) as e:
        run(capi, "decompress_aggregate_rows", 1, 0, blocks, (KEY_INT64, 8, 8, nf, aggs), 1 << 16)
    assert e.value.code == capi.E_ARG


def test_null_aggregate_arrays_and_row_sort_argument_errors(capi):
    rng = np.random.default_rng(64)
    arena, off, ln, _, _, _ = build_blocks(capi, 1, 0, 0, [stream(good_rows(rng))])
    dst = np.zeros(1 << 16, np.uint8)
    total, nrec, ngrp = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    st, bad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = capi.load().b2s_decompress_aggregate_rows_packed(
        1, 0, 1, arena.ctypes.data, off.ctypes.data, ln.ctypes.data, None, None, None, KEY_INT64, 8, 8, -1, 1,
        None, None, None, dst.ctypes.data, dst.size, C.byref(total), C.byref(nrec), C.byref(ngrp), st.ctypes.data,
        bad.ctypes.data)
    assert rc == capi.E_ARG
    for kt, kl in ((3, 8), (KEY_INT64, 4)):
        with pytest.raises(capi.B2SError) as e:
            run(capi, "decompress_aggregate_rows", 1, 0, (arena, off, ln, None, None, None), (kt, 8, kl, -1, AGG1),
                1 << 16)
        assert e.value.code == capi.E_ARG


# ---------------------------------------------------------------------------------------------------------------
# 4. end to end: partial-aggregate rows written by several maps, each reducer's rows merged
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,codec,level", [("snappy", 2, 0), ("lz4", 1, 0), ("none", 0, 0)])
def test_partition_then_aggregate_end_to_end(capi, name, codec, level):
    M, R, per_map = 4, 6, 4000
    maps = []
    for m in range(M):
        rng = np.random.default_rng(70 + m)
        rows, aggs = make_rows(rng, per_map, KEY_INT64, rng.integers(0, 500, per_map), [SUM_I64, SUM_F64, MAX_I32],
                               key_null=0, key_null_frac=0.02)
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
        got, _ = check(capi, codec, level, 3, plain, KEY_INT64, 8, 8, 0, aggs,
                       blocks=(arena, off, lens, np.arange(M + 1, dtype=np.uint32), lens, ck))
        direct, _ = check(capi, 0, 0, 0, [b"".join(plain)], KEY_INT64, 8, 8, 0, aggs)
        assert got == direct


# ---------------------------------------------------------------------------------------------------------------
# 5. the host mirror: b2sh_reader_read_aggregated_rows over the serialized writer's files
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("codec", ["lz4", "none"])
def test_host_mirror_reads_rows_aggregated(tmp_path, codec):
    host = pkg.host
    d = mirror(tmp_path, codec)
    M, R, per_map = 3, 3, 2000
    maps = []
    for m in range(M):
        rng = np.random.default_rng(80 + m)
        rows, aggs = make_rows(rng, per_map, KEY_INT32, rng.integers(-50, 50, per_map), [SUM_I64, MIN_F64, MAX_I64],
                               key_null=0, key_null_frac=0.05)
        maps.append((rows, rng.integers(0, R, per_map)))
    write_maps(host, d, maps, R)
    for red in range(R):
        rd = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        data, n, g = rd.readAggregatedRows(KEY_INT32, 8, 4, 0, aggs)
        rd.close()
        want, wn, wg = model_aggregate([stream([r for r, p in zip(rows, ids) if p == red]) for rows, ids in maps],
                                       [(KEY_INT32, 8, 4, 0)], aggs)
        assert (n, g) == (wn, wg) and data == want
    d.close()


def test_host_mirror_checksum_and_malformed_errors(tmp_path):
    host = pkg.host
    d = mirror(tmp_path, "lz4")
    rng = np.random.default_rng(90)
    write_maps(host, d, [(good_rows(rng, 2000), np.zeros(2000, np.int64))], 2)
    w = host.S3SerializedShuffleWriter(d, 0, 1, 2)  # map 1: a row cut short by 3 bytes
    w.insertRecord(0, (40).to_bytes(4, "big") + bytes(37))
    w.commit()
    w.close()
    rd = host.S3ShuffleReader(d, 0, [1], 0, 1)
    with pytest.raises(host.IOException):
        rd.readAggregatedRows(KEY_INT64, 8, 8, -1, AGG1)
    rd.close()
    path = d.getPath("data", 0, 0)
    raw = bytearray(open(path, "rb").read())
    raw[30] ^= 0x04
    open(path, "wb").write(raw)
    rd = host.S3ShuffleReader(d, 0, [0], 0, 1)
    with pytest.raises(host.SparkException, match=r"Invalid checksum detected for shuffle_0_0_0$"):
        rd.readAggregatedRows(KEY_INT64, 8, 8, -1, AGG1)
    rd.close()
    d.close()
