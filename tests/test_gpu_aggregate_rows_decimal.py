"""The Decimal aggregate ops of the row aggregation (B2S_AGG_SUM_DECIMAL | P << 8, MIN / MAX_DECIMAL) on the GPU,
against the Python-integer model of tests/decimal_model.py: Spark's Sum and Average decimal buffers, compact and out of
line, null on a null input or a running sum out of range, and Min / Max of Decimal(p > 18); the single-key and
composite-key calls, packed and _dev, codec NONE and Snappy; the corrupt-record rules; a q67-shaped exchange end to
end."""
import ctypes as C

import numpy as np
import pytest

import spark_s3_shuffle_b200 as pkg
from decimal_model import MAX_DEC, MIN_DEC, model_aggregate_decimal, sum_decimal, to_byte_array, wide
from rows_model import KEY_INT32, KEY_INT64, MIN_I32, STRING, SUM_I64, blocks_of, build_blocks, mirror, parse, run, \
    stream, write_maps

pytestmark = pytest.mark.gpu

CODECS = [("none", 0, 0), ("snappy", 2, 0)]
KEY = (KEY_INT64, 8, 8, 0)


# ---------------------------------------------------------------------------------------------------------------
# rows: one null word, field 0 the int64 key (null bit 0), field a + 1 aggregate a (null bit a + 1), then 16 bytes per
# out-of-line decimal, then a random tail
# ---------------------------------------------------------------------------------------------------------------
def make_rows(rng, keys, ops, vals, extra_len=None, tail=True):
    """vals[a][i]: aggregate a of row i (an int; None = null; for a plain op the 8-byte slot's int).  extra_len[a][i]:
    an out-of-line value's byte length (sign-extended past the minimal one; default minimal)"""
    m = len(ops)
    nwide = sum(1 for op in ops if wide(op))
    fixed = 8 + 8 * (m + 1)
    rows = []
    for i, k in enumerate(keys):
        t = int(rng.integers(0, 24)) if tail else 0
        r = bytearray(rng.integers(0, 256, fixed + 16 * nwide + t, dtype=np.uint8).tobytes())
        word = 0
        r[8:16] = int(k).to_bytes(8, "little", signed=True)
        w = 0
        for a, op in enumerate(ops):
            off = 16 + 8 * a
            v = vals[a][i]
            if v is None:
                word |= 1 << (a + 1)
            if wide(op):
                o = fixed + 16 * w
                w += 1
                r[o:o + 16] = rng.integers(0, 256, 16, dtype=np.uint8).tobytes()  # garbage the merge must zero
                if v is None:
                    r[off:off + 8] = (o << 32).to_bytes(8, "little")
                else:
                    b = to_byte_array(v)
                    n = max(len(b), extra_len[a][i]) if extra_len and extra_len[a] is not None else len(b)
                    b = v.to_bytes(n, "big", signed=True)
                    r[o:o + n] = b
                    r[off:off + 8] = ((o << 32) | n).to_bytes(8, "little")
            else:
                r[off:off + 8] = (0 if v is None else v & (2**64 - 1)).to_bytes(8, "little")
        r[0:8] = word.to_bytes(8, "little")
        rows.append(bytes(r))
    aggs = [(op, 16 + 8 * a, a + 1 if op & 0xFF != MIN_I32 else -1) for a, op in enumerate(ops)]
    return rows, aggs


def check(capi, codec, plain, aggs, keys=(KEY,), dev=False, composite=False):
    blocks = build_blocks(capi, codec, 0, 3, plain)
    total = sum(len(b) for b in plain)
    if composite:
        got, r = run(capi, "decompress_aggregate_rows_keys", codec, 3, blocks, (list(keys), aggs), total, dev)
    else:
        got, r = run(capi, "decompress_aggregate_rows", codec, 3, blocks, (*keys[0], aggs), total, dev)
    assert (r["status"] == 0).all(), r["status"]
    want, n, g = model_aggregate_decimal(plain, list(keys), aggs)
    assert (r["n_records"], r["n_groups"], r["total"]) == (n, g, len(want))
    assert got == want
    return got


def group_keys(rng, sizes):
    keys = np.concatenate([np.full(s, g) for g, s in enumerate(sizes)])
    return rng.permutation(keys)


def rand_dec(rng, p, n, null_frac=0.0):
    """values below 10^p in magnitude, many of them near it"""
    out = []
    for _ in range(n):
        if rng.random() < null_frac:
            out.append(None)
            continue
        digits = int(rng.integers(1, p + 1))
        v = int(rng.integers(0, 10**min(digits, 18))) * 10**max(0, digits - 18)
        out.append(v if rng.random() < 0.5 else -v)
    return out


SIZES = [1] * 40 + [16] * 20 + [17] * 20 + [130, 300, 1000, 129]


# ---------------------------------------------------------------------------------------------------------------
# 1. Sum and Average layouts against the model
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["sum", "avg"])
@pytest.mark.parametrize("p", [7, 17, 18, 19, 28, 38])
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_sum_and_average_buffers_like_the_model(capi, name, codec, level, p, layout):
    rng = np.random.default_rng(p * 10 + codec + (layout == "avg"))
    keys = group_keys(rng, SIZES)
    n = len(keys)
    sums = rand_dec(rng, p, n, null_frac=0.01)
    second = [int(x) for x in rng.integers(0, 2, n)] if layout == "sum" else [int(x) for x in rng.integers(0, 9, n)]
    ops = [sum_decimal(p), MIN_I32 if layout == "sum" else SUM_I64]
    rows, aggs = make_rows(rng, keys, ops, [sums, second])
    plain = blocks_of(rows, [n // 3, 0, n - n // 3])
    a = check(capi, codec, plain, aggs)
    b = check(capi, codec, plain, aggs, dev=True)
    c = check(capi, codec, plain, aggs, composite=True)
    assert a == b == c


# ---------------------------------------------------------------------------------------------------------------
# 2. where the overflow and the null input fall
# ---------------------------------------------------------------------------------------------------------------
def overflow_group(p, size, at, kind):
    """a group of size records whose running sum first leaves the range at record at (kind "over"), whose prefix
    leaves it while the total is back in range ("prefix"), or whose record at is null ("null")"""
    big = 10**p - 1
    vals = [0] * size
    if kind == "null":
        vals = [1] * size
        vals[at] = None
        return vals
    if at == 0:
        vals[0] = 10**p if p <= 18 or kind == "over" else -(10**p)
    else:
        vals[0] = big
        vals[at] = 1
    if kind == "prefix" and at + 1 < size:
        vals[at + 1] = -big
    return vals


CASES = [(size, at) for size in (1, 5, 16, 17, 40, 300)
         for at in sorted({0, size // 2, 31, 127, size - 1}) if at < size]


@pytest.mark.parametrize("kind", ["over", "prefix", "null"])
@pytest.mark.parametrize("p", [17, 38])
def test_overflow_and_null_positions(capi, p, kind):
    rng = np.random.default_rng(p + len(kind))
    keys, vals = [], []
    for g, (size, at) in enumerate(CASES):
        keys += [g] * size
        vals += overflow_group(p, size, at, kind)
    g_ok = len(CASES)  # a group in range throughout: not null
    keys += [g_ok] * 200
    vals += [10**p // 300] * 200
    rows, aggs = make_rows(rng, keys, [sum_decimal(p)], [vals])
    for codec in (0, 2):
        got = check(capi, codec, blocks_of(rows, [len(rows) // 2, len(rows) - len(rows) // 2]), aggs)
        out = [got[o + 4:o + ln] for o, ln in parse(got)]
        nulls = [(int.from_bytes(r[:8], "little") >> 1) & 1 for r in out]
        if kind != "prefix":
            assert nulls == [1] * len(CASES) + [0]
        else:  # the prefix cases whose next record exists end in range yet stay null
            assert all(nulls[:-1]) and nulls[-1] == 0


def test_composite_key_and_dev_on_overflowing_groups(capi):
    rng = np.random.default_rng(7)
    keys, vals = [], []
    for g, (size, at) in enumerate(CASES):
        keys += [g] * size
        vals += overflow_group(28, size, at, "over")
    rows, aggs = make_rows(rng, keys, [sum_decimal(28)], [vals])
    plain = blocks_of(rows, [len(rows)])
    for dev in (False, True):
        check(capi, 2, plain, aggs, dev=dev, composite=True)


# ---------------------------------------------------------------------------------------------------------------
# 3. min / max of Decimal(p > 18)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,codec,level", CODECS)
def test_min_max_with_negatives_and_mixed_lengths(capi, name, codec, level):
    rng = np.random.default_rng(30 + codec)
    keys = group_keys(rng, SIZES + [3] * 30)
    n = len(keys)
    edges = [0, 1, -1, 127, 128, -128, -129, 10**38 - 1, -(10**38 - 1), 2**63, -2**63 - 1]
    mins = [int(rng.choice(edges)) if rng.random() < 0.3 else v for v in rand_dec(rng, 38, n, null_frac=0.2)]
    maxs = rand_dec(rng, 30, n, null_frac=0.2)
    extra = [[int(x) for x in rng.integers(1, 17, n)] for _ in range(2)]
    all_null = [None] * n  # a group with no non-null input is null
    rows, aggs = make_rows(rng, keys, [MIN_DEC, MAX_DEC, MAX_DEC], [mins, maxs, all_null], extra_len=extra + [None])
    plain = blocks_of(rows, [n // 2, n - n // 2])
    a = check(capi, codec, plain, aggs)
    b = check(capi, codec, plain, aggs, dev=True)
    assert a == b
    assert check(capi, codec, plain, aggs, composite=True) == a


# ---------------------------------------------------------------------------------------------------------------
# 4. one hot reducer: a single group of more than a million rows
# ---------------------------------------------------------------------------------------------------------------
def test_one_group_of_more_than_a_million_rows(capi):
    n = 1 << 20
    rng = np.random.default_rng(40)
    # rows of 64 bytes: null word, key, sum slot, isEmpty slot, count slot, 16 value bytes, 8 spare
    vals = rng.integers(-4 * 10**18, 4 * 10**18, n)  # the sum needs more than 64 bits, far below 10^28
    rows = np.zeros((n, 64), np.uint8)
    rows[:, 8:16] = np.frombuffer(np.int64(5).tobytes(), np.uint8)
    slot = (np.uint64(40) << np.uint64(32)) | np.uint64(16)
    rows[:, 16:24] = np.frombuffer(slot.tobytes(), np.uint8)
    rows[:, 32:40] = np.frombuffer(np.int64(1).tobytes(), np.uint8)
    hi = np.where(vals < 0, -1, 0).astype(">i8")
    rows[:, 40:48] = hi.view(np.uint8).reshape(n, 8)
    rows[:, 48:56] = vals.astype(">i8").view(np.uint8).reshape(n, 8)
    rec = np.zeros((n, 68), np.uint8)
    rec[:, 0:4] = np.frombuffer((64).to_bytes(4, "big"), np.uint8)
    rec[:, 4:] = rows
    plain = [rec[: n // 2].tobytes(), rec[n // 2:].tobytes()]
    aggs = [(sum_decimal(28), 16, 1), (MIN_I32, 24, -1), (SUM_I64, 32, 3)]
    want = int(vals.sum(dtype=object))
    for codec in (0, 2):
        blocks = build_blocks(capi, codec, 0, 3, plain)
        for dev in (False, True):
            got, r = run(capi, "decompress_aggregate_rows", codec, 3, blocks, (*KEY, aggs), 68 * n, dev)
            assert (r["n_records"], r["n_groups"], r["total"]) == (n, 1, 68)
            row = got[4:]
            assert int.from_bytes(row[:8], "little") & 0b1110 == 0
            s = int.from_bytes(row[16:24], "little")
            o, ln = s >> 32, s & 0xFFFFFFFF
            assert o == 40 and int.from_bytes(row[o:o + ln], "big", signed=True) == want
            assert bytes(row[o:o + ln]) == to_byte_array(want) and row[o + ln:o + 16] == bytes(16 - ln)
            assert int.from_bytes(row[32:40], "little") == n


# ---------------------------------------------------------------------------------------------------------------
# 5. corrupt records and argument errors
# ---------------------------------------------------------------------------------------------------------------
def one_wide_row(key, size, region, value=5, null=False, row_len=48):
    """null word, key, a Decimal(28) sum slot naming size bytes at region, then the region"""
    r = bytearray(row_len)
    b = value.to_bytes(16, "big", signed=True)[16 - min(max(size, 1), 16):]
    r[region:region + len(b)] = b[: max(0, row_len - region)]
    r[0:8] = ((1 << 1) if null else 0).to_bytes(8, "little")
    r[8:16] = key.to_bytes(8, "little")
    r[16:24] = ((region << 32) | size).to_bytes(8, "little")
    return bytes(r[:row_len])


@pytest.mark.parametrize("rule,row,why", [
    ("size_zero", one_wide_row(1, 0, 24), b"size is not in [1, 16]"),
    ("size_17", one_wide_row(1, 17, 24, row_len=48), b"size is not in [1, 16]"),
    ("bytes_past_row", one_wide_row(1, 16, 36, row_len=48), b"bytes run past the end of its row"),
    ("region_past_row_null", one_wide_row(1, 0, 40, null=True, row_len=48), b"16-byte region runs past"),
    ("region_in_slots", one_wide_row(1, 4, 16, row_len=48), b"starts before the end of a slot"),
    ("region_in_null_word", one_wide_row(1, 4, 4, row_len=48), b"starts before the end of a slot"),
])
def test_each_corrupt_decimal_rule_fails_its_block(capi, rule, row, why):
    good = [stream([one_wide_row(k % 7, 16, 24, value=k * 10**20) for k in range(200)]) for _ in range(3)]
    head = stream([one_wide_row(k, 16, 24) for k in range(10)])
    plain = [good[0], head + stream([row]), good[1], good[2]]
    aggs = [(sum_decimal(28), 16, 1)]
    for codec in (0, 2):
        blocks = build_blocks(capi, codec, 0, 3, plain)
        for dev in (False, True):
            for composite in (False, True):
                name = "decompress_aggregate_rows" + ("_keys" if composite else "")
                args = ([KEY], aggs) if composite else (*KEY, aggs)
                got, r = run(capi, name, codec, 3, blocks, args, sum(map(len, plain)), dev)
                assert list(r["status"]) == [0, capi.E_CORRUPT, 0, 0]
                assert r["n_records"] == 0 and r["n_groups"] == 0 and r["total"] == 0 and got == b""
                err = capi.load().b2s_last_error()
                assert b"block 1: " in err and (b"at byte %d:" % len(head)) in err and why in err, err


def test_nothing_is_written_when_a_decimal_is_corrupt(capi):
    plain = [stream([one_wide_row(1, 16, 24), one_wide_row(1, 0, 24)])]
    blocks = build_blocks(capi, 0, 0, 0, plain)
    arena, off, ln, _, _, _ = blocks
    d_src = capi.dev_alloc(arena.size)
    d_dst = capi.dev_alloc(4096)
    try:
        capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        marker = np.full(4096, 0xA5, np.uint8)
        capi.dev_memcpy(d_dst, marker.ctypes.data, 4096, 1)
        r = capi.decompress_aggregate_rows_dev(0, d_src, off, ln, d_dst, 4096, *KEY, aggs=[(sum_decimal(28), 16, 1)])
        assert list(r["status"]) == [capi.E_CORRUPT] and r["total"] == 0
        back = np.zeros(4096, np.uint8)
        capi.dev_memcpy(back.ctypes.data, d_dst, 4096, 2)
        assert (back == 0xA5).all()
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)


@pytest.mark.parametrize("aggs", [
    [(sum_decimal(0), 16, 1)],            # precision 0
    [(sum_decimal(39), 16, 1)],           # precision above 38
    [(9 | (255 << 8), 16, 1)],            # precision 255
    [(SUM_I64 | (10 << 8), 16, 1)],       # precision bits on another op
    [(MAX_DEC | (20 << 8), 16, 1)],
    [(sum_decimal(20), 16, -1)],          # SUM_DECIMAL without a null field
    [(sum_decimal(10), 16, -1)],
    [(12, 16, 1)],                        # unknown ops
    [(8 | (20 << 8), 16, 1)],
    [(sum_decimal(20) | (1 << 16), 16, 1)],
])
def test_bad_decimal_arguments(capi, aggs):
    blocks = build_blocks(capi, 0, 0, 0, [stream([one_wide_row(1, 16, 24)])])
    for name, args in (("decompress_aggregate_rows", (*KEY, aggs)),
                       ("decompress_aggregate_rows_keys", ([KEY], aggs))):
        with pytest.raises(capi.B2SError) as e:
            run(capi, name, 0, 0, blocks, args, 1 << 16)
        assert e.value.code == capi.E_ARG


# ---------------------------------------------------------------------------------------------------------------
# 6. the host mirror, and a q67-shaped exchange end to end
# ---------------------------------------------------------------------------------------------------------------
def test_host_mirror_reads_decimal_aggregates_by_composite_key(tmp_path):
    host = pkg.host
    d = mirror(tmp_path, "lz4")
    M, R, per_map = 3, 2, 1500
    maps, aggs = [], None
    for m in range(M):
        rng = np.random.default_rng(50 + m)
        keys = rng.integers(-40, 40, per_map)
        ops = [sum_decimal(28), MIN_I32, MAX_DEC]
        rows, aggs = make_rows(rng, keys, ops, [rand_dec(rng, 24, per_map, 0.01),
                                                 [int(x) for x in rng.integers(0, 2, per_map)],
                                                 rand_dec(rng, 38, per_map, 0.1)])
        maps.append((rows, rng.integers(0, R, per_map)))
    write_maps(host, d, maps, R)
    keys = [KEY]
    for red in range(R):
        rd = host.S3ShuffleReader(d, 0, list(range(M)), red, red + 1)
        data, n, g = rd.readAggregatedRowsKeys(keys, aggs)
        rd.close()
        want, wn, wg = model_aggregate_decimal([stream([r for r, p in zip(rows, ids) if p == red])
                                                for rows, ids in maps], keys, aggs)
        assert (n, g) == (wn, wg) and data == want
    d.close()


def q67_rows(rng, n, n_keys):
    """q67's partial rows: 8 grouping columns (5 strings, 3 ints), a Decimal(28, 2) sum and isEmpty"""
    cats = [b"Books", b"Music", b"Home", b"Sports", b"Electronics and more"]
    key_tuples = [(cats[k % 5], b"class%d" % (k % 3), b"brand-%d" % (k % 11), b"product-%04d" % k,
                   1998 + k % 5, 1 + k % 4, 1 + k % 12, b"AAAAAAAAB%02dAAAA" % (k % 7)) for k in range(n_keys)]
    rows, truth = [], {}
    for _ in range(n):
        kt = key_tuples[int(rng.integers(0, n_keys))]
        v = int(rng.integers(-10**15, 10**15)) * 10**5 + int(rng.integers(0, 10**5))
        truth[kt] = truth.get(kt, 0) + v
        fixed = 8 + 8 * 10
        var = bytearray()
        r = bytearray(fixed)
        for c, x in enumerate(kt):
            o = 8 + 8 * c
            if isinstance(x, bytes):
                r[o:o + 8] = ((fixed + len(var)) << 32 | len(x)).to_bytes(8, "little")
                var += x + bytes((-len(x)) % 8)
            else:
                r[o:o + 8] = x.to_bytes(8, "little")
        b = to_byte_array(v)
        r[8 + 64:8 + 72] = ((fixed + len(var)) << 32 | len(b)).to_bytes(8, "little")
        var += b + bytes(16 - len(b))
        r[8 + 72:8 + 80] = (0).to_bytes(8, "little")  # isEmpty = false
        rows.append(bytes(r + var))
    return rows, truth


def test_q67_exchange_end_to_end(capi):
    M, R, per_map = 4, 5, 3000
    kinds = [STRING] * 4 + [KEY_INT32] * 3 + [STRING]
    keys = [(kinds[c], 8 + 8 * c, 8 if kinds[c] == STRING else 4, c) for c in range(8)]
    aggs = [(sum_decimal(28), 8 + 64, 8), (MIN_I32, 8 + 72, -1)]
    truth, outs = {}, []
    for m in range(M):
        rng = np.random.default_rng(90 + m)
        rows, t = q67_rows(rng, per_map, 600)
        for k, v in t.items():
            truth[k] = truth.get(k, 0) + v
        recs = np.frombuffer(stream(rows), np.uint8)
        rec_len = np.array([4 + len(r) for r in rows], np.uint32)
        dst = np.zeros(capi.partition_compress_bound(2, 0, R, recs.size), np.uint8)
        r = capi.partition_compress_rows_hash_packed(2, recs, rec_len, keys, R, dst, checksum_alg=3)
        outs.append((dst[: r["total"]].copy(), r))
    got = {}
    for red in range(R):
        blocks = [o[int(r["dst_off"][red]):int(r["dst_off"][red] + r["dst_len"][red])] for o, r in outs]
        lens = np.array([b.size for b in blocks], np.uint64)
        arena = np.concatenate(blocks + [np.zeros(1, np.uint8)])
        off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        ck = np.array([r["checksums"][red] for _, r in outs], np.uint64)
        data, res = run(capi, "decompress_aggregate_rows_keys", 2, 3,
                        (arena, off, lens, np.arange(M + 1, dtype=np.uint32), lens, ck), (keys, aggs),
                        int(lens.sum()) * 8 + 4096)
        assert (res["status"] == 0).all()
        for o, ln in parse(data):
            row = data[o + 4:o + ln]
            kt = []
            for c in range(8):
                s = int.from_bytes(row[8 + 8 * c:16 + 8 * c], "little")
                kt.append(bytes(row[s >> 32:(s >> 32) + (s & 0xFFFFFFFF)]) if kinds[c] == STRING
                          else int.from_bytes(row[8 + 8 * c:12 + 8 * c], "little", signed=True))
            s = int.from_bytes(row[72:80], "little")
            assert (int.from_bytes(row[:8], "little") >> 8) & 1 == 0
            assert tuple(kt) not in got
            got[tuple(kt)] = int.from_bytes(row[s >> 32:(s >> 32) + (s & 0xFFFFFFFF)], "big", signed=True)
    assert got == truth
