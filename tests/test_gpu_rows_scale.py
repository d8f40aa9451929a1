"""The UnsafeRow reduce calls and the row partitioners past 4 GiB of rows, and at Spark's 2^31 - 1 byte row limit.

The row code keeps 64-bit byte offsets next to 32-bit record positions, counts and lengths: the framing's bitmap and
its per-tile counts, the packed (count | s << 32) scans, the radix scatter's bucket bases, group, partition and partner
positions, and the span copies' lengths.  Each is right only while the arithmetic around it stays 64-bit, and only an
input past 2^32 bytes (and 2^26 records) shows it.  Every case here asserts the sizes it exists to reach.

Inputs are generated with numpy and every expected output comes from a plain vectorised reference over them (order
from a stable argsort, integer aggregates from reduceat, double sums added in record order, windows from cumsum and
shifted indices, joins from repeat over the matched ranges, partitions from a stable argsort of the ids).  The
references are checked against the scalar models on small inputs in test_rows_scale_reference.py.  Outputs are copied
back and compared in slices of at most 256 MiB.

The shared arena is 68 M records of 68 bytes (4.62 GB, one group and one window partition of 2.3 GB), generated once
for the row sorts, the aggregate, the window and the partitioners; the composite-key sort generates its own arena of the
same size and frees it.  Measured over the whole module on an H100 80GB HBM3 (700 W power limit): about 8 minutes,
device memory in use peaking at 29 GiB and the host's resident memory at 20.9 GB.
A card that cannot give the memory fails the case with the library's E_NOMEM; nothing here skips.
"""
import ctypes as C
import functools
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import hash_model as hm

pytestmark = pytest.mark.gpu

MiB, GiB = 1 << 20, 1 << 30
PIECE = 256 * MiB  # the most of one device buffer held on the host at a time
LIMIT = (1 << 31) - 1  # Spark's largest row

KEY_INT64 = 2
INT64_MIN = np.iinfo(np.int64).min

# ---------------------------------------------------------------------------------------------------------------
# the arena's rows: a null word (bit 0: the key is null), then seven 8-byte fields
# ---------------------------------------------------------------------------------------------------------------
NF = 7
KEY, V, D, LO, HI, ONE, IDX = 8, 16, 24, 32, 40, 48, 56  # row offsets: key, int64, double, int64, double, 1, index
ROW = 8 + 8 * NF
REC = 4 + ROW
N = 68_000_000  # 4.62e9 bytes > 2^32, > 2^26 records
GIANT_KEY = 7
N_BLOCKS = 40


def make_rows(n, seed, giant=0.5, nulls=0.03, domain=500_000):
    """n records of REC bytes as an (n, REC) uint8 array.  A share `giant` of the keys is GIANT_KEY, a share `nulls`
    is null (their key bytes stay random), the rest are uniform in [-domain, domain]: many ties, one huge group"""
    rng = np.random.default_rng(seed)
    rec = np.empty((n, REC), np.uint8)
    rec[:, :4] = np.frombuffer(ROW.to_bytes(4, "big"), np.uint8)
    w = rec[:, 4:].view("<i8")  # (n, 8): null word, then the fields
    u = rng.random(n)
    key = rng.integers(-domain, domain + 1, n)
    key[u < giant] = GIANT_KEY
    w[:, 0] = u >= 1 - nulls
    w[:, KEY // 8] = key
    del key, u
    w[:, V // 8] = rng.integers(-2**35, 2**35, n)  # |any sum| < 2^62: the int64 references cannot wrap
    w[:, D // 8] = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 30, n))).view("<i8")
    w[:, LO // 8] = rng.integers(INT64_MIN, 2**63 - 1, n)
    w[:, HI // 8] = rng.standard_normal(n).view("<i8")  # no NaN, no -0.0: numpy's max is Spark's here
    w[:, ONE // 8] = 1
    w[:, IDX // 8] = np.arange(n)
    return rec


def field(rec, off, dt="<i8"):
    return rec[:, 4 + off:4 + off + 8].view(dt)[:, 0]


def is_null(rec):
    return (field(rec, 0) & 1).astype(bool)


def sort_order(rec):
    """the stable order of a nullable int64 key, nulls first (a null's key bytes ignored)"""
    null = is_null(rec)
    return np.lexsort((np.where(null, 0, field(rec, KEY)), ~null))


# the composite key: an int32 DESC column and a string of 25..32 bytes that all share their first 24, so the refine
# rounds past the first string bytes decide.  Row: null word (bit 0: the int is null, bit 1: the string), the int32,
# the string's slot, the index, then the string's 32-byte var region (zero past the string).
KEY_INT32, STRING_KEY, DESC = 1, 3, 1 << 8
S_OFF, S_PREFIX = 32, 24
COMPOSITE_KEYS = [(KEY_INT32 | DESC, 8, 4, 0), (STRING_KEY, 16, 8, 1)]


def make_keyed_rows(n, seed, nulls=0.02, domain=40):
    rng = np.random.default_rng(seed)
    rec = np.zeros((n, REC), np.uint8)
    rec[:, :4] = np.frombuffer(ROW.to_bytes(4, "big"), np.uint8)
    w = rec[:, 4:].view("<i8")
    w[:, 0] = (rng.random(n) < nulls) | (rng.random(n) < nulls) << 1
    rec[:, 12:16].view("<i4")[:, 0] = rng.integers(-domain, domain + 1, n)
    w[:, 2] = S_OFF << 32 | rng.integers(S_PREFIX + 1, S_PREFIX + 9, n)
    w[:, 3] = np.arange(n)
    rec[:, 4 + S_OFF:4 + S_OFF + S_PREFIX] = np.random.default_rng(0).integers(0, 256, S_PREFIX, dtype=np.uint8)
    alphabet = np.array([0, 1, 0x7F, 0x80, 0xFF], np.uint8)  # few values: many equal suffixes, and proper prefixes
    for j in range(8):
        live = S_PREFIX + j < (w[:, 2] & 0xFFFFFFFF)
        rec[live, 4 + S_OFF + S_PREFIX + j] = alphabet[rng.integers(0, alphabet.size, int(live.sum()))]
    return rec


def keyed_order(rec):
    """the stable order of COMPOSITE_KEYS: int32 descending, then the string's unsigned bytes (a proper prefix first),
    nulls first in each column.  Past the shared prefix a string is its suffix zero-padded to 8 bytes, as a big-endian
    u64, then its length"""
    nw = field(rec, 0)
    inull, snull = (nw & 1).astype(bool), (nw & 2).astype(bool)
    i32 = rec[:, 12:16].view("<i4")[:, 0].astype(np.int64)
    suffix = rec[:, 4 + S_OFF + S_PREFIX:4 + S_OFF + 32].copy().view(">u8")[:, 0]
    length = field(rec, 16) & 0xFFFFFFFF
    return np.lexsort((np.where(snull, 0, length), np.where(snull, 0, suffix), ~snull, np.where(inull, 0, -i32),
                       ~inull))


def group_starts(rec, order):
    """-> (starts, lengths) of the runs of equal keys in `order` (all nulls one run)"""
    null = is_null(rec)[order]
    key = np.where(null, INT64_MIN, field(rec, KEY)[order])  # no generated key is INT64_MIN
    starts = np.flatnonzero(np.concatenate([[True], key[1:] != key[:-1]]))
    return starts, np.diff(np.concatenate([starts, [order.size]]))


def sequential_sums(x, starts, lens, long_group=4096):
    """((0.0 + x[s]) + x[s + 1]) + ... for every group, in that order, bit for bit: short groups by rounds (round r adds
    the r-th value of every group longer than r), long ones by np.add.accumulate, which is sequential"""
    acc = np.zeros(starts.size)
    short = np.flatnonzero(lens <= long_group)
    for r in range(int(lens[short].max()) if short.size else 0):
        sel = short[lens[short] > r]
        acc[sel] = acc[sel] + x[starts[sel] + r]
    for g in np.flatnonzero(lens > long_group):
        acc[g] = np.add.accumulate(np.concatenate([[0.0], x[starts[g]:starts[g] + lens[g]]]))[-1]
    return acc


AGGS = [(0, V, -1), (1, D, -1), (4, LO, -1), (7, HI, -1), (0, ONE, -1), (5, IDX, -1)]  # AGG_* op, slot, null field


def aggregate_ref(rec, order, long_group=4096):
    """the aggregate call's rows for AGGS: each group's first record with int64 sum, double sum, int64 min, double max,
    count (the sum of ONE) and int64 max merged in"""
    starts, lens = group_starts(rec, order)
    out = rec[order[starts]]
    f = lambda off, dt="<i8": field(rec, off, dt)[order]  # noqa: E731
    field(out, V)[:] = np.add.reduceat(f(V), starts)
    field(out, D, "<f8")[:] = sequential_sums(f(D, "<f8"), starts, lens, long_group)
    field(out, LO)[:] = np.minimum.reduceat(f(LO), starts)
    field(out, HI, "<f8")[:] = np.maximum.reduceat(f(HI, "<f8"), starts)
    field(out, ONE)[:] = lens
    field(out, IDX)[:] = np.maximum.reduceat(f(IDX), starts)
    return out


# the window: PARTITION BY key ORDER BY index; row_number(), sum(v) ROWS UNBOUNDED PRECEDING, lag(v, 1, LAG_DEFAULT)
LAG_DEFAULT = -777
W_FNS = [0, (6, 2, 4, V, -1), (11, 1, 0, 4, V, -1, 2, LAG_DEFAULT % 2**64)]
W_KEYS = [(KEY_INT64, KEY, 8, 0), (KEY_INT64, IDX, 8, -1)]
W_ROW = 8 + 8 * (NF + 3)
W_REC = 4 + W_ROW


class WindowRef:
    """the window call's output rows, by sorted position"""

    def __init__(self, rec, order):
        self.rec, self.order = rec, order
        starts, lens = group_starts(rec, order)
        self.pstart = np.repeat(starts, lens)
        self.v = field(rec, V)[order]
        self.csum = np.cumsum(self.v)  # |partial sums| < 2^62: no wrap
        self.parts = (starts, lens)

    def rows(self, a, b):
        n = b - a
        out = np.zeros((n, W_REC), np.uint8)
        out[:, :4] = np.frombuffer(W_ROW.to_bytes(4, "big"), np.uint8)
        src = self.rec[self.order[a:b]]
        out[:, 4:4 + ROW] = src[:, 4:]
        w = out[:, 4:].view("<i8")
        w[:, 0] = field(src, 0) & ((1 << NF) - 1)  # the joined null bits: the input's, the values' are all clear
        pos, ps = np.arange(a, b), self.pstart[a:b]
        w[:, 1 + NF] = pos - ps + 1
        base = np.where(ps > 0, self.csum[np.maximum(ps - 1, 0)], 0)
        w[:, 2 + NF] = self.csum[a:b] - base
        w[:, 3 + NF] = np.where(pos > ps, self.v[np.maximum(pos - 1, 0)], LAG_DEFAULT)
        return out


# ---------------------------------------------------------------------------------------------------------------
# the join's rows: left (null word, key, index), right (null word, key, index, payload); joined: one null word, 5 slots
# ---------------------------------------------------------------------------------------------------------------
JL_ROW, JR_ROW = 24, 32
J_ROW = 8 + 8 * 5
J_REC = 4 + J_ROW
JOIN_KEYS = [(KEY_INT64, 8, 8, 0)]


def side_rows(key, null, row_bytes, rng):
    n = key.size
    rec = np.zeros((n, 4 + row_bytes), np.uint8)
    rec[:, :4] = np.frombuffer(row_bytes.to_bytes(4, "big"), np.uint8)
    w = rec[:, 4:].view("<i8")
    w[:, 0] = null
    w[:, 1] = np.where(null, rng.integers(-9, 9, n), key)
    w[:, 2] = np.arange(n)
    if row_bytes > 24:
        w[:, 3] = rng.integers(INT64_MIN, 2**63 - 1, n)
    return rec


def make_join(seed, hot=(8000, 12000), small_keys=20_000, small=(2, 3), unmatched=300_000, nulls=100_000):
    """(left, right) records: a hot key with hot[0] x hot[1] rows, small_keys keys with small[0] x small[1] rows,
    unmatched keys on each side and null keys, in a random input order"""
    rng = np.random.default_rng(seed)
    sides = []
    for s in (0, 1):
        key = np.concatenate([np.full(hot[s], 3, np.int64), np.repeat(np.arange(10, 10 + small_keys), small[s]),
                              2 * rng.integers(10**6, 10**9, unmatched) + s, np.zeros(nulls, np.int64)])
        null = np.zeros(key.size, np.int64)
        null[-nulls:] = 1
        p = rng.permutation(key.size)
        sides.append(side_rows(key[p], null[p], (JL_ROW, JR_ROW)[s], rng))
    return sides


def join_index(left, right, outer):
    """(left index, right index or -1) of every output row, in output order: left rows in key order (stable, nulls
    first), each repeated over its right matches in the right's stable order (a null key matches nothing); with outer
    an unmatched left row once, with -1"""
    lo, ro = sort_order(left), sort_order(right)
    rv = ro[~is_null(right)[ro]]
    rk = field(right, KEY)[rv]
    lk = field(left, KEY)[lo]
    a, b = np.searchsorted(rk, lk, "left"), np.searchsorted(rk, lk, "right")
    cnt = np.where(is_null(left)[lo], 0, b - a)
    emit = np.maximum(cnt, 1) if outer else cnt
    li = np.repeat(lo, emit)
    within = np.arange(li.size) - np.repeat(np.cumsum(emit) - emit, emit)
    ri = np.where(np.repeat(cnt, emit) > 0, rv[np.minimum(np.repeat(a, emit) + within, max(rv.size - 1, 0))], -1)
    return li, ri


def joined_rows(left, right, li, ri):
    out = np.zeros((li.size, J_REC), np.uint8)
    out[:, :4] = np.frombuffer(J_ROW.to_bytes(4, "big"), np.uint8)
    w = out[:, 4:].view("<i8")
    lw, rw = left[li, 4:].view("<i8"), right[np.maximum(ri, 0), 4:].view("<i8")
    none = ri < 0
    w[:, 0] = (lw[:, 0] & 3) | np.where(none, 7, rw[:, 0] & 7) << 2
    w[:, 1:3] = lw[:, 1:3]
    w[:, 3:6] = np.where(none[:, None], 0, rw[:, 1:4])
    return out


# ---------------------------------------------------------------------------------------------------------------
# the partitioners
# ---------------------------------------------------------------------------------------------------------------
def hash_ids(rec, R):
    """Spark's pmod(Murmur3Hash(key, 42), R) of each record; a null key leaves the seed"""
    h = np.full(rec.shape[0], hm.SEED, np.uint32)
    live = ~is_null(rec)
    h[live] = hm._v_hash_long(field(rec, KEY)[live], h[live])
    return (h.view(np.int32).astype(np.int64) % R).astype(np.uint32)


def row_hashes(rec):
    """UnsafeRow.hashCode (hashUnsafeWords of the whole row, seed 42) of every record, as Java's signed int"""
    words = rec[:, 4:].view("<u4")
    h = np.full(rec.shape[0], hm.SEED, np.uint32)
    for k in range(words.shape[1]):
        h = hm._v_mix_h1(h, hm._v_mix_k1(words[:, k].copy()))
    return hm._v_fmix(h, np.uint32(words.shape[1] * 4)).view(np.int32)


def round_robin_order(rec):
    """the sort before repartition(n): signed row hash, then (all rows one length) the row bytes unsigned"""
    h = row_hashes(rec)
    order = np.argsort(h, kind="stable")
    hs = h[order]
    tie = np.flatnonzero(np.concatenate([[False], hs[1:] == hs[:-1]]) | np.concatenate([hs[:-1] == hs[1:], [False]]))
    if tie.size:
        grp = order[tie]
        be = rec[grp, 4:].view(">u8")  # big-endian words: their order is the bytes' unsigned order
        sub = np.lexsort(tuple(be[:, k] for k in range(be.shape[1] - 1, -1, -1)) + (hs[tie],))
        order[tie] = grp[sub]
    return order


def partition_perm(ids, R):
    """the records of each partition in order, partition after partition -> (permutation, per-partition counts)"""
    return np.argsort(ids, kind="stable"), np.bincount(ids, minlength=R)


# ---------------------------------------------------------------------------------------------------------------
# device buffers, LZ4Block blocks and the slice-by-slice comparison
# ---------------------------------------------------------------------------------------------------------------
class Dev:
    """device buffers freed together"""

    def __init__(self, capi):
        self.capi, self.ptrs = capi, []

    def alloc(self, n):
        p = self.capi.dev_alloc(max(int(n), 1))  # B2SError(E_NOMEM) when the card cannot give it: the case fails
        self.ptrs.append(p)
        return p

    def put(self, d, a):
        a = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
        for o in range(0, a.size, PIECE):
            k = min(PIECE, a.size - o)
            self.capi.dev_memcpy(d + o, a[o:o + k].ctypes.data, k, 1)

    def get(self, d, n):
        out = np.empty(n, np.uint8)
        if n:
            self.capi.dev_memcpy(out.ctypes.data, d, n, 2)
        return out

    def free(self):
        for p in self.ptrs:
            self.capi.dev_free(p)
        self.ptrs = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.free()


def first_diff(got, want, rec_bytes, row0):
    """None when equal, else the first differing record and byte, with its absolute output offset"""
    got, want = got.reshape(-1), want.reshape(-1)
    if got.size == want.size and np.array_equal(got, want):
        return None
    if got.size != want.size:
        return "sizes %d != %d" % (got.size, want.size)
    i = int(np.flatnonzero(got != want)[0])
    at = row0 * rec_bytes + i
    return "record %d byte %d (output offset %d = 2^31 %+d = 2^32 %+d): got %d, want %d" % (
        row0 + i // rec_bytes, i % rec_bytes, at, at - 2**31, at - 2**32, got[i], want[i])


def compare_records(dev, d, n, rec_bytes, want):
    """the n records of rec_bytes at device d against want(a, b) -> the (b - a, rec_bytes) expected records"""
    step = max(1, PIECE // rec_bytes)
    for a in range(0, n, step):
        b = min(n, a + step)
        bad = first_diff(dev.get(d + a * rec_bytes, (b - a) * rec_bytes), want(a, b), rec_bytes, a)
        assert bad is None, bad


def compare_segments(dev, d, segments):
    """the device bytes at d against the concatenation of segments (uint8 arrays of any size)"""
    at = 0
    for s in segments:
        for o in range(0, s.size, PIECE):
            k = min(PIECE, s.size - o)
            bad = first_diff(dev.get(d + at + o, k), s[o:o + k], 1, at + o)
            assert bad is None, bad
        at += s.size


@functools.lru_cache(maxsize=None)
def liblz4():
    L = C.CDLL("liblz4.so.1")
    L.LZ4_compress_default.restype = C.c_int
    L.LZ4_compress_default.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    return L


def lz4_block(oracle, data, block_size=65536):
    """one LZ4Block stream of data (a uint8 array), codec blocks compressed by liblz4 as
    test_gpu_lz4_warp_decode.liblz4_stream makes them.  That helper grows its stream by bytes concatenation, which is
    quadratic: over a block of hundreds of MB it would run for hours, so the frames are joined once here."""
    from test_gpu_lz4_warp_decode import END_MARK, frame
    L = liblz4()
    parts = []
    out = C.create_string_buffer(block_size + block_size // 255 + 64)
    for i in range(0, data.size, block_size):
        piece = np.ascontiguousarray(data[i:i + block_size])
        k = L.LZ4_compress_default(piece.ctypes.data, out, piece.size, len(out))
        assert k > 0
        parts.append(frame(oracle, out.raw[:k], piece.size, piece.tobytes()))
    return b"".join(parts) + END_MARK


def upload_lz4(oracle, dev, flat, cuts):
    """flat cut into blocks at the byte offsets cuts, each compressed as one LZ4Block stream and copied to the device
    -> (device arena, offsets, lengths)"""
    with ThreadPoolExecutor(8) as ex:  # liblz4 and the oracle's xxh32 release the GIL
        blocks = list(ex.map(lambda k: lz4_block(oracle, flat[cuts[k]:cuts[k + 1]]), range(len(cuts) - 1)))
    ln = np.array([len(b) for b in blocks], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    d = dev.alloc(int(ln.sum()))
    for o, b in zip(off, blocks):
        dev.put(d + int(o), np.frombuffer(b, np.uint8))
    return d, off, ln


def record_cuts(n, rec_bytes, k):
    return (np.linspace(0, n, k + 1).astype(np.int64) * rec_bytes)


# ---------------------------------------------------------------------------------------------------------------
# after every case: a small known call must still be exact, and device memory must be back where the module started
# but for the library's grow-only workspaces.  The reduce calls keep buffers of up to 1 GiB each and free larger ones
# when they return (the 1 GiB buffer trim).  The header says nothing about the row partitioners' write-side workspaces;
# after the 4.6 GB calls here between 0 and 8.6 GiB of device memory have been measured kept, so their cases allow
# WRITE_KEEPS and run last.
# ---------------------------------------------------------------------------------------------------------------
READ_KEEPS = 6 * GiB
WRITE_KEEPS = 10 * GiB


def small_sort_is_exact(capi):
    rec = make_rows(5000, 99, giant=0.1, nulls=0.1, domain=100)
    flat = rec.reshape(-1)
    dst = np.zeros(flat.size, np.uint8)
    cuts = record_cuts(5000, REC, 3)
    r = capi.decompress_sort_rows_packed(0, flat, cuts[:-1], np.diff(cuts), dst, KEY_INT64, KEY, 8, 0)
    assert (r["status"] == 0).all() and r["n_records"] == 5000
    assert np.array_equal(dst.reshape(-1, REC), rec[sort_order(rec)])


def after_case(capi, free_at_start, keeps=READ_KEEPS):
    small_sort_is_exact(capi)
    import torch
    kept = free_at_start - torch.cuda.mem_get_info(0)[0]
    assert kept < keeps, "%.2f GiB of device memory kept (at most %.0f GiB)" % (kept / GiB, keeps / GiB)


# ---------------------------------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def free_at_start(capi):
    torch = pytest.importorskip("torch")
    return torch.cuda.mem_get_info(0)[0]


@pytest.fixture(scope="module")
def arena(free_at_start):
    rec = make_rows(N, 2026)
    order = sort_order(rec)
    starts, lens = group_starts(rec, order)
    assert rec.nbytes > 2**32 and N > 2**26
    assert lens.max() * REC > 2**31  # one group / window partition past 2^31 bytes
    return rec, order


# ---------------------------------------------------------------------------------------------------------------
# 1. row sort past 4 GiB
# ---------------------------------------------------------------------------------------------------------------
def test_row_sort_packed_codec_none_past_4_gib(capi, free_at_start, arena):
    """the host-side chunk pipeline and the framing over 4.6 GB in 40 blocks"""
    rec, order = arena
    flat = rec.reshape(-1)
    cuts = record_cuts(N, REC, N_BLOCKS)
    dst = np.empty(flat.size, np.uint8)
    r = capi.decompress_sort_rows_packed(0, flat, cuts[:-1], np.diff(cuts), dst, KEY_INT64, KEY, 8, 0)
    assert (r["status"] == 0).all() and r["n_records"] == N and r["total"] == flat.size
    out = dst.reshape(N, REC)
    step = PIECE // REC
    for a in range(0, N, step):
        bad = first_diff(out[a:a + step], rec[order[a:a + step]], REC, a)
        assert bad is None, bad
    del dst, out
    after_case(capi, free_at_start)


def test_row_sort_dev_lz4_past_4_gib(capi, free_at_start, oracle, arena):
    """liblz4's LZ4Block blocks: the decoder's destination offsets cross 2^32 too"""
    rec, order = arena
    with Dev(capi) as dev:
        d_src, off, ln = upload_lz4(oracle, dev, rec.reshape(-1), record_cuts(N, REC, N_BLOCKS))
        d_dst = dev.alloc(rec.nbytes)
        r = capi.decompress_sort_rows_dev(1, d_src, off, ln, d_dst, rec.nbytes, KEY_INT64, KEY, 8, 0)
        assert (r["status"] == 0).all() and r["n_records"] == N and r["total"] == rec.nbytes
        compare_records(dev, d_dst, N, REC, lambda a, b: rec[order[a:b]])
    after_case(capi, free_at_start)


# ---------------------------------------------------------------------------------------------------------------
# 2. composite-key sort past 4 GiB: int32 DESC and a string with a long shared prefix
# ---------------------------------------------------------------------------------------------------------------
def test_composite_key_sort_past_4_gib(capi, free_at_start):
    rec = make_keyed_rows(N, 2027)
    order = keyed_order(rec)
    assert rec.nbytes > 2**32 and N > 2**26
    with Dev(capi) as dev:
        d_src = dev.alloc(rec.nbytes)
        dev.put(d_src, rec)
        d_dst = dev.alloc(rec.nbytes)
        cuts = record_cuts(N, REC, N_BLOCKS)
        r = capi.decompress_sort_rows_keys_dev(0, d_src, cuts[:-1], np.diff(cuts), d_dst, rec.nbytes, COMPOSITE_KEYS)
        assert (r["status"] == 0).all() and r["n_records"] == N and r["total"] == rec.nbytes
        compare_records(dev, d_dst, N, REC, lambda a, b: rec[order[a:b]])
    del rec, order
    after_case(capi, free_at_start)


# ---------------------------------------------------------------------------------------------------------------
# 3. aggregate past 4 GiB, one group past 2^31 bytes
# ---------------------------------------------------------------------------------------------------------------
def test_aggregate_past_4_gib(capi, free_at_start, arena):
    rec, order = arena
    want = aggregate_ref(rec, order)
    G = want.shape[0]
    assert G > 900_000 and field(want, ONE).max() * REC > 2**31
    with Dev(capi) as dev:
        d_src = dev.alloc(rec.nbytes)
        dev.put(d_src, rec)
        d_dst = dev.alloc(G * REC)
        cuts = record_cuts(N, REC, N_BLOCKS)
        r = capi.decompress_aggregate_rows_dev(0, d_src, cuts[:-1], np.diff(cuts), d_dst, G * REC, KEY_INT64, KEY, 8,
                                               0, AGGS)
        assert (r["status"] == 0).all() and r["n_records"] == N and r["n_groups"] == G and r["total"] == G * REC
        compare_records(dev, d_dst, G, REC, lambda a, b: want[a:b])
    after_case(capi, free_at_start)


# ---------------------------------------------------------------------------------------------------------------
# 5. window past 4 GiB of input and 6 GiB of output, one partition past 2^31 bytes
# ---------------------------------------------------------------------------------------------------------------
def test_window_past_4_gib(capi, free_at_start, arena):
    rec, order = arena
    ref = WindowRef(rec, order)
    out_bytes = N * W_REC
    assert out_bytes > 2**32 and ref.parts[1].max() * W_REC > 2**31
    with Dev(capi) as dev:
        d_src = dev.alloc(rec.nbytes)
        dev.put(d_src, rec)
        d_dst = dev.alloc(out_bytes)
        cuts = record_cuts(N, REC, N_BLOCKS)
        r = capi.decompress_window_offset_rows_keys_dev(0, d_src, cuts[:-1], np.diff(cuts), d_dst, out_bytes, W_KEYS,
                                                        1, NF, [0] * NF, W_FNS)
        assert (r["status"] == 0).all() and r["n_records"] == N and r["n_out_records"] == N
        assert r["total"] == out_bytes
        compare_records(dev, d_dst, N, W_REC, ref.rows)
    after_case(capi, free_at_start)


# ---------------------------------------------------------------------------------------------------------------
# 4. join past 4 GiB of output
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("join_type", [0, 1], ids=["inner", "left_outer"])
def test_join_past_4_gib_of_output(capi, free_at_start, oracle, join_type):
    left, right = make_join(31)
    li, ri = join_index(left, right, outer=join_type == 1)
    n_out = li.size
    assert n_out > 2**26 and n_out * J_REC > 2**32
    with Dev(capi) as dev:
        flat = np.concatenate([left.reshape(-1), right.reshape(-1)])
        cuts = np.concatenate([record_cuts(left.shape[0], left.shape[1], 3),
                               left.nbytes + record_cuts(right.shape[0], right.shape[1], 4)[1:]])
        d_src, off, ln = upload_lz4(oracle, dev, flat, cuts)
        del flat
        cap = n_out * J_REC
        d_dst = dev.alloc(cap)
        r = capi.decompress_join_rows_keys_dev(join_type, 1, d_src, off, ln, 3, d_dst, cap, JOIN_KEYS, JOIN_KEYS, 2, 3,
                                               [0, 0], [0, 0, 0])
        assert (r["status"] == 0).all() and r["total"] == cap and r["n_out_records"] == n_out
        assert r["n_left_records"] == left.shape[0] and r["n_right_records"] == right.shape[0]
        compare_records(dev, d_dst, n_out, J_REC, lambda a, b: joined_rows(left, right, li[a:b], ri[a:b]))
    after_case(capi, free_at_start)


# ---------------------------------------------------------------------------------------------------------------
# 7. rows at Spark's 2^31 - 1 byte limit
# ---------------------------------------------------------------------------------------------------------------
def pattern(n, seed):
    """n compressible bytes (a 251-byte period)"""
    return np.resize(np.random.default_rng(seed).integers(0, 256, 251, dtype=np.uint8), n)


def small_records(n, fixed_words, key, seed):
    """n records of a null word and fixed_words 8-byte fields, the first the key, the second the index"""
    rng = np.random.default_rng(seed)
    row = 8 + 8 * fixed_words
    rec = np.zeros((n, 4 + row), np.uint8)
    rec[:, :4] = np.frombuffer(row.to_bytes(4, "big"), np.uint8)
    w = rec[:, 4:].view("<i8")
    w[:, 1] = key
    if fixed_words > 1:
        w[:, 2] = np.arange(n)
    if fixed_words > 2:
        w[:, 3:] = rng.integers(INT64_MIN, 2**63 - 1, (n, fixed_words - 2))
    return rec


def giant_record(key, fixed, var, extra=()):
    """(header: size prefix, null word, key, *extra, the var slot; var bytes) of one row with var bytes after `fixed`
    bytes of null word and slots"""
    row = fixed + var.size
    words = [0, key, *extra, (fixed << 32) | var.size]
    assert 8 * len(words) == fixed and row <= LIMIT
    head = np.frombuffer(row.to_bytes(4, "big") + b"".join((w % 2**64).to_bytes(8, "little") for w in words),
                         np.uint8)
    return head, var


def run_giant(capi, oracle, dev, blocks, call):
    """blocks: lists of uint8 segments, each list one LZ4Block block -> (device arena, offsets, lengths)"""
    streams = [lz4_block(oracle, np.concatenate(segs)) for segs in blocks]
    ln = np.array([len(s) for s in streams], np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    d = dev.alloc(int(ln.sum()))
    for o, s in zip(off, streams):
        dev.put(d + int(o), np.frombuffer(s, np.uint8))
    return call(d, off, ln)


def test_row_sort_of_a_row_at_the_limit(capi, free_at_start, oracle):
    var = pattern(LIMIT - 24, 1)
    head, _ = giant_record(0, 24, var)
    assert int.from_bytes(head[:4].tobytes(), "big") == 0x7FFFFFFF
    a = small_records(3000, 2, np.arange(3000) % 7 - 3, 2)  # keys -3..3; the giant's key 0 sorts among them
    b = small_records(2000, 2, np.arange(2000) % 5 - 2, 3)
    total = a.nbytes + b.nbytes + head.size + var.size
    with Dev(capi) as dev:
        d_dst = dev.alloc(total)
        r = run_giant(capi, oracle, dev, [[a[:1000].reshape(-1)], [a[1000:].reshape(-1), head, var, b[:10].reshape(-1)],
                                          [b[10:].reshape(-1)]],
                      lambda d, off, ln: capi.decompress_sort_rows_dev(1, d, off, ln, d_dst, total, KEY_INT64, KEY, 8,
                                                                       0))
        assert (r["status"] == 0).all() and r["n_records"] == 5001 and r["total"] == total
        # stable order: a's rows, the giant (after a[1000:], before b) and b's rows, by key
        ka, kb = field(a, KEY), field(b, KEY)
        segs = []
        for k in range(-3, 4):
            segs.append(a[ka == k].reshape(-1))
            if k == 0:
                segs += [head, var]
            segs.append(b[kb == k].reshape(-1))
        compare_segments(dev, d_dst, segs)
    after_case(capi, free_at_start)


def join_giant_sides(var_bytes, match):
    """left: small unmatched rows and one giant row (key 5, string field of var_bytes); right: small unmatched rows and,
    when match, one row of key 5"""
    lsmall = small_records(1000, 2, 2 * np.arange(1000) + 100, 4)  # keys even
    lsmall[:, 4 + 16:] = 0  # the string field: empty
    rsmall = small_records(1500, 2, 2 * np.arange(1500) + 101, 5)  # keys odd
    var = pattern(var_bytes, 6)
    lhead, _ = giant_record(5, 24, var)
    rrow = small_records(1, 2, 5, 7) if match else small_records(0, 2, 5, 7)
    return lsmall, lhead, var, rsmall, rrow


def join_giant(capi, oracle, dev, join_type, var_bytes, match, cap):
    lsmall, lhead, var, rsmall, rrow = join_giant_sides(var_bytes, match)
    d_dst = dev.alloc(cap)
    r = run_giant(capi, oracle, dev, [[lsmall[:500].reshape(-1), lhead, var, lsmall[500:].reshape(-1)],
                                      [rsmall.reshape(-1), rrow.reshape(-1)]],
                  lambda d, off, ln: capi.decompress_join_rows_keys_dev(join_type, 1, d, off, ln, 1, d_dst, cap,
                                                                        JOIN_KEYS, JOIN_KEYS, 2, 2, [0, 1], [0, 0]))
    return r, d_dst, var, rrow


def test_join_row_at_the_limit_and_one_past(capi, free_at_start, oracle):
    fixed_out = 8 + 8 * 4
    var_bytes = LIMIT - fixed_out  # the joined row is exactly 2^31 - 1 bytes
    with Dev(capi) as dev:
        r, d_dst, var, rrow = join_giant(capi, oracle, dev, 0, var_bytes, True, LIMIT + 4)
        assert (r["status"] == 0).all() and r["n_out_records"] == 1 and r["total"] == LIMIT + 4
        rw = rrow[0, 4:].view("<i8")
        words = [0, 5, (fixed_out << 32) | var_bytes, int(rw[1]), int(rw[2])]
        head = np.frombuffer(LIMIT.to_bytes(4, "big") + b"".join((w % 2**64).to_bytes(8, "little") for w in words),
                             np.uint8)
        compare_segments(dev, d_dst, [head, var])
    after_case(capi, free_at_start)
    with Dev(capi) as dev:
        with pytest.raises(capi.B2SError) as e:
            join_giant(capi, oracle, dev, 0, var_bytes + 1, True, LIMIT + 8)
        assert e.value.code == capi.E_UNSUPPORTED
    after_case(capi, free_at_start)


def test_left_outer_null_side_row_past_the_limit(capi, free_at_start, oracle):
    """an unmatched left row whose row with the right side null is one byte past the limit: refused by the left outer
    join; the inner join of the same blocks emits nothing and succeeds"""
    var_bytes = LIMIT - 40 + 1
    with Dev(capi) as dev:
        with pytest.raises(capi.B2SError) as e:
            join_giant(capi, oracle, dev, 1, var_bytes, False, 1 << 31)
        assert e.value.code == capi.E_UNSUPPORTED
    with Dev(capi) as dev:
        r, _, _, _ = join_giant(capi, oracle, dev, 0, var_bytes, False, 4096)
        assert (r["status"] == 0).all() and r["n_out_records"] == 0 and r["total"] == 0
    after_case(capi, free_at_start)


def window_giant(capi, oracle, dev, out_row):
    """small rows (null word, key, index, string slot 0) and one giant of the same key in the middle; row_number over
    PARTITION BY key ORDER BY index: every output row is its input row plus 8 bytes"""
    fixed = 32
    var = pattern(out_row - 8 - fixed, 8)
    small = small_records(2000, 3, np.arange(2000) % 3, 9)  # the third field (the string slot) is random: zero it
    small[:, 4 + 24:4 + 32] = 0
    head, _ = giant_record(1, fixed, var, extra=(1000,))
    cap = small.size + 2000 * 8 + out_row + 4 + 64
    d_dst = dev.alloc(cap)
    keys = [(KEY_INT64, KEY, 8, 0), (KEY_INT64, 16, 8, -1)]
    r = run_giant(capi, oracle, dev, [[small[:1000].reshape(-1), head, var], [small[1000:].reshape(-1)]],
                  lambda d, off, ln: capi.decompress_window_rows_keys_dev(1, d, off, ln, d_dst, cap, keys, 1, 3,
                                                                          [0, 0, 1], [0]))
    return r, d_dst, small, var


def test_window_row_at_the_limit_and_one_past(capi, free_at_start, oracle):
    with Dev(capi) as dev:
        r, d_dst, small, var = window_giant(capi, oracle, dev, LIMIT)
        assert (r["status"] == 0).all() and r["n_out_records"] == 2001
        # output rows: [size][null word][key][index][string slot + 8 << 32][row_number] then the var bytes
        segs = []
        for k in range(3):
            idx = np.flatnonzero(field(small, KEY) == k)
            rows = [(int(field(small, 16)[i]), i) for i in idx]  # (index, row) by the ORDER BY column
            if k == 1:
                rows.append((1000, -1))  # ties small row 1000, which follows it in the blocks
            rows.sort()
            for rn, (_, i) in enumerate(rows, 1):
                if i < 0:
                    words = [0, 1, 1000, (40 << 32) | var.size, rn]
                    segs += [np.frombuffer(LIMIT.to_bytes(4, "big") + b"".join(w.to_bytes(8, "little") for w in words),
                                           np.uint8), var]
                else:
                    w = small[i, 4:].view("<i8")
                    words = [0, int(w[1]), int(w[2]), 0, rn]
                    segs.append(np.frombuffer((40).to_bytes(4, "big") + b"".join(
                        (x % 2**64).to_bytes(8, "little") for x in words), np.uint8))
        compare_segments(dev, d_dst, segs)
    after_case(capi, free_at_start)
    with Dev(capi) as dev:
        with pytest.raises(capi.B2SError) as e:
            window_giant(capi, oracle, dev, LIMIT + 1)
        assert e.value.code == capi.E_UNSUPPORTED
    after_case(capi, free_at_start)


# ---------------------------------------------------------------------------------------------------------------
# 6. row partitioners past 4 GiB, 200 partitions, codec NONE
# ---------------------------------------------------------------------------------------------------------------
R_PARTS = 200


def check_partitions(dev, d_dst, r, rec, perm, counts):
    assert list(r["status"]) == [0] * R_PARTS
    ln = np.asarray(r["dst_len"], np.int64)
    off = np.asarray(r["dst_off"], np.int64)
    assert np.array_equal(ln, counts * REC)
    assert np.array_equal(off, np.concatenate([[0], np.cumsum(ln)[:-1]]))
    compare_records(dev, d_dst, rec.shape[0], REC, lambda a, b: rec[perm[a:b]])


@pytest.mark.parametrize("kind", ["hash", "round_robin"])
def test_row_partitioner_past_4_gib(capi, free_at_start, arena, kind):
    rec, _ = arena
    start = 57
    if kind == "hash":
        perm, counts = partition_perm(hash_ids(rec, R_PARTS), R_PARTS)
    else:
        order = round_robin_order(rec)
        ids = ((start + 1 + np.arange(N)) % R_PARTS).astype(np.uint32)
        perm, counts = partition_perm(ids, R_PARTS)
        perm = order[perm]
        del order, ids
    assert rec.nbytes > 2**32 and N > 2**26
    if kind == "hash":  # the giant key's partition
        assert counts.max() * REC > 2**31
    with Dev(capi) as dev:
        d_rec = dev.alloc(rec.nbytes)
        dev.put(d_rec, rec)
        d_len = dev.alloc(4 * N)
        dev.put(d_len, np.full(N, REC, np.uint32))
        cap = capi.partition_compress_bound(0, 0, R_PARTS, rec.nbytes)
        d_dst = dev.alloc(cap)
        if kind == "hash":
            r = capi.partition_compress_rows_hash_dev(0, d_rec, rec.nbytes, d_len, N, [(KEY_INT64, KEY, 8, 0)],
                                                      R_PARTS, d_dst, cap)
        else:
            r = capi.partition_compress_rows_round_robin_dev(0, d_rec, rec.nbytes, d_len, N, R_PARTS, start, 1, d_dst,
                                                             cap)
        assert r["total"] == rec.nbytes
        check_partitions(dev, d_dst, r, rec, perm, counts)
    after_case(capi, free_at_start, WRITE_KEEPS)
