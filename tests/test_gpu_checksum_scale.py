"""The checksum kernels (csrc/checksum.cu, K1) at the scales the rest of the suite never reaches, against the CPU.

A checksum call cuts every slice into work items of 2^s bytes.  api.cu's pick_tile_shift chooses s from the call's total
bytes: s = 14 below ITEMS << 15, then s is the largest value up to 20 with total >= ITEMS << s, where ITEMS = 132 SMs x
32 x 4 = 16896 work items.  So items of 32 KiB to 1 MiB only occur in calls of 0.52 GiB to 16.5 GiB and more.  The CRC
kernels also shift each item to its place in the slice, and the finalize shifts the init term over the whole slice, by
x^(8e) mod P built from one table entry per bit of the byte count e; counts of 2^29 bytes and more use entries past
x^(2^32).

Every expected value here comes from the CPU (zlib.adler32, zlib.crc32 and the oracle's CRC32C, each in its continuation
form) over bytes copied back from the device in pieces of at most 256 MiB.  The module allocates one ~16.6 GiB device
buffer, filled with non-zero bytes so that a byte masked in or out by mistake next to a slice always changes its CRC.
"""
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MiB, GiB = 1 << 20, 1 << 30
PIECE = 256 * MiB  # host-side piece: the most this file holds of the device buffer at a time
ITEMS = 132 * 32 * 4  # pick_tile_shift's work-item target (kSMs x 32 x 4)
SHIFTS = range(14, 21)


def threshold(s):
    """total bytes from which a checksum call uses work items of 2^s bytes (for s = 15..20)"""
    return ITEMS << s


# the filler slice of (a) for work-item size 2^s: a prefix of the buffer that puts its batch's total just past
# threshold(s); the odd term leaves its end unaligned.  FILLER[20] > 2^34.
FILLER = {s: threshold(s) + 12345 + 2 * s for s in SHIFTS}
EDGE0 = (FILLER[20] + 8191) // 4096 * 4096  # the edge slices of (a) live in [EDGE0, EDGE0 + EDGE_BYTES)
EDGE_BYTES = 48 * MiB
BUF_BYTES = EDGE0 + EDGE_BYTES  # ~16.56 GiB

# (b): byte counts across bits 29..32 of the power tables, at phase 0 (offset 0) and at an odd phase
BIG_LENGTHS = [(1 << 29) - 1, 1 << 29, (1 << 29) + 1, (1 << 30) + (1 << 29) + 13, (1 << 32) - 1, (1 << 32) + 17]
ODD = 1 * GiB + 9  # off & 15 = 9
SCRATCH = 8 * GiB  # (c) and the 0xFF slice overwrite [SCRATCH, ...) or [0, ...) and restore them afterwards

ALGS = {"ADLER32": 1, "CRC32": 2, "CRC32C": 3}


def _crc32c(state, a):
    from oracle import oracle
    return oracle.lib().orc_crc32c(state, a.ctypes.data if a.size else None, a.size)


UPDATE = {1: lambda st, a: zlib.adler32(a, st), 2: lambda st, a: zlib.crc32(a, st), 3: _crc32c}
INIT = {1: 1, 2: 0, 3: 0}


def cpu(alg, a):
    return UPDATE[alg](INIT[alg], np.ascontiguousarray(a, dtype=np.uint8))


class DeviceBuffer:
    """BUF_BYTES of device memory with deterministic non-zero content: piece k of PIECE bytes is BASE + (k mod 67)
    (BASE in 1..188, so no byte is ever 0)."""

    def __init__(self, capi):
        self.capi = capi
        self.d = capi.dev_alloc(BUF_BYTES)
        self.base = np.random.default_rng(2029).integers(1, 189, PIECE, dtype=np.uint8)

    def fill(self, lo, hi):
        tmp = np.empty(PIECE, np.uint8)
        k = lo // PIECE
        while k * PIECE < hi:
            a, b = max(lo, k * PIECE), min(hi, (k + 1) * PIECE, BUF_BYTES)
            np.add(self.base, k % 67, out=tmp)
            self.write(a, tmp[a - k * PIECE:b - k * PIECE])
            k += 1

    def write(self, off, a):
        a = np.ascontiguousarray(a)
        self.capi.dev_memcpy(self.d + off, a.ctypes.data, a.size, 1)

    def read(self, off, n):
        out = np.empty(n, np.uint8)
        if n:
            self.capi.dev_memcpy(out.ctypes.data, self.d + off, n, 2)
        return out

    def pieces(self, off, n):
        end = off + n
        while off < end:
            k = min(PIECE, end - off)
            yield self.read(off, k)
            off += k

    def states(self, lo, ends, algs=(1, 2, 3)):
        """{end: {alg: CPU checksum of [lo, end)}} for every end, in one streaming pass from lo"""
        st = {g: INIT[g] for g in algs}
        out, pos = {}, lo
        with ThreadPoolExecutor(len(algs)) as ex:  # zlib and ctypes release the GIL on large buffers
            for end in sorted(set(ends)):
                for a in self.pieces(pos, end - pos):
                    st = dict(zip(algs, ex.map(lambda g: UPDATE[g](st[g], a), algs)))
                pos = end
                out[end] = dict(st)
        return out

    def checksum(self, alg, lo, n):
        return self.states(lo, [lo + n], (alg,))[lo + n][alg]

    def free(self):
        self.capi.dev_free(self.d)


@pytest.fixture(scope="module")
def buf(capi):
    b = DeviceBuffer(capi)  # raises B2SError(E_NOMEM) when the card cannot give ~16.6 GiB: the test fails, never skips
    try:
        b.fill(0, BUF_BYTES)
        yield b
    finally:
        b.free()


@pytest.fixture(scope="module")
def ref(buf):
    """CPU checksums of every filler prefix and of the (b) slices at phase 0 (one pass from 0), and of the (b) slices
    at the odd phase (one pass from ODD)"""
    r = buf.states(0, list(FILLER.values()) + BIG_LENGTHS)
    odd = buf.states(ODD, [ODD + n for n in BIG_LENGTHS])
    r.update({(ODD, n): odd[ODD + n] for n in BIG_LENGTHS})
    return r


def mismatches(got, want, labels):
    return [(lab, hex(int(g)), hex(int(w))) for g, w, lab in zip(got, want, labels) if int(g) != int(w)]


# ---------------------------------------------------------------------------------------------------------------
# (a) every work-item size
# ---------------------------------------------------------------------------------------------------------------
def edge_slices(s):
    """(off, len, label) slices in the edge region, for work items of T = 2^s bytes: every start phase with padded
    lengths ((off & 15) + len) T, T +- 1 and 3T; last rows of 1..511 bytes; one slice inside a single row and one inside
    a single 16-byte word (masked at both ends); 1-byte slices; zero-length slices between the others"""
    T = 1 << s
    want = []
    for ph in (0, 1, 7, 15):
        for pad in (T, T - 1, T + 1, 3 * T):
            want.append((ph, pad - ph, "phase %d padded %d" % (ph, pad)))
    for ph in (0, 7):
        for last in (1, 15, 16, 17, 496, 511):
            pad = T + 5 * 512 + last
            want.append((ph, pad - ph, "phase %d, last row of %d bytes" % (ph, last)))
    want += [(5, 300, "one row, masked at both ends"), (3, 9, "one word, masked at both ends"),
             (15, 1, "1 byte at phase 15"), (0, 1, "1 byte at phase 0")]
    out, cur = [], EDGE0 + 4096
    for i, (ph, n, lab) in enumerate(want):
        off = (cur + 4095) // 4096 * 4096 + ph
        if i % 3 == 0:
            out.append((off, 0, "empty"))
        out.append((off, n, lab))
        cur = off + n + 4096 + 37
    assert cur < EDGE0 + EDGE_BYTES
    return out


@pytest.mark.parametrize("s", SHIFTS)
def test_every_work_item_size(capi, buf, ref, s):
    edges = edge_slices(s)
    edge_host = buf.read(EDGE0, EDGE_BYTES)
    half = len(edges) // 2
    sl = edges[:half] + [(0, FILLER[s], "filler of %d bytes" % FILLER[s])] + edges[half:]
    total = sum(n for _, n, _ in sl)
    # the batch must be cut into items of exactly 2^s bytes
    assert total >= threshold(s) or s == 14
    assert s == 20 or total < threshold(s + 1)
    off = [o for o, _, _ in sl]
    ln = [n for _, n, _ in sl]
    bad = {}
    for name, alg in ALGS.items():
        want = [ref[n][alg] if o == 0 and n == FILLER[s] else cpu(alg, edge_host[o - EDGE0:o - EDGE0 + n])
                for o, n, _ in sl]
        got = capi.checksum_dev(alg, buf.d, off, ln)
        m = mismatches(got, want, [lab for _, _, lab in sl])
        if m:
            bad[name] = m
    assert not bad, ("2^%d-byte work items" % s, bad)


# ---------------------------------------------------------------------------------------------------------------
# (b) byte counts across the power-table bits
# ---------------------------------------------------------------------------------------------------------------
def test_byte_counts_across_power_table_bits(capi, buf, ref):
    """each slice alone (its own size picks the work item) and all of them in one batch"""
    sl = [(0, n) for n in BIG_LENGTHS] + [(ODD, n) for n in BIG_LENGTHS] + [(0, FILLER[20])]
    bad = {}
    for name, alg in ALGS.items():
        want = [ref[n][alg] if o == 0 else ref[(o, n)][alg] for o, n in sl]
        labels = ["%d bytes at offset %d" % (n, o) for o, n in sl]
        alone = [int(capi.checksum_dev(alg, buf.d, [o], [n])[0]) for o, n in sl]
        batch = capi.checksum_dev(alg, buf.d, [o for o, _ in sl], [n for _, n in sl])
        m = mismatches(alone, want, labels) + mismatches(batch, want, ["batch: " + x for x in labels])
        if m:
            bad[name] = m
    assert not bad, bad


def test_adler32_largest_item_sums(capi, buf):
    """> 4 GiB of 0xFF bytes: every byte at its largest, so the per-item sums A and B are at their largest"""
    lo, n = 3, (1 << 32) + 4097
    ff = np.full(PIECE, 0xFF, np.uint8)
    try:
        for o in range(lo, lo + n, PIECE):
            buf.write(o, ff[:min(PIECE, lo + n - o)])
        want = buf.states(lo, [lo + n])[lo + n]
        for name, alg in ALGS.items():
            got = int(capi.checksum_dev(alg, buf.d, [lo], [n])[0])
            assert got == want[alg], (name, hex(got), hex(want[alg]))
            got = capi.checksum_dev(alg, buf.d, [lo, lo + n - 7], [n, 7])
            exp = [want[alg], cpu(alg, ff[:7])]
            assert [int(g) for g in got] == exp, (name, [hex(int(g)) for g in got], [hex(e) for e in exp])
    finally:
        buf.fill(0, lo + n + 1)


# ---------------------------------------------------------------------------------------------------------------
# (c) every call site with one slice of 512 MiB or more, CRC32C
# ---------------------------------------------------------------------------------------------------------------
CRC32C = 3


def test_host_and_dev_checksum_calls(capi, buf):
    """checksum_batch (the large stream is a chunk of its own), checksum_packed and checksum_dev"""
    n = (1 << 29) + 13
    host = np.concatenate(list(buf.pieces(0, n)))  # the one host array this file holds beyond a piece
    small = buf.read(EDGE0, 1000)
    streams = [small, host, small[:0], small[:5]]
    got = capi.checksum_batch(CRC32C, streams)
    want = [cpu(CRC32C, x) for x in streams]
    assert got == want, ([hex(g) for g in got], [hex(w) for w in want])
    sl = [(0, n), (7, 1 << 29), (17, 100), (n - 1, 1), (9, 0)]
    want = [cpu(CRC32C, host[o:o + k]) for o, k in sl]
    got = capi.checksum_packed(CRC32C, host, [o for o, _ in sl], [k for _, k in sl])
    assert [int(g) for g in got] == want
    got = capi.checksum_dev(CRC32C, buf.d, [o for o, _ in sl], [k for _, k in sl])
    assert [int(g) for g in got] == want


def test_compress_and_decompress_dev_large_stream(capi, buf):
    """write side: compress_dev of ~600 MiB of incompressible bytes into one LZ4Block stream of raw blocks (> 512 MiB)
    reports the CRC32C of that stream.  Read side: a block of two slices, the second one that stream, verifies,
    decodes to the input, and names slice 1 when its checksum is wrong."""
    src = [(4 * GiB + 3, 100003), (5 * GiB + 11, 600 * MiB + 7)]
    cap = sum(capi.compress_bound(capi.CODEC_LZ4BLOCK, 0, n) for _, n in src)
    d_comp, d_out = buf.d + SCRATCH, buf.d + SCRATCH + (cap + 4095) // 4096 * 4096
    out_bytes = sum(n for _, n in src)
    try:
        r = capi.compress_dev(capi.CODEC_LZ4BLOCK, buf.d, [o for o, _ in src], [n for _, n in src], d_comp, cap,
                              checksum_alg=CRC32C)
        assert list(r["status"]) == [0, 0]
        off, ln = [int(x) for x in r["dst_off"]], [int(x) for x in r["dst_len"]]
        assert ln[1] > 1 << 29 and off[1] == off[0] + ln[0]
        want = [buf.checksum(CRC32C, SCRATCH + o, n) for o, n in zip(off, ln)]
        assert [int(c) for c in r["checksums"]] == want, ([hex(int(c)) for c in r["checksums"]], [hex(w) for w in want])

        blk = ([off[0]], [ln[0] + ln[1]])
        d = capi.decompress_dev(capi.CODEC_LZ4BLOCK, d_comp, *blk, d_out, out_bytes, checksum_alg=CRC32C,
                                slice_base=[0, 2], slice_len=ln, slice_checksum=want)
        assert int(d["status"][0]) == 0 and int(d["dst_len"][0]) == out_bytes
        o0 = SCRATCH + (cap + 4095) // 4096 * 4096 + int(d["dst_off"][0])
        pos = 0
        for o, n in src:
            for a, b in zip(buf.pieces(o0 + pos, n), buf.pieces(o, n)):
                assert np.array_equal(a, b)
            pos += n
        d = capi.decompress_dev(capi.CODEC_LZ4BLOCK, d_comp, *blk, d_out, out_bytes, checksum_alg=CRC32C,
                                slice_base=[0, 2], slice_len=ln, slice_checksum=[want[0], want[1] ^ 1])
        assert int(d["status"][0]) == capi.E_CHECKSUM and int(d["bad_slice"][0]) == 1
    finally:
        buf.fill(SCRATCH, SCRATCH + 2 * cap + 8192)


def test_partition_compress_dev_codec_none(capi, buf):
    """codec NONE: one partition of > 512 MiB beside small and empty ones; every partition's checksum is the CPU
    CRC32C of its output, and that output is its records in order"""
    R = 6  # 1 and 4 stay empty
    big, n_big = MiB + 3, 560
    recs = []
    for i in range(n_big):
        recs.append((big, 2))
        if i % 100 == 0:
            recs += [(1000 + i, 0), (777, 3), (13, 0)]
    recs += [(1, 5), (4096, 3)]
    lens = np.array([n for n, _ in recs], np.uint32)
    parts = np.array([p for _, p in recs], np.uint32)
    rec_lo = 2 * GiB
    rec_bytes = int(lens.sum(dtype=np.uint64))
    assert int(lens[parts == 2].sum(dtype=np.uint64)) >= 1 << 29
    cap = capi.partition_compress_bound(capi.CODEC_NONE, 0, R, rec_bytes)
    d_len, d_part = capi.dev_alloc(lens.nbytes), capi.dev_alloc(parts.nbytes)
    try:
        capi.dev_memcpy(d_len, lens.ctypes.data, lens.nbytes, 1)
        capi.dev_memcpy(d_part, parts.ctypes.data, parts.nbytes, 1)
        r = capi.partition_compress_dev(capi.CODEC_NONE, buf.d + rec_lo, rec_bytes, d_len, d_part, len(recs), R,
                                        buf.d + SCRATCH, cap, checksum_alg=CRC32C)
        assert list(r["status"]) == [0] * R
        # the model: each partition's records in input order, checksummed from the source bytes
        model = {p: 0 for p in range(R)}
        size = {p: 0 for p in range(R)}
        o = rec_lo
        for n, p in recs:
            model[p] = _crc32c(model[p], buf.read(o, n))
            size[p] += n
            o += n
        assert [int(x) for x in r["dst_len"]] == [size[p] for p in range(R)]
        got = [int(c) for c in r["checksums"]]
        out = [buf.checksum(CRC32C, SCRATCH + int(r["dst_off"][p]), int(r["dst_len"][p])) for p in range(R)]
        assert got == out == [model[p] for p in range(R)], ([hex(x) for x in got], [hex(x) for x in out])
    finally:
        capi.dev_free(d_len)
        capi.dev_free(d_part)
        buf.fill(SCRATCH, SCRATCH + cap)
