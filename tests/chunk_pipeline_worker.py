"""One process, one pipeline configuration: runs the host-pointer codec calls (checksum, compress, decompress) over a
seeded mixed workload and checks every output byte for byte against the CPU reference of its kernel.

The chunk size, the slot count, the read pipeline's lag and the codec-block group sizes are read once, by b2s_init, from
B2S_HOST_CHUNK_MB / B2S_SLOTS / B2S_READ_LAG / B2S_LZ4_CHUNK_BLOCKS / B2S_LZ4D_CHUNK_BLOCKS, so
tests/test_gpu_chunk_pipelines.py starts this worker once per configuration with the environment set.  It prints one
JSON line: each check's name with "ok" or its failure, and what the calls reached (chunks, slot reuses, block groups),
computed on the host from the same chunking rule as chunk_schedule.h's chunk_starts.

    python tests/chunk_pipeline_worker.py <config name> <libzc.so: the Zstd encoder's CPU model>
"""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import spark_s3_shuffle_b200 as pkg  # noqa: E402
import zstd_ref  # noqa: E402
from conftest import KINDS, corpus  # noqa: E402
from oracle import oracle  # noqa: E402

capi = pkg.capi
LZ4, SNAPPY, ZSTD = capi.CODEC_LZ4BLOCK, capi.CODEC_SNAPPY_XERIAL, capi.CODEC_ZSTD
ALGS = [capi.CHECKSUM_NONE, capi.CHECKSUM_ADLER32, capi.CHECKSUM_CRC32, capi.CHECKSUM_CRC32C]


def env_int(name, default):
    return int(os.environ.get(name, default))


CHUNK_BYTES = env_int("B2S_HOST_CHUNK_MB", 256) << 20
CHUNK_STREAMS = 1 << 18
SLOTS = min(8, max(2, env_int("B2S_SLOTS", 6)))
LAG = max(1, min(env_int("B2S_READ_LAG", 1), (SLOTS - 1) // 2))
COMPRESS_GROUP = max(1, env_int("B2S_LZ4_CHUNK_BLOCKS", 32768))
SNAPPY_DECODE_GROUP = max(1, env_int("B2S_LZ4D_CHUNK_BLOCKS", 65536))

# (name, codec, level, codec block size) of every compress setting
SETTINGS = [("lz4-32k", LZ4, 0, 32768), ("lz4-4k", LZ4, 0, 4096), ("snappy", SNAPPY, 0, 32768),
            ("zstd1", ZSTD, 1, 32768), ("zstd3", ZSTD, 3, 32768)]
# the decompress runs: codec, the setting whose GPU streams are among the inputs, slice checksum
DECODES = [("lz4", LZ4, "lz4-32k", capi.CHECKSUM_CRC32C), ("snappy", SNAPPY, "snappy", capi.CHECKSUM_ADLER32),
           ("zstd", ZSTD, "zstd1", capi.CHECKSUM_CRC32)]

RESULTS = {}
REACH = {}


def check(name, fn, *args):
    try:
        fn(*args)
        RESULTS[name] = "ok"
    except Exception as e:  # noqa: BLE001  (the failure is reported, and the other checks still run)
        RESULTS[name] = "%s: %s" % (type(e).__name__, str(e)[:400])


# ---------------------------------------------------------------------------------------------------------------------
# the chunking rule of the host-pointer calls, and what a call reached
# ---------------------------------------------------------------------------------------------------------------------
def make_chunks(lens):
    """chunk_schedule.h chunk_starts: a chunk takes streams while it has fewer than 2^18 and its bytes stay within the chunk size
    (its first stream always) -> chunk start indices followed by len(lens)"""
    starts, i, n = [], 0, len(lens)
    while i < n:
        starts.append(i)
        b = cnt = 0
        while i < n and cnt < CHUNK_STREAMS and (cnt == 0 or b + lens[i] <= CHUNK_BYTES):
            b += lens[i]
            i += 1
            cnt += 1
    return starts + [n]


def chunk_of(starts, i):
    return int(np.searchsorted(starts, i, side="right")) - 1


def late_stream(starts, pick=lambda i: True):
    """the first stream from the second-to-last chunk on (the middle of the only chunk when there is one) for which
    pick holds, else the last one in front of it"""
    c = max(0, len(starts) - 3)
    first = starts[c] if len(starts) > 2 else starts[-1] // 2
    for i in list(range(first, starts[-1])) + list(range(first - 1, -1, -1)):
        if pick(i):
            return i
    raise AssertionError("no stream to pick")


def reach(call, lens, pipelined=True):
    starts = make_chunks(lens)
    chunks = len(starts) - 1
    counts = [starts[c + 1] - starts[c] for c in range(chunks)]
    r = {"streams": len(lens), "chunks": chunks, "streams_per_chunk": [min(counts), max(counts)]}
    if pipelined:
        r["slot_reuses"] = max(0, chunks - SLOTS)
        # chunks c and c - 2 on one slot (two slots) with a different stream count: the case the read pipeline
        # must order correctly
        r["count_changes_c_vs_c2"] = sum(counts[c] != counts[c - 2] for c in range(2, chunks))
    REACH[call] = r
    return starts


def groups(nb, per):
    """(groups, blocks in the last group) of nb codec blocks split into groups of per"""
    return [-(-nb // per), nb - (-(-nb // per) - 1) * per if nb else 0]


# ---------------------------------------------------------------------------------------------------------------------
# the workload and the CPU references
# ---------------------------------------------------------------------------------------------------------------------
N_MID = 445  # with the blocks configuration's groups of 3 and 5 codec blocks, every last group is a short one


def workload(seed=2024):
    """~29 MiB: 0 B and 1 B streams, 32 KiB +- 1, and seven of 1.5-3 MiB, each of which fills a 1 MiB chunk alone,
    shuffled so that neighbouring chunks hold very different numbers of streams"""
    rng = np.random.default_rng(seed)
    sizes = [0] * 12 + [1] * 12 + [int(32768 + d) for d in rng.integers(-1, 2, N_MID)]
    sizes += [int(s) for s in rng.integers(3 << 19, 3 << 20, 7)]
    rng.shuffle(sizes)
    return [corpus(oracle, KINDS[i % len(KINDS)], n, seed=i) for i, n in enumerate(sizes)]


def load_zmodel(path):
    L = C.CDLL(path)
    L.zc_compress_model_hlog.restype = C.c_longlong
    L.zc_compress_model_hlog.argtypes = [C.c_char_p, C.c_ulonglong, C.c_uint, C.c_char_p, C.c_ulonglong, C.c_int]

    def model(data, block_size, hash_log):
        cap = len(data) + len(data) // 64 + 1024
        buf = C.create_string_buffer(cap)
        n = L.zc_compress_model_hlog(data, len(data), block_size, buf, cap, hash_log)
        assert n > 0
        return buf.raw[:n]
    return model


def spec(zmodel, codec, level, bs, p):
    """the stream the compress kernels must write for p: their executable CPU specification"""
    if codec == LZ4:
        return oracle.lz4block_compress(p, bs, compressor=1)
    if codec == SNAPPY:
        return oracle.xerial_compress(p, bs, compressor=1)
    return zmodel(p, bs, 11 if level == 1 else 13)


def ck(alg, b):
    return oracle.checksum(alg, b) if alg else 0


def packed(parts):
    """parts back to back -> (arena, offsets, lengths)"""
    ln = np.array([len(p) for p in parts], dtype=np.uint64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
    arena = np.frombuffer(b"".join(parts), dtype=np.uint8) if ln.sum() else np.zeros(1, np.uint8)
    return arena, off, ln


def same(what, got, want, starts):
    assert len(got) == len(want), "%s: %d results for %d streams" % (what, len(got), len(want))
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, "%s: %d of %d differ, first: stream %d in chunk %d of %d" % (
        what, len(bad), len(want), bad[0], chunk_of(starts, bad[0]), len(starts) - 1)


def exclusive_sum(v):
    v = np.asarray(v, dtype=np.uint64)
    return np.concatenate([[0], np.cumsum(v)[:-1]]).astype(np.uint64) if v.size else v


# ---------------------------------------------------------------------------------------------------------------------
# checksum
# ---------------------------------------------------------------------------------------------------------------------
def check_checksums(parts):
    starts = reach("checksum", [len(p) for p in parts], pipelined=False)
    arena, off, ln = packed(parts)
    for alg in ALGS[1:]:
        want = [oracle.checksum(alg, p) for p in parts]
        check("checksum_batch/%d" % alg, lambda: same("checksum_batch", capi.checksum_batch(alg, parts), want, starts))
        check("checksum_packed/%d" % alg,
              lambda: same("checksum_packed", [int(v) for v in capi.checksum_packed(alg, arena, off, ln)], want, starts))


# ---------------------------------------------------------------------------------------------------------------------
# compress
# ---------------------------------------------------------------------------------------------------------------------
def compress_batch_check(codec, level, bs, alg, parts, want, starts):
    got, cks, st = capi.compress_batch(codec, parts, bs, alg, level)
    assert st == [0] * len(parts), "status %s" % sorted(set(st))
    same("streams", got, want, starts)
    same("checksums", cks, [ck(alg, w) for w in want], starts)
    # one stream of a late chunk gets a destination one byte short of its stream
    j = late_stream(starts)
    caps = [capi.compress_bound(codec, bs, len(p)) for p in parts]
    caps[j] = len(want[j]) - 1
    got, cks, st = capi.compress_batch(codec, parts, bs, alg, level, dst_caps=caps)
    assert st[j] == capi.E_DST_TOO_SMALL, "short dst_caps entry: status %d" % st[j]
    assert st[:j] + st[j + 1:] == [0] * (len(parts) - 1), "a short dst_caps entry changed another stream's status"
    same("streams beside a short dst_caps entry", got[:j] + got[j + 1:], want[:j] + want[j + 1:], starts)


def compress_packed_check(codec, level, bs, alg, parts, want, starts):
    arena, off, ln = packed(parts)
    cap = sum(capi.compress_bound(codec, bs, len(p)) for p in parts) + 64
    dst = np.zeros(cap, np.uint8)
    r = capi.compress_packed(codec, arena, off, ln, dst, bs, alg, level)
    assert (r["status"] == 0).all(), "status %s" % sorted(set(r["status"].tolist()))
    assert [int(v) for v in r["dst_len"]] == [len(w) for w in want], "dst_len differs from the specification's lengths"
    assert np.array_equal(r["dst_off"], exclusive_sum(r["dst_len"])), "dst_off is not the exclusive sum of dst_len"
    assert r["total"] == sum(len(w) for w in want), "total %d" % r["total"]
    got = [dst[int(o):int(o + l)].tobytes() for o, l in zip(r["dst_off"], r["dst_len"])]
    same("streams", got, want, starts)
    same("checksums", [int(v) for v in r["checksums"]], [ck(alg, w) for w in want], starts)
    # a destination that ends one byte into a stream of a late chunk: the streams in front are intact and OK, that
    # stream and every later one B2S_E_DST_TOO_SMALL
    j = late_stream(starts)
    short = int(r["dst_off"][j]) + 1
    dst2 = np.zeros(short, np.uint8)
    r2 = capi.compress_packed(codec, arena, off, ln, dst2, bs, alg, level)
    st = r2["status"].tolist()
    assert st[:j] == [0] * j, "a stream in front of the short end lost its OK status"
    assert st[j:] == [capi.E_DST_TOO_SMALL] * (len(parts) - j), "streams at and past the short end: %s" % sorted(set(st[j:]))
    assert dst2[:short - 1].tobytes() == dst[:short - 1].tobytes(), "streams in front of the short end differ"


def check_compress(parts, zmodel, gpu_streams):
    starts = reach("compress", [len(p) for p in parts])
    for i, (name, codec, level, bs) in enumerate(SETTINGS):
        want = [spec(zmodel, codec, level, bs, p) for p in parts]
        if len(starts) == 2:  # one chunk: all its codec blocks go through the group pipeline of one call
            REACH["compress_groups/" + name] = groups(sum(-(-len(p) // bs) for p in parts), COMPRESS_GROUP)
        check("compress_batch/" + name, compress_batch_check, codec, level, bs, ALGS[i % 4], parts, want, starts)
        check("compress_packed/" + name, compress_packed_check, codec, level, bs, ALGS[(i + 1) % 4], parts, want,
              starts)
        gpu_streams[name] = want if RESULTS["compress_batch/" + name] == "ok" else None  # what the GPU wrote


# ---------------------------------------------------------------------------------------------------------------------
# decompress
# ---------------------------------------------------------------------------------------------------------------------
def read_inputs(codec, parts, gpu):
    """Streams of every part: the reference writers' for even parts (the oracle's liblz4-style LZ4Block and Snappy,
    libzstd's streaming frames), the GPU's for odd ones.  Consecutive streams are grouped into shuffle blocks of one to
    three streams (ShuffleBlockBatchId), each stream one slice. -> (blocks, their plaintexts, per block [streams])"""
    rng = np.random.default_rng(7 + codec)
    streams = []
    for i, p in enumerate(parts):
        if i % 2 and gpu is not None:
            streams.append(gpu[i])
        elif codec == LZ4:
            streams.append(oracle.lz4block_compress(p, 32768))
        elif codec == SNAPPY:
            streams.append(oracle.xerial_compress(p, 32768))
        else:
            streams.append(zstd_ref.compress_stream(p, level=1 if i % 4 == 1 else 3))
    blocks, plain, members, i = [], [], [], 0
    while i < len(parts):
        g = min(int(rng.choice([1, 1, 1, 2, 3])), len(parts) - i)
        blocks.append(b"".join(streams[i:i + g]))
        plain.append(b"".join(parts[i:i + g]))
        members.append(streams[i:i + g])
        i += g
    return blocks, plain, members


def slice_arrays(slices):
    """per block [(length, checksum)] -> (slice_base, slice_len, slice_checksum)"""
    sb = np.concatenate([[0], np.cumsum([len(s) for s in slices])]).astype(np.uint32)
    sl = np.array([l for s in slices for l, _ in s] or [0], dtype=np.uint64)
    sc = np.array([c for s in slices for _, c in s] or [0], dtype=np.uint64)
    return sb, sl, sc


def decompress_batch_check(codec, alg, blocks, plain, members, starts, bad_block, bad_k):
    sizes, st = capi.decompressed_size_batch(codec, blocks)
    assert st == [0] * len(blocks), "decompressed_size_batch status %s" % sorted(set(st))
    same("decompressed sizes", sizes, [len(p) for p in plain], starts)
    slices = [[(len(s), oracle.checksum(alg, s)) for s in m] for m in members]
    slices[bad_block][bad_k] = (slices[bad_block][bad_k][0], slices[bad_block][bad_k][1] ^ 0x10)
    out, st, bad = capi.decompress_batch(codec, blocks, alg, slices, dst_caps=[len(p) for p in plain])
    want_st = [0] * len(blocks)
    want_st[bad_block] = capi.E_CHECKSUM
    want_bad = [-1] * len(blocks)
    want_bad[bad_block] = bad_k
    same("status", st, want_st, starts)
    same("bad_slice", bad, want_bad, starts)
    want = list(plain)
    want[bad_block] = None
    same("outputs", out, want, starts)


def decompress_packed_check(codec, alg, blocks, plain, members, bad_block, bad_k, dev):
    """decompress_packed (or decompress_dev) with one wrong slice checksum; the packed form also gets one block whose
    slices do not tile it, in front of the wrong checksum's block"""
    blocks, plain = list(blocks), list(plain)
    slices = [[(len(s), oracle.checksum(alg, s)) for s in m] for m in members]
    slices[bad_block][bad_k] = (slices[bad_block][bad_k][0], slices[bad_block][bad_k][1] ^ 0x10)
    want_st = [0] * len(blocks)
    want_st[bad_block] = capi.E_CHECKSUM
    want_bad = [-1] * len(blocks)
    want_bad[bad_block] = bad_k
    if not dev:  # a copy of a two-stream block whose second slice claims 5 bytes more than the block has
        t = next(k for k in range(bad_block - 1, -1, -1) if len(members[k]) == 2)
        blocks.insert(bad_block, blocks[t])
        plain.insert(bad_block, plain[t])
        slices.insert(bad_block, [slices[t][0], (slices[t][1][0] + 5, slices[t][1][1])])
        want_st.insert(bad_block, capi.E_CHECKSUM)
        want_bad.insert(bad_block, 1)
    sb, sl, sc = slice_arrays(slices)
    starts = make_chunks([len(b) for b in blocks])
    arena, off, ln = packed(blocks)
    total_plain = sum(len(p) for p in plain)
    if dev:
        d_src, d_dst = capi.dev_alloc(arena.size), capi.dev_alloc(total_plain)
        try:
            capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
            r = capi.decompress_dev(codec, d_src, off, ln, d_dst, total_plain, alg, sb, sl, sc)
            dst = np.zeros(max(r["total"], 1), np.uint8)
            if r["total"]:
                capi.dev_memcpy(dst.ctypes.data, d_dst, r["total"], 2)
        finally:
            capi.dev_free(d_src)
            capi.dev_free(d_dst)
    else:
        dst = np.zeros(total_plain, np.uint8)
        r = capi.decompress_packed(codec, arena, off, ln, dst, alg, sb, sl, sc)
    same("status", r["status"].tolist(), want_st, starts)
    same("bad_slice", r["bad_slice"].tolist(), want_bad, starts)
    assert np.array_equal(r["dst_off"], exclusive_sum(r["dst_len"])), "dst_off is not the exclusive sum of dst_len"
    assert r["total"] == int(np.sum(r["dst_len"])), "total %d is not the sum of dst_len" % r["total"]
    ok = [i for i in range(len(blocks)) if want_st[i] == 0]
    same("dst_len", [int(r["dst_len"][i]) for i in ok], [len(plain[i]) for i in ok], starts)
    got = [dst[int(r["dst_off"][i]):int(r["dst_off"][i] + r["dst_len"][i])].tobytes() for i in ok]
    same("outputs", got, [plain[i] for i in ok], starts)


def check_decompress(parts, gpu_streams, dev=False):
    for name, codec, setting, alg in DECODES:
        blocks, plain, members = read_inputs(codec, parts, gpu_streams.get(setting))
        starts = reach("decompress/" + name, [len(b) for b in blocks])
        if codec == SNAPPY and len(starts) == 2:
            REACH["snappy_decode_groups"] = groups(sum(-(-len(p) // 32768) for p in parts), SNAPPY_DECODE_GROUP)
        bad_block = late_stream(starts, lambda i: len(members[i]) >= 2 and i > 0)
        bad_k = len(members[bad_block]) - 1
        if dev:
            check("decompress_dev/" + name, decompress_packed_check, codec, alg, blocks, plain, members, bad_block,
                  bad_k, True)
            continue
        check("decompress_batch/" + name, decompress_batch_check, codec, alg, blocks, plain, members, starts,
              bad_block, bad_k)
        check("decompress_packed/" + name, decompress_packed_check, codec, alg, blocks, plain, members, bad_block,
              bad_k, False)


# ---------------------------------------------------------------------------------------------------------------------
# device-resident forms and the one-call families (the codec-block group pipelines inside a single slot)
# ---------------------------------------------------------------------------------------------------------------------
def compress_dev_check(codec, level, bs, alg, parts, want):
    arena, off, ln = packed(parts)
    cap = sum(capi.compress_bound(codec, bs, len(p)) for p in parts) + 64
    d_src, d_dst = capi.dev_alloc(arena.size), capi.dev_alloc(cap)
    try:
        capi.dev_memcpy(d_src, arena.ctypes.data, arena.size, 1)
        r = capi.compress_dev(codec, d_src, off, ln, d_dst, cap, bs, alg, level)
        dst = np.zeros(max(r["total"], 1), np.uint8)
        capi.dev_memcpy(dst.ctypes.data, d_dst, r["total"], 2)
    finally:
        capi.dev_free(d_src)
        capi.dev_free(d_dst)
    starts = [0, len(parts)]
    assert (r["status"] == 0).all(), "status %s" % sorted(set(r["status"].tolist()))
    assert np.array_equal(r["dst_off"], exclusive_sum(r["dst_len"])), "dst_off is not the exclusive sum of dst_len"
    got = [dst[int(o):int(o + l)].tobytes() for o, l in zip(r["dst_off"], r["dst_len"])]
    same("streams", got, want, starts)
    same("checksums", [int(v) for v in r["checksums"]], [ck(alg, w) for w in want], starts)


def check_dev_forms(parts, zmodel, gpu_streams):
    for i, (name, codec, level, bs) in enumerate(SETTINGS):
        want = gpu_streams.get(name) or [spec(zmodel, codec, level, bs, p) for p in parts]
        check("compress_dev/" + name, compress_dev_check, codec, level, bs, ALGS[(i + 2) % 4], parts, want)
    check_decompress(parts, gpu_streams, dev=True)


REC = 104  # a TeraSort record: 2-byte header, 10-byte key, the rest


def partition_check(codec, level, alg):
    rng = np.random.default_rng(codec)
    n, R = 60000, 24
    recs = np.frombuffer(oracle.gen_terasort(1000 * codec, n).tobytes(), np.uint8)
    part = rng.integers(0, R - 1, n).astype(np.uint32)  # partition R - 1 stays empty
    part[:500] = 3  # one large partition
    order = np.argsort(part, kind="stable")
    body = recs.reshape(n, REC)[order].ravel()
    bounds = np.concatenate([[0], np.cumsum(np.bincount(part, minlength=R))]) * REC
    parts = [body[bounds[p]:bounds[p + 1]].tobytes() for p in range(R)]
    ne = [p for p in range(R) if parts[p]]
    arena, off, ln = packed([parts[p] for p in ne])
    cap = sum(capi.compress_bound(codec, 0, len(parts[p])) for p in ne) + 64
    dst = np.zeros(cap, np.uint8)
    want = capi.compress_packed(codec, arena, off, ln, dst, 0, alg, level)
    assert (want["status"] == 0).all()
    pcap = capi.partition_compress_bound(codec, 0, R, recs.size)
    pdst = np.zeros(pcap, np.uint8)
    r = capi.partition_compress_packed(codec, recs, np.full(n, REC, np.uint32), part, R, pdst, 0, alg, level)
    assert (r["status"] == 0).all(), "status %s" % sorted(set(r["status"].tolist()))
    assert r["total"] == want["total"] and pdst[:r["total"]].tobytes() == dst[:want["total"]].tobytes(), \
        "the .data arena differs from compress_packed over the partitioned records"
    assert [int(r["dst_len"][p]) for p in ne] == [int(v) for v in want["dst_len"]], "partition lengths differ"
    assert all(r["dst_len"][p] == 0 for p in range(R) if p not in ne), "an empty partition has bytes"
    assert [int(r["checksums"][p]) for p in ne] == [int(v) for v in want["checksums"]], "partition checksums differ"


def sort_check():
    n = 30000
    recs = np.frombuffer(oracle.gen_terasort(77, n).tobytes(), np.uint8).reshape(n, REC)
    cuts = np.sort(np.random.default_rng(5).choice(np.arange(1, n), 19, replace=False))
    plain = [b.tobytes() for b in np.split(recs, cuts)]
    streams = [oracle.xerial_compress(p, 32768) for p in plain]
    arena, off, ln = packed(streams)
    alg = capi.CHECKSUM_CRC32C
    sb = np.arange(len(streams) + 1, dtype=np.uint32)
    sc = np.array([oracle.checksum(alg, s) for s in streams], dtype=np.uint64)
    dst = np.zeros(n * REC, np.uint8)
    r = capi.decompress_sort_packed(SNAPPY, arena, off, ln, dst, REC, 2, 10, alg, sb, ln, sc)
    assert (r["status"] == 0).all() and r["n_records"] == n and r["total"] == n * REC, r
    order = np.lexsort([recs[:, 2 + j] for j in range(9, -1, -1)])  # stable; the first key byte is the primary one
    assert dst.tobytes() == recs[order].tobytes(), "sorted records differ from a stable sort by the key bytes"
    REACH["sort_snappy_decode_groups"] = groups(sum(-(-len(p) // 32768) for p in plain), SNAPPY_DECODE_GROUP)


def main():
    config, zc = sys.argv[1], sys.argv[2]
    zmodel = load_zmodel(zc)
    capi.init(1)  # device 0 only: the batch calls are not sharded, so every call runs the chunking computed here
    parts = workload()
    gpu_streams = {}
    check_checksums(parts)
    check_compress(parts, zmodel, gpu_streams)
    check_decompress(parts, gpu_streams)
    if config == "blocks":
        check_dev_forms(parts, zmodel, gpu_streams)
        for name, codec, level, alg in (("lz4", LZ4, 0, capi.CHECKSUM_CRC32C), ("snappy", SNAPPY, 0, capi.CHECKSUM_ADLER32),
                                        ("zstd", ZSTD, 1, capi.CHECKSUM_CRC32)):
            check("partition_compress_packed/" + name, partition_check, codec, level, alg)
        check("decompress_sort_packed/snappy", sort_check)
    capi.shutdown()
    print(json.dumps({"config": config, "slots": SLOTS, "read_lag": LAG, "chunk_bytes": CHUNK_BYTES,
                      "compress_group": COMPRESS_GROUP, "snappy_decode_group": SNAPPY_DECODE_GROUP,
                      "checks": RESULTS, "reach": REACH}))


if __name__ == "__main__":
    main()
