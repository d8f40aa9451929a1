"""A model of what Spark's RoundRobinPartitioning writer sees of a map task's UnsafeRows (ShuffleExchangeExec,
Spark 3.5), for the tests of b2s_partition_compress_rows_round_robin_*:

- with spark.sql.execution.sortBeforeRepartition and R > 1 the rows are sorted first: by row.hashCode() =
  Murmur3_x86_32.hashUnsafeWords(row, 42) as a signed int, then by RecordBinaryComparator (the shorter row first, then
  unsigned bytes); otherwise they stay in input order;
- the k-th row of that order goes to partition (position + 1 + k) mod R, position = XORShiftRandom(partitionId)
  .nextInt(R), which the caller passes as start.

In two forms: scalar (plain Python over row bytes) and vectorised (numpy lexsort over the hash and size, ties of both
broken in Python over the tied groups only), which the GPU tests use at scale.  Also: the records reordered as the
writer sees them with their ids, to feed b2s_partition_compress_packed."""
import numpy as np

import hash_model as hm

SEED = 42  # UnsafeRow.hashCode's seed


def hash_unsafe_words(b, seed=SEED):
    """Murmur3_x86_32.hashUnsafeWords: whole little-endian 4-byte words only (len(b) % 4 == 0)"""
    assert len(b) % 4 == 0
    h = seed & hm.M32
    for i in range(0, len(b), 4):
        h = hm._mix_h1(h, hm._mix_k1(int.from_bytes(b[i:i + 4], "little")))
    return hm._fmix(h, len(b))


def row_hash(row):
    """row.hashCode() as Java's signed int"""
    return hm.signed(hash_unsafe_words(row))


def sort_key(row):
    """the sort's order: signed hash, then RecordBinaryComparator (length first, then unsigned lexicographic)"""
    return (row_hash(row), len(row), bytes(row))


def sorted_order(rows, sort, R):
    """indices of rows in the order the writer sees them"""
    if not sort or R == 1:
        return list(range(len(rows)))
    return sorted(range(len(rows)), key=lambda i: sort_key(rows[i]))


def ids(n, start, R):
    """the partition of the k-th row the writer sees"""
    return [(start + 1 + k) % R for k in range(n)]


def record_hashes_np(records, rec_len):
    """signed row hash of every framed record ([int32 big-endian size][row], rows of whole words), vectorised; rows
    longer than hm.LONG_BYTES are hashed by the scalar form"""
    rl = np.asarray(rec_len, np.int64)
    start = np.concatenate([[0], np.cumsum(rl)[:-1]]).astype(np.int64)
    size = rl - 4
    h = np.full(rl.size, SEED, np.uint32)
    short = np.nonzero(size <= hm.LONG_BYTES)[0]
    if short.size:
        h[short] = hm._v_hash_bytes(records, start[short] + 4, size[short], h[short])
    for i in np.nonzero(size > hm.LONG_BYTES)[0]:
        h[i] = hash_unsafe_words(records[start[i] + 4:start[i] + 4 + size[i]].tobytes())
    return h.view(np.int32), start, size


def sorted_order_np(records, rec_len, sort, R):
    """sorted_order over framed records, vectorised"""
    n = len(rec_len)
    if not sort or R == 1 or n < 2:
        return np.arange(n, dtype=np.int64)
    h, start, size = record_hashes_np(records, rec_len)
    order = np.lexsort((size, h))
    hs, ss = h[order], size[order]
    brk = np.concatenate([[True], (hs[1:] != hs[:-1]) | (ss[1:] != ss[:-1]), [True]])
    edges = np.nonzero(brk)[0]
    for a, b in zip(edges[:-1], edges[1:]):
        if b - a > 1:  # equal hash and size: the row bytes decide
            grp = order[a:b]
            order[a:b] = sorted(grp, key=lambda i: records[start[i] + 4:start[i] + 4 + size[i]].tobytes())
    return order


def writer_records(records, rec_len, start, R, sort):
    """(records in the writer's order, their rec_len, their ids): b2s_partition_compress_packed of these is what the
    round-robin call must return"""
    rl = np.asarray(rec_len, np.uint32)
    order = sorted_order_np(records, rl, sort, R)
    off = np.concatenate([[0], np.cumsum(rl.astype(np.int64))]).astype(np.int64)
    parts = [records[off[i]:off[i + 1]] for i in order]
    recs = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    return recs, rl[order], np.array(ids(len(order), start, R), np.uint32)
