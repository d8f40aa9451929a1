/*
 * b200shuffle.h — flat C ABI of libb200shuffle.so, the H100-native (sm_90a) shuffle-block codec path.
 *
 * This is the drop-in boundary for IBM/spark-s3-shuffle's codec hot path.  The reference has no FFI of its own
 * (it is pure Scala and reaches native code only through lz4-java / snappy-java / zstd-jni / java.util.zip); each
 * entry point below names the reference interface (file:line under /root/reference/src/main/scala/org/apache/spark)
 * whose work it replaces.  INTEGRATION.md shows the JNI stub + Scala classes a maintainer adds on the JVM side.
 *
 *   write side  (map task)   : per-partition  compress  + checksum          -> b2s_compress_*
 *       replaces the CompressionCodec.compressedOutputStream + MutableCheckedOutputStream chain that feeds
 *       shuffle/S3ShuffleMapOutputWriter.scala:140-146,168-202 and whose results arrive at :91,113-115
 *   read side   (reduce task): checksum-verify + decompress per block        -> b2s_decompress_*
 *       replaces storage/S3ChecksumValidationStream.scala:54-86 and serializerManager.wrapStream at
 *       storage/S3ShuffleReader.scala:99-110
 *   checksums only                                                           -> b2s_checksum_*
 *       replaces helper/S3ShuffleHelper.scala:94-103 (ADLER32 | CRC32) and adds CRC32C
 *
 * Conventions: plain pointers and sizes, no C++ or torch types.  Every call is synchronous (returns when results
 * are in the caller's buffers) and re-entrant.  Function return: 0 = call completed (inspect per-block status[]),
 * negative B2S_E_* = the call itself failed.  The library never aborts the process and has NO CPU fallback: without
 * a usable CUDA device every compute entry point returns B2S_E_CUDA.
 *
 * "_packed" variants take/produce one contiguous arena plus offsets — the layout of a .data object
 * (concatenated per-partition streams, ascending reduceId; SURVEY.md appendix A) — so one H2D/D2H moves a whole
 * batch and dst_len[] *is* the partitionLengths array handed to helper/S3ShuffleHelper.scala:44-47.
 * "_dev" variants take device pointers for data (descriptor arrays stay on the host) and are what the
 * device-resident roofline measurement in bench.py drives.
 */
#ifndef B200SHUFFLE_H
#define B200SHUFFLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_VERSION 0x000100

/* codecs — Spark's spark.io.compression.codec short names (storage/S3ShuffleReader.scala:57-60 probes the codec) */
#define B2S_CODEC_NONE 0
#define B2S_CODEC_LZ4BLOCK 1      /* "lz4"   : lz4-java LZ4Block stream, XXH32 seed 0x9747b28c & 0x0FFFFFFF */
#define B2S_CODEC_SNAPPY_XERIAL 2 /* "snappy": xerial SnappyOutputStream framing over raw snappy */
#define B2S_CODEC_ZSTD 3          /* "zstd"  : RFC 8878 frames, concatenation allowed; a frame's Content_Checksum
                                   * is skipped, not verified (Spark's ZStdCompressionCodec never sets the flag), so
                                   * a frame that libzstd rejects for a wrong content checksum alone decodes here */

/* checksum algorithms — spark.shuffle.checksum.algorithm (helper/S3ShuffleHelper.scala:94-103) */
#define B2S_CHECKSUM_NONE 0
#define B2S_CHECKSUM_ADLER32 1
#define B2S_CHECKSUM_CRC32 2
#define B2S_CHECKSUM_CRC32C 3 /* north-star addition; the Scala shim adds the "CRC32C" case */

/* key types of the row sort (b2s_decompress_sort_rows_*) */
#define B2S_KEY_BYTES 0 /* key_len (1..16) bytes, unsigned, lexicographic */
#define B2S_KEY_INT32 1 /* 4 bytes, little-endian two's complement: UnsafeRow's IntegerType / DateType slot */
#define B2S_KEY_INT64 2 /* 8 bytes, little-endian two's complement: LongType, TimestampType, Decimal(p <= 18) */
/* the composite-key calls (b2s_decompress_*_rows_keys_*) also take: an 8-byte UnsafeRow slot (offset << 32) | size
 * naming the size bytes at row offset offset, unsigned lexicographic, a proper prefix first (StringType under
 * UTF8_BINARY, BinaryType) */
#define B2S_STRING_KEY 3
/* ... and these column types (4 is unassigned); BooleanType needs none: it is B2S_KEY_BYTES with key_len 1 (0 / 1) */
#define B2S_KEY_INT16 (5)   /* 2 bytes, little-endian two's complement: ShortType */
#define B2S_KEY_INT8 (6)    /* 1 byte, signed: ByteType */
#define B2S_KEY_FLOAT32 (7) /* 4 bytes, IEEE float, Spark SQL's order: -0.0 == 0.0, NaN == NaN above +inf: FloatType */
#define B2S_KEY_FLOAT64 (8) /* 8 bytes, IEEE double, the same order: DoubleType */
/* an 8-byte UnsafeRow slot (offset << 32) | size naming size (1..16) bytes at row offset offset: the unscaled value of
 * a Decimal(p > 18), big-endian two's complement (BigInteger.toByteArray), ordered as a signed integer */
#define B2S_DECIMAL_KEY (9)
/* order flags, OR-ed into a composite-key column's key_type: its non-null values sort in reverse; its nulls sort after
 * its non-null values (Spark's SortOrder direction and null ordering; NULLS_LAST on a column without a null bit is
 * accepted and changes nothing) */
#define B2S_KEY_DESCENDING (1u << 8)
#define B2S_KEY_NULLS_LAST (1u << 9)
/* a null-safe (<=>) key column, OR-ed into key_type: Spark's ExtractEquiJoinKeys expands l <=> r into the key pairs
 * (Coalesce(l, Literal.default(t)), Coalesce(r, ...)) and (IsNull(l), IsNull(r)), so the column is the pair
 * (coalesce(v, default), isnull(v)): default 0 for numbers, dates and timestamps, 0 for decimals (a wide one as
 * BigInteger.ZERO.toByteArray(), the one byte 0x00), empty for strings and binary, false for booleans.  Accepted only by
 * the join calls (b2s_decompress_join_rows_keys_*) and the hash calls (b2s_partition_compress_rows_hash_*, their cached
 * form included); every other call that takes key types returns B2S_E_ARG for it. */
#define B2S_KEY_NULL_SAFE (1u << 10)

/* aggregate ops of the row aggregation (b2s_decompress_aggregate_rows_*), each over an 8-byte slot of the row */
#define B2S_AGG_SUM_INT64 0   /* wrapping two's-complement sum: Sum(long), Count, Average's count */
#define B2S_AGG_SUM_FLOAT64 1 /* IEEE double sum: Sum(double), Average's sum */
#define B2S_AGG_MIN_INT32 2
#define B2S_AGG_MAX_INT32 3
#define B2S_AGG_MIN_INT64 4
#define B2S_AGG_MAX_INT64 5
#define B2S_AGG_MIN_FLOAT64 6
#define B2S_AGG_MAX_FLOAT64 7
/* Decimal buffers (8 is unassigned).  SUM_DECIMAL carries the buffer's precision P (1..38) in bits 8..15:
 * B2S_AGG_SUM_DECIMAL | (P << 8).  P <= 18: the slot holds the unscaled long; P > 18: the slot is (offset << 32) | size
 * naming 1..16 big-endian two's-complement bytes, as B2S_DECIMAL_KEY reads them.  MIN / MAX_DECIMAL take a
 * Decimal(p > 18) slot in that out-of-line form; a Decimal(p <= 18) min / max is MIN / MAX_INT64. */
#define B2S_AGG_SUM_DECIMAL (9)  /* Sum(decimal)'s and Average(decimal)'s sum: exact, null on overflow of 10^P */
#define B2S_AGG_MIN_DECIMAL (10) /* Min(decimal p > 18) */
#define B2S_AGG_MAX_DECIMAL (11) /* Max(decimal p > 18) */
/* Spark's CentralMomentAgg buffers of order 2 (stddev_*, var_*): one entry over three consecutive 8-byte double slots,
 * n at agg_off, avg at agg_off + 8, m2 at agg_off + 16; never null (agg_null_field -1), no precision bits.  The group's
 * buffer starts at (0.0, 0.0, 0.0) and merges each record's (n2, avg2, m2b) in stable order by mergeExpressions:
 *   newN = n1 + n2; delta = avg2 - avg1; deltaN = newN == 0.0 ? 0.0 : delta / newN;
 *   avg' = avg1 + deltaN * n2; m2' = (m2a + m2b) + ((delta * deltaN) * n1) * n2; n' = newN
 * every operation one IEEE double operation rounded to nearest, left to right, no FMA. */
#define B2S_AGG_VARIANCE (B2S_AGG_MAX_DECIMAL + 1)

/* per-block status / call errors.  The Scala shim maps them to the reference's exception types:            */
#define B2S_OK 0
#define B2S_E_CORRUPT (-1)       /* IOException("Stream is corrupted")  (LZ4BlockInputStream et al. [U])   */
#define B2S_E_CHECKSUM (-2)      /* SparkException("Invalid checksum detected for <block>") S3ChecksumValidationStream.scala:72-74 */
#define B2S_E_DST_TOO_SMALL (-3) /* retry with a larger destination                                          */
#define B2S_E_UNSUPPORTED (-4)   /* UnsupportedOperationException (S3ShuffleHelper.scala:100-101)            */
#define B2S_E_ARG (-5)           /* RuntimeException("Precondition: ...")                                    */
#define B2S_E_CUDA (-6)          /* no device / CUDA failure; b2s_last_error() has the text                  */
#define B2S_E_NOT_INIT (-7)
#define B2S_E_NOMEM (-8)
#define B2S_E_NOT_CACHED (-9) /* an exchange-cache source is not resident (evicted, removed, other device): fetch it */

/* ---- lifecycle: call once per executor, beside S3ShuffleDataIO.initializeExecutor (shuffle/S3ShuffleDataIO.scala:30-32) ---- */
/* gpu_mask: bit i selects CUDA device i (0 = all visible devices).  The per-stream-pointer calls (b2s_*_batch) shard
 * their streams round-robin over the selected devices (stream i -> device i mod D), one host thread, pinned staging and
 * streams per device, nothing exchanged between devices.  Packed and device-resident calls run on ONE device: the calling
 * thread's (b2s_set_thread_device, default 0) — an executor pins each task thread to a device, or, as bench.py does,
 * runs one process per GPU.  streams_per_gpu = pipeline slots (stream pair + staging) per lane, 2..8, 0 = default 6;
 * pinned_bytes_per_gpu = the library's own pinned descriptor blocks are allocated up front from this budget (0 = grow on
 * demand; payload staging is the caller's, b2s_host_alloc).  Every device runs two LANES — write-side calls take one,
 * read-side calls the other — so a compress and a decompress call from different threads overlap on the full-duplex
 * link.  Idempotent. */
int b2s_init(uint32_t gpu_mask, uint64_t pinned_bytes_per_gpu, uint32_t streams_per_gpu);
void b2s_shutdown(void);
int b2s_device_count(void); /* devices selected by b2s_init, or B2S_E_NOT_INIT */
int b2s_set_thread_device(uint32_t dev_index); /* device used by this thread's packed / host-pointer calls */
/* NUMA placement (SURVEY.md §8e "NUMA-pin staging buffers to the GPU's socket"; the reference's task threads are the
 * ones of storage/S3BufferedPrefetchIterator.scala:78-92 and the map task).  b2s_bind_thread_to_device = set_thread_device
 * + pin the calling thread to the CPUs of the device's NUMA node + prefer that node for its allocations (best effort;
 * a no-op returning 0 when the topology is unknown or B2S_NUMA=0).  b2s_host_alloc always places its pages next to the
 * calling thread's device.  b2s_device_numa_node: the node, -1000 if unknown. */
int b2s_bind_thread_to_device(uint32_t dev_index);
int b2s_device_numa_node(uint32_t dev_index);
const char* b2s_strerror(int32_t code);
const char* b2s_last_error(void); /* thread-local text of the last B2S_E_CUDA / B2S_E_ARG */
uint32_t b2s_version(void);

/* pinned host memory the JVM side wraps as direct ByteBuffers (replaces the byte[] of
 * storage/S3BufferedInputStreamAdaptor.scala:11 and the BufferedOutputStream of S3ShuffleMapOutputWriter.scala:46-47) */
void* b2s_host_alloc(uint64_t bytes);
void b2s_host_free(void* p);
int b2s_host_register(void* p, uint64_t bytes);
int b2s_host_unregister(void* p);

/* ---- sizing ---- */
/* worst-case compressed size of one stream of src_len bytes (codec_block_size 0 = Spark default 32 KiB) */
uint64_t b2s_compress_bound(uint32_t codec, uint32_t codec_block_size, uint64_t src_len);
/* decompressed size of each compressed stream (LZ4Block: sum of originalLen; Snappy: sum of chunk varints).  A stream
 * whose framing, or a Snappy chunk's claim, fails the rules of b2s_decompress_batch gets its status here, per stream. */
int b2s_decompressed_size_batch(uint32_t codec, uint32_t n, const uint8_t* const* src, const uint64_t* src_len,
                                uint64_t* out_len, int32_t* status);

/* ---- checksums: one value per slice of bytes (low 32 bits significant, as in the .checksum file) ---- */
int b2s_checksum_batch(uint32_t alg, uint32_t n, const uint8_t* const* src, const uint64_t* len, uint64_t* out);
int b2s_checksum_packed(uint32_t alg, uint32_t n, const uint8_t* base, const uint64_t* off, const uint64_t* len,
                        uint64_t* out);

/* ---- write side ---- */
/* n independent streams (one per (map,reduce) partition).  Each output is a complete, self-terminated stream in the
 * codec's JVM wire format; checksum_out[i] (if checksum_alg != 0) is over the *compressed* bytes of stream i. */
int b2s_compress_batch(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t n,
                       const uint8_t* const* src, const uint64_t* src_len, uint8_t* const* dst,
                       const uint64_t* dst_cap, uint64_t* dst_len, uint64_t* checksum_out, int32_t* status);
/* packed: stream i is src_base[src_off[i] .. +src_len[i]); outputs are written back to back into dst_base in index
 * order: dst_off[i], dst_len[i].  *dst_total receives the arena bytes used. */
int b2s_compress_packed(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t n,
                        const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len, uint8_t* dst_base,
                        uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                        uint64_t* checksum_out, int32_t* status);

/* ---- write side, serialized shuffle: partition + compress in one call ----
 * Replaces what ShuffleExternalSorter / UnsafeShuffleWriter (serialized shuffle, spark.shuffle.sort) and the Bypass
 * writer do on the CPU before S3ShuffleMapOutputWriter sees a byte: split the map task's serialized records by reduce
 * id, then compress + checksum each partition.  With a relocatable serializer a partition's stream is the
 * concatenation of its records in insertion order, so the caller hands over the records back to back plus one
 * partition id per record and gets the finished .data arena, partitionLengths and .checksum values back.
 *
 * Records: record i is rec_len[i] bytes of rec_base, back to back (sum rec_len == rec_bytes), reduce id rec_part[i].
 * Output, per partition p of num_partitions (empty ones included): dst_off[p], dst_len[p], checksum_out[p] (may be
 * NULL), status[p].  Partitions come in ascending id; the records of a partition keep their input order (a stable
 * partition, as Spark's writers produce).  A partition with no bytes has dst_len 0, takes no room in the arena (its
 * dst_off is where the next partition starts) and has the checksum of a zero-length slice; every other partition is a
 * complete, self-terminated stream in the codec's JVM wire format, byte for byte what b2s_compress_packed makes of it.
 * codec B2S_CODEC_NONE partitions and checksums only: the arena holds the partitioned records
 * (spark.shuffle.compress=false).  *dst_total = arena bytes.
 * Errors: num_partitions outside [1, 2^24] (PackedRecordPointer's 24-bit partition id), an id >= num_partitions or
 * sum rec_len != rec_bytes -> B2S_E_ARG, nothing reported as written, b2s_last_error() names the first offending
 * record.  dst_cap below the arena -> B2S_E_DST_TOO_SMALL, status[p] = B2S_E_DST_TOO_SMALL for the partitions that do
 * not fit and *dst_total = the bytes needed.  Device memory for the records, their partitioned copy and the codec
 * workspace that cannot be had -> B2S_E_NOMEM.  n_records = 0 is valid: every partition is empty.
 * Runs on the calling thread's device, on its write lane (like b2s_compress_*), and fills b2s_last_timing. */
/* worst-case .data bytes for rec_bytes of records spread over num_partitions partitions, any distribution */
uint64_t b2s_partition_compress_bound(uint32_t codec, uint32_t codec_block_size, uint32_t num_partitions,
                                      uint64_t rec_bytes);
/* host records (ideally b2s_host_alloc memory): one upload, the partition step, compression, one download */
int b2s_partition_compress_packed(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
                                  uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base,
                                  uint64_t rec_bytes, const uint32_t* rec_len, const uint32_t* rec_part,
                                  uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                                  uint64_t* dst_total, uint64_t* checksum_out, int32_t* status);
/* same, with rec_base / rec_len / rec_part / dst_base in device memory of dev_index (they are data-sized); the
 * per-partition outputs stay host arrays, as in the other _dev calls */
int b2s_partition_compress_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                               uint32_t checksum_alg, uint32_t num_partitions, uint64_t n_records,
                               const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
                               const uint32_t* rec_part, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                               uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status);

/* ---- write side, hash-partitioned rows: Spark's HashPartitioning ids computed on the GPU ----
 * b2s_partition_compress_* for a HashPartitioning exchange of UnsafeRows: the reduce id of every record is Spark's
 * pmod(Murmur3Hash(key columns, 42), num_partitions), bit for bit, so the caller passes no rec_part.  Record i is
 * rec_len[i] bytes as UnsafeRowSerializer writes a row: [size s: int32 big-endian][s bytes of row], rec_len[i] = 4 + s.
 * The key columns are given as to the composite-key calls (b2s_decompress_*_rows_keys_*, below): n_keys (1..16),
 * key_type[c] at row offset key_off[c], key_len[c] bytes, null bit key_null_field[c] (-1: never null).  Starting from
 * h = 42, each column left to right sets h = its hash with seed h; a null column leaves h as it is (all null: 42).
 * A B2S_KEY_NULL_SAFE column takes two steps, as HashPartitioning over its expanded key pair does: h = the hash of its
 * value by its type's rule below, of the type's default when the column is null (so a null changes h), then
 * h = hashInt(isnull ? 1 : 0).  A column without a null bit (-1) is never null: its second step is hashInt(0).
 *   B2S_KEY_BYTES, key_len 1 (BooleanType): hashInt(byte != 0 ? 1 : 0)
 *   B2S_KEY_INT8 / B2S_KEY_INT16 / B2S_KEY_INT32 (ByteType, ShortType, IntegerType, DateType): hashInt of the value
 *   B2S_KEY_INT64 (LongType, TimestampType, Decimal(p <= 18)): hashLong
 *   B2S_KEY_FLOAT32 / B2S_KEY_FLOAT64: hashInt(floatToIntBits) / hashLong(doubleToLongBits), -0.0 as 0.0 and every NaN
 *     as the canonical NaN (Spark >= 3.2)
 *   B2S_STRING_KEY (StringType, BinaryType) / B2S_DECIMAL_KEY (Decimal(p > 18), 1..16 bytes): hashUnsafeBytes of the
 *     slot's bytes, with Spark's tail (every byte after the last whole 4-byte word mixed on its own, sign-extended)
 * Outputs: byte for byte what b2s_partition_compress_packed / _dev return for the same records and those ids.
 * Errors, B2S_E_ARG: what b2s_partition_compress_* rejects; n_keys outside 1..16, a type not listed, a key_len that does
 * not match its type, an order flag (B2S_KEY_NULL_SAFE is not one), key_null_field < -1.  A bad record -> B2S_E_ARG,
 * nothing reported as written, and
 * b2s_last_error() names the lowest bad record and why: rec_len < 4, a size prefix other than rec_len - 4, a row that
 * does not hold a key slot or a key's null word, a non-null string past the row, a non-null decimal whose size is not
 * 1..16 or that runs past the row.  No usable device -> B2S_E_CUDA.  b2s_last_timing as for the partition calls, plus
 * dominant_ms / dominant_launches = the hash step alone.  Exchange-cache form: b2s_partition_compress_rows_hash_cached_packed
 * (below, with the exchange cache). */
int b2s_partition_compress_rows_hash_packed(uint32_t codec, int32_t level, uint32_t codec_block_size,
                                            uint32_t checksum_alg, uint32_t num_partitions, uint64_t n_records,
                                            const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
                                            uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
                                            const uint32_t* key_len, const int32_t* key_null_field, uint8_t* dst_base,
                                            uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                                            uint64_t* dst_total, uint64_t* checksum_out, int32_t* status);
/* same, with rec_base / rec_len / dst_base in device memory of dev_index */
int b2s_partition_compress_rows_hash_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                                         uint32_t checksum_alg, uint32_t num_partitions, uint64_t n_records,
                                         const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
                                         uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
                                         const uint32_t* key_len, const int32_t* key_null_field, uint8_t* dst_base,
                                         uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                         uint64_t* checksum_out, int32_t* status);

/* ---- write side, partial aggregation: Spark's HashAggregateExec(Partial) and its hash exchange on the GPU ----
 * The map side of a grouped aggregation's shuffle (HashAggregateExec(Partial) -> Exchange hashpartitioning(keys)) in
 * one call: the map task's rows are grouped by the key columns, Spark's aggregation buffers are folded over each group,
 * one partial row is written per key, and the partial rows are hash-partitioned and compressed into the .data object.
 * A reducer merges them with b2s_decompress_aggregate_rows_keys_* (the merge ops below).
 * Records: as for b2s_partition_compress_rows_hash_*: [size: int32 big-endian][row], rec_len[i] = 4 + size.
 * Key columns: exactly those of the hash call (n_keys 1..16, its types, no order flags; B2S_KEY_BYTES is a 1-byte
 * boolean).  n_keys = 0, a global aggregate, is B2S_E_ARG: Spark does not hash-partition it.
 * Grouping: a group is a maximal set of records whose every key column is equal by the composite-key aggregation's
 * rule: nulls equal nulls, strings are equal when their lengths and bytes are, 0.0 equals -0.0, every NaN equals every
 * NaN.
 * Aggregates: agg_fn[a] (a < n_aggs, at most 16; 0 is DISTINCT) is B2S_WINDOW_SUM .. B2S_WINDOW_AVG or
 * B2S_WINDOW_VARIANCE, val_type[a] a
 * B2S_WINDOW_VAL_* (a decimal(p, s): B2S_WINDOW_VAL_DECIMAL | p << 8 | s << 16), val_off[a] the input's 8-byte slot
 * (for p > 18 the slot (offset << 32) | size names 1..16 big-endian two's-complement bytes), val_null_field[a] its
 * null bit or -1, as in the window aggregate call.  The semantics are Spark 3.5's DeclarativeAggregate.updateExpressions
 * with ANSI off, folded over the group's records in input order.  Each function writes its buffers (Spark's
 * aggBufferAttributes order), in function order:
 *   SUM int8/16/32/64        long: the wrapping sum of the non-null inputs, sign-extended; null if none.
 *                            Merge: B2S_AGG_SUM_INT64
 *   SUM float / double       double: ((0.0 + x1) + x2) + ... over the non-null inputs, floats widened exactly, each add
 *                            rounded to nearest (a lone -0.0 gives +0.0); null if none.  Merge: B2S_AGG_SUM_FLOAT64
 *   SUM decimal(p, s), p<=28 decimal(p + 10, s): the exact sum, 0 if no input is non-null (below 2^32 records it never
 *                            overflows); boolean isEmpty: 1 iff no input is non-null.  Never null.
 *                            Merge: B2S_AGG_SUM_DECIMAL | (p + 10) << 8, B2S_AGG_MIN_INT32
 *   COUNT, any val_type,     long: the non-null inputs (every record for VAL_NONE, count(*)); never null.
 *   VAL_NONE or VAL_BYTES    Merge: B2S_AGG_SUM_INT64
 *   AVG int8 .. double       double sum ((0.0 + c1) + c2) + ..., c the input cast to double (a long rounded to nearest),
 *                            0.0 when null; long count of the non-null inputs.  Never null.
 *                            Merge: B2S_AGG_SUM_FLOAT64, B2S_AGG_SUM_INT64
 *   AVG decimal(p, s), p<=27 decimal(p + 10, s) exact sum (0 if none), long count.  Merge: B2S_AGG_SUM_DECIMAL |
 *                            (p + 10) << 8, B2S_AGG_SUM_INT64.  Spark's Average adds with Add, whose result type for
 *                            (P, s) + (P, s) is decimal(P + 1, s), exact only while P + 1 <= 38; Sum adds with
 *                            DecimalAddNoOverflowCheck into its buffer type, so it takes p 28.
 *   MIN / MAX int / date     int; long / timestamp / decimal(p <= 18): long; double: double; decimal(p > 18): decimal.
 *                            Spark's Least / Greatest in Spark SQL's order (-0.0 equals 0.0, NaN above every other value
 *                            and equal to every NaN): among equal values the first is kept, with its exact bits.  Null
 *                            if none.  Merge: B2S_AGG_MIN / MAX_INT32, _INT64, _FLOAT64, _DECIMAL
 *   VARIANCE (16) int8 ..    stddev / stddev_samp / stddev_pop / variance / var_samp / var_pop (CentralMomentAgg, order
 *   int64, float, double     2): three doubles n, avg, m2, from (0, 0, 0), each non-null input x = Cast(child, Double) (a
 *                            long rounded to nearest, a float widened) in input order by updateExpressions: newN = n +
 *                            1.0; delta = x - avg; deltaN = delta / newN; avg' = avg + deltaN; m2' = m2 + delta * (delta
 *                            - deltaN); every operation one IEEE double operation rounded to nearest, no FMA.  Never
 *                            null.  One buffer, three fields.  Merge: B2S_AGG_VARIANCE at n's slot (null field -1)
 * Partial row: as UnsafeProjection(groupingAttributes ++ aggBufferAttributes) writes it, with nf = n_keys + fields,
 * the fields being 1 per buffer and 3 per VARIANCE (at most 32, so one null word, b = 1): field c < n_keys is key column
 * c, then the buffers' fields in order, whose null bit is set only for a null value.  Fixed values are written as UnsafeRowWriter writes them (the 8-byte slot zeroed, then
 * the type's width; an isEmpty boolean one byte).  Key values come from the group's first record in input order; float
 * and double keys are normalized as NormalizeNaNAndZero leaves them (-0.0 as 0.0, any NaN as the canonical NaN).  Var
 * regions follow the fixed region 8 (b + nf), in field order: a string or binary key its bytes zero-padded to 8 (a null
 * one: slot 0, no bytes); a decimal(p > 18) key or buffer 16 bytes holding BigInteger.toByteArray's minimal bytes,
 * zero-padded, slot (offset << 32) | length (a null one: 16 zero bytes, slot offset << 32).
 * Order and outputs: the partial rows are produced in the composite-key sort's order (ascending, nulls first) and then
 * partitioned stably by pmod(Murmur3Hash(key columns, 42), num_partitions).  dst_off / dst_len / checksum_out / status,
 * *dst_total and the return value are byte for byte what b2s_partition_compress_rows_hash_packed returns for those
 * partial rows in that order, keyed by the key columns at their output slots (8 + 8 c, null bit c when key_null_field[c]
 * >= 0).  *n_groups (required) = the partial rows.
 * Sizing: dst_cap below the arena -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes needed, as the partition calls.
 * With W the decimal(p > 18) fields (keys and buffers) and S the string / binary key columns, an arena of
 *   b2s_partition_compress_bound(codec, codec_block_size, num_partitions,
 *                                n_records * (4 + 8 (1 + nf) + 16 W + 8 S) + S * rec_bytes)
 * bytes always suffices: a partial row's string key holds at most its input row's bytes plus 7 of padding, so the bound
 * holds even when several key columns name the same bytes.
 * Errors, B2S_E_ARG, checked before the device: what the hash call rejects; n_records >= 2^32; n_aggs above 16 or a
 * NULL aggregate array (n_aggs > 0) or n_groups; an unknown function or val_type; a decimal p outside 1..38 or s > p;
 * VAL_NONE or VAL_BYTES with a function other than COUNT; MIN / MAX of byte, short, float or bytes (the reducer cannot
 * merge them); decimal SUM with p > 28 or AVG with p > 27; VARIANCE of a decimal, VAL_NONE or VAL_BYTES; more than 16
 * buffers in all (the reduce-side merge's limit; a VARIANCE is one); n_keys + fields above 32;
 * a val_off that is not a multiple of 8 of at least 8 (a field's slot), or a val_null_field outside -1..65535.  A bad
 * record -> B2S_E_ARG, nothing reported as written, b2s_last_error() names the lowest bad record and why: the hash call's
 * record checks, a row that does not hold a value slot or a value's null word, a non-null decimal(p > 18) value whose
 * size is not 1..16 or that runs past its row.  Device memory that cannot be had -> B2S_E_NOMEM (the caller keeps
 * Spark's partial aggregation).  No usable device -> B2S_E_CUDA.
 * Runs on the write lane.  b2s_last_timing: kernel_ms the whole call's device work, dominant_ms / dominant_launches the
 * aggregation step (from the input records to the written partial rows). */
int b2s_aggregate_partition_compress_rows_hash_packed(
    uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len, uint32_t n_keys,
    const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
    uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type, const uint32_t* val_off,
    const int32_t* val_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
    uint64_t* dst_total, uint64_t* checksum_out, int32_t* status, uint64_t* n_groups);
/* same, with rec_base / rec_len / dst_base in device memory of dev_index; the other arrays stay host arrays */
int b2s_aggregate_partition_compress_rows_hash_dev(
    uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
    uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
    uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
    const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
    uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status, uint64_t* n_groups);

/* ---- write side, grouping sets: Spark's Expand and HashAggregateExec(Partial) and its hash exchange on the GPU ----
 * The map side of a ROLLUP, CUBE or GROUPING SETS aggregation's shuffle (Expand -> HashAggregateExec(Partial) ->
 * Exchange hashpartitioning(grouping columns, spark_grouping_id)) in one call.  The arguments are those of
 * b2s_aggregate_partition_compress_rows_hash_* in the same order, with n_sets / set_mask after the aggregate arrays:
 * bit c of set_mask[k] is set when key column c belongs to grouping set k.  The semantics are Spark 3.5's Expand
 * followed by HashAggregateExec(Partial), ANSI off, spark.sql.legacy.integerGroupingId off:
 * Input records: as for b2s_aggregate_partition_compress_rows_hash_*.  Record r stands for the n_sets projected records
 * (r, k), in row-major order (0, 0), (0, 1), .., (1, 0), ..: ExpandExec's output order.  Every record of a group comes
 * from one set, so each group's fold order is the input order.
 * Projected record (r, k): key column c takes record r's value if bit c of set_mask[k] is set, and null otherwise; one
 * more key column follows them: gid, a never-null long, the sum of 1 << (n_keys - 1 - c) over the columns c outside the
 * set (Spark's spark_grouping_id: ROLLUP(a, b, c)'s sets give 0, 1, 3, 7; CUBE(a, b)'s 0, 1, 2, 3).  Aggregate inputs
 * are read from record r unmasked: Spark's aggregate functions reference the child's attribute, not the nulled
 * grouping alias.
 * Partial rows: n_keys grouping columns, every one nullable, then gid (INT64, slot 8 + 8 n_keys), then the buffers, as
 * UnsafeProjection(groupingAttributes ++ aggBufferAttributes) writes them; nf = n_keys + 1 + fields <= 32 (3 fields
 * per VARIANCE, 1 per other buffer).  They come
 * in the composite-key order of (grouping columns ascending, nulls first; gid) and are partitioned by
 * pmod(Murmur3Hash(grouping columns, gid; 42), num_partitions).
 * Defining contract: dst_off / dst_len / checksum_out / status, *dst_total, *n_groups and the return value are byte for
 * byte what b2s_aggregate_partition_compress_rows_hash_packed returns for the materialized Expand output in row-major
 * order, keyed by the n_keys grouping columns (each with a real null bit) and gid (B2S_KEY_INT64, null bit -1), with the
 * same aggregates at their projected slots.
 * Errors, B2S_E_ARG, checked before the device: what b2s_aggregate_partition_compress_rows_hash_* rejects; n_keys outside
 * 1..15 (gid takes the 16th key column); n_sets == 0 or a NULL set_mask; a mask bit at or above n_keys; two equal masks
 * (Spark adds a _gen_grouping_pos column for duplicate sets); n_records * n_sets >= 2^32; n_keys + 1 + fields above 32
 * (only VARIANCE buffers can pass it).  The empty set (mask 0, the grand total) and a single full set are allowed.  A bad record -> B2S_E_ARG
 * naming its input index, for the reasons b2s_aggregate_partition_compress_rows_hash_* gives.  A record whose row,
 * projected for a set (its in-set strings, 16 bytes per decimal(p > 18) key or input, 8 (2 + nf') bytes of fixed region),
 * would pass 2^31 - 1 bytes -> B2S_E_UNSUPPORTED.  Device memory that cannot be had -> B2S_E_NOMEM (the caller keeps
 * Spark's Expand and partial aggregation).  No usable device -> B2S_E_CUDA.
 * Sizing: dst_cap below the arena -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes needed.  The bound of
 * b2s_aggregate_partition_compress_rows_hash_* with n_records and rec_bytes multiplied by n_sets and nf as above,
 *   b2s_partition_compress_bound(codec, codec_block_size, num_partitions,
 *                                n_sets * (n_records * (4 + 8 (1 + nf) + 16 W + 8 S) + S * rec_bytes))
 * always suffices.
 * Runs on the write lane.  b2s_last_timing: kernel_ms the whole call's device work, dominant_ms / dominant_launches the
 * aggregation step, the expansion included. */
int b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed(
    uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len, uint32_t n_keys,
    const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
    uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type, const uint32_t* val_off,
    const int32_t* val_null_field, uint32_t n_sets, const uint32_t* set_mask, uint8_t* dst_base, uint64_t dst_cap,
    uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status,
    uint64_t* n_groups);
/* same, with rec_base / rec_len / dst_base in device memory of dev_index; the other arrays stay host arrays */
int b2s_aggregate_grouping_sets_partition_compress_rows_hash_dev(
    uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
    uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
    uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
    const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, uint32_t n_sets, const uint32_t* set_mask,
    uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
    uint64_t* checksum_out, int32_t* status, uint64_t* n_groups);

/* ---- read + write, one DISTINCT group: Spark's PartialMerge and Partial aggregates between two exchanges on the GPU ----
 * The middle stage of an aggregate with one DISTINCT group (AggUtils.planAggregateWithOneDistinct, Spark 3.5): on the
 * reducer of the exchange by G ++ X, HashAggregate(G ++ X, F: PartialMerge) then HashAggregate(G, F: PartialMerge, D:
 * Partial), then the exchange by G, in one call per reduce task.  G are the grouping columns, X the distinct columns, F
 * the non-distinct functions and D the distinct ones.  The map side is b2s_aggregate_partition_compress_rows_hash_*
 * with key columns G ++ X and functions F; the final merge of this call's output is b2s_decompress_aggregate_rows_keys_*
 * keyed by G with the merge ops of F's and D's buffers.
 * Read side: codec, checksum_alg, the n fetched blocks (src_off / src_len, slices and checksums) and the per-block
 * status[n] / bad_slice[n] exactly as b2s_decompress_aggregate_rows_keys_*.
 * Input rows: the map side's partial rows for key columns G ++ X and functions F: one null word (n_keys + F's fields
 * <= 32), key column c at slot 8 + 8 c with null bit c, then F's buffer fields in function order (1 per buffer, 3 per
 * VARIANCE).  n_keys (1..16) key columns, the first n_group_keys (0..15) G and at least one X; key_type[c] / key_len[c]
 * as the composite-key calls take them, no order flags (a G column of B2S_KEY_BYTES is a 1-byte boolean).  F:
 * (agg_fn[a], val_type[a]), a < n_aggs, exactly as the map side took them (its rules apply); the call derives every
 * buffer's slot, merge and initial value from them.
 * D: (distinct_fn[a], distinct_val_type[a], distinct_column[a]), a < n_distinct (1..16): COUNT, SUM, AVG or VARIANCE
 * with the map side's val_type rules (decimal SUM p <= 28, AVG p <= 27, VARIANCE not decimal), over distinct column
 * distinct_column[a] (in [n_group_keys, n_keys)), whose key type must agree with val_type: INT8 .. INT64 with
 * VAL_INT8 .. VAL_INT64, INT64 also with VAL_DECIMAL p <= 18, FLOAT32 / FLOAT64 with VAL_FLOAT32 / VAL_FLOAT64,
 * B2S_DECIMAL_KEY with VAL_DECIMAL p > 18, string, binary and boolean with COUNT and VAL_BYTES only.  Or
 * distinct_column[a] = B2S_DISTINCT_ALL_COLUMNS with COUNT and VAL_NONE: count(DISTINCT every distinct column), which
 * counts the (G, X) groups in which no distinct column is null (Spark's Count of several children).  One DISTINCT
 * group means every distinct function's children are all of X, so with several distinct columns only
 * B2S_DISTINCT_ALL_COLUMNS is accepted (a function over one of them would fold a value once per (G, X) row, not once
 * per distinct value).  MIN / MAX are B2S_E_ARG: Spark's optimizer removes their DISTINCT.
 * Semantics (Spark 3.5, ANSI off), in the order this contract fixes (Spark's own is its hash maps' iteration order):
 *   stage 2: the rows are sorted and grouped by G ++ X, and F's buffers merged per (G, X) group in stable (block)
 *            order, byte for byte as b2s_decompress_aggregate_rows_keys_* merges them;
 *   stage 3: the merged (G, X) rows in that order; for each G group, in ascending X order, F's buffers merged by
 *            mergeExpressions from their initial values (a decimal sum is null once an input sum is null, which is an
 *            overflow, or the running sum reaches 10^P; isEmpty is the AND; a variance is merged by CentralMomentAgg's
 *            mergeExpressions) and D's buffers updated by updateExpressions over the column's value in each (G, X) row.
 *            Double chains are one rounded add, or one rounded central-moment step, at a time, no FMA.
 * Output rows: what b2s_aggregate_partition_compress_rows_hash_* writes for key columns G and functions F ++ D
 * (UnsafeProjection(G ++ F's buffers ++ D's buffers)), key values from the G group's first row, in the composite-key
 * order of G, partitioned stably by pmod(Murmur3Hash(G, 42), num_partitions) and compressed with codec, level,
 * codec_block_size and checksum_alg.  n_group_keys == 0 is SinglePartition: num_partitions must be 1, and the call
 * writes exactly one row, the initial buffers (Sum null, Count 0, Avg 0 and 0, decimal Sum 0 and isEmpty true, Variance
 * (0, 0, 0)) when the task has no rows (HashAggregateExec's outputForEmptyGroupingKeyWithoutInput).
 * Defining contract: dst_off / dst_len / checksum_out (may be NULL) / part_status (per output partition), *dst_total and
 * the return value are byte for byte what b2s_partition_compress_rows_hash_packed returns for those rows in that order,
 * keyed by G at its output slots (8 + 8 c, null bit c); without G, what b2s_partition_compress_packed returns with one
 * partition and every id 0.  counts[3] (required): the input rows, the (G, X) groups, the rows written.
 * A corrupt or mis-framed block: as in the aggregated read, its status is set, nothing is written, every partition's
 * outputs are 0 and the call returns 0.  dst_cap below the arena -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes
 * needed (the caller cannot bound the output before decoding: retry once with that).
 * Errors, B2S_E_ARG, checked before the device: every rule above (a single-column distinct function with more than
 * one distinct column included); n_keys + F's fields above 32; more than 16 buffers in
 * the input (F) or the output (F ++ D; a VARIANCE is one); n_group_keys + the output's fields above 32; n_distinct 0;
 * the aggregated read's checks on the blocks and slices; the partition call's on codec, codec_block_size,
 * num_partitions and the output arrays.  Device memory that cannot be had -> B2S_E_NOMEM; no usable device ->
 * B2S_E_CUDA.
 * Runs on the read lane's slot 0, as the aggregated read does (one lock, one stream).  b2s_last_timing: kernel_ms the
 * whole call's device work, dominant_ms / dominant_launches stage 3 (from the merged (G, X) rows to the written rows). */
#define B2S_DISTINCT_ALL_COLUMNS (-1)
int b2s_decompress_aggregate_distinct_partition_compress_rows_hash_packed(
    uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t n,
    const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
    const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_group_keys, uint32_t n_keys,
    const uint32_t* key_type, const uint32_t* key_len, uint32_t n_aggs, const uint32_t* agg_fn,
    const uint32_t* val_type, uint32_t n_distinct, const uint32_t* distinct_fn, const uint32_t* distinct_val_type,
    const int32_t* distinct_column, uint32_t num_partitions, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
    uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* part_status, uint64_t* counts,
    int32_t* status, int32_t* bad_slice);
/* same, with src_base and dst_base in device memory of dev_index; the other arrays stay host arrays */
int b2s_decompress_aggregate_distinct_partition_compress_rows_hash_dev(
    uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t n,
    const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
    const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_group_keys, uint32_t n_keys,
    const uint32_t* key_type, const uint32_t* key_len, uint32_t n_aggs, const uint32_t* agg_fn,
    const uint32_t* val_type, uint32_t n_distinct, const uint32_t* distinct_fn, const uint32_t* distinct_val_type,
    const int32_t* distinct_column, uint32_t num_partitions, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
    uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* part_status, uint64_t* counts,
    int32_t* status, int32_t* bad_slice);

/* ---- write side, window group limit: Spark's Sort and WindowGroupLimitExec(Partial) and its exchange on the GPU ----
 * The map side of a top-N-per-group window's shuffle (Sort(pk ++ ord, global = false) -> WindowGroupLimitExec(pk, ord,
 * rank_fn, limit, Partial) -> Exchange hashpartitioning(pk) | SinglePartition) in one call.  A reducer finishes it with
 * b2s_decompress_window_rows_keys_* and the same limit (WindowGroupLimitExec(Final) and the window).
 * Records: as for b2s_partition_compress_rows_hash_*: [size: int32 big-endian][row], rec_len[i] = 4 + size.
 * Key columns: as for b2s_decompress_window_rows_keys_*: n_keys (1..16) composite-key columns, the first
 * n_partition_keys (0..15) the PARTITION BY columns, with the hash call's types (B2S_KEY_BYTES only as a 1-byte boolean)
 * and no order flag; the rest, at least one, the ORDER BY columns, of any composite-key type and any order flags.
 * Sort: the records are sorted stably by the whole key exactly as b2s_decompress_sort_rows_keys_* sorts them, ties in
 * input order (the local SortExec in front of the Partial limit).
 * Limit: partitions and peers follow the window call's rules (nulls equal nulls, 0.0 equals -0.0, NaN equals NaN).
 * limit_fn is B2S_WINDOW_ROW_NUMBER, B2S_WINDOW_RANK or B2S_WINDOW_DENSE_RANK and limit at least 1; a record is kept
 * when its limit_fn value within its partition is at most limit, so every rank tie at the boundary is kept and
 * ROW_NUMBER cuts ties in input order.
 * Outputs: the kept records, unchanged and in sorted order, partitioned stably by pmod(Murmur3Hash(partition columns,
 * 42), num_partitions) and compressed.  n_partition_keys == 0 is Spark's SinglePartition exchange: num_partitions must
 * be 1 and every kept record goes to partition 0.  *n_out_records (required) = the kept records.
 * Defining contract: dst_off / dst_len / checksum_out / status, *dst_total and the return value are byte for byte what
 * b2s_partition_compress_rows_hash_packed returns for the kept records in sorted order, keyed by the partition columns
 * at their input slots and null bits; without partition columns, what b2s_partition_compress_packed returns for them
 * with num_partitions 1 and every id 0.
 * Sizing: the kept records never outgrow the input, so an arena of
 *   b2s_partition_compress_bound(codec, codec_block_size, num_partitions, rec_bytes)
 * always suffices; dst_cap below the arena -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes needed, as the partition
 * calls.
 * Errors, B2S_E_ARG, checked before the device: what the hash call rejects for the partition columns; what the window
 * call rejects for the key (n_keys outside 1..16, a type not listed, a key_len that does not match its type, an order
 * flag on a partition column, n_partition_keys above 15 or leaving no ORDER BY column); limit_fn not one of the three or
 * limit < 1; n_partition_keys == 0 with num_partitions != 1; n_records >= 2^32; a NULL n_out_records.  A bad record ->
 * B2S_E_ARG, nothing reported as written, b2s_last_error() names the lowest bad record and why, by the hash call's
 * record checks applied to every key column.  A partition of more than 2^31 - 1 records -> B2S_E_UNSUPPORTED, as in the
 * window call.  Device memory that cannot be had -> B2S_E_NOMEM (the caller keeps Spark's Sort and partial limit).  No
 * usable device -> B2S_E_CUDA.
 * Runs on the write lane.  b2s_last_timing: kernel_ms the whole call's device work, dominant_ms / dominant_launches the
 * limit step (from the input records to the gathered kept records, the sort included).  No exchange-cache form. */
int b2s_window_limit_partition_compress_rows_hash_packed(
    uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t limit_fn, int32_t limit, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out,
    int32_t* status, uint64_t* n_out_records);
/* same, with rec_base / rec_len / dst_base in device memory of dev_index; the other arrays stay host arrays */
int b2s_window_limit_partition_compress_rows_hash_dev(
    uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
    uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t limit_fn, int32_t limit, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out,
    int32_t* status, uint64_t* n_out_records);

/* ---- write side, range-partitioned rows: Spark's RangePartitioner ids computed on the GPU ----
 * b2s_partition_compress_* for a RangePartitioning exchange of UnsafeRows (a global ORDER BY's map side): the reduce id
 * of every record is what Spark's RangePartitioner.getPartition returns for its sort key over the n_bounds range
 * bounds, so the caller passes no rec_part, and num_partitions = n_bounds + 1 (dst_off / dst_len / checksum_out /
 * status have that many entries).  The id is the number of bounds strictly below the record's key (with strictly
 * increasing bounds both of getPartition's branches, the linear scan and the binary search, return it): a key equal
 * to bound p goes to partition p.  Records are framed as for the hash call ([size: int32 big-endian][row], rec_len[i] =
 * 4 + size).  The key columns are given as to the composite-key calls, order flags included (B2S_KEY_DESCENDING,
 * B2S_KEY_NULLS_LAST), and compared in Spark SQL's order: -0.0 equals 0.0, NaN equals NaN and sorts above +inf,
 * strings and binary as unsigned bytes, decimals by value, a null string is not an empty one.
 * Bounds: n_bounds (0..2^24 - 1) rows framed the same way, back to back in bound_base (bound_bytes, bound_len[j] each),
 * as Spark holds them: UnsafeProjection(sort order children) rows, so key column c is field c of a bound row (its slot
 * at 8 * ceil(n_keys / 64) + 8 c, its null bit c when key_null_field[c] >= 0, else never null; type, flags and key_len
 * those of the records' column c).  The bound arrays are host memory in both forms; they are uploaded once per call.
 * n_bounds = 0 sends every record to partition 0; n_records = 0 is valid.
 * Outputs: byte for byte what b2s_partition_compress_packed / _dev return for the same records and those ids.
 * Errors, B2S_E_ARG, nothing reported as written, b2s_last_error() says why: what the hash call rejects, except that
 * order flags and B2S_KEY_BYTES of key_len 1..16 are allowed; n_bounds above 2^24 - 1; a null bound array with n_bounds
 * > 0; bound_len not summing to bound_bytes; a bad bound (bound_len < 4, a size prefix other than bound_len - 4, a row
 * that does not hold a key slot or null word, a string past its row, a bad decimal) or a bound whose key is not above
 * the one before it (equal ones included, such as -0.0 after 0.0, two NaNs or two nulls): the lowest such bound is named;
 * a bad record, as for the hash call.  A bad bound is named before a bad record.  No usable device -> B2S_E_CUDA.
 * b2s_last_timing as for the partition calls, plus dominant_ms / dominant_launches = the range step (the bound checks
 * and the id kernel).  Exchange-cache form: b2s_partition_compress_rows_range_cached_packed (below). */
int b2s_partition_compress_rows_range_packed(uint32_t codec, int32_t level, uint32_t codec_block_size,
                                             uint32_t checksum_alg, uint64_t n_records, const uint8_t* rec_base,
                                             uint64_t rec_bytes, const uint32_t* rec_len, uint32_t n_keys,
                                             const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                             const int32_t* key_null_field, uint32_t n_bounds,
                                             const uint8_t* bound_base, uint64_t bound_bytes,
                                             const uint32_t* bound_len, uint8_t* dst_base, uint64_t dst_cap,
                                             uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                             uint64_t* checksum_out, int32_t* status);
/* same, with rec_base / rec_len / dst_base in device memory of dev_index (the bound arrays stay in host memory) */
int b2s_partition_compress_rows_range_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                                          uint32_t checksum_alg, uint64_t n_records, const uint8_t* rec_base,
                                          uint64_t rec_bytes, const uint32_t* rec_len, uint32_t n_keys,
                                          const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                          const int32_t* key_null_field, uint32_t n_bounds, const uint8_t* bound_base,
                                          uint64_t bound_bytes, const uint32_t* bound_len, uint8_t* dst_base,
                                          uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                          uint64_t* checksum_out, int32_t* status);

/* ---- write side, round-robin-partitioned rows: Spark's repartition(n) order and ids computed on the GPU ----
 * b2s_partition_compress_* for a RoundRobinPartitioning exchange of UnsafeRows (Dataset.repartition(n) without
 * columns, the REPARTITION(n) hint): the caller passes no rec_part.  Records are framed as for the hash call ([size:
 * int32 big-endian][row], rec_len[i] = 4 + size).  start_position is Spark's position before the task's first row,
 * new XORShiftRandom(partitionId).nextInt(num_partitions), computed by the caller.  sort_rows (0 or 1) is
 * spark.sql.execution.sortBeforeRepartition: with num_partitions > 1 the rows are first sorted as Spark's
 * UnsafeExternalRowSorter does, by row.hashCode() (Murmur3 hashUnsafeWords of the row, seed 42) as a signed int, then
 * by RecordBinaryComparator (the shorter row first, then unsigned bytes); rows tied on both are identical, so the order
 * is unique.  With num_partitions == 1, or sort_rows == 0, the rows stay in input order.  The k-th row of that order
 * (0-based) goes to partition (start_position + 1 + k) mod num_partitions.
 * Outputs: byte for byte what b2s_partition_compress_packed / _dev return for the records in that order with those ids.
 * Errors, B2S_E_ARG, nothing reported as written, b2s_last_error() says why: what b2s_partition_compress_* rejects;
 * start_position outside [0, num_partitions); sort_rows above 1; start_position + n_records above 2^31 - 1 (Spark's
 * position would wrap: keep such a task on the CPU path); a bad record (rec_len < 4, a size prefix other than rec_len -
 * 4, a row size that is not a multiple of 8), the lowest one named, in both modes.  No usable device -> B2S_E_CUDA.
 * b2s_last_timing as for the partition calls, plus dominant_ms / dominant_launches = the round-robin step (the checks
 * and hash, the sort with its refinement rounds, the ids).  Exchange-cache form:
 * b2s_partition_compress_rows_round_robin_cached_packed (below). */
int b2s_partition_compress_rows_round_robin_packed(uint32_t codec, int32_t level, uint32_t codec_block_size,
                                                   uint32_t checksum_alg, uint32_t num_partitions,
                                                   int32_t start_position, uint32_t sort_rows, uint64_t n_records,
                                                   const uint8_t* rec_base, uint64_t rec_bytes,
                                                   const uint32_t* rec_len, uint8_t* dst_base, uint64_t dst_cap,
                                                   uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                                   uint64_t* checksum_out, int32_t* status);
/* same, with rec_base / rec_len / dst_base in device memory of dev_index */
int b2s_partition_compress_rows_round_robin_dev(uint32_t dev_index, uint32_t codec, int32_t level,
                                                uint32_t codec_block_size, uint32_t checksum_alg,
                                                uint32_t num_partitions, int32_t start_position, uint32_t sort_rows,
                                                uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes,
                                                const uint32_t* rec_len, uint8_t* dst_base, uint64_t dst_cap,
                                                uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                                uint64_t* checksum_out, int32_t* status);

/* ---- read side ---- */
/* n compressed blocks as produced by S3BufferedPrefetchIterator.next() (storage/S3BufferedPrefetchIterator.scala:196-212).
 * Block i covers n_slices[i] consecutive reduce partitions (1 for ShuffleBlockId, >1 for ShuffleBlockBatchId,
 * storage/S3ChecksumValidationStream.scala:22-27); slice_len[i][k] / slice_checksum[i][k] are the .index differences and
 * .checksum values of those partitions.  With checksum_alg != 0 every slice is verified over the compressed bytes
 * before decoding; a mismatch yields status[i] = B2S_E_CHECKSUM and bad_slice[i] = k (may be NULL).
 * n_slices / slice_* may be NULL when checksum_alg == 0.
 * A block whose status is not B2S_OK leaves the bytes of its own output range unspecified (the decoder may have
 * written part of it before it met the corruption); the output ranges of the other blocks are never touched by it.
 * Verdicts are per block: B2S_E_CORRUPT for a stream that breaks its codec's format, and B2S_E_UNSUPPORTED for a
 * well-formed stream this decoder does not take: a Zstandard frame with a Dictionary_ID, or a Snappy chunk of more
 * than 65536 decoded bytes or of 65536 compressed bytes or more (snappy-java's blockSize above 64 KiB).  A Snappy
 * chunk that claims more than 64 decoded bytes per 3 compressed bytes (more than any element sequence yields) is
 * B2S_E_CORRUPT.  Neither claim counts towards any decoded length or size: the call, and the other blocks, go on. */
int b2s_decompress_batch(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* const* src,
                         const uint64_t* src_len, const uint32_t* n_slices, const uint64_t* const* slice_len,
                         const uint64_t* const* slice_checksum, uint8_t* const* dst, const uint64_t* dst_cap,
                         uint64_t* dst_len, int32_t* status, int32_t* bad_slice);
/* packed: slices are flattened — block i owns slice_len[slice_base[i] .. slice_base[i+1]) */
int b2s_decompress_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                          const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                          const uint64_t* slice_len, const uint64_t* slice_checksum, uint8_t* dst_base,
                          uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                          int32_t* status, int32_t* bad_slice);

/* ---- read side, key-sorted: verify + decompress + sort a reduce task's records in one call ----
 * Replaces, for a shuffle with a key ordering and no aggregator (sortByKey, repartitionAndSortWithinPartitions,
 * TeraSort), the ExternalSorter that storage/S3ShuffleReader.scala:141-149 feeds with the decoded records.  The n blocks
 * are the task's fetched blocks, with the slice and checksum arguments of b2s_decompress_packed; slices are verified
 * before decoding.  Every decoded record is record_bytes long (a fixed-size serialized record, e.g. TeraSort's Kryo
 * record: 104 bytes, key at 2, 10 bytes), and its key is bytes [key_off, key_off + key_len), compared as unsigned bytes,
 * lexicographically, ascending.
 * Output: the arena holds every record of every block exactly once, sorted by key; the sort is stable (equal keys keep
 * block order, then their order within the block), so with a relocatable serializer the arena is again a valid
 * serialized stream.  *dst_total = sum of the decoded lengths, *n_records = record count.  codec B2S_CODEC_NONE
 * verifies and sorts only (spark.shuffle.compress=false).
 * Per block: a corrupt stream, or a decoded length that is not a multiple of record_bytes (b2s_last_error() names the
 * block), sets status[i] = B2S_E_CORRUPT; a checksum mismatch sets B2S_E_CHECKSUM and bad_slice[i] (may be NULL).  When
 * a block fails, nothing is sorted, *n_records = *dst_total = 0 and the call returns 0; blocks whose slices fail
 * verification are not decoded.
 * Errors: key_len outside [1, 16], key_off + key_len > record_bytes, record_bytes == 0 or more than 2^32 - 1 records ->
 * B2S_E_ARG; dst_cap below the decoded bytes -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes needed; device memory
 * for the whole task (compressed blocks, decoded records, sorted copy, sort workspace) that cannot be had -> B2S_E_NOMEM,
 * and the caller keeps its CPU sorter.  Runs on the read lane without chunking — the whole task is resident at once —
 * and fills b2s_last_timing (top_kernel_ms = the sort step).  The device buffers of the task stay allocated for the
 * next call up to 1 GiB each; larger ones are freed when the call returns. */
int b2s_decompress_sort_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                               const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                               const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t record_bytes,
                               uint32_t key_off, uint32_t key_len, uint8_t* dst_base, uint64_t dst_cap,
                               uint64_t* dst_total, uint64_t* n_records, int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; the descriptor arrays stay host arrays */
int b2s_decompress_sort_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                            const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                            const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                            uint32_t record_bytes, uint32_t key_off, uint32_t key_len, uint8_t* dst_base,
                            uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                            int32_t* bad_slice);

/* ---- read side, row-sorted: verify + decompress + sort a reduce task's UnsafeRow records by one typed key ----
 * The Spark SQL counterpart of b2s_decompress_sort_*: the SortExec that a sort-merge join runs on every reducer right
 * after the shuffle read.  Blocks, slices and checksums are those of b2s_decompress_sort_packed.  A decoded block is a
 * sequence of records as UnsafeRowSerializer writes them: [s: int32 big-endian][s bytes of row], s >= 0, no end
 * marker (the last record ends exactly at the block's decoded end).  A block of several concatenated streams
 * (ShuffleBlockBatchId) is still a whole number of records; an empty block holds none.
 * Key (offsets count from the start of the row, after the 4-byte size):
 *   B2S_KEY_BYTES: key_len (1..16) bytes at key_off, unsigned, lexicographic (the fixed-size call's meaning)
 *   B2S_KEY_INT32: 4 bytes at key_off (key_len 4), little-endian two's complement, ordered as signed
 *   B2S_KEY_INT64: the same with 8 bytes (key_len 8)
 * Nulls: null_field = -1 means the key has no null bit.  With null_field >= 0 a record is null when bit
 * (null_field & 63) of the little-endian u64 at row offset 8 * (null_field >> 6) is set (UnsafeRow's null bitset);
 * null records sort before every other record (ASC NULLS FIRST) and their key bytes are ignored.
 * Output: every record, size prefix included, back to back in ascending key order — again a valid UnsafeRowSerializer
 * stream.  The sort is stable: equal keys, and nulls among themselves, keep block order, then their order within the
 * block.  *dst_total = decoded bytes, *n_records = record count.
 * Per block, B2S_E_CORRUPT (b2s_last_error() names the block and the byte offset of its first bad record) when a size is
 * negative, a record runs past the block end, the block ends inside a size prefix, a row is shorter than key_off +
 * key_len, or (null_field >= 0) a row does not hold the null-bit word.  Checksums, B2S_E_DST_TOO_SMALL, B2S_E_NOMEM,
 * "nothing is sorted when a block fails", codec NONE, the read lane and the 1 GiB buffer trim are as in
 * b2s_decompress_sort_*.
 * Errors -> B2S_E_ARG: an unknown key_type; key_len outside [1, 16] for BYTES, other than 4 / 8 for INT32 / INT64;
 * null_field < -1; more than 2^32 - 1 records.
 * Timing (b2s_last_timing): kernel_ms = verification + decode + framing + sort; top_kernel_ms = framing + sort (from
 * the end of decoding, including the one readback that sizes the sort: the record count and the per-block framing
 * verdicts); dominant_ms / dominant_launches = the framing step alone. */
int b2s_decompress_sort_rows_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                                    const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t key_type,
                                    uint32_t key_off, uint32_t key_len, int32_t null_field, uint8_t* dst_base,
                                    uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                                    int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; the descriptor arrays stay host arrays */
int b2s_decompress_sort_rows_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                 const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                 const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                                 uint32_t key_type, uint32_t key_off, uint32_t key_len, int32_t null_field,
                                 uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                                 int32_t* status, int32_t* bad_slice);

/* ---- read side, aggregated: verify + decompress + group a reduce task's UnsafeRow records by key and merge ----
 * The HashAggregateExec(Final) that a grouped aggregation runs on every reducer right after the shuffle read: the rows
 * are the partial aggregates of the map side, one per map per key, and the call merges them into one row per key.
 * Blocks, slices, checksums, key_type, key_off, key_len and null_field mean exactly what they mean in
 * b2s_decompress_sort_rows_packed.  A group is a maximal set of records with equal keys; all null keys form one group.
 * Aggregates: n_aggs (0..16) of them; aggregate a reads the 8-byte little-endian slot at row offset agg_off[a] with
 * op agg_op[a] and null bit agg_null_field[a] (-1: never null; else as null_field).  An aggregate is taken over the
 * group's non-null inputs, in stable order (block order, then order within the block), as one HashAggregateExec
 * buffer merges them:
 *   B2S_AGG_SUM_INT64   : 64-bit wrapping sum (non-ANSI Add)
 *   B2S_AGG_SUM_FLOAT64 : ((0.0 + x1) + x2) + ... in double, left to right, no reassociation, no FMA — bit for bit
 *                         coalesce(coalesce(sum.left, 0) + sum.right, sum.left); a lone -0.0 gives +0.0
 *   B2S_AGG_MIN/MAX_INT32   : signed, on the low 4 bytes of the slot; written with the high 4 bytes zero
 *   B2S_AGG_MIN/MAX_INT64   : signed
 *   B2S_AGG_MIN/MAX_FLOAT64 : Spark SQL's double order: -0.0 == 0.0, NaN == NaN and above every other value; among
 *                             equal values the first in stable order is kept with its exact bits (Least / Greatest)
 * A group with no non-null input for aggregate a gets its null bit set and an all-zero slot (UnsafeRow.setNullAt);
 * otherwise the null bit is cleared and the slot holds the result.  n_aggs = 0 keeps the first row of every key.
 * The Decimal ops:
 *   B2S_AGG_SUM_DECIMAL | P << 8 : Spark's Sum / Average decimal merge into an UnsafeRow buffer (Sum.mergeExpressions
 *       with DecimalAddNoOverflowCheck, Average's sum.left + sum.right, each result written by UnsafeRow.setDecimal(...,
 *       P), whose changePrecision(P) turns an overflow into null).  Over the group's records in stable order, starting
 *       from 0, the result is null when some input is null (a decimal sum buffer is null only after an overflow; its
 *       initial value is 0) or some running sum S_k has |S_k| >= 10^P; the null sticks, later inputs do not clear it.
 *       Otherwise it is the exact sum.  Unlike the other ops it propagates nulls, so it needs agg_null_field[a] >= 0.
 *   B2S_AGG_MIN/MAX_DECIMAL : the signed minimum / maximum of the non-null inputs; null when there is none.
 *   A result is written as UnsafeRow.setDecimal writes it.  P <= 18: the long, or an all-zero slot when null.  Out of
 *   line (P > 18, and MIN / MAX_DECIMAL): the 16 bytes at the head row's offset are zeroed; a non-null result's minimal
 *   two's-complement bytes (BigInteger.toByteArray: bitlen(x >= 0 ? x : ~x) / 8 + 1 of them, so 0 is 00, 128 is
 *   00 80, -128 is 80) go there and the slot becomes (offset << 32) | length; a null result leaves the slot
 *   offset << 32 ("keep the offset for future update") with the null bit set.
 *   Spark's buffers map to them so (the final If(isEmpty, null, sum), overflow check or ANSI error stay on the CPU):
 *     Sum(decimal) [sum, isEmpty]     : SUM_DECIMAL | P << 8 on sum, MIN_INT32 on isEmpty (a BooleanType slot is byte 0
 *                                       with bytes 1..7 zero, so the minimum is the AND Spark merges with)
 *     Average(decimal) [sum, count]   : SUM_DECIMAL | P << 8, SUM_INT64
 *     Min / Max(decimal p > 18)       : MIN / MAX_DECIMAL
 *     CentralMomentAgg [n, avg, m2]   : B2S_AGG_VARIANCE at n's slot, agg_null_field -1 (stddev_* / var_*)
 *   B2S_AGG_VARIANCE : one entry over three consecutive double slots (agg_off, + 8, + 16), merged by mergeExpressions
 *       from (0, 0, 0) over every record of the group in stable order (see its define); never null, so no null bit
 *       is written.  Its 24 bytes count in every overlap check and in the row length a record must have.
 * Output: one record per group, back to back, groups in the row sort's order (ascending, nulls first) — again a valid
 * UnsafeRowSerializer stream.  A group's record is its first record in stable order, byte for byte (size prefix and
 * variable-length region included) except each aggregate's slot and null bit.  *dst_total = output bytes, *n_records =
 * input records, *n_groups = output records.  The output is never longer than the decoded input, so a dst_cap of at
 * least the decoded bytes never gets B2S_E_DST_TOO_SMALL.
 * Per block, B2S_E_CORRUPT for every framing rule of b2s_decompress_sort_rows_packed and when a row is shorter than an
 * aggregate slot (agg_off[a] + 8) or an aggregate's null word.  With an out-of-line Decimal aggregate also, for the
 * block of the first bad record: a non-null input whose size is not 1..16 or whose bytes run past its row; a record
 * whose 16-byte region [offset, offset + 16) is not inside its row (any record can be a group's head), or starts
 * before the end of a key or aggregate slot or a null word the call uses.  The region is not checked against a string
 * or decimal key's out-of-line bytes or another decimal's region: Spark gives each its own bytes, and a row that
 * shares them gets a merged decimal written over them.  Checksums, "nothing is written when a block fails"
 * (*n_records = *n_groups = 0, the call returns 0), B2S_E_NOMEM, codec NONE, the read lane and the 1 GiB buffer trim
 * are as in b2s_decompress_sort_*.  dst_cap below the output bytes -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes
 * needed.
 * Errors -> B2S_E_ARG: those of b2s_decompress_sort_rows_packed; n_aggs > 16; an unknown op; precision bits on any op
 * but SUM_DECIMAL, or a SUM_DECIMAL precision of 0 or above 38; SUM_DECIMAL with agg_null_field[a] = -1; VARIANCE with
 * agg_null_field[a] >= 0;
 * agg_null_field[a] < -1;
 * NULL agg arrays with n_aggs > 0; an aggregate slot that overlaps another slot, the key bytes, or an 8-byte null word
 * that the key or an aggregate uses.
 * Timing (b2s_last_timing): kernel_ms = the whole call; top_kernel_ms = framing + keys + radix + aggregation;
 * dominant_ms / dominant_launches = the aggregation step alone, from the sorted indices to the written output. */
int b2s_decompress_aggregate_rows_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                         const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                                         const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t key_type,
                                         uint32_t key_off, uint32_t key_len, int32_t null_field, uint32_t n_aggs,
                                         const uint32_t* agg_op, const uint32_t* agg_off, const int32_t* agg_null_field,
                                         uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                                         uint64_t* n_groups, int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; the descriptor and aggregate arrays stay host arrays */
int b2s_decompress_aggregate_rows_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                      const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                      const uint32_t* slice_base, const uint64_t* slice_len,
                                      const uint64_t* slice_checksum, uint32_t key_type, uint32_t key_off,
                                      uint32_t key_len, int32_t null_field, uint32_t n_aggs, const uint32_t* agg_op,
                                      const uint32_t* agg_off, const int32_t* agg_null_field, uint8_t* dst_base,
                                      uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_groups,
                                      int32_t* status, int32_t* bad_slice);

/* ---- read side, composite key: the row sort and the row aggregation by several key columns, strings included ----
 * b2s_decompress_sort_rows_* and b2s_decompress_aggregate_rows_* with a key of n_keys (1..16) columns, given as
 * parallel arrays: column c is key_type[c] at row offset key_off[c], key_len[c] bytes, null bit key_null_field[c].
 * Columns compare left to right; each is read exactly as the single-key calls read their key (B2S_KEY_BYTES,
 * B2S_KEY_INT32, B2S_KEY_INT64: the same key_len rules), and a null sorts first within its column (-1: never null).
 * These calls only:
 *   B2S_STRING_KEY: key_len 8, the slot of a variable-length value; a null string and an empty string are different
 *   B2S_KEY_INT16 / B2S_KEY_INT8: key_len 2 / 1, signed; BooleanType is B2S_KEY_BYTES with key_len 1
 *   B2S_KEY_FLOAT32 / B2S_KEY_FLOAT64: key_len 4 / 8, Spark SQL's order (SQLOrderingUtil.compareDoubles): -0.0 == 0.0,
 *     every NaN equals every other NaN and sorts above +inf
 *   B2S_DECIMAL_KEY: key_len 8, the slot of a Decimal(p > 18): size (1..16) bytes of the unscaled value, big-endian
 *     two's complement, compared as signed integers (one column has one scale, so this is value order); a null
 *     decimal's slot is not read
 *   order flags OR-ed into key_type[c]: B2S_KEY_DESCENDING reverses the order of the column's non-null values;
 *     B2S_KEY_NULLS_LAST puts its nulls after them (no effect with key_null_field[c] == -1).  Independent, as Spark's
 *     SortOrder direction and null ordering.
 * Two columns may share a slot or a null word.
 * Sort: every record, stably sorted by the composite key (per column: ascending, nulls first, unless flagged).
 * Aggregate: a group is a maximal run of records whose every column is equal (both null, or both non-null with equal
 * values; strings: equal length and bytes; floats: as compared, so 0.0 and -0.0 form one group and all NaNs one);
 * aggregates, output rows (each group's first record, its key bytes as they were), group order (the sort's) and
 * *n_groups are as in b2s_decompress_aggregate_rows_*.
 * With n_keys == 1, a fixed-width column of a single-key type and no flag the output is byte for byte that of the
 * single-key call.
 * Per block, B2S_E_CORRUPT for every framing rule of the single-key calls, applied with the largest key_off + key_len
 * and null word of all columns, when a non-null string's offset + size runs past the end of its row, and when a
 * non-null decimal's size is 0 or above 16 or its offset + size runs past the end of its row (b2s_last_error() names
 * the block and the byte offset of its first bad record).  When a block fails nothing is written: *n_records
 * (= *n_groups) = 0 and the call returns 0.
 * Errors -> B2S_E_ARG: n_keys outside [1, 16]; NULL key arrays; an unknown key_type or a key_type bit above the low 8
 * other than the two flags; a key_len its type does not allow; key_null_field[c] < -1; the aggregate checks of
 * b2s_decompress_aggregate_rows_* against every column (no aggregate slot overlaps any key slot, a string's or
 * decimal's 8-byte slot included, or a null word any column uses).  Checksums, codec NONE, B2S_E_DST_TOO_SMALL,
 * B2S_E_NOMEM, the read lane, the 1 GiB buffer trim and b2s_last_timing are as in the single-key calls.
 * The key is sorted by its first 20 encoded bytes (a column takes its value bytes — a decimal 16 — plus one for its
 * null bit; a string 9 per started 8 bytes of value, at least 9).  A key longer than that — any string column, or
 * fixed-width columns of more than 20 bytes — is refined in rounds of 16 more bytes over the records still tied, and
 * each round makes one small blocking readback (the count of tied records; the first round also brings the string and
 * decimal checks' verdicts).  A key with a decimal column always takes that first round, for its verdicts, even when
 * it fits in 20 bytes.  DESCENDING and NULLS_LAST change no widths: a flagged key costs what the unflagged one does. */
int b2s_decompress_sort_rows_keys_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                         const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                                         const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_keys,
                                         const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                         const int32_t* key_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                         uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                                         int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; the descriptor and key arrays stay host arrays */
int b2s_decompress_sort_rows_keys_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                      const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                      const uint32_t* slice_base, const uint64_t* slice_len,
                                      const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type,
                                      const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
                                      uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                                      int32_t* status, int32_t* bad_slice);
int b2s_decompress_aggregate_rows_keys_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                              const uint8_t* src_base, const uint64_t* src_off,
                                              const uint64_t* src_len, const uint32_t* slice_base,
                                              const uint64_t* slice_len, const uint64_t* slice_checksum,
                                              uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
                                              const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_aggs,
                                              const uint32_t* agg_op, const uint32_t* agg_off,
                                              const int32_t* agg_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                              uint64_t* dst_total, uint64_t* n_records, uint64_t* n_groups,
                                              int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; the descriptor, key and aggregate arrays stay host
 * arrays */
int b2s_decompress_aggregate_rows_keys_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                           const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                           const uint32_t* slice_base, const uint64_t* slice_len,
                                           const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type,
                                           const uint32_t* key_off, const uint32_t* key_len,
                                           const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_op,
                                           const uint32_t* agg_off, const int32_t* agg_null_field, uint8_t* dst_base,
                                           uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                                           uint64_t* n_groups, int32_t* status, int32_t* bad_slice);

/* ---- read side, sort-merge join: a reducer's two shuffled UnsafeRow inputs joined in one call ----
 * Spark SQL's SortMergeJoinExec on a reducer: both children's shuffle reads sorted by the join key and merged into
 * joined rows (UnsafeRowJoiner), for an equi-join without a further condition.
 * Sides.  Blocks [0, n_left) are the left (streamed) side's fetched blocks, blocks [n_left, n) the right (buffered)
 * side's.  Both sides share one codec and one checksum algorithm.  Blocks, slices, checksums and framing as in
 * b2s_decompress_sort_rows_packed: [size: int32 BE][row], no end marker.
 * Keys.  Column c has one key_type[c] and key_len[c] for both sides (Spark coerces join keys to one type) and its own
 * slot and null bit on each side: left_key_off[c] / left_key_null_field[c] and right_key_off[c] /
 * right_key_null_field[c] (-1: never null on that side).  Every type of the composite-key calls is accepted; the order
 * flags are not (the join orders ascending, nulls first).  Two keys are equal when every column is non-null on both
 * sides and the values are equal by the composite-key aggregation's grouping rule (strings by length and bytes, 0.0
 * equal to -0.0, every NaN equal to every other NaN: Spark's NormalizeFloatingNumbers).  A key with a null column
 * matches nothing.
 * Null-safe columns.  A column whose key_type has B2S_KEY_NULL_SAFE (l <=> r) compares and orders as the pair
 * (coalesce(v, default), isnull(v)), both ascending: a null equals a null and sorts directly after the non-null default
 * value, and it does not make the key unmatchable; only a null in a plain column does.  A side whose null field is -1
 * has isnull false.  Either side's pair form (Spark folds a non-nullable side's pair to (col, false)) is this one.
 * Order.  Ls: the left records stably sorted by the key (ascending, nulls first, ties in block order, then in their
 * order in the block); Rs: the right records sorted the same way.
 *   B2S_JOIN_INNER: for each l of Ls, for each r of Rs whose key equals l's, in Rs order: join(l, r).
 *   B2S_JOIN_LEFT_OUTER: the same; a left record without an equal right key (a null key included) gives join(l, null).
 *   B2S_JOIN_LEFT_SEMI: l itself, byte for byte, once, when it has a match.
 *   B2S_JOIN_LEFT_ANTI: l itself when it has no match, null keys included (NOT EXISTS; not the null-aware form).
 *   B2S_JOIN_RIGHT_OUTER: for each r of Rs, for each l of Ls whose key equals r's, in Ls order: join(l, r); a right
 *     record without an equal left key (a null key included) gives join(null, r).  SortMergeJoinExec's RightOuter
 *     order (the right side streamed, the left buffered), so its outputOrdering, the right keys, holds.
 *   B2S_JOIN_FULL_OUTER: by runs.  A run is a maximal set of records of both sides whose keys are equal in the sort
 *     order, nulls equal to nulls there; it matches when its key has no null column and it holds records of both sides
 *     (its records all have the same null columns).  Runs are taken in ascending key order, nulls first; within a run,
 *     first each left record l in Ls order: join(l, r) for each right record r of the run in Rs order if the run
 *     matches, else join(l, null); then, if the run does not match, each right record r in Rs order: join(null, r).
 *     Spark declares no outputOrdering for a full outer sort-merge join; this order makes the output deterministic,
 *     and without null keys it is the order of Spark's full outer scanner.  A run matches when its key has no null in a
 *     plain column and it holds records of both sides.
 *   B2S_JOIN_EXISTENCE: for each l of Ls, once: l joined with one non-null boolean field, 1 when l has a match, else 0
 *     (SortMergeJoinExec(ExistenceJoin(exists)), whose output is left.output :+ exists).  The row is the window call's
 *     output row with one value: b = ceil((nL + 1) / 64) null words holding the left's bits and zeros above them, the
 *     left slots, the boolean slot (8 bytes, 0 or 1), the left var bytes; every VAR or DECIMAL_WIDE slot that is not
 *     zero has its offset moved by 8 (b - bL + 1).  *n_out_records = the left record count.
 * Joined row: UnsafeRowJoiner's, which is UnsafeProjection(left.output ++ right.output) when each input's
 * variable-length data is laid out as UnsafeProjection writes it.  nL, nR: the sides' field counts (n_left_fields,
 * n_right_fields); bL, bR, b: the null-bitset words of the left row, the right row and the output, ceil(nL / 64),
 * ceil(nR / 64), ceil((nL + nR) / 64); varX = size(X) - 8 (bX + nX), side X's variable-length bytes.  The output is
 * [b words of null bits][left's 8 nL bytes of slots][right's 8 nR][left's var bytes][right's var bytes].  Null bit i
 * is left bit i for i < nL, right bit i - nL below nL + nR, zero past it.  Every VAR or DECIMAL_WIDE field whose slot
 * is not zero has its offset (the high 32 bits) moved by 8 (b - bL + nR) on the left, by 8 (b - bR + nL) + varL on
 * the right; a zero slot (a null string) stays zero, and a null wide decimal (offset << 32) is moved.
 * The null right side (left and full outer): every right null bit set, every right slot zero, except that each
 * DECIMAL_WIDE right field gets 16 zero bytes appended to the var bytes, in field order, and its slot is offset << 32
 * (what UnsafeRowWriter.write(i, (Decimal) null, p, s) writes).  The null left side (right and full outer) mirrors it:
 * every left null bit set, every left slot zero, and each DECIMAL_WIDE left field k (in field order) 16 zero bytes in
 * the left var bytes, its slot (8 (b + nL + nR) + 16 k) << 32; so varL = 16 * (the left DECIMAL_WIDE fields) and the
 * right side's offsets move by 8 (b - bR + nL) + varL as above.  A joined row never has both sides null.
 * Outputs.  [size BE][row] records, an UnsafeRowSerializer stream, *n_out_records of them, *dst_total bytes; dst_cap
 * below that -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes needed.  *n_left_records / *n_right_records: the input
 * record counts.  The field-kind arrays (B2S_FIELD_*, one per field) may be NULL for semi and anti joins, and the right
 * one for the existence join.
 * Errors -> B2S_E_ARG: an unknown join_type; n_left > n; a key column the composite-key calls reject (B2S_KEY_NULL_SAFE
 * aside), or any order flag; a key slot outside its side's slots [8 bX, 8 (bX + nX)) or a null bit not below its side's field count; a field
 * count outside 1..65536; NULL or unknown field kinds for every type but semi and anti (the existence join: the left
 * side's); more than 2^32 - 1 input records.
 * Per block, B2S_E_CORRUPT for every framing rule of the composite-key calls with that block's side's key columns, and
 * when a row is shorter than its side's fixed region 8 (bX + nX); b2s_last_error() names the block and the byte offset
 * of the bad record.  A joined row longer than 2^31 - 1 bytes -> B2S_E_UNSUPPORTED.  Checksums and bad_slice as in the
 * sorts.  When a block fails nothing is written, every count is 0 and the call returns 0.  The task or its output not
 * fitting in device memory -> B2S_E_NOMEM (the caller keeps Spark's join).
 * Runs on the read lane with the sorts' 1 GiB buffer trim.  b2s_last_timing: kernel_ms the whole call, top_kernel_ms
 * framing, keys, sort and join, dominant_ms / dominant_launches the join step alone (from the sorted order to the
 * written output). */
#define B2S_JOIN_INNER 0
#define B2S_JOIN_LEFT_OUTER 1
#define B2S_JOIN_LEFT_SEMI 2
#define B2S_JOIN_LEFT_ANTI 3
/* 4 is not assigned */
#define B2S_JOIN_RIGHT_OUTER 5
#define B2S_JOIN_FULL_OUTER 6
/* 7 is not assigned */
#define B2S_JOIN_EXISTENCE 8
/* field kinds of a side's schema (the joined row's offset fix-up and an outer join's null side) */
#define B2S_FIELD_FIXED 0        /* a fixed-width value in its 8-byte slot */
#define B2S_FIELD_VAR 1          /* (offset << 32) | size: string, binary, array, map, struct */
#define B2S_FIELD_DECIMAL_WIDE 2 /* Decimal(p > 18): (offset << 32) | size, 16 bytes reserved */
int b2s_decompress_join_rows_keys_packed(
    uint32_t join_type, uint32_t codec, uint32_t checksum_alg, uint32_t n_left, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_len,
    const uint32_t* left_key_off, const int32_t* left_key_null_field, const uint32_t* right_key_off,
    const int32_t* right_key_null_field, uint32_t n_left_fields, const uint8_t* left_field_kind,
    uint32_t n_right_fields, const uint8_t* right_field_kind, uint8_t* dst_base, uint64_t dst_cap,
    uint64_t* dst_total, uint64_t* n_left_records, uint64_t* n_right_records, uint64_t* n_out_records, int32_t* status,
    int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; the descriptor, key and field-kind arrays stay host
 * arrays */
int b2s_decompress_join_rows_keys_dev(
    uint32_t dev_index, uint32_t join_type, uint32_t codec, uint32_t checksum_alg, uint32_t n_left, uint32_t n,
    const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
    const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_len, const uint32_t* left_key_off, const int32_t* left_key_null_field,
    const uint32_t* right_key_off, const int32_t* right_key_null_field, uint32_t n_left_fields,
    const uint8_t* left_field_kind, uint32_t n_right_fields, const uint8_t* right_field_kind, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_left_records, uint64_t* n_right_records,
    uint64_t* n_out_records, int32_t* status, int32_t* bad_slice);

/* ---- read side, window: Spark's WindowExec (ranking functions) on a reducer's shuffled UnsafeRows ----
 * Spark SQL's Sort -> [WindowGroupLimit(Final) ->] Window over a shuffle read, for window expressions that are ranking
 * functions with their default frame, in one call: the rows are sorted by the window's key, each record gets the
 * values of the n_fns functions over its partition, and each output row is the input row joined with those values.
 * Blocks, slices, checksums and framing as in b2s_decompress_sort_rows_packed: [size: int32 BE][row], no end marker.
 * Keys.  The composite key of the *_keys calls: n_keys (at most 16) columns key_type[c] / key_off[c] / key_len[c] /
 * key_null_field[c], every type of those calls.  Its first n_partition_keys columns (0..15) are the PARTITION BY
 * columns and take no order flag (WindowExec.requiredChildOrdering sorts them ascending, nulls first); the remaining
 * columns (at least one) are the ORDER BY columns, with any flags.  Records are stably sorted by the whole key, exactly
 * as b2s_decompress_sort_rows_keys_* sorts them (ties in block order, then in their order in the block).
 * Partitions and peers.  A partition is a maximal run of sorted records that are equal on the partition columns, by
 * the composite-key aggregation's grouping rule: nulls equal nulls, strings are equal by length and bytes, 0.0 equals
 * -0.0 and every NaN equals every other NaN (on input NormalizeFloatingNumbers has normalised, WindowExec's equality
 * of the projected partition rows).  With n_partition_keys == 0 the whole reducer is one partition.  Peers are records
 * of one partition that are equal on the order columns by the same rule (RankLike's EqualNullSafe).
 * Functions.  fn[j] (j < n_fns, 1..16 of them, in any order, repeats allowed) is one of B2S_WINDOW_*.  With N the
 * partition's size, i the record's 0-based position in it and [gs, ge) its peer group's positions in it:
 *   ROW_NUMBER    int     i + 1
 *   RANK          int     gs + 1
 *   DENSE_RANK    int     the number of peer groups of the partition up to and including this one
 *   PERCENT_RANK  double  N > 1 ? (double) gs / (N - 1) : 0.0
 *   CUME_DIST     double  (double) ge / N
 *   NTILE         int     NTile(k)'s bucket, k = fn_arg[j] (at least 1): the first N % k buckets hold N / k + 1 rows
 *                         each, the rest N / k, numbered from 1 in sorted order
 * fn_arg[j] must be 0 for every function but NTILE.
 * Limit (WindowGroupLimitExec).  limit_fn is B2S_WINDOW_NO_LIMIT with limit 0 (every record is output), or one of
 * ROW_NUMBER, RANK and DENSE_RANK with limit at least 1: then only the records whose value of limit_fn is at most limit
 * are output, so rank ties at the boundary are all kept.  With a limit every fn[j] must be ROW_NUMBER, RANK or
 * DENSE_RANK: the only case Spark's InferWindowGroupLimit plans, and the only one where the values of the kept rows do
 * not depend on the dropped ones.
 * Output row.  The input row joined with a row of the n_fns values, laid out as UnsafeRowJoiner joins them: the join's
 * joined row (b2s_decompress_join_rows_keys_*) with a right side of n_fns non-null FIXED fields and no var bytes.  With
 * nC = n_fields, bC = ceil(nC / 64) and b = ceil((nC + n_fns) / 64):
 *   [b words: the input's nC null bits, zeros above][the input's 8 nC bytes of slots][8 bytes per function, in fn
 *   order][the input's var bytes]
 * An int value is written as UnsafeRowWriter writes it, the 8-byte slot zeroed and then 4 little-endian bytes; a double
 * as its 8 bytes.  Every VAR or DECIMAL_WIDE field (field_kind, B2S_FIELD_* as for the join; required) whose slot is
 * not zero has its offset (the high 32 bits) moved by 8 (b - bC + n_fns).
 * Outputs.  The output rows in sorted order as [size BE][row] records, an UnsafeRowSerializer stream: *n_out_records of
 * them, *dst_total bytes; dst_cap below that -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes needed.  *n_records:
 * the input record count.
 * Errors -> B2S_E_ARG: a key column the composite-key calls reject; an order flag on a partition column; no order
 * column (n_partition_keys >= n_keys, or above 15); a key slot outside the input's slots [8 bC, 8 (bC + nC)) or a key
 * null bit not below nC; n_fields outside 1..65536; NULL or unknown field kinds; n_fns outside 1..16, NULL fn or fn_arg,
 * an unknown fn, an NTILE bucket count below 1 or a non-zero fn_arg of another function; a limit_fn that is none of
 * the four, B2S_WINDOW_NO_LIMIT with a non-zero limit, a limit below 1, or a limit with a function other than the
 * three; a NULL count pointer; more than 2^32 - 1 input records.
 * Per block, B2S_E_CORRUPT for every framing rule of the composite-key calls and when a row is shorter than the input's
 * fixed region 8 (bC + nC); b2s_last_error() names the block and the byte offset of the bad record.  A partition of
 * more than 2^31 - 1 records (Spark's int values would wrap) or an output row longer than 2^31 - 1 bytes ->
 * B2S_E_UNSUPPORTED.  When a block fails nothing is written, every count is 0 and the call returns 0.  Checksums and
 * bad_slice, codec NONE and B2S_E_NOMEM (the caller keeps Spark's window) are as in the sorts.
 * Runs on the read lane with the sorts' 1 GiB buffer trim.  b2s_last_timing: kernel_ms the whole call, top_kernel_ms
 * framing through emit, dominant_ms / dominant_launches the window step alone (from the sorted order to the written
 * rows). */
#define B2S_WINDOW_ROW_NUMBER 0
#define B2S_WINDOW_RANK 1
#define B2S_WINDOW_DENSE_RANK 2
#define B2S_WINDOW_PERCENT_RANK 3
#define B2S_WINDOW_CUME_DIST 4
#define B2S_WINDOW_NTILE 5
#define B2S_WINDOW_NO_LIMIT 0xffffffffu
int b2s_decompress_window_rows_keys_packed(
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, uint32_t limit_fn, int32_t limit,
    uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_out_records,
    int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; every array stays a host array */
int b2s_decompress_window_rows_keys_dev(
    uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields,
    const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, uint32_t limit_fn,
    int32_t limit, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
    uint64_t* n_out_records, int32_t* status, int32_t* bad_slice);

/* ---- read side, window aggregates: Spark's WindowExec with aggregate functions on a reducer's shuffled UnsafeRows ----
 * b2s_decompress_window_rows_keys_* without a limit, where fn[j] may also be an aggregate function over a frame.  Blocks,
 * keys, partitions, peers, the ranking functions, the output stream, the counts and everything not stated here are that
 * call's.  The semantics are Spark 3.5's AggregateProcessor running each DeclarativeAggregate's update and evaluate
 * expressions with spark.sql.ansi.enabled off.
 * Per function j: fn[j], fn_arg[j] (NTILE's bucket count, else 0), fn_frame[j], val_type[j], val_off[j] and
 * val_null_field[j].  A ranking function takes frame 0 (its own) and B2S_WINDOW_VAL_NONE.  An aggregate function
 * (B2S_WINDOW_SUM .. B2S_WINDOW_AVG) takes one of the frames, with i the record's 0-based position in its partition of N
 * and [gs, ge) its peer group's positions:
 *   B2S_WINDOW_FRAME_PARTITION      positions [0, N): no ORDER BY, or UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING with
 *                                   either frame type
 *   B2S_WINDOW_FRAME_ROWS_RUNNING   positions [0, i]: ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW
 *   B2S_WINDOW_FRAME_RANGE_RUNNING  positions [0, ge), through the last peer: RANGE BETWEEN UNBOUNDED PRECEDING AND
 *                                   CURRENT ROW, the default with ORDER BY
 * With every function on FRAME_PARTITION the key may have no ORDER BY column (n_partition_keys == n_keys).
 * Input.  val_type[j] is B2S_WINDOW_VAL_INT8, _INT16, _INT32, _INT64, _FLOAT32 or _FLOAT64, read from the field whose
 * 8-byte slot is at byte val_off[j] (8 (bC + f) for a field f < nC) as UnsafeRowWriter writes it; or
 * B2S_WINDOW_VAL_DECIMAL | p << 8 | s << 16 for decimal(p, s), 1 <= p <= 38, s <= p: for p <= 18 the slot holds the
 * unscaled long, for p > 18 the field is DECIMAL_WIDE and its slot (offset << 32) | size points at the unscaled value's
 * big-endian two's-complement bytes.  The field's kind must be DECIMAL_WIDE exactly when p > 18 and FIXED otherwise.
 * val_null_field[j] is the field's null bit, or -1 (never null).  B2S_WINDOW_VAL_NONE is count(*) (COUNT only; val_off
 * and val_null_field are then ignored).
 * Fold order.  Every frame is folded over its records in sorted order from the partition's first record.  The sort is
 * stable, so this is the order Spark's UnboundedWindowFunctionFrame and UnboundedPrecedingWindowFunctionFrame fold in
 * whenever Spark's sort keeps ties in read order.  Only the double sums and the first-of-equal choice of MIN / MAX
 * depend on it.
 *   SUM    integral input: the 64-bit wrapping sum of the non-null inputs, sign-extended, a long.  Float or double
 *          input: ((0.0 + x1) + x2) + ... over the non-null inputs in double, each add rounded to nearest (no
 *          reassociation, no FMA; a float widened exactly; a lone -0.0 gives +0.0), a double.  decimal(p, s) with
 *          p <= 28: the exact sum, a decimal(p + 10, s); below 2^31 records |S| < 2^31 10^p < 10^(p + 10) < 2^127, so it
 *          never overflows.  Null when the frame has no non-null input.
 *   COUNT  the number of non-null inputs (every record for VAL_NONE), a long; never null.
 *   MIN / MAX  the input's type.  Spark SQL's order: -0.0 equals 0.0 and NaN is above every other value and equal to
 *          every NaN; decimals compare as signed unscaled values.  Among equal values the first in fold order is kept
 *          with its exact bits (Least / Greatest, as B2S_AGG_MIN / MAX_FLOAT64).  Null when no input is non-null.
 *   AVG    numeric input: the SUM fold in double (integral inputs converted to double rounded to nearest) divided by
 *          (double) count, a double.  decimal(p, s) with p <= 24: the exact sum divided by the count and rounded
 *          HALF_UP (ties away from zero) to scale s + 4, a decimal(p + 4, s + 4).  Null when the count is 0.
 *          Spark first divides to at least 38 significant digits (Decimal./, rounding HALF_UP) and then rounds that
 *          to scale s + 4; for p <= 24 and counts c < 2^31 the two roundings equal this one.  |S| < c 10^p, so the
 *          quotient has at most p - s <= 24 - s digits before the point and the first rounding keeps at least 14 + s
 *          after it: an error of at most 10^-(14+s) / 2, which is 10^-10 / 2 units of 10^-(s+4).  In those units the
 *          exact quotient is k + m / c (0 <= m < c): on a half-point (2m = c) it has s + 5 digits after the point and
 *          the first rounding is exact; elsewhere it is at least 1 / (2c) > 2^-32 > 10^-10 / 2 units from every
 *          half-point, so the first rounding cannot carry it across one.
 * Output row.  The input row joined with the row of the n_fns values as UnsafeRowJoiner joins them, as in the ranking
 * call, except that a value can be null and carry bytes.  With b = ceil((nC + n_fns) / 64): value j's null bit is
 * nC + j, set exactly when its result is null (its slot is then zero).  Ints, longs, floats and doubles are written as
 * UnsafeRowWriter writes them: the slot zeroed, then the value's bytes.  A decimal result of precision <= 18 is its
 * unscaled long; a wider one takes 16 bytes appended after the input's var bytes, in function order, at offset
 * 8 (b + nC + n_fns) + varC + 16 k for the k-th such function (varC: the input's var bytes), its slot (offset << 32) | len
 * and its bytes BigInteger.toByteArray's minimal len, zero-padded to 16.  A null one keeps its 16 zero bytes and the
 * slot offset << 32 (the join's null-side rule).
 * Errors -> B2S_E_ARG: everything the ranking call rejects (except no ORDER BY column as above); n_fns outside 1..16;
 * NULL fn, fn_arg, fn_frame, val_type, val_off or val_null_field; an unknown function or frame, or a frame the function
 * does not take; a val_type the function does not take (SUM and AVG: the numeric types and decimals up to p 28 and 24;
 * MIN and MAX: numeric and decimal; COUNT: those and VAL_NONE; ranking: VAL_NONE); a decimal precision or scale out of
 * range or a field kind that does not match; a value slot that is not one of the input's slots, or a value null bit
 * below -1 or not below nC.  These are checked before the device.  Per block, B2S_E_CORRUPT for the ranking call's
 * rules and when a non-null DECIMAL_WIDE input's size is not 1..16 or its bytes run past its row; nothing is written
 * when a block fails.  A partition of more than 2^31 - 1 records or an output row longer than 2^31 - 1 bytes ->
 * B2S_E_UNSUPPORTED.  B2S_E_DST_TOO_SMALL, B2S_E_NOMEM, the read lane, the buffer trim and b2s_last_timing as in the
 * ranking call (dominant_ms the window step). */
#define B2S_WINDOW_SUM 6
#define B2S_WINDOW_COUNT 7
#define B2S_WINDOW_MIN 8
#define B2S_WINDOW_MAX 9
#define B2S_WINDOW_AVG 10
#define B2S_WINDOW_FRAME_PARTITION 1
#define B2S_WINDOW_FRAME_ROWS_RUNNING 2
#define B2S_WINDOW_FRAME_RANGE_RUNNING 3
#define B2S_WINDOW_VAL_NONE 0
#define B2S_WINDOW_VAL_INT8 1
#define B2S_WINDOW_VAL_INT16 2
#define B2S_WINDOW_VAL_INT32 3
#define B2S_WINDOW_VAL_INT64 4
#define B2S_WINDOW_VAL_FLOAT32 5
#define B2S_WINDOW_VAL_FLOAT64 6
#define B2S_WINDOW_VAL_DECIMAL 7
int b2s_decompress_window_aggregate_rows_keys_packed(
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
    uint64_t* n_records, uint64_t* n_out_records, int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; every array stays a host array */
int b2s_decompress_window_aggregate_rows_keys_dev(
    uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields,
    const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame,
    const uint32_t* val_type, const uint32_t* val_off, const int32_t* val_null_field, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_out_records, int32_t* status,
    int32_t* bad_slice);

/* ---- read side, window offsets: Spark's WindowExec with offset functions on a reducer's shuffled UnsafeRows ----
 * b2s_decompress_window_aggregate_rows_keys_*, where fn[j] may also be an offset function, with two more per-function
 * arrays: fn_flags[j] and fn_default[j].  Everything not stated here is that call's, and one fn array mixes ranking,
 * aggregate and offset functions as one WindowExec does.  The semantics are Spark 3.5's FrameLessOffsetWindowFunctionFrame
 * (Lag, Lead), First, Last and NthValue.  With N the partition's size, i the record's 0-based position in it and e its
 * frame's last position (N - 1 for FRAME_PARTITION, i for FRAME_ROWS_RUNNING, ge - 1 for FRAME_RANGE_RUNNING):
 *   fn          fn_arg          fn_frame        value
 *   LEAD        offset k >= 1   0 (its own)     the input at position i + k if that is inside the partition, else the
 *                                               default.  IGNORE_NULLS: the k-th non-null input after i in the partition,
 *                                               else the default
 *   LAG         offset k >= 1   0               the same backwards: i - k, or the k-th non-null input before i
 *   FIRST       0               one of the      the input at position 0.  IGNORE_NULLS: the first non-null input in
 *                               three frames    [0, e], or null
 *   LAST        0               the three       the input at e.  IGNORE_NULLS: the last non-null input in [0, e], or null
 *   NTH_VALUE   n >= 1          the three       the input at n - 1 if n - 1 <= e, else null.  IGNORE_NULLS: the n-th
 *                                               non-null input in [0, e], or null
 * A null input at the chosen position gives null, not the default.  The default is null unless fn_flags[j] has
 * B2S_WINDOW_HAS_DEFAULT; then fn_default[j] holds the literal's slot bits as UnsafeRowWriter writes the input type
 * (the slot zeroed, then the type's width).  HAS_DEFAULT is allowed only for LAG and LEAD of a fixed-width type (not
 * VAL_BYTES, not a decimal above p 18).  B2S_WINDOW_IGNORE_NULLS is Spark's ignoreNulls.  LAG and LEAD need an ORDER BY
 * column, as Spark's analyzer requires; FIRST, LAST and NTH_VALUE with every frame FRAME_PARTITION may have none, as
 * aggregates may.  The result type is the input's type.
 * Input.  val_type[j] / val_off[j] / val_null_field[j] as for an aggregate: every B2S_WINDOW_VAL_INT8 .. _FLOAT64 (the
 * planner maps boolean to INT8, date to INT32 and timestamp to INT64), decimals of every precision 1..38, or
 * B2S_WINDOW_VAL_BYTES: a B2S_FIELD_VAR field (string or binary) whose slot is (offset << 32) | size.  VAL_NONE is not an
 * offset function's type, and an aggregate function does not take VAL_BYTES.
 * Output row.  The input row joined with the value row, as in the aggregate call.  A null value sets bit nC + j.  A
 * fixed-width value is written as UnsafeRowWriter writes it (the slot zeroed, then the type's width; floats keep their
 * exact bits).  Every var-valued function has a region after the input's var bytes, the regions in function order: a
 * wide decimal value (an offset function's or an aggregate's result) 16 bytes, BigInteger.toByteArray's minimal bytes
 * re-encoded from the value and zero-padded, its slot (offset << 32) | len, a null one 16 zero bytes and slot
 * offset << 32; a VAL_BYTES value its bytes zero-padded to a multiple of 8 as UnsafeRowWriter pads them, its slot
 * (offset << 32) | size, a null one no bytes and a zero slot.  Without offset functions this is the aggregate call's row.
 * Errors -> B2S_E_ARG: everything the aggregate call rejects (an offset function and VAL_BYTES aside); NULL fn_flags or
 * fn_default; an offset or n below 1; a non-zero fn_arg for FIRST and LAST; a frame an offset function does not take;
 * VAL_NONE for an offset function or VAL_BYTES for any other; an unknown flag bit, or flags on a function that is not an
 * offset function; HAS_DEFAULT where it is not allowed; a non-zero fn_default without it; default bits above the
 * type's width; VAL_BYTES on a field whose kind is not VAR.  These are checked before the device.  Per block,
 * B2S_E_CORRUPT for the aggregate call's rules and when a non-null VAL_BYTES input's bytes lie outside its row's var
 * region [8 (bC + nC), size) or a non-null DECIMAL_WIDE input of an offset function is bad as the aggregate call defines
 * it; every non-null input of an offset function is checked, whether or not an output row takes it, so the verdict does
 * not depend on the offsets; b2s_last_error() names the block and the record's offset, and nothing is written.  A
 * partition of more than 2^31 - 1 records or an output row longer than 2^31 - 1 bytes -> B2S_E_UNSUPPORTED.
 * B2S_E_DST_TOO_SMALL (with the exact size), B2S_E_NOMEM, the read lane, the buffer trim and b2s_last_timing
 * (dominant_ms the window step) as in the aggregate call. */
#define B2S_WINDOW_LAG 11
#define B2S_WINDOW_LEAD 12
#define B2S_WINDOW_FIRST 13
#define B2S_WINDOW_LAST 14
#define B2S_WINDOW_NTH_VALUE 15
/* the partial aggregation's central-moment function (stddev / variance, b2s_aggregate_*partition_compress_rows_hash_*
 * only; every window call rejects it) */
#define B2S_WINDOW_VARIANCE 16
#define B2S_WINDOW_VAL_BYTES 8
#define B2S_WINDOW_IGNORE_NULLS 1
#define B2S_WINDOW_HAS_DEFAULT 2
int b2s_decompress_window_offset_rows_keys_packed(
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, const uint32_t* fn_flags, const uint64_t* fn_default,
    uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_out_records,
    int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; every array stays a host array */
int b2s_decompress_window_offset_rows_keys_dev(
    uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields,
    const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame,
    const uint32_t* val_type, const uint32_t* val_off, const int32_t* val_null_field, const uint32_t* fn_flags,
    const uint64_t* fn_default, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
    uint64_t* n_out_records, int32_t* status, int32_t* bad_slice);

/* ---- read side, window frames: Spark's WindowExec over sliding ROWS and RANGE frames on a reducer's UnsafeRows ----
 * b2s_decompress_window_offset_rows_keys_*, with two more per-function arrays after fn_default: frame_lower[j] and
 * frame_upper[j].  Everything not stated here is that call's, and one fn array mixes ranking functions, LAG / LEAD, the
 * older frames and the new ones.  fn_frame[j] may also be B2S_WINDOW_FRAME_ROWS or B2S_WINDOW_FRAME_RANGE, for SUM,
 * COUNT, MIN, MAX, AVG, FIRST, LAST and NTH_VALUE (not ranking functions, LAG or LEAD); then frame_lower[j] /
 * frame_upper[j] are the frame's bounds: B2S_WINDOW_UNBOUNDED_PRECEDING (lower only), B2S_WINDOW_UNBOUNDED_FOLLOWING
 * (upper only), 0 CURRENT ROW, -k k PRECEDING, +k k FOLLOWING.  Frames 0..3 keep their meaning with both bounds 0.
 * Frames.  With [ps, pe) the partition's sorted positions and i a record's, its frame is the span [s, e] (possibly
 * empty) that Spark 3.5's frame classes produce for these bounds: UnboundedPreceding (lower unbounded: the running
 * fold, read at e), UnboundedFollowing (upper unbounded: a fresh fold from s to the partition's end), Unbounded (both:
 * the partition) and Sliding (any other: a fresh fold of the buffered rows from s).
 *   ROWS   [max(ps, i + lower), min(pe - 1, i + upper)]: RowBoundOrdering's j - (i + k).  Offsets fit in an int.
 *   RANGE  the positions whose order value lies between the bounds in the column's sort order (RangeBoundOrdering):
 *          CURRENT ROW is the peer group's edge and takes any order key; an offset bound is v + k ascending and
 *          v + (-k) descending in the column type's arithmetic, null when v is null (a null bound equals the null
 *          inputs and sorts before or after every value by the null order, so a null-keyed row's frame is its null
 *          peers).  An offset needs exactly one ORDER BY column (n_keys - n_partition_keys == 1) of type B2S_KEY_INT8,
 *          _INT16, _INT32 (int or date) or _INT64, any direction and null order; it must fit the column's type and,
 *          descending, not be the type's minimum.  Float, double, decimal and interval offsets are not taken.
 * Values, folded over [s, e] in sorted order from s: SUM of an integral the wrapping 64-bit sum, of a decimal exact;
 * COUNT the non-null inputs (0 on an empty frame, never null); MIN / MAX the first of equal values with its bits; SUM of
 * a float or double and AVG of a non-decimal ((0.0 + x_s) + x_{s+1}) + ... in double (for an unbounded lower end the
 * running fold at e); AVG of a decimal the exact sum rounded HALF_UP as in the aggregate call; FIRST / LAST /
 * NTH_VALUE the input at s, at e, or at s + n - 1 if that is <= e (IGNORE_NULLS: the first, last or n-th non-null
 * input in [s, e]).  An empty frame gives null for everything but COUNT.
 * Errors -> B2S_E_ARG, before the device: everything the offset call rejects (with frames 4 and 5 accepted as above);
 * NULL frame_lower or frame_upper; non-zero bounds on frames 0..3; UNBOUNDED FOLLOWING as a lower or UNBOUNDED
 * PRECEDING as an upper bound; lower above upper; a ROWS offset outside the int range; a RANGE offset without exactly
 * one ORDER BY column of the four integral key types, or that does not fit the column (descending: or is its minimum).
 * B2S_E_UNSUPPORTED (the caller keeps Spark's window; nothing is written), where Spark's int compare or bound arithmetic
 * would wrap and its buffer loop no longer matches these frames: a partition of N records with N - 1 + |k| > 2^31 - 1
 * for a finite ROWS offset k, or a non-null order value v whose exact v +- k leaves the column's type.  Everything else
 * (the output row, B2S_E_CORRUPT, B2S_E_DST_TOO_SMALL, B2S_E_NOMEM, the lane, the trim, b2s_last_timing) is the offset
 * call's.  b2s_decompress_window_aggregate_rows_keys_* and b2s_decompress_window_offset_rows_keys_* keep rejecting
 * frames 4 and 5. */
#define B2S_WINDOW_FRAME_ROWS 4
#define B2S_WINDOW_FRAME_RANGE 5
#define B2S_WINDOW_UNBOUNDED_PRECEDING INT64_MIN
#define B2S_WINDOW_UNBOUNDED_FOLLOWING INT64_MAX
int b2s_decompress_window_frame_rows_keys_packed(
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, const uint32_t* fn_flags, const uint64_t* fn_default,
    const int64_t* frame_lower, const int64_t* frame_upper, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
    uint64_t* n_records, uint64_t* n_out_records, int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index; every array stays a host array */
int b2s_decompress_window_frame_rows_keys_dev(
    uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields,
    const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame,
    const uint32_t* val_type, const uint32_t* val_off, const int32_t* val_null_field, const uint32_t* fn_flags,
    const uint64_t* fn_default, const int64_t* frame_lower, const int64_t* frame_upper, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_out_records, int32_t* status,
    int32_t* bad_slice);

/* ---- exchange cache: map outputs kept resident in HBM for reducers on the same device ----
 * (docs/f4_gpu_resident_exchange.md steps 2 and 3, local half.)  The serialized writer's partition step already leaves
 * a map task's records partitioned by reduce id in HBM; the cached store keeps that arena, keyed by (shuffle_id,
 * map_id), on the calling thread's device, and a reducer on the same device reads its partitions of it with one gather
 * instead of fetching, verifying and decoding the .data ranges.  The object store stays the source of truth: an entry is
 * never the only copy, and a miss is served by the usual fetch.  An entry on another device of the process is a miss.
 *
 * Budget: per device, in bytes of cached records and of the row writers' record boundaries (8 per record); 0 (the
 * default) turns the cache off.  Stores evict least recently used
 * entries that no read is using until the new entry fits; a read counts as a use.  Lowering a budget evicts down to it.
 * Device memory: when one of the library's own workspaces cannot grow, unreferenced entries of that device are evicted
 * and the allocation is retried once, so a generous budget does not make another call fail with B2S_E_NOMEM.
 * Concurrency: every read references the entries it uses from its lookup until its stream has synchronised; eviction
 * and removal unlink an entry at once and free its memory when its last reader is done.
 * Without a usable device every call returns B2S_E_CUDA; before b2s_init, B2S_E_NOT_INIT. */
int b2s_exchange_set_budget(uint32_t dev_index, uint64_t bytes);
/* b2s_partition_compress_packed, byte for byte (outputs, status and return value), that also keeps the partitioned
 * records and their partition offsets as the entry (shuffle_id, map_id), replacing an existing entry of that key.  The
 * records are copied device to device into an exact-size allocation.  *cached = 1 when the entry was stored, 0 when it
 * does not fit (the budget is 0 or below its size, or the rest of the cache is in use) or the call did not succeed. */
int b2s_partition_compress_cached_packed(int32_t shuffle_id, int64_t map_id, uint32_t codec, int32_t level,
                                         uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
                                         uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes,
                                         const uint32_t* rec_len, const uint32_t* rec_part, uint8_t* dst_base,
                                         uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                         uint64_t* checksum_out, int32_t* status, int32_t* cached);
/* len[i] = bytes of partitions [start_reduce, end_reduce) of map_ids[i] when that map output is resident on the calling
 * thread's device, UINT64_MAX otherwise.  Returns the number of hits.  Nothing is referenced: a later read can still
 * find an entry gone.  start_reduce < 0, end_reduce < start_reduce, NULL arrays, or a resident entry with fewer than
 * end_reduce partitions -> B2S_E_ARG. */
int b2s_exchange_lookup(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, uint32_t n_maps,
                        const int64_t* map_ids, uint64_t* len);
/* the partitions [start_reduce, end_reduce) of each map output, back to back in map_ids order, copied to host memory:
 * dst_off[i] / dst_len[i], status[i] = B2S_OK or B2S_E_NOT_CACHED (dst_len 0).  For shuffles without a key ordering.
 * dst_cap below the bytes -> B2S_E_DST_TOO_SMALL with *dst_total = the bytes needed.  Runs on the read lane. */
int b2s_exchange_read_packed(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, uint32_t n_maps,
                             const int64_t* map_ids, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                             uint64_t* dst_len, uint64_t* dst_total, int32_t* status);
/* b2s_decompress_sort_packed over n sources of which some are served from the cache.  Source i is the cached range
 * [start_reduce, end_reduce) of map_ids[i] when cached[i] != 0 (its src_off / src_len and slices are ignored; its slice
 * range may be empty), fetched block i otherwise.  The contract is decompress_sort's with source order as block order:
 * the sort is stable, fetched blocks are verified and decoded as there, and when any source fails nothing is sorted,
 * *n_records = 0 and the call returns 0.  A cached source that is not resident sets status[i] = B2S_E_NOT_CACHED; one
 * that is not a whole number of records, B2S_E_CORRUPT.  Cached sources are not checksum-verified (they never left the
 * device).  Decoded blocks are written straight to their place among the cached ranges; one gather moves the cached
 * ranges.  kernel_ms covers gather, verification, decode and sort; top_kernel_ms the sort. */
int b2s_exchange_read_sort_packed(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids,
                                  const uint8_t* cached, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                  const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                  const uint32_t* slice_base, const uint64_t* slice_len,
                                  const uint64_t* slice_checksum, uint32_t record_bytes, uint32_t key_off,
                                  uint32_t key_len, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
                                  uint64_t* n_records, int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index (and the cache entries of that device) */
int b2s_exchange_read_sort_dev(uint32_t dev_index, int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce,
                               const int64_t* map_ids, const uint8_t* cached, uint32_t codec, uint32_t checksum_alg,
                               uint32_t n, const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                               const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                               uint32_t record_bytes, uint32_t key_off, uint32_t key_len, uint8_t* dst_base,
                               uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                               int32_t* bad_slice);
/* The row writers' cached forms: b2s_partition_compress_rows_{hash,range,round_robin}_packed, byte for byte (outputs,
 * status and return value), that also keep the partitioned rows as the entry (shuffle_id, map_id), as
 * b2s_partition_compress_cached_packed does, together with their record boundaries: every record's offset in the entry
 * (device memory, 8 bytes per record, counted against the budget beside the records' bytes rounded up to 8) and each
 * partition's first record index.  A read of such an entry marks its records from the boundaries, a thread per record,
 * instead of walking the size chain (b2s_exchange_read_*_rows_keys_*).  b2s_exchange_lookup's len stays the bytes of records.  The entry
 * is also served by b2s_exchange_read_packed.  cached NULL -> B2S_E_ARG; otherwise the argument errors of the uncached
 * form, then the exchange cache's (B2S_E_CUDA without a usable device, B2S_E_NOT_INIT before b2s_init). */
int b2s_partition_compress_rows_hash_cached_packed(int32_t shuffle_id, int64_t map_id, uint32_t codec, int32_t level,
                                                   uint32_t codec_block_size, uint32_t checksum_alg,
                                                   uint32_t num_partitions, uint64_t n_records,
                                                   const uint8_t* rec_base, uint64_t rec_bytes,
                                                   const uint32_t* rec_len, uint32_t n_keys, const uint32_t* key_type,
                                                   const uint32_t* key_off, const uint32_t* key_len,
                                                   const int32_t* key_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                                   uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                                   uint64_t* checksum_out, int32_t* status, int32_t* cached);
int b2s_partition_compress_rows_range_cached_packed(int32_t shuffle_id, int64_t map_id, uint32_t codec, int32_t level,
                                                    uint32_t codec_block_size, uint32_t checksum_alg,
                                                    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes,
                                                    const uint32_t* rec_len, uint32_t n_keys,
                                                    const uint32_t* key_type, const uint32_t* key_off,
                                                    const uint32_t* key_len, const int32_t* key_null_field,
                                                    uint32_t n_bounds, const uint8_t* bound_base,
                                                    uint64_t bound_bytes, const uint32_t* bound_len,
                                                    uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                                                    uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out,
                                                    int32_t* status, int32_t* cached);
int b2s_partition_compress_rows_round_robin_cached_packed(int32_t shuffle_id, int64_t map_id, uint32_t codec,
                                                          int32_t level, uint32_t codec_block_size,
                                                          uint32_t checksum_alg, uint32_t num_partitions,
                                                          int32_t start_position, uint32_t sort_rows,
                                                          uint64_t n_records, const uint8_t* rec_base,
                                                          uint64_t rec_bytes, const uint32_t* rec_len,
                                                          uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                                                          uint64_t* dst_len, uint64_t* dst_total,
                                                          uint64_t* checksum_out, int32_t* status, int32_t* cached);
/* b2s_decompress_sort_rows_keys_* and b2s_decompress_aggregate_rows_keys_* over n sources of which some are served
 * from the cache, with b2s_exchange_read_sort_packed's contract: source i is the cached range [start_reduce,
 * end_reduce) of map_ids[i] when cached[i] != 0, fetched block i otherwise; source order is block order and the sort is
 * stable; a cached source that is not resident sets status[i] = B2S_E_NOT_CACHED; cached sources are not
 * checksum-verified; when any source fails nothing is sorted or written (*n_records = 0, and *n_groups = 0, the call
 * returns 0).  Every row rule of the composite-key calls applies to cached sources too: a cached row too short for the
 * read's key, null word or aggregate slot fails its source with B2S_E_CORRUPT, and b2s_last_error() names "cached source
 * i" and the byte offset of its lowest bad record, as for a fetched block.  A cached range of a row writer's entry is
 * framed from its stored record boundaries; one of an id-taking entry (b2s_partition_compress_cached_packed) is walked
 * as a fetched block is.  With n_keys = 1 these serve the single-key calls' reads.  Errors -> B2S_E_ARG: those of the
 * composite-key calls, and b2s_exchange_read_sort_packed's (NULL map_ids / cached / status, a bad reduce range). */
int b2s_exchange_read_sort_rows_keys_packed(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce,
                                            const int64_t* map_ids, const uint8_t* cached, uint32_t codec,
                                            uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                            const uint64_t* src_off, const uint64_t* src_len,
                                            const uint32_t* slice_base, const uint64_t* slice_len,
                                            const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type,
                                            const uint32_t* key_off, const uint32_t* key_len,
                                            const int32_t* key_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                            uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                                            int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index (and the cache entries of that device) */
int b2s_exchange_read_sort_rows_keys_dev(uint32_t dev_index, int32_t shuffle_id, int32_t start_reduce,
                                         int32_t end_reduce, const int64_t* map_ids, const uint8_t* cached,
                                         uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                         const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                                         const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_keys,
                                         const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                         const int32_t* key_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                         uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                                         int32_t* bad_slice);
int b2s_exchange_read_aggregate_rows_keys_packed(
    int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids, const uint8_t* cached,
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
    const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_op, const uint32_t* agg_off,
    const int32_t* agg_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
    uint64_t* n_groups, int32_t* status, int32_t* bad_slice);
/* same, with src_base / dst_base in device memory of dev_index (and the cache entries of that device) */
int b2s_exchange_read_aggregate_rows_keys_dev(
    uint32_t dev_index, int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids,
    const uint8_t* cached, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_op,
    const uint32_t* agg_off, const int32_t* agg_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
    uint64_t* n_records, uint64_t* n_groups, int32_t* status, int32_t* bad_slice);
/* removes the entry (shuffle_id, map_id) — map_id -1: every map output of the shuffle — on every device (the hook for
 * removeShuffle).  Returns the number of entries removed. */
int b2s_exchange_remove(int32_t shuffle_id, int64_t map_id);

/* ---- device-resident variants (data pointers are device memory on device `dev_index` of the b2s_init selection;
 *      descriptor arrays are host memory).  Synchronous; timings retrievable with b2s_last_timing. ---- */
int b2s_checksum_dev(uint32_t dev_index, uint32_t alg, uint32_t n, const void* d_base, const uint64_t* off,
                     const uint64_t* len, uint64_t* out);
int b2s_compress_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                     uint32_t checksum_alg, uint32_t n, const void* d_src_base, const uint64_t* src_off,
                     const uint64_t* src_len, void* d_dst_base, uint64_t dst_cap, uint64_t* dst_off,
                     uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status);
int b2s_decompress_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const void* d_src_base,
                       const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                       const uint64_t* slice_len, const uint64_t* slice_checksum, void* d_dst_base, uint64_t dst_cap,
                       uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total, int32_t* status,
                       int32_t* bad_slice);
void* b2s_dev_alloc(uint32_t dev_index, uint64_t bytes);
void b2s_dev_free(uint32_t dev_index, void* p);
int b2s_dev_memcpy(uint32_t dev_index, void* dst, const void* src, uint64_t bytes, int kind /*1=H2D 2=D2H 3=D2D*/);

/* ---- observability (the reference logs bytes/ms/MiB/s per block: shuffle/S3MeasureOutputStream.scala:55-63,
 *      storage/S3BufferedPrefetchIterator.scala:155-186) ---- */
typedef struct b2s_timing {
  double total_ms;        /* host wall time of the last call on this thread */
  double h2d_ms, d2h_ms;  /* CUDA-event time of the copies (0 for _dev calls) */
  double kernel_ms;       /* CUDA-event time from first to last kernel of the call */
  double top_kernel_ms;   /* CUDA-event time of the codec step (lz4 match+parse+emit / decompress / checksum) */
  uint64_t h2d_bytes, d2h_bytes;
  uint64_t kernel_launches; /* kernels launched by the call */
  uint64_t src_bytes, dst_bytes;
  double dominant_ms;       /* CUDA-event time of the single dominant kernel (lz4_match_kernel / lz4 decode), summed over its launches */
  uint64_t dominant_launches;
} b2s_timing;
int b2s_last_timing(b2s_timing* out);
/* CUDA-event stopwatch on the library's own stream of device dev_index (torch.cuda.Event only sees torch's stream):
 * b2s_mark(dev, 0) ... calls ... b2s_mark(dev, 1); b2s_marks_elapsed_ms(dev, &ms) synchronises on mark 1 */
int b2s_mark(uint32_t dev_index, uint32_t which);
int b2s_marks_elapsed_ms(uint32_t dev_index, double* ms);
uint64_t b2s_total_kernel_launches(void); /* process-wide counter since b2s_init */

/* ---- synthetic workload generator for the benchmark (device-side TeraGen-style 104-byte records; not on the
 *      product path).  Writes n_records*104 bytes at d_dst. ---- */
int b2s_gen_terasort_dev(uint32_t dev_index, void* d_dst, uint64_t first_record, uint64_t n_records, uint64_t seed);

#ifdef __cplusplus
}
#endif
#endif
