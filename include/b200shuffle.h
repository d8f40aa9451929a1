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
/* decompressed size of each compressed stream (LZ4Block: sum of originalLen; Snappy: sum of chunk varints) */
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
 *   B2S_KEY_BYTES, key_len 1 (BooleanType): hashInt(byte != 0 ? 1 : 0)
 *   B2S_KEY_INT8 / B2S_KEY_INT16 / B2S_KEY_INT32 (ByteType, ShortType, IntegerType, DateType): hashInt of the value
 *   B2S_KEY_INT64 (LongType, TimestampType, Decimal(p <= 18)): hashLong
 *   B2S_KEY_FLOAT32 / B2S_KEY_FLOAT64: hashInt(floatToIntBits) / hashLong(doubleToLongBits), -0.0 as 0.0 and every NaN
 *     as the canonical NaN (Spark >= 3.2)
 *   B2S_STRING_KEY (StringType, BinaryType) / B2S_DECIMAL_KEY (Decimal(p > 18), 1..16 bytes): hashUnsafeBytes of the
 *     slot's bytes, with Spark's tail (every byte after the last whole 4-byte word mixed on its own, sign-extended)
 * Outputs: byte for byte what b2s_partition_compress_packed / _dev return for the same records and those ids.
 * Errors, B2S_E_ARG: what b2s_partition_compress_* rejects; n_keys outside 1..16, a type not listed, a key_len that does
 * not match its type, an order flag, key_null_field < -1.  A bad record -> B2S_E_ARG, nothing reported as written, and
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
 * written part of it before it met the corruption); the output ranges of the other blocks are never touched by it. */
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
 * but SUM_DECIMAL, or a SUM_DECIMAL precision of 0 or above 38; SUM_DECIMAL with agg_null_field[a] = -1;
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
 *     and without null keys it is the order of Spark's full outer scanner.
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
 * record counts.  The field-kind arrays (B2S_FIELD_*, one per field) may be NULL for semi and anti joins.
 * Errors -> B2S_E_ARG: an unknown join_type; n_left > n; a key column the composite-key calls reject, or any order
 * flag; a key slot outside its side's slots [8 bX, 8 (bX + nX)) or a null bit not below its side's field count; a field
 * count outside 1..65536; NULL or unknown field kinds for every type but semi and anti; more than 2^32 - 1 input
 * records.
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
