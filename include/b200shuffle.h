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
#define B2S_CODEC_ZSTD 3          /* "zstd"  : RFC 8878 frames, concatenation allowed */

/* checksum algorithms — spark.shuffle.checksum.algorithm (helper/S3ShuffleHelper.scala:94-103) */
#define B2S_CHECKSUM_NONE 0
#define B2S_CHECKSUM_ADLER32 1
#define B2S_CHECKSUM_CRC32 2
#define B2S_CHECKSUM_CRC32C 3 /* north-star addition; the Scala shim adds the "CRC32C" case */

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

/* ---- read side ---- */
/* n compressed blocks as produced by S3BufferedPrefetchIterator.next() (storage/S3BufferedPrefetchIterator.scala:196-212).
 * Block i covers n_slices[i] consecutive reduce partitions (1 for ShuffleBlockId, >1 for ShuffleBlockBatchId,
 * storage/S3ChecksumValidationStream.scala:22-27); slice_len[i][k] / slice_checksum[i][k] are the .index differences and
 * .checksum values of those partitions.  With checksum_alg != 0 every slice is verified over the compressed bytes
 * before decoding; a mismatch yields status[i] = B2S_E_CHECKSUM and bad_slice[i] = k (may be NULL).
 * n_slices / slice_* may be NULL when checksum_alg == 0. */
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
 * a block fails, nothing is sorted, *n_records = 0 and the call returns 0; blocks whose slices fail verification are
 * not decoded.
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

/* ---- exchange cache: map outputs kept resident in HBM for reducers on the same device ----
 * (docs/f4_gpu_resident_exchange.md steps 2 and 3, local half.)  The serialized writer's partition step already leaves
 * a map task's records partitioned by reduce id in HBM; the cached store keeps that arena, keyed by (shuffle_id,
 * map_id), on the calling thread's device, and a reducer on the same device reads its partitions of it with one gather
 * instead of fetching, verifying and decoding the .data ranges.  The object store stays the source of truth: an entry is
 * never the only copy, and a miss is served by the usual fetch.  An entry on another device of the process is a miss.
 *
 * Budget: per device, in bytes of cached records; 0 (the default) turns the cache off.  Stores evict least recently used
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
