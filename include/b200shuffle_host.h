/*
 * b200shuffle_host.h — C entry points of libb200shuffle_host.so: the HOST-SIDE MIRROR of the reference's plugin
 * surface for the codec path, written in C++ because the reference is compiled (Scala/JVM) code and no JVM exists
 * in this image.  It sits *above* the C ABI of include/b200shuffle.h exactly where the Scala classes sit above the
 * JNI shim (INTEGRATION.md), keeps their names, argument meaning, on-disk layout and error behaviour, and exists so
 * that parity tests can read like the reference's own tests (src/test/scala/org/apache/spark/shuffle/S3ShuffleManagerTest.scala).
 *
 * Mirrored classes (C++ in spark-s3-shuffle_b200/host/, namespace b2s::host):
 *   S3ShuffleDispatcher        helper/S3ShuffleDispatcher.scala:39-70 (config), :120-144 (paths), :190-237 (open/create)
 *   S3ShuffleHelper            helper/S3ShuffleHelper.scala:44-59 (.index/.checksum), :67-92 (cached readers), :94-103 (algorithms)
 *   S3ShuffleMapOutputWriter   shuffle/S3ShuffleMapOutputWriter.scala:67-83 (getPartitionWriter), :91-118 (commitAllPartitions),
 *                              :168-202 (partition stream), + the GPU "compress on commit" mode of SURVEY.md §3.2 option B
 *   S3SerializedShuffleWriter  UnsafeShuffleWriter + ShuffleExternalSorter.insertRecord [U] for a SerializedShuffleHandle:
 *                              records + reduce ids -> GPU partition + compress -> commitAllPartitions' output path
 *   S3MeasureOutputStream      shuffle/S3MeasureOutputStream.scala:8-65 (timing + byte counters of the .data stream)
 *   S3SingleSpillShuffleMapOutputWriter  shuffle/S3SingleSpillShuffleMapOutputWriter.scala:24-64 (+ GPU checksum verification)
 *   S3ShuffleReader            storage/S3ShuffleReader.scala:77-110 (block list -> prefetch -> verify -> decompress),
 *                              storage/S3ShuffleBlockIterator.scala:36-43, storage/S3ShuffleBlockStream.scala:36-40,73-92
 *   S3BufferedPrefetchIterator storage/S3BufferedPrefetchIterator.scala:16-213 (threads, memory budget, LIFO, ThreadPredictor)
 *   S3BufferedInputStreamAdaptor  storage/S3BufferedInputStreamAdaptor.scala:7-59 (owns the block buffer, returns budget on close)
 *   B200CompressionCodec       the Spark CompressionCodec seam [U] of SURVEY.md §8(f)-1 (compressedOutputStream / compressedInputStream)
 *   CoalescingQueue            (no counterpart in the reference) group commit of the codec calls of concurrent task threads,
 *                              owned by the dispatcher like the reference's executor-wide singletons; SURVEY.md §8(b) threading
 * Only file:// roots are implemented (S3/Hadoop I/O is out of scope, DESIGN.md §6).
 *
 * Errors: functions return 0 or a negative B2SH_E_* code; b2sh_last_error() holds the reference's exception text
 * (e.g. "Precondition: Expect a monotonically increasing reducePartitionId.", "Invalid checksum detected for shuffle_0_1_2").
 */
#ifndef B200SHUFFLE_HOST_H
#define B200SHUFFLE_HOST_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2SH_OK 0
#define B2SH_E_RUNTIME (-101)     /* RuntimeException (preconditions, length mismatch)                   */
#define B2SH_E_IO (-102)          /* IOException (closed stream, "Stream is corrupted")                  */
#define B2SH_E_SPARK (-103)       /* SparkException (invalid checksum, unexpected file length)           */
#define B2SH_E_UNSUPPORTED (-104) /* UnsupportedOperationException (unknown checksum algorithm / codec)  */
#define B2SH_E_CODEC (-105)       /* the C ABI below reported a call-level failure (no GPU, CUDA error)  */

const char* b2sh_last_error(void);

/* ---- dispatcher: conf is "key=value\n" lines using the reference's keys (spark.shuffle.s3.rootDir, .bufferSize,
 * .folderPrefixes, .alwaysCreateIndex, .cleanup, spark.shuffle.checksum.enabled/.algorithm, spark.io.compression.codec,
 * spark.io.compression.lz4.blockSize, spark.app.id) plus the additive spark.shuffle.s3.gpu.enabled (default true) and
 * spark.shuffle.s3.gpu.exchangeCacheBytes (default 0 = off; INTEGRATION.md §3f): the per-device budget of the exchange
 * cache, which keeps the serialized writer's partitioned map outputs in HBM for reducers on the same device.
 * remove_shuffle also removes the shuffle's cached map outputs. ---- */
typedef struct b2sh_dispatcher b2sh_dispatcher;
int b2sh_dispatcher_create(const char* conf, b2sh_dispatcher** out);
void b2sh_dispatcher_destroy(b2sh_dispatcher* d);
/* kind: 0 = .data, 1 = .index, 2 = .checksum ; writes the path (helper/S3ShuffleDispatcher.scala:142-143) into buf */
int b2sh_dispatcher_get_path(b2sh_dispatcher* d, int kind, int32_t shuffle_id, int64_t map_id, char* buf, uint32_t cap);
int b2sh_dispatcher_remove_shuffle(b2sh_dispatcher* d, int32_t shuffle_id);

/* ---- group commit of the codec calls of concurrent task threads (SURVEY.md §8b, threading row).  The dispatcher — one
 * per executor, like the reference's singleton (helper/S3ShuffleDispatcher.scala:240-254) — owns a queue: the first
 * caller runs at once, whatever other threads submit while the GPU is busy is merged into ONE b2s_compress_batch /
 * b2s_decompress_batch in the next round (no timer, no added latency for a single thread).  Same arguments and per-stream
 * results as the C-ABI batch calls; a call-level failure returns B2SH_E_CODEC.  The writer and the reader go through it
 * when spark.shuffle.s3.gpu.coalesce=true (additive key, default false).  out4: calls, batches, largest number of
 * calls merged into one batch, streams. ---- */
int b2sh_dispatcher_queue_compress(b2sh_dispatcher* d, uint32_t codec, int32_t level, uint32_t codec_block_size,
                                   uint32_t checksum_alg, uint32_t n, const uint8_t* const* src, const uint64_t* src_len,
                                   uint8_t* const* dst, const uint64_t* dst_cap, uint64_t* dst_len,
                                   uint64_t* checksum_out, int32_t* status);
int b2sh_dispatcher_queue_decompress(b2sh_dispatcher* d, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                     const uint8_t* const* src, const uint64_t* src_len, const uint32_t* n_slices,
                                     const uint64_t* const* slice_len, const uint64_t* const* slice_checksum,
                                     uint8_t* const* dst, const uint64_t* dst_cap, uint64_t* dst_len, int32_t* status,
                                     int32_t* bad_slice);
int b2sh_dispatcher_queue_statistics(b2sh_dispatcher* d, uint64_t* out4);

/* ---- helper ---- */
int b2sh_helper_checksum_algorithm(const char* name); /* -> B2S_CHECKSUM_* id or B2SH_E_UNSUPPORTED */
int b2sh_helper_get_partition_lengths(b2sh_dispatcher* d, int32_t shuffle_id, int64_t map_id, int64_t* out,
                                      uint32_t cap, uint32_t* count); /* the cumulative offsets stored in .index */
int b2sh_helper_get_checksums(b2sh_dispatcher* d, int32_t shuffle_id, int64_t map_id, int64_t* out, uint32_t cap,
                              uint32_t* count);

/* ---- map output writer ---- */
typedef struct b2sh_writer b2sh_writer;
int b2sh_writer_create(b2sh_dispatcher* d, int32_t shuffle_id, int64_t map_id, int32_t num_partitions,
                       b2sh_writer** out);
/* getPartitionWriter(reducePartitionId).openStream().write(bytes): ids must increase monotonically */
int b2sh_writer_open_partition(b2sh_writer* w, int32_t reduce_id);
int b2sh_writer_write(b2sh_writer* w, const uint8_t* bytes, uint64_t n);
int b2sh_writer_close_partition(b2sh_writer* w);
/* commitAllPartitions: GPU mode compresses + checksums every partition in one batch, then writes .data/.index/.checksum.
 * checksums_in is used only in pass-through mode (spark.shuffle.s3.gpu.enabled=false: bytes arrive already compressed,
 * exactly the reference's behaviour).  partition_lengths_out receives num_partitions values (MapOutputCommitMessage). */
int b2sh_writer_commit_all_partitions(b2sh_writer* w, const int64_t* checksums_in, int64_t* partition_lengths_out);
int b2sh_writer_abort(b2sh_writer* w);
/* S3MeasureOutputStream counters of the .data stream after commit: bytes written, nanoseconds spent inside
 * write/flush/close, and the reference's log line ("Statistics: Stage .. -- Writing shuffle_0_1_0.data N took T ms (B MiB/s)"). */
int b2sh_writer_statistics(b2sh_writer* w, uint64_t* bytes, uint64_t* nanos, char* line, uint32_t cap);
void b2sh_writer_destroy(b2sh_writer* w);

/* ---- GPU serialized writer: UnsafeShuffleWriter / ShuffleExternalSorter for a SerializedShuffleHandle (relocatable
 * serializer, no map-side aggregation; INTEGRATION.md §3d).  insert() = ShuffleExternalSorter.insertRecord(record,
 * partitionId), in any partition order; commit() partitions, compresses and checksums every partition in ONE
 * b2s_partition_compress_packed call and writes .data/.index/.checksum like b2sh_writer_commit_all_partitions — the
 * files are byte-identical to that writer's when it is fed the same records partition by partition, every partition
 * opened in ascending order.  partition_lengths_out receives num_partitions values.  Needs
 * spark.shuffle.s3.gpu.enabled; codec "none" partitions and checksums only.  With the exchange cache on the call is
 * b2s_partition_compress_cached_packed: the same files, and the partitioned records stay in HBM. ---- */
typedef struct b2sh_serialized_writer b2sh_serialized_writer;
int b2sh_serialized_writer_create(b2sh_dispatcher* d, int32_t shuffle_id, int64_t map_id, int32_t num_partitions,
                                  b2sh_serialized_writer** out);
int b2sh_serialized_writer_insert(b2sh_serialized_writer* w, int32_t partition_id, const uint8_t* bytes, uint64_t len);
int b2sh_serialized_writer_commit(b2sh_serialized_writer* w, int64_t* partition_lengths_out);
int b2sh_serialized_writer_statistics(b2sh_serialized_writer* w, uint64_t* bytes, uint64_t* nanos, char* line,
                                      uint32_t cap);
void b2sh_serialized_writer_destroy(b2sh_serialized_writer* w);

/* ---- single-spill writer (shuffle/S3SingleSpillShuffleMapOutputWriter.scala:24-64): moves an already compressed +
 * checksummed spill file to the .data object, then writes .checksum and .index.  verify_on_transfer != 0 recomputes the
 * per-partition checksums over the file on the GPU (b2s_checksum_packed) and fails with B2SH_E_SPARK on a mismatch. ---- */
int b2sh_single_spill_transfer(b2sh_dispatcher* d, int32_t shuffle_id, int64_t map_id, const char* spill_file,
                               const int64_t* partition_lengths, const int64_t* checksums, uint32_t num_partitions,
                               int verify_on_transfer);

/* ---- reader: blocks [start_partition, end_partition) of the given maps ---- */
typedef struct b2sh_reader b2sh_reader;
int b2sh_reader_create(b2sh_dispatcher* d, int32_t shuffle_id, const int64_t* map_ids, uint32_t n_maps,
                       int32_t start_partition, int32_t end_partition, int do_batch_fetch, b2sh_reader** out);
/* read(): resolves block ranges from .index, drops empty blocks, fetches the remaining ones, verifies every
 * partition slice against .checksum and decompresses — all blocks of the task in one C-ABI batch.  Afterwards
 * block k's decoded stream is at data + off[k].  A checksum mismatch returns B2SH_E_SPARK with the reference's message,
 * a malformed stream B2SH_E_IO.  With the exchange cache on, the maps resident on the calling thread's device are read
 * from it first (one block per map covering [start_partition, end_partition)); only the others are fetched, and only
 * their bytes count in remote_bytes_read. */
int b2sh_reader_read(b2sh_reader* r, uint32_t* n_blocks);
/* read_sorted(): read() for a shuffle with a key ordering, no aggregator and fixed-size records (INTEGRATION.md §3e,
 * spark.shuffle.s3.gpu.sortKey).  Resolves and fetches the task's non-empty blocks as read() does, then makes ONE
 * b2s_decompress_sort_packed call: *data / *len / *n_records receive every record of the task sorted by the unsigned
 * bytes [key_off, key_off + key_len) of each record_bytes-long record (stable: equal keys in map, then reduce-id
 * order).  The buffer stays valid until the reader's next read or its destruction.  A checksum mismatch returns
 * B2SH_E_SPARK with the reference's message, a malformed stream (or one that does not hold whole records) B2SH_E_IO.
 * Codec "none" is verified and sorted only.  With the exchange cache on, a map resident on the calling thread's device
 * is one cached source in that order (b2s_exchange_read_sort_packed) instead of its fetched blocks; maps evicted before
 * the call are fetched and the call is repeated. */
int b2sh_reader_read_sorted(b2sh_reader* r, uint32_t record_bytes, uint32_t key_off, uint32_t key_len,
                            const uint8_t** data, uint64_t* len, uint64_t* n_records);
int b2sh_reader_block(b2sh_reader* r, uint32_t k, int64_t* map_id, int32_t* start_reduce, int32_t* end_reduce,
                      const uint8_t** data, uint64_t* len);
uint64_t b2sh_reader_remote_bytes_read(b2sh_reader* r); /* metric parity with storage/S3ShuffleReader.scala:94-95 */
/* Pipelined form of read() (SURVEY.md §8(f)-2).  b2sh_reader_open() starts the prefetcher (1..maxConcurrencyTask threads
 * under maxBufferSizeTask bytes of compressed blocks, storage/S3BufferedPrefetchIterator.scala); every
 * b2sh_reader_next_batch() drains the blocks that are complete (at most max_blocks; 0 = no limit), verifies + decodes
 * them in ONE C-ABI batch and returns their buffers to the budget.  *n_blocks == 0 marks the end; b2sh_reader_block()
 * addresses the blocks of the current batch only.  b2sh_reader_read() is open() + next_batch() until the end, keeping
 * every decoded block.  Block order is unspecified, as in the reference (its completed list is LIFO, :146,:209). */
int b2sh_reader_open(b2sh_reader* r);
int b2sh_reader_next_batch(b2sh_reader* r, uint32_t max_blocks, uint32_t* n_blocks);
/* out8: bytesRead, numStreams, timeWaiting ns, timePrefetching ns, totalRuntime ns, active threads, peak buffered
 * bytes, peak threads.  line: the reference's statistics line (:162-175), available once hasNext turned false. */
int b2sh_reader_statistics(b2sh_reader* r, uint64_t* out8, uint64_t* batches, char* line, uint32_t cap);
void b2sh_reader_destroy(b2sh_reader* r);

/* ---- the prefetcher on its own: compressed blocks as S3BufferedPrefetchIterator.next() yields them.  The buffer of a
 * block stays valid (and charged to the budget) until b2sh_prefetch_close_stream(); max_buffer_size / max_threads <= 0
 * take spark.shuffle.s3.maxBufferSizeTask / .maxConcurrencyTask. ---- */
typedef struct b2sh_prefetch b2sh_prefetch;
int b2sh_prefetch_create(b2sh_dispatcher* d, int32_t shuffle_id, const int64_t* map_ids, uint32_t n_maps,
                         int32_t start_partition, int32_t end_partition, int do_batch_fetch, int64_t max_buffer_size,
                         int32_t max_threads, b2sh_prefetch** out);
int b2sh_prefetch_has_next(b2sh_prefetch* p);
int b2sh_prefetch_next(b2sh_prefetch* p, int64_t* map_id, int32_t* start_reduce, int32_t* end_reduce,
                       const uint8_t** data, uint64_t* len, uint64_t* stream);
int b2sh_prefetch_close_stream(b2sh_prefetch* p, uint64_t stream);
int b2sh_prefetch_statistics(b2sh_prefetch* p, uint64_t* out8, char* line, uint32_t cap);
void b2sh_prefetch_destroy(b2sh_prefetch* p);

/* ---- Spark CompressionCodec seam (SURVEY.md §8(f)-1): codec and block size come from the dispatcher's conf
 * (spark.io.compression.codec, spark.io.compression.lz4.blockSize; additive spark.shuffle.s3.gpu.codecBufferSize,
 * default 64m).  compressedOutputStream(sink): written bytes are collected and leave as complete streams of the codec's
 * JVM wire format, one per codecBufferSize and one at close.  compressedInputStream(source): the first read drains the
 * source and decodes it in one batch.  sink returns < 0 to fail; source returns bytes read, <= 0 at the end. ---- */
typedef int64_t (*b2sh_sink_fn)(void* ctx, const uint8_t* bytes, uint64_t n);
typedef int64_t (*b2sh_source_fn)(void* ctx, uint8_t* buf, uint64_t cap);
typedef struct b2sh_codec b2sh_codec;
typedef struct b2sh_ostream b2sh_ostream;
typedef struct b2sh_istream b2sh_istream;
int b2sh_codec_create(b2sh_dispatcher* d, b2sh_codec** out);
int b2sh_codec_supports_concatenation(b2sh_codec* c); /* supportsConcatenationOfSerializedStreams, storage/S3ShuffleReader.scala:57-60 */
void b2sh_codec_destroy(b2sh_codec* c);
int b2sh_codec_output_stream(b2sh_codec* c, b2sh_sink_fn sink, void* ctx, b2sh_ostream** out);
int b2sh_ostream_write(b2sh_ostream* s, const uint8_t* bytes, uint64_t n);
int b2sh_ostream_flush(b2sh_ostream* s);
int b2sh_ostream_close(b2sh_ostream* s, uint64_t* bytes_in, uint64_t* bytes_out, uint32_t* streams);
void b2sh_ostream_destroy(b2sh_ostream* s);
int b2sh_codec_input_stream(b2sh_codec* c, b2sh_source_fn source, void* ctx, b2sh_istream** out);
int b2sh_istream_read(b2sh_istream* s, uint8_t* buf, uint64_t cap, int64_t* got); /* *got = -1 at the end of the stream */
int b2sh_istream_close(b2sh_istream* s);
void b2sh_istream_destroy(b2sh_istream* s);

#ifdef __cplusplus
}
#endif
#endif
