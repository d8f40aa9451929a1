/*
 * b200shuffle_jni.c — the thin JNI layer between the Scala side of IBM/spark-s3-shuffle and libb200shuffle.so.
 *
 * One native method per C entry point a JVM needs (include/b200shuffle.h); the Scala object that declares them is
 * org.apache.spark.shuffle.gpu.B200Codec (INTEGRATION.md §2).  Call sites on the reference side:
 *   init / shutdown / bindThreadToDevice   shuffle/S3ShuffleDataIO.scala:30-32 (initializeExecutor), task threads
 *   compressPacked                         shuffle/S3ShuffleMapOutputWriter.scala:91-118 (commitAllPartitions)
 *   partitionCompressPacked                the GPU serialized writer (INTEGRATION.md §3d): records + reduce ids of a
 *                                          map task in, .data arena + partitionLengths + checksums out
 *   partitionCompressRowsHashPacked        the same for a HashPartitioning exchange (INTEGRATION.md §3j): rows and
 *                                          their key columns in, the reduce ids computed on the GPU
 *   partitionCompressRowsRangePacked       the same for a RangePartitioning exchange (INTEGRATION.md §3k): rows,
 *                                          their sort-key columns and the partitioner's bound rows in
 *   partitionCompressRowsRoundRobinPacked  the same for a RoundRobinPartitioning exchange (INTEGRATION.md §3l): rows,
 *                                          the task's start position and sortBeforeRepartition in
 *   partitionCompressRows*CachedPacked     the three row writers keeping their map output in the exchange cache
 *                                          (INTEGRATION.md §3m); exchangeRead{Sort,Aggregate}RowsKeysPacked read it
 *   decompressPacked / decompressedSize    storage/S3ShuffleReader.scala:98-110 (the codec seam, batched drain of
 *                                          storage/S3BufferedPrefetchIterator.scala:196-212)
 *   checksumPacked                         shuffle/S3SingleSpillShuffleMapOutputWriter.scala:54-63,
 *                                          helper/S3ShuffleHelper.scala:94-103
 * Payload travels in pinned direct ByteBuffers (hostAlloc/wrap): the methods take raw addresses (jlong), so no
 * jbyteArray is ever pinned or copied.  The small descriptor arrays (offsets, lengths, checksums, status) are Java
 * long[]/int[]/byte[]: compressPacked, decompressPacked, decompressedSizePacked, checksumPacked and lastTiming hold
 * them with Get/ReleasePrimitiveArrayCritical (every Get paired with a Release on every path); every other native
 * copies them through Get/Set<Type>ArrayRegion, so no Java array is held while the GPU works.  Every native checks
 * each array's length against the count that sizes it, and each required array against null, before the library
 * sees a pointer: a bad argument is B2S_E_ARG, never a read or write past a Java array.
 *
 * Build (reference side):  cc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude \
 *                              jni/b200shuffle_jni.c -L. -lb200shuffle -o libb200shuffle_jni.so
 * Without a JDK: tests/test_jni_shim.py compiles this file against jni/stub/jni.h with -Wall -Wextra -Werror and runs
 * every native through a stand-in JNIEnv (tests/native/jni_env_host.c) that checks each call as -Xcheck:jni would.
 */
#include <jni.h>
#include <stdint.h>
#include <stdlib.h>

#include "b200shuffle.h"

#define J(name) Java_org_apache_spark_shuffle_gpu_B200Codec_##name
#define PTR(T, a) ((T*)(uintptr_t)(a))

/* critical-section helper: NULL arrays are allowed where the C ABI allows NULL */
static void* crit_get(JNIEnv* e, jarray a) { return a ? (*e)->GetPrimitiveArrayCritical(e, a, 0) : 0; }
static void crit_put(JNIEnv* e, jarray a, void* p, jint mode) {
  if (a && p) (*e)->ReleasePrimitiveArrayCritical(e, a, p, mode);
}

/* ---- lifecycle ---- */
JNIEXPORT jint JNICALL J(init)(JNIEnv* e, jclass c, jint gpuMask, jlong pinnedBytesPerGpu, jint streamsPerGpu) {
  (void)e; (void)c;
  return b2s_init((uint32_t)gpuMask, (uint64_t)pinnedBytesPerGpu, (uint32_t)streamsPerGpu);
}
JNIEXPORT void JNICALL J(shutdown)(JNIEnv* e, jclass c) {
  (void)e; (void)c;
  b2s_shutdown();
}
JNIEXPORT jint JNICALL J(deviceCount)(JNIEnv* e, jclass c) {
  (void)e; (void)c;
  return b2s_device_count();
}
JNIEXPORT jint JNICALL J(setThreadDevice)(JNIEnv* e, jclass c, jint dev) {
  (void)e; (void)c;
  return b2s_set_thread_device((uint32_t)dev);
}
JNIEXPORT jint JNICALL J(bindThreadToDevice)(JNIEnv* e, jclass c, jint dev) {
  (void)e; (void)c;
  return b2s_bind_thread_to_device((uint32_t)dev);
}
JNIEXPORT jstring JNICALL J(lastError)(JNIEnv* e, jclass c) {
  (void)c;
  return (*e)->NewStringUTF(e, b2s_last_error());
}
JNIEXPORT jstring JNICALL J(strerror)(JNIEnv* e, jclass c, jint code) {
  (void)c;
  return (*e)->NewStringUTF(e, b2s_strerror((int32_t)code));
}

/* ---- pinned host memory, handed to the JVM as direct ByteBuffers ---- */
JNIEXPORT jlong JNICALL J(hostAlloc)(JNIEnv* e, jclass c, jlong bytes) {
  (void)e; (void)c;
  return (jlong)(uintptr_t)b2s_host_alloc((uint64_t)bytes);
}
JNIEXPORT void JNICALL J(hostFree)(JNIEnv* e, jclass c, jlong addr) {
  (void)e; (void)c;
  b2s_host_free(PTR(void, addr));
}
JNIEXPORT jobject JNICALL J(wrap)(JNIEnv* e, jclass c, jlong addr, jlong bytes) {
  (void)c;
  return (*e)->NewDirectByteBuffer(e, PTR(void, addr), bytes);
}
JNIEXPORT jlong JNICALL J(addressOf)(JNIEnv* e, jclass c, jobject directBuffer) {
  (void)c;
  return (jlong)(uintptr_t)(*e)->GetDirectBufferAddress(e, directBuffer);
}
JNIEXPORT jint JNICALL J(hostRegister)(JNIEnv* e, jclass c, jlong addr, jlong bytes) {
  (void)e; (void)c;
  return b2s_host_register(PTR(void, addr), (uint64_t)bytes);
}
JNIEXPORT jint JNICALL J(hostUnregister)(JNIEnv* e, jclass c, jlong addr) {
  (void)e; (void)c;
  return b2s_host_unregister(PTR(void, addr));
}

/* ---- sizing ---- */
JNIEXPORT jlong JNICALL J(compressBound)(JNIEnv* e, jclass c, jint codec, jint blockSize, jlong n) {
  (void)e; (void)c;
  return (jlong)b2s_compress_bound((uint32_t)codec, (uint32_t)blockSize, (uint64_t)n);
}

/* ---- write side: n partition streams of one map task, packed arena in, packed .data arena out.
 *      off/len/dstOff/dstLen/checksums: long[n]; meta: long[1] = {dst_total}; status: int[n] ---- */
JNIEXPORT jint JNICALL J(compressPacked)(JNIEnv* e, jclass c, jint codec, jint level, jint blockSize, jint alg, jint n,
                                         jlong src, jlongArray off, jlongArray len, jlong dst, jlong dstCap,
                                         jlongArray dstOff, jlongArray dstLen, jlongArray meta, jlongArray checksums,
                                         jintArray status) {
  (void)c;
  if (n < 0 || !meta || (*e)->GetArrayLength(e, meta) < 1) return B2S_E_ARG;
  if (n > 0 && (!off || !len || !dstOff || !dstLen || !status || (*e)->GetArrayLength(e, off) < n ||
                (*e)->GetArrayLength(e, len) < n || (*e)->GetArrayLength(e, dstOff) < n ||
                (*e)->GetArrayLength(e, dstLen) < n || (*e)->GetArrayLength(e, status) < n ||
                (checksums && (*e)->GetArrayLength(e, checksums) < n)))
    return B2S_E_ARG;
  jlong* o = crit_get(e, off);
  jlong* l = crit_get(e, len);
  jlong* dO = crit_get(e, dstOff);
  jlong* dL = crit_get(e, dstLen);
  jlong* m = crit_get(e, meta);
  jlong* k = crit_get(e, checksums);
  jint* st = crit_get(e, status);
  const int rc = b2s_compress_packed((uint32_t)codec, (int32_t)level, (uint32_t)blockSize, (uint32_t)alg, (uint32_t)n,
                                     PTR(const uint8_t, src), (const uint64_t*)o, (const uint64_t*)l, PTR(uint8_t, dst),
                                     (uint64_t)dstCap, (uint64_t*)dO, (uint64_t*)dL, (uint64_t*)m, (uint64_t*)k,
                                     (int32_t*)st);
  crit_put(e, status, st, 0);
  crit_put(e, checksums, k, 0);
  crit_put(e, meta, m, 0);
  crit_put(e, dstLen, dL, 0);
  crit_put(e, dstOff, dO, 0);
  crit_put(e, len, l, JNI_ABORT); /* inputs: nothing to copy back */
  crit_put(e, off, o, JNI_ABORT);
  return rc;
}

/* ---- write side, serialized shuffle (ShuffleExternalSorter.insertRecord's records + partition ids): partition by
 *      reduce id and compress every partition in one call.  records / recLen (u32) / recPart (u32) / dst are direct
 *      buffer addresses (data-sized); dstOff/dstLen/checksums: long[numPartitions], status: int[numPartitions],
 *      meta: long[1] = {dst_total}.  The per-partition results are collected in native memory during the blocking
 *      call and copied out with Set<Type>ArrayRegion afterwards: no Java array is held in a critical region while the
 *      GPU works. ---- */
/* a composite key: int[n] key_type / key_off / key_len / key_null_field, as the C ABI's *_keys calls take them */
typedef struct {
  jint n; /* 1..16 columns */
  jintArray type, off, len, nullField;
} composite_key;
static int bad_keys(JNIEnv* e, const composite_key* keys) {
  return keys->n < 1 || keys->n > 16 || !keys->type || !keys->off || !keys->len || !keys->nullField ||
         (*e)->GetArrayLength(e, keys->type) < keys->n || (*e)->GetArrayLength(e, keys->off) < keys->n ||
         (*e)->GetArrayLength(e, keys->len) < keys->n || (*e)->GetArrayLength(e, keys->nullField) < keys->n;
}

/* a RangePartitioner's bounds: n rows framed as UnsafeRowSerializer writes them, back to back at the direct buffer
 * address rows (bytes long), their lengths int[n] len */
typedef struct {
  jint n;
  jlong rows, bytes;
  jintArray len;
} range_bounds;

/* cached (may be NULL): int[1], the cached store's flag; then (shuffleId, mapId) keys the exchange-cache entry.
 * hash (may be NULL): the records are serialized rows whose reduce ids are computed on the GPU
 * from these key columns, recPart is not read: Spark's HashPartitioning ids (partitionCompressRowsHashPacked), or with
 * range its RangePartitioner ids over those bounds (partitionCompressRowsRangePacked; numPartitions = range->n + 1).
 * rr (may be NULL; then hash is NULL): {startPosition, sortRows}, the records are serialized rows dealt out in Spark's
 * repartition(n) order (partitionCompressRowsRoundRobinPacked); recPart is not read */
static jint partition_compress(JNIEnv* e, jint shuffleId, jlong mapId, jintArray cached, const composite_key* hash,
                               const range_bounds* range, const jint* rr, jint codec, jint level, jint blockSize,
                               jint alg, jint numPartitions, jlong nRecords, jlong records, jlong recBytes, jlong recLen,
                               jlong recPart, jlong dst, jlong dstCap, jlongArray dstOff, jlongArray dstLen,
                               jlongArray meta, jlongArray checksums, jintArray status) {
  if ((cached && (*e)->GetArrayLength(e, cached) < 1) || numPartitions < 1 || !dstOff || !dstLen || !meta || !status || (*e)->GetArrayLength(e, dstOff) < numPartitions ||
      (*e)->GetArrayLength(e, dstLen) < numPartitions || (*e)->GetArrayLength(e, status) < numPartitions ||
      (*e)->GetArrayLength(e, meta) < 1 || (checksums && (*e)->GetArrayLength(e, checksums) < numPartitions))
    return B2S_E_ARG;
  if (hash && bad_keys(e, hash)) return B2S_E_ARG;
  if (range && (range->n < 0 || (range->n && (!range->len || (*e)->GetArrayLength(e, range->len) < range->n))))
    return B2S_E_ARG;
  uint32_t kt[16], ko[16], kl[16];
  int32_t knf[16];
  if (hash) {
    (*e)->GetIntArrayRegion(e, hash->type, 0, hash->n, (jint*)kt);
    (*e)->GetIntArrayRegion(e, hash->off, 0, hash->n, (jint*)ko);
    (*e)->GetIntArrayRegion(e, hash->len, 0, hash->n, (jint*)kl);
    (*e)->GetIntArrayRegion(e, hash->nullField, 0, hash->n, (jint*)knf);
  }
  const size_t R = (size_t)numPartitions;
  uint64_t* buf = (uint64_t*)malloc(R * 3 * sizeof(uint64_t));
  int32_t* st = (int32_t*)malloc(R * sizeof(int32_t));
  /* the bound lengths, copied out of the Java array so that none is held while the GPU works */
  uint32_t* bl = range ? (uint32_t*)malloc(((size_t)range->n + 1) * sizeof(uint32_t)) : 0;
  if (!buf || !st || (range && !bl)) {
    free(buf);
    free(st);
    free(bl);
    return B2S_E_NOMEM;
  }
  if (range && range->n) (*e)->GetIntArrayRegion(e, range->len, 0, range->n, (jint*)bl);
  uint64_t total = 0;
  int32_t stored = 0;
  const int rc =
      rr && cached ? b2s_partition_compress_rows_round_robin_cached_packed(
               (int32_t)shuffleId, (int64_t)mapId, (uint32_t)codec, (int32_t)level, (uint32_t)blockSize, (uint32_t)alg,
               (uint32_t)numPartitions, rr[0], (uint32_t)rr[1], (uint64_t)nRecords, PTR(const uint8_t, records),
               (uint64_t)recBytes, PTR(const uint32_t, recLen), PTR(uint8_t, dst), (uint64_t)dstCap, buf, buf + R,
               &total, buf + 2 * R, st, &stored)
      : rr ? b2s_partition_compress_rows_round_robin_packed(
               (uint32_t)codec, (int32_t)level, (uint32_t)blockSize, (uint32_t)alg, (uint32_t)numPartitions, rr[0],
               (uint32_t)rr[1], (uint64_t)nRecords, PTR(const uint8_t, records), (uint64_t)recBytes,
               PTR(const uint32_t, recLen), PTR(uint8_t, dst), (uint64_t)dstCap, buf, buf + R, &total, buf + 2 * R, st)
      : range && cached ? b2s_partition_compress_rows_range_cached_packed(
                  (int32_t)shuffleId, (int64_t)mapId, (uint32_t)codec, (int32_t)level, (uint32_t)blockSize,
                  (uint32_t)alg, (uint64_t)nRecords, PTR(const uint8_t, records), (uint64_t)recBytes,
                  PTR(const uint32_t, recLen), (uint32_t)hash->n, kt, ko, kl, knf, (uint32_t)range->n,
                  PTR(const uint8_t, range->rows), (uint64_t)range->bytes, bl, PTR(uint8_t, dst), (uint64_t)dstCap,
                  buf, buf + R, &total, buf + 2 * R, st, &stored)
      : range ? b2s_partition_compress_rows_range_packed(
                  (uint32_t)codec, (int32_t)level, (uint32_t)blockSize, (uint32_t)alg, (uint64_t)nRecords,
                  PTR(const uint8_t, records), (uint64_t)recBytes, PTR(const uint32_t, recLen), (uint32_t)hash->n, kt,
                  ko, kl, knf, (uint32_t)range->n, PTR(const uint8_t, range->rows), (uint64_t)range->bytes, bl,
                  PTR(uint8_t, dst), (uint64_t)dstCap, buf, buf + R, &total, buf + 2 * R, st)
      : hash && cached ? b2s_partition_compress_rows_hash_cached_packed(
                 (int32_t)shuffleId, (int64_t)mapId, (uint32_t)codec, (int32_t)level, (uint32_t)blockSize,
                 (uint32_t)alg, (uint32_t)numPartitions, (uint64_t)nRecords, PTR(const uint8_t, records),
                 (uint64_t)recBytes, PTR(const uint32_t, recLen), (uint32_t)hash->n, kt, ko, kl, knf, PTR(uint8_t, dst),
                 (uint64_t)dstCap, buf, buf + R, &total, buf + 2 * R, st, &stored)
      : hash ? b2s_partition_compress_rows_hash_packed(
                 (uint32_t)codec, (int32_t)level, (uint32_t)blockSize, (uint32_t)alg, (uint32_t)numPartitions,
                 (uint64_t)nRecords, PTR(const uint8_t, records), (uint64_t)recBytes, PTR(const uint32_t, recLen),
                 (uint32_t)hash->n, kt, ko, kl, knf, PTR(uint8_t, dst), (uint64_t)dstCap, buf, buf + R, &total,
                 buf + 2 * R, st)
      : cached ? b2s_partition_compress_cached_packed(
                   (int32_t)shuffleId, (int64_t)mapId, (uint32_t)codec, (int32_t)level, (uint32_t)blockSize,
                   (uint32_t)alg, (uint32_t)numPartitions, (uint64_t)nRecords, PTR(const uint8_t, records),
                   (uint64_t)recBytes, PTR(const uint32_t, recLen), PTR(const uint32_t, recPart), PTR(uint8_t, dst),
                   (uint64_t)dstCap, buf, buf + R, &total, buf + 2 * R, st, &stored)
             : b2s_partition_compress_packed(
                   (uint32_t)codec, (int32_t)level, (uint32_t)blockSize, (uint32_t)alg, (uint32_t)numPartitions,
                   (uint64_t)nRecords, PTR(const uint8_t, records), (uint64_t)recBytes, PTR(const uint32_t, recLen),
                   PTR(const uint32_t, recPart), PTR(uint8_t, dst), (uint64_t)dstCap, buf, buf + R, &total,
                   buf + 2 * R, st);
  if (cached) (*e)->SetIntArrayRegion(e, cached, 0, 1, (const jint*)&stored);
  if (rc == 0 || rc == B2S_E_DST_TOO_SMALL) {
    (*e)->SetLongArrayRegion(e, dstOff, 0, numPartitions, (const jlong*)buf);
    (*e)->SetLongArrayRegion(e, dstLen, 0, numPartitions, (const jlong*)(buf + R));
    if (checksums) (*e)->SetLongArrayRegion(e, checksums, 0, numPartitions, (const jlong*)(buf + 2 * R));
    (*e)->SetIntArrayRegion(e, status, 0, numPartitions, (const jint*)st);
  }
  const jlong m = (jlong)total;
  (*e)->SetLongArrayRegion(e, meta, 0, 1, &m);
  free(bl);
  free(st);
  free(buf);
  return rc;
}
JNIEXPORT jint JNICALL J(partitionCompressPacked)(JNIEnv* e, jclass c, jint codec, jint level, jint blockSize, jint alg,
                                                  jint numPartitions, jlong nRecords, jlong records, jlong recBytes,
                                                  jlong recLen, jlong recPart, jlong dst, jlong dstCap,
                                                  jlongArray dstOff, jlongArray dstLen, jlongArray meta,
                                                  jlongArray checksums, jintArray status) {
  (void)c;
  return partition_compress(e, 0, 0, 0, 0, 0, 0, codec, level, blockSize, alg, numPartitions, nRecords, records,
                            recBytes, recLen, recPart, dst, dstCap, dstOff, dstLen, meta, checksums, status);
}
/* HashPartitioning exchange of UnsafeRows (INTEGRATION.md §3j): records as UnsafeRowSerializer writes them, recLen
 * (u32) per record, no reduce ids: the GPU computes Spark's pmod(Murmur3Hash(key columns, 42), numPartitions).  The key
 * columns are int[nKeys] keyType / keyOff / keyLen / keyNullField; the rest as partitionCompressPacked */
JNIEXPORT jint JNICALL J(partitionCompressRowsHashPacked)(JNIEnv* e, jclass c, jint codec, jint level, jint blockSize,
                                                          jint alg, jint numPartitions, jlong nRecords, jlong records,
                                                          jlong recBytes, jlong recLen, jint nKeys, jintArray keyType,
                                                          jintArray keyOff, jintArray keyLen, jintArray keyNullField,
                                                          jlong dst, jlong dstCap, jlongArray dstOff,
                                                          jlongArray dstLen, jlongArray meta, jlongArray checksums,
                                                          jintArray status) {
  (void)c;
  const composite_key keys = {nKeys, keyType, keyOff, keyLen, keyNullField};
  return partition_compress(e, 0, 0, 0, &keys, 0, 0, codec, level, blockSize, alg, numPartitions, nRecords, records,
                            recBytes, recLen, 0, dst, dstCap, dstOff, dstLen, meta, checksums, status);
}
/* RangePartitioning exchange of UnsafeRows (INTEGRATION.md §3k): records and key columns as
 * partitionCompressRowsHashPacked (order flags allowed), no numPartitions: the RangePartitioner's nBounds bound rows
 * (UnsafeProjection(sort order children) rows, each with its int32 big-endian size prefix) lie back to back at the
 * direct buffer address bounds, boundBytes long, their lengths in int[nBounds] boundLen; the GPU computes every
 * record's RangePartitioner id, and dstOff / dstLen / checksums / status have nBounds + 1 entries.  The bounds are an
 * address rather than a byte[]: the exchange serialises them once into a direct buffer its map tasks share, and no
 * Java array is held while the GPU works (boundLen is copied out first) */
JNIEXPORT jint JNICALL J(partitionCompressRowsRangePacked)(JNIEnv* e, jclass c, jint codec, jint level, jint blockSize,
                                                           jint alg, jlong nRecords, jlong records, jlong recBytes,
                                                           jlong recLen, jint nKeys, jintArray keyType,
                                                           jintArray keyOff, jintArray keyLen, jintArray keyNullField,
                                                           jint nBounds, jlong bounds, jlong boundBytes,
                                                           jintArray boundLen, jlong dst, jlong dstCap,
                                                           jlongArray dstOff, jlongArray dstLen, jlongArray meta,
                                                           jlongArray checksums, jintArray status) {
  (void)c;
  if (nBounds < 0 || nBounds > (1 << 24) - 1) return B2S_E_ARG;
  const composite_key keys = {nKeys, keyType, keyOff, keyLen, keyNullField};
  const range_bounds range = {nBounds, bounds, boundBytes, boundLen};
  return partition_compress(e, 0, 0, 0, &keys, &range, 0, codec, level, blockSize, alg, nBounds + 1, nRecords, records,
                            recBytes, recLen, 0, dst, dstCap, dstOff, dstLen, meta, checksums, status);
}
/* RoundRobinPartitioning exchange of UnsafeRows (INTEGRATION.md §3l): records as partitionCompressRowsHashPacked, no
 * key columns: startPosition is new XORShiftRandom(partitionId).nextInt(numPartitions), sortRows (0 / 1) is
 * spark.sql.execution.sortBeforeRepartition; the GPU sorts the rows as UnsafeExternalRowSorter would and deals the
 * k-th to (startPosition + 1 + k) % numPartitions */
JNIEXPORT jint JNICALL J(partitionCompressRowsRoundRobinPacked)(JNIEnv* e, jclass c, jint codec, jint level,
                                                                jint blockSize, jint alg, jint numPartitions,
                                                                jint startPosition, jint sortRows, jlong nRecords,
                                                                jlong records, jlong recBytes, jlong recLen, jlong dst,
                                                                jlong dstCap, jlongArray dstOff, jlongArray dstLen,
                                                                jlongArray meta, jlongArray checksums,
                                                                jintArray status) {
  (void)c;
  const jint rr[2] = {startPosition, sortRows};
  return partition_compress(e, 0, 0, 0, 0, 0, rr, codec, level, blockSize, alg, numPartitions, nRecords, records,
                            recBytes, recLen, 0, dst, dstCap, dstOff, dstLen, meta, checksums, status);
}
/* the row writers' cached forms (INTEGRATION.md §3m): their arguments behind (shuffleId, mapId), and cached: int[1] =
 * stored; the entry keeps every record's offset, so a reducer's read marks its rows instead of walking them */
JNIEXPORT jint JNICALL J(partitionCompressRowsHashCachedPacked)(JNIEnv* e, jclass c, jint shuffleId, jlong mapId,
                                                                jint codec, jint level, jint blockSize, jint alg,
                                                                jint numPartitions, jlong nRecords, jlong records,
                                                                jlong recBytes, jlong recLen, jint nKeys,
                                                                jintArray keyType, jintArray keyOff, jintArray keyLen,
                                                                jintArray keyNullField, jlong dst, jlong dstCap,
                                                                jlongArray dstOff, jlongArray dstLen, jlongArray meta,
                                                                jlongArray checksums, jintArray status,
                                                                jintArray cached) {
  (void)c;
  if (!cached) return B2S_E_ARG;
  const composite_key keys = {nKeys, keyType, keyOff, keyLen, keyNullField};
  return partition_compress(e, shuffleId, mapId, cached, &keys, 0, 0, codec, level, blockSize, alg, numPartitions,
                            nRecords, records, recBytes, recLen, 0, dst, dstCap, dstOff, dstLen, meta, checksums,
                            status);
}
JNIEXPORT jint JNICALL J(partitionCompressRowsRangeCachedPacked)(JNIEnv* e, jclass c, jint shuffleId, jlong mapId,
                                                                 jint codec, jint level, jint blockSize, jint alg,
                                                                 jlong nRecords, jlong records, jlong recBytes,
                                                                 jlong recLen, jint nKeys, jintArray keyType,
                                                                 jintArray keyOff, jintArray keyLen,
                                                                 jintArray keyNullField, jint nBounds, jlong bounds,
                                                                 jlong boundBytes, jintArray boundLen, jlong dst,
                                                                 jlong dstCap, jlongArray dstOff, jlongArray dstLen,
                                                                 jlongArray meta, jlongArray checksums,
                                                                 jintArray status, jintArray cached) {
  (void)c;
  if (!cached || nBounds < 0 || nBounds > (1 << 24) - 1) return B2S_E_ARG;
  const composite_key keys = {nKeys, keyType, keyOff, keyLen, keyNullField};
  const range_bounds range = {nBounds, bounds, boundBytes, boundLen};
  return partition_compress(e, shuffleId, mapId, cached, &keys, &range, 0, codec, level, blockSize, alg, nBounds + 1,
                            nRecords, records, recBytes, recLen, 0, dst, dstCap, dstOff, dstLen, meta, checksums,
                            status);
}
JNIEXPORT jint JNICALL J(partitionCompressRowsRoundRobinCachedPacked)(JNIEnv* e, jclass c, jint shuffleId,
                                                                      jlong mapId, jint codec, jint level,
                                                                      jint blockSize, jint alg, jint numPartitions,
                                                                      jint startPosition, jint sortRows,
                                                                      jlong nRecords, jlong records, jlong recBytes,
                                                                      jlong recLen, jlong dst, jlong dstCap,
                                                                      jlongArray dstOff, jlongArray dstLen,
                                                                      jlongArray meta, jlongArray checksums,
                                                                      jintArray status, jintArray cached) {
  (void)c;
  if (!cached) return B2S_E_ARG;
  const jint rr[2] = {startPosition, sortRows};
  return partition_compress(e, shuffleId, mapId, cached, 0, 0, rr, codec, level, blockSize, alg, numPartitions,
                            nRecords, records, recBytes, recLen, 0, dst, dstCap, dstOff, dstLen, meta, checksums,
                            status);
}
/* the same, keeping the partitioned records in the exchange cache as (shuffleId, mapId); cached: int[1] = stored */
JNIEXPORT jint JNICALL J(partitionCompressCachedPacked)(JNIEnv* e, jclass c, jint shuffleId, jlong mapId, jint codec,
                                                        jint level, jint blockSize, jint alg, jint numPartitions,
                                                        jlong nRecords, jlong records, jlong recBytes, jlong recLen,
                                                        jlong recPart, jlong dst, jlong dstCap, jlongArray dstOff,
                                                        jlongArray dstLen, jlongArray meta, jlongArray checksums,
                                                        jintArray status, jintArray cached) {
  (void)c;
  if (!cached) return B2S_E_ARG;
  return partition_compress(e, shuffleId, mapId, cached, 0, 0, 0, codec, level, blockSize, alg, numPartitions,
                            nRecords, records, recBytes, recLen, recPart, dst, dstCap, dstOff, dstLen, meta, checksums,
                            status);
}

/* ---- read side: n prefetched blocks; block i owns slices [sliceBase[i], sliceBase[i+1]) of sliceLen/sliceChecksum
 *      (.index differences and .checksum values).  meta: long[1] = {dst_total}; status, badSlice: int[n] ---- */
JNIEXPORT jint JNICALL J(decompressPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n, jlong src, jlongArray off,
                                           jlongArray len, jintArray sliceBase, jlongArray sliceLen,
                                           jlongArray sliceChecksum, jlong dst, jlong dstCap, jlongArray dstOff,
                                           jlongArray dstLen, jlongArray meta, jintArray status, jintArray badSlice) {
  (void)c;
  if (n < 0 || !meta || (*e)->GetArrayLength(e, meta) < 1) return B2S_E_ARG;
  if (n > 0 && (!off || !len || !dstOff || !dstLen || !status || (*e)->GetArrayLength(e, off) < n ||
                (*e)->GetArrayLength(e, len) < n || (*e)->GetArrayLength(e, dstOff) < n ||
                (*e)->GetArrayLength(e, dstLen) < n || (*e)->GetArrayLength(e, status) < n ||
                (badSlice && (*e)->GetArrayLength(e, badSlice) < n)))
    return B2S_E_ARG;
  if (alg != 0 && n > 0) { /* block i's slices are [sliceBase[i], sliceBase[i+1]): sliceBase[n] sizes the slice arrays */
    if (!sliceBase || !sliceLen || !sliceChecksum || (*e)->GetArrayLength(e, sliceBase) < n + 1) return B2S_E_ARG;
    jint ns = 0;
    (*e)->GetIntArrayRegion(e, sliceBase, n, 1, &ns);
    if (ns < 0 || (*e)->GetArrayLength(e, sliceLen) < ns || (*e)->GetArrayLength(e, sliceChecksum) < ns)
      return B2S_E_ARG;
  }
  jlong* o = crit_get(e, off);
  jlong* l = crit_get(e, len);
  jint* sb = crit_get(e, sliceBase);
  jlong* sl = crit_get(e, sliceLen);
  jlong* sc = crit_get(e, sliceChecksum);
  jlong* dO = crit_get(e, dstOff);
  jlong* dL = crit_get(e, dstLen);
  jlong* m = crit_get(e, meta);
  jint* st = crit_get(e, status);
  jint* bad = crit_get(e, badSlice);
  const int rc = b2s_decompress_packed((uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src),
                                       (const uint64_t*)o, (const uint64_t*)l, (const uint32_t*)sb, (const uint64_t*)sl,
                                       (const uint64_t*)sc, PTR(uint8_t, dst), (uint64_t)dstCap, (uint64_t*)dO,
                                       (uint64_t*)dL, (uint64_t*)m, (int32_t*)st, (int32_t*)bad);
  crit_put(e, badSlice, bad, 0);
  crit_put(e, status, st, 0);
  crit_put(e, meta, m, 0);
  crit_put(e, dstLen, dL, 0);
  crit_put(e, dstOff, dO, 0);
  crit_put(e, sliceChecksum, sc, JNI_ABORT);
  crit_put(e, sliceLen, sl, JNI_ABORT);
  crit_put(e, sliceBase, sb, JNI_ABORT);
  crit_put(e, len, l, JNI_ABORT);
  crit_put(e, off, o, JNI_ABORT);
  return rc;
}

/* ---- read side, key-sorted (S3ShuffleReader.read with a key ordering, INTEGRATION.md §3e): verify, decode and sort
 *      the task's fixed-size records by key in one call.  src / dst are direct buffer addresses (data-sized); off/len:
 *      long[n], sliceBase: int[n+1], sliceLen/sliceChecksum: long[slices] (inputs, copied in with Get<Type>ArrayRegion);
 *      meta: long[2] = {dst_total, n_records}; status, badSlice: int[n].  All arrays go through native copies, so no
 *      Java array is held in a critical region while the GPU works. ---- */
/* mapIds (NULL: a plain decompressSortPacked): long[n] and cached: int[n] make it an exchange-cache read of the
 * partitions [startReduce, endReduce) of shuffleId (with keys: exchangeRead{Sort,Aggregate}RowsKeysPacked).  rows: a row sort (decompressSortRowsPacked) of UnsafeRow records
 * by the key keyType at keyOff (recordBytes unused, mapIds NULL).  aggOp (rows only; NULL otherwise): a row
 * aggregation (decompressAggregateRowsPacked) with int[nAggs] aggOp / aggOff / aggNullField, and meta long[3] =
 * {dst_total, n_records, n_groups}.  keys (rows only; NULL: the one key keyType / keyOff / keyLen / nullField): a
 * composite key (decompressSortRowsKeysPacked / decompressAggregateRowsKeysPacked) */
static jint sort_packed(JNIEnv* e, jint shuffleId, jint startReduce, jint endReduce, jlongArray mapIds,
                        jintArray cached, jint codec, jint alg, jint n, jlong src, jlongArray off, jlongArray len,
                        jintArray sliceBase, jlongArray sliceLen, jlongArray sliceChecksum, jint recordBytes,
                        int rows, jint keyType, jint keyOff, jint keyLen, jint nullField, const composite_key* keys,
                        jint nAggs, jintArray aggOp, jintArray aggOff, jintArray aggNullField, jlong dst, jlong dstCap,
                        jlongArray meta, jintArray status, jintArray badSlice) {
  const jsize n_meta = aggOp ? 3 : 2;
  if (n < 0 || !meta || (*e)->GetArrayLength(e, meta) < n_meta) return B2S_E_ARG;
  if (keys && bad_keys(e, keys)) return B2S_E_ARG;
  if (aggOp && (nAggs < 0 || nAggs > 16 || !aggOff || !aggNullField || (*e)->GetArrayLength(e, aggOp) < nAggs ||
                (*e)->GetArrayLength(e, aggOff) < nAggs || (*e)->GetArrayLength(e, aggNullField) < nAggs))
    return B2S_E_ARG;
  if (mapIds && n > 0 && (!cached || (*e)->GetArrayLength(e, mapIds) < n || (*e)->GetArrayLength(e, cached) < n))
    return B2S_E_ARG;
  if (n > 0 && (!off || !len || !status || (*e)->GetArrayLength(e, off) < n || (*e)->GetArrayLength(e, len) < n ||
                (*e)->GetArrayLength(e, status) < n || (badSlice && (*e)->GetArrayLength(e, badSlice) < n)))
    return B2S_E_ARG;
  const int with_slices = alg != 0 && n > 0;
  if (with_slices && (!sliceBase || !sliceLen || !sliceChecksum || (*e)->GetArrayLength(e, sliceBase) < n + 1))
    return B2S_E_ARG;
  const size_t N = (size_t)n;
  uint64_t* blk = (uint64_t*)malloc((N * 2 + 1) * sizeof(uint64_t));
  int32_t* st = (int32_t*)malloc((N * 2 + 1) * sizeof(int32_t));
  uint32_t* sb = (uint32_t*)malloc((N + 1) * sizeof(uint32_t));
  int64_t* ids = (int64_t*)malloc((N + 1) * sizeof(int64_t));
  uint8_t* hit = (uint8_t*)malloc(N + 1);
  uint64_t* sl = 0;
  int rc = blk && st && sb && ids && hit ? 0 : B2S_E_NOMEM;
  if (rc == 0 && n > 0) {
    (*e)->GetLongArrayRegion(e, off, 0, n, (jlong*)blk);
    (*e)->GetLongArrayRegion(e, len, 0, n, (jlong*)(blk + N));
    if (mapIds) {
      (*e)->GetLongArrayRegion(e, mapIds, 0, n, (jlong*)ids);
      (*e)->GetIntArrayRegion(e, cached, 0, n, (jint*)st); /* st is scratch until the call */
      for (size_t i = 0; i < N; i++) hit[i] = st[i] != 0;
    }
  }
  if (rc == 0 && with_slices) {
    (*e)->GetIntArrayRegion(e, sliceBase, 0, n + 1, (jint*)sb);
    const jsize ns = (jsize)sb[n];
    if (ns < 0 || (*e)->GetArrayLength(e, sliceLen) < ns || (*e)->GetArrayLength(e, sliceChecksum) < ns) {
      rc = B2S_E_ARG;
    } else if (!(sl = (uint64_t*)malloc(((size_t)ns * 2 + 1) * sizeof(uint64_t)))) {
      rc = B2S_E_NOMEM;
    } else {
      (*e)->GetLongArrayRegion(e, sliceLen, 0, ns, (jlong*)sl);
      (*e)->GetLongArrayRegion(e, sliceChecksum, 0, ns, (jlong*)(sl + ns));
    }
  }
  uint64_t total = 0, nrec = 0, ngrp = 0;
  if (rc == 0) {
    const size_t ns = with_slices ? (size_t)sb[n] : 0;
    uint32_t kt[16], ko[16], kl[16];
    int32_t knf[16];
    if (keys) {
      (*e)->GetIntArrayRegion(e, keys->type, 0, keys->n, (jint*)kt);
      (*e)->GetIntArrayRegion(e, keys->off, 0, keys->n, (jint*)ko);
      (*e)->GetIntArrayRegion(e, keys->len, 0, keys->n, (jint*)kl);
      (*e)->GetIntArrayRegion(e, keys->nullField, 0, keys->n, (jint*)knf);
    }
    if (aggOp) {
      uint32_t aop[16], aoff[16];
      int32_t anf[16];
      if (nAggs > 0) {
        (*e)->GetIntArrayRegion(e, aggOp, 0, nAggs, (jint*)aop);
        (*e)->GetIntArrayRegion(e, aggOff, 0, nAggs, (jint*)aoff);
        (*e)->GetIntArrayRegion(e, aggNullField, 0, nAggs, (jint*)anf);
      }
      if (keys && mapIds)
        rc = b2s_exchange_read_aggregate_rows_keys_packed(
            (int32_t)shuffleId, (int32_t)startReduce, (int32_t)endReduce, ids, hit, (uint32_t)codec, (uint32_t)alg,
            (uint32_t)n, PTR(const uint8_t, src), blk, blk + N, with_slices ? sb : 0, with_slices ? sl : 0,
            with_slices ? sl + ns : 0, (uint32_t)keys->n, kt, ko, kl, knf, (uint32_t)nAggs, aop, aoff, anf,
            PTR(uint8_t, dst), (uint64_t)dstCap, &total, &nrec, &ngrp, st, st + N);
      else if (keys)
        rc = b2s_decompress_aggregate_rows_keys_packed(
            (uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src), blk, blk + N, with_slices ? sb : 0,
            with_slices ? sl : 0, with_slices ? sl + ns : 0, (uint32_t)keys->n, kt, ko, kl, knf, (uint32_t)nAggs, aop,
            aoff, anf, PTR(uint8_t, dst), (uint64_t)dstCap, &total, &nrec, &ngrp, st, st + N);
      else
        rc = b2s_decompress_aggregate_rows_packed(
            (uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src), blk, blk + N, with_slices ? sb : 0,
            with_slices ? sl : 0, with_slices ? sl + ns : 0, (uint32_t)keyType, (uint32_t)keyOff, (uint32_t)keyLen,
            (int32_t)nullField, (uint32_t)nAggs, aop, aoff, anf, PTR(uint8_t, dst), (uint64_t)dstCap, &total, &nrec,
            &ngrp, st, st + N);
    } else if (keys && mapIds)
      rc = b2s_exchange_read_sort_rows_keys_packed(
          (int32_t)shuffleId, (int32_t)startReduce, (int32_t)endReduce, ids, hit, (uint32_t)codec, (uint32_t)alg,
          (uint32_t)n, PTR(const uint8_t, src), blk, blk + N, with_slices ? sb : 0, with_slices ? sl : 0,
          with_slices ? sl + ns : 0, (uint32_t)keys->n, kt, ko, kl, knf, PTR(uint8_t, dst), (uint64_t)dstCap, &total,
          &nrec, st, st + N);
    else if (keys)
      rc = b2s_decompress_sort_rows_keys_packed((uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src),
                                                blk, blk + N, with_slices ? sb : 0, with_slices ? sl : 0,
                                                with_slices ? sl + ns : 0, (uint32_t)keys->n, kt, ko, kl, knf,
                                                PTR(uint8_t, dst), (uint64_t)dstCap, &total, &nrec, st, st + N);
    else if (rows)
      rc = b2s_decompress_sort_rows_packed((uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src), blk,
                                           blk + N, with_slices ? sb : 0, with_slices ? sl : 0,
                                           with_slices ? sl + ns : 0, (uint32_t)keyType, (uint32_t)keyOff,
                                           (uint32_t)keyLen, (int32_t)nullField, PTR(uint8_t, dst), (uint64_t)dstCap,
                                           &total, &nrec, st, st + N);
    else if (mapIds)
      rc = b2s_exchange_read_sort_packed((int32_t)shuffleId, (int32_t)startReduce, (int32_t)endReduce, ids, hit,
                                         (uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src), blk,
                                         blk + N, with_slices ? sb : 0, with_slices ? sl : 0,
                                         with_slices ? sl + ns : 0, (uint32_t)recordBytes, (uint32_t)keyOff,
                                         (uint32_t)keyLen, PTR(uint8_t, dst), (uint64_t)dstCap, &total, &nrec, st,
                                         st + N);
    else
      rc = b2s_decompress_sort_packed((uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src), blk,
                                      blk + N, with_slices ? sb : 0, with_slices ? sl : 0, with_slices ? sl + ns : 0,
                                      (uint32_t)recordBytes, (uint32_t)keyOff, (uint32_t)keyLen, PTR(uint8_t, dst),
                                      (uint64_t)dstCap, &total, &nrec, st, st + N);
    if ((rc == 0 || rc == B2S_E_DST_TOO_SMALL) && n > 0) {
      (*e)->SetIntArrayRegion(e, status, 0, n, (const jint*)st);
      if (badSlice) (*e)->SetIntArrayRegion(e, badSlice, 0, n, (const jint*)(st + N));
    }
    const jlong m[3] = {(jlong)total, (jlong)nrec, (jlong)ngrp};
    (*e)->SetLongArrayRegion(e, meta, 0, n_meta, m);
  }
  free(hit);
  free(ids);
  free(sl);
  free(sb);
  free(st);
  free(blk);
  return rc;
}
JNIEXPORT jint JNICALL J(decompressSortPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n, jlong src,
                                               jlongArray off, jlongArray len, jintArray sliceBase, jlongArray sliceLen,
                                               jlongArray sliceChecksum, jint recordBytes, jint keyOff, jint keyLen,
                                               jlong dst, jlong dstCap, jlongArray meta, jintArray status,
                                               jintArray badSlice) {
  (void)c;
  return sort_packed(e, 0, 0, 0, 0, 0, codec, alg, n, src, off, len, sliceBase, sliceLen, sliceChecksum, recordBytes,
                     0, 0, keyOff, keyLen, -1, 0, 0, 0, 0, 0, dst, dstCap, meta, status, badSlice);
}

/* ---- read side, row-sorted (a Spark SQL exchange read followed by a SortExec, INTEGRATION.md §3g): verify, decode and
 *      sort the task's length-prefixed UnsafeRow records by one typed key (keyType B2S_KEY_*, keyOff in the row,
 *      nullField -1 or the key's null bit).  Arrays as decompressSortPacked. ---- */
JNIEXPORT jint JNICALL J(decompressSortRowsPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n, jlong src,
                                                   jlongArray off, jlongArray len, jintArray sliceBase,
                                                   jlongArray sliceLen, jlongArray sliceChecksum, jint keyType,
                                                   jint keyOff, jint keyLen, jint nullField, jlong dst, jlong dstCap,
                                                   jlongArray meta, jintArray status, jintArray badSlice) {
  (void)c;
  return sort_packed(e, 0, 0, 0, 0, 0, codec, alg, n, src, off, len, sliceBase, sliceLen, sliceChecksum, 0, 1, keyType,
                     keyOff, keyLen, nullField, 0, 0, 0, 0, 0, dst, dstCap, meta, status, badSlice);
}

/* ---- read side, aggregated (a Spark SQL exchange read followed by a HashAggregateExec(Final), INTEGRATION.md §3h):
 *      verify, decode, group the task's UnsafeRow records by one typed key and merge nAggs aggregates (aggOp /
 *      aggOff / aggNullField: int[nAggs], B2S_AGG_* ops, B2S_AGG_SUM_DECIMAL with its precision in bits 8..15).
 *      meta: long[3] = {dst_total, n_records, n_groups}; other arrays as decompressSortRowsPacked. ---- */
JNIEXPORT jint JNICALL J(decompressAggregateRowsPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n, jlong src,
                                                        jlongArray off, jlongArray len, jintArray sliceBase,
                                                        jlongArray sliceLen, jlongArray sliceChecksum, jint keyType,
                                                        jint keyOff, jint keyLen, jint nullField, jint nAggs,
                                                        jintArray aggOp, jintArray aggOff, jintArray aggNullField,
                                                        jlong dst, jlong dstCap, jlongArray meta, jintArray status,
                                                        jintArray badSlice) {
  (void)c;
  if (!aggOp) return B2S_E_ARG;
  return sort_packed(e, 0, 0, 0, 0, 0, codec, alg, n, src, off, len, sliceBase, sliceLen, sliceChecksum, 0, 1, keyType,
                     keyOff, keyLen, nullField, 0, nAggs, aggOp, aggOff, aggNullField, dst, dstCap, meta, status,
                     badSlice);
}

/* ---- read side, composite key (INTEGRATION.md §3g / §3h): the row sort and the row aggregation by nKeys (1..16)
 *      columns, strings included: keyType (B2S_KEY_*, B2S_STRING_KEY or B2S_DECIMAL_KEY, OR-ed with the order flags
 *      B2S_KEY_DESCENDING / B2S_KEY_NULLS_LAST; as a Java int the flags are plain bits 8 and 9) / keyOff / keyLen /
 *      keyNullField are int[nKeys], passed through unchanged; other arrays and meta as decompressSortRowsPacked /
 *      decompressAggregateRowsPacked. ---- */
JNIEXPORT jint JNICALL J(decompressSortRowsKeysPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n, jlong src,
                                                       jlongArray off, jlongArray len, jintArray sliceBase,
                                                       jlongArray sliceLen, jlongArray sliceChecksum, jint nKeys,
                                                       jintArray keyType, jintArray keyOff, jintArray keyLen,
                                                       jintArray keyNullField, jlong dst, jlong dstCap,
                                                       jlongArray meta, jintArray status, jintArray badSlice) {
  (void)c;
  const composite_key k = {nKeys, keyType, keyOff, keyLen, keyNullField};
  return sort_packed(e, 0, 0, 0, 0, 0, codec, alg, n, src, off, len, sliceBase, sliceLen, sliceChecksum, 0, 1, 0, 0, 0,
                     -1, &k, 0, 0, 0, 0, dst, dstCap, meta, status, badSlice);
}
JNIEXPORT jint JNICALL J(decompressAggregateRowsKeysPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n,
                                                            jlong src, jlongArray off, jlongArray len,
                                                            jintArray sliceBase, jlongArray sliceLen,
                                                            jlongArray sliceChecksum, jint nKeys, jintArray keyType,
                                                            jintArray keyOff, jintArray keyLen,
                                                            jintArray keyNullField, jint nAggs, jintArray aggOp,
                                                            jintArray aggOff, jintArray aggNullField, jlong dst,
                                                            jlong dstCap, jlongArray meta, jintArray status,
                                                            jintArray badSlice) {
  (void)c;
  if (!aggOp) return B2S_E_ARG;
  const composite_key k = {nKeys, keyType, keyOff, keyLen, keyNullField};
  return sort_packed(e, 0, 0, 0, 0, 0, codec, alg, n, src, off, len, sliceBase, sliceLen, sliceChecksum, 0, 1, 0, 0, 0,
                     -1, &k, nAggs, aggOp, aggOff, aggNullField, dst, dstCap, meta, status, badSlice);
}

/* ---- exchange cache (INTEGRATION.md §3f): map outputs kept in HBM for reducers on the same device ---- */
JNIEXPORT jint JNICALL J(exchangeSetBudget)(JNIEnv* e, jclass c, jint dev, jlong bytes) {
  (void)e; (void)c;
  return b2s_exchange_set_budget((uint32_t)dev, (uint64_t)bytes);
}
JNIEXPORT jint JNICALL J(exchangeRemove)(JNIEnv* e, jclass c, jint shuffleId, jlong mapId) {
  (void)e; (void)c;
  return b2s_exchange_remove((int32_t)shuffleId, (int64_t)mapId);
}
/* len: long[n] = bytes of [startReduce, endReduce) of each resident map, -1 (UINT64_MAX) otherwise; returns the hits */
JNIEXPORT jint JNICALL J(exchangeLookup)(JNIEnv* e, jclass c, jint shuffleId, jint startReduce, jint endReduce, jint n,
                                         jlongArray mapIds, jlongArray len) {
  (void)c;
  if (n < 0 || (n > 0 && (!mapIds || !len || (*e)->GetArrayLength(e, mapIds) < n || (*e)->GetArrayLength(e, len) < n)))
    return B2S_E_ARG;
  const size_t N = (size_t)n;
  uint64_t* buf = (uint64_t*)malloc((N * 2 + 1) * sizeof(uint64_t));
  if (!buf) return B2S_E_NOMEM;
  if (n > 0) (*e)->GetLongArrayRegion(e, mapIds, 0, n, (jlong*)buf);
  const int rc = b2s_exchange_lookup((int32_t)shuffleId, (int32_t)startReduce, (int32_t)endReduce, (uint32_t)n,
                                     (const int64_t*)buf, buf + N);
  if (rc >= 0 && n > 0) (*e)->SetLongArrayRegion(e, len, 0, n, (const jlong*)(buf + N));
  free(buf);
  return rc;
}
/* the cached ranges back to back into dst (a direct buffer address); dstOff/dstLen: long[n], status: int[n],
 * meta: long[1] = {dst_total} */
JNIEXPORT jint JNICALL J(exchangeReadPacked)(JNIEnv* e, jclass c, jint shuffleId, jint startReduce, jint endReduce,
                                             jint n, jlongArray mapIds, jlong dst, jlong dstCap, jlongArray dstOff,
                                             jlongArray dstLen, jlongArray meta, jintArray status) {
  (void)c;
  if (n < 0 || !meta || (*e)->GetArrayLength(e, meta) < 1) return B2S_E_ARG;
  if (n > 0 && (!mapIds || !dstOff || !dstLen || !status || (*e)->GetArrayLength(e, mapIds) < n ||
                (*e)->GetArrayLength(e, dstOff) < n || (*e)->GetArrayLength(e, dstLen) < n ||
                (*e)->GetArrayLength(e, status) < n))
    return B2S_E_ARG;
  const size_t N = (size_t)n;
  uint64_t* buf = (uint64_t*)malloc((N * 3 + 1) * sizeof(uint64_t));
  int32_t* st = (int32_t*)malloc((N + 1) * sizeof(int32_t));
  if (!buf || !st) {
    free(buf);
    free(st);
    return B2S_E_NOMEM;
  }
  if (n > 0) (*e)->GetLongArrayRegion(e, mapIds, 0, n, (jlong*)buf);
  uint64_t total = 0;
  const int rc = b2s_exchange_read_packed((int32_t)shuffleId, (int32_t)startReduce, (int32_t)endReduce, (uint32_t)n,
                                          (const int64_t*)buf, PTR(uint8_t, dst), (uint64_t)dstCap, buf + N,
                                          buf + 2 * N, &total, st);
  if (rc == 0 && n > 0) {
    (*e)->SetLongArrayRegion(e, dstOff, 0, n, (const jlong*)(buf + N));
    (*e)->SetLongArrayRegion(e, dstLen, 0, n, (const jlong*)(buf + 2 * N));
    (*e)->SetIntArrayRegion(e, status, 0, n, (const jint*)st);
  }
  const jlong m = (jlong)total;
  (*e)->SetLongArrayRegion(e, meta, 0, 1, &m);
  free(st);
  free(buf);
  return rc;
}
/* decompressSortPacked over sources of which those with cached[i] != 0 are the cached range of mapIds[i]
 * (mapIds: long[n], cached: int[n]); the other arguments as decompressSortPacked */
JNIEXPORT jint JNICALL J(exchangeReadSortPacked)(JNIEnv* e, jclass c, jint shuffleId, jint startReduce, jint endReduce,
                                                 jlongArray mapIds, jintArray cached, jint codec, jint alg, jint n,
                                                 jlong src, jlongArray off, jlongArray len, jintArray sliceBase,
                                                 jlongArray sliceLen, jlongArray sliceChecksum, jint recordBytes,
                                                 jint keyOff, jint keyLen, jlong dst, jlong dstCap, jlongArray meta,
                                                 jintArray status, jintArray badSlice) {
  (void)c;
  if (!mapIds) return B2S_E_ARG;
  return sort_packed(e, shuffleId, startReduce, endReduce, mapIds, cached, codec, alg, n, src, off, len, sliceBase,
                     sliceLen, sliceChecksum, recordBytes, 0, 0, keyOff, keyLen, -1, 0, 0, 0, 0, 0, dst, dstCap,
                     meta, status, badSlice);
}

/* a native copy of the first n elements (elem bytes each: 1 byte, 4 int, 8 long) of a Java array; NULL for a NULL
 * array.  *rc: B2S_E_ARG when the array is shorter than n, B2S_E_NOMEM when the copy cannot be had (nothing is done
 * once *rc is set) */
static void* region(JNIEnv* e, jarray a, jsize n, size_t elem, int* rc) {
  if (!a || *rc) return 0;
  if (n < 0 || (*e)->GetArrayLength(e, a) < n) {
    *rc = B2S_E_ARG;
    return 0;
  }
  void* p = malloc((size_t)n * elem + 1);
  if (!p) {
    *rc = B2S_E_NOMEM;
    return 0;
  }
  if (elem == 1) (*e)->GetByteArrayRegion(e, (jbyteArray)a, 0, n, (jbyte*)p);
  else if (elem == 4) (*e)->GetIntArrayRegion(e, (jintArray)a, 0, n, (jint*)p);
  else (*e)->GetLongArrayRegion(e, (jlongArray)a, 0, n, (jlong*)p);
  return p;
}
/* region of an array the call requires: a NULL one is B2S_E_ARG too */
static void* need(JNIEnv* e, jarray a, jsize n, size_t elem, int* rc) {
  if (!a && !*rc) *rc = B2S_E_ARG;
  return region(e, a, n, elem, rc);
}

/* ---- read side, sort-merge join (INTEGRATION.md §3n): blocks [0, nLeft) are the left side's, the rest the right's;
 *      joinType: B2S_JOIN_* (inner, left outer, left semi, left anti, right outer, full outer, existence).
 *      keyType / keyLen: int[nKeys] for both sides, a type OR-ed with B2S_KEY_NULL_SAFE for a <=> column;
 *      left/rightKeyOff and left/rightKeyNullField: int[nKeys] per side; left/rightFieldKind: byte[nFields] of
 *      B2S_FIELD_* (null for semi and anti joins; rightFieldKind null for existence joins); meta: long[4] = {dst_total,
 *      n_left_records, n_right_records, n_out_records}; other arrays as decompressSortRowsPacked.  Every array goes
 *      through a native copy. ---- */
JNIEXPORT jint JNICALL J(decompressJoinRowsKeysPacked)(JNIEnv* e, jclass c, jint joinType, jint codec, jint alg,
                                                       jint nLeft, jint n, jlong src, jlongArray off, jlongArray len,
                                                       jintArray sliceBase, jlongArray sliceLen,
                                                       jlongArray sliceChecksum, jint nKeys, jintArray keyType,
                                                       jintArray keyLen, jintArray leftKeyOff,
                                                       jintArray leftKeyNullField, jintArray rightKeyOff,
                                                       jintArray rightKeyNullField, jint nLeftFields,
                                                       jbyteArray leftFieldKind, jint nRightFields,
                                                       jbyteArray rightFieldKind, jlong dst, jlong dstCap,
                                                       jlongArray meta, jintArray status, jintArray badSlice) {
  (void)c;
  if (n < 0 || nKeys < 1 || nKeys > 16 || !meta || (*e)->GetArrayLength(e, meta) < 4) return B2S_E_ARG;
  if (n > 0 && (!status || (*e)->GetArrayLength(e, status) < n || (badSlice && (*e)->GetArrayLength(e, badSlice) < n)))
    return B2S_E_ARG;
  const int with_slices = alg != 0 && n > 0;
  int rc = 0;
  uint64_t* o = n > 0 ? need(e, off, n, 8, &rc) : 0;
  uint64_t* l = n > 0 ? need(e, len, n, 8, &rc) : 0;
  uint32_t* sb = with_slices ? need(e, sliceBase, n + 1, 4, &rc) : 0;
  const jsize ns = sb && !rc ? (jsize)sb[n] : 0;
  uint64_t* sl = with_slices ? need(e, sliceLen, ns, 8, &rc) : 0;
  uint64_t* sc = with_slices ? need(e, sliceChecksum, ns, 8, &rc) : 0;
  uint32_t* kt = need(e, keyType, nKeys, 4, &rc);
  uint32_t* kl = need(e, keyLen, nKeys, 4, &rc);
  uint32_t* lo = need(e, leftKeyOff, nKeys, 4, &rc);
  int32_t* ln = need(e, leftKeyNullField, nKeys, 4, &rc);
  uint32_t* ro = need(e, rightKeyOff, nKeys, 4, &rc);
  int32_t* rn = need(e, rightKeyNullField, nKeys, 4, &rc);
  uint8_t* lk = region(e, leftFieldKind, nLeftFields, 1, &rc);
  uint8_t* rk = region(e, rightFieldKind, nRightFields, 1, &rc);
  int32_t* st = (int32_t*)malloc((size_t)n * 2 * sizeof(int32_t) + 1);
  if (!rc && !st) rc = B2S_E_NOMEM;
  uint64_t m[4] = {0, 0, 0, 0};
  if (!rc) {
    rc = b2s_decompress_join_rows_keys_packed(
        (uint32_t)joinType, (uint32_t)codec, (uint32_t)alg, (uint32_t)nLeft, (uint32_t)n, PTR(const uint8_t, src), o,
        l, sb, sl, sc, (uint32_t)nKeys, kt, kl, lo, ln, ro, rn, (uint32_t)nLeftFields, lk, (uint32_t)nRightFields, rk,
        PTR(uint8_t, dst), (uint64_t)dstCap, &m[0], &m[1], &m[2], &m[3], st, st + n);
    (*e)->SetLongArrayRegion(e, meta, 0, 4, (const jlong*)m);
    if ((rc == 0 || rc == B2S_E_DST_TOO_SMALL) && n > 0) { /* a failed call leaves st unwritten */
      (*e)->SetIntArrayRegion(e, status, 0, n, (const jint*)st);
      if (badSlice) (*e)->SetIntArrayRegion(e, badSlice, 0, n, (const jint*)(st + n));
    }
  }
  void* owned[] = {o, l, sb, sl, sc, kt, kl, lo, ln, ro, rn, lk, rk, st};
  for (size_t i = 0; i < sizeof owned / sizeof owned[0]; i++) free(owned[i]);
  return rc;
}

/* ---- read side, window (INTEGRATION.md §3o): WindowExec's ranking functions over the task's rows; the first
 *      nPartitionKeys of the nKeys key columns (keyType / keyOff / keyLen / keyNullField: int[nKeys]) partition, the
 *      rest order; fieldKind: byte[nFields] of B2S_FIELD_*; fn / fnArg: int[nFns] (B2S_WINDOW_*, NTILE's bucket
 *      count); limitFn: B2S_WINDOW_NO_LIMIT (-1 as a Java int) or ROW_NUMBER / RANK / DENSE_RANK with limit; meta:
 *      long[3] = {dst_total, n_records, n_out_records}; other arrays as decompressSortRowsPacked.  Every array goes
 *      through a native copy. ---- */
JNIEXPORT jint JNICALL J(decompressWindowRowsKeysPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n, jlong src,
                                                         jlongArray off, jlongArray len, jintArray sliceBase,
                                                         jlongArray sliceLen, jlongArray sliceChecksum,
                                                         jint nPartitionKeys, jint nKeys, jintArray keyType,
                                                         jintArray keyOff, jintArray keyLen, jintArray keyNullField,
                                                         jint nFields, jbyteArray fieldKind, jint nFns, jintArray fn,
                                                         jintArray fnArg, jint limitFn, jint limit, jlong dst,
                                                         jlong dstCap, jlongArray meta, jintArray status,
                                                         jintArray badSlice) {
  (void)c;
  if (n < 0 || nKeys < 1 || nKeys > 16 || nFns < 1 || nFns > 16 || !meta || (*e)->GetArrayLength(e, meta) < 3)
    return B2S_E_ARG;
  if (n > 0 && (!status || (*e)->GetArrayLength(e, status) < n || (badSlice && (*e)->GetArrayLength(e, badSlice) < n)))
    return B2S_E_ARG;
  const int with_slices = alg != 0 && n > 0;
  int rc = 0;
  uint64_t* o = n > 0 ? need(e, off, n, 8, &rc) : 0;
  uint64_t* l = n > 0 ? need(e, len, n, 8, &rc) : 0;
  uint32_t* sb = with_slices ? need(e, sliceBase, n + 1, 4, &rc) : 0;
  const jsize ns = sb && !rc ? (jsize)sb[n] : 0;
  uint64_t* sl = with_slices ? need(e, sliceLen, ns, 8, &rc) : 0;
  uint64_t* sc = with_slices ? need(e, sliceChecksum, ns, 8, &rc) : 0;
  uint32_t* kt = need(e, keyType, nKeys, 4, &rc);
  uint32_t* ko = need(e, keyOff, nKeys, 4, &rc);
  uint32_t* kl = need(e, keyLen, nKeys, 4, &rc);
  int32_t* kn = need(e, keyNullField, nKeys, 4, &rc);
  uint8_t* fk = need(e, fieldKind, nFields, 1, &rc);
  uint32_t* fs = need(e, fn, nFns, 4, &rc);
  int32_t* fa = need(e, fnArg, nFns, 4, &rc);
  int32_t* st = (int32_t*)malloc((size_t)n * 2 * sizeof(int32_t) + 1);
  if (!rc && !st) rc = B2S_E_NOMEM;
  uint64_t m[3] = {0, 0, 0};
  if (!rc) {
    rc = b2s_decompress_window_rows_keys_packed(
        (uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src), o, l, sb, sl, sc,
        (uint32_t)nPartitionKeys, (uint32_t)nKeys, kt, ko, kl, kn, (uint32_t)nFields, fk, (uint32_t)nFns, fs, fa,
        (uint32_t)limitFn, (int32_t)limit, PTR(uint8_t, dst), (uint64_t)dstCap, &m[0], &m[1], &m[2], st, st + n);
    (*e)->SetLongArrayRegion(e, meta, 0, 3, (const jlong*)m);
    if ((rc == 0 || rc == B2S_E_DST_TOO_SMALL) && n > 0) { /* a failed call leaves st unwritten */
      (*e)->SetIntArrayRegion(e, status, 0, n, (const jint*)st);
      if (badSlice) (*e)->SetIntArrayRegion(e, badSlice, 0, n, (const jint*)(st + n));
    }
  }
  void* owned[] = {o, l, sb, sl, sc, kt, ko, kl, kn, fk, fs, fa, st};
  for (size_t i = 0; i < sizeof owned / sizeof owned[0]; i++) free(owned[i]);
  return rc;
}

/* ---- read side, window aggregates (INTEGRATION.md §3o): decompressWindowRowsKeysPacked without a limit, where fn may
 *      also hold aggregate functions (B2S_WINDOW_SUM .. AVG); fnFrame / valType / valOff / valNullField: int[nFns]
 *      (B2S_WINDOW_FRAME_*, B2S_WINDOW_VAL_* with a decimal's p << 8 | s << 16, the input's slot offset, its null bit
 *      or -1; 0, VAL_NONE, 0, -1 for a ranking function).  Every array goes through a native copy. ---- */
JNIEXPORT jint JNICALL J(decompressWindowAggregateRowsKeysPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n,
                                                                  jlong src, jlongArray off, jlongArray len,
                                                                  jintArray sliceBase, jlongArray sliceLen,
                                                                  jlongArray sliceChecksum, jint nPartitionKeys,
                                                                  jint nKeys, jintArray keyType, jintArray keyOff,
                                                                  jintArray keyLen, jintArray keyNullField,
                                                                  jint nFields, jbyteArray fieldKind, jint nFns,
                                                                  jintArray fn, jintArray fnArg, jintArray fnFrame,
                                                                  jintArray valType, jintArray valOff,
                                                                  jintArray valNullField, jlong dst, jlong dstCap,
                                                                  jlongArray meta, jintArray status,
                                                                  jintArray badSlice) {
  (void)c;
  if (n < 0 || nKeys < 1 || nKeys > 16 || nFns < 1 || nFns > 16 || !meta || (*e)->GetArrayLength(e, meta) < 3)
    return B2S_E_ARG;
  if (n > 0 && (!status || (*e)->GetArrayLength(e, status) < n || (badSlice && (*e)->GetArrayLength(e, badSlice) < n)))
    return B2S_E_ARG;
  const int with_slices = alg != 0 && n > 0;
  int rc = 0;
  uint64_t* o = n > 0 ? need(e, off, n, 8, &rc) : 0;
  uint64_t* l = n > 0 ? need(e, len, n, 8, &rc) : 0;
  uint32_t* sb = with_slices ? need(e, sliceBase, n + 1, 4, &rc) : 0;
  const jsize ns = sb && !rc ? (jsize)sb[n] : 0;
  uint64_t* sl = with_slices ? need(e, sliceLen, ns, 8, &rc) : 0;
  uint64_t* sc = with_slices ? need(e, sliceChecksum, ns, 8, &rc) : 0;
  uint32_t* kt = need(e, keyType, nKeys, 4, &rc);
  uint32_t* ko = need(e, keyOff, nKeys, 4, &rc);
  uint32_t* kl = need(e, keyLen, nKeys, 4, &rc);
  int32_t* kn = need(e, keyNullField, nKeys, 4, &rc);
  uint8_t* fk = need(e, fieldKind, nFields, 1, &rc);
  uint32_t* fs = need(e, fn, nFns, 4, &rc);
  int32_t* fa = need(e, fnArg, nFns, 4, &rc);
  uint32_t* fr = need(e, fnFrame, nFns, 4, &rc);
  uint32_t* vt = need(e, valType, nFns, 4, &rc);
  uint32_t* vo = need(e, valOff, nFns, 4, &rc);
  int32_t* vn = need(e, valNullField, nFns, 4, &rc);
  int32_t* st = (int32_t*)malloc((size_t)n * 2 * sizeof(int32_t) + 1);
  if (!rc && !st) rc = B2S_E_NOMEM;
  uint64_t m[3] = {0, 0, 0};
  if (!rc) {
    rc = b2s_decompress_window_aggregate_rows_keys_packed(
        (uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src), o, l, sb, sl, sc,
        (uint32_t)nPartitionKeys, (uint32_t)nKeys, kt, ko, kl, kn, (uint32_t)nFields, fk, (uint32_t)nFns, fs, fa, fr,
        vt, vo, vn, PTR(uint8_t, dst), (uint64_t)dstCap, &m[0], &m[1], &m[2], st, st + n);
    (*e)->SetLongArrayRegion(e, meta, 0, 3, (const jlong*)m);
    if ((rc == 0 || rc == B2S_E_DST_TOO_SMALL) && n > 0) { /* a failed call leaves st unwritten */
      (*e)->SetIntArrayRegion(e, status, 0, n, (const jint*)st);
      if (badSlice) (*e)->SetIntArrayRegion(e, badSlice, 0, n, (const jint*)(st + n));
    }
  }
  void* owned[] = {o, l, sb, sl, sc, kt, ko, kl, kn, fk, fs, fa, fr, vt, vo, vn, st};
  for (size_t i = 0; i < sizeof owned / sizeof owned[0]; i++) free(owned[i]);
  return rc;
}

/* ---- read side, window offsets (INTEGRATION.md §3o): decompressWindowAggregateRowsKeysPacked where fn may also hold
 *      offset functions (B2S_WINDOW_LAG .. NTH_VALUE, fnArg their offset or n, valType B2S_WINDOW_VAL_BYTES too);
 *      fnFlags: int[nFns] (B2S_WINDOW_IGNORE_NULLS | B2S_WINDOW_HAS_DEFAULT, 0 for every other function), fnDefault:
 *      long[nFns] (the default's slot bits).  Every array goes through a native copy. ---- */
JNIEXPORT jint JNICALL J(decompressWindowOffsetRowsKeysPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n,
                                                               jlong src, jlongArray off, jlongArray len,
                                                               jintArray sliceBase, jlongArray sliceLen,
                                                               jlongArray sliceChecksum, jint nPartitionKeys,
                                                               jint nKeys, jintArray keyType, jintArray keyOff,
                                                               jintArray keyLen, jintArray keyNullField,
                                                               jint nFields, jbyteArray fieldKind, jint nFns,
                                                               jintArray fn, jintArray fnArg, jintArray fnFrame,
                                                               jintArray valType, jintArray valOff,
                                                               jintArray valNullField, jintArray fnFlags,
                                                               jlongArray fnDefault, jlong dst, jlong dstCap,
                                                               jlongArray meta, jintArray status,
                                                               jintArray badSlice) {
  (void)c;
  if (n < 0 || nKeys < 1 || nKeys > 16 || nFns < 1 || nFns > 16 || !meta || (*e)->GetArrayLength(e, meta) < 3)
    return B2S_E_ARG;
  if (n > 0 && (!status || (*e)->GetArrayLength(e, status) < n || (badSlice && (*e)->GetArrayLength(e, badSlice) < n)))
    return B2S_E_ARG;
  const int with_slices = alg != 0 && n > 0;
  int rc = 0;
  uint64_t* o = n > 0 ? need(e, off, n, 8, &rc) : 0;
  uint64_t* l = n > 0 ? need(e, len, n, 8, &rc) : 0;
  uint32_t* sb = with_slices ? need(e, sliceBase, n + 1, 4, &rc) : 0;
  const jsize ns = sb && !rc ? (jsize)sb[n] : 0;
  uint64_t* sl = with_slices ? need(e, sliceLen, ns, 8, &rc) : 0;
  uint64_t* sc = with_slices ? need(e, sliceChecksum, ns, 8, &rc) : 0;
  uint32_t* kt = need(e, keyType, nKeys, 4, &rc);
  uint32_t* ko = need(e, keyOff, nKeys, 4, &rc);
  uint32_t* kl = need(e, keyLen, nKeys, 4, &rc);
  int32_t* kn = need(e, keyNullField, nKeys, 4, &rc);
  uint8_t* fk = need(e, fieldKind, nFields, 1, &rc);
  uint32_t* fs = need(e, fn, nFns, 4, &rc);
  int32_t* fa = need(e, fnArg, nFns, 4, &rc);
  uint32_t* fr = need(e, fnFrame, nFns, 4, &rc);
  uint32_t* vt = need(e, valType, nFns, 4, &rc);
  uint32_t* vo = need(e, valOff, nFns, 4, &rc);
  int32_t* vn = need(e, valNullField, nFns, 4, &rc);
  uint32_t* ff = need(e, fnFlags, nFns, 4, &rc);
  uint64_t* fd = need(e, fnDefault, nFns, 8, &rc);
  int32_t* st = (int32_t*)malloc((size_t)n * 2 * sizeof(int32_t) + 1);
  if (!rc && !st) rc = B2S_E_NOMEM;
  uint64_t m[3] = {0, 0, 0};
  if (!rc) {
    rc = b2s_decompress_window_offset_rows_keys_packed(
        (uint32_t)codec, (uint32_t)alg, (uint32_t)n, PTR(const uint8_t, src), o, l, sb, sl, sc,
        (uint32_t)nPartitionKeys, (uint32_t)nKeys, kt, ko, kl, kn, (uint32_t)nFields, fk, (uint32_t)nFns, fs, fa, fr,
        vt, vo, vn, ff, fd, PTR(uint8_t, dst), (uint64_t)dstCap, &m[0], &m[1], &m[2], st, st + n);
    (*e)->SetLongArrayRegion(e, meta, 0, 3, (const jlong*)m);
    if ((rc == 0 || rc == B2S_E_DST_TOO_SMALL) && n > 0) { /* a failed call leaves st unwritten */
      (*e)->SetIntArrayRegion(e, status, 0, n, (const jint*)st);
      if (badSlice) (*e)->SetIntArrayRegion(e, badSlice, 0, n, (const jint*)(st + n));
    }
  }
  void* owned[] = {o, l, sb, sl, sc, kt, ko, kl, kn, fk, fs, fa, fr, vt, vo, vn, ff, fd, st};
  for (size_t i = 0; i < sizeof owned / sizeof owned[0]; i++) free(owned[i]);
  return rc;
}

/* decompressSortRowsKeysPacked / decompressAggregateRowsKeysPacked over sources of which those with cached[i] != 0
 * are the cached range of mapIds[i] (INTEGRATION.md §3m; mapIds: long[n], cached: int[n]) */
JNIEXPORT jint JNICALL J(exchangeReadSortRowsKeysPacked)(JNIEnv* e, jclass c, jint shuffleId, jint startReduce,
                                                         jint endReduce, jlongArray mapIds, jintArray cached,
                                                         jint codec, jint alg, jint n, jlong src, jlongArray off,
                                                         jlongArray len, jintArray sliceBase, jlongArray sliceLen,
                                                         jlongArray sliceChecksum, jint nKeys, jintArray keyType,
                                                         jintArray keyOff, jintArray keyLen, jintArray keyNullField,
                                                         jlong dst, jlong dstCap, jlongArray meta, jintArray status,
                                                         jintArray badSlice) {
  (void)c;
  if (!mapIds) return B2S_E_ARG;
  const composite_key k = {nKeys, keyType, keyOff, keyLen, keyNullField};
  return sort_packed(e, shuffleId, startReduce, endReduce, mapIds, cached, codec, alg, n, src, off, len, sliceBase,
                     sliceLen, sliceChecksum, 0, 1, 0, 0, 0, -1, &k, 0, 0, 0, 0, dst, dstCap, meta, status,
                     badSlice);
}
JNIEXPORT jint JNICALL J(exchangeReadAggregateRowsKeysPacked)(JNIEnv* e, jclass c, jint shuffleId,
                                                              jint startReduce, jint endReduce, jlongArray mapIds,
                                                              jintArray cached, jint codec, jint alg, jint n,
                                                              jlong src, jlongArray off, jlongArray len,
                                                              jintArray sliceBase, jlongArray sliceLen,
                                                              jlongArray sliceChecksum, jint nKeys, jintArray keyType,
                                                              jintArray keyOff, jintArray keyLen,
                                                              jintArray keyNullField, jint nAggs, jintArray aggOp,
                                                              jintArray aggOff, jintArray aggNullField, jlong dst,
                                                              jlong dstCap, jlongArray meta, jintArray status,
                                                              jintArray badSlice) {
  (void)c;
  if (!mapIds || !aggOp) return B2S_E_ARG;
  const composite_key k = {nKeys, keyType, keyOff, keyLen, keyNullField};
  return sort_packed(e, shuffleId, startReduce, endReduce, mapIds, cached, codec, alg, n, src, off, len, sliceBase,
                     sliceLen, sliceChecksum, 0, 1, 0, 0, 0, -1, &k, nAggs, aggOp, aggOff, aggNullField, dst, dstCap,
                     meta, status, badSlice);
}

/* decoded size of each of n compressed streams laid out in one arena (sizes the destination of decompressPacked) */
JNIEXPORT jint JNICALL J(decompressedSizePacked)(JNIEnv* e, jclass c, jint codec, jint n, jlong src, jlongArray off,
                                                 jlongArray len, jlongArray outLen, jintArray status) {
  (void)c;
  enum { kStack = 256 };
  const uint8_t* ptrs_stack[kStack];
  const uint8_t** ptrs = ptrs_stack;
  if (n < 0 || (n > 0 && (!off || !len || !outLen || !status || (*e)->GetArrayLength(e, off) < n ||
                          (*e)->GetArrayLength(e, len) < n || (*e)->GetArrayLength(e, outLen) < n ||
                          (*e)->GetArrayLength(e, status) < n)))
    return B2S_E_ARG;
  jlong* o = crit_get(e, off);
  jlong* l = crit_get(e, len);
  jlong* out = crit_get(e, outLen);
  jint* st = crit_get(e, status);
  int rc = 0;
  /* the C entry point takes per-stream pointers; chunks of kStack streams keep the critical section allocation-free */
  for (jint i0 = 0; i0 < n && rc == 0; i0 += kStack) {
    const jint m = n - i0 < kStack ? n - i0 : kStack;
    for (jint i = 0; i < m; i++) ptrs[i] = PTR(const uint8_t, src) + (uint64_t)o[i0 + i];
    rc = b2s_decompressed_size_batch((uint32_t)codec, (uint32_t)m, ptrs, (const uint64_t*)(l + i0),
                                     (uint64_t*)(out + i0), (int32_t*)(st + i0));
  }
  crit_put(e, status, st, 0);
  crit_put(e, outLen, out, 0);
  crit_put(e, len, l, JNI_ABORT);
  crit_put(e, off, o, JNI_ABORT);
  return rc;
}

/* ---- checksums only: one value per slice of a packed arena ---- */
JNIEXPORT jint JNICALL J(checksumPacked)(JNIEnv* e, jclass c, jint alg, jint n, jlong base, jlongArray off, jlongArray len,
                                         jlongArray out) {
  (void)c;
  if (n < 0 || (n > 0 && (!off || !len || !out || (*e)->GetArrayLength(e, off) < n ||
                          (*e)->GetArrayLength(e, len) < n || (*e)->GetArrayLength(e, out) < n)))
    return B2S_E_ARG;
  jlong* o = crit_get(e, off);
  jlong* l = crit_get(e, len);
  jlong* r = crit_get(e, out);
  const int rc = b2s_checksum_packed((uint32_t)alg, (uint32_t)n, PTR(const uint8_t, base), (const uint64_t*)o,
                                     (const uint64_t*)l, (uint64_t*)r);
  crit_put(e, out, r, 0);
  crit_put(e, len, l, JNI_ABORT);
  crit_put(e, off, o, JNI_ABORT);
  return rc;
}

/* ---- observability: {total_ms, h2d_ms, d2h_ms, kernel_ms} x 1000 (microseconds) + byte counters of the calling
 *      thread's last call, for the MiB/s log lines of shuffle/S3MeasureOutputStream.scala:55-63 ---- */
JNIEXPORT jint JNICALL J(lastTiming)(JNIEnv* e, jclass c, jlongArray out8) {
  (void)c;
  if (!out8 || (*e)->GetArrayLength(e, out8) < 8) return B2S_E_ARG;
  b2s_timing t;
  const int rc = b2s_last_timing(&t);
  jlong* o = crit_get(e, out8);
  if (o) {
    o[0] = (jlong)(t.total_ms * 1000.0);
    o[1] = (jlong)(t.h2d_ms * 1000.0);
    o[2] = (jlong)(t.d2h_ms * 1000.0);
    o[3] = (jlong)(t.kernel_ms * 1000.0);
    o[4] = (jlong)t.h2d_bytes;
    o[5] = (jlong)t.d2h_bytes;
    o[6] = (jlong)t.src_bytes;
    o[7] = (jlong)t.dst_bytes;
  }
  crit_put(e, out8, o, 0);
  return rc;
}
