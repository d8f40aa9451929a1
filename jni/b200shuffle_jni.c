/*
 * b200shuffle_jni.c — the thin JNI layer between the Scala side of IBM/spark-s3-shuffle and libb200shuffle.so.
 *
 * One native method per C entry point a JVM needs (include/b200shuffle.h); the Scala object that declares them is
 * org.apache.spark.shuffle.gpu.B200Codec (INTEGRATION.md §2).  Call sites on the reference side:
 *   init / shutdown / bindThreadToDevice   shuffle/S3ShuffleDataIO.scala:30-32 (initializeExecutor), task threads
 *   compressPacked                         shuffle/S3ShuffleMapOutputWriter.scala:91-118 (commitAllPartitions)
 *   partitionCompressPacked                the GPU serialized writer (INTEGRATION.md §3d): records + reduce ids of a
 *                                          map task in, .data arena + partitionLengths + checksums out
 *   decompressPacked / decompressedSize    storage/S3ShuffleReader.scala:98-110 (the codec seam, batched drain of
 *                                          storage/S3BufferedPrefetchIterator.scala:196-212)
 *   checksumPacked                         shuffle/S3SingleSpillShuffleMapOutputWriter.scala:54-63,
 *                                          helper/S3ShuffleHelper.scala:94-103
 * Payload travels in pinned direct ByteBuffers (hostAlloc/wrap): the methods take raw addresses (jlong), so no
 * jbyteArray is ever pinned or copied; the small descriptor arrays (offsets, lengths, checksums, status) are Java
 * long[]/int[] accessed with Get/ReleasePrimitiveArrayCritical — every Get is paired with a Release on every path.
 *
 * Build (reference side):  cc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude \
 *                              jni/b200shuffle_jni.c -L. -lb200shuffle -o libb200shuffle_jni.so
 * Here (no JDK): tests/test_jni_shim.py compiles this file against jni/stub/jni.h with -Wall -Werror, so signatures,
 * argument order against b200shuffle.h and the Get/Release pairing are at least compiler- and script-checked.
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
/* cached (may be NULL): int[1], the cached store's flag; then (shuffleId, mapId) keys the exchange-cache entry */
static jint partition_compress(JNIEnv* e, jint shuffleId, jlong mapId, jintArray cached, jint codec, jint level,
                               jint blockSize, jint alg, jint numPartitions, jlong nRecords, jlong records,
                               jlong recBytes, jlong recLen, jlong recPart, jlong dst, jlong dstCap, jlongArray dstOff,
                               jlongArray dstLen, jlongArray meta, jlongArray checksums, jintArray status) {
  if ((cached && (*e)->GetArrayLength(e, cached) < 1) || numPartitions < 1 || !dstOff || !dstLen || !meta || !status || (*e)->GetArrayLength(e, dstOff) < numPartitions ||
      (*e)->GetArrayLength(e, dstLen) < numPartitions || (*e)->GetArrayLength(e, status) < numPartitions ||
      (*e)->GetArrayLength(e, meta) < 1 || (checksums && (*e)->GetArrayLength(e, checksums) < numPartitions))
    return B2S_E_ARG;
  const size_t R = (size_t)numPartitions;
  uint64_t* buf = (uint64_t*)malloc(R * 3 * sizeof(uint64_t));
  int32_t* st = (int32_t*)malloc(R * sizeof(int32_t));
  if (!buf || !st) {
    free(buf);
    free(st);
    return B2S_E_NOMEM;
  }
  uint64_t total = 0;
  int32_t stored = 0;
  const int rc =
      cached ? b2s_partition_compress_cached_packed(
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
  return partition_compress(e, 0, 0, 0, codec, level, blockSize, alg, numPartitions, nRecords, records, recBytes, recLen,
                            recPart, dst, dstCap, dstOff, dstLen, meta, checksums, status);
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
  return partition_compress(e, shuffleId, mapId, cached, codec, level, blockSize, alg, numPartitions, nRecords, records,
                            recBytes, recLen, recPart, dst, dstCap, dstOff, dstLen, meta, checksums, status);
}

/* ---- read side: n prefetched blocks; block i owns slices [sliceBase[i], sliceBase[i+1]) of sliceLen/sliceChecksum
 *      (.index differences and .checksum values).  meta: long[1] = {dst_total}; status, badSlice: int[n] ---- */
JNIEXPORT jint JNICALL J(decompressPacked)(JNIEnv* e, jclass c, jint codec, jint alg, jint n, jlong src, jlongArray off,
                                           jlongArray len, jintArray sliceBase, jlongArray sliceLen,
                                           jlongArray sliceChecksum, jlong dst, jlong dstCap, jlongArray dstOff,
                                           jlongArray dstLen, jlongArray meta, jintArray status, jintArray badSlice) {
  (void)c;
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
 * partitions [startReduce, endReduce) of shuffleId */
static jint sort_packed(JNIEnv* e, jint shuffleId, jint startReduce, jint endReduce, jlongArray mapIds,
                        jintArray cached, jint codec, jint alg, jint n, jlong src, jlongArray off, jlongArray len,
                        jintArray sliceBase, jlongArray sliceLen, jlongArray sliceChecksum, jint recordBytes,
                        jint keyOff, jint keyLen, jlong dst, jlong dstCap, jlongArray meta, jintArray status,
                        jintArray badSlice) {
  if (n < 0 || !meta || (*e)->GetArrayLength(e, meta) < 2) return B2S_E_ARG;
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
  uint64_t total = 0, nrec = 0;
  if (rc == 0) {
    const size_t ns = with_slices ? (size_t)sb[n] : 0;
    if (mapIds)
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
    const jlong m[2] = {(jlong)total, (jlong)nrec};
    (*e)->SetLongArrayRegion(e, meta, 0, 2, m);
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
                     keyOff, keyLen, dst, dstCap, meta, status, badSlice);
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
                     sliceLen, sliceChecksum, recordBytes, keyOff, keyLen, dst, dstCap, meta, status, badSlice);
}

/* decoded size of each of n compressed streams laid out in one arena (sizes the destination of decompressPacked) */
JNIEXPORT jint JNICALL J(decompressedSizePacked)(JNIEnv* e, jclass c, jint codec, jint n, jlong src, jlongArray off,
                                                 jlongArray len, jlongArray outLen, jintArray status) {
  (void)c;
  enum { kStack = 256 };
  const uint8_t* ptrs_stack[kStack];
  const uint8_t** ptrs = ptrs_stack;
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
  b2s_timing t;
  const int rc = b2s_last_timing(&t);
  if ((*e)->GetArrayLength(e, out8) < 8) return B2S_E_ARG;
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
