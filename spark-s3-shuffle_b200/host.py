"""ctypes binding of include/b200shuffle_host.h (libb200shuffle_host.so, the C++ host mirror of the reference's
plugin classes on the codec path).  Class and method names follow the reference so the tests read like
src/test/scala/org/apache/spark/shuffle/S3ShuffleManagerTest.scala; nothing here computes.
"""
import ctypes as C

import numpy as np

from . import _build
from .capi import (_agg_arrays, _arg, _join_arrays, _key_arrays, _window_aggregate_arrays, _window_arrays,
                   _window_offset_arrays, _window_frame_arrays)

OK, E_RUNTIME, E_IO, E_SPARK, E_UNSUPPORTED, E_CODEC = 0, -101, -102, -103, -104, -105


class RuntimeException(RuntimeError):
    """java.lang.RuntimeException (preconditions, length mismatch: shuffle/S3ShuffleMapOutputWriter.scala:68-73,96-100)"""


class IOException(IOError):
    """java.io.IOException (closed stream :175-177; "Stream is corrupted")"""


class SparkException(Exception):
    """org.apache.spark.SparkException (storage/S3ChecksumValidationStream.scala:72-74, helper/S3ShuffleHelper.scala:112-114)"""


class UnsupportedOperationException(Exception):
    """java.lang.UnsupportedOperationException (helper/S3ShuffleHelper.scala:100-101)"""


class CodecException(RuntimeError):
    """The C ABI reported a call-level failure (no GPU / CUDA error) — there is no CPU fallback."""


_EXC = {E_RUNTIME: RuntimeException, E_IO: IOException, E_SPARK: SparkException,
        E_UNSUPPORTED: UnsupportedOperationException, E_CODEC: CodecException}

_vp, _i32, _i64, _u32, _u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64
PROTOTYPES = [
    ("b2sh_last_error", C.c_char_p, []),
    ("b2sh_dispatcher_create", C.c_int, [C.c_char_p, C.POINTER(_vp)]),
    ("b2sh_dispatcher_destroy", None, [_vp]),
    ("b2sh_dispatcher_get_path", C.c_int, [_vp, C.c_int, _i32, _i64, C.c_char_p, _u32]),
    ("b2sh_dispatcher_remove_shuffle", C.c_int, [_vp, _i32]),
    ("b2sh_dispatcher_queue_compress", C.c_int,
     [_vp, _u32, _i32, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("b2sh_dispatcher_queue_decompress", C.c_int,
     [_vp, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("b2sh_dispatcher_queue_statistics", C.c_int, [_vp, C.POINTER(_u64)]),
    ("b2sh_helper_checksum_algorithm", C.c_int, [C.c_char_p]),
    ("b2sh_helper_get_partition_lengths", C.c_int, [_vp, _i32, _i64, _vp, _u32, C.POINTER(_u32)]),
    ("b2sh_helper_get_checksums", C.c_int, [_vp, _i32, _i64, _vp, _u32, C.POINTER(_u32)]),
    ("b2sh_writer_create", C.c_int, [_vp, _i32, _i64, _i32, C.POINTER(_vp)]),
    ("b2sh_writer_open_partition", C.c_int, [_vp, _i32]),
    ("b2sh_writer_write", C.c_int, [_vp, _vp, _u64]),
    ("b2sh_writer_close_partition", C.c_int, [_vp]),
    ("b2sh_writer_commit_all_partitions", C.c_int, [_vp, _vp, _vp]),
    ("b2sh_writer_abort", C.c_int, [_vp]),
    ("b2sh_writer_destroy", None, [_vp]),
    ("b2sh_single_spill_transfer", C.c_int, [_vp, _i32, _i64, C.c_char_p, _vp, _vp, _u32, C.c_int]),
    ("b2sh_reader_create", C.c_int, [_vp, _i32, _vp, _u32, _i32, _i32, C.c_int, C.POINTER(_vp)]),
    ("b2sh_reader_read", C.c_int, [_vp, C.POINTER(_u32)]),
    ("b2sh_reader_read_sorted", C.c_int,
     [_vp, _u32, _u32, _u32, C.POINTER(_vp), C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_reader_read_sorted_rows", C.c_int,
     [_vp, _u32, _u32, _u32, _i32, C.POINTER(_vp), C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_reader_read_aggregated_rows", C.c_int,
     [_vp, _u32, _u32, _u32, _i32, _u32, _vp, _vp, _vp, C.POINTER(_vp), C.POINTER(_u64), C.POINTER(_u64),
      C.POINTER(_u64)]),
    ("b2sh_reader_read_sorted_rows_keys", C.c_int,
     [_vp, _u32, _vp, _vp, _vp, _vp, C.POINTER(_vp), C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_reader_read_aggregated_rows_keys", C.c_int,
     [_vp, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _vp, _vp, C.POINTER(_vp), C.POINTER(_u64), C.POINTER(_u64),
      C.POINTER(_u64)]),
    ("b2sh_reader_read_joined_rows", C.c_int,
     [_vp, _vp, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _u32, _vp, _u32, _vp, C.POINTER(_vp), C.POINTER(_u64),
      C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_reader_aggregate_distinct_rows", C.c_int,
     [_vp, _vp, _u32, _u32, _vp, _vp, _u32, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp]),
    ("b2sh_reader_read_window_rows", C.c_int,
     [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _u32, _vp, _vp, _u32, _i32, C.POINTER(_vp), C.POINTER(_u64),
      C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_reader_read_window_aggregate_rows", C.c_int,
     [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(_vp),
      C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_reader_read_window_offset_rows", C.c_int,
     [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(_vp),
      C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_reader_read_window_frame_rows", C.c_int,
     [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
      C.POINTER(_vp), C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_reader_block", C.c_int,
     [_vp, _u32, C.POINTER(_i64), C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_vp), C.POINTER(_u64)]),
    ("b2sh_reader_remote_bytes_read", _u64, [_vp]),
    ("b2sh_reader_destroy", None, [_vp]),
    ("b2sh_serialized_writer_create", C.c_int, [_vp, _i32, _i64, _i32, C.POINTER(_vp)]),
    ("b2sh_serialized_writer_hash_rows", C.c_int, [_vp, _u32, _vp, _vp, _vp, _vp]),
    ("b2sh_serialized_writer_range_rows", C.c_int, [_vp, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _u64, _vp]),
    ("b2sh_serialized_writer_round_robin_rows", C.c_int, [_vp, _u32, _i32, _u32]),
    ("b2sh_serialized_writer_aggregate_rows", C.c_int, [_vp, _u32, _vp, _vp, _vp, _vp]),
    ("b2sh_serialized_writer_grouping_sets", C.c_int, [_vp, _u32, _vp]),
    ("b2sh_serialized_writer_window_limit", C.c_int, [_vp, _u32, _u32, _vp, _vp, _vp, _vp, _u32, _i32]),
    ("b2sh_serialized_writer_insert", C.c_int, [_vp, _i32, _vp, _u64]),
    ("b2sh_serialized_writer_commit", C.c_int, [_vp, _vp]),
    ("b2sh_serialized_writer_statistics", C.c_int, [_vp, C.POINTER(_u64), C.POINTER(_u64), C.c_char_p, _u32]),
    ("b2sh_serialized_writer_destroy", None, [_vp]),
    ("b2sh_writer_statistics", C.c_int, [_vp, C.POINTER(_u64), C.POINTER(_u64), C.c_char_p, _u32]),
    ("b2sh_reader_open", C.c_int, [_vp]),
    ("b2sh_reader_next_batch", C.c_int, [_vp, _u32, C.POINTER(_u32)]),
    ("b2sh_reader_statistics", C.c_int, [_vp, C.POINTER(_u64), C.POINTER(_u64), C.c_char_p, _u32]),
    ("b2sh_prefetch_create", C.c_int, [_vp, _i32, _vp, _u32, _i32, _i32, C.c_int, _i64, _i32, C.POINTER(_vp)]),
    ("b2sh_prefetch_has_next", C.c_int, [_vp]),
    ("b2sh_prefetch_next", C.c_int,
     [_vp, C.POINTER(_i64), C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_vp), C.POINTER(_u64), C.POINTER(_u64)]),
    ("b2sh_prefetch_close_stream", C.c_int, [_vp, _u64]),
    ("b2sh_prefetch_statistics", C.c_int, [_vp, C.POINTER(_u64), C.c_char_p, _u32]),
    ("b2sh_prefetch_destroy", None, [_vp]),
    ("b2sh_codec_create", C.c_int, [_vp, C.POINTER(_vp)]),
    ("b2sh_codec_supports_concatenation", C.c_int, [_vp]),
    ("b2sh_codec_destroy", None, [_vp]),
    ("b2sh_codec_output_stream", C.c_int, [_vp, _vp, _vp, C.POINTER(_vp)]),
    ("b2sh_ostream_write", C.c_int, [_vp, _vp, _u64]),
    ("b2sh_ostream_flush", C.c_int, [_vp]),
    ("b2sh_ostream_close", C.c_int, [_vp, C.POINTER(_u64), C.POINTER(_u64), C.POINTER(_u32)]),
    ("b2sh_ostream_destroy", None, [_vp]),
    ("b2sh_codec_input_stream", C.c_int, [_vp, _vp, _vp, C.POINTER(_vp)]),
    ("b2sh_istream_read", C.c_int, [_vp, _vp, _u64, C.POINTER(_i64)]),
    ("b2sh_istream_close", C.c_int, [_vp]),
    ("b2sh_istream_destroy", None, [_vp]),
]
SINK_FN = C.CFUNCTYPE(_i64, _vp, _vp, _u64)
SOURCE_FN = C.CFUNCTYPE(_i64, _vp, _vp, _u64)
STAT_KEYS = ("bytesRead", "numStreams", "timeWaiting", "timePrefetching", "totalRuntime", "activeThreads",
             "peakMemoryUsage", "peakThreads")
SYMBOLS = [p[0] for p in PROTOTYPES]
_lib = None


def load():
    global _lib
    if _lib is None:
        L = C.CDLL(_build.build_host())
        for name, res, args in PROTOTYPES:
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


def _check(rc):
    if rc < 0:
        raise _EXC.get(rc, RuntimeException)(load().b2sh_last_error().decode())
    return rc


class S3ShuffleDispatcher:
    """helper/S3ShuffleDispatcher.scala — conf is a dict of the reference's SparkConf keys."""

    def __init__(self, conf):
        text = "".join("%s=%s\n" % (k, str(v).lower() if isinstance(v, bool) else v) for k, v in conf.items())
        self._h = _vp()
        _check(load().b2sh_dispatcher_create(text.encode(), C.byref(self._h)))

    def getPath(self, kind, shuffleId, mapId):
        """kind: 'data' | 'index' | 'checksum' (helper/S3ShuffleDispatcher.scala:142-143)"""
        buf = C.create_string_buffer(4096)
        _check(load().b2sh_dispatcher_get_path(self._h, {"data": 0, "index": 1, "checksum": 2}[kind], shuffleId, mapId,
                                               buf, 4096))
        return buf.value.decode()

    def removeShuffle(self, shuffleId):
        _check(load().b2sh_dispatcher_remove_shuffle(self._h, shuffleId))

    # ---- the executor's group-commit queue (spark-s3-shuffle_b200/host/coalesce.h) ----
    def queueStatistics(self):
        v = (_u64 * 4)()
        _check(load().b2sh_dispatcher_queue_statistics(self._h, v))
        return dict(zip(("calls", "batches", "maxMerged", "streams"), list(v)))

    def queueCompress(self, codec, parts, blockSize=32768, checksumAlg=0, bound=None):
        """parts: list of bytes -> (streams, checksums, status); merged with whatever other threads submit meanwhile"""
        n = len(parts)
        srcs = [np.frombuffer(p, dtype=np.uint8) if len(p) else np.zeros(1, np.uint8) for p in parts]
        lens = np.array([len(p) for p in parts], dtype=np.uint64)
        caps = np.array([bound(len(p)) for p in parts], dtype=np.uint64)
        dsts = [np.empty(max(int(c), 1), dtype=np.uint8) for c in caps]
        sp = (_vp * n)(*[a.ctypes.data for a in srcs])
        dp = (_vp * n)(*[a.ctypes.data for a in dsts])
        dlen, cks, st = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.int32)
        _check(load().b2sh_dispatcher_queue_compress(self._h, codec, 0, blockSize, checksumAlg, n, sp, lens.ctypes.data,
                                                     dp, caps.ctypes.data, dlen.ctypes.data, cks.ctypes.data,
                                                     st.ctypes.data))
        return [d[: int(l)].tobytes() for d, l in zip(dsts, dlen)], [int(x) for x in cks], [int(x) for x in st]

    def queueDecompress(self, codec, streams, sizes):
        """streams: list of bytes, sizes: their decoded sizes -> (outputs, status)"""
        n = len(streams)
        srcs = [np.frombuffer(p, dtype=np.uint8) for p in streams]
        lens = np.array([len(p) for p in streams], dtype=np.uint64)
        caps = np.array(sizes, dtype=np.uint64)
        dsts = [np.empty(max(int(c), 1), dtype=np.uint8) for c in caps]
        sp = (_vp * n)(*[a.ctypes.data for a in srcs])
        dp = (_vp * n)(*[a.ctypes.data for a in dsts])
        dlen, st = np.zeros(n, np.uint64), np.zeros(n, np.int32)
        _check(load().b2sh_dispatcher_queue_decompress(self._h, codec, 0, n, sp, lens.ctypes.data, None, None, None, dp,
                                                       caps.ctypes.data, dlen.ctypes.data, st.ctypes.data, None))
        return [d[: int(l)].tobytes() for d, l in zip(dsts, dlen)], [int(x) for x in st]

    def close(self):
        if self._h:
            load().b2sh_dispatcher_destroy(self._h)
            self._h = None


class S3ShuffleHelper:
    """helper/S3ShuffleHelper.scala"""

    @staticmethod
    def createChecksumAlgorithm(name):
        return _check(load().b2sh_helper_checksum_algorithm(name.encode()))

    @staticmethod
    def _array(fn, d, shuffleId, mapId):
        cap = 1 << 16
        while True:
            out = np.zeros(cap, dtype=np.int64)
            cnt = _u32(0)
            rc = fn(d._h, shuffleId, mapId, out.ctypes.data, cap, C.byref(cnt))
            if rc == E_RUNTIME and cnt.value > cap:
                cap = cnt.value
                continue
            _check(rc)
            return out[: cnt.value].copy()

    @staticmethod
    def getPartitionLengths(d, shuffleId, mapId):
        """the cumulative offsets stored in .index (:67-81)"""
        return S3ShuffleHelper._array(load().b2sh_helper_get_partition_lengths, d, shuffleId, mapId)

    @staticmethod
    def getChecksums(d, shuffleId, mapId):
        return S3ShuffleHelper._array(load().b2sh_helper_get_checksums, d, shuffleId, mapId)


class S3ShuffleMapOutputWriter:
    """shuffle/S3ShuffleMapOutputWriter.scala — getPartitionWriter(p) returns a stream-like object."""

    class _PartitionStream:
        def __init__(self, w):
            self._w = w

        def write(self, data):
            a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
            _check(load().b2sh_writer_write(self._w._h, a.ctypes.data if a.size else None, a.size))

        def close(self):
            _check(load().b2sh_writer_close_partition(self._w._h))

        def __enter__(self):
            return self

        def __exit__(self, *a):
            self.close()

    def __init__(self, dispatcher, shuffleId, mapId, numPartitions):
        self._h = _vp()
        self.numPartitions = numPartitions
        _check(load().b2sh_writer_create(dispatcher._h, shuffleId, mapId, numPartitions, C.byref(self._h)))

    def getPartitionWriter(self, reducePartitionId):
        _check(load().b2sh_writer_open_partition(self._h, reducePartitionId))
        return self._PartitionStream(self)

    def commitAllPartitions(self, checksums=None):
        """-> partitionLengths (MapOutputCommitMessage).  checksums are only consumed in pass-through mode."""
        out = np.zeros(max(self.numPartitions, 1), dtype=np.int64)
        ck = None
        if checksums is not None:
            ck = np.ascontiguousarray(checksums, dtype=np.int64)
            assert ck.size == self.numPartitions
        _check(load().b2sh_writer_commit_all_partitions(self._h, ck.ctypes.data if ck is not None else None,
                                                        out.ctypes.data))
        return out[: self.numPartitions]

    def abort(self):
        _check(load().b2sh_writer_abort(self._h))

    def statistics(self):
        """S3MeasureOutputStream's counters for the .data stream: (bytes, nanoseconds, log line)"""
        b, ns, line = _u64(), _u64(), C.create_string_buffer(512)
        _check(load().b2sh_writer_statistics(self._h, C.byref(b), C.byref(ns), line, 512))
        return b.value, ns.value, line.value.decode()

    def close(self):
        if self._h:
            load().b2sh_writer_destroy(self._h)
            self._h = None


class S3SerializedShuffleWriter:
    """The GPU serialized writer (UnsafeShuffleWriter + ShuffleExternalSorter for a SerializedShuffleHandle):
    insertRecord(partitionId, record) in any partition order; commit() partitions, compresses and checksums on the GPU
    in one call and writes .data/.index/.checksum as S3ShuffleMapOutputWriter.commitAllPartitions does."""

    def __init__(self, dispatcher, shuffleId, mapId, numPartitions):
        self._h = _vp()
        self.numPartitions = numPartitions
        _check(load().b2sh_serialized_writer_create(dispatcher._h, shuffleId, mapId, numPartitions, C.byref(self._h)))

    def hashRows(self, keys):
        """HashPartitioning by keys = [(key_type, key_off, key_len, null_field), ...], before the first insert: each
        later record is one serialized row, its partitionId ignored; commit() computes Spark's ids on the GPU"""
        keys = list(keys)
        arrs = [np.array([k[i] for k in keys] or [0], dtype=np.int32 if i == 3 else np.uint32) for i in range(4)]
        _check(load().b2sh_serialized_writer_hash_rows(self._h, len(keys), *[a.ctypes.data for a in arrs]))

    def rangeRows(self, keys, bounds):
        """RangePartitioning by keys (as hashRows, order flags allowed) over bounds = the RangePartitioner's bound rows,
        each framed as UnsafeRowSerializer writes it, before the first insert; len(bounds) + 1 must be numPartitions"""
        keys, bounds = list(keys), [bytes(b) for b in bounds]
        arrs = [np.array([k[i] for k in keys] or [0], dtype=np.int32 if i == 3 else np.uint32) for i in range(4)]
        base = np.frombuffer(b"".join(bounds) or b"\0", dtype=np.uint8).copy()
        bl = np.array([len(b) for b in bounds] or [0], dtype=np.uint32)
        _check(load().b2sh_serialized_writer_range_rows(self._h, len(keys), *[a.ctypes.data for a in arrs], len(bounds),
                                                        base.ctypes.data, sum(len(b) for b in bounds), bl.ctypes.data))

    def roundRobinRows(self, numPartitions, startPosition, sortRows):
        """RoundRobinPartitioning (Spark's repartition(n)) from startPosition, the rows sorted first when sortRows,
        before the first insert; numPartitions must be the writer's"""
        _check(load().b2sh_serialized_writer_round_robin_rows(self._h, numPartitions, startPosition, int(sortRows)))

    def aggregateRows(self, aggs):
        """the map side's partial aggregation, after hashRows and before the first insert: aggs = [(fn, val_type,
        val_off, val_null_field), ...] as capi.aggregate_partition_compress_rows_hash_packed takes them; commit() writes
        one partial row per key of hashRows' key columns, hash-partitioned"""
        aggs = list(aggs)
        arrs = [np.array([a[i] for a in aggs] or [0], dtype=np.int32 if i == 3 else np.uint32) for i in range(4)]
        _check(load().b2sh_serialized_writer_aggregate_rows(self._h, len(aggs), *[a.ctypes.data for a in arrs]))

    def groupingSets(self, masks):
        """the grouping sets of a ROLLUP, CUBE or GROUPING SETS aggregation, after aggregateRows and before the first
        insert: masks = [bit c set when hashRows' key column c is in the set, ...]; commit() writes the partial rows
        keyed by the grouping columns and spark_grouping_id"""
        m = np.array(list(masks) or [0], dtype=np.uint32)
        _check(load().b2sh_serialized_writer_grouping_sets(self._h, len(masks), m.ctypes.data))

    def windowLimitRows(self, keys, nPartitionKeys, limitFn, limit):
        """the partial limit of a top-N-per-group window, in place of hashRows and before the first insert: keys = the
        window key as hashRows takes it (the first nPartitionKeys the PARTITION BY columns, then the ORDER BY columns,
        order flags allowed); commit() sorts the rows, keeps those whose limitFn value in their partition is at most
        limit and hash-partitions them by the partition columns"""
        keys = list(keys)
        arrs = [np.array([k[i] for k in keys] or [0], dtype=np.int32 if i == 3 else np.uint32) for i in range(4)]
        _check(load().b2sh_serialized_writer_window_limit(self._h, nPartitionKeys, len(keys),
                                                          *[a.ctypes.data for a in arrs], limitFn, limit))

    def insertRecord(self, partitionId, record):
        a = np.frombuffer(record, dtype=np.uint8) if not isinstance(record, np.ndarray) else np.ascontiguousarray(record)
        _check(load().b2sh_serialized_writer_insert(self._h, partitionId, a.ctypes.data if a.size else None, a.size))

    def commit(self):
        """-> partitionLengths (MapOutputCommitMessage)"""
        out = np.zeros(self.numPartitions, dtype=np.int64)
        _check(load().b2sh_serialized_writer_commit(self._h, out.ctypes.data))
        return out

    def statistics(self):
        b, ns, line = _u64(), _u64(), C.create_string_buffer(512)
        _check(load().b2sh_serialized_writer_statistics(self._h, C.byref(b), C.byref(ns), line, 512))
        return b.value, ns.value, line.value.decode()

    def close(self):
        if self._h:
            load().b2sh_serialized_writer_destroy(self._h)
            self._h = None


class S3SingleSpillShuffleMapOutputWriter:
    """shuffle/S3SingleSpillShuffleMapOutputWriter.scala"""

    def __init__(self, dispatcher, shuffleId, mapId):
        self._d, self.shuffleId, self.mapId = dispatcher, shuffleId, mapId

    def transferMapSpillFile(self, mapSpillFile, partitionLengths, checksums, verifyOnTransfer=False):
        pl = np.ascontiguousarray(partitionLengths, dtype=np.int64)
        ck = np.ascontiguousarray(checksums, dtype=np.int64)
        assert pl.size == ck.size
        _check(load().b2sh_single_spill_transfer(self._d._h, self.shuffleId, self.mapId, str(mapSpillFile).encode(),
                                                 pl.ctypes.data, ck.ctypes.data, pl.size, int(verifyOnTransfer)))


def _read_sorted(h, fn, *args, groups=False):
    """fn(h, *args, &data, &len, &records[, &groups]): one of the reader's sorted reads, numpy arrays in args passed as
    pointers.  -> (bytes, number of records[, number of groups])"""
    p, ln, nrec, ngrp = _vp(), _u64(), _u64(), _u64()
    counts = (nrec, ngrp) if groups else (nrec,)
    _check(fn(h, *map(_arg, args), C.byref(p), C.byref(ln), *map(C.byref, counts)))
    return ((C.string_at(p.value, ln.value) if ln.value else b""),) + tuple(c.value for c in counts)


class S3ShuffleReader:
    """storage/S3ShuffleReader.scala — read() yields (blockName-parts, decoded bytes) per non-empty block."""

    def __init__(self, dispatcher, shuffleId, mapIds, startPartition, endPartition, doBatchFetch=False):
        self._h = _vp()
        ids = np.ascontiguousarray(mapIds, dtype=np.int64)
        _check(load().b2sh_reader_create(dispatcher._h, shuffleId, ids.ctypes.data, ids.size, startPartition,
                                         endPartition, int(doBatchFetch), C.byref(self._h)))

    def read(self):
        n = _u32(0)
        _check(load().b2sh_reader_read(self._h, C.byref(n)))
        return self._blocks(n.value)

    def readSorted(self, recordBytes, keyOffset, keyLength):
        """read() with a key ordering (spark.shuffle.s3.gpu.sortKey=recordBytes,keyOffset,keyLength): every record
        of the task in ascending unsigned-byte key order, stable.  -> (bytes, number of records)"""
        return _read_sorted(self._h, load().b2sh_reader_read_sorted, recordBytes, keyOffset, keyLength)

    def readSortedRows(self, keyType, keyOffset, keyLength, nullField=-1):
        """read() of a SQL exchange sorted by one typed key (spark.shuffle.s3.gpu.sortRows): every UnsafeRowSerializer
        record of the task in ascending key order, nulls first, stable.  With the exchange cache on, resident maps are
        read from it.  -> (bytes, number of records)"""
        return _read_sorted(self._h, load().b2sh_reader_read_sorted_rows, keyType, keyOffset, keyLength, nullField)

    def readAggregatedRows(self, keyType, keyOffset, keyLength, nullField=-1, aggs=()):
        """read() of a SQL exchange whose partial aggregates are merged by one typed key
        (spark.shuffle.s3.gpu.aggregateRows): one UnsafeRowSerializer record per key, in the row sort's order, with
        each aggregate (op, offset, null field) merged over the key's records.  With the exchange cache on, resident
        maps are read from it.  -> (bytes, number of input records, number of groups)"""
        return _read_sorted(self._h, load().b2sh_reader_read_aggregated_rows, keyType, keyOffset, keyLength,
                            nullField, *_agg_arrays(aggs), groups=True)

    def readSortedRowsKeys(self, keys):
        """readSortedRows by a composite key: keys = [(keyType, keyOffset, keyLength, nullField), ...], compared left
        to right.  keyType: KEY_* or STRING_KEY / DECIMAL_KEY, OR-ed with KEY_DESCENDING and / or KEY_NULLS_LAST
        (capi.decompress_sort_rows_keys_packed).  -> (bytes, number of records)"""
        return _read_sorted(self._h, load().b2sh_reader_read_sorted_rows_keys, *_key_arrays(keys))

    def readAggregatedRowsKeys(self, keys, aggs=()):
        """readAggregatedRows grouped by a composite key (keys as in readSortedRowsKeys, flags included: groups come
        out in that order; floats group by Spark SQL's equality, 0.0 with -0.0 and NaN with NaN).
        -> (bytes, number of input records, number of groups)"""
        return _read_sorted(self._h, load().b2sh_reader_read_aggregated_rows_keys, *_key_arrays(keys),
                            *_agg_arrays(aggs), groups=True)

    def readJoinedRows(self, right, joinType, leftKeys, rightKeys, nLeftFields, nRightFields, leftKinds=None,
                       rightKinds=None):
        """Spark's sort-merge join of this reader's partitions (the left side) with right's (the same partitions of
        another shuffle): both readers' blocks through ONE capi.decompress_join_rows_keys_packed call, whose arguments
        these are (joinType: any capi.JOIN_*, right and full outer included).
        -> (joined rows, n_left_records, n_right_records, n_out_records)"""
        n, kt, kl, lo, ln, ro, rn, lk, rk = _join_arrays(leftKeys, rightKeys, leftKinds, rightKinds)
        p, size = _vp(), _u64()
        counts = [_u64(), _u64(), _u64()]
        _check(load().b2sh_reader_read_joined_rows(self._h, right._h, joinType, n, *map(_arg, (kt, kl, lo, ln, ro, rn)),
                                                   nLeftFields, _arg(lk), nRightFields, _arg(rk), C.byref(p),
                                                   C.byref(size), *map(C.byref, counts)))
        return ((C.string_at(p.value, size.value) if size.value else b""),) + tuple(c.value for c in counts)

    def aggregateDistinctRows(self, writer, nGroupKeys, keys, aggs, distinctAggs):
        """One DISTINCT group's middle stage: this reader's blocks of the exchange by G ++ X (keys = [(key_type,
        key_len), ...], the first nGroupKeys G; the map side's partial rows for functions aggs = [(fn, val_type), ...])
        merged per (G, X), folded per G (aggs merged, distinctAggs = [(fn, val_type, column or
        capi.DISTINCT_ALL_COLUMNS), ...] updated) and partitioned by G into writer, a S3SerializedShuffleWriter of the
        exchange by G with no partitioning and no records, which commits its files.
        -> (partitionLengths, [input rows, (G, X) groups, rows written])"""
        arr = lambda vals, t: np.array(list(vals) or [0], dtype=t)  # noqa: E731
        kt, kl = arr((k[0] for k in keys), np.uint32), arr((k[1] for k in keys), np.uint32)
        fn, vt = arr((a[0] for a in aggs), np.uint32), arr((a[1] for a in aggs), np.uint32)
        dfn, dvt = arr((a[0] for a in distinctAggs), np.uint32), arr((a[1] for a in distinctAggs), np.uint32)
        dcol = arr((a[2] for a in distinctAggs), np.int32)
        lengths = np.zeros(writer.numPartitions, dtype=np.int64)
        counts = np.zeros(3, dtype=np.uint64)
        _check(load().b2sh_reader_aggregate_distinct_rows(
            self._h, writer._h, nGroupKeys, len(keys), kt.ctypes.data, kl.ctypes.data, len(aggs), fn.ctypes.data,
            vt.ctypes.data, len(distinctAggs), dfn.ctypes.data, dvt.ctypes.data, dcol.ctypes.data, lengths.ctypes.data,
            counts.ctypes.data))
        return lengths, [int(c) for c in counts]

    def readWindowRows(self, keys, nPartitionKeys, nFields, kinds, fns, limit=None):
        """Spark's ranking window over this reader's partitions: its blocks through ONE
        capi.decompress_window_rows_keys_packed call, whose arguments these are (keys: the partition columns, then the
        order columns; fns: WINDOW_* or (WINDOW_NTILE, k); limit: None or (limit function, limit)).
        -> (output rows, n_records, n_out_records)"""
        a = _window_arrays(keys, nPartitionKeys, nFields, kinds, fns, limit)
        p, size = _vp(), _u64()
        counts = [_u64(), _u64()]
        _check(load().b2sh_reader_read_window_rows(self._h, *map(_arg, a), C.byref(p), C.byref(size),
                                                   *map(C.byref, counts)))
        return ((C.string_at(p.value, size.value) if size.value else b""),) + tuple(c.value for c in counts)

    def readWindowAggregateRows(self, keys, nPartitionKeys, nFields, kinds, fns):
        """Spark's window with aggregate functions over this reader's partitions: its blocks through ONE
        capi.decompress_window_aggregate_rows_keys_packed call, whose arguments these are (fns: ranking functions as
        in readWindowRows, or (fn, frame, val_type, val_off, val_null_field)).  -> (output rows, n_records,
        n_out_records)"""
        a = _window_aggregate_arrays(keys, nPartitionKeys, nFields, kinds, fns)
        p, size = _vp(), _u64()
        counts = [_u64(), _u64()]
        _check(load().b2sh_reader_read_window_aggregate_rows(self._h, *map(_arg, a), C.byref(p), C.byref(size),
                                                             *map(C.byref, counts)))
        return ((C.string_at(p.value, size.value) if size.value else b""),) + tuple(c.value for c in counts)

    def readWindowOffsetRows(self, keys, nPartitionKeys, nFields, kinds, fns):
        """Spark's window with offset (and ranking and aggregate) functions over this reader's partitions: its blocks
        through ONE capi.decompress_window_offset_rows_keys_packed call, whose arguments these are (fns: as in
        readWindowAggregateRows, or (fn, arg, frame, val_type, val_off, val_null_field, flags, default)).
        -> (output rows, n_records, n_out_records)"""
        a = _window_offset_arrays(keys, nPartitionKeys, nFields, kinds, fns)
        p, size = _vp(), _u64()
        counts = [_u64(), _u64()]
        _check(load().b2sh_reader_read_window_offset_rows(self._h, *map(_arg, a), C.byref(p), C.byref(size),
                                                          *map(C.byref, counts)))
        return ((C.string_at(p.value, size.value) if size.value else b""),) + tuple(c.value for c in counts)

    def readWindowFrameRows(self, keys, nPartitionKeys, nFields, kinds, fns):
        """Spark's window over sliding ROWS and RANGE frames (with ranking, aggregate and offset functions) over this
        reader's partitions: its blocks through ONE capi.decompress_window_frame_rows_keys_packed call, whose arguments
        these are (fns: as in readWindowOffsetRows, or (fn, arg, frame, val_type, val_off, val_null_field, flags,
        default, lower, upper)).  -> (output rows, n_records, n_out_records)"""
        a = _window_frame_arrays(keys, nPartitionKeys, nFields, kinds, fns)
        p, size = _vp(), _u64()
        counts = [_u64(), _u64()]
        _check(load().b2sh_reader_read_window_frame_rows(self._h, *map(_arg, a), C.byref(p), C.byref(size),
                                                         *map(C.byref, counts)))
        return ((C.string_at(p.value, size.value) if size.value else b""),) + tuple(c.value for c in counts)

    def _blocks(self, n):
        out = []
        for k in range(n):
            m, rs, re, p, ln = _i64(), _i32(), _i32(), _vp(), _u64()
            _check(load().b2sh_reader_block(self._h, k, C.byref(m), C.byref(rs), C.byref(re), C.byref(p), C.byref(ln)))
            out.append(((m.value, rs.value, re.value), C.string_at(p.value, ln.value) if ln.value else b""))
        return out

    def open(self):
        """start the prefetcher (storage/S3BufferedPrefetchIterator.scala); then call nextBatch() until it returns None"""
        _check(load().b2sh_reader_open(self._h))

    def nextBatch(self, maxBlocks=0):
        n = _u32(0)
        _check(load().b2sh_reader_next_batch(self._h, maxBlocks, C.byref(n)))
        return self._blocks(n.value) if n.value else None

    def statistics(self):
        v, nb, line = (_u64 * 8)(), _u64(), C.create_string_buffer(1024)
        _check(load().b2sh_reader_statistics(self._h, v, C.byref(nb), line, 1024))
        d = dict(zip(STAT_KEYS, list(v)))
        d["batches"], d["line"] = nb.value, line.value.decode()
        return d

    @property
    def remoteBytesRead(self):
        return load().b2sh_reader_remote_bytes_read(self._h)

    def close(self):
        if self._h:
            load().b2sh_reader_destroy(self._h)
            self._h = None


class S3BufferedPrefetchIterator:
    """storage/S3BufferedPrefetchIterator.scala on its own: yields ((mapId, startReduce, endReduce), compressed bytes,
    stream handle); the block stays charged to the budget until closeStream(handle)."""

    def __init__(self, dispatcher, shuffleId, mapIds, startPartition, endPartition, doBatchFetch=False,
                 maxBufferSize=0, maxThreads=0):
        self._h = _vp()
        ids = np.ascontiguousarray(mapIds, dtype=np.int64)
        _check(load().b2sh_prefetch_create(dispatcher._h, shuffleId, ids.ctypes.data, ids.size, startPartition,
                                           endPartition, int(doBatchFetch), maxBufferSize, maxThreads,
                                           C.byref(self._h)))

    def hasNext(self):
        return bool(load().b2sh_prefetch_has_next(self._h))

    def next(self):
        m, rs, re, p, ln, h = _i64(), _i32(), _i32(), _vp(), _u64(), _u64()
        _check(load().b2sh_prefetch_next(self._h, C.byref(m), C.byref(rs), C.byref(re), C.byref(p), C.byref(ln),
                                         C.byref(h)))
        return (m.value, rs.value, re.value), (C.string_at(p.value, ln.value) if ln.value else b""), h.value

    def closeStream(self, handle):
        _check(load().b2sh_prefetch_close_stream(self._h, handle))

    def statistics(self):
        v, line = (_u64 * 8)(), C.create_string_buffer(1024)
        _check(load().b2sh_prefetch_statistics(self._h, v, line, 1024))
        d = dict(zip(STAT_KEYS, list(v)))
        d["line"] = line.value.decode()
        return d

    def close(self):
        if self._h:
            load().b2sh_prefetch_destroy(self._h)
            self._h = None


class B200CompressionCodec:
    """The Spark CompressionCodec seam (SURVEY.md §8f-1): compressedOutputStream(sink) / compressedInputStream(source)
    over file-like objects.  Codec and block size come from the dispatcher's conf."""

    class _Out:
        def __init__(self, codec, sink):
            self._sink, self._err = sink, None

            def cb(ctx, p, n):
                try:
                    sink.write(C.string_at(p, n))
                    return n
                except Exception as e:  # surfaces as IOException from the C side
                    self._err = e
                    return -1

            self._cb = SINK_FN(cb)
            self._h = _vp()
            _check(load().b2sh_codec_output_stream(codec._h, C.cast(self._cb, _vp), None, C.byref(self._h)))
            self.bytesIn = self.bytesOut = self.streams = 0

        def write(self, data):
            a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
            _check(load().b2sh_ostream_write(self._h, a.ctypes.data if a.size else None, a.size))

        def flush(self):
            _check(load().b2sh_ostream_flush(self._h))

        def close(self):
            if not self._h:
                return
            bi, bo, ns = _u64(), _u64(), _u32()
            try:
                _check(load().b2sh_ostream_close(self._h, C.byref(bi), C.byref(bo), C.byref(ns)))
                self.bytesIn, self.bytesOut, self.streams = bi.value, bo.value, ns.value
            finally:
                load().b2sh_ostream_destroy(self._h)
                self._h = None

        def __enter__(self):
            return self

        def __exit__(self, *a):
            self.close()

    class _In:
        def __init__(self, codec, source):
            def cb(ctx, p, cap):
                b = source.read(min(cap, 1 << 24))
                if not b:
                    return 0
                C.memmove(p, b, len(b))
                return len(b)

            self._cb = SOURCE_FN(cb)
            self._h = _vp()
            _check(load().b2sh_codec_input_stream(codec._h, C.cast(self._cb, _vp), None, C.byref(self._h)))

        def read(self, n=-1):
            """n < 0: everything that is left; else up to n bytes (b"" at the end, like a Python file object)"""
            out = []
            want = n
            while want != 0:
                k = (1 << 24) if want < 0 else min(want, 1 << 24)
                buf = np.empty(k, dtype=np.uint8)
                got = _i64()
                _check(load().b2sh_istream_read(self._h, buf.ctypes.data, k, C.byref(got)))
                if got.value < 0:
                    break
                out.append(buf[: got.value].tobytes())
                if want > 0:
                    want -= got.value
            return b"".join(out)

        def close(self):
            if self._h:
                load().b2sh_istream_close(self._h)
                load().b2sh_istream_destroy(self._h)
                self._h = None

    def __init__(self, dispatcher):
        self._h = _vp()
        _check(load().b2sh_codec_create(dispatcher._h, C.byref(self._h)))

    def supportsConcatenationOfSerializedStreams(self):
        return bool(load().b2sh_codec_supports_concatenation(self._h))

    def compressedOutputStream(self, sink):
        return self._Out(self, sink)

    def compressedInputStream(self, source):
        return self._In(self, source)

    def close(self):
        if self._h:
            load().b2sh_codec_destroy(self._h)
            self._h = None
