"""ctypes binding of include/b200shuffle.h — the same entry points the JNI shim binds (INTEGRATION.md §2).

Nothing here computes: every helper marshals numpy/bytes into plain pointers + sizes and calls libb200shuffle.so.
"""
import ctypes as C
import os

import numpy as np

from . import _build

# ---- constants mirrored from b200shuffle.h ----
CODEC_NONE, CODEC_LZ4BLOCK, CODEC_SNAPPY_XERIAL, CODEC_ZSTD = 0, 1, 2, 3
CHECKSUM_NONE, CHECKSUM_ADLER32, CHECKSUM_CRC32, CHECKSUM_CRC32C = 0, 1, 2, 3
OK, E_CORRUPT, E_CHECKSUM, E_DST_TOO_SMALL, E_UNSUPPORTED, E_ARG, E_CUDA, E_NOT_INIT, E_NOMEM, E_NOT_CACHED = (
    0, -1, -2, -3, -4, -5, -6, -7, -8, -9)
NOT_RESIDENT = 2**64 - 1  # b2s_exchange_lookup's length of a map output that is not resident
CODEC_BY_NAME = {"lz4": CODEC_LZ4BLOCK, "snappy": CODEC_SNAPPY_XERIAL, "zstd": CODEC_ZSTD}
CHECKSUM_BY_NAME = {"ADLER32": CHECKSUM_ADLER32, "CRC32": CHECKSUM_CRC32, "CRC32C": CHECKSUM_CRC32C}

_u8p, _u64p, _u32p, _i32p, _vp = C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
_u32, _u64, _i32 = C.c_uint32, C.c_uint64, C.c_int32


class Timing(C.Structure):
    _fields_ = [
        ("total_ms", C.c_double), ("h2d_ms", C.c_double), ("d2h_ms", C.c_double), ("kernel_ms", C.c_double),
        ("top_kernel_ms", C.c_double), ("h2d_bytes", _u64), ("d2h_bytes", _u64), ("kernel_launches", _u64),
        ("src_bytes", _u64), ("dst_bytes", _u64), ("dominant_ms", C.c_double), ("dominant_launches", _u64),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# every symbol include/b200shuffle.h declares: (name, restype, argtypes)
PROTOTYPES = [
    ("b2s_init", C.c_int, [_u32, _u64, _u32]),
    ("b2s_shutdown", None, []),
    ("b2s_device_count", C.c_int, []),
    ("b2s_set_thread_device", C.c_int, [_u32]),
    ("b2s_bind_thread_to_device", C.c_int, [_u32]),
    ("b2s_device_numa_node", C.c_int, [_u32]),
    ("b2s_strerror", C.c_char_p, [_i32]),
    ("b2s_last_error", C.c_char_p, []),
    ("b2s_version", _u32, []),
    ("b2s_host_alloc", C.c_void_p, [_u64]),
    ("b2s_host_free", None, [C.c_void_p]),
    ("b2s_host_register", C.c_int, [C.c_void_p, _u64]),
    ("b2s_host_unregister", C.c_int, [C.c_void_p]),
    ("b2s_compress_bound", _u64, [_u32, _u32, _u64]),
    ("b2s_decompressed_size_batch", C.c_int, [_u32, _u32, _vp, _u64p, _u64p, _i32p]),
    ("b2s_checksum_batch", C.c_int, [_u32, _u32, _vp, _u64p, _u64p]),
    ("b2s_checksum_packed", C.c_int, [_u32, _u32, _u8p, _u64p, _u64p, _u64p]),
    ("b2s_compress_batch", C.c_int, [_u32, _i32, _u32, _u32, _u32, _vp, _u64p, _vp, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_compress_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u8p, _u64p, _u64p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_partition_compress_bound", _u64, [_u32, _u32, _u32, _u64]),
    ("b2s_partition_compress_packed", C.c_int,
     [_u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32p, _u8p, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_partition_compress_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _u64, _vp, _u64, _u32p, _u32p, _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_decompress_batch", C.c_int,
     [_u32, _u32, _u32, _vp, _u64p, _u32p, _vp, _vp, _vp, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u8p, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_decompress_sort_packed", C.c_int,
     [_u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _u8p, _u64, _u64p, _u64p, _i32p,
      _i32p]),
    ("b2s_decompress_sort_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _vp, _u64, _u64p, _u64p, _i32p,
      _i32p]),
    ("b2s_exchange_set_budget", C.c_int, [_u32, _u64]),
    ("b2s_partition_compress_cached_packed", C.c_int,
     [_i32, C.c_int64, _u32, _i32, _u32, _u32, _u32, _u64, _u8p, _u64, _u32p, _u32p, _u8p, _u64, _u64p, _u64p, _u64p,
      _u64p, _i32p, _i32p]),
    ("b2s_exchange_lookup", C.c_int, [_i32, _i32, _i32, _u32, _vp, _u64p]),
    ("b2s_exchange_read_packed", C.c_int, [_i32, _i32, _i32, _u32, _vp, _u8p, _u64, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_exchange_read_sort_packed", C.c_int,
     [_i32, _i32, _i32, _vp, _vp, _u32, _u32, _u32, _u8p, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32, _u8p,
      _u64, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_exchange_read_sort_dev", C.c_int,
     [_u32, _i32, _i32, _i32, _vp, _vp, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _u32, _u32, _u32,
      _vp, _u64, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_exchange_remove", C.c_int, [_i32, C.c_int64]),
    ("b2s_checksum_dev", C.c_int, [_u32, _u32, _u32, _vp, _u64p, _u64p, _u64p]),
    ("b2s_compress_dev", C.c_int,
     [_u32, _u32, _i32, _u32, _u32, _u32, _vp, _u64p, _u64p, _vp, _u64, _u64p, _u64p, _u64p, _u64p, _i32p]),
    ("b2s_decompress_dev", C.c_int,
     [_u32, _u32, _u32, _u32, _vp, _u64p, _u64p, _u32p, _u64p, _u64p, _vp, _u64, _u64p, _u64p, _u64p, _i32p, _i32p]),
    ("b2s_dev_alloc", C.c_void_p, [_u32, _u64]),
    ("b2s_dev_free", None, [_u32, C.c_void_p]),
    ("b2s_dev_memcpy", C.c_int, [_u32, C.c_void_p, C.c_void_p, _u64, C.c_int]),
    ("b2s_last_timing", C.c_int, [C.POINTER(Timing)]),
    ("b2s_total_kernel_launches", _u64, []),
    ("b2s_mark", C.c_int, [_u32, _u32]),
    ("b2s_marks_elapsed_ms", C.c_int, [_u32, C.POINTER(C.c_double)]),
    ("b2s_gen_terasort_dev", C.c_int, [_u32, C.c_void_p, _u64, _u64, _u64]),
]
SYMBOLS = [p[0] for p in PROTOTYPES]

_lib = None


def load(build_if_needed=True):
    """Loads libb200shuffle.so (building it with nvcc when stale).  Raises if that is impossible — no fallback."""
    global _lib
    if _lib is None:
        path = _build.build() if build_if_needed else _build.LIB
        if not os.path.exists(path):
            raise RuntimeError("libb200shuffle.so is missing and could not be built; there is no CPU fallback")
        L = C.CDLL(path)
        for name, res, args in PROTOTYPES:
            f = getattr(L, name)  # AttributeError if the library does not export a declared symbol
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib


class B2SError(RuntimeError):
    def __init__(self, code, where):
        L = load()
        self.code = code
        msg = L.b2s_strerror(code).decode()
        detail = L.b2s_last_error().decode()
        super().__init__("%s: %s (%d)%s" % (where, msg, code, (": " + detail) if detail else ""))


def _check(rc, where):
    if rc != 0:
        raise B2SError(rc, where)


def init(gpu_mask=0, pinned_bytes_per_gpu=0, streams_per_gpu=0):
    _check(load().b2s_init(gpu_mask, pinned_bytes_per_gpu, streams_per_gpu), "b2s_init")


def bind_thread_to_device(dev=0):
    """pins the calling thread to the CPUs of the device's NUMA node and prefers that node for its allocations"""
    _check(load().b2s_bind_thread_to_device(dev), "b2s_bind_thread_to_device")
    return load().b2s_device_numa_node(dev)


def shutdown():
    load().b2s_shutdown()


def last_timing():
    t = Timing()
    load().b2s_last_timing(C.byref(t))
    return t.as_dict()


def mark(which, dev=0):
    _check(load().b2s_mark(dev, which), "b2s_mark")


def marks_elapsed_ms(dev=0):
    ms = C.c_double(0)
    _check(load().b2s_marks_elapsed_ms(dev, C.byref(ms)), "b2s_marks_elapsed_ms")
    return ms.value


def compress_bound(codec, block_size, n):
    return load().b2s_compress_bound(codec, block_size, n)


# ---------------------------------------------------------------------------------------------------------------
# marshalling helpers
# ---------------------------------------------------------------------------------------------------------------
def _as_u8(b):
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b, dtype=np.uint8)
    return np.frombuffer(b, dtype=np.uint8)


def _ptr(a):
    return a.ctypes.data if a is not None and a.size else None


def _ptr_array(arrs):
    out = np.zeros(max(len(arrs), 1), dtype=np.uint64)
    for i, a in enumerate(arrs):
        out[i] = a.ctypes.data if a.size else 0
    return out


class HostBuffer:
    """Pinned host memory from b2s_host_alloc, viewed as a numpy uint8 array (what the JVM wraps as a direct buffer)."""

    def __init__(self, nbytes):
        self.nbytes = int(nbytes)
        self.ptr = load().b2s_host_alloc(max(self.nbytes, 1))
        if not self.ptr:
            raise B2SError(E_NOMEM, "b2s_host_alloc")
        buf = (C.c_uint8 * max(self.nbytes, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=np.uint8, count=self.nbytes)

    def free(self):
        if self.ptr:
            self.array = None
            load().b2s_host_free(self.ptr)
            self.ptr = None


# ---------------------------------------------------------------------------------------------------------------
# host-pointer API
# ---------------------------------------------------------------------------------------------------------------
def checksum_batch(alg, blocks):
    arrs = [_as_u8(b) for b in blocks]
    n = len(arrs)
    ptrs = _ptr_array(arrs)
    lens = np.array([a.size for a in arrs] or [0], dtype=np.uint64)
    out = np.zeros(max(n, 1), dtype=np.uint64)
    _check(load().b2s_checksum_batch(alg, n, _ptr(ptrs), _ptr(lens), _ptr(out)), "b2s_checksum_batch")
    return [int(v) for v in out[:n]]


def checksum_packed(alg, base, off, length):
    base = _as_u8(base)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    out = np.zeros(max(off.size, 1), dtype=np.uint64)
    _check(load().b2s_checksum_packed(alg, off.size, _ptr(base), _ptr(off), _ptr(length), _ptr(out)),
           "b2s_checksum_packed")
    return out[: off.size]


def compress_batch(codec, blocks, block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dst_caps=None):
    """-> (list of compressed streams (bytes or None on error), checksums, status)"""
    arrs = [_as_u8(b) for b in blocks]
    n = len(arrs)
    lens = np.array([a.size for a in arrs] or [0], dtype=np.uint64)
    caps = np.array(
        (dst_caps if dst_caps is not None else [compress_bound(codec, block_size, a.size) for a in arrs]) or [0],
        dtype=np.uint64)
    outs = [np.empty(int(c), dtype=np.uint8) for c in caps[:n]]
    sp, dp = _ptr_array(arrs), _ptr_array(outs)
    dlen = np.zeros(max(n, 1), dtype=np.uint64)
    cks = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    _check(load().b2s_compress_batch(codec, level, block_size, checksum_alg, n, _ptr(sp), _ptr(lens), _ptr(dp),
                                     _ptr(caps), _ptr(dlen), _ptr(cks), _ptr(st)), "b2s_compress_batch")
    res = [outs[i][: int(dlen[i])].tobytes() if st[i] == 0 else None for i in range(n)]
    return res, [int(v) for v in cks[:n]], [int(v) for v in st[:n]]


def compress_packed(codec, src, off, length, dst, block_size=0, checksum_alg=CHECKSUM_NONE, level=0):
    """src/dst: uint8 arrays (ideally HostBuffer.array).  -> dict(dst_off, dst_len, total, checksums, status)"""
    src, dst = _as_u8(src), _as_u8(dst)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    cks = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_compress_packed(codec, level, block_size, checksum_alg, n, _ptr(src), _ptr(off), _ptr(length),
                                      _ptr(dst), dst.size, _ptr(dst_off), _ptr(dst_len), C.addressof(total),
                                      _ptr(cks), _ptr(st)), "b2s_compress_packed")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, checksums=cks[:n], status=st[:n])


def partition_compress_bound(codec, block_size, num_partitions, rec_bytes):
    return load().b2s_partition_compress_bound(codec, block_size, num_partitions, rec_bytes)


def _partition_out(num_partitions):
    return (np.zeros(num_partitions, dtype=np.uint64), np.zeros(num_partitions, dtype=np.uint64),
            np.zeros(num_partitions, dtype=np.uint64), np.zeros(num_partitions, dtype=np.int32))


def partition_compress_packed(codec, records, rec_len, rec_part, num_partitions, dst, block_size=0,
                              checksum_alg=CHECKSUM_NONE, level=0):
    """records: the serialized records back to back (uint8 array, ideally HostBuffer.array); rec_len / rec_part: one
    length and one reduce id per record.  -> dict(dst_off, dst_len, total, checksums, status), one entry per partition"""
    records, dst = _as_u8(records), _as_u8(dst)
    rec_len = np.ascontiguousarray(rec_len, dtype=np.uint32)
    rec_part = np.ascontiguousarray(rec_part, dtype=np.uint32)
    dst_off, dst_len, cks, st = _partition_out(num_partitions)
    total = _u64(0)
    _check(load().b2s_partition_compress_packed(codec, level, block_size, checksum_alg, num_partitions, rec_len.size,
                                                _ptr(records), records.size, _ptr(rec_len), _ptr(rec_part), _ptr(dst),
                                                dst.size, _ptr(dst_off), _ptr(dst_len), C.addressof(total), _ptr(cks),
                                                _ptr(st)), "b2s_partition_compress_packed")
    return dict(dst_off=dst_off, dst_len=dst_len, total=total.value, checksums=cks, status=st)


def decompressed_size_batch(codec, blocks):
    arrs = [_as_u8(b) for b in blocks]
    n = len(arrs)
    sp = _ptr_array(arrs)
    lens = np.array([a.size for a in arrs] or [0], dtype=np.uint64)
    out = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    _check(load().b2s_decompressed_size_batch(codec, n, _ptr(sp), _ptr(lens), _ptr(out), _ptr(st)),
           "b2s_decompressed_size_batch")
    return [int(v) for v in out[:n]], [int(v) for v in st[:n]]


def decompress_batch(codec, blocks, checksum_alg=CHECKSUM_NONE, slices=None, dst_caps=None):
    """slices: per block a list of (length, checksum) pairs (the block's .index differences / .checksum values).
    -> (list of decoded bytes or None, status, bad_slice)"""
    arrs = [_as_u8(b) for b in blocks]
    n = len(arrs)
    if dst_caps is None:
        sizes, _ = decompressed_size_batch(codec, blocks)
        dst_caps = sizes
    caps = np.array(list(dst_caps) or [0], dtype=np.uint64)
    outs = [np.empty(max(int(c), 1), dtype=np.uint8) for c in caps[:n]]
    sp, dp = _ptr_array(arrs), _ptr_array(outs)
    lens = np.array([a.size for a in arrs] or [0], dtype=np.uint64)
    dlen = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    ns = sl_ptrs = sc_ptrs = None
    keep = []
    if checksum_alg != CHECKSUM_NONE:
        ns = np.array([len(s) for s in slices] or [0], dtype=np.uint32)
        sl = [np.array([p[0] for p in s] or [0], dtype=np.uint64) for s in slices]
        sc = [np.array([p[1] for p in s] or [0], dtype=np.uint64) for s in slices]
        keep = [sl, sc]
        sl_ptrs = np.array([a.ctypes.data for a in sl] or [0], dtype=np.uint64)
        sc_ptrs = np.array([a.ctypes.data for a in sc] or [0], dtype=np.uint64)
    _check(load().b2s_decompress_batch(codec, checksum_alg, n, _ptr(sp), _ptr(lens), _ptr(ns), _ptr(sl_ptrs),
                                       _ptr(sc_ptrs), _ptr(dp), _ptr(caps), _ptr(dlen), _ptr(st), _ptr(bad)),
           "b2s_decompress_batch")
    del keep
    res = [outs[i][: int(dlen[i])].tobytes() if st[i] == 0 else None for i in range(n)]
    return res, [int(v) for v in st[:n]], [int(v) for v in bad[:n]]


def decompress_packed(codec, src, off, length, dst, checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None,
                      slice_checksum=None):
    src, dst = _as_u8(src), _as_u8(dst)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    sb = sl = sc = None
    if checksum_alg != CHECKSUM_NONE:
        sb = np.ascontiguousarray(slice_base, dtype=np.uint32)
        sl = np.ascontiguousarray(slice_len, dtype=np.uint64)
        sc = np.ascontiguousarray(slice_checksum, dtype=np.uint64)
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_decompress_packed(codec, checksum_alg, n, _ptr(src), _ptr(off), _ptr(length), _ptr(sb), _ptr(sl),
                                        _ptr(sc), _ptr(dst), dst.size, _ptr(dst_off), _ptr(dst_len),
                                        C.addressof(total), _ptr(st), _ptr(bad)), "b2s_decompress_packed")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, status=st[:n], bad_slice=bad[:n])


def _sort_slices(checksum_alg, slice_base, slice_len, slice_checksum):
    if checksum_alg == CHECKSUM_NONE:
        return None, None, None
    return (np.ascontiguousarray(slice_base, dtype=np.uint32), np.ascontiguousarray(slice_len, dtype=np.uint64),
            np.ascontiguousarray(slice_checksum, dtype=np.uint64))


def decompress_sort_packed(codec, src, off, length, dst, record_bytes, key_off, key_len, checksum_alg=CHECKSUM_NONE,
                           slice_base=None, slice_len=None, slice_checksum=None):
    """Verifies and decodes a reduce task's blocks and sorts their fixed-size records by the unsigned bytes
    [key_off, key_off + key_len) into dst (stable).  -> dict(total, n_records, status, bad_slice)"""
    src, dst = _as_u8(src), _as_u8(dst)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    sb, sl, sc = _sort_slices(checksum_alg, slice_base, slice_len, slice_checksum)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    total, nrec = _u64(0), _u64(0)
    _check(load().b2s_decompress_sort_packed(codec, checksum_alg, n, _ptr(src), _ptr(off), _ptr(length), _ptr(sb),
                                             _ptr(sl), _ptr(sc), record_bytes, key_off, key_len, _ptr(dst), dst.size,
                                             C.addressof(total), C.addressof(nrec), _ptr(st), _ptr(bad)),
           "b2s_decompress_sort_packed")
    return dict(total=total.value, n_records=nrec.value, status=st[:n], bad_slice=bad[:n])


# ---------------------------------------------------------------------------------------------------------------
# device-resident API (bench.py roofline leg); d_* are raw device addresses (ints)
# ---------------------------------------------------------------------------------------------------------------
def dev_alloc(nbytes, dev=0):
    p = load().b2s_dev_alloc(dev, nbytes)
    if not p:
        raise B2SError(E_NOMEM, "b2s_dev_alloc")
    return p


def dev_free(p, dev=0):
    load().b2s_dev_free(dev, p)


def dev_memcpy(dst, src, nbytes, kind, dev=0):
    _check(load().b2s_dev_memcpy(dev, dst, src, nbytes, kind), "b2s_dev_memcpy")


def gen_terasort_dev(d_dst, first_record, n_records, seed=42, dev=0):
    _check(load().b2s_gen_terasort_dev(dev, d_dst, first_record, n_records, seed), "b2s_gen_terasort_dev")


def checksum_dev(alg, d_base, off, length, dev=0):
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    out = np.zeros(max(off.size, 1), dtype=np.uint64)
    _check(load().b2s_checksum_dev(dev, alg, off.size, d_base, _ptr(off), _ptr(length), _ptr(out)), "b2s_checksum_dev")
    return out[: off.size]


def compress_dev(codec, d_src, off, length, d_dst, dst_cap, block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    cks = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_compress_dev(dev, codec, level, block_size, checksum_alg, n, d_src, _ptr(off), _ptr(length),
                                   d_dst, dst_cap, _ptr(dst_off), _ptr(dst_len), C.addressof(total), _ptr(cks),
                                   _ptr(st)), "b2s_compress_dev")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, checksums=cks[:n], status=st[:n])


def decompress_dev(codec, d_src, off, length, d_dst, dst_cap, checksum_alg=CHECKSUM_NONE, slice_base=None,
                   slice_len=None, slice_checksum=None, dev=0):
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    sb = sl = sc = None
    if checksum_alg != CHECKSUM_NONE:
        sb = np.ascontiguousarray(slice_base, dtype=np.uint32)
        sl = np.ascontiguousarray(slice_len, dtype=np.uint64)
        sc = np.ascontiguousarray(slice_checksum, dtype=np.uint64)
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_decompress_dev(dev, codec, checksum_alg, n, d_src, _ptr(off), _ptr(length), _ptr(sb), _ptr(sl),
                                     _ptr(sc), d_dst, dst_cap, _ptr(dst_off), _ptr(dst_len), C.addressof(total),
                                     _ptr(st), _ptr(bad)), "b2s_decompress_dev")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, status=st[:n], bad_slice=bad[:n])


def decompress_sort_dev(codec, d_src, off, length, d_dst, dst_cap, record_bytes, key_off, key_len,
                        checksum_alg=CHECKSUM_NONE, slice_base=None, slice_len=None, slice_checksum=None, dev=0):
    """decompress_sort_packed on device-resident blocks (d_src) into a device arena (d_dst)"""
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = off.size
    sb, sl, sc = _sort_slices(checksum_alg, slice_base, slice_len, slice_checksum)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    total, nrec = _u64(0), _u64(0)
    _check(load().b2s_decompress_sort_dev(dev, codec, checksum_alg, n, d_src, _ptr(off), _ptr(length), _ptr(sb),
                                          _ptr(sl), _ptr(sc), record_bytes, key_off, key_len, d_dst, dst_cap,
                                          C.addressof(total), C.addressof(nrec), _ptr(st), _ptr(bad)),
           "b2s_decompress_sort_dev")
    return dict(total=total.value, n_records=nrec.value, status=st[:n], bad_slice=bad[:n])


def partition_compress_dev(codec, d_records, rec_bytes, d_rec_len, d_rec_part, n_records, num_partitions, d_dst,
                           dst_cap, block_size=0, checksum_alg=CHECKSUM_NONE, level=0, dev=0):
    """d_*: device addresses (records, u32 lengths, u32 reduce ids, destination arena)"""
    dst_off, dst_len, cks, st = _partition_out(num_partitions)
    total = _u64(0)
    _check(load().b2s_partition_compress_dev(dev, codec, level, block_size, checksum_alg, num_partitions, n_records,
                                             d_records, rec_bytes, d_rec_len, d_rec_part, d_dst, dst_cap,
                                             _ptr(dst_off), _ptr(dst_len), C.addressof(total), _ptr(cks), _ptr(st)),
           "b2s_partition_compress_dev")
    return dict(dst_off=dst_off, dst_len=dst_len, total=total.value, checksums=cks, status=st)


# ---------------------------------------------------------------------------------------------------------------
# exchange cache: map outputs kept resident in HBM for reducers on the same device
# ---------------------------------------------------------------------------------------------------------------
def exchange_set_budget(nbytes, dev=0):
    """per-device budget in bytes of cached records; 0 (the default) turns the cache off"""
    _check(load().b2s_exchange_set_budget(dev, nbytes), "b2s_exchange_set_budget")


def partition_compress_cached_packed(shuffle_id, map_id, codec, records, rec_len, rec_part, num_partitions, dst,
                                     block_size=0, checksum_alg=CHECKSUM_NONE, level=0):
    """partition_compress_packed that also keeps the partitioned records as the cache entry (shuffle_id, map_id).
    -> dict(dst_off, dst_len, total, checksums, status, cached)"""
    records, dst = _as_u8(records), _as_u8(dst)
    rec_len = np.ascontiguousarray(rec_len, dtype=np.uint32)
    rec_part = np.ascontiguousarray(rec_part, dtype=np.uint32)
    dst_off, dst_len, cks, st = _partition_out(num_partitions)
    total, cached = _u64(0), _i32(0)
    _check(load().b2s_partition_compress_cached_packed(
        shuffle_id, map_id, codec, level, block_size, checksum_alg, num_partitions, rec_len.size, _ptr(records),
        records.size, _ptr(rec_len), _ptr(rec_part), _ptr(dst), dst.size, _ptr(dst_off), _ptr(dst_len),
        C.addressof(total), _ptr(cks), _ptr(st), C.addressof(cached)), "b2s_partition_compress_cached_packed")
    return dict(dst_off=dst_off, dst_len=dst_len, total=total.value, checksums=cks, status=st, cached=cached.value)


def exchange_lookup(shuffle_id, start_reduce, end_reduce, map_ids):
    """-> (hits, lengths): lengths[i] = bytes of the range of map_ids[i], NOT_RESIDENT when it is not resident"""
    ids = np.ascontiguousarray(map_ids, dtype=np.int64)
    ln = np.zeros(max(ids.size, 1), dtype=np.uint64)
    rc = load().b2s_exchange_lookup(shuffle_id, start_reduce, end_reduce, ids.size, _ptr(ids), _ptr(ln))
    if rc < 0:
        raise B2SError(rc, "b2s_exchange_lookup")
    return rc, ln[: ids.size]


def exchange_read_packed(shuffle_id, start_reduce, end_reduce, map_ids, dst):
    """the cached ranges back to back into dst.  -> dict(dst_off, dst_len, total, status)"""
    ids = np.ascontiguousarray(map_ids, dtype=np.int64)
    dst = _as_u8(dst)
    n = ids.size
    dst_off = np.zeros(max(n, 1), dtype=np.uint64)
    dst_len = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    total = _u64(0)
    _check(load().b2s_exchange_read_packed(shuffle_id, start_reduce, end_reduce, n, _ptr(ids), _ptr(dst), dst.size,
                                           _ptr(dst_off), _ptr(dst_len), C.addressof(total), _ptr(st)),
           "b2s_exchange_read_packed")
    return dict(dst_off=dst_off[:n], dst_len=dst_len[:n], total=total.value, status=st[:n])


def _exchange_sources(map_ids, cached):
    return (np.ascontiguousarray(map_ids, dtype=np.int64),
            np.ascontiguousarray(np.asarray(cached, dtype=bool), dtype=np.uint8))


def exchange_read_sort_packed(shuffle_id, start_reduce, end_reduce, map_ids, cached, codec, src, off, length, dst,
                              record_bytes, key_off, key_len, checksum_alg=CHECKSUM_NONE, slice_base=None,
                              slice_len=None, slice_checksum=None):
    """decompress_sort_packed over sources of which those with cached[i] set are the cached range of map_ids[i].
    -> dict(total, n_records, status, bad_slice)"""
    ids, cm = _exchange_sources(map_ids, cached)
    src, dst = _as_u8(src), _as_u8(dst)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = ids.size
    sb, sl, sc = _sort_slices(checksum_alg, slice_base, slice_len, slice_checksum)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    total, nrec = _u64(0), _u64(0)
    _check(load().b2s_exchange_read_sort_packed(shuffle_id, start_reduce, end_reduce, _ptr(ids), _ptr(cm), codec,
                                                checksum_alg, n, _ptr(src), _ptr(off), _ptr(length), _ptr(sb),
                                                _ptr(sl), _ptr(sc), record_bytes, key_off, key_len, _ptr(dst),
                                                dst.size, C.addressof(total), C.addressof(nrec), _ptr(st), _ptr(bad)),
           "b2s_exchange_read_sort_packed")
    return dict(total=total.value, n_records=nrec.value, status=st[:n], bad_slice=bad[:n])


def exchange_read_sort_dev(shuffle_id, start_reduce, end_reduce, map_ids, cached, codec, d_src, off, length, d_dst,
                           dst_cap, record_bytes, key_off, key_len, checksum_alg=CHECKSUM_NONE, slice_base=None,
                           slice_len=None, slice_checksum=None, dev=0):
    """exchange_read_sort_packed with the fetched blocks (d_src) and the output (d_dst) in device memory"""
    ids, cm = _exchange_sources(map_ids, cached)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    length = np.ascontiguousarray(length, dtype=np.uint64)
    n = ids.size
    sb, sl, sc = _sort_slices(checksum_alg, slice_base, slice_len, slice_checksum)
    st = np.zeros(max(n, 1), dtype=np.int32)
    bad = np.zeros(max(n, 1), dtype=np.int32)
    total, nrec = _u64(0), _u64(0)
    _check(load().b2s_exchange_read_sort_dev(dev, shuffle_id, start_reduce, end_reduce, _ptr(ids), _ptr(cm), codec,
                                             checksum_alg, n, d_src, _ptr(off), _ptr(length), _ptr(sb), _ptr(sl),
                                             _ptr(sc), record_bytes, key_off, key_len, d_dst, dst_cap,
                                             C.addressof(total), C.addressof(nrec), _ptr(st), _ptr(bad)),
           "b2s_exchange_read_sort_dev")
    return dict(total=total.value, n_records=nrec.value, status=st[:n], bad_slice=bad[:n])


def exchange_remove(shuffle_id, map_id=-1):
    """removes (shuffle_id, map_id), or every map output of the shuffle (map_id -1), on every device -> count"""
    rc = load().b2s_exchange_remove(shuffle_id, map_id)
    if rc < 0:
        raise B2SError(rc, "b2s_exchange_remove")
    return rc
