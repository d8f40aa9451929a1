"""ctypes wrapper around oracle/libb2s_oracle.so — CPU ORACLE, TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this module.
The product package (spark-s3-shuffle_b200/) never does.  See oracle/b2s_oracle.h for what is restated and
which reference file:line each function follows.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libb2s_oracle.so")

ADLER32, CRC32, CRC32C = 1, 2, 3
ALG_BY_NAME = {"ADLER32": ADLER32, "CRC32": CRC32, "CRC32C": CRC32C}


def build(force=False):
    src = os.path.join(_HERE, "b2s_oracle.c")
    hdr = os.path.join(_HERE, "b2s_oracle.h")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["make", "-C", _HERE, "-B", "libb2s_oracle.so"], stdout=subprocess.DEVNULL)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        u8p, i64p = C.c_void_p, C.c_void_p
        L.orc_crc32.restype = C.c_uint32
        L.orc_crc32.argtypes = [C.c_uint32, u8p, C.c_size_t]
        L.orc_crc32c.restype = C.c_uint32
        L.orc_crc32c.argtypes = [C.c_uint32, u8p, C.c_size_t]
        L.orc_adler32.restype = C.c_uint32
        L.orc_adler32.argtypes = [C.c_uint32, u8p, C.c_size_t]
        L.orc_checksum.restype = C.c_uint32
        L.orc_checksum.argtypes = [C.c_uint32, u8p, C.c_size_t]
        L.orc_xxh32.restype = C.c_uint32
        L.orc_xxh32.argtypes = [u8p, C.c_size_t, C.c_uint32]
        L.orc_lz4_compress_block.restype = C.c_int
        L.orc_lz4_compress_block.argtypes = [u8p, C.c_int, u8p, C.c_int]
        L.orc_lz4_compress_block_win.restype = C.c_int
        L.orc_lz4_compress_block_win.argtypes = [u8p, C.c_int, u8p, C.c_int, C.c_int]
        L.orc_lz4_decompress_block.restype = C.c_int
        L.orc_lz4_decompress_block.argtypes = [u8p, C.c_int, u8p, C.c_int]
        L.orc_lz4block_bound.restype = C.c_uint64
        L.orc_lz4block_bound.argtypes = [C.c_uint64, C.c_uint32]
        L.orc_lz4block_compress.restype = C.c_int64
        L.orc_lz4block_compress.argtypes = [u8p, C.c_uint64, C.c_uint32, u8p, C.c_uint64, C.c_int]
        L.orc_lz4block_decompress.restype = C.c_int64
        L.orc_lz4block_decompress.argtypes = [u8p, C.c_uint64, u8p, C.c_uint64]
        L.orc_lz4block_decompressed_size.restype = C.c_int64
        L.orc_lz4block_decompressed_size.argtypes = [u8p, C.c_uint64]
        L.orc_snappy_max_compressed.restype = C.c_uint64
        L.orc_snappy_max_compressed.argtypes = [C.c_uint64]
        L.orc_snappy_compress_raw.restype = C.c_int64
        L.orc_snappy_compress_raw.argtypes = [u8p, C.c_uint64, u8p, C.c_uint64]
        L.orc_snappy_uncompressed_length.restype = C.c_int64
        L.orc_snappy_uncompressed_length.argtypes = [u8p, C.c_uint64]
        L.orc_snappy_uncompress_raw.restype = C.c_int64
        L.orc_snappy_uncompress_raw.argtypes = [u8p, C.c_uint64, u8p, C.c_uint64]
        L.orc_xerial_bound.restype = C.c_uint64
        L.orc_xerial_bound.argtypes = [C.c_uint64, C.c_uint32]
        L.orc_xerial_compress.restype = C.c_int64
        L.orc_xerial_compress.argtypes = [u8p, C.c_uint64, C.c_uint32, u8p, C.c_uint64]
        L.orc_xerial_compress2.restype = C.c_int64
        L.orc_xerial_compress2.argtypes = [u8p, C.c_uint64, C.c_uint32, u8p, C.c_uint64, C.c_int]
        L.orc_xerial_decompress.restype = C.c_int64
        L.orc_xerial_decompress.argtypes = [u8p, C.c_uint64, u8p, C.c_uint64]
        L.orc_xerial_decompressed_size.restype = C.c_int64
        L.orc_xerial_decompressed_size.argtypes = [u8p, C.c_uint64]
        L.orc_validate_slices.restype = C.c_int64
        L.orc_validate_slices.argtypes = [C.c_uint32, u8p, i64p, i64p, C.c_int, C.c_int]
        L.orc_index_from_lengths.restype = None
        L.orc_index_from_lengths.argtypes = [i64p, C.c_int, u8p]
        L.orc_be64_array.restype = None
        L.orc_be64_array.argtypes = [i64p, C.c_int, u8p]
        L.orc_read_be64_array.restype = C.c_int
        L.orc_read_be64_array.argtypes = [u8p, C.c_uint64, i64p]
        L.orc_gen_terasort.restype = None
        L.orc_gen_terasort.argtypes = [u8p, C.c_uint64, C.c_uint64, C.c_uint64]
        L.orc_baseline_run.restype = C.c_int
        L.orc_baseline_run.argtypes = [C.c_void_p]
        L.orc_baseline_run_codec.restype = C.c_int
        L.orc_baseline_run_codec.argtypes = [C.c_void_p]
        _lib = L
    return _lib


def _u8(b):
    """bytes / bytearray / ndarray -> contiguous uint8 ndarray (no copy when possible)."""
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b, dtype=np.uint8)
    return np.frombuffer(bytes(b) if not isinstance(b, (bytes, bytearray, memoryview)) else b, dtype=np.uint8)


def _p(a):
    return a.ctypes.data if a.size else None


# ---- checksums ----
def crc32(b):
    a = _u8(b)
    return lib().orc_crc32(0, _p(a), a.size)


def crc32c(b):
    a = _u8(b)
    return lib().orc_crc32c(0, _p(a), a.size)


def adler32(b):
    a = _u8(b)
    return lib().orc_adler32(1, _p(a), a.size)


def checksum(alg, b):
    a = _u8(b)
    return lib().orc_checksum(alg, _p(a), a.size)


def xxh32(b, seed=0x9747B28C):
    a = _u8(b)
    return lib().orc_xxh32(_p(a), a.size, seed)


# ---- raw LZ4 block ----
def lz4_compress_block(b, win=False, hash_log=12, cap=None):
    """win=True: the CPU model of the GPU compressor"""
    a = _u8(b)
    cap = cap if cap is not None else a.size + a.size // 255 + 32
    out = np.empty(max(cap, 1), dtype=np.uint8)
    if win:
        n = lib().orc_lz4_compress_block_win(_p(a), a.size, out.ctypes.data, cap, hash_log)
    else:
        n = lib().orc_lz4_compress_block(_p(a), a.size, out.ctypes.data, cap)
    return out[:n].tobytes() if n > 0 else None


def lz4_decompress_block(b, orig_len):
    a = _u8(b)
    out = np.empty(max(orig_len, 1), dtype=np.uint8)
    used = lib().orc_lz4_decompress_block(_p(a), a.size, out.ctypes.data, orig_len)
    if used < 0:
        return None, used
    return out[:orig_len].tobytes(), used


# ---- LZ4Block streams ----
def lz4block_compress(b, block_size=32768, compressor=0):
    a = _u8(b)
    cap = lib().orc_lz4block_bound(a.size, block_size)
    out = np.empty(cap, dtype=np.uint8)
    n = lib().orc_lz4block_compress(_p(a), a.size, block_size, out.ctypes.data, cap, compressor)
    if n < 0:
        raise ValueError("orc_lz4block_compress failed: %d" % n)
    return out[:n].tobytes()


def lz4block_decompressed_size(b):
    a = _u8(b)
    return lib().orc_lz4block_decompressed_size(_p(a), a.size)


def lz4block_decompress(b):
    """Returns bytes, or raises IOError('Stream is corrupted') like LZ4BlockInputStream."""
    a = _u8(b)
    n = lib().orc_lz4block_decompressed_size(_p(a), a.size)
    if n < 0:
        raise IOError("Stream is corrupted")
    out = np.empty(max(n, 1), dtype=np.uint8)
    r = lib().orc_lz4block_decompress(_p(a), a.size, out.ctypes.data, n)
    if r < 0:
        raise IOError("Stream is corrupted")
    return out[:r].tobytes()


# ---- snappy ----
def snappy_compress_raw(b):
    a = _u8(b)
    cap = lib().orc_snappy_max_compressed(a.size)
    out = np.empty(cap, dtype=np.uint8)
    n = lib().orc_snappy_compress_raw(_p(a), a.size, out.ctypes.data, cap)
    if n < 0:
        raise ValueError("snappy compress failed")
    return out[:n].tobytes()


def snappy_uncompress_raw(b):
    a = _u8(b)
    n = lib().orc_snappy_uncompressed_length(_p(a), a.size)
    if n < 0:
        raise IOError("snappy: corrupt input")
    out = np.empty(max(n, 1), dtype=np.uint8)
    r = lib().orc_snappy_uncompress_raw(_p(a), a.size, out.ctypes.data, n)
    if r < 0:
        raise IOError("snappy: corrupt input")
    return out[:r].tobytes()


def xerial_compress(b, block_size=32768, compressor=0):
    """compressor: 0 = restated snappy-style greedy, 1 = CPU model of the GPU compressor"""
    a = _u8(b)
    cap = lib().orc_xerial_bound(a.size, block_size)
    out = np.empty(cap, dtype=np.uint8)
    n = lib().orc_xerial_compress2(_p(a), a.size, block_size, out.ctypes.data, cap, compressor)
    if n < 0:
        raise ValueError("xerial compress failed")
    return out[:n].tobytes()


def xerial_decompress(b):
    a = _u8(b)
    n = lib().orc_xerial_decompressed_size(_p(a), a.size)
    if n < 0:
        raise IOError("snappy stream corrupt")
    out = np.empty(max(n, 1), dtype=np.uint8)
    r = lib().orc_xerial_decompress(_p(a), a.size, out.ctypes.data, n)
    if r < 0:
        raise IOError("snappy stream corrupt")
    return out[:r].tobytes()


# ---- shuffle metadata ----
def index_bytes(lengths):
    l = np.ascontiguousarray(lengths, dtype=np.int64)
    out = np.empty((l.size + 1) * 8, dtype=np.uint8)
    lib().orc_index_from_lengths(_p(l), l.size, out.ctypes.data)
    return out.tobytes()


def be64_bytes(values):
    v = np.ascontiguousarray(values, dtype=np.int64)
    out = np.empty(v.size * 8, dtype=np.uint8)
    lib().orc_be64_array(_p(v), v.size, out.ctypes.data)
    return out.tobytes()


def read_be64(b):
    a = _u8(b)
    out = np.empty(max(a.size // 8, 1), dtype=np.int64)
    n = lib().orc_read_be64_array(_p(a), a.size, out.ctypes.data)
    if n < 0:
        raise ValueError("Unexpected file length")  # SparkException in helper/S3ShuffleHelper.scala:112-114
    return out[:n].copy()


def validate_slices(alg, block, cumulative, ref, start_reduce, end_reduce):
    a = _u8(block)
    c = np.ascontiguousarray(cumulative, dtype=np.int64)
    r = np.ascontiguousarray(ref, dtype=np.int64)
    return lib().orc_validate_slices(alg, _p(a), c.ctypes.data, r.ctypes.data, start_reduce, end_reduce)


# ---- workload ----
def gen_terasort(first_record, n_records, seed=42):
    out = np.empty(n_records * 104, dtype=np.uint8)
    lib().orc_gen_terasort(out.ctypes.data, first_record, n_records, seed)
    return out


# ---- baseline ----
class _Job(C.Structure):
    _fields_ = [
        ("src", C.c_void_p),
        ("block_bytes", C.c_uint64),
        ("n_blocks", C.c_uint64),
        ("lz4_block_size", C.c_uint32),
        ("checksum_alg", C.c_uint32),
        ("threads", C.c_int),
        ("lz4_compress", C.c_void_p),
        ("lz4_decompress", C.c_void_p),
        ("write_seconds", C.c_double),
        ("read_seconds", C.c_double),
        ("compressed_bytes", C.c_uint64),
        ("errors", C.c_int),
    ]


def _liblz4():
    try:
        L = C.CDLL("liblz4.so.1")
        return (C.cast(L.LZ4_compress_default, C.c_void_p).value, C.cast(L.LZ4_decompress_fast, C.c_void_p).value)
    except OSError:
        return (None, None)


class _CodecJob(C.Structure):
    _fields_ = [("base", _Job), ("codec", C.c_uint32), ("level", C.c_int32), ("zstd_compress", C.c_void_p),
                ("zstd_decompress", C.c_void_p), ("zstd_is_error", C.c_void_p)]


def _libzstd():
    L = C.CDLL("libzstd.so.1")
    return tuple(C.cast(getattr(L, n), C.c_void_p).value for n in ("ZSTD_compress", "ZSTD_decompress", "ZSTD_isError"))


def baseline_run_codec(codec, data, block_bytes, block_size=32768, checksum_alg=CRC32C, threads=1, level=3):
    """baseline_run for codec "lz4" | "snappy" | "zstd" (zstd = libzstd.so.1 at `level`, snappy = the restated
    compressor under xerial framing).  Same result dict."""
    if codec == "lz4":
        return baseline_run(data, block_bytes, block_size, checksum_alg, threads, True)
    a = _u8(data)
    n_blocks = a.size // block_bytes
    zc, zd, ze = _libzstd() if codec == "zstd" else (None, None, None)
    job = _CodecJob(_Job(a.ctypes.data, block_bytes, n_blocks, block_size, checksum_alg, threads, None, None, 0, 0, 0, 0),
                    {"snappy": 2, "zstd": 3}[codec], level, zc, zd, ze)
    rc = lib().orc_baseline_run_codec(C.byref(job))
    b = job.base
    return dict(rc=rc, write_s=b.write_seconds, read_s=b.read_seconds, compressed_bytes=b.compressed_bytes,
                errors=b.errors, liblz4=False, bytes=n_blocks * block_bytes)


def baseline_run(data, block_bytes, lz4_block_size=32768, checksum_alg=CRC32C, threads=1, use_liblz4=True):
    """Times the reference's CPU arithmetic (LZ4Block stream + checksum) on `data` split into shuffle blocks of
    block_bytes.  Returns dict(write_s, read_s, compressed_bytes, errors, liblz4)."""
    a = _u8(data)
    n_blocks = a.size // block_bytes
    comp, decomp = _liblz4() if use_liblz4 else (None, None)
    job = _Job(a.ctypes.data, block_bytes, n_blocks, lz4_block_size, checksum_alg, threads, comp, decomp, 0, 0, 0, 0)
    rc = lib().orc_baseline_run(C.byref(job))
    return dict(
        rc=rc,
        write_s=job.write_seconds,
        read_s=job.read_seconds,
        compressed_bytes=job.compressed_bytes,
        errors=job.errors,
        liblz4=bool(comp),
        bytes=n_blocks * block_bytes,
    )
