"""A model of Spark's HashPartitioning id of an UnsafeRow, pmod(Murmur3Hash(key columns, 42), R), for the tests of
b2s_partition_compress_rows_hash_*, in two forms:

- scalar: one row at a time, in plain Python ints, straight from org.apache.spark.unsafe.hash.Murmur3_x86_32 and
  Murmur3HashFunction (pinned by the vectors of Spark's Murmur3_x86_32Suite and its SQL documentation);
- vectorised: numpy over every record of a buffer at once (uint32 arithmetic wraps), which the GPU tests use at scale;
  a string longer than LONG_BYTES is hashed by the scalar form, since a hash is sequential along its bytes.

A key column is (key_type, key_off, key_len, null_field) as the composite-key calls take it.  Also here: a builder of
UnsafeRows with typed fields, and serialized records ([int32 big-endian size][row])."""
import math
import struct

import numpy as np

KEY_BYTES, KEY_INT32, KEY_INT64, STRING, KEY_INT16, KEY_INT8, KEY_FLOAT32, KEY_FLOAT64, DECIMAL = 0, 1, 2, 3, 5, 6, 7, 8, 9
SEED = 42
M32 = 0xFFFFFFFF
LONG_BYTES = 1 << 16


# ---------------------------------------------------------------------------------------------------------------
# scalar
# ---------------------------------------------------------------------------------------------------------------
def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & M32


def _mix_k1(k):
    return (_rotl((k * 0xCC9E2D51) & M32, 15) * 0x1B873593) & M32


def _mix_h1(h, k):
    return (_rotl(h ^ k, 13) * 5 + 0xE6546B64) & M32


def _fmix(h, n):
    h ^= n
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    return h ^ (h >> 16)


def hash_int(v, seed):
    return _fmix(_mix_h1(seed & M32, _mix_k1(v & M32)), 4)


def hash_long(v, seed):
    v &= (1 << 64) - 1
    return _fmix(_mix_h1(_mix_h1(seed & M32, _mix_k1(v & M32)), _mix_k1(v >> 32)), 8)


def hash_bytes(b, seed):
    """hashUnsafeBytes: whole little-endian words, then every tail byte on its own, sign-extended"""
    h, n = seed & M32, len(b)
    whole = n - n % 4
    for i in range(0, whole, 4):
        h = _mix_h1(h, _mix_k1(int.from_bytes(b[i:i + 4], "little")))
    for i in range(whole, n):
        h = _mix_h1(h, _mix_k1((b[i] - 256 if b[i] > 127 else b[i]) & M32))
    return _fmix(h, n)


def signed(h):
    return h - (1 << 32) if h >> 31 else h


def pmod(h, R):
    """Java's r = h % R; if (r < 0) r += R, of a signed 32-bit h (Python's % of a positive R is that already)"""
    return signed(h) % R


def is_null(row, f):
    return f >= 0 and (int.from_bytes(row[8 * (f >> 6):8 * (f >> 6) + 8], "little") >> (f & 63)) & 1


def col_hash(row, col, h):
    """one key column of a row folded into h (a null one leaves it)"""
    kt, ko, kl, nf = col
    if is_null(row, nf):
        return h
    raw = bytes(row[ko:ko + kl])
    if kt == KEY_BYTES:
        return hash_int(1 if raw[0] else 0, h)
    if kt in (KEY_INT8, KEY_INT16, KEY_INT32):
        return hash_int(int.from_bytes(raw, "little", signed=True), h)
    if kt == KEY_INT64:
        return hash_long(int.from_bytes(raw, "little", signed=True), h)
    if kt == KEY_FLOAT32:
        f = struct.unpack("<f", raw)[0]
        bits = 0 if f == 0.0 else 0x7FC00000 if math.isnan(f) else int.from_bytes(raw, "little")
        return hash_int(bits, h)
    if kt == KEY_FLOAT64:
        f = struct.unpack("<d", raw)[0]
        bits = 0 if f == 0.0 else 0x7FF8000000000000 if math.isnan(f) else int.from_bytes(raw, "little")
        return hash_long(bits, h)
    assert kt in (STRING, DECIMAL)
    slot = int.from_bytes(raw, "little")
    o, s = slot >> 32, slot & M32
    return hash_bytes(bytes(row[o:o + s]), h)


def row_hash(row, keys):
    """Murmur3Hash(keys, 42) of a row (bytes without the size prefix), unsigned 32 bits"""
    h = SEED
    for col in keys:
        h = col_hash(row, col, h)
    return h


def ids_scalar(rows, keys, R):
    return np.array([pmod(row_hash(r, keys), R) for r in rows], dtype=np.uint32)


# ---------------------------------------------------------------------------------------------------------------
# vectorised
# ---------------------------------------------------------------------------------------------------------------
def _v_rotl(x, r):
    return (x << np.uint32(r)) | (x >> np.uint32(32 - r))


def _v_mix_k1(k):
    return _v_rotl(k * np.uint32(0xCC9E2D51), 15) * np.uint32(0x1B873593)


def _v_mix_h1(h, k):
    return _v_rotl(h ^ k, 13) * np.uint32(5) + np.uint32(0xE6546B64)


def _v_fmix(h, n):
    h = h ^ n
    h ^= h >> np.uint32(16)
    h *= np.uint32(0x85EBCA6B)
    h ^= h >> np.uint32(13)
    h *= np.uint32(0xC2B2AE35)
    return h ^ (h >> np.uint32(16))


def _v_hash_int(v, h):
    return _v_fmix(_v_mix_h1(h, _v_mix_k1(v.astype(np.uint32))), np.uint32(4))


def _v_hash_long(v, h):
    v = v.astype(np.uint64)
    lo = (v & np.uint64(M32)).astype(np.uint32)
    hi = (v >> np.uint64(32)).astype(np.uint32)
    return _v_fmix(_v_mix_h1(_v_mix_h1(h, _v_mix_k1(lo)), _v_mix_k1(hi)), np.uint32(8))


def _v_read(buf, pos, n):
    """the n-byte (n <= 8) little-endian unsigned values at buf[pos]"""
    v = np.zeros(pos.size, np.uint64)
    for b in range(n):
        v |= buf[pos + b].astype(np.uint64) << np.uint64(8 * b)
    return v


def _v_hash_bytes(buf, p, n, h):
    """hashUnsafeBytes of the n[i] bytes at buf[p[i]], seeds h (all n <= LONG_BYTES)"""
    h = h.copy()
    nw = n // 4
    for w in range(int(nw.max()) if n.size else 0):
        sel = np.nonzero(nw > w)[0]
        word = _v_read(buf, p[sel] + 4 * w, 4).astype(np.uint32)
        h[sel] = _v_mix_h1(h[sel], _v_mix_k1(word))
    for t in range(3):
        sel = np.nonzero(n % 4 > t)[0]
        byte = buf[p[sel] + 4 * nw[sel] + t].astype(np.int8).astype(np.int32).astype(np.uint32)
        h[sel] = _v_mix_h1(h[sel], _v_mix_k1(byte))
    return _v_fmix(h, n.astype(np.uint32))


def row_hash_np(buf, row_start, keys):
    """Murmur3Hash(keys, 42) of the rows starting at buf[row_start[i]] (uint8 buffer), as uint32"""
    buf = np.asarray(buf, np.uint8)
    row_start = np.asarray(row_start, np.int64)
    h = np.full(row_start.size, SEED, np.uint32)
    for kt, ko, kl, nf in keys:
        live = np.ones(row_start.size, bool)
        if nf >= 0:
            word = _v_read(buf, row_start + 8 * (nf >> 6), 8)
            live = ((word >> np.uint64(nf & 63)) & np.uint64(1)) == 0
        idx = np.nonzero(live)[0]
        v = _v_read(buf, row_start[idx] + ko, kl)
        if kt == KEY_BYTES:
            new = _v_hash_int((v & np.uint64(0xFF)) != 0, h[idx])
        elif kt in (KEY_INT8, KEY_INT16, KEY_INT32):
            sdt = {KEY_INT8: np.int8, KEY_INT16: np.int16, KEY_INT32: np.int32}[kt]
            udt = {KEY_INT8: np.uint8, KEY_INT16: np.uint16, KEY_INT32: np.uint32}[kt]
            new = _v_hash_int(v.astype(udt).view(sdt).astype(np.int32).view(np.uint32), h[idx])
        elif kt == KEY_INT64:
            new = _v_hash_long(v, h[idx])
        elif kt == KEY_FLOAT32:
            f = v.astype(np.uint32).view(np.float32)
            bits = np.where(f == 0, np.uint32(0), np.where(np.isnan(f), np.uint32(0x7FC00000), v.astype(np.uint32)))
            new = _v_hash_int(bits, h[idx])
        elif kt == KEY_FLOAT64:
            f = v.view(np.float64)
            bits = np.where(f == 0, np.uint64(0), np.where(np.isnan(f), np.uint64(0x7FF8000000000000), v))
            new = _v_hash_long(bits, h[idx])
        else:
            so = (v >> np.uint64(32)).astype(np.int64)
            sz = (v & np.uint64(M32)).astype(np.int64)
            new = np.empty(idx.size, np.uint32)
            short = sz <= LONG_BYTES
            s = np.nonzero(short)[0]
            new[s] = _v_hash_bytes(buf, row_start[idx[s]] + so[s], sz[s], h[idx[s]])
            for j in np.nonzero(~short)[0]:
                p = int(row_start[idx[j]] + so[j])
                new[j] = hash_bytes(bytes(buf[p:p + int(sz[j])]), int(h[idx[j]]))
        h[idx] = new
    return h


def ids_np(buf, row_start, keys, R):
    """the partition ids pmod(hash, R) of the rows at row_start"""
    h = row_hash_np(buf, row_start, keys).view(np.int32).astype(np.int64)
    return (h % R).astype(np.uint32)


def record_ids_np(records, rec_len, keys, R):
    """ids of serialized records back to back in records (uint8), rec_len[i] bytes each"""
    rec_len = np.asarray(rec_len, np.int64)
    start = np.concatenate([[0], np.cumsum(rec_len)[:-1]]).astype(np.int64) if rec_len.size else np.zeros(0, np.int64)
    return ids_np(records, start + 4, keys, R)


# ---------------------------------------------------------------------------------------------------------------
# rows
# ---------------------------------------------------------------------------------------------------------------
# field types of the row builder -> (key_type, key_len)
FIELD = {"bool": (KEY_BYTES, 1), "byte": (KEY_INT8, 1), "short": (KEY_INT16, 2), "int": (KEY_INT32, 4),
         "long": (KEY_INT64, 8), "float": (KEY_FLOAT32, 4), "double": (KEY_FLOAT64, 8), "string": (STRING, 8),
         "decimal": (DECIMAL, 8)}


def decimal_bytes(unscaled):
    """BigInteger.toByteArray: the minimal big-endian two's complement bytes (1 at least)"""
    n = 1
    while not -(1 << (8 * n - 1)) <= unscaled < (1 << (8 * n - 1)):
        n += 1
    return unscaled.to_bytes(n, "big", signed=True)


def make_row(types, values):
    """an UnsafeRow of fields types[i] = values[i] (None: null); strings are bytes, decimals unscaled ints, floats
    either Python floats or raw bit patterns given as ("bits", int)"""
    nf = len(types)
    bitset = 8 * ((nf + 63) // 64)
    fixed = bytearray(bitset + 8 * nf)
    var = bytearray()
    base = bitset + 8 * nf
    for i, (t, v) in enumerate(zip(types, values)):
        slot = bitset + 8 * i
        if v is None:
            w = 8 * (i >> 6)
            fixed[w:w + 8] = (int.from_bytes(fixed[w:w + 8], "little") | (1 << (i & 63))).to_bytes(8, "little")
            continue
        if t in ("string", "decimal"):
            data = bytes(v) if t == "string" else decimal_bytes(v)
            fixed[slot:slot + 8] = (((base + len(var)) << 32) | len(data)).to_bytes(8, "little")
            var += data + bytes(-len(data) % 8)
        elif t in ("float", "double"):
            if isinstance(v, tuple):
                raw = v[1].to_bytes(4 if t == "float" else 8, "little")
            else:
                raw = struct.pack("<f" if t == "float" else "<d", v)
            fixed[slot:slot + len(raw)] = raw
        elif t == "bool":
            fixed[slot] = 1 if v else 0
        else:
            kl = FIELD[t][1]
            fixed[slot:slot + kl] = int(v).to_bytes(kl, "little", signed=True)
    return bytes(fixed + var)


def keys_of(types, fields, nullable=True):
    """the key columns (type, off, len, null field) of fields (indices into types) of make_row's rows"""
    bitset = 8 * ((len(types) + 63) // 64)
    return [(FIELD[types[f]][0], bitset + 8 * f, FIELD[types[f]][1], f if nullable else -1) for f in fields]


def records_of(rows):
    """serialized records back to back -> (uint8 buffer, rec_len uint32)"""
    buf = b"".join(len(r).to_bytes(4, "big") + r for r in rows)
    return (np.frombuffer(buf, np.uint8).copy() if buf else np.zeros(0, np.uint8),
            np.array([4 + len(r) for r in rows], np.uint32))


# a composite key of every type: (string, int, decimal(28), double, boolean, short, byte, float)
COMPOSITE = ["string", "int", "decimal", "double", "bool", "short", "byte", "float"]
SPECIAL_F64 = [0.0, -0.0, ("bits", 0x7FF8000000000000), ("bits", 0x7FF0000000000001), ("bits", 0xFFF8000000000123),
               ("bits", 0x7FFFFFFFFFFFFFFF), float("inf"), -float("inf"), 1.5]
SPECIAL_F32 = [0.0, -0.0, ("bits", 0x7FC00000), ("bits", 0x7F800001), ("bits", 0xFFC00123), ("bits", 0x7FFFFFFF),
               float("inf"), -2.5]


def random_rows(rng, n, types=COMPOSITE, null_rate=0.15, max_str=40):
    rows = []
    for i in range(n):
        vals = []
        for t in types:
            if rng.random() < null_rate:
                vals.append(None)
            elif t == "string":
                ln = int(rng.integers(0, max_str)) if rng.random() < 0.8 else int(rng.integers(0, 4))
                vals.append(bytes(rng.integers(0, 256, ln, dtype=np.uint8)))
            elif t == "decimal":
                nb = int(rng.integers(1, 17))
                vals.append(int.from_bytes(bytes(rng.integers(0, 256, nb, dtype=np.uint8)), "big", signed=True))
            elif t == "double":
                vals.append(SPECIAL_F64[rng.integers(len(SPECIAL_F64))] if rng.random() < 0.4
                            else float(rng.normal() * 1e6))
            elif t == "float":
                vals.append(SPECIAL_F32[rng.integers(len(SPECIAL_F32))] if rng.random() < 0.4
                            else float(np.float32(rng.normal() * 1e3)))
            elif t == "bool":
                vals.append(bool(rng.integers(2)))
            else:
                bits = {"byte": 8, "short": 16, "int": 32, "long": 64}[t]
                vals.append(int(rng.integers(-(1 << (bits - 1)), 1 << (bits - 1), dtype=np.int64)) if bits < 64
                            else int(rng.integers(-(1 << 62), 1 << 62)) * 2 + int(rng.integers(2)))
        if i % 17 == 0:
            vals = [None] * len(types)
        rows.append(make_row(types, vals))
    return rows
