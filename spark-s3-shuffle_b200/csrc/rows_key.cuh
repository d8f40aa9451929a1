// rows_key.cuh — the order-preserving, prefix-free encoding of a row's composite key (kernels.h, KeySpec), one window
// at a time.  Shared by the row sort's key and refinement passes (rows.cu) and the range-partition step (rows_range.cu):
// comparing two encodings with memcmp is Spark SQL's ordering of the keys.
#pragma once

#include "kernels.h"

namespace b2s {

// Bytes [d, d + nb) (nb <= 20) of one record's encoded key (kernels.h, KeySpec), as five big-endian u32 words.  Named
// words, not an array: an array indexed by the byte position would live in local memory.
struct KeyWindow {
  uint32_t w0, w1, w2, w3, w4;
  uint32_t d, nb;
  __device__ __forceinline__ void put(uint32_t p, uint32_t v) {
    const uint32_t q = p - d;
    if (q >= nb) return;
    const uint32_t x = v << (8 * (3 - (q & 3))), k = q >> 2;
    w0 |= k == 0 ? x : 0u;
    w1 |= k == 1 ? x : 0u;
    w2 |= k == 2 ? x : 0u;
    w3 |= k == 3 ? x : 0u;
    w4 |= k == 4 ? x : 0u;
  }
  __device__ __forceinline__ uint32_t word(uint32_t k) const {
    return k == 0 ? w0 : k == 1 ? w1 : k == 2 ? w2 : k == 3 ? w3 : w4;
  }
};

__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
  return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
}

// A fixed-width number's len (1..8) bytes v (little-endian; bytes past len unspecified) as an unsigned number of len
// bytes whose order is the column's: an int with its sign bit flipped; a float (Spark SQL's order) with -0.0 made +0.0
// and every NaN the canonical quiet NaN, then every bit flipped when negative, else the sign bit.
__device__ __forceinline__ uint64_t ordered_bits(uint32_t ty, uint32_t len, uint64_t v) {
  const uint64_t sign = 1ull << (8 * len - 1), mag = v & (sign - 1);
  if (ty != B2S_KEY_FLOAT32 && ty != B2S_KEY_FLOAT64) return v ^ sign;
  const bool f32 = ty == B2S_KEY_FLOAT32;
  if (mag == 0) return sign;                                                   // +-0.0
  if (mag > (f32 ? 0x7f800000ull : 0x7ff0000000000000ull))                     // NaN
    return (f32 ? 0x7fc00000ull : 0x7ff8000000000000ull) | sign;
  return (v & sign) ? ~v & (sign | (sign - 1)) : v ^ sign;
}

// A decimal's slot (offset << 32) | size -> (hi, lo): its size bytes of the row, big-endian two's complement,
// sign-extended to 128 bits with the sign bit flipped.  *bad: the size is not 1..16 or the bytes run past the row; they
// are then clamped to 16 and to the row, so no load leaves it.
__device__ __forceinline__ void decimal_bits(const uint8_t* row, uint32_t row_size, uint64_t slot, uint64_t& hi,
                                             uint64_t& lo, bool* bad) {
  uint32_t so = (uint32_t)(slot >> 32), sz = (uint32_t)slot;
  if (sz - 1 >= 16u || (uint64_t)so + sz > row_size) {
    *bad = true;
    so = min(so, row_size);
    sz = min(min(sz, 16u), row_size - so);
  }
  hi = lo = 0;
  if (sz) {
    uint64_t a, b;
    ld_span16<true>(row + so, (int)sz, a, b);
    hi = bswap64(a);  // the 16 bytes from the value's first as a big-endian number: the value is its top sz bytes
    lo = bswap64(b);
    const uint32_t s = 8 * (16 - sz);  // an arithmetic shift right by s sign-extends it
    if (s >= 64) {
      lo = (uint64_t)((int64_t)hi >> (s - 64));
      hi = (uint64_t)((int64_t)hi >> 63);
    } else if (s) {
      lo = (lo >> s) | (hi << (64 - s));
      hi = (uint64_t)((int64_t)hi >> s);
    }
  }
  hi ^= 1ull << 63;
}

// The window kw of the encoded key of a row of row_size bytes.  whole: every column is walked and the return value is
// the key's encoded length (else the walk stops at the window's end); every non-null decimal slot is then checked.
// *bad: a non-null string slot runs past the row, or a decimal slot is bad (decimal_bits); the bytes read are then
// clamped to the row, so no load leaves it.  Join (the join's key pass): a column whose null_field is kNullByteOnly
// takes the null byte of a non-null value without reading a null word (its other side's column is nullable).  NullSafe
// (a join key with a B2S_KEY_NULL_SAFE column): such a column is (coalesce(v, default), isnull(v)): no leading null
// byte, its value's bytes or the type's default's when null (a null's slot is not read), then a trailing 0 / 1 byte.
template <bool Join = false, bool NullSafe = false>
__device__ __forceinline__ uint32_t encode_key(const uint8_t* row, uint32_t row_size, const KeySpec& ks, KeyWindow& kw,
                                               bool whole, bool* bad) {
  const uint32_t wend = kw.d + kw.nb;
  uint32_t p = 0;
  for (uint32_t c = 0; c < ks.n; c++) {
    if (!whole && p >= wend) break;
    const uint32_t ty = ks.type[c] & kKeyTypeMask, off = ks.off[c], len = ks.len[c];
    const uint32_t flip = ks.type[c] & B2S_KEY_DESCENDING ? 0xff : 0;  // DESC: every value byte complemented
    const int32_t nf = ks.null_field[c];
    const bool safe = Join && NullSafe && (ks.type[c] & B2S_KEY_NULL_SAFE);
    bool is_null = false;
    if (nf >= 0) {
      uint64_t nw, unused;
      ld_span16<true>(row + 8 * (uint32_t)(nf >> 6), 8, nw, unused);
      is_null = (nw >> (nf & 63)) & 1;
      if (!safe) kw.put(p++, is_null == ((ks.type[c] & B2S_KEY_NULLS_LAST) != 0) ? 1 : 0);
    } else if (Join && nf == kNullByteOnly) {
      kw.put(p++, 1);
    }
    if (ty == kStringKey) {
      if (is_null && !safe) continue;
      uint64_t slot, unused;
      if (safe && is_null) slot = 0;  // a null-safe null: the empty string
      else ld_span16<true>(row + off, 8, slot, unused);
      uint32_t so = (uint32_t)(slot >> 32), sz = (uint32_t)slot;
      if ((uint64_t)so + sz > row_size) {
        *bad = true;
        so = min(so, row_size);
        sz = min(sz, row_size - so);
      }
      const uint32_t groups = sz ? (sz + 7) / 8 : 1;
      for (uint32_t g = kw.d > p ? (kw.d - p) / 9 : 0; g < groups && p + 9 * g < wend; g++) {
        const uint32_t base = p + 9 * g, real = min(8u, sz - 8 * g);
        uint64_t v = 0, unused2;
        if (real) {
          ld_span16<true>(row + so + 8 * g, (int)real, v, unused2);
          if (real < 8) v &= (1ull << (8 * real)) - 1;
        }
        for (uint32_t b = 0; b < 8; b++) kw.put(base + b, ((uint32_t)(v >> (8 * b)) & 0xff) ^ flip);
        kw.put(base + 8, (g + 1 < groups ? 9 : real) ^ flip);
      }
      p += 9 * groups;
    } else {
      const uint32_t w = key_value_bytes(ty, len);
      const bool in_window = p < wend && p + w > kw.d;
      if (!is_null && (in_window || (whole && ty == kDecimalKey))) {  // a null's bytes stay zero
        uint64_t lo, hi;
        ld_span16<true>(row + off, (int)len, lo, hi);
        if (ty == kDecimalKey) decimal_bits(row, row_size, /* the slot */ lo, hi, lo, bad);
        else if (ty != B2S_KEY_BYTES) lo = ordered_bits(ty, len, lo);
        // BYTES in memory order; a number (lo, or hi:lo for a decimal) most significant byte first
        for (uint32_t b = 0; in_window && b < w; b++) {
          const uint32_t s = ty == B2S_KEY_BYTES ? b : w - 1 - b;
          kw.put(p + b, ((uint32_t)(s < 8 ? lo >> (8 * s) : hi >> (8 * (s - 8))) & 0xff) ^ flip);
        }
      } else if (safe && is_null && in_window) {  // the default, 0 (false; BYTES all zero), encoded as a value
        const uint64_t lo = ty == B2S_KEY_BYTES || ty == kDecimalKey ? 0 : ordered_bits(ty, len, 0);
        const uint64_t hi = ty == kDecimalKey ? 1ull << 63 : 0;
        for (uint32_t b = 0; b < w; b++) {
          const uint32_t s = ty == B2S_KEY_BYTES ? b : w - 1 - b;
          kw.put(p + b, (uint32_t)(s < 8 ? lo >> (8 * s) : hi >> (8 * (s - 8))) & 0xff);
        }
      }
      p += w;
    }
    if (safe) kw.put(p++, is_null ? 1 : 0);
  }
  return p;
}

// Two rows' keys ks are equal: their encodings compared kKeyChunkBytes at a time.  Equal so far and one key ended inside
// the window: the encoding is prefix-free, so both did.  For keys whose strings and decimals have been checked.
__device__ __forceinline__ bool encoded_keys_equal(const uint8_t* ra, uint32_t sa, const uint8_t* rb, uint32_t sb,
                                                   const KeySpec& ks) {
  bool bad = false;
  for (uint32_t d = 0;; d += kKeyChunkBytes) {
    KeyWindow wa{0, 0, 0, 0, 0, d, kKeyChunkBytes}, wb{0, 0, 0, 0, 0, d, kKeyChunkBytes};
    const uint32_t la = encode_key(ra, sa, ks, wa, false, &bad);
    const uint32_t lb = encode_key(rb, sb, ks, wb, false, &bad);
    if (wa.w0 != wb.w0 || wa.w1 != wb.w1 || wa.w2 != wb.w2 || wa.w3 != wb.w3) return false;
    if (min(la, lb) < d + kKeyChunkBytes) return true;
  }
}

}  // namespace b2s
