// rows_hash.cu — Spark's HashPartitioning id of length-prefixed UnsafeRow records: pmod(Murmur3Hash(keys, 42), R),
// the map side of a hash exchange (ShuffleExchangeExec computes it per row before the writer sees the record).
// Murmur3_x86_32 (murmur3.cuh), byte strings with Spark's legacy tail: every tail byte mixed on its own,
// sign-extended.  A thread per record; the ids go to the partition step's id array.
#include <algorithm>

#include "kernels.h"
#include "murmur3.cuh"

namespace b2s {

namespace {

constexpr int kHashThreads = 256;
constexpr uint32_t kHashSeed = 42;  // HashPartitioning's Murmur3Hash seed

__device__ __forceinline__ uint32_t hash_int(uint32_t v, uint32_t seed) { return fmix(mix_h1(seed, mix_k1(v)), 4); }
__device__ __forceinline__ uint32_t hash_long(uint64_t v, uint32_t seed) {
  const uint32_t h = mix_h1(seed, mix_k1((uint32_t)v));
  return fmix(mix_h1(h, mix_k1((uint32_t)(v >> 32))), 8);
}

// ids[i] = record i's partition id; a bad record lowers *bad to (i << 3) | kHashBad* and takes id 0.  A record that
// ends past rec_bytes is not read (the partition step's length sum reports it).  min_key / min_null: the row bytes that
// hold every key slot / every null word of a nullable key column.  NullSafe: a B2S_KEY_NULL_SAFE column hashes its
// value, or its type's default when null (a null's slot is not read), then hashInt(isnull); without it a key type
// carries no flag.
template <bool NullSafe>
__device__ __forceinline__ void hash_rows(const uint8_t* __restrict__ rec, uint64_t rec_bytes,
                                          const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
                                          uint64_t n, const KeySpec& ks, uint32_t min_key, uint32_t min_null,
                                          uint32_t num_partitions, uint32_t* __restrict__ ids,
                                          unsigned long long* __restrict__ bad) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t o = rec_off[i];
    const uint32_t len = rec_len[i];
    uint32_t id = 0;
    uint64_t why = 0;
    if (o + len <= rec_bytes) {
      uint64_t lo, hi;
      uint32_t size = 0;
      if (len >= 4) {
        ld_span16<true>(rec + o, 4, lo, hi);
        size = __byte_perm((uint32_t)lo, 0, 0x0123);
      }
      const uint8_t* row = rec + o + 4;
      if (len < 4) why = kHashBadShort;
      else if (size != len - 4) why = kHashBadSize;
      else if (size < min_key) why = kHashBadKey;
      else if (size < min_null) why = kHashBadNull;
      uint32_t h = kHashSeed;
      for (uint32_t c = 0; !why && c < ks.n; c++) {
        const int32_t nf = ks.null_field[c];
        const bool safe = NullSafe && (ks.type[c] & B2S_KEY_NULL_SAFE);
        bool is_null = false;
        if (nf >= 0) {
          ld_span16<true>(row + 8 * (uint32_t)(nf >> 6), 8, lo, hi);
          is_null = (lo >> (nf & 63)) & 1;
          if (is_null && !safe) continue;  // a null column leaves the hash as it is
        }
        const uint32_t ty = NullSafe ? ks.type[c] & kKeyTypeMask : ks.type[c];
        if (NullSafe && is_null) {  // the default: 0, false, the empty string, a wide decimal's one byte 0x00
          lo = hi = 0;
        } else {
          ld_span16<true>(row + ks.off[c], (int)ks.len[c], lo, hi);
        }
        if (NullSafe && is_null && (ty == kStringKey || ty == kDecimalKey)) {
          h = ty == kStringKey ? fmix(h, 0) : fmix(mix_h1(h, mix_k1(0)), 1);
        } else switch (ty) {
          case B2S_KEY_BYTES: h = hash_int((lo & 0xff) ? 1u : 0u, h); break;  // BooleanType
          case B2S_KEY_INT8: h = hash_int((uint32_t)(int32_t)(int8_t)lo, h); break;
          case B2S_KEY_INT16: h = hash_int((uint32_t)(int32_t)(int16_t)lo, h); break;
          case B2S_KEY_INT32: h = hash_int((uint32_t)lo, h); break;
          case B2S_KEY_INT64: h = hash_long(lo, h); break;
          case B2S_KEY_FLOAT32: {  // -0.0 as 0, every NaN as floatToIntBits' canonical one
            uint32_t v = (uint32_t)lo;
            const uint32_t mag = v & 0x7fffffffu;
            v = mag == 0 ? 0u : mag > 0x7f800000u ? 0x7fc00000u : v;
            h = hash_int(v, h);
            break;
          }
          case B2S_KEY_FLOAT64: {
            const uint64_t mag = lo & 0x7fffffffffffffffull;
            h = hash_long(mag == 0 ? 0ull : mag > 0x7ff0000000000000ull ? 0x7ff8000000000000ull : lo, h);
            break;
          }
          default: {  // a string's or a wide decimal's (offset << 32) | size slot
            const uint32_t so = (uint32_t)(lo >> 32), sz = (uint32_t)lo;
            if (ty == kDecimalKey && sz - 1 >= 16u) why = kHashBadDecimal;
            else if ((uint64_t)so + sz > size) why = ty == kDecimalKey ? kHashBadDecimal : kHashBadString;
            else h = hash_bytes(row + so, sz, h);
          }
        }
        if (safe) h = hash_int(is_null ? 1u : 0u, h);
      }
      if (why) atomicMin(bad, (unsigned long long)((i << 3) | why));
      else {
        const int32_t m = (int32_t)h % (int32_t)num_partitions;  // num_partitions <= 2^24: Java's pmod
        id = (uint32_t)(m < 0 ? m + (int32_t)num_partitions : m);
      }
    }
    ids[i] = id;
  }
}

__global__ void __launch_bounds__(kHashThreads) rows_hash_kernel(
    const uint8_t* __restrict__ rec, uint64_t rec_bytes, const uint64_t* __restrict__ rec_off,
    const uint32_t* __restrict__ rec_len, uint64_t n, const __grid_constant__ KeySpec ks, uint32_t min_key,
    uint32_t min_null, uint32_t num_partitions, uint32_t* __restrict__ ids, unsigned long long* __restrict__ bad) {
  hash_rows<false>(rec, rec_bytes, rec_off, rec_len, n, ks, min_key, min_null, num_partitions, ids, bad);
}

// the hash call's kernel for keys with a B2S_KEY_NULL_SAFE column; every other caller keeps rows_hash_kernel
__global__ void __launch_bounds__(kHashThreads) rows_hash_null_safe_kernel(
    const uint8_t* __restrict__ rec, uint64_t rec_bytes, const uint64_t* __restrict__ rec_off,
    const uint32_t* __restrict__ rec_len, uint64_t n, const __grid_constant__ KeySpec ks, uint32_t min_key,
    uint32_t min_null, uint32_t num_partitions, uint32_t* __restrict__ ids, unsigned long long* __restrict__ bad) {
  hash_rows<true>(rec, rec_bytes, rec_off, rec_len, n, ks, min_key, min_null, num_partitions, ids, bad);
}

}  // namespace

void launch_rows_hash(const uint8_t* rec, uint64_t rec_bytes, const uint64_t* rec_off, const uint32_t* rec_len,
                      uint64_t n, const KeySpec& ks, uint32_t num_partitions, uint32_t* ids, uint64_t* bad,
                      cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  uint64_t min_key = 0, min_null = 0;
  bool null_safe = false;
  for (uint32_t c = 0; c < ks.n; c++) {
    null_safe |= (ks.type[c] & B2S_KEY_NULL_SAFE) != 0;
    min_key = std::max<uint64_t>(min_key, (uint64_t)ks.off[c] + ks.len[c]);
    if (ks.null_field[c] >= 0) min_null = std::max<uint64_t>(min_null, 8ull * (uint32_t)(ks.null_field[c] >> 6) + 8);
  }
  min_key = std::min<uint64_t>(min_key, 0xffffffffull);  // a row is below 2^32 - 4 bytes: no slot past that is held
  const uint64_t want = (n + kHashThreads - 1) / kHashThreads;
  const unsigned grid = (unsigned)(want < (uint64_t)kSMs * 16 ? want : (uint64_t)kSMs * 16);
  auto kernel = null_safe ? rows_hash_null_safe_kernel : rows_hash_kernel;
  kernel<<<grid, kHashThreads, 0, st>>>(rec, rec_bytes, rec_off, rec_len, n, ks, (uint32_t)min_key, (uint32_t)min_null,
                                        num_partitions, ids, (unsigned long long*)bad);
  if (launches) *launches += 1;
}

}  // namespace b2s
