// murmur3.cuh — Murmur3_x86_32 as org.apache.spark.unsafe.hash.Murmur3_x86_32 has it, on the device.  Shared by the
// HashPartitioning ids (rows_hash.cu) and the round-robin sort's row hash (rows_round_robin.cu).
#pragma once

#include "kernels.h"

namespace b2s {

// rotl32: common.cuh
__device__ __forceinline__ uint32_t mix_k1(uint32_t k) { return rotl32(k * 0xcc9e2d51u, 15) * 0x1b873593u; }
__device__ __forceinline__ uint32_t mix_h1(uint32_t h, uint32_t k) { return rotl32(h ^ k, 13) * 5u + 0xe6546b64u; }
__device__ __forceinline__ uint32_t fmix(uint32_t h, uint32_t n) {
  h ^= n;
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  return h ^ (h >> 16);
}

// hashUnsafeBytes of the n bytes at p: 16 bytes per load, their four words mixed in order; then the last n % 16
// bytes: their whole words, then each tail byte sign-extended.  Over n % 4 == 0 it is hashUnsafeWords.
__device__ __forceinline__ uint32_t hash_bytes(const uint8_t* p, uint32_t n, uint32_t h) {
  uint64_t lo, hi;
  uint32_t q = 0;
  for (; q + 16 <= n; q += 16) {
    ld_span16<true>(p + q, 16, lo, hi);
    h = mix_h1(h, mix_k1((uint32_t)lo));
    h = mix_h1(h, mix_k1((uint32_t)(lo >> 32)));
    h = mix_h1(h, mix_k1((uint32_t)hi));
    h = mix_h1(h, mix_k1((uint32_t)(hi >> 32)));
  }
  const uint32_t r = n - q;
  if (r) {
    ld_span16<true>(p + q, (int)r, lo, hi);
    const uint32_t whole = r & ~3u;
    for (uint32_t b = 0; b < whole; b += 4)
      h = mix_h1(h, mix_k1((uint32_t)(b < 8 ? lo >> (8 * b) : hi >> (8 * (b - 8)))));
    for (uint32_t b = whole; b < r; b++) {
      const uint8_t v = (uint8_t)(b < 8 ? lo >> (8 * b) : hi >> (8 * (b - 8)));
      h = mix_h1(h, mix_k1((uint32_t)(int32_t)(int8_t)v));
    }
  }
  return fmix(h, n);
}

}  // namespace b2s
