// decimal128.h — the 128-bit integer arithmetic of the Decimal aggregate ops (B2S_AGG_SUM_DECIMAL, MIN / MAX_DECIMAL):
// the add with its overflow, the |x| < 10^P range check, the signed order and BigInteger.toByteArray's minimal
// big-endian encoding, written once for host and device.
//
// aggregate.cu's merge kernels call these.  tests/native/decimal128_host.cpp compiles the same functions with g++, and
// tests/test_decimal128.py checks them against Python integers without a GPU.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2S_HD __host__ __device__
#else
#ifndef B2S_HD
#define B2S_HD
#endif
#endif

namespace b2s {

// a signed 128-bit integer, two's complement
struct Dec128 {
  uint64_t lo, hi;
};

// 10^P for P = 0..38 as (lo, hi); the device reads its copy from constant memory
#define B2S_DEC_POW10                                                                                               \
  {{0x0000000000000001ull, 0}, {0x000000000000000aull, 0}, {0x0000000000000064ull, 0},                              \
   {0x00000000000003e8ull, 0}, {0x0000000000002710ull, 0}, {0x00000000000186a0ull, 0},                              \
   {0x00000000000f4240ull, 0}, {0x0000000000989680ull, 0}, {0x0000000005f5e100ull, 0},                              \
   {0x000000003b9aca00ull, 0}, {0x00000002540be400ull, 0}, {0x000000174876e800ull, 0},                              \
   {0x000000e8d4a51000ull, 0}, {0x000009184e72a000ull, 0}, {0x00005af3107a4000ull, 0},                              \
   {0x00038d7ea4c68000ull, 0}, {0x002386f26fc10000ull, 0}, {0x016345785d8a0000ull, 0},                              \
   {0x0de0b6b3a7640000ull, 0}, {0x8ac7230489e80000ull, 0}, {0x6bc75e2d63100000ull, 0x0000000000000005ull},          \
   {0x35c9adc5dea00000ull, 0x0000000000000036ull}, {0x19e0c9bab2400000ull, 0x000000000000021eull},                  \
   {0x02c7e14af6800000ull, 0x000000000000152dull}, {0x1bcecceda1000000ull, 0x000000000000d3c2ull},                  \
   {0x161401484a000000ull, 0x0000000000084595ull}, {0xdcc80cd2e4000000ull, 0x000000000052b7d2ull},                  \
   {0x9fd0803ce8000000ull, 0x00000000033b2e3cull}, {0x3e25026110000000ull, 0x00000000204fce5eull},                  \
   {0x6d7217caa0000000ull, 0x00000001431e0faeull}, {0x4674edea40000000ull, 0x0000000c9f2c9cd0ull},                  \
   {0xc0914b2680000000ull, 0x0000007e37be2022ull}, {0x85acef8100000000ull, 0x000004ee2d6d415bull},                  \
   {0x38c15b0a00000000ull, 0x0000314dc6448d93ull}, {0x378d8e6400000000ull, 0x0001ed09bead87c0ull},                  \
   {0x2b878fe800000000ull, 0x0013426172c74d82ull}, {0xb34b9f1000000000ull, 0x00c097ce7bc90715ull},                  \
   {0x00f436a000000000ull, 0x0785ee10d5da46d9ull}, {0x098a224000000000ull, 0x4b3b4ca85a86c47aull}}
#if defined(__CUDACC__)
static __constant__ uint64_t kDecPow10Dev[39][2] = B2S_DEC_POW10;
#endif
static constexpr uint64_t kDecPow10Host[39][2] = B2S_DEC_POW10;
#undef B2S_DEC_POW10

B2S_HD inline Dec128 dec_pow10(uint32_t p) {
#if defined(__CUDA_ARCH__)
  return {kDecPow10Dev[p][0], kDecPow10Dev[p][1]};
#else
  return {kDecPow10Host[p][0], kDecPow10Host[p][1]};
#endif
}

B2S_HD inline uint64_t dec_bswap64(uint64_t x) {
#if defined(__CUDA_ARCH__)
  return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
#else
  return __builtin_bswap64(x);
#endif
}

B2S_HD inline uint32_t dec_clz64(uint64_t x) {  // x != 0
#if defined(__CUDA_ARCH__)
  return (uint32_t)__clzll((long long)x);
#else
  return (uint32_t)__builtin_clzll(x);
#endif
}

B2S_HD inline Dec128 dec_of_long(uint64_t v) { return {v, (uint64_t)((int64_t)v >> 63)}; }

// a + b modulo 2^128, with the carry out of bit 127.  *ovf: the signed sum needs a 129th bit (both operands have one
// sign and the sum the other), so |a + b| >= 2^127 > 10^38.
B2S_HD inline Dec128 dec_add(Dec128 a, Dec128 b, bool* ovf) {
  Dec128 s;
  s.lo = a.lo + b.lo;
  s.hi = a.hi + b.hi + (s.lo < a.lo ? 1 : 0);
  *ovf = ((~(a.hi ^ b.hi) & (a.hi ^ s.hi)) >> 63) != 0;
  return s;
}

// |x| < 10^p (p <= 38): the range of Decimal(p, s)'s unscaled value
B2S_HD inline bool dec_fits(Dec128 x, uint32_t p) {
  uint64_t ml = x.lo, mh = x.hi;
  if (mh >> 63) {  // |x| as an unsigned 128-bit number (2^127 for the most negative x)
    ml = ~ml + 1;
    mh = ~mh + (ml == 0 ? 1 : 0);
  }
  const Dec128 lim = dec_pow10(p);
  return mh < lim.hi || (mh == lim.hi && ml < lim.lo);
}

// signed a < b
B2S_HD inline bool dec_less(Dec128 a, Dec128 b) {
  return (int64_t)a.hi < (int64_t)b.hi || (a.hi == b.hi && a.lo < b.lo);
}

// the length of BigInteger.toByteArray(x): bitlen(x >= 0 ? x : ~x) / 8 + 1, so 0 is one byte 00, 128 is 00 80 and
// -128 is 80 (1..16)
B2S_HD inline uint32_t dec_bytes(Dec128 x) {
  const uint64_t s = (uint64_t)((int64_t)x.hi >> 63);
  const uint64_t h = x.hi ^ s, l = x.lo ^ s;
  const uint32_t bits = h ? 128 - dec_clz64(h) : l ? 64 - dec_clz64(l) : 0;
  return bits / 8 + 1;
}

// The len (1..16) low bytes of x big-endian, then 16 - len zero bytes: memory bytes 0..7 and 8..15 as little-endian
// words (*m0, *m1).  With len = dec_bytes(x) that is BigInteger.toByteArray(x), zero-padded to 16 bytes.
B2S_HD inline void dec_encode(Dec128 x, uint32_t len, uint64_t* m0, uint64_t* m1) {
  const uint32_t s = 8 * (16 - len);  // x << s puts its len low bytes at the top
  uint64_t h = x.hi, l = x.lo;
  if (s >= 64) {
    h = l << (s - 64);
    l = 0;
  } else if (s) {
    h = (h << s) | (l >> (64 - s));
    l <<= s;
  }
  *m0 = dec_bswap64(h);
  *m1 = dec_bswap64(l);
}

}  // namespace b2s
