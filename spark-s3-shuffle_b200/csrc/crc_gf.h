// crc_gf.h — GF(2) arithmetic modulo a CRC polynomial and the power tables of the K1 checksum kernels, written once
// for host and device.
//
// checksum.cu builds the tables on the host (build_crc_tables) and its kernels shift partial CRCs with gf_mul /
// gf_xpow8.  tests/native/crc_gf_host.cpp compiles the same functions with g++, and tests/test_crc_gf.py checks them
// against plain polynomial arithmetic without a GPU.
//
// Representation: reflected, as the CRC registers are — bit 31 holds x^0, bit 0 holds x^31; poly is the reflected
// polynomial without its x^32 term (0xEDB88320 for CRC32, 0x82F63B78 for CRC32C).
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

constexpr uint32_t kGfOne = 0x80000000u;  // x^0 in the reflected representation

// misc table layout, per polynomial: x^(2^k) and x^-(2^k) for k = 0 .. kPowBits-1 (a byte count e shifts by x^(8e), so
// bit j of a 64-bit e needs k = j + 3 <= 66), then the 32 lane-fold constants, then poly.
constexpr int kPowBits = 64 + 3;
constexpr int kMiscXPow = 0;
constexpr int kMiscXInv = kMiscXPow + kPowBits;
constexpr int kMiscLane = kMiscXInv + kPowBits;
constexpr int kMiscPoly = kMiscLane + 32;
constexpr int kMiscWords = kMiscPoly + 1;

// a * b mod P
B2S_HD inline uint32_t gf_mul(uint32_t a, uint32_t b, uint32_t poly) {
  uint32_t p = 0;
#pragma unroll 8
  for (int i = 0; i < 32; i++) {
    p ^= (uint32_t)((int32_t)a >> 31) & b;
    a <<= 1;
    b = (b >> 1) ^ ((0u - (b & 1u)) & poly);
  }
  return p;
}

// x^(8*e) mod P for e bytes; tab = x^(2^k) (or x^-(2^k) for x^(-8*e)), k = 3 .. 66.  Every k has its own entry: the
// powers x^(2^k) mod P repeat with a period that depends on how P factors (32 for CRC32, 31 for CRC32C).
B2S_HD inline uint32_t gf_xpow8(uint64_t e, const uint32_t* tab, uint32_t poly) {
  uint32_t p = kGfOne;
  unsigned k = 3;
  while (e) {
    if (e & 1) p = gf_mul(tab[k], p, poly);
    e >>= 1;
    k++;
  }
  return p;
}

// rows[16*256]: R[k][b] = register after byte b followed by 511-k zero bytes (Z_496..Z_511); misc[kMiscWords] as above
inline void build_crc_tables(uint32_t poly, uint32_t* rows, uint32_t* misc) {
  uint32_t t0[256];
  for (uint32_t i = 0; i < 256; i++) {
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ poly : (c >> 1);
    t0[i] = c;
  }
  // Z_j[b] = register after byte b followed by j zero bytes
  uint32_t z[256];
  for (int b = 0; b < 256; b++) z[b] = t0[b];
  for (int j = 0; j <= 511; j++) {
    if (j >= 496) {
      int k = 511 - j;  // R[k] = Z_{511-k}
      for (int b = 0; b < 256; b++) rows[k * 256 + b] = z[b];
    }
    for (int b = 0; b < 256; b++) z[b] = (z[b] >> 8) ^ t0[z[b] & 0xff];
  }
  uint32_t* x2n = misc + kMiscXPow;
  uint32_t* xinv2n = misc + kMiscXInv;
  uint32_t p = 1u << 30;  // x^1
  x2n[0] = p;
  for (int k = 1; k < kPowBits; k++) {
    p = gf_mul(p, p, poly);
    x2n[k] = p;
  }
  p = (((kGfOne ^ poly) << 1) | 1u);  // x^-1
  xinv2n[0] = p;
  for (int k = 1; k < kPowBits; k++) {
    p = gf_mul(p, p, poly);
    xinv2n[k] = p;
  }
  for (int l = 0; l < 32; l++) misc[kMiscLane + l] = gf_xpow8((uint64_t)16 * (31 - l), x2n, poly);
  misc[kMiscPoly] = poly;
}

}  // namespace b2s
