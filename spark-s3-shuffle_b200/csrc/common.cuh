// common.cuh — shared device helpers for libb200shuffle (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200shuffle.h"

namespace b2s {

constexpr int kSMs = 132;  // H100 SXM; grids are sized in multiples of this

// ---- unaligned little-endian 32-bit load from global memory: two aligned words + funnel shift.
// Only ever touches the aligned words that contain bytes p..p+3 (safe at allocation edges).
__device__ __forceinline__ uint32_t ld32u(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const unsigned sh = (a & 3u) * 8u;
  const uint32_t lo = w[0];
  const uint32_t hi = sh ? w[1] : 0u;
  return __funnelshift_r(lo, hi, sh);
}
__device__ __forceinline__ uint32_t ld32u_ro(const uint8_t* p) {  // read-only data path (ld.global.nc)
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const unsigned sh = (a & 3u) * 8u;
  const uint32_t lo = __ldg(w);
  const uint32_t hi = sh ? __ldg(w + 1) : 0u;
  return __funnelshift_r(lo, hi, sh);
}

// ---- the n bytes at p (1 <= n <= 16) as two little-endian 8-byte values: lo = bytes 0..7, hi = bytes 8..15 (bytes
// past n are unspecified).  Reads only the aligned 8-byte words that contain a byte of [p, p+n) — one, two or three
// of them — so it cannot cross an allocation edge that the span itself does not cross.  RO selects the read-only data
// path (__ldg), which is right only for memory that no thread writes while the kernel runs.
template <bool RO>
__device__ __forceinline__ void ld_span16(const uint8_t* p, int n, uint64_t& lo, uint64_t& hi) {
  const int b = (int)(reinterpret_cast<uintptr_t>(p) & 7u);  // position of byte 0 in the first word
  // (p - b, not an integer cast: the compiler keeps p's address space and emits global loads)
  const uint64_t* w = reinterpret_cast<const uint64_t*>(p - b);
  const uint64_t w0 = RO ? __ldg(w) : w[0];
  const uint64_t w1 = b + n > 8 ? (RO ? __ldg(w + 1) : w[1]) : 0ull;
  const uint64_t w2 = b + n > 16 ? (RO ? __ldg(w + 2) : w[2]) : 0ull;
  const unsigned s = 8u * (unsigned)b;
  lo = (w0 >> s) | ((w1 << 1) << (63u - s));  // (x << 1) << (63 - s): no shift by 64 when s == 0
  hi = (w1 >> s) | ((w2 << 1) << (63u - s));
}
// ---- stores bytes 0..n-1 (0 <= n <= 16) of (lo, hi) as ld_span16 returns them at p, with naturally aligned 1, 2, 4
// and 8-byte stores (at most seven; each writes only bytes of [p, p+n))
__device__ __forceinline__ void st_span16(uint8_t* p, int n, uint64_t lo, uint64_t hi) {
  // head: up to 8-byte alignment, while the bytes last
  if ((reinterpret_cast<uintptr_t>(p) & 1u) && n >= 1) {
    *p = (uint8_t)lo;
    lo = (lo >> 8) | (hi << 56);
    hi >>= 8;
    p += 1;
    n -= 1;
  }
  if ((reinterpret_cast<uintptr_t>(p) & 2u) && n >= 2) {
    *reinterpret_cast<uint16_t*>(p) = (uint16_t)lo;
    lo = (lo >> 16) | (hi << 48);
    hi >>= 16;
    p += 2;
    n -= 2;
  }
  if ((reinterpret_cast<uintptr_t>(p) & 4u) && n >= 4) {
    *reinterpret_cast<uint32_t*>(p) = (uint32_t)lo;
    lo = (lo >> 32) | (hi << 32);
    hi >>= 32;
    p += 4;
    n -= 4;
  }
  // body and tail: sizes only shrink from here, so every store stays naturally aligned
  if (n >= 8) {
    *reinterpret_cast<uint64_t*>(p) = lo;
    lo = hi;
    p += 8;
    n -= 8;
  }
  if (n >= 8) {
    *reinterpret_cast<uint64_t*>(p) = lo;
    p += 8;
    n -= 8;
  }
  if (n >= 4) {
    *reinterpret_cast<uint32_t*>(p) = (uint32_t)lo;
    lo >>= 32;
    p += 4;
    n -= 4;
  }
  if (n >= 2) {
    *reinterpret_cast<uint16_t*>(p) = (uint16_t)lo;
    lo >>= 16;
    p += 2;
    n -= 2;
  }
  if (n >= 1) *p = (uint8_t)lo;
}

// ---- the whole warp copies n bytes (any alignment): aligned 16-byte destination pieces, one per lane per step, sources
// read with ld_span16 (read-only path: s must not be written while the kernel runs)
__device__ __forceinline__ void warp_copy(uint8_t* d, const uint8_t* s, uint64_t n, uint32_t lane) {
  uint64_t lo, hi;
  uint32_t head = (uint32_t)((16u - (reinterpret_cast<uintptr_t>(d) & 15u)) & 15u);
  if (head > n) head = (uint32_t)n;
  if (lane == 0 && head) {
    ld_span16<true>(s, (int)head, lo, hi);
    st_span16(d, (int)head, lo, hi);
  }
  d += head;
  s += head;
  n -= head;
  const uint64_t body = n & ~uint64_t(15);
  for (uint64_t q = (uint64_t)lane * 16; q < body; q += 32 * 16) {
    ld_span16<true>(s + q, 16, lo, hi);
    *reinterpret_cast<ulonglong2*>(d + q) = make_ulonglong2(lo, hi);
  }
  if (lane == 0 && n > body) {
    ld_span16<true>(s + body, (int)(n - body), lo, hi);
    st_span16(d + body, (int)(n - body), lo, hi);
  }
}

// ---- cooperative byte copy by a group of G lanes (lane in [0,G)), arbitrary alignment.
// Fast path moves 16 bytes per lane per step with aligned 128-bit stores; source words are re-aligned with
// funnel shifts so the loads stay aligned too.
template <int G>
__device__ __forceinline__ void group_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n,
                                           int lane) {
  // head: bring dst to 16-byte alignment
  uint32_t head = (uint32_t)((16u - (reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u);
  if (head > n) head = n;
  for (uint32_t i = lane; i < head; i += G) dst[i] = src[i];
  dst += head;
  src += head;
  n -= head;
  const uint32_t nvec = n >> 4;
  if (nvec) {
    const uintptr_t sa = reinterpret_cast<uintptr_t>(src);
    const unsigned sh = (sa & 3u) * 8u;
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(sa & ~uintptr_t(3));
    uint4* dv = reinterpret_cast<uint4*>(dst);
    if ((sa & 15u) == 0) {
      const uint4* sv = reinterpret_cast<const uint4*>(src);
      for (uint32_t i = lane; i < nvec; i += G) dv[i] = sv[i];
    } else {
      for (uint32_t i = lane; i < nvec; i += G) {
        const uint32_t* q = sw + i * 4;
        uint32_t a = q[0], b = q[1], c = q[2], d = q[3];
        uint32_t e = sh ? q[4] : 0u;
        uint4 o;
        o.x = __funnelshift_r(a, b, sh);
        o.y = __funnelshift_r(b, c, sh);
        o.z = __funnelshift_r(c, d, sh);
        o.w = __funnelshift_r(d, e, sh);
        dv[i] = o;
      }
    }
  }
  const uint32_t done = nvec << 4;
  for (uint32_t i = done + lane; i < n; i += G) dst[i] = src[i];
}

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return __funnelshift_l(x, x, r); }

// first error wins: status[i] is 0 until some thread records a negative code
__device__ __forceinline__ void set_status(int32_t* status, uint32_t i, int32_t code) {
  atomicCAS(reinterpret_cast<int*>(status + i), 0, code);
}

// ---- per-LZ4-block work descriptors shared by the codec kernels ----
struct BlockDesc {
  uint64_t src;     // byte offset of the payload (after the 21-byte header) in the source arena
  uint64_t dst;     // byte offset of the decoded bytes in the destination arena
  uint32_t clen;    // payload bytes
  uint32_t olen;    // decoded bytes
  uint32_t check;   // stored checksum field (XXH32 & 0x0FFFFFFF for LZ4Block)
  uint32_t stream;  // owning stream index; bit 31 set = stored RAW
};

}  // namespace b2s
