// lz4_decode.cu — the read side of LZ4Block: the lz4-java stream framing and K4, LZ4 block decompression
// (LZ4_decompress_fast semantics: driven by originalLen, must consume exactly compressedLen; oracle:
// orc_lz4_decompress_block).  K3, the compressor, and the write-side framing live in lz4_compress.cu.
//
// Replaces liblz4's LZ4_decompress_fast as driven by lz4-java's LZ4BlockInputStream [U] under
// serializerManager.wrapStream at storage/S3ShuffleReader.scala:107-109.
// Wire format (oracle/b2s_oracle.c restates it): per <= blockSize bytes of input a 21-byte header
//   "LZ4Block" | token = method(0x10 RAW, 0x20 LZ4) | level | compressedLen LE32 | originalLen LE32 | XXH32&0x0FFFFFFF LE32
// then the payload; a stream ends with a header whose three ints are zero.
//
//   lz4block_walk_kernel    THREAD per stream: header walk, run twice (count codec blocks and decoded bytes, then write
//                           one descriptor per codec block).
//   lz4_decode_warp_kernel  WARP per LZ4 codec block of any size lz4-java writes (up to 32 MiB), persistent grid: the
//                           token chain is resolved 32 sequences at a time by pointer doubling over speculative headers
//                           in a 128-byte window, then the batch's literals and matches are copied (lz_batch.cuh).
//                           Nothing goes through HBM between parse and copy.
#include "kernels.h"
#include "lz_batch.cuh"

namespace b2s {

constexpr int kMinMatch = 4, kMFLimit = 12, kLastLiterals = 5;

// ------------------------------------------------------------------------------------------------------------
// LZ4Block framing, read side: header walk (LZ4BlockInputStream.refill [U])
// ------------------------------------------------------------------------------------------------------------
struct Lz4bHeader {
  int method;
  int level;
  int32_t clen, olen;
  uint32_t check;
  bool magic_ok;
};
__device__ __forceinline__ Lz4bHeader lz4b_read_header(const uint8_t* p) {
  Lz4bHeader h;
  h.magic_ok = ld32u_ro(p) == 0x42345A4Cu && ld32u_ro(p + 4) == 0x6B636F6Cu;
  const int token = p[8];
  h.method = token & 0xF0;
  h.level = 10 + (token & 0x0F);
  h.clen = (int32_t)ld32u_ro(p + 9);
  h.olen = (int32_t)ld32u_ro(p + 13);
  h.check = ld32u_ro(p + 17);
  return h;
}
__device__ __forceinline__ bool lz4b_header_valid(const Lz4bHeader& h) {
  if (!h.magic_ok) return false;
  if (h.method != 0x10 && h.method != 0x20) return false;
  if (h.olen > (1 << h.level) || h.olen < 0 || h.clen < 0 || (h.olen == 0 && h.clen != 0) ||
      (h.olen != 0 && h.clen == 0) || (h.method == 0x10 && h.olen != h.clen))
    return false;
  return true;
}

// FILL=false: count blocks/bytes per stream.  FILL=true: write descriptors.
template <bool FILL>
__global__ void lz4block_walk_kernel(const uint8_t* __restrict__ src_base, const uint64_t* __restrict__ src_off,
                                     const uint64_t* __restrict__ src_len, uint32_t n, uint64_t* __restrict__ nblk,
                                     uint64_t* __restrict__ olen_total, const uint64_t* __restrict__ blk_base,
                                     const uint64_t* __restrict__ dst_off, uint64_t dst_cap,
                                     int32_t* __restrict__ status, BlockDesc* __restrict__ desc) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (FILL && status[i] != 0 && status[i] != B2S_E_DST_TOO_SMALL) return;
  if (!FILL && status[i] != 0) {  // failed checksum verification: nothing of this block is decoded
    nblk[i] = 0;
    olen_total[i] = 0;
    return;
  }
  const uint8_t* p = src_base + src_off[i];
  const uint64_t len = src_len[i];
  uint64_t ip = 0, cnt = 0, total = 0;
  bool bad = false;
  bool too_small = false;
  if (FILL) too_small = (dst_off[i] + olen_total[i] > dst_cap);
  while (ip < len) {
    if (len - ip < 21) {
      bad = true;
      break;
    }
    const Lz4bHeader h = lz4b_read_header(p + ip);
    if (!lz4b_header_valid(h)) {
      bad = true;
      break;
    }
    ip += 21;
    if (h.olen == 0 && h.clen == 0) {
      if (h.check != 0) {
        bad = true;
        break;
      }
      continue;  // end mark; stopOnEmptyBlock=false: a concatenated stream may follow
    }
    if ((uint64_t)h.clen > len - ip) {
      bad = true;
      break;
    }
    if (FILL) {
      BlockDesc d;
      d.src = src_off[i] + ip;
      d.dst = dst_off[i] + total;
      d.clen = too_small ? 0u : (uint32_t)h.clen;
      d.olen = too_small ? 0u : (uint32_t)h.olen;
      d.check = h.check;
      d.stream = i | (h.method == 0x10 ? 0x80000000u : 0u);
      desc[blk_base[i] + cnt] = d;
    }
    cnt++;
    total += (uint64_t)h.olen;
    ip += (uint64_t)h.clen;
  }
  if (!FILL) {
    if (bad) {
      status[i] = B2S_E_CORRUPT;
      cnt = 0;
      total = 0;
    }
    nblk[i] = cnt;
    olen_total[i] = total;
  } else if (too_small) {
    status[i] = B2S_E_DST_TOO_SMALL;
  }
}

void launch_lz4block_count(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                           uint64_t* d_nblk, uint64_t* d_olen, int32_t* d_status, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  lz4block_walk_kernel<false><<<(n + 127) / 128, 128, 0, st>>>(src_base, d_src_off, d_src_len, n, d_nblk, d_olen,
                                                              nullptr, nullptr, 0, d_status, nullptr);
  *launches += 1;
}

void launch_lz4block_fill(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                          const uint64_t* d_blk_base, const uint64_t* d_dst_off, uint64_t* d_olen, uint64_t dst_cap,
                          int32_t* d_status, BlockDesc* d_desc, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  lz4block_walk_kernel<true><<<(n + 127) / 128, 128, 0, st>>>(src_base, d_src_off, d_src_len, n, nullptr, d_olen,
                                                             d_blk_base, d_dst_off, dst_cap, d_status, d_desc);
  *launches += 1;
}

// ---- lz4_decode_warp_kernel: WARP per LZ4 codec block, token parse and copies in one pass, no per-sequence records.
//
// Each step loads the 128 compressed bytes from the cursor ip into shared memory (aligned words that hold block bytes
// only).  Lane l owns window positions 4l..4l+3 and computes the header a token at each of them would have — ll with
// at most one extension byte, the offset, ml with at most one extension byte — and next(p), the position of the token
// after it.  A header that needs a byte at or past the window's end (or the block's), or a second extension byte, is
// "unresolved".  Pointer doubling over next (four rounds of shuffles on four byte-packed tables J_k = next^(2^k)) then
// gives lane s the s-th token of the chain from ip in five more shuffles.  The resolved prefix of the chain, up to 32
// tokens, is one batch; an unresolved token after it (a long length, a header across the window end, the final
// literals-only sequence) is decoded by its lane alone from global memory with every check of the serial walk.
//
// Every sequence of the batch is validated against the same bounds as LZ4_decompress_fast's safe reader before any of
// its bytes is written; the batch is cut at the first bad sequence, so a corrupt block writes nothing outside its own
// output range (what lies inside it is unspecified).  Speculative headers at literal bytes are never validated, copied
// or read past the window.
constexpr int kWarpDecWarps = 8, kWin = 128;
constexpr uint32_t kUnresolved = 0xffu;

// one token at ip, serially, with the checks of the JVM reader; false = corrupt.  last = literals-only final sequence.
__device__ __noinline__ bool lz4_token_serial(const uint8_t* __restrict__ in, int clen, int olen, int op, int& ip,
                                             int& ll, int& lip, int& off, int& ml, bool& last) {
  last = false;
  off = 0;
  ml = 0;
  if (ip >= clen) return false;
  const int token = __ldg(in + ip++);
  ll = token >> 4;
  if (ll == 15) {
    int bb;
    do {
      if (ip >= clen) return false;
      bb = __ldg(in + ip++);
      ll += bb;
      if (ll > olen) return false;  // cannot be valid, and a long run of 0xFF bytes must not wrap the counter
    } while (bb == 255);
  }
  if (ll > olen - op || ll > clen - ip) return false;
  lip = ip;
  ip += ll;
  const int opl = op + ll;
  if (olen - opl < kMFLimit) {  // last sequence: literals only; a match may not start < 12 bytes before the end
    last = true;
    return opl == olen && ip == clen;
  }
  if (ip + 2 > clen) return false;
  off = __ldg(in + ip) | (__ldg(in + ip + 1) << 8);
  ip += 2;
  ml = token & 15;
  if (ml == 15) {
    int bb;
    do {
      if (ip >= clen) return false;
      bb = __ldg(in + ip++);
      ml += bb;
      if (ml > olen) return false;
    } while (bb == 255);
  }
  ml += kMinMatch;
  if (ml > olen - opl || off == 0 || off > opl) return false;
  return olen - (opl + ml) >= kLastLiterals;  // the last 5 bytes of a block are literals
}

// J_{k+1} = J_k o J_k on the four positions this lane owns (byte b of a table = entry of position 4*lane + b; entries
// >= kWin — the window's end or kUnresolved — map to themselves)
__device__ __forceinline__ uint32_t lz4_compose(uint32_t jt) {
  uint32_t r = 0;
#pragma unroll
  for (int b = 0; b < 4; b++) {
    const uint32_t q = (jt >> (8 * b)) & 0xffu;
    const uint32_t v = __shfl_sync(0xffffffffu, jt, (int)(q >> 2) & 31);
    const uint32_t e = q < (uint32_t)kWin ? (v >> (8 * (q & 3u))) & 0xffu : q;
    r |= e << (8 * b);
  }
  return r;
}
__device__ __forceinline__ uint32_t lz4_lookup(uint32_t jt, uint32_t p) {
  const uint32_t v = __shfl_sync(0xffffffffu, jt, (int)(p >> 2) & 31);
  return p < (uint32_t)kWin ? (v >> (8 * (p & 3u))) & 0xffu : p;
}

__global__ void __launch_bounds__(kWarpDecWarps * 32, 4)
    lz4_decode_warp_kernel(const BlockDesc* __restrict__ desc, uint32_t nb, const uint8_t* __restrict__ src_base,
                           uint8_t* dst_base, int32_t* __restrict__ status, unsigned int* __restrict__ work_counter) {
  constexpr unsigned FULL = 0xffffffffu;
  __shared__ __align__(16) uint32_t s_win_all[kWarpDecWarps][kWin / 4];
  __shared__ __align__(16) uint2 s_hdr_all[kWarpDecWarps][kWin];
  const int lane = threadIdx.x & 31;
  uint32_t* s_win = s_win_all[threadIdx.x >> 5];
  const uint8_t* s_wb = reinterpret_cast<const uint8_t*>(s_win);
  uint2* s_hdr = s_hdr_all[threadIdx.x >> 5];

  for (;;) {
    uint32_t b = 0;
    if (lane == 0) b = atomicAdd(work_counter, 1u);
    b = __shfl_sync(FULL, b, 0);
    if (b >= nb) break;
    const BlockDesc d = desc[b];
    if (d.olen == 0) continue;  // no-op descriptor
    const uint8_t* __restrict__ in = src_base + d.src;
    uint8_t* out = dst_base + d.dst;
    if (d.stream & 0x80000000u) {  // stored RAW
      group_copy<32>(out, in, d.olen, lane);
      continue;
    }
    const int clen = (int)d.clen, olen = (int)d.olen;
    int ip = 0, base_op = 0;
    bool err = false;
    for (;;) {
      if (ip >= clen) {  // a token must start here
        err = true;
        break;
      }
      // ---- window: bytes ip .. ip + lim - 1 of the block, from the aligned words that contain them
      const int lim = min(clen - ip, kWin);
      const uintptr_t wa = reinterpret_cast<uintptr_t>(in) + (uintptr_t)ip;
      const uint32_t* wp = reinterpret_cast<const uint32_t*>(wa & ~uintptr_t(3));
      const int a = (int)(wa & 3u);
      const unsigned wsh = 8u * (unsigned)a;
      const uint32_t w = 4 * lane < a + lim ? __ldg(wp + lane) : 0u;
      const uint32_t w32 = (lane == 31 && kWin < a + lim) ? __ldg(wp + 32) : 0u;
      uint32_t wn = __shfl_down_sync(FULL, w, 1);
      if (lane == 31) wn = w32;
      const uint32_t mine = __funnelshift_r(w, wn, wsh);  // window bytes 4*lane .. 4*lane + 3
      s_win[lane] = mine;
      __syncwarp();

      // ---- speculative header at each of my four positions
      uint32_t j0 = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int p = 4 * lane + k;
        const int token = (int)((mine >> (8 * k)) & 0xffu);
        int q = p + 1;
        int ll = token >> 4;
        bool ok = p < lim;
        if (ll == 15) {
          const int e = s_wb[q & (kWin - 1)];
          ok = ok && q < lim && e != 255;
          ll += e;
          q++;
        }
        const int lit = q;
        q += ll;
        ok = ok && q + 1 < lim;
        const int off = s_wb[q & (kWin - 1)] | (s_wb[(q + 1) & (kWin - 1)] << 8);
        q += 2;
        int ml = token & 15;
        if (ml == 15) {
          const int e = s_wb[q & (kWin - 1)];
          ok = ok && q < lim && e != 255;
          ml += e;
          q++;
        }
        ml += kMinMatch;
        if (ok) s_hdr[p] = make_uint2((uint32_t)ll | ((uint32_t)ml << 16), (uint32_t)off | ((uint32_t)lit << 16));
        j0 |= (ok ? (uint32_t)q : kUnresolved) << (8 * k);
      }
      __syncwarp();

      // ---- chain from position 0: lane s gets its s-th token (>= kWin: past the chain's resolved part)
      const uint32_t j1 = lz4_compose(j0), j2 = lz4_compose(j1), j3 = lz4_compose(j2), j4 = lz4_compose(j3);
      uint32_t c = 0, t;
      t = lz4_lookup(j0, c); if (lane & 1) c = t;
      t = lz4_lookup(j1, c); if (lane & 2) c = t;
      t = lz4_lookup(j2, c); if (lane & 4) c = t;
      t = lz4_lookup(j3, c); if (lane & 8) c = t;
      t = lz4_lookup(j4, c); if (lane & 16) c = t;
      const uint32_t nxt = lz4_lookup(j0, c);
      const bool resolved = c < (uint32_t)kWin && nxt != kUnresolved;
      const unsigned resmask = __ballot_sync(FULL, resolved);
      const int nres = __popc(resmask);  // the chain is monotone: the resolved lanes are 0 .. nres-1
      const bool serial = nres < 32 && __shfl_sync(FULL, c, nres & 31) < (uint32_t)kWin;  // unresolved token at lane nres

      int ll = 0, ml = 0, off = 0, lip = 0;
      if (resolved) {
        const uint2 h = s_hdr[c];
        ll = (int)(h.x & 0xffffu);
        ml = (int)(h.x >> 16);
        off = (int)(h.y & 0xffffu);
        lip = ip + (int)(h.y >> 16);
      }
      // output positions: inclusive scan of ll + ml over the resolved lanes
      int inc = ll + ml;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        const int u = __shfl_up_sync(FULL, inc, s);
        if (lane >= s) inc += u;
      }
      bool bad = false, last = false;
      int nip = ip + (nres == 32 ? (int)__shfl_sync(FULL, nxt, 31) : kWin);  // cursor after the batch
      if (serial && lane == nres) {
        const int op0 = base_op + inc;  // inc = sum over the resolved lanes here
        int tip = ip + (int)c;
        bad = !lz4_token_serial(in, clen, olen, op0, tip, ll, lip, off, ml, last);
        inc += ll + ml;
        nip = tip;
      }
      const int nbatch = nres + (serial ? 1 : 0);
      if (serial) nip = __shfl_sync(FULL, nip, nres);
      const int op = base_op + inc - (ll + ml);
      if (resolved) {  // the serial lane has checked itself; a resolved token is never the final one
        const int opl = op + ll;
        bad = ll > olen - op || olen - opl < kMFLimit || ml > olen - opl || off == 0 || off > opl ||
              olen - (opl + ml) < kLastLiterals;
      }
      const unsigned badmask = __ballot_sync(FULL, bad) & (nbatch == 32 ? FULL : (1u << nbatch) - 1u);
      const int nok = badmask ? __ffs(badmask) - 1 : nbatch;
      if (lane >= nok) ll = ml = 0;
      const int total = __shfl_sync(FULL, inc, nbatch - 1);  // only used when the batch is copied whole

      lz_copy_literals(in, out, lip, ll, op, lane);
      lz_execute_matches<true>(out, op + ll, ml, off, lane);
      if (badmask) {
        err = true;
        break;
      }
      if (__shfl_sync(FULL, last ? 1 : 0, nbatch - 1)) break;  // the final sequence is done
      base_op += total;
      ip = nip;
      __syncwarp();  // the next window overwrites s_win / s_hdr
    }
    if (err && lane == 0) set_status(status, d.stream & 0x7fffffffu, B2S_E_CORRUPT);
  }
}

void launch_lz4_decode_warp(const BlockDesc* d_desc, uint32_t nb, const uint8_t* src_base, uint8_t* dst_base,
                            int32_t* d_status, unsigned int* d_counter, cudaStream_t st, uint64_t* launches) {
  if (!nb) return;
  cudaMemsetAsync(d_counter, 0, sizeof(unsigned int), st);
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lz4_decode_warp_kernel, kWarpDecWarps * 32, 0);
  if (per_sm < 1) per_sm = 1;
  const uint64_t want = ((uint64_t)nb + kWarpDecWarps - 1) / kWarpDecWarps;
  uint64_t grid = (uint64_t)kSMs * per_sm;  // persistent: one wave, warps pull blocks from the counter
  if (grid > want) grid = want;
  lz4_decode_warp_kernel<<<(unsigned)grid, kWarpDecWarps * 32, 0, st>>>(d_desc, nb, src_base, dst_base, d_status,
                                                                         d_counter);
  *launches += 1;
}

}  // namespace b2s
