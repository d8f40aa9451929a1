// lz4_decode.cu — K4: LZ4 block decompression as two kernels (LZ4_decompress_fast semantics: driven by originalLen,
// must consume exactly compressedLen; oracle: orc_lz4_decompress_block).
//
// Replaces liblz4's LZ4_decompress_fast as driven by lz4-java's LZ4BlockInputStream [U] under
// serializerManager.wrapStream at storage/S3ShuffleReader.scala:107-109.
//
// Same split as the compressor (lz4_compress.cu): the token chain of a block is inherently serial, the byte copies
// are not.  The first, single-kernel decoder (kept below in lz4.cu as the path for codec blocks > 64 KiB) carried the
// serial chain on 8-lane tiles and spent several warp-instructions per output byte.
//
//   P1 lz4_tokens_kernel  THREAD per codec block: walks tokens / length bytes / offsets, validates every bound the
//                         JVM reader would trip over, and writes one 8-byte record per sequence
//                         (literal count, match length, offset, literal source position).
//   P2 lz4_copy_kernel    warp per codec block, LANE per sequence: output positions by a warp scan, all literals of a
//                         batch of 32 sequences copied at once, then the matches in dependency rounds — a match is
//                         ready when its source lies entirely below the output of the earliest unfinished match;
//                         short matches are copied by their lanes, long ones by the whole warp.
#include "kernels.h"
#include "lz_batch.cuh"
#include "tma_ring.cuh"

namespace b2s {

constexpr int kMinMatch = 4, kMFLimit = 12, kLastLiterals = 5;
int g_lz4d_tokens = 1;  // B2S_LZ4D_TOKENS: 1 = global loads + L1 prefetch, 2 = TMA ring (tma_ring.cuh)

// record: x = literal count | match length << 16 (0 = final sequence) ; y = offset | literal source position << 16
__global__ void __launch_bounds__(64) lz4_tokens_kernel(const BlockDesc* __restrict__ desc, uint32_t b0, uint32_t m,
                                                        const uint8_t* __restrict__ src_base, uint2* __restrict__ rec,
                                                        uint32_t rec_stride, uint32_t* __restrict__ nrec,
                                                        int32_t* __restrict__ status) {
  const uint32_t bl = blockIdx.x * blockDim.x + threadIdx.x;
  if (bl >= m) return;
  const uint32_t b = b0 + bl;
  const BlockDesc d = desc[b];
  if (d.olen == 0 || (d.stream & 0x80000000u)) {  // no-op descriptor or stored RAW (copied by P2)
    nrec[b] = 0;
    return;
  }
  const uint8_t* __restrict__ in = src_base + d.src;
  const int clen = (int)d.clen, olen = (int)d.olen;
  uint2* __restrict__ r = rec + (size_t)bl * rec_stride;
  int ip = 0, op = 0;
  uint32_t ns = 0;
  bool err = false;
  int pf_sector = -1;
  for (int k = 64; k < 512 && k < clen; k += 64) asm volatile("prefetch.global.L1 [%0];" ::"l"(in + k));
  // The token chain is what bounds this kernel (one dependent L1 round trip per field).  Every sequence therefore
  // starts with ONE 8-byte window read at ip — three independent aligned word loads — which holds the token, and for
  // the common short sequence (literals <= 5) also the offset: one round trip instead of two or three.
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(in);
  while (true) {
    if (ip >= clen) {
      err = true;
      break;
    }
    if ((ip >> 5) != pf_sector) {  // entering a new 32-byte sector: pull the sector 16 ahead towards L1/L2 now
      pf_sector = ip >> 5;
      if (ip + 512 < clen) asm volatile("prefetch.global.L1 [%0];" ::"l"(in + ip + 512));
    }
    // window: bytes ip .. ip+7 (only aligned words that contain bytes of the block are read: ip + 7 may pass the end
    // of the block by < 8 bytes, inside the same or the next aligned word of the arena's 256-byte granule)
    const uintptr_t wa = a0 + (uintptr_t)ip;
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(wa & ~uintptr_t(3));
    const unsigned wsh = (wa & 3u) * 8u;
    const int avail = clen - ip;  // >= 1
    const uint32_t x0 = __ldg(wp);
    const uint32_t x1 = ((int)(wa & 3u) + avail > 4) ? __ldg(wp + 1) : 0u;
    const uint32_t x2 = ((int)(wa & 3u) + avail > 8) ? __ldg(wp + 2) : 0u;
    const uint32_t lo = __funnelshift_r(x0, x1, wsh), hi = __funnelshift_r(x1, x2, wsh);
    const int token = (int)(lo & 0xffu);
    ip++;
    int ll = token >> 4;
    if (ll == 15) {
      int bb;
      do {
        if (ip >= clen) {
          err = true;
          break;
        }
        bb = __ldg(in + ip++);
        ll += bb;
      } while (bb == 255);
      if (err) break;
    }
    if (ll > olen - op || ll > clen - ip) {
      err = true;
      break;
    }
    const int lit_ip = ip;
    ip += ll;
    op += ll;
    if (olen - op < kMFLimit) {  // last sequence: literals only; a match may not start < 12 bytes before the end
      if (op != olen || ip != clen) err = true;
      else r[ns++] = make_uint2((uint32_t)ll, (uint32_t)lit_ip << 16);
      break;
    }
    if (ip + 2 > clen) {
      err = true;
      break;
    }
    int off;
    if (ll <= 5 && (token >> 4) != 15) {  // offset bytes sit at window bytes 1+ll, 2+ll (<= 7)
      const unsigned sb = 8u * (unsigned)(1 + ll);
      const uint32_t w = sb < 32 ? __funnelshift_r(lo, hi, sb) : hi >> (sb - 32);
      off = (int)(w & 0xffffu);
    } else {
      off = __ldg(in + ip) | (__ldg(in + ip + 1) << 8);
    }
    ip += 2;
    int ml = token & 15;
    if (ml == 15) {
      int bb;
      do {
        if (ip >= clen) {
          err = true;
          break;
        }
        bb = __ldg(in + ip++);
        ml += bb;
      } while (bb == 255);
      if (err) break;
    }
    ml += kMinMatch;
    if (ml > olen - op || off == 0 || off > op) {
      err = true;
      break;
    }
    r[ns++] = make_uint2((uint32_t)ll | ((uint32_t)ml << 16), (uint32_t)off | ((uint32_t)lit_ip << 16));
    op += ml;
    if (olen - op < kLastLiterals) {  // the last 5 bytes of a block are literals
      err = true;
      break;
    }
  }
  if (err) {
    set_status(status, d.stream & 0x7fffffffu, B2S_E_CORRUPT);
    ns = 0;
  }
  nrec[b] = ns;
}

// The same walk with the compressed stream arriving through the TMA ring of tma_ring.cuh (B2S_LZ4D_TOKENS=2): the
// stream is requested in 64-byte bulk copies four pieces ahead of the cursor and read from shared memory — no global
// load instruction in the token chain, no prefetch bookkeeping.  Literal bytes are skipped over, not read; pieces the
// walk jumps across are still fetched (the ring is strictly sequential) but never waited for longer than they take.
constexpr int kTokThreads = 64;
__global__ void __launch_bounds__(kTokThreads) lz4_tokens_tma_kernel(const BlockDesc* __restrict__ desc, uint32_t b0,
                                                                     uint32_t m, const uint8_t* __restrict__ src_base,
                                                                     uint2* __restrict__ rec, uint32_t rec_stride,
                                                                     uint32_t* __restrict__ nrec,
                                                                     int32_t* __restrict__ status) {
  __shared__ __align__(128) uint8_t s_ring[kTokThreads * kRingBytes];
  __shared__ __align__(8) uint64_t s_bars[kTokThreads * kRingStages];
  const uint32_t bl = blockIdx.x * blockDim.x + threadIdx.x;
  if (bl >= m) return;
  const uint32_t b = b0 + bl;
  const BlockDesc d = desc[b];
  if (d.olen == 0 || (d.stream & 0x80000000u)) {  // no-op descriptor or stored RAW (copied by P2)
    nrec[b] = 0;
    return;
  }
  const uint8_t* __restrict__ in = src_base + d.src;
  const int clen = (int)d.clen, olen = (int)d.olen;
  uint2* __restrict__ r = rec + (size_t)bl * rec_stride;
  TmaRing R;
  R.init(s_ring + threadIdx.x * kRingBytes, s_bars + threadIdx.x * kRingStages, in, clen);
  const int sh0 = (int)(reinterpret_cast<uintptr_t>(in) & 15u);  // stream position of block byte 0
  int ip = 0, op = 0;
  uint32_t ns = 0;
  bool err = false;
  while (true) {
    if (ip >= clen) {
      err = true;
      break;
    }
    // window: bytes ip .. ip+7 from three aligned words of the ring (bytes past the block's end are never used)
    const int u = sh0 + ip;
    R.consume_to(u);
    R.ensure(u + 11);
    const int w = u & ~3;
    const unsigned wsh = (unsigned)(u & 3) * 8u;
    const uint32_t x0 = R.word(w), x1 = R.word(w + 4), x2 = R.word(w + 8);
    const uint32_t lo = __funnelshift_r(x0, x1, wsh), hi = __funnelshift_r(x1, x2, wsh);
    const int token = (int)(lo & 0xffu);
    ip++;
    int ll = token >> 4;
    if (ll == 15) {
      int bb;
      do {
        if (ip >= clen) {
          err = true;
          break;
        }
        R.ensure(sh0 + ip);
        bb = (int)R.byte(sh0 + ip);
        ip++;
        ll += bb;
      } while (bb == 255);
      if (err) break;
    }
    if (ll > olen - op || ll > clen - ip) {
      err = true;
      break;
    }
    const int lit_ip = ip;
    ip += ll;
    op += ll;
    if (olen - op < kMFLimit) {  // last sequence: literals only; a match may not start < 12 bytes before the end
      if (op != olen || ip != clen) err = true;
      else r[ns++] = make_uint2((uint32_t)ll, (uint32_t)lit_ip << 16);
      break;
    }
    if (ip + 2 > clen) {
      err = true;
      break;
    }
    int off;
    if (ll <= 5 && (token >> 4) != 15) {  // offset bytes sit at window bytes 1+ll, 2+ll (<= 7)
      const unsigned sb = 8u * (unsigned)(1 + ll);
      const uint32_t wv = sb < 32 ? __funnelshift_r(lo, hi, sb) : hi >> (sb - 32);
      off = (int)(wv & 0xffffu);
    } else {
      R.consume_to(sh0 + ip);
      R.ensure(sh0 + ip + 1);
      off = (int)(R.byte(sh0 + ip) | (R.byte(sh0 + ip + 1) << 8));
    }
    ip += 2;
    int ml = token & 15;
    if (ml == 15) {
      int bb;
      do {
        if (ip >= clen) {
          err = true;
          break;
        }
        R.ensure(sh0 + ip);
        bb = (int)R.byte(sh0 + ip);
        ip++;
        ml += bb;
      } while (bb == 255);
      if (err) break;
    }
    ml += kMinMatch;
    if (ml > olen - op || off == 0 || off > op) {
      err = true;
      break;
    }
    r[ns++] = make_uint2((uint32_t)ll | ((uint32_t)ml << 16), (uint32_t)off | ((uint32_t)lit_ip << 16));
    op += ml;
    if (olen - op < kLastLiterals) {  // the last 5 bytes of a block are literals
      err = true;
      break;
    }
  }
  R.drain();
  if (err) {
    set_status(status, d.stream & 0x7fffffffu, B2S_E_CORRUPT);
    ns = 0;
  }
  nrec[b] = ns;
}

constexpr int kCopyThreads = 256;
__global__ void __launch_bounds__(kCopyThreads) lz4_copy_kernel(const BlockDesc* __restrict__ desc, uint32_t b0,
                                                                uint32_t m, const uint8_t* __restrict__ src_base,
                                                                uint8_t* dst_base, const uint2* __restrict__ rec,
                                                                uint32_t rec_stride,
                                                                const uint32_t* __restrict__ nrec) {
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const uint32_t bl = blockIdx.x * (kCopyThreads / 32) + (threadIdx.x >> 5);
  if (bl >= m) return;
  const uint32_t b = b0 + bl;
  const BlockDesc d = desc[b];
  if (d.olen == 0) return;
  const uint8_t* __restrict__ in = src_base + d.src;
  uint8_t* out = dst_base + d.dst;
  if (d.stream & 0x80000000u) {
    group_copy<32>(out, in, d.olen, lane);
    return;
  }
  const uint32_t n = nrec[b];
  const uint2* __restrict__ r = rec + (size_t)bl * rec_stride;
  int base_op = 0;
  for (uint32_t i0 = 0; i0 < n; i0 += 32) {
    const uint32_t i = i0 + lane;
    uint2 q = make_uint2(0, 0);
    if (i < n) q = r[i];
    const int lit = (int)(q.x & 0xffffu), ml = (int)(q.x >> 16);
    const int off = (int)(q.y & 0xffffu), lip = (int)(q.y >> 16);
    // output position of every sequence of the batch: exclusive scan of lit + ml
    int inc = lit + ml;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int t = __shfl_up_sync(FULL, inc, s);
      if (lane >= s) inc += t;
    }
    const int op = base_op + inc - (lit + ml);
    base_op += __shfl_sync(FULL, inc, 31);

    // ---- literals: independent of everything, all lanes at once; long runs go through the whole warp
    if (lit > 0 && lit <= 16) {  // aligned 8-byte words of the compressed block (read-only: __ldg)
      uint64_t lo, hi;
      ld_span16<true>(in + lip, lit, lo, hi);
      st_span16(out + op, lit, lo, hi);
    }
    unsigned biglit = __ballot_sync(FULL, lit > 16);
    while (biglit) {
      const int l = __ffs(biglit) - 1;
      biglit &= biglit - 1;
      const int n_l = __shfl_sync(FULL, lit, l), op_l = __shfl_sync(FULL, op, l), ip_l = __shfl_sync(FULL, lip, l);
      if (n_l >= 96) group_copy<32>(out + op_l, in + ip_l, (uint32_t)n_l, lane);
      else
        for (int j = lane; j < n_l; j += 32) out[op_l + j] = __ldg(in + ip_l + j);
    }
    __syncwarp();

    // ---- matches, in dependency rounds (lz_batch.cuh)
    lz_execute_matches<true>(out, op + lit, ml, off, lane);
  }
}

// records per codec block: an LZ4 sequence takes >= 3 compressed bytes and (all but the last) >= 4 output bytes; a
// Snappy element takes >= 2 compressed bytes and may produce a single byte
uint32_t lz4_decode_rec_stride(uint32_t codec, uint32_t max_olen, uint32_t max_clen) {
  if (codec == B2S_CODEC_SNAPPY_XERIAL) return max_clen / 2 + 2;
  const uint32_t a = max_olen / 4 + 2, b = max_clen / 3 + 2;
  return a < b ? a : b;
}
size_t lz4_decode_ws_bytes(uint32_t chunk_blocks, uint32_t rec_stride) {
  return (size_t)chunk_blocks * rec_stride * 8 + 256;
}

// tokens and copy are launched separately so the runtime can put the (latency-bound) token walk of chunk k+1 on a side
// stream beside the (issue-bound) copies of chunk k
void launch_lz4_tokens(uint32_t codec, const BlockDesc* d_desc, uint32_t b0, uint32_t m, uint32_t rec_stride,
                       const uint8_t* src_base, uint8_t* d_ws, uint32_t* d_nrec, int32_t* d_status, cudaStream_t st,
                       uint64_t* launches) {
  if (!m) return;
  uint2* rec = reinterpret_cast<uint2*>(d_ws);
  if (codec == B2S_CODEC_SNAPPY_XERIAL) {
    launch_snappy_tokens(d_desc, b0, m, src_base, rec, rec_stride, d_nrec, d_status, st, launches);
  } else if (g_lz4d_tokens == 2) {
    lz4_tokens_tma_kernel<<<(m + kTokThreads - 1) / kTokThreads, kTokThreads, 0, st>>>(d_desc, b0, m, src_base, rec,
                                                                                     rec_stride, d_nrec, d_status);
    *launches += 1;
  } else {
    lz4_tokens_kernel<<<(m + 63) / 64, 64, 0, st>>>(d_desc, b0, m, src_base, rec, rec_stride, d_nrec, d_status);
    *launches += 1;
  }
}
void launch_lz4_copy(const BlockDesc* d_desc, uint32_t b0, uint32_t m, uint32_t rec_stride, const uint8_t* src_base,
                     uint8_t* dst_base, const uint8_t* d_ws, const uint32_t* d_nrec, cudaStream_t st,
                     uint64_t* launches) {
  if (!m) return;
  lz4_copy_kernel<<<(m + kCopyThreads / 32 - 1) / (kCopyThreads / 32), kCopyThreads, 0, st>>>(
      d_desc, b0, m, src_base, dst_base, reinterpret_cast<const uint2*>(d_ws), rec_stride, d_nrec);
  *launches += 1;
}

}  // namespace b2s
