// lz4_compress.cu — K3: LZ4 block compression as three kernels (specification: orc_lz4_compress_block_win in oracle/).
//
// Replaces liblz4's LZ4_compress_default as driven by lz4-java's LZ4BlockOutputStream [U] under
// SerializerManager.wrapStream on the streams of shuffle/S3ShuffleMapOutputWriter.scala:140-146.
//
// Why three kernels: an LZ77 coder has one inherently serial piece — the greedy parse — and two pieces that are not.
// The first, single-kernel version spent many warp-instructions per input byte because the serial parse ran on a
// whole warp (4 of 32 lanes useful), while HBM sat almost idle.  So the
// serial piece is isolated and given one THREAD per codec block, and the abundant HBM bandwidth carries small
// intermediates between the phases:
//
//   A  lz4_match_kernel   warp per block, all lanes busy, no parse dependency: for every position p of a FIXED window
//                         of 32 positions look the 4 bytes up in a per-warp u16 hash table in shared memory (state
//                         before the window; byte runs use the offset-1 candidate), verify the candidate, measure
//                         the match locally up to 8 bytes  ->  off[p] (u16, 0 = none), ml8[p] (u8);
//                         then insert the 32 positions (highest position wins a slot, deterministic).
//   B  lz4_parse_kernel   THREAD per block: greedy walk over ml8[] (8 positions per 64-bit load), long matches
//                         extended on the source; emits one 8-byte record per sequence with its output offset
//                         (running sum — no scan needed later), decides RAW (compressedLength >= originalLength).
//   C  lz4_emit_kernel    warp per block, LANE per sequence (dense): token, literals, offset, length bytes written
//                         straight to the block's final position in the packed destination (after an exclusive scan
//                         of the block sizes), together with the 21-byte LZ4Block header.  No scratch copy.
//
// Intermediates per input byte: off 2 B + ml8 1 B + records <= 2 B; the runtime processes at most kChunk blocks per
// pass so the workspace stays bounded.  Algorithmic bytes stay (1 + r) per input byte; the extra traffic is the off/ml
// intermediate.
#include "kernels.h"

namespace b2s {

constexpr int kMinMatch = 4, kMFLimit = 12, kLastLiterals = 5;
constexpr int kMatchWarps = 9;  // 9 warps x 8 KiB tables = 72 KiB per CTA, 3 CTAs per SM = 27 warps

__device__ __forceinline__ uint32_t find_stream_of_block(const uint32_t* __restrict__ blk_base, uint32_t n_streams,
                                                         uint32_t b) {
  uint32_t lo = 0, hi = n_streams;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (blk_base[mid] <= b) lo = mid; else hi = mid;
  }
  return lo;
}

struct BlockSpan {
  const uint8_t* s;
  int n;
  uint32_t stream;
};
__device__ __forceinline__ BlockSpan block_span(const uint8_t* __restrict__ src_base, const uint64_t* __restrict__ src_off,
                                                const uint64_t* __restrict__ src_len,
                                                const uint32_t* __restrict__ blk_base, uint32_t n_streams, uint32_t b,
                                                uint32_t block_size) {
  BlockSpan r;
  r.stream = find_stream_of_block(blk_base, n_streams, b);
  const uint64_t boff = (uint64_t)(b - blk_base[r.stream]) * block_size;
  const uint64_t rem = src_len[r.stream] - boff;
  r.n = (int)(rem < block_size ? rem : block_size);
  r.s = src_base + src_off[r.stream] + boff;
  return r;
}

// ------------------------------------------------------------------------------------------------------------
// A: match finding
// ------------------------------------------------------------------------------------------------------------
// Candidate words of one window, requested in iteration k and consumed in iteration k+1 so that their latency is
// covered by a whole iteration of table work (the hash-table chain window -> insert -> next lookup never waits on
// a global load).
struct PendingWindow {
  uint32_t c0, c1, c2, v, v2;
  int p, cand, pos;
  unsigned csh;
  bool live;  // lane holds a position <= mflimit whose candidate is older than the position
};

template <int HLOG>
__global__ void __launch_bounds__(kMatchWarps * 32, 3) lz4_match_kernel(
    const uint8_t* __restrict__ src_base, const uint64_t* __restrict__ src_off, const uint64_t* __restrict__ src_len,
    const uint32_t* __restrict__ blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
    uint32_t stride, uint32_t near_limit, uint16_t* __restrict__ offarr, uint16_t* __restrict__ mlarr,
    unsigned int* __restrict__ work_counter) {
  extern __shared__ __align__(16) uint16_t smem_tables[];
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  uint16_t* table = smem_tables + (size_t)(threadIdx.x >> 5) * (1 << HLOG);
  // Lane l owns window position r = 31 - l: same-address shared stores resolve in favour of the lowest lane on this
  // part, so a contested hash slot receives the highest position on the first store and the read-back that
  // guarantees determinism almost never iterates.
  const int r_me = 31 - lane;

  for (;;) {
    uint32_t bl = 0;
    if (lane == 0) bl = atomicAdd(work_counter, 1u);
    bl = __shfl_sync(FULL, bl, 0);
    if (bl >= m) break;
    const BlockSpan B = block_span(src_base, src_off, src_len, blk_base, n_streams, b0 + bl, block_size);
    const uint8_t* __restrict__ s = B.s;
    const int n = B.n;
    uint16_t* oq = offarr + (size_t)bl * stride + r_me;
    uint16_t* mq = mlarr + (size_t)bl * stride + r_me;
    {
      uint4* t4 = reinterpret_cast<uint4*>(table);
      for (int j = lane; j < (1 << HLOG) / 8; j += 32) t4[j] = make_uint4(0, 0, 0, 0);
    }
    __syncwarp();
    if (n < kMFLimit + 1) continue;
    const int mflimit = n - kMFLimit;
    const int matchlimit = n - kLastLiterals;

    // carry of the previous window's last position (window position 31 = lane 0): its offset and full length
    uint32_t carry_off = 0;
    int carry_L = 0;

    // Finishes a window whose candidate words have arrived: verify, local match length (<= 8), FULL match length,
    // stores.  Full lengths come without touching the source almost always: if positions p and p+1 both matched with
    // the same offset, then L[p] = L[p+1] + 1 (same alignment of the comparison).  So inside a window every segment
    // of equal offsets takes its lengths from the segment's last position q: L[p] = L[q] + (q - p), and L[q] is the
    // local length unless q is itself "long" (8 local bytes equal, room to grow) — only those segment ends are
    // measured on the source, cooperatively, 32 bytes per ballot round.  A run that fills the whole window and
    // continues the previous window's run takes the length of its last position from the carry instead.
    auto finish = [&](const PendingWindow& W) {
      const bool ok = W.live && __funnelshift_r(W.c0, W.c1, W.csh) == W.v;
      const uint32_t x = __funnelshift_r(W.c1, W.c2, W.csh) ^ W.v2;
      int ml = x ? 4 + ((__ffs(x) - 1) >> 3) : 8;
      const int lim = matchlimit - W.p;
      ml = ml < lim ? ml : lim;
      const bool lng = ok && x == 0 && lim > 8;
      const uint32_t off = ok ? (uint32_t)(W.p - W.cand) : 0u;
      int L = ok ? ml : 0;
      const unsigned lngmask = __brev(__ballot_sync(FULL, lng));  // bit r <-> window position r
      if (lngmask) {
        const uint32_t next_off = __shfl_up_sync(FULL, off, 1);   // position r+1 lives in lane-1
        const bool brk = lane == 0 || off == 0 || off != next_off;
        const unsigned brkmask = __brev(__ballot_sync(FULL, brk));  // segment ends; bit 31 always set
        unsigned extmask = brkmask & lngmask;
        const uint32_t off0 = __shfl_sync(FULL, off, 31);  // position 0
        if ((extmask >> 31) && (brkmask & 0x7fffffffu) == 0 && off0 == carry_off) {
          extmask &= 0x7fffffffu;  // one run through the whole window, continuing the carried one
          if (lane == 0) L = carry_L - 32;
        }
        while (extmask) {
          const int q = __ffs(extmask) - 1;
          extmask &= extmask - 1;
          const int oq_ = (int)__shfl_sync(FULL, off, 31 - q);
          const int mpos = W.pos + q;
          const int maxl = matchlimit - mpos;
          const uint8_t* a = s + mpos + lane;
          const uint8_t* c = a - oq_;
          int Lq = maxl;
          for (int base = 8;; base += 32) {
            const int k = base + lane;
            const bool stop = k >= maxl || __ldg(a + base) != __ldg(c + base);
            const unsigned bm = __ballot_sync(FULL, stop);
            if (bm) {
              const int e = base + __ffs(bm) - 1;
              Lq = e < maxl ? e : maxl;
              break;
            }
          }
          if (r_me == q) L = Lq;
        }
        // lengths inside segments from their ends
        const int d = __ffs(brkmask >> r_me) - 1;  // distance to my segment's last position
        const int Lend = __shfl_sync(FULL, L, lane - d);
        if (off) L = Lend + d;
      }
      carry_off = __shfl_sync(FULL, off, 0);
      carry_L = __shfl_sync(FULL, L, 0);
      __stcs(oq, (uint16_t)off);  // position < stride always (stride = block_size rounded up to 32)
      // Snappy (near_limit = 2048, blocks <= 32 KiB so L < 2^15): bit 15 tells the parse kernel that the offset fits
      // the 2-byte copy element, sparing it a dependent load of off[]
      __stcs(mq, (uint16_t)(L | ((off != 0u && off < near_limit) ? 0x8000 : 0)));
      oq += 32;
      mq += 32;
    };

    // per-lane word pointer for the prefetched source words of full windows; (s + pos + r) & 3 is window-invariant
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(s + (r_me <= mflimit ? r_me : mflimit));
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(a0 & ~uintptr_t(3));
    const unsigned sh = (reinterpret_cast<uintptr_t>(s + r_me) & 3u) * 8u;
    uint32_t w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2);
    uint32_t carry_v = 0;
    // one window: hash + lookup, request the candidate words into N, finish the previous window F, insert
    auto step = [&](int pos, PendingWindow& N, const PendingWindow& F, bool have_prev) {
      const bool full = pos + 31 <= mflimit;  // uniform
      const int p = pos + r_me;
      const bool valid = p <= mflimit;
      const int pc = valid ? p : mflimit;
      uint32_t v, v2;
      if (full) {
        v = __funnelshift_r(w0, w1, sh);
        v2 = __funnelshift_r(w1, w2, sh);
        if (pos + 63 <= mflimit) {  // the next window is full as well: request its words now
          wp += 8;
          w0 = __ldg(wp);
          w1 = __ldg(wp + 1);
          w2 = __ldg(wp + 2);
        }
      } else {  // last, partial window: clamped positions, plain loads
        v = ld32u_ro(s + pc);
        v2 = ld32u_ro(s + pc + 4);
      }
      // byte run: the 4 bytes at p-1 equal those at p, i.e. v(p-1) == v(p) — the neighbour lane's value
      const uint32_t vprev = __shfl_down_sync(FULL, v, 1);
      bool rle = vprev == v;
      if (lane == 31) rle = pos > 0 && carry_v == v;
      carry_v = __shfl_sync(FULL, v, 0);
      const uint32_t h = (v * 2654435761u) >> (32 - HLOG);
      int cand = table[h];
      if (rle) cand = pc - 1;
      const bool older = cand < pc;
      if (!older) cand = 0;  // keep the loads in bounds; the result is discarded
      {
        const uintptr_t ca = reinterpret_cast<uintptr_t>(s + cand);
        const uint32_t* cw = reinterpret_cast<const uint32_t*>(ca & ~uintptr_t(3));
        N.csh = (ca & 3u) * 8u;
        N.c0 = __ldg(cw);
        N.c1 = __ldg(cw + 1);
        N.c2 = __ldg(cw + 2);  // cand + 11 < p + 11 <= n - 1
      }
      N.v = v;
      N.v2 = v2;
      N.p = pc;
      N.cand = cand;
      N.pos = pos;
      N.live = valid && older;

      if (have_prev) finish(F);  // window k-1: its candidate words were requested one iteration ago

      // insert window k; a read-back settles slots hit twice so that the highest position wins
      __syncwarp();
      if (valid) table[h] = (uint16_t)p;
      __syncwarp();
      for (;;) {
        const bool lost = valid && table[h] < (uint16_t)p;
        if (!__ballot_sync(FULL, lost)) break;
        if (lost) table[h] = (uint16_t)p;
        __syncwarp();
      }
    };

    // two windows per trip, the pending-window registers ping-pong (no copies)
    PendingWindow PA, PB;
    PA.live = PB.live = false;
    PA.c0 = PA.c1 = PA.c2 = PA.v = PA.v2 = PA.csh = 0;
    PA.p = PA.cand = PA.pos = 0;
    PB = PA;
    bool last_is_a = true;
    for (int pos = 0; pos <= mflimit; pos += 64) {
      step(pos, PA, PB, pos > 0);
      last_is_a = true;
      if (pos + 32 > mflimit) break;
      step(pos + 32, PB, PA, true);
      last_is_a = false;
    }
    if (last_is_a) finish(PA); else finish(PB);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------------------
// B: greedy parse, one thread per codec block
// ------------------------------------------------------------------------------------------------------------
// record: x = literal start | literal count << 16 ; y = match length (0 = final literal run) | output offset << 16
//
// The walk is a fixed-trip loop over groups of 4 positions (one 64-bit load of ml[], next group prefetched).  A match
// is at least 4 long, so at most one sequence starts per group: every iteration is the same straight-line code for
// all 32 lanes (= 32 blocks), no source access, no data-dependent trip counts.
// CODEC: 0 = LZ4; 1 = Snappy: same walk, Snappy element sizes (no RAW fallback, varint preamble, copies split at 64
// bytes); 2 = Zstandard: same walk, the record carries the running literal count instead of an output offset (sizes
// are only known after the entropy stage, zstd_enc.cu) and the block's trailing literals become a final ml == 0 record.
template <int CODEC>
__global__ void __launch_bounds__(64) lz4_parse_kernel(
    const uint64_t* __restrict__ src_len, const uint32_t* __restrict__ blk_base, uint32_t n_streams, uint32_t b0,
    uint32_t m, uint32_t block_size, uint32_t stride, uint32_t max_seq, const uint16_t* __restrict__ mlarr,
    uint2* __restrict__ seqarr, uint32_t* __restrict__ nseq, uint32_t* __restrict__ csize,
    uint64_t* __restrict__ sizes) {
  constexpr bool SNAPPY = CODEC == 1, ZSTD = CODEC == 2;
  const uint32_t bl = blockIdx.x * blockDim.x + threadIdx.x;
  if (bl >= m) return;
  const uint32_t b = b0 + bl;
  const uint32_t si = find_stream_of_block(blk_base, n_streams, b);
  const uint64_t rem = src_len[si] - (uint64_t)(b - blk_base[si]) * block_size;
  const int n = (int)(rem < block_size ? rem : block_size);
  // LZ4BlockOutputStream stores RAW when compressedLength >= originalLength; SnappyOutputStream never does
  const int cap = (SNAPPY || ZSTD) ? 0x7fffffff : n - 1;
  const unsigned long long* __restrict__ mlw =
      reinterpret_cast<const unsigned long long*>(mlarr + (size_t)bl * stride);
  uint2* __restrict__ seq = seqarr + (size_t)bl * max_seq;
  int p = 0, anchor = 0, op = SNAPPY ? (n < 128 ? 1 : n < 16384 ? 2 : 3) : 0;  // Snappy: varint(n) comes first
  uint32_t ns = 0;
  bool fail = false;
  const int mflimit = n - kMFLimit;
  if (n >= kMFLimit + 1) {  // shorter blocks hold no match; the match kernel skipped them (nothing was written to ml[])
    // 8 positions (one 16-byte load) per group; a match is >= 4 long, so at most two sequences start in a group: the
    // body is two copies of the same straight-line "take" code, 32-bit arithmetic only.  Each lane streams through its
    // own block, so every load is a trip to L2/DRAM (no L1 to speak of while the match kernel of the next chunk holds
    // the SM's shared memory): a ring of four groups is kept in flight in registers, i.e. every load is issued four
    // trips (~800 cycles of work) before its use.
    const uint4* __restrict__ mlv = reinterpret_cast<const uint4*>(mlw);
    const int groups = (mflimit >> 3) + 1;
    auto ld = [&](int g) { return __ldcs(mlv + (g < groups ? g : groups - 1)); };
    auto body = [&](const uint4 cur, int g) {
      const int base = 8 * g;
      if (fail || p >= base + 8) return;  // a match taken earlier covers the whole group
      const unsigned nz = (cur.x & 0xffffu ? 1u : 0u) | (cur.x >> 16 ? 2u : 0u) | (cur.y & 0xffffu ? 4u : 0u) |
                          (cur.y >> 16 ? 8u : 0u) | (cur.z & 0xffffu ? 16u : 0u) | (cur.z >> 16 ? 32u : 0u) |
                          (cur.w & 0xffffu ? 64u : 0u) | (cur.w >> 16 ? 128u : 0u);
#pragma unroll
      for (int t = 0; t < 2; t++) {
        const int rel = p - base;  // >= 0
        const unsigned m = rel < 8 ? (nz & (0xffu << rel)) : 0u;
        if (m) {
          const int idx = __ffs(m) - 1;
          const uint32_t word = idx < 4 ? (idx < 2 ? cur.x : cur.y) : (idx < 6 ? cur.z : cur.w);
          const int mlw16 = (int)((idx & 1) ? word >> 16 : word & 0xffffu);
          const int ml = SNAPPY ? (mlw16 & 0x7fff) : mlw16;
          p = base + idx;
          const int lit = p - anchor;
          int size;
          if (ZSTD) {
            size = lit;  // "op" counts literal bytes: where this sequence's literals go in the literals section
          } else if (SNAPPY) {
            size = lit ? lit + (lit - 1 < 60 ? 1 : lit - 1 < 256 ? 2 : 3) : 0;
            int len = ml;
            if (len >= 68) {
              const int k = (len - 68) / 64 + 1;
              size += 3 * k;
              len -= 64 * k;
            }
            if (len > 64) {
              size += 3;
              len -= 60;
            }
            size += (len < 12 && (mlw16 & 0x8000)) ? 2 : 3;
          } else {
            const int mlc = ml - kMinMatch;
            size = 3 + lit;
            if (lit >= 15) size += (lit - 15) / 255 + 1;
            if (mlc >= 15) size += (mlc - 15) / 255 + 1;
          }
          if (op + size > cap) {
            fail = true;
          } else {
            seq[ns++] = make_uint2((uint32_t)anchor | ((uint32_t)lit << 16), (uint32_t)ml | ((uint32_t)op << 16));
            op += size;
            p += ml;
            anchor = p;
          }
        } else if (rel < 8) {
          p = base + 8;
        }
      }
    };
    uint4 r0 = ld(0), r1 = ld(1), r2 = ld(2), r3 = ld(3);
    for (int g = 0; g < groups && !fail; g += 4) {
      {
        const uint4 c = r0;
        r0 = ld(g + 4);
        body(c, g);
      }
      if (g + 1 < groups) {
        const uint4 c = r1;
        r1 = ld(g + 5);
        body(c, g + 1);
      }
      if (g + 2 < groups) {
        const uint4 c = r2;
        r2 = ld(g + 6);
        body(c, g + 2);
      }
      if (g + 3 < groups) {
        const uint4 c = r3;
        r3 = ld(g + 7);
        body(c, g + 3);
      }
    }
  }
  if (ZSTD) {  // trailing literals as a final ml == 0 record; sizes are decided by the entropy stage
    seq[ns++] = make_uint2((uint32_t)anchor | ((uint32_t)(n - anchor) << 16), (uint32_t)op << 16);
    nseq[b] = ns;
    return;
  }
  if (SNAPPY) {
    const int lit = n - anchor;
    if (lit) {
      seq[ns++] = make_uint2((uint32_t)anchor | ((uint32_t)lit << 16), (uint32_t)op << 16);
      op += lit + (lit - 1 < 60 ? 1 : lit - 1 < 256 ? 2 : 3);
    }
    nseq[b] = ns;
    csize[b] = (uint32_t)op;
    sizes[b] = 4u + (uint64_t)op;  // BE32 chunk length + raw snappy block
    return;
  }
  if (!fail) {
    const int lit = n - anchor;
    const int need = 1 + lit + (lit >= 15 ? (lit - 15) / 255 + 1 : 0);
    if (op + need > cap) {
      fail = true;
    } else {
      seq[ns++] = make_uint2((uint32_t)anchor | ((uint32_t)lit << 16), (uint32_t)op << 16);
      op += need;
    }
  }
  nseq[b] = ns;
  csize[b] = fail ? ((uint32_t)n | 0x80000000u) : (uint32_t)op;
  sizes[b] = 21u + (uint64_t)(fail ? n : op);
}

// ------------------------------------------------------------------------------------------------------------
// C: emission, one lane per sequence, into the block's final packed position; also writes the LZ4Block header
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int lz4b_level(uint32_t block_size) {
  int bits = 32 - __clz(block_size - 1);
  int lvl = bits - 10;
  return lvl < 0 ? 0 : lvl;
}
__device__ __forceinline__ uint8_t lz4b_header_byte(int j, int token, uint32_t clen, uint32_t olen, uint32_t check) {
  const uint64_t magic = 0x6B636F6C42345A4Cull;  // "LZ4Block"
  if (j < 8) return (uint8_t)(magic >> (8 * j));
  if (j == 8) return (uint8_t)token;
  if (j < 13) return (uint8_t)(clen >> (8 * (j - 9)));
  if (j < 17) return (uint8_t)(olen >> (8 * (j - 13)));
  return (uint8_t)(check >> (8 * (j - 17)));
}
__device__ __forceinline__ void warp_store_len_ext(uint8_t* o, int nb, int r, int lane) {
  for (int j = lane; j < nb; j += 32) o[j] = (j == nb - 1) ? (uint8_t)(r - 255 * (nb - 1)) : (uint8_t)255;
}
// cooperative emit of one sequence (mlen == 0: final literal run without a match part)
__device__ __forceinline__ void warp_emit_seq(uint8_t* __restrict__ o, const uint8_t* __restrict__ lit_src, int lit,
                                              int off, int mlen, int lane) {
  const int ml = mlen - kMinMatch;
  const int nbL = lit >= 15 ? (lit - 15) / 255 + 1 : 0;
  if (lane == 0) o[0] = (uint8_t)(((lit < 15 ? lit : 15) << 4) | (mlen ? (ml < 15 ? ml : 15) : 0));
  if (nbL) warp_store_len_ext(o + 1, nbL, lit - 15, lane);
  if (lit >= 96) {
    group_copy<32>(o + 1 + nbL, lit_src, (uint32_t)lit, lane);
  } else {
    for (int j = lane; j < lit; j += 32) o[1 + nbL + j] = __ldg(lit_src + j);
  }
  if (mlen) {
    uint8_t* q = o + 1 + nbL + lit;
    if (lane == 0) q[0] = (uint8_t)off;
    if (lane == 1) q[1] = (uint8_t)(off >> 8);
    if (ml >= 15) warp_store_len_ext(q + 2, (ml - 15) / 255 + 1, ml - 15, lane);
  }
}

constexpr int kEmitThreads = 256;
__global__ void __launch_bounds__(kEmitThreads) lz4_emit_kernel(
    const uint8_t* __restrict__ src_base, const uint64_t* __restrict__ src_off, const uint64_t* __restrict__ src_len,
    const uint32_t* __restrict__ blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
    uint32_t stride, uint32_t max_seq, const uint16_t* __restrict__ offarr, const uint2* __restrict__ seqarr,
    const uint32_t* __restrict__ nseq, const uint32_t* __restrict__ csize, const uint32_t* __restrict__ hash,
    const uint64_t* __restrict__ scan, uint8_t* __restrict__ dst_base, uint64_t dst_cap) {
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const uint32_t bl = blockIdx.x * (kEmitThreads / 32) + (threadIdx.x >> 5);
  if (bl >= m) return;
  const uint32_t b = b0 + bl;
  const BlockSpan B = block_span(src_base, src_off, src_len, blk_base, n_streams, b, block_size);
  const uint8_t* __restrict__ s = B.s;
  const uint32_t cs = csize[b];
  const bool raw = cs & 0x80000000u;
  const uint32_t clen = cs & 0x7fffffffu;
  const uint64_t o0 = scan[b] + 21ull * B.stream;
  if (o0 + 21ull + clen > dst_cap) return;  // the stream-meta kernel reports B2S_E_DST_TOO_SMALL for this stream
  uint8_t* __restrict__ o = dst_base + o0;
  const int token = (raw ? 0x10 : 0x20) | lz4b_level(block_size);
  if (lane < 21) o[lane] = lz4b_header_byte(lane, token, clen, (uint32_t)B.n, hash[b] & 0x0FFFFFFFu);
  uint8_t* __restrict__ out = o + 21;
  if (raw) {
    group_copy<32>(out, s, clen, lane);
    return;
  }
  const uint32_t ns = nseq[b];
  const uint2* __restrict__ seq = seqarr + (size_t)bl * max_seq;
  const uint16_t* __restrict__ offp = offarr + (size_t)bl * stride;
  const int omask = stride <= 32768u ? 0x7fff : 0xffff;
  for (uint32_t i0 = 0; i0 < ns; i0 += 32) {
    const uint32_t i = i0 + lane;
    bool slow = false;
    int anchor = 0, lit = 0, ml = 0, op = 0, off = 0;
    if (i < ns) {
      const uint2 r = seq[i];
      anchor = (int)(r.x & 0xffffu);
      lit = (int)(r.x >> 16);
      ml = (int)(r.y & 0xffffu);
      op = (int)(r.y >> 16);
      const int mlc = ml - kMinMatch;
      if (ml) off = offp[anchor + lit] & omask;  // bit 15 of off[] is the parse kernel's "exactly 4" flag (blocks <= 32 KiB)
      if (lit <= 16 && ml && mlc < 15 + 510) {
        uint8_t* q = out + op;
        *q++ = (uint8_t)(((lit < 15 ? lit : 15) << 4) | (mlc < 15 ? mlc : 15));
        if (lit >= 15) *q++ = (uint8_t)(lit - 15);
        // literals (<= 16 bytes): aligned word loads + funnel shifts into four registers, then predicated byte stores
        // — a per-byte load loop would be one L2 round trip per byte whenever L1 is not there to absorb it
        if (lit) {
          const uintptr_t la = reinterpret_cast<uintptr_t>(s + anchor);
          const uint32_t* lw = reinterpret_cast<const uint32_t*>(la & ~uintptr_t(3));
          const unsigned lsh = (la & 3u) * 8u;
          const int need = (int)(la & 3u) + lit;  // bytes from the first aligned word on
          const uint32_t w0 = __ldg(lw), w1 = need > 4 ? __ldg(lw + 1) : 0u, w2 = need > 8 ? __ldg(lw + 2) : 0u,
                         w3 = need > 12 ? __ldg(lw + 3) : 0u, w4 = need > 16 ? __ldg(lw + 4) : 0u;
          const uint32_t r0 = __funnelshift_r(w0, w1, lsh), r1 = __funnelshift_r(w1, w2, lsh),
                         r2 = __funnelshift_r(w2, w3, lsh), r3 = __funnelshift_r(w3, w4, lsh);
#pragma unroll
          for (int j = 0; j < 16; j++) {
            const uint32_t r = j < 4 ? r0 : j < 8 ? r1 : j < 12 ? r2 : r3;
            if (j < lit) q[j] = (uint8_t)(r >> (8 * (j & 3)));
          }
        }
        q += lit;
        q[0] = (uint8_t)off;
        q[1] = (uint8_t)(off >> 8);
        if (mlc >= 15) {
          int rem = mlc - 15;
          q += 2;
          if (rem >= 255) {
            *q++ = 255;
            rem -= 255;
          }
          *q = (uint8_t)rem;
        }
      } else {
        slow = true;
      }
    }
    unsigned slowmask = __ballot_sync(FULL, slow);
    while (slowmask) {
      const int l = __ffs(slowmask) - 1;
      slowmask &= slowmask - 1;
      const int a_r = __shfl_sync(FULL, anchor, l);
      const int lit_r = __shfl_sync(FULL, lit, l);
      const int ml_r = __shfl_sync(FULL, ml, l);
      const int op_r = __shfl_sync(FULL, op, l);
      const int off_r = __shfl_sync(FULL, off, l);
      warp_emit_seq(out + op_r, s + a_r, lit_r, off_r, ml_r, lane);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------------------
int g_lz4_hlog = 12;  // B2S_LZ4_HLOG (api.cu reads it once at init); 12 is the specified default

template <int HLOG>
static void launch_match_t(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                           const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m,
                           uint32_t block_size, uint32_t stride, uint32_t near_limit, uint16_t* d_off,
                           uint16_t* d_ml, unsigned int* d_counter, cudaStream_t st) {
  const size_t smem = (size_t)kMatchWarps * (2u << HLOG);
  cudaFuncSetAttribute(lz4_match_kernel<HLOG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);  // per device and cheap: set on every launch
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lz4_match_kernel<HLOG>, kMatchWarps * 32, smem);
  if (per_sm < 1) per_sm = 1;
  uint64_t want = ((uint64_t)m + kMatchWarps - 1) / kMatchWarps;
  uint64_t grid = (uint64_t)kSMs * per_sm;  // persistent: one wave, warps pull blocks from the counter
  if (grid > want) grid = want;
  lz4_match_kernel<HLOG><<<(unsigned)grid, kMatchWarps * 32, smem, st>>>(
      src_base, d_src_off, d_src_len, d_blk_base, n_streams, b0, m, block_size, stride, near_limit, d_off, d_ml,
      d_counter);
}

// Workspace of one pass over `m` codec blocks:
//   off   u16 per position
//   ml    u16 per position
//   seq   8-byte records, max_seq per block
//   bits  zstd_bits_stride(): sequence-section header + bitstream (Zstandard only)
struct Lz4Ws {
  uint32_t stride, max_seq;
  uint16_t *off, *ml;
  uint2* seq;
  uint8_t* bits;
};
static size_t ws_max_seq(size_t stride) { return stride / 4 + 2; }
size_t lz4_compress_ws_bytes(uint32_t chunk_blocks, uint32_t block_size, uint32_t codec) {
  const size_t stride = (block_size + 31u) & ~31u;
  const size_t per_block = stride * 2 + stride * 2 + ws_max_seq(stride) * 8 +
                           (codec == B2S_CODEC_ZSTD ? zstd_bits_stride(stride) : 0);
  return (size_t)chunk_blocks * per_block + 1024;
}
static Lz4Ws carve_ws(uint8_t* d_ws, uint32_t m, uint32_t block_size) {
  Lz4Ws w;
  w.stride = (block_size + 31u) & ~31u;
  w.max_seq = (uint32_t)ws_max_seq(w.stride);
  size_t at = 0;
  w.off = reinterpret_cast<uint16_t*>(d_ws);
  at += (size_t)m * w.stride * 2;
  w.ml = reinterpret_cast<uint16_t*>(d_ws + at);
  at += (size_t)m * w.stride * 2;
  at = (at + 15) & ~size_t(15);
  w.seq = reinterpret_cast<uint2*>(d_ws + at);
  at += (size_t)m * w.max_seq * 8;
  w.bits = d_ws + at;
  return w;
}

template <int CODEC>
static void launch_parse_t(const uint64_t* d_src_len, const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0,
                           uint32_t m, uint32_t block_size, const Lz4Ws& w, uint32_t* d_nseq, uint32_t* d_csize,
                           uint64_t* d_sizes, cudaStream_t st) {
  lz4_parse_kernel<CODEC><<<(m + 63) / 64, 64, 0, st>>>(d_src_len, d_blk_base, n_streams, b0, m, block_size, w.stride,
                                                        w.max_seq, w.ml, w.seq, d_nseq, d_csize, d_sizes);
}

void launch_lz4_match(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                      const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
                      uint32_t codec, uint8_t* d_ws, unsigned int* d_counter, cudaStream_t st, uint64_t* launches,
                      cudaEvent_t ev0, cudaEvent_t ev1, int hlog) {
  if (!m) return;
  const uint32_t near_limit = codec == B2S_CODEC_SNAPPY_XERIAL ? 2048u : 0u;
  const Lz4Ws w = carve_ws(d_ws, m, block_size);
  cudaMemsetAsync(d_counter, 0, sizeof(unsigned int), st);
  if (ev0) cudaEventRecord(ev0, st);
#define B2S_LZ4M(H)                                                                                        \
  launch_match_t<H>(src_base, d_src_off, d_src_len, d_blk_base, n_streams, b0, m, block_size, w.stride, near_limit, \
                    w.off, w.ml, d_counter, st)
  switch (hlog > 0 ? hlog : g_lz4_hlog) {
    case 10: B2S_LZ4M(10); break;
    case 11: B2S_LZ4M(11); break;
    case 13: B2S_LZ4M(13); break;
    default: B2S_LZ4M(12); break;
  }
#undef B2S_LZ4M
  if (ev1) cudaEventRecord(ev1, st);
  *launches += 1;
}

void launch_lz4_parse_emit(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                           const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m,
                           uint32_t block_size, uint32_t codec, uint8_t* d_ws, uint32_t* d_nseq, uint32_t* d_csize,
                           const uint32_t* d_hash, uint64_t* d_sizes, uint64_t* d_running_total, uint64_t* d_scan_ws,
                           uint8_t* dst_base, uint64_t dst_cap, cudaStream_t st, uint64_t* launches) {
  if (!m) return;
  const Lz4Ws w = carve_ws(d_ws, m, block_size);
  if (codec == B2S_CODEC_ZSTD) {
    launch_parse_t<2>(d_src_len, d_blk_base, n_streams, b0, m, block_size, w, d_nseq, d_csize, d_sizes, st);
    uint8_t* d_bits = w.bits;
    // d_hash is unused by this codec and carries the bitstream sizes from the entropy stage to the emit kernel
    launch_zstd_seqenc(src_base, d_src_off, d_src_len, d_blk_base, n_streams, b0, m, block_size, w.stride, w.max_seq,
                       w.off, w.seq, d_nseq, d_bits, const_cast<uint32_t*>(d_hash), d_csize, d_sizes, st, launches);
    launch_exclusive_scan_u64(d_sizes + b0, m, d_running_total, d_scan_ws, st, launches, d_running_total);
    launch_zstd_emit(src_base, d_src_off, d_src_len, d_blk_base, n_streams, b0, m, block_size, w.stride, w.max_seq,
                     w.seq, d_nseq, d_bits, d_hash, d_csize, d_sizes, dst_base, dst_cap, st, launches);
    *launches += 1;
    return;
  }
  if (codec == B2S_CODEC_SNAPPY_XERIAL) {
    launch_parse_t<1>(d_src_len, d_blk_base, n_streams, b0, m, block_size, w, d_nseq, d_csize, d_sizes, st);
    launch_exclusive_scan_u64(d_sizes + b0, m, d_running_total, d_scan_ws, st, launches, d_running_total);
    launch_snappy_emit(src_base, d_src_off, d_src_len, d_blk_base, n_streams, b0, m, block_size, w.stride, w.max_seq,
                       w.off, w.seq, d_nseq, d_csize, d_sizes, dst_base, dst_cap, st, launches);
    *launches += 1;
    return;
  }
  launch_parse_t<0>(d_src_len, d_blk_base, n_streams, b0, m, block_size, w, d_nseq, d_csize, d_sizes, st);
  // packed offsets of this chunk's blocks, chained onto the running total of the chunks before it
  launch_exclusive_scan_u64(d_sizes + b0, m, d_running_total, d_scan_ws, st, launches, d_running_total);
  lz4_emit_kernel<<<(m + kEmitThreads / 32 - 1) / (kEmitThreads / 32), kEmitThreads, 0, st>>>(
      src_base, d_src_off, d_src_len, d_blk_base, n_streams, b0, m, block_size, w.stride, w.max_seq, w.off, w.seq,
      d_nseq, d_csize, d_hash, d_sizes, dst_base, dst_cap);
  *launches += 2;
}

// per stream: packed offset/length, end mark, capacity check (runs once all chunks have been scanned)
__global__ void lz4block_stream_meta_kernel(const uint32_t* __restrict__ blk_base, uint32_t n_streams,
                                            uint32_t n_blocks, uint32_t block_size, const uint64_t* __restrict__ scan,
                                            const uint64_t* __restrict__ scan_total, uint8_t* __restrict__ dst_base,
                                            uint64_t dst_cap, uint64_t* __restrict__ dst_off,
                                            uint64_t* __restrict__ dst_len, int32_t* __restrict__ status) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_streams) return;
  const uint32_t b0 = blk_base[i], b1 = blk_base[i + 1];
  const uint64_t s0 = b0 < n_blocks ? scan[b0] : *scan_total;
  const uint64_t s1 = b1 < n_blocks ? scan[b1] : *scan_total;
  const uint64_t off = s0 + 21ull * i;
  const uint64_t len = (s1 - s0) + 21ull;
  dst_off[i] = off;
  dst_len[i] = len;
  if (off + len > dst_cap) {
    status[i] = B2S_E_DST_TOO_SMALL;
    return;
  }
  uint8_t* e = dst_base + off + len - 21;
  const int token = 0x10 | lz4b_level(block_size);
#pragma unroll
  for (int j = 0; j < 21; j++) e[j] = lz4b_header_byte(j, token, 0, 0, 0);
}

void launch_lz4block_stream_meta(const uint32_t* d_blk_base, uint32_t n_streams, uint32_t n_blocks, uint32_t block_size,
                                 const uint64_t* d_scan, const uint64_t* d_scan_total, uint8_t* dst_base,
                                 uint64_t dst_cap, uint64_t* d_dst_off, uint64_t* d_dst_len, int32_t* d_status,
                                 cudaStream_t st, uint64_t* launches) {
  if (!n_streams) return;
  lz4block_stream_meta_kernel<<<(n_streams + 255) / 256, 256, 0, st>>>(d_blk_base, n_streams, n_blocks, block_size,
                                                                       d_scan, d_scan_total, dst_base, dst_cap,
                                                                       d_dst_off, d_dst_len, d_status);
  *launches += 1;
}

}  // namespace b2s
