// lz4.cu — K4 (LZ4 block decompress) and the read side of the lz4-java LZ4Block stream framing (K3, the compressor,
// and the write-side framing live in lz4_compress.cu).
//
// Replaces, for spark.io.compression.codec=lz4, what Spark's SerializerManager.wrapStream puts around the streams
// of shuffle/S3ShuffleMapOutputWriter.scala:140-146 (write) and storage/S3ShuffleReader.scala:107-109 (read):
//   net.jpountz.lz4.LZ4BlockOutputStream -> LZ4JNICompressor  -> liblz4 LZ4_compress_default      [U]
//   net.jpountz.lz4.LZ4BlockInputStream  -> LZ4JNIFastDecompressor -> liblz4 LZ4_decompress_fast  [U]
// Wire format (oracle/b2s_oracle.c restates it): per <= blockSize bytes of input a 21-byte header
//   "LZ4Block" | token = method(0x10 RAW, 0x20 LZ4) | level | compressedLen LE32 | originalLen LE32 | XXH32&0x0FFFFFFF LE32
// then the payload; a stream ends with a header whose three ints are zero.
//
// Parallelism: every codec block (<= 64 KiB here) is independent.
//  compress : one warp per block, window-batched greedy parse (see K3 below).  Deterministic; the CPU model
//             orc_lz4_compress_block_win() in oracle/ produces identical bytes.
//  decompress: blocks up to 64 KiB take one warp each (lz4_decode_warp_kernel, lz4_decode.cu); a batch with a larger
//             block takes a tile of 8 lanes per block here: the token chain is serial, the tile parses uniformly and
//             copies literals / (overlapping) matches 8 bytes per step.
// This is latency/issue-bound byte-stream work (no tensor cores, HBM far from saturated by one block per tile), so
// the levers are blocks in flight per SM (small per-tile state: 4-8 KiB hash table, no staged copy of the block)
// and instructions per sequence.
#include "kernels.h"

namespace b2s {

constexpr int kLz4Threads = 128;
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
                                     uint64_t* __restrict__ olen_total, unsigned long long* __restrict__ maxima,
                                     const uint64_t* __restrict__ blk_base,
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
  uint32_t max_olen = 0, max_clen = 0;
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
    if (!FILL) {
      max_olen = max_olen > (uint32_t)h.olen ? max_olen : (uint32_t)h.olen;
      max_clen = max_clen > (uint32_t)h.clen ? max_clen : (uint32_t)h.clen;
    }
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
    if (cnt) {  // largest codec block of the batch (selects the decode path and sizes its records)
      atomicMax(maxima, (unsigned long long)max_olen);
      atomicMax(maxima + 1, (unsigned long long)max_clen);
    }
  } else if (too_small) {
    status[i] = B2S_E_DST_TOO_SMALL;
  }
}

void launch_lz4block_count(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                           uint64_t* d_nblk, uint64_t* d_olen, uint64_t* d_maxima, int32_t* d_status, cudaStream_t st,
                           uint64_t* launches) {
  if (!n) return;
  lz4block_walk_kernel<false><<<(n + 127) / 128, 128, 0, st>>>(src_base, d_src_off, d_src_len, n, d_nblk, d_olen,
                                                              (unsigned long long*)d_maxima, nullptr, nullptr, 0,
                                                              d_status, nullptr);
  *launches += 1;
}

void launch_lz4block_fill(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                          const uint64_t* d_blk_base, const uint64_t* d_dst_off, uint64_t* d_olen, uint64_t dst_cap,
                          int32_t* d_status, BlockDesc* d_desc, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  lz4block_walk_kernel<true><<<(n + 127) / 128, 128, 0, st>>>(src_base, d_src_off, d_src_len, n, nullptr, d_olen,
                                                             nullptr, d_blk_base, d_dst_off, dst_cap, d_status,
                                                             d_desc);
  *launches += 1;
}

// ------------------------------------------------------------------------------------------------------------
// K4: decompress (LZ4_decompress_fast semantics: driven by originalLen, must consume exactly compressedLen)
//
// A warp carries 32/TILE independent blocks ("tiles" of TILE lanes) through ONE warp-uniform instruction stream:
// every iteration decodes one sequence per tile (token, literal run, offset, match), with the copy loops bounded by
// the warp-wide maximum (REDUX.MAX) and predicated per tile.  All synchronisation is full-mask __syncwarp().
// (Per-tile control flow with partial-mask sync looked natural but ptxas guards every non-uniform-mask
// __syncwarp/__ballot with MATCH.ANY — a long-latency, low-throughput instruction — so it is avoided.)
// Sequences in shuffle data are short (terasort: 0.8 literal + 6.7 match bytes), hence small tiles.
// ------------------------------------------------------------------------------------------------------------
template <int TILE>
__global__ void __launch_bounds__(kLz4Threads) lz4_decompress_kernel(const BlockDesc* __restrict__ desc,
                                                                     uint32_t n_blocks,
                                                                     const uint8_t* __restrict__ src_base,
                                                                     uint8_t* __restrict__ dst_base,
                                                                     int32_t* __restrict__ status,
                                                                     unsigned int* __restrict__ work_counter) {
  constexpr unsigned FULL = 0xffffffffu;
  const int tl = threadIdx.x % TILE;  // lane within the tile
  bool active = false, exhausted = false;
  const uint8_t* __restrict__ in = nullptr;
  uint8_t* out = nullptr;
  int ip = 0, op = 0, clen = 0, olen = 0;
  uint32_t stream = 0;

  for (;;) {
    // ---- refill tiles that have no block (rare: once per codec block)
    if (!active && !exhausted) {
      uint32_t b = 0;
      if (tl == 0) b = atomicAdd(work_counter, 1u);
      b = __shfl_sync(tile_mask<TILE>(), b, 0, TILE);
      if (b >= n_blocks) {
        exhausted = true;
      } else {
        const BlockDesc d = desc[b];
        if (d.olen != 0) {
          in = src_base + d.src;
          out = dst_base + d.dst;
          if (d.stream & 0x80000000u) {  // stored RAW
            group_copy<TILE>(out, in, d.olen, tl);
          } else {
            active = true;
            ip = op = 0;
            clen = (int)d.clen;
            olen = (int)d.olen;
            stream = d.stream;
          }
        }
      }
    }
    if (__all_sync(FULL, exhausted && !active)) break;

    // ---- one sequence per active tile, warp-uniform control flow
    bool err = false;
    int token = 0, ll = 0;
    if (active) {
      if (ip >= clen) err = true;
      else {
        token = __ldg(in + ip++);
        ll = token >> 4;
      }
    }
    bool more = active && !err && ll == 15;
    while (__any_sync(FULL, more)) {
      if (more) {
        if (ip >= clen) {
          err = true;
          more = false;
        } else {
          const int bb = __ldg(in + ip++);
          ll += bb;
          more = (bb == 255);
          if (ll > olen) {  // cannot be valid, and an unbounded run of 0xFF bytes must not wrap the counter
            err = true;
            more = false;
          }
        }
      }
    }
    if (active && !err && (ll > olen - op || ll > clen - ip)) err = true;
    {
      const int cl = (active && !err) ? ll : 0;
      const int maxl = __reduce_max_sync(FULL, cl);
      for (int j = tl; j < maxl; j += TILE)
        if (j < cl) out[op + j] = __ldg(in + ip + j);
    }
    if (active && !err) {
      op += ll;
      ip += ll;
    }
    const bool last = active && !err && (olen - op < kMFLimit);  // last match must start >= 12 bytes before the end
    if (last && (op != olen || ip != clen)) err = true;
    const bool cont = active && !err && !last;
    int off = 0, ml = 0;
    if (cont) {
      if (ip + 2 > clen) err = true;
      else {
        off = __ldg(in + ip) | (__ldg(in + ip + 1) << 8);
        ip += 2;
        ml = token & 15;
      }
    }
    more = cont && !err && ml == 15;
    while (__any_sync(FULL, more)) {
      if (more) {
        if (ip >= clen) {
          err = true;
          more = false;
        } else {
          const int bb = __ldg(in + ip++);
          ml += bb;
          more = (bb == 255);
          if (ml > olen) {
            err = true;
            more = false;
          }
        }
      }
    }
    if (cont && !err) {
      ml += kMinMatch;
      if (ml > olen - op || off == 0 || off > op) err = true;
    }
    __syncwarp();  // literals of this sequence are visible to the whole warp
    {
      const int cm = (cont && !err) ? ml : 0;
      const int maxm = __reduce_max_sync(FULL, cm);
      const uint8_t* msrc = out + op - off;
      for (int j = tl; j < maxm; j += TILE) {
        if (j < cm) {
          // overlapping match (off < ml): every byte comes from the already complete window [op-off, op)
          const int k = (j >= off) ? (int)((unsigned)j % (unsigned)off) : j;
          out[op + j] = msrc[k];
        }
      }
    }
    if (cont && !err) {
      op += ml;
      if (olen - op < kLastLiterals) err = true;  // the last 5 bytes of a block are literals
    }
    __syncwarp();
    if (active && (err || last)) {
      if (err && tl == 0) set_status(status, stream & 0x7fffffffu, B2S_E_CORRUPT);
      active = false;
    }
  }
}

template <int TILE>
static void launch_lz4_decompress_t(const BlockDesc* d_desc, uint32_t n_blocks, const uint8_t* src_base,
                                    uint8_t* dst_base, int32_t* d_status, unsigned int* d_counter, cudaStream_t st) {
  constexpr int kTiles = kLz4Threads / TILE;
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lz4_decompress_kernel<TILE>, kLz4Threads, 0);
  if (per_sm < 1) per_sm = 1;
  uint64_t want = ((uint64_t)n_blocks + kTiles - 1) / kTiles;
  uint64_t grid = (uint64_t)kSMs * per_sm;
  if (grid > want) grid = want;
  lz4_decompress_kernel<TILE><<<(unsigned)grid, kLz4Threads, 0, st>>>(d_desc, n_blocks, src_base, dst_base, d_status,
                                                                     d_counter);
}

void launch_lz4_decompress(const BlockDesc* d_desc, uint32_t n_blocks, const uint8_t* src_base, uint8_t* dst_base,
                           int32_t* d_status, unsigned int* d_counter, cudaStream_t st, uint64_t* launches) {
  if (!n_blocks) return;
  cudaMemsetAsync(d_counter, 0, sizeof(unsigned int), st);
  launch_lz4_decompress_t<8>(d_desc, n_blocks, src_base, dst_base, d_status, d_counter, st);
  *launches += 1;
}

}  // namespace b2s
