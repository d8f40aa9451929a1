// exchange.cu — the copy step of the exchange cache's reads (b2s_exchange_read_*): one launch moves every cached range
// of a call, and for an uncompressed sorted read every fetched block, to its place in the output arena.  A reducer of
// config 3 reads one small range from each of up to thousands of map outputs, so a copy call per range would make
// launch overhead the cost of a cache hit.  The host cuts each range into pieces of at most kExchangePieceBytes, so a
// long range is spread over many warps (and CTAs); a warp copies one piece with destination-aligned 16-byte stores and
// aligned source loads (warp_copy: ld_span16), whatever the byte offsets of the range (104-byte records put them at
// multiples of 8).
#include <algorithm>

#include "kernels.h"

namespace b2s {

namespace {

constexpr int kExThreads = 256;
constexpr int kExWarps = kExThreads / 32;

__global__ void __launch_bounds__(kExThreads) exchange_gather_kernel(const ExchangePiece* __restrict__ pieces,
                                                                     uint32_t n, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint64_t w = (uint64_t)blockIdx.x * kExWarps + (threadIdx.x >> 5); w < n; w += (uint64_t)gridDim.x * kExWarps) {
    const ExchangePiece p = pieces[w];
    warp_copy(dst + p.dst, p.src, p.len, lane);
  }
}

}  // namespace

void exchange_add_pieces(std::vector<ExchangePiece>& pieces, const uint8_t* src, uint64_t dst, uint64_t len) {
  for (uint64_t at = 0; at < len; at += kExchangePieceBytes)
    pieces.push_back(ExchangePiece{src + at, dst + at, std::min<uint64_t>(kExchangePieceBytes, len - at)});
}

void launch_exchange_gather(const ExchangePiece* d_pieces, uint32_t n, uint8_t* d_dst, cudaStream_t st,
                            uint64_t* launches) {
  if (!n) return;
  const uint64_t blocks = ((uint64_t)n + kExWarps - 1) / kExWarps;
  const unsigned grid = (unsigned)std::min<uint64_t>(blocks, (uint64_t)kSMs * 16);
  exchange_gather_kernel<<<grid, kExThreads, 0, st>>>(d_pieces, n, d_dst);
  if (launches) *launches += 1;
}

}  // namespace b2s
