// sort.cu — stable sort of fixed-size records by an unsigned byte key (the reduce side of an ordered RDD shuffle: what
// Spark's ExternalSorter does with a key ordering, for keys whose ordering is unsigned byte order, e.g. TeraSort's
// 10-byte keys).  Three steps, all on the device:
//   keys   : one thread per record loads its key bytes (any alignment, ld_span16) and stores them as ceil(key_len/4)
//            big-endian u32 words, word-major, zero-padded on the right
//   radix  : LSD radix sort of (key word, record index) pairs with the partition step's pass (launch_radix_pass),
//            8 bits per pass, one pass per real key byte, least significant byte first.  Before the first pass on each
//            more significant word, that word is gathered into the current order (k[j] = word[idx[j]])
//   gather : records copied in sorted order with the partition step's gather (launch_partition_gather); for
//            fixed-size records the offsets are i * record_bytes
#include <algorithm>

#include "kernels.h"

namespace b2s {

namespace {

constexpr int kSortThreads = 256;

inline unsigned grid_for(uint64_t n) {
  const uint64_t want = (n + kSortThreads - 1) / kSortThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

// words[w * n + i] = key bytes [4w, 4w + 4) of record i as a big-endian u32, bytes past key_len zero
__global__ void __launch_bounds__(kSortThreads) sort_keys_kernel(const uint8_t* __restrict__ rec, uint64_t n,
                                                                 uint32_t record_bytes, uint32_t key_off,
                                                                 uint32_t key_len, uint32_t* __restrict__ words) {
  const uint32_t W = (key_len + 3) / 4;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t lo, hi;
    ld_span16<true>(rec + i * record_bytes + key_off, (int)key_len, lo, hi);
    if (key_len < 8) {
      lo &= (1ull << (8 * key_len)) - 1;
      hi = 0;
    } else if (key_len < 16) {
      hi &= (1ull << (8 * (key_len - 8))) - 1;
    }
#pragma unroll
    for (uint32_t w = 0; w < 4; w++)
      if (w < W) {
        const uint32_t x = (uint32_t)((w < 2 ? lo : hi) >> (32 * (w & 1)));
        words[(size_t)w * n + i] = __byte_perm(x, 0, 0x0123);
      }
  }
}

// out[j] = word[idx[j]]: a key word in the current sorted order
__global__ void __launch_bounds__(kSortThreads) sort_word_gather_kernel(const uint32_t* __restrict__ word,
                                                                        const uint32_t* __restrict__ idx, uint64_t n,
                                                                        uint32_t* __restrict__ out) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
    out[j] = word[idx[j]];
}

// the gather's per-record arrays for fixed-size records: source and destination offsets i * record_bytes
__global__ void __launch_bounds__(kSortThreads) sort_fixed_offsets_kernel(uint64_t n, uint32_t record_bytes,
                                                                          uint64_t* __restrict__ src_off,
                                                                          uint64_t* __restrict__ sdst,
                                                                          uint32_t* __restrict__ len) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    src_off[i] = i * record_bytes;
    sdst[i] = i * record_bytes;
    len[i] = record_bytes;
  }
}

inline size_t a256(size_t b) { return (b + 255) / 256 * 256; }

}  // namespace

size_t key_sort_ws_bytes(uint64_t n, uint32_t key_len) {
  const size_t W = (key_len + 3) / 4, hist = radix_hist_elems(n);
  return a256(n * 4 * W) + a256(n * 4) * 5 + a256(n * 8) * 2 + a256(hist * 8) + a256(scan_ws_elems(hist) * 8) + 256;
}

void launch_key_sort(const uint8_t* d_rec, uint64_t n, uint32_t record_bytes, uint32_t key_off, uint32_t key_len,
                     uint8_t* d_ws, uint8_t* d_dst, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  const uint32_t W = (key_len + 3) / 4;
  const size_t hist_elems = radix_hist_elems(n);
  uint8_t* p = d_ws;
  uint32_t* words = (uint32_t*)p;  p += a256(n * 4 * W);  // W arrays of n words: word w at words + w * n
  uint32_t* K[2];
  uint32_t* I[2];
  K[0] = (uint32_t*)p;  p += a256(n * 4);
  K[1] = (uint32_t*)p;  p += a256(n * 4);
  I[0] = (uint32_t*)p;  p += a256(n * 4);
  I[1] = (uint32_t*)p;  p += a256(n * 4);
  uint32_t* len = (uint32_t*)p;     p += a256(n * 4);
  uint64_t* src_off = (uint64_t*)p; p += a256(n * 8);
  uint64_t* sdst = (uint64_t*)p;    p += a256(n * 8);
  uint64_t* hist = (uint64_t*)p;    p += a256(hist_elems * 8);
  uint64_t* ws = (uint64_t*)p;      p += a256(scan_ws_elems(hist_elems) * 8);
  uint64_t* unused_total = (uint64_t*)p;  // grand totals of the histogram scans

  sort_keys_kernel<<<grid_for(n), kSortThreads, 0, st>>>(d_rec, n, record_bytes, key_off, key_len, words);
  if (launches) *launches += 1;

  const uint32_t* idx = nullptr;  // current order; nullptr = input order
  if (n > 1) {
    uint32_t pass = 0;
    for (int w = (int)W - 1; w >= 0; w--) {
      const uint32_t* kin = words + (size_t)w * n;
      if (idx) {  // the current keys' buffer is free again: put this word there, in the current order
        uint32_t* kg = K[(pass - 1) & 1];
        sort_word_gather_kernel<<<grid_for(n), kSortThreads, 0, st>>>(kin, idx, n, kg);
        if (launches) *launches += 1;
        kin = kg;
      }
      // the last word holds key_len - 4 (W - 1) real bytes in its high end; the others hold four
      const uint32_t real = w == (int)W - 1 ? key_len - 4 * (W - 1) : 4;
      for (uint32_t shift = 32 - 8 * real; shift < 32; shift += 8, pass++) {
        launch_radix_pass(kin, idx, (uint32_t)n, (int)shift, 256, hist, unused_total, ws, K[pass & 1], I[pass & 1],
                          st, launches);
        kin = K[pass & 1];
        idx = I[pass & 1];
      }
    }
  }

  sort_fixed_offsets_kernel<<<grid_for(n), kSortThreads, 0, st>>>(n, record_bytes, src_off, sdst, len);
  if (launches) *launches += 1;
  PartitionPlan plan;
  plan.src_off = src_off;
  plan.sdst = sdst;
  plan.idx = idx;
  launch_partition_gather(d_rec, len, n, plan, d_dst, st, launches);
}

}  // namespace b2s
