// partition.cu — stable partition of serialized records by reduce id (the map side of Spark's serialized shuffle:
// ShuffleExternalSorter.insertRecord stores (record, partitionId) pairs, sorts the pointers by partition id and writes
// each partition in insertion order).  Four steps, all on the device:
//   prep    : rec_len (u32) widened into the u64 offset array that the scan turns into record offsets; ids validated
//   radix   : LSD radix sort of (id, record index) pairs, <= 8 bits per pass; per pass a per-tile digit histogram,
//             one scan over the digit-major histogram, and a stable scatter (warp match + per-warp shared counters)
//   bounds  : sorted record lengths -> scan -> destination offsets; the first sorted record of each partition gives
//             the partition's offset in the arena
//   gather  : records copied in sorted order into the partitioned arena (lane per short record, warp per long one;
//             stores go to 16-byte aligned destination pieces, sources are read as aligned 8-byte words)
#include <algorithm>

#include "kernels.h"

namespace b2s {

namespace {

constexpr int kPartThreads = 256;
constexpr int kPartWarps = kPartThreads / 32;
constexpr int kPartItems = 16;  // keys per thread per tile
constexpr uint32_t kPartTile = kPartThreads * kPartItems;
constexpr uint32_t kLaneCopyMax = 256;  // longer records are copied by the whole warp

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// off[i] = rec_len[i] (scanned in place afterwards); the first record with an id >= num_partitions goes to *bad
__global__ void __launch_bounds__(kPartThreads) part_prep_kernel(const uint32_t* __restrict__ rec_len,
                                                                 const uint32_t* __restrict__ rec_part, uint64_t n,
                                                                 uint32_t num_partitions, uint64_t* __restrict__ off,
                                                                 unsigned long long* __restrict__ bad) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    off[i] = rec_len[i];
    if (rec_part[i] >= num_partitions) atomicMin(bad, (unsigned long long)i);
  }
}

// hist[d * ntiles + tile] = number of keys of the tile whose digit is d
__global__ void __launch_bounds__(kPartThreads) part_hist_kernel(const uint32_t* __restrict__ keys, uint32_t n,
                                                                 int shift, uint32_t nd, uint32_t ntiles,
                                                                 uint64_t* __restrict__ hist) {
  __shared__ uint32_t cnt[256];
  const uint32_t tile = blockIdx.x;
  if (threadIdx.x < nd) cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t base = tile * kPartTile;
  for (int r = 0; r < kPartItems; r++) {
    const uint32_t i = base + (uint32_t)r * kPartThreads + threadIdx.x;
    const bool valid = i < n;
    const uint32_t d = valid ? (keys[i] >> shift) & (nd - 1) : 0x100u;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (valid && (peers & lanemask_lt()) == 0) atomicAdd(&cnt[d], (uint32_t)__popc(peers));
  }
  __syncthreads();
  if (threadIdx.x < nd) hist[(size_t)threadIdx.x * ntiles + tile] = cnt[threadIdx.x];
}

// Stable scatter: keys of a tile are taken 256 at a time in input order; within a warp __match_any_sync ranks equal
// digits, per-warp counts in shared memory rank them across warps, and a per-digit running count carries the rank
// across the rounds of the tile.  hist = exclusive scan of part_hist_kernel's output (the digit's base in the tile).
// idx_in == nullptr: the key's index is its position (first pass).
__global__ void __launch_bounds__(kPartThreads) part_scatter_kernel(const uint32_t* __restrict__ keys_in,
                                                                    const uint32_t* __restrict__ idx_in, uint32_t n,
                                                                    int shift, uint32_t nd, uint32_t ntiles,
                                                                    const uint64_t* __restrict__ hist,
                                                                    uint32_t* __restrict__ keys_out,
                                                                    uint32_t* __restrict__ idx_out) {
  __shared__ uint32_t wcnt[kPartWarps][256];
  __shared__ uint32_t run[256];
  __shared__ uint32_t base_of[256];
  const uint32_t tile = blockIdx.x, w = threadIdx.x >> 5, t = threadIdx.x;
  if (t < nd) {
    run[t] = 0;
    base_of[t] = (uint32_t)hist[(size_t)t * ntiles + tile];  // < n < 2^32
  }
  const uint32_t base = tile * kPartTile;
  for (int r = 0; r < kPartItems; r++) {
    if (base + (uint32_t)r * kPartThreads >= n) break;  // uniform over the block
    if (t < nd)
#pragma unroll
      for (int k = 0; k < kPartWarps; k++) wcnt[k][t] = 0;
    __syncthreads();
    const uint32_t i = base + (uint32_t)r * kPartThreads + t;
    const bool valid = i < n;
    const uint32_t key = valid ? keys_in[i] : 0u;
    const uint32_t idx = valid ? (idx_in ? idx_in[i] : i) : 0u;
    const uint32_t d = valid ? (key >> shift) & (nd - 1) : 0x100u;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned before = peers & lanemask_lt();
    if (valid && before == 0) wcnt[w][d] = (uint32_t)__popc(peers);
    __syncthreads();
    if (t < nd) {
      uint32_t acc = run[t];
#pragma unroll
      for (int k = 0; k < kPartWarps; k++) {
        const uint32_t c = wcnt[k][t];
        wcnt[k][t] = acc;
        acc += c;
      }
      run[t] = acc;
    }
    __syncthreads();
    if (valid) {
      const uint32_t pos = base_of[d] + wcnt[w][d] + (uint32_t)__popc(before);
      keys_out[pos] = key;
      idx_out[pos] = idx;
    }
    __syncthreads();
  }
}

// slen[j] = length of the j-th record in sorted order (scanned in place afterwards into its arena offset)
__global__ void __launch_bounds__(kPartThreads) part_sorted_len_kernel(const uint32_t* __restrict__ idx,
                                                                       const uint32_t* __restrict__ rec_len, uint64_t n,
                                                                       uint64_t* __restrict__ slen) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
    slen[j] = rec_len[idx ? idx[j] : j];
}

// part_start[p] = arena offset of partition p's first record (untouched, i.e. ~0, for partitions without records).
// keys == nullptr (no radix pass: one partition) reads the ids in input order.
__global__ void __launch_bounds__(kPartThreads) part_bounds_kernel(const uint32_t* __restrict__ keys,
                                                                   const uint32_t* __restrict__ rec_part, uint64_t n,
                                                                   uint32_t num_partitions,
                                                                   const uint64_t* __restrict__ sdst,
                                                                   uint64_t* __restrict__ part_start) {
  const uint32_t* k = keys ? keys : rec_part;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t p = k[j];
    if (p < num_partitions && (j == 0 || k[j - 1] != p)) part_start[p] = sdst[j];
  }
}

// one lane copies n bytes: destination-aligned 16-byte stores, sources read as aligned 8-byte words (ld_span16)
__device__ __forceinline__ void lane_copy(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, uint32_t n) {
  uint64_t lo, hi;
  uint32_t head = (uint32_t)((16u - (reinterpret_cast<uintptr_t>(d) & 15u)) & 15u);
  if (head > n) head = n;
  if (head) {
    ld_span16<true>(s, (int)head, lo, hi);
    st_span16(d, (int)head, lo, hi);
    d += head;
    s += head;
    n -= head;
  }
  for (; n >= 16; n -= 16, d += 16, s += 16) {
    ld_span16<true>(s, 16, lo, hi);
    *reinterpret_cast<ulonglong2*>(d) = make_ulonglong2(lo, hi);
  }
  if (n) {
    ld_span16<true>(s, (int)n, lo, hi);
    st_span16(d, (int)n, lo, hi);
  }
}

// A warp takes 32 consecutive sorted records, so its stores land in one contiguous stretch of the arena.  Records up to
// kLaneCopyMax bytes are copied by their own lane; longer ones afterwards by the whole warp, one at a time.
__global__ void __launch_bounds__(kPartThreads) part_gather_kernel(const uint8_t* __restrict__ src,
                                                                   const uint64_t* __restrict__ src_off,
                                                                   const uint32_t* __restrict__ rec_len,
                                                                   const uint32_t* __restrict__ idx,
                                                                   const uint64_t* __restrict__ sdst, uint64_t n,
                                                                   uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * kPartWarps;
  for (uint64_t g = (uint64_t)blockIdx.x * kPartWarps + (threadIdx.x >> 5); g * 32 < n; g += warps) {
    const uint64_t j = g * 32 + lane;
    uint32_t len = 0;
    uint64_t so = 0, dof = 0;
    if (j < n) {
      const uint32_t i = idx ? idx[j] : (uint32_t)j;
      len = rec_len[i];
      so = src_off[i];
      dof = sdst[j];
    }
    const bool long_rec = len > kLaneCopyMax;
    if (len && !long_rec) lane_copy(dst + dof, src + so, len);
    unsigned todo = __ballot_sync(0xffffffffu, long_rec);
    while (todo) {
      const int l = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint32_t ln = __shfl_sync(0xffffffffu, len, l);
      const uint64_t s = __shfl_sync(0xffffffffu, so, l), d = __shfl_sync(0xffffffffu, dof, l);
      warp_copy(dst + d, src + s, ln, lane);
    }
  }
}

inline unsigned grid_for(uint64_t n) {
  const uint64_t want = (n + kPartThreads - 1) / kPartThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

}  // namespace

uint32_t partition_radix_passes(uint32_t num_partitions) {
  uint32_t bits = 0;
  while (bits < 32 && (1ull << bits) < num_partitions) bits++;
  return (bits + 7) / 8;
}

size_t radix_hist_elems(uint64_t n) {
  const uint64_t ntiles = (n + kPartTile - 1) / kPartTile;
  return (size_t)256 * (ntiles ? ntiles : 1);
}

void launch_radix_pass(const uint32_t* keys_in, const uint32_t* idx_in, uint32_t n, int shift, uint32_t nd,
                       uint64_t* hist, uint64_t* hist_total, uint64_t* scan_ws, uint32_t* keys_out, uint32_t* idx_out,
                       cudaStream_t st, uint64_t* launches) {
  const uint32_t ntiles = (uint32_t)(((uint64_t)n + kPartTile - 1) / kPartTile);
  part_hist_kernel<<<ntiles, kPartThreads, 0, st>>>(keys_in, n, shift, nd, ntiles, hist);
  launch_exclusive_scan_u64(hist, (size_t)nd * ntiles, hist_total, scan_ws, st, launches);
  part_scatter_kernel<<<ntiles, kPartThreads, 0, st>>>(keys_in, idx_in, n, shift, nd, ntiles, hist, keys_out, idx_out);
  if (launches) *launches += 2;
}

size_t partition_ws_bytes(uint64_t n, uint32_t num_partitions) {
  const size_t hist = radix_hist_elems(n);
  auto a = [](size_t b) { return (b + 255) / 256 * 256; };
  return a((n + 1) * 8) * 2 + a(n * 4) * 4 + a(hist * 8) + a(scan_ws_elems(std::max<size_t>(hist, n + 1)) * 8) +
         256 + a(((size_t)num_partitions + 2) * 8) + 1024;
}

void launch_partition(const uint32_t* d_rec_len, const uint32_t* d_rec_part, uint64_t n, uint32_t num_partitions,
                      uint8_t* d_ws, PartitionPlan* plan, cudaStream_t st,
                      uint64_t* launches) {
  auto a = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t hist_elems = radix_hist_elems(n);
  uint8_t* p = d_ws;
  plan->src_off = (uint64_t*)p;  p += a((n + 1) * 8);
  plan->sdst = (uint64_t*)p;     p += a((n + 1) * 8);
  uint32_t* kA = (uint32_t*)p;   p += a(n * 4);
  uint32_t* iA = (uint32_t*)p;   p += a(n * 4);
  uint32_t* kB = (uint32_t*)p;   p += a(n * 4);
  uint32_t* iB = (uint32_t*)p;   p += a(n * 4);
  uint64_t* hist = (uint64_t*)p; p += a(hist_elems * 8);
  uint64_t* ws = (uint64_t*)p;   p += a(scan_ws_elems(std::max<size_t>(hist_elems, n + 1)) * 8);
  uint64_t* unused_total = (uint64_t*)p;  p += 256;  // grand totals of the histogram scans and of the sorted-length scan
  // readback block: [bad, total, part_start[num_partitions]]
  plan->readback = (uint64_t*)p;
  plan->readback_bytes = ((size_t)num_partitions + 2) * 8;
  uint64_t* bad = plan->readback;
  uint64_t* total = plan->readback + 1;
  uint64_t* part_start = plan->readback + 2;
  cudaMemsetAsync(plan->readback, 0xff, plan->readback_bytes, st);

  part_prep_kernel<<<grid_for(n), kPartThreads, 0, st>>>(d_rec_len, d_rec_part, n, num_partitions, plan->src_off,
                                                         (unsigned long long*)bad);
  launch_exclusive_scan_u64(plan->src_off, n, total, ws, st, launches);

  const uint32_t passes = partition_radix_passes(num_partitions);
  uint32_t bits = 0;
  while (bits < 32 && (1ull << bits) < num_partitions) bits++;
  const uint32_t* keys = nullptr;
  const uint32_t* idx = nullptr;
  int shift = 0;
  for (uint32_t k = 0; k < passes; k++) {
    const uint32_t pb = (bits - (uint32_t)shift + (passes - k) - 1) / (passes - k);  // spread the bits evenly
    const uint32_t nd = 1u << pb;
    const uint32_t* kin = keys ? keys : d_rec_part;
    uint32_t* kout = (k & 1) ? kB : kA;
    uint32_t* iout = (k & 1) ? iB : iA;
    launch_radix_pass(kin, idx, (uint32_t)n, shift, nd, hist, unused_total, ws, kout, iout, st, launches);
    keys = kout;
    idx = iout;
    shift += (int)pb;
  }
  plan->idx = idx;
  part_sorted_len_kernel<<<grid_for(n), kPartThreads, 0, st>>>(idx, d_rec_len, n, plan->sdst);
  launch_exclusive_scan_u64(plan->sdst, n, unused_total, ws, st, launches);
  part_bounds_kernel<<<grid_for(n), kPartThreads, 0, st>>>(keys, d_rec_part, n, num_partitions, plan->sdst, part_start);
  if (launches) *launches += 3;
}

void launch_partition_gather(const uint8_t* rec_base, const uint32_t* d_rec_len, uint64_t n, const PartitionPlan& plan,
                             uint8_t* d_dst, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  const uint64_t groups = (n + 31) / 32;
  const uint64_t blocks = (groups + kPartWarps - 1) / kPartWarps;
  const unsigned grid = (unsigned)std::min<uint64_t>(blocks, (uint64_t)kSMs * 16);
  part_gather_kernel<<<grid, kPartThreads, 0, st>>>(rec_base, plan.src_off, d_rec_len, plan.idx, plan.sdst, n, d_dst);
  if (launches) *launches += 1;
}

}  // namespace b2s
