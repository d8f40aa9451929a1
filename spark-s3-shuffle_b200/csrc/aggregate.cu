// aggregate.cu — group a reduce task's key-sorted UnsafeRow records by key and merge their aggregate buffers (the
// HashAggregateExec(Final) that Spark SQL runs right after the shuffle read of a grouped aggregation).  The records have
// been framed, keyed and radix-sorted by rows.cu; from the sorted indices, all on the device:
//   heads   : one thread per sorted position j: flag = the key words of idx[j] differ from those of idx[j - 1] (or
//             j = 0); the same thread loads every aggregate's 8-byte slot and null bit of the record into dense,
//             sorted-order arrays (vals[a * n + j], nulls[j] bit a), so that the merge below reads coalesced memory
//   scan    : the flags scanned: the group of every position and the group count
//   compact : per group its first position, the first record's index and length (0 past the last group), whose scan
//             (launch_sorted_offsets) is the group's output offset and the output bytes; both totals come back in one
//             readback, which sizes the output
//   gather  : the group heads' records, whole, to the output (launch_partition_gather); no other record is copied
//   merge   : every aggregate over each group's records, in sorted (stable) order, patched into the gathered row: a
//             thread per group of up to kSmallGroup records, a warp per larger group (32 records at a time, loads in
//             parallel).  Sums and min / max combine exactly across lanes; the double sum adds in record order (each
//             lane's value broadcast in turn), so it is bit for bit the sequential sum.  One thread writes an output
//             row's slots and then its null words, one read-modify-write per aggregate, so aggregates (and the key)
//             that share a null word never race.
#include <algorithm>

#include "kernels.h"

namespace b2s {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kAggThreads = 256;
constexpr uint32_t kSmallGroup = 16;

inline size_t a256(size_t b) { return (b + 255) / 256 * 256; }

inline unsigned grid_for(uint64_t n) {
  const uint64_t want = (n + kAggThreads - 1) / kAggThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

// the aggregate workspace: heads (scanned in place), readback [groups, output bytes], per group the head's record
// index, first position (+ n at the end) and record length, the dense null bits and values, the spec
struct AggWs {
  uint64_t* head;
  uint64_t* readback;
  uint32_t* hidx;
  uint32_t* gpos;
  uint32_t* glen;
  uint32_t* nulls;
  uint64_t* vals;
  AggSpec* spec;
};

AggWs carve_agg_ws(uint8_t* d_aws, uint64_t n, uint32_t n_aggs) {
  AggWs a;
  uint8_t* p = d_aws;
  a.head = (uint64_t*)p;     p += a256(n * 8);
  a.readback = (uint64_t*)p; p += a256(16);
  a.hidx = (uint32_t*)p;     p += a256(n * 4);
  a.gpos = (uint32_t*)p;     p += a256((n + 1) * 4);
  a.glen = (uint32_t*)p;     p += a256(n * 4);
  a.nulls = (uint32_t*)p;    p += a256(n * 4);
  a.vals = (uint64_t*)p;     p += a256(n * n_aggs * 8);
  a.spec = (AggSpec*)p;
  return a;
}

__device__ __forceinline__ bool bit_set(const uint8_t* row, int32_t field) {
  uint64_t w, unused;
  ld_span16<true>(row + 8 * (uint32_t)(field >> 6), 8, w, unused);
  return (w >> (field & 63)) & 1;
}

__global__ void __launch_bounds__(kAggThreads) agg_heads_kernel(const uint8_t* __restrict__ arena,
                                                                const uint64_t* __restrict__ rec_off,
                                                                const uint32_t* __restrict__ idx, uint64_t n,
                                                                const uint32_t* __restrict__ words, uint32_t W,
                                                                const uint32_t* __restrict__ heads,
                                                                const AggSpec* __restrict__ spec,
                                                                uint64_t* __restrict__ head, uint32_t* __restrict__ nulls,
                                                                uint64_t* __restrict__ vals) {
  const uint32_t n_aggs = spec->n;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = idx ? idx[j] : (uint32_t)j;
    bool h = j == 0;
    if (heads) {
      h = heads[j] != 0;
    } else if (!h) {
      const uint32_t p = idx ? idx[j - 1] : (uint32_t)(j - 1);
#pragma unroll
      for (uint32_t k = 0; k < 5; k++)
        if (k < W) h |= words[(size_t)k * n + i] != words[(size_t)k * n + p];
    }
    head[j] = h;
    const uint8_t* row = arena + rec_off[i] + 4;
    uint32_t nm = 0;
    for (uint32_t a = 0; a < n_aggs; a++) {
      uint64_t v, unused;
      ld_span16<true>(row + spec->off[a], 8, v, unused);
      vals[(size_t)a * n + j] = v;
      const int32_t nf = spec->null_field[a];
      if (nf >= 0 && bit_set(row, nf)) nm |= 1u << a;
    }
    nulls[j] = nm;
  }
}

// head holds the exclusive scan of the flags, *groups their total
__global__ void __launch_bounds__(kAggThreads) agg_compact_kernel(const uint64_t* __restrict__ head,
                                                                  const uint64_t* __restrict__ groups,
                                                                  const uint32_t* __restrict__ idx,
                                                                  const uint32_t* __restrict__ rec_len, uint64_t n,
                                                                  uint32_t* __restrict__ hidx,
                                                                  uint32_t* __restrict__ gpos,
                                                                  uint32_t* __restrict__ glen) {
  const uint64_t G = *groups;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = head[j], next = j + 1 < n ? head[j + 1] : G;
    if (next != g) {
      const uint32_t i = idx ? idx[j] : (uint32_t)j;
      hidx[g] = i;
      gpos[g] = (uint32_t)j;
      glen[g] = rec_len[i];
    }
    if (j >= G) glen[j] = 0;
    if (j == n - 1) gpos[G] = (uint32_t)n;
  }
}

// Spark SQL's double order as an unsigned key: -0.0 == 0.0, every NaN equal and above +inf
__device__ __forceinline__ uint64_t double_key(uint64_t b) {
  if ((b & ~(1ull << 63)) > 0x7ff0000000000000ull) return ~0ull;
  if (b == (1ull << 63)) b = 0;
  return (b >> 63) ? ~b : (b | (1ull << 63));
}

// the order key of a min / max op (larger key = larger value); other ops: unused
__device__ __forceinline__ uint64_t order_key(uint32_t op, uint64_t v) {
  if (op == B2S_AGG_MIN_INT32 || op == B2S_AGG_MAX_INT32) return (uint32_t)v ^ 0x80000000u;
  if (op == B2S_AGG_MIN_INT64 || op == B2S_AGG_MAX_INT64) return v ^ (1ull << 63);
  return double_key(v);
}

__device__ __forceinline__ bool is_max(uint32_t op) {
  return op == B2S_AGG_MAX_INT32 || op == B2S_AGG_MAX_INT64 || op == B2S_AGG_MAX_FLOAT64;
}

// x replaces the best so far when it is strictly better: among equal values the first in stable order stays
__device__ __forceinline__ bool better(bool mx, uint64_t kx, uint64_t kbest) { return mx ? kx > kbest : kx < kbest; }

// the slot a result is written as: an INT32 result with its high 4 bytes zero, as UnsafeRowWriter writes it
__device__ __forceinline__ uint64_t slot_of(uint32_t op, uint64_t v) {
  return (op == B2S_AGG_MIN_INT32 || op == B2S_AGG_MAX_INT32) ? (uint32_t)v : v;
}

// aggregate a of the records at positions [s, e), by one thread; returns false when none of them is non-null
__device__ __forceinline__ bool merge_thread(uint32_t op, uint32_t a, const uint64_t* __restrict__ vals,
                             const uint32_t* __restrict__ nulls, uint64_t n, uint32_t s, uint32_t e, uint64_t* out) {
  bool has = false;
  uint64_t acc = 0, best = 0, kbest = 0;
  double fs = 0.0;
  const bool mx = is_max(op);
  for (uint32_t j = s; j < e; j++) {
    if ((__ldg(nulls + j) >> a) & 1) continue;
    const uint64_t v = __ldg(vals + (size_t)a * n + j);
    if (op == B2S_AGG_SUM_INT64) {
      acc += v;
    } else if (op == B2S_AGG_SUM_FLOAT64) {
      fs = __dadd_rn(fs, __longlong_as_double((long long)v));
    } else {
      const uint64_t k = order_key(op, v);
      if (!has || better(mx, k, kbest)) {
        kbest = k;
        best = v;
      }
    }
    has = true;
  }
  *out = op == B2S_AGG_SUM_INT64 ? acc : op == B2S_AGG_SUM_FLOAT64 ? (uint64_t)__double_as_longlong(fs) : best;
  return has;
}

// aggregate a of the records at positions [s, e), by the whole warp (every lane returns the result)
__device__ __forceinline__ bool merge_warp(uint32_t op, uint32_t a, const uint64_t* __restrict__ vals, const uint32_t* __restrict__ nulls,
                           uint64_t n, uint32_t s, uint32_t e, uint32_t lane, uint64_t* out) {
  const uint64_t* va = vals + (size_t)a * n;
  if (op == B2S_AGG_SUM_FLOAT64) {  // loads in parallel, four rounds of 32 ahead; the adds in record order
    double fs = 0.0;
    bool any = false;
    for (uint32_t b = s; b < e; b += 128) {
      uint64_t v[4];
      unsigned ok[4];
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const uint32_t j = b + 32 * r + lane;
        const bool in = j < e && !((__ldg(nulls + j) >> a) & 1);
        v[r] = in ? __ldg(va + j) : 0;
        ok[r] = __ballot_sync(FULL, in);
      }
#pragma unroll
      for (int r = 0; r < 4; r++) {
        any |= ok[r] != 0;
#pragma unroll
        for (int l = 0; l < 32; l++) {
          const double x = __longlong_as_double((long long)__shfl_sync(FULL, v[r], l));
          if ((ok[r] >> l) & 1) fs = __dadd_rn(fs, x);
        }
      }
    }
    *out = (uint64_t)__double_as_longlong(fs);
    return any;
  }
  // integer sum and min / max: each lane over its records (positions s + lane, s + lane + 32, ...), then the lanes
  // combined; min / max keep the earliest position among equal keys
  const bool mx = is_max(op);
  bool has = false;
  uint64_t acc = 0, best = 0, kbest = 0;
  uint32_t pbest = 0;
  for (uint32_t b = s; b < e; b += 128) {
    uint64_t v[4];
    bool in[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const uint32_t j = b + 32 * r + lane;
      in[r] = j < e && !((__ldg(nulls + j) >> a) & 1);
      v[r] = in[r] ? __ldg(va + j) : 0;
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
      if (!in[r]) continue;
      if (op == B2S_AGG_SUM_INT64) {
        acc += v[r];
      } else {
        const uint64_t k = order_key(op, v[r]);
        if (!has || better(mx, k, kbest)) {
          kbest = k;
          best = v[r];
          pbest = b + 32 * r + lane;
        }
      }
      has = true;
    }
  }
  const bool any = __any_sync(FULL, has);
  if (op == B2S_AGG_SUM_INT64) {
#pragma unroll
    for (int d = 16; d; d >>= 1) acc += __shfl_xor_sync(FULL, acc, d);
    *out = acc;
    return any;
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    const bool oh = __shfl_xor_sync(FULL, has, d);
    const uint64_t ok = __shfl_xor_sync(FULL, kbest, d), ob = __shfl_xor_sync(FULL, best, d);
    const uint32_t op_ = __shfl_xor_sync(FULL, pbest, d);
    if (oh && (!has || better(mx, ok, kbest) || (ok == kbest && op_ < pbest))) {
      has = true;
      kbest = ok;
      best = ob;
      pbest = op_;
    }
  }
  *out = best;
  return any;
}

// the result of aggregate a into the output row (slot, and null bit in *null_mask)
__device__ __forceinline__ void put(uint8_t* row, uint32_t op, uint32_t off, uint32_t a, bool has, uint64_t v,
                                    uint32_t* null_mask) {
  st_span16(row + off, 8, has ? slot_of(op, v) : 0ull, 0);
  if (!has) *null_mask |= 1u << a;
}

// after every slot: each aggregate's null bit, one read-modify-write of its null word at a time
__device__ __forceinline__ void put_null_bits(uint8_t* row, const AggSpec* __restrict__ spec, uint32_t n_aggs,
                                              uint32_t null_mask) {
  for (uint32_t a = 0; a < n_aggs; a++) {
    const int32_t nf = spec->null_field[a];
    if (nf < 0) continue;
    uint8_t* p = row + 8 * (uint32_t)(nf >> 6);
    uint64_t w, unused;
    ld_span16<false>(p, 8, w, unused);
    const uint64_t bit = 1ull << (nf & 63);
    w = ((null_mask >> a) & 1) ? (w | bit) : (w & ~bit);
    st_span16(p, 8, w, 0);
  }
}

// groups of up to kSmallGroup records: a thread each
__global__ void __launch_bounds__(kAggThreads) agg_merge_small_kernel(const uint32_t* __restrict__ gpos, uint64_t G,
                                                                      uint64_t n, const uint64_t* __restrict__ vals,
                                                                      const uint32_t* __restrict__ nulls,
                                                                      const AggSpec* __restrict__ spec, uint32_t n_aggs,
                                                                      const uint64_t* __restrict__ gdst,
                                                                      uint8_t* __restrict__ dst) {
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < G; g += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t s = gpos[g], e = gpos[g + 1];
    if (e - s > kSmallGroup) continue;
    uint8_t* row = dst + gdst[g] + 4;
    uint32_t null_mask = 0;
    for (uint32_t a = 0; a < n_aggs; a++) {
      const uint32_t op = spec->op[a];
      uint64_t v;
      const bool has = merge_thread(op, a, vals, nulls, n, s, e, &v);
      put(row, op, spec->off[a], a, has, v, &null_mask);
    }
    put_null_bits(row, spec, n_aggs, null_mask);
  }
}

// the larger groups: a warp each (warps step through the groups and skip the small ones)
__global__ void __launch_bounds__(kAggThreads) agg_merge_large_kernel(const uint32_t* __restrict__ gpos, uint64_t G,
                                                                      uint64_t n, const uint64_t* __restrict__ vals,
                                                                      const uint32_t* __restrict__ nulls,
                                                                      const AggSpec* __restrict__ spec, uint32_t n_aggs,
                                                                      const uint64_t* __restrict__ gdst,
                                                                      uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (kAggThreads / 32);
  for (uint64_t g = (uint64_t)blockIdx.x * (kAggThreads / 32) + (threadIdx.x >> 5); g < G; g += warps) {
    const uint32_t s = gpos[g], e = gpos[g + 1];
    if (e - s <= kSmallGroup) continue;  // uniform over the warp
    uint8_t* row = dst + gdst[g] + 4;
    uint32_t null_mask = 0;
    for (uint32_t a = 0; a < n_aggs; a++) {
      const uint32_t op = spec->op[a];
      uint64_t v;
      const bool has = merge_warp(op, a, vals, nulls, n, s, e, lane, &v);
      if (lane == 0) put(row, op, spec->off[a], a, has, v, &null_mask);
    }
    if (lane == 0) put_null_bits(row, spec, n_aggs, null_mask);
  }
}

}  // namespace

size_t rows_aggregate_ws_bytes(uint64_t n, uint32_t n_aggs) {
  return a256(n * 8) + a256(16) + 3 * a256(n * 4) + a256((n + 1) * 4) + a256(n * n_aggs * 8) + a256(sizeof(AggSpec));
}

uint64_t* rows_aggregate_readback(uint8_t* d_aws, uint64_t n, uint32_t n_aggs) {
  return carve_agg_ws(d_aws, n, n_aggs).readback;
}

void launch_rows_group(const uint8_t* arena, uint64_t n, const uint32_t* idx, const uint32_t* heads,
                       uint32_t key_bytes, const AggSpec& spec, uint8_t* d_ws, uint8_t* d_aws, cudaStream_t st,
                       uint64_t* launches) {
  const AggWs a = carve_agg_ws(d_aws, n, spec.n);
  if (!n) {
    cudaMemsetAsync(a.readback, 0, 16, st);
    return;
  }
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  uint64_t* scan_ws = (uint64_t*)(d_ws + key_sort_ws_bytes(n, key_bytes));
  cudaMemcpyAsync(a.spec, &spec, sizeof(AggSpec), cudaMemcpyHostToDevice, st);
  agg_heads_kernel<<<grid_for(n), kAggThreads, 0, st>>>(arena, w.src_off, idx, n, w.words, (key_bytes + 3) / 4, heads,
                                                        a.spec, a.head, a.nulls, a.vals);
  launch_exclusive_scan_u64(a.head, n, a.readback, scan_ws, st, launches);
  agg_compact_kernel<<<grid_for(n), kAggThreads, 0, st>>>(a.head, a.readback, idx, w.len, n, a.hidx, a.gpos, a.glen);
  // the group lengths are already in group order: no index
  launch_sorted_offsets(nullptr, a.glen, n, w.sdst, a.readback + 1, scan_ws, st, launches);
  if (launches) *launches += 2;
}

void launch_rows_aggregate(const uint8_t* arena, uint64_t n, uint64_t groups, uint32_t key_bytes, uint32_t n_aggs,
                           uint8_t* d_ws, uint8_t* d_aws, uint8_t* d_dst, cudaStream_t st, uint64_t* launches) {
  if (!groups) return;
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  const AggWs a = carve_agg_ws(d_aws, n, n_aggs);
  PartitionPlan plan;
  plan.src_off = w.src_off;
  plan.sdst = w.sdst;
  plan.idx = a.hidx;
  launch_partition_gather(arena, w.len, groups, plan, d_dst, st, launches);
  if (!n_aggs) return;
  agg_merge_small_kernel<<<grid_for(groups), kAggThreads, 0, st>>>(a.gpos, groups, n, a.vals, a.nulls, a.spec, n_aggs,
                                                                    w.sdst, d_dst);
  const uint64_t ctas = (groups + kAggThreads / 32 - 1) / (kAggThreads / 32);
  agg_merge_large_kernel<<<(unsigned)std::min<uint64_t>(ctas, (uint64_t)kSMs * 16), kAggThreads, 0, st>>>(
      a.gpos, groups, n, a.vals, a.nulls, a.spec, n_aggs, w.sdst, d_dst);
  if (launches) *launches += 2;
}

}  // namespace b2s
