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
// The Decimal ops (B2S_AGG_*_DECIMAL) are merged by kernels of their own (the *_dec kernels, launched only when the spec
// has one), so the kernels of the other ops keep their code and registers.  An out-of-line decimal is staged by the
// heads step as 16 bytes (the value's low words in vals, its high words in vhi), which also checks every record's
// 16-byte region.  The sum is exact and null once an input is null or a running sum leaves (-10^P, 10^P): a thread adds
// with the 128-bit overflow of decimal128.h; a warp scans each round of 32 inputs in three 64-bit words (33 * 10^38 <
// 2^133), adds the rounds before it and checks every lane's running sum with one vote.
// B2S_AGG_VARIANCE (Spark's CentralMomentAgg [n, avg, m2]) is merged by kernels of its own too (the *_var kernels,
// which also know the Decimal ops): the heads step stages n with the other slots and avg, m2 in arrays of their own; a
// thread per small group, or a warp per large one (loads in parallel, each lane's triple broadcast in turn), runs
// mergeExpressions in stable order from (0, 0, 0), one rounded double operation at a time.
#include <algorithm>

#include "decimal128.h"
#include "kernels.h"
#include "rows_key.cuh"

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

// the aggregate workspace: heads (scanned in place), readback [groups, output bytes, decimal verdict], per group the
// head's record index, first position (+ n at the end) and record length, the dense null bits and values, the high
// words of the out-of-line decimals, the spec, the variance entries' avg and m2 words
struct AggWs {
  uint64_t* head;
  uint64_t* readback;
  uint32_t* hidx;
  uint32_t* gpos;
  uint32_t* glen;
  uint32_t* nulls;
  uint64_t* vals;
  uint64_t* vhi;
  AggSpec* spec;
  uint64_t* vmom;
};

AggWs carve_agg_ws(uint8_t* d_aws, uint64_t n, uint32_t n_aggs, uint32_t n_wide, uint32_t n_var = 0) {
  AggWs a;
  uint8_t* p = d_aws;
  a.head = (uint64_t*)p;     p += a256(n * 8);
  a.readback = (uint64_t*)p; p += a256(24);
  a.hidx = (uint32_t*)p;     p += a256(n * 4);
  a.gpos = (uint32_t*)p;     p += a256((n + 1) * 4);
  a.glen = (uint32_t*)p;     p += a256(n * 4);
  a.nulls = (uint32_t*)p;    p += a256(n * 4);
  a.vals = (uint64_t*)p;     p += a256(n * n_aggs * 8);
  a.vhi = (uint64_t*)p;      p += a256(n * n_wide * 8);
  a.spec = (AggSpec*)p;      p += a256(sizeof(AggSpec));
  a.vmom = n_var ? (uint64_t*)p : nullptr;
  return a;
}

__device__ __forceinline__ bool bit_set(const uint8_t* row, int32_t field) {
  uint64_t w, unused;
  ld_span16<true>(row + 8 * (uint32_t)(field >> 6), 8, w, unused);
  return (w >> (field & 63)) & 1;
}

// Dec (a spec with an out-of-line decimal): such an aggregate's value is staged as (vals, vhi) = its (lo, hi), 0 when
// null, and a record whose value or 16-byte region is bad lowers *bad to its arena offset << 2 | kAggBad*.  Var (a spec
// with a variance entry): its avg and m2 words (slots off + 8, off + 16) into vmom.
template <bool Dec, bool Var>
__device__ __forceinline__ void agg_heads(const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off,
                                          const uint32_t* __restrict__ rec_len, const uint32_t* __restrict__ idx,
                                          uint64_t n, const uint32_t* __restrict__ words, uint32_t W,
                                          const uint32_t* __restrict__ heads, const AggSpec* __restrict__ spec,
                                          uint64_t* __restrict__ head, uint32_t* __restrict__ nulls,
                                          uint64_t* __restrict__ vals, uint64_t* __restrict__ vhi,
                                          uint64_t* __restrict__ vmom, unsigned long long* __restrict__ bad) {
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
      const int32_t nf = spec->null_field[a];
      const bool null = nf >= 0 && bit_set(row, nf);
      if (null) nm |= 1u << a;
      if (Dec && agg_decimal_wide(spec->op[a])) {
        const uint32_t size = rec_len[i] - 4, so = (uint32_t)(v >> 32);
        uint64_t hi = 0, lo = 0;
        bool bad_value = false;
        if (!null) {
          decimal_bits(row, size, v, hi, lo, &bad_value);
          hi ^= 1ull << 63;  // decimal_bits flips the sign bit for the sort
        }
        const uint64_t why = bad_value                      ? kAggBadDecimal
                             : (uint64_t)so + 16 > size     ? kAggBadRegionEnd
                             : so < spec->region_from       ? kAggBadRegionStart
                                                            : 0;
        if (why) atomicMin(bad, (unsigned long long)((rec_off[i] << 2) | why));
        v = lo;
        vhi[(size_t)spec->wide[a] * n + j] = hi;
      }
      if (Var && spec->op[a] == B2S_AGG_VARIANCE) {
        uint64_t avg, m2;
        ld_span16<true>(row + spec->off[a] + 8, 16, avg, m2);
        vmom[(size_t)(2 * spec->var[a]) * n + j] = avg;
        vmom[(size_t)(2 * spec->var[a] + 1) * n + j] = m2;
      }
      vals[(size_t)a * n + j] = v;
    }
    nulls[j] = nm;
  }
}

template <bool Dec>
__global__ void __launch_bounds__(kAggThreads) agg_heads_kernel(const uint8_t* __restrict__ arena,
                                                                const uint64_t* __restrict__ rec_off,
                                                                const uint32_t* __restrict__ rec_len,
                                                                const uint32_t* __restrict__ idx, uint64_t n,
                                                                const uint32_t* __restrict__ words, uint32_t W,
                                                                const uint32_t* __restrict__ heads,
                                                                const AggSpec* __restrict__ spec,
                                                                uint64_t* __restrict__ head, uint32_t* __restrict__ nulls,
                                                                uint64_t* __restrict__ vals, uint64_t* __restrict__ vhi,
                                                                unsigned long long* __restrict__ bad) {
  agg_heads<Dec, false>(arena, rec_off, rec_len, idx, n, words, W, heads, spec, head, nulls, vals, vhi, nullptr, bad);
}

// agg_heads_kernel for a spec with a variance entry
template <bool Dec>
__global__ void __launch_bounds__(kAggThreads) agg_heads_var_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t n, const uint32_t* __restrict__ words, uint32_t W,
    const uint32_t* __restrict__ heads, const AggSpec* __restrict__ spec, uint64_t* __restrict__ head,
    uint32_t* __restrict__ nulls, uint64_t* __restrict__ vals, uint64_t* __restrict__ vhi, uint64_t* __restrict__ vmom,
    unsigned long long* __restrict__ bad) {
  agg_heads<Dec, true>(arena, rec_off, rec_len, idx, n, words, W, heads, spec, head, nulls, vals, vhi, vmom, bad);
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

// ---- the Decimal ops ----
// aggregate a (a Decimal op; wa: its index among the out-of-line ones) of the records at positions [s, e), by one
// thread; returns false when the result is null
__device__ __forceinline__ bool merge_thread_dec(uint32_t op, uint32_t a, uint32_t wa,
                                                 const uint64_t* __restrict__ vals, const uint64_t* __restrict__ vhi,
                                                 const uint32_t* __restrict__ nulls, uint64_t n, uint32_t s, uint32_t e,
                                                 Dec128* out) {
  const uint64_t* va = vals + (size_t)a * n;
  const uint64_t* ha = vhi + (size_t)wa * n;
  const bool wide = agg_decimal_wide(op);
  if (agg_base_op(op) == B2S_AGG_SUM_DECIMAL) {  // stable order from 0: null at the first null input or overflow
    const uint32_t P = agg_precision(op);
    Dec128 acc{0, 0};
    for (uint32_t j = s; j < e; j++) {
      if ((__ldg(nulls + j) >> a) & 1) return false;
      const Dec128 x = wide ? Dec128{__ldg(va + j), __ldg(ha + j)} : dec_of_long(__ldg(va + j));
      bool ovf;
      acc = dec_add(acc, x, &ovf);
      if (ovf || !dec_fits(acc, P)) return false;
    }
    *out = acc;
    return true;
  }
  const bool mx = agg_base_op(op) == B2S_AGG_MAX_DECIMAL;
  bool has = false;
  Dec128 best{0, 0};
  for (uint32_t j = s; j < e; j++) {
    if ((__ldg(nulls + j) >> a) & 1) continue;
    const Dec128 x{__ldg(va + j), __ldg(ha + j)};
    if (!has || (mx ? dec_less(best, x) : dec_less(x, best))) best = x;
    has = true;
  }
  *out = best;
  return has;
}

// (a2, a1, a0) += (b2, b1, b0): 192-bit two's complement
__device__ __forceinline__ void add192(uint64_t& a0, uint64_t& a1, uint64_t& a2, uint64_t b0, uint64_t b1,
                                       uint64_t b2) {
  a0 += b0;
  const uint64_t c0 = a0 < b0 ? 1 : 0;
  uint64_t t = a1 + b1;
  uint64_t c1 = t < b1 ? 1 : 0;
  t += c0;
  c1 += t < c0 ? 1 : 0;
  a1 = t;
  a2 += b2 + c1;
}

// merge_thread_dec by the whole warp (every lane returns the result).  The sum: per round of 32 records an inclusive
// scan of the inputs in three 64-bit words plus the running sum of the rounds before; the result is null as soon as
// any lane's input is null or any lane's running sum is out of range (one vote each, so the decision is warp-uniform),
// and no further rounds are loaded.  Min / max: each lane over its records, then the lanes combined, the earliest
// position kept among equal values.  Loads: four rounds of 32 in flight, as merge_warp.
__device__ __forceinline__ bool merge_warp_dec(uint32_t op, uint32_t a, uint32_t wa, const uint64_t* __restrict__ vals,
                                               const uint64_t* __restrict__ vhi, const uint32_t* __restrict__ nulls,
                                               uint64_t n, uint32_t s, uint32_t e, uint32_t lane, Dec128* out) {
  const uint64_t* va = vals + (size_t)a * n;
  const uint64_t* ha = vhi + (size_t)wa * n;
  const bool wide = agg_decimal_wide(op);
  if (agg_base_op(op) == B2S_AGG_SUM_DECIMAL) {
    const uint32_t P = agg_precision(op);
    uint64_t c0 = 0, c1 = 0, c2 = 0;  // the running sum before the round
    bool null = false;
    for (uint32_t b = s; b < e && !null; b += 128) {
      Dec128 x[4];
      bool nl[4];
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const uint32_t j = b + 32 * r + lane;
        nl[r] = j < e && ((__ldg(nulls + j) >> a) & 1);
        const bool in = j < e && !nl[r];
        const uint64_t lo = in ? __ldg(va + j) : 0;
        x[r] = wide ? Dec128{lo, in ? __ldg(ha + j) : 0} : dec_of_long(lo);
      }
#pragma unroll
      for (int r = 0; r < 4; r++) {
        if (__any_sync(FULL, nl[r])) {
          null = true;
          break;
        }
        uint64_t p0 = x[r].lo, p1 = x[r].hi, p2 = (uint64_t)((int64_t)x[r].hi >> 63);
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint64_t q0 = __shfl_up_sync(FULL, p0, d), q1 = __shfl_up_sync(FULL, p1, d),
                         q2 = __shfl_up_sync(FULL, p2, d);
          if (lane >= (uint32_t)d) add192(p0, p1, p2, q0, q1, q2);
        }
        add192(p0, p1, p2, c0, c1, c2);
        const bool ok = p2 == (uint64_t)((int64_t)p1 >> 63) && dec_fits(Dec128{p0, p1}, P);
        if (__any_sync(FULL, !ok)) {
          null = true;
          break;
        }
        c0 = __shfl_sync(FULL, p0, 31);
        c1 = __shfl_sync(FULL, p1, 31);
        c2 = __shfl_sync(FULL, p2, 31);
      }
    }
    *out = Dec128{c0, c1};
    return !null;
  }
  const bool mx = agg_base_op(op) == B2S_AGG_MAX_DECIMAL;
  bool has = false;
  Dec128 best{0, 0};
  uint32_t pbest = 0;
  for (uint32_t b = s; b < e; b += 128) {
    Dec128 x[4];
    bool in[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const uint32_t j = b + 32 * r + lane;
      in[r] = j < e && !((__ldg(nulls + j) >> a) & 1);
      x[r] = in[r] ? Dec128{__ldg(va + j), __ldg(ha + j)} : Dec128{0, 0};
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
      if (!in[r]) continue;
      if (!has || (mx ? dec_less(best, x[r]) : dec_less(x[r], best))) {
        best = x[r];
        pbest = b + 32 * r + lane;
      }
      has = true;
    }
  }
  const bool any = __any_sync(FULL, has);
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    const bool oh = __shfl_xor_sync(FULL, has, d);
    const Dec128 o{__shfl_xor_sync(FULL, best.lo, d), __shfl_xor_sync(FULL, best.hi, d)};
    const uint32_t op_ = __shfl_xor_sync(FULL, pbest, d);
    const bool eq = o.lo == best.lo && o.hi == best.hi;
    if (oh && (!has || (mx ? dec_less(best, o) : dec_less(o, best)) || (eq && op_ < pbest))) {
      has = true;
      best = o;
      pbest = op_;
    }
  }
  *out = best;
  return any;
}

// a Decimal op's result into the output row.  A compact sum (P <= 18): as put.  Out of line: the 16 bytes at the row's
// own offset zeroed, the minimal bytes written there and the slot (offset << 32) | length; null: the slot offset << 32
// (UnsafeRow.setDecimal keeps the offset for a later update) and the null bit.
__device__ __forceinline__ void put_decimal(uint8_t* row, uint32_t op, uint32_t off, uint32_t a, bool has, Dec128 x,
                                            uint32_t* null_mask) {
  if (!agg_decimal_wide(op)) {
    put(row, op, off, a, has, x.lo, null_mask);
    return;
  }
  uint64_t slot, unused;
  ld_span16<false>(row + off, 8, slot, unused);
  const uint32_t so = (uint32_t)(slot >> 32);
  uint64_t m0 = 0, m1 = 0;
  uint32_t len = 0;
  if (has) {
    len = dec_bytes(x);
    dec_encode(x, len, &m0, &m1);
  }
  st_span16(row + so, 16, m0, m1);
  st_span16(row + off, 8, ((uint64_t)so << 32) | len, 0);
  if (!has) *null_mask |= 1u << a;
}

__device__ __forceinline__ bool is_decimal(uint32_t op) { return agg_base_op(op) >= B2S_AGG_SUM_DECIMAL; }

// agg_merge_small_kernel for a spec with a Decimal op
__global__ void __launch_bounds__(kAggThreads) agg_merge_small_dec_kernel(
    const uint32_t* __restrict__ gpos, uint64_t G, uint64_t n, const uint64_t* __restrict__ vals,
    const uint64_t* __restrict__ vhi, const uint32_t* __restrict__ nulls, const AggSpec* __restrict__ spec,
    uint32_t n_aggs, const uint64_t* __restrict__ gdst, uint8_t* __restrict__ dst) {
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < G; g += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t s = gpos[g], e = gpos[g + 1];
    if (e - s > kSmallGroup) continue;
    uint8_t* row = dst + gdst[g] + 4;
    uint32_t null_mask = 0;
    for (uint32_t a = 0; a < n_aggs; a++) {
      const uint32_t op = spec->op[a];
      if (is_decimal(op)) {
        Dec128 x;
        const bool has = merge_thread_dec(op, a, spec->wide[a], vals, vhi, nulls, n, s, e, &x);
        put_decimal(row, op, spec->off[a], a, has, x, &null_mask);
      } else {
        uint64_t v;
        const bool has = merge_thread(op, a, vals, nulls, n, s, e, &v);
        put(row, op, spec->off[a], a, has, v, &null_mask);
      }
    }
    put_null_bits(row, spec, n_aggs, null_mask);
  }
}

// agg_merge_large_kernel for a spec with a Decimal op
__global__ void __launch_bounds__(kAggThreads) agg_merge_large_dec_kernel(
    const uint32_t* __restrict__ gpos, uint64_t G, uint64_t n, const uint64_t* __restrict__ vals,
    const uint64_t* __restrict__ vhi, const uint32_t* __restrict__ nulls, const AggSpec* __restrict__ spec,
    uint32_t n_aggs, const uint64_t* __restrict__ gdst, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (kAggThreads / 32);
  for (uint64_t g = (uint64_t)blockIdx.x * (kAggThreads / 32) + (threadIdx.x >> 5); g < G; g += warps) {
    const uint32_t s = gpos[g], e = gpos[g + 1];
    if (e - s <= kSmallGroup) continue;  // uniform over the warp
    uint8_t* row = dst + gdst[g] + 4;
    uint32_t null_mask = 0;
    for (uint32_t a = 0; a < n_aggs; a++) {
      const uint32_t op = spec->op[a];
      if (is_decimal(op)) {
        Dec128 x;
        const bool has = merge_warp_dec(op, a, spec->wide[a], vals, vhi, nulls, n, s, e, lane, &x);
        if (lane == 0) put_decimal(row, op, spec->off[a], a, has, x, &null_mask);
      } else {
        uint64_t v;
        const bool has = merge_warp(op, a, vals, nulls, n, s, e, lane, &v);
        if (lane == 0) put(row, op, spec->off[a], a, has, v, &null_mask);
      }
    }
    if (lane == 0) put_null_bits(row, spec, n_aggs, null_mask);
  }
}

// ---- the variance ----
// one mergeExpressions step of CentralMomentAgg (order 2): (n1, avg1, m2a) merged with (n2, avg2, m2b), every operation
// one double operation rounded to nearest, in Spark's order
__device__ __forceinline__ void var_merge(double& n1, double& avg1, double& m2a, double n2, double avg2, double m2b) {
  const double newN = __dadd_rn(n1, n2);
  const double delta = __dsub_rn(avg2, avg1);
  const double deltaN = newN == 0.0 ? 0.0 : __ddiv_rn(delta, newN);
  avg1 = __dadd_rn(avg1, __dmul_rn(deltaN, n2));
  m2a = __dadd_rn(__dadd_rn(m2a, m2b), __dmul_rn(__dmul_rn(__dmul_rn(delta, deltaN), n1), n2));
  n1 = newN;
}

__device__ __forceinline__ double dbl(uint64_t b) { return __longlong_as_double((long long)b); }
__device__ __forceinline__ uint64_t bits(double x) { return (uint64_t)__double_as_longlong(x); }

// variance entry a (v: its index among them) of the records at positions [s, e), by one thread, from (0, 0, 0)
__device__ __forceinline__ void merge_thread_var(uint32_t a, uint32_t v, const uint64_t* __restrict__ vals,
                                                 const uint64_t* __restrict__ vmom, uint64_t n, uint32_t s,
                                                 uint32_t e, double r[3]) {
  const uint64_t *vn = vals + (size_t)a * n, *va = vmom + (size_t)(2 * v) * n, *vm = va + n;
  double n1 = 0.0, avg = 0.0, m2 = 0.0;
  for (uint32_t j = s; j < e; j++) var_merge(n1, avg, m2, dbl(__ldg(vn + j)), dbl(__ldg(va + j)), dbl(__ldg(vm + j)));
  r[0] = n1;
  r[1] = avg;
  r[2] = m2;
}

// merge_thread_var by the whole warp (every lane returns the result): four rounds of 32 triples loaded in parallel,
// then each lane's triple broadcast in record order into the one chain
__device__ __forceinline__ void merge_warp_var(uint32_t a, uint32_t v, const uint64_t* __restrict__ vals,
                                               const uint64_t* __restrict__ vmom, uint64_t n, uint32_t s, uint32_t e,
                                               uint32_t lane, double r[3]) {
  const uint64_t *vn = vals + (size_t)a * n, *va = vmom + (size_t)(2 * v) * n, *vm = va + n;
  double n1 = 0.0, avg = 0.0, m2 = 0.0;
  for (uint32_t b = s; b < e; b += 128) {
    uint64_t x[4][3];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const uint32_t j = b + 32 * q + lane;
      const bool in = j < e;
      x[q][0] = in ? __ldg(vn + j) : 0;
      x[q][1] = in ? __ldg(va + j) : 0;
      x[q][2] = in ? __ldg(vm + j) : 0;
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const uint32_t m = min(32u, e - min(e, b + 32 * q));
      for (uint32_t l = 0; l < m; l++) {
        const double n2 = dbl(__shfl_sync(FULL, x[q][0], l)), a2 = dbl(__shfl_sync(FULL, x[q][1], l)),
                     m2b = dbl(__shfl_sync(FULL, x[q][2], l));
        var_merge(n1, avg, m2, n2, a2, m2b);
      }
    }
  }
  r[0] = n1;
  r[1] = avg;
  r[2] = m2;
}

// a variance entry's three slots (never null)
__device__ __forceinline__ void put_var(uint8_t* row, uint32_t off, const double r[3]) {
  st_span16(row + off, 16, bits(r[0]), bits(r[1]));
  st_span16(row + off + 16, 8, bits(r[2]), 0);
}

// agg_merge_small_kernel for a spec with a variance entry (and any other op)
__global__ void __launch_bounds__(kAggThreads) agg_merge_small_var_kernel(
    const uint32_t* __restrict__ gpos, uint64_t G, uint64_t n, const uint64_t* __restrict__ vals,
    const uint64_t* __restrict__ vhi, const uint64_t* __restrict__ vmom, const uint32_t* __restrict__ nulls,
    const AggSpec* __restrict__ spec, uint32_t n_aggs, const uint64_t* __restrict__ gdst, uint8_t* __restrict__ dst) {
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < G; g += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t s = gpos[g], e = gpos[g + 1];
    if (e - s > kSmallGroup) continue;
    uint8_t* row = dst + gdst[g] + 4;
    uint32_t null_mask = 0;
    for (uint32_t a = 0; a < n_aggs; a++) {
      const uint32_t op = spec->op[a];
      if (op == B2S_AGG_VARIANCE) {
        double r[3];
        merge_thread_var(a, spec->var[a], vals, vmom, n, s, e, r);
        put_var(row, spec->off[a], r);
      } else if (agg_decimal_op(op)) {
        Dec128 x;
        const bool has = merge_thread_dec(op, a, spec->wide[a], vals, vhi, nulls, n, s, e, &x);
        put_decimal(row, op, spec->off[a], a, has, x, &null_mask);
      } else {
        uint64_t v;
        const bool has = merge_thread(op, a, vals, nulls, n, s, e, &v);
        put(row, op, spec->off[a], a, has, v, &null_mask);
      }
    }
    put_null_bits(row, spec, n_aggs, null_mask);
  }
}

// agg_merge_large_kernel for a spec with a variance entry (and any other op)
__global__ void __launch_bounds__(kAggThreads) agg_merge_large_var_kernel(
    const uint32_t* __restrict__ gpos, uint64_t G, uint64_t n, const uint64_t* __restrict__ vals,
    const uint64_t* __restrict__ vhi, const uint64_t* __restrict__ vmom, const uint32_t* __restrict__ nulls,
    const AggSpec* __restrict__ spec, uint32_t n_aggs, const uint64_t* __restrict__ gdst, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (kAggThreads / 32);
  for (uint64_t g = (uint64_t)blockIdx.x * (kAggThreads / 32) + (threadIdx.x >> 5); g < G; g += warps) {
    const uint32_t s = gpos[g], e = gpos[g + 1];
    if (e - s <= kSmallGroup) continue;  // uniform over the warp
    uint8_t* row = dst + gdst[g] + 4;
    uint32_t null_mask = 0;
    for (uint32_t a = 0; a < n_aggs; a++) {
      const uint32_t op = spec->op[a];
      if (op == B2S_AGG_VARIANCE) {
        double r[3];
        merge_warp_var(a, spec->var[a], vals, vmom, n, s, e, lane, r);
        if (lane == 0) put_var(row, spec->off[a], r);
      } else if (agg_decimal_op(op)) {
        Dec128 x;
        const bool has = merge_warp_dec(op, a, spec->wide[a], vals, vhi, nulls, n, s, e, lane, &x);
        if (lane == 0) put_decimal(row, op, spec->off[a], a, has, x, &null_mask);
      } else {
        uint64_t v;
        const bool has = merge_warp(op, a, vals, nulls, n, s, e, lane, &v);
        if (lane == 0) put(row, op, spec->off[a], a, has, v, &null_mask);
      }
    }
    if (lane == 0) put_null_bits(row, spec, n_aggs, null_mask);
  }
}

}  // namespace

size_t rows_aggregate_ws_bytes(uint64_t n, uint32_t n_aggs, uint32_t n_wide, uint32_t n_var) {
  return a256(n * 8) + a256(24) + 3 * a256(n * 4) + a256((n + 1) * 4) + a256(n * n_aggs * 8) + a256(n * n_wide * 8) +
         a256(sizeof(AggSpec)) + a256(n * n_var * 16);
}

uint64_t* rows_aggregate_readback(uint8_t* d_aws, uint64_t n, uint32_t n_aggs, uint32_t n_wide) {
  return carve_agg_ws(d_aws, n, n_aggs, n_wide).readback;
}

const uint64_t* rows_group_heads_before(uint8_t* d_aws, uint64_t n) { return carve_agg_ws(d_aws, n, 0, 0).head; }
const uint32_t* rows_group_starts(uint8_t* d_aws, uint64_t n) { return carve_agg_ws(d_aws, n, 0, 0).gpos; }
const uint32_t* rows_group_lengths(uint8_t* d_aws, uint64_t n) { return carve_agg_ws(d_aws, n, 0, 0).glen; }

void launch_rows_group(const uint8_t* arena, uint64_t n, const uint32_t* idx, const uint32_t* heads,
                       uint32_t key_bytes, const AggSpec& spec, uint8_t* d_ws, uint8_t* d_aws, cudaStream_t st,
                       uint64_t* launches) {
  const AggWs a = carve_agg_ws(d_aws, n, spec.n, spec.n_wide, spec.n_var);
  if (!n) {
    cudaMemsetAsync(a.readback, 0, 16, st);
    return;
  }
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  uint64_t* scan_ws = (uint64_t*)(d_ws + key_sort_ws_bytes(n, key_bytes));
  cudaMemcpyAsync(a.spec, &spec, sizeof(AggSpec), cudaMemcpyHostToDevice, st);
  if (spec.n_var) {
    if (spec.n_wide) cudaMemsetAsync(a.readback + 2, 0xff, 8, st);
    auto heads_var = spec.n_wide ? agg_heads_var_kernel<true> : agg_heads_var_kernel<false>;
    heads_var<<<grid_for(n), kAggThreads, 0, st>>>(arena, w.src_off, w.len, idx, n, w.words, (key_bytes + 3) / 4, heads,
                                                   a.spec, a.head, a.nulls, a.vals, a.vhi, a.vmom,
                                                   (unsigned long long*)(a.readback + 2));
  } else if (spec.n_wide) {
    cudaMemsetAsync(a.readback + 2, 0xff, 8, st);
    agg_heads_kernel<true><<<grid_for(n), kAggThreads, 0, st>>>(
        arena, w.src_off, w.len, idx, n, w.words, (key_bytes + 3) / 4, heads, a.spec, a.head, a.nulls, a.vals, a.vhi,
        (unsigned long long*)(a.readback + 2));
  } else {
    agg_heads_kernel<false><<<grid_for(n), kAggThreads, 0, st>>>(arena, w.src_off, w.len, idx, n, w.words,
                                                                 (key_bytes + 3) / 4, heads, a.spec, a.head, a.nulls,
                                                                 a.vals, nullptr, nullptr);
  }
  launch_exclusive_scan_u64(a.head, n, a.readback, scan_ws, st, launches);
  agg_compact_kernel<<<grid_for(n), kAggThreads, 0, st>>>(a.head, a.readback, idx, w.len, n, a.hidx, a.gpos, a.glen);
  // the group lengths are already in group order: no index
  launch_sorted_offsets(nullptr, a.glen, n, w.sdst, a.readback + 1, scan_ws, st, launches);
  if (launches) *launches += 2;
}

void launch_rows_aggregate(const uint8_t* arena, uint64_t n, uint64_t groups, uint32_t key_bytes, const AggSpec& spec,
                           uint8_t* d_ws, uint8_t* d_aws, uint8_t* d_dst, cudaStream_t st, uint64_t* launches) {
  if (!groups) return;
  const uint32_t n_aggs = spec.n;
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  const AggWs a = carve_agg_ws(d_aws, n, n_aggs, spec.n_wide, spec.n_var);
  PartitionPlan plan;
  plan.src_off = w.src_off;
  plan.sdst = w.sdst;
  plan.idx = a.hidx;
  launch_partition_gather(arena, w.len, groups, plan, d_dst, st, launches);
  if (!n_aggs) return;
  const uint64_t ctas = (groups + kAggThreads / 32 - 1) / (kAggThreads / 32);
  const unsigned large_grid = (unsigned)std::min<uint64_t>(ctas, (uint64_t)kSMs * 16);
  if (spec.n_var) {
    agg_merge_small_var_kernel<<<grid_for(groups), kAggThreads, 0, st>>>(a.gpos, groups, n, a.vals, a.vhi, a.vmom,
                                                                          a.nulls, a.spec, n_aggs, w.sdst, d_dst);
    agg_merge_large_var_kernel<<<large_grid, kAggThreads, 0, st>>>(a.gpos, groups, n, a.vals, a.vhi, a.vmom, a.nulls,
                                                                   a.spec, n_aggs, w.sdst, d_dst);
  } else if (spec.decimal) {
    agg_merge_small_dec_kernel<<<grid_for(groups), kAggThreads, 0, st>>>(a.gpos, groups, n, a.vals, a.vhi, a.nulls,
                                                                          a.spec, n_aggs, w.sdst, d_dst);
    agg_merge_large_dec_kernel<<<large_grid, kAggThreads, 0, st>>>(a.gpos, groups, n, a.vals, a.vhi, a.nulls, a.spec,
                                                                   n_aggs, w.sdst, d_dst);
  } else {
    agg_merge_small_kernel<<<grid_for(groups), kAggThreads, 0, st>>>(a.gpos, groups, n, a.vals, a.nulls, a.spec,
                                                                      n_aggs, w.sdst, d_dst);
    agg_merge_large_kernel<<<large_grid, kAggThreads, 0, st>>>(a.gpos, groups, n, a.vals, a.nulls, a.spec, n_aggs,
                                                               w.sdst, d_dst);
  }
  if (launches) *launches += 2;
}

}  // namespace b2s
