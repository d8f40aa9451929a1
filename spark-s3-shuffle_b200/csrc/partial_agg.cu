// partial_agg.cu — a map task's partial aggregation (Spark SQL's HashAggregateExec(Partial) under a hash exchange):
// its UnsafeRow records grouped by the key and Spark's aggregation buffers folded over each group, one partial row per
// key written as UnsafeProjection(groupingAttributes ++ aggBufferAttributes) writes it.  The records are the caller's
// ([size: int32 big-endian][row] back to back, rec_len each); the key sort and the grouping are rows.cu's and
// aggregate.cu's (launch_rows_order, the refinement rounds, launch_rows_group).  All on the device:
//   offsets : rec_len scanned into the sort workspace's record offsets and lengths, as launch_rows_emit leaves them
//   check   : a thread per record: every value slot, value null word and out-of-line decimal input inside its row
//             (the key columns are checked by launch_rows_hash); the lowest bad record lowers one verdict word
//   stage   : a thread per sorted position: each buffer's input as the reduce side's merge op reads it (vals[k n + j],
//             a decimal's high word in vhi, nulls[j] bit k for a null); a null decimal or AVG input is a present 0, a
//             COUNT or isEmpty input a present 0 / 1, a null double input a +0.0 (its sum chain starts at +0.0, so the
//             accumulator is never -0.0 and adding +0.0 leaves it as it is)
//   fold    : groups of up to kSmallGroup records a thread each; up to kChunk records a warp each; larger groups over
//             the grid: a warp per aligned chunk of kChunk positions folds the (at most two) large groups it meets into
//             a partial, and a warp per large group combines its chunks' partials.  Sums of integers and decimals are
//             exact and so in any order; min / max keep the earliest position among equal values, so they too.  A
//             double sum is one add chain per group in position order: a warp stages 256 values in shared memory and
//             its lane 0 adds them, the next tile's loads in flight meanwhile.  A variance (CentralMomentAgg's
//             [n, avg, m2]) is one update chain per group in position order the same way; it is not associative, so
//             the warp, chunk and combine folds skip it, as they skip the double sums.
//   size    : a thread per group: its partial row's length, scanned into the output offsets (the last scan total is the
//             output bytes, read back with the group count)
//   emit    : a warp per partial row, lane f writing field f (n_keys + fields <= 32, so one null word; a variance
//             buffer is three fields)
// The distinct aggregation's step (a spec with merge entries, the kernels' Merge instantiations) runs the same steps
// over a reducer's merged rows, already in the key's order: no sort, the group heads where the key's encoding changes
// (pa_heads_kernel).  Its merge entries (a decimal sum's or a variance's mergeExpressions) are chains in position
// order, as the double sums are: a thread per small group, else pa_var_merge_kernel (a chain over shared-memory tiles)
// or pa_dec_merge_kernel (a CTA's warps scan segments and check every prefix sum); the other merges are the update folds over the
// buffer, which give the same bits.
#include <algorithm>

#include "decimal128.h"
#include "kernels.h"
#include "rows_key.cuh"

namespace b2s {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kPaThreads = 256;
constexpr uint32_t kSmallGroup = 32;
constexpr uint32_t kChunk = 2048;
constexpr uint32_t kTile = 256;  // the double chain's values per shared-memory tile

inline size_t a256(size_t b) { return (b + 255) / 256 * 256; }

inline unsigned grid_for(uint64_t n) {
  const uint64_t want = (n + kPaThreads - 1) / kPaThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

inline unsigned warp_grid_for(uint64_t warps) {
  const uint64_t want = (warps + kPaThreads / 32 - 1) / (kPaThreads / 32);
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

// one buffer's fold so far: (lo, hi) its value (hi: a decimal's high word), pos the position it came from (min / max)
struct PAcc {
  uint64_t lo, hi;
  uint32_t pos, has;
};

// the workspace (partial_agg_ws_bytes): header [check verdict, record bytes, check detail, range 0 (= 0), groups,
// output bytes], staged values, decimal high words, null bits, the folded buffers (per group; a variance's avg and m2
// in rmom), the chunk partials, the partial rows' lengths and offsets and the offsets' scan workspace
struct PaWs {
  uint64_t* hdr;
  uint64_t* vals;
  uint64_t* vhi;
  uint32_t* nulls;
  uint64_t* rlo;
  uint64_t* rhi;
  uint32_t* rnull;
  uint64_t* rmom;
  PAcc* part;
  uint32_t* rowlen;
  uint64_t* rowoff;
  uint64_t* scan_ws;
};

__host__ __device__ inline uint64_t n_chunks(uint64_t n) { return (n + kChunk - 1) / kChunk; }

PaWs carve_pa_ws(uint8_t* d, uint64_t n, const PartialAggSpec& s) {
  PaWs w;
  uint8_t* p = d;
  w.hdr = (uint64_t*)p;    p += 256;
  w.vals = (uint64_t*)p;   p += a256(n * s.n_bufs * 8);
  w.vhi = (uint64_t*)p;    p += a256(n * s.n_dec * 8);
  w.nulls = (uint32_t*)p;  p += a256(n * 4);
  w.rlo = (uint64_t*)p;    p += a256(n * s.n_bufs * 8);
  w.rhi = (uint64_t*)p;    p += a256(n * s.n_dec * 8);
  w.rnull = (uint32_t*)p;  p += a256(n * 4);
  w.rmom = (uint64_t*)p;   p += a256(n * s.n_var * 16);
  w.part = (PAcc*)p;       p += a256(n_chunks(n) * 2 * s.n_bufs * sizeof(PAcc));
  w.rowlen = (uint32_t*)p; p += a256(n * 4);
  w.rowoff = (uint64_t*)p; p += a256(n * 8);
  w.scan_ws = (uint64_t*)p;
  return w;
}

__device__ __forceinline__ bool bit_at(const uint8_t* row, int32_t f) {
  uint64_t w, unused;
  ld_span16<true>(row + 8 * (uint32_t)(f >> 6), 8, w, unused);
  return (w >> (f & 63)) & 1;
}

__device__ __forceinline__ uint32_t vkind(uint32_t vt) { return vt & 0xff; }
__device__ __forceinline__ bool wide_input(uint32_t vt) {
  return vkind(vt) == B2S_WINDOW_VAL_DECIMAL && ((vt >> 8) & 0xff) > 18;
}
// the buffer's input is read from its slot (COUNT reads only its null bit)
__device__ __forceinline__ bool reads_value(uint32_t stage) { return stage != kStageCount && stage != kStageIsEmpty; }

__device__ __forceinline__ uint32_t row_size_at(const uint8_t* rec, uint64_t o) {
  uint64_t lo, hi;
  ld_span16<true>(rec + o, 4, lo, hi);
  return __byte_perm((uint32_t)lo, 0, 0x0123);
}

// rec_len into the sort workspace: len[i] = rec_len[i], off[i] = rec_len[i] (scanned in place after)
__global__ void __launch_bounds__(kPaThreads) pa_offsets_kernel(const uint32_t* __restrict__ rec_len, uint64_t n,
                                                                uint32_t* __restrict__ len, uint64_t* __restrict__ off) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t l = rec_len[i];
    len[i] = l;
    off[i] = l;
  }
}

// Record i's value slots, value null words and out-of-line decimal inputs inside its row.  A record that is not a
// framed row or ends past rec_bytes is launch_rows_hash's to report, so it is not read here.  A bad one lowers *bad to
// (i << 3) | kPaBadValue and *detail to (i << 2) | its first failing check (kPaBad*).
__global__ void __launch_bounds__(kPaThreads) pa_check_kernel(const uint8_t* __restrict__ rec, uint64_t rec_bytes,
                                                              const uint64_t* __restrict__ rec_off,
                                                              const uint32_t* __restrict__ rec_len, uint64_t n,
                                                              const __grid_constant__ PartialAggSpec s,
                                                              unsigned long long* __restrict__ bad,
                                                              unsigned long long* __restrict__ detail) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t o = rec_off[i];
    const uint32_t len = rec_len[i];
    if (len < 4 || o + len > rec_bytes) continue;
    const uint32_t size = row_size_at(rec, o);
    if (size != len - 4) continue;
    const uint8_t* row = rec + o + 4;
    uint64_t why = 0;
    for (uint32_t k = 0; k < s.n_bufs && !why; k++) {
      const uint32_t vt = s.vtype[k];
      if (vkind(vt) == B2S_WINDOW_VAL_NONE) continue;
      const int32_t nf = s.vnull[k];
      if (nf >= 0 && 8ull * (uint32_t)(nf >> 6) + 8 > size) {
        why = kPaBadNull;
        break;
      }
      if (!reads_value(s.stage[k])) continue;
      if ((uint64_t)s.voff[k] + 8 > size) {
        why = kPaBadSlot;
        break;
      }
      if (wide_input(vt) && !(nf >= 0 && bit_at(row, nf))) {
        uint64_t slot, unused;
        ld_span16<true>(row + s.voff[k], 8, slot, unused);
        const uint32_t so = (uint32_t)(slot >> 32), sz = (uint32_t)slot;
        if (sz - 1 >= 16u || (uint64_t)so + sz > size) why = kPaBadDecimal;
      }
    }
    if (why) {
      atomicMin(bad, (unsigned long long)((i << 3) | kPaBadValue));
      atomicMin(detail, (unsigned long long)((i << 2) | why));
    }
  }
}

// buffer k's staged input from a checked row: (lo, hi) and whether it is null (then (0, 0))
__device__ __forceinline__ bool stage_one(const uint8_t* row, uint32_t size, const PartialAggSpec& s, uint32_t k,
                                          uint32_t st, uint64_t& lo, uint64_t& hi) {
  const uint32_t vt = s.vtype[k], kind = vkind(vt);
  const bool null = kind != B2S_WINDOW_VAL_NONE && s.vnull[k] >= 0 && bit_at(row, s.vnull[k]);
  lo = hi = 0;
  if (st == kStageCount) {
    lo = null ? 0 : 1;
    return false;
  }
  if (st == kStageIsEmpty) {
    lo = null ? 1 : 0;
    return false;
  }
  if (null) return st == kStageValue;  // a null SUM / MIN / MAX input is skipped; a null sum-or-zero input is 0
  uint64_t v, unused;
  ld_span16<true>(row + s.voff[k], 8, v, unused);
  switch (kind) {
    case B2S_WINDOW_VAL_INT8: v = (uint64_t)(int64_t)(int8_t)v; break;
    case B2S_WINDOW_VAL_INT16: v = (uint64_t)(int64_t)(int16_t)v; break;
    case B2S_WINDOW_VAL_INT32: v = (uint64_t)(int64_t)(int32_t)v; break;
    case B2S_WINDOW_VAL_FLOAT32: v = (uint64_t)__double_as_longlong((double)__int_as_float((int)(uint32_t)v)); break;
    default: break;
  }
  if (kind == B2S_WINDOW_VAL_DECIMAL) {
    if (wide_input(vt)) {
      bool bad = false;
      decimal_bits(row, size, v, hi, lo, &bad);
      hi ^= 1ull << 63;  // decimal_bits flips the sign bit for the sort
    } else {
      lo = v;
      hi = (uint64_t)((int64_t)v >> 63);
    }
    return false;
  }
  if (s.to_double[k] && kind <= B2S_WINDOW_VAL_INT64) v = (uint64_t)__double_as_longlong(__ll2double_rn((long long)v));
  lo = v;
  return false;
}

// Merge (a spec with merge entries: the distinct aggregation's step over merged rows): kStageCountAll stages 1 when no
// bit of the mask voff[k] is set in the row's null word; kStageMerge stages a decimal sum buffer as kStageValue does, and
// a variance buffer's n into vals and its avg and m2 into vhi words wide[k] and wide[k] + 1
template <bool Merge>
__global__ void __launch_bounds__(kPaThreads) pa_stage_kernel(const uint8_t* __restrict__ rec,
                                                              const uint64_t* __restrict__ rec_off,
                                                              const uint32_t* __restrict__ rec_len,
                                                              const uint32_t* __restrict__ idx, uint64_t n,
                                                              const __grid_constant__ PartialAggSpec s,
                                                              uint64_t* __restrict__ vals, uint64_t* __restrict__ vhi,
                                                              uint32_t* __restrict__ nulls) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = idx ? idx[j] : (uint32_t)j;
    const uint8_t* row = rec + rec_off[i] + 4;
    const uint32_t size = rec_len[i] - 4;
    uint32_t nm = 0;
    for (uint32_t k = 0; k < s.n_bufs; k++) {
      uint64_t lo, hi;
      const uint32_t st = s.stage[k];
      if (Merge && st == kStageCountAll) {
        uint64_t w, unused;
        ld_span16<true>(row, 8, w, unused);
        vals[(size_t)k * n + j] = (w & s.voff[k]) ? 0 : 1;
        continue;
      }
      if (Merge && st == kStageMerge && s.op[k] == B2S_AGG_VARIANCE) {
        uint64_t cn, avg, m2, unused;
        ld_span16<true>(row + s.voff[k], 8, cn, unused);
        ld_span16<true>(row + s.voff[k] + 8, 16, avg, m2);
        vals[(size_t)k * n + j] = cn;
        vhi[(size_t)s.wide[k] * n + j] = avg;
        vhi[(size_t)(s.wide[k] + 1) * n + j] = m2;
        continue;
      }
      if (stage_one(row, size, s, k, Merge && st == kStageMerge ? kStageValue : st, lo, hi)) nm |= 1u << k;
      vals[(size_t)k * n + j] = lo;
      if (agg_decimal_op(s.op[k])) vhi[(size_t)s.wide[k] * n + j] = hi;
    }
    nulls[j] = nm;
  }
}

// ---- the associative folds ----
__device__ __forceinline__ bool is_sum(uint32_t op) {
  return op == B2S_AGG_SUM_INT64 || agg_base_op(op) == B2S_AGG_SUM_DECIMAL;
}
__device__ __forceinline__ bool is_max_op(uint32_t op) {
  return op == B2S_AGG_MAX_INT32 || op == B2S_AGG_MAX_INT64 || op == B2S_AGG_MAX_FLOAT64 ||
         op == B2S_AGG_MAX_DECIMAL;
}
// a min / max value's order as an unsigned 128-bit key (larger key = larger value): Spark SQL's double order (-0.0 ==
// 0.0, every NaN equal and above +inf), signed integers and decimals
__device__ __forceinline__ void order_of(uint32_t op, uint64_t lo, uint64_t hi, uint64_t& khi, uint64_t& klo) {
  klo = 0;
  if (op == B2S_AGG_MIN_INT32 || op == B2S_AGG_MAX_INT32) {
    khi = (uint32_t)lo ^ 0x80000000u;
  } else if (op == B2S_AGG_MIN_INT64 || op == B2S_AGG_MAX_INT64) {
    khi = lo ^ (1ull << 63);
  } else if (op == B2S_AGG_MIN_FLOAT64 || op == B2S_AGG_MAX_FLOAT64) {
    uint64_t b = lo;
    if ((b & ~(1ull << 63)) > 0x7ff0000000000000ull) b = ~0ull;
    else {
      if (b == (1ull << 63)) b = 0;
      b = (b >> 63) ? ~b : (b | (1ull << 63));
    }
    khi = b;
  } else {
    khi = hi ^ (1ull << 63);
    klo = lo;
  }
}

// a folded with b (either order): a sum adds, a min / max keeps the better value, the earlier position among equal ones
__device__ __forceinline__ PAcc combine(uint32_t op, PAcc a, PAcc b) {
  if (!b.has) return a;
  if (!a.has) return b;
  if (is_sum(op)) {
    PAcc r;
    r.lo = a.lo + b.lo;
    r.hi = a.hi + b.hi + (r.lo < a.lo ? 1 : 0);
    r.pos = 0;
    r.has = 1;
    return r;
  }
  uint64_t ah, al, bh, bl;
  order_of(op, a.lo, a.hi, ah, al);
  order_of(op, b.lo, b.hi, bh, bl);
  const bool mx = is_max_op(op);
  const bool b_better = mx ? (bh > ah || (bh == ah && bl > al)) : (bh < ah || (bh == ah && bl < al));
  const bool eq = ah == bh && al == bl;
  return b_better || (eq && b.pos < a.pos) ? b : a;
}

__device__ __forceinline__ PAcc load_acc(const PartialAggSpec& s, uint32_t k, const uint64_t* __restrict__ vals,
                                         const uint64_t* __restrict__ vhi, const uint32_t* __restrict__ nulls,
                                         uint64_t n, uint32_t j) {
  PAcc x;
  x.has = !((__ldg(nulls + j) >> k) & 1);
  x.lo = x.has ? __ldg(vals + (size_t)k * n + j) : 0;
  x.hi = x.has && agg_decimal_op(s.op[k]) ? __ldg(vhi + (size_t)s.wide[k] * n + j) : 0;
  x.pos = j;
  return x;
}

__device__ __forceinline__ PAcc shfl_acc(PAcc a, int d) {
  PAcc o;
  o.lo = __shfl_xor_sync(FULL, a.lo, d);
  o.hi = __shfl_xor_sync(FULL, a.hi, d);
  o.pos = __shfl_xor_sync(FULL, a.pos, d);
  o.has = __shfl_xor_sync(FULL, a.has, d);
  return o;
}

__device__ __forceinline__ PAcc warp_reduce(uint32_t op, PAcc a) {
#pragma unroll
  for (int d = 16; d; d >>= 1) a = combine(op, a, shfl_acc(a, d));
  return a;
}

// buffer k over positions [s0, e0) by the whole warp (every lane returns the fold); not a double sum
__device__ __forceinline__ PAcc fold_warp(const PartialAggSpec& s, uint32_t k, const uint64_t* __restrict__ vals,
                                          const uint64_t* __restrict__ vhi, const uint32_t* __restrict__ nulls,
                                          uint64_t n, uint32_t s0, uint32_t e0, uint32_t lane) {
  const uint32_t op = s.op[k];
  PAcc acc{0, 0, 0, 0};
  for (uint32_t b = s0; b < e0; b += 128) {
    PAcc x[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const uint32_t j = b + 32 * r + lane;
      x[r] = j < e0 ? load_acc(s, k, vals, vhi, nulls, n, j) : PAcc{0, 0, 0, 0};
    }
#pragma unroll
    for (int r = 0; r < 4; r++) acc = combine(op, acc, x[r]);
  }
  return warp_reduce(op, acc);
}

__device__ __forceinline__ bool dsum_op(uint32_t op) { return op == B2S_AGG_SUM_FLOAT64; }
// a buffer folded by one chain in position order (pa_chain_kernel's), not by the associative folds
__device__ __forceinline__ bool chain_op(uint32_t op) { return op == B2S_AGG_SUM_FLOAT64 || op == B2S_AGG_VARIANCE; }

// a buffer the associative folds and the update chains skip: a chain's, or (Merge) a merge entry (pa_var_merge_kernel, pa_dec_merge_kernel)
template <bool Merge>
__device__ __forceinline__ bool skips(const PartialAggSpec& s, uint32_t k) {
  return chain_op(s.op[k]) || (Merge && s.stage[k] == kStageMerge);
}

__device__ __forceinline__ double dbl(uint64_t b) { return __longlong_as_double((long long)b); }
__device__ __forceinline__ uint64_t bits(double x) { return (uint64_t)__double_as_longlong(x); }

// one updateExpressions step of CentralMomentAgg (order 2) with the non-null input x, every operation one double
// operation rounded to nearest, in Spark's order
__device__ __forceinline__ void var_update(double& cn, double& avg, double& m2, double x) {
  const double newN = __dadd_rn(cn, 1.0);
  const double delta = __dsub_rn(x, avg);
  const double deltaN = __ddiv_rn(delta, newN);
  avg = __dadd_rn(avg, deltaN);
  m2 = __dadd_rn(m2, __dmul_rn(delta, __dsub_rn(delta, deltaN)));
  cn = newN;
}

// one mergeExpressions step of CentralMomentAgg (order 2): the group's buffer (cn, avg, m2) merged with (n2, avg2, m2b),
// every operation one double operation rounded to nearest, in Spark's order
__device__ __forceinline__ void var_merge(double& cn, double& avg, double& m2, double n2, double avg2, double m2b) {
  const double newN = __dadd_rn(cn, n2);
  const double delta = __dsub_rn(avg2, avg);
  const double deltaN = newN == 0.0 ? 0.0 : __ddiv_rn(delta, newN);
  const double n1 = cn;
  avg = __dadd_rn(avg, __dmul_rn(deltaN, n2));
  m2 = __dadd_rn(__dadd_rn(m2, m2b), __dmul_rn(__dmul_rn(__dmul_rn(delta, deltaN), n1), n2));
  cn = newN;
}

// one step of a decimal sum's merge (Sum / Average mergeExpressions into a decimal(P) buffer): a null input, or a sum
// reaching 10^P, makes the result null for good (*gone)
__device__ __forceinline__ void dec_merge(Dec128& acc, bool& gone, bool null, Dec128 v, uint32_t P) {
  if (gone) return;
  bool ovf = false;
  acc = dec_add(acc, v, &ovf);
  gone = null || ovf || !dec_fits(acc, P);
}

// a variance buffer's fold of group g: n into rlo, avg and m2 into rmom
__device__ __forceinline__ void put_var(const PartialAggSpec& s, uint32_t k, uint64_t g, uint64_t n, double cn,
                                        double avg, double m2, uint64_t* __restrict__ rlo,
                                        uint64_t* __restrict__ rmom) {
  rlo[(size_t)k * n + g] = bits(cn);
  rmom[(size_t)(2 * s.var[k]) * n + g] = bits(avg);
  rmom[(size_t)(2 * s.var[k] + 1) * n + g] = bits(m2);
}

__device__ __forceinline__ void put_result(const PartialAggSpec& s, uint32_t k, uint64_t g, uint64_t n, PAcc r,
                                           uint64_t* __restrict__ rlo, uint64_t* __restrict__ rhi) {
  rlo[(size_t)k * n + g] = r.lo;
  if (agg_decimal_op(s.op[k])) rhi[(size_t)s.wide[k] * n + g] = r.hi;
}

// the group of sorted position j, from the heads-before scan of launch_rows_group
__device__ __forceinline__ uint64_t group_of(const uint64_t* __restrict__ hb, uint64_t n, uint64_t G, uint64_t j) {
  return (j + 1 < n ? hb[j + 1] : G) - 1;
}

// groups of up to kSmallGroup records: a thread each, every buffer in position order (the chains included; Merge:
// the merge entries' chains too)
template <bool Merge>
__global__ void __launch_bounds__(kPaThreads) pa_fold_small_kernel(const uint32_t* __restrict__ gpos,
                                                                   const uint64_t* __restrict__ groups, uint64_t n,
                                                                   const __grid_constant__ PartialAggSpec s,
                                                                   const uint64_t* __restrict__ vals,
                                                                   const uint64_t* __restrict__ vhi,
                                                                   const uint32_t* __restrict__ nulls,
                                                                   uint64_t* __restrict__ rlo, uint64_t* __restrict__ rhi,
                                                                   uint32_t* __restrict__ rnull,
                                                                   uint64_t* __restrict__ rmom) {
  const uint64_t G = *groups;
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < G; g += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t s0 = gpos[g], e0 = gpos[g + 1];
    if (e0 - s0 > kSmallGroup) continue;
    uint32_t nm = 0;
    for (uint32_t k = 0; k < s.n_bufs; k++) {
      const uint32_t op = s.op[k];
      PAcc acc{0, 0, 0, 0};
      if (Merge && s.stage[k] == kStageMerge) {
        if (op == B2S_AGG_VARIANCE) {
          double cn = 0.0, avg = 0.0, m2 = 0.0;
          for (uint32_t j = s0; j < e0; j++)
            var_merge(cn, avg, m2, dbl(__ldg(vals + (size_t)k * n + j)), dbl(__ldg(vhi + (size_t)s.wide[k] * n + j)),
                      dbl(__ldg(vhi + (size_t)(s.wide[k] + 1) * n + j)));
          put_var(s, k, g, n, cn, avg, m2, rlo, rmom);
        } else {
          Dec128 sum{0, 0};
          bool gone = false;
          for (uint32_t j = s0; j < e0; j++)
            dec_merge(sum, gone, (__ldg(nulls + j) >> k) & 1,
                      Dec128{__ldg(vals + (size_t)k * n + j), __ldg(vhi + (size_t)s.wide[k] * n + j)},
                      agg_precision(op));
          if (gone) nm |= 1u << k;
          put_result(s, k, g, n, PAcc{sum.lo, sum.hi, 0, 1}, rlo, rhi);
        }
        continue;
      }
      if (op == B2S_AGG_VARIANCE) {  // never null
        double cn = 0.0, avg = 0.0, m2 = 0.0;
        for (uint32_t j = s0; j < e0; j++)
          if (!((__ldg(nulls + j) >> k) & 1)) var_update(cn, avg, m2, dbl(__ldg(vals + (size_t)k * n + j)));
        put_var(s, k, g, n, cn, avg, m2, rlo, rmom);
        continue;
      }
      if (dsum_op(op)) {
        double fs = 0.0;
        for (uint32_t j = s0; j < e0; j++) {
          fs = __dadd_rn(fs, __longlong_as_double((long long)__ldg(vals + (size_t)k * n + j)));
          acc.has |= !((__ldg(nulls + j) >> k) & 1);
        }
        acc.lo = (uint64_t)__double_as_longlong(fs);
      } else {
        for (uint32_t j = s0; j < e0; j++) acc = combine(op, acc, load_acc(s, k, vals, vhi, nulls, n, j));
      }
      if (!acc.has) nm |= 1u << k;
      put_result(s, k, g, n, acc, rlo, rhi);
    }
    rnull[g] = nm;
  }
}

// groups of kSmallGroup + 1 .. kChunk records: a warp each (not the chains: pa_chain_kernel)
template <bool Merge>
__global__ void __launch_bounds__(kPaThreads) pa_fold_warp_kernel(const uint32_t* __restrict__ gpos,
                                                                  const uint64_t* __restrict__ groups, uint64_t n,
                                                                  const __grid_constant__ PartialAggSpec s,
                                                                  const uint64_t* __restrict__ vals,
                                                                  const uint64_t* __restrict__ vhi,
                                                                  const uint32_t* __restrict__ nulls,
                                                                  uint64_t* __restrict__ rlo, uint64_t* __restrict__ rhi,
                                                                  uint32_t* __restrict__ rnull) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t G = *groups, warps = (uint64_t)gridDim.x * (kPaThreads / 32);
  for (uint64_t g = (uint64_t)blockIdx.x * (kPaThreads / 32) + (threadIdx.x >> 5); g < G; g += warps) {
    const uint32_t s0 = gpos[g], e0 = gpos[g + 1];
    if (e0 - s0 <= kSmallGroup || e0 - s0 > kChunk) continue;  // uniform over the warp
    uint32_t nm = 0;
    for (uint32_t k = 0; k < s.n_bufs; k++) {
      if (skips<Merge>(s, k)) continue;
      const PAcc r = fold_warp(s, k, vals, vhi, nulls, n, s0, e0, lane);
      if (!r.has) nm |= 1u << k;
      if (lane == 0) put_result(s, k, g, n, r, rlo, rhi);
    }
    if (lane == 0) rnull[g] = nm;  // a double sum's bit: pa_chain_kernel's atomicOr
  }
}

// a warp per aligned chunk c of kChunk positions: the large groups (over kChunk records) it meets, at most two: the one
// holding its first position (partial slot 0) and, if another, the one holding its last (slot 1)
template <bool Merge>
__global__ void __launch_bounds__(kPaThreads) pa_fold_chunk_kernel(const uint32_t* __restrict__ gpos,
                                                                   const uint64_t* __restrict__ hb,
                                                                   const uint64_t* __restrict__ groups, uint64_t n,
                                                                   const __grid_constant__ PartialAggSpec s,
                                                                   const uint64_t* __restrict__ vals,
                                                                   const uint64_t* __restrict__ vhi,
                                                                   const uint32_t* __restrict__ nulls,
                                                                   PAcc* __restrict__ part) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t G = *groups, C = n_chunks(n), warps = (uint64_t)gridDim.x * (kPaThreads / 32);
  for (uint64_t c = (uint64_t)blockIdx.x * (kPaThreads / 32) + (threadIdx.x >> 5); c < C; c += warps) {
    const uint64_t p0 = c * kChunk, p1 = std::min<uint64_t>(n, p0 + kChunk);
    const uint64_t g0 = group_of(hb, n, G, p0), g1 = group_of(hb, n, G, p1 - 1);
    for (uint32_t slot = 0; slot < 2; slot++) {
      const uint64_t g = slot ? g1 : g0;
      if (slot && g1 == g0) break;
      const uint32_t s0 = gpos[g], e0 = gpos[g + 1];
      if (e0 - s0 <= kChunk) continue;
      const uint32_t a = (uint32_t)std::max<uint64_t>(s0, p0), b = (uint32_t)std::min<uint64_t>(e0, p1);
      for (uint32_t k = 0; k < s.n_bufs; k++) {
        if (skips<Merge>(s, k)) continue;
        const PAcc r = fold_warp(s, k, vals, vhi, nulls, n, a, b, lane);
        if (lane == 0) part[(c * 2 + slot) * s.n_bufs + k] = r;
      }
    }
  }
}

// a warp per large group: its chunks' partials combined (chunk c holds it in slot 0 when it holds c's first position)
template <bool Merge>
__global__ void __launch_bounds__(kPaThreads) pa_fold_combine_kernel(const uint32_t* __restrict__ gpos,
                                                                     const uint64_t* __restrict__ groups, uint64_t n,
                                                                     const __grid_constant__ PartialAggSpec s,
                                                                     const PAcc* __restrict__ part,
                                                                     uint64_t* __restrict__ rlo,
                                                                     uint64_t* __restrict__ rhi,
                                                                     uint32_t* __restrict__ rnull) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t G = *groups, warps = (uint64_t)gridDim.x * (kPaThreads / 32);
  for (uint64_t g = (uint64_t)blockIdx.x * (kPaThreads / 32) + (threadIdx.x >> 5); g < G; g += warps) {
    const uint32_t s0 = gpos[g], e0 = gpos[g + 1];
    if (e0 - s0 <= kChunk) continue;
    const uint64_t c0 = s0 / kChunk, c1 = (e0 - 1) / kChunk;
    uint32_t nm = 0;
    for (uint32_t k = 0; k < s.n_bufs; k++) {
      const uint32_t op = s.op[k];
      if (chain_op(op) || (Merge && s.stage[k] == kStageMerge)) continue;
      PAcc acc{0, 0, 0, 0};
      for (uint64_t c = c0 + lane; c <= c1; c += 32) {
        const uint32_t slot = (uint64_t)s0 <= c * kChunk ? 0 : 1;
        acc = combine(op, acc, part[(c * 2 + slot) * s.n_bufs + k]);
      }
      acc = warp_reduce(op, acc);
      if (!acc.has) nm |= 1u << k;
      if (lane == 0) put_result(s, k, g, n, acc, rlo, rhi);
    }
    if (lane == 0) rnull[g] = nm;
  }
}

// The chains of the groups over kSmallGroup records, a warp each, one chain per buffer in position order: the double
// sums (Var false: the adds, a null staged as +0.0) or the variances (Var true: var_update over the non-null inputs).
// The warp loads a tile of kTile values (coalesced) into shared memory, with a variance's null bits, and lane 0 runs
// the chain over them; the next tile's loads are issued before the chain, so they are in flight while it runs.  Runs
// after the other folds, which wrote rnull[g] without a double sum's bit (a variance is never null).  Merge: the merge
// entries are pa_var_merge_kernel's and pa_dec_merge_kernel's.
template <bool Var, bool Merge>
__global__ void __launch_bounds__(kPaThreads) pa_chain_kernel(const uint32_t* __restrict__ gpos,
                                                              const uint64_t* __restrict__ groups, uint64_t n,
                                                              const __grid_constant__ PartialAggSpec s,
                                                              const uint64_t* __restrict__ vals,
                                                              const uint32_t* __restrict__ nulls,
                                                              uint64_t* __restrict__ rlo, uint32_t* __restrict__ rnull,
                                                              uint64_t* __restrict__ rmom) {
  __shared__ double tile[kPaThreads / 32][kTile];
  __shared__ uint32_t tnull[kPaThreads / 32][Var ? kTile / 32 : 1];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint64_t G = *groups, warps = (uint64_t)gridDim.x * (kPaThreads / 32);
  constexpr uint32_t kPer = kTile / 32;
  for (uint64_t g = (uint64_t)blockIdx.x * (kPaThreads / 32) + wid; g < G; g += warps) {
    const uint32_t s0 = gpos[g], e0 = gpos[g + 1];
    if (e0 - s0 <= kSmallGroup) continue;
    uint32_t nm = 0;
    for (uint32_t k = 0; k < s.n_bufs; k++) {
      if (s.op[k] != (Var ? B2S_AGG_VARIANCE : B2S_AGG_SUM_FLOAT64) || (Merge && s.stage[k] == kStageMerge)) continue;
      const uint64_t* va = vals + (size_t)k * n;
      double next[kPer];
      uint32_t next_null[kPer];
      bool any = false;
      auto load = [&](uint32_t b) {
#pragma unroll
        for (uint32_t r = 0; r < kPer; r++) {
          const uint32_t j = b + r * 32 + lane;
          next[r] = j < e0 ? __longlong_as_double((long long)__ldg(va + j)) : 0.0;
          if (Var) {
            next_null[r] = __ballot_sync(FULL, j < e0 && ((__ldg(nulls + j) >> k) & 1));
          } else {
            any |= j < e0 && !((__ldg(nulls + j) >> k) & 1);
          }
        }
      };
      load(s0);
      double fs = 0.0, cn = 0.0, avg = 0.0, m2 = 0.0;
      for (uint32_t b = s0; b < e0; b += kTile) {
#pragma unroll
        for (uint32_t r = 0; r < kPer; r++) tile[wid][r * 32 + lane] = next[r];
        if (Var && lane == 0) {
#pragma unroll
          for (uint32_t r = 0; r < kPer; r++) tnull[wid][r] = next_null[r];
        }
        __syncwarp();
        if (b + kTile < e0) load(b + kTile);
        if (lane == 0) {
          const uint32_t m = min(kTile, e0 - b);
          if (Var) {
            for (uint32_t t = 0; t < m; t++)
              if (!((tnull[wid][t >> 5] >> (t & 31)) & 1)) var_update(cn, avg, m2, tile[wid][t]);
          } else if (m == kTile) {
#pragma unroll 16
            for (uint32_t t = 0; t < kTile; t++) fs = __dadd_rn(fs, tile[wid][t]);
          } else {
            for (uint32_t t = 0; t < m; t++) fs = __dadd_rn(fs, tile[wid][t]);
          }
        }
        __syncwarp();
      }
      if (Var) {
        if (lane == 0) put_var(s, k, g, n, cn, avg, m2, rlo, rmom);
      } else {
        if (!__any_sync(FULL, any)) nm |= 1u << k;
        if (lane == 0) rlo[(size_t)k * n + g] = (uint64_t)__double_as_longlong(fs);
      }
    }
    if (lane == 0 && nm) atomicOr(rnull + g, nm);
  }
}

// The variance merge entries (Merge) of the groups over kSmallGroup records, a warp each, as pa_chain_kernel runs the
// update chains: the warp loads a tile of kMergeTile [n, avg, m2] triples (vals, vhi words wide[k] and wide[k] + 1;
// coalesced) into shared memory and lane 0 runs CentralMomentAgg's mergeExpressions over them in position order from
// (0, 0, 0), the next tile's loads in flight meanwhile.
constexpr uint32_t kMergeTile = 64;
__global__ void __launch_bounds__(kPaThreads) pa_var_merge_kernel(const uint32_t* __restrict__ gpos,
                                                                  const uint64_t* __restrict__ groups, uint64_t n,
                                                                  const __grid_constant__ PartialAggSpec s,
                                                                  const uint64_t* __restrict__ vals,
                                                                  const uint64_t* __restrict__ vhi,
                                                                  uint64_t* __restrict__ rlo,
                                                                  uint64_t* __restrict__ rmom) {
  constexpr uint32_t kPer = kMergeTile / 32;
  __shared__ uint64_t tile[kPaThreads / 32][3][kMergeTile];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint64_t G = *groups, warps = (uint64_t)gridDim.x * (kPaThreads / 32);
  for (uint64_t g = (uint64_t)blockIdx.x * (kPaThreads / 32) + wid; g < G; g += warps) {
    const uint32_t s0 = gpos[g], e0 = gpos[g + 1];
    if (e0 - s0 <= kSmallGroup) continue;
    for (uint32_t k = 0; k < s.n_bufs; k++) {
      if (s.stage[k] != kStageMerge || s.op[k] != B2S_AGG_VARIANCE) continue;
      const uint64_t *v0 = vals + (size_t)k * n, *v1 = vhi + (size_t)s.wide[k] * n, *v2 = v1 + n;
      uint64_t next[3][kPer];
      auto load = [&](uint32_t b) {
#pragma unroll
        for (uint32_t r = 0; r < kPer; r++) {
          const uint32_t j = b + r * 32 + lane;
          next[0][r] = j < e0 ? __ldg(v0 + j) : 0;
          next[1][r] = j < e0 ? __ldg(v1 + j) : 0;
          next[2][r] = j < e0 ? __ldg(v2 + j) : 0;
        }
      };
      load(s0);
      double cn = 0.0, avg = 0.0, m2 = 0.0;
      for (uint32_t b = s0; b < e0; b += kMergeTile) {
#pragma unroll
        for (uint32_t r = 0; r < kPer; r++)
#pragma unroll
          for (uint32_t w = 0; w < 3; w++) tile[wid][w][r * 32 + lane] = next[w][r];
        __syncwarp();
        if (b + kMergeTile < e0) load(b + kMergeTile);
        if (lane == 0) {
          const uint32_t m = min(kMergeTile, e0 - b);
          for (uint32_t t = 0; t < m; t++)
            var_merge(cn, avg, m2, dbl(tile[wid][0][t]), dbl(tile[wid][1][t]), dbl(tile[wid][2][t]));
        }
        __syncwarp();
      }
      if (lane == 0) put_var(s, k, g, n, cn, avg, m2, rlo, rmom);
    }
  }
}

// a + b of 128-bit two's-complement words (mod 2^128)
__device__ __forceinline__ Dec128 add128(Dec128 a, Dec128 b) {
  Dec128 r;
  r.lo = a.lo + b.lo;
  r.hi = a.hi + b.hi + (r.lo < a.lo ? 1 : 0);
  return r;
}

// The decimal sum merge entries (Merge) of the groups over kSmallGroup records, a CTA each.  The sequential merge
// (dec_merge: null once an input is null or a running sum reaches 10^P) is null exactly when some input is null or some
// prefix sum is out of range, so the prefixes are checked in parallel: each warp sums its segment of the group, the
// segment sums give each warp the sum before its segment, and each warp then scans its segment 32 positions a round
// (an inclusive 128-bit warp scan on top of the sum so far) and checks every prefix.  Prefixes are taken mod 2^128:
// every input is below 10^P in magnitude (the read's merge nulls larger sums) and so is every prefix before the first
// bad one, so that one is below 2 * 10^38 and still at least 10^38 in magnitude once wrapped, and it is found; with no
// bad prefix every wrapped prefix is the true one.  Its null bit is ORed in.
__global__ void __launch_bounds__(kPaThreads) pa_dec_merge_kernel(const uint32_t* __restrict__ gpos,
                                                                  const uint64_t* __restrict__ groups, uint64_t n,
                                                                  const __grid_constant__ PartialAggSpec s,
                                                                  const uint64_t* __restrict__ vals,
                                                                  const uint64_t* __restrict__ vhi,
                                                                  const uint32_t* __restrict__ nulls,
                                                                  uint64_t* __restrict__ rlo, uint64_t* __restrict__ rhi,
                                                                  uint32_t* __restrict__ rnull) {
  constexpr uint32_t kWarps = kPaThreads / 32;
  __shared__ uint64_t seg_lo[kWarps], seg_hi[kWarps];
  __shared__ uint32_t bad[kWarps];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint64_t G = *groups;
  for (uint64_t g = blockIdx.x; g < G; g += gridDim.x) {
    const uint32_t s0 = gpos[g], e0 = gpos[g + 1];
    if (e0 - s0 <= kSmallGroup) continue;  // uniform over the CTA
    const uint32_t L = ((e0 - s0 + kWarps - 1) / kWarps + 31) / 32 * 32;
    const uint32_t a = min(e0, s0 + wid * L), b = min(e0, a + L);
    uint32_t nm = 0;
    for (uint32_t k = 0; k < s.n_bufs; k++) {
      if (s.stage[k] != kStageMerge || agg_base_op(s.op[k]) != B2S_AGG_SUM_DECIMAL) continue;
      const uint64_t *v0 = vals + (size_t)k * n, *v1 = vhi + (size_t)s.wide[k] * n;
      const uint32_t P = agg_precision(s.op[k]);
      // pass 1: the segment's sum
      Dec128 part{0, 0};
      for (uint32_t j = a + lane; j < b; j += 32) part = add128(part, Dec128{__ldg(v0 + j), __ldg(v1 + j)});
#pragma unroll
      for (int d = 16; d; d >>= 1)
        part = add128(part, Dec128{__shfl_xor_sync(FULL, part.lo, d), __shfl_xor_sync(FULL, part.hi, d)});
      if (lane == 0) {
        seg_lo[wid] = part.lo;
        seg_hi[wid] = part.hi;
      }
      __syncthreads();
      Dec128 sum{0, 0}, total{0, 0};
      for (uint32_t w = 0; w < kWarps; w++) {
        if (w == wid) sum = total;
        total = add128(total, Dec128{seg_lo[w], seg_hi[w]});
      }
      // pass 2: every prefix of the segment, on top of the sum before it
      bool gone = false;
      for (uint32_t c = a; c < b && !gone; c += 32) {
        const uint32_t j = c + lane;
        const bool in = j < b;
        const bool null = in && ((__ldg(nulls + j) >> k) & 1);
        Dec128 x{in && !null ? __ldg(v0 + j) : 0, in && !null ? __ldg(v1 + j) : 0};
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const Dec128 y{__shfl_up_sync(FULL, x.lo, d), __shfl_up_sync(FULL, x.hi, d)};
          if (lane >= (uint32_t)d) x = add128(x, y);
        }
        x = add128(sum, x);
        gone = __any_sync(FULL, in && (null || !dec_fits(x, P)));
        sum = Dec128{__shfl_sync(FULL, x.lo, 31), __shfl_sync(FULL, x.hi, 31)};
      }
      if (lane == 0) bad[wid] = gone;
      __syncthreads();
      bool any = false;
      for (uint32_t w = 0; w < kWarps; w++) any |= bad[w] != 0;
      if (any) nm |= 1u << k;
      if (threadIdx.x == 0) put_result(s, k, g, n, PAcc{total.lo, total.hi, 0, 1}, rlo, rhi);
      __syncthreads();  // the shared words are reused by the next entry
    }
    if (threadIdx.x == 0 && nm) atomicOr(rnull + g, nm);
  }
}

// Position j of the merged rows (in their key order) starts a group of the key columns ks (a prefix of the order's
// columns): j == 0, or its encoded key differs from j - 1's (encoded_keys_equal, as the window's partition heads
// compare theirs; the read's key pass has checked every string and decimal).  No key columns: only position 0.
__global__ void __launch_bounds__(kPaThreads) pa_heads_kernel(const uint8_t* __restrict__ rec,
                                                              const uint64_t* __restrict__ rec_off,
                                                              const uint32_t* __restrict__ rec_len, uint64_t n,
                                                              const __grid_constant__ KeySpec ks,
                                                              uint32_t* __restrict__ heads) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t h = j == 0;
    if (j && ks.n)
      h = !encoded_keys_equal(rec + rec_off[j] + 4, rec_len[j] - 4, rec + rec_off[j - 1] + 4, rec_len[j - 1] - 4, ks);
    heads[j] = h;
  }
}

// ---- the partial rows ----
// a key column's var bytes in the partial row (c < n_keys): a non-null string its length padded to 8, a wide decimal
// (null or not) 16
__device__ __forceinline__ uint32_t key_var_bytes(const uint8_t* row, const KeySpec& ks, uint32_t c, bool null) {
  const uint32_t ty = ks.type[c];
  if (ty == kDecimalKey) return 16;
  if (ty != kStringKey || null) return 0;
  uint64_t slot, unused;
  ld_span16<true>(row + ks.off[c], 8, slot, unused);
  return ((uint32_t)slot + 7) & ~7u;
}

__device__ __forceinline__ bool key_null(const uint8_t* row, const KeySpec& ks, uint32_t c) {
  return ks.null_field[c] >= 0 && bit_at(row, ks.null_field[c]);
}

// a buffer's result is out of line: a decimal of precision above 18
__device__ __forceinline__ bool wide_buffer(uint32_t op) { return agg_decimal_wide(op); }

// per group g < G its partial row's record length (4 + row) into rowlen and rowoff (0 past the last group), for the scan
__global__ void __launch_bounds__(kPaThreads) pa_size_kernel(const uint8_t* __restrict__ rec,
                                                             const uint64_t* __restrict__ rec_off,
                                                             const uint32_t* __restrict__ idx,
                                                             const uint32_t* __restrict__ gpos,
                                                             const uint64_t* __restrict__ groups, uint64_t n,
                                                             const __grid_constant__ PartialAggSpec s,
                                                             uint32_t* __restrict__ rowlen,
                                                             uint64_t* __restrict__ rowoff) {
  const uint64_t G = *groups;
  const uint32_t nf = s.keys.n + s.n_fields, fixed = 8 * (1 + nf);
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t len = 0;
    if (g < G) {
      const uint32_t j = gpos[g], i = idx ? idx[j] : j;
      const uint8_t* row = rec + rec_off[i] + 4;
      len = 4 + fixed;
      for (uint32_t c = 0; c < s.keys.n; c++) len += key_var_bytes(row, s.keys, c, key_null(row, s.keys, c));
      for (uint32_t k = 0; k < s.n_bufs; k++) len += wide_buffer(s.op[k]) ? 16 : 0;
      rowlen[g] = len;
    }
    rowoff[g] = len;
  }
}

// Partial row g (rowoff: its scanned offset), a warp: lane f < nf is field f.  The key values come from the group's
// first row; float keys normalized (-0.0 -> 0.0, any NaN -> the canonical one); a wide decimal key or buffer re-encoded
// as BigInteger.toByteArray's minimal bytes.  Lane 0 writes the size prefix and the null word.
__global__ void __launch_bounds__(kPaThreads) pa_emit_kernel(const uint8_t* __restrict__ rec,
                                                             const uint64_t* __restrict__ rec_off,
                                                             const uint32_t* __restrict__ rec_len,
                                                             const uint32_t* __restrict__ idx,
                                                             const uint32_t* __restrict__ gpos, uint64_t G, uint64_t n,
                                                             const __grid_constant__ PartialAggSpec s,
                                                             const uint64_t* __restrict__ rlo,
                                                             const uint64_t* __restrict__ rhi,
                                                             const uint32_t* __restrict__ rnull,
                                                             const uint64_t* __restrict__ rmom,
                                                             const uint32_t* __restrict__ rowlen,
                                                             const uint64_t* __restrict__ rowoff,
                                                             uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nk = s.keys.n, nf = nk + s.n_fields, fixed = 8 * (1 + nf);
  const uint64_t warps = (uint64_t)gridDim.x * (kPaThreads / 32);
  for (uint64_t g = (uint64_t)blockIdx.x * (kPaThreads / 32) + (threadIdx.x >> 5); g < G; g += warps) {
    const uint32_t j = gpos[g], i = idx ? idx[j] : j;
    const uint8_t* row = rec + rec_off[i] + 4;
    const uint32_t size = rec_len[i] - 4;
    uint8_t* out = dst + rowoff[g];
    uint8_t* orow = out + 4;
    // this lane's field: its slot, null bit, var bytes and, for a wide decimal, its 16 bytes
    bool null = false, dec = false, str = false;
    uint64_t slot = 0, m0 = 0, m1 = 0;
    uint32_t var = 0, slen = 0, sfrom = 0;
    if (lane < nk) {
      const uint32_t c = lane, ty = s.keys.type[c];
      null = key_null(row, s.keys, c);
      var = key_var_bytes(row, s.keys, c, null);
      if (!null) {
        uint64_t v, unused;
        ld_span16<true>(row + s.keys.off[c], (int)s.keys.len[c], v, unused);
        if (ty == kStringKey) {
          str = true;
          sfrom = (uint32_t)(v >> 32);
          slen = (uint32_t)v;
        } else if (ty == kDecimalKey) {
          uint64_t hi, lo;
          bool bad = false;
          decimal_bits(row, size, v, hi, lo, &bad);
          const Dec128 x{lo, hi ^ (1ull << 63)};
          slen = dec_bytes(x);
          dec_encode(x, slen, &m0, &m1);
          dec = true;
        } else if (ty == B2S_KEY_FLOAT32) {
          const uint32_t b = (uint32_t)v, mag = b & 0x7fffffffu;
          slot = mag == 0 ? 0u : mag > 0x7f800000u ? 0x7fc00000u : b;
        } else if (ty == B2S_KEY_FLOAT64) {
          const uint64_t mag = v & 0x7fffffffffffffffull;
          slot = mag == 0 ? 0ull : mag > 0x7ff0000000000000ull ? 0x7ff8000000000000ull : v;
        } else {
          const uint32_t len = s.keys.len[c];
          slot = len >= 8 ? v : v & ((1ull << (8 * len)) - 1);
        }
      } else if (ty == kDecimalKey) {
        dec = true;  // 16 zero bytes, slot offset << 32
      }
    } else if (lane < nf) {
      // the lane's buffer k and, for a variance, which of its three fields (n, avg, m2)
      uint32_t k = 0, part = lane - nk;
      for (; k + 1 < s.n_bufs; k++) {
        const uint32_t w = s.op[k] == B2S_AGG_VARIANCE ? 3 : 1;
        if (part < w) break;
        part -= w;
      }
      const uint32_t op = s.op[k];
      null = (rnull[g] >> k) & 1;
      const uint64_t lo = part ? rmom[(size_t)(2 * s.var[k] + part - 1) * n + g] : rlo[(size_t)k * n + g];
      if (wide_buffer(op)) {
        var = 16;
        dec = true;
        if (!null) {
          const Dec128 x{lo, rhi[(size_t)s.wide[k] * n + g]};
          slen = dec_bytes(x);
          dec_encode(x, slen, &m0, &m1);
        }
      } else if (!null) {
        slot = op == B2S_AGG_MIN_INT32 || op == B2S_AGG_MAX_INT32 ? (uint32_t)lo : lo;
      }
    }
    // var regions in field order
    uint32_t at = var;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(FULL, at, d);
      if (lane >= (uint32_t)d) at += t;
    }
    const uint32_t voff = fixed + at - var;
    if (dec) {
      st_span16(orow + voff, 16, m0, m1);
      slot = ((uint64_t)voff << 32) | (null ? 0 : slen);
    } else if (str) {
      for (uint32_t b = 0; b < var; b++) orow[voff + b] = b < slen ? row[sfrom + b] : 0;
      slot = ((uint64_t)voff << 32) | slen;
    }
    if (lane < nf) st_span16(orow + 8 + 8 * lane, 8, slot, 0);
    const uint32_t nulls = __ballot_sync(FULL, lane < nf && null);
    if (lane == 0) {
      const uint32_t sz = rowlen[g] - 4;
      st_span16(out, 4, __byte_perm(sz, 0, 0x0123), 0);
      st_span16(orow, 8, nulls, 0);
    }
  }
}

// the staging, the folds and the chains of launch_partial_agg_fold (Merge: a spec with merge entries)
template <bool Merge>
void launch_fold(const uint8_t* rec, uint64_t n, const uint32_t* idx, const KeySortWs& w, const PaWs& a,
                 const uint32_t* gpos, const uint64_t* hb, const uint64_t* groups, const PartialAggSpec& spec,
                 cudaStream_t st, uint64_t* launches) {
  pa_stage_kernel<Merge><<<grid_for(n), kPaThreads, 0, st>>>(rec, w.src_off, w.len, idx, n, spec, a.vals, a.vhi,
                                                             a.nulls);
  pa_fold_small_kernel<Merge><<<grid_for(n), kPaThreads, 0, st>>>(gpos, groups, n, spec, a.vals, a.vhi, a.nulls, a.rlo,
                                                                  a.rhi, a.rnull, a.rmom);
  const unsigned wg = warp_grid_for(n / kSmallGroup + 1);
  pa_fold_warp_kernel<Merge><<<wg, kPaThreads, 0, st>>>(gpos, groups, n, spec, a.vals, a.vhi, a.nulls, a.rlo, a.rhi,
                                                        a.rnull);
  uint32_t launched = 3;
  if (n > kChunk) {
    pa_fold_chunk_kernel<Merge><<<warp_grid_for(n_chunks(n)), kPaThreads, 0, st>>>(gpos, hb, groups, n, spec, a.vals,
                                                                                   a.vhi, a.nulls, a.part);
    pa_fold_combine_kernel<Merge><<<warp_grid_for(n / kChunk + 1), kPaThreads, 0, st>>>(gpos, groups, n, spec, a.part,
                                                                                        a.rlo, a.rhi, a.rnull);
    launched += 2;
  }
  if (spec.dsum) {
    pa_chain_kernel<false, Merge><<<wg, kPaThreads, 0, st>>>(gpos, groups, n, spec, a.vals, a.nulls, a.rlo, a.rnull,
                                                             a.rmom);
    launched++;
  }
  if (spec.n_var) {
    pa_chain_kernel<true, Merge><<<wg, kPaThreads, 0, st>>>(gpos, groups, n, spec, a.vals, a.nulls, a.rlo, a.rnull,
                                                            a.rmom);
    launched++;
  }
  if (Merge && spec.n_merge_var) {
    pa_var_merge_kernel<<<wg, kPaThreads, 0, st>>>(gpos, groups, n, spec, a.vals, a.vhi, a.rlo, a.rmom);
    launched++;
  }
  if (Merge && spec.n_merge_dec) {
    pa_dec_merge_kernel<<<grid_for(n), kPaThreads, 0, st>>>(gpos, groups, n, spec, a.vals, a.vhi, a.nulls, a.rlo,
                                                            a.rhi, a.rnull);
    launched++;
  }
  if (launches) *launches += launched;
}

}  // namespace

size_t partial_agg_ws_bytes(uint64_t n, const PartialAggSpec& s) {
  return 256 + 2 * a256(n * s.n_bufs * 8) + 2 * a256(n * s.n_dec * 8) + 2 * a256(n * 4) + a256(n * s.n_var * 16) +
         a256(n_chunks(n) * 2 * s.n_bufs * sizeof(PAcc)) + a256(n * 4) + a256(n * 8) + a256(scan_ws_elems(n) * 8);
}

uint64_t* partial_agg_header(uint8_t* d_paws) { return (uint64_t*)d_paws; }

void launch_partial_agg_offsets(const uint32_t* rec_len, uint64_t n, uint32_t key_bytes, uint8_t* d_ws,
                                uint8_t* d_paws, cudaStream_t st, uint64_t* launches) {
  uint64_t* hdr = partial_agg_header(d_paws);
  cudaMemsetAsync(hdr, 0, 256, st);
  cudaMemsetAsync(hdr, 0xff, 8, st);      // check verdict
  cudaMemsetAsync(hdr + 2, 0xff, 8, st);  // check detail
  if (!n) return;
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  uint64_t* scan_ws = (uint64_t*)(d_ws + key_sort_ws_bytes(n, key_bytes));
  pa_offsets_kernel<<<grid_for(n), kPaThreads, 0, st>>>(rec_len, n, w.len, w.src_off);
  launch_exclusive_scan_u64(w.src_off, n, hdr + 1, scan_ws, st, launches);
  if (launches) *launches += 1;
}

void launch_partial_agg_check(const uint8_t* rec, uint64_t rec_bytes, uint64_t n, uint32_t key_bytes,
                              const PartialAggSpec& spec, uint8_t* d_ws, uint8_t* d_paws, uint32_t* ids,
                              cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  uint64_t* hdr = partial_agg_header(d_paws);
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  launch_rows_hash(rec, rec_bytes, w.src_off, w.len, n, spec.keys, 1, ids, hdr, st, launches);
  pa_check_kernel<<<grid_for(n), kPaThreads, 0, st>>>(rec, rec_bytes, w.src_off, w.len, n, spec,
                                                      (unsigned long long*)hdr, (unsigned long long*)(hdr + 2));
  if (launches) *launches += 1;
}

void launch_partial_agg_fold(const uint8_t* rec, uint64_t n, const uint32_t* idx, uint32_t key_bytes,
                             const PartialAggSpec& spec, uint8_t* d_ws, uint8_t* d_gws, uint8_t* d_paws,
                             cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  const PaWs a = carve_pa_ws(d_paws, n, spec);
  const uint64_t* groups = rows_aggregate_readback(d_gws, n, 0, 0);
  const uint32_t* gpos = rows_group_starts(d_gws, n);
  const uint64_t* hb = rows_group_heads_before(d_gws, n);
  cudaMemcpyAsync(a.hdr + 4, groups, 8, cudaMemcpyDeviceToDevice, st);
  if (spec.n_bufs) {
    if (spec.merge) launch_fold<true>(rec, n, idx, w, a, gpos, hb, groups, spec, st, launches);
    else launch_fold<false>(rec, n, idx, w, a, gpos, hb, groups, spec, st, launches);
  }
  pa_size_kernel<<<grid_for(n), kPaThreads, 0, st>>>(rec, w.src_off, idx, gpos, groups, n, spec, a.rowlen, a.rowoff);
  launch_exclusive_scan_u64(a.rowoff, n, a.hdr + 5, a.scan_ws, st, launches);
  if (launches) *launches += 1;
}

const uint32_t* partial_agg_row_len(uint8_t* d_paws, uint64_t n, const PartialAggSpec& spec) {
  return carve_pa_ws(d_paws, n, spec).rowlen;
}

void launch_partial_agg_emit(const uint8_t* rec, uint64_t n, uint64_t groups, const uint32_t* idx, uint32_t key_bytes,
                             const PartialAggSpec& spec, uint8_t* d_ws, uint8_t* d_gws, uint8_t* d_paws,
                             uint8_t* d_dst, cudaStream_t st, uint64_t* launches) {
  if (!groups) return;
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  const PaWs a = carve_pa_ws(d_paws, n, spec);
  pa_emit_kernel<<<warp_grid_for(groups), kPaThreads, 0, st>>>(rec, w.src_off, w.len, idx, rows_group_starts(d_gws, n),
                                                              groups, n, spec, a.rlo, a.rhi, a.rnull, a.rmom,
                                                              a.rowlen, a.rowoff, d_dst);
  if (launches) *launches += 1;
}

void launch_partial_agg_heads(const uint8_t* rec, uint64_t n, uint32_t key_bytes, const KeySpec& ks, uint8_t* d_ws,
                              uint32_t* heads, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  pa_heads_kernel<<<grid_for(n), kPaThreads, 0, st>>>(rec, w.src_off, w.len, n, ks, heads);
  if (launches) *launches += 1;
}

}  // namespace b2s
