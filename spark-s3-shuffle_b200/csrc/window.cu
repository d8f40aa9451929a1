// window.cu — Spark's WindowExec on a reducer for the ranking functions (row_number, rank, dense_rank, percent_rank,
// cume_dist, ntile), with WindowGroupLimitExec's limit, for the aggregate functions (sum, count, min, max, avg) over
// whole-partition and running frames, and for the offset functions (lag, lead, first, last, nth_value), and the output
// rows built as UnsafeRowJoiner joins the input row with the row of values.  The records have been framed, keyed by the
// whole window key (partition columns, then order columns), stably sorted by rows.cu and grouped by aggregate.cu's
// launch_rows_group, whose groups are the peer groups.  All on the device:
//   heads  : one thread per sorted position: a partition starts at a peer head whose partition columns differ from its
//            predecessor's, compared by encode_key 16 encoded bytes at a time until they differ or both keys end (so
//            the equality is the sort's: strings by length and bytes, -0.0 with 0.0, NaN with NaN, null with null);
//            the flags scanned, and each partition's first position compacted
//   nonnull: (offset functions with IGNORE_NULLS over a nullable input) per function a present flag per sorted position,
//            exclusive-scanned to r(j) (the total at r(n)), and the present positions compacted into pres[]; a
//            partition [ps, pe)'s present positions are then pres[r(ps) .. r(pe)), so every skip-nulls lookup is index
//            arithmetic bounded by the partition or the frame
//   stage  : (aggregate functions) one thread per sorted position: each aggregate's input, null flag and, for a
//            DECIMAL_WIDE input, its 16 bytes checked, into dense sorted-order state arrays (lo, hi, count)
//   fold   : each state becomes its fold over the partition's positions up to it.  Integer sums, counts, decimal sums
//            and min / max are associative: a log-step segmented scan, one pass per power of two below n, each
//            position combining with the one d before it while that is in its partition (min / max keep the earlier
//            of equal values).  Double sums are serial by contract: a warp per partition, 32 positions a round loaded
//            one round ahead, each lane's value broadcast in turn and added in order, each lane keeping its prefix
//   frames : (sliding ROWS / RANGE frames) one thread per sorted position: each distinct bounds set's frame [fs, ft),
//            by arithmetic, the peer group, or a binary search over the staged RANGE column; then, from the staged
//            inputs, range-minimum passes for MIN / MAX and a fresh double fold per row for double sums whose frame's
//            lower end is bounded (every other aggregate reads the prefix folds at both ends of its frame)
//   values : one thread per sorted position: from its partition's bounds and its peer group's bounds and index, every
//            function's value (into a per-function array in sorted order; an aggregate's read from the fold at its
//            frame's last position, with its null flag and a wide decimal's high word; an offset function's source
//            position, read for a fixed-width value), whether the limit keeps it, and its output bytes (a string
//            value's bytes padded to 8 make them per row); each record's own string and wide decimal inputs of offset
//            functions are checked; the kept records and the bytes scanned, and the totals, the too-long and
//            too-large-partition flags and the first bad input come back in one readback
//   emit   : a warp per output row (with a limit, over the compacted kept positions only): its null words widened (with
//            the values' null bits), its slots, the function slots, its var bytes and the var-valued functions' bytes in
//            function order (16 per wide decimal, a string's padded to 8; with offset functions each region's offset is
//            a warp scan of the sizes before it), then the VAR and DECIMAL_WIDE slots' offsets moved
// A map task's partial limit (WindowGroupLimitExec(Partial), in front of the shuffle) takes the same heads, then a
// thread per sorted position for its limit value, keep flag and kept length (scanned), and a warp per kept record that
// copies it unchanged: the partition + compress step's input.
#include <algorithm>

#include "decimal128.h"
#include "rows_key.cuh"

namespace b2s {

namespace {

constexpr int kWindowThreads = 256;

inline size_t a256(size_t b) { return (b + 255) / 256 * 256; }

inline unsigned grid_for(uint64_t n) {
  const uint64_t want = (n + kWindowThreads - 1) / kWindowThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

// the window workspace: per position the partition-head flags (scanned in place, the partition count at [n]), the
// partitions' first positions (n after the last), every function's value (function f at [f n, f n + n)), the kept
// records and the output bytes (scanned in place), the kept positions compacted; scan workspace, readback, the shape
// and its field list; then, with aggregate functions, two sets of fold state (aggregate a at [a n, a n + n) of each
// array), the values' null bits per position (with aggregate or offset functions) and the wide decimal results' high
// words (wide ordinal k at [k n, k n + n)); then per non-null index x the scanned present flags (n + 1 at [x stride,
// x stride + n]) and the present positions (at [x n, x n + n))
struct WindowWs {
  uint64_t* phead;
  uint32_t* pstart;
  uint64_t* vals;
  uint64_t* rows;
  uint64_t* bytes;
  uint32_t* kept;
  uint64_t* scan_ws;
  uint64_t* readback;
  WindowShape* shape;
  uint32_t* fields;
  uint64_t* lo[2];
  uint64_t* hi[2];
  uint32_t* cnt[2];
  uint32_t* vnul;
  uint64_t* vhi;
  uint64_t* rnk;
  uint32_t* pres;
  uint64_t stride;
  uint32_t* fs;
  uint32_t* ft;
  uint64_t* ov;
  uint8_t* onull;
  uint64_t* rlo[3];
  uint64_t* rhi[3];
  uint32_t* rcnt[3];
  uint8_t* end;
};

WindowWs carve_window_ws(uint8_t* d_wws, uint64_t n, const WindowShape& sh) {
  WindowWs w;
  uint8_t* p = d_wws;
  w.phead = (uint64_t*)p;    p += a256((n + 1) * 8);
  w.pstart = (uint32_t*)p;   p += a256((n + 1) * 4);
  w.vals = (uint64_t*)p;     p += a256((size_t)sh.n_fns * n * 8);
  w.rows = (uint64_t*)p;     p += a256(n * 8);
  w.bytes = (uint64_t*)p;    p += a256(n * 8);
  w.kept = (uint32_t*)p;     p += a256(n * 4);
  w.scan_ws = (uint64_t*)p;  p += a256(scan_ws_elems(n + 1) * 8);
  w.readback = (uint64_t*)p; p += a256(kWindowReadbackBytes);
  w.shape = (WindowShape*)p; p += a256(sizeof(WindowShape));
  w.fields = (uint32_t*)p;   p += a256((size_t)sh.n * 4);
  const size_t m = (size_t)sh.n_agg * n;
  for (int b = 0; b < 2; b++) {
    w.lo[b] = (uint64_t*)p;  p += a256(m * 8);
    w.hi[b] = (uint64_t*)p;  p += a256(m * 8);
    w.cnt[b] = (uint32_t*)p; p += a256(m * 4);
  }
  w.vnul = (uint32_t*)p;     p += a256(sh.n_agg || sh.n_off ? n * 4 : 0);
  w.vhi = (uint64_t*)p;      p += a256((size_t)sh.n_wide * n * 8);
  w.stride = a256((n + 1) * 8) / 8;
  w.rnk = (uint64_t*)p;      p += (size_t)sh.n_nn * w.stride * 8;
  w.pres = (uint32_t*)p;     p += a256((size_t)sh.n_nn * n * 4);
  // sliding frames: per bounds set b each position's frame [fs, ft) (at [b n, b n + n)), the staged order column, and
  // per result state r (at [r n, r n + n)) its value, then with range-minimum passes two sets of level state
  w.fs = (uint32_t*)p;       p += a256((size_t)sh.n_bnd * n * 4);
  w.ft = (uint32_t*)p;       p += a256((size_t)sh.n_bnd * n * 4);
  w.ov = (uint64_t*)p;       p += a256(sh.ord_staged ? n * 8 : 0);
  w.onull = p;               p += a256(sh.ord_staged ? n : 0);
  for (int b = 0; b < 3; b++) {
    const size_t r = b == 0 || sh.rmq_width > 1 ? (size_t)sh.n_res * n : 0;
    w.rlo[b] = (uint64_t*)p;  p += a256(r * 8);
    w.rhi[b] = (uint64_t*)p;  p += a256(r * 8);
    w.rcnt[b] = (uint32_t*)p; p += a256(r * 4);
  }
  w.end = p;
  return w;
}

__device__ __forceinline__ uint32_t at(const uint32_t* idx, uint64_t j) { return idx ? idx[j] : (uint32_t)j; }

__device__ __forceinline__ uint64_t ld64(const uint8_t* p) {
  uint64_t lo, unused;
  ld_span16<true>(p, 8, lo, unused);
  return lo;
}

// the exclusive scan of some flags after position j: scanned[j + 1], or the total after the last position.  So j is
// flagged when it differs from scanned[j], and next_scanned - 1 is the index of the run that holds j.
__device__ __forceinline__ uint64_t next_scanned(const uint64_t* scanned, uint64_t j, uint64_t n, uint64_t total) {
  return j + 1 < n ? scanned[j + 1] : total;
}

// Position j starts a partition: it is a peer head (its group starts there) and its partition columns differ from
// j - 1's.  Position 0 always does; without partition columns no other one.
__global__ void __launch_bounds__(kWindowThreads) window_part_heads_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t n, const WindowShape* __restrict__ sh,
    const uint64_t* __restrict__ heads_before, const uint64_t* __restrict__ groups, uint64_t* __restrict__ phead) {
  const uint64_t G = *groups;
  const KeySpec& ks = sh->part;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t h = j == 0;
    if (j && ks.n && next_scanned(heads_before, j, n, G) != heads_before[j]) {
      const uint32_t a = at(idx, j), b = at(idx, j - 1);
      // the sort's key pass has checked every string and decimal
      h = !encoded_keys_equal(arena + rec_off[a] + 4, rec_len[a] - 4, arena + rec_off[b] + 4, rec_len[b] - 4, ks);
    }
    phead[j] = h;
  }
}

// pstart[p] = partition p's first position (phead: the scanned flags, phead[n] the partition count), pstart[P] = n
__global__ void __launch_bounds__(kWindowThreads) window_part_starts_kernel(const uint64_t* __restrict__ phead,
                                                                            uint64_t n, uint32_t* __restrict__ pstart) {
  const uint64_t P = phead[n];
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (next_scanned(phead, j, n, P) != phead[j]) pstart[phead[j]] = (uint32_t)j;
    if (j == n - 1) pstart[P] = (uint32_t)n;
  }
}

__device__ __forceinline__ uint64_t int_slot(uint64_t v) { return (uint32_t)v; }  // the slot zeroed, 4 LE bytes

// NTile(k)'s bucket (1-based) of the 0-based position i of a partition of N: the first N % k buckets hold N / k + 1
// rows, the rest N / k
__device__ __forceinline__ uint64_t ntile(uint64_t i, uint64_t N, uint64_t k) {
  const uint64_t q = N / k, r = N % k, big = r * (q + 1);
  return i < big ? i / (q + 1) + 1 : r + (i - big) / q + 1;
}

// ---- aggregate functions ----
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ uint32_t val_kind(uint32_t vt) { return vt & 0xff; }
__device__ __forceinline__ uint32_t dec_p(uint32_t vt) { return (vt >> 8) & 0xff; }

// an aggregate function (offset functions are numbered after them)
__host__ __device__ __forceinline__ bool is_agg(uint32_t fn) { return fn >= B2S_WINDOW_SUM && fn <= B2S_WINDOW_AVG; }

// SUM of a float or double and AVG of anything but a decimal fold in double, serially; every other aggregate is a
// group operation (or min / max) and scans
__device__ __forceinline__ bool folds_double(uint32_t fn, uint32_t vt) {
  const uint32_t k = val_kind(vt);
  return (fn == B2S_WINDOW_SUM && (k == B2S_WINDOW_VAL_FLOAT32 || k == B2S_WINDOW_VAL_FLOAT64)) ||
         (fn == B2S_WINDOW_AVG && k != B2S_WINDOW_VAL_DECIMAL);
}

// a decimal result's precision: SUM p + 10, AVG p + 4, MIN / MAX p
__device__ __forceinline__ uint32_t result_p(uint32_t fn, uint32_t vt) {
  return dec_p(vt) + (fn == B2S_WINDOW_SUM ? 10 : fn == B2S_WINDOW_AVG ? 4 : 0);
}

__device__ __forceinline__ bool null_bit(const uint8_t* row, int32_t field) {
  return field >= 0 && (ld64(row + 8 * (uint32_t)(field >> 6)) >> (field & 63)) & 1;
}

// Stage: per aggregate a (function f) and position j, (lo, hi) = the input as a signed 128-bit integer (ints and
// decimals), its float or double bits (MIN / MAX of floats), or its double bits (double folds); count = 1 when it is
// present (always for VAL_NONE), else 0 with (lo, hi) = 0.  A bad non-null DECIMAL_WIDE input lowers *bad to its
// record's arena offset << 2 | kAggBadDecimal.
__global__ void __launch_bounds__(kWindowThreads) window_stage_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t n, const WindowShape* __restrict__ sh, uint64_t* __restrict__ lo,
    uint64_t* __restrict__ hi, uint32_t* __restrict__ cnt, unsigned long long* __restrict__ bad) {
  const uint32_t n_fns = sh->n_fns;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = at(idx, j);
    const uint8_t* row = arena + rec_off[i] + 4;
    for (uint32_t f = 0; f < n_fns; f++) {
      const uint32_t fn = sh->fn[f];
      if (!is_agg(fn)) continue;
      const uint32_t vt = sh->vtype[f], k = val_kind(vt);
      uint64_t l = 0, h = 0;
      uint32_t c = 1;
      if (k != B2S_WINDOW_VAL_NONE) {
        c = !null_bit(row, sh->vnull[f]);
        if (c) {
          const uint64_t v = ld64(row + sh->voff[f]);
          switch (k) {
            case B2S_WINDOW_VAL_INT8: l = (uint64_t)(int64_t)(int8_t)v; break;
            case B2S_WINDOW_VAL_INT16: l = (uint64_t)(int64_t)(int16_t)v; break;
            case B2S_WINDOW_VAL_INT32: l = (uint64_t)(int64_t)(int32_t)v; break;
            case B2S_WINDOW_VAL_FLOAT32: l = (uint32_t)v; break;
            default: l = v; break;  // INT64, FLOAT64, a decimal's long
          }
          h = (uint64_t)((int64_t)l >> 63);
          if (k == B2S_WINDOW_VAL_DECIMAL && dec_p(vt) > 18) {
            bool b = false;
            decimal_bits(row, rec_len[i] - 4, v, h, l, &b);
            h ^= 1ull << 63;  // decimal_bits flips the sign bit for the sort
            if (b) atomicMin(bad, (unsigned long long)((rec_off[i] << 2) | kAggBadDecimal));
          }
          if (folds_double(fn, vt))
            l = k == B2S_WINDOW_VAL_FLOAT32   ? __double_as_longlong((double)__int_as_float((int)l))
                : k == B2S_WINDOW_VAL_FLOAT64 ? l
                                              : __double_as_longlong(__ll2double_rn((long long)l));
        }
      }
      const size_t at_a = (size_t)sh->agg[f] * n + j;
      lo[at_a] = l;
      hi[at_a] = h;
      cnt[at_a] = c;
    }
  }
}

// Spark SQL's a < b for floats (k FLOAT32: the low 32 bits) or doubles: -0.0 == 0.0, NaN above everything else
__device__ __forceinline__ bool float_less(uint32_t k, uint64_t a, uint64_t b) {
  const double x = k == B2S_WINDOW_VAL_FLOAT32 ? (double)__int_as_float((int)a) : __longlong_as_double(a);
  const double y = k == B2S_WINDOW_VAL_FLOAT32 ? (double)__int_as_float((int)b) : __longlong_as_double(b);
  if (isnan(y)) return !isnan(x);
  return x < y;
}

// MIN / MAX of an earlier state (l0, h0, c0) and a later one (l, h, c), into (l, h): the later value is kept only when
// it is present and strictly better (or the earlier is absent), so the first of equal values keeps its exact bits
__device__ __forceinline__ void minmax_keep(uint32_t fn, uint32_t vt, uint64_t l0, uint64_t h0, uint32_t c0,
                                            uint64_t& l, uint64_t& h, uint32_t c) {
  const uint32_t k = val_kind(vt);
  const bool fl = k == B2S_WINDOW_VAL_FLOAT32 || k == B2S_WINDOW_VAL_FLOAT64;
  const bool later_wins = fn == B2S_WINDOW_MIN ? (fl ? float_less(k, l, l0) : dec_less(Dec128{l, h}, Dec128{l0, h0}))
                                               : (fl ? float_less(k, l0, l) : dec_less(Dec128{l0, h0}, Dec128{l, h}));
  if (c0 && !(c && later_wins)) {
    l = l0;
    h = h0;
  }
}

// One pass of the segmented scan: position j takes the combination of j - d's state (earlier) and its own when j - d
// is in its partition, else keeps its own.  Only the scanning aggregates are touched.
__global__ void __launch_bounds__(kWindowThreads) window_scan_pass_kernel(
    uint64_t n, const WindowShape* __restrict__ sh, const uint64_t* __restrict__ phead,
    const uint32_t* __restrict__ pstart, uint64_t d, const uint64_t* __restrict__ lo_in,
    const uint64_t* __restrict__ hi_in, const uint32_t* __restrict__ cnt_in, uint64_t* __restrict__ lo_out,
    uint64_t* __restrict__ hi_out, uint32_t* __restrict__ cnt_out) {
  const uint64_t P = phead[n];
  const uint32_t n_fns = sh->n_fns;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const bool take = j >= pstart[next_scanned(phead, j, n, P) - 1] + d;
    for (uint32_t f = 0; f < n_fns; f++) {
      const uint32_t fn = sh->fn[f], vt = sh->vtype[f];
      if (!is_agg(fn) || folds_double(fn, vt)) continue;
      const size_t x = (size_t)sh->agg[f] * n + j;
      uint64_t l = lo_in[x], h = hi_in[x];
      uint32_t c = cnt_in[x];
      if (take) {
        const uint64_t l0 = lo_in[x - d], h0 = hi_in[x - d];
        const uint32_t c0 = cnt_in[x - d];
        if (fn == B2S_WINDOW_MIN || fn == B2S_WINDOW_MAX) {
          minmax_keep(fn, vt, l0, h0, c0, l, h, c);
        } else {  // sums and counts, modulo 2^128
          bool unused;
          const Dec128 s = dec_add(Dec128{l0, h0}, Dec128{l, h}, &unused);
          l = s.lo;
          h = s.hi;
        }
        c += c0;
      }
      lo_out[x] = l;
      hi_out[x] = h;
      cnt_out[x] = c;
    }
  }
}

// The double folds: a warp per partition, ((0.0 + x1) + x2) + ... over the present inputs in sorted order, the running
// sum and count written at every position.  lo_in / cnt_in may be lo_out / cnt_out: a position is read a round before
// it is written, by the lane that writes it.
__global__ void __launch_bounds__(kWindowThreads) window_fold_kernel(
    uint64_t n, const WindowShape* __restrict__ sh, const uint64_t* __restrict__ phead,
    const uint32_t* __restrict__ pstart, const uint64_t* lo_in, const uint32_t* cnt_in, uint64_t* lo_out,
    uint32_t* cnt_out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
  const uint64_t P = phead[n];
  const uint32_t n_fns = sh->n_fns;
  for (uint64_t p = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; p < P; p += warps) {
    const uint64_t s = pstart[p], e = pstart[p + 1];
    for (uint32_t f = 0; f < n_fns; f++) {
      if (!is_agg(sh->fn[f]) || !folds_double(sh->fn[f], sh->vtype[f])) continue;
      const size_t base = (size_t)sh->agg[f] * n;
      double acc = 0.0;
      uint32_t seen = 0;
      uint64_t j = s + lane;
      double x = j < e ? __longlong_as_double(lo_in[base + j]) : 0.0;
      uint32_t c = j < e ? cnt_in[base + j] : 0;
      for (uint64_t r = s; r < e; r += 32) {
        const uint64_t jn = r + 32 + lane;
        const double xn = jn < e ? __longlong_as_double(lo_in[base + jn]) : 0.0;
        const uint32_t cn = jn < e ? cnt_in[base + jn] : 0;
        const unsigned present = __ballot_sync(kFull, c != 0);
        double mine = acc;
#pragma unroll
        for (uint32_t k = 0; k < 32; k++) {
          const double y = __shfl_sync(kFull, x, k);
          if ((present >> k) & 1) acc = __dadd_rn(acc, y);
          if (lane == k) mine = acc;
        }
        j = r + lane;
        if (j < e) {
          lo_out[base + j] = __double_as_longlong(mine);
          cnt_out[base + j] = seen + __popc(present & (0xffffffffu >> (31 - lane)));
        }
        seen += __popc(present);
        x = xn;
        c = cn;
      }
    }
  }
}

// ---- sliding frames ----
__host__ __device__ __forceinline__ bool is_sliding(uint32_t frame) { return frame >= B2S_WINDOW_FRAME_ROWS; }
constexpr int64_t kUnboundedPreceding = INT64_MIN, kUnboundedFollowing = INT64_MAX;

// Stage the RANGE order column: per sorted position its value sign-extended from the column's width, and its null flag
__global__ void __launch_bounds__(kWindowThreads) window_order_stage_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ idx, uint64_t n,
    const WindowShape* __restrict__ sh, uint64_t* __restrict__ ov, uint8_t* __restrict__ onull) {
  const uint32_t len = sh->ord_len, off = sh->ord_off;
  const int32_t nf = sh->ord_null;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* row = arena + rec_off[at(idx, j)] + 4;
    uint64_t v, unused;
    ld_span16<true>(row + off, (int)len, v, unused);
    const int sh_bits = 64 - 8 * (int)len;
    ov[j] = (uint64_t)(((int64_t)(v << sh_bits)) >> sh_bits);
    onull[j] = null_bit(row, nf);
  }
}

// The first position p in [a, b) whose staged order value is not before (upper: is after) the bound B in the column's
// sort order; b when there is none.  Both predicates are monotone over a partition's sorted positions.
__device__ __forceinline__ uint64_t range_search(const uint64_t* __restrict__ ov, const uint8_t* __restrict__ onull,
                                                 uint64_t a, uint64_t b, int64_t B, bool desc, bool nulls_first,
                                                 bool upper) {
  while (a < b) {
    const uint64_t m = a + (b - a) / 2;
    bool hit;
    if (onull[m]) {
      hit = !nulls_first;  // B is not null: a null sorts before it with NULLS FIRST, after it with NULLS LAST
    } else {
      const int64_t v = (int64_t)ov[m];
      hit = upper ? (desc ? v < B : v > B) : (desc ? v <= B : v >= B);
    }
    if (hit) b = m;
    else a = m + 1;
  }
  return a;
}

// Per sorted position j and bounds set b, the frame [fs, ft) of j's partition [ps, pe) (ft == fs: empty).  ROWS: j + lo
// .. j + hi clipped; RANGE: CURRENT ROW the peer group's edge, an offset the binary search for v + k (v - k
// descending) over the partition's staged order values, a null-keyed row's the null peers.  A partition whose ROWS
// offset k has N - 1 + |k| > 2^31 - 1, or a non-null v +- k outside the column's type, sets readback[5].
__global__ void __launch_bounds__(kWindowThreads) window_bounds_kernel(
    uint64_t n, const WindowShape* __restrict__ sh, const uint64_t* __restrict__ heads_before,
    const uint32_t* __restrict__ gpos, const uint64_t* __restrict__ groups, const uint64_t* __restrict__ phead,
    const uint32_t* __restrict__ pstart, const uint64_t* __restrict__ ov, const uint8_t* __restrict__ onull,
    uint32_t* __restrict__ fs, uint32_t* __restrict__ ft, uint64_t* __restrict__ readback) {
  const uint64_t G = *groups, P = phead[n];
  const uint32_t n_bnd = sh->n_bnd;
  const bool desc = sh->ord_type & B2S_KEY_DESCENDING, nulls_first = !(sh->ord_type & B2S_KEY_NULLS_LAST);
  const int64_t tmax = sh->ord_len >= 8 ? INT64_MAX : (int64_t)((1ull << (8 * sh->ord_len - 1)) - 1);
  const int64_t tmin = -tmax - 1;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = next_scanned(heads_before, j, n, G) - 1, p = next_scanned(phead, j, n, P) - 1;
    const uint64_t ps = pstart[p], pe = pstart[p + 1], gs = gpos[g], ge = gpos[g + 1];
    bool wraps = false;
    for (uint32_t b = 0; b < n_bnd; b++) {
      const int64_t lo = sh->blo[b], hi = sh->bhi[b];
      int64_t s, t;  // the frame's first position and one past its last, before clipping to the partition
      if (sh->bkind[b] == B2S_WINDOW_FRAME_ROWS) {
        s = lo == kUnboundedPreceding ? (int64_t)ps : (int64_t)j + lo;
        t = hi == kUnboundedFollowing ? (int64_t)pe : (int64_t)j + hi + 1;
        const uint64_t N1 = pe - ps - 1;
        if (j == ps && ((lo != kUnboundedPreceding && N1 + (uint64_t)(lo < 0 ? -lo : lo) > 0x7fffffffull) ||
                        (hi != kUnboundedFollowing && N1 + (uint64_t)(hi < 0 ? -hi : hi) > 0x7fffffffull)))
          wraps = true;
      } else {
        const bool null = ov && onull[j];
        const int64_t v = ov ? (int64_t)ov[j] : 0;
        int64_t e[2];
        for (int u = 0; u < 2; u++) {
          const int64_t k = u ? hi : lo;
          if (k == kUnboundedPreceding) e[u] = (int64_t)ps;
          else if (k == kUnboundedFollowing) e[u] = (int64_t)pe;
          else if (k == 0 || null) e[u] = (int64_t)(u ? ge : gs);  // the peer group: with an offset, the null peers
          else {
            const int64_t d = desc ? -k : k;  // the column's checks keep -k in range
            const bool ovf = d > 0 ? v > tmax - d : v < tmin - d;
            if (ovf) {
              wraps = true;
              e[u] = (int64_t)j;
            } else {
              e[u] = (int64_t)range_search(ov, onull, ps, pe, v + d, desc, nulls_first, u);
            }
          }
        }
        s = e[0];
        t = e[1];
      }
      s = s < (int64_t)ps ? (int64_t)ps : s > (int64_t)pe ? (int64_t)pe : s;
      t = t < s ? s : t > (int64_t)pe ? (int64_t)pe : t;
      fs[(size_t)b * n + j] = (uint32_t)s;
      ft[(size_t)b * n + j] = (uint32_t)t;
    }
    if (wraps) readback[5] = 1;
  }
}

// A MIN / MAX whose frame's lower end is bounded (res[f] >= 0, not a double fold): level k of the range-minimum passes
// holds per position j the state of [j, j + 2^k) (clipped to n); level 0 is the staged input.  Pass k writes the result
// of every position whose frame width w has floor(log2 w) == k, as the earlier of level k at fs and at ft - 2^k (the
// earlier wins ties, so the first of equal values is kept), then (build) level k + 1.  An empty frame's state is zero.
__global__ void __launch_bounds__(kWindowThreads) window_rmq_pass_kernel(
    uint64_t n, const WindowShape* __restrict__ sh, const uint32_t* __restrict__ fs, const uint32_t* __restrict__ ft,
    uint32_t k, bool staged, bool build, const uint64_t* __restrict__ lo_in, const uint64_t* __restrict__ hi_in,
    const uint32_t* __restrict__ cnt_in, uint64_t* __restrict__ lo_out, uint64_t* __restrict__ hi_out,
    uint32_t* __restrict__ cnt_out, uint64_t* __restrict__ rlo, uint64_t* __restrict__ rhi,
    uint32_t* __restrict__ rcnt) {
  const uint32_t n_fns = sh->n_fns;
  const uint64_t d = 1ull << k;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    for (uint32_t f = 0; f < n_fns; f++) {
      const uint32_t fn = sh->fn[f], vt = sh->vtype[f];
      if (sh->res[f] < 0 || (fn != B2S_WINDOW_MIN && fn != B2S_WINDOW_MAX)) continue;
      const size_t in = (size_t)(staged ? sh->agg[f] : (uint32_t)sh->res[f]) * n, r = (size_t)sh->res[f] * n;
      const size_t bx = (size_t)sh->bnd[f] * n + j;
      const uint64_t s = fs[bx], t = ft[bx];
      if (t > s && 63 - __clzll(t - s) == (int)k) {
        uint64_t l = lo_in[in + t - d], h = hi_in[in + t - d];
        const uint32_t c = cnt_in[in + t - d], c0 = cnt_in[in + s];
        minmax_keep(fn, vt, lo_in[in + s], hi_in[in + s], c0, l, h, c);
        rlo[r + j] = l;
        rhi[r + j] = h;
        rcnt[r + j] = c0 + c;
      } else if (k == 0 && t <= s) {
        rlo[r + j] = rhi[r + j] = 0;
        rcnt[r + j] = 0;
      }
      if (build) {
        uint64_t l = lo_in[in + j], h = hi_in[in + j];
        uint32_t c = cnt_in[in + j];
        if (j + d < n) {
          const uint64_t l1 = lo_in[in + j + d], h1 = hi_in[in + j + d];
          const uint32_t c1 = cnt_in[in + j + d];
          uint64_t a = l1, b = h1;
          minmax_keep(fn, vt, l, h, c, a, b, c1);
          l = a;
          h = b;
          c += c1;
        }
        lo_out[r + j] = l;
        hi_out[r + j] = h;
        cnt_out[r + j] = c;
      }
    }
  }
}

// A double fold whose frame's lower end is bounded (Spark's sliding and shrinking frames re-fold the frame from its
// first row): per position, ((0.0 + x_s) + x_{s+1}) + ... over the frame's present staged inputs, with their count.
// One thread per position, so the cost is the sum of the frame widths, as Spark's own.
__global__ void __launch_bounds__(kWindowThreads) window_frame_fold_kernel(
    uint64_t n, const WindowShape* __restrict__ sh, const uint32_t* __restrict__ fs, const uint32_t* __restrict__ ft,
    const uint64_t* __restrict__ lo_in, const uint32_t* __restrict__ cnt_in, uint64_t* __restrict__ rlo,
    uint32_t* __restrict__ rcnt) {
  const uint32_t n_fns = sh->n_fns;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    for (uint32_t f = 0; f < n_fns; f++) {
      if (sh->res[f] < 0 || !folds_double(sh->fn[f], sh->vtype[f])) continue;
      const size_t in = (size_t)sh->agg[f] * n, bx = (size_t)sh->bnd[f] * n + j;
      const uint64_t s = fs[bx], t = ft[bx];
      double acc = 0.0;
      uint32_t c = 0;
      for (uint64_t p = s; p < t; p++) {
        if (!cnt_in[in + p]) continue;
        // a NaN sum keeps its own payload, as Java's (x86's) acc + x does when both are NaN; the add alone may return
        // x's
        if (!isnan(acc)) acc = __dadd_rn(acc, __longlong_as_double(lo_in[in + p]));
        c++;
      }
      rlo[(size_t)sh->res[f] * n + j] = __double_as_longlong(acc);
      rcnt[(size_t)sh->res[f] * n + j] = c;
    }
  }
}

// the exact decimal average: S / c rounded HALF_UP to 4 more digits, as q0 10^4 + round(r0 10^4 / c) with
// q0 = |S| / c and r0 = |S| % c (c < 2^32, so each 32-bit limb's step divides a 64-bit number)
__device__ __forceinline__ Dec128 dec_avg(Dec128 x, uint32_t c) {
  const bool neg = x.hi >> 63;
  if (neg) {
    x.lo = ~x.lo + 1;
    x.hi = ~x.hi + (x.lo == 0);
  }
  const uint32_t limb[4] = {(uint32_t)(x.hi >> 32), (uint32_t)x.hi, (uint32_t)(x.lo >> 32), (uint32_t)x.lo};
  uint64_t r = 0, q[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint64_t cur = (r << 32) | limb[k];
    q[k] = cur / c;
    r = cur % c;
  }
  const uint64_t ql = (q[2] << 32) | q[3], qh = (q[0] << 32) | q[1];
  const uint64_t frac = (r * 20000 + c) / (2ull * c);  // r 10^4 / c rounded half up, 0..10^4
  Dec128 y;
  y.lo = ql * 10000;
  y.hi = qh * 10000 + __umul64hi(ql, 10000);
  const uint64_t lo = y.lo + frac;
  y.hi += lo < y.lo;
  y.lo = lo;
  if (neg) {
    y.lo = ~y.lo + 1;
    y.hi = ~y.hi + (y.lo == 0);
  }
  return y;
}

// The state arrays an aggregate's value is read from (the folds), and where the values kernel puts the values' null
// bits (a mask per position) and wide decimal results' high words; all nullptr without aggregate functions, but for
// the null bits with offset functions
struct WindowAggIo {
  const uint64_t* lo;
  const uint64_t* hi;
  const uint32_t* cnt;
  uint32_t* vnul;
  uint64_t* vhi;
};

// aggregate f's value at position j from its frame's state (l, h, c); *null when it is null (slot 0)
__device__ uint64_t agg_finish(const WindowShape* __restrict__ sh, uint32_t f, const WindowAggIo& io, uint64_t n,
                               uint64_t j, uint64_t l, uint64_t h, uint32_t c, bool* null) {
  const uint32_t fn = sh->fn[f], vt = sh->vtype[f], k = val_kind(vt);
  if (fn == B2S_WINDOW_COUNT) return c;
  *null = c == 0;
  if (!c) return 0;
  if (folds_double(fn, vt))
    return fn == B2S_WINDOW_AVG ? __double_as_longlong(__ddiv_rn(__longlong_as_double(l), (double)c)) : l;
  if (k != B2S_WINDOW_VAL_DECIMAL) {
    if (fn == B2S_WINDOW_SUM) return l;
    return k == B2S_WINDOW_VAL_INT8 ? l & 0xff : k == B2S_WINDOW_VAL_INT16 ? l & 0xffff
           : k == B2S_WINDOW_VAL_INT32 || k == B2S_WINDOW_VAL_FLOAT32 ? l & 0xffffffffull : l;
  }
  Dec128 v{l, h};
  if (fn == B2S_WINDOW_AVG) v = dec_avg(v, c);
  if (result_p(fn, vt) > 18) io.vhi[(size_t)sh->wide[f] * n + j] = v.hi;
  return v.lo;
}

// aggregate f's value at position j from the fold at its frame's last position e
__device__ uint64_t agg_value(const WindowShape* __restrict__ sh, uint32_t f, const WindowAggIo& io, uint64_t n,
                              uint64_t e, uint64_t j, bool* null) {
  const size_t x = (size_t)sh->agg[f] * n + e;
  return agg_finish(sh, f, io, n, j, io.lo[x], io.hi[x], io.cnt[x], null);
}

// What the values kernel reads for sliding frames: each bounds set's frames, and the result states
struct WindowFrameIo {
  const uint32_t* fs;
  const uint32_t* ft;
  const uint64_t* rlo;
  const uint64_t* rhi;
  const uint32_t* rcnt;
};

// aggregate f's value at position j of partition [ps, pe) over the sliding frame [s, t): its own result state, or the
// prefix folds' state at t - 1, less (sums and counts, exact modulo 2^128 and 2^32) the state at s - 1 when s > ps.  A
// frame whose lower end is unbounded (s == ps) reads the running fold as the older frames do.
__device__ uint64_t frame_agg_value(const WindowShape* __restrict__ sh, uint32_t f, const WindowAggIo& io,
                                    const WindowFrameIo& fio, uint64_t n, uint64_t ps, uint64_t s, uint64_t t,
                                    uint64_t j, bool* null) {
  if (sh->res[f] >= 0) {
    const size_t x = (size_t)sh->res[f] * n + j;
    return agg_finish(sh, f, io, n, j, fio.rlo[x], fio.rhi[x], fio.rcnt[x], null);
  }
  if (t <= s) return agg_finish(sh, f, io, n, j, 0, 0, 0, null);
  const size_t base = (size_t)sh->agg[f] * n;
  uint64_t l = io.lo[base + t - 1], h = io.hi[base + t - 1];
  uint32_t c = io.cnt[base + t - 1];
  if (s > ps) {
    const size_t x = base + s - 1;
    const uint64_t nl = ~io.lo[x] + 1, nh = ~io.hi[x] + (io.lo[x] == 0);  // -state(s - 1)
    bool unused;
    const Dec128 d = dec_add(Dec128{l, h}, Dec128{nl, nh}, &unused);
    l = d.lo;
    h = d.hi;
    c -= io.cnt[x];
  }
  return agg_finish(sh, f, io, n, j, l, h, c, null);
}

// ---- offset functions ----
__device__ __forceinline__ bool is_offset(uint32_t fn) { return fn >= B2S_WINDOW_LAG; }
__device__ __forceinline__ bool wide_input(uint32_t vt) {
  return val_kind(vt) == B2S_WINDOW_VAL_DECIMAL && dec_p(vt) > 18;
}
// the slot bits UnsafeRowWriter writes for a fixed-width value of kind k: the slot zeroed, then the type's width
__device__ __forceinline__ uint64_t width_mask(uint32_t k) {
  return k == B2S_WINDOW_VAL_INT8 ? 0xffull : k == B2S_WINDOW_VAL_INT16 ? 0xffffull
         : k == B2S_WINDOW_VAL_INT32 || k == B2S_WINDOW_VAL_FLOAT32 ? 0xffffffffull : ~0ull;
}
constexpr uint64_t kNoSource = ~0ull;

// Non-null index, step 1: per sorted position j and non-null index x (function f, nn[f] = x), rnk[x stride + j] = 1
// when f's input is present
__global__ void __launch_bounds__(kWindowThreads) window_present_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ idx, uint64_t n,
    const WindowShape* __restrict__ sh, uint64_t stride, uint64_t* __restrict__ rnk) {
  const uint32_t n_fns = sh->n_fns;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* row = arena + rec_off[at(idx, j)] + 4;
    for (uint32_t f = 0; f < n_fns; f++)
      if (sh->nn[f] >= 0) rnk[(size_t)sh->nn[f] * stride + j] = !null_bit(row, sh->vnull[f]);
  }
}

// step 3, after each index's scan: pres[x n + r(j)] = j for each present position j
__global__ void __launch_bounds__(kWindowThreads) window_pres_kernel(uint64_t n, uint32_t n_nn, uint64_t stride,
                                                                     const uint64_t* __restrict__ rnk,
                                                                     uint32_t* __restrict__ pres) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
    for (uint32_t x = 0; x < n_nn; x++) {
      const uint64_t* r = rnk + (size_t)x * stride;
      if (r[j + 1] != r[j]) pres[(size_t)x * n + r[j]] = (uint32_t)j;
    }
}

// What the values kernel reads for offset functions: the records, and the non-null indexes (nullptr without one)
struct WindowOffIo {
  const uint8_t* arena;
  const uint64_t* rec_off;
  const uint64_t* rnk;
  const uint32_t* pres;
  uint64_t stride;
};

// Offset function f's source sorted position for position j of partition [ps, pe) whose frame is [s, e] (FIRST, LAST
// and NTH_VALUE; e + 1 == s: empty), or kNoSource: outside the partition or the frame (LAG / LEAD's default, else
// null).  With a non-null index the partition's present positions are pres[r(ps) .. r(pe)) and the frame's
// pres[r(s) .. r(e + 1)).
__device__ __forceinline__ uint64_t offset_source(const WindowShape* __restrict__ sh, uint32_t f,
                                                  const WindowOffIo& io, uint64_t n, uint64_t j, uint64_t ps,
                                                  uint64_t pe, uint64_t s, uint64_t e) {
  const uint32_t fn = sh->fn[f];
  const uint64_t k = sh->arg[f];  // LAG / LEAD's offset, NTH_VALUE's n; 0 for FIRST and LAST
  const int32_t x = sh->nn[f];
  if (x < 0) {  // every position is present
    switch (fn) {
      case B2S_WINDOW_LEAD: return j + k < pe ? j + k : kNoSource;
      case B2S_WINDOW_LAG: return j - ps >= k ? j - k : kNoSource;
      case B2S_WINDOW_FIRST: return s < e + 1 ? s : kNoSource;
      case B2S_WINDOW_LAST: return s < e + 1 ? e : kNoSource;
      default: return s + k - 1 < e + 1 ? s + k - 1 : kNoSource;
    }
  }
  const uint64_t* r = io.rnk + (size_t)x * io.stride;
  const uint64_t lo = r[s];
  uint64_t q;
  switch (fn) {
    case B2S_WINDOW_LEAD:
      q = r[j + 1] + k - 1;
      if (q >= r[pe]) return kNoSource;
      break;
    case B2S_WINDOW_LAG:
      q = r[j];
      if (q < r[ps] + k) return kNoSource;
      q -= k;
      break;
    case B2S_WINDOW_FIRST:
      q = lo;
      if (q >= r[e + 1]) return kNoSource;
      break;
    case B2S_WINDOW_LAST:
      q = r[e + 1];
      if (q <= lo) return kNoSource;
      q -= 1;
      break;
    default:
      q = lo + k - 1;
      if (q >= r[e + 1]) return kNoSource;
      break;
  }
  return io.pres[(size_t)x * n + q];
}

// Offset function f's value at position j: a fixed-width value's slot bits, LAG / LEAD's default, or (strings and wide
// decimals) the source's sorted position for the emit; *null when it is null.  *extra grows by a string's bytes padded
// to 8.  Position j's own input is checked (so the verdict does not depend on the offsets): a bad one lowers *bad to its
// record's arena offset << 2 | kAggBadDecimal or kWindowBadBytes.
__device__ __forceinline__ uint64_t offset_value(const uint32_t* __restrict__ rec_len, const uint32_t* __restrict__ idx,
                                                 const WindowShape* __restrict__ sh, uint32_t f, const WindowOffIo& io,
                                                 uint64_t n, uint64_t j, uint64_t ps, uint64_t pe, uint64_t s,
                                                 uint64_t e, bool* null, uint64_t* extra, unsigned long long* bad) {
  const uint32_t vt = sh->vtype[f], k = val_kind(vt), voff = sh->voff[f];
  const int32_t vnull = sh->vnull[f];
  if (k == B2S_WINDOW_VAL_BYTES || wide_input(vt)) {
    const uint32_t i = at(idx, j);
    const uint8_t* row = io.arena + io.rec_off[i] + 4;
    if (!null_bit(row, vnull)) {
      const uint64_t slot = ld64(row + voff);
      const uint32_t size = rec_len[i] - 4;
      bool b = false;
      if (k == B2S_WINDOW_VAL_BYTES) {
        b = (slot >> 32) < 8ull * (sh->bw + sh->n) || (slot >> 32) + (uint32_t)slot > size;
      } else {
        uint64_t h, l;
        decimal_bits(row, size, slot, h, l, &b);
      }
      if (b)
        atomicMin(bad, (unsigned long long)((io.rec_off[i] << 2) |
                                            (k == B2S_WINDOW_VAL_BYTES ? kWindowBadBytes : kAggBadDecimal)));
    }
  }
  const uint64_t src = offset_source(sh, f, io, n, j, ps, pe, s, e);
  if (src == kNoSource) {
    *null = !(sh->flags[f] & B2S_WINDOW_HAS_DEFAULT);
    return *null ? 0 : sh->dflt[f];
  }
  const uint32_t i = at(idx, src);
  const uint8_t* row = io.arena + io.rec_off[i] + 4;
  *null = null_bit(row, vnull);
  if (*null) return 0;
  if (k == B2S_WINDOW_VAL_BYTES) {
    *extra += ((uint64_t)(uint32_t)ld64(row + voff) + 7) & ~7ull;
    return src;
  }
  return wide_input(vt) ? src : ld64(row + voff) & width_mask(k);
}

__global__ void __launch_bounds__(kWindowThreads) window_values_kernel(
    const uint32_t* __restrict__ rec_len, const uint32_t* __restrict__ idx, uint64_t n,
    const WindowShape* __restrict__ sh, const uint64_t* __restrict__ heads_before, const uint32_t* __restrict__ gpos,
    const uint64_t* __restrict__ groups, const uint64_t* __restrict__ phead, const uint32_t* __restrict__ pstart,
    uint64_t* __restrict__ vals, uint64_t* __restrict__ rows, uint64_t* __restrict__ bytes,
    uint64_t* __restrict__ readback, WindowAggIo io, WindowOffIo oio, WindowFrameIo fio) {
  const uint64_t G = *groups, P = phead[n];
  const uint32_t n_fns = sh->n_fns, limit_fn = sh->limit_fn;
  // what the output row adds to the input row, past the offset functions' strings
  const uint64_t grow = 8ull * (sh->out_bw - sh->bw + n_fns) + 16ull * (sh->n_wide + sh->n_wide_off);
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = next_scanned(heads_before, j, n, G) - 1, p = next_scanned(phead, j, n, P) - 1;
    const uint64_t ps = pstart[p], N = pstart[p + 1] - ps;
    const uint64_t i = j - ps, gs = gpos[g] - ps, ge = gpos[g + 1] - ps;
    const uint64_t dense = g - heads_before[ps] + 1;  // ps is a peer head: heads_before[ps] is its group
    if (N > 0x7fffffffull) readback[3] = 1;
    uint32_t nul = 0;
    uint64_t extra = 0;
    for (uint32_t f = 0; f < n_fns; f++) {
      uint64_t v;
      bool null = false;
      switch (sh->fn[f]) {
        case B2S_WINDOW_ROW_NUMBER: v = int_slot(i + 1); break;
        case B2S_WINDOW_RANK: v = int_slot(gs + 1); break;
        case B2S_WINDOW_DENSE_RANK: v = int_slot(dense); break;
        case B2S_WINDOW_PERCENT_RANK: v = __double_as_longlong(N > 1 ? (double)gs / (double)(N - 1) : 0.0); break;
        case B2S_WINDOW_CUME_DIST: v = __double_as_longlong((double)ge / (double)N); break;
        case B2S_WINDOW_NTILE: v = int_slot(ntile(i, N, sh->arg[f])); break;
        default: {
          const uint32_t fr = sh->frame[f];
          uint64_t s = ps, e = fr == B2S_WINDOW_FRAME_ROWS_RUNNING ? j
                               : fr == B2S_WINDOW_FRAME_RANGE_RUNNING ? ps + ge - 1 : ps + N - 1;
          if (is_sliding(fr)) {  // [s, e]: empty when e + 1 == s
            const size_t bx = (size_t)sh->bnd[f] * n + j;
            s = fio.fs[bx];
            e = (uint64_t)fio.ft[bx] - 1;
          }
          v = is_offset(sh->fn[f]) ? offset_value(rec_len, idx, sh, f, oio, n, j, ps, ps + N, s, e, &null, &extra,
                                                  (unsigned long long*)(readback + 4))
              : is_sliding(fr)     ? frame_agg_value(sh, f, io, fio, n, ps, s, e + 1, j, &null)
                                   : agg_value(sh, f, io, n, e, j, &null);
          break;
        }
      }
      vals[(size_t)f * n + j] = v;
      nul |= (uint32_t)null << f;
    }
    if (io.vnul) io.vnul[j] = nul;
    bool keep = true;
    if (limit_fn != B2S_WINDOW_NO_LIMIT) {
      const uint64_t lv = limit_fn == B2S_WINDOW_ROW_NUMBER ? i + 1 : limit_fn == B2S_WINDOW_RANK ? gs + 1 : dense;
      keep = lv <= (uint64_t)sh->limit;
    }
    const uint64_t size = rec_len[at(idx, j)] - 4 + extra;
    if (keep && size + grow > 0x7fffffffull) readback[2] = 1;
    rows[j] = keep;
    bytes[j] = keep ? 4 + size + grow : 0;
  }
}

// with a limit: kept[rows[j]] = j for each kept position j (rows: the scanned kept flags)
__global__ void __launch_bounds__(kWindowThreads) window_compact_kernel(uint64_t n, const uint64_t* __restrict__ rows,
                                                                        uint64_t out_rows, uint32_t* __restrict__ kept) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
    if (next_scanned(rows, j, n, out_rows) != rows[j]) kept[rows[j]] = (uint32_t)j;
}

// The map side's partial limit, a thread per sorted position j: its limit_fn value within its partition (row number,
// rank or dense rank, as window_values_kernel derives them), rows[j] = whether it is at most limit, bytes[j] = the
// kept record's length (else 0), and readback[3] = 1 for a partition of more than 2^31 - 1 records
__global__ void __launch_bounds__(kWindowThreads) window_limit_kernel(
    const uint32_t* __restrict__ rec_len, const uint32_t* __restrict__ idx, uint64_t n, uint32_t limit_fn,
    uint64_t limit, const uint64_t* __restrict__ heads_before, const uint32_t* __restrict__ gpos,
    const uint64_t* __restrict__ groups, const uint64_t* __restrict__ phead, const uint32_t* __restrict__ pstart,
    uint64_t* __restrict__ rows, uint64_t* __restrict__ bytes, uint64_t* __restrict__ readback) {
  const uint64_t G = *groups, P = phead[n];
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = next_scanned(heads_before, j, n, G) - 1, p = next_scanned(phead, j, n, P) - 1;
    const uint64_t ps = pstart[p];
    if (pstart[p + 1] - ps > 0x7fffffffull) readback[3] = 1;
    const uint64_t lv = limit_fn == B2S_WINDOW_ROW_NUMBER ? j - ps + 1
                        : limit_fn == B2S_WINDOW_RANK     ? gpos[g] - ps + 1
                                                          : g - heads_before[ps] + 1;  // ps is a peer head
    const bool keep = lv <= limit;
    rows[j] = keep;
    bytes[j] = keep ? rec_len[at(idx, j)] : 0;
  }
}

// Kept record t, by a warp: the record of the sorted position kept[t], unchanged, to dst + bytes[kept[t]] (the scanned
// kept lengths), its length to out_len[t]
__global__ void __launch_bounds__(kWindowThreads) window_limit_gather_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t out_rows, const uint32_t* __restrict__ kept,
    const uint64_t* __restrict__ bytes, uint32_t* __restrict__ out_len, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
  for (uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; t < out_rows; t += warps) {
    const uint64_t j = kept[t];
    const uint32_t i = at(idx, j), len = rec_len[i];
    warp_copy(dst + bytes[j], arena + rec_off[i], len, lane);
    if (lane == 0) out_len[t] = len;
  }
}

// Output row t, by a warp: the sorted position j = kept[t] (no limit: t) and its record; the output row is
// [out_bw null words: the input's n bits][the input's slots][the function slots][the input's var bytes]
__global__ void __launch_bounds__(kWindowThreads) window_emit_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t n, uint64_t out_rows, const uint32_t* __restrict__ kept,
    const WindowShape* __restrict__ sh, const uint64_t* __restrict__ vals, const uint64_t* __restrict__ bytes,
    const uint32_t* __restrict__ vnul, const uint64_t* __restrict__ vhi, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
  const uint32_t nf = sh->n, bw = sh->bw, b = sh->out_bw, n_fns = sh->n_fns, n_wide = sh->n_wide, n_off = sh->n_off;
  const uint32_t fixed_in = 8 * (bw + nf);
  const uint64_t fixed_out = 8ull * (b + nf + n_fns);
  const uint64_t shift = 8ull * (b - bw + n_fns) << 32;
  for (uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; t < out_rows; t += warps) {
    const uint64_t j = kept ? kept[t] : t;
    const uint32_t i = at(idx, j);
    const uint8_t* src = arena + rec_off[i] + 4;
    const uint64_t var = rec_len[i] - 4 - fixed_in;
    uint8_t* d = dst + bytes[j];
    uint8_t* row = d + 4;
    const uint32_t nul = vnul ? vnul[j] : 0;
    // lane f's var region (function f's, past the input's var bytes) starts vpre bytes in; every region's bytes: vall.
    // With offset functions the regions are sized per row: a lane per function, its source row (vrow) and an inclusive
    // warp scan of the sizes (16 per wide decimal, a non-null string's bytes padded to 8)
    uint64_t vpre = lane < n_fns && sh->wide[lane] >= 0 ? 16ull * (uint32_t)sh->wide[lane] : 0, vall = 16ull * n_wide;
    const uint8_t* vrow = nullptr;
    uint32_t vlen = 0;
    if (n_off) {
      uint64_t sz = 0;
      if (lane < n_fns) {
        const uint32_t vt = sh->vtype[lane];
        if (is_offset(sh->fn[lane]) && !((nul >> lane) & 1) && (val_kind(vt) == B2S_WINDOW_VAL_BYTES || wide_input(vt))) {
          const uint32_t s = at(idx, vals[(size_t)lane * n + j]);
          vrow = arena + rec_off[s] + 4;
          vlen = val_kind(vt) == B2S_WINDOW_VAL_BYTES ? (uint32_t)ld64(vrow + sh->voff[lane]) : rec_len[s] - 4;
        }
        sz = sh->wide[lane] >= 0 || (is_offset(sh->fn[lane]) && wide_input(vt)) ? 16
             : vrow ? ((uint64_t)vlen + 7) & ~7ull : 0;
      }
      uint64_t incl = sz;
#pragma unroll
      for (uint32_t o = 1; o < 32; o *= 2) {
        const uint64_t y = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += y;
      }
      vpre = incl - sz;
      vall = __shfl_sync(kFull, incl, 31);
    }
    if (lane == 0) st_span16(d, 4, __byte_perm((uint32_t)(fixed_out + var + vall), 0, 0x0123), 0);
    for (uint32_t w = lane; w < b; w += 32) {
      uint64_t bits = 0;
      if (w < bw) {
        bits = ld64(src + 8 * w);
        const uint64_t left = nf - 64ull * w;
        if (left < 64) bits &= (1ull << left) - 1;
      }
      for (uint32_t f = 0; f < n_fns; f++)  // the values' null bits nf + f
        if ((nul >> f) & 1 && (nf + f) >> 6 == w) bits |= 1ull << ((nf + f) & 63);
      st_span16(row + 8 * w, 8, bits, 0);
    }
    warp_copy(row + 8 * b, src + 8 * bw, 8ull * nf, lane);
    if (lane < n_fns) {
      const uint32_t f = lane;
      uint64_t slot = vals[(size_t)f * n + j];
      const int32_t k = sh->wide[f];
      const uint64_t off = fixed_out + var + vpre;
      const bool wide_off = n_off && is_offset(sh->fn[f]) && wide_input(sh->vtype[f]);
      if (k >= 0 || wide_off) {  // 16 bytes in its region: BigInteger.toByteArray's, or zeros when null
        uint64_t m0 = 0, m1 = 0;
        if ((nul >> f) & 1) {
          slot = off << 32;
        } else {
          Dec128 x{slot, 0};
          if (wide_off) {  // the source's bytes, re-encoded minimally
            bool unused = false;
            decimal_bits(vrow, vlen, ld64(vrow + sh->voff[f]), x.hi, x.lo, &unused);
            x.hi ^= 1ull << 63;
          } else {
            x.hi = vhi[(size_t)k * n + j];
          }
          const uint32_t len = dec_bytes(x);
          dec_encode(x, len, &m0, &m1);
          slot = off << 32 | len;
        }
        st_span16(row + off, 16, m0, m1);
      } else if (vrow) {  // a string: its bytes follow below
        slot = off << 32 | vlen;
      }
      st_span16(row + 8 * (b + nf + f), 8, slot, 0);
    }
    warp_copy(row + fixed_out, src + fixed_in, var, lane);
    // the offset functions' strings, each by the whole warp, zero-padded to 8 bytes
    for (uint32_t f = 0; n_off && f < n_fns; f++) {
      const uint8_t* s = (const uint8_t*)__shfl_sync(kFull, (unsigned long long)vrow, f);
      if (!s || val_kind(sh->vtype[f]) != B2S_WINDOW_VAL_BYTES) continue;
      const uint32_t len = __shfl_sync(kFull, vlen, f);
      const uint64_t off = fixed_out + var + __shfl_sync(kFull, vpre, f);
      warp_copy(row + off, s + (uint32_t)(ld64(s + sh->voff[f]) >> 32), len, lane);
      if (lane == 0 && (len & 7)) st_span16(row + off + len, 8 - (len & 7), 0, 0);
    }
    __syncwarp();
    // a zero slot (a null string) stays zero
    for (uint32_t x = lane; x < sh->n_var; x += 32) {
      const uint32_t f = sh->var[x];
      const uint64_t slot = ld64(src + 8 * (bw + f));
      if (slot) st_span16(row + 8 * (b + f), 8, slot + shift, 0);
    }
    __syncwarp();
  }
}

}  // namespace

size_t window_ws_bytes(uint64_t n, const WindowShape& shape) {
  return reinterpret_cast<uintptr_t>(carve_window_ws(nullptr, n, shape).end);  // the parts' offsets from 0
}

uint64_t* window_readback(uint8_t* d_wws, uint64_t n, const WindowShape& shape) {
  return carve_window_ws(d_wws, n, shape).readback;
}

// the partitions of the peer groups in d_aws (the shape uploaded to w.shape): head flags scanned into w.phead (the count
// at [n]), the partitions' first positions into w.pstart
static void launch_window_partitions(const uint8_t* arena, uint64_t n, const uint32_t* idx, const KeySortWs& k,
                                     const WindowWs& w, uint8_t* d_aws, cudaStream_t st, uint64_t* launches) {
  window_part_heads_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(arena, k.src_off, k.len, idx, n, w.shape,
                                                                   rows_group_heads_before(d_aws, n),
                                                                   rows_aggregate_readback(d_aws, n, 0, 0), w.phead);
  launch_exclusive_scan_u64(w.phead, n, w.phead + n, w.scan_ws, st, launches);
  window_part_starts_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(w.phead, n, w.pstart);
  if (launches) *launches += 2;
}

void launch_window_values(const uint8_t* arena, uint64_t n, const uint32_t* idx, WindowShape shape,
                          const uint32_t* h_fields, uint32_t key_bytes, uint8_t* d_ws, uint8_t* d_aws, uint8_t* d_wws,
                          cudaStream_t st, uint64_t* launches) {
  const WindowWs w = carve_window_ws(d_wws, n, shape);
  const KeySortWs k = carve_key_sort_ws(d_ws, n, key_bytes);
  shape.var = w.fields;
  cudaMemcpyAsync(w.shape, &shape, sizeof(WindowShape), cudaMemcpyHostToDevice, st);
  if (shape.n_var) cudaMemcpyAsync(w.fields, h_fields, (size_t)shape.n_var * 4, cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(w.readback, 0, kWindowReadbackBytes, st);
  cudaMemsetAsync(w.readback + 4, 0xff, 8, st);
  const uint64_t* heads_before = rows_group_heads_before(d_aws, n);
  const uint64_t* groups = rows_aggregate_readback(d_aws, n, 0, 0);
  launch_window_partitions(arena, n, idx, k, w, d_aws, st, launches);
  const WindowFrameIo fio{w.fs, w.ft, w.rlo[0], w.rhi[0], w.rcnt[0]};
  if (shape.n_bnd) {  // sliding frames: the order column staged for a RANGE offset, then every bounds set's frames
    if (shape.ord_staged)
      window_order_stage_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(arena, k.src_off, idx, n, w.shape, w.ov,
                                                                         w.onull);
    window_bounds_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(
        n, w.shape, heads_before, rows_group_starts(d_aws, n), groups, w.phead, w.pstart,
        shape.ord_staged ? w.ov : nullptr, w.onull, w.fs, w.ft, w.readback);
    if (launches) *launches += 1 + shape.ord_staged;
  }
  WindowOffIo oio{arena, k.src_off, nullptr, nullptr, w.stride};
  if (shape.n_nn) {  // the non-null indexes: present flags, a scan each, the present positions compacted
    window_present_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(arena, k.src_off, idx, n, w.shape, w.stride, w.rnk);
    for (uint32_t x = 0; x < shape.n_nn; x++) {
      uint64_t* r = w.rnk + (size_t)x * w.stride;
      launch_exclusive_scan_u64(r, n, r + n, w.scan_ws, st, launches);
    }
    window_pres_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(n, shape.n_nn, w.stride, w.rnk, w.pres);
    oio.rnk = w.rnk;
    oio.pres = w.pres;
    if (launches) *launches += 2;
  }
  WindowAggIo io{};
  io.vnul = shape.n_off ? w.vnul : nullptr;
  if (shape.n_agg) {
    bool scans = false, folds = false, rmq = false, frame_folds = false;
    for (uint32_t f = 0; f < shape.n_fns; f++) {
      if (!is_agg(shape.fn[f])) continue;
      const uint32_t kind = shape.vtype[f] & 0xff;
      const bool dbl = (shape.fn[f] == B2S_WINDOW_SUM &&
                        (kind == B2S_WINDOW_VAL_FLOAT32 || kind == B2S_WINDOW_VAL_FLOAT64)) ||
                       (shape.fn[f] == B2S_WINDOW_AVG && kind != B2S_WINDOW_VAL_DECIMAL);
      // a sliding frame's own result state replaces the prefix folds
      if (shape.res[f] >= 0) (dbl ? frame_folds : rmq) = true;
      else (dbl ? folds : scans) = true;
    }
    window_stage_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(arena, k.src_off, k.len, idx, n, w.shape, w.lo[0],
                                                                w.hi[0], w.cnt[0],
                                                                (unsigned long long*)(w.readback + 4));
    // the sliding frames read the staged inputs (set 0) before the scans and the running fold overwrite them; the
    // range-minimum passes read levels 0 .. floor(log2(the widest frame))
    uint32_t levels = 0;
    for (uint64_t wmax = std::min<uint64_t>(shape.rmq_width, n); rmq && wmax; wmax >>= 1) levels++;
    for (uint32_t lv = 0; lv < levels; lv++) {
      const int in = lv & 1 ? 1 : 2, out = lv & 1 ? 2 : 1;  // level lv in rlo[in] (level 0: the staged set)
      window_rmq_pass_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(
          n, w.shape, w.fs, w.ft, lv, lv == 0, lv + 1 < levels, lv ? w.rlo[in] : w.lo[0],
          lv ? w.rhi[in] : w.hi[0], lv ? w.rcnt[in] : w.cnt[0], w.rlo[out], w.rhi[out], w.rcnt[out], w.rlo[0],
          w.rhi[0], w.rcnt[0]);
    }
    if (frame_folds)
      window_frame_fold_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(n, w.shape, w.fs, w.ft, w.lo[0], w.cnt[0],
                                                                       w.rlo[0], w.rcnt[0]);
    if (launches) *launches += levels + frame_folds;
    int cur = 0;  // the set holding the scanned folds
    for (uint64_t d = 1; scans && d < n; d *= 2, cur ^= 1)
      window_scan_pass_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(n, w.shape, w.phead, w.pstart, d, w.lo[cur],
                                                                      w.hi[cur], w.cnt[cur], w.lo[cur ^ 1],
                                                                      w.hi[cur ^ 1], w.cnt[cur ^ 1]);
    if (folds) {
      const uint64_t want = (n + kWindowThreads / 32 - 1) / (kWindowThreads / 32);  // at most a warp per partition
      const unsigned grid = (unsigned)std::min<uint64_t>(want, (uint64_t)kSMs * 16);
      window_fold_kernel<<<grid, kWindowThreads, 0, st>>>(n, w.shape, w.phead, w.pstart, w.lo[0], w.cnt[0],
                                                          w.lo[cur], w.cnt[cur]);
    }
    io = WindowAggIo{w.lo[cur], w.hi[cur], w.cnt[cur], w.vnul, w.vhi};
    if (launches) {
      uint64_t passes = 0;
      for (uint64_t d = 1; scans && d < n; d *= 2) passes++;
      *launches += 1 + passes + folds;
    }
  }
  window_values_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(k.len, idx, n, w.shape, heads_before,
                                                               rows_group_starts(d_aws, n), groups, w.phead, w.pstart,
                                                               w.vals, w.rows, w.bytes, w.readback, io, oio, fio);
  launch_exclusive_scan_u64(w.rows, n, w.readback, w.scan_ws, st, launches);
  launch_exclusive_scan_u64(w.bytes, n, w.readback + 1, w.scan_ws, st, launches);
  if (launches) *launches += 1;
}

void launch_window_emit(const uint8_t* arena, uint64_t n, const uint32_t* idx, uint64_t out_rows, uint32_t key_bytes,
                        const WindowShape& shape, bool limited, uint8_t* d_ws, uint8_t* d_wws, uint8_t* d_dst,
                        cudaStream_t st, uint64_t* launches) {
  if (!out_rows) return;
  const WindowWs w = carve_window_ws(d_wws, n, shape);
  const KeySortWs k = carve_key_sort_ws(d_ws, n, key_bytes);
  if (limited) {
    window_compact_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(n, w.rows, out_rows, w.kept);
    if (launches) *launches += 1;
  }
  const uint64_t want = (out_rows + kWindowThreads / 32 - 1) / (kWindowThreads / 32);
  const unsigned grid = (unsigned)std::min<uint64_t>(want, (uint64_t)kSMs * 16);
  window_emit_kernel<<<grid, kWindowThreads, 0, st>>>(arena, k.src_off, k.len, idx, n, out_rows,
                                                      limited ? w.kept : nullptr, w.shape, w.vals, w.bytes,
                                                      shape.n_agg || shape.n_off ? w.vnul : nullptr, w.vhi, d_dst);
  if (launches) *launches += 1;
}

void launch_window_limit(const uint8_t* arena, uint64_t n, const uint32_t* idx, const WindowShape& shape,
                         uint32_t key_bytes, uint8_t* d_ws, uint8_t* d_aws, uint8_t* d_wws, cudaStream_t st,
                         uint64_t* launches) {
  const WindowWs w = carve_window_ws(d_wws, n, shape);
  const KeySortWs k = carve_key_sort_ws(d_ws, n, key_bytes);
  cudaMemcpyAsync(w.shape, &shape, sizeof(WindowShape), cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(w.readback, 0, kWindowReadbackBytes, st);
  launch_window_partitions(arena, n, idx, k, w, d_aws, st, launches);
  window_limit_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(
      k.len, idx, n, shape.limit_fn, (uint64_t)shape.limit, rows_group_heads_before(d_aws, n),
      rows_group_starts(d_aws, n), rows_aggregate_readback(d_aws, n, 0, 0), w.phead, w.pstart, w.rows, w.bytes,
      w.readback);
  launch_exclusive_scan_u64(w.rows, n, w.readback, w.scan_ws, st, launches);
  launch_exclusive_scan_u64(w.bytes, n, w.readback + 1, w.scan_ws, st, launches);
  if (launches) *launches += 1;
}

void launch_window_limit_gather(const uint8_t* arena, uint64_t n, const uint32_t* idx, uint64_t out_rows,
                                uint32_t key_bytes, const WindowShape& shape, uint8_t* d_ws, uint8_t* d_wws,
                                uint32_t* d_out_len, uint8_t* d_out, cudaStream_t st, uint64_t* launches) {
  if (!out_rows) return;
  const WindowWs w = carve_window_ws(d_wws, n, shape);
  const KeySortWs k = carve_key_sort_ws(d_ws, n, key_bytes);
  window_compact_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(n, w.rows, out_rows, w.kept);
  const uint64_t want = (out_rows + kWindowThreads / 32 - 1) / (kWindowThreads / 32);
  const unsigned grid = (unsigned)std::min<uint64_t>(want, (uint64_t)kSMs * 16);
  window_limit_gather_kernel<<<grid, kWindowThreads, 0, st>>>(arena, k.src_off, k.len, idx, out_rows, w.kept, w.bytes,
                                                              d_out_len, d_out);
  if (launches) *launches += 2;
}

}  // namespace b2s
