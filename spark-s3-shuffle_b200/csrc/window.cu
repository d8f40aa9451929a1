// window.cu — Spark's WindowExec on a reducer for the ranking functions (row_number, rank, dense_rank, percent_rank,
// cume_dist, ntile), with WindowGroupLimitExec's limit, and the output rows built as UnsafeRowJoiner joins the input
// row with the row of values.  The records have been framed, keyed by the whole window key (partition columns, then
// order columns), stably sorted by rows.cu and grouped by aggregate.cu's launch_rows_group, whose groups are the peer
// groups.  All on the device:
//   heads  : one thread per sorted position: a partition starts at a peer head whose partition columns differ from its
//            predecessor's, compared by encode_key 16 encoded bytes at a time until they differ or both keys end (so
//            the equality is the sort's: strings by length and bytes, -0.0 with 0.0, NaN with NaN, null with null);
//            the flags scanned, and each partition's first position compacted
//   values : one thread per sorted position: from its partition's bounds and its peer group's bounds and index, every
//            function's value (into a per-function array in sorted order), whether the limit keeps it, and its output
//            bytes; the kept records and the bytes scanned, and the totals and the too-long and too-large-partition
//            flags come back in one readback
//   emit   : a warp per output row (with a limit, over the compacted kept positions only): its null words widened, its
//            slots, the function slots and its var bytes, then the VAR and DECIMAL_WIDE slots' offsets moved
#include <algorithm>

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
// and its field list
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
};

WindowWs carve_window_ws(uint8_t* d_wws, uint64_t n, uint32_t n_fns) {
  WindowWs w;
  uint8_t* p = d_wws;
  w.phead = (uint64_t*)p;    p += a256((n + 1) * 8);
  w.pstart = (uint32_t*)p;   p += a256((n + 1) * 4);
  w.vals = (uint64_t*)p;     p += a256((size_t)n_fns * n * 8);
  w.rows = (uint64_t*)p;     p += a256(n * 8);
  w.bytes = (uint64_t*)p;    p += a256(n * 8);
  w.kept = (uint32_t*)p;     p += a256(n * 4);
  w.scan_ws = (uint64_t*)p;  p += a256(scan_ws_elems(n + 1) * 8);
  w.readback = (uint64_t*)p; p += a256(kWindowReadbackBytes);
  w.shape = (WindowShape*)p; p += a256(sizeof(WindowShape));
  w.fields = (uint32_t*)p;
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
      const uint8_t *ra = arena + rec_off[a] + 4, *rb = arena + rec_off[b] + 4;
      const uint32_t sa = rec_len[a] - 4, sb = rec_len[b] - 4;
      bool bad = false;  // the sort's key pass has checked every string and decimal
      for (uint32_t d = 0;; d += kKeyChunkBytes) {
        KeyWindow wa{0, 0, 0, 0, 0, d, kKeyChunkBytes}, wb{0, 0, 0, 0, 0, d, kKeyChunkBytes};
        const uint32_t la = encode_key(ra, sa, ks, wa, false, &bad);
        const uint32_t lb = encode_key(rb, sb, ks, wb, false, &bad);
        if (wa.w0 != wb.w0 || wa.w1 != wb.w1 || wa.w2 != wb.w2 || wa.w3 != wb.w3) {
          h = 1;
          break;
        }
        // equal so far and one key ended inside the window: the encoding is prefix-free, so both did
        if (min(la, lb) < d + kKeyChunkBytes) break;
      }
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

__global__ void __launch_bounds__(kWindowThreads) window_values_kernel(
    const uint32_t* __restrict__ rec_len, const uint32_t* __restrict__ idx, uint64_t n,
    const WindowShape* __restrict__ sh, const uint64_t* __restrict__ heads_before, const uint32_t* __restrict__ gpos,
    const uint64_t* __restrict__ groups, const uint64_t* __restrict__ phead, const uint32_t* __restrict__ pstart,
    uint64_t* __restrict__ vals, uint64_t* __restrict__ rows, uint64_t* __restrict__ bytes,
    uint64_t* __restrict__ readback) {
  const uint64_t G = *groups, P = phead[n];
  const uint32_t n_fns = sh->n_fns, limit_fn = sh->limit_fn;
  const uint64_t grow = 8ull * (sh->out_bw - sh->bw + n_fns);  // what the output row adds to the input row
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t g = next_scanned(heads_before, j, n, G) - 1, p = next_scanned(phead, j, n, P) - 1;
    const uint64_t ps = pstart[p], N = pstart[p + 1] - ps;
    const uint64_t i = j - ps, gs = gpos[g] - ps, ge = gpos[g + 1] - ps;
    const uint64_t dense = g - heads_before[ps] + 1;  // ps is a peer head: heads_before[ps] is its group
    if (N > 0x7fffffffull) readback[3] = 1;
    for (uint32_t f = 0; f < n_fns; f++) {
      uint64_t v;
      switch (sh->fn[f]) {
        case B2S_WINDOW_ROW_NUMBER: v = int_slot(i + 1); break;
        case B2S_WINDOW_RANK: v = int_slot(gs + 1); break;
        case B2S_WINDOW_DENSE_RANK: v = int_slot(dense); break;
        case B2S_WINDOW_PERCENT_RANK: v = __double_as_longlong(N > 1 ? (double)gs / (double)(N - 1) : 0.0); break;
        case B2S_WINDOW_CUME_DIST: v = __double_as_longlong((double)ge / (double)N); break;
        default: v = int_slot(ntile(i, N, sh->arg[f])); break;
      }
      vals[(size_t)f * n + j] = v;
    }
    bool keep = true;
    if (limit_fn != B2S_WINDOW_NO_LIMIT) {
      const uint64_t lv = limit_fn == B2S_WINDOW_ROW_NUMBER ? i + 1 : limit_fn == B2S_WINDOW_RANK ? gs + 1 : dense;
      keep = lv <= (uint64_t)sh->limit;
    }
    const uint64_t size = rec_len[at(idx, j)] - 4;
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

// Output row t, by a warp: the sorted position j = kept[t] (no limit: t) and its record; the output row is
// [out_bw null words: the input's n bits][the input's slots][the function slots][the input's var bytes]
__global__ void __launch_bounds__(kWindowThreads) window_emit_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t n, uint64_t out_rows, const uint32_t* __restrict__ kept,
    const WindowShape* __restrict__ sh, const uint64_t* __restrict__ vals, const uint64_t* __restrict__ bytes,
    uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
  const uint32_t nf = sh->n, bw = sh->bw, b = sh->out_bw, n_fns = sh->n_fns;
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
    if (lane == 0) st_span16(d, 4, __byte_perm((uint32_t)(fixed_out + var), 0, 0x0123), 0);
    for (uint32_t w = lane; w < b; w += 32) {
      uint64_t bits = 0;
      if (w < bw) {
        bits = ld64(src + 8 * w);
        const uint64_t left = nf - 64ull * w;
        if (left < 64) bits &= (1ull << left) - 1;
      }
      st_span16(row + 8 * w, 8, bits, 0);
    }
    warp_copy(row + 8 * b, src + 8 * bw, 8ull * nf, lane);
    for (uint32_t f = lane; f < n_fns; f += 32) st_span16(row + 8 * (b + nf + f), 8, vals[(size_t)f * n + j], 0);
    warp_copy(row + fixed_out, src + fixed_in, var, lane);
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

size_t window_ws_bytes(uint64_t n, uint32_t n_fns, uint32_t n_fields) {
  return a256((n + 1) * 8) + a256((n + 1) * 4) + a256((size_t)n_fns * n * 8) + 2 * a256(n * 8) + a256(n * 4) +
         a256(scan_ws_elems(n + 1) * 8) + a256(kWindowReadbackBytes) + a256(sizeof(WindowShape)) +
         a256((size_t)n_fields * 4);
}

uint64_t* window_readback(uint8_t* d_wws, uint64_t n, uint32_t n_fns) {
  return carve_window_ws(d_wws, n, n_fns).readback;
}

void launch_window_values(const uint8_t* arena, uint64_t n, const uint32_t* idx, WindowShape shape,
                          const uint32_t* h_fields, uint32_t key_bytes, uint8_t* d_ws, uint8_t* d_aws, uint8_t* d_wws,
                          cudaStream_t st, uint64_t* launches) {
  const WindowWs w = carve_window_ws(d_wws, n, shape.n_fns);
  const KeySortWs k = carve_key_sort_ws(d_ws, n, key_bytes);
  shape.var = w.fields;
  cudaMemcpyAsync(w.shape, &shape, sizeof(WindowShape), cudaMemcpyHostToDevice, st);
  if (shape.n_var) cudaMemcpyAsync(w.fields, h_fields, (size_t)shape.n_var * 4, cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(w.readback, 0, kWindowReadbackBytes, st);
  const uint64_t* heads_before = rows_group_heads_before(d_aws, n);
  const uint64_t* groups = rows_aggregate_readback(d_aws, n, 0, 0);
  window_part_heads_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(arena, k.src_off, k.len, idx, n, w.shape,
                                                                   heads_before, groups, w.phead);
  launch_exclusive_scan_u64(w.phead, n, w.phead + n, w.scan_ws, st, launches);
  window_part_starts_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(w.phead, n, w.pstart);
  window_values_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(k.len, idx, n, w.shape, heads_before,
                                                               rows_group_starts(d_aws, n), groups, w.phead, w.pstart,
                                                               w.vals, w.rows, w.bytes, w.readback);
  launch_exclusive_scan_u64(w.rows, n, w.readback, w.scan_ws, st, launches);
  launch_exclusive_scan_u64(w.bytes, n, w.readback + 1, w.scan_ws, st, launches);
  if (launches) *launches += 3;
}

void launch_window_emit(const uint8_t* arena, uint64_t n, const uint32_t* idx, uint64_t out_rows, uint32_t key_bytes,
                        uint32_t n_fns, bool limited, uint8_t* d_ws, uint8_t* d_wws, uint8_t* d_dst, cudaStream_t st,
                        uint64_t* launches) {
  if (!out_rows) return;
  const WindowWs w = carve_window_ws(d_wws, n, n_fns);
  const KeySortWs k = carve_key_sort_ws(d_ws, n, key_bytes);
  if (limited) {
    window_compact_kernel<<<grid_for(n), kWindowThreads, 0, st>>>(n, w.rows, out_rows, w.kept);
    if (launches) *launches += 1;
  }
  const uint64_t want = (out_rows + kWindowThreads / 32 - 1) / (kWindowThreads / 32);
  const unsigned grid = (unsigned)std::min<uint64_t>(want, (uint64_t)kSMs * 16);
  window_emit_kernel<<<grid, kWindowThreads, 0, st>>>(arena, k.src_off, k.len, idx, n, out_rows,
                                                      limited ? w.kept : nullptr, w.shape, w.vals, w.bytes, d_dst);
  if (launches) *launches += 1;
}

}  // namespace b2s
