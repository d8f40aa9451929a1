// join.cu — the merge of a sort-merge join on a reducer: Spark's SortMergeJoinExec over its two shuffled inputs, with
// the joined rows built as UnsafeRowJoiner builds them.  Both sides' records have been framed, keyed (each with its own
// layout) and stably sorted together by rows.cu, and grouped by aggregate.cu's launch_rows_group, so every group of
// equal keys holds that key's left records in their sorted order followed by its right ones.  All on the device:
//   var   : one thread per sorted position: its record's variable-length bytes (its row past the null words and
//           slots), scanned in sorted order, so a group's var bytes of either side are a difference of two prefixes
//           (its left records span [group start, first right), its right ones [first right, group end)); each group's
//           largest per side, for the 2^31 - 1 row limit
//   count : one thread per sorted position of either side: its group's first right position (a search: left records
//           come first), so the group's left and right counts, its key's nulls (a null key matches nothing; a group
//           matches when its key has no null and it holds records of both sides), and from the join type the output
//           records and bytes the record drives: a left record its rows with the group's right records (inner, left
//           and full outer), a right record its rows with the group's left records (right outer), either one row with
//           a null other side when its group does not match (left, right and full outer: a full outer join's right
//           records only then), or (existence) a left record its own row with the exists field; both are scanned, and the totals, the left record count and the too-long flag come
//           back in one readback
//   emit  : a warp per output record, whose driving position is found by a search in the scanned output record counts,
//           so a hot key's many joined rows spread over the whole GPU; its partner is the k-th record of the other
//           side's part of the group, or a null side.  A joined row is [null words][left slots][right slots][left
//           var][right var]: the four spans are copied 16 bytes per lane, the null words built from both sides' bits,
//           and the slots of VAR and DECIMAL_WIDE fields moved by their side's shift; a null side has its bits set, its
//           slots zero and 16 zero bytes for each DECIMAL_WIDE field.  A semi or anti join compacts its kept left
//           positions and gathers those records with the row sort's gather.  An existence join's rows are emitted by a
//           warp per left position: the record with one more fixed field, as the window emit builds its rows.
#include <algorithm>

#include "kernels.h"

namespace b2s {

namespace {

constexpr int kJoinThreads = 256;

inline size_t a256(size_t b) { return (b + 255) / 256 * 256; }

inline unsigned grid_for(uint64_t n) {
  const uint64_t want = (n + kJoinThreads - 1) / kJoinThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

// the join workspace: per position the output records and bytes (scanned in place), the var bytes (scanned, the total
// at [n]), the first position of its partners (semi and anti joins: the kept records, in output order); per group and
// side the largest var bytes; scan workspace, readback, the shape and its field lists
struct JoinWs {
  uint64_t* rows;
  uint64_t* bytes;
  uint64_t* var;
  uint32_t* rpos;
  uint32_t* gmax;
  uint64_t* scan_ws;
  uint64_t* readback;
  JoinShape* shape;
  uint32_t* fields;
};

JoinWs carve_join_ws(uint8_t* d_jws, uint64_t n, uint32_t n_ranges) {
  JoinWs j;
  uint8_t* p = d_jws;
  j.rows = (uint64_t*)p;     p += a256(n * 8);
  j.bytes = (uint64_t*)p;    p += a256(n * 8);
  j.var = (uint64_t*)p;      p += a256((n + 1) * 8);
  j.rpos = (uint32_t*)p;     p += a256(n * 4);
  j.gmax = (uint32_t*)p;     p += a256(2 * n * 4);
  j.scan_ws = (uint64_t*)p;  p += a256(scan_ws_elems(n + 1) * 8);
  j.readback = (uint64_t*)p; p += a256(join_readback_bytes(n_ranges));
  j.shape = (JoinShape*)p;   p += a256(sizeof(JoinShape));
  j.fields = (uint32_t*)p;
  return j;
}

__device__ __forceinline__ uint32_t at(const uint32_t* idx, uint64_t j) { return idx ? idx[j] : (uint32_t)j; }

__device__ __forceinline__ uint64_t ld64(const uint8_t* p) {
  uint64_t lo, unused;
  ld_span16<true>(p, 8, lo, unused);
  return lo;
}

// word k of the first nbits bits of a row's null bitset (ones: every one of them set), 0 outside it
__device__ __forceinline__ uint64_t bits_word(const uint8_t* row, uint32_t nbits, int64_t k, bool ones) {
  if (k < 0 || (uint64_t)k * 64 >= nbits) return 0;
  const uint64_t w = ones ? ~0ull : ld64(row + 8 * k);
  const uint64_t left = nbits - (uint64_t)k * 64;
  return left >= 64 ? w : w & ((1ull << left) - 1);
}

// the group of position j (heads_before: the heads before each position; G groups)
__device__ __forceinline__ uint64_t group_of(const uint64_t* heads_before, uint64_t j, uint64_t n, uint64_t G) {
  return (j + 1 < n ? heads_before[j + 1] : G) - 1;
}

__global__ void __launch_bounds__(kJoinThreads) join_var_kernel(const uint64_t* __restrict__ rec_off,
                                                                const uint32_t* __restrict__ rec_len,
                                                                const uint32_t* __restrict__ idx, uint64_t n,
                                                                const JoinShape* __restrict__ sh,
                                                                const uint64_t* __restrict__ heads_before,
                                                                const uint64_t* __restrict__ groups,
                                                                uint64_t* __restrict__ var, uint32_t* __restrict__ gmax,
                                                                uint64_t* __restrict__ readback) {
  const uint64_t split = sh->split, G = *groups;
  const uint32_t fixed_l = 8 * (sh->bw[0] + sh->n[0]), fixed_r = 8 * (sh->bw[1] + sh->n[1]);
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    // arena order: the last left record gives the left count
    if (rec_off[j] < split && (j + 1 == n || rec_off[j + 1] >= split)) readback[2] = j + 1;
    const uint32_t i = at(idx, j);
    const bool right = rec_off[i] >= split;
    const uint32_t fixed = right ? fixed_r : fixed_l;
    uint32_t v = 0;
    if (rec_len[i] - 4 >= fixed) {  // a shorter row fails the call (the key pass's verdict)
      v = rec_len[i] - 4 - fixed;
      uint32_t* m = gmax + 2 * group_of(heads_before, j, n, G) + right;
      if (v > *m) atomicMax(m, v);
    }
    var[j] = v;
  }
}

constexpr uint32_t kNoMatch = 0xffffffffu;  // rpos of a position without partners (none, or a null other side)

__global__ void __launch_bounds__(kJoinThreads) join_count_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t n, const JoinShape* __restrict__ sh,
    const uint64_t* __restrict__ heads_before, const uint32_t* __restrict__ gpos, const uint64_t* __restrict__ groups,
    const uint64_t* __restrict__ var, const uint32_t* __restrict__ gmax, uint64_t* __restrict__ rows,
    uint64_t* __restrict__ bytes, uint32_t* __restrict__ rpos, uint64_t* __restrict__ readback) {
  const uint64_t split = sh->split, G = *groups;
  const uint32_t type = sh->type;
  const uint64_t fixed_out = 8ull * (sh->out_bw + sh->n[0] + sh->n[1]);
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = at(idx, j);
    const uint32_t right = rec_off[i] >= split;
    const uint32_t size = rec_len[i] - 4, fixed = 8 * (sh->bw[right] + sh->n[right]);
    uint64_t r = 0, b = 0;
    uint32_t partner = kNoMatch;
    // a row shorter than its fixed region fails the call (the key pass's verdict): not read, no output
    if (size >= fixed && !(right && (join_keeps_whole(type) || type == kJoinExistence))) {
      const uint64_t g = group_of(heads_before, j, n, G), s = gpos[g], e = gpos[g + 1];
      uint64_t lo = right ? s : j + 1, hi = right ? j : e;  // the group's first right position: left records come first
      while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        if (rec_off[at(idx, mid)] >= split) hi = mid;
        else lo = mid + 1;
      }
      const uint8_t* row = arena + rec_off[i] + 4;
      const KeySpec& ks = sh->keys[right];
      bool null = false;
      for (uint32_t c = 0; c < ks.n; c++) {
        const int32_t f = ks.null_field[c];
        if (f >= 0) null |= (ld64(row + 8 * (uint32_t)(f >> 6)) >> (f & 63)) & 1;
      }
      const uint64_t L = lo - s, R = e - lo;
      const bool matched = L && R && !null;
      const uint64_t var_own = size - fixed;
      // a left record drives its rows in every join but right outer, a right record only there
      const bool drives = right ? type == kJoinRightOuter : type != kJoinRightOuter;
      if (join_keeps_whole(type)) {
        r = matched == (type == kJoinLeftSemi);
        b = r ? 4 + (uint64_t)size : 0;
      } else if (type == kJoinExistence) {  // its row grows by the null words it adds and the exists slot
        r = 1;
        b = 4 + (uint64_t)size + 8ull * (sh->out_bw - sh->bw[0] + 1);
        if (b - 4 > 0x7fffffffull) readback[3] = 1;
        partner = matched;
      } else if (drives && matched) {  // one row with each record of the other side's part of the group
        r = right ? L : R;
        b = r * (4 + fixed_out + var_own) + (right ? var[lo] - var[s] : var[e] - var[lo]);
        if (fixed_out + var_own + gmax[2 * g + !right] > 0x7fffffffull) readback[3] = 1;
        partner = (uint32_t)(right ? s : lo);
      } else if (drives ? type != kJoinInner : type == kJoinFullOuter && !matched) {  // one row, the other side null
        r = 1;
        b = 4 + fixed_out + var_own + 16ull * sh->n_wide[!right];
        if (b - 4 > 0x7fffffffull) readback[3] = 1;
      }
    }
    rpos[j] = partner;
    rows[j] = r;
    bytes[j] = b;
  }
}

// semi and anti joins: the kept left positions (one output row each) compacted, kept[rows[j]] = the record at j
__global__ void __launch_bounds__(kJoinThreads) join_compact_kernel(const uint32_t* __restrict__ idx, uint64_t n,
                                                                    const uint64_t* __restrict__ rows,
                                                                    uint64_t out_rows, uint32_t* __restrict__ kept) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
    if ((j + 1 < n ? rows[j + 1] : out_rows) != rows[j]) kept[rows[j]] = at(idx, j);
}

// Output record t, by a warp: its driving position j (the last whose first output record is at or before t) and the
// k-th record of its partners, or a null other side (rpos[j] = kNoMatch)
__global__ void __launch_bounds__(kJoinThreads) join_emit_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t n, uint64_t out_rows, const JoinShape* __restrict__ sh,
    const uint64_t* __restrict__ rows, const uint64_t* __restrict__ bytes, const uint64_t* __restrict__ var,
    const uint32_t* __restrict__ rpos, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
  const uint64_t split = sh->split;
  const uint32_t nl = sh->n[0], nr = sh->n[1], bl = sh->bw[0], br = sh->bw[1], b = sh->out_bw;
  const uint32_t fixed_l = 8 * (bl + nl), fixed_r = 8 * (br + nr);
  const uint64_t fixed_out = 8ull * (b + nl + nr);
  for (uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; t < out_rows; t += warps) {
    uint64_t lo = 0, hi = n;
    while (hi - lo > 1) {
      const uint64_t mid = (lo + hi) / 2;
      if (rows[mid] <= t) lo = mid;
      else hi = mid;
    }
    const uint64_t j = lo, k = t - rows[j];
    const uint32_t di = at(idx, j);
    const bool right = rec_off[di] >= split;  // the driving record's side
    const uint8_t* D = arena + rec_off[di] + 4;
    const uint64_t var_d = rec_len[di] - 4 - (right ? fixed_r : fixed_l);
    uint8_t* d = dst + bytes[j];
    const uint32_t ps = rpos[j];
    const uint8_t* P = nullptr;
    uint64_t var_p = 16ull * sh->n_wide[!right];
    if (ps != kNoMatch) {
      const uint32_t pi = at(idx, ps + k);
      P = arena + rec_off[pi] + 4;
      var_p = rec_len[pi] - 4 - (right ? fixed_l : fixed_r);
      d += k * (4 + fixed_out + var_d) + (var[ps + k] - var[ps]);
    }
    const uint8_t *L = right ? P : D, *R = right ? D : P;  // nullptr: a null side
    const uint64_t var_l = right ? var_p : var_d, var_r = right ? var_d : var_p;
    uint8_t* row = d + 4;
    if (lane == 0) st_span16(d, 4, __byte_perm((uint32_t)(fixed_out + var_l + var_r), 0, 0x0123), 0);
    // null word w: left bits [64 w, 64 w + 64), then right bit q at output bit nl + q
    for (uint32_t w = lane; w < b; w += 32) {
      const int64_t q0 = 64 * (int64_t)w - nl, a = q0 >> 6;  // floor
      const uint32_t s = (uint32_t)(q0 & 63);
      const uint64_t r0 = bits_word(R, nr, a, !R), r1 = s ? bits_word(R, nr, a + 1, !R) : 0;
      st_span16(row + 8 * w, 8, bits_word(L, nl, w, !L) | (r0 >> s) | (s ? r1 << (64 - s) : 0), 0);
    }
    // a null side: zero slots, and each DECIMAL_WIDE field's 16 zero bytes
    if (L) {
      warp_copy(row + 8 * b, L + 8 * bl, 8ull * nl, lane);
      warp_copy(row + fixed_out, L + fixed_l, var_l, lane);
    } else {
      for (uint32_t f = lane; f < nl; f += 32) st_span16(row + 8 * (b + f), 8, 0, 0);
      for (uint32_t q = lane; q < var_l / 8; q += 32) st_span16(row + fixed_out + 8 * q, 8, 0, 0);
    }
    if (R) {
      warp_copy(row + 8 * (b + nl), R + 8 * br, 8ull * nr, lane);
      warp_copy(row + fixed_out + var_l, R + fixed_r, var_r, lane);
    } else {
      for (uint32_t f = lane; f < nr; f += 32) st_span16(row + 8 * (b + nl + f), 8, 0, 0);
      for (uint32_t q = lane; q < var_r / 8; q += 32) st_span16(row + fixed_out + var_l + 8 * q, 8, 0, 0);
    }
    __syncwarp();
    // the slots whose offsets move: a zero slot (a null string) stays; a null side's wide decimals get their region's
    // offset, size 0 (UnsafeRowWriter.write of a null Decimal)
    const uint64_t shift_l = 8ull * (b - bl + nr) << 32, shift_r = (8ull * (b - br + nl) + var_l) << 32;
    if (L) {
      for (uint32_t x = lane; x < sh->n_var[0]; x += 32) {
        const uint32_t f = sh->var[0][x];
        const uint64_t slot = ld64(L + 8 * (bl + f));
        if (slot) st_span16(row + 8 * (b + f), 8, slot + shift_l, 0);
      }
    } else {
      for (uint32_t x = lane; x < sh->n_wide[0]; x += 32)
        st_span16(row + 8 * (b + sh->wide[0][x]), 8, (fixed_out + 16ull * x) << 32, 0);
    }
    if (R) {
      for (uint32_t x = lane; x < sh->n_var[1]; x += 32) {
        const uint32_t f = sh->var[1][x];
        const uint64_t slot = ld64(R + 8 * (br + f));
        if (slot) st_span16(row + 8 * (b + nl + f), 8, slot + shift_r, 0);
      }
    } else {
      for (uint32_t x = lane; x < sh->n_wide[1]; x += 32)
        st_span16(row + 8 * (b + nl + sh->wide[1][x]), 8, (fixed_out + var_l + 16ull * x) << 32, 0);
    }
    __syncwarp();
  }
}

// An existence join's row of left position j (right positions have none), by a warp: [out_bw null words: the left's
// bits][the left's slots][the exists slot: rpos[j]][the left's var bytes], its var slots moved past the added words
__global__ void __launch_bounds__(kJoinThreads) join_exists_emit_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    const uint32_t* __restrict__ idx, uint64_t n, const JoinShape* __restrict__ sh, const uint64_t* __restrict__ bytes,
    const uint32_t* __restrict__ rpos, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
  const uint64_t split = sh->split;
  const uint32_t nl = sh->n[0], bl = sh->bw[0], b = sh->out_bw;
  const uint32_t fixed_in = 8 * (bl + nl);
  const uint64_t fixed_out = 8ull * (b + nl + 1);
  const uint64_t shift = 8ull * (b - bl + 1) << 32;
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; j < n; j += warps) {
    const uint32_t i = at(idx, j);
    if (rec_off[i] >= split) continue;
    const uint8_t* src = arena + rec_off[i] + 4;
    const uint64_t var = rec_len[i] - 4 - fixed_in;
    uint8_t* d = dst + bytes[j];
    uint8_t* row = d + 4;
    if (lane == 0) {
      st_span16(d, 4, __byte_perm((uint32_t)(fixed_out + var), 0, 0x0123), 0);
      st_span16(row + 8 * (b + nl), 8, rpos[j], 0);
    }
    for (uint32_t w = lane; w < b; w += 32) st_span16(row + 8 * w, 8, bits_word(src, nl, w, false), 0);
    warp_copy(row + 8 * b, src + 8 * bl, 8ull * nl, lane);
    warp_copy(row + fixed_out, src + fixed_in, var, lane);
    __syncwarp();
    // a zero slot (a null string) stays zero
    for (uint32_t x = lane; x < sh->n_var[0]; x += 32) {
      const uint32_t f = sh->var[0][x];
      const uint64_t slot = ld64(src + 8 * (bl + f));
      if (slot) st_span16(row + 8 * (b + f), 8, slot + shift, 0);
    }
    __syncwarp();
  }
}

}  // namespace

size_t join_ws_bytes(uint64_t n, uint32_t n_ranges, uint32_t n_fields) {
  return 2 * a256(n * 8) + a256((n + 1) * 8) + a256(n * 4) + a256(2 * n * 4) + a256(scan_ws_elems(n + 1) * 8) +
         a256(join_readback_bytes(n_ranges)) + a256(sizeof(JoinShape)) + a256((size_t)n_fields * 4);
}

uint64_t* join_readback(uint8_t* d_jws, uint64_t n, uint32_t n_ranges) {
  return carve_join_ws(d_jws, n, n_ranges).readback;
}

void launch_join_count(const uint8_t* arena, uint64_t n, const uint32_t* idx, JoinShape shape,
                       const uint32_t* h_fields, uint32_t n_fields, uint32_t key_bytes, uint8_t* d_ws,
                       uint8_t* d_aws, uint8_t* d_jws, uint32_t n_ranges, cudaStream_t st, uint64_t* launches) {
  const JoinWs j = carve_join_ws(d_jws, n, n_ranges);
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  shape.var[0] = j.fields;
  shape.var[1] = j.fields + shape.n_var[0];
  shape.wide[1] = shape.var[1] + shape.n_var[1];
  shape.wide[0] = shape.wide[1] + shape.n_wide[1];
  cudaMemcpyAsync(j.shape, &shape, sizeof(JoinShape), cudaMemcpyHostToDevice, st);
  if (n_fields) cudaMemcpyAsync(j.fields, h_fields, (size_t)n_fields * 4, cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(j.readback, 0, 32, st);
  cudaMemsetAsync(j.gmax, 0, 2 * n * 4, st);
  const uint64_t* heads_before = rows_group_heads_before(d_aws, n);
  const uint64_t* groups = rows_aggregate_readback(d_aws, n, 0, 0);
  join_var_kernel<<<grid_for(n), kJoinThreads, 0, st>>>(w.src_off, w.len, idx, n, j.shape, heads_before, groups, j.var,
                                                        j.gmax, j.readback);
  launch_exclusive_scan_u64(j.var, n, j.var + n, j.scan_ws, st, launches);
  join_count_kernel<<<grid_for(n), kJoinThreads, 0, st>>>(arena, w.src_off, w.len, idx, n, j.shape, heads_before,
                                                          rows_group_starts(d_aws, n), groups, j.var, j.gmax, j.rows,
                                                          j.bytes, j.rpos, j.readback);
  launch_exclusive_scan_u64(j.rows, n, j.readback, j.scan_ws, st, launches);
  launch_exclusive_scan_u64(j.bytes, n, j.readback + 1, j.scan_ws, st, launches);
  if (launches) *launches += 2;
}

void launch_join_emit(const uint8_t* arena, uint64_t n, const uint32_t* idx, uint64_t out_rows, uint32_t key_bytes,
                      uint32_t type, uint8_t* d_ws, uint8_t* d_jws, uint32_t n_ranges, uint8_t* d_dst, cudaStream_t st,
                      uint64_t* launches) {
  if (!out_rows) return;
  const JoinWs j = carve_join_ws(d_jws, n, n_ranges);
  if (join_keeps_whole(type)) {  // the kept left records' indices (in rpos, which these joins do not use), then the row sort's gather
    join_compact_kernel<<<grid_for(n), kJoinThreads, 0, st>>>(idx, n, j.rows, out_rows, j.rpos);
    if (launches) *launches += 1;
    launch_rows_gather(arena, n, key_bytes, j.rpos, d_ws, d_dst, st, launches, out_rows);
    return;
  }
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  if (type == kJoinExistence) {  // a warp per sorted position
    const uint64_t want = (n + kJoinThreads / 32 - 1) / (kJoinThreads / 32);
    join_exists_emit_kernel<<<(unsigned)std::min<uint64_t>(want, (uint64_t)kSMs * 16), kJoinThreads, 0, st>>>(
        arena, w.src_off, w.len, idx, n, j.shape, j.bytes, j.rpos, d_dst);
    if (launches) *launches += 1;
    return;
  }
  const uint64_t want = (out_rows + kJoinThreads / 32 - 1) / (kJoinThreads / 32);
  const unsigned grid = (unsigned)std::min<uint64_t>(want, (uint64_t)kSMs * 16);
  join_emit_kernel<<<grid, kJoinThreads, 0, st>>>(arena, w.src_off, w.len, idx, n, out_rows, j.shape, j.rows, j.bytes,
                                                  j.var, j.rpos, d_dst);
  if (launches) *launches += 1;
}

}  // namespace b2s
