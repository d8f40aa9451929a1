// rows_expand.cu — Spark SQL's Expand for grouping sets (ROLLUP, CUBE, GROUPING SETS) in front of a map task's partial
// aggregation: every record of the caller's once per grouping set, in ExpandExec's row-major order, as a compact
// UnsafeRow that holds only what the aggregation reads.  Projected record p = r * n_sets + k is input record r under set
// k; its row's fields are
//   c < n_keys          key column c: the input's value when bit c of set k's mask is set, else null
//   n_keys              gid, a never-null long: Spark's spark_grouping_id, the sum of 1 << (n_keys - 1 - c) over the
//                       key columns c outside the set
//   n_keys + 1 + i      aggregate input i, read from the input unmasked (a COUNT's input: its null bit alone)
// at most 32 fields, so one null word.  Fixed values are copied as the slot holds them (the bytes past a key's width
// zeroed); a string key its bytes zero-padded to 8; a decimal(p > 18) key or input 16 bytes (its 1..16 bytes as the
// input holds them, zero-padded; a null one 16 zero bytes, slot offset << 32).  An out-of-set column or a null string
// has slot 0 and no bytes.  The records' framing, key columns and values are checked before (launch_partial_agg_check),
// so every slot read here lies inside its row.
//   size  : a thread per projected record: its length (4 + row) into len and off, off scanned into the projected offsets
//           (64-bit: the projected arena is n_sets times the input); the lowest record whose projected row passes
//           2^31 - 1 bytes into header word 1
//   write : a warp per projected record, lane f writing field f's slot, the strings copied by the whole warp with
//           16-byte loads; lane 0 the size prefix, the null word and the record length
#include "kernels.h"
#include "rows_key.cuh"

namespace b2s {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kXThreads = 256;

inline size_t a256(size_t b) { return (b + 255) / 256 * 256; }

inline unsigned grid_for(uint64_t n) {
  const uint64_t want = (n + kXThreads - 1) / kXThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

inline unsigned warp_grid_for(uint64_t warps) {
  const uint64_t want = (warps + kXThreads / 32 - 1) / (kXThreads / 32);
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

// the workspace (expand_ws_bytes): header [projected bytes, lowest over-long record (~0: none)], the set masks, the
// projected records' lengths and offsets, the offsets' scan workspace
struct XWs {
  uint64_t* hdr;
  uint32_t* masks;
  uint32_t* len;
  uint64_t* off;
  uint64_t* scan_ws;
};

XWs carve_x_ws(uint8_t* d, uint64_t n, uint32_t n_sets) {
  const uint64_t N = n * n_sets;
  XWs w;
  uint8_t* p = d;
  w.hdr = (uint64_t*)p;    p += 256;
  w.masks = (uint32_t*)p;  p += a256((size_t)n_sets * 4);
  w.len = (uint32_t*)p;    p += a256(N * 4);
  w.off = (uint64_t*)p;    p += a256(N * 8);
  w.scan_ws = (uint64_t*)p;
  return w;
}

__device__ __forceinline__ bool bit_at(const uint8_t* row, int32_t f) {
  uint64_t w, unused;
  ld_span16<true>(row + 8 * (uint32_t)(f >> 6), 8, w, unused);
  return (w >> (f & 63)) & 1;
}

__device__ __forceinline__ bool wide_input(uint32_t vt) {
  return (vt & 0xff) == B2S_WINDOW_VAL_DECIMAL && ((vt >> 8) & 0xff) > 18;
}

__device__ __forceinline__ uint32_t gid_of(uint32_t mask, uint32_t nk) {
  return __brev(~mask & ((1u << nk) - 1)) >> (32 - nk);
}

// key column c's var bytes in the projected row: an in-set non-null string its length padded to 8, an in-set decimal
// (null or not) 16
__device__ __forceinline__ uint32_t x_key_var(const uint8_t* row, const KeySpec& ks, uint32_t c, bool in, bool null) {
  if (!in) return 0;
  const uint32_t ty = ks.type[c];
  if (ty == kDecimalKey) return 16;
  if (ty != kStringKey || null) return 0;
  uint64_t slot, unused;
  ld_span16<true>(row + ks.off[c], 8, slot, unused);
  return ((uint32_t)slot + 7) & ~7u;
}

__device__ __forceinline__ bool x_key_null(const uint8_t* row, const KeySpec& ks, uint32_t c) {
  return ks.null_field[c] >= 0 && bit_at(row, ks.null_field[c]);
}

__device__ __forceinline__ uint32_t row_p_sets(uint32_t p, uint32_t n_sets, uint32_t& k) {
  const uint32_t r = p / n_sets;
  k = p - r * n_sets;
  return r;
}

__global__ void __launch_bounds__(kXThreads) x_size_kernel(const uint8_t* __restrict__ rec,
                                                           const uint64_t* __restrict__ rec_off, uint32_t N,
                                                           const __grid_constant__ ExpandSpec s,
                                                           const uint32_t* __restrict__ masks,
                                                           uint32_t* __restrict__ len, uint64_t* __restrict__ off,
                                                           unsigned long long* __restrict__ too_long) {
  const uint32_t nk = s.keys.n, nf = nk + 1 + s.n_in;
  for (uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < N; p += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t k;
    const uint32_t r = row_p_sets((uint32_t)p, s.n_sets, k), mask = __ldg(masks + k);
    const uint8_t* row = rec + rec_off[r] + 4;
    uint64_t l = 4 + 8 * (1 + nf);
    for (uint32_t c = 0; c < nk; c++) {
      const bool in = (mask >> c) & 1;
      l += x_key_var(row, s.keys, c, in, in && x_key_null(row, s.keys, c));
    }
    for (uint32_t i = 0; i < s.n_in; i++) l += wide_input(s.vtype[i]) ? 16 : 0;
    if (l - 4 > 0x7fffffffull) {
      atomicMin(too_long, (unsigned long long)r);
      l = 4;
    }
    len[p] = (uint32_t)l;
    off[p] = l;
  }
}

// Projected record p, a warp: lane f < nf is field f (see the top of the file)
__global__ void __launch_bounds__(kXThreads) x_write_kernel(const uint8_t* __restrict__ rec,
                                                            const uint64_t* __restrict__ rec_off, uint32_t N,
                                                            const __grid_constant__ ExpandSpec s,
                                                            const uint32_t* __restrict__ masks,
                                                            const uint32_t* __restrict__ len,
                                                            const uint64_t* __restrict__ off,
                                                            uint32_t* __restrict__ out_len, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nk = s.keys.n, nf = nk + 1 + s.n_in, fixed = 8 * (1 + nf);
  const uint64_t warps = (uint64_t)gridDim.x * (kXThreads / 32);
  for (uint64_t p = (uint64_t)blockIdx.x * (kXThreads / 32) + (threadIdx.x >> 5); p < N; p += warps) {
    uint32_t k;
    const uint32_t r = row_p_sets((uint32_t)p, s.n_sets, k), mask = __ldg(masks + k);
    const uint8_t* row = rec + rec_off[r] + 4;
    uint8_t* out = dst + off[p];
    uint8_t* orow = out + 4;
    bool null = false, dec = false, str = false;
    uint64_t slot = 0, m0 = 0, m1 = 0;
    uint32_t var = 0, slen = 0, sfrom = 0;
    if (lane < nk) {
      const uint32_t c = lane, ty = s.keys.type[c];
      const bool in = (mask >> c) & 1;
      null = !in || x_key_null(row, s.keys, c);
      var = x_key_var(row, s.keys, c, in, null);
      dec = in && ty == kDecimalKey;
      if (!null) {
        uint64_t v, unused;
        ld_span16<true>(row + s.keys.off[c], (int)s.keys.len[c], v, unused);
        if (ty == kStringKey) {
          str = true;
          sfrom = (uint32_t)(v >> 32);
          slen = (uint32_t)v;
        } else if (ty == kDecimalKey) {
          sfrom = (uint32_t)(v >> 32);
          slen = (uint32_t)v;
        } else {
          const uint32_t w = s.keys.len[c];
          slot = w >= 8 ? v : v & ((1ull << (8 * w)) - 1);
        }
      }
    } else if (lane == nk) {
      slot = gid_of(mask, nk);
    } else if (lane < nf) {
      const uint32_t i = lane - nk - 1, vt = s.vtype[i];
      null = s.vnull[i] >= 0 && bit_at(row, s.vnull[i]);
      dec = wide_input(vt);
      var = dec ? 16 : 0;
      if (!null && s.reads[i]) {
        uint64_t v, unused;
        ld_span16<true>(row + s.voff[i], 8, v, unused);
        if (dec) {
          sfrom = (uint32_t)(v >> 32);
          slen = (uint32_t)v;
        } else {
          slot = v;
        }
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
      if (slen) {
        ld_span16<true>(row + sfrom, (int)slen, m0, m1);
        if (slen < 8) m0 &= (1ull << (8 * slen)) - 1;
        if (slen <= 8) m1 = 0;
        else if (slen < 16) m1 &= (1ull << (8 * (slen - 8))) - 1;
      }
      st_span16(orow + voff, 16, m0, m1);
      slot = ((uint64_t)voff << 32) | slen;
    } else if (str) {
      slot = ((uint64_t)voff << 32) | slen;
    }
    if (lane < nf) st_span16(orow + 8 + 8 * lane, 8, slot, 0);
    // the strings, one at a time by the whole warp, then their padding
    for (uint32_t todo = __ballot_sync(FULL, str); todo; todo &= todo - 1) {
      const int src = __ffs(todo) - 1;
      const uint32_t from = __shfl_sync(FULL, sfrom, src), n = __shfl_sync(FULL, slen, src);
      const uint32_t to = __shfl_sync(FULL, voff, src), pad = __shfl_sync(FULL, var, src) - n;
      warp_copy(orow + to, row + from, n, lane);
      if (lane == 0 && pad) st_span16(orow + to + n, (int)pad, 0, 0);
    }
    const uint32_t nulls = __ballot_sync(FULL, lane < nf && null);
    if (lane == 0) {
      const uint32_t l = len[p];
      st_span16(out, 4, __byte_perm(l - 4, 0, 0x0123), 0);
      st_span16(orow, 8, nulls, 0);
      out_len[p] = l;
    }
  }
}

}  // namespace

size_t expand_ws_bytes(uint64_t n, uint32_t n_sets) {
  const uint64_t N = n * n_sets;
  return 256 + a256((size_t)n_sets * 4) + a256(N * 4) + a256(N * 8) + a256(scan_ws_elems(N) * 8);
}

uint64_t* expand_header(uint8_t* d_xws) { return (uint64_t*)d_xws; }

uint32_t* expand_masks(uint8_t* d_xws, uint64_t n, uint32_t n_sets) { return carve_x_ws(d_xws, n, n_sets).masks; }

void launch_expand_size(const uint8_t* rec, const uint64_t* rec_off, uint64_t n, const ExpandSpec& spec,
                        uint8_t* d_xws, cudaStream_t st, uint64_t* launches) {
  const XWs w = carve_x_ws(d_xws, n, spec.n_sets);
  cudaMemsetAsync(w.hdr, 0, 256, st);
  cudaMemsetAsync(w.hdr + 1, 0xff, 8, st);
  const uint64_t N = n * spec.n_sets;
  if (!N) return;
  x_size_kernel<<<grid_for(N), kXThreads, 0, st>>>(rec, rec_off, (uint32_t)N, spec, w.masks, w.len, w.off,
                                                   (unsigned long long*)(w.hdr + 1));
  launch_exclusive_scan_u64(w.off, N, w.hdr, w.scan_ws, st, launches);
  if (launches) *launches += 1;
}

void launch_expand_write(const uint8_t* rec, const uint64_t* rec_off, uint64_t n, const ExpandSpec& spec,
                         uint8_t* d_xws, uint32_t* d_out_len, uint8_t* d_out, cudaStream_t st, uint64_t* launches) {
  const XWs w = carve_x_ws(d_xws, n, spec.n_sets);
  const uint64_t N = n * spec.n_sets;
  if (!N) return;
  x_write_kernel<<<warp_grid_for(N), kXThreads, 0, st>>>(rec, rec_off, (uint32_t)N, spec, w.masks, w.len, w.off,
                                                         d_out_len, d_out);
  if (launches) *launches += 1;
}

}  // namespace b2s
