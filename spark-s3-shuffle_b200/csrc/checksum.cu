// checksum.cu — K1: batched CRC32 / CRC32C / Adler32 over slices of (compressed) bytes.
//
// Replaces java.util.zip.{CRC32,Adler32} as used by helper/S3ShuffleHelper.scala:94-103 and driven by
// storage/S3ChecksumValidationStream.scala:54-86 (read side) and Spark's MutableCheckedOutputStream (write side),
// and adds CRC32C (north-star).
//
// HBM-bound design: a slice is cut into work items of 2^tile_shift bytes (16-byte aligned in memory); one warp per
// item, lanes interleaved at 16-byte granularity so every global load is a fully coalesced 512-byte row.
//   CRC: each lane keeps a zero-init register advanced by "my 16 bytes + 496 zero bytes" per row through 16 byte-indexed
//        tables Z_496..Z_511 in shared memory (1 lookup per input byte, 12 of 16 independent of the loop-carried
//        register).  Lane registers are folded with constant GF(2) multipliers, the item is shifted to its place in the
//        slice with x^(8e) mod P built lane-parallel from x^(2^k) tables (negative e via x^-1 powers), and XORed
//        into the slice accumulator.  init/xorout are applied algebraically at the end.
//   Adler32: two dp4a per 32-bit word, 64-bit weighted sums, same work-item combine.
// Algorithmic traffic: 1 byte read per input byte, nothing written but 8 bytes per slice.
#include "crc_gf.h"
#include "kernels.h"

namespace b2s {

constexpr int kCkThreads = 256;  // 8 warps per CTA

// ---------------- table construction (host, once per device; crc_gf.h) ----------------
int checksum_tables_create(ChecksumTables* t) {
  static const uint32_t polys[2] = {0xEDB88320u, 0x82F63B78u};
  for (int w = 0; w < 2; w++) {
    uint32_t* rows = new uint32_t[16 * 256];
    uint32_t misc[kMiscWords];
    build_crc_tables(polys[w], rows, misc);
    if (cudaMalloc(&t->d_crc_rows[w], 16 * 256 * 4) != cudaSuccess) return -1;
    if (cudaMalloc(&t->d_crc_misc[w], kMiscWords * 4) != cudaSuccess) return -1;
    cudaMemcpy(t->d_crc_rows[w], rows, 16 * 256 * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(t->d_crc_misc[w], misc, kMiscWords * 4, cudaMemcpyHostToDevice);
    delete[] rows;
  }
  return 0;
}
void checksum_tables_destroy(ChecksumTables* t) {
  for (int w = 0; w < 2; w++) {
    cudaFree(t->d_crc_rows[w]);
    cudaFree(t->d_crc_misc[w]);
    t->d_crc_rows[w] = t->d_crc_misc[w] = nullptr;
  }
}

// ---------------- work decomposition ----------------
// items[i] = number of work items of slice i ; then exclusive-scanned in place (d_work_base[n] = total)
__global__ void ck_count_items_kernel(const uint64_t* __restrict__ off, const uint64_t* __restrict__ len, uint32_t n,
                                      uint32_t tile_shift, uint64_t* __restrict__ items, uint32_t* __restrict__ acc,
                                      uint64_t* __restrict__ acc64) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t v = len[i] ? (off[i] & 15u) + len[i] : 0;
  items[i] = (v + ((1ull << tile_shift) - 1)) >> tile_shift;
  if (acc) acc[i] = 0;
  if (acc64) {
    acc64[2 * i] = 0;
    acc64[2 * i + 1] = 0;
  }
}

struct ItemGeom {
  uint32_t slice;
  uint64_t vbase;   // virtual offset of the item inside the slice's padded stream
  uint64_t vlen;    // padded stream length a + len
  uint32_t a;       // front padding (off & 15)
  uint32_t ibytes;  // bytes of the padded stream inside this item
};

__device__ __forceinline__ ItemGeom locate_item(uint64_t item, const uint64_t* __restrict__ work_base, uint32_t n,
                                                const uint64_t* __restrict__ off, const uint64_t* __restrict__ len,
                                                uint32_t tile_shift) {
  // largest i with work_base[i] <= item
  uint32_t lo = 0, hi = n;  // invariant: work_base[lo] <= item < work_base[hi]
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (work_base[mid] <= item) lo = mid; else hi = mid;
  }
  ItemGeom g;
  g.slice = lo;
  g.a = (uint32_t)(off[lo] & 15u);
  g.vlen = g.a + len[lo];
  g.vbase = (item - work_base[lo]) << tile_shift;
  uint64_t rem = g.vlen - g.vbase;
  g.ibytes = (uint32_t)(rem < (1ull << tile_shift) ? rem : (1ull << tile_shift));
  return g;
}

// keep bytes k of a 16-byte word whose stream index is in [lo, hi); idx = stream index of byte 0 of the word
__device__ __forceinline__ uint4 mask16(uint4 w, int64_t idx, int64_t lo, int64_t hi) {
  uint32_t c[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int j = 0; j < 4; j++) {
    int64_t b0 = idx + 4 * j;
    int64_t f = lo - b0;  // first valid byte in this component
    int64_t e = hi - b0;  // end valid byte
    uint32_t m = 0xffffffffu;
    if (f >= 4 || e <= 0) m = 0;
    else {
      if (f > 0) m &= 0xffffffffu << (8 * (int)f);
      if (e < 4) m &= 0xffffffffu >> (8 * (4 - (int)e));
    }
    c[j] &= m;
  }
  return make_uint4(c[0], c[1], c[2], c[3]);
}

__device__ __forceinline__ uint4 ldg16(const uint8_t* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// ---------------- CRC kernel ----------------
__device__ __forceinline__ uint32_t crc_row(const uint32_t (*R)[256], uint32_t s, uint4 w) {
  const uint32_t x = w.x ^ s;
  uint32_t r = R[0][x & 255] ^ R[1][(x >> 8) & 255] ^ R[2][(x >> 16) & 255] ^ R[3][x >> 24];
  r ^= R[4][w.y & 255] ^ R[5][(w.y >> 8) & 255] ^ R[6][(w.y >> 16) & 255] ^ R[7][w.y >> 24];
  r ^= R[8][w.z & 255] ^ R[9][(w.z >> 8) & 255] ^ R[10][(w.z >> 16) & 255] ^ R[11][w.z >> 24];
  r ^= R[12][w.w & 255] ^ R[13][(w.w >> 8) & 255] ^ R[14][(w.w >> 16) & 255] ^ R[15][w.w >> 24];
  return r;
}

__global__ void __launch_bounds__(kCkThreads) crc_items_kernel(const uint8_t* __restrict__ base,
                                                               const uint64_t* __restrict__ off,
                                                               const uint64_t* __restrict__ len, uint32_t n,
                                                               uint32_t tile_shift,
                                                               const uint64_t* __restrict__ work_base,
                                                               const uint32_t* __restrict__ g_rows,
                                                               const uint32_t* __restrict__ g_misc,
                                                               uint32_t* __restrict__ acc) {
  __shared__ uint32_t R[16][256];
  __shared__ uint32_t misc[kMiscWords];
  for (int i = threadIdx.x; i < 16 * 256; i += kCkThreads) (&R[0][0])[i] = g_rows[i];
  for (int i = threadIdx.x; i < kMiscWords; i += kCkThreads) misc[i] = g_misc[i];
  __syncthreads();
  const uint32_t poly = misc[kMiscPoly];
  const int lane = threadIdx.x & 31;
  const uint64_t total = work_base[n];
  const uint64_t wstride = (uint64_t)gridDim.x * (kCkThreads / 32);
  for (uint64_t item = (uint64_t)blockIdx.x * (kCkThreads / 32) + (threadIdx.x >> 5); item < total; item += wstride) {
    const ItemGeom g = locate_item(item, work_base, n, off, len, tile_shift);
    const uint32_t rows = (g.ibytes + 511u) >> 9;
    const uint32_t zpad = rows * 512u - g.ibytes;
    const uint64_t after = g.vlen - (g.vbase + g.ibytes);
    // memory address of padded-stream byte 0 of this item (16-byte aligned)
    const uint8_t* p = base + (off[g.slice] - g.a) + g.vbase + 16 * lane;
    const int64_t lo = (int64_t)g.a - (int64_t)g.vbase;  // first valid stream index relative to the item
    const int64_t hi = (int64_t)g.ibytes;
    uint32_t s = 0;
    // rows that need masking: row 0 if lo > 0, last row if zpad > 0
    uint32_t r = 0;
    if (lo > 0 && rows) {
      int64_t idx = 16 * lane;
      uint4 w = (idx < hi && idx + 16 > lo) ? mask16(ldg16(p), idx, lo, hi) : make_uint4(0, 0, 0, 0);
      s = crc_row(R, s, w);
      r = 1;
    }
    const uint32_t full_end = zpad ? rows - 1 : rows;
    // steady state: unmasked, software-pipelined two rows deep
    if (r < full_end) {
      uint4 w0 = ldg16(p + (uint64_t)r * 512);
      for (; r + 1 < full_end; r++) {
        uint4 w1 = ldg16(p + (uint64_t)(r + 1) * 512);
        s = crc_row(R, s, w0);
        w0 = w1;
      }
      s = crc_row(R, s, w0);
      r++;
    }
    if (r < rows) {  // masked last row
      int64_t idx = (int64_t)r * 512 + 16 * lane;
      uint4 w = (idx < hi && idx + 16 > lo) ? mask16(ldg16(p + (uint64_t)r * 512), idx, lo, hi) : make_uint4(0, 0, 0, 0);
      s = crc_row(R, s, w);
    }
    // fold lanes: lane l is over-advanced by 16*l bytes relative to lane 31's frame -> bring all to "row end + 496"
    uint32_t v = gf_mul(s, misc[kMiscLane + lane], poly);
#pragma unroll
    for (int d = 16; d; d >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, d);
    // shift to the item's place in the slice: x^(8*(after - zpad - 496)), built lane-parallel from bit factors
    int64_t e = (int64_t)after - (int64_t)zpad - 496;
    const uint32_t* tab = misc + (e >= 0 ? kMiscXPow : kMiscXInv);
    uint64_t ue = (uint64_t)(e >= 0 ? e : -e);
    uint32_t f = ((ue >> lane) & 1) ? tab[lane + 3] : kGfOne;
    if ((ue >> (lane + 32)) & 1) f = gf_mul(f, tab[lane + 35], poly);
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      uint32_t o = __shfl_xor_sync(0xffffffffu, f, d);
      f = gf_mul(f, o, poly);
    }
    if (lane == 0) atomicXor(acc + g.slice, gf_mul(f, v, poly));
  }
}

__global__ void crc_finalize_kernel(const uint32_t* __restrict__ acc, const uint64_t* __restrict__ len, uint32_t n,
                                    const uint32_t* __restrict__ g_misc, uint64_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t poly = g_misc[kMiscPoly];
  // crc(M) = raw0(M) ^ 0xFFFFFFFF * x^(8|M|) ^ 0xFFFFFFFF
  uint32_t init = gf_mul(gf_xpow8(len[i], g_misc + kMiscXPow, poly), 0xffffffffu, poly);
  out[i] = (uint64_t)(acc[i] ^ init ^ 0xffffffffu);
}

// ---------------- Adler32 kernel ----------------
constexpr uint32_t kAdlerMod = 65521u;

__global__ void __launch_bounds__(kCkThreads) adler_items_kernel(const uint8_t* __restrict__ base,
                                                                 const uint64_t* __restrict__ off,
                                                                 const uint64_t* __restrict__ len, uint32_t n,
                                                                 uint32_t tile_shift,
                                                                 const uint64_t* __restrict__ work_base,
                                                                 unsigned long long* __restrict__ acc64) {
  const int lane = threadIdx.x & 31;
  const uint64_t total = work_base[n];
  const uint64_t wstride = (uint64_t)gridDim.x * (kCkThreads / 32);
  for (uint64_t item = (uint64_t)blockIdx.x * (kCkThreads / 32) + (threadIdx.x >> 5); item < total; item += wstride) {
    const ItemGeom g = locate_item(item, work_base, n, off, len, tile_shift);
    const uint32_t rows = (g.ibytes + 511u) >> 9;
    const uint64_t after = g.vlen - (g.vbase + g.ibytes);
    const uint8_t* p = base + (off[g.slice] - g.a) + g.vbase + 16 * lane;
    const int64_t lo = (int64_t)g.a - (int64_t)g.vbase;
    const int64_t hi = (int64_t)g.ibytes;
    // A = sum b ; B = sum (ibytes - idx) * b   (front-padding zeros contribute nothing)
    uint32_t A = 0;
    uint64_t B = 0;
    for (uint32_t r = 0; r < rows; r++) {
      int64_t idx = (int64_t)r * 512 + 16 * lane;
      uint4 w = make_uint4(0, 0, 0, 0);
      if (idx < hi && idx + 16 > lo) {
        w = ldg16(p + (uint64_t)r * 512);
        if (idx < lo || idx + 16 > hi) w = mask16(w, idx, lo, hi);
      }
      const uint32_t c[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        uint32_t S = __dp4a(c[j], 0x01010101u, 0u);
        uint32_t Wt = __dp4a(c[j], 0x01020304u, 0u);  // 4*b0 + 3*b1 + 2*b2 + 1*b3
        A += S;
        int64_t wgt = hi - (idx + 4 * j) - 4;  // weight of the word's last byte minus one (may be negative only when S == 0)
        B += (uint64_t)Wt + (uint64_t)((int64_t)S * wgt);
      }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      A += __shfl_xor_sync(0xffffffffu, A, d);
      B += __shfl_xor_sync(0xffffffffu, B, d);
    }
    if (lane == 0) {
      uint64_t a_mod = A % kAdlerMod;
      uint64_t contrib = (B % kAdlerMod + (after % kAdlerMod) * a_mod) % kAdlerMod;
      atomicAdd(acc64 + 2 * g.slice, (unsigned long long)a_mod);
      atomicAdd(acc64 + 2 * g.slice + 1, (unsigned long long)contrib);
    }
  }
}

__global__ void adler_finalize_kernel(const unsigned long long* __restrict__ acc64, const uint64_t* __restrict__ len,
                                      uint32_t n, uint64_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t a = (1 + acc64[2 * i]) % kAdlerMod;
  uint64_t b = (len[i] % kAdlerMod + acc64[2 * i + 1]) % kAdlerMod;
  out[i] = (b << 16) | a;
}

// ---------------- launch ----------------
void launch_checksum(const ChecksumTables& t, uint32_t alg, const uint8_t* base, const uint64_t* d_off,
                     const uint64_t* d_len, uint32_t n, uint32_t tile_shift, uint64_t* d_work_base, uint64_t* d_ws,
                     uint64_t* d_out, cudaStream_t st, uint64_t* launches) {
  if (n == 0) return;
  // accumulators live in the output array's tail-free scratch: reuse d_ws after the scan partials
  uint64_t* d_acc = d_ws + scan_ws_elems((size_t)n + 1);  // 2*n uint64 (adler) or n uint32 (crc)
  const bool crc = (alg == B2S_CHECKSUM_CRC32 || alg == B2S_CHECKSUM_CRC32C);
  ck_count_items_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_off, d_len, n, tile_shift, d_work_base,
                                                       crc ? reinterpret_cast<uint32_t*>(d_acc) : nullptr,
                                                       crc ? nullptr : d_acc);
  cudaMemsetAsync(d_work_base + n, 0, sizeof(uint64_t), st);
  *launches += 1;
  launch_exclusive_scan_u64(d_work_base, (size_t)n + 1, d_ws + scan_ws_elems((size_t)n + 1) - 1, d_ws, st, launches);
  // note: the scan's grand-total slot is the last element of its own workspace region; d_work_base[n] holds the total
  const int grid = kSMs * 4;
  if (crc) {
    const int w = alg == B2S_CHECKSUM_CRC32 ? 0 : 1;
    crc_items_kernel<<<grid, kCkThreads, 0, st>>>(base, d_off, d_len, n, tile_shift, d_work_base, t.d_crc_rows[w],
                                                  t.d_crc_misc[w], reinterpret_cast<uint32_t*>(d_acc));
    crc_finalize_kernel<<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<uint32_t*>(d_acc), d_len, n, t.d_crc_misc[w],
                                                        d_out);
  } else {
    adler_items_kernel<<<grid, kCkThreads, 0, st>>>(base, d_off, d_len, n, tile_shift, d_work_base,
                                                    reinterpret_cast<unsigned long long*>(d_acc));
    adler_finalize_kernel<<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<unsigned long long*>(d_acc), d_len, n,
                                                          d_out);
  }
  *launches += 2;
}

// got[s] vs expected[s] for flattened slices; owner[s] = block index, slice_base[owner] = first slice of the block
__global__ void ck_compare_kernel(const uint64_t* __restrict__ got, const uint64_t* __restrict__ expected,
                                  const uint32_t* __restrict__ owner, const uint32_t* __restrict__ slice_base,
                                  uint32_t n_slices, int32_t* __restrict__ status, int32_t* __restrict__ bad_slice) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_slices) return;
  if ((uint32_t)got[s] != (uint32_t)expected[s] || (expected[s] >> 32) != 0) {
    uint32_t i = owner[s];
    // report the lowest mismatching slice of the block (the reference stops at the first one it meets)
    atomicMin(reinterpret_cast<unsigned int*>(bad_slice + i), s - slice_base[i]);
    status[i] = B2S_E_CHECKSUM;
  }
}

void launch_checksum_compare(const uint64_t* d_got, const uint64_t* d_expected, const uint32_t* d_slice_owner,
                             const uint32_t* d_slice_base, uint32_t n_slices, int32_t* d_status, int32_t* d_bad_slice,
                             cudaStream_t st, uint64_t* launches) {
  if (!n_slices) return;
  ck_compare_kernel<<<(n_slices + 255) / 256, 256, 0, st>>>(d_got, d_expected, d_slice_owner, d_slice_base, n_slices,
                                                           d_status, d_bad_slice);
  *launches += 1;
}

}  // namespace b2s
