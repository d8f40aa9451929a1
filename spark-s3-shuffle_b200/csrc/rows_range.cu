// rows_range.cu — Spark's RangePartitioner id of length-prefixed UnsafeRow records, the map side of a range exchange
// (ShuffleExchangeExec(RangePartitioning) projects each row to its sort key and searches the sampled bounds).  The id
// of a record is the number of bounds whose key is below the record's: with strictly increasing bounds that is what
// both of RangePartitioner.getPartition's branches (linear scan, binary search) return.  Keys are compared as their
// encodings (rows_key.cuh), whose memcmp order is Spark SQL's order of the sort key.
//   bounds : a thread per bound checks the bound row, stores its first kKeyPrefixBytes encoded bytes as five big-endian
//            words and its encoded length (0: a bad bound), then a thread per bound compares it with its predecessor
//   ids    : a thread per record checks the record, encodes its first window, and binary-searches the bounds' windows;
//            where a record and a bound agree on the whole window and both keys go on, further windows of
//            kKeyChunkBytes are encoded from both rows until they differ (the encoding is prefix-free, so zero-padded
//            windows compare exactly)
#include <algorithm>

#include "kernels.h"
#include "rows_key.cuh"

namespace b2s {

namespace {

constexpr int kRangeThreads = 256;

inline unsigned range_grid(uint64_t n) {
  const uint64_t want = (n + kRangeThreads - 1) / kRangeThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? want : (uint64_t)kSMs * 16);
}

// Why the framed row at p (len bytes: [size: int32 big-endian][row]) cannot be encoded, kHashBad*, or 0; *size = the
// row's size.  min_key / min_null: the row bytes that hold every key slot / every null word of a nullable key column.
__device__ __forceinline__ uint64_t frame_why(const uint8_t* p, uint32_t len, uint32_t min_key, uint32_t min_null,
                                              uint32_t* size) {
  if (len < 4) return kHashBadShort;
  uint64_t lo, hi;
  ld_span16<true>(p, 4, lo, hi);
  *size = __byte_perm((uint32_t)lo, 0, 0x0123);
  if (*size != len - 4) return kHashBadSize;
  if (*size < min_key) return kHashBadKey;
  if (*size < min_null) return kHashBadNull;
  return 0;
}

// The reason encode_key found a row bad: its first non-null string or decimal column (left to right) whose slot does
// not name bytes inside the row, as the hash kernel reports it.  Only on a bad row.
__device__ __noinline__ uint64_t slot_why(const uint8_t* row, uint32_t size, const KeySpec& ks) {
  for (uint32_t c = 0; c < ks.n; c++) {
    const uint32_t ty = ks.type[c] & kKeyTypeMask;
    if (ty != kStringKey && ty != kDecimalKey) continue;
    const int32_t nf = ks.null_field[c];
    uint64_t lo, hi;
    if (nf >= 0) {
      ld_span16<true>(row + 8 * (uint32_t)(nf >> 6), 8, lo, hi);
      if ((lo >> (nf & 63)) & 1) continue;
    }
    ld_span16<true>(row + ks.off[c], 8, lo, hi);
    const uint32_t so = (uint32_t)(lo >> 32), sz = (uint32_t)lo;
    if (ty == kDecimalKey && sz - 1 >= 16u) return kHashBadDecimal;
    if ((uint64_t)so + sz > size) return ty == kDecimalKey ? kHashBadDecimal : kHashBadString;
  }
  return kHashBadString;
}

// The first window and the encoded length of the framed row at p (0 and why != 0 when it is bad); *size = its size
__device__ __forceinline__ uint32_t first_window(const uint8_t* p, uint32_t len, const KeySpec& ks, uint32_t min_key,
                                                 uint32_t min_null, KeyWindow& kw, uint32_t* size, uint64_t* why) {
  *why = frame_why(p, len, min_key, min_null, size);
  if (*why) return 0;
  bool bad = false;
  const uint32_t klen = encode_key(p + 4, *size, ks, kw, true, &bad);
  if (bad) *why = slot_why(p + 4, *size, ks);
  return *why ? 0 : klen;
}

__device__ __forceinline__ int cmp_u32(uint32_t a, uint32_t b) { return a < b ? -1 : a > b ? 1 : 0; }

// Keys a (row ra, spec ka) and b (row rb, spec kb), both longer than kKeyPrefixBytes and equal over it: the sign of
// memcmp over the rest, a window of kKeyChunkBytes at a time.  Both rows are good, so their slots lie inside them.
__device__ __noinline__ int cmp_rest(const uint8_t* ra, uint32_t sa, const KeySpec& ka, const uint8_t* rb, uint32_t sb,
                                     const KeySpec& kb, uint32_t klen) {
  for (uint32_t d = kKeyPrefixBytes; d < klen; d += kKeyChunkBytes) {
    KeyWindow x{0, 0, 0, 0, 0, d, kKeyChunkBytes}, y{0, 0, 0, 0, 0, d, kKeyChunkBytes};
    bool bad = false;
    encode_key(ra, sa, ka, x, false, &bad);
    encode_key(rb, sb, kb, y, false, &bad);
    int c = cmp_u32(x.w0, y.w0);
    if (!c) c = cmp_u32(x.w1, y.w1);
    if (!c) c = cmp_u32(x.w2, y.w2);
    if (!c) c = cmp_u32(x.w3, y.w3);
    if (c) return c;
  }
  return 0;
}

// A good key (window kw, encoded length klen, row of size bytes) against bound j (bw: its words, bnd / boff: its row)
__device__ __forceinline__ int cmp_bound(const KeyWindow& kw, uint32_t klen, const uint8_t* row, uint32_t size,
                                         const KeySpec& ks, const uint4* __restrict__ bw,
                                         const uint8_t* __restrict__ bnd, const uint64_t* __restrict__ boff,
                                         const KeySpec& bks, uint32_t j) {
  const uint4 a = __ldg(bw + 2 * j), b = __ldg(bw + 2 * j + 1);
  int c = cmp_u32(kw.w0, a.x);
  if (!c) c = cmp_u32(kw.w1, a.y);
  if (!c) c = cmp_u32(kw.w2, a.z);
  if (!c) c = cmp_u32(kw.w3, a.w);
  if (!c) c = cmp_u32(kw.w4, b.x);
  // equal windows: both keys end inside it (and are equal) or both go on; a bad bound (length 0) is not read further
  if (c || klen <= kKeyPrefixBytes || b.y <= kKeyPrefixBytes) return c;
  const uint64_t o = boff[j];
  return cmp_rest(row, size, ks, bnd + o + 4, (uint32_t)(boff[j + 1] - o - 4), bks, klen);
}

// bw[2j], bw[2j + 1] = bound j's first window (w0..w3; w4, encoded length or 0 when bad); a bad bound lowers *bad to
// (j << 3) | its kHashBad* reason
__global__ void __launch_bounds__(kRangeThreads) bounds_encode_kernel(
    const uint8_t* __restrict__ bnd, const uint64_t* __restrict__ boff, uint32_t nb, const __grid_constant__ KeySpec bks,
    uint32_t min_key, uint32_t min_null, uint4* __restrict__ bw, unsigned long long* __restrict__ bad) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < nb; j += gridDim.x * blockDim.x) {
    KeyWindow kw{0, 0, 0, 0, 0, 0, kKeyPrefixBytes};
    uint32_t size = 0;
    uint64_t why;
    const uint32_t klen = first_window(bnd + boff[j], (uint32_t)(boff[j + 1] - boff[j]), bks, min_key, min_null, kw,
                                       &size, &why);
    bw[2 * j] = make_uint4(kw.w0, kw.w1, kw.w2, kw.w3);
    bw[2 * j + 1] = make_uint4(kw.w4, klen, 0, 0);
    if (why) atomicMin(bad, (unsigned long long)(((uint64_t)j << 3) | why));
  }
}

// bound j >= 1 whose key is not above bound j - 1's lowers *bad to (j << 3) | kRangeBadOrder (a bad pair is skipped:
// the bad bound already lowered it further)
__global__ void __launch_bounds__(kRangeThreads) bounds_order_kernel(
    const uint8_t* __restrict__ bnd, const uint64_t* __restrict__ boff, uint32_t nb, const __grid_constant__ KeySpec bks,
    const uint4* __restrict__ bw, unsigned long long* __restrict__ bad) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x + 1; j < nb; j += gridDim.x * blockDim.x) {
    const uint4 a = __ldg(bw + 2 * j), b = __ldg(bw + 2 * j + 1);
    if (!b.y || !__ldg(bw + 2 * j - 1).y) continue;
    const KeyWindow kw{a.x, a.y, a.z, a.w, b.x, 0, kKeyPrefixBytes};
    if (cmp_bound(kw, b.y, bnd + boff[j] + 4, (uint32_t)(boff[j + 1] - boff[j] - 4), bks, bw, bnd, boff, bks, j - 1) <=
        0)
      atomicMin(bad, (unsigned long long)(((uint64_t)j << 3) | kRangeBadOrder));
  }
}

// ids[i] = the bounds below record i's key (a lower-bound search over the bounds' windows); a bad record takes id 0
// and lowers *bad to kRangeBadRecord | (i << 3) | its kHashBad* reason.  A record that ends past rec_bytes is not read
// (the partition step's length sum reports it).
__global__ void __launch_bounds__(kRangeThreads) rows_range_kernel(
    const uint8_t* __restrict__ rec, uint64_t rec_bytes, const uint64_t* __restrict__ rec_off,
    const uint32_t* __restrict__ rec_len, uint64_t n, const __grid_constant__ KeySpec ks, uint32_t min_key,
    uint32_t min_null, const uint8_t* __restrict__ bnd, const uint64_t* __restrict__ boff, uint32_t nb,
    const __grid_constant__ KeySpec bks, const uint4* __restrict__ bw, uint32_t* __restrict__ ids,
    unsigned long long* __restrict__ bad) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t o = rec_off[i];
    const uint32_t len = rec_len[i];
    uint32_t id = 0;
    if (o + len <= rec_bytes) {
      KeyWindow kw{0, 0, 0, 0, 0, 0, kKeyPrefixBytes};
      uint32_t size = 0;
      uint64_t why;
      const uint32_t klen = first_window(rec + o, len, ks, min_key, min_null, kw, &size, &why);
      if (why) {
        atomicMin(bad, (unsigned long long)(kRangeBadRecord | (i << 3) | why));
      } else {
        uint32_t lo = 0, hi = nb;
        while (lo < hi) {
          const uint32_t mid = (lo + hi) / 2;
          if (cmp_bound(kw, klen, rec + o + 4, size, ks, bw, bnd, boff, bks, mid) > 0) lo = mid + 1;
          else hi = mid;
        }
        id = lo;
      }
    }
    ids[i] = id;
  }
}

// the row bytes that hold every key slot / every null word of a nullable column
void key_extent(const KeySpec& ks, uint32_t* min_key, uint32_t* min_null) {
  uint64_t k = 0, z = 0;
  for (uint32_t c = 0; c < ks.n; c++) {
    k = std::max<uint64_t>(k, (uint64_t)ks.off[c] + ks.len[c]);
    if (ks.null_field[c] >= 0) z = std::max<uint64_t>(z, 8ull * (uint32_t)(ks.null_field[c] >> 6) + 8);
  }
  *min_key = (uint32_t)std::min<uint64_t>(k, 0xffffffffull);  // a row is below 2^32 - 4 bytes: no slot past that
  *min_null = (uint32_t)z;
}

// The key columns of a bound row, UnsafeProjection(sort order children)'s row: column c is field c (its slot after the
// null words, its null bit c when the records' column is nullable), with the records' column's type, flags and key_len
KeySpec range_bound_keys(const KeySpec& ks) {
  KeySpec b = ks;
  for (uint32_t c = 0; c < ks.n; c++) {
    b.off[c] = 8 * ((ks.n + 63) / 64) + 8 * c;
    b.null_field[c] = ks.null_field[c] >= 0 ? (int32_t)c : -1;
  }
  return b;
}

}  // namespace

size_t rows_range_ws_bytes(uint32_t n_bounds, uint64_t bound_bytes) {
  auto a = [](size_t b) { return (b + 255) / 256 * 256; };
  return a((size_t)n_bounds * 32) + a(((size_t)n_bounds + 1) * 8) + a(bound_bytes + 16) + 256;
}

RangeWs carve_rows_range_ws(uint8_t* d_ws, uint32_t n_bounds, uint64_t bound_bytes) {
  auto a = [](size_t b) { return (b + 255) / 256 * 256; };
  RangeWs w;
  uint8_t* p = d_ws;
  w.words = (uint4*)p; p += a((size_t)n_bounds * 32);
  w.off = (uint64_t*)p;  p += a(((size_t)n_bounds + 1) * 8);
  w.rows = p;            p += a(bound_bytes + 16);
  w.verdict = (uint64_t*)p;
  return w;
}

void launch_rows_range(const uint8_t* rec, uint64_t rec_bytes, const uint64_t* rec_off, const uint32_t* rec_len,
                       uint64_t n, const KeySpec& ks, const RangeWs& w, uint32_t n_bounds, uint32_t* ids,
                       uint64_t* bad, cudaStream_t st, uint64_t* launches) {
  const KeySpec bks = range_bound_keys(ks);
  uint32_t min_key, min_null;
  if (n_bounds) {
    key_extent(bks, &min_key, &min_null);
    bounds_encode_kernel<<<range_grid(n_bounds), kRangeThreads, 0, st>>>(w.rows, w.off, n_bounds, bks, min_key,
                                                                          min_null, w.words, (unsigned long long*)bad);
    if (launches) *launches += 1;
    if (n_bounds > 1) {
      bounds_order_kernel<<<range_grid(n_bounds - 1), kRangeThreads, 0, st>>>(w.rows, w.off, n_bounds, bks, w.words,
                                                                             (unsigned long long*)bad);
      if (launches) *launches += 1;
    }
  }
  if (!n) return;
  key_extent(ks, &min_key, &min_null);
  rows_range_kernel<<<range_grid(n), kRangeThreads, 0, st>>>(rec, rec_bytes, rec_off, rec_len, n, ks, min_key, min_null,
                                                             w.rows, w.off, n_bounds, bks, w.words, ids,
                                                             (unsigned long long*)bad);
  if (launches) *launches += 1;
}

}  // namespace b2s
