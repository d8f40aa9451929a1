// rows.cu — stable sort of length-prefixed UnsafeRow records by one typed key (the reduce side of a Spark SQL exchange:
// the SortExec a sort-merge join runs right after the shuffle read).  A decoded block is a sequence of
// [size: int32 big-endian][size bytes of row] records, as UnsafeRowSerializer writes them.  Steps, all on the device:
//   frame  : a warp per block (persistent grid, blocks taken from a counter) walks the size chain.  The walk only moves
//            forward, so the block is staged through a per-warp shared-memory ring of windows with cp.async, several
//            windows ahead of the walk; each hop is a shared-memory load.  A record longer than a window restarts the
//            staging at the next record.  Every record is validated; its start sets one bit of a bitmap over the decoded
//            arena (1 bit per byte), and a block's first bad record goes to its verdict
//   count  : set bits per 64 KiB tile of the arena, scanned: the record count, read back with the verdicts
//   emit   : the bitmap compacted into dense record offsets (u64) and lengths (u32, prefix included), arena order
//   keys   : one thread per record: the first bytes (at most kKeyPrefixBytes) of the encoded key (kernels.h, KeySpec)
//            as big-endian u32 words (one column: int32 / int64 byte-swapped, sign bit flipped; a nullable key gets a
//            leading byte 0 = null, 1 = non-null, and a null record's key bytes are 0; the composite calls' types and
//            order flags are further column encodings of the same function, encode_key)
//   radix  : the fixed-size sort's radix passes (launch_key_radix): the sorted record indices
//   refine : only for keys longer than the first pass: rounds over the records still tied (runs of equal first bytes
//            whose keys go on): compacted in order, their next kKeyChunkBytes bytes extracted behind their run number,
//            radix-sorted stably and put back into their runs' positions, until no run is tied.  A whole-row key (the
//            round-robin exchange's sort, launch_rows_whole_*) refines the same way, its rows read where they lie
//   gather : sorted lengths -> scan -> destination offsets (launch_sorted_offsets), the partition step's gather (a row
//            sort; a grouped aggregation gathers only each group's first record, aggregate.cu)
#include <algorithm>

#include "kernels.h"
#include "rows_key.cuh"

namespace b2s {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kFrameWarps = 4;
constexpr uint32_t kFrameWin = 1024;                     // bytes per staged window
constexpr uint32_t kFrameRing = 8;                       // windows per warp: the walk's two and six in flight
constexpr uint32_t kFrameRingBytes = kFrameWin * kFrameRing;
constexpr uint32_t kFrameChunks = kFrameWin / (16 * 32);  // 16-byte copies per lane per window
constexpr int kRowThreads = 256;
constexpr uint32_t kTileWords = kRowThreads * 8;          // bitmap words per count / emit tile (64 KiB of arena)

inline size_t a256(size_t b) { return (b + 255) / 256 * 256; }

inline unsigned grid_for(uint64_t n) {
  const uint64_t want = (n + kRowThreads - 1) / kRowThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

// Block b = arena bytes [r_off[b], r_off[b] + r_len[b]).  Window k of a block is arena bytes [A + k W, A + (k + 1) W)
// with A the block start rounded down to 16; it is staged in ring slot k mod R.  While the walk is in window k, windows
// k .. k + R - 1 have been issued (one cp.async group each, in order), so waiting until at most R - 2 groups are pending
// makes windows k and k + 1 resident: every size prefix that starts in window k lies in them.  A slot is refilled only
// once its window has landed and been walked (a pending copy into it could otherwise land after the new one).  16-byte
// pieces are copied while they start before the block end; the last may reach 15 bytes past it, into the arena's slack.
__global__ void __launch_bounds__(kFrameWarps * 32) rows_frame_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ r_off, const uint64_t* __restrict__ r_len,
    uint32_t n, uint64_t min_key, uint64_t min_null, uint64_t min_agg, uint32_t* __restrict__ bitmap,
    uint64_t* __restrict__ verdict,
    unsigned int* __restrict__ counter) {
  __shared__ __align__(16) uint32_t s_ring[kFrameWarps][kFrameRingBytes / 4];
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t* ring = s_ring[threadIdx.x >> 5];
  const uint32_t ring_s = (uint32_t)__cvta_generic_to_shared(ring);
  for (;;) {
    uint32_t b = 0;
    if (lane == 0) b = atomicAdd(counter, 1u);
    b = __shfl_sync(FULL, b, 0);
    if (b >= n) break;
    const uint64_t start = r_off[b], end = start + r_len[b];
    const uint64_t A = start & ~15ull;
    auto issue = [&](uint64_t k) {
      const uint64_t w0 = A + k * kFrameWin;
      const uint32_t slot = (uint32_t)(k % kFrameRing) * kFrameWin;
#pragma unroll
      for (uint32_t c = 0; c < kFrameChunks; c++) {
        const uint32_t o = (c * 32 + lane) * 16;
        if (w0 + o < end) cp_async16(ring_s + slot + o, arena + w0 + o);
      }
      cp_async_commit();
    };
    for (uint32_t j = 0; j < kFrameRing; j++) issue(j);
    uint64_t k = 0, p = start, bad = ~0ull;
    while (p < end) {
      const uint64_t kp = (p - A) / kFrameWin;
      if (kp != k) {
        if (kp == k + 1) {  // window k is resident and walked: its slot takes window k + R
          issue(k + kFrameRing);
        } else {  // a record longer than a window: let what is in flight land, restage from the next record
          cp_async_wait<0>();
          __syncwarp();
          for (uint32_t j = 0; j < kFrameRing; j++) issue(kp + j);
        }
        k = kp;
      }
      cp_async_wait<kFrameRing - 2>();
      __syncwarp();
      if (lane == 0) {  // the records that start in window k
        const uint64_t wend = A + (k + 1) * kFrameWin;
        uint64_t q = p, cw = q >> 5;
        uint32_t acc = 0;
        while (q < wend && q < end) {
          uint64_t why = 0;
          int32_t s = 0;
          if (q + 4 > end) {
            why = kRowsBadPrefix;
          } else {
            const uint32_t o = (uint32_t)(q - A) & (kFrameRingBytes - 1);
            const uint32_t lo = ring[o >> 2], hi = ring[((o >> 2) + 1) & (kFrameRingBytes / 4 - 1)];
            s = (int32_t)__byte_perm(__funnelshift_r(lo, hi, (o & 3) * 8), 0, 0x0123);
            if (s < 0) why = kRowsBadNegative;
            else if (q + 4 + (uint32_t)s > end) why = kRowsBadPastEnd;
            else if ((uint64_t)s < min_key) why = kRowsBadKey;
            else if ((uint64_t)s < min_null) why = kRowsBadNull;
            else if ((uint64_t)s < min_agg) why = kRowsBadAgg;
          }
          if (why) {
            bad = (why << 61) | (q - start);
            break;
          }
          if ((q >> 5) != cw) {
            if (acc) atomicOr(bitmap + cw, acc);
            cw = q >> 5;
            acc = 0;
          }
          acc |= 1u << (q & 31);
          q += 4 + (uint32_t)s;
        }
        if (acc) atomicOr(bitmap + cw, acc);
        p = q;
      }
      p = __shfl_sync(FULL, p, 0);
      bad = __shfl_sync(FULL, bad, 0);
      __syncwarp();  // lane 0's ring reads are done before the next refill overwrites a slot
      if (bad != ~0ull) break;
    }
    cp_async_wait<0>();  // nothing in flight into the ring when the next block starts
    __syncwarp();
    if (lane == 0) verdict[b] = bad;
  }
}

// Marks the records of ranges whose offsets are known (kernels.h, RowsMark), a thread per record: t-th marked record ->
// its mark by a binary search over the marks' first record numbers, its start from its stored offset, its size prefix
// from the arena.  A record the read's checks reject lowers its range's verdict, offset-major ((offset << 3) | why, so
// the lowest bad record wins; re-packed on the host); a good one sets its start bit.
__global__ void __launch_bounds__(kRowThreads) rows_mark_kernel(const uint8_t* __restrict__ arena,
                                                                const RowsMark* __restrict__ marks, uint32_t n_marks,
                                                                uint64_t total, uint64_t min_key, uint64_t min_null,
                                                                uint64_t min_agg, uint32_t* __restrict__ bitmap,
                                                                uint64_t* __restrict__ verdict) {
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = n_marks;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) / 2;
      if (marks[mid].first <= t) lo = mid;
      else hi = mid;
    }
    const RowsMark& m = marks[lo];
    const uint64_t q = m.base + m.off[t - m.first];
    const uint64_t s = __byte_perm(ld32u_ro(arena + q), 0, 0x0123);
    const uint64_t why = s < min_key ? kRowsBadKey : s < min_null ? kRowsBadNull : s < min_agg ? kRowsBadAgg : 0;
    if (why) atomicMin((unsigned long long*)(verdict + m.range), (unsigned long long)(((q - m.place) << 3) | why));
    else atomicOr(bitmap + (q >> 5), 1u << (q & 31));
  }
}

// exclusive scan of one u32 per thread over the CTA (kRowThreads threads)
__device__ __forceinline__ uint32_t cta_exclusive_scan(uint32_t v) {
  __shared__ uint32_t warp_sums[kRowThreads / 32];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(FULL, inc, d);
    if (lane >= (uint32_t)d) inc += t;
  }
  if (lane == 31) warp_sums[wid] = inc;
  __syncthreads();
  uint32_t before = 0;
  for (uint32_t w = 0; w < wid; w++) before += warp_sums[w];
  return before + inc - v;
}

// cnt[tile] = records starting in the tile's 64 KiB of arena; a thread takes 8 consecutive bitmap words
__global__ void __launch_bounds__(kRowThreads) rows_count_kernel(const uint32_t* __restrict__ bitmap,
                                                                 uint64_t* __restrict__ cnt) {
  __shared__ uint32_t warp_sums[kRowThreads / 32];
  const uint4* w = reinterpret_cast<const uint4*>(bitmap + (size_t)blockIdx.x * kTileWords) + threadIdx.x * 2;
  const uint4 a = w[0], b = w[1];
  uint32_t c = __popc(a.x) + __popc(a.y) + __popc(a.z) + __popc(a.w) + __popc(b.x) + __popc(b.y) + __popc(b.z) +
               __popc(b.w);
#pragma unroll
  for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(FULL, c, d);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int k = 0; k < kRowThreads / 32; k++) t += warp_sums[k];
    cnt[blockIdx.x] = t;
  }
}

// record j of the arena (tile_base: the scanned tile counts): rec_off[j] = its offset, rec_len[j] = 4 + its size
__global__ void __launch_bounds__(kRowThreads) rows_emit_kernel(const uint8_t* __restrict__ arena,
                                                                const uint32_t* __restrict__ bitmap,
                                                                const uint64_t* __restrict__ tile_base,
                                                                uint64_t* __restrict__ rec_off,
                                                                uint32_t* __restrict__ rec_len) {
  const uint64_t w0 = (uint64_t)blockIdx.x * kTileWords + threadIdx.x * 8;
  const uint4* w = reinterpret_cast<const uint4*>(bitmap + w0);
  const uint4 a = w[0], b = w[1];
  const uint32_t words[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint32_t c = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) c += __popc(words[k]);
  uint64_t j = tile_base[blockIdx.x] + cta_exclusive_scan(c);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    uint32_t m = words[k];
    while (m) {
      const uint64_t off = (w0 + k) * 32 + (uint32_t)(__ffs(m) - 1);
      m &= m - 1;
      rec_off[j] = off;
      rec_len[j] = 4 + __byte_perm(ld32u_ro(arena + off), 0, 0x0123);
      j++;
    }
  }
}

// The first pass: words[k * n + i] = word k of record i's encoded key, k < ceil(key_bytes / 4).  klen (keys that
// refine): klen[i] = the encoded length, and a record whose string runs past its row lowers its range's verdict
// (verdict[r], ranges: the ranges' arena offsets, ascending) to its offset in the range.  Eight CTAs per SM: the key
// pass of every row sort keeps full occupancy (32 registers, no spills with the wider encodings' branches).
__global__ void __launch_bounds__(kRowThreads, 8) rows_keys_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    uint64_t n, const __grid_constant__ KeySpec ks, uint32_t key_bytes, uint32_t* __restrict__ words,
    uint32_t* __restrict__ klen, const uint64_t* __restrict__ ranges, uint32_t n_ranges, uint64_t* __restrict__ verdict) {
  const uint32_t W = (key_bytes + 3) / 4;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t ro = rec_off[i];
    KeyWindow kw{0, 0, 0, 0, 0, 0, key_bytes};
    bool bad = false;
    const uint32_t len = encode_key(arena + ro + 4, rec_len[i] - 4, ks, kw, klen != nullptr, &bad);
#pragma unroll
    for (uint32_t k = 0; k < 5; k++)
      if (k < W) words[(size_t)k * n + i] = kw.word(k);
    if (klen) klen[i] = len;
    if (bad) {  // the range holding the record: the last that starts at or before it
      uint32_t lo = 0, hi = n_ranges;
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (ranges[mid] <= ro) lo = mid;
        else hi = mid;
      }
      atomicMin((unsigned long long*)(verdict + lo), (unsigned long long)((kRowsBadString << 61) | (ro - ranges[lo])));
    }
  }
}

// The join's key pass (kernels.h, JoinKeys): rows_keys_kernel with each record's side's columns and its fixed-region
// check.  A kernel of its own, so that the single-spec sorts keep theirs; NullSafe: a key with a B2S_KEY_NULL_SAFE
// column (encode_key), its own instantiation so that plain keys keep theirs.
template <bool NullSafe>
__global__ void __launch_bounds__(kRowThreads) rows_join_keys_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    uint64_t n, const __grid_constant__ JoinKeys jk, uint32_t key_bytes, uint32_t* __restrict__ words,
    uint32_t* __restrict__ klen, const uint64_t* __restrict__ ranges, uint32_t n_ranges,
    uint64_t* __restrict__ verdict) {
  const uint32_t W = (key_bytes + 3) / 4;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t ro = rec_off[i];
    const uint32_t s = ro >= jk.split, size = rec_len[i] - 4;
    KeyWindow kw{0, 0, 0, 0, 0, 0, key_bytes};
    bool bad = false;
    uint32_t len = 0;
    uint64_t why = 0;
    if (size < jk.fixed[s]) {  // its key slots and null words are not all inside it: not read
      why = kRowsBadKey;
    } else {
      len = encode_key<true, NullSafe>(arena + ro + 4, size, jk.side[s], kw, klen != nullptr, &bad);
      if (bad) why = kRowsBadString;
    }
#pragma unroll
    for (uint32_t k = 0; k < 5; k++)
      if (k < W) words[(size_t)k * n + i] = kw.word(k);
    if (klen) klen[i] = why ? 0 : len;
    if (why) {  // the range holding the record: the last that starts at or before it
      uint32_t lo = 0, hi = n_ranges;
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (ranges[mid] <= ro) lo = mid;
        else hi = mid;
      }
      atomicMin((unsigned long long*)(verdict + lo), (unsigned long long)((why << 61) | (ro - ranges[lo])));
    }
  }
}

// ---- refinement (keys longer than the first pass: kernels.h, launch_rows_refine_*) ----
// ord[j] = the record at position j of the current order, head[j] = 1 where a new key (so far) starts
__global__ void __launch_bounds__(kRowThreads) refine_init_kernel(const uint32_t* __restrict__ idx, uint64_t n,
                                                                  const uint32_t* __restrict__ words, uint32_t W,
                                                                  uint32_t* __restrict__ ord,
                                                                  uint32_t* __restrict__ head) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = idx ? idx[j] : (uint32_t)j;
    ord[j] = i;
    bool h = j == 0;
    if (!h) {
      const uint32_t p = idx ? idx[j - 1] : (uint32_t)(j - 1);
#pragma unroll
      for (uint32_t k = 0; k < 5; k++)
        if (k < W) h |= words[(size_t)k * n + i] != words[(size_t)k * n + p];
    }
    head[j] = h;
  }
}

// Position j is tied at byte d: its run of equal keys so far has two or more records, and its key goes on past d.
// Keys equal over [0, d) end together or both go on (the encoding is prefix-free), so a run is tied as a whole.
__device__ __forceinline__ bool tied(uint64_t j, uint64_t n, uint32_t d, const uint32_t* __restrict__ ord,
                                     const uint32_t* __restrict__ head, const uint32_t* __restrict__ klen) {
  return klen[ord[j]] > d && (!head[j] || (j + 1 < n && !head[j + 1]));
}

// scan[j] = head[j] << 32 | 1 for a tied position, else 0: its exclusive scan numbers the tied records and their runs
__global__ void __launch_bounds__(kRowThreads) refine_mark_kernel(const uint32_t* __restrict__ ord,
                                                                  const uint32_t* __restrict__ head,
                                                                  const uint32_t* __restrict__ klen, uint64_t n,
                                                                  uint32_t d, uint64_t* __restrict__ scan) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
    scan[j] = tied(j, n, d, ord, head, klen) ? ((uint64_t)head[j] << 32) | 1 : 0;
}

// tied position j, the k-th tied record, of run s: cpos[k] = j, cidx[k] = its record; its sort key (stride m) = s,
// then its encoded key bytes [d, d + kKeyChunkBytes)
__global__ void __launch_bounds__(kRowThreads) refine_extract_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    uint64_t n, const __grid_constant__ KeySpec ks, const uint32_t* __restrict__ ord, const uint32_t* __restrict__ head,
    const uint32_t* __restrict__ klen, const uint64_t* __restrict__ scan, uint64_t m, uint32_t d,
    uint32_t* __restrict__ cpos, uint32_t* __restrict__ cidx, uint32_t* __restrict__ words) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (!tied(j, n, d, ord, head, klen)) continue;
    const uint32_t k = (uint32_t)scan[j], s = (uint32_t)(scan[j] >> 32) + head[j] - 1;
    const uint32_t i = ord[j];
    cpos[k] = (uint32_t)j;
    cidx[k] = i;
    KeyWindow kw{0, 0, 0, 0, 0, d, kKeyChunkBytes};
    bool bad = false;
    encode_key(arena + rec_off[i] + 4, rec_len[i] - 4, ks, kw, false, &bad);
    words[k] = s;
#pragma unroll
    for (uint32_t q = 0; q < 4; q++) words[(size_t)(q + 1) * m + k] = kw.word(q);
  }
}

// refine_extract_kernel for a join's keys: each record with its side's columns (a bad record has key length 0: never
// tied, never read here)
template <bool NullSafe>
__global__ void __launch_bounds__(kRowThreads) refine_extract_join_kernel(
    const uint8_t* __restrict__ arena, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    uint64_t n, const __grid_constant__ JoinKeys jk, const uint32_t* __restrict__ ord,
    const uint32_t* __restrict__ head, const uint32_t* __restrict__ klen, const uint64_t* __restrict__ scan, uint64_t m,
    uint32_t d,
    uint32_t* __restrict__ cpos, uint32_t* __restrict__ cidx, uint32_t* __restrict__ words) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (!tied(j, n, d, ord, head, klen)) continue;
    const uint32_t k = (uint32_t)scan[j], s = (uint32_t)(scan[j] >> 32) + head[j] - 1;
    const uint32_t i = ord[j];
    cpos[k] = (uint32_t)j;
    cidx[k] = i;
    KeyWindow kw{0, 0, 0, 0, 0, d, kKeyChunkBytes};
    bool bad = false;
    encode_key<true, NullSafe>(arena + rec_off[i] + 4, rec_len[i] - 4, jk.side[rec_off[i] >= jk.split], kw, false, &bad);
    words[k] = s;
#pragma unroll
    for (uint32_t q = 0; q < 4; q++) words[(size_t)(q + 1) * m + k] = kw.word(q);
  }
}

// Bytes [d, d + kKeyChunkBytes) of a whole-row key (kernels.h, launch_rows_whole_order) as four big-endian words, for
// d = 4 + 16 r: the size word and row bytes [0, 12) when d == 4, else row bytes [d - 8, d + 8); zero past the row.
// The row's size is a multiple of 8, so every word lies wholly inside or wholly past it.
__device__ __forceinline__ uint4 row_key_window(const uint8_t* row, uint32_t size, uint32_t d) {
  const uint32_t from = d == 4 ? 0 : d - 8, want = d == 4 ? 12 : 16;
  const uint32_t take = from < size ? min(size - from, want) : 0;
  uint64_t lo = 0, hi = 0;
  if (take) {
    ld_span16<true>(row + from, (int)take, lo, hi);
    if (take < 8) lo &= (1ull << (8 * take)) - 1;
    hi = take <= 8 ? 0 : take < 16 ? hi & ((1ull << (8 * (take - 8))) - 1) : hi;
  }
  const uint32_t a = __byte_perm((uint32_t)lo, 0, 0x0123), b = __byte_perm((uint32_t)(lo >> 32), 0, 0x0123);
  const uint32_t c = __byte_perm((uint32_t)hi, 0, 0x0123), e = __byte_perm((uint32_t)(hi >> 32), 0, 0x0123);
  return d == 4 ? make_uint4(size, a, b, c) : make_uint4(a, b, c, e);
}

// refine_extract_kernel for whole-row keys: the records are read where they lie (rec + rec_off[i], rec_len[i] bytes,
// framed), only tied ones, whose key length (klen) says they are whole rows inside the records
__global__ void __launch_bounds__(kRowThreads) refine_extract_row_kernel(
    const uint8_t* __restrict__ rec, const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ rec_len,
    uint64_t n, const uint32_t* __restrict__ ord, const uint32_t* __restrict__ head, const uint32_t* __restrict__ klen,
    const uint64_t* __restrict__ scan, uint64_t m, uint32_t d, uint32_t* __restrict__ cpos, uint32_t* __restrict__ cidx,
    uint32_t* __restrict__ words) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    if (!tied(j, n, d, ord, head, klen)) continue;
    const uint32_t k = (uint32_t)scan[j], s = (uint32_t)(scan[j] >> 32) + head[j] - 1;
    const uint32_t i = ord[j];
    cpos[k] = (uint32_t)j;
    cidx[k] = i;
    const uint4 w = row_key_window(rec + rec_off[i] + 4, rec_len[i] - 4, d);
    words[k] = s;
    words[m + k] = w.x;
    words[2 * m + k] = w.y;
    words[3 * m + k] = w.z;
    words[4 * m + k] = w.w;
  }
}

// the k-th of the sorted tied records (sidx) to the k-th tied position; a new key starts where (run, bytes) changes
__global__ void __launch_bounds__(kRowThreads) refine_scatter_kernel(const uint32_t* __restrict__ sidx, uint64_t m,
                                                                     const uint32_t* __restrict__ words,
                                                                     const uint32_t* __restrict__ cpos,
                                                                     const uint32_t* __restrict__ cidx,
                                                                     uint32_t* __restrict__ ord,
                                                                     uint32_t* __restrict__ head) {
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = sidx ? sidx[k] : (uint32_t)k, j = cpos[k];
    ord[j] = cidx[r];
    bool h = k == 0;
    if (!h) {
      const uint32_t p = sidx ? sidx[k - 1] : (uint32_t)(k - 1);
#pragma unroll
      for (uint32_t q = 0; q < 5; q++) h |= words[(size_t)q * m + r] != words[(size_t)q * m + p];
    }
    head[j] = h;
  }
}

// the refinement workspace (kernels.h, rows_refine_ws_bytes)
struct RefineWs {
  uint32_t* ord;
  uint32_t* head;
  uint32_t* klen;
  uint32_t* cpos;
  uint32_t* cidx;
  uint64_t* scan;
  uint64_t* scan_ws;
  uint64_t* readback;
};

RefineWs carve_refine_ws(uint8_t* d_rws, uint64_t n) {
  RefineWs r;
  uint8_t* p = d_rws;
  r.ord = (uint32_t*)p;     p += a256(n * 4);
  r.head = (uint32_t*)p;    p += a256(n * 4);
  r.klen = (uint32_t*)p;    p += a256(n * 4);
  r.cpos = (uint32_t*)p;    p += a256(n * 4);
  r.cidx = (uint32_t*)p;    p += a256(n * 4);
  r.scan = (uint64_t*)p;    p += a256(n * 8);
  r.scan_ws = (uint64_t*)p; p += a256(scan_ws_elems(n) * 8);
  r.readback = (uint64_t*)p;
  return r;
}

// a refinement round's end: the m extracted (run, bytes) keys sorted stably and put back into their runs' positions
void refine_sort_scatter(const KeySortWs& w, const RefineWs& r, uint64_t m, uint64_t segs, cudaStream_t st,
                         uint64_t* launches) {
  // the run number takes as many passes as it has bytes (none for a single run)
  const uint32_t lead = segs <= 1 ? 0 : segs <= 256 ? 1 : segs <= 65536 ? 2 : segs <= (1u << 24) ? 3 : 4;
  const uint32_t* sidx = launch_key_radix(w, m, 4 + kKeyChunkBytes, st, launches, lead);
  refine_scatter_kernel<<<grid_for(m), kRowThreads, 0, st>>>(sidx, m, w.words, r.cpos, r.cidx, r.ord, r.head);
}

// the framing workspace: bitmap (whole tiles), tile counts, their scan workspace, readback, ranges, work counter
struct FrameWs {
  uint32_t* bitmap;
  uint64_t* tile_cnt;
  uint64_t* scan_ws;
  uint64_t* readback;
  uint64_t* r_off;
  uint64_t* r_len;
  unsigned int* counter;
  RowsMark* marks;
  uint64_t tiles;
};

inline uint64_t frame_tiles(uint64_t arena_bytes) {
  const uint64_t words = (arena_bytes + 31) / 32;
  return std::max<uint64_t>((words + kTileWords - 1) / kTileWords, 1);
}

FrameWs carve_frame_ws(uint8_t* d_fws, uint64_t arena_bytes, uint32_t n_ranges) {
  FrameWs f;
  f.tiles = frame_tiles(arena_bytes);
  uint8_t* p = d_fws;
  f.bitmap = (uint32_t*)p;   p += a256(f.tiles * kTileWords * 4);
  f.tile_cnt = (uint64_t*)p; p += a256(f.tiles * 8);
  f.scan_ws = (uint64_t*)p;  p += a256(scan_ws_elems(f.tiles) * 8);
  f.readback = (uint64_t*)p; p += a256(rows_frame_readback_bytes(n_ranges));
  f.r_off = (uint64_t*)p;    p += a256((size_t)n_ranges * 8);
  f.r_len = (uint64_t*)p;    p += a256((size_t)n_ranges * 8);
  f.counter = (unsigned int*)p; p += 256;
  f.marks = (RowsMark*)p;
  return f;
}

}  // namespace

size_t rows_frame_ws_bytes(uint64_t arena_bytes, uint32_t n_ranges, uint32_t n_marks) {
  const uint64_t tiles = frame_tiles(arena_bytes);
  return a256(tiles * kTileWords * 4) + a256(tiles * 8) + a256(scan_ws_elems(tiles) * 8) +
         a256(rows_frame_readback_bytes(n_ranges)) + 2 * a256((size_t)n_ranges * 8) + 256 +
         a256((size_t)n_marks * sizeof(RowsMark));
}

uint64_t* rows_frame_readback(uint8_t* d_fws, uint64_t arena_bytes, uint32_t n_ranges) {
  return carve_frame_ws(d_fws, arena_bytes, n_ranges).readback;
}

void launch_rows_frame(const uint8_t* arena, uint64_t arena_bytes, const uint64_t* h_off, const uint64_t* h_len,
                       uint32_t n_ranges, uint64_t min_key, uint64_t min_null, uint64_t min_agg, uint8_t* d_fws,
                       cudaStream_t st, uint64_t* launches, const RowsMark* h_marks, uint32_t n_marks) {
  const FrameWs f = carve_frame_ws(d_fws, arena_bytes, n_ranges);
  cudaMemsetAsync(f.bitmap, 0, f.tiles * kTileWords * 4, st);
  cudaMemsetAsync(f.readback, 0xff, rows_frame_readback_bytes(n_ranges), st);
  cudaMemsetAsync(f.counter, 0, sizeof(unsigned int), st);
  if (n_ranges) {
    cudaMemcpyAsync(f.r_off, h_off, (size_t)n_ranges * 8, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(f.r_len, h_len, (size_t)n_ranges * 8, cudaMemcpyHostToDevice, st);
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rows_frame_kernel, kFrameWarps * 32, 0);
    if (per_sm < 1) per_sm = 1;
    const uint64_t want = ((uint64_t)n_ranges + kFrameWarps - 1) / kFrameWarps;
    const uint64_t grid = std::min<uint64_t>((uint64_t)kSMs * per_sm, want);  // persistent: one wave
    rows_frame_kernel<<<(unsigned)grid, kFrameWarps * 32, 0, st>>>(arena, f.r_off, f.r_len, n_ranges, min_key,
                                                                    min_null, min_agg, f.bitmap, f.readback + 1,
                                                                    f.counter);
    if (launches) *launches += 1;
  }
  // after the walk, which writes every range's verdict (a marked range's walk is empty)
  const uint64_t marked = n_marks ? h_marks[n_marks - 1].first + h_marks[n_marks - 1].count : 0;
  if (marked) {
    cudaMemcpyAsync(f.marks, h_marks, (size_t)n_marks * sizeof(RowsMark), cudaMemcpyHostToDevice, st);
    rows_mark_kernel<<<grid_for(marked), kRowThreads, 0, st>>>(arena, f.marks, n_marks, marked, min_key, min_null,
                                                               min_agg, f.bitmap, f.readback + 1);
    if (launches) *launches += 1;
  }
  rows_count_kernel<<<(unsigned)f.tiles, kRowThreads, 0, st>>>(f.bitmap, f.tile_cnt);
  launch_exclusive_scan_u64(f.tile_cnt, f.tiles, f.readback, f.scan_ws, st, launches);
  if (launches) *launches += 1;
}

size_t rows_sort_ws_bytes(uint64_t n, uint32_t key_bytes) {
  return key_sort_ws_bytes(n, key_bytes) + a256(scan_ws_elems(n) * 8);
}

void launch_rows_emit(const uint8_t* arena, uint64_t arena_bytes, uint32_t n_ranges, uint8_t* d_fws, uint64_t n,
                      uint32_t key_bytes, uint8_t* d_ws, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  const FrameWs f = carve_frame_ws(d_fws, arena_bytes, n_ranges);
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  rows_emit_kernel<<<(unsigned)f.tiles, kRowThreads, 0, st>>>(arena, f.bitmap, f.tile_cnt, w.src_off, w.len);
  if (launches) *launches += 1;
}

const uint64_t* rows_frame_ranges(uint8_t* d_fws, uint64_t arena_bytes, uint32_t n_ranges) {
  return carve_frame_ws(d_fws, arena_bytes, n_ranges).r_off;
}

size_t rows_refine_ws_bytes(uint64_t n, uint32_t n_ranges) {
  return 5 * a256(n * 4) + a256(n * 8) + a256(scan_ws_elems(n) * 8) + a256(((size_t)n_ranges + 1) * 8);
}

uint64_t* rows_refine_readback(uint8_t* d_rws, uint64_t n, uint32_t) { return carve_refine_ws(d_rws, n).readback; }
const uint32_t* rows_refine_order(uint8_t* d_rws, uint64_t n, uint32_t) { return carve_refine_ws(d_rws, n).ord; }
const uint32_t* rows_refine_heads(uint8_t* d_rws, uint64_t n, uint32_t) { return carve_refine_ws(d_rws, n).head; }

const uint32_t* launch_rows_order(const uint8_t* arena, uint64_t n, const KeySpec& ks, const uint64_t* ranges,
                                  uint32_t n_ranges, uint8_t* d_ws, uint8_t* d_rws, cudaStream_t st,
                                  uint64_t* launches) {
  if (!n) return nullptr;
  const uint32_t key_bytes = rows_key_bytes(ks);
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  RefineWs r{};
  if (d_rws) {
    r = carve_refine_ws(d_rws, n);
    cudaMemsetAsync(r.readback + 1, 0xff, (size_t)n_ranges * 8, st);
  }
  rows_keys_kernel<<<grid_for(n), kRowThreads, 0, st>>>(arena, w.src_off, w.len, n, ks, key_bytes, w.words, r.klen,
                                                        ranges, n_ranges, d_rws ? r.readback + 1 : nullptr);
  if (launches) *launches += 1;
  const uint32_t* idx = launch_key_radix(w, n, key_bytes, st, launches);
  if (d_rws) {
    refine_init_kernel<<<grid_for(n), kRowThreads, 0, st>>>(idx, n, w.words, (key_bytes + 3) / 4, r.ord, r.head);
    if (launches) *launches += 1;
  }
  return idx;
}

// a join key with a B2S_KEY_NULL_SAFE column (both sides have the same types)
static bool join_null_safe(const JoinKeys& jk) {
  for (uint32_t c = 0; c < jk.side[0].n; c++)
    if (jk.side[0].type[c] & B2S_KEY_NULL_SAFE) return true;
  return false;
}

const uint32_t* launch_rows_join_order(const uint8_t* arena, uint64_t n, const JoinKeys& jk, const uint64_t* ranges,
                                       uint32_t n_ranges, uint64_t* verdict, uint8_t* d_ws, uint8_t* d_rws,
                                       cudaStream_t st, uint64_t* launches) {
  cudaMemsetAsync(verdict, 0xff, (size_t)n_ranges * 8, st);
  if (!n) return nullptr;
  const uint32_t key_bytes = rows_key_bytes(jk.side[0]);
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  RefineWs r{};
  if (d_rws) {  // the verdicts are the join's: the refinement's first readback finds none
    r = carve_refine_ws(d_rws, n);
    cudaMemsetAsync(r.readback + 1, 0xff, (size_t)n_ranges * 8, st);
  }
  auto keys = join_null_safe(jk) ? rows_join_keys_kernel<true> : rows_join_keys_kernel<false>;
  keys<<<grid_for(n), kRowThreads, 0, st>>>(arena, w.src_off, w.len, n, jk, key_bytes, w.words, r.klen, ranges, n_ranges,
                                            verdict);
  if (launches) *launches += 1;
  const uint32_t* idx = launch_key_radix(w, n, key_bytes, st, launches);
  if (d_rws) {
    refine_init_kernel<<<grid_for(n), kRowThreads, 0, st>>>(idx, n, w.words, (key_bytes + 3) / 4, r.ord, r.head);
    if (launches) *launches += 1;
  }
  return idx;
}

void launch_rows_join_refine_round(const uint8_t* arena, uint64_t n, const JoinKeys& jk, uint64_t m, uint64_t segs,
                                   uint32_t d, uint8_t* d_ws, uint8_t* d_rws, cudaStream_t st, uint64_t* launches) {
  const KeySortWs w = carve_key_sort_ws(d_ws, n, kKeyPrefixBytes);
  const RefineWs r = carve_refine_ws(d_rws, n);
  auto extract = join_null_safe(jk) ? refine_extract_join_kernel<true> : refine_extract_join_kernel<false>;
  extract<<<grid_for(n), kRowThreads, 0, st>>>(arena, w.src_off, w.len, n, jk, r.ord, r.head, r.klen, r.scan, m, d,
                                               r.cpos, r.cidx, w.words);
  refine_sort_scatter(w, r, m, segs, st, launches);
  if (launches) *launches += 2;
}

void launch_rows_refine_mark(uint64_t n, uint32_t d, uint8_t* d_rws, uint32_t, cudaStream_t st, uint64_t* launches) {
  const RefineWs r = carve_refine_ws(d_rws, n);
  refine_mark_kernel<<<grid_for(n), kRowThreads, 0, st>>>(r.ord, r.head, r.klen, n, d, r.scan);
  launch_exclusive_scan_u64(r.scan, n, r.readback, r.scan_ws, st, launches);
  if (launches) *launches += 1;
}

void launch_rows_refine_round(const uint8_t* arena, uint64_t n, const KeySpec& ks, uint64_t m, uint64_t segs,
                              uint32_t d, uint8_t* d_ws, uint8_t* d_rws, uint32_t, cudaStream_t st,
                              uint64_t* launches) {
  // the first pass's workspace, its key words no longer needed: the m tied records' keys at stride m
  const KeySortWs w = carve_key_sort_ws(d_ws, n, kKeyPrefixBytes);
  const RefineWs r = carve_refine_ws(d_rws, n);
  refine_extract_kernel<<<grid_for(n), kRowThreads, 0, st>>>(arena, w.src_off, w.len, n, ks, r.ord, r.head, r.klen,
                                                             r.scan, m, d, r.cpos, r.cidx, w.words);
  refine_sort_scatter(w, r, m, segs, st, launches);
  if (launches) *launches += 2;
}

uint32_t* rows_whole_words(uint8_t* d_ws, uint64_t n) { return carve_key_sort_ws(d_ws, n, kKeyPrefixBytes).words; }
uint32_t* rows_refine_klen(uint8_t* d_rws, uint64_t n) { return carve_refine_ws(d_rws, n).klen; }

void launch_rows_whole_order(uint64_t n, uint8_t* d_ws, uint8_t* d_rws, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  const KeySortWs w = carve_key_sort_ws(d_ws, n, kKeyPrefixBytes);
  const RefineWs r = carve_refine_ws(d_rws, n);
  const uint32_t* idx = launch_key_radix(w, n, 4, st, launches);
  refine_init_kernel<<<grid_for(n), kRowThreads, 0, st>>>(idx, n, w.words, 1, r.ord, r.head);
  if (launches) *launches += 1;
}

void launch_rows_whole_refine_round(const uint8_t* rec, const uint64_t* rec_off, const uint32_t* rec_len, uint64_t n,
                                    uint64_t m, uint64_t segs, uint32_t d, uint8_t* d_ws, uint8_t* d_rws,
                                    cudaStream_t st, uint64_t* launches) {
  const KeySortWs w = carve_key_sort_ws(d_ws, n, kKeyPrefixBytes);
  const RefineWs r = carve_refine_ws(d_rws, n);
  refine_extract_row_kernel<<<grid_for(n), kRowThreads, 0, st>>>(rec, rec_off, rec_len, n, r.ord, r.head, r.klen,
                                                                 r.scan, m, d, r.cpos, r.cidx, w.words);
  refine_sort_scatter(w, r, m, segs, st, launches);
  if (launches) *launches += 2;
}

void launch_rows_gather(const uint8_t* arena, uint64_t n, uint32_t key_bytes, const uint32_t* idx, uint8_t* d_ws,
                        uint8_t* d_dst, cudaStream_t st, uint64_t* launches, uint64_t count) {
  const uint64_t m = count < n ? count : n;
  if (!m) return;
  const KeySortWs w = carve_key_sort_ws(d_ws, n, key_bytes);
  uint64_t* offsets_scan_ws = (uint64_t*)(d_ws + key_sort_ws_bytes(n, key_bytes));
  PartitionPlan plan;
  plan.src_off = w.src_off;
  plan.sdst = w.sdst;
  plan.idx = idx;
  launch_sorted_offsets(plan.idx, w.len, m, w.sdst, w.total, offsets_scan_ws, st, launches);
  launch_partition_gather(arena, w.len, m, plan, d_dst, st, launches);
}

}  // namespace b2s
