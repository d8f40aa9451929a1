// snappy.cu — K5: Snappy (xerial SnappyOutputStream framing) on the same multi-kernel skeleton as LZ4.
//
// Replaces, for spark.io.compression.codec=snappy, org.xerial.snappy.SnappyOutputStream / SnappyInputStream [U]
// (snappy-java 1.1.10.x -> native snappy::RawCompress / RawUncompress) under SerializerManager.wrapStream at
// shuffle/S3ShuffleMapOutputWriter.scala:140-146 (write) and storage/S3ShuffleReader.scala:107-109 (read).
// Wire format (oracle/b2s_oracle.c restates it): 16-byte stream header {0x82 "SNAPPY" 0x00, BE32 version=1, BE32 compat=1},
// then per <= blockSize (32 KiB) bytes of input: BE32 compressedLength | raw snappy block (varint uncompressed length,
// literal / copy elements).  A header may re-occur mid-stream (concatenated streams).
//
// write: lz4_match_kernel (shared, lz4_compress.cu) -> lz4_parse_kernel<SNAPPY> (shared, element sizes differ)
//        -> snappy_emit_kernel (lane per sequence, Snappy element grammar) ; specification: orc_snappy_compress_raw_win
// read : xerial_walk_kernel (chunk descriptors) -> snappy_tokens_kernel (thread per chunk: elements -> 8-byte records)
//        -> snappy_copy_kernel (warp per chunk, lane per record; literal and match copies shared with the LZ4 decoder,
//        lz_batch.cuh)
#include "kernels.h"
#include "lz_batch.cuh"

namespace b2s {

__device__ __forceinline__ uint32_t find_stream_sn(const uint32_t* __restrict__ blk_base, uint32_t n_streams, uint32_t b) {
  uint32_t lo = 0, hi = n_streams;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (blk_base[mid] <= b) lo = mid; else hi = mid;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------------------------
// write side: emission
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int sn_varint_len(uint32_t n) { return n < 128 ? 1 : n < 16384 ? 2 : 3; }
__device__ __forceinline__ int sn_literal_header(int lit) { return lit - 1 < 60 ? 1 : lit - 1 < 256 ? 2 : 3; }
// one copy element of 4..64 bytes
__device__ __forceinline__ uint8_t* sn_put_copy(uint8_t* q, int off, int len) {
  if (len < 12 && off < 2048) {
    *q++ = (uint8_t)(1 | ((len - 4) << 2) | ((off >> 8) << 5));
    *q++ = (uint8_t)off;
  } else {
    *q++ = (uint8_t)(2 | ((len - 1) << 2));
    *q++ = (uint8_t)off;
    *q++ = (uint8_t)(off >> 8);
  }
  return q;
}
__device__ __forceinline__ uint8_t* sn_put_copies(uint8_t* q, int off, int len) {  // snappy's EmitCopy
  while (len >= 68) {
    q = sn_put_copy(q, off, 64);
    len -= 64;
  }
  if (len > 64) {
    q = sn_put_copy(q, off, 60);
    len -= 60;
  }
  return sn_put_copy(q, off, len);
}
__device__ __forceinline__ uint8_t* sn_put_literal_header(uint8_t* q, int lit) {
  const int n1 = lit - 1;
  if (n1 < 60) {
    *q++ = (uint8_t)(n1 << 2);
  } else if (n1 < 256) {
    *q++ = (uint8_t)(60 << 2);
    *q++ = (uint8_t)n1;
  } else {
    *q++ = (uint8_t)(61 << 2);
    *q++ = (uint8_t)n1;
    *q++ = (uint8_t)(n1 >> 8);
  }
  return q;
}

constexpr int kSnEmitThreads = 256;
// records as written by lz4_parse_kernel<SNAPPY>: x = literal start | literal count << 16 ; y = match length | op << 16
__global__ void __launch_bounds__(kSnEmitThreads) snappy_emit_kernel(
    const uint8_t* __restrict__ src_base, const uint64_t* __restrict__ src_off, const uint64_t* __restrict__ src_len,
    const uint32_t* __restrict__ blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
    uint32_t stride, uint32_t max_seq, const uint16_t* __restrict__ offarr, const uint2* __restrict__ seqarr,
    const uint32_t* __restrict__ nseq, const uint32_t* __restrict__ csize, const uint64_t* __restrict__ scan,
    uint8_t* __restrict__ dst_base, uint64_t dst_cap) {
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const uint32_t bl = blockIdx.x * (kSnEmitThreads / 32) + (threadIdx.x >> 5);
  if (bl >= m) return;
  const uint32_t b = b0 + bl;
  const uint32_t si = find_stream_sn(blk_base, n_streams, b);
  const uint64_t boff = (uint64_t)(b - blk_base[si]) * block_size;
  const uint64_t rem = src_len[si] - boff;
  const uint32_t n = (uint32_t)(rem < block_size ? rem : block_size);
  const uint8_t* __restrict__ s = src_base + src_off[si] + boff;
  const uint32_t clen = csize[b];
  const uint64_t o0 = scan[b] + 16ull * (si + 1);  // every stream up to and including mine starts with a 16-byte header
  if (o0 + 4ull + clen > dst_cap) return;          // the stream-meta kernel reports B2S_E_DST_TOO_SMALL
  uint8_t* __restrict__ o = dst_base + o0;
  if (lane < 4) o[lane] = (uint8_t)(clen >> (8 * (3 - lane)));  // BE32 compressed length
  uint8_t* __restrict__ out = o + 4;
  if (lane == 0) {  // varint(uncompressed length)
    uint8_t* q = out;
    uint32_t v = n;
    while (v >= 0x80) {
      *q++ = (uint8_t)(v | 0x80);
      v >>= 7;
    }
    *q = (uint8_t)v;
  }
  const uint32_t ns = nseq[b];
  const uint2* __restrict__ seq = seqarr + (size_t)bl * max_seq;
  const uint16_t* __restrict__ offp = offarr + (size_t)bl * stride;
  for (uint32_t i0 = 0; i0 < ns; i0 += 32) {
    const uint32_t i = i0 + lane;
    bool slow = false;
    int anchor = 0, lit = 0, ml = 0, op = 0, off = 0;
    if (i < ns) {
      const uint2 r = seq[i];
      anchor = (int)(r.x & 0xffffu);
      lit = (int)(r.x >> 16);
      ml = (int)(r.y & 0xffffu);
      op = (int)(r.y >> 16);
      if (ml) off = offp[anchor + lit] & (stride <= 32768u ? 0x7fff : 0xffff);  // bit 15: parse flag (lz4_compress.cu)
      if (lit <= 16) {
        uint8_t* q = out + op;
        if (lit) {
          *q++ = (uint8_t)((lit - 1) << 2);
          const uint8_t* ls = s + anchor;
          for (int j = 0; j < lit; j++) q[j] = __ldg(ls + j);
          q += lit;
        }
        if (ml) sn_put_copies(q, off, ml);
      } else {
        slow = true;
      }
    }
    unsigned slowmask = __ballot_sync(FULL, slow);
    while (slowmask) {  // long literal run: header + copy elements by the owner, the bytes by the whole warp
      const int l = __ffs(slowmask) - 1;
      slowmask &= slowmask - 1;
      const int a_r = __shfl_sync(FULL, anchor, l);
      const int lit_r = __shfl_sync(FULL, lit, l);
      const int op_r = __shfl_sync(FULL, op, l);
      const int hdr = sn_literal_header(lit_r);
      if (lane == l) {
        uint8_t* q = sn_put_literal_header(out + op_r, lit);
        if (ml) sn_put_copies(q + lit, off, ml);
      }
      uint8_t* q = out + op_r + hdr;
      if (lit_r >= 96) group_copy<32>(q, s + a_r, (uint32_t)lit_r, lane);
      else
        for (int j = lane; j < lit_r; j += 32) q[j] = __ldg(s + a_r + j);
    }
  }
}

// per stream: 16-byte header at the stream's start, packed offset/length, capacity check
__global__ void xerial_stream_meta_kernel(const uint32_t* __restrict__ blk_base, uint32_t n_streams, uint32_t n_blocks,
                                          const uint64_t* __restrict__ scan, const uint64_t* __restrict__ scan_total,
                                          uint8_t* __restrict__ dst_base, uint64_t dst_cap,
                                          uint64_t* __restrict__ dst_off, uint64_t* __restrict__ dst_len,
                                          int32_t* __restrict__ status) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_streams) return;
  const uint32_t b0 = blk_base[i], b1 = blk_base[i + 1];
  const uint64_t s0 = b0 < n_blocks ? scan[b0] : *scan_total;
  const uint64_t s1 = b1 < n_blocks ? scan[b1] : *scan_total;
  const uint64_t off = s0 + 16ull * i;
  const uint64_t len = (s1 - s0) + 16ull;
  dst_off[i] = off;
  dst_len[i] = len;
  if (off + len > dst_cap) {
    status[i] = B2S_E_DST_TOO_SMALL;
    return;
  }
  const uint8_t hdr[16] = {0x82, 'S', 'N', 'A', 'P', 'P', 'Y', 0, 0, 0, 0, 1, 0, 0, 0, 1};
  uint8_t* e = dst_base + off;
#pragma unroll
  for (int j = 0; j < 16; j++) e[j] = hdr[j];
}

void launch_snappy_emit(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                        const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
                        uint32_t stride, uint32_t max_seq, const uint16_t* d_off, const uint2* d_seq,
                        const uint32_t* d_nseq, const uint32_t* d_csize, const uint64_t* d_scan, uint8_t* dst_base,
                        uint64_t dst_cap, cudaStream_t st, uint64_t* launches) {
  if (!m) return;
  snappy_emit_kernel<<<(m + kSnEmitThreads / 32 - 1) / (kSnEmitThreads / 32), kSnEmitThreads, 0, st>>>(
      src_base, d_src_off, d_src_len, d_blk_base, n_streams, b0, m, block_size, stride, max_seq, d_off, d_seq, d_nseq,
      d_csize, d_scan, dst_base, dst_cap);
  *launches += 1;
}

void launch_xerial_stream_meta(const uint32_t* d_blk_base, uint32_t n_streams, uint32_t n_blocks, const uint64_t* d_scan,
                               const uint64_t* d_scan_total, uint8_t* dst_base, uint64_t dst_cap, uint64_t* d_dst_off,
                               uint64_t* d_dst_len, int32_t* d_status, cudaStream_t st, uint64_t* launches) {
  if (!n_streams) return;
  xerial_stream_meta_kernel<<<(n_streams + 255) / 256, 256, 0, st>>>(d_blk_base, n_streams, n_blocks, d_scan,
                                                                     d_scan_total, dst_base, dst_cap, d_dst_off,
                                                                     d_dst_len, d_status);
  *launches += 1;
}

// ------------------------------------------------------------------------------------------------------------
// read side: xerial chunk walk (SnappyInputStream.hasNextChunk / readHeader [U])
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_be32(const uint8_t* p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
// varint at p (at most `avail` bytes): returns bytes used (0 = malformed) and the value
__device__ __forceinline__ int sn_read_varint(const uint8_t* p, uint64_t avail, uint32_t* out) {
  uint64_t v = 0;
  for (int i = 0; i < 5; i++) {
    if ((uint64_t)i >= avail) return 0;
    const uint8_t b = p[i];
    v |= (uint64_t)(b & 0x7f) << (7 * i);
    if (!(b & 0x80)) {
      if (v > 0xffffffffull) return 0;
      *out = (uint32_t)v;
      return i + 1;
    }
  }
  return 0;
}

template <bool FILL>
__global__ void xerial_walk_kernel(const uint8_t* __restrict__ src_base, const uint64_t* __restrict__ src_off,
                                   const uint64_t* __restrict__ src_len, uint32_t n, uint64_t* __restrict__ nblk,
                                   uint64_t* __restrict__ olen_total, unsigned long long* __restrict__ maxima,
                                   const uint64_t* __restrict__ blk_base, const uint64_t* __restrict__ dst_off,
                                   uint64_t dst_cap, int32_t* __restrict__ status, BlockDesc* __restrict__ desc) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (FILL && status[i] != 0 && status[i] != B2S_E_DST_TOO_SMALL) return;
  if (!FILL && status[i] != 0) {
    nblk[i] = 0;
    olen_total[i] = 0;
    return;
  }
  const uint8_t* p = src_base + src_off[i];
  const uint64_t len = src_len[i];
  uint64_t ip = 0, cnt = 0, total = 0;
  uint32_t max_olen = 0, max_clen = 0;
  bool bad = false, too_small = false;
  if (FILL) too_small = (dst_off[i] + olen_total[i] > dst_cap);
  // stream header: magic 82 53 4E 41 50 50 59 00, then version / compatible version (not checked beyond presence).
  // No bytes at all is an empty stream, as SnappyInputStream.readHeader takes it (a partition the map side wrote
  // nothing for, fetched alone).
  if (len && (len < 16 || ld_be32(p) != 0x82534E41u || ld_be32(p + 4) != 0x50505900u)) bad = true;
  ip = 16;
  while (!bad && ip < len) {
    if (len - ip < 4) {
      bad = true;
      break;
    }
    const uint32_t clen = ld_be32(p + ip);
    ip += 4;
    if (clen == 0x82534E41u) {  // a concatenated stream's header sits in the length slot
      if (len - ip < 12 || ld_be32(p + ip) != 0x50505900u) {
        bad = true;
        break;
      }
      ip += 12;
      continue;
    }
    if ((uint64_t)clen > len - ip) {
      bad = true;
      break;
    }
    uint32_t ulen = 0;
    const int vb = sn_read_varint(p + ip, clen, &ulen);
    if (!vb) {
      bad = true;
      break;
    }
    if (FILL) {
      BlockDesc d;
      d.src = src_off[i] + ip + vb;  // elements start after the varint
      d.dst = dst_off[i] + total;
      d.clen = too_small ? 0u : clen - (uint32_t)vb;
      d.olen = too_small ? 0u : ulen;
      d.check = 0;
      d.stream = i;
      desc[blk_base[i] + cnt] = d;
    } else {
      max_olen = max_olen > ulen ? max_olen : ulen;
      max_clen = max_clen > clen ? max_clen : clen;
    }
    cnt++;
    total += ulen;
    ip += clen;
  }
  if (!FILL) {
    if (bad) {
      status[i] = B2S_E_CORRUPT;
      cnt = 0;
      total = 0;
    }
    nblk[i] = cnt;
    olen_total[i] = total;
    if (cnt) {
      atomicMax(maxima, (unsigned long long)max_olen);
      atomicMax(maxima + 1, (unsigned long long)max_clen);
    }
  } else if (too_small) {
    status[i] = B2S_E_DST_TOO_SMALL;
  }
}

void launch_xerial_count(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                         uint64_t* d_nblk, uint64_t* d_olen, uint64_t* d_maxima, int32_t* d_status, cudaStream_t st,
                         uint64_t* launches) {
  if (!n) return;
  xerial_walk_kernel<false><<<(n + 127) / 128, 128, 0, st>>>(src_base, d_src_off, d_src_len, n, d_nblk, d_olen,
                                                            (unsigned long long*)d_maxima, nullptr, nullptr, 0,
                                                            d_status, nullptr);
  *launches += 1;
}
void launch_xerial_fill(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                        const uint64_t* d_blk_base, const uint64_t* d_dst_off, uint64_t* d_olen, uint64_t dst_cap,
                        int32_t* d_status, BlockDesc* d_desc, cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  xerial_walk_kernel<true><<<(n + 127) / 128, 128, 0, st>>>(src_base, d_src_off, d_src_len, n, nullptr, d_olen, nullptr,
                                                           d_blk_base, d_dst_off, dst_cap, d_status, d_desc);
  *launches += 1;
}

// ------------------------------------------------------------------------------------------------------------
// read side: elements -> records (thread per chunk).  A literal element followed by a copy element becomes one
// record for the copy kernel (snappy_copy_kernel).
// record: x = literal count | match length << 16 ; y = offset | literal source position << 16
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64) snappy_tokens_kernel(const BlockDesc* __restrict__ desc, uint32_t b0, uint32_t m,
                                                           const uint8_t* __restrict__ src_base,
                                                           uint2* __restrict__ rec, uint32_t rec_stride,
                                                           uint32_t* __restrict__ nrec, int32_t* __restrict__ status) {
  const uint32_t bl = blockIdx.x * blockDim.x + threadIdx.x;
  if (bl >= m) return;
  const uint32_t b = b0 + bl;
  const BlockDesc d = desc[b];
  if (d.olen == 0 && d.clen == 0) {  // no-op descriptor (or an empty chunk)
    nrec[b] = 0;
    return;
  }
  const uint8_t* __restrict__ in = src_base + d.src;
  const int clen = (int)d.clen, olen = (int)d.olen;
  uint2* __restrict__ r = rec + (size_t)bl * rec_stride;
  int ip = 0, op = 0;
  uint32_t ns = 0;
  bool err = false;
  int plit = 0, plip = 0;  // pending literal element waiting for a copy to pair with
  while (ip < clen) {
    if ((ip & 31) < 3 && ip + 256 < clen) asm volatile("prefetch.global.L1 [%0];" ::"l"(in + ip + 256));
    const int tag = __ldg(in + ip++);
    const int kind = tag & 3;
    if (kind == 0) {
      int len = (tag >> 2) + 1;
      if (len > 60) {
        const int nbytes = len - 60;
        if (ip + nbytes > clen) {
          err = true;
          break;
        }
        len = 0;
        for (int k = 0; k < nbytes; k++) len |= (int)__ldg(in + ip + k) << (8 * k);
        if (len < 0 || len >= (1 << 24)) {  // cannot fit a chunk that passed the size limits
          err = true;
          break;
        }
        len += 1;
        ip += nbytes;
      }
      if (len > clen - ip || len > olen - op) {
        err = true;
        break;
      }
      if (plit) r[ns++] = make_uint2((uint32_t)plit, (uint32_t)plip << 16);  // two literals in a row
      plit = len;
      plip = ip;
      ip += len;
      op += len;
      continue;
    }
    int len, off;
    if (kind == 1) {
      if (ip + 1 > clen) {
        err = true;
        break;
      }
      len = 4 + ((tag >> 2) & 7);
      off = ((tag >> 5) << 8) | __ldg(in + ip);
      ip += 1;
    } else if (kind == 2) {
      if (ip + 2 > clen) {
        err = true;
        break;
      }
      len = (tag >> 2) + 1;
      off = __ldg(in + ip) | (__ldg(in + ip + 1) << 8);
      ip += 2;
    } else {
      if (ip + 4 > clen) {
        err = true;
        break;
      }
      len = (tag >> 2) + 1;
      const uint32_t o32 = (uint32_t)__ldg(in + ip) | ((uint32_t)__ldg(in + ip + 1) << 8) |
                           ((uint32_t)__ldg(in + ip + 2) << 16) | ((uint32_t)__ldg(in + ip + 3) << 24);
      ip += 4;
      if (o32 > 65535u) {  // farther back than a <= 64 KiB chunk can reach
        err = true;
        break;
      }
      off = (int)o32;
    }
    if (off == 0 || off > op || len > olen - op) {
      err = true;
      break;
    }
    r[ns++] = make_uint2((uint32_t)plit | ((uint32_t)len << 16), (uint32_t)off | ((uint32_t)plip << 16));
    plit = 0;
    op += len;
  }
  if (!err && plit) r[ns++] = make_uint2((uint32_t)plit, (uint32_t)plip << 16);
  if (!err && op != olen) err = true;
  if (err) {
    set_status(status, d.stream & 0x7fffffffu, B2S_E_CORRUPT);
    ns = 0;
  }
  nrec[b] = ns;
}

void launch_snappy_tokens(const BlockDesc* d_desc, uint32_t b0, uint32_t m, const uint8_t* src_base, uint2* d_rec,
                          uint32_t rec_stride, uint32_t* d_nrec, int32_t* d_status, cudaStream_t st,
                          uint64_t* launches) {
  if (!m) return;
  snappy_tokens_kernel<<<(m + 63) / 64, 64, 0, st>>>(d_desc, b0, m, src_base, d_rec, rec_stride, d_nrec, d_status);
  *launches += 1;
}

// ------------------------------------------------------------------------------------------------------------
// read side: records -> bytes.  Warp per codec block, LANE per sequence: output positions by a warp scan, all literals
// of a batch of 32 sequences at once, then the matches in dependency rounds (lz_batch.cuh).
// ------------------------------------------------------------------------------------------------------------
constexpr int kCopyThreads = 256;
__global__ void __launch_bounds__(kCopyThreads) snappy_copy_kernel(const BlockDesc* __restrict__ desc, uint32_t b0,
                                                                   uint32_t m, const uint8_t* __restrict__ src_base,
                                                                   uint8_t* dst_base, const uint2* __restrict__ rec,
                                                                   uint32_t rec_stride,
                                                                   const uint32_t* __restrict__ nrec) {
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const uint32_t bl = blockIdx.x * (kCopyThreads / 32) + (threadIdx.x >> 5);
  if (bl >= m) return;
  const uint32_t b = b0 + bl;
  const BlockDesc d = desc[b];
  if (d.olen == 0) return;
  const uint8_t* __restrict__ in = src_base + d.src;
  uint8_t* out = dst_base + d.dst;
  if (d.stream & 0x80000000u) {
    group_copy<32>(out, in, d.olen, lane);
    return;
  }
  const uint32_t n = nrec[b];
  const uint2* __restrict__ r = rec + (size_t)bl * rec_stride;
  int base_op = 0;
  for (uint32_t i0 = 0; i0 < n; i0 += 32) {
    const uint32_t i = i0 + lane;
    uint2 q = make_uint2(0, 0);
    if (i < n) q = r[i];
    const int lit = (int)(q.x & 0xffffu), ml = (int)(q.x >> 16);
    const int off = (int)(q.y & 0xffffu), lip = (int)(q.y >> 16);
    // output position of every sequence of the batch: exclusive scan of lit + ml
    int inc = lit + ml;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int t = __shfl_up_sync(FULL, inc, s);
      if (lane >= s) inc += t;
    }
    const int op = base_op + inc - (lit + ml);
    base_op += __shfl_sync(FULL, inc, 31);

    // ---- literals: independent of everything, all lanes at once; long runs go through the whole warp
    lz_copy_literals(in, out, lip, lit, op, lane);

    // ---- matches, in dependency rounds (lz_batch.cuh)
    lz_execute_matches<true>(out, op + lit, ml, off, lane);
  }
}

// records per codec block: a Snappy element takes >= 2 compressed bytes and may produce a single byte
uint32_t snappy_decode_rec_stride(uint32_t max_clen) { return max_clen / 2 + 2; }
size_t snappy_decode_ws_bytes(uint32_t chunk_blocks, uint32_t rec_stride) {
  return (size_t)chunk_blocks * rec_stride * 8 + 256;
}

void launch_snappy_copy(const BlockDesc* d_desc, uint32_t b0, uint32_t m, uint32_t rec_stride, const uint8_t* src_base,
                        uint8_t* dst_base, const uint8_t* d_ws, const uint32_t* d_nrec, cudaStream_t st,
                        uint64_t* launches) {
  if (!m) return;
  snappy_copy_kernel<<<(m + kCopyThreads / 32 - 1) / (kCopyThreads / 32), kCopyThreads, 0, st>>>(
      d_desc, b0, m, src_base, dst_base, reinterpret_cast<const uint2*>(d_ws), rec_stride, d_nrec);
  *launches += 1;
}

}  // namespace b2s
