// zstd_core.h — Zstandard (RFC 8878) frame decoding, written once for host and device.
//
// Replaces, for spark.io.compression.codec=zstd, com.github.luben.zstd.ZstdInputStreamNoFinalizer [U] (zstd-jni 1.5.5-x ->
// libzstd ZSTD_decompressStream) under serializerManager.wrapStream at storage/S3ShuffleReader.scala:107-109.
// The same functions are compiled by nvcc into the kernels of zstd.cu (the product) and by the host compiler into the
// unit tests tests/test_zstd_core.py and tests/test_zstd_levels.py, which check them against libzstd.so.1 on frames
// produced by libzstd itself (levels -5 to 22 — every strategy — in streaming mode without content size as zstd-jni
// writes them, with content checksum, with 2 workers, with long distance matching and a 2^27 window; raw/RLE/compressed
// blocks, raw literals inside compressed blocks, Huffman 1- and 4-stream literals, treeless literals,
// predefined/RLE/FSE/repeat sequence tables, all six repeat-offset forms, concatenated and skippable frames).
// tests/test_gpu_zstd_levels.py sends the same frames through the kernels.  Nothing here is a CPU fallback: the C ABI
// only ever launches the device build.
//
// Scope: frames without dictionary; window <= the decoded size the caller provides room for; Content_Checksum is
// skipped, not verified (Spark's ZStdCompressionCodec leaves it off).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2S_HD __host__ __device__
#else
#define B2S_HD
#endif
#if defined(B2S_ZSTD_WARP) && defined(__CUDACC__)
#include "lz_batch.cuh"  // lz_execute_matches: the dependency-round executor shared with the LZ4 / Snappy copy kernel
#endif

// Cooperative execution.  On the device the decoder runs with ALL 32 lanes of a warp executing the same control flow on
// the same data (the serial parts are simply computed redundantly, which costs a warp no more than one lane would),
// so that the byte-copy loops can be split across the lanes and the four Huffman streams of a literals section across
// four lanes (zstd_par.h, the block-parallel decomposition the kernels run).  zstd.cu defines B2S_ZSTD_WARP before
// including this header; everywhere else one "lane" does everything.  decode_stream() below is the single-pass
// statement of the format, kept as the reference the decomposition is tested against on the host.
#if defined(B2S_ZSTD_WARP) && defined(__CUDA_ARCH__)
#define B2S_LANE ((int)(threadIdx.x & 31))
#define B2S_NLANES 32
#define B2S_SYNC() __syncwarp()
#define B2S_ALL(pred) (__all_sync(0xffffffffu, (pred)))
#else
#define B2S_LANE 0
#define B2S_NLANES 1
#define B2S_SYNC() ((void)0)
#define B2S_ALL(pred) (pred)
#endif

namespace b2s {
namespace zstd {

constexpr int kErrCorrupt = -1;      // -> B2S_E_CORRUPT
constexpr int kErrDstTooSmall = -3;  // -> B2S_E_DST_TOO_SMALL
constexpr int kErrUnsupported = -4;  // -> B2S_E_UNSUPPORTED (dictionary)
constexpr uint32_t kBlockMax = 128 * 1024;

struct FseEntry {
  uint8_t sym, nbits;
  uint16_t base;
};
static_assert(sizeof(FseEntry) == 4, "zstd_par.h reads an entry as one little-endian 32-bit word");

// per-stream decoder state: ~11 KB of tables (shared memory on the device) + a pointer to the literals buffer
struct Workspace {
#ifdef B2S_ZSTD_UNION_TABLES
  // Block-parallel decoding (zstd_par.h) rebuilds every table per block and is done with the literals before it
  // starts on the sequences, so the Huffman tables and the three sequence tables can share their bytes: 6.6 KB instead
  // of 11 KB per warp, i.e. 32 instead of 20 resident warps per SM.  (decode_stream keeps tables across blocks and
  // must not be built this way.)
  union {
    struct {
      FseEntry ll[512], of[256], ml[512];
    };
    struct {
      uint16_t huf[2048];  // Huffman decoding table: symbol | nbits << 8, 2^maxbits entries (maxbits <= 11)
      FseEntry wt[64];     // Huffman weights (FSE, accuracy <= 6)
      uint8_t weights[256];
    };
  };
#else
  FseEntry ll[512], of[256], ml[512];
  FseEntry wt[64];        // Huffman weights (FSE, accuracy <= 6)
  uint16_t huf[2048];     // Huffman decoding table: symbol | nbits << 8, 2^maxbits entries (maxbits <= 11)
  uint8_t weights[256];
#endif
  uint8_t* lit;           // kBlockMax + 64 bytes (global memory on the device; the tables above sit in shared memory)
  int16_t norm[64];
  uint16_t next[64];
  int ll_log, of_log, ml_log, huf_bits;
  bool ll_ok, of_ok, ml_ok, huf_ok;
  uint32_t rep[3];
};

B2S_HD inline int highbit32(uint32_t v) {  // position of the highest set bit, v != 0
#if defined(__CUDA_ARCH__)
  return 31 - __clz((int)v);
#endif
  int r = 0;
  while (v >>= 1) r++;
  return r;
}

// ---- LSB-first forward bit reader (FSE table descriptions) --------------------------------------------------
struct BitsFwd {
  const uint8_t* p;
  uint64_t n;
  uint64_t pos;  // bit position
  B2S_HD uint32_t peek(int nb) const {
    uint64_t v = 0;
    const uint64_t b = pos >> 3;
    for (int i = 0; i < 5; i++)
      if (b + i < n) v |= (uint64_t)p[b + i] << (8 * i);
    return (uint32_t)((v >> (pos & 7)) & ((1ull << nb) - 1));
  }
};

// ---- backward bit reader (Huffman streams, sequence bitstream): starts below the final 1-bit marker ----------
// Keeps up to 64 upcoming bits in a register (`buf` holds stream bits [lo, lo+64), refilled with one 8-byte gather
// when the cursor leaves it) so a read is a shift and a mask, not a fresh walk over memory.
struct BitsRev {
  const uint8_t* p;
  int32_t n;    // bytes (a literals stream or a sequence bitstream is at most one block: < 2^17 bytes, 2^20 bits)
  int32_t pos;  // bits still unread; may go negative (over-read: zeros), checked by the callers
  uint64_t buf;
  int32_t lo;   // bit index of buf's bit 0 (multiple of 8; may be negative: bits below the stream start are zero)
  B2S_HD void fill(int32_t want_lo) {  // buf := stream bits [want_lo, want_lo + 64)
    lo = want_lo;
    uint64_t v = 0;
    const int32_t b = want_lo >> 3;  // arithmetic shift: negative byte indices read as zero
    if (b >= 0 && b + 16 <= n) {     // away from both ends: two aligned 8-byte loads instead of eight byte loads
#ifdef __CUDA_ARCH__
      const uintptr_t a = reinterpret_cast<uintptr_t>(p + b);
      const uint64_t* wp = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
      const unsigned sh = (unsigned)(a & 7u) * 8u;
      const uint64_t x0 = wp[0], x1 = wp[1];  // wp[1] ends at most 15 bytes after p + b: inside the stream
      buf = sh ? (x0 >> sh) | (x1 << (64u - sh)) : x0;
#else
      for (int i = 0; i < 8; i++) v |= (uint64_t)p[b + i] << (8 * i);
      buf = v;
#endif
      return;
    }
    for (int i = 0; i < 8; i++) {
      const int32_t k = b + i;
      if (k >= 0 && k < n) v |= (uint64_t)p[k] << (8 * i);
    }
    buf = v;
  }
  B2S_HD bool init(const uint8_t* src, uint64_t len) {
    p = src;
    if (len == 0 || len > (1u << 24) || src[len - 1] == 0) return false;
    n = (int32_t)len;
    pos = (int32_t)(len - 1) * 8 + highbit32(src[len - 1]);
    fill(((pos - 57) >> 3) * 8);  // pos lies within the top byte of the buffer
    return true;
  }
  B2S_HD uint32_t read(int nb) {  // nb <= 32
    if (nb == 0) return 0;
    pos -= nb;
    if (pos < lo) fill(((pos - 24) >> 3) * 8);  // keep >= 32 bits above pos available: pos - lo in [24, 31]
    return (uint32_t)(buf >> (pos - lo)) & (0xffffffffu >> (32 - nb));
  }
};

// ---- FSE -------------------------------------------------------------------------------------------------------
// normalized counts -> decoding table (RFC 8878 4.1.1)
B2S_HD inline bool fse_build(FseEntry* t, const int16_t* norm, int nsym, int log, uint16_t* next) {
  const int size = 1 << log;
  int high = size - 1;
  for (int s = 0; s < nsym; s++) {
    if (norm[s] == -1) {
      t[high--].sym = (uint8_t)s;
      next[s] = 1;
    } else {
      next[s] = (uint16_t)norm[s];
    }
  }
  const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  int pos = 0;
  for (int s = 0; s < nsym; s++) {
    for (int i = 0; i < norm[s]; i++) {
      t[pos].sym = (uint8_t)s;
      do pos = (pos + step) & mask;
      while (pos > high);
    }
  }
  if (pos != 0) return false;
  for (int i = 0; i < size; i++) {
    const int s = t[i].sym;
    const uint32_t x = next[s]++;
    const int nb = log - highbit32(x);
    t[i].nbits = (uint8_t)nb;
    t[i].base = (uint16_t)((x << nb) - size);
  }
  return true;
}

// reads a table description; returns bytes consumed (0 = malformed)
B2S_HD inline uint64_t fse_read_header(const uint8_t* src, uint64_t n, int16_t* norm, int max_sym, int max_log, int* log_out,
                                       int* nsym_out) {
  BitsFwd b{src, n, 0};
  if (n == 0) return 0;
  const int log = (int)b.peek(4) + 5;
  b.pos += 4;
  if (log > max_log) return 0;
  int remaining = 1 << log;
  int sym = 0;
  while (remaining > 0 && sym <= max_sym) {
    const int bits = highbit32((uint32_t)(remaining + 1)) + 1;
    uint32_t val = b.peek(bits);
    const uint32_t lower = (1u << (bits - 1)) - 1;
    const uint32_t threshold = (1u << bits) - 1 - (uint32_t)(remaining + 1);
    if ((val & lower) < threshold) {
      b.pos += bits - 1;
      val &= lower;
    } else if (val > lower) {
      b.pos += bits;
      val -= threshold;
    } else {
      b.pos += bits;
    }
    const int prob = (int)val - 1;
    remaining -= prob < 0 ? -prob : prob;
    norm[sym++] = (int16_t)prob;
    if (prob == 0) {
      uint32_t rep = b.peek(2);
      b.pos += 2;
      for (;;) {
        for (uint32_t i = 0; i < rep && sym <= max_sym; i++) norm[sym++] = 0;
        if (rep != 3) break;
        rep = b.peek(2);
        b.pos += 2;
      }
    }
    if ((b.pos >> 3) > n) return 0;
  }
  if (remaining != 0 || sym > max_sym + 1) return 0;
  *log_out = log;
  *nsym_out = sym;
  const uint64_t used = (b.pos + 7) >> 3;
  return used <= n ? used : 0;
}

// ---- Huffman ---------------------------------------------------------------------------------------------------
// weights[0..nw) given (the last one is implied) -> decoding table; returns false when malformed
B2S_HD inline bool huf_build(Workspace* w, int nw) {
  uint32_t sum = 0;
  for (int i = 0; i < nw; i++) {
    if (w->weights[i] > 11) return false;
    if (w->weights[i]) sum += 1u << (w->weights[i] - 1);
  }
  if (sum == 0) return false;
  const int maxbits = highbit32(sum) + 1;
  if (maxbits > 11) return false;
  const uint32_t left = (1u << maxbits) - sum;
  if (left & (left - 1)) return false;  // the implied weight must complete a power of two
  w->weights[nw] = (uint8_t)(highbit32(left) + 1);
  const int nsym = nw + 1;
  // number of codes per length, first table index per length (longest codes first)
  uint32_t rank_count[13] = {0}, rank_idx[13];
  for (int i = 0; i < nsym; i++) {
    const int wt = w->weights[i];
    rank_count[wt ? maxbits + 1 - wt : 0]++;
  }
  rank_idx[maxbits] = 0;
  for (int i = maxbits; i >= 1; i--) rank_idx[i - 1] = rank_idx[i] + rank_count[i] * (1u << (maxbits - i));
  if (rank_idx[0] != (1u << maxbits)) return false;
  for (int i = 0; i < nsym; i++) {
    const int wt = w->weights[i];
    if (!wt) continue;
    const int bits = maxbits + 1 - wt;
    const uint32_t code = rank_idx[bits], len = 1u << (maxbits - bits);
    for (uint32_t k = 0; k < len; k++) w->huf[code + k] = (uint16_t)(i | (bits << 8));
    rank_idx[bits] += len;
  }
  w->huf_bits = maxbits;
  return true;
}

// Huffman tree description; returns bytes consumed (0 = malformed)
B2S_HD inline uint64_t huf_read_tree(Workspace* w, const uint8_t* src, uint64_t n) {
  if (n == 0) return 0;
  const int hb = src[0];
  int nw = 0;
  uint64_t used;
  if (hb >= 128) {  // direct: 4 bits per weight
    nw = hb - 127;
    const uint64_t bytes = (uint64_t)(nw + 1) / 2;
    if (1 + bytes > n) return 0;
    for (int i = 0; i < nw; i++) {
      const uint8_t v = src[1 + i / 2];
      w->weights[i] = (i & 1) ? (v & 15) : (v >> 4);
    }
    used = 1 + bytes;
  } else {  // FSE-compressed weights, two interleaved states
    const uint64_t clen = (uint64_t)hb;
    if (clen == 0 || 1 + clen > n) return 0;
    int log = 0, nsym = 0;
    const uint64_t h = fse_read_header(src + 1, clen, w->norm, 12, 6, &log, &nsym);  // weights 0..12 (only <= 11 are legal)
    if (!h || h >= clen) return 0;
    for (int i = nsym; i < 13; i++) w->norm[i] = 0;
    if (!fse_build(w->wt, w->norm, nsym, log, w->next)) return 0;
    BitsRev br;
    if (!br.init(src + 1 + h, clen - h)) return 0;
    uint32_t s1 = br.read(log), s2 = br.read(log);
    for (;;) {
      if (nw >= 254) return 0;
      w->weights[nw++] = w->wt[s1].sym;
      if (br.pos < w->wt[s1].nbits) {  // not enough bits for another update: flush the other state and stop
        if (br.pos < 0) return 0;
        w->weights[nw++] = w->wt[s2].sym;
        break;
      }
      s1 = w->wt[s1].base + br.read(w->wt[s1].nbits);
      if (nw >= 254) return 0;
      w->weights[nw++] = w->wt[s2].sym;
      if (br.pos < w->wt[s2].nbits) {
        if (br.pos < 0) return 0;
        w->weights[nw++] = w->wt[s1].sym;
        break;
      }
      s2 = w->wt[s2].base + br.read(w->wt[s2].nbits);
    }
    used = 1 + clen;
  }
  if (nw < 1 || nw > 255) return 0;
  if (!huf_build(w, nw)) return 0;
  return used;
}

B2S_HD inline bool huf_decode_stream(const Workspace* w, const uint8_t* src, uint64_t n, uint8_t* out, uint64_t count) {
  BitsRev br;
  if (!br.init(src, n)) return false;
  const int mb = w->huf_bits;
  const uint32_t mask = (1u << mb) - 1;
  uint32_t state = br.read(mb);
  for (uint64_t i = 0; i < count; i++) {
    const uint16_t e = w->huf[state];
    out[i] = (uint8_t)e;
    const int nb = e >> 8;
    state = ((state << nb) & mask) | br.read(nb);
  }
  // every stream must be consumed exactly: the over-read equals the initial state's width
  return br.pos == -mb;
}

// ---- sequences ---------------------------------------------------------------------------------------------------
// Code -> (baseline, extra bits), RFC 8878 tables 3.1.1.3.2.1.1, in closed form: a function-local lookup table would be
// rebuilt on the (local-memory) stack for every sequence on the device.
B2S_HD inline void ll_code(int c, uint32_t* base, int* bits) {
  if (c < 16) { *base = (uint32_t)c; *bits = 0; }
  else if (c < 20) { *base = 16u + 2u * (uint32_t)(c - 16); *bits = 1; }
  else if (c < 22) { *base = 24u + 4u * (uint32_t)(c - 20); *bits = 2; }
  else if (c < 24) { *base = 32u + 8u * (uint32_t)(c - 22); *bits = 3; }
  else if (c == 24) { *base = 48u; *bits = 4; }
  else if (c == 25) { *base = 64u; *bits = 6; }
  else { *base = 1u << (c - 19); *bits = c - 19; }
}
B2S_HD inline void ml_code(int c, uint32_t* base, int* bits) {
  if (c < 32) { *base = (uint32_t)c + 3u; *bits = 0; }
  else if (c < 36) { *base = 35u + 2u * (uint32_t)(c - 32); *bits = 1; }
  else if (c < 38) { *base = 43u + 4u * (uint32_t)(c - 36); *bits = 2; }
  else if (c < 40) { *base = 51u + 8u * (uint32_t)(c - 38); *bits = 3; }
  else if (c < 42) { *base = 67u + 16u * (uint32_t)(c - 40); *bits = 4; }
  else if (c == 42) { *base = 99u; *bits = 5; }
  else if (c == 43) { *base = 131u; *bits = 7; }
  else { *base = (1u << (c - 36)) + 3u; *bits = c - 36; }
}

// kind: 0 = literal lengths, 1 = offsets, 2 = match lengths
B2S_HD inline bool seq_default_table(Workspace* w, int kind) {
  const int16_t LL[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
  const int16_t OF[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
  const int16_t ML[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                          1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
  if (kind == 0) {
    for (int i = 0; i < 36; i++) w->norm[i] = LL[i];
    w->ll_log = 6;
    return fse_build(w->ll, w->norm, 36, 6, w->next);
  }
  if (kind == 1) {
    for (int i = 0; i < 29; i++) w->norm[i] = OF[i];
    w->of_log = 5;
    return fse_build(w->of, w->norm, 29, 5, w->next);
  }
  for (int i = 0; i < 53; i++) w->norm[i] = ML[i];
  w->ml_log = 6;
  return fse_build(w->ml, w->norm, 53, 6, w->next);
}

// sets up one of the three sequence tables per its compression mode; returns bytes consumed or -1
B2S_HD inline int64_t seq_setup_table(Workspace* w, int kind, int mode, const uint8_t* src, uint64_t n) {
  FseEntry* t = kind == 0 ? w->ll : kind == 1 ? w->of : w->ml;
  int* log = kind == 0 ? &w->ll_log : kind == 1 ? &w->of_log : &w->ml_log;
  bool* ok = kind == 0 ? &w->ll_ok : kind == 1 ? &w->of_ok : &w->ml_ok;
  const int max_sym = kind == 0 ? 35 : kind == 1 ? 31 : 52;
  const int max_log = kind == 0 ? 9 : kind == 1 ? 8 : 9;
  if (mode == 0) {
    if (!seq_default_table(w, kind)) return -1;
    *ok = true;
    return 0;
  }
  if (mode == 1) {  // RLE: a single symbol, zero state bits
    if (n < 1 || src[0] > max_sym) return -1;
    t[0].sym = src[0];
    t[0].nbits = 0;
    t[0].base = 0;
    *log = 0;
    *ok = true;
    return 1;
  }
  if (mode == 2) {
    int l = 0, nsym = 0;
    const uint64_t h = fse_read_header(src, n, w->norm, max_sym, max_log, &l, &nsym);
    if (!h) return -1;
    if (!fse_build(t, w->norm, nsym, l, w->next)) return -1;
    *log = l;
    *ok = true;
    return (int64_t)h;
  }
  return *ok ? 0 : -1;  // repeat: the previous block's table must exist
}

// ---- blocks --------------------------------------------------------------------------------------------------------
// Decodes one compressed block of `n` bytes.  out = start of the frame's output, op = bytes of the frame produced so
// far (matches may reach back to out[0]); cap = room in out.  size_only: only count the regenerated size.
// Returns the number of bytes the block regenerates, or a negative error.
B2S_HD inline int64_t decode_compressed_block(Workspace* w, const uint8_t* src, uint64_t n, uint8_t* out, uint64_t op,
                                              uint64_t cap, bool size_only) {
  if (n < 1) return kErrCorrupt;
  // ---- literals section
  const int ltype = src[0] & 3, sf = (src[0] >> 2) & 3;
  uint64_t hdr, regen, csize = 0;
  int streams = 1;
  if (ltype < 2) {
    if (sf == 0 || sf == 2) {
      hdr = 1;
      regen = src[0] >> 3;
    } else if (sf == 1) {
      if (n < 2) return kErrCorrupt;
      hdr = 2;
      regen = (src[0] >> 4) | ((uint64_t)src[1] << 4);
    } else {
      if (n < 3) return kErrCorrupt;
      hdr = 3;
      regen = (src[0] >> 4) | ((uint64_t)src[1] << 4) | ((uint64_t)src[2] << 12);
    }
  } else {
    if (sf < 2) {
      if (n < 3) return kErrCorrupt;
      hdr = 3;
      const uint32_t v = src[0] | (src[1] << 8) | ((uint32_t)src[2] << 16);
      regen = (v >> 4) & 0x3ff;
      csize = (v >> 14) & 0x3ff;
      streams = sf == 0 ? 1 : 4;
    } else if (sf == 2) {
      if (n < 4) return kErrCorrupt;
      hdr = 4;
      const uint32_t v = src[0] | (src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24);
      regen = (v >> 4) & 0x3fff;
      csize = v >> 18;
      streams = 4;
    } else {
      if (n < 5) return kErrCorrupt;
      hdr = 5;
      const uint64_t v = src[0] | (src[1] << 8) | ((uint64_t)src[2] << 16) | ((uint64_t)src[3] << 24) | ((uint64_t)src[4] << 32);
      regen = (v >> 4) & 0x3ffff;
      csize = v >> 22;
      streams = 4;
    }
  }
  if (regen > kBlockMax) return kErrCorrupt;
  const uint8_t* lit = nullptr;  // literal bytes of this block (either inside src or in w->lit)
  uint64_t ip = hdr;
  if (ltype == 0) {
    if (ip + regen > n) return kErrCorrupt;
    lit = src + ip;
    ip += regen;
  } else if (ltype == 1) {
    if (ip + 1 > n) return kErrCorrupt;
    if (!size_only)
    {
      for (uint64_t i = B2S_LANE; i < regen; i += B2S_NLANES) w->lit[i] = src[ip];
      B2S_SYNC();
    }
    lit = w->lit;
    ip += 1;
  } else {
    if (ip + csize > n) return kErrCorrupt;
    const uint8_t* ls = src + ip;
    uint64_t ln = csize;
    if (ltype == 2) {
      const uint64_t t = huf_read_tree(w, ls, ln);
      if (!t) return kErrCorrupt;
      w->huf_ok = true;
      ls += t;
      ln -= t;
    } else if (!w->huf_ok) {
      return kErrCorrupt;  // treeless without a previous table
    }
    if (!size_only) {
      if (streams == 1) {
        bool ok1 = true;
        if (B2S_LANE == 0) ok1 = huf_decode_stream(w, ls, ln, w->lit, regen);
        B2S_SYNC();
        if (!B2S_ALL(ok1)) return kErrCorrupt;
      } else {
        if (ln < 6) return kErrCorrupt;
        const uint64_t s1 = ls[0] | (ls[1] << 8), s2 = ls[2] | (ls[3] << 8), s3 = ls[4] | (ls[5] << 8);
        if (6 + s1 + s2 + s3 > ln) return kErrCorrupt;
        const uint64_t s4 = ln - 6 - s1 - s2 - s3;
        const uint64_t q = (regen + 3) / 4;
        if (3 * q > regen) return kErrCorrupt;
        const uint8_t* a = ls + 6;
        if (!huf_decode_stream(w, a, s1, w->lit, q)) return kErrCorrupt;
        if (!huf_decode_stream(w, a + s1, s2, w->lit + q, q)) return kErrCorrupt;
        if (!huf_decode_stream(w, a + s1 + s2, s3, w->lit + 2 * q, q)) return kErrCorrupt;
        if (!huf_decode_stream(w, a + s1 + s2 + s3, s4, w->lit + 3 * q, regen - 3 * q)) return kErrCorrupt;
      }
    }
    lit = w->lit;
    ip += csize;
  }
  // ---- sequences section
  if (ip >= n) return kErrCorrupt;
  uint32_t nseq = src[ip++];
  if (nseq >= 128) {
    if (nseq == 255) {
      if (ip + 2 > n) return kErrCorrupt;
      nseq = src[ip] + (src[ip + 1] << 8) + 0x7F00;
      ip += 2;
    } else {
      if (ip + 1 > n) return kErrCorrupt;
      nseq = ((nseq - 128) << 8) + src[ip];
      ip += 1;
    }
  }
  uint64_t produced = 0;
  uint64_t lpos = 0;
  if (nseq) {
    if (ip >= n) return kErrCorrupt;
    const int modes = src[ip++];
    if (modes & 3) return kErrCorrupt;
    for (int kind = 0; kind < 3; kind++) {
      const int mode = (modes >> (6 - 2 * kind)) & 3;
      const int64_t used = seq_setup_table(w, kind, mode, src + ip, n - ip);
      if (used < 0) return kErrCorrupt;
      ip += (uint64_t)used;
    }
    BitsRev br;
    if (ip >= n || !br.init(src + ip, n - ip)) return kErrCorrupt;
    uint32_t sl = br.read(w->ll_log), so = br.read(w->of_log), sm = br.read(w->ml_log);
    for (uint32_t i = 0; i < nseq; i++) {
      const int oc = w->of[so].sym, mc = w->ml[sm].sym, lc = w->ll[sl].sym;
      if (oc > 31 || mc > 52 || lc > 35) return kErrCorrupt;
      uint32_t mlb, llb;
      int mle, lle;
      ml_code(mc, &mlb, &mle);
      ll_code(lc, &llb, &lle);
      // extra bits: offset, match length, literal length — in that order
      const uint32_t ofv = (oc ? (1u << oc) : 1u) + br.read(oc);
      const uint32_t mlen = mlb + br.read(mle);
      const uint32_t llen = llb + br.read(lle);
      // offset: values 1..3 are repeat codes
      uint32_t offset;
      if (ofv > 3) {
        offset = ofv - 3;
        w->rep[2] = w->rep[1];
        w->rep[1] = w->rep[0];
        w->rep[0] = offset;
      } else {
        uint32_t idx = ofv - 1;
        if (llen == 0) idx++;
        if (idx == 0) {
          offset = w->rep[0];
        } else {
          offset = idx < 3 ? w->rep[idx] : w->rep[0] - 1;
          if (idx > 1) w->rep[2] = w->rep[1];
          w->rep[1] = w->rep[0];
          w->rep[0] = offset;
        }
      }
      if (offset == 0) return kErrCorrupt;
      if (lpos + llen > regen) return kErrCorrupt;
      if (produced + llen + mlen > kBlockMax) return kErrCorrupt;
      if (!size_only) {
        const uint64_t o = op + produced;
        if (o + llen + mlen > cap) return kErrDstTooSmall;
        if ((uint64_t)offset > o + llen) return kErrCorrupt;  // reaches before the start of the frame
        for (uint32_t k = 0; k < llen; k++) out[o + k] = lit[lpos + k];
        uint8_t* d = out + o + llen;
        const uint8_t* s = d - offset;
        for (uint32_t k = 0; k < mlen; k++) d[k] = s[k];
      }
      lpos += llen;
      produced += (uint64_t)llen + mlen;
      if (i + 1 < nseq) {  // state updates: literal length, match length, offset
        sl = w->ll[sl].base + br.read(w->ll[sl].nbits);
        sm = w->ml[sm].base + br.read(w->ml[sm].nbits);
        so = w->of[so].base + br.read(w->of[so].nbits);
      }
    }
    if (br.pos != 0) return kErrCorrupt;  // the bitstream must be consumed exactly
  }
  // remaining literals
  const uint64_t tail = regen - lpos;
  if (produced + tail > kBlockMax) return kErrCorrupt;
  if (!size_only) {
    const uint64_t o = op + produced;
    if (o + tail > cap) return kErrDstTooSmall;
    for (uint64_t k = B2S_LANE; k < tail; k += B2S_NLANES) out[o + k] = lit[lpos + k];
    B2S_SYNC();
  }
  return (int64_t)(produced + tail);
}

// Decodes every frame in src[0..n) (concatenated frames, skippable frames) into dst; returns the decoded size or a
// negative error.  size_only: dst/cap are ignored.
B2S_HD inline int64_t decode_stream(Workspace* w, const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t cap, bool size_only) {
  uint64_t ip = 0, total = 0;
  while (ip < n) {
    if (n - ip < 4) return kErrCorrupt;
    const uint32_t magic = src[ip] | (src[ip + 1] << 8) | ((uint32_t)src[ip + 2] << 16) | ((uint32_t)src[ip + 3] << 24);
    ip += 4;
    if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {  // skippable frame
      if (n - ip < 4) return kErrCorrupt;
      const uint64_t sz = src[ip] | (src[ip + 1] << 8) | ((uint64_t)src[ip + 2] << 16) | ((uint64_t)src[ip + 3] << 24);
      ip += 4;
      if (sz > n - ip) return kErrCorrupt;
      ip += sz;
      continue;
    }
    if (magic != 0xFD2FB528u) return kErrCorrupt;
    if (ip >= n) return kErrCorrupt;
    const int fhd = src[ip++];
    const int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, did_flag = fhd & 3;
    if (fhd & 0x08) return kErrCorrupt;  // reserved bit
    if (!single) {
      if (ip >= n) return kErrCorrupt;
      ip++;  // window descriptor: the whole frame output is addressable here, so the size itself is not needed
    }
    const int did_bytes = did_flag == 0 ? 0 : did_flag == 1 ? 1 : did_flag == 2 ? 2 : 4;
    if (ip + did_bytes > n) return kErrCorrupt;
    uint32_t did = 0;
    for (int i = 0; i < did_bytes; i++) did |= (uint32_t)src[ip + i] << (8 * i);
    ip += did_bytes;
    if (did != 0) return kErrUnsupported;
    const int fcs_bytes = fcs_flag == 0 ? (single ? 1 : 0) : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
    if (ip + fcs_bytes > n) return kErrCorrupt;
    uint64_t fcs = 0;
    for (int i = 0; i < fcs_bytes; i++) fcs |= (uint64_t)src[ip + i] << (8 * i);
    if (fcs_bytes == 2) fcs += 256;
    ip += fcs_bytes;
    // frame state
    w->rep[0] = 1;
    w->rep[1] = 4;
    w->rep[2] = 8;
    w->ll_ok = w->of_ok = w->ml_ok = w->huf_ok = false;
    uint8_t* out = size_only ? nullptr : dst + total;
    const uint64_t room = size_only ? 0 : cap - total;
    uint64_t op = 0;
    for (;;) {
      if (ip + 3 > n) return kErrCorrupt;
      const uint32_t bh = src[ip] | (src[ip + 1] << 8) | ((uint32_t)src[ip + 2] << 16);
      ip += 3;
      const int last = bh & 1, type = (bh >> 1) & 3;
      const uint32_t bsize = bh >> 3;
      if (type == 3 || bsize > kBlockMax) return kErrCorrupt;
      if (type == 0) {
        if (bsize > n - ip) return kErrCorrupt;
        if (!size_only) {
          if (op + bsize > room) return kErrDstTooSmall;
          for (uint32_t k = B2S_LANE; k < bsize; k += B2S_NLANES) out[op + k] = src[ip + k];
          B2S_SYNC();
        }
        ip += bsize;
        op += bsize;
      } else if (type == 1) {
        if (ip >= n) return kErrCorrupt;
        if (!size_only) {
          if (op + bsize > room) return kErrDstTooSmall;
          for (uint32_t k = B2S_LANE; k < bsize; k += B2S_NLANES) out[op + k] = src[ip];
          B2S_SYNC();
        }
        ip += 1;
        op += bsize;
      } else {
        if (bsize > n - ip) return kErrCorrupt;
        const int64_t r = decode_compressed_block(w, src + ip, bsize, out, op, room, size_only);
        if (r < 0) return r;
        ip += bsize;
        op += (uint64_t)r;
      }
      if (last) break;
    }
    if (fcs_bytes && fcs != op) return kErrCorrupt;
    if (checksum) {
      if (ip + 4 > n) return kErrCorrupt;
      ip += 4;
    }
    total += op;
  }
  return (int64_t)total;
}

}  // namespace zstd
}  // namespace b2s
