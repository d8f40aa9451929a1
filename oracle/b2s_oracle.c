/*
 * b2s_oracle.c — CPU ORACLE (plain C).  TEST INFRASTRUCTURE ONLY — see b2s_oracle.h for scope and pinning.
 * Never linked into, imported by, or executed from the product library (spark-s3-shuffle_b200/).
 */
#include "b2s_oracle.h"

#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ======================================================================================================
 * Checksums.  java.util.zip.CRC32 / Adler32 are what S3ShuffleHelper.createChecksumAlgorithm returns
 * (helper/S3ShuffleHelper.scala:94-103); CRC32C (java.util.zip.CRC32C, Castagnoli) is the north-star's addition.
 * Bitwise-definition tables built at first use; slicing-by-8 for speed (the baseline leg times this).
 * ====================================================================================================== */
static uint32_t g_crc_tab[2][8][256];
static int g_crc_init_done[2];

static void crc_init(int which, uint32_t poly_reflected) {
  if (g_crc_init_done[which]) return;
  for (uint32_t i = 0; i < 256; i++) {
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ poly_reflected : (c >> 1);
    g_crc_tab[which][0][i] = c;
  }
  for (uint32_t i = 0; i < 256; i++)
    for (int s = 1; s < 8; s++) {
      uint32_t c = g_crc_tab[which][s - 1][i];
      g_crc_tab[which][s][i] = g_crc_tab[which][0][c & 0xff] ^ (c >> 8);
    }
  g_crc_init_done[which] = 1;
}

static uint32_t crc_generic(int which, uint32_t crc, const uint8_t* p, size_t n) {
  uint32_t(*T)[256] = g_crc_tab[which];
  crc = ~crc;
  while (n && ((uintptr_t)p & 7)) {
    crc = T[0][(crc ^ *p++) & 0xff] ^ (crc >> 8);
    n--;
  }
  while (n >= 8) {
    uint32_t a, b;
    memcpy(&a, p, 4);
    memcpy(&b, p + 4, 4);
    a ^= crc;
    crc = T[7][a & 0xff] ^ T[6][(a >> 8) & 0xff] ^ T[5][(a >> 16) & 0xff] ^ T[4][a >> 24] ^ T[3][b & 0xff] ^
          T[2][(b >> 8) & 0xff] ^ T[1][(b >> 16) & 0xff] ^ T[0][b >> 24];
    p += 8;
    n -= 8;
  }
  while (n--) crc = T[0][(crc ^ *p++) & 0xff] ^ (crc >> 8);
  return ~crc;
}

uint32_t orc_crc32(uint32_t crc, const uint8_t* p, size_t n) {
  crc_init(0, 0xEDB88320u);
  return crc_generic(0, crc, p, n);
}
uint32_t orc_crc32c(uint32_t crc, const uint8_t* p, size_t n) {
  crc_init(1, 0x82F63B78u);
  return crc_generic(1, crc, p, n);
}

uint32_t orc_adler32(uint32_t adler, const uint8_t* p, size_t n) {
  uint32_t a = adler & 0xffff, b = adler >> 16;
  while (n) {
    size_t k = n < 5552 ? n : 5552; /* largest run before 32-bit overflow, as in zlib */
    n -= k;
    while (k--) {
      a += *p++;
      b += a;
    }
    a %= 65521u;
    b %= 65521u;
  }
  return (b << 16) | a;
}

uint32_t orc_checksum(uint32_t alg, const uint8_t* p, size_t n) {
  switch (alg) {
    case 1: return orc_adler32(1, p, n);
    case 2: return orc_crc32(0, p, n);
    case 3: return orc_crc32c(0, p, n);
    default: return 0;
  }
}

/* XXH32 — lz4-java's StreamingXXHash32(seed 0x9747b28c) [U]; published algorithm (xxHash spec). */
#define XP1 2654435761u
#define XP2 2246822519u
#define XP3 3266489917u
#define XP4 668265263u
#define XP5 374761393u
static inline uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
static inline uint32_t rd32(const uint8_t* p) {
  uint32_t v;
  memcpy(&v, p, 4);
  return v;
}
uint32_t orc_xxh32(const uint8_t* p, size_t n, uint32_t seed) {
  const uint8_t* end = p + n;
  uint32_t h;
  if (n >= 16) {
    uint32_t v1 = seed + XP1 + XP2, v2 = seed + XP2, v3 = seed, v4 = seed - XP1;
    const uint8_t* lim = end - 16;
    do {
      v1 = rotl32(v1 + rd32(p) * XP2, 13) * XP1;
      v2 = rotl32(v2 + rd32(p + 4) * XP2, 13) * XP1;
      v3 = rotl32(v3 + rd32(p + 8) * XP2, 13) * XP1;
      v4 = rotl32(v4 + rd32(p + 12) * XP2, 13) * XP1;
      p += 16;
    } while (p <= lim);
    h = rotl32(v1, 1) + rotl32(v2, 7) + rotl32(v3, 12) + rotl32(v4, 18);
  } else {
    h = seed + XP5;
  }
  h += (uint32_t)n;
  while (p + 4 <= end) {
    h = rotl32(h + rd32(p) * XP3, 17) * XP4;
    p += 4;
  }
  while (p < end) {
    h = rotl32(h + (*p++) * XP5, 11) * XP1;
  }
  h ^= h >> 15;
  h *= XP2;
  h ^= h >> 13;
  h *= XP3;
  h ^= h >> 16;
  return h;
}

/* ======================================================================================================
 * Raw LZ4 block format (lz4 "block format description"): sequences of token | [litlen ext] | literals |
 * offset LE16 | [matchlen ext]; end-of-block rules: last 5 bytes literal, last match starts >= 12 bytes
 * before the end.  The JVM path calls liblz4's LZ4_compress_default / LZ4_decompress_fast through lz4-java [U].
 * ====================================================================================================== */
#define LZ4_MINMATCH 4
#define LZ4_MFLIMIT 12
#define LZ4_LASTLITERALS 5

static inline uint32_t lz4_hash(uint32_t v, int hash_log) { return (v * 2654435761u) >> (32 - hash_log); }

/* emits one sequence; returns new op or -1 when the output would not fit */
static int lz4_emit_seq(const uint8_t* src, int anchor, int lit, int off, int mlen, uint8_t* dst, int op, int cap) {
  int need = 1 + lit + (lit >= 15 ? (lit - 15) / 255 + 1 : 0);
  if (mlen) need += 2 + (mlen - 4 >= 15 ? (mlen - 4 - 15) / 255 + 1 : 0);
  if (op + need > cap) return -1;
  int tok = op++;
  if (lit >= 15) {
    int r = lit - 15;
    dst[tok] = 15 << 4;
    while (r >= 255) {
      dst[op++] = 255;
      r -= 255;
    }
    dst[op++] = (uint8_t)r;
  } else {
    dst[tok] = (uint8_t)(lit << 4);
  }
  memcpy(dst + op, src + anchor, (size_t)lit);
  op += lit;
  if (mlen) {
    dst[op++] = (uint8_t)off;
    dst[op++] = (uint8_t)(off >> 8);
    int m = mlen - 4;
    if (m >= 15) {
      dst[tok] |= 15;
      m -= 15;
      while (m >= 255) {
        dst[op++] = 255;
        m -= 255;
      }
      dst[op++] = (uint8_t)m;
    } else {
      dst[tok] |= (uint8_t)m;
    }
  }
  return op;
}

int orc_lz4_compress_block(const uint8_t* src, int n, uint8_t* dst, int cap) {
  enum { HL = 12 };
  int table[1 << HL];
  int op = 0, anchor = 0;
  if (n >= LZ4_MFLIMIT + 1) {
    const int mflimit = n - LZ4_MFLIMIT;  /* last position a match may start at */
    const int matchlimit = n - LZ4_LASTLITERALS;
    memset(table, 0, sizeof table);
    table[lz4_hash(rd32(src), HL)] = 0;
    int ip = 1;
    for (;;) {
      /* search with liblz4-style acceleration: step grows after 64 misses */
      int cand, misses = 1 << 6, step;
      for (;;) {
        if (ip > mflimit) goto last_literals;
        uint32_t h = lz4_hash(rd32(src + ip), HL);
        cand = table[h];
        table[h] = ip;
        if (ip - cand <= 65535 && cand < ip && rd32(src + cand) == rd32(src + ip)) break;
        step = misses++ >> 6;
        ip += step;
      }
      /* extend backwards */
      while (ip > anchor && cand > 0 && src[ip - 1] == src[cand - 1]) {
        ip--;
        cand--;
      }
      int mlen = LZ4_MINMATCH;
      while (ip + mlen < matchlimit && src[ip + mlen] == src[cand + mlen]) mlen++;
      op = lz4_emit_seq(src, anchor, ip - anchor, ip - cand, mlen, dst, op, cap);
      if (op < 0) return 0;
      ip += mlen;
      anchor = ip;
      if (ip > mflimit) break;
      table[lz4_hash(rd32(src + ip - 2), HL)] = ip - 2;
    }
  }
last_literals:
  op = lz4_emit_seq(src, anchor, n - anchor, 0, 0, dst, op, cap);
  return op < 0 ? 0 : op;
}

/*
 * CPU model of the GPU compressor (DESIGN.md K3) — the kernels' executable specification, bit-identical output.
 * Three phases, mirroring the three kernels:
 *  A  match finding, parse-independent: the block is cut into FIXED windows of 32 positions.  Every position
 *     p <= mflimit of a window looks its 4 bytes up in a u16 hash table holding the state *before* the window
 *     (zero-initialised, so position 0 is a legal candidate); a byte run (the 4 bytes at p-1 equal those at p) uses
 *     the offset-1 candidate instead.  A verified candidate yields off[p] = p - cand, else 0.  Then all positions
 *     of the window are inserted (highest position wins a slot).
 *  B  greedy parse over off[]: the lowest p >= cursor with off[p] != 0 starts a match, extended forward to
 *     matchlimit; the cursor jumps to its end.
 *  C  LZ4 sequence emission.
 */
/* phase A of the GPU model: off[p] for every p <= n - 12 (0 = no match); off has n entries, zero-initialised */
static void win_find_offsets(const uint8_t* src, int n, int hash_log, uint16_t* off) {
  enum { W = 32 };
  uint16_t* table = (uint16_t*)calloc((size_t)1 << hash_log, sizeof(uint16_t));
  const int mflimit = n - LZ4_MFLIMIT;
  for (int pos = 0; pos <= mflimit; pos += W) {
    const int last = pos + W - 1 < mflimit ? pos + W - 1 : mflimit;
    for (int p = pos; p <= last; p++) {
      const uint32_t v = rd32(src + p);
      const int c = table[lz4_hash(v, hash_log)];
      if (p > 0 && rd32(src + p - 1) == v) off[p] = 1;
      else if (c < p && rd32(src + c) == v) off[p] = (uint16_t)(p - c);
    }
    for (int p = pos; p <= last; p++) table[lz4_hash(rd32(src + p), hash_log)] = (uint16_t)p;
  }
  free(table);
}

/* The greedy walk shared by the CPU models of the three GPU encoders: from cursor *p, the next match the parse takes
 * (its position in *p, its length in *mlen), or 0 when the block holds no further match. */
static int win_next_match(const uint8_t* src, const uint16_t* off, int n, int* p, int* mlen) {
  const int mflimit = n - LZ4_MFLIMIT, matchlimit = n - LZ4_LASTLITERALS;
  int q = *p;
  while (q <= mflimit) {
    if (!off[q]) {
      q++;
      continue;
    }
    const int c = q - off[q];
    int l = LZ4_MINMATCH;
    while (q + l < matchlimit && src[q + l] == src[c + l]) l++;
    *p = q;
    *mlen = l;
    return 1;
  }
  return 0;
}

int orc_lz4_compress_block_win(const uint8_t* src, int n, uint8_t* dst, int cap, int hash_log) {
  if (n > 65536 || hash_log > 16 || hash_log < 4) return 0;
  uint16_t* off = (uint16_t*)calloc((size_t)(n > 0 ? n : 1), sizeof(uint16_t));
  int op = 0, anchor = 0;
  if (n >= LZ4_MFLIMIT + 1) {
    win_find_offsets(src, n, hash_log, off); /* phase A */
    int p = 0, mlen = 0;                      /* phase B + C */
    while (win_next_match(src, off, n, &p, &mlen)) {
      op = lz4_emit_seq(src, anchor, p - anchor, off[p], mlen, dst, op, cap);
      if (op < 0) {
        free(off);
        return 0;
      }
      p += mlen;
      anchor = p;
    }
  }
  op = lz4_emit_seq(src, anchor, n - anchor, 0, 0, dst, op, cap);
  free(off);
  return op < 0 ? 0 : op;
}

/* LZ4_decompress_fast semantics (lz4 1.9.4 LZ4_decompress_unsafe_generic), plus input bounds checks */
int orc_lz4_decompress_block(const uint8_t* src, int src_len, uint8_t* dst, int orig_len) {
  int ip = 0, op = 0;
  for (;;) {
    if (ip >= src_len) return -1;
    int token = src[ip++];
    int ll = token >> 4;
    if (ll == 15) {
      int b;
      do {
        if (ip >= src_len) return -1;
        b = src[ip++];
        ll += b;
        if (ll > orig_len) return -1; /* cannot be valid, and a long run of 0xFF bytes must not wrap the counter */
      } while (b == 255);
    }
    if (ll > orig_len - op || ll > src_len - ip) return -1;
    memcpy(dst + op, src + ip, (size_t)ll);
    op += ll;
    ip += ll;
    if (orig_len - op < LZ4_MFLIMIT) {
      if (op == orig_len) return ip;
      return -1; /* last match must start >= 12 bytes before the end */
    }
    if (ip + 2 > src_len) return -1;
    int off = src[ip] | (src[ip + 1] << 8);
    ip += 2;
    int ml = token & 15;
    if (ml == 15) {
      int b;
      do {
        if (ip >= src_len) return -1;
        b = src[ip++];
        ml += b;
        if (ml > orig_len) return -1;
      } while (b == 255);
    }
    ml += LZ4_MINMATCH;
    if (ml > orig_len - op) return -1;
    if (off == 0 || off > op) return -1;
    for (int i = 0; i < ml; i++) dst[op + i] = dst[op - off + i];
    op += ml;
    if (orig_len - op < LZ4_LASTLITERALS) return -1;
  }
}

/* ======================================================================================================
 * lz4-java LZ4BlockOutputStream / LZ4BlockInputStream framing [U] (net.jpountz.lz4, 1.8.0), as constructed by
 * Spark's LZ4CompressionCodec: blockSize = spark.io.compression.lz4.blockSize (32 KiB), syncFlush=false,
 * checksum = XXH32(seed 0x9747b28c) & 0x0FFFFFFF, reader with stopOnEmptyBlock=false (concatenation allowed).
 * header: "LZ4Block" | token(method|level) | compressedLen LE32 | originalLen LE32 | check LE32
 * ====================================================================================================== */
static const uint8_t LZ4B_MAGIC[8] = {'L', 'Z', '4', 'B', 'l', 'o', 'c', 'k'};
#define LZ4B_RAW 0x10
#define LZ4B_LZ4 0x20
#define LZ4B_LEVEL_BASE 10
#define LZ4B_SEED 0x9747b28cu

static int lz4b_level(uint32_t block_size) {
  int bits = 0;
  uint32_t v = block_size - 1;
  while (v) {
    bits++;
    v >>= 1;
  }
  int lvl = bits - LZ4B_LEVEL_BASE;
  return lvl < 0 ? 0 : lvl;
}
static void wr_le32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)v;
  p[1] = (uint8_t)(v >> 8);
  p[2] = (uint8_t)(v >> 16);
  p[3] = (uint8_t)(v >> 24);
}
static uint32_t rd_le32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

uint64_t orc_lz4block_bound(uint64_t n, uint32_t block_size) {
  uint64_t nb = (n + block_size - 1) / block_size;
  return n + (nb + 1) * ORC_LZ4B_HEADER;
}

static int64_t lz4block_compress_impl(const uint8_t* src, uint64_t n, uint32_t block_size, uint8_t* dst, uint64_t cap,
                                      int compressor, orc_lz4_compress_fn ext) {
  if (block_size < 64 || block_size > (1u << 25) || compressor < 0 || compressor > 1) return -3;
  const int level = lz4b_level(block_size);
  uint64_t op = 0;
  uint8_t* tmp = (uint8_t*)malloc(block_size + block_size / 255 + 32);
  for (uint64_t off = 0; off < n; off += block_size) {
    uint32_t o = (uint32_t)(n - off < block_size ? n - off : block_size);
    if (op + ORC_LZ4B_HEADER + o > cap) {
      free(tmp);
      return -2;
    }
    uint32_t check = orc_xxh32(src + off, o, LZ4B_SEED) & 0x0FFFFFFFu;
    int clen;
    int tcap = (int)(block_size + block_size / 255 + 32);
    if (ext)
      clen = ext((const char*)(src + off), (char*)tmp, (int)o, tcap);
    else if (compressor == 1) /* the GPU pipeline: single-cursor greedy parse */
      clen = (o <= 65536) ? orc_lz4_compress_block_win(src + off, (int)o, tmp, (int)o - 1, 12) : 0;
    else
      clen = orc_lz4_compress_block(src + off, (int)o, tmp, tcap);
    int method = LZ4B_LZ4;
    if (clen <= 0 || (uint32_t)clen >= o) { /* LZ4BlockOutputStream.flushBufferedData: RAW if compressedLength >= o */
      method = LZ4B_RAW;
      clen = (int)o;
    }
    memcpy(dst + op, LZ4B_MAGIC, 8);
    dst[op + 8] = (uint8_t)(method | level);
    wr_le32(dst + op + 9, (uint32_t)clen);
    wr_le32(dst + op + 13, o);
    wr_le32(dst + op + 17, check);
    memcpy(dst + op + ORC_LZ4B_HEADER, method == LZ4B_RAW ? src + off : tmp, (size_t)clen);
    op += ORC_LZ4B_HEADER + (uint64_t)clen;
  }
  free(tmp);
  if (op + ORC_LZ4B_HEADER > cap) return -2;
  /* finish(): end mark = RAW|level, three zero ints */
  memcpy(dst + op, LZ4B_MAGIC, 8);
  dst[op + 8] = (uint8_t)(LZ4B_RAW | level);
  memset(dst + op + 9, 0, 12);
  return (int64_t)(op + ORC_LZ4B_HEADER);
}

int64_t orc_lz4block_compress(const uint8_t* src, uint64_t n, uint32_t block_size, uint8_t* dst, uint64_t cap,
                              int compressor) {
  return lz4block_compress_impl(src, n, block_size, dst, cap, compressor, NULL);
}

/* walks the stream like LZ4BlockInputStream.refill(); dst==NULL => size only */
static int64_t lz4block_walk(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t cap, orc_lz4_decompress_fast_fn ext) {
  uint64_t ip = 0, op = 0;
  while (ip < n) {
    if (n - ip < ORC_LZ4B_HEADER) return -1; /* truncated header: EOFException("Stream ended prematurely") */
    if (memcmp(src + ip, LZ4B_MAGIC, 8)) return -1;
    int token = src[ip + 8];
    int method = token & 0xF0, level = LZ4B_LEVEL_BASE + (token & 0x0F);
    if (method != LZ4B_RAW && method != LZ4B_LZ4) return -1;
    int32_t clen = (int32_t)rd_le32(src + ip + 9), olen = (int32_t)rd_le32(src + ip + 13);
    uint32_t check = rd_le32(src + ip + 17);
    if (olen > (1 << level) || olen < 0 || clen < 0 || (olen == 0 && clen != 0) || (olen != 0 && clen == 0) ||
        (method == LZ4B_RAW && olen != clen))
      return -1;
    ip += ORC_LZ4B_HEADER;
    if (olen == 0 && clen == 0) {
      if (check != 0) return -1;
      continue; /* end mark; stopOnEmptyBlock=false => try the next concatenated stream */
    }
    if ((uint64_t)clen > n - ip) return -1;
    if (dst) {
      if (op + (uint64_t)olen > cap) return -2;
      if (method == LZ4B_RAW) {
        memcpy(dst + op, src + ip, (size_t)olen);
      } else {
        int used = ext ? ext((const char*)(src + ip), (char*)(dst + op), olen)
                       : orc_lz4_decompress_block(src + ip, clen, dst + op, olen);
        if (used != clen) return -1;
      }
      if ((orc_xxh32(dst + op, (size_t)olen, LZ4B_SEED) & 0x0FFFFFFFu) != check) return -1;
    }
    ip += (uint64_t)clen;
    op += (uint64_t)olen;
  }
  return (int64_t)op;
}
int64_t orc_lz4block_decompress(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t cap) {
  static uint8_t dummy;
  return lz4block_walk(src, n, dst ? dst : &dummy, cap, NULL);
}
int64_t orc_lz4block_decompressed_size(const uint8_t* src, uint64_t n) { return lz4block_walk(src, n, NULL, 0, NULL); }

/* ======================================================================================================
 * Raw Snappy (format_description.txt of google/snappy) + xerial SnappyOutputStream framing [U]
 * (org.xerial.snappy 1.1.10.x): 16-byte header {0x82 'S' 'N' 'A' 'P' 'P' 'Y' 0x00, BE32 version=1, BE32 compat=1},
 * then chunks: BE32 compressed length | raw snappy block of <= blockSize (32 KiB) input bytes.
 * ====================================================================================================== */
uint64_t orc_snappy_max_compressed(uint64_t n) { return 32 + n + n / 6; }

static uint64_t snappy_emit_literal(uint8_t* dst, uint64_t op, const uint8_t* lit, uint64_t len) {
  uint64_t n1 = len - 1;
  if (n1 < 60) {
    dst[op++] = (uint8_t)(n1 << 2);
  } else {
    int bytes = n1 < (1u << 8) ? 1 : n1 < (1u << 16) ? 2 : n1 < (1u << 24) ? 3 : 4;
    dst[op++] = (uint8_t)((59 + bytes) << 2);
    for (int i = 0; i < bytes; i++) dst[op++] = (uint8_t)(n1 >> (8 * i));
  }
  memcpy(dst + op, lit, len);
  return op + len;
}
static uint64_t snappy_emit_copy_le64(uint8_t* dst, uint64_t op, uint32_t off, uint32_t len) {
  if (len < 12 && off < 2048) {
    dst[op++] = (uint8_t)(1 | ((len - 4) << 2) | ((off >> 8) << 5));
    dst[op++] = (uint8_t)off;
  } else {
    dst[op++] = (uint8_t)(2 | ((len - 1) << 2));
    dst[op++] = (uint8_t)off;
    dst[op++] = (uint8_t)(off >> 8);
  }
  return op;
}
static uint64_t snappy_emit_copy(uint8_t* dst, uint64_t op, uint32_t off, uint32_t len) {
  while (len >= 68) {
    op = snappy_emit_copy_le64(dst, op, off, 64);
    len -= 64;
  }
  if (len > 64) {
    op = snappy_emit_copy_le64(dst, op, off, 60);
    len -= 60;
  }
  return snappy_emit_copy_le64(dst, op, off, len);
}

int64_t orc_snappy_compress_raw(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t cap) {
  if (cap < orc_snappy_max_compressed(n) || n > 0xffffffffu) return -2;
  uint64_t op = 0;
  uint64_t v = n;
  while (v >= 0x80) {
    dst[op++] = (uint8_t)(v | 0x80);
    v >>= 7;
  }
  dst[op++] = (uint8_t)v;
  /* snappy compresses independent 64 KiB fragments */
  enum { HL = 14 };
  static __thread uint16_t table[1 << HL];
  for (uint64_t base = 0; base < n; base += 65536) {
    const uint8_t* f = src + base;
    uint32_t fn = (uint32_t)(n - base < 65536 ? n - base : 65536);
    uint32_t ip = 0, anchor = 0;
    memset(table, 0, sizeof table);
    if (fn >= 15) {
      const uint32_t ip_limit = fn - 15;
      ip = 1;
      while (ip <= ip_limit) {
        uint32_t h = (rd32(f + ip) * 0x1e35a7bdu) >> (32 - HL);
        uint32_t cand = table[h];
        table[h] = (uint16_t)ip;
        if (cand < ip && rd32(f + cand) == rd32(f + ip)) {
          uint32_t mlen = 4;
          while (ip + mlen < fn && f[ip + mlen] == f[cand + mlen]) mlen++;
          if (ip > anchor) op = snappy_emit_literal(dst, op, f + anchor, ip - anchor);
          op = snappy_emit_copy(dst, op, ip - cand, mlen);
          ip += mlen;
          anchor = ip;
        } else {
          ip++;
        }
      }
    }
    if (anchor < fn) op = snappy_emit_literal(dst, op, f + anchor, fn - anchor);
  }
  return (int64_t)op;
}

/* CPU model of the GPU Snappy compressor: the same match finding and greedy parse as orc_lz4_compress_block_win
 * (including its end-of-block margins: no match starts in the last 12 bytes or covers the last 5 — legal, merely
 * conservative, for Snappy), emitted in the Snappy element grammar.  One chunk <= 32 KiB (the xerial block size). */
int64_t orc_snappy_compress_raw_win(const uint8_t* src, uint64_t n64, uint8_t* dst, uint64_t cap, int hash_log) {
  if (n64 > 32768 || cap < orc_snappy_max_compressed(n64)) return -2;
  const int n = (int)n64;
  uint64_t op = 0;
  uint64_t v = n64;
  while (v >= 0x80) {
    dst[op++] = (uint8_t)(v | 0x80);
    v >>= 7;
  }
  dst[op++] = (uint8_t)v;
  int anchor = 0;
  if (n >= LZ4_MFLIMIT + 1) {
    uint16_t* off = (uint16_t*)calloc((size_t)n, sizeof(uint16_t));
    win_find_offsets(src, n, hash_log, off);
    int p = 0, mlen = 0;
    while (win_next_match(src, off, n, &p, &mlen)) {
      if (p > anchor) op = snappy_emit_literal(dst, op, src + anchor, (uint64_t)(p - anchor));
      op = snappy_emit_copy(dst, op, off[p], (uint32_t)mlen);
      p += mlen;
      anchor = p;
    }
    free(off);
  }
  if (anchor < n) op = snappy_emit_literal(dst, op, src + anchor, (uint64_t)(n - anchor));
  return (int64_t)op;
}

int64_t orc_snappy_uncompressed_length(const uint8_t* src, uint64_t n) {
  uint64_t v = 0;
  for (int i = 0; i < 5; i++) {
    if ((uint64_t)i >= n) return -1;
    uint8_t b = src[i];
    v |= (uint64_t)(b & 0x7f) << (7 * i);
    if (!(b & 0x80)) return v > 0xffffffffu ? -1 : (int64_t)v;
  }
  return -1;
}

int64_t orc_snappy_uncompress_raw(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t cap) {
  int64_t ulen = orc_snappy_uncompressed_length(src, n);
  if (ulen < 0) return -1;
  if ((uint64_t)ulen > cap) return -2;
  uint64_t ip = 0, op = 0;
  while (src[ip++] & 0x80) {
  }
  while (ip < n) {
    uint8_t tag = src[ip++];
    uint32_t len, off;
    switch (tag & 3) {
      case 0: {
        len = (tag >> 2) + 1;
        if (len > 60) {
          uint32_t nb = len - 60;
          if (ip + nb > n) return -1;
          len = 0;
          for (uint32_t i = 0; i < nb; i++) len |= (uint32_t)src[ip + i] << (8 * i);
          len += 1;
          ip += nb;
        }
        if (len > n - ip || len > (uint64_t)ulen - op) return -1;
        memcpy(dst + op, src + ip, len);
        ip += len;
        op += len;
        continue;
      }
      case 1:
        if (ip + 1 > n) return -1;
        len = 4 + ((tag >> 2) & 7);
        off = ((uint32_t)(tag >> 5) << 8) | src[ip];
        ip += 1;
        break;
      case 2:
        if (ip + 2 > n) return -1;
        len = (tag >> 2) + 1;
        off = src[ip] | (src[ip + 1] << 8);
        ip += 2;
        break;
      default:
        if (ip + 4 > n) return -1;
        len = (tag >> 2) + 1;
        off = rd_le32(src + ip);
        ip += 4;
        break;
    }
    if (off == 0 || off > op || len > (uint64_t)ulen - op) return -1;
    for (uint32_t i = 0; i < len; i++) dst[op + i] = dst[op - off + i];
    op += len;
  }
  return op == (uint64_t)ulen ? (int64_t)op : -1;
}

static const uint8_t XERIAL_HEADER[16] = {0x82, 'S', 'N', 'A', 'P', 'P', 'Y', 0, 0, 0, 0, 1, 0, 0, 0, 1};
static void wr_be32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24);
  p[1] = (uint8_t)(v >> 16);
  p[2] = (uint8_t)(v >> 8);
  p[3] = (uint8_t)v;
}
static uint32_t rd_be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; }

uint64_t orc_xerial_bound(uint64_t n, uint32_t block_size) {
  uint64_t nb = (n + block_size - 1) / block_size;
  return ORC_XERIAL_HEADER + nb * (4 + orc_snappy_max_compressed(block_size));
}
static int64_t xerial_compress_impl(const uint8_t* src, uint64_t n, uint32_t block_size, uint8_t* dst, uint64_t cap,
                                    int compressor) {
  if (compressor < 0 || compressor > 1) return -3;
  if (cap < ORC_XERIAL_HEADER) return -2;
  memcpy(dst, XERIAL_HEADER, 16);
  uint64_t op = 16;
  for (uint64_t off = 0; off < n; off += block_size) {
    uint64_t o = n - off < block_size ? n - off : block_size;
    if (op + 4 + orc_snappy_max_compressed(o) > cap) return -2;
    int64_t c = compressor == 1 ? orc_snappy_compress_raw_win(src + off, o, dst + op + 4, cap - op - 4, 12)
                                : orc_snappy_compress_raw(src + off, o, dst + op + 4, cap - op - 4);
    if (c < 0) return c;
    wr_be32(dst + op, (uint32_t)c);
    op += 4 + (uint64_t)c;
  }
  return (int64_t)op;
}
int64_t orc_xerial_compress(const uint8_t* src, uint64_t n, uint32_t block_size, uint8_t* dst, uint64_t cap) {
  return xerial_compress_impl(src, n, block_size, dst, cap, 0);
}
/* compressor: 0 = restated snappy-style greedy, 1 = GPU window model (hash_log 12, block_size <= 32 KiB);
 * any other value returns -3 */
int64_t orc_xerial_compress2(const uint8_t* src, uint64_t n, uint32_t block_size, uint8_t* dst, uint64_t cap,
                             int compressor) {
  return xerial_compress_impl(src, n, block_size, dst, cap, compressor);
}
static int64_t xerial_walk(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t cap) {
  if (n == 0) return 0; /* SnappyInputStream.readHeader: no bytes at all is an empty stream */
  if (n < 16 || memcmp(src, XERIAL_HEADER, 8)) return -1;
  uint64_t ip = 16, op = 0;
  while (ip < n) {
    if (n - ip < 4) return -1;
    uint32_t clen = rd_be32(src + ip);
    ip += 4;
    if (clen == 0x82534E41u) { /* SnappyInputStream.hasNextChunk: concatenated stream header */
      if (n - ip < 12 || memcmp(src + ip, XERIAL_HEADER + 4, 4)) return -1;
      ip += 12;
      continue;
    }
    if (clen > n - ip) return -1;
    int64_t u = orc_snappy_uncompressed_length(src + ip, clen);
    if (u < 0) return -1;
    if (dst) {
      if (op + (uint64_t)u > cap) return -2;
      if (orc_snappy_uncompress_raw(src + ip, clen, dst + op, cap - op) != u) return -1;
    }
    ip += clen;
    op += (uint64_t)u;
  }
  return (int64_t)op;
}
int64_t orc_xerial_decompress(const uint8_t* src, uint64_t n, uint8_t* dst, uint64_t cap) {
  static uint8_t dummy;
  return xerial_walk(src, n, dst ? dst : &dummy, cap);
}
int64_t orc_xerial_decompressed_size(const uint8_t* src, uint64_t n) { return xerial_walk(src, n, NULL, 0); }

/* ======================================================================================================
 * S3ChecksumValidationStream.validateChecksum (storage/S3ChecksumValidationStream.scala:63-86): per-partition
 * checksum of the compressed bytes compared with .checksum[reduceId]; zero-length partitions are skipped only
 * in the sense that their (empty-input) checksum must still equal the stored one (:80-82 recurses).
 * ====================================================================================================== */
int64_t orc_validate_slices(uint32_t alg, const uint8_t* block, const int64_t* cumulative, const int64_t* ref,
                            int start_reduce, int end_reduce) {
  int64_t base = cumulative[start_reduce];
  for (int r = start_reduce; r < end_reduce; r++) {
    int64_t len = cumulative[r + 1] - cumulative[r];
    uint32_t c = orc_checksum(alg, block + (cumulative[r] - base), (size_t)len);
    if ((int64_t)c != ref[r]) return r;
  }
  return -1;
}

/* helper/S3ShuffleHelper.scala:44-47: Array(0) ++ lengths.tail.scan(lengths.head)(_ + _), DataOutputStream.writeLong */
void orc_be64_array(const int64_t* v, int n, uint8_t* out) {
  for (int i = 0; i < n; i++)
    for (int b = 0; b < 8; b++) out[i * 8 + b] = (uint8_t)((uint64_t)v[i] >> (56 - 8 * b));
}
void orc_index_from_lengths(const int64_t* lengths, int n, uint8_t* out) {
  int64_t acc = 0;
  orc_be64_array(&acc, 1, out);
  for (int i = 0; i < n; i++) {
    acc += lengths[i];
    orc_be64_array(&acc, 1, out + 8 * (i + 1));
  }
}
int orc_read_be64_array(const uint8_t* in, uint64_t nbytes, int64_t* out) {
  if (nbytes % 8) return -1;
  for (uint64_t i = 0; i < nbytes / 8; i++) {
    uint64_t v = 0;
    for (int b = 0; b < 8; b++) v = (v << 8) | in[i * 8 + b];
    out[i] = (int64_t)v;
  }
  return (int)(nbytes / 8);
}

/* ======================================================================================================
 * Synthetic terasort-shaped records (SURVEY.md §8d config 2/3).  104 bytes:
 *   01 0B | key[10] random | 01 5B | 00 11 | rowid 32 hex | 88 99 AA BB | 12 random hex digits x4 | CC DD EE FF
 * Counter-based (splitmix64) so the GPU generator in the bench produces identical bytes.
 * ====================================================================================================== */
static inline uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
void orc_gen_terasort(uint8_t* dst, uint64_t first_record, uint64_t n_records, uint64_t seed) {
  static const char HEX[] = "0123456789ABCDEF";
  for (uint64_t i = 0; i < n_records; i++) {
    uint64_t g = first_record + i;
    uint8_t* r = dst + i * 104;
    uint64_t a = mix64(seed ^ mix64(g * 4 + 0)), b = mix64(seed ^ mix64(g * 4 + 1)), c = mix64(seed ^ mix64(g * 4 + 2));
    r[0] = 0x01;
    r[1] = 0x0B;
    for (int k = 0; k < 8; k++) r[2 + k] = (uint8_t)(a >> (8 * k));
    r[10] = (uint8_t)b;
    r[11] = (uint8_t)(b >> 8);
    r[12] = 0x01;
    r[13] = 0x5B;
    r[14] = 0x00;
    r[15] = 0x11;
    for (int k = 0; k < 32; k++) r[16 + k] = (k < 16) ? '0' : (uint8_t)HEX[(g >> (4 * (31 - k))) & 15];
    r[48] = 0x88;
    r[49] = 0x99;
    r[50] = 0xAA;
    r[51] = 0xBB;
    for (int k = 0; k < 12; k++) {
      uint8_t ch = (uint8_t)HEX[(c >> (4 * k)) & 15];
      r[52 + 4 * k] = r[53 + 4 * k] = r[54 + 4 * k] = r[55 + 4 * k] = ch;
    }
    r[100] = 0xCC;
    r[101] = 0xDD;
    r[102] = 0xEE;
    r[103] = 0xFF;
  }
}

/* ======================================================================================================
 * CPU baseline: what the reference's JVM path computes per shuffle block, natively, one worker per thread.
 *   write: LZ4Block stream compress (+XXH32) then checksum over the compressed stream  (call stack SURVEY §3.1)
 *   read : checksum verify over compressed bytes, then LZ4Block stream decompress (+XXH32) (storage/S3ShuffleReader.scala:99-110)
 * ====================================================================================================== */
typedef struct {
  orc_baseline_job* job;
  int tid;
  uint8_t** comp;
  uint64_t* comp_len;
  uint32_t* sums;
  int phase;
  int errors;
  const orc_codec_job* cj; /* NULL: LZ4Block */
} bl_worker;

static double now_s(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec + ts.tv_nsec * 1e-9;
}

static void* bl_thread(void* arg) {
  bl_worker* w = (bl_worker*)arg;
  orc_baseline_job* j = w->job;
  uint8_t* outbuf = NULL;
  if (w->phase == 1) outbuf = (uint8_t*)malloc(j->block_bytes + 64);
  for (uint64_t i = (uint64_t)w->tid; i < j->n_blocks; i += (uint64_t)j->threads) {
    const uint8_t* s = j->src + i * j->block_bytes;
    const uint32_t codec = w->cj ? w->cj->codec : 1u;
    if (w->phase == 0) {
      uint64_t cap = codec == 3   ? j->block_bytes + j->block_bytes / 128 + 1024
                     : codec == 2 ? orc_xerial_bound(j->block_bytes, j->lz4_block_size)
                                  : orc_lz4block_bound(j->block_bytes, j->lz4_block_size);
      if (!w->comp[i]) w->comp[i] = (uint8_t*)malloc(cap);
      int64_t c;
      if (codec == 3) {
        size_t r = w->cj->zstd_compress(w->comp[i], cap, s, j->block_bytes, w->cj->level);
        c = w->cj->zstd_is_error(r) ? -1 : (int64_t)r;
      } else if (codec == 2) {
        c = orc_xerial_compress2(s, j->block_bytes, j->lz4_block_size, w->comp[i], cap, 0);
      } else {
        c = lz4block_compress_impl(s, j->block_bytes, j->lz4_block_size, w->comp[i], cap, 0, j->lz4_compress);
      }
      if (c < 0) {
        w->errors++;
        continue;
      }
      w->comp_len[i] = (uint64_t)c;
      if (j->checksum_alg) w->sums[i] = orc_checksum(j->checksum_alg, w->comp[i], (size_t)c);
    } else {
      if (j->checksum_alg && orc_checksum(j->checksum_alg, w->comp[i], (size_t)w->comp_len[i]) != w->sums[i]) w->errors++;
      int64_t u;
      if (codec == 3) {
        size_t r = w->cj->zstd_decompress(outbuf, j->block_bytes, w->comp[i], w->comp_len[i]);
        u = w->cj->zstd_is_error(r) ? -1 : (int64_t)r;
      } else if (codec == 2) {
        u = orc_xerial_decompress(w->comp[i], w->comp_len[i], outbuf, j->block_bytes);
      } else {
        u = lz4block_walk(w->comp[i], w->comp_len[i], outbuf, j->block_bytes, j->lz4_decompress);
      }
      if (u != (int64_t)j->block_bytes || memcmp(outbuf, s, (size_t)j->block_bytes)) w->errors++;
    }
  }
  free(outbuf);
  return NULL;
}

static int baseline_run_impl(orc_baseline_job* job, const orc_codec_job* cj);
int orc_baseline_run(orc_baseline_job* job) { return baseline_run_impl(job, NULL); }
int orc_baseline_run_codec(orc_codec_job* job) {
  if (job->codec < 1 || job->codec > 3) return -2;
  if (job->codec == 3 && (!job->zstd_compress || !job->zstd_decompress || !job->zstd_is_error)) return -2;
  return baseline_run_impl(&job->base, job->codec == 1 ? NULL : job);
}
static int baseline_run_impl(orc_baseline_job* job, const orc_codec_job* cj) {
  int T = job->threads < 1 ? 1 : job->threads;
  job->threads = T;
  uint8_t** comp = (uint8_t**)calloc(job->n_blocks, sizeof(uint8_t*));
  uint64_t* comp_len = (uint64_t*)calloc(job->n_blocks, sizeof(uint64_t));
  uint32_t* sums = (uint32_t*)calloc(job->n_blocks, sizeof(uint32_t));
  pthread_t* th = (pthread_t*)calloc((size_t)T, sizeof(pthread_t));
  bl_worker* ws = (bl_worker*)calloc((size_t)T, sizeof(bl_worker));
  job->errors = 0;
  for (int phase = 0; phase < 2; phase++) {
    double t0 = now_s();
    for (int t = 0; t < T; t++) {
      ws[t] = (bl_worker){job, t, comp, comp_len, sums, phase, 0, cj};
      pthread_create(&th[t], NULL, bl_thread, &ws[t]);
    }
    for (int t = 0; t < T; t++) {
      pthread_join(th[t], NULL);
      job->errors += ws[t].errors;
    }
    double dt = now_s() - t0;
    if (phase == 0)
      job->write_seconds = dt;
    else
      job->read_seconds = dt;
  }
  job->compressed_bytes = 0;
  for (uint64_t i = 0; i < job->n_blocks; i++) {
    job->compressed_bytes += comp_len[i];
    free(comp[i]);
  }
  free(comp);
  free(comp_len);
  free(sums);
  free(th);
  free(ws);
  return job->errors ? -1 : 0;
}
