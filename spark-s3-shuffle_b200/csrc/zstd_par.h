// zstd_par.h — Zstandard decoding split so that the BLOCKS of a frame decode in parallel (host + device, like
// zstd_core.h whose table/bit-stream functions it reuses).
//
// A frame is serial in three ways only: (1) a block may reuse the previous block's entropy tables (Repeat_Mode,
// treeless literals), (2) the three repeat offsets run across blocks, (3) matches reach back into earlier output.
// None of them needs the expensive part — Huffman literals and the FSE sequence decoder — to be serial:
//
//   walk      THREAD per stream.  Reads only headers (frame, block, literals-section sizes, Number_of_Sequences, the
//             compression-modes byte) and records one BlockInfo per block, including which earlier block DEFINES each
//             table a Repeat_Mode block uses (table provenance).  Run twice: counting, then filling.
//   entropy   WARP per block, all blocks of all streams at once.  Builds the block's tables — from its own descriptions
//             or by re-reading the defining block's — decodes the literals into a workspace and the sequences into
//             (literal length, match length, offset value) triples; offset values 1..3 stay unresolved.  Also yields the
//             block's regenerated size, which is all the size pass needs.
//   execute   WARP per stream, blocks in order.  Resolves repeat offsets, places literals and matches: ~15
//             warp-instructions per sequence instead of the ~300 of the FSE decoder, so the serial tail is short.
//
// decode_stream() of zstd_core.h stays as the single-pass statement of the same semantics; the host unit test
// (tests/native/zstd_core_host.cpp) checks both against libzstd.
#pragma once
#include "zstd_core.h"

namespace b2s {
namespace zstd {

struct BlockInfo {
  uint64_t src;       // offset of the block's content from src_base
  uint64_t lit_base;  // literals workspace offset (Huffman / RLE literals); raw literals are read in place
  uint64_t seq_base;  // first slot of this block's sequences in the ll / ml / ofv arrays
  uint64_t fcs;       // Frame_Content_Size, on the last block of a frame that declares one (has_fcs)
  uint32_t bsize;     // Block_Size (RLE block: the regenerated size; its content is one byte)
  uint32_t stream;    // owning stream (index into the call's stream arrays)
  uint32_t regen;     // regenerated size of the literals section
  uint32_t lit_hdr;   // literals section header bytes
  uint32_t lit_csize; // compressed size of Huffman literals (tree included)
  uint32_t nseq;
  uint32_t seq_off;   // offset, inside the block content, of the byte after Number_of_Sequences
  uint32_t out_size;  // regenerated size of the block (entropy pass; raw / RLE blocks: walk)
  int32_t huf_src;    // block holding the Huffman tree of these literals (itself for ltype 2), -1 = none
  int32_t tab_src[3]; // block holding the LL / OF / ML table description (itself unless Repeat_Mode), -1 = none
  uint8_t type;       // 0 raw, 1 RLE, 2 compressed
  uint8_t first;      // first block of a frame: repeat offsets and the match window start here
  uint8_t ltype;      // 0 raw, 1 RLE, 2 Huffman with tree, 3 Huffman treeless
  uint8_t lstreams;   // 1 or 4
  uint8_t modes;      // Symbol_Compression_Modes byte (0 when nseq == 0)
  uint8_t last;       // last block of its frame
  uint8_t has_fcs;
  uint8_t pad;
};

struct StreamTotals {
  uint64_t nblk, nseq, lit;
};

// literals section header -> (type, streams, header bytes, regenerated size, compressed size); false = malformed
B2S_HD inline bool parse_literals_header(const uint8_t* src, uint64_t n, int* ltype, int* streams, uint32_t* hdr,
                                         uint32_t* regen, uint32_t* csize) {
  if (n < 1) return false;
  const int t = src[0] & 3, sf = (src[0] >> 2) & 3;
  *ltype = t;
  *streams = 1;
  *csize = 0;
  if (t < 2) {
    if (sf == 0 || sf == 2) {
      *hdr = 1;
      *regen = src[0] >> 3;
    } else if (sf == 1) {
      if (n < 2) return false;
      *hdr = 2;
      *regen = (src[0] >> 4) | ((uint32_t)src[1] << 4);
    } else {
      if (n < 3) return false;
      *hdr = 3;
      *regen = (src[0] >> 4) | ((uint32_t)src[1] << 4) | ((uint32_t)src[2] << 12);
    }
  } else if (sf < 2) {
    if (n < 3) return false;
    *hdr = 3;
    const uint32_t v = src[0] | (src[1] << 8) | ((uint32_t)src[2] << 16);
    *regen = (v >> 4) & 0x3ff;
    *csize = (v >> 14) & 0x3ff;
    *streams = sf == 0 ? 1 : 4;
  } else if (sf == 2) {
    if (n < 4) return false;
    *hdr = 4;
    const uint32_t v = src[0] | (src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24);
    *regen = (v >> 4) & 0x3fff;
    *csize = v >> 18;
    *streams = 4;
  } else {
    if (n < 5) return false;
    *hdr = 5;
    const uint64_t v = src[0] | (src[1] << 8) | ((uint64_t)src[2] << 16) | ((uint64_t)src[3] << 24) | ((uint64_t)src[4] << 32);
    *regen = (uint32_t)((v >> 4) & 0x3ffff);
    *csize = (uint32_t)(v >> 22);
    *streams = 4;
  }
  return *regen <= kBlockMax;
}

// Walks the frames and blocks of one stream.  out == nullptr: count only.  Otherwise writes BlockInfo records starting at
// out[0] (the caller passes the stream's slice); blk0 is the GLOBAL index of out[0] (provenance fields are global),
// lit_base / seq_base the stream's first workspace positions, src_abs the stream's offset from src_base.
// Returns 0 or a negative error; tot receives the stream's totals either way.
B2S_HD inline int walk_stream(const uint8_t* src, uint64_t n, BlockInfo* out, uint32_t blk0, uint32_t stream,
                              uint64_t src_abs, uint64_t lit_base, uint64_t seq_base, StreamTotals* tot) {
  uint64_t ip = 0;
  uint32_t k = 0;  // blocks so far
  uint64_t lit = 0, nsq = 0;
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
    if (fhd & 0x08) return kErrCorrupt;
    if (!single) {
      if (ip >= n) return kErrCorrupt;
      ip++;
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
    bool first = true;
    int32_t huf_src = -1, tab_src[3] = {-1, -1, -1};
    for (;;) {
      if (ip + 3 > n) return kErrCorrupt;
      const uint32_t bh = src[ip] | (src[ip + 1] << 8) | ((uint32_t)src[ip + 2] << 16);
      ip += 3;
      const int last = bh & 1, type = (bh >> 1) & 3;
      const uint32_t bsize = bh >> 3;
      if (type == 3 || bsize > kBlockMax) return kErrCorrupt;
      BlockInfo b;
      b.src = src_abs + ip;
      b.lit_base = lit_base + lit;
      b.seq_base = seq_base + nsq;
      b.bsize = bsize;
      b.stream = stream;
      b.regen = b.lit_hdr = b.lit_csize = b.nseq = b.seq_off = 0;
      b.out_size = bsize;
      b.huf_src = -1;
      b.tab_src[0] = b.tab_src[1] = b.tab_src[2] = -1;
      b.type = (uint8_t)type;
      b.first = first ? 1 : 0;
      b.ltype = 0;
      b.lstreams = 1;
      b.modes = 0;
      b.last = (uint8_t)last;
      b.has_fcs = (last && fcs_bytes) ? 1 : 0;
      b.fcs = fcs;
      b.pad = 0;
      if (type == 0) {
        if (bsize > n - ip) return kErrCorrupt;
        ip += bsize;
      } else if (type == 1) {
        if (ip >= n) return kErrCorrupt;
        ip += 1;
      } else {
        if (bsize > n - ip) return kErrCorrupt;
        const uint8_t* c = src + ip;
        int ltype, streams;
        uint32_t hdr, regen, csize;
        if (!parse_literals_header(c, bsize, &ltype, &streams, &hdr, &regen, &csize)) return kErrCorrupt;
        uint64_t q = hdr;
        if (ltype == 0) q += regen;
        else if (ltype == 1) q += 1;
        else q += csize;
        if (q >= bsize) return kErrCorrupt;  // at least the Number_of_Sequences byte follows
        uint32_t nseq = c[q++];
        if (nseq >= 128) {
          if (nseq == 255) {
            if (q + 2 > bsize) return kErrCorrupt;
            nseq = c[q] + (c[q + 1] << 8) + 0x7F00;
            q += 2;
          } else {
            if (q + 1 > bsize) return kErrCorrupt;
            nseq = ((nseq - 128) << 8) + c[q];
            q += 1;
          }
        }
        b.out_size = 0;
        b.regen = regen;
        b.lit_hdr = hdr;
        b.lit_csize = csize;
        b.ltype = (uint8_t)ltype;
        b.lstreams = (uint8_t)streams;
        b.nseq = nseq;
        b.seq_off = (uint32_t)q;
        if (ltype == 2) huf_src = (int32_t)(blk0 + k);
        if (ltype >= 2) {
          if (huf_src < 0) return kErrCorrupt;  // treeless literals without an earlier tree
          b.huf_src = huf_src;
        }
        if (nseq) {
          if (q >= bsize) return kErrCorrupt;
          const int modes = c[q];
          if (modes & 3) return kErrCorrupt;
          b.modes = (uint8_t)modes;
          for (int kind = 0; kind < 3; kind++) {
            const int mode = (modes >> (6 - 2 * kind)) & 3;
            if (mode != 3) tab_src[kind] = (int32_t)(blk0 + k);
            else if (tab_src[kind] < 0) return kErrCorrupt;  // Repeat_Mode without an earlier table
            b.tab_src[kind] = tab_src[kind];
          }
        }
        if (ltype != 0) lit += ((uint64_t)regen + 15) & ~(uint64_t)15;
        nsq += nseq;
        ip += bsize;
      }
      if (out) out[k] = b;
      k++;
      first = false;
      if (last) break;
    }
    if (checksum) {
      if (ip + 4 > n) return kErrCorrupt;
      ip += 4;
    }
  }
  tot->nblk = k;
  tot->nseq = nsq;
  tot->lit = lit;
  return 0;
}

// Positions `*p` on the description of table `kind` inside the sequences section that starts at s (the modes byte) and
// returns that table's mode; the descriptions before it are skipped (their lengths come from parsing them).
B2S_HD inline int seek_table_description(Workspace* w, const uint8_t* s, uint64_t n, int kind, uint64_t* p) {
  if (n < 1) return -1;
  const int modes = s[0];
  uint64_t ip = 1;
  for (int k = 0; k < kind; k++) {
    const int m = (modes >> (6 - 2 * k)) & 3;
    if (m == 1) {
      ip += 1;
    } else if (m == 2) {
      int l = 0, ns = 0;
      if (ip > n) return -1;
      const uint64_t h = fse_read_header(s + ip, n - ip, w->norm, k == 0 ? 35 : 31, k == 0 ? 9 : 8, &l, &ns);
      if (!h) return -1;
      ip += h;
    }
  }
  if (ip > n) return -1;
  *p = ip;
  return (modes >> (6 - 2 * kind)) & 3;
}

// Entropy stage of one compressed block (cooperative on the device: every lane runs it, see zstd_core.h).
// Decodes the literals to lit_ws + lit_base (unless raw) and the sequences to ll/ml/ofv[seq_base ..), returns the
// block's regenerated size or a negative error.  size_only: nothing is stored.
B2S_HD inline int64_t entropy_block(Workspace* w, const BlockInfo* blocks, uint32_t bi, const uint8_t* src_base,
                                    uint8_t* lit_ws, uint32_t* sq_ll, uint32_t* sq_ml, uint32_t* sq_ofv,
                                    bool size_only) {
  const BlockInfo b = blocks[bi];
  if (b.type != 2) return (int64_t)b.bsize;
  const uint8_t* c = src_base + b.src;
  const uint64_t n = b.bsize;
  // ---- literals
  if (!size_only && b.ltype != 0) {
    uint8_t* lit = lit_ws + b.lit_base;
    if (b.ltype == 1) {
      const uint8_t v = c[b.lit_hdr];
      for (uint32_t i = B2S_LANE; i < b.regen; i += B2S_NLANES) lit[i] = v;
      B2S_SYNC();
    } else {
      const BlockInfo hb = blocks[b.huf_src];
      const uint8_t* hs = src_base + hb.src + hb.lit_hdr;  // the defining block's literals start with the tree
      const uint64_t t = huf_read_tree(w, hs, hb.lit_csize);
      if (!t) return kErrCorrupt;
      const uint8_t* ls = c + b.lit_hdr;
      uint64_t ln = b.lit_csize;
      if (b.ltype == 2) {
        ls += t;
        ln -= t;
      }
      if (b.lstreams == 1) {
        bool ok1 = true;
        if (B2S_LANE == 0) ok1 = huf_decode_stream(w, ls, ln, lit, b.regen);
        B2S_SYNC();
        if (!B2S_ALL(ok1)) return kErrCorrupt;
      } else {
        if (ln < 6) return kErrCorrupt;
        const uint64_t s1 = ls[0] | (ls[1] << 8), s2 = ls[2] | (ls[3] << 8), s3 = ls[4] | (ls[5] << 8);
        if (6 + s1 + s2 + s3 > ln) return kErrCorrupt;
        const uint64_t s4 = ln - 6 - s1 - s2 - s3;
        const uint64_t q = ((uint64_t)b.regen + 3) / 4;
        if (3 * q > b.regen) return kErrCorrupt;
        const uint8_t* a = ls + 6;
#if defined(B2S_ZSTD_WARP) && defined(__CUDA_ARCH__)
        {
          bool ok = true;
          const int l = B2S_LANE;
          if (l == 0) ok = huf_decode_stream(w, a, s1, lit, q);
          else if (l == 1) ok = huf_decode_stream(w, a + s1, s2, lit + q, q);
          else if (l == 2) ok = huf_decode_stream(w, a + s1 + s2, s3, lit + 2 * q, q);
          else if (l == 3) ok = huf_decode_stream(w, a + s1 + s2 + s3, s4, lit + 3 * q, b.regen - 3 * q);
          B2S_SYNC();
          if (!B2S_ALL(ok)) return kErrCorrupt;
        }
#else
        if (!huf_decode_stream(w, a, s1, lit, q)) return kErrCorrupt;
        if (!huf_decode_stream(w, a + s1, s2, lit + q, q)) return kErrCorrupt;
        if (!huf_decode_stream(w, a + s1 + s2, s3, lit + 2 * q, q)) return kErrCorrupt;
        if (!huf_decode_stream(w, a + s1 + s2 + s3, s4, lit + 3 * q, b.regen - 3 * q)) return kErrCorrupt;
#endif
      }
    }
  }
  // ---- sequences
  uint32_t produced = 0, lpos = 0;  // both <= kBlockMax
  if (b.nseq) {
    uint64_t ip = (uint64_t)b.seq_off + 1;  // past the modes byte
    for (int kind = 0; kind < 3; kind++) {
      const int mode = (b.modes >> (6 - 2 * kind)) & 3;
      if (mode == 3) {  // Repeat_Mode: rebuild from the block that defined the table
        const BlockInfo pb = blocks[b.tab_src[kind]];
        const uint8_t* ps = src_base + pb.src + pb.seq_off;
        uint64_t at = 0;
        const int pm = seek_table_description(w, ps, pb.bsize - pb.seq_off, kind, &at);
        if (pm < 0 || pm == 3) return kErrCorrupt;
        if (seq_setup_table(w, kind, pm, ps + at, pb.bsize - pb.seq_off - at) < 0) return kErrCorrupt;
      } else {
        if (ip > n) return kErrCorrupt;
        const int64_t used = seq_setup_table(w, kind, mode, c + ip, n - ip);
        if (used < 0) return kErrCorrupt;
        ip += (uint64_t)used;
      }
    }
    BitsRev br;
    if (ip >= n || !br.init(c + ip, n - ip)) return kErrCorrupt;
    uint32_t sl = br.read(w->ll_log), so = br.read(w->of_log), sm = br.read(w->ml_log);
    uint32_t my_ll = 0, my_ml = 0, my_ofv = 0;
    int nb = 0;
    // one 32-bit load per table entry (sym | nbits << 8 | base << 16): the entry feeds both the symbol and, at the end of
    // the iteration, the state update — through a generic pointer the compiler would otherwise re-read it field by field
    const uint32_t* tll = reinterpret_cast<const uint32_t*>(w->ll);
    const uint32_t* tof = reinterpret_cast<const uint32_t*>(w->of);
    const uint32_t* tml = reinterpret_cast<const uint32_t*>(w->ml);
    for (uint32_t i = 0; i < b.nseq; i++) {
      const uint32_t eo = tof[so], em = tml[sm], el = tll[sl];
      const int oc = (int)(eo & 0xffu), mc = (int)(em & 0xffu), lc = (int)(el & 0xffu);
      if (oc > 31 || mc > 52 || lc > 35) return kErrCorrupt;
      uint32_t mlb, llb;
      int mle, lle;
      ml_code(mc, &mlb, &mle);
      ll_code(lc, &llb, &lle);
      const uint32_t ofv = (oc ? (1u << oc) : 1u) + br.read(oc);
      const uint32_t mlen = mlb + br.read(mle);
      const uint32_t llen = llb + br.read(lle);
      if (lpos + llen > b.regen) return kErrCorrupt;
      if (produced + llen + mlen > kBlockMax) return kErrCorrupt;
      lpos += llen;
      produced += llen + mlen;
      if (!size_only) {  // lane (i mod NLANES) latches the triple; stored NLANES at a time (coalesced on the device)
        if (B2S_LANE == nb) {
          my_ll = llen;
          my_ml = mlen;
          my_ofv = ofv;
        }
        nb++;
        if (nb == B2S_NLANES || i + 1 == b.nseq) {
          if (B2S_LANE < nb) {
            const uint64_t at = b.seq_base + (i + 1 - (uint32_t)nb) + (uint32_t)B2S_LANE;
            sq_ll[at] = my_ll;
            sq_ml[at] = my_ml;
            sq_ofv[at] = my_ofv;
          }
          nb = 0;
        }
      }
      if (i + 1 < b.nseq) {  // state updates: literal length, match length, offset
        sl = (el >> 16) + br.read((int)((el >> 8) & 0xffu));
        sm = (em >> 16) + br.read((int)((em >> 8) & 0xffu));
        so = (eo >> 16) + br.read((int)((eo >> 8) & 0xffu));
      }
    }
    if (br.pos != 0) return kErrCorrupt;
  }
  const uint32_t total = produced + (b.regen - lpos);
  if (total > kBlockMax) return kErrCorrupt;
  return (int64_t)total;
}

// Decoded size of a stream from its blocks' sizes (after the entropy stage); checks every declared Frame_Content_Size.
B2S_HD inline int64_t stream_size(const BlockInfo* blocks, uint64_t nb) {
  uint64_t sum = 0, frame = 0;
  for (uint64_t k = 0; k < nb; k++) {
    frame += blocks[k].out_size;
    if (blocks[k].last) {
      if (blocks[k].has_fcs && frame != blocks[k].fcs) return kErrCorrupt;
      sum += frame;
      frame = 0;
    }
  }
  return (int64_t)(sum + frame);
}

// one step of the repeat-offset state machine (RFC 8878 3.1.1.5); returns the resolved offset (0 = corrupt)
B2S_HD inline uint32_t resolve_offset(uint32_t ofv, bool ll0, uint32_t* r0, uint32_t* r1, uint32_t* r2) {
  uint32_t offset;
  if (ofv > 3) {
    offset = ofv - 3;
    *r2 = *r1;
    *r1 = *r0;
    *r0 = offset;
  } else {
    uint32_t idx = ofv - 1;
    if (ll0) idx++;
    if (idx == 0) {
      offset = *r0;
    } else {
      offset = idx == 1 ? *r1 : idx == 2 ? *r2 : *r0 - 1;
      if (idx > 1) *r2 = *r1;
      *r1 = *r0;
      *r0 = offset;
    }
  }
  return offset;
}

// Execute stage of one stream: blocks[0..nb) in order into dst[0..cap).  Returns the decoded size or a negative error.
B2S_HD inline int64_t execute_stream(const BlockInfo* blocks, uint32_t nb, const uint8_t* src_base, const uint8_t* lit_ws,
                                     const uint32_t* sq_ll, const uint32_t* sq_ml, const uint32_t* sq_ofv, uint8_t* dst,
                                     uint64_t cap) {
  uint64_t total = 0, frame_start = 0;
  uint32_t r0 = 1, r1 = 4, r2 = 8;
  for (uint32_t k = 0; k < nb; k++) {
    const BlockInfo b = blocks[k];
    if (b.first) {
      frame_start = total;
      r0 = 1;
      r1 = 4;
      r2 = 8;
    }
    if (total + b.out_size > cap) return kErrDstTooSmall;
    uint8_t* ob = dst + total;  // block base: positions inside a block fit an int
    const uint8_t* c = src_base + b.src;
    if (b.type == 0) {
      for (uint32_t i = B2S_LANE; i < b.bsize; i += B2S_NLANES) ob[i] = c[i];
      B2S_SYNC();
    } else if (b.type == 1) {
      const uint8_t v = c[0];
      for (uint32_t i = B2S_LANE; i < b.bsize; i += B2S_NLANES) ob[i] = v;
      B2S_SYNC();
    } else {
      const uint8_t* lit = b.ltype == 0 ? c + b.lit_hdr : lit_ws + b.lit_base;
      const uint64_t back = total - frame_start;  // bytes of this frame before the block: the match window
      uint32_t produced = 0, lpos = 0;
#if defined(B2S_ZSTD_WARP) && defined(__CUDA_ARCH__)
      constexpr unsigned FULL = 0xffffffffu;
      const int lane = B2S_LANE;
      // the next batch's triples are loaded while this one executes (a lone warp has nothing else to hide DRAM behind)
      uint32_t n_ll = 0, n_ml = 0, n_ofv = 4;  // idle lanes: an empty sequence with a fresh (harmless) offset
      if ((uint32_t)lane < b.nseq) {
        n_ll = sq_ll[b.seq_base + lane];
        n_ml = sq_ml[b.seq_base + lane];
        n_ofv = sq_ofv[b.seq_base + lane];
      }
      for (uint32_t i0 = 0; i0 < b.nseq; i0 += 32) {
        const int cnt = (int)(b.nseq - i0 < 32u ? b.nseq - i0 : 32u);
        const uint32_t ll = n_ll, ml = n_ml, ofv = n_ofv;
        n_ll = 0;
        n_ml = 0;
        n_ofv = 4;
        if (i0 + 32 + lane < b.nseq) {
          n_ll = sq_ll[b.seq_base + i0 + 32 + lane];
          n_ml = sq_ml[b.seq_base + i0 + 32 + lane];
          n_ofv = sq_ofv[b.seq_base + i0 + 32 + lane];
        }
        // repeat offsets: sequences before the first repeat code resolve independently; from there on, in order
        const unsigned repmask = __ballot_sync(FULL, lane < cnt && ofv <= 3u);
        const int f = repmask ? __ffs(repmask) - 1 : cnt;
        uint32_t off = ofv - 3u;
        if (f >= 1) {  // reps after the prefix [0, f): its last three offsets, older ones shift out
          const uint32_t a = __shfl_sync(FULL, off, f - 1), bb = __shfl_sync(FULL, off, f >= 2 ? f - 2 : 0),
                         cc = __shfl_sync(FULL, off, f >= 3 ? f - 3 : 0);
          if (f >= 3) { r2 = cc; r1 = bb; r0 = a; }
          else if (f == 2) { r2 = r0; r1 = bb; r0 = a; }
          else { r2 = r1; r1 = r0; r0 = a; }
        }
        for (int j = f; j < cnt; j++) {
          const uint32_t v = __shfl_sync(FULL, ofv, j);
          const uint32_t l = __shfl_sync(FULL, ll, j);
          const uint32_t o = resolve_offset(v, l == 0, &r0, &r1, &r2);
          if (lane == j) off = o;
        }
        // positions: exclusive scans of ll + ml (output) and ll (literals)
        uint32_t inc = ll + ml, linc = ll;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
          const uint32_t t = __shfl_up_sync(FULL, inc, s), u = __shfl_up_sync(FULL, linc, s);
          if (lane >= s) {
            inc += t;
            linc += u;
          }
        }
        const uint32_t o = produced + inc - (ll + ml), lp = lpos + linc - ll;
        const uint32_t sum = __shfl_sync(FULL, inc, 31), lsum = __shfl_sync(FULL, linc, 31);
        bool bad = lane < cnt && (off == 0 || (uint64_t)off > back + o + ll);
        if (lpos + lsum > b.regen || produced + sum > b.out_size) bad = true;
        if (__any_sync(FULL, bad)) return kErrCorrupt;
        if (ll <= 32) {  // loads first, then stores: one memory round trip per 8 bytes instead of one per byte
          for (uint32_t q0 = 0; q0 < ll; q0 += 8) {
            uint8_t t[8];
#pragma unroll
            for (int u = 0; u < 8; u++)
              if (q0 + u < ll) t[u] = lit[lp + q0 + u];
#pragma unroll
            for (int u = 0; u < 8; u++)
              if (q0 + u < ll) ob[o + q0 + u] = t[u];
          }
        }
        unsigned big = __ballot_sync(FULL, ll > 32);
        while (big) {
          const int l = __ffs(big) - 1;
          big &= big - 1;
          const uint32_t n_l = __shfl_sync(FULL, ll, l), o_l = __shfl_sync(FULL, o, l), p_l = __shfl_sync(FULL, lp, l);
          for (uint32_t q = lane; q < n_l; q += 32) ob[o_l + q] = lit[p_l + q];
        }
        __syncwarp();
        lz_execute_matches<false>(ob, (int)(o + ll), (int)ml, (int)off, lane);
        produced += sum;
        lpos += lsum;
      }
#else
      for (uint32_t i = 0; i < b.nseq; i++) {
        const uint32_t ll = sq_ll[b.seq_base + i], ml = sq_ml[b.seq_base + i];
        const uint32_t off = resolve_offset(sq_ofv[b.seq_base + i], ll == 0, &r0, &r1, &r2);
        if (off == 0 || (uint64_t)off > back + produced + ll) return kErrCorrupt;
        if (lpos + ll > b.regen || produced + ll + ml > b.out_size) return kErrCorrupt;
        for (uint32_t q = 0; q < ll; q++) ob[produced + q] = lit[lpos + q];
        uint8_t* d = ob + produced + ll;
        const uint8_t* s = d - off;
        for (uint32_t q = 0; q < ml; q++) d[q] = s[q];
        produced += ll + ml;
        lpos += ll;
      }
#endif
      const uint32_t tail = b.regen - lpos;
      if (produced + tail != b.out_size) return kErrCorrupt;
      for (uint32_t q = B2S_LANE; q < tail; q += B2S_NLANES) ob[produced + q] = lit[lpos + q];
      B2S_SYNC();
    }
    total += b.out_size;
    if (b.has_fcs && total - frame_start != b.fcs) return kErrCorrupt;
  }
  return (int64_t)total;
}

}  // namespace zstd
}  // namespace b2s
