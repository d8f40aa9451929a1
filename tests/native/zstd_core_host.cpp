// Host build of spark-s3-shuffle_b200/csrc/zstd_core.h for tests/test_zstd_core.py: the very functions the CUDA
// kernels of zstd.cu call, compiled by g++ so they can be checked against libzstd.so.1 without a GPU.
// Test infrastructure only — the C ABI never runs this.
#include <stdlib.h>

#include "../../spark-s3-shuffle_b200/csrc/zstd_core.h"

extern "C" {
long long zc_decode(const unsigned char* src, unsigned long long n, unsigned char* dst, unsigned long long cap) {
  b2s::zstd::Workspace* w = (b2s::zstd::Workspace*)malloc(sizeof(b2s::zstd::Workspace));
  w->lit = (unsigned char*)malloc(b2s::zstd::kBlockMax + 64);
  long long r = b2s::zstd::decode_stream(w, src, n, dst, cap, false);
  free(w->lit);
  free(w);
  return r;
}
long long zc_size(const unsigned char* src, unsigned long long n) {
  b2s::zstd::Workspace* w = (b2s::zstd::Workspace*)malloc(sizeof(b2s::zstd::Workspace));
  w->lit = (unsigned char*)malloc(b2s::zstd::kBlockMax + 64);
  long long r = b2s::zstd::decode_stream(w, src, n, nullptr, 0, true);
  free(w->lit);
  free(w);
  return r;
}
unsigned long long zc_workspace_bytes() { return sizeof(b2s::zstd::Workspace); }
}

// the block-parallel decomposition (zstd_par.h): walk (count, fill) -> entropy per block -> execute, run one after the
// other exactly as the three kernels of zstd.cu do
#include <vector>

#include "../../spark-s3-shuffle_b200/csrc/zstd_par.h"
extern "C" long long zc_decode_par(const unsigned char* src, unsigned long long n, unsigned char* dst,
                                   unsigned long long cap, int size_only) {
  using namespace b2s::zstd;
  StreamTotals t{0, 0, 0};
  int rc = walk_stream(src, n, nullptr, 0, 0, 0, 0, 0, &t);
  if (rc < 0) return rc;
  std::vector<BlockInfo> blocks(t.nblk ? t.nblk : 1);
  StreamTotals t2{0, 0, 0};
  rc = walk_stream(src, n, blocks.data(), 0, 0, 0, 0, 0, &t2);
  if (rc < 0 || t2.nblk != t.nblk || t2.nseq != t.nseq || t2.lit != t.lit) return -100;
  std::vector<unsigned char> lit(t.lit + 64);
  std::vector<uint32_t> ll(t.nseq + 1), ml(t.nseq + 1), ofv(t.nseq + 1);
  Workspace* w = (Workspace*)malloc(sizeof(Workspace));
  w->lit = nullptr;
  long long total = 0;
  for (uint32_t b = 0; b < t.nblk; b++) {
    const long long r = entropy_block(w, blocks.data(), b, src, lit.data(), ll.data(), ml.data(), ofv.data(), size_only != 0);
    if (r < 0) {
      free(w);
      return r;
    }
    blocks[b].out_size = (uint32_t)r;
    total += r;
  }
  free(w);
  if (size_only) return stream_size(blocks.data(), t.nblk);
  return execute_stream(blocks.data(), (uint32_t)t.nblk, src, lit.data(), ll.data(), ml.data(), ofv.data(), dst, cap);
}

// Coverage probes: what a frame really contains, read with the same walk and entropy stages.
// zc_frame_sequences: every sequence of every block as (literal length, match length, offset VALUE) — repeat codes stay
// 1..3, new offsets are offset + 3.  Returns the sequence count (cap too small: the count, nothing beyond cap written)
// or a negative error.
extern "C" long long zc_frame_sequences(const unsigned char* src, unsigned long long n, unsigned* ll_out,
                                        unsigned* ml_out, unsigned* ofv_out, unsigned long long cap) {
  using namespace b2s::zstd;
  StreamTotals t{0, 0, 0};
  int rc = walk_stream(src, n, nullptr, 0, 0, 0, 0, 0, &t);
  if (rc < 0) return rc;
  std::vector<BlockInfo> blocks(t.nblk ? t.nblk : 1);
  rc = walk_stream(src, n, blocks.data(), 0, 0, 0, 0, 0, &t);
  if (rc < 0) return rc;
  std::vector<unsigned char> lit(t.lit + 64);
  std::vector<uint32_t> ll(t.nseq + 1), ml(t.nseq + 1), ofv(t.nseq + 1);
  Workspace* w = (Workspace*)malloc(sizeof(Workspace));
  w->lit = nullptr;
  for (uint32_t b = 0; b < t.nblk; b++) {
    const long long r = entropy_block(w, blocks.data(), b, src, lit.data(), ll.data(), ml.data(), ofv.data(), false);
    if (r < 0) {
      free(w);
      return r;
    }
  }
  free(w);
  for (uint64_t i = 0; i < t.nseq && i < cap; i++) {
    ll_out[i] = ll[i];
    ml_out[i] = ml[i];
    ofv_out[i] = ofv[i];
  }
  return (long long)t.nseq;
}

// zc_frame_blocks: six ints per block — block type (0 raw, 1 RLE, 2 compressed), literals type (0 raw, 1 RLE,
// 2 Huffman, 3 treeless), Huffman stream count (1 / 4), the Symbol_Compression_Modes byte, the Huffman weights' form
// (1 FSE-compressed, 0 direct, -1 no tree in this block) and the sequence count.  Returns the block count (at most cap
// blocks written) or a negative error.
extern "C" long long zc_frame_blocks(const unsigned char* src, unsigned long long n, int* out, unsigned long long cap) {
  using namespace b2s::zstd;
  StreamTotals t{0, 0, 0};
  int rc = walk_stream(src, n, nullptr, 0, 0, 0, 0, 0, &t);
  if (rc < 0) return rc;
  std::vector<BlockInfo> blocks(t.nblk ? t.nblk : 1);
  rc = walk_stream(src, n, blocks.data(), 0, 0, 0, 0, 0, &t);
  if (rc < 0) return rc;
  for (uint64_t k = 0; k < t.nblk && k < cap; k++) {
    const BlockInfo& b = blocks[k];
    int* o = out + 6 * k;
    o[0] = b.type;
    o[1] = b.type == 2 ? b.ltype : -1;
    o[2] = b.type == 2 ? b.lstreams : 0;
    o[3] = b.modes;
    o[4] = (b.type == 2 && b.ltype == 2) ? (src[b.src + b.lit_hdr] < 128 ? 1 : 0) : -1;  // Huffman header byte
    o[5] = (int)b.nseq;
  }
  return (long long)t.nblk;
}

// ------------------------------------------------------------------------------------------------------------------
// CPU model of the GPU Zstandard ENCODER (zstd_enc.cu): the shared window match finder + greedy parse (the same
// specification as orc_lz4_compress_block_win in oracle/), then the encoder core of zstd_enc_core.h.
// ------------------------------------------------------------------------------------------------------------------
#include <string.h>

#include <vector>

#include "../../spark-s3-shuffle_b200/csrc/zstd_enc_core.h"

namespace {
inline uint32_t rd32(const uint8_t* p) {
  uint32_t v;
  memcpy(&v, p, 4);
  return v;
}
// phase A of the GPU compressor: fixed windows of 32 positions, table state before the window, offset-1 for byte runs
void win_find_offsets(const uint8_t* src, int n, int hash_log, std::vector<uint16_t>& off) {
  std::vector<uint16_t> table((size_t)1 << hash_log, 0);
  const int mflimit = n - 12;
  for (int pos = 0; pos <= mflimit; pos += 32) {
    const int last = pos + 31 < mflimit ? pos + 31 : mflimit;
    for (int p = pos; p <= last; p++) {
      const uint32_t v = rd32(src + p);
      const int c = table[(v * 2654435761u) >> (32 - hash_log)];
      if (p > 0 && rd32(src + p - 1) == v) off[p] = 1;
      else if (c < p && rd32(src + c) == v) off[p] = (uint16_t)(p - c);
    }
    for (int p = pos; p <= last; p++) table[(rd32(src + p) * 2654435761u) >> (32 - hash_log)] = (uint16_t)p;
  }
}
}  // namespace

extern "C" long long zc_compress_model_hlog(const unsigned char* src, unsigned long long n, unsigned block_size,
                                            unsigned char* dst, unsigned long long cap, int hash_log);
extern "C" long long zc_compress_model(const unsigned char* src, unsigned long long n, unsigned block_size,
                                       unsigned char* dst, unsigned long long cap) {
  return zc_compress_model_hlog(src, n, block_size, dst, cap, 12);
}
static int g_model_subchunk = 0;  // 1: the sub-chunk parallel parse of B2S_LZ4_PIPE=4
extern "C" void zc_model_subchunk(int on) { g_model_subchunk = on; }
// hash_log: 12 = unspecified level / level 2; level 1 -> 11, level >= 3 -> 13 (hlog_for_level in csrc/api.cu)
extern "C" long long zc_compress_model_hlog(const unsigned char* src, unsigned long long n, unsigned block_size,
                                            unsigned char* dst, unsigned long long cap, int hash_log) {
  using namespace b2s::zstdenc;
  static CTables T;
  static bool built = false;
  if (!built) {
    build_predefined(&T);
    built = true;
  }
  unsigned long long op = 0;
  if (cap < kFrameHeaderBytes + kEndBlockBytes) return -3;
  put_frame_header(dst);
  op = kFrameHeaderBytes;
  std::vector<uint8_t> lits, bits;
  for (unsigned long long b0 = 0; b0 < n; b0 += block_size) {
    const int bn = (int)(n - b0 < block_size ? n - b0 : block_size);
    const uint8_t* s = src + b0;
    std::vector<Seq> seqs;
    lits.clear();
    int anchor = 0;
    if (bn >= 13) {
      std::vector<uint16_t> off((size_t)bn, 0);
      win_find_offsets(s, bn, hash_log, off);
      const int mflimit = bn - 12, matchlimit = bn - 5;
      // the warp-parallel parse restarts in every sub-chunk of 1/32 block (rounded up to 32 positions); a match neither
      // starts in a sub-chunk's last three positions nor extends past its end (oracle: orc_lz4_compress_block_win_sub)
      const int stride = (int)((block_size + 31u) & ~31u);
      const int sub = g_model_subchunk ? ((stride >> 5) + 31) & ~31 : bn + 1;  // bn + 1: one cursor over the block
      int p = 0;
      while (p <= mflimit) {
        int chunk_hi = (p / sub + 1) * sub;
        if (chunk_hi > bn) chunk_hi = bn;
        const int plim = mflimit < chunk_hi - 4 ? mflimit : chunk_hi - 4;
        const int elim = matchlimit < chunk_hi ? matchlimit : chunk_hi;
        if (p > plim) {
          p = chunk_hi;
          continue;
        }
        if (!off[p]) {
          p++;
          continue;
        }
        const int c = p - off[p];
        int ml = 4;
        while (p + ml < elim && s[p + ml] == s[c + ml]) ml++;
        seqs.push_back(Seq{(uint32_t)(p - anchor), (uint32_t)ml, off[p]});
        lits.insert(lits.end(), s + anchor, s + p);
        p += ml;
        anchor = p;
      }
    }
    lits.insert(lits.end(), s + anchor, s + bn);
    // compressed block: raw literals + FSE sequences (own or predefined tables), when smaller than the raw block
    bool raw = seqs.empty();
    uint32_t csize = 0, nbits = 0, hb = 0;
    uint8_t hdr[kSeqHeaderMax];
    if (!raw) {
      bits.assign((size_t)bn + 16, 0);
      BlockTables B;
      nbits = encode_block_sequences(&T, &B, (uint32_t)seqs.size(), [&](uint32_t i) { return seqs[i]; }, hdr, &hb,
                                     bits.data(), (uint32_t)bn);
      csize = raw_literals_header_bytes((uint32_t)lits.size()) + (uint32_t)lits.size() + nseq_header_bytes((uint32_t)seqs.size()) + hb + nbits;
      if (nbits > (uint32_t)bn || csize >= (uint32_t)bn) raw = true;
    }
    const uint32_t payload = raw ? (uint32_t)bn : csize;
    if (op + 3 + payload + kEndBlockBytes > cap) return -3;
    put_block_header(dst + op, 0, raw ? 0 : 2, payload);
    op += 3;
    if (raw) {
      memcpy(dst + op, s, (size_t)bn);
    } else {
      uint8_t* q = dst + op;
      put_raw_literals_header(q, (uint32_t)lits.size());
      q += raw_literals_header_bytes((uint32_t)lits.size());
      memcpy(q, lits.data(), lits.size());
      q += lits.size();
      put_nseq(q, (uint32_t)seqs.size());
      q += nseq_header_bytes((uint32_t)seqs.size());
      memcpy(q, hdr, hb);  // Compression_Modes + the block's own table descriptions
      q += hb;
      memcpy(q, bits.data(), nbits);
    }
    op += payload;
  }
  put_block_header(dst + op, 1, 0, 0);  // empty Raw_Block with Last_Block
  op += kEndBlockBytes;
  return (long long)op;
}

// ---- the per-block FSE table helpers of zstd_enc_core.h, exposed for property tests ---------------------------------
extern "C" void zc_normalize(const uint16_t* cnt, int nsym, unsigned total, int log, int16_t* norm) {
  b2s::zstdenc::normalize_counts(cnt, nsym, total, log, norm);
}
// writes the description of norm[0..nsym) (norm[nsym] must be addressable: the sentinel) and reads it back with the
// DECODER's header reader; returns the description's bytes, or -1 when the round trip differs
extern "C" int zc_ncount_roundtrip(int16_t* norm, int nsym, int log, int max_sym, int max_log) {
  uint8_t buf[256];
  norm[nsym] = 1;
  const uint32_t n = b2s::zstdenc::write_ncount(buf, norm, log);
  int16_t back[64];
  for (int i = 0; i < 64; i++) back[i] = 0;
  int log2 = 0, nsym2 = 0;
  const uint64_t used = b2s::zstd::fse_read_header(buf, n, back, max_sym, max_log, &log2, &nsym2);
  if (used != n || log2 != log) return -1;
  for (int s = 0; s < nsym; s++)
    if ((s < nsym2 ? back[s] : 0) != norm[s]) return -1;
  return (int)n;
}
