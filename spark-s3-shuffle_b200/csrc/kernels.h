// kernels.h — internal launch interface between the C-ABI runtime (api.cu) and the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "common.cuh"

namespace b2s {

// ---------------- scan.cu ----------------
// in-place exclusive prefix sum over d_v[0..n); d_total (device, 1 element) receives the grand total.
// d_ws must hold scan_ws_elems(n) uint64.
size_t scan_ws_elems(size_t n);
// d_base (optional, device): offset added to every result and to the total; d_total may alias d_base, which chains
// the scans of consecutive chunks into one running prefix.
void launch_exclusive_scan_u64(uint64_t* d_v, size_t n, uint64_t* d_total, uint64_t* d_ws, cudaStream_t st,
                               uint64_t* launches, const uint64_t* d_base = nullptr);

// ---------------- checksum.cu (K1) ----------------
struct ChecksumTables {
  uint32_t* d_crc_rows[2];  // [crc32, crc32c] : 16 x 256 row-advance tables (Z_496..Z_511)
  uint32_t* d_crc_misc[2];  // x2n[32] | xinv2n[32] | lane_const[32] | poly
};
int checksum_tables_create(ChecksumTables* t);  // on the current device
void checksum_tables_destroy(ChecksumTables* t);
inline size_t checksum_ws_elems(size_t n) { return scan_ws_elems(n + 1) + 2 * n + 2; }
// slices i = [d_off[i], d_off[i]+d_len[i]) of base; d_out[i] = checksum (low 32 bits).  tile_shift: log2 bytes per
// warp work item (>= 9).  d_work_base[n+1] is scratch for the work-item prefix; d_ws >= checksum_ws_elems(n).
void launch_checksum(const ChecksumTables& t, uint32_t alg, const uint8_t* base, const uint64_t* d_off,
                     const uint64_t* d_len, uint32_t n, uint32_t tile_shift, uint64_t* d_work_base, uint64_t* d_ws,
                     uint64_t* d_out, cudaStream_t st, uint64_t* launches);
// verify: slice s of block owner[s] mismatching -> status[owner]=B2S_E_CHECKSUM, bad_slice[owner]=min(s-slice_base[owner])
void launch_checksum_compare(const uint64_t* d_got, const uint64_t* d_expected, const uint32_t* d_slice_owner,
                             const uint32_t* d_slice_base, uint32_t n_slices, int32_t* d_status, int32_t* d_bad_slice,
                             cudaStream_t st, uint64_t* launches);

// ---------------- xxh32.cu (K2) ----------------
void launch_xxh32_encode(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                         const uint32_t* d_blk_base, uint32_t n_streams, uint32_t n_blocks, uint32_t block_size,
                         uint32_t seed, uint32_t* d_hash, cudaStream_t st, uint64_t* launches);
void launch_xxh32_verify(const BlockDesc* d_desc, uint32_t n_blocks, const uint8_t* dst_base, uint32_t seed,
                         uint32_t mask, int32_t* d_status, cudaStream_t st, uint64_t* launches);

// ---------------- lz4_compress.cu (K3: match / parse / emit + write-side LZ4Block framing) ----------------
extern int g_lz4_hlog;
// bytes of workspace for one pass over `chunk_blocks` codec blocks (off u16 + ml8 u8 per position, 8-byte records)
size_t lz4_compress_ws_bytes(uint32_t chunk_blocks, uint32_t block_size, uint32_t codec);
// Codec blocks [b0, b0+m) of the batch, in two halves that may run on different streams (d_ws is handed from one to
// the other):  launch_lz4_match = phase A (per-position off/ml into d_ws; ev0/ev1 bracket the kernel);
// launch_lz4_parse_emit = parse -> scan(d_sizes[b0..b0+m), chained on *d_running_total) -> emit (+ 21-byte headers)
// straight into the blocks' packed positions in dst_base.  d_nseq/d_csize/d_hash/d_sizes are indexed by global block
// id; afterwards d_sizes[b] holds the packed offset (without the per-stream end marks) and d_csize[b] the payload
// bytes (bit 31 = stored RAW).
void launch_lz4_match(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                      const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
                      uint32_t codec, uint8_t* d_ws, unsigned int* d_counter, cudaStream_t st, uint64_t* launches,
                      cudaEvent_t ev0, cudaEvent_t ev1, int hlog = 0 /* 0 = B2S_LZ4_HLOG (12) */);
void launch_lz4_parse_emit(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                           const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m,
                           uint32_t block_size, uint32_t codec, uint8_t* d_ws, uint32_t* d_nseq, uint32_t* d_csize,
                           const uint32_t* d_hash, uint64_t* d_sizes, uint64_t* d_running_total, uint64_t* d_scan_ws,
                           uint8_t* dst_base, uint64_t dst_cap, cudaStream_t st, uint64_t* launches);
// per stream: dst_off/dst_len, end mark, B2S_E_DST_TOO_SMALL (d_scan = packed block offsets, d_scan_total = their sum)
void launch_lz4block_stream_meta(const uint32_t* d_blk_base, uint32_t n_streams, uint32_t n_blocks, uint32_t block_size,
                                 const uint64_t* d_scan, const uint64_t* d_scan_total, uint8_t* dst_base,
                                 uint64_t dst_cap, uint64_t* d_dst_off, uint64_t* d_dst_len, int32_t* d_status,
                                 cudaStream_t st, uint64_t* launches);

// ---------------- lz4_decode.cu (read-side LZ4Block framing + K4) ----------------
// header walk pass 1: per stream block count + decoded bytes; malformed -> status CORRUPT (streams already failed are skipped)
void launch_lz4block_count(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                           uint64_t* d_nblk, uint64_t* d_olen, int32_t* d_status, cudaStream_t st, uint64_t* launches);
// header walk pass 2: descriptors at d_blk_base[i]+k; streams that overflow dst_cap get status DST_TOO_SMALL + no-op descriptors
void launch_lz4block_fill(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                          const uint64_t* d_blk_base, const uint64_t* d_dst_off, uint64_t* d_olen, uint64_t dst_cap,
                          int32_t* d_status, BlockDesc* d_desc, cudaStream_t st, uint64_t* launches);
// LZ4 codec blocks [0, nb) in one launch, a warp per block (parse + copies; malformed blocks set status[stream] =
// B2S_E_CORRUPT).  d_counter: one device word of scratch.
void launch_lz4_decode_warp(const BlockDesc* d_desc, uint32_t nb, const uint8_t* src_base, uint8_t* dst_base,
                            int32_t* d_status, unsigned int* d_counter, cudaStream_t st, uint64_t* launches);

// ---------------- snappy.cu (K5: xerial framing, Snappy emit / tokens / copy; match and parse kernels are shared) ------
void launch_snappy_emit(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                        const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
                        uint32_t stride, uint32_t max_seq, const uint16_t* d_off, const uint2* d_seq,
                        const uint32_t* d_nseq, const uint32_t* d_csize, const uint64_t* d_scan, uint8_t* dst_base,
                        uint64_t dst_cap, cudaStream_t st, uint64_t* launches);
void launch_xerial_stream_meta(const uint32_t* d_blk_base, uint32_t n_streams, uint32_t n_blocks, const uint64_t* d_scan,
                               const uint64_t* d_scan_total, uint8_t* dst_base, uint64_t dst_cap, uint64_t* d_dst_off,
                               uint64_t* d_dst_len, int32_t* d_status, cudaStream_t st, uint64_t* launches);
// d_maxima[0..1] (pre-zeroed) receive the largest uncompressed / compressed length of any chunk of the batch (the
// decoder takes chunks up to 64 KiB and sizes its records by the largest)
void launch_xerial_count(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                         uint64_t* d_nblk, uint64_t* d_olen, uint64_t* d_maxima, int32_t* d_status, cudaStream_t st,
                         uint64_t* launches);
void launch_xerial_fill(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                        const uint64_t* d_blk_base, const uint64_t* d_dst_off, uint64_t* d_olen, uint64_t dst_cap,
                        int32_t* d_status, BlockDesc* d_desc, cudaStream_t st, uint64_t* launches);
void launch_snappy_tokens(const BlockDesc* d_desc, uint32_t b0, uint32_t m, const uint8_t* src_base, uint2* d_rec,
                          uint32_t rec_stride, uint32_t* d_nrec, int32_t* d_status, cudaStream_t st,
                          uint64_t* launches);
// Snappy record workspace: records per codec block, and bytes for chunk_blocks codec blocks
uint32_t snappy_decode_rec_stride(uint32_t max_clen);
size_t snappy_decode_ws_bytes(uint32_t chunk_blocks, uint32_t rec_stride);
// codec blocks [b0, b0+m): the byte copies from the per-sequence records of launch_snappy_tokens in d_ws (d_nrec is
// indexed by global block id).  A separate launch so that the token walk of chunk k+1 can run beside the copies of
// chunk k.
void launch_snappy_copy(const BlockDesc* d_desc, uint32_t b0, uint32_t m, uint32_t rec_stride, const uint8_t* src_base,
                        uint8_t* dst_base, const uint8_t* d_ws, const uint32_t* d_nrec, cudaStream_t st,
                        uint64_t* launches);

// ---------------- zstd.cu (K6: Zstandard frame decoding, block-parallel; core in zstd_core.h + zstd_par.h) ----------------
// d_cnt / d_base: three arrays of n u64 each (blocks, sequences, literal-workspace bytes per stream); d_base holds their
// exclusive scans.  d_blocks: zstd_block_info_bytes() per block.  d_ws: zstd_ws_bytes(total literals, total sequences).
size_t zstd_block_info_bytes();
size_t zstd_ws_bytes(uint64_t lit_bytes, uint64_t nseq);
void launch_zstd_count(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                       uint64_t* d_cnt, int32_t* d_status, cudaStream_t st, uint64_t* launches);
void launch_zstd_fill(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len, uint32_t n,
                      uint64_t* d_cnt, const uint64_t* d_base, void* d_blocks, int32_t* d_status, cudaStream_t st,
                      uint64_t* launches);
// warp per block: literals + sequences into d_ws (size_only: nothing stored), block sizes into d_blocks
void launch_zstd_entropy(bool size_only, const uint8_t* src_base, void* d_blocks, uint64_t nb, uint8_t* d_ws,
                         uint64_t lit_bytes, uint64_t nseq, int32_t* d_status, cudaStream_t st, uint64_t* launches);
void launch_zstd_sum(const void* d_blocks, const uint64_t* d_cnt, const uint64_t* d_base, uint32_t n, uint64_t* d_olen,
                     int32_t* d_status, cudaStream_t st, uint64_t* launches);
// warp per stream: decodes stream i to dst_base + d_dst_off[i] (d_olen[i] bytes, as computed by launch_zstd_sum)
void launch_zstd_execute(const uint8_t* src_base, const void* d_blocks, const uint64_t* d_cnt, const uint64_t* d_base,
                         uint32_t n, const uint8_t* d_ws, uint64_t lit_bytes, uint64_t nseq, const uint64_t* d_olen,
                         uint8_t* dst_base, const uint64_t* d_dst_off, uint64_t dst_cap, int32_t* d_status,
                         cudaStream_t st, uint64_t* launches);

// ---------------- zstd_enc.cu (K7: Zstandard frame encoding: raw literals + predefined-FSE sequences) ----------------
int zstd_ctables_create(void** d_tables);  // predefined FSE compression tables, on the current device
void zstd_ctables_destroy(void* d_tables);
void zstd_set_ctables(int ordinal, const void* d_tables);
// per-block scratch of the Zstandard entropy stage: 192 bytes of sequence-section header (modes + table descriptions,
// zstdenc::kSeqHeaderMax) + one byte per position + 32 for the bitstream
inline size_t zstd_bits_stride(size_t stride) { return stride + 32 + 192; }
void launch_zstd_seqenc(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                        const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
                        uint32_t stride, uint32_t max_seq, const uint16_t* d_off, const uint2* d_seq,
                        const uint32_t* d_nseq, uint8_t* d_bits, uint32_t* d_nbits, uint32_t* d_csize,
                        uint64_t* d_sizes, cudaStream_t st, uint64_t* launches);
void launch_zstd_emit(const uint8_t* src_base, const uint64_t* d_src_off, const uint64_t* d_src_len,
                      const uint32_t* d_blk_base, uint32_t n_streams, uint32_t b0, uint32_t m, uint32_t block_size,
                      uint32_t stride, uint32_t max_seq, const uint2* d_seq, const uint32_t* d_nseq,
                      const uint8_t* d_bits, const uint32_t* d_nbits, const uint32_t* d_csize, const uint64_t* d_scan,
                      uint8_t* dst_base, uint64_t dst_cap, cudaStream_t st, uint64_t* launches);
void launch_zstd_stream_meta(const uint32_t* d_blk_base, uint32_t n_streams, uint32_t n_blocks, const uint64_t* d_scan,
                             const uint64_t* d_scan_total, uint8_t* dst_base, uint64_t dst_cap, uint64_t* d_dst_off,
                             uint64_t* d_dst_len, int32_t* d_status, cudaStream_t st, uint64_t* launches);

// ---------------- partition.cu (stable partition of serialized records by reduce id) ----------------
// Record i is rec_base[src_off[i] .. + rec_len[i]) with id rec_part[i]; n < 2^32.  After launch_partition the records
// of partition p, in input order, belong at part_start[p] .. (the arena offsets of the records in sorted order are in
// sdst; idx = sorted record indices, nullptr = identity).  readback = [first record with an id >= num_partitions
// (~0 = none), sum of rec_len, part_start[num_partitions] (~0 = no records)], readback_bytes long.
struct PartitionPlan {
  uint64_t* src_off = nullptr;
  uint64_t* sdst = nullptr;
  const uint32_t* idx = nullptr;
  uint64_t* readback = nullptr;
  size_t readback_bytes = 0;
};
// One stable LSD radix pass over n (key, record index) pairs (n < 2^32), digit (key >> shift) & (nd - 1), nd a power of
// two <= 256: a per-tile histogram, one scan over the digit-major histogram, a stable scatter.  idx_in == nullptr: the
// index is the position.  hist: radix_hist_elems(n) u64, hist_total: one u64, scan_ws: scan_ws_elems(that) u64.
// Shared by the partition step and the key sort (sort.cu).
size_t radix_hist_elems(uint64_t n);
void launch_radix_pass(const uint32_t* keys_in, const uint32_t* idx_in, uint32_t n, int shift, uint32_t nd,
                       uint64_t* hist, uint64_t* hist_total, uint64_t* scan_ws, uint32_t* keys_out, uint32_t* idx_out,
                       cudaStream_t st, uint64_t* launches);
uint32_t partition_radix_passes(uint32_t num_partitions);
size_t partition_ws_bytes(uint64_t n, uint32_t num_partitions);  // d_ws of launch_partition
void launch_partition(const uint32_t* d_rec_len, const uint32_t* d_rec_part, uint64_t n, uint32_t num_partitions,
                      uint8_t* d_ws, PartitionPlan* plan, cudaStream_t st,
                      uint64_t* launches);
// copies the records into d_dst in sorted order (only once the readback has shown every id valid and the lengths sum
// to the arena size)
void launch_partition_gather(const uint8_t* rec_base, const uint32_t* d_rec_len, uint64_t n, const PartitionPlan& plan,
                             uint8_t* d_dst, cudaStream_t st, uint64_t* launches);
// sdst[j] = arena offset of the j-th record in the order idx (nullptr = identity): rec_len[idx[j]] scanned.
// total: one u64 (the grand total); scan_ws: scan_ws_elems(n) u64
void launch_sorted_offsets(const uint32_t* idx, const uint32_t* d_rec_len, uint64_t n, uint64_t* sdst, uint64_t* total,
                           uint64_t* scan_ws, cudaStream_t st, uint64_t* launches);

// ---------------- sort.cu (stable sort of fixed-size records by an unsigned byte key) ----------------
// n records of record_bytes each, back to back at d_rec (n < 2^32); the key of a record is its bytes
// [key_off, key_off + key_len), 1 <= key_len <= 16, compared as unsigned bytes, lexicographically.  Writes the records
// to d_dst in ascending key order, equal keys in input order.  d_ws: key_sort_ws_bytes(n, key_len).
size_t key_sort_ws_bytes(uint64_t n, uint32_t key_bytes);
void launch_key_sort(const uint8_t* d_rec, uint64_t n, uint32_t record_bytes, uint32_t key_off, uint32_t key_len,
                     uint8_t* d_ws, uint8_t* d_dst, cudaStream_t st, uint64_t* launches);
// The per-record arrays of a key sort of n records with key_bytes key bytes, carved from key_sort_ws_bytes(n, key_bytes)
// bytes: the key as ceil(key_bytes / 4) big-endian u32 words, word-major (words[k * n + i], zero-padded on the right);
// radix buffers; the gather's per-record length, source and destination offsets; histogram and its scan workspace.
struct KeySortWs {
  uint32_t* words;
  uint32_t* K[2];
  uint32_t* I[2];
  uint32_t* len;
  uint64_t* src_off;
  uint64_t* sdst;
  uint64_t* hist;
  uint64_t* scan_ws;
  uint64_t* total;
};
KeySortWs carve_key_sort_ws(uint8_t* d_ws, uint64_t n, uint32_t key_bytes);
// LSD radix sort of the key words (one 8-bit pass per key byte, least significant first), stable; returns the sorted
// record indices (nullptr when n < 2: input order)
const uint32_t* launch_key_radix(const KeySortWs& w, uint64_t n, uint32_t key_bytes, cudaStream_t st,
                                 uint64_t* launches);

// ---------------- rows.cu (stable sort of length-prefixed UnsafeRow records by a typed key) ----------------
// Framing: the n_ranges decoded blocks [off[i], off[i] + len[i]) of the arena (arena_bytes long, 64 bytes of slack
// after it) are walked as [size: int32 big-endian][size bytes] records.  d_fws: rows_frame_ws_bytes(arena_bytes,
// n_ranges).  Afterwards rows_frame_readback(d_fws) holds rows_frame_readback_bytes(n_ranges) bytes: [record count,
// verdict of range 0, 1, ...]; a verdict is ~0 when the range is whole records, else kRowsBad* << 61 | the offset of the
// range's first bad record.  A record is bad when its prefix is cut by the range end, its size is negative, it runs past
// the range end, its row is shorter than min_key bytes, or shorter than min_null bytes.
constexpr uint64_t kRowsBadPrefix = 1, kRowsBadNegative = 2, kRowsBadPastEnd = 3, kRowsBadKey = 4, kRowsBadNull = 5;
size_t rows_frame_ws_bytes(uint64_t arena_bytes, uint32_t n_ranges);
inline size_t rows_frame_readback_bytes(uint32_t n_ranges) { return ((size_t)n_ranges + 1) * 8; }
uint64_t* rows_frame_readback(uint8_t* d_fws, uint64_t arena_bytes, uint32_t n_ranges);
void launch_rows_frame(const uint8_t* arena, uint64_t arena_bytes, const uint64_t* h_off, const uint64_t* h_len,
                       uint32_t n_ranges, uint64_t min_key, uint64_t min_null, uint8_t* d_fws, cudaStream_t st,
                       uint64_t* launches);
// key bytes of the sort: key_len, plus the leading null byte of a nullable key
inline uint32_t rows_key_bytes(uint32_t key_len, int32_t null_field) { return key_len + (null_field >= 0 ? 1 : 0); }
size_t rows_sort_ws_bytes(uint64_t n, uint32_t key_bytes);
// the framed records (n = the read-back count) as dense offsets and lengths in arena order, into the sort workspace
void launch_rows_emit(const uint8_t* arena, uint64_t arena_bytes, uint32_t n_ranges, uint8_t* d_fws, uint64_t n,
                      uint32_t key_bytes, uint8_t* d_ws, cudaStream_t st, uint64_t* launches);
// the emitted records to d_dst, ascending by key (nulls first), stable.  key_type B2S_KEY_*
void launch_rows_sort(const uint8_t* arena, uint64_t n, uint32_t key_type, uint32_t key_off, uint32_t key_len,
                      int32_t null_field, uint8_t* d_ws, uint8_t* d_dst, cudaStream_t st, uint64_t* launches);

// ---------------- exchange.cu (exchange-cache reads: ranges of device memory gathered into one arena) ----------------
// piece: len bytes at src (device pointer, any alignment) go to d_dst + dst
struct ExchangePiece {
  const uint8_t* src;
  uint64_t dst;
  uint64_t len;
};
constexpr uint64_t kExchangePieceBytes = 32 << 10;
// appends the range [src, src + len) -> dst, cut into pieces of at most kExchangePieceBytes
void exchange_add_pieces(std::vector<ExchangePiece>& pieces, const uint8_t* src, uint64_t dst, uint64_t len);
// one launch copies every piece (d_pieces: device copy of the pieces)
void launch_exchange_gather(const ExchangePiece* d_pieces, uint32_t n, uint8_t* d_dst, cudaStream_t st,
                            uint64_t* launches);

// ---------------- gen.cu (bench utility) ----------------
void launch_gen_terasort(uint8_t* d_dst, uint64_t first_record, uint64_t n_records, uint64_t seed, cudaStream_t st);

}  // namespace b2s
