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
  uint32_t* d_crc_misc[2];  // x2n[67] | xinv2n[67] | lane_const[32] | poly (crc_gf.h: kMisc*)
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
// ids: the id array of a workspace sized with hashed ids (partition_ws_bytes(n, R, true)), else nullptr.
struct PartitionPlan {
  uint64_t* src_off = nullptr;
  uint64_t* sdst = nullptr;
  const uint32_t* idx = nullptr;
  uint64_t* readback = nullptr;
  size_t readback_bytes = 0;
  uint32_t* ids = nullptr;
  const uint32_t* keys = nullptr;  // the sorted ids (nullptr: no radix pass, one partition)
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
// d_ws of launch_partition; hashed_ids: with room for the id array (plan->ids) behind the rest
size_t partition_ws_bytes(uint64_t n, uint32_t num_partitions, bool hashed_ids = false);
// launch_partition = launch_partition_offsets, then launch_partition_order over the same d_ws and plan.  Between the
// two, src_off holds the record offsets and the readback's first word is ~0, so ids can be computed there (rows_hash).
// offsets: the readback reset, the offsets (rec_len scanned); d_rec_part == nullptr skips the id check.
void launch_partition_offsets(const uint32_t* d_rec_len, const uint32_t* d_rec_part, uint64_t n,
                              uint32_t num_partitions, uint8_t* d_ws, PartitionPlan* plan, cudaStream_t st,
                              uint64_t* launches);
// order: the radix passes over the ids, the sorted offsets and the partition bounds.  idx_in (nullptr: the position):
// the record index of position k, whose id is d_rec_part[k]; the passes are stable, so a partition keeps that order.
void launch_partition_order(const uint32_t* d_rec_len, const uint32_t* d_rec_part, uint64_t n, uint32_t num_partitions,
                            uint8_t* d_ws, PartitionPlan* plan, cudaStream_t st, uint64_t* launches,
                            const uint32_t* idx_in = nullptr);
void launch_partition(const uint32_t* d_rec_len, const uint32_t* d_rec_part, uint64_t n, uint32_t num_partitions,
                      uint8_t* d_ws, PartitionPlan* plan, cudaStream_t st,
                      uint64_t* launches);
// rec_start[p] (num_partitions + 1 u64, device memory) = the sorted index of partition p's first record, n past the
// last record (an empty partition: the next non-empty one's first), from the sorted ids of launch_partition_order; n > 0
void launch_partition_rec_start(const PartitionPlan& plan, uint64_t n, uint32_t num_partitions, uint64_t* rec_start,
                                cudaStream_t st, uint64_t* launches);
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
// record indices (nullptr when n < 2: input order).  lead_bytes (a key of more than one word): only the low lead_bytes
// bytes of word 0 can be non-zero, so only they take passes.
const uint32_t* launch_key_radix(const KeySortWs& w, uint64_t n, uint32_t key_bytes, cudaStream_t st,
                                 uint64_t* launches, uint32_t lead_bytes = 4);

// ---------------- rows.cu (stable sort of length-prefixed UnsafeRow records by a typed key) ----------------
// Framing: the n_ranges decoded blocks [off[i], off[i] + len[i]) of the arena (arena_bytes long, 64 bytes of slack
// after it) are walked as [size: int32 big-endian][size bytes] records.  d_fws: rows_frame_ws_bytes(arena_bytes,
// n_ranges).  Afterwards rows_frame_readback(d_fws) holds rows_frame_readback_bytes(n_ranges) bytes: [record count,
// verdict of range 0, 1, ...]; a verdict is ~0 when the range is whole records, else kRowsBad* << 61 | the offset of the
// range's first bad record.  A record is bad when its prefix is cut by the range end, its size is negative, it runs past
// the range end, its row is shorter than min_key bytes, shorter than min_null bytes, or shorter than min_agg bytes.
// kRowsBadString is the key pass's verdict (launch_rows_order): a non-null string key runs past its row, or a non-null
// decimal's slot does not name 1..16 bytes inside its row.
constexpr uint64_t kRowsBadPrefix = 1, kRowsBadNegative = 2, kRowsBadPastEnd = 3, kRowsBadKey = 4, kRowsBadNull = 5,
                   kRowsBadAgg = 6, kRowsBadString = 7;
// Marked ranges (n_marks of them, h_marks in host memory): ranges whose record offsets are known, so they are not
// walked (their h_len entries are 0) but marked, a thread per record.  Mark k covers count records: record j's start is
// arena offset base + off[j] (mod 2^64); it is checked against min_key, min_null and min_agg only (its size prefix was
// checked when the offsets were taken), and the verdict of its range (index `range`) is lowered to the lowest bad
// record, offset-major: rows_mark_verdict turns it into the walk's form.  `first` numbers the marks' records in order
// (a prefix sum of count).
struct RowsMark {
  const uint64_t* off;
  uint64_t base;   // the range's arena offset minus the offset of its first record in off's numbering
  uint64_t place;  // the range's arena offset
  uint64_t first;
  uint64_t count;
  uint32_t range;
};
// a marked range's verdict as the readback brings it, re-packed into the walk's form (kRowsBad* << 61 | offset)
inline uint64_t rows_mark_verdict(uint64_t v) { return v == ~0ull ? v : ((v & 7) << 61) | (v >> 3); }
size_t rows_frame_ws_bytes(uint64_t arena_bytes, uint32_t n_ranges, uint32_t n_marks = 0);
inline size_t rows_frame_readback_bytes(uint32_t n_ranges) { return ((size_t)n_ranges + 1) * 8; }
uint64_t* rows_frame_readback(uint8_t* d_fws, uint64_t arena_bytes, uint32_t n_ranges);
// the ranges' arena offsets on the device (ascending), as launch_rows_frame uploaded them
const uint64_t* rows_frame_ranges(uint8_t* d_fws, uint64_t arena_bytes, uint32_t n_ranges);
void launch_rows_frame(const uint8_t* arena, uint64_t arena_bytes, const uint64_t* h_off, const uint64_t* h_len,
                       uint32_t n_ranges, uint64_t min_key, uint64_t min_null, uint64_t min_agg, uint8_t* d_fws,
                       cudaStream_t st, uint64_t* launches, const RowsMark* h_marks = nullptr, uint32_t n_marks = 0);
// The sort key of a row: n columns compared left to right.  Column c: type[c] (low 8 bits: B2S_KEY_*, B2S_STRING_KEY or
// B2S_DECIMAL_KEY; above them the order flags B2S_KEY_DESCENDING / B2S_KEY_NULLS_LAST) at row offset off[c], len[c]
// bytes (a string or a decimal: its 8-byte slot, (offset << 32) | size), null bit null_field[c] (-1: never null).
// It is encoded as one byte string compared by memcmp, prefix-free, column after column: a nullable column's null byte
// (0 null, 1 not; NULLS_LAST: 1 null, 0 not), then the value (all zero when null): BYTES as they are; an int big-endian
// with its sign bit flipped; a float with -0.0 made +0.0 and every NaN the canonical NaN, then every bit flipped when
// negative, else the sign bit, big-endian; a decimal's 1..16 bytes sign-extended to 16, sign bit flipped; a non-null
// string as groups of 8 bytes zero-padded, each followed by a marker: 9 when more bytes follow, else the number of real
// bytes in the group (0..8) (an empty string is one group of zeros with marker 0, a null string nothing).  DESCENDING
// complements every value byte of the column (a string's markers included): the column's code stays prefix-free and
// its order reverses.
constexpr uint32_t kMaxKeys = 16;
// a join's key column that is never null on its side but nullable on the other: it encodes the null byte of a non-null
// value, so that equal keys of the two sides encode equal (rows_key.cuh, encode_key<true>)
constexpr int32_t kNullByteOnly = -2;
constexpr uint32_t kStringKey = B2S_STRING_KEY, kDecimalKey = B2S_DECIMAL_KEY;
constexpr uint32_t kKeyTypeMask = 0xff;
// the encoded value bytes of a fixed-width column of type ty (low 8 bits) and key_len len: a decimal's 16, else len
__host__ __device__ inline uint32_t key_value_bytes(uint32_t ty, uint32_t len) { return ty == kDecimalKey ? 16 : len; }
struct KeySpec {
  uint32_t n = 0;
  uint32_t type[kMaxKeys] = {};
  uint32_t off[kMaxKeys] = {};
  uint32_t len[kMaxKeys] = {};
  int32_t null_field[kMaxKeys] = {};
};
// The first pass radix-sorts the first kKeyPrefixBytes bytes of every encoded key (fewer when every key is shorter);
// keys longer than that are refined in rounds of kKeyChunkBytes more bytes over the records still tied.
constexpr uint32_t kKeyPrefixBytes = 20, kKeyChunkBytes = 16;
// the encoded key's length when it is the same for every row (no string column), else ~0u
inline uint32_t rows_key_encoded_bytes(const KeySpec& ks) {
  uint32_t b = 0;
  for (uint32_t c = 0; c < ks.n; c++) {
    const uint32_t ty = ks.type[c] & kKeyTypeMask;
    if (ty == kStringKey) return ~0u;
    // a null byte (leading), or a null-safe column's isnull byte (trailing, with or without a null field)
    b += key_value_bytes(ty, ks.len[c]) + (ks.null_field[c] != -1 || (ks.type[c] & B2S_KEY_NULL_SAFE) ? 1 : 0);
  }
  return b;
}
// key bytes of the first pass; a single column: key_len, plus the leading null byte of a nullable key
inline uint32_t rows_key_bytes(const KeySpec& ks) {
  const uint32_t b = rows_key_encoded_bytes(ks);
  return b < kKeyPrefixBytes ? b : kKeyPrefixBytes;
}
// The key takes the refinement path: it is longer than the first pass, or it has a decimal column, whose slots are
// checked there (the first round's readback brings the verdicts; when the key fits the first pass no record is tied).
inline bool rows_key_refines(const KeySpec& ks) {
  if (rows_key_encoded_bytes(ks) > kKeyPrefixBytes) return true;
  for (uint32_t c = 0; c < ks.n; c++)
    if ((ks.type[c] & kKeyTypeMask) == kDecimalKey) return true;
  return false;
}
size_t rows_sort_ws_bytes(uint64_t n, uint32_t key_bytes);
// the framed records (n = the read-back count) as dense offsets and lengths in arena order, into the sort workspace
void launch_rows_emit(const uint8_t* arena, uint64_t arena_bytes, uint32_t n_ranges, uint8_t* d_fws, uint64_t n,
                      uint32_t key_bytes, uint8_t* d_ws, cudaStream_t st, uint64_t* launches);
// The refinement workspace (keys that refine): per record the encoded key length, per position the current order and
// its group-head flags, the compaction's scan and maps, and the readback [tied records | segments << 32, string verdict
// of range 0, 1, ...] (a verdict as rows_frame_readback's: ~0 or kRowsBadString << 61 | offset).
size_t rows_refine_ws_bytes(uint64_t n, uint32_t n_ranges);
uint64_t* rows_refine_readback(uint8_t* d_rws, uint64_t n, uint32_t n_ranges);
// keys + radix: the emitted records' order by their first key_bytes encoded bytes, stable, as sorted record indices
// (nullptr when n < 2: arena order).  The key words stay in the workspace in record order.  With d_rws (keys that
// refine): also every key's encoded length and the string verdicts (ranges: rows_frame_ranges), and the order and
// head flags that launch_rows_refine_* start from.
const uint32_t* launch_rows_order(const uint8_t* arena, uint64_t n, const KeySpec& ks, const uint64_t* ranges,
                                  uint32_t n_ranges, uint8_t* d_ws, uint8_t* d_rws, cudaStream_t st,
                                  uint64_t* launches);
// Refinement round at encoded byte d (kKeyPrefixBytes, then + kKeyChunkBytes per round).  mark: the tied records (a
// run of equal first-d-byte keys of two or more whose keys go on past d) counted into the readback.  round (m tied
// records in segs runs, as read back): their next kKeyChunkBytes bytes extracted, the m records sorted stably by (run,
// bytes) and put back into their runs' positions, the head flags split where the bytes differ.
void launch_rows_refine_mark(uint64_t n, uint32_t d, uint8_t* d_rws, uint32_t n_ranges, cudaStream_t st,
                             uint64_t* launches);
void launch_rows_refine_round(const uint8_t* arena, uint64_t n, const KeySpec& ks, uint64_t m, uint64_t segs,
                              uint32_t d, uint8_t* d_ws, uint8_t* d_rws, uint32_t n_ranges, cudaStream_t st,
                              uint64_t* launches);
// after the last round (no tied record): the sorted record indices, and per position 1 where a new key starts
const uint32_t* rows_refine_order(uint8_t* d_rws, uint64_t n, uint32_t n_ranges);
const uint32_t* rows_refine_heads(uint8_t* d_rws, uint64_t n, uint32_t n_ranges);
// Whole-row sort (a round-robin exchange's sortBeforeRepartition order): the key of record i (rec_len[i] bytes at
// rec + rec_off[i], [size: int32 big-endian][row], size a multiple of 8) is [hash ^ 0x80000000: 4 B][size: 4 B][row]
// (big-endian words), prefix-free: rows of different sizes differ within the first 8 bytes, rows of equal size end
// together.  d_ws: rows_sort_ws_bytes(n, kKeyPrefixBytes); d_rws: rows_refine_ws_bytes(n, 0).  The caller stores each
// key's first word at rows_whole_words(d_ws, n)[i] and its length at rows_refine_klen(d_rws, n)[i] (0: never read);
// launch_rows_whole_order radix-sorts the first word only (4 passes) and sets up the order and head flags; the rounds
// are launch_rows_refine_mark and launch_rows_whole_refine_round from d = 4, kKeyChunkBytes more each; the order ends
// in rows_refine_order.
uint32_t* rows_whole_words(uint8_t* d_ws, uint64_t n);
uint32_t* rows_refine_klen(uint8_t* d_rws, uint64_t n);
void launch_rows_whole_order(uint64_t n, uint8_t* d_ws, uint8_t* d_rws, cudaStream_t st, uint64_t* launches);
void launch_rows_whole_refine_round(const uint8_t* rec, const uint64_t* rec_off, const uint32_t* rec_len, uint64_t n,
                                    uint64_t m, uint64_t segs, uint32_t d, uint8_t* d_ws, uint8_t* d_rws,
                                    cudaStream_t st, uint64_t* launches);
// A join's key pass (two row layouts in one sort): record i is a left record when its arena offset is below split (the
// left blocks come first, so the left records are a prefix), else a right one, and it is keyed with its side's columns
// side[0] / side[1] (encoded to equal widths: a plain column nullable on one side only has kNullByteOnly on the other;
// a B2S_KEY_NULL_SAFE column encodes its trailing isnull byte on both sides, whatever their null fields).  A
// row shorter than its side's fixed region fixed[s] lowers its range's verdict (verdict[r], as rows_keys_kernel's) with
// kRowsBadKey; a bad string or decimal with kRowsBadString.  Such a record gets key length 0 (never refined).
struct JoinKeys {
  KeySpec side[2];
  uint64_t split;
  uint32_t fixed[2];
};
// launch_rows_order for a join: the same workspaces and order, the key words from each record's side; verdict
// (n_ranges words, device) is reset here
const uint32_t* launch_rows_join_order(const uint8_t* arena, uint64_t n, const JoinKeys& jk, const uint64_t* ranges,
                                       uint32_t n_ranges, uint64_t* verdict, uint8_t* d_ws, uint8_t* d_rws,
                                       cudaStream_t st, uint64_t* launches);
// launch_rows_refine_round for a join's keys
void launch_rows_join_refine_round(const uint8_t* arena, uint64_t n, const JoinKeys& jk, uint64_t m, uint64_t segs,
                                   uint32_t d, uint8_t* d_ws, uint8_t* d_rws, cudaStream_t st, uint64_t* launches);
// the emitted records to d_dst in the order idx; count (below n): only the records idx[0 .. count), a subset
void launch_rows_gather(const uint8_t* arena, uint64_t n, uint32_t key_bytes, const uint32_t* idx, uint8_t* d_ws,
                        uint8_t* d_dst, cudaStream_t st, uint64_t* launches, uint64_t count = ~0ull);

// ---------------- rows_hash.cu (Spark's HashPartitioning ids of length-prefixed UnsafeRow records) ----------------
// Record i: rec_len[i] bytes at rec + rec_off[i], [size: int32 big-endian][row].  ids[i] = pmod(Murmur3Hash(key
// columns, 42), num_partitions), the columns (ks, no order flags; B2S_KEY_BYTES is a 1-byte boolean) folded left to
// right, a null one skipped.  A bad record takes id 0 and lowers *bad (device, ~0 = none) to (i << 3) | its reason:
// kHashBadShort rec_len < 4, kHashBadSize the size prefix is not rec_len - 4, kHashBadKey / kHashBadNull the row does
// not hold a key slot / a key's null word, kHashBadString a non-null string runs past the row, kHashBadDecimal a
// non-null decimal's size is not 1..16 or it runs past the row.  Records ending past rec_bytes are not read.
constexpr uint64_t kHashBadShort = 1, kHashBadSize = 2, kHashBadKey = 3, kHashBadNull = 4, kHashBadString = 5,
                   kHashBadDecimal = 6;
void launch_rows_hash(const uint8_t* rec, uint64_t rec_bytes, const uint64_t* rec_off, const uint32_t* rec_len,
                      uint64_t n, const KeySpec& ks, uint32_t num_partitions, uint32_t* ids, uint64_t* bad,
                      cudaStream_t st, uint64_t* launches);

// ---------------- rows_range.cu (Spark's RangePartitioner ids of length-prefixed UnsafeRow records) ----------------
// n_bounds bound rows (< 2^24), framed as records ([size: int32 big-endian][row]) back to back: w.rows[w.off[j] ..
// w.off[j + 1]), both uploaded by the caller into a workspace of rows_range_ws_bytes(n_bounds, bound_bytes) bytes.  Bound
// j's key column c is its field c (the records' column's type, flags and key_len; slot 8 * ceil(n / 64) + 8 c, null bit
// c when the records' column is nullable).  Records and key columns ks (order flags allowed) as launch_rows_hash's.
// ids[i] = the number of bounds whose key is below record i's, by the key encoding (KeySpec): Spark's
// RangePartitioner.getPartition over strictly increasing bounds.  Verdicts lower *bad (device, ~0 = none):
//   a bad bound j: (j << 3) | its kHashBad* reason (as a record's), or kRangeBadOrder when its key is not above bound
//   j - 1's; a bad record i: kRangeBadRecord | (i << 3) | its kHashBad* reason, so a bad bound always wins.
// n == 0: only the bound step runs.
constexpr uint64_t kRangeBadOrder = 7, kRangeBadRecord = 1ull << 63;
struct RangeWs {
  uint4* words;       // bound j: its first kKeyPrefixBytes encoded bytes (five big-endian words), its encoded length
  uint64_t* off;      // n_bounds + 1 row offsets
  uint8_t* rows;      // bound_bytes, with 16 bytes of slack
  uint64_t* verdict;  // one word for a call without records
};
size_t rows_range_ws_bytes(uint32_t n_bounds, uint64_t bound_bytes);
RangeWs carve_rows_range_ws(uint8_t* d_ws, uint32_t n_bounds, uint64_t bound_bytes);
void launch_rows_range(const uint8_t* rec, uint64_t rec_bytes, const uint64_t* rec_off, const uint32_t* rec_len,
                       uint64_t n, const KeySpec& ks, const RangeWs& w, uint32_t n_bounds, uint32_t* ids,
                       uint64_t* bad, cudaStream_t st, uint64_t* launches);

// ---------------- rows_round_robin.cu (Spark's RoundRobinPartitioning of length-prefixed UnsafeRow records) ---------
// Records as launch_rows_hash's.  A bad record lowers *bad (device, ~0 = none) to (i << 3) | its reason: kHashBadShort,
// kHashBadSize, or kRowsBadWords (its row size is not a multiple of 8: not an UnsafeRow).  words / klen (nullptr: no
// sort, only the checks): the whole-row sort's first key word, hashUnsafeWords(row, 42) ^ 0x80000000 (signed order as
// unsigned), and key length 8 + size; a bad record, or one ending past rec_bytes, gets length 0: it is not read again.
constexpr uint64_t kRowsBadWords = 7;
void launch_rows_round_robin_hash(const uint8_t* rec, uint64_t rec_bytes, const uint64_t* rec_off,
                                  const uint32_t* rec_len, uint64_t n, uint32_t* words, uint32_t* klen, uint64_t* bad,
                                  cudaStream_t st, uint64_t* launches);
// ids[k] = (start + 1 + k) mod num_partitions, k < n: the id of the k-th row the writer sees (start + n < 2^31)
void launch_rows_round_robin_ids(uint64_t n, uint32_t start, uint32_t num_partitions, uint32_t* ids, cudaStream_t st,
                                 uint64_t* launches);

// ---------------- aggregate.cu (group key-sorted rows and merge their aggregate buffers) ----------------
// Aggregate a: op[a] (B2S_AGG_*, with SUM_DECIMAL's precision in bits 8..15) over the 8-byte slot at row offset off[a],
// null bit null_field[a] (-1: never null).  An out-of-line decimal (agg_decimal_wide) is staged as 16 bytes: its high
// words at index wide[a] of n_wide; its 16-byte region must start at or after region_from (the end of every slot and
// null word the call uses).
constexpr uint32_t kMaxAggs = 16;
struct AggSpec {
  uint32_t n = 0;
  uint32_t op[kMaxAggs] = {};
  uint32_t off[kMaxAggs] = {};
  int32_t null_field[kMaxAggs] = {};
  uint32_t wide[kMaxAggs] = {};
  uint32_t n_wide = 0;
  uint32_t region_from = 0;
  bool decimal = false;  // some op is a Decimal op: the merge runs the kernels that know them
  // B2S_AGG_VARIANCE entries: n staged as the other slots, avg and m2 as words 2 var[a] and 2 var[a] + 1 of 2 n_var;
  // with one, the merge runs the kernels that know them (which know the Decimal ops too)
  uint32_t var[kMaxAggs] = {};
  uint32_t n_var = 0;
};
__host__ __device__ inline uint32_t agg_base_op(uint32_t op) { return op & 0xff; }
__host__ __device__ inline uint32_t agg_precision(uint32_t op) { return (op >> 8) & 0xff; }
// a Decimal op (SUM / MIN / MAX_DECIMAL): its value is staged in 128 bits
__host__ __device__ inline bool agg_decimal_op(uint32_t op) {
  return agg_base_op(op) >= B2S_AGG_SUM_DECIMAL && agg_base_op(op) <= B2S_AGG_MAX_DECIMAL;
}
// the op's value is out of line: 16 bytes at (offset << 32) | size
__host__ __device__ inline bool agg_decimal_wide(uint32_t op) {
  const uint32_t b = agg_base_op(op);
  return b == B2S_AGG_MIN_DECIMAL || b == B2S_AGG_MAX_DECIMAL || (b == B2S_AGG_SUM_DECIMAL && agg_precision(op) > 18);
}
// the verdict of the decimal region checks (rows_aggregate_readback's third word): ~0, or the lowest bad record's arena
// offset << 2 | one of these
constexpr uint64_t kAggBadDecimal = 1, kAggBadRegionEnd = 2, kAggBadRegionStart = 3;
// d_aws: rows_aggregate_ws_bytes(n, n_aggs, n_wide, n_var), beside the sort workspace d_ws of the same n records
size_t rows_aggregate_ws_bytes(uint64_t n, uint32_t n_aggs, uint32_t n_wide, uint32_t n_var = 0);
// after launch_rows_group: [group count, output bytes, decimal verdict (only with an out-of-line decimal)] (device)
uint64_t* rows_aggregate_readback(uint8_t* d_aws, uint64_t n, uint32_t n_aggs, uint32_t n_wide);
// the groups of the records in the order idx (launch_rows_order): heads, group starts, the heads' output offsets and
// the readback.  Also stages every aggregate's inputs in sorted order.  heads (keys that refine: rows_refine_heads)
// flags where a new key starts; nullptr: where the key words differ.
void launch_rows_group(const uint8_t* arena, uint64_t n, const uint32_t* idx, const uint32_t* heads,
                       uint32_t key_bytes, const AggSpec& spec, uint8_t* d_ws, uint8_t* d_aws, cudaStream_t st,
                       uint64_t* launches);
// the groups (count read back) to d_dst: the first record of each, whole, with the aggregates' slots and null bits
// replaced by the merged values
void launch_rows_aggregate(const uint8_t* arena, uint64_t n, uint64_t groups, uint32_t key_bytes, const AggSpec& spec,
                           uint8_t* d_ws, uint8_t* d_aws, uint8_t* d_dst, cudaStream_t st, uint64_t* launches);

// after launch_rows_group: per sorted position the number of group heads before it (a head's group index), and per
// group its first position (n after the last group)
const uint64_t* rows_group_heads_before(uint8_t* d_aws, uint64_t n);
const uint32_t* rows_group_starts(uint8_t* d_aws, uint64_t n);
// per group its head's record length, after launch_rows_group: the merged records' lengths, in output order
const uint32_t* rows_group_lengths(uint8_t* d_aws, uint64_t n);

// ---------------- partial_agg.cu (a map task's partial aggregation: one partial row per key) ----------------
// The caller's records ([size: int32 big-endian][row], rec_len each, back to back), sorted by the key columns keys
// (launch_rows_order) and grouped (launch_rows_group, an AggSpec of no aggregates, in d_gws).  Buffer k < n_bufs:
// merge op op[k] (B2S_AGG_*; SUM_DECIMAL | P << 8), staged from its input (B2S_WINDOW_VAL_* vtype[k], a decimal's p in
// bits 8..15; slot voff[k], null bit vnull[k] or -1) by stage[k]: kStageValue the value (a null is skipped),
// kStageZero the value or 0 when null (to_double[k]: an integer cast to double, rounded to nearest), kStageCount 1 per
// non-null input (every input for VAL_NONE), kStageIsEmpty 1 per null input.  A decimal buffer (op >= SUM_DECIMAL) is
// staged in 128 bits: wide[k] is its index among the n_dec of them.  dsum: some buffer is a double sum.  A variance
// buffer (op B2S_AGG_VARIANCE, kStageValue with to_double: the input cast to double, a null skipped) folds into three
// fields (n, avg, m2); var[k] is its index among the n_var of them.  n_fields: the partial row's buffer fields.
// Merge entries (merge: some buffer has one; the distinct aggregation's step over merged rows): kStageCountAll stages 1
// per row with no null bit of the mask voff[k] set (SUM_INT64: count(DISTINCT a, b, ..)); kStageMerge folds a buffer by
// its mergeExpressions in position order: a SUM_DECIMAL | P << 8 buffer (vtype its decimal(P)) is null once an input is
// null or the sum reaches 10^P; a VARIANCE buffer reads [n, avg, m2] at voff (staged in vhi words wide[k], wide[k] + 1
// of n_dec).
constexpr uint32_t kStageValue = 0, kStageZero = 1, kStageCount = 2, kStageIsEmpty = 3, kStageCountAll = 4,
                   kStageMerge = 5;
struct PartialAggSpec {
  KeySpec keys;
  uint32_t n_bufs = 0;
  uint32_t op[kMaxAggs] = {};
  uint32_t stage[kMaxAggs] = {};
  uint32_t to_double[kMaxAggs] = {};
  uint32_t vtype[kMaxAggs] = {};
  uint32_t voff[kMaxAggs] = {};
  int32_t vnull[kMaxAggs] = {};
  uint32_t wide[kMaxAggs] = {};
  uint32_t n_dec = 0;
  bool dsum = false;
  uint32_t var[kMaxAggs] = {};
  uint32_t n_var = 0;
  uint32_t n_fields = 0;
  bool merge = false;
  uint32_t n_merge_dec = 0, n_merge_var = 0;  // the kStageMerge entries of each kind (pa_merge_chain_kernel's)
};
// the check verdict (header word 0) of a record whose value is bad: (i << 3) | kPaBadValue, beside launch_rows_hash's
// kHashBad* reasons; header word 2 then holds (i << 2) | kPaBadSlot, kPaBadNull or kPaBadDecimal
constexpr uint64_t kPaBadValue = 7, kPaBadSlot = 1, kPaBadNull = 2, kPaBadDecimal = 3;
size_t partial_agg_ws_bytes(uint64_t n, const PartialAggSpec& spec);
// the workspace's header (device): [check verdict (~0: none), record bytes, check detail (~0: none), 0 (the one range's
// offset), groups, partial-row bytes]
uint64_t* partial_agg_header(uint8_t* d_paws);
// the record offsets: rec_len scanned into the sort workspace d_ws (key_bytes: its key width), as launch_rows_emit
// leaves them; their total into header word 1.  Resets the header.
void launch_partial_agg_offsets(const uint32_t* rec_len, uint64_t n, uint32_t key_bytes, uint8_t* d_ws,
                                uint8_t* d_paws, cudaStream_t st, uint64_t* launches);
// every record checked (its framing and key columns by launch_rows_hash, into ids, n u32 of scratch; its values here):
// the lowest bad record into header words 0 and 2
void launch_partial_agg_check(const uint8_t* rec, uint64_t rec_bytes, uint64_t n, uint32_t key_bytes,
                              const PartialAggSpec& spec, uint8_t* d_ws, uint8_t* d_paws, uint32_t* ids,
                              cudaStream_t st, uint64_t* launches);
// after launch_rows_group: staging, the folds, the partial rows' lengths and offsets; header words 4, 5
void launch_partial_agg_fold(const uint8_t* rec, uint64_t n, const uint32_t* idx, uint32_t key_bytes,
                             const PartialAggSpec& spec, uint8_t* d_ws, uint8_t* d_gws, uint8_t* d_paws,
                             cudaStream_t st, uint64_t* launches);
// per partial row its record length (4 + row), after launch_partial_agg_fold
const uint32_t* partial_agg_row_len(uint8_t* d_paws, uint64_t n, const PartialAggSpec& spec);
// per position j < n of records already in the order of a key whose first columns are ks (offsets and lengths in the
// sort workspace d_ws, as launch_partial_agg_offsets leaves them): heads[j] = 1 where ks's value differs from j - 1's
// (and at 0), for launch_rows_group
void launch_partial_agg_heads(const uint8_t* rec, uint64_t n, uint32_t key_bytes, const KeySpec& ks, uint8_t* d_ws,
                              uint32_t* heads, cudaStream_t st, uint64_t* launches);
// the groups (count read back) as partial rows, [size: int32 big-endian][row] back to back, to d_dst
void launch_partial_agg_emit(const uint8_t* rec, uint64_t n, uint64_t groups, const uint32_t* idx, uint32_t key_bytes,
                             const PartialAggSpec& spec, uint8_t* d_ws, uint8_t* d_gws, uint8_t* d_paws,
                             uint8_t* d_dst, cudaStream_t st, uint64_t* launches);

// ---------------- rows_expand.cu (Spark's Expand for grouping sets, in front of the partial aggregation) ----------------
// The caller's records (checked by launch_partial_agg_check; offsets rec_off as launch_partial_agg_offsets leaves them),
// each projected once per grouping set into a compact UnsafeRow: key column c (nullable; null outside the set), gid
// (Spark's spark_grouping_id, a long), then input i < n_in of the aggregates that read one (type vtype[i], slot voff[i],
// null bit vnull[i] or -1; reads[i]: its value is read, not only its null bit).  Set k's mask is device word k of
// expand_masks; projected record r * n_sets + k is record r under set k.
struct ExpandSpec {
  KeySpec keys;
  uint32_t n_in = 0;
  uint32_t vtype[kMaxAggs] = {};
  uint32_t voff[kMaxAggs] = {};
  int32_t vnull[kMaxAggs] = {};
  uint32_t reads[kMaxAggs] = {};
  uint32_t n_sets = 0;
};
size_t expand_ws_bytes(uint64_t n, uint32_t n_sets);
// the workspace's header (device): [projected bytes, the lowest record whose projected row passes 2^31 - 1 bytes
// (~0: none)]
uint64_t* expand_header(uint8_t* d_xws);
// the n_sets set masks (device), for the caller to fill
uint32_t* expand_masks(uint8_t* d_xws, uint64_t n, uint32_t n_sets);
// the projected records' lengths and 64-bit offsets; header words 0 and 1.  Resets the header.
void launch_expand_size(const uint8_t* rec, const uint64_t* rec_off, uint64_t n, const ExpandSpec& spec,
                        uint8_t* d_xws, cudaStream_t st, uint64_t* launches);
// the projected records ([size: int32 big-endian][row], header word 0 bytes) to d_out, their lengths to d_out_len
void launch_expand_write(const uint8_t* rec, const uint64_t* rec_off, uint64_t n, const ExpandSpec& spec,
                         uint8_t* d_xws, uint32_t* d_out_len, uint8_t* d_out, cudaStream_t st, uint64_t* launches);

// ---------------- join.cu (sort-merge join of a reducer's two sorted sides into Spark's joined UnsafeRows) -----------
// The records of both sides, stably sorted together by the join key (launch_rows_join_order) and grouped
// (launch_rows_group): each group holds its key's left records, then its right ones.  The shape of the joined row:
// field counts n[s], null-bitset words bw[s] and out_bw of the inputs and the output, and the non-fixed fields (VAR and
// DECIMAL_WIDE: their slots' offsets move) of each side, and each side's DECIMAL_WIDE fields (a null side's 16-byte
// regions), as device lists.
constexpr uint32_t kJoinInner = B2S_JOIN_INNER, kJoinLeftOuter = B2S_JOIN_LEFT_OUTER,
                   kJoinLeftSemi = B2S_JOIN_LEFT_SEMI, kJoinLeftAnti = B2S_JOIN_LEFT_ANTI,
                   kJoinRightOuter = B2S_JOIN_RIGHT_OUTER, kJoinFullOuter = B2S_JOIN_FULL_OUTER,
                   kJoinExistence = B2S_JOIN_EXISTENCE;
// a semi or anti join: its output is the kept left records themselves, not joined rows
__host__ __device__ inline bool join_keeps_whole(uint32_t type) {
  return type == kJoinLeftSemi || type == kJoinLeftAnti;
}
struct JoinShape {
  uint32_t type;
  uint64_t split;      // the arena offset of the first right record (JoinKeys::split)
  uint32_t n[2], bw[2], out_bw;
  uint32_t n_var[2], n_wide[2];
  const uint32_t* var[2];
  const uint32_t* wide[2];
  KeySpec keys[2];     // each side's key columns whose null makes a key unmatchable (a null-safe column's is -1)
};
// d_jws: join_ws_bytes(n, n_ranges, n_fields) bytes; launch_join_count uploads the shape and its field lists (h_fields:
// the left's non-fixed fields, the right's, the right's DECIMAL_WIDE ones, the left's DECIMAL_WIDE ones)
size_t join_ws_bytes(uint64_t n, uint32_t n_ranges, uint32_t n_fields);
// the readback: [output records, output bytes, left records, a joined row is too long (0 / 1), verdict of range 0, 1,
// ...] (the verdicts: launch_rows_join_order's)
uint64_t* join_readback(uint8_t* d_jws, uint64_t n, uint32_t n_ranges);
inline size_t join_readback_bytes(uint32_t n_ranges) { return (4 + (size_t)n_ranges) * 8; }
// per sorted position (of either side) its output records and bytes, scanned; the totals and the left record count
// into the readback (its first four words).  idx: the sorted order (nullptr: arena order), heads as
// launch_rows_group's.
void launch_join_count(const uint8_t* arena, uint64_t n, const uint32_t* idx, JoinShape shape,
                       const uint32_t* h_fields, uint32_t n_fields, uint32_t key_bytes, uint8_t* d_ws,
                       uint8_t* d_aws, uint8_t* d_jws, uint32_t n_ranges, cudaStream_t st, uint64_t* launches);
// the out_rows joined records (read back) to d_dst, a warp per record; semi and anti joins (join_keeps_whole): the
// kept left records, compacted and gathered by launch_rows_gather; the existence join: a warp per left record, the
// record with its exists field
void launch_join_emit(const uint8_t* arena, uint64_t n, const uint32_t* idx, uint64_t out_rows, uint32_t key_bytes,
                      uint32_t type, uint8_t* d_ws, uint8_t* d_jws, uint32_t n_ranges, uint8_t* d_dst, cudaStream_t st,
                      uint64_t* launches);

// ---------------- window.cu (Spark's WindowExec ranking and aggregate functions over a reducer's key-sorted rows) -------
// The records, stably sorted by the window's key (partition columns, then order columns: launch_rows_order) and grouped
// by the whole key (launch_rows_group: the peer groups).  The shape of the output row: the input's field count n,
// null-bitset words bw, the output's out_bw = ceil((n + n_fns) / 64), the functions (B2S_WINDOW_*) and their
// arguments, the limit (limit_fn B2S_WINDOW_NO_LIMIT: none), the partition columns (the key's first part.n columns),
// and the input's VAR and DECIMAL_WIDE fields (their slots' offsets move), as a device list.  An aggregate function f
// (fn[f] >= B2S_WINDOW_SUM) has its frame, input type (B2S_WINDOW_VAL_*, a decimal's p and s above), slot and null bit
// (-1: never null), its index agg[f] among the n_agg aggregate functions, and wide[f], its ordinal among the n_wide
// functions with a DECIMAL_WIDE result (-1 for every other function).  An offset function (fn[f] >= B2S_WINDOW_LAG)
// has the same input fields (B2S_WINDOW_VAL_BYTES too), its flags and default slot bits, and nn[f], its index among the
// n_nn non-null indexes (IGNORE_NULLS over a nullable input; -1 for every other function); n_off offset functions, of
// which n_wide_off take a DECIMAL_WIDE input (their values take 16 bytes each, as wide aggregate results do).
constexpr uint32_t kMaxWindowFns = 16;
struct WindowShape {
  uint32_t n, bw, out_bw;
  uint32_t n_fns;
  uint32_t fn[kMaxWindowFns];
  uint32_t arg[kMaxWindowFns];
  uint32_t limit_fn;
  int32_t limit;
  uint32_t n_var;
  const uint32_t* var;
  KeySpec part;
  uint32_t frame[kMaxWindowFns];
  uint32_t vtype[kMaxWindowFns];
  uint32_t voff[kMaxWindowFns];
  int32_t vnull[kMaxWindowFns];
  uint32_t agg[kMaxWindowFns];
  int32_t wide[kMaxWindowFns];
  uint32_t n_agg, n_wide;
  uint32_t flags[kMaxWindowFns];
  uint64_t dflt[kMaxWindowFns];
  int32_t nn[kMaxWindowFns];
  uint32_t n_off, n_nn, n_wide_off;
  // Sliding frames (fn_frame B2S_WINDOW_FRAME_ROWS / _RANGE): function f's frame is bounds set bnd[f] (-1: an older
  // frame), one per distinct (frame, lower, upper): its frame code bkind, and its bounds blo / bhi (INT64_MIN /
  // INT64_MAX unbounded, 0 CURRENT ROW, else the signed offset).  An aggregate whose frame value is not read from the
  // prefix folds has its own result state at index res[f] among n_res (-1 otherwise): a MIN / MAX with a bounded lower
  // end (range-minimum passes over frames of at most rmq_width positions; 0: none, ~0: unbounded) or a double fold with
// one (a fold per row).  The
  // order column of a RANGE offset (ord_type with its flags, slot, width and null bit) is staged when ord_staged.
  int32_t bnd[kMaxWindowFns];
  uint32_t n_bnd;
  uint32_t bkind[kMaxWindowFns];
  int64_t blo[kMaxWindowFns], bhi[kMaxWindowFns];
  int32_t res[kMaxWindowFns];
  uint32_t n_res;
  uint64_t rmq_width;
  bool ord_staged;
  uint32_t ord_type, ord_off, ord_len;
  int32_t ord_null;
};
// d_wws: window_ws_bytes(n, shape) bytes
size_t window_ws_bytes(uint64_t n, const WindowShape& shape);
// the readback: [output records, output bytes, an output row is too long (0 / 1), a partition is too large (0 / 1),
// the first bad DECIMAL_WIDE or string input (its arena offset << 2 | kAggBadDecimal or kWindowBadBytes; ~0: none),
// a sliding frame's bound would wrap in Spark's arithmetic (0 / 1)]
uint64_t* window_readback(uint8_t* d_wws, uint64_t n, const WindowShape& shape);
constexpr size_t kWindowReadbackBytes = 48;
constexpr uint64_t kWindowBadBytes = 2;  // an offset function's string input lies outside its row's var region
// Per sorted position: whether it starts a partition (only peer heads compare their partition columns with their
// predecessor's, encoded 16 bytes at a time), scanned, and the partitions' starts compacted; with aggregate functions,
// their inputs staged and folded from each partition's start; with offset functions that skip nulls, a non-null index
// each (present flags scanned, present positions compacted); then every function's value, whether the limit keeps
// the record and its output bytes, the kept records and bytes scanned, the totals and the verdicts into the readback.
// Uploads the shape and its field list (h_fields: shape.n_var fields).  idx: the sorted order (nullptr: arena order);
// d_aws: launch_rows_group's workspace.
void launch_window_values(const uint8_t* arena, uint64_t n, const uint32_t* idx, WindowShape shape,
                          const uint32_t* h_fields, uint32_t key_bytes, uint8_t* d_ws, uint8_t* d_aws, uint8_t* d_wws,
                          cudaStream_t st, uint64_t* launches);
// the out_rows output records (read back) to d_dst, a warp per record; with a limit the kept positions are compacted
// first, so only they are read
void launch_window_emit(const uint8_t* arena, uint64_t n, const uint32_t* idx, uint64_t out_rows, uint32_t key_bytes,
                        const WindowShape& shape, bool limited, uint8_t* d_ws, uint8_t* d_wws, uint8_t* d_dst,
                        cudaStream_t st, uint64_t* launches);
// The map side's partial limit (WindowGroupLimitExec(Partial)) with a shape of no functions: the partition columns
// (part), limit_fn and limit.  Per sorted position: whether it starts a partition (as launch_window_values finds it),
// its limit_fn value, whether the limit keeps it and its record length when kept; the kept records and bytes scanned,
// and readback words 0, 1 and 3 (the kept records, their bytes, a partition too large).  Uploads the shape.
void launch_window_limit(const uint8_t* arena, uint64_t n, const uint32_t* idx, const WindowShape& shape,
                         uint32_t key_bytes, uint8_t* d_ws, uint8_t* d_aws, uint8_t* d_wws, cudaStream_t st,
                         uint64_t* launches);
// the out_rows kept records (read back), unchanged and in sorted order, to d_out back to back, a warp per record, and
// their lengths to d_out_len; the kept positions are compacted first
void launch_window_limit_gather(const uint8_t* arena, uint64_t n, const uint32_t* idx, uint64_t out_rows,
                                uint32_t key_bytes, const WindowShape& shape, uint8_t* d_ws, uint8_t* d_wws,
                                uint32_t* d_out_len, uint8_t* d_out, cudaStream_t st, uint64_t* launches);

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
