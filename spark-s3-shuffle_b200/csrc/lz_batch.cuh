// lz_batch.cuh — copies the LITERALS and executes the MATCH copies of a batch of up to 32 LZ sequences, one lane per
// sequence (device only).  The literal copy is shared by the two LZ decoders, lz4_decode_warp_kernel (lz4_decode.cu)
// and snappy_copy_kernel (snappy.cu); the match copy by those and the Zstandard warp decoder (zstd_core.h under
// B2S_ZSTD_WARP).
//
// Match preconditions: the literals of the whole batch are already in place (and made visible with __syncwarp);
// positions are relative to `out`; lane l's match writes [mdst, mdst+ml) and reads [mdst-off, mdst-off+ml) (ml == 0:
// no match); mdst is non-decreasing with the lane index and the output intervals are disjoint; everything below the
// batch's first output byte is final.
//
// The matches a lane depends on — those whose output intersects its source [msrc, min(msrc+ml, mdst)) (the part of
// the source that is its OWN output is produced by the sequential copy itself) — form a contiguous lane range
// [jlo, jhi], found by two 5-step binary searches over the lane-sorted interval ends / starts.  A lane copies as soon
// as every match in its range is done; the number of rounds is the depth of the dependency chain, not its length.
#pragma once
#include "common.cuh"

namespace b2s {

// The literals of a batch of up to 32 sequences (lane l: lit bytes from in + lip to out + op; lit == 0: none): all
// lanes at once, runs longer than 16 bytes by the whole warp.  Ends with __syncwarp, so the literals are visible to the
// match copies that follow.
__device__ __forceinline__ void lz_copy_literals(const uint8_t* __restrict__ in, uint8_t* out, int lip, int lit, int op,
                                                 int lane) {
  constexpr unsigned FULL = 0xffffffffu;
  if (lit > 0 && lit <= 16) {  // aligned 8-byte words of the compressed block (read-only: __ldg)
    uint64_t lo, hi;
    ld_span16<true>(in + lip, lit, lo, hi);
    st_span16(out + op, lit, lo, hi);
  }
  unsigned biglit = __ballot_sync(FULL, lit > 16);
  while (biglit) {
    const int l = __ffs(biglit) - 1;
    biglit &= biglit - 1;
    const int n_l = __shfl_sync(FULL, lit, l), op_l = __shfl_sync(FULL, op, l), ip_l = __shfl_sync(FULL, lip, l);
    if (n_l >= 96) group_copy<32>(out + op_l, in + ip_l, (uint32_t)n_l, lane);
    else
      for (int j = lane; j < n_l; j += 32) out[op_l + j] = __ldg(in + ip_l + j);
  }
  __syncwarp();
}

// (Tried: moving a short match in groups of four bytes — four independent loads, then four stores — when the group's
// source cannot be its own output: the read pass got slower.  Those were still byte loads; see WIDE below.)
//
// WIDE: a short match (ml <= 16) whose source is apart from its output (off >= ml) reads that source as one to three
// aligned 8-byte words (ld_span16) instead of ml byte loads.  The 32 lanes' sources lie in up to 32 different places,
// so every warp-wide load instruction touches up to 32 sectors; fewer, wider loads cut those instructions (and their
// round trips) by the match length.  The Zstandard executor passes WIDE = false and keeps the byte loop: inlined into
// its larger kernel, the wide copy raised the register count from 64 to 80 and its execute stage measured slower.
template <bool WIDE>
__device__ __forceinline__ void lz_execute_matches(uint8_t* out, int mdst, int ml, int off, int lane) {
  constexpr unsigned FULL = 0xffffffffu;
  const int msrc = mdst - off;
  const int mend = mdst + ml;  // non-decreasing across lanes (ml == 0: empty interval)
  const int send = msrc + ml < mdst ? msrc + ml : mdst;
  const unsigned matchmask = __ballot_sync(FULL, ml > 0);
  if (!matchmask) return;
  int jlo = 0, jhi1 = 0;  // first lane whose output ends above msrc ; number of lanes whose output starts below send
#pragma unroll
  for (int step = 16; step >= 1; step >>= 1) {
    const int e = __shfl_sync(FULL, mend, jlo + step - 1);
    const int b = __shfl_sync(FULL, mdst, jhi1 + step - 1);
    if (e <= msrc) jlo += step;
    if (b < send) jhi1 += step;
  }
  // (32 lanes: the searches cover indices 0..30; lane 31 can only matter to itself)
  unsigned need = 0;
  if (ml > 0) {
    const int hi = jhi1 < lane ? jhi1 : lane;  // exclusive upper bound, only lanes below me
    if (jlo < hi) need = (((1u << hi) - 1u) & ~((1u << jlo) - 1u)) & matchmask;
  }
  unsigned done = ~matchmask;
  bool pending = ml > 0;
  while (done != FULL) {
    const bool ready = pending && (need & ~done) == 0;
    if (ready && ml <= 16) {
      if (WIDE && off >= ml) {  // the source is complete and apart from the output: read it in aligned 8-byte words
        uint64_t lo, hi;
        ld_span16<false>(out + msrc, ml, lo, hi);  // plain loads: `out` is written by this warp
        st_span16(out + mdst, ml, lo, hi);
      } else {
        // overlapping match (off < ml): sequential byte copy, later bytes are read from bytes it has just written
        for (int j = 0; j < ml; j++) out[mdst + j] = out[msrc + j];
      }
    }
    unsigned longmask = __ballot_sync(FULL, ready && ml > 16);
    while (longmask) {
      const int l = __ffs(longmask) - 1;
      longmask &= longmask - 1;
      const int ml_l = __shfl_sync(FULL, ml, l), off_l = __shfl_sync(FULL, off, l);
      uint8_t* o = out + __shfl_sync(FULL, mdst, l);
      const uint8_t* sp = o - off_l;
      if (off_l >= ml_l) {  // disjoint source: plain cooperative copy
        if (ml_l >= 96) group_copy<32>(o, sp, (uint32_t)ml_l, lane);
        else
          for (int j = lane; j < ml_l; j += 32) o[j] = sp[j];
      } else if (off_l == 1) {  // byte run (the commonest overlapping match)
        const uint8_t v = sp[0];
        for (int j = lane; j < ml_l; j += 32) o[j] = v;
      } else {
        // overlapping match (off < ml): every byte comes from the already complete window [o - off, o)
        for (int j = lane; j < ml_l; j += 32) o[j] = sp[(unsigned)j % (unsigned)off_l];
      }
    }
    done |= __ballot_sync(FULL, ready);
    pending = pending && !ready;
    __syncwarp();  // this round's bytes are visible to the next round's loads
  }
}

}  // namespace b2s
