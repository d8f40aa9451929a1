// rows_round_robin.cu — Spark's RoundRobinPartitioning of length-prefixed UnsafeRow records, the map side of
// Dataset.repartition(n) (ShuffleExchangeExec deals a map task's rows out in turn, from a position the task's
// partition id seeds).  With spark.sql.execution.sortBeforeRepartition the task's rows are first sorted by
// (row.hashCode(), RecordBinaryComparator), so that a retried task deals the same rows to the same partitions:
//   hash : a thread per record checks it and hashes its whole row (hashUnsafeWords, seed 42), the first key word of
//          the whole-row sort (rows.cu, launch_rows_whole_*), whose rounds break hash ties by size, then row bytes
//   ids  : a thread per sorted position k: (start + 1 + k) mod R; the partition step's stable radix passes over
//          (id, record) then keep the sorted order inside each partition
#include "kernels.h"
#include "murmur3.cuh"

namespace b2s {

namespace {

constexpr int kRoundRobinThreads = 256;
constexpr uint32_t kRowHashSeed = 42;  // UnsafeRow.hashCode's Murmur3 seed

inline unsigned rr_grid(uint64_t n) {
  const uint64_t want = (n + kRoundRobinThreads - 1) / kRoundRobinThreads;
  return (unsigned)(want < (uint64_t)kSMs * 16 ? (want ? want : 1) : (uint64_t)kSMs * 16);
}

// kernels.h, launch_rows_round_robin_hash.  A record that ends past rec_bytes is not read (the partition step's
// length sum reports it).
__global__ void __launch_bounds__(kRoundRobinThreads) rows_rr_hash_kernel(
    const uint8_t* __restrict__ rec, uint64_t rec_bytes, const uint64_t* __restrict__ rec_off,
    const uint32_t* __restrict__ rec_len, uint64_t n, uint32_t* __restrict__ words, uint32_t* __restrict__ klen,
    unsigned long long* __restrict__ bad) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t o = rec_off[i];
    const uint32_t len = rec_len[i];
    uint32_t h = 0, kl = 0;
    if (o + len <= rec_bytes) {
      uint32_t size = 0;
      if (len >= 4) {
        uint64_t lo, hi;
        ld_span16<true>(rec + o, 4, lo, hi);
        size = __byte_perm((uint32_t)lo, 0, 0x0123);
      }
      const uint64_t why = len < 4 ? kHashBadShort : size != len - 4 ? kHashBadSize : (size & 7) ? kRowsBadWords : 0;
      if (why) {
        atomicMin(bad, (unsigned long long)((i << 3) | why));
      } else if (words) {
        h = hash_bytes(rec + o + 4, size, kRowHashSeed);
        kl = 8 + size;
      }
    }
    if (words) {
      words[i] = h ^ 0x80000000u;
      klen[i] = kl;
    }
  }
}

__global__ void __launch_bounds__(kRoundRobinThreads) rows_rr_ids_kernel(uint64_t n, uint32_t start,
                                                                         uint32_t num_partitions,
                                                                         uint32_t* __restrict__ ids) {
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x)
    ids[k] = (start + 1 + (uint32_t)k) % num_partitions;  // start + 1 + k <= 2^31 - 1
}

}  // namespace

void launch_rows_round_robin_hash(const uint8_t* rec, uint64_t rec_bytes, const uint64_t* rec_off,
                                  const uint32_t* rec_len, uint64_t n, uint32_t* words, uint32_t* klen, uint64_t* bad,
                                  cudaStream_t st, uint64_t* launches) {
  if (!n) return;
  rows_rr_hash_kernel<<<rr_grid(n), kRoundRobinThreads, 0, st>>>(rec, rec_bytes, rec_off, rec_len, n, words, klen,
                                                                 (unsigned long long*)bad);
  if (launches) *launches += 1;
}

void launch_rows_round_robin_ids(uint64_t n, uint32_t start, uint32_t num_partitions, uint32_t* ids, cudaStream_t st,
                                 uint64_t* launches) {
  if (!n) return;
  rows_rr_ids_kernel<<<rr_grid(n), kRoundRobinThreads, 0, st>>>(n, start, num_partitions, ids);
  if (launches) *launches += 1;
}

}  // namespace b2s
