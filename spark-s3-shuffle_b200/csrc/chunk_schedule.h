// chunk_schedule.h — the chunks of a host-pointer call (compress_host, decompress_host in api.cu) and the order of
// their pipeline stages over rotating slots.  No CUDA: tests/test_chunk_schedule.py checks the order with g++.
#pragma once
#include <cstdint>
#include <functional>
#include <utility>
#include <vector>

namespace b2s {

// Chunk c holds streams [starts[c], starts[c + 1]): up to max_streams streams and max_bytes bytes, or one longer one.
inline std::vector<uint32_t> chunk_starts(uint32_t n, const uint64_t* len, uint32_t max_streams, uint64_t max_bytes) {
  std::vector<uint32_t> starts;
  for (uint32_t i = 0; i < n;) {
    starts.push_back(i);
    uint64_t bytes = 0;
    for (uint32_t cnt = 0; i < n && cnt < max_streams && (cnt == 0 || bytes + len[i] <= max_bytes); cnt++)
      bytes += len[i++];
  }
  starts.push_back(n);
  return starts;
}

// {lag, run}: step t calls run(slot, chunk, first stream, stream count) for chunk t - lag
template <class Slot>
using ChunkStage = std::pair<size_t, std::function<int(Slot&, size_t, uint32_t, uint32_t)>>;

// Runs every chunk through `stages` (lags increasing from 0) on slots[0 .. nslot), chunk c on slot c % nslot; step t
// runs each stage for chunk t - lag, in stage order.  Slot reuse: stage 0 of chunk c restages its slot (the staged
// sources, and the pinned block whose statuses, lengths and offsets later stages read), so every stage of chunk
// c - nslot runs before it (a lag of nslot or more: first in step c, past the last chunk too), and then
// retire(slot, true) waits for that chunk's queued work.  At the end retire(slots[s], s < chunk count) drains every
// slot.  The first non-zero return of a stage or of retire ends the run and is returned.
template <class Slot, class Retire>
int run_chunks(Slot* slots, int nslot, const std::vector<uint32_t>& starts, const std::vector<ChunkStage<Slot>>& stages,
               Retire&& retire) {
  const size_t n = starts.size() - 1, ns = (size_t)nslot;
  auto call = [&](const auto& run, size_t c) { return run(slots[c % ns], c, starts[c], starts[c + 1] - starts[c]); };
  for (size_t t = 0; t < n + stages.back().first; t++) {
    for (const auto& [lag, run] : stages)
      if (lag >= ns && t >= ns && t - ns < n)
        if (int rc = call(run, t - ns)) return rc;
    if (t >= ns && t < n)
      if (int rc = retire(slots[t % ns], true)) return rc;
    for (const auto& [lag, run] : stages)
      if (lag < ns && t >= lag && t - lag < n)
        if (int rc = call(run, t - lag)) return rc;
  }
  for (size_t s = 0; s < ns; s++)
    if (int rc = retire(slots[s], s < n)) return rc;
  return 0;
}

}  // namespace b2s
