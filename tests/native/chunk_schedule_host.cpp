// Host build of spark-s3-shuffle_b200/csrc/chunk_schedule.h for tests/test_chunk_schedule.py: run_chunks drives stages
// that only record what ran, so the order the host-pointer calls issue their chunk stages and slot retires in can be
// checked without a GPU.  Test infrastructure only — the C ABI never runs this.
#include <vector>

#include "../../spark-s3-shuffle_b200/csrc/chunk_schedule.h"

namespace {
struct FakeSlot {
  int id;
};
}  // namespace

extern "C" {
// Runs n one-stream chunks through stages of the given lags on `slots` slots.  Events go to ev as triples: (0, stage,
// chunk) for a stage, (1, slot, used) for a retire; the call that would be event number fail_at returns 7 instead of
// running (fail_at < 0: none).  Returns the event count and stores run_chunks' result in *rc.
int cs_run(int slots, int nstage, const unsigned long long* lags, int n, int fail_at, int* ev, int* rc) {
  std::vector<FakeSlot> s(slots);
  for (int i = 0; i < slots; i++) s[i].id = i;
  std::vector<uint32_t> starts;
  for (int c = 0; c <= n; c++) starts.push_back((uint32_t)c);
  int count = 0;
  auto record = [&](int kind, int a, int b) {
    if (count == fail_at) return 7;
    ev[3 * count] = kind;
    ev[3 * count + 1] = a;
    ev[3 * count + 2] = b;
    count++;
    return 0;
  };
  std::vector<b2s::ChunkStage<FakeSlot>> stages;
  for (int k = 0; k < nstage; k++)
    stages.push_back({(size_t)lags[k], [&record, k, slots](FakeSlot& slot, size_t c, uint32_t first, uint32_t cnt) {
                        // chunk c holds stream c alone and runs on slot c % slots; 99 reports anything else
                        if (first != c || cnt != 1 || slot.id != (int)(c % (size_t)slots)) return 99;
                        return record(0, k, (int)c);
                      }});
  *rc = b2s::run_chunks(s.data(), slots, starts, stages,
                        [&](FakeSlot& slot, bool used) { return record(1, slot.id, used ? 1 : 0); });
  return count;
}

// chunk_starts over n streams; out receives the starts (at most n + 1), the return value their count
int cs_chunk_starts(uint32_t n, const unsigned long long* len, uint32_t max_streams, unsigned long long max_bytes,
                    uint32_t* out) {
  std::vector<uint64_t> l(len, len + n);
  const std::vector<uint32_t> starts = b2s::chunk_starts(n, l.data(), max_streams, max_bytes);
  for (size_t i = 0; i < starts.size(); i++) out[i] = starts[i];
  return (int)starts.size();
}
}
