// api.cu — runtime + C ABI of libb200shuffle.so (see include/b200shuffle.h for the contract and the reference
// interfaces each entry point replaces).
//
// Structure: a process-wide context with one Device per selected GPU.  A Device runs two lanes (write side, read side),
// each with up to NSLOT pipeline slots; a slot is a pair of CUDA streams plus grow-only device buffers (staged
// source/destination arenas, descriptor "meta" block, codec scratch) and a pinned host block for descriptor traffic.
// Host-pointer entry points cut a batch into chunks of ~256 MiB, and run H2D -> kernels -> (size readback) -> D2H per
// chunk on rotating slots so copies of one chunk overlap kernels of another.  "_dev" entry points run the same
// kernel sequence on caller-owned device arenas.
// There is no CPU fallback anywhere in this file: without a device every compute entry point fails with B2S_E_CUDA.
#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <optional>
#include <string>
#include <thread>
#include <vector>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "chunk_schedule.h"
#include "kernels.h"

using namespace b2s;

namespace {

thread_local std::string t_last_error;
thread_local b2s_timing t_timing;
// the timed call this thread is running (begin_call): marks and dominant pairs another call recorded are never read
thread_local uint64_t t_call = 0;
std::atomic<uint64_t> g_calls{0};
thread_local uint32_t t_device = 0;  // device (index into the b2s_init selection) used by this thread's host-pointer calls

int fail(int code, const char* fmt, const char* a = "") {
  char buf[512];
  snprintf(buf, sizeof buf, fmt, a);
  t_last_error = buf;
  return code;
}
int fail_cuda(const char* what, cudaError_t e) {
  t_last_error = std::string(what) + ": " + cudaGetErrorString(e);
  return B2S_E_CUDA;
}
#define CU(call)                                           \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) return fail_cuda(#call, e__);  \
  } while (0)

constexpr int NSLOT = 8;  // upper bound; g_nslot (b2s_init streams_per_gpu, default 6) are used
int g_nslot = 6;
uint64_t g_host_chunk_bytes = 256ull << 20;  // host-pointer calls: bytes per pipeline chunk (B2S_HOST_CHUNK_MB).  The thread-per-block
                                              // kernels cost ~2 ms per launch whatever the block count, so chunks must be large enough to amortise them
constexpr uint32_t kChunkStreams = 1u << 18;
constexpr uint32_t kXxhSeed = 0x9747b28cu;
uint32_t g_lz4_chunk_blocks = 32768;  // codec blocks per match/parse/emit (or tokens/copy) pass: bounds the workspace; B2S_LZ4_CHUNK_BLOCKS
uint32_t g_lz4d_chunk_blocks = 65536;  // Snappy decode only (LZ4 decodes in one launch): codec blocks per token walk + copy pair; the walk is latency bound, more blocks per launch = more loads in flight; B2S_LZ4D_CHUNK_BLOCKS

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int g_read_lag = 1;            // B2S_READ_LAG: chunks between the stages of the read pipeline (upload+sizes | decode | download)

// --------------------------------------------------------------------------------------------------------------
// NUMA placement of pinned staging (SURVEY.md §8e: "NUMA-pin staging buffers to the GPU's socket").  On the 8-GPU boxes
// GPUs 0-3 hang off socket 0 and 4-7 off socket 1; pinned arenas that land on the other socket send every H2D/D2H
// byte across the socket interconnect, which is what capped the host-staged path at 4 and 8 ranks (VERDICT round 1).
// Raw syscalls (no libnuma in the image).  B2S_NUMA=0 disables all of it.
// --------------------------------------------------------------------------------------------------------------
int g_numa = 1;
namespace numa {
constexpr int kDefault = 0, kPreferred = 1;
constexpr unsigned long kMaskBits = 1024;
struct Mask {
  unsigned long w[kMaskBits / (8 * sizeof(unsigned long))] = {};
};
inline long set_policy(int mode, const Mask* m) {
  return syscall(SYS_set_mempolicy, mode, m ? m->w : nullptr, m ? kMaskBits + 1 : 0ul);
}
inline long get_policy(int* mode, Mask* m) {
  return syscall(SYS_get_mempolicy, mode, m->w, kMaskBits + 1, nullptr, 0ul);
}
int node_of_pci(const char* busid) {  // "0000:40:00.0" -> /sys/bus/pci/devices/0000:40:00.0/numa_node
  char path[256], low[64];
  size_t k = 0;
  for (; busid[k] && k + 1 < sizeof low; k++) low[k] = (char)((busid[k] >= 'A' && busid[k] <= 'F') ? busid[k] + 32 : busid[k]);
  low[k] = 0;
  snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", low);
  FILE* f = fopen(path, "r");
  if (!f) return -1;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  return node;
}
bool node_cpus(int node, cpu_set_t* set) {  // parses /sys/devices/system/node/nodeN/cpulist ("0-31,64-95")
  char path[128], buf[4096];
  snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
  FILE* f = fopen(path, "r");
  if (!f) return false;
  const bool got = fgets(buf, sizeof buf, f) != nullptr;
  fclose(f);
  if (!got) return false;
  CPU_ZERO(set);
  int count = 0;
  for (char* q = buf; *q && *q != '\n';) {
    char* e = nullptr;
    long a = strtol(q, &e, 10), b = a;
    if (e == q) break;
    q = e;
    if (*q == '-') {
      b = strtol(q + 1, &e, 10);
      q = e;
    }
    for (long c = a; c <= b && c < CPU_SETSIZE; c++) {
      CPU_SET((int)c, set);
      count++;
    }
    if (*q == ',') q++;
  }
  return count > 0;
}
// allocations made while one of these is alive come from `node` when it has room (MPOL_PREFERRED); the thread's
// previous policy is put back afterwards
struct PreferNode {
  bool active = false;
  int old_mode = 0;
  Mask old_mask;
  explicit PreferNode(int node) {
    if (!g_numa || node < 0 || node >= (int)kMaskBits) return;
    if (get_policy(&old_mode, &old_mask) != 0) return;
    Mask m;
    m.w[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    active = set_policy(kPreferred, &m) == 0;
  }
  ~PreferNode() {
    if (active) set_policy(old_mode, old_mode == kDefault ? nullptr : &old_mask);
  }
};
}  // namespace numa
thread_local int t_numa_node = -1;  // node of the device this thread's pinned allocations should sit next to

bool exchange_shed_current_device();  // exchange cache (below): frees the current device's unreferenced entries

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = align_up(bytes + bytes / 8, 1 << 20);
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();  // an allocation failure is reported as B2S_E_NOMEM, not left for a later CU() check
      e = cudaMalloc(&p, bytes);
      want = bytes;
    }
    // a workspace never fails for want of memory the exchange cache holds: it gives back what no read uses, once
    if (e != cudaSuccess && exchange_shed_current_device()) {
      (void)cudaGetLastError();
      e = cudaMalloc(&p, bytes);
    }
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      p = nullptr;
      return fail(B2S_E_NOMEM, "cudaMalloc: %s", cudaGetErrorString(e));
    }
    cap = want;
    return 0;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};
struct PinBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    size_t want = align_up(bytes + bytes / 4, 1 << 16);
    numa::PreferNode near(t_numa_node);
    cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();  // reported as B2S_E_NOMEM, not left for a later CU() check
      p = nullptr;
      return fail(B2S_E_NOMEM, "cudaHostAlloc: %s", cudaGetErrorString(e));
    }
    cap = want;
    return 0;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
};

// bump allocator over one buffer
struct Carver {
  uint8_t* base;
  size_t off = 0;
  explicit Carver(void* b) : base((uint8_t*)b) {}
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 16);
    T* r = (T*)(base + off);
    off += n * sizeof(T);
    return r;
  }
};

double ms_between(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0;
  if (cudaEventElapsedTime(&ms, a, b) != cudaSuccess) {
    (void)cudaGetLastError();  // unrecorded event: not an error of the call being timed
    return 0;
  }
  return ms;
}

// The timed marks of a slot's main stream, which b2s_last_timing is read from (add_times): kernel region (K), codec
// step (T), upload (H), download (D), partition or sort step (P), row framing: walk + count, emit (F0-F1, F2-F3; the
// hash step of a hash partition, the range step of a range partition, the round-robin step: F0-F1), grouping + merge
// of an aggregation (G).  Stop: where a call that did not record the end of a span it reads stopped.
enum Mark { K0, K1, T0, T1, H0, H1, D0, D1, P0, P1, F0, F1, F2, F3, G0, G1, kStop, kMarks };

struct Slot {
  cudaStream_t st = nullptr;
  cudaStream_t st2 = nullptr;                               // side stream: match kernels of chunk k+1 overlap parse/emit of chunk k
  cudaEvent_t ev_fork = nullptr, ev_match[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;              // readback milestones
  cudaEvent_t ev_mark[kMarks] = {};
  uint64_t mark_call[kMarks] = {};      // the call (t_call) that last recorded each mark
  uint64_t mark_launches[kMarks] = {};  // the call's launch count at the mark, where the step passed it
  DevBuf meta, scratch, desc, src, dst, zmeta;
  DevBuf pws, parena;  // partition workspace (sort keys, offsets) and the partitioned arena in front of compression
  DevBuf xpieces;      // the copy pieces of an exchange-cache read (exchange.cu)
  DevBuf fws;          // row framing workspace: bitmap over the decoded arena, tile counts, verdicts (rows.cu)
  DevBuf aggrows;      // a partial aggregation's partial rows (partial_agg.cu) or a window limit's kept rows and their
                       // lengths (window.cu), in front of the partition step
  DevBuf xrows;        // grouping sets: the projected records' lengths, then the records (rows_expand.cu)
  PinBuf hmeta;
  // per-launch event pairs around the dominant kernel of a call (grow-only pool; dom_used pairs of call dom_call)
  std::vector<cudaEvent_t> ev_dom;
  size_t dom_used = 0;
  uint64_t dom_call = 0;
  int dom_pair(cudaEvent_t* a, cudaEvent_t* b) {
    if (dom_call != t_call) dom_used = 0;  // what another call left is not this call's
    dom_call = t_call;
    if (dom_used * 2 + 2 > ev_dom.size()) {
      cudaEvent_t x = nullptr, y = nullptr;
      if (cudaEventCreate(&x) != cudaSuccess || cudaEventCreate(&y) != cudaSuccess) return -1;
      ev_dom.push_back(x);
      ev_dom.push_back(y);
    }
    *a = ev_dom[dom_used * 2];
    *b = ev_dom[dom_used * 2 + 1];
    dom_used++;
    return 0;
  }
  // adds this call's dominant pairs to b2s_last_timing and empties the pool
  void take_pairs() {
    const size_t n = dom_call == t_call ? dom_used : 0;
    for (size_t k = 0; k < n; k++) t_timing.dominant_ms += ms_between(ev_dom[2 * k], ev_dom[2 * k + 1]);
    t_timing.dominant_launches += n;
    dom_used = 0;
  }
  cudaError_t mark(Mark m, cudaStream_t s, uint64_t launches = 0) {
    mark_call[m] = t_call;
    mark_launches[m] = launches;
    return cudaEventRecord(ev_mark[m], s);
  }
  bool mine(Mark m) const { return mark_call[m] == t_call; }
  // this call's ms from a to b: 0 when the call did not record a; up to where the call stopped when it did not record b
  // (the stop mark, recorded and waited for once)
  double span(Mark a, Mark b) {
    if (!mine(a)) return 0;
    if (!mine(b)) {
      if (!mine(kStop) && (mark(kStop, st) != cudaSuccess || cudaEventSynchronize(ev_mark[kStop]) != cudaSuccess)) {
        (void)cudaGetLastError();  // the call's work is done: an unreadable time is 0, not a failure
        return 0;
      }
      b = kStop;
    }
    return ms_between(ev_mark[a], ev_mark[b]);
  }
  // the fixed events, created by create() and destroyed by release(); the first kUntimed only order the two streams
  static constexpr int kUntimed = 5;
  std::array<cudaEvent_t*, 7 + kMarks> events() {
    std::array<cudaEvent_t*, 7 + kMarks> e{&ev_fork, &ev_match[0], &ev_match[1], &ev_free[0], &ev_free[1], &ev_a, &ev_b};
    for (int m = 0; m < kMarks; m++) e[7 + m] = &ev_mark[m];
    return e;
  }
  int create(int prio) {
    CU(cudaStreamCreateWithPriority(&st, cudaStreamNonBlocking, prio));
    CU(cudaStreamCreateWithPriority(&st2, cudaStreamNonBlocking, prio));
    const auto evs = events();
    for (int k = 0; k < (int)evs.size(); k++)
      CU(k < kUntimed ? cudaEventCreateWithFlags(evs[k], cudaEventDisableTiming) : cudaEventCreate(evs[k]));
    return 0;
  }
  // frees whatever the slot holds (buffers, events, streams); a slot that was never created holds nothing
  void release() {
    for (DevBuf* b : {&meta, &scratch, &desc, &src, &dst, &zmeta, &pws, &parena, &xpieces, &fws, &aggrows, &xrows}) b->release();
    hmeta.release();
    for (cudaEvent_t* e : events())
      if (*e) cudaEventDestroy(*e);
    for (cudaEvent_t e : ev_dom) cudaEventDestroy(e);
    ev_dom.clear();
    if (st2) cudaStreamDestroy(st2);
    if (st) cudaStreamDestroy(st);
  }
};

// A device runs two independent LANES: write-side calls (compress) take lane 0, read-side calls (decompress,
// checksum) lane 1.  Each lane has its own lock, pipeline slots, streams and staging, so a map task's compress call
// (H2D-heavy) and a reduce task's decompress call (D2H-heavy) from different threads overlap on the full-duplex PCIe
// link instead of queueing behind one per-device mutex (VERDICT round 1: the two directions were never busy together).
constexpr int kLaneWrite = 0, kLaneRead = 1, kLanes = 2;
struct Lane {
  Slot slot[NSLOT];
  std::mutex mtx;
};
struct Device {
  int ordinal = 0;
  int numa_node = -1;            // /sys/bus/pci/devices/<bdf>/numa_node, -1 = unknown
  Lane lane[kLanes];
  ChecksumTables tabs{};
  void* zstd_ctables = nullptr;  // predefined FSE compression tables (zstd_enc.cu)
  cudaEvent_t ev_mark[2] = {nullptr, nullptr};  // b2s_mark stopwatch
};

struct Context {
  std::vector<Device*> devs;
  std::atomic<uint64_t> launches{0};
};
Context* g_ctx = nullptr;
std::mutex g_init_mtx;

int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v && *v ? atoi(v) : dflt;
}

uint32_t block_size_or_default(uint32_t bs) { return bs ? bs : 32768u; }

// B2S_E_CUDA (and the reason) when the process sees no CUDA device; otherwise 0 and, when asked, the device count
int no_device(int* count_out = nullptr) {
  int count = 0;
  const cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0)
    return fail(B2S_E_CUDA, "no CUDA device: %s", e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
  if (count_out) *count_out = count;
  return 0;
}

// pick the checksum work-item size: enough items to fill the machine, big enough to amortise the combine
uint32_t pick_tile_shift(uint64_t total_bytes) {
  uint32_t s = 20;  // 1 MiB
  const uint64_t want_items = (uint64_t)kSMs * 32 * 4;
  while (s > 14 && (total_bytes >> s) < want_items) s--;
  return s;
}

struct WallTimer {
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  double ms() const { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
};

// Starts a timed call: a new call id, an empty b2s_last_timing and the wall clock
WallTimer begin_call() {
  t_call = ++g_calls;
  t_timing = b2s_timing{};
  return WallTimer{};
}

// --------------------------------------------------------------------------------------------------------------
// compress job: one chunk of n streams living in a device source arena
// --------------------------------------------------------------------------------------------------------------
// bytes every stream adds around its codec blocks: LZ4Block end mark (21) / xerial stream header (16)
inline uint64_t stream_overhead(uint32_t codec) {
  return codec == B2S_CODEC_SNAPPY_XERIAL ? 16ull : codec == B2S_CODEC_ZSTD ? 9ull : 21ull;  // + zstd: frame header 6 + end block 3
}

// A compress chunk's descriptor block: the upload region (copied host -> device in one piece), the download region
// (device -> host in one piece), then, on the device only, the work arrays.  The pinned block and the device "meta"
// block are both carved by compress_layout, so the two copies move the same arrays.
struct CompressLayout {
  uint8_t *up = nullptr, *down = nullptr;
  size_t up_bytes = 0, down_bytes = 0;
  uint64_t *src_off = nullptr, *src_len = nullptr;  // upload
  uint32_t* blk_base = nullptr;
  uint64_t *dst_off = nullptr, *dst_len = nullptr, *cks = nullptr, *total = nullptr;  // download
  int32_t* status = nullptr;
  uint32_t *csize = nullptr, *hash = nullptr, *nseq = nullptr;  // device only
  uint64_t *sizes = nullptr, *work_base = nullptr, *ws = nullptr;
  unsigned int* counter = nullptr;
};
// ws_elems < 0: the pinned block, which ends after the download region
CompressLayout compress_layout(void* base, uint32_t n, uint32_t nb, ptrdiff_t ws_elems) {
  CompressLayout L;
  Carver c(base);
  L.up = (uint8_t*)c.take<uint64_t>(0);
  L.src_off = c.take<uint64_t>(n);
  L.src_len = c.take<uint64_t>(n);
  L.blk_base = c.take<uint32_t>(n + 1);
  c.off = align_up(c.off, 16);
  L.up_bytes = c.off;
  L.down = (uint8_t*)c.take<uint64_t>(0);
  L.dst_off = c.take<uint64_t>(n);
  L.dst_len = c.take<uint64_t>(n);
  L.cks = c.take<uint64_t>(n);
  L.total = c.take<uint64_t>(2);
  L.status = c.take<int32_t>(n);
  c.off = align_up(c.off, 16);
  L.down_bytes = c.off - L.up_bytes;
  if (ws_elems < 0) return L;
  L.csize = c.take<uint32_t>(nb);
  L.hash = c.take<uint32_t>(nb);
  L.nseq = c.take<uint32_t>(nb);
  L.sizes = c.take<uint64_t>((size_t)nb + 1);
  L.work_base = c.take<uint64_t>((size_t)n + 1);
  L.ws = c.take<uint64_t>((size_t)ws_elems);
  L.counter = c.take<unsigned int>(4);
  return L;
}

// a compress chunk: h is the pinned block (the host reads dst_off, dst_len, cks, total and status there after ev_a),
// d the device meta block
struct CompressJob {
  uint32_t n = 0, nb = 0;
  CompressLayout h, d;
};

// codec and codec block size a compress job accepts
int check_codec_block(uint32_t codec, uint32_t bs) {
  if (codec != B2S_CODEC_LZ4BLOCK && codec != B2S_CODEC_SNAPPY_XERIAL && codec != B2S_CODEC_ZSTD)
    return fail(B2S_E_UNSUPPORTED, "codec %s not supported by this build", "");
  if (codec != B2S_CODEC_SNAPPY_XERIAL && (bs < 64 || bs > 65536))
    return fail(B2S_E_UNSUPPORTED, "lz4 / zstd block size must be in [64, 65536]%s");
  if (codec == B2S_CODEC_SNAPPY_XERIAL && (bs < 64 || bs > 32768))
    return fail(B2S_E_UNSUPPORTED, "snappy block size must be in [64, 32768]%s");
  return 0;
}

// Compression level.  LZ4Block and Snappy have none in the reference either (lz4-java's fast compressor, snappy-java);
// for Zstandard (spark.io.compression.zstd.level, codec chosen at storage/S3ShuffleReader.scala:57-60) the level sets the
// match finder's hash-table size: 1 -> 2^11 entries per block (fastest), 2 / unspecified -> 2^12, >= 3 -> 2^13 (more
// shared memory per warp, fewer resident warps, more matches found).
int hlog_for_level(uint32_t codec, int32_t level) {
  if (codec != B2S_CODEC_ZSTD || level <= 0) return 0;
  return level == 1 ? 11 : level == 2 ? 12 : 13;
}

// Runs codec blocks [0, nb) in groups of `group`, group k in workspace par = k & 1 (ws_bytes at ws0): first(b0, m, ws,
// par, e0, e1) enqueues its first pass on S.st2, second(...) its second pass on S.st, beside the first pass of group
// k+1.  e0 / e1 (S.dom_pair) time whichever pass the caller counts as dominant.  The caller has forked S.st2 from S.st.
template <class First, class Second>
int run_block_groups(Slot& S, uint32_t nb, uint32_t group, uint8_t* ws0, size_t ws_bytes, First first, Second second) {
  for (uint32_t b0 = 0, k = 0; b0 < nb; b0 += group, k++) {
    const uint32_t m = std::min<uint32_t>(group, nb - b0);
    const int par = (int)(k & 1);
    uint8_t* ws = ws0 + (size_t)par * ws_bytes;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    S.dom_pair(&e0, &e1);
    if (k >= 2) CU(cudaStreamWaitEvent(S.st2, S.ev_free[par], 0));  // group k-2's second pass has released ws
    if (int rc = first(b0, m, ws, par, e0, e1)) return rc;
    CU(cudaEventRecord(S.ev_match[par], S.st2));
    CU(cudaStreamWaitEvent(S.st, S.ev_match[par], 0));
    if (int rc = second(b0, m, ws, par, e0, e1)) return rc;
    CU(cudaEventRecord(S.ev_free[par], S.st));
  }
  return 0;
}

// Enqueues the compression of n streams at d_src + src_off[i] (src_len[i] bytes) into d_dst on S.st.  The results
// are in J.h once ev_a has completed.
int compress_chunk(Slot& S, const ChecksumTables& tabs, uint32_t codec, int32_t level, uint32_t bs, uint32_t alg,
                   uint32_t n, const uint64_t* src_off, const uint64_t* src_len, const uint8_t* d_src, uint8_t* d_dst,
                   uint64_t dst_cap, CompressJob& J, uint64_t* launches) {
  if (int rc = check_codec_block(codec, bs)) return rc;
  uint64_t nb64 = 0;
  for (uint32_t i = 0; i < n; i++) nb64 += (src_len[i] + bs - 1) / bs;
  if (nb64 >= 0x7fffffffull) return fail(B2S_E_ARG, "too many codec blocks in one chunk%s");
  const uint32_t nb = (uint32_t)nb64;
  J.n = n;
  J.nb = nb;
  size_t up = align_up(n * 8, 16) * 2 + align_up((n + 1) * 4, 16);
  size_t down = align_up(n * 8, 16) * 3 + 16 + align_up(n * 4, 16);
  int rc = S.hmeta.ensure(up + down + 64);
  if (rc) return rc;
  J.h = compress_layout(S.hmeta.p, n, nb, -1);
  memcpy(J.h.src_off, src_off, (size_t)n * 8);
  memcpy(J.h.src_len, src_len, (size_t)n * 8);
  uint64_t acc = 0;
  for (uint32_t i = 0; i < n; i++) {
    J.h.blk_base[i] = (uint32_t)acc;
    acc += (src_len[i] + bs - 1) / bs;
  }
  J.h.blk_base[n] = (uint32_t)acc;

  const uint32_t chunk = std::min<uint32_t>(nb ? nb : 1, g_lz4_chunk_blocks);
  size_t ws_elems = std::max(scan_ws_elems(nb + 1), checksum_ws_elems(n)) + 4;
  size_t need = J.h.up_bytes + J.h.down_bytes + align_up((size_t)nb * 4, 16) * 3 + align_up(((size_t)nb + 1) * 8, 16) +
                align_up(((size_t)n + 1) * 8, 16) + ws_elems * 8 + 256;
  rc = S.meta.ensure(need);
  if (rc) return rc;
  const size_t ws_bytes = align_up(lz4_compress_ws_bytes(chunk, bs, codec), 256);
  rc = S.scratch.ensure(ws_bytes * (nb > chunk ? 2 : 1));
  if (rc) return rc;
  const CompressLayout M = J.d = compress_layout(S.meta.p, n, nb, (ptrdiff_t)ws_elems);

  cudaStream_t st = S.st;
  CU(cudaMemcpyAsync(M.up, J.h.up, M.up_bytes, cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(M.down, 0, M.down_bytes, st));
  CU(S.mark(K0, st));
  CU(S.mark(T0, st));
  // Match kernels (issue bound, shared-memory limited) on the side stream, parse (latency bound), scan and emit on st.
  // The side stream forks BEFORE the per-block XXH32 pass (LZ4Block headers; only the emit kernel needs it), so that
  // pass runs beside the first group's match kernel instead of in front of it.
  CU(cudaEventRecord(S.ev_fork, st));
  CU(cudaStreamWaitEvent(S.st2, S.ev_fork, 0));
  if (codec == B2S_CODEC_LZ4BLOCK)
    launch_xxh32_encode(d_src, M.src_off, M.src_len, M.blk_base, n, nb, bs, kXxhSeed, M.hash, st, launches);
  CU(cudaMemsetAsync(M.total, 0, 16, st));
  auto match = [&](uint32_t b0, uint32_t m, uint8_t* ws, int par, cudaEvent_t e0, cudaEvent_t e1) {
    launch_lz4_match(d_src, M.src_off, M.src_len, M.blk_base, n, b0, m, bs, codec, ws, M.counter + par, S.st2, launches,
                     e0, e1, hlog_for_level(codec, level));
    return 0;
  };
  auto parse_emit = [&](uint32_t b0, uint32_t m, uint8_t* ws, int, cudaEvent_t, cudaEvent_t) {
    launch_lz4_parse_emit(d_src, M.src_off, M.src_len, M.blk_base, n, b0, m, bs, codec, ws, M.nseq, M.csize, M.hash,
                          M.sizes, M.total, M.ws, d_dst, dst_cap, st, launches);
    return 0;
  };
  if (int r = run_block_groups(S, nb, chunk, (uint8_t*)S.scratch.p, ws_bytes, match, parse_emit)) return r;
  CU(S.mark(T1, st));
  if (codec == B2S_CODEC_ZSTD)
    launch_zstd_stream_meta(M.blk_base, n, nb, M.sizes, M.total, d_dst, dst_cap, M.dst_off, M.dst_len, M.status, st,
                            launches);
  else if (codec == B2S_CODEC_SNAPPY_XERIAL)
    launch_xerial_stream_meta(M.blk_base, n, nb, M.sizes, M.total, d_dst, dst_cap, M.dst_off, M.dst_len, M.status, st,
                              launches);
  else
    launch_lz4block_stream_meta(M.blk_base, n, nb, bs, M.sizes, M.total, d_dst, dst_cap, M.dst_off, M.dst_len,
                                M.status, st, launches);
  if (alg != B2S_CHECKSUM_NONE) {
    uint32_t shift = pick_tile_shift(dst_cap < (uint64_t)nb * bs ? dst_cap : (uint64_t)nb * bs);
    launch_checksum(tabs, alg, d_dst, M.dst_off, M.dst_len, n, shift, M.work_base, M.ws, M.cks, st, launches);
  }
  CU(S.mark(K1, st));
  CU(cudaMemcpyAsync(J.h.down, M.down, M.down_bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(S.ev_a, st));
  CU(cudaGetLastError());
  return 0;
}

// --------------------------------------------------------------------------------------------------------------
// decompress job
// --------------------------------------------------------------------------------------------------------------
// A decompress chunk's descriptor block, carved like a compress chunk's (compress_layout): upload region, download
// region, device-only work arrays.  dst_len is the decoded length of every stream.
struct DecompressLayout {
  uint8_t *up = nullptr, *down = nullptr;
  size_t up_bytes = 0, down_bytes = 0;
  uint64_t *src_off = nullptr, *src_len = nullptr, *slice_off = nullptr, *slice_len = nullptr, *slice_sum = nullptr;
  uint32_t *slice_owner = nullptr, *slice_base = nullptr;  // upload
  uint64_t* totals = nullptr;  // download: [nb_total, olen_total, Snappy: largest chunk olen, clen]
  uint64_t *dst_off = nullptr, *dst_len = nullptr;
  int32_t *status = nullptr, *bad = nullptr;
  uint64_t *nblk = nullptr, *cks_got = nullptr, *work_base = nullptr, *ws = nullptr;  // device only
  unsigned int* counter = nullptr;
};
// ws_elems < 0: the pinned block, which ends after the download region
DecompressLayout decompress_layout(void* base, uint32_t n, uint32_t s, ptrdiff_t ws_elems) {
  DecompressLayout L;
  Carver c(base);
  L.up = (uint8_t*)c.take<uint64_t>(0);
  L.src_off = c.take<uint64_t>(n);
  L.src_len = c.take<uint64_t>(n);
  L.slice_off = c.take<uint64_t>(s);
  L.slice_len = c.take<uint64_t>(s);
  L.slice_sum = c.take<uint64_t>(s);
  L.slice_owner = c.take<uint32_t>(s);
  L.slice_base = c.take<uint32_t>((size_t)n + 1);
  c.off = align_up(c.off, 16);
  L.up_bytes = c.off;
  L.down = (uint8_t*)c.take<uint64_t>(0);
  L.totals = c.take<uint64_t>(4);
  L.dst_off = c.take<uint64_t>(n);
  L.dst_len = c.take<uint64_t>(n);
  L.status = c.take<int32_t>(n);
  L.bad = c.take<int32_t>(n);
  c.off = align_up(c.off, 16);
  L.down_bytes = c.off - L.up_bytes;
  if (ws_elems < 0) return L;
  L.nblk = c.take<uint64_t>(n);
  L.cks_got = c.take<uint64_t>(s);
  L.work_base = c.take<uint64_t>((size_t)s + 1);
  L.ws = c.take<uint64_t>((size_t)ws_elems);
  L.counter = c.take<unsigned int>(4);
  return L;
}

// a decompress chunk: h is the pinned block (the host reads totals after ev_a, the rest after ev_b), d the device
// meta block
struct DecompressJob {
  uint32_t n = 0, n_slices = 0, codec = 0;
  uint64_t nb = 0, total_out = 0;
  DecompressLayout h, d;
  // zstd: per-stream counts / bases (blocks, sequences, literal bytes) and their totals
  uint64_t *zcnt = nullptr, *zbase = nullptr;
  uint64_t znb = 0, znseq = 0, zlit = 0;
  bool size_only = false;
};

// allow_none: codec NONE verifies the slices only and reports the stored lengths as decoded lengths in phase A (the
// key sort of uncompressed blocks); phase B is not run for it
int check_decode_codec(uint32_t codec, bool allow_none) {
  if (codec != B2S_CODEC_LZ4BLOCK && codec != B2S_CODEC_SNAPPY_XERIAL && codec != B2S_CODEC_ZSTD &&
      !(allow_none && codec == B2S_CODEC_NONE))
    return fail(B2S_E_UNSUPPORTED, "codec %s not supported by this build", "");
  return 0;
}

// Phase A of decoding n streams at d_src + src_off[i] (src_len[i] bytes; src_bytes in all), enqueued on S.st: checksum
// verify of their n_slices slices (slice_base[0..n], indices into slice_len / slice_sum), header count, scans, and
// the readback of J.h.totals, there once ev_a has completed.
int decompress_phase_a(Slot& S, const ChecksumTables& tabs, uint32_t codec, uint32_t alg, uint32_t n,
                       const uint64_t* src_off, const uint64_t* src_len, uint32_t n_slices, const uint32_t* slice_base,
                       const uint64_t* slice_len, const uint64_t* slice_sum, const uint8_t* d_src, uint64_t src_bytes,
                       DecompressJob& J, uint64_t* launches, bool allow_none = false) {
  if (int rc = check_decode_codec(codec, allow_none)) return rc;
  J.n = n;
  J.codec = codec;
  J.n_slices = alg ? n_slices : 0;
  const uint32_t s = J.n_slices;
  size_t up = align_up(n * 8, 16) * 2 + align_up((size_t)s * 8, 16) * 3 + align_up((size_t)s * 4, 16) +
              align_up(((size_t)n + 1) * 4, 16);
  size_t down = 32 + align_up(n * 8, 16) * 2 + align_up(n * 4, 16) * 2;
  int rc = S.hmeta.ensure(up + down + 128);
  if (rc) return rc;
  const DecompressLayout H = J.h = decompress_layout(S.hmeta.p, n, s, -1);
  memcpy(H.src_off, src_off, (size_t)n * 8);
  memcpy(H.src_len, src_len, (size_t)n * 8);
  uint32_t q0 = 0;  // the slices of stream k are checked where the stream sits on the device
  for (uint32_t k = 0; k < n; k++) {
    H.slice_base[k] = q0;
    if (!s) continue;
    uint64_t o = src_off[k];
    for (uint32_t q = slice_base[k]; q < slice_base[k + 1]; q++, q0++) {
      H.slice_off[q0] = o;
      H.slice_len[q0] = slice_len[q];
      H.slice_sum[q0] = slice_sum[q];
      H.slice_owner[q0] = k;
      o += slice_len[q];
    }
  }
  H.slice_base[n] = q0;

  size_t ws_elems = std::max(scan_ws_elems((size_t)n + 1), checksum_ws_elems(s)) + 4;
  size_t need = H.up_bytes + H.down_bytes + align_up((size_t)n * 8, 16) * 1 + align_up((size_t)s * 8, 16) +
                align_up(((size_t)s + 1) * 8, 16) + ws_elems * 8 + 256;
  rc = S.meta.ensure(need);
  if (rc) return rc;
  const DecompressLayout M = J.d = decompress_layout(S.meta.p, n, s, (ptrdiff_t)ws_elems);

  cudaStream_t st = S.st;
  CU(cudaMemcpyAsync(M.up, H.up, M.up_bytes, cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(M.down, 0, M.down_bytes, st));
  CU(cudaMemsetAsync(M.bad, 0xff, (size_t)n * 4, st));
  CU(S.mark(K0, st));
  if (alg != B2S_CHECKSUM_NONE && s) {
    launch_checksum(tabs, alg, d_src, M.slice_off, M.slice_len, s, pick_tile_shift(src_bytes), M.work_base, M.ws,
                    M.cks_got, st, launches);
    launch_checksum_compare(M.cks_got, M.slice_sum, M.slice_owner, M.slice_base, s, M.status, M.bad, st, launches);
  }
  if (codec == B2S_CODEC_ZSTD) {
    // walk (count) -> totals to the host -> walk (fill) -> entropy decode of every block in parallel -> stream sizes.
    // The one blocking readback sizes the descriptor array and the literal / sequence workspace (zstd_par.h).
    rc = S.zmeta.ensure(((size_t)n * 6 + 8) * 8);
    if (rc) return rc;
    J.zcnt = (uint64_t*)S.zmeta.p;
    J.zbase = J.zcnt + (size_t)n * 3;
    uint64_t* ztot = J.zbase + (size_t)n * 3;
    launch_zstd_count(d_src, M.src_off, M.src_len, n, J.zcnt, M.status, st, launches);
    CU(cudaMemcpyAsync(J.zbase, J.zcnt, (size_t)n * 24, cudaMemcpyDeviceToDevice, st));
    for (int k = 0; k < 3; k++) launch_exclusive_scan_u64(J.zbase + (size_t)n * k, n, ztot + k, M.ws, st, launches);
    uint64_t h[3] = {0, 0, 0};
    CU(cudaMemcpyAsync(h, ztot, 24, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    J.znb = h[0];
    J.znseq = h[1];
    J.zlit = h[2];
    if (J.znb >= 0x7fffffffull) return fail(B2S_E_ARG, "too many Zstandard blocks in one chunk%s");
    rc = S.desc.ensure((size_t)(J.znb + 1) * zstd_block_info_bytes());
    if (rc) return rc;
    if (!J.size_only) {
      rc = S.scratch.ensure(zstd_ws_bytes(J.zlit, J.znseq));
      if (rc) return rc;
    }
    launch_zstd_fill(d_src, M.src_off, M.src_len, n, J.zcnt, J.zbase, S.desc.p, M.status, st, launches);
    launch_zstd_entropy(J.size_only, d_src, S.desc.p, J.znb, (uint8_t*)S.scratch.p, J.zlit, J.znseq, M.status, st,
                        launches);
    launch_zstd_sum(S.desc.p, J.zcnt, J.zbase, n, M.dst_len, M.status, st, launches);
    CU(cudaMemsetAsync(M.nblk, 0, (size_t)n * 8, st));
  } else if (codec == B2S_CODEC_SNAPPY_XERIAL)
    launch_xerial_count(d_src, M.src_off, M.src_len, n, M.nblk, M.dst_len, M.totals + 2, M.status, st, launches);
  else if (codec == B2S_CODEC_NONE) {  // stored bytes: decoded length = block length, no codec blocks
    CU(cudaMemcpyAsync(M.dst_len, M.src_len, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
    CU(cudaMemsetAsync(M.nblk, 0, (size_t)n * 8, st));
  } else
    launch_lz4block_count(d_src, M.src_off, M.src_len, n, M.nblk, M.dst_len, M.status, st, launches);
  // dst_off = exclusive scan(dst_len) ; blk_base = exclusive scan(nblk) (in place)
  CU(cudaMemcpyAsync(M.dst_off, M.dst_len, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
  launch_exclusive_scan_u64(M.dst_off, n, M.totals + 1, M.ws, st, launches);
  launch_exclusive_scan_u64(M.nblk, n, M.totals + 0, M.ws, st, launches);
  CU(cudaMemcpyAsync(H.totals, M.totals, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(S.ev_a, st));
  CU(cudaGetLastError());
  return 0;
}

// phase B (after ev_a): descriptors, decode, XXH32 verify, meta readback
int decompress_enqueue_b(Slot& S, DecompressJob& J, const uint8_t* d_src, uint8_t* d_dst, uint64_t dst_cap,
                         uint64_t* launches) {
  J.nb = J.h.totals[0];
  J.total_out = J.h.totals[1];
  if (J.codec == B2S_CODEC_ZSTD) {
    cudaStream_t zst = S.st;
    CU(S.mark(T0, zst));
    launch_zstd_execute(d_src, S.desc.p, J.zcnt, J.zbase, J.n, (const uint8_t*)S.scratch.p, J.zlit, J.znseq, J.d.dst_len,
                        d_dst, J.d.dst_off, dst_cap, J.d.status, zst, launches);
    CU(S.mark(T1, zst));
    CU(S.mark(K1, zst));
    CU(cudaMemcpyAsync(J.h.down, J.d.down, J.d.down_bytes, cudaMemcpyDeviceToHost, zst));
    CU(cudaEventRecord(S.ev_b, zst));
    CU(cudaGetLastError());
    return 0;
  }
  if (J.nb >= 0xffffffffull) return fail(B2S_E_ARG, "too many codec blocks in one chunk%s");
  int rc = S.desc.ensure((size_t)(J.nb + 1) * sizeof(BlockDesc));
  if (rc) return rc;
  cudaStream_t st = S.st;
  BlockDesc* desc = (BlockDesc*)S.desc.p;
  CU(cudaMemsetAsync(desc, 0, (size_t)J.nb * sizeof(BlockDesc), st));
  if (J.codec == B2S_CODEC_SNAPPY_XERIAL)
    launch_xerial_fill(d_src, J.d.src_off, J.d.src_len, J.n, J.d.nblk, J.d.dst_off, J.d.dst_len, dst_cap, J.d.status, desc, st,
                       launches);
  else
    launch_lz4block_fill(d_src, J.d.src_off, J.d.src_len, J.n, J.d.nblk, J.d.dst_off, J.d.dst_len, dst_cap, J.d.status, desc, st,
                         launches);
  CU(S.mark(T0, st));
  if (J.nb && J.codec == B2S_CODEC_LZ4BLOCK) {
    // one launch over every codec block: warp per block, parse and copies together (lz4_decode.cu)
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    S.dom_pair(&e0, &e1);
    CU(cudaEventRecord(e0, st));
    launch_lz4_decode_warp(desc, (uint32_t)J.nb, d_src, d_dst, J.d.status, J.d.counter, st, launches);
    CU(cudaEventRecord(e1, st));
  } else if (J.nb && J.codec == B2S_CODEC_SNAPPY_XERIAL) {
    // the walk has failed every stream with a chunk of more than 64 KiB (B2S_E_UNSUPPORTED for that stream alone), so
    // the largest chunk left is under 64 KiB compressed: the records' 16-bit fields hold every count and position
    const uint64_t max_clen = J.h.totals[3];
    // tokens (thread per block) + copy (lane per sequence), in chunks that bound the record workspace
    const uint32_t nb = (uint32_t)J.nb;
    const uint32_t rec_stride = snappy_decode_rec_stride((uint32_t)max_clen);
    const uint32_t chunk = std::min<uint32_t>(nb, g_lz4d_chunk_blocks);
    const size_t nrec_bytes = align_up((size_t)nb * 4, 256);
    const size_t ws_bytes = align_up(snappy_decode_ws_bytes(chunk, rec_stride), 256);
    rc = S.scratch.ensure(nrec_bytes + ws_bytes * (nb > chunk ? 2 : 1));
    if (rc) return rc;
    uint32_t* nrec = (uint32_t*)S.scratch.p;
    // token walk (thread per block, latency bound) of group k+1 on the side stream, copies of group k on the main one
    CU(cudaEventRecord(S.ev_fork, st));
    CU(cudaStreamWaitEvent(S.st2, S.ev_fork, 0));
    auto tokens = [&](uint32_t b0, uint32_t m, uint8_t* ws, int, cudaEvent_t, cudaEvent_t) {
      launch_snappy_tokens(desc, b0, m, d_src, reinterpret_cast<uint2*>(ws), rec_stride, nrec, J.d.status, S.st2,
                           launches);
      return 0;
    };
    auto copy = [&](uint32_t b0, uint32_t m, uint8_t* ws, int, cudaEvent_t e0, cudaEvent_t e1) -> int {
      CU(cudaEventRecord(e0, st));
      launch_snappy_copy(desc, b0, m, rec_stride, d_src, d_dst, ws, nrec, st, launches);
      CU(cudaEventRecord(e1, st));
      return 0;
    };
    if (int r = run_block_groups(S, nb, chunk, (uint8_t*)S.scratch.p + nrec_bytes, ws_bytes, tokens, copy)) return r;
  }
  CU(S.mark(T1, st));
  // One XXH32 pass over all decoded blocks after the last chunk.  Queueing it chunk by chunk on the side stream (beside
  // the next chunk's copy kernel) was measured slower: both kernels are
  // memory-latency bound and take each other's L2 / DRAM queue slots.
  if (J.codec == B2S_CODEC_LZ4BLOCK)
    launch_xxh32_verify(desc, (uint32_t)J.nb, d_dst, kXxhSeed, 0x0FFFFFFFu, J.d.status, st, launches);
  CU(S.mark(K1, st));
  CU(cudaMemcpyAsync(J.h.down, J.d.down, J.d.down_bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(S.ev_b, st));
  CU(cudaGetLastError());
  return 0;
}

int get_device(uint32_t dev_index, Device** out) {
  if (!g_ctx) return fail(B2S_E_NOT_INIT, "b2s_init has not been called%s");
  if (dev_index >= g_ctx->devs.size()) return fail(B2S_E_ARG, "device index out of range%s");
  *out = g_ctx->devs[dev_index];
  t_numa_node = (*out)->numa_node;
  CU(cudaSetDevice((*out)->ordinal));
  return 0;
}

// the kinds of call whose steps add_times reads into b2s_last_timing, one rule each
enum class Family {
  kCodec, kPartition, kPartitionNone, kSort, kSortRows, kAggregate, kJoin, kWindow, kPartialAggregate
};

// Adds the times of this call's steps on S to b2s_last_timing: kernel_ms, top_kernel_ms, dominant_ms / _launches by
// the rule of its family, and h2d_ms.  A step the call did not run reads 0; one it started but did not finish ends
// where the call stopped (Slot::span).  d2h_ms is read once the payload copy has run (end_call, retire_slot).
void add_times(Slot& S, Family f) {
  b2s_timing& t = t_timing;
  auto dominant = [&](Mark a, Mark b) {  // a dominant step and the launches in it (the step passed its launch count)
    t.dominant_ms += S.span(a, b);
    t.dominant_launches += S.mine(a) && S.mine(b) ? S.mark_launches[b] - S.mark_launches[a] : 0;
  };
  switch (f) {
    case Family::kCodec:  // checksum, compress, decompress, exchange read, and each chunk of a pipelined call: the
                          // kernel region; the codec step; the dominant pairs (match, LZ4 decode, Snappy copy)
      t.kernel_ms += S.span(K0, K1);
      t.top_kernel_ms += S.span(T0, T1);
      S.take_pairs();
      break;
    case Family::kPartition:      // partition step + compression; the codec step; the match launches
    case Family::kPartitionNone:  // partition step + checksum (without one, the gather); the partition step
      t.kernel_ms += S.span(P0, f == Family::kPartitionNone && !S.mine(K1) ? P1 : K1);
      t.top_kernel_ms += f == Family::kPartition ? S.span(T0, T1) : S.span(P0, P1);
      if (S.mine(F0)) dominant(F0, F1);  // a hash, range or round-robin partition: its id step
      else S.take_pairs();
      break;
    case Family::kSort:       // verification + decode + sort; the sort step; the decoder's dominant pairs
    case Family::kSortRows:   // the same; framing + order + gather; the framing (walk + count, emit)
    case Family::kAggregate:  // the same; framing through merge; grouping + merge
    case Family::kJoin:       // the same; framing through join; the join step (grouping, counts, emit)
    case Family::kWindow:     // the same; framing through emit; the window step (grouping, values, emit)
      t.kernel_ms += S.span(K0, P1);
      t.top_kernel_ms += S.span(P0, P1);
      if (f == Family::kSort) S.take_pairs();
      if (f == Family::kSortRows) {
        dominant(F0, F1);
        dominant(F2, F3);
      }
      if (f == Family::kAggregate || f == Family::kJoin || f == Family::kWindow) dominant(G0, G1);
      break;
    case Family::kPartialAggregate:  // a map-side step (aggregation, window limit, or the DISTINCT call's stage 3, whose
                                     // read and stage 2 the call adds) + partition step + compression (or checksums);
                                     // the codec step (or the partition step); the map-side step
      t.kernel_ms += S.span(G0, S.mine(K1) ? K1 : P1);
      t.top_kernel_ms += S.mine(T0) ? S.span(T0, T1) : S.span(P0, P1);
      dominant(G0, G1);
      break;
  }
  t.h2d_ms += S.span(H0, H1);
}

// what a call moved: bytes into and out of its kernels, and over PCIe
struct CallBytes {
  uint64_t src = 0, dst = 0, h2d = 0, d2h = 0;
};

// Ends a successful call's b2s_last_timing: its bytes, its launches (also counted for the process) and its wall time.
// S: the one slot the call ran on, whose steps give the times (add_times); nullptr for a call pipelined over slots,
// whose chunks added their own times.
void end_call(const WallTimer& wt, uint64_t launches, const CallBytes& b, Slot* S = nullptr,
              Family f = Family::kCodec) {
  if (S) {
    add_times(*S, f);
    t_timing.d2h_ms += S->span(D0, D1);
  }
  t_timing.src_bytes += b.src;
  t_timing.dst_bytes += b.dst;
  t_timing.h2d_bytes += b.h2d;
  t_timing.d2h_bytes += b.d2h;
  t_timing.kernel_launches = launches;
  g_ctx->launches += launches;
  t_timing.total_ms = wt.ms();
}

// run_chunks' retire: the slot's stream has drained, the payload download of its last chunk included
int retire_slot(Slot& S, bool used) {
  CU(cudaStreamSynchronize(S.st));
  if (used) t_timing.d2h_ms += S.span(D0, D1);
  return 0;
}

// device layout of a chunk's sources: runs that are contiguous in host memory stay contiguous (one memcpy each)
struct Run {
  const uint8_t* host;
  uint64_t dev_off;
  uint64_t bytes;
};
uint64_t plan_runs(uint32_t cnt, const uint8_t* const* ptr, const uint64_t* len, uint64_t* dev_off,
                   std::vector<Run>& runs) {
  runs.clear();
  uint64_t cur = 0;
  for (uint32_t i = 0; i < cnt; i++) {
    if (len[i] == 0) {
      dev_off[i] = cur;
      continue;
    }
    if (!runs.empty() && runs.back().host + runs.back().bytes == ptr[i]) {
      dev_off[i] = runs.back().dev_off + runs.back().bytes;
      runs.back().bytes += len[i];
    } else {
      // keep the host pointer's 16-byte phase so aligned fast paths behave the same as in host memory
      cur = align_up(cur, 16) + ((uintptr_t)ptr[i] & 15u);
      dev_off[i] = cur;
      runs.push_back(Run{ptr[i], cur, len[i]});
    }
    cur = dev_off[i] + len[i];
  }
  return cur;
}

// Stages the cnt sources of a chunk in S.src: dev_off[i] receives where source i sits, the return value the arena's
// bytes (what the chunk uploads).  The copies run between marks H0 and H1.
int upload_chunk(Slot& S, uint32_t cnt, const uint8_t* const* ptr, const uint64_t* len, uint64_t* dev_off,
                 std::vector<Run>& runs, uint64_t* bytes) {
  *bytes = plan_runs(cnt, ptr, len, dev_off, runs);
  if (int rc = S.src.ensure(*bytes + 64)) return rc;
  CU(S.mark(H0, S.st));
  for (const Run& r : runs)
    CU(cudaMemcpyAsync((uint8_t*)S.src.p + r.dev_off, r.host, r.bytes, cudaMemcpyHostToDevice, S.st));
  CU(S.mark(H1, S.st));
  return 0;
}

// Copies a finished chunk of n streams (stream k: len[k] bytes at off[k] of S.dst, chunk_total bytes in all) to the
// host between marks D0 and D1, and adds what it copied to d2h_bytes.  packed_dst: the whole chunk at run_off of that
// arena, as much of it as fits in packed_cap, and every stream still OK that does not fit entirely gets
// B2S_E_DST_TOO_SMALL.  dst: stream k of an OK status to dst[k], or B2S_E_DST_TOO_SMALL when it exceeds dst_cap[k].
// Neither: nothing is copied.
int download_chunk(Slot& S, uint32_t n, const uint64_t* off, const uint64_t* len, uint64_t chunk_total,
                   uint8_t* packed_dst, uint64_t packed_cap, uint64_t run_off, uint8_t* const* dst,
                   const uint64_t* dst_cap, int32_t* status) {
  CU(S.mark(D0, S.st));
  if (packed_dst) {
    uint64_t fit = chunk_total;
    if (run_off + chunk_total > packed_cap) {
      fit = packed_cap > run_off ? packed_cap - run_off : 0;
      for (uint32_t k = 0; k < n; k++)
        if (status[k] == B2S_OK && run_off + off[k] + len[k] > packed_cap) status[k] = B2S_E_DST_TOO_SMALL;
    }
    // what fits is copied, so that the streams in front of the first one that does not stay valid
    if (fit) CU(cudaMemcpyAsync(packed_dst + run_off, S.dst.p, fit, cudaMemcpyDeviceToHost, S.st));
    t_timing.d2h_bytes += fit;
  } else if (dst) {
    for (uint32_t k = 0; k < n; k++) {
      if (status[k] != B2S_OK || len[k] == 0) continue;
      if (len[k] > dst_cap[k]) {
        status[k] = B2S_E_DST_TOO_SMALL;
        continue;
      }
      CU(cudaMemcpyAsync(dst[k], (uint8_t*)S.dst.p + off[k], len[k], cudaMemcpyDeviceToHost, S.st));
      t_timing.d2h_bytes += len[k];
    }
  }
  CU(S.mark(D1, S.st));
  return 0;
}


// ---- in-process multi-GPU: the per-stream-pointer batch calls shard their streams round-robin (stream i -> device
// i mod D) over every device selected by b2s_init, one host thread per device, each driving its own pipeline slots,
// pinned staging and streams; nothing is exchanged between devices (SURVEY.md §8e).  Packed calls and the calling
// thread's own work stay on the thread's device (b2s_set_thread_device).
template <typename F>
int shard_over_devices(uint32_t n, F&& run_subset) {
  const uint32_t D = g_ctx ? (uint32_t)g_ctx->devs.size() : 0;
  std::vector<int> rcs(D, 0);
  std::vector<std::string> errs(D);
  std::vector<b2s_timing> tms(D);
  std::vector<std::thread> th;
  for (uint32_t d = 0; d < D; d++) {
    th.emplace_back([&, d] {
      t_device = d;
      std::vector<uint32_t> idx;
      for (uint32_t i = d; i < n; i += D) idx.push_back(i);
      rcs[d] = idx.empty() ? 0 : run_subset(idx);
      errs[d] = t_last_error;
      tms[d] = t_timing;
    });
  }
  for (auto& t : th) t.join();
  t_timing = b2s_timing{};
  int rc = 0;
  for (uint32_t d = 0; d < D; d++) {
    if (rcs[d] && !rc) {
      rc = rcs[d];
      t_last_error = errs[d];
    }
    // devices work concurrently: times are the slowest device's, byte and launch counters add up
    t_timing.total_ms = std::max(t_timing.total_ms, tms[d].total_ms);
    t_timing.h2d_ms = std::max(t_timing.h2d_ms, tms[d].h2d_ms);
    t_timing.d2h_ms = std::max(t_timing.d2h_ms, tms[d].d2h_ms);
    t_timing.kernel_ms = std::max(t_timing.kernel_ms, tms[d].kernel_ms);
    t_timing.top_kernel_ms = std::max(t_timing.top_kernel_ms, tms[d].top_kernel_ms);
    t_timing.dominant_ms = std::max(t_timing.dominant_ms, tms[d].dominant_ms);
    t_timing.h2d_bytes += tms[d].h2d_bytes;
    t_timing.d2h_bytes += tms[d].d2h_bytes;
    t_timing.kernel_launches += tms[d].kernel_launches;
    t_timing.dominant_launches += tms[d].dominant_launches;
    t_timing.src_bytes += tms[d].src_bytes;
    t_timing.dst_bytes += tms[d].dst_bytes;
  }
  return rc;
}
bool want_sharding(uint32_t n) { return g_ctx && g_ctx->devs.size() > 1 && n >= 2 * g_ctx->devs.size(); }

// --------------------------------------------------------------------------------------------------------------
// exchange cache (docs/f4_gpu_resident_exchange.md steps 2-3): partitioned map outputs kept in HBM, per CUDA device,
// under a byte budget, least recently used out first.  An entry is linked in `by_key` while it can be found; a read
// references the entries it uses until its stream has synchronised, and an entry unlinked (evicted, removed, replaced)
// while referenced is freed by its last reader.  `used` counts the bytes of linked entries.  The lock is never held
// across a CUDA call: device memory is allocated and freed outside it.
// --------------------------------------------------------------------------------------------------------------
constexpr int kMaxOrdinals = 32;  // b2s_init selects devices 0..31
struct ExEntry {
  int32_t shuffle = 0;
  int64_t map = 0;
  int ordinal = 0;  // CUDA device holding buf
  uint8_t* buf = nullptr;
  uint64_t bytes = 0;                // of records
  std::vector<uint64_t> part_start;  // R + 1 offsets of the partitions in buf
  // Record boundaries (entries of the row writers; empty / nullptr for the id-taking store): every record's offset in
  // buf, in order (device memory, in buf's allocation behind the records), and the R + 1 indices in rec_off of each
  // partition's first record
  const uint64_t* rec_off = nullptr;
  std::vector<uint64_t> rec_start;
  uint64_t charged = 0;  // what counts against the budget: the records' bytes (8-aligned with boundaries), 8 per boundary
  uint32_t refs = 0;
  uint64_t last_use = 0;
  bool linked = true;
};
struct ExCache {
  std::mutex mtx;
  std::map<std::pair<int32_t, int64_t>, ExEntry*> by_key;
  uint64_t budget[kMaxOrdinals] = {}, used[kMaxOrdinals] = {};
  uint64_t tick = 0;
};
ExCache g_ex;

// unlinks e (caller holds g_ex.mtx); an unreferenced entry goes to `dead`, for the caller to free outside the lock
void ex_unlink(ExEntry* e, std::vector<ExEntry*>& dead) {
  g_ex.by_key.erase({e->shuffle, e->map});
  g_ex.used[e->ordinal] -= e->charged;
  e->linked = false;
  if (!e->refs) dead.push_back(e);
}

void ex_free(const std::vector<ExEntry*>& dead) {
  if (dead.empty()) return;
  int cur = 0;
  cudaGetDevice(&cur);
  for (ExEntry* e : dead) {
    if (e->buf) {
      cudaSetDevice(e->ordinal);
      cudaFree(e->buf);
    }
    delete e;
  }
  cudaSetDevice(cur);
  (void)cudaGetLastError();
}

// unlinks least recently used unreferenced entries of `ordinal` until `bytes` more fit under its budget (caller holds
// the lock).  When they cannot be made to fit it returns false, having evicted nothing unless `partial` (a lowered
// budget: evict what can go, the referenced rest goes when it is released and evicted later).
bool ex_make_room(int ordinal, uint64_t bytes, std::vector<ExEntry*>& dead, bool partial = false) {
  const uint64_t budget = g_ex.budget[ordinal];
  uint64_t idle = 0;
  for (auto& kv : g_ex.by_key)
    if (kv.second->ordinal == ordinal && !kv.second->refs) idle += kv.second->charged;
  const bool fits = bytes <= budget && g_ex.used[ordinal] - idle <= budget - bytes;
  if (!fits && !partial) return false;
  while (g_ex.used[ordinal] + bytes > budget) {
    ExEntry* victim = nullptr;
    for (auto& kv : g_ex.by_key) {
      ExEntry* e = kv.second;
      if (e->ordinal == ordinal && !e->refs && (!victim || e->last_use < victim->last_use)) victim = e;
    }
    if (!victim) break;
    ex_unlink(victim, dead);
  }
  return fits;
}

bool exchange_shed_current_device() {
  int ordinal = 0;
  if (cudaGetDevice(&ordinal) != cudaSuccess || ordinal < 0 || ordinal >= kMaxOrdinals) return false;
  std::vector<ExEntry*> dead;
  {
    std::lock_guard<std::mutex> lk(g_ex.mtx);
    std::vector<ExEntry*> idle;
    for (auto& kv : g_ex.by_key)
      if (kv.second->ordinal == ordinal && !kv.second->refs) idle.push_back(kv.second);
    for (ExEntry* e : idle) ex_unlink(e, dead);
  }
  ex_free(dead);
  return !dead.empty();
}

// The entries a read uses, referenced from its lookup until the read's stream has synchronised.  entry[i]: the
// resident entry of map_ids[i] on `ordinal` (nullptr: not resident, or want[i] == 0); each use counts for the LRU order.
struct ExRefs {
  std::vector<ExEntry*> entry;
  ExRefs(int ordinal, int32_t shuffle, uint32_t n, const int64_t* map_ids, const uint8_t* want) : entry(n, nullptr) {
    std::lock_guard<std::mutex> lk(g_ex.mtx);
    for (uint32_t i = 0; i < n; i++) {
      if (want && !want[i]) continue;
      auto it = g_ex.by_key.find({shuffle, map_ids[i]});
      if (it == g_ex.by_key.end() || it->second->ordinal != ordinal) continue;
      entry[i] = it->second;
      entry[i]->refs++;
      entry[i]->last_use = ++g_ex.tick;
    }
  }
  ~ExRefs() {
    std::vector<ExEntry*> dead;
    {
      std::lock_guard<std::mutex> lk(g_ex.mtx);
      for (ExEntry* e : entry)
        if (e && --e->refs == 0 && !e->linked) dead.push_back(e);
    }
    ex_free(dead);
  }
  // B2S_E_ARG when a resident entry has fewer than end_reduce partitions
  int check_range(int32_t end_reduce) const {
    for (const ExEntry* e : entry)
      if (e && (uint64_t)end_reduce + 1 > e->part_start.size())
        return fail(B2S_E_ARG, "end_reduce exceeds the partitions of a cached map output%s");
    return 0;
  }
  // the bytes of partitions [start, end) of source i inside its entry
  const uint8_t* range(uint32_t i, int32_t start, int32_t end, uint64_t* len) const {
    const ExEntry* e = entry[i];
    *len = e->part_start[(size_t)end] - e->part_start[(size_t)start];
    return e->buf + e->part_start[(size_t)start];
  }
  // the record boundaries of partitions [start, end) of source i (false: its entry keeps none): *off = the first
  // record's offset in rec_off's numbering (the entry's), *first = its offsets, *count = how many
  bool bounds(uint32_t i, int32_t start, int32_t end, uint64_t* off, const uint64_t** first, uint64_t* count) const {
    const ExEntry* e = entry[i];
    if (e->rec_start.empty()) return false;
    *off = e->part_start[(size_t)start];
    *first = e->rec_off + e->rec_start[(size_t)start];
    *count = e->rec_start[(size_t)end] - e->rec_start[(size_t)start];
    return true;
  }
};

// The record boundaries a row writer's store keeps (ex_store): its partition plan (launch_partition_order's, over n
// records: sdst holds every record's offset in the partitioned arena, and the readback block, already read back, is
// free to take rec_start), and pinned host memory for rec_start's readback (R + 1 u64)
struct ExBounds {
  const PartitionPlan* plan;
  uint64_t n;
  uint64_t* host;
  uint64_t* launches;
};

// Keeps `bytes` of partitioned records at d_rec (device memory of the current device `ordinal`, stream st) as the
// entry (shuffle, map): exact-size allocation, device-to-device copy.  rb (rows): the record boundaries too, their
// offsets copied behind the records and rec_start computed from the sorted ids and read back, all before the one
// synchronisation.  Returns 1 when stored, 0 when it does not fit.
int ex_store(int ordinal, cudaStream_t st, int32_t shuffle, int64_t map, const uint8_t* d_rec, uint64_t bytes,
             std::vector<uint64_t>&& part_start, const ExBounds* rb = nullptr) {
  // the charge is what the entry holds: the records, and for a row entry their 8-aligned size and the offsets
  const uint64_t rec_sz = align_up(bytes, 8), n = rb ? rb->n : 0, charged = (n ? rec_sz : bytes) + 8 * n;
  std::vector<ExEntry*> dead;
  bool fits;
  {
    std::lock_guard<std::mutex> lk(g_ex.mtx);
    auto it = g_ex.by_key.find({shuffle, map});
    if (it != g_ex.by_key.end()) ex_unlink(it->second, dead);  // a stale output of this map is never served again
    fits = g_ex.budget[ordinal] > 0 && ex_make_room(ordinal, charged, dead);
    if (fits) g_ex.used[ordinal] += charged;  // reserved until the entry is linked
  }
  ex_free(dead);
  dead.clear();
  if (!fits) return 0;
  ExEntry* e = new ExEntry();
  e->shuffle = shuffle;
  e->map = map;
  e->ordinal = ordinal;
  e->bytes = bytes;
  e->charged = charged;
  const uint32_t R = (uint32_t)part_start.size() - 1;
  e->part_start = std::move(part_start);
  if (rb) e->rec_start.assign((size_t)R + 1, 0);
  bool ok = true;
  if (bytes) {
    ok = cudaMalloc(&e->buf, rec_sz + 8 * n) == cudaSuccess &&
         cudaMemcpyAsync(e->buf, d_rec, bytes, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
    if (ok && n) {
      e->rec_off = (const uint64_t*)(e->buf + rec_sz);
      launch_partition_rec_start(*rb->plan, n, R, rb->plan->readback, st, rb->launches);
      ok = cudaMemcpyAsync(e->buf + rec_sz, rb->plan->sdst, 8 * n, cudaMemcpyDeviceToDevice, st) == cudaSuccess &&
           cudaMemcpyAsync(rb->host, rb->plan->readback, ((size_t)R + 1) * 8, cudaMemcpyDeviceToHost, st) ==
               cudaSuccess;
    }
    ok = ok && cudaStreamSynchronize(st) == cudaSuccess && cudaGetLastError() == cudaSuccess;
    if (!ok) (void)cudaGetLastError();  // not stored; the call's own outputs are unaffected
    if (ok && n) e->rec_start.assign(rb->host, rb->host + (size_t)R + 1);
  }
  {
    std::lock_guard<std::mutex> lk(g_ex.mtx);
    g_ex.used[ordinal] -= charged;
    if (!ok) {
      dead.push_back(e);
    } else {
      auto it = g_ex.by_key.find({shuffle, map});
      if (it != g_ex.by_key.end()) ex_unlink(it->second, dead);  // stored by another thread meanwhile
      g_ex.used[ordinal] += charged;
      e->last_use = ++g_ex.tick;
      g_ex.by_key[{shuffle, map}] = e;
    }
  }
  ex_free(dead);
  return ok ? 1 : 0;
}

// without a usable device the exchange calls report B2S_E_CUDA (b2s_init has failed for that reason)
int exchange_ready() {
  if (g_ctx) return 0;
  if (int rc = no_device()) return rc;
  return fail(B2S_E_NOT_INIT, "b2s_init has not been called%s");
}

int reduce_range_args(int32_t start_reduce, int32_t end_reduce) {
  if (start_reduce < 0 || end_reduce < start_reduce || end_reduce > (1 << 24))
    return fail(B2S_E_ARG, "reduce range must satisfy 0 <= start_reduce <= end_reduce <= 2^24%s");
  return 0;
}

// creates the streams, events and tables of CUDA device d for D (b2s_init); on failure destroy_device frees what it made
int create_device(Device& D, int d, uint64_t pinned_bytes_per_gpu) {
  D.ordinal = d;
  CU(cudaSetDevice(d));
  char busid[32] = {0};
  if (g_numa && cudaDeviceGetPCIBusId(busid, sizeof busid, d) == cudaSuccess) D.numa_node = numa::node_of_pci(busid);
  (void)cudaGetLastError();
  t_numa_node = D.numa_node;
  for (int l = 0; l < kLanes; l++)
    for (int k = 0; k < g_nslot; k++) {
      Slot& S = D.lane[l].slot[k];
      // the read lane's kernels are short and latency bound (token walks, per-stream header walks, two host round
      // trips per chunk): they get the higher stream priority so they are not queued behind the write lane's grids
      int prio_lo = 0, prio_hi = 0;
      cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
      if (int rc = S.create(l == kLaneRead ? prio_hi : prio_lo)) return rc;
      // pinned_bytes_per_gpu: the library's own pinned descriptor blocks are sized up front (split over the slots)
      // instead of growing on first use; 0 = grow on demand.  Payload staging is the caller's (b2s_host_alloc).
      if (pinned_bytes_per_gpu) {
        const uint64_t per = std::min<uint64_t>(pinned_bytes_per_gpu / (uint64_t)(kLanes * g_nslot), 64ull << 20);
        if (per >= 4096 && S.hmeta.ensure(per)) return B2S_E_NOMEM;
      }
    }
  if (checksum_tables_create(&D.tabs)) return fail(B2S_E_CUDA, "checksum table upload failed%s");
  if (zstd_ctables_create(&D.zstd_ctables)) return fail(B2S_E_CUDA, "zstd table upload failed%s");
  zstd_set_ctables(d, D.zstd_ctables);
  CU(cudaEventCreate(&D.ev_mark[0]));
  CU(cudaEventCreate(&D.ev_mark[1]));
  return 0;
}

void destroy_device(Device* D) {
  cudaSetDevice(D->ordinal);
  cudaDeviceSynchronize();
  for (Lane& Ln : D->lane)
    for (Slot& S : Ln.slot) S.release();
  checksum_tables_destroy(&D->tabs);
  zstd_set_ctables(D->ordinal, nullptr);
  zstd_ctables_destroy(D->zstd_ctables);
  for (auto ev : D->ev_mark)
    if (ev) cudaEventDestroy(ev);
  delete D;
}

void destroy_context(Context* C) {
  for (Device* D : C->devs) destroy_device(D);
  delete C;
}

}  // namespace

// ==============================================================================================================
// C ABI
// ==============================================================================================================
extern "C" {

uint32_t b2s_version(void) { return B2S_VERSION; }

const char* b2s_strerror(int32_t code) {
  switch (code) {
    case B2S_OK: return "ok";
    case B2S_E_CORRUPT: return "Stream is corrupted";
    case B2S_E_CHECKSUM: return "Invalid checksum detected";
    case B2S_E_DST_TOO_SMALL: return "destination too small";
    case B2S_E_UNSUPPORTED: return "unsupported codec, checksum algorithm or parameter";
    case B2S_E_ARG: return "invalid argument";
    case B2S_E_CUDA: return "CUDA failure or no usable device";
    case B2S_E_NOT_INIT: return "b2s_init has not been called";
    case B2S_E_NOMEM: return "out of memory";
    case B2S_E_NOT_CACHED: return "not resident in the exchange cache";
    default: return "unknown error";
  }
}
const char* b2s_last_error(void) { return t_last_error.c_str(); }

int b2s_init(uint32_t gpu_mask, uint64_t pinned_bytes_per_gpu, uint32_t streams_per_gpu) {
  std::lock_guard<std::mutex> lk(g_init_mtx);
  if (g_ctx) return 0;
  // Hardware work queues.  A device runs 2 lanes x B2S_SLOTS slots x 2 streams (24 by default); CUDA multiplexes streams
  // onto CUDA_DEVICE_MAX_CONNECTIONS queues (8 unless set) and streams that share a queue run in submission order — the
  // read lane's uploads then wait behind whole chunks of the write lane.  With 32 queues a write call
  // and a read call in flight together overlap instead of running one after the other.  The
  // variable is read when the CUDA context is created, so it only helps if the library gets here first (a host that
  // creates the context earlier sets it itself: bench.py does); an explicit setting is never overridden.
  if (env_int("B2S_MAX_CONNECTIONS", 32) > 0 && !getenv("CUDA_DEVICE_MAX_CONNECTIONS")) {
    char v[16];
    snprintf(v, sizeof v, "%d", std::min(32, env_int("B2S_MAX_CONNECTIONS", 32)));
    setenv("CUDA_DEVICE_MAX_CONNECTIONS", v, 0);
  }
  int count = 0;
  if (int rc = no_device(&count)) return rc;
  g_lz4_hlog = env_int("B2S_LZ4_HLOG", g_lz4_hlog);
  g_lz4_chunk_blocks = (uint32_t)std::max(1, env_int("B2S_LZ4_CHUNK_BLOCKS", (int)g_lz4_chunk_blocks));
  g_numa = env_int("B2S_NUMA", 1);
  g_read_lag = std::max(1, env_int("B2S_READ_LAG", g_read_lag));
  g_lz4d_chunk_blocks = (uint32_t)std::max(1, env_int("B2S_LZ4D_CHUNK_BLOCKS", (int)g_lz4d_chunk_blocks));
  g_host_chunk_bytes = (uint64_t)std::max(1, env_int("B2S_HOST_CHUNK_MB", (int)(g_host_chunk_bytes >> 20))) << 20;
  // streams_per_gpu: pipeline slots (stream pairs + staging) per lane, 0 = default; B2S_SLOTS overrides
  g_nslot = std::min(NSLOT, std::max(2, env_int("B2S_SLOTS", streams_per_gpu ? (int)streams_per_gpu : g_nslot)));
  Context* C = new Context();
  for (int d = 0; d < count && d < 32; d++) {
    if (gpu_mask && !(gpu_mask & (1u << d))) continue;
    Device* D = new Device();
    C->devs.push_back(D);
    if (int rc = create_device(*D, d, pinned_bytes_per_gpu)) {
      destroy_context(C);
      return rc;
    }
  }
  if (C->devs.empty()) {
    delete C;
    return fail(B2S_E_ARG, "gpu_mask selects no visible device%s");
  }
  t_numa_node = C->devs[0]->numa_node;
  g_ctx = C;
  return 0;
}

void b2s_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_init_mtx);
  if (!g_ctx) return;
  std::vector<ExEntry*> dead;
  {
    std::lock_guard<std::mutex> lx(g_ex.mtx);
    while (!g_ex.by_key.empty()) ex_unlink(g_ex.by_key.begin()->second, dead);
    for (int d = 0; d < kMaxOrdinals; d++) g_ex.budget[d] = 0;
  }
  ex_free(dead);
  destroy_context(g_ctx);
  g_ctx = nullptr;
}

int b2s_device_count(void) { return g_ctx ? (int)g_ctx->devs.size() : B2S_E_NOT_INIT; }

int b2s_set_thread_device(uint32_t dev_index) {
  if (!g_ctx) return fail(B2S_E_NOT_INIT, "b2s_init has not been called%s");
  if (dev_index >= g_ctx->devs.size()) return fail(B2S_E_ARG, "device index out of range%s");
  t_device = dev_index;
  t_numa_node = g_ctx->devs[dev_index]->numa_node;
  return 0;
}

int b2s_bind_thread_to_device(uint32_t dev_index) {
  int rc = b2s_set_thread_device(dev_index);
  if (rc) return rc;
  const int node = g_ctx->devs[dev_index]->numa_node;
  if (!g_numa || node < 0) return 0;  // topology unknown (or B2S_NUMA=0): nothing to do, not an error
  cpu_set_t set;
  if (numa::node_cpus(node, &set)) sched_setaffinity(0, sizeof set, &set);  // best effort: a cpuset cgroup may refuse
  numa::Mask m;
  m.w[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
  numa::set_policy(numa::kPreferred, &m);
  return 0;
}
int b2s_device_numa_node(uint32_t dev_index) {
  if (!g_ctx) return B2S_E_NOT_INIT;
  if (dev_index >= g_ctx->devs.size()) return B2S_E_ARG;
  return g_ctx->devs[dev_index]->numa_node < 0 ? -1000 : g_ctx->devs[dev_index]->numa_node;
}

void* b2s_host_alloc(uint64_t bytes) {
  void* p = nullptr;
  // next to the calling thread's device (b2s_set_thread_device / b2s_bind_thread_to_device; device 0 by default)
  if (g_ctx && t_device < g_ctx->devs.size()) t_numa_node = g_ctx->devs[t_device]->numa_node;
  numa::PreferNode near(t_numa_node);
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) {
    fail(B2S_E_NOMEM, "cudaHostAlloc failed%s");
    return nullptr;
  }
  return p;
}
void b2s_host_free(void* p) {
  if (p) cudaFreeHost(p);
}
int b2s_host_register(void* p, uint64_t bytes) {
  CU(cudaHostRegister(p, bytes, cudaHostRegisterPortable));
  return 0;
}
int b2s_host_unregister(void* p) {
  CU(cudaHostUnregister(p));
  return 0;
}

uint64_t b2s_compress_bound(uint32_t codec, uint32_t codec_block_size, uint64_t src_len) {
  const uint64_t bs = block_size_or_default(codec_block_size);
  const uint64_t nb = (src_len + bs - 1) / bs;
  switch (codec) {
    case B2S_CODEC_LZ4BLOCK: return src_len + (nb + 1) * 21;  // RAW fallback bounds every block by its input
    case B2S_CODEC_SNAPPY_XERIAL: return 16 + nb * 37 + src_len + src_len / 6;  // per chunk: BE32 + 32 + n + n/6
    case B2S_CODEC_ZSTD: return src_len + nb * 3 + 9;  // Raw_Block fallback bounds every block by its input
    default: return src_len;
  }
}

void* b2s_dev_alloc(uint32_t dev_index, uint64_t bytes) {
  Device* D;
  if (get_device(dev_index, &D)) return nullptr;
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
  if (e != cudaSuccess) {
    fail(B2S_E_NOMEM, "cudaMalloc: %s", cudaGetErrorString(e));
    return nullptr;
  }
  return p;
}
void b2s_dev_free(uint32_t dev_index, void* p) {
  Device* D;
  if (get_device(dev_index, &D)) return;
  if (p) cudaFree(p);
}
int b2s_dev_memcpy(uint32_t dev_index, void* dst, const void* src, uint64_t bytes, int kind) {
  Device* D;
  int rc = get_device(dev_index, &D);
  if (rc) return rc;
  cudaMemcpyKind k = kind == 1 ? cudaMemcpyHostToDevice : kind == 2 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  CU(cudaMemcpy(dst, src, bytes, k));
  return 0;
}

int b2s_last_timing(b2s_timing* out) {
  if (!out) return B2S_E_ARG;
  *out = t_timing;
  return 0;
}
uint64_t b2s_total_kernel_launches(void) { return g_ctx ? g_ctx->launches.load() : 0; }

int b2s_mark(uint32_t dev_index, uint32_t which) {
  Device* D;
  int rc = get_device(dev_index, &D);
  if (rc) return rc;
  if (which > 1) return fail(B2S_E_ARG, "mark index must be 0 or 1%s");
  // every entry point is synchronous, so an event on the first slot's stream brackets whatever ran in between
  CU(cudaEventRecord(D->ev_mark[which], D->lane[kLaneWrite].slot[0].st));
  return 0;
}
int b2s_marks_elapsed_ms(uint32_t dev_index, double* ms) {
  Device* D;
  int rc = get_device(dev_index, &D);
  if (rc) return rc;
  if (!ms) return fail(B2S_E_ARG, "null argument%s");
  CU(cudaEventSynchronize(D->ev_mark[1]));
  float f = 0;
  CU(cudaEventElapsedTime(&f, D->ev_mark[0], D->ev_mark[1]));
  *ms = f;
  return 0;
}

int b2s_gen_terasort_dev(uint32_t dev_index, void* d_dst, uint64_t first_record, uint64_t n_records, uint64_t seed) {
  Device* D;
  int rc = get_device(dev_index, &D);
  if (rc) return rc;
  Lane& Ln = D->lane[kLaneWrite];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  launch_gen_terasort((uint8_t*)d_dst, first_record, n_records, seed, Ln.slot[0].st);
  CU(cudaStreamSynchronize(Ln.slot[0].st));
  CU(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// checksums
// ------------------------------------------------------------------------------------------------------------
static int checksum_chunk_dev(Device* D, Slot& S, uint32_t alg, uint32_t n, const uint8_t* d_base, const uint64_t* off,
                              const uint64_t* len, uint64_t* out, uint64_t total_bytes, uint64_t* launches) {
  if (alg < B2S_CHECKSUM_ADLER32 || alg > B2S_CHECKSUM_CRC32C)
    return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  size_t up = align_up((size_t)n * 8, 16) * 2, down = align_up((size_t)n * 8, 16);
  int rc = S.hmeta.ensure(up + down + 64);
  if (rc) return rc;
  size_t ws_elems = checksum_ws_elems(n) + 4;
  rc = S.meta.ensure(up + down + align_up(((size_t)n + 1) * 8, 16) + ws_elems * 8 + 128);
  if (rc) return rc;
  Carver hc(S.hmeta.p), dc(S.meta.p);
  uint64_t* h_off = hc.take<uint64_t>(n);
  uint64_t* h_len = hc.take<uint64_t>(n);
  hc.off = align_up(hc.off, 16);
  uint64_t* h_out = hc.take<uint64_t>(n);
  uint64_t* d_off = dc.take<uint64_t>(n);
  uint64_t* d_len = dc.take<uint64_t>(n);
  dc.off = align_up(dc.off, 16);
  uint64_t* d_out = dc.take<uint64_t>(n);
  uint64_t* d_work = dc.take<uint64_t>((size_t)n + 1);
  uint64_t* d_ws = dc.take<uint64_t>(ws_elems);
  memcpy(h_off, off, (size_t)n * 8);
  memcpy(h_len, len, (size_t)n * 8);
  cudaStream_t st = S.st;
  CU(cudaMemcpyAsync(d_off, h_off, up, cudaMemcpyHostToDevice, st));
  CU(S.mark(K0, st));
  CU(S.mark(T0, st));
  launch_checksum(D->tabs, alg, d_base, d_off, d_len, n, pick_tile_shift(total_bytes), d_work, d_ws, d_out, st,
                  launches);
  CU(S.mark(T1, st));
  CU(S.mark(K1, st));
  CU(cudaMemcpyAsync(h_out, d_out, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  memcpy(out, h_out, (size_t)n * 8);
  return 0;
}

int b2s_checksum_dev(uint32_t dev_index, uint32_t alg, uint32_t n, const void* d_base, const uint64_t* off,
                     const uint64_t* len, uint64_t* out) {
  const WallTimer wt = begin_call();
  Device* D;
  int rc = get_device(dev_index, &D);
  if (rc) return rc;
  if (!n) return 0;
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  uint64_t total = 0, launches = 0;
  for (uint32_t i = 0; i < n; i++) total += len[i];
  rc = checksum_chunk_dev(D, Ln.slot[0], alg, n, (const uint8_t*)d_base, off, len, out, total, &launches);
  if (rc) return rc;
  end_call(wt, launches, CallBytes{total, 0, 0, 0}, &Ln.slot[0]);
  return 0;
}

static int checksum_host(uint32_t alg, uint32_t n, const uint8_t* const* ptr, const uint64_t* len, uint64_t* out) {
  const WallTimer wt = begin_call();
  Device* D;
  int rc = get_device(t_device, &D);
  if (rc) return rc;
  if (!n) return 0;
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  const std::vector<uint32_t> starts = chunk_starts(n, len, kChunkStreams, g_host_chunk_bytes);
  std::vector<uint64_t> dev_off;
  std::vector<Run> runs;
  uint64_t launches = 0;
  for (size_t c = 0; c + 1 < starts.size(); c++) {
    Slot& S = Ln.slot[0];
    const uint32_t i0 = starts[c], cnt = starts[c + 1] - starts[c];
    dev_off.resize(cnt);
    uint64_t bytes = 0;
    if ((rc = upload_chunk(S, cnt, ptr + i0, len + i0, dev_off.data(), runs, &bytes))) return rc;
    rc = checksum_chunk_dev(D, S, alg, cnt, (const uint8_t*)S.src.p, dev_off.data(), len + i0, out + i0, bytes,
                            &launches);
    if (rc) return rc;
    add_times(S, Family::kCodec);
    t_timing.h2d_bytes += bytes;
    t_timing.d2h_bytes += (uint64_t)cnt * 8;
    t_timing.src_bytes += bytes;
  }
  end_call(wt, launches, CallBytes{});
  return 0;
}


int b2s_checksum_batch(uint32_t alg, uint32_t n, const uint8_t* const* src, const uint64_t* len, uint64_t* out) {
  if (n && (!src || !len || !out)) return fail(B2S_E_ARG, "null argument%s");
  if (!want_sharding(n)) return checksum_host(alg, n, src, len, out);
  return shard_over_devices(n, [&](const std::vector<uint32_t>& idx) {
    const uint32_t m = (uint32_t)idx.size();
    std::vector<const uint8_t*> p(m);
    std::vector<uint64_t> l(m), o(m);
    for (uint32_t k = 0; k < m; k++) {
      p[k] = src[idx[k]];
      l[k] = len[idx[k]];
    }
    int rc = checksum_host(alg, m, p.data(), l.data(), o.data());
    if (!rc)
      for (uint32_t k = 0; k < m; k++) out[idx[k]] = o[k];
    return rc;
  });
}
int b2s_checksum_packed(uint32_t alg, uint32_t n, const uint8_t* base, const uint64_t* off, const uint64_t* len,
                        uint64_t* out) {
  if (n && (!base || !off || !len || !out)) return fail(B2S_E_ARG, "null argument%s");
  std::vector<const uint8_t*> ptr(n);
  for (uint32_t i = 0; i < n; i++) ptr[i] = base + off[i];
  return checksum_host(alg, n, ptr.data(), len, out);
}

// ------------------------------------------------------------------------------------------------------------
// write side
// ------------------------------------------------------------------------------------------------------------
int b2s_compress_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                     uint32_t checksum_alg, uint32_t n, const void* d_src_base, const uint64_t* src_off,
                     const uint64_t* src_len, void* d_dst_base, uint64_t dst_cap, uint64_t* dst_off,
                     uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  Device* D;
  int rc = get_device(dev_index, &D);
  if (rc) return rc;
  if (checksum_alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (dst_total) *dst_total = 0;
  if (!n) return 0;
  if (!src_off || !src_len || !dst_off || !dst_len || !status) return fail(B2S_E_ARG, "null argument%s");
  Lane& Ln = D->lane[kLaneWrite];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  CompressJob J;
  uint64_t launches = 0;
  rc = compress_chunk(S, D->tabs, codec, level, block_size_or_default(codec_block_size), checksum_alg, n, src_off,
                      src_len, (const uint8_t*)d_src_base, (uint8_t*)d_dst_base, dst_cap, J, &launches);
  if (rc) return rc;
  CU(cudaEventSynchronize(S.ev_a));
  CU(cudaGetLastError());
  memcpy(dst_off, J.h.dst_off, (size_t)n * 8);
  memcpy(dst_len, J.h.dst_len, (size_t)n * 8);
  memcpy(status, J.h.status, (size_t)n * 4);
  if (checksum_out) {
    if (checksum_alg) memcpy(checksum_out, J.h.cks, (size_t)n * 8);
    else memset(checksum_out, 0, (size_t)n * 8);
  }
  uint64_t total = J.h.total[0] + stream_overhead(codec) * n, srcb = 0;
  for (uint32_t i = 0; i < n; i++) srcb += src_len[i];
  if (dst_total) *dst_total = total;
  end_call(wt, launches, CallBytes{srcb, total, 0, 0}, &S);
  return 0;
}

// shared engine for the host-pointer write path.  packed_dst != nullptr: outputs back to back into that arena.
static int compress_host(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t alg, uint32_t n,
                         const uint8_t* const* src, const uint64_t* src_len, uint8_t* packed_dst, uint64_t packed_cap,
                         uint8_t* const* dst, const uint64_t* dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                         uint64_t* dst_total, uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  Device* D;
  int rc = get_device(t_device, &D);
  if (rc) return rc;
  if (alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (dst_total) *dst_total = 0;
  if (!n) return 0;
  Lane& Ln = D->lane[kLaneWrite];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  const uint32_t bs = block_size_or_default(codec_block_size);
  if ((rc = check_codec_block(codec, bs))) return rc;  // before anything is staged
  const std::vector<uint32_t> starts = chunk_starts(n, src_len, kChunkStreams, g_host_chunk_bytes);
  std::vector<CompressJob> jobs(starts.size() - 1);
  std::vector<Run> runs;
  std::vector<uint64_t> dev_off;
  uint64_t launches = 0, run_off = 0;

  auto enqueue = [&](Slot& S, size_t c, uint32_t i0, uint32_t cnt) -> int {
    uint64_t bound = 0, bytes = 0;
    for (uint32_t k = 0; k < cnt; k++) bound += b2s_compress_bound(codec, bs, src_len[i0 + k]);
    if (int r = S.dst.ensure(bound + 64)) return r;
    dev_off.resize(cnt);
    if (int r = upload_chunk(S, cnt, src + i0, src_len + i0, dev_off.data(), runs, &bytes)) return r;
    t_timing.h2d_bytes += bytes;
    t_timing.src_bytes += bytes;
    return compress_chunk(S, D->tabs, codec, level, bs, alg, cnt, dev_off.data(), src_len + i0,
                          (const uint8_t*)S.src.p, (uint8_t*)S.dst.p, S.dst.cap, jobs[c], &launches);
  };
  auto finish = [&](Slot& S, size_t c, uint32_t i0, uint32_t cnt) -> int {
    const CompressLayout& H = jobs[c].h;
    CU(cudaEventSynchronize(S.ev_a));
    add_times(S, Family::kCodec);
    const uint64_t chunk_total = H.total[0] + stream_overhead(codec) * cnt;
    for (uint32_t k = 0; k < cnt; k++) {
      status[i0 + k] = H.status[k];
      dst_len[i0 + k] = H.dst_len[k];
      dst_off[i0 + k] = run_off + H.dst_off[k];
      if (checksum_out) checksum_out[i0 + k] = alg ? H.cks[k] : 0;
    }
    // a stream has at least its framing bytes, and no status but B2S_E_DST_TOO_SMALL
    const int r = download_chunk(S, cnt, H.dst_off, H.dst_len, chunk_total, packed_dst, packed_cap, run_off,
                                 dst ? dst + i0 : nullptr, dst_cap ? dst_cap + i0 : nullptr, status + i0);
    run_off += chunk_total;
    t_timing.dst_bytes += chunk_total;
    return r;
  };

  if (int r = run_chunks(Ln.slot, g_nslot, starts, {{0, enqueue}, {(size_t)g_nslot, finish}}, retire_slot))
    return r;
  CU(cudaGetLastError());
  if (dst_total) *dst_total = run_off;
  end_call(wt, launches, CallBytes{});
  return 0;
}

int b2s_compress_batch(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t n,
                       const uint8_t* const* src, const uint64_t* src_len, uint8_t* const* dst,
                       const uint64_t* dst_cap, uint64_t* dst_len, uint64_t* checksum_out, int32_t* status) {
  if (n && (!src || !src_len || !dst || !dst_cap || !dst_len || !status)) return fail(B2S_E_ARG, "null argument%s");
  if (!want_sharding(n)) {
    std::vector<uint64_t> off(n);
    return compress_host(codec, level, codec_block_size, checksum_alg, n, src, src_len, nullptr, 0, dst, dst_cap, off.data(),
                         dst_len, nullptr, checksum_out, status);
  }
  return shard_over_devices(n, [&](const std::vector<uint32_t>& idx) {
    const uint32_t m = (uint32_t)idx.size();
    std::vector<const uint8_t*> sp(m);
    std::vector<uint8_t*> dp(m);
    std::vector<uint64_t> sl(m), dc(m), dl(m), ck(m), off(m);
    std::vector<int32_t> st(m);
    for (uint32_t k = 0; k < m; k++) {
      sp[k] = src[idx[k]];
      sl[k] = src_len[idx[k]];
      dp[k] = dst[idx[k]];
      dc[k] = dst_cap[idx[k]];
    }
    int rc = compress_host(codec, level, codec_block_size, checksum_alg, m, sp.data(), sl.data(), nullptr, 0, dp.data(),
                           dc.data(), off.data(), dl.data(), nullptr, ck.data(), st.data());
    if (!rc)
      for (uint32_t k = 0; k < m; k++) {
        dst_len[idx[k]] = dl[k];
        status[idx[k]] = st[k];
        if (checksum_out) checksum_out[idx[k]] = ck[k];
      }
    return rc;
  });
}

int b2s_compress_packed(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t n,
                        const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len, uint8_t* dst_base,
                        uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                        uint64_t* checksum_out, int32_t* status) {
  if (n && (!src_base || !src_off || !src_len || !dst_base || !dst_off || !dst_len || !status))
    return fail(B2S_E_ARG, "null argument%s");
  std::vector<const uint8_t*> ptr(n);
  for (uint32_t i = 0; i < n; i++) ptr[i] = src_base + src_off[i];
  return compress_host(codec, level, codec_block_size, checksum_alg, n, ptr.data(), src_len, dst_base, dst_cap, nullptr,
                       nullptr, dst_off, dst_len, dst_total, checksum_out, status);
}

// ------------------------------------------------------------------------------------------------------------
// write side, serialized shuffle: partition records by reduce id, then compress every partition
// ------------------------------------------------------------------------------------------------------------
uint64_t b2s_partition_compress_bound(uint32_t codec, uint32_t codec_block_size, uint32_t num_partitions,
                                      uint64_t rec_bytes) {
  if (codec == B2S_CODEC_NONE) return rec_bytes;
  // k non-empty partitions of L_p bytes: sum ceil(L_p / bs) <= (rec_bytes + k (bs - 1)) / bs, and every bound below
  // grows with k, which is at most min(num_partitions, rec_bytes)
  const uint64_t bs = block_size_or_default(codec_block_size);
  const uint64_t k = std::min<uint64_t>(num_partitions, rec_bytes);
  const uint64_t nb = (rec_bytes + k * (bs - 1)) / bs;
  switch (codec) {
    case B2S_CODEC_LZ4BLOCK: return rec_bytes + (nb + k) * 21;
    case B2S_CODEC_SNAPPY_XERIAL: return 16 * k + nb * 37 + rec_bytes + rec_bytes / 6;
    case B2S_CODEC_ZSTD: return rec_bytes + nb * 3 + 9 * k;
    default: return rec_bytes;
  }
}

// checksum of a zero-length slice (what b2s_checksum_* returns for it): Adler-32 starts at 1, the CRCs at 0
static uint64_t empty_checksum(uint32_t alg) { return alg == B2S_CHECKSUM_ADLER32 ? 1 : 0; }

// first record whose bytes reach past rec_bytes, by bisection over the device record offsets (error path only)
static uint64_t first_record_past(const uint64_t* d_off, const uint32_t* d_len, uint64_t n, uint64_t rec_bytes) {
  uint64_t lo = 0, hi = n;  // answer in [lo, hi)
  while (lo + 1 < hi) {
    const uint64_t mid = lo + (hi - lo) / 2;
    uint64_t o = 0;
    if (cudaMemcpy(&o, d_off + mid, 8, cudaMemcpyDeviceToHost) != cudaSuccess) break;
    if (o > rec_bytes) hi = mid;  // record mid starts past the end: the first offender is earlier
    else lo = mid;
  }
  for (uint64_t i = lo; i < hi; i++) {  // lo is the last record starting within rec_bytes
    uint64_t o = 0;
    uint32_t l = 0;
    if (cudaMemcpy(&o, d_off + i, 8, cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(&l, d_len + i, 4, cudaMemcpyDeviceToHost) != cudaSuccess)
      break;
    if (o + l > rec_bytes) return i;
  }
  return lo;
}

// Where a partition call's reduce ids come from: the caller's (kGiven, one per record), or computed from the rows on
// the device: Spark's HashPartitioning ids by the key columns (kHash), its RangePartitioner ids over n_bounds bound rows
// of bound_bytes in host memory, bound_len[j] each (kRange), or its RoundRobinPartitioning ids from position start, the
// rows sorted first when sort is set (kRoundRobin)
struct RowIds {
  enum Kind { kGiven, kHash, kRange, kRoundRobin } kind = kGiven;
  KeySpec keys;
  uint32_t n_bounds = 0;
  const uint8_t* bound_base = nullptr;
  uint64_t bound_bytes = 0;
  const uint32_t* bound_len = nullptr;
  uint32_t start = 0;
  bool sort = false;

  static RowIds hash(const KeySpec& keys) {
    RowIds ids;
    ids.kind = kHash;
    ids.keys = keys;
    return ids;
  }
  static RowIds range(const KeySpec& keys, uint32_t n_bounds, const uint8_t* bound_base, uint64_t bound_bytes,
                      const uint32_t* bound_len) {
    RowIds ids;
    ids.kind = kRange;
    ids.keys = keys;
    ids.n_bounds = n_bounds;
    ids.bound_base = bound_base;
    ids.bound_bytes = bound_bytes;
    ids.bound_len = bound_len;
    return ids;
  }
  // SinglePartition: the range ids of no bounds, every id 0, with every record still checked by the range kernel
  static RowIds single_partition(const KeySpec& keys) { return range(keys, 0, nullptr, 0, nullptr); }
  static RowIds round_robin(int32_t start, uint32_t sort) {
    RowIds ids;
    ids.kind = kRoundRobin;
    ids.start = (uint32_t)start;
    ids.sort = sort != 0;
    return ids;
  }
};

// The B2S_E_ARG of a rows call's verdict word (~0: none): a bad record (kHashBad*, launch_rows_hash), or for a range
// call a bad bound or a bad record (launch_rows_range), or for a round-robin call a bad record
// (launch_rows_round_robin_hash)
static int row_ids_verdict(const RowIds& ids, uint64_t v) {
  static const char* const why[] = {"", "bound_len is below 4", "its size prefix is not bound_len - 4",
                                    "its row does not hold a key slot", "its row does not hold a key's null word",
                                    "a string key runs past its row",
                                    "a decimal key's size is not 1..16 or it runs past its row"};
  static const char* const rec_why[] = {"", "rec_len is below 4", "its size prefix is not rec_len - 4"};
  char msg[256];
  if (ids.kind == RowIds::kRoundRobin) {
    snprintf(msg, sizeof msg, "record %llu is not a serialized UnsafeRow: %s", (unsigned long long)(v >> 3),
             (v & 7) == kRowsBadWords ? "its row size is not a multiple of 8" : rec_why[v & 7]);
    return fail(B2S_E_ARG, "%s", msg);
  }
  if (ids.kind == RowIds::kRange && !(v & kRangeBadRecord)) {
    if ((v & 7) == kRangeBadOrder)
      snprintf(msg, sizeof msg, "bound %llu is not above the bound before it: the bounds must be strictly increasing",
               (unsigned long long)(v >> 3));
    else
      snprintf(msg, sizeof msg, "bound %llu is not a serialized row of the key columns: %s",
               (unsigned long long)(v >> 3), why[v & 7]);
    return fail(B2S_E_ARG, "%s", msg);
  }
  v &= ~kRangeBadRecord;
  snprintf(msg, sizeof msg, "record %llu is not a serialized row of the key columns: %s", (unsigned long long)(v >> 3),
           (v & 7) < 3 ? rec_why[v & 7] : why[v & 7]);
  return fail(B2S_E_ARG, "%s", msg);
}

// the range call's bounds into their workspace at d_ws: the rows and their offsets, one upload each
static int upload_bounds(const RowIds& ids, uint8_t* d_ws, RangeWs* w, cudaStream_t st) {
  *w = carve_rows_range_ws(d_ws, ids.n_bounds, ids.bound_bytes);
  if (!ids.n_bounds) return 0;
  std::vector<uint64_t> off(ids.n_bounds + 1, 0);
  for (uint32_t j = 0; j < ids.n_bounds; j++) off[j + 1] = off[j] + ids.bound_len[j];
  CU(cudaMemcpyAsync(w->off, off.data(), off.size() * 8, cudaMemcpyHostToDevice, st));
  if (ids.bound_bytes) CU(cudaMemcpyAsync(w->rows, ids.bound_base, ids.bound_bytes, cudaMemcpyHostToDevice, st));
  return 0;  // a copy from pageable memory has taken its source when it returns, so off may go
}

// The round-robin step's order: every record checked (lowering P's bad-record word) and, with the sort (sws / rws:
// the whole-row sort's workspaces, else nullptr), hashed and sorted by its whole-row key.  *order = the record at each
// sorted position (nullptr: input order).  One 8-byte readback per refinement round; the first also brings the
// bad-record word and the byte total, so a bad record fails the call, and a record past rec_bytes ends the sort,
// before any round reads it (the partition step's readback then names that record).
static int round_robin_order(Slot& S, const RowIds& ids, uint64_t n, const uint8_t* d_rec, uint64_t rec_bytes,
                             const uint32_t* d_len, const PartitionPlan& P, uint8_t* sws, uint8_t* rws,
                             const uint32_t** order, uint64_t* launches) {
  cudaStream_t st = S.st;
  *order = nullptr;
  launch_rows_round_robin_hash(d_rec, rec_bytes, P.src_off, d_len, n, rws ? rows_whole_words(sws, n) : nullptr,
                               rws ? rows_refine_klen(rws, n) : nullptr, P.readback, st, launches);
  if (!rws) return 0;
  launch_rows_whole_order(n, sws, rws, st, launches);
  if (int rc = S.hmeta.ensure(24)) return rc;
  uint64_t* rb = (uint64_t*)S.hmeta.p;  // [tied records | runs << 32, bad record, byte total]
  for (uint32_t d = 4, round = 0;; d += kKeyChunkBytes, round++) {
    launch_rows_refine_mark(n, d, rws, 0, st, launches);
    CU(cudaMemcpyAsync(rb, rows_refine_readback(rws, n, 0), 8, cudaMemcpyDeviceToHost, st));
    if (!round) CU(cudaMemcpyAsync(rb + 1, P.readback, 16, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    if (!round && rb[1] != ~0ull) return row_ids_verdict(ids, rb[1]);
    if (!round && rb[2] != rec_bytes) return 0;
    const uint64_t tied = rb[0] & 0xffffffffull, runs = rb[0] >> 32;
    if (!tied) break;
    launch_rows_whole_refine_round(d_rec, P.src_off, d_len, n, tied, runs, d, sws, rws, st, launches);
  }
  *order = rows_refine_order(rws, n, 0);
  return 0;
}

// The partition step and the compression of the non-empty partitions, on device-resident records.  d_dst receives the
// .data arena (dst_cap bytes); *arena_bytes the bytes it needs.  Returns B2S_E_DST_TOO_SMALL (status[] set for the
// partitions that do not fit) when dst_cap is short.  part_start (optional) receives the R + 1 partition offsets of the
// partitioned records, which are in d_dst (codec NONE) or S.parena.  ids: given (d_part), or computed from the rows on
// the device between the offsets and the radix passes (marks F0 and F1 bracket that step: the hash kernel, the range
// call's bound checks and id kernel, or the round-robin call's hash, sort and id kernel), where a bad record or bound
// fails the call.  plan (optional, n > 0): receives the partition plan, whose arrays in S.pws outlive the call until
// the slot's next use (compression does not touch them).
static int partition_compress_run(Device* D, Slot& S, uint32_t codec, int32_t level, uint32_t bs, uint32_t alg,
                                  uint32_t R, uint64_t n, const uint8_t* d_rec, uint64_t rec_bytes,
                                  const uint32_t* d_len, const uint32_t* d_part, uint8_t* d_dst, uint64_t dst_cap,
                                  uint64_t* dst_off, uint64_t* dst_len, uint64_t* checksum_out, int32_t* status,
                                  uint64_t* arena_bytes, uint64_t* launches, std::vector<uint64_t>* part_start,
                                  const RowIds& ids, PartitionPlan* plan) {
  cudaStream_t st = S.st;
  std::vector<uint64_t> pstart(R), plen(R);
  const bool given = ids.kind == RowIds::kGiven, range = ids.kind == RowIds::kRange;
  const bool rr_sort = ids.kind == RowIds::kRoundRobin && ids.sort && R > 1;  // R == 1: Spark does not sort
  CU(S.mark(P0, st));
  PartitionPlan P;
  if (n) {
    const size_t pws = partition_ws_bytes(n, R, !given);
    const size_t sws = rr_sort ? rows_sort_ws_bytes(n, kKeyPrefixBytes) : 0;
    int rc = S.pws.ensure(pws + (range ? rows_range_ws_bytes(ids.n_bounds, ids.bound_bytes) : 0) +
                          (rr_sort ? sws + rows_refine_ws_bytes(n, 0) : 0));
    if (rc) return rc;
    uint8_t* ws = (uint8_t*)S.pws.p;
    RangeWs rw;
    if (range)
      if (int rc = upload_bounds(ids, ws + pws, &rw, st)) return rc;
    if (given) {
      launch_partition(d_len, d_part, n, R, ws, &P, st, launches);
    } else {
      launch_partition_offsets(d_len, nullptr, n, R, ws, &P, st, launches);
      CU(S.mark(F0, st, *launches));
      const uint32_t* order = nullptr;
      switch (ids.kind) {
        case RowIds::kRoundRobin:
          if (int rc = round_robin_order(S, ids, n, d_rec, rec_bytes, d_len, P, rr_sort ? ws + pws : nullptr,
                                         rr_sort ? ws + pws + sws : nullptr, &order, launches))
            return rc;
          launch_rows_round_robin_ids(n, ids.start, R, P.ids, st, launches);
          break;
        case RowIds::kRange:
          launch_rows_range(d_rec, rec_bytes, P.src_off, d_len, n, ids.keys, rw, ids.n_bounds, P.ids, P.readback, st,
                            launches);
          break;
        default:
          launch_rows_hash(d_rec, rec_bytes, P.src_off, d_len, n, ids.keys, R, P.ids, P.readback, st, launches);
      }
      CU(S.mark(F1, st, *launches));
      launch_partition_order(d_len, P.ids, n, R, ws, &P, st, launches, order);
    }
    // the one readback between the partition step and compression: [bad id (ids: bad record or bound), byte total,
    // partition offsets]
    rc = S.hmeta.ensure(P.readback_bytes);
    if (rc) return rc;
    const uint64_t* rb = (const uint64_t*)S.hmeta.p;
    CU(cudaMemcpyAsync(S.hmeta.p, P.readback, P.readback_bytes, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    char msg[256];
    if (!given && rb[0] != ~0ull) return row_ids_verdict(ids, rb[0]);
    if (rb[0] != ~0ull) {
      uint32_t id = 0;
      CU(cudaMemcpy(&id, d_part + rb[0], 4, cudaMemcpyDeviceToHost));
      snprintf(msg, sizeof msg, "record %llu has partition id %u, num_partitions is %u", (unsigned long long)rb[0], id, R);
      return fail(B2S_E_ARG, "%s", msg);
    }
    if (rb[1] != rec_bytes) {
      if (rb[1] > rec_bytes)
        snprintf(msg, sizeof msg, "rec_len sums to %llu bytes, rec_bytes is %llu: record %llu ends past rec_bytes",
                 (unsigned long long)rb[1], (unsigned long long)rec_bytes,
                 (unsigned long long)first_record_past(P.src_off, d_len, n, rec_bytes));
      else
        snprintf(msg, sizeof msg, "rec_len sums to %llu bytes, rec_bytes is %llu", (unsigned long long)rb[1],
                 (unsigned long long)rec_bytes);
      return fail(B2S_E_ARG, "%s", msg);
    }
    uint64_t next = rec_bytes;
    for (uint32_t p = R; p-- > 0;) {
      const uint64_t s = rb[2 + p];
      pstart[p] = s == ~0ull ? next : s;
      plen[p] = next - pstart[p];
      next = pstart[p];
    }
    if (plan) *plan = P;
  } else if (rec_bytes) {
    return fail(B2S_E_ARG, "rec_len sums to 0 bytes, rec_bytes is %s", std::to_string(rec_bytes).c_str());
  } else if (range && ids.n_bounds) {  // no records: the bounds are still checked, with a readback of their verdict
    int rc = S.pws.ensure(rows_range_ws_bytes(ids.n_bounds, ids.bound_bytes));
    if (rc) return rc;
    RangeWs rw;
    if (int rc = upload_bounds(ids, (uint8_t*)S.pws.p, &rw, st)) return rc;
    CU(cudaMemsetAsync(rw.verdict, 0xff, 8, st));
    CU(S.mark(F0, st, *launches));
    launch_rows_range(nullptr, 0, nullptr, nullptr, 0, ids.keys, rw, ids.n_bounds, nullptr, rw.verdict, st,
                      launches);
    CU(S.mark(F1, st, *launches));
    rc = S.hmeta.ensure(8);
    if (rc) return rc;
    CU(cudaMemcpyAsync(S.hmeta.p, rw.verdict, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    const uint64_t v = *(const uint64_t*)S.hmeta.p;
    if (v != ~0ull) return row_ids_verdict(ids, v);
  }
  if (part_start) {
    part_start->assign(pstart.begin(), pstart.end());
    part_start->push_back(rec_bytes);
  }

  if (codec == B2S_CODEC_NONE) {
    *arena_bytes = rec_bytes;
    memcpy(dst_off, pstart.data(), (size_t)R * 8);
    memcpy(dst_len, plen.data(), (size_t)R * 8);
    if (rec_bytes > dst_cap) {
      for (uint32_t p = 0; p < R; p++) status[p] = pstart[p] + plen[p] > dst_cap ? B2S_E_DST_TOO_SMALL : B2S_OK;
      return fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s bytes of records", std::to_string(rec_bytes).c_str());
    }
    launch_partition_gather(d_rec, d_len, n, P, d_dst, st, launches);
    CU(S.mark(P1, st));
    if (alg && rec_bytes) {  // over every partition, empty ones included
      int rc = checksum_chunk_dev(D, S, alg, R, d_dst, pstart.data(), plen.data(), checksum_out, rec_bytes, launches);
      if (rc) return rc;
    } else {
      CU(cudaStreamSynchronize(st));
      for (uint32_t p = 0; p < R; p++) checksum_out[p] = alg ? empty_checksum(alg) : 0;
    }
    CU(cudaGetLastError());
    for (uint32_t p = 0; p < R; p++) status[p] = B2S_OK;
    return 0;
  }

  // compress the non-empty partitions of the partitioned arena with the pipeline behind b2s_compress_dev
  std::vector<uint32_t> ne;
  for (uint32_t p = 0; p < R; p++)
    if (plen[p]) ne.push_back(p);
  const uint32_t m = (uint32_t)ne.size();
  std::vector<uint64_t> ne_off(m), ne_len(m);
  for (uint32_t k = 0; k < m; k++) {
    ne_off[k] = pstart[ne[k]];
    ne_len[k] = plen[ne[k]];
  }
  CompressJob J;
  uint64_t total = 0;
  if (m) {
    int rc = S.parena.ensure(rec_bytes + 64);
    if (rc) return rc;
    launch_partition_gather(d_rec, d_len, n, P, (uint8_t*)S.parena.p, st, launches);
    CU(S.mark(P1, st));
    rc = compress_chunk(S, D->tabs, codec, level, bs, alg, m, ne_off.data(), ne_len.data(),
                        (const uint8_t*)S.parena.p, d_dst, dst_cap, J, launches);
    if (rc) return rc;
    CU(cudaEventSynchronize(S.ev_a));
    CU(cudaGetLastError());
    total = J.h.total[0] + stream_overhead(codec) * m;
  }
  *arena_bytes = total;
  bool short_dst = false;
  uint64_t at = 0;  // an empty partition sits where the next non-empty one starts
  for (uint32_t p = 0, k = 0; p < R; p++) {
    if (k < m && ne[k] == p) {
      dst_off[p] = J.h.dst_off[k];
      dst_len[p] = J.h.dst_len[k];
      checksum_out[p] = alg ? J.h.cks[k] : 0;
      status[p] = J.h.status[k];
      if (dst_off[p] + dst_len[p] > dst_cap) status[p] = B2S_E_DST_TOO_SMALL;
      short_dst |= status[p] == B2S_E_DST_TOO_SMALL;
      at = dst_off[p] + dst_len[p];
      k++;
    } else {
      dst_off[p] = at;
      dst_len[p] = 0;
      checksum_out[p] = alg ? empty_checksum(alg) : 0;
      status[p] = B2S_OK;
    }
  }
  if (short_dst) return fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s bytes of the .data arena",
                             std::to_string(total).c_str());
  return 0;
}

// What every map-side partition call takes besides its records: the device (packed: the thread's), the codec step's
// settings, num_partitions, and the caller's .data arena with its per-partition outputs
struct MapCall {
  bool packed;
  uint32_t dev_index;
  uint32_t codec;
  int32_t level;
  uint32_t bs;  // block_size_or_default's
  uint32_t alg;
  uint32_t R;
  uint8_t* dst_base;
  uint64_t dst_cap;
  uint64_t* dst_off;
  uint64_t* dst_len;
  uint64_t* dst_total;
  uint64_t* checksum_out;
  int32_t* status;
};

// n records of bytes at rec, their lengths at len: a call's input (host memory when packed), or the rows its own step
// left on the slot
struct MapRows {
  uint64_t n;
  const uint8_t* rec;
  uint64_t bytes;
  const uint32_t* len;
};

// rec_part is read only for given ids
static int partition_args(const MapCall& c, const MapRows& in, const uint32_t* rec_part, const RowIds& ids) {
  if (c.alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (c.codec != B2S_CODEC_NONE)
    if (int rc = check_codec_block(c.codec, c.bs)) return rc;
  if (c.R < 1 || c.R > (1u << 24)) return fail(B2S_E_ARG, "num_partitions must be in [1, 2^24]%s");
  if (in.n > 0xffffffffull) return fail(B2S_E_ARG, "more than 2^32 - 1 records in one call%s");
  if ((in.n && (!in.len || (!rec_part && ids.kind == RowIds::kGiven))) || (in.bytes && !in.rec) || !c.dst_off ||
      !c.dst_len || !c.status)
    return fail(B2S_E_ARG, "null argument%s");
  if (in.bytes && !c.dst_base) return fail(B2S_E_ARG, "null argument%s");
  return 0;
}

static Family partition_family(uint32_t codec) {
  return codec == B2S_CODEC_NONE ? Family::kPartitionNone : Family::kPartition;
}

// what a cached store keeps: the exchange-cache key and where to report whether it was stored
struct ExStore {
  int32_t shuffle;
  int64_t map;
  int32_t* cached;
};

// the largest whole-task buffer a call keeps for the next one (SortBufferTrim, PartialAggTrim)
constexpr size_t kSortKeepBytes = 1ull << 30;

// The aggregation step's buffers, sized by the call's records (staged and folded values, the partial rows), are given
// back when the call ends if they are larger than the sorts keep, so one large map task does not hold them for the life
// of the process
struct PartialAggTrim {
  Slot& S;
  ~PartialAggTrim() {
    for (DevBuf* b : {&S.fws, &S.aggrows, &S.xrows})
      if (b->cap > kSortKeepBytes) b->release();
  }
};

// The partition + compress step of a map-side call over the rows on S (its own step's, or its records), with the ids
// of ids (given: d_part), into the caller's arena, or (packed) into S.dst, sized by the bound, then one download of what
// fits (*fit bytes), a short caller arena flagged after the run.  Sets the per-partition outputs and *dst_total to the
// *arena bytes the arena needs; B2S_E_DST_TOO_SMALL leaves them set.  store (packed): the partitioned records, with a
// rows call's record boundaries, kept as an exchange-cache entry when the call succeeds.
static int partition_tail(Device* D, Slot& S, const MapCall& c, const MapRows& rows, const uint32_t* d_part,
                          const RowIds& ids, const ExStore* store, uint64_t* arena, uint64_t* fit,
                          uint64_t* launches) {
  cudaStream_t st = S.st;
  uint8_t* d_dst = c.dst_base;
  uint64_t cap = c.dst_cap;
  if (c.packed) {
    if (int rc = S.dst.ensure(b2s_partition_compress_bound(c.codec, c.bs, c.R, rows.bytes) + 64)) return rc;
    d_dst = (uint8_t*)S.dst.p;
    cap = S.dst.cap;
  }
  std::vector<uint64_t> cks(c.R), part_start;
  PartitionPlan P;
  int rc = partition_compress_run(D, S, c.codec, c.level, c.bs, c.alg, c.R, rows.n, rows.rec, rows.bytes, rows.len,
                                  d_part, d_dst, cap, c.dst_off, c.dst_len, cks.data(), c.status, arena, launches,
                                  store ? &part_start : nullptr, ids, &P);
  if (rc && rc != B2S_E_DST_TOO_SMALL) return rc;
  *fit = 0;
  if (c.packed) {
    *fit = std::min(*arena, c.dst_cap);
    if (*arena > c.dst_cap) {
      for (uint32_t p = 0; p < c.R; p++)
        if (c.dst_len[p] && c.dst_off[p] + c.dst_len[p] > c.dst_cap) c.status[p] = B2S_E_DST_TOO_SMALL;
      rc = fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s bytes of the .data arena", std::to_string(*arena).c_str());
    }
    CU(S.mark(D0, st));
    if (*fit) CU(cudaMemcpyAsync(c.dst_base, S.dst.p, *fit, cudaMemcpyDeviceToHost, st));
    CU(S.mark(D1, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
  }
  if (c.checksum_out) memcpy(c.checksum_out, cks.data(), (size_t)c.R * 8);
  if (c.dst_total) *c.dst_total = *arena;
  if (store && !rc) {
    // the partitioned records are still in this slot (its lane is held): in front of compression, or the arena itself
    // for codec NONE
    const uint8_t* parts = (const uint8_t*)(c.codec == B2S_CODEC_NONE ? S.dst.p : S.parena.p);
    // a rows call's entry keeps its record boundaries: the plan's offsets, also still in this slot (S.pws); S.hmeta
    // (only grown) has held the partition step's readback of R + 2 words
    ExBounds rb{&P, rows.n, (uint64_t*)S.hmeta.p, launches};
    *store->cached = ex_store(D->ordinal, st, store->shuffle, store->map, parts, rows.bytes, std::move(part_start),
                              ids.kind == RowIds::kGiven ? nullptr : &rb);
  }
  return rc;
}

// A map-side call's own step on S: from its records on the device to the rows it partitions (launches: its count)
using MapStep = std::function<int(Slot& S, const MapRows& records, MapRows* rows, uint64_t* launches)>;

// the step of a call that partitions its records as they are
static int pass_through(Slot&, const MapRows& in, MapRows* rows, uint64_t*) {
  *rows = in;
  return 0;
}

// A map-side call on the write lane's slot 0, after its checks.  Without a usable device a rows call reports B2S_E_CUDA
// (as the sort calls do) and a call with given ids B2S_E_NOT_INIT.  Then (packed) one upload of [records | rec_len |
// rec_part, for given ids] between marks H0 and H1 (the whole map output is partitioned at once: no chunking), the
// call's step to the rows it partitions (*n_out: how many), and the partition + compress step over them.
static int write_lane_run(const WallTimer& wt, const MapCall& c, const MapRows& in, const uint32_t* rec_part,
                          const RowIds& ids, const ExStore* store, Family f, uint64_t* n_out, const MapStep& step) {
  const bool given = ids.kind == RowIds::kGiven;
  if (!given && !g_ctx)
    if (int rc = no_device()) return rc;
  Device* D;
  if (int rc = get_device(c.packed ? t_device : c.dev_index, &D)) return rc;
  Lane& Ln = D->lane[kLaneWrite];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  const PartialAggTrim trim{S};
  cudaStream_t st = S.st;
  MapRows d_in = in;
  const uint32_t* d_part = rec_part;
  if (c.packed) {
    const size_t rec_sz = align_up(in.bytes, 16), len_sz = align_up(in.n * 4, 16);
    if (int rc = S.src.ensure(rec_sz + (given ? 2 : 1) * len_sz + 64)) return rc;
    uint8_t* d = (uint8_t*)S.src.p;
    d_in.rec = d;
    d_in.len = (const uint32_t*)(d + rec_sz);
    d_part = (const uint32_t*)(d + rec_sz + len_sz);
    CU(S.mark(H0, st));
    if (in.bytes) CU(cudaMemcpyAsync(d, in.rec, in.bytes, cudaMemcpyHostToDevice, st));
    if (in.n) {
      CU(cudaMemcpyAsync(d + rec_sz, in.len, in.n * 4, cudaMemcpyHostToDevice, st));
      if (given) CU(cudaMemcpyAsync(d + rec_sz + len_sz, rec_part, in.n * 4, cudaMemcpyHostToDevice, st));
    }
    CU(S.mark(H1, st));
  }
  uint64_t launches = 0, arena = 0, fit = 0;
  MapRows rows{};
  if (int rc = step(S, d_in, &rows, &launches)) return rc;
  const int rc = partition_tail(D, S, c, rows, d_part, ids, store, &arena, &fit, &launches);
  if (rc && rc != B2S_E_DST_TOO_SMALL) return rc;
  if (n_out) *n_out = rows.n;
  const uint64_t h2d =
      c.packed ? in.bytes + in.n * (given ? 8 : 4) + (ids.kind == RowIds::kRange ? ids.bound_bytes : 0) : 0;
  end_call(wt, launches, CallBytes{in.bytes, arena, h2d, fit}, &S, f);
  return rc;
}

int b2s_partition_compress_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                               uint32_t checksum_alg, uint32_t num_partitions, uint64_t n_records,
                               const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
                               const uint32_t* rec_part, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                               uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{false, dev_index, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RowIds ids;
  if (int rc = partition_args(c, in, rec_part, ids)) return rc;
  return write_lane_run(wt, c, in, rec_part, ids, nullptr, partition_family(codec), nullptr, pass_through);
}

int b2s_partition_compress_packed(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
                                  uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base,
                                  uint64_t rec_bytes, const uint32_t* rec_len, const uint32_t* rec_part,
                                  uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                                  uint64_t* dst_total, uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{true, 0, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RowIds ids;
  if (int rc = partition_args(c, in, rec_part, ids)) return rc;
  return write_lane_run(wt, c, in, rec_part, ids, nullptr, partition_family(codec), nullptr, pass_through);
}

int b2s_partition_compress_cached_packed(int32_t shuffle_id, int64_t map_id, uint32_t codec, int32_t level,
                                         uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
                                         uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes,
                                         const uint32_t* rec_len, const uint32_t* rec_part, uint8_t* dst_base,
                                         uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                         uint64_t* checksum_out, int32_t* status, int32_t* cached) {
  if (!cached) return fail(B2S_E_ARG, "null argument%s");
  *cached = 0;
  if (int rc = exchange_ready()) return rc;
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{true, 0, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RowIds ids;
  if (int rc = partition_args(c, in, rec_part, ids)) return rc;
  const ExStore store{shuffle_id, map_id, cached};
  return write_lane_run(wt, c, in, rec_part, ids, &store, partition_family(codec), nullptr, pass_through);
}

// ------------------------------------------------------------------------------------------------------------
// read side
// ------------------------------------------------------------------------------------------------------------
// slices of a block must tile it exactly (S3ChecksumValidationStream walks .index differences over the block)
static int check_slices(uint32_t n, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len) {
  for (uint32_t i = 0; i < n; i++) {
    uint64_t sum = 0;
    if (slice_base[i + 1] < slice_base[i]) return fail(B2S_E_ARG, "slice_base must be non-decreasing%s");
    for (uint32_t q = slice_base[i]; q < slice_base[i + 1]; q++) sum += slice_len[q];
    if (sum != src_len[i]) return fail(B2S_E_ARG, "slice lengths of a block must sum to its length%s");
  }
  return 0;
}

int b2s_decompress_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const void* d_src_base,
                       const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                       const uint64_t* slice_len, const uint64_t* slice_checksum, void* d_dst_base, uint64_t dst_cap,
                       uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total, int32_t* status,
                       int32_t* bad_slice) {
  const WallTimer wt = begin_call();
  Device* D;
  int rc = get_device(dev_index, &D);
  if (rc) return rc;
  if (checksum_alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (dst_total) *dst_total = 0;
  if (!n) return 0;
  if (!src_off || !src_len || !dst_off || !dst_len || !status) return fail(B2S_E_ARG, "null argument%s");
  if (checksum_alg && (!slice_base || !slice_len || !slice_checksum)) return fail(B2S_E_ARG, "slice arrays required%s");
  if (checksum_alg && (rc = check_slices(n, src_len, slice_base, slice_len))) return rc;
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  DecompressJob J;
  uint64_t srcb = 0, launches = 0;
  for (uint32_t i = 0; i < n; i++) srcb += src_len[i];
  rc = decompress_phase_a(S, D->tabs, codec, checksum_alg, n, src_off, src_len, checksum_alg ? slice_base[n] : 0,
                          slice_base, slice_len, slice_checksum, (const uint8_t*)d_src_base, srcb, J, &launches);
  if (rc) return rc;
  CU(cudaEventSynchronize(S.ev_a));
  rc = decompress_enqueue_b(S, J, (const uint8_t*)d_src_base, (uint8_t*)d_dst_base, dst_cap, &launches);
  if (rc) return rc;
  CU(cudaEventSynchronize(S.ev_b));
  CU(cudaGetLastError());
  memcpy(dst_off, J.h.dst_off, (size_t)n * 8);
  memcpy(dst_len, J.h.dst_len, (size_t)n * 8);
  memcpy(status, J.h.status, (size_t)n * 4);
  if (bad_slice) memcpy(bad_slice, J.h.bad, (size_t)n * 4);
  if (dst_total) *dst_total = J.total_out;
  end_call(wt, launches, CallBytes{srcb, J.total_out, 0, 0}, &S);
  return 0;
}

static int decompress_host(uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* const* src,
                           const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
                           const uint64_t* slice_sum, uint8_t* packed_dst, uint64_t packed_cap, uint8_t* const* dst,
                           const uint64_t* dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                           int32_t* status, int32_t* bad_slice, bool size_only) {
  const WallTimer wt = begin_call();
  Device* D;
  int rc = get_device(t_device, &D);
  if (rc) return rc;
  if (alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (dst_total) *dst_total = 0;
  if (!n) return 0;
  if (alg) {
    // A block whose slices do not tile it (a fetch that came back short: storage/S3ShuffleBlockStream.scala:66-69,88-91
    // turns I/O errors into a silent EOF) is that block's problem, not the call's: the reference's validation stream
    // would run out of bytes inside some slice and raise "Invalid checksum detected" for this block only
    // (storage/S3ChecksumValidationStream.scala:72-74).  Such blocks get B2S_E_CHECKSUM + the slice index and are left
    // out of the batch; everything else is processed normally.
    std::vector<uint32_t> good;
    std::vector<int32_t> where(n, -1);
    for (uint32_t i = 0; i < n; i++) {
      if (slice_base[i + 1] < slice_base[i]) return fail(B2S_E_ARG, "slice_base must be non-decreasing%s");
      uint64_t sum = 0;
      int32_t first_short = -1;
      for (uint32_t q = slice_base[i]; q < slice_base[i + 1]; q++) {
        sum += slice_len[q];
        if (first_short < 0 && sum > src_len[i]) first_short = (int32_t)(q - slice_base[i]);
      }
      if (sum == src_len[i]) good.push_back(i);
      else where[i] = first_short >= 0 ? first_short : (int32_t)(slice_base[i + 1] - slice_base[i]) - (slice_base[i + 1] > slice_base[i] ? 1 : 0);
    }
    if (good.size() != n) {
      const uint32_t m = (uint32_t)good.size();
      std::vector<const uint8_t*> sp(m);
      std::vector<uint64_t> sl(m), dc(m), doff(m), dl(m), l, c;
      std::vector<uint8_t*> dp(m);
      std::vector<uint32_t> sb(m + 1, 0);
      std::vector<int32_t> st(m), bd(m, -1);
      for (uint32_t k = 0; k < m; k++) {
        const uint32_t i = good[k];
        sp[k] = src[i];
        sl[k] = src_len[i];
        if (dst) dp[k] = dst[i];
        if (dst_cap) dc[k] = dst_cap[i];
        for (uint32_t q = slice_base[i]; q < slice_base[i + 1]; q++) {
          l.push_back(slice_len[q]);
          c.push_back(slice_sum[q]);
        }
        sb[k + 1] = (uint32_t)l.size();
      }
      uint64_t total = 0;
      rc = m ? decompress_host(codec, alg, m, sp.data(), sl.data(), sb.data(), l.data(), c.data(), packed_dst, packed_cap,
                               dst ? dp.data() : nullptr, dst_cap ? dc.data() : nullptr, doff.data(), dl.data(), &total,
                               st.data(), bd.data(), size_only)
             : 0;
      if (rc) return rc;
      uint32_t k = 0;
      uint64_t at = 0;
      for (uint32_t i = 0; i < n; i++) {
        if (k < m && good[k] == i) {
          status[i] = st[k];
          dst_len[i] = dl[k];
          if (dst_off) dst_off[i] = doff[k];
          if (bad_slice) bad_slice[i] = bd[k];
          at = doff[k] + dl[k];
          k++;
        } else {
          status[i] = B2S_E_CHECKSUM;
          dst_len[i] = 0;
          if (dst_off) dst_off[i] = at;
          if (bad_slice) bad_slice[i] = where[i];
        }
      }
      if (dst_total) *dst_total = total;
      return 0;
    }
  }
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  if ((rc = check_decode_codec(codec, false))) return rc;  // before anything is staged
  const std::vector<uint32_t> starts = chunk_starts(n, src_len, kChunkStreams, g_host_chunk_bytes);
  std::vector<DecompressJob> jobs(starts.size() - 1);
  std::vector<Run> runs;
  std::vector<uint64_t> dev_off;
  uint64_t launches = 0, run_off = 0;

  auto stage_a = [&](Slot& S, size_t c, uint32_t i0, uint32_t cnt) -> int {
    DecompressJob& J = jobs[c];
    J.size_only = size_only;
    dev_off.resize(cnt);
    uint64_t bytes = 0;
    if (int r = upload_chunk(S, cnt, src + i0, src_len + i0, dev_off.data(), runs, &bytes)) return r;
    t_timing.h2d_bytes += bytes;
    t_timing.src_bytes += bytes;
    const uint32_t ns = alg ? slice_base[i0 + cnt] - slice_base[i0] : 0;
    return decompress_phase_a(S, D->tabs, codec, alg, cnt, dev_off.data(), src_len + i0, ns,
                              alg ? slice_base + i0 : nullptr, slice_len, slice_sum, (const uint8_t*)S.src.p, bytes,
                              J, &launches);
  };
  auto stage_b = [&](Slot& S, size_t c, uint32_t, uint32_t) -> int {
    DecompressJob& J = jobs[c];
    CU(cudaEventSynchronize(S.ev_a));
    if (size_only) {
      J.total_out = J.h.totals[1];
      CU(cudaMemcpyAsync(J.h.down, J.d.down, J.d.down_bytes, cudaMemcpyDeviceToHost, S.st));
      CU(cudaEventRecord(S.ev_b, S.st));
      return 0;
    }
    int r = S.dst.ensure(J.h.totals[1] + 64);
    if (r) return r;
    return decompress_enqueue_b(S, J, (const uint8_t*)S.src.p, (uint8_t*)S.dst.p, S.dst.cap, &launches);
  };
  auto stage_c = [&](Slot& S, size_t c, uint32_t i0, uint32_t) -> int {
    const DecompressJob& J = jobs[c];
    CU(cudaEventSynchronize(S.ev_b));
    if (!size_only) add_times(S, Family::kCodec);
    for (uint32_t k = 0; k < J.n; k++) {
      const uint32_t i = i0 + k;
      status[i] = J.h.status[k];
      dst_len[i] = J.h.dst_len[k];  // size_only: the decoded lengths of phase A
      if (bad_slice) bad_slice[i] = J.h.bad[k];
      if (dst_off) dst_off[i] = run_off + J.h.dst_off[k];
    }
    // a size_only call has no destination: nothing is copied
    const int r = download_chunk(S, J.n, J.h.dst_off, J.h.dst_len, J.total_out, packed_dst, packed_cap, run_off,
                                 dst ? dst + i0 : nullptr, dst_cap ? dst_cap + i0 : nullptr, status + i0);
    run_off += J.total_out;
    t_timing.dst_bytes += J.total_out;
    return r;
  };

  // lag chunks between the stages keep lag uploads / decodes queued on the device while the host waits for one chunk's
  // sizes (the write lane keeps g_nslot chunks in flight and would otherwise own the copy queues).
  const size_t lag = (size_t)std::max(1, std::min(g_read_lag, (g_nslot - 1) / 2));
  if (int r = run_chunks(Ln.slot, g_nslot, starts, {{0, stage_a}, {lag, stage_b}, {2 * lag, stage_c}}, retire_slot))
    return r;
  CU(cudaGetLastError());
  if (dst_total) *dst_total = run_off;
  end_call(wt, launches, CallBytes{});
  return 0;
}

// builds the flattened slice arrays used by the engine from the per-block pointer form
static void flatten_slices(uint32_t n, const uint32_t* n_slices, const uint64_t* const* slice_len,
                           const uint64_t* const* slice_checksum, std::vector<uint32_t>& base,
                           std::vector<uint64_t>& len, std::vector<uint64_t>& sum) {
  base.assign((size_t)n + 1, 0);
  for (uint32_t i = 0; i < n; i++) base[i + 1] = base[i] + n_slices[i];
  len.resize(base[n]);
  sum.resize(base[n]);
  for (uint32_t i = 0; i < n; i++)
    for (uint32_t k = 0; k < n_slices[i]; k++) {
      len[base[i] + k] = slice_len[i][k];
      sum[base[i] + k] = slice_checksum[i][k];
    }
}

int b2s_decompress_batch(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* const* src,
                         const uint64_t* src_len, const uint32_t* n_slices, const uint64_t* const* slice_len,
                         const uint64_t* const* slice_checksum, uint8_t* const* dst, const uint64_t* dst_cap,
                         uint64_t* dst_len, int32_t* status, int32_t* bad_slice) {
  if (n && (!src || !src_len || !dst || !dst_cap || !dst_len || !status)) return fail(B2S_E_ARG, "null argument%s");
  if (checksum_alg && n && (!n_slices || !slice_len || !slice_checksum)) return fail(B2S_E_ARG, "slice arrays required%s");
  std::vector<uint32_t> base;
  std::vector<uint64_t> len, sum;
  if (!want_sharding(n)) {
    if (checksum_alg) flatten_slices(n, n_slices, slice_len, slice_checksum, base, len, sum);
    return decompress_host(codec, checksum_alg, n, src, src_len, base.data(), len.data(), sum.data(), nullptr, 0, dst,
                           dst_cap, nullptr, dst_len, nullptr, status, bad_slice, false);
  }
  return shard_over_devices(n, [&](const std::vector<uint32_t>& idx) {
    const uint32_t m = (uint32_t)idx.size();
    std::vector<const uint8_t*> sp(m);
    std::vector<uint8_t*> dp(m);
    std::vector<uint64_t> sl(m), dc(m), dl(m);
    std::vector<uint32_t> ns(m), b;
    std::vector<const uint64_t*> slp(m), scp(m);
    std::vector<uint64_t> l, c;
    std::vector<int32_t> st(m), bad(m);
    for (uint32_t k = 0; k < m; k++) {
      const uint32_t i = idx[k];
      sp[k] = src[i];
      sl[k] = src_len[i];
      dp[k] = dst[i];
      dc[k] = dst_cap[i];
      if (checksum_alg) {
        ns[k] = n_slices[i];
        slp[k] = slice_len[i];
        scp[k] = slice_checksum[i];
      }
    }
    if (checksum_alg) flatten_slices(m, ns.data(), slp.data(), scp.data(), b, l, c);
    int rc = decompress_host(codec, checksum_alg, m, sp.data(), sl.data(), b.data(), l.data(), c.data(), nullptr, 0,
                             dp.data(), dc.data(), nullptr, dl.data(), nullptr, st.data(), bad.data(), false);
    if (!rc)
      for (uint32_t k = 0; k < m; k++) {
        dst_len[idx[k]] = dl[k];
        status[idx[k]] = st[k];
        if (bad_slice) bad_slice[idx[k]] = bad[k];
      }
    return rc;
  });
}

int b2s_decompress_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                          const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                          const uint64_t* slice_len, const uint64_t* slice_checksum, uint8_t* dst_base,
                          uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                          int32_t* status, int32_t* bad_slice) {
  if (n && (!src_base || !src_off || !src_len || !dst_base || !dst_off || !dst_len || !status))
    return fail(B2S_E_ARG, "null argument%s");
  if (checksum_alg && n && (!slice_base || !slice_len || !slice_checksum))
    return fail(B2S_E_ARG, "slice arrays required%s");
  std::vector<const uint8_t*> ptr(n);
  for (uint32_t i = 0; i < n; i++) ptr[i] = src_base + src_off[i];
  return decompress_host(codec, checksum_alg, n, ptr.data(), src_len, slice_base, slice_len, slice_checksum, dst_base,
                         dst_cap, nullptr, nullptr, dst_off, dst_len, dst_total, status, bad_slice, false);
}

// ------------------------------------------------------------------------------------------------------------
// read side, key-sorted: verify + decode a reduce task's blocks, then sort its records by key
// ------------------------------------------------------------------------------------------------------------
// What the records of a sort call are: fixed-size (record_bytes long, an unsigned byte key) or length-prefixed UnsafeRow
// records (rows: [size: int32 big-endian][row], key columns in the row, each with its null bit).  aggregate: rows
// grouped by the key and merged (b2s_decompress_aggregate_rows_*: the caller's n_aggs aggregates), not sorted.
struct JoinSpec;
struct WindowSpec;
struct RecordSpec {
  bool is_rows = false;
  uint32_t record_bytes = 0;
  KeySpec keys;             // rows: the key columns; fixed-size records: one B2S_KEY_BYTES column
  uint32_t n_keys = 1;      // as the caller passed it; keys holds the columns when it is in [1, 16]
  bool key_arrays = true;   // the caller's key arrays are not NULL
  bool composite = false;   // the *_keys calls: string, decimal, 16 / 8-bit and float columns and order flags accepted
  bool null_safe = false;   // the join and hash calls: B2S_KEY_NULL_SAFE accepted too
  bool aggregate = false;
  uint32_t n_aggs = 0;
  const uint32_t* agg_op = nullptr;
  const uint32_t* agg_off = nullptr;
  const int32_t* agg_null_field = nullptr;
  const JoinSpec* join = nullptr;  // a join: keys are the left side's columns
  const WindowSpec* window = nullptr;  // a window: keys are the partition columns, then the order columns
  bool rows() const { return is_rows; }
  Family family() const {
    return join ? Family::kJoin : window ? Family::kWindow : aggregate ? Family::kAggregate
           : is_rows ? Family::kSortRows : Family::kSort;
  }
};
// A join's other arguments (b2s_decompress_join_rows_keys_*): its type, the left blocks, the right side's key columns,
// both sides' field counts and kinds, and the per-side record counts it returns.  Side 0 is the left.
struct JoinSpec {
  uint32_t type = 0;
  uint32_t n_left = 0;
  KeySpec right;
  bool right_arrays = true;  // the right side's key arrays are not NULL
  uint32_t n_fields[2] = {};
  const uint8_t* kind[2] = {};
  uint64_t* n_side[2] = {};
};
// A window's other arguments (b2s_decompress_window_rows_keys_*): how many key columns partition, the input's fields
// and kinds, the functions and their arguments, the limit, and the input record count it returns.  The aggregate call
// (b2s_decompress_window_aggregate_rows_keys_*, agg) adds each function's frame and input column, and has no limit; the
// offset call (b2s_decompress_window_offset_rows_keys_*, agg and offset) adds each function's flags and default.
struct WindowSpec {
  uint32_t n_partition_keys = 0;
  uint32_t n_fields = 0;
  const uint8_t* kind = nullptr;
  uint32_t n_fns = 0;
  const uint32_t* fn = nullptr;
  const int32_t* fn_arg = nullptr;
  uint32_t limit_fn = B2S_WINDOW_NO_LIMIT;
  int32_t limit = 0;
  uint64_t* n_in = nullptr;
  bool agg = false;
  const uint32_t* frame = nullptr;
  const uint32_t* val_type = nullptr;
  const uint32_t* val_off = nullptr;
  const int32_t* val_null = nullptr;
  bool offset = false;
  const uint32_t* flags = nullptr;
  const uint64_t* dflt = nullptr;
  bool frames = false;  // the frame call (b2s_decompress_window_frame_rows_keys_*, agg and offset): sliding bounds
  const int64_t* lower = nullptr;
  const int64_t* upper = nullptr;
};
static RecordSpec fixed_spec(uint32_t record_bytes, uint32_t key_off, uint32_t key_len) {
  RecordSpec r;
  r.record_bytes = record_bytes;
  r.keys.n = 1;
  r.keys.off[0] = key_off;
  r.keys.len[0] = key_len;
  r.keys.null_field[0] = -1;
  return r;
}
static RecordSpec rows_spec(uint32_t key_type, uint32_t key_off, uint32_t key_len, int32_t null_field) {
  RecordSpec r = fixed_spec(0, key_off, key_len);
  r.is_rows = true;
  r.keys.type[0] = key_type;
  r.keys.null_field[0] = null_field;
  return r;
}
// the *_keys calls: n_keys parallel columns; checked by sort_args, after the device
static RecordSpec keys_spec(uint32_t n_keys, const uint32_t* type, const uint32_t* off, const uint32_t* len,
                            const int32_t* null_field) {
  RecordSpec r;
  r.is_rows = true;
  r.composite = true;
  r.n_keys = n_keys;
  r.key_arrays = type && off && len && null_field;
  if (r.key_arrays && n_keys >= 1 && n_keys <= kMaxKeys) {
    r.keys.n = n_keys;
    for (uint32_t c = 0; c < n_keys; c++) {
      r.keys.type[c] = type[c];
      r.keys.off[c] = off[c];
      r.keys.len[c] = len[c];
      r.keys.null_field[c] = null_field[c];
    }
  }
  return r;
}

static bool overlaps(uint64_t a0, uint64_t a1, uint64_t b0, uint64_t b1) { return a0 < b1 && b0 < a1; }
// the bytes an aggregate's slots take from agg_off: a variance entry's three doubles, every other op's one slot
static uint64_t agg_width(uint32_t op) { return agg_base_op(op) == B2S_AGG_VARIANCE ? 24 : 8; }
// the row offset of field f's 8-byte null word
static uint64_t null_word(int32_t f) { return 8ull * (uint32_t)(f >> 6); }

static RecordSpec with_aggregates(RecordSpec r, uint32_t n_aggs, const uint32_t* op, const uint32_t* off,
                                  const int32_t* agg_null) {
  r.aggregate = true;
  r.n_aggs = n_aggs;
  r.agg_op = op;
  r.agg_off = off;
  r.agg_null_field = agg_null;
  return r;
}
static RecordSpec aggregate_spec(uint32_t key_type, uint32_t key_off, uint32_t key_len, int32_t null_field,
                                 uint32_t n_aggs, const uint32_t* op, const uint32_t* off, const int32_t* agg_null) {
  return with_aggregates(rows_spec(key_type, key_off, key_len, null_field), n_aggs, op, off, agg_null);
}

// each aggregate is a known op on 8 bytes (a variance entry: 24) that touch no other slot, a key column, or a null word
// in use
static int agg_args(const RecordSpec& spec) {
  const uint32_t n = spec.n_aggs;
  const KeySpec& ks = spec.keys;
  if (n > kMaxAggs) return fail(B2S_E_ARG, "n_aggs must be at most 16%s");
  if (n && (!spec.agg_op || !spec.agg_off || !spec.agg_null_field)) return fail(B2S_E_ARG, "null argument%s");
  std::vector<std::pair<uint64_t, uint64_t>> words;  // the null words the key and the aggregates use
  for (uint32_t c = 0; c < ks.n; c++)
    if (ks.null_field[c] >= 0) words.push_back({null_word(ks.null_field[c]), null_word(ks.null_field[c]) + 8});
  for (uint32_t k = 0; k < n; k++) {
    const uint32_t op = spec.agg_op[k], base = agg_base_op(op), precision = agg_precision(op);
    if ((op >> 16) || (base > B2S_AGG_MAX_FLOAT64 && base < B2S_AGG_SUM_DECIMAL) || base > B2S_AGG_VARIANCE)
      return fail(B2S_E_ARG, "unknown aggregate op%s");
    if (base != B2S_AGG_SUM_DECIMAL && precision)
      return fail(B2S_E_ARG, "only B2S_AGG_SUM_DECIMAL takes a precision%s");
    if (base == B2S_AGG_SUM_DECIMAL && (precision < 1 || precision > 38))
      return fail(B2S_E_ARG, "B2S_AGG_SUM_DECIMAL's precision must be in [1, 38]%s");
    const int32_t f = spec.agg_null_field[k];
    if (f < -1) return fail(B2S_E_ARG, "agg_null_field must be -1 or a field ordinal%s");
    if (base == B2S_AGG_SUM_DECIMAL && f < 0)
      return fail(B2S_E_ARG, "B2S_AGG_SUM_DECIMAL needs an agg_null_field: its result can be null%s");
    if (base == B2S_AGG_VARIANCE && f >= 0)
      return fail(B2S_E_ARG, "B2S_AGG_VARIANCE takes agg_null_field -1: its buffers are never null%s");
    if (f >= 0) words.push_back({null_word(f), null_word(f) + 8});
  }
  for (uint32_t k = 0; k < n; k++) {
    const uint64_t s0 = spec.agg_off[k], s1 = s0 + agg_width(spec.agg_op[k]);
    for (uint32_t c = 0; c < ks.n; c++)
      if (overlaps(s0, s1, ks.off[c], (uint64_t)ks.off[c] + ks.len[c]))
        return fail(B2S_E_ARG, "an aggregate slot overlaps the key%s");
    for (uint32_t m = 0; m < k; m++)
      if (overlaps(s0, s1, spec.agg_off[m], (uint64_t)spec.agg_off[m] + agg_width(spec.agg_op[m])))
        return fail(B2S_E_ARG, "aggregate slots overlap%s");
    for (const auto& w : words)
      if (overlaps(s0, s1, w.first, w.second)) return fail(B2S_E_ARG, "an aggregate slot overlaps a null word%s");
  }
  return 0;
}

// The device form of the aggregates: ops, slots and null bits; the index of every out-of-line decimal among them; where
// their 16-byte regions may start (past every key and aggregate slot and every null word the call uses); the index of
// every variance entry among them.
static AggSpec agg_spec(const RecordSpec& spec) {
  AggSpec agg;
  agg.n = spec.n_aggs;
  uint64_t from = 0;
  const KeySpec& ks = spec.keys;
  for (uint32_t c = 0; c < ks.n; c++) {
    from = std::max<uint64_t>(from, (uint64_t)ks.off[c] + ks.len[c]);
    if (ks.null_field[c] >= 0) from = std::max<uint64_t>(from, null_word(ks.null_field[c]) + 8);
  }
  for (uint32_t k = 0; k < agg.n; k++) {
    const uint32_t op = spec.agg_op[k];
    agg.op[k] = op;
    agg.off[k] = spec.agg_off[k];
    agg.null_field[k] = spec.agg_null_field[k];
    if (agg_decimal_wide(op)) agg.wide[k] = agg.n_wide++;
    if (op == B2S_AGG_VARIANCE) agg.var[k] = agg.n_var++;
    agg.decimal |= agg_decimal_op(op);
    from = std::max<uint64_t>(from, (uint64_t)spec.agg_off[k] + agg_width(op));
    if (spec.agg_null_field[k] >= 0) from = std::max<uint64_t>(from, null_word(spec.agg_null_field[k]) + 8);
  }
  agg.region_from = (uint32_t)std::min<uint64_t>(from, 0xffffffffull);
  return agg;
}

// the bytes a row must hold for the aggregates: every slot and every aggregate null word (0 without aggregates)
static uint64_t agg_min_row(const RecordSpec& spec) {
  uint64_t m = 0;
  for (uint32_t k = 0; k < spec.n_aggs; k++) {
    m = std::max<uint64_t>(m, (uint64_t)spec.agg_off[k] + agg_width(spec.agg_op[k]));
    if (spec.agg_null_field[k] >= 0) m = std::max<uint64_t>(m, null_word(spec.agg_null_field[k]) + 8);
  }
  return m;
}

// the key columns of rows: n_keys, the arrays, and each column's type, flags, key_len and null field
static int key_columns_args(const RecordSpec& spec) {
  const KeySpec& ks = spec.keys;
  if (spec.n_keys < 1 || spec.n_keys > kMaxKeys) return fail(B2S_E_ARG, "n_keys must be in [1, 16]%s");
  if (!spec.key_arrays) return fail(B2S_E_ARG, "null argument%s");
  for (uint32_t c = 0; c < ks.n; c++) {
    const uint32_t type = ks.type[c] & kKeyTypeMask, flags = ks.type[c] & ~kKeyTypeMask, key_len = ks.len[c];
    const bool composite_type = type == kStringKey || (type >= B2S_KEY_INT16 && type <= kDecimalKey);
    if (type > B2S_KEY_INT64 && !(spec.composite && composite_type)) return fail(B2S_E_ARG, "unknown key_type%s");
    const uint32_t known = B2S_KEY_DESCENDING | B2S_KEY_NULLS_LAST | (spec.null_safe ? B2S_KEY_NULL_SAFE : 0);
    if (flags && (!spec.composite || (flags & ~known))) return fail(B2S_E_ARG, "unknown key_type flag%s");
    if (type == B2S_KEY_BYTES && (key_len < 1 || key_len > 16))
      return fail(B2S_E_ARG, "key_len must be in [1, 16]%s");
    // the fixed key_len of every other type: the value's bytes, or a string's or decimal's 8-byte slot
    static const uint32_t fixed_len[] = {0, 4, 8, 8, 0, 2, 1, 4, 8, 8};
    if (type != B2S_KEY_BYTES && key_len != fixed_len[type])
      return fail(B2S_E_ARG, "key_len does not match the key_type (INT8 1, INT16 2, INT32 / FLOAT32 4, else 8)%s");
    if (ks.null_field[c] < -1) return fail(B2S_E_ARG, "null_field must be -1 or a field ordinal%s");
  }
  return 0;
}

// the null-bitset words of n fields
static uint32_t bitset_words(uint32_t n) { return (n + 63) / 64; }

// a join's checks past the composite key's (the left columns): its type and blocks, the right columns, no order flag,
// each side's fields, and every key slot and null bit inside its side's fixed region
static int join_args(const RecordSpec& spec, uint32_t n) {
  const JoinSpec& js = *spec.join;
  if ((js.type > B2S_JOIN_FULL_OUTER && js.type != B2S_JOIN_EXISTENCE) || js.type == B2S_JOIN_LEFT_ANTI + 1)
    return fail(B2S_E_ARG, "unknown join_type%s");  // 4 and 7 are not assigned
  if (js.n_left > n) return fail(B2S_E_ARG, "n_left must be at most n%s");
  RecordSpec right = spec;
  right.keys = js.right;
  right.key_arrays = js.right_arrays;
  if (int rc = key_columns_args(right)) return rc;
  const KeySpec* side[2] = {&spec.keys, &js.right};
  const bool kinds = !join_keeps_whole(js.type);
  for (uint32_t s = 0; s < 2; s++) {
    const uint32_t nf = js.n_fields[s];
    if (nf < 1 || nf > 65536) return fail(B2S_E_ARG, "a side's field count must be in [1, 65536]%s");
    const uint64_t lo = 8ull * bitset_words(nf), hi = lo + 8ull * nf;
    for (uint32_t c = 0; c < side[s]->n; c++) {
      if (side[s]->type[c] & ~kKeyTypeMask & ~B2S_KEY_NULL_SAFE)
        return fail(B2S_E_ARG, "a join key column takes no order flag%s");
      if (side[s]->off[c] < lo || (uint64_t)side[s]->off[c] + side[s]->len[c] > hi)
        return fail(B2S_E_ARG, "a key slot lies outside its side's field slots%s");
      if (side[s]->null_field[c] >= (int64_t)nf)
        return fail(B2S_E_ARG, "a key null bit is not below its side's field count%s");
    }
    if (kinds && (s == 0 || js.type != B2S_JOIN_EXISTENCE)) {  // an existence join's row holds no right field
      if (!js.kind[s]) return fail(B2S_E_ARG, "field kinds are required for joins that build joined rows%s");
      for (uint32_t f = 0; f < nf; f++)
        if (js.kind[s][f] > B2S_FIELD_DECIMAL_WIDE) return fail(B2S_E_ARG, "unknown field kind%s");
    }
  }
  for (uint32_t s = 0; s < 2; s++)
    if (!js.n_side[s]) return fail(B2S_E_ARG, "null argument%s");
  return 0;
}

// a window's checks past the composite key's: the partition columns (no flag, at least one order column after them),
// the input's fields and every key slot and null bit inside them, the functions and the limit
static int window_args(const RecordSpec& spec) {
  const WindowSpec& ws = *spec.window;
  const KeySpec& ks = spec.keys;
  // the aggregate call has checked its functions (window_agg_fn_args); with every frame the whole partition it needs
  // no ORDER BY column
  bool whole = ws.agg;
  for (uint32_t j = 0; whole && j < ws.n_fns; j++) whole = ws.frame[j] == B2S_WINDOW_FRAME_PARTITION;
  if (whole ? ws.n_partition_keys > spec.n_keys
            : ws.n_partition_keys >= spec.n_keys || ws.n_partition_keys >= kMaxKeys)
    return fail(B2S_E_ARG, "n_partition_keys must be in [0, 15] and leave at least one ORDER BY column%s");
  for (uint32_t c = 0; c < ws.n_partition_keys; c++)
    if (ks.type[c] & ~kKeyTypeMask) return fail(B2S_E_ARG, "a partition column takes no order flag%s");
  const uint32_t nf = ws.n_fields;
  if (nf < 1 || nf > 65536) return fail(B2S_E_ARG, "n_fields must be in [1, 65536]%s");
  const uint64_t lo = 8ull * bitset_words(nf), hi = lo + 8ull * nf;
  for (uint32_t c = 0; c < ks.n; c++) {
    if (ks.off[c] < lo || (uint64_t)ks.off[c] + ks.len[c] > hi)
      return fail(B2S_E_ARG, "a key slot lies outside the input's field slots%s");
    if (ks.null_field[c] >= (int64_t)nf) return fail(B2S_E_ARG, "a key null bit is not below n_fields%s");
  }
  if (!ws.kind) return fail(B2S_E_ARG, "field kinds are required%s");
  for (uint32_t f = 0; f < nf; f++)
    if (ws.kind[f] > B2S_FIELD_DECIMAL_WIDE) return fail(B2S_E_ARG, "unknown field kind%s");
  if (ws.n_fns < 1 || ws.n_fns > kMaxWindowFns) return fail(B2S_E_ARG, "n_fns must be in [1, 16]%s");
  if (!ws.fn || !ws.fn_arg || !ws.n_in) return fail(B2S_E_ARG, "null argument%s");
  if (ws.agg) return 0;
  const bool limited = ws.limit_fn != B2S_WINDOW_NO_LIMIT;
  auto rank_like = [](uint32_t f) { return f <= B2S_WINDOW_DENSE_RANK; };
  for (uint32_t j = 0; j < ws.n_fns; j++) {
    if (ws.fn[j] > B2S_WINDOW_NTILE) return fail(B2S_E_ARG, "unknown window function%s");
    if (ws.fn[j] == B2S_WINDOW_NTILE ? ws.fn_arg[j] < 1 : ws.fn_arg[j] != 0)
      return fail(B2S_E_ARG, "fn_arg must be NTILE's bucket count (at least 1), and 0 for every other function%s");
    if (limited && !rank_like(ws.fn[j]))
      return fail(B2S_E_ARG, "with a limit every function must be ROW_NUMBER, RANK or DENSE_RANK%s");
  }
  if (limited ? !rank_like(ws.limit_fn) || ws.limit < 1 : ws.limit != 0)
    return fail(B2S_E_ARG, "limit_fn must be B2S_WINDOW_NO_LIMIT with limit 0, or ROW_NUMBER, RANK or DENSE_RANK with "
                           "a limit of at least 1%s");
  return 0;
}

// The aggregate window call's checks of its functions, before the device: the input's fields and kinds, and per
// function its argument, frame, input type, slot and null bit (b2s_decompress_window_aggregate_rows_keys_*).  With
// ws.offset (the offset call) the offset functions and VAL_BYTES are accepted too.
static int window_agg_fn_args(const WindowSpec& ws) {
  const uint32_t nf = ws.n_fields;
  if (nf < 1 || nf > 65536) return fail(B2S_E_ARG, "n_fields must be in [1, 65536]%s");
  if (!ws.kind) return fail(B2S_E_ARG, "field kinds are required%s");
  for (uint32_t f = 0; f < nf; f++)
    if (ws.kind[f] > B2S_FIELD_DECIMAL_WIDE) return fail(B2S_E_ARG, "unknown field kind%s");
  if (ws.n_fns < 1 || ws.n_fns > kMaxWindowFns) return fail(B2S_E_ARG, "n_fns must be in [1, 16]%s");
  if (!ws.fn || !ws.fn_arg || !ws.frame || !ws.val_type || !ws.val_off || !ws.val_null || !ws.n_in)
    return fail(B2S_E_ARG, "null argument%s");
  const uint64_t lo = 8ull * bitset_words(nf);
  for (uint32_t j = 0; j < ws.n_fns; j++) {
    const uint32_t fn = ws.fn[j], frame = ws.frame[j], vt = ws.val_type[j], kind = vt & 0xff;
    if (fn > (ws.offset ? B2S_WINDOW_NTH_VALUE : B2S_WINDOW_AVG)) return fail(B2S_E_ARG, "unknown window function%s");
    const bool offset = fn >= B2S_WINDOW_LAG, lag_lead = fn == B2S_WINDOW_LAG || fn == B2S_WINDOW_LEAD;
    const bool counted = fn == B2S_WINDOW_NTILE || lag_lead || fn == B2S_WINDOW_NTH_VALUE;
    if (counted ? ws.fn_arg[j] < 1 : ws.fn_arg[j] != 0)
      return fail(B2S_E_ARG, ws.offset ? "fn_arg must be NTILE's bucket count, LAG / LEAD's offset or NTH_VALUE's n "
                                         "(at least 1), and 0 for every other function%s"
                                       : "fn_arg must be NTILE's bucket count (at least 1), and 0 for every other "
                                         "function%s");
    const bool ranking = fn <= B2S_WINDOW_NTILE;
    const uint32_t max_frame = ws.frames ? B2S_WINDOW_FRAME_RANGE : B2S_WINDOW_FRAME_RANGE_RUNNING;
    if (ranking || lag_lead ? frame != 0 : frame < B2S_WINDOW_FRAME_PARTITION || frame > max_frame)
      return fail(B2S_E_ARG, ws.offset ? "fn_frame must be 0 for a ranking function, LAG and LEAD, and a "
                                         "B2S_WINDOW_FRAME_* for an aggregate, FIRST, LAST and NTH_VALUE%s"
                                       : "fn_frame must be 0 for a ranking function and a B2S_WINDOW_FRAME_* for an "
                                         "aggregate%s");
    const uint32_t max_kind = ws.offset ? B2S_WINDOW_VAL_BYTES : B2S_WINDOW_VAL_DECIMAL;
    if (kind > max_kind || (kind != B2S_WINDOW_VAL_DECIMAL && (vt >> 8)) || (vt >> 24))
      return fail(B2S_E_ARG, "unknown val_type%s");
    if (kind == B2S_WINDOW_VAL_BYTES && !offset)
      return fail(B2S_E_ARG, "only an offset function takes B2S_WINDOW_VAL_BYTES%s");
    if (kind == B2S_WINDOW_VAL_NONE) {
      if (fn != B2S_WINDOW_COUNT && !ranking) return fail(B2S_E_ARG, "only COUNT takes B2S_WINDOW_VAL_NONE%s");
      continue;
    }
    if (ranking) return fail(B2S_E_ARG, "a ranking function takes B2S_WINDOW_VAL_NONE%s");
    const uint32_t p = (vt >> 8) & 0xff, sc = vt >> 16;
    if (kind == B2S_WINDOW_VAL_DECIMAL) {
      const uint32_t max_p = fn == B2S_WINDOW_SUM ? 28 : fn == B2S_WINDOW_AVG ? 24 : 38;  // offset functions: 38
      if (p < 1 || p > max_p || sc > p)
        return fail(B2S_E_ARG, "a decimal input needs 1 <= p <= 38 (SUM 28, AVG 24) and s <= p%s");
    }
    const uint32_t off = ws.val_off[j];
    if (off < lo || (off - lo) % 8 || (off - lo) / 8 >= nf)
      return fail(B2S_E_ARG, "val_off is not one of the input's field slots%s");
    const uint8_t want = kind == B2S_WINDOW_VAL_BYTES                   ? B2S_FIELD_VAR
                         : kind == B2S_WINDOW_VAL_DECIMAL && p > 18 ? B2S_FIELD_DECIMAL_WIDE
                                                                    : B2S_FIELD_FIXED;
    if (ws.kind[(off - lo) / 8] != want)
      return fail(B2S_E_ARG, ws.offset ? "a value field's kind must be VAR for VAL_BYTES, DECIMAL_WIDE for a decimal "
                                         "above p 18, else FIXED%s"
                                       : "a value field's kind must be DECIMAL_WIDE for a decimal above p 18, else "
                                         "FIXED%s");
    if (ws.val_null[j] < -1 || ws.val_null[j] >= (int64_t)nf)
      return fail(B2S_E_ARG, "val_null_field must be -1 or a field ordinal below n_fields%s");
  }
  return 0;
}

// The offset window call's checks of its functions, before the device (b2s_decompress_window_offset_rows_keys_*): the
// aggregate call's, with offset functions and VAL_BYTES, then each function's flags and default
static int window_offset_fn_args(const WindowSpec& ws) {
  if (int rc = window_agg_fn_args(ws)) return rc;
  if (!ws.flags || !ws.dflt) return fail(B2S_E_ARG, "null argument%s");
  for (uint32_t j = 0; j < ws.n_fns; j++) {
    const uint32_t fn = ws.fn[j], fl = ws.flags[j], kind = ws.val_type[j] & 0xff, p = (ws.val_type[j] >> 8) & 0xff;
    if (fl & ~(uint32_t)(B2S_WINDOW_IGNORE_NULLS | B2S_WINDOW_HAS_DEFAULT) || (fl && fn < B2S_WINDOW_LAG))
      return fail(B2S_E_ARG, "fn_flags takes B2S_WINDOW_IGNORE_NULLS and B2S_WINDOW_HAS_DEFAULT, on offset functions "
                             "only%s");
    if (!(fl & B2S_WINDOW_HAS_DEFAULT)) {
      if (ws.dflt[j]) return fail(B2S_E_ARG, "a non-zero fn_default needs B2S_WINDOW_HAS_DEFAULT%s");
      continue;
    }
    if ((fn != B2S_WINDOW_LAG && fn != B2S_WINDOW_LEAD) || kind == B2S_WINDOW_VAL_BYTES ||
        (kind == B2S_WINDOW_VAL_DECIMAL && p > 18))
      return fail(B2S_E_ARG, "B2S_WINDOW_HAS_DEFAULT is for LAG and LEAD of a fixed-width type%s");
    const uint32_t width = kind == B2S_WINDOW_VAL_INT8 ? 1 : kind == B2S_WINDOW_VAL_INT16 ? 2
                           : kind == B2S_WINDOW_VAL_INT32 || kind == B2S_WINDOW_VAL_FLOAT32 ? 4 : 8;
    if (width < 8 && ws.dflt[j] >> (8 * width))
      return fail(B2S_E_ARG, "fn_default has bits above its type's width%s");
  }
  return 0;
}

// The frame window call's checks of its functions, before the device (b2s_decompress_window_frame_rows_keys_*): the
// offset call's, with frames 4 and 5 for the functions that take a frame, then each function's bounds, and a RANGE
// offset's order column (n_keys, key_type: the caller's key; the key itself is checked with the sort's)
static int window_frame_fn_args(const WindowSpec& ws, uint32_t n_keys, const uint32_t* key_type) {
  if (int rc = window_offset_fn_args(ws)) return rc;
  if (!ws.lower || !ws.upper) return fail(B2S_E_ARG, "null argument%s");
  for (uint32_t j = 0; j < ws.n_fns; j++) {
    const int64_t lo = ws.lower[j], hi = ws.upper[j];
    const uint32_t frame = ws.frame[j];
    if (frame != B2S_WINDOW_FRAME_ROWS && frame != B2S_WINDOW_FRAME_RANGE) {
      if (lo || hi) return fail(B2S_E_ARG, "frame_lower and frame_upper must be 0 unless fn_frame is "
                                           "B2S_WINDOW_FRAME_ROWS or B2S_WINDOW_FRAME_RANGE%s");
      continue;
    }
    if (lo == B2S_WINDOW_UNBOUNDED_FOLLOWING || hi == B2S_WINDOW_UNBOUNDED_PRECEDING)
      return fail(B2S_E_ARG, "UNBOUNDED FOLLOWING is an upper bound and UNBOUNDED PRECEDING a lower one%s");
    if (lo > hi) return fail(B2S_E_ARG, "a frame's lower bound must not exceed its upper bound%s");
    if (frame == B2S_WINDOW_FRAME_ROWS)
      for (const int64_t k : {lo, hi})
        if (k != B2S_WINDOW_UNBOUNDED_PRECEDING && k != B2S_WINDOW_UNBOUNDED_FOLLOWING &&
            (k < INT32_MIN || k > INT32_MAX))
          return fail(B2S_E_ARG, "a ROWS frame's offset must fit in an int%s");
    if (frame != B2S_WINDOW_FRAME_RANGE) continue;
    for (const int64_t k : {lo, hi}) {  // an offset: one integral ORDER BY column whose type the offset fits
      if (k == 0 || k == B2S_WINDOW_UNBOUNDED_PRECEDING || k == B2S_WINDOW_UNBOUNDED_FOLLOWING) continue;
      if (n_keys != ws.n_partition_keys + 1 || n_keys > kMaxKeys || !key_type)
        return fail(B2S_E_ARG, "a RANGE frame with an offset needs exactly one ORDER BY column%s");
      const uint32_t ty = key_type[ws.n_partition_keys], base = ty & kKeyTypeMask;
      const int bits = base == B2S_KEY_INT8 ? 8 : base == B2S_KEY_INT16 ? 16 : base == B2S_KEY_INT32 ? 32
                       : base == B2S_KEY_INT64 ? 64 : 0;
      if (!bits)
        return fail(B2S_E_ARG, "a RANGE frame's offset needs a byte, short, int, date or long ORDER BY column%s");
      const int64_t tmax = bits == 64 ? INT64_MAX : (int64_t)((1ull << (bits - 1)) - 1), tmin = -tmax - 1;
      if (k < tmin || k > tmax || ((ty & B2S_KEY_DESCENDING) && k == tmin))
        return fail(B2S_E_ARG, "a RANGE frame's offset must fit its ORDER BY column's type (and not be its minimum "
                               "when descending)%s");
    }
  }
  return 0;
}

static int sort_args(uint32_t codec, uint32_t alg, uint32_t n, const uint64_t* src_off, const uint64_t* src_len,
                     const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                     const RecordSpec& spec, const void* src_base, const void* dst_base, uint64_t dst_cap,
                     const uint64_t* dst_total, const uint64_t* n_records, const int32_t* status) {
  if (alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (codec > B2S_CODEC_ZSTD) return fail(B2S_E_UNSUPPORTED, "codec %s not supported by this build", "");
  const KeySpec& ks = spec.keys;
  if (spec.rows()) {
    if (int rc = key_columns_args(spec)) return rc;
    if (spec.aggregate)
      if (int rc = agg_args(spec)) return rc;
    if (spec.join)
      if (int rc = join_args(spec, n)) return rc;
    if (spec.window)
      if (int rc = window_args(spec)) return rc;
  } else {
    const uint32_t key_len = ks.len[0];
    if (spec.record_bytes == 0) return fail(B2S_E_ARG, "record_bytes must be at least 1%s");
    if (key_len < 1 || key_len > 16) return fail(B2S_E_ARG, "key_len must be in [1, 16]%s");
    if ((uint64_t)ks.off[0] + key_len > spec.record_bytes)
      return fail(B2S_E_ARG, "key_off + key_len exceeds record_bytes%s");
  }
  if (!dst_total || !n_records) return fail(B2S_E_ARG, "null argument%s");
  if (n && (!src_base || !src_off || !src_len || !status)) return fail(B2S_E_ARG, "null argument%s");
  if (dst_cap && !dst_base) return fail(B2S_E_ARG, "null argument%s");
  if (alg && n && (!slice_base || !slice_len || !slice_checksum)) return fail(B2S_E_ARG, "slice arrays required%s");
  if (alg && n) return check_slices(n, src_len, slice_base, slice_len);
  return 0;
}

// without a usable device the sort calls report B2S_E_CUDA (b2s_init has failed for that reason), otherwise as get_device
static int sort_device(uint32_t dev_index, Device** out) {
  if (!g_ctx)
    if (int rc = no_device()) return rc;
  return get_device(dev_index, out);
}

// ------------------------------------------------------------------------------------------------------------
// write side, hash-partitioned rows: Spark's HashPartitioning id of every row, then the partition + compress step
// ------------------------------------------------------------------------------------------------------------
// The composite calls' column rules, then what a hash takes: no order flags, B2S_KEY_BYTES only as a 1-byte boolean.
// With the partition step's own checks first.  Like every rows call's checks, these come before the device, so that
// without a usable device a well-formed call reports B2S_E_CUDA (as the sort calls do) and an ill-formed one B2S_E_ARG.
static int hash_args(const MapCall& c, const MapRows& in, const RecordSpec& spec) {
  if (int rc = partition_args(c, in, nullptr, RowIds::hash(spec.keys))) return rc;
  if (int rc = key_columns_args(spec)) return rc;
  for (uint32_t k = 0; k < spec.keys.n; k++) {
    const uint32_t flags = spec.keys.type[k] & ~kKeyTypeMask;
    if (flags & ~(spec.null_safe ? B2S_KEY_NULL_SAFE : 0))
      return fail(B2S_E_ARG, "a hashed key column takes no order flag%s");
    if ((spec.keys.type[k] & kKeyTypeMask) == B2S_KEY_BYTES && spec.keys.len[k] != 1)
      return fail(B2S_E_ARG, "a hashed B2S_KEY_BYTES column is a boolean: key_len must be 1%s");
  }
  return 0;
}

// the outputs a cached store zeroes before its checks: *dst_total, and *cached (B2S_E_ARG when it is NULL)
static int cached_args(uint64_t* dst_total, int32_t* cached) {
  if (dst_total) *dst_total = 0;
  if (!cached) return fail(B2S_E_ARG, "null argument%s");
  *cached = 0;
  return 0;
}

// the hash call's key columns: null-safe ones allowed
static RecordSpec hash_spec(uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                            const int32_t* key_null_field) {
  RecordSpec spec = keys_spec(n_keys, key_type, key_off, key_len, key_null_field);
  spec.null_safe = true;
  return spec;
}

int b2s_partition_compress_rows_hash_packed(uint32_t codec, int32_t level, uint32_t codec_block_size,
                                            uint32_t checksum_alg, uint32_t num_partitions, uint64_t n_records,
                                            const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
                                            uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
                                            const uint32_t* key_len, const int32_t* key_null_field, uint8_t* dst_base,
                                            uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                                            uint64_t* dst_total, uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{true, 0, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RecordSpec spec = hash_spec(n_keys, key_type, key_off, key_len, key_null_field);
  if (int rc = hash_args(c, in, spec)) return rc;
  return write_lane_run(wt, c, in, nullptr, RowIds::hash(spec.keys), nullptr, partition_family(codec), nullptr,
                        pass_through);
}

int b2s_partition_compress_rows_hash_cached_packed(int32_t shuffle_id, int64_t map_id, uint32_t codec, int32_t level,
                                                   uint32_t codec_block_size, uint32_t checksum_alg,
                                                   uint32_t num_partitions, uint64_t n_records,
                                                   const uint8_t* rec_base, uint64_t rec_bytes,
                                                   const uint32_t* rec_len, uint32_t n_keys, const uint32_t* key_type,
                                                   const uint32_t* key_off, const uint32_t* key_len,
                                                   const int32_t* key_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                                   uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                                   uint64_t* checksum_out, int32_t* status, int32_t* cached) {
  const WallTimer wt = begin_call();
  if (int rc = cached_args(dst_total, cached)) return rc;
  const MapCall c{true, 0, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RecordSpec spec = hash_spec(n_keys, key_type, key_off, key_len, key_null_field);
  if (int rc = hash_args(c, in, spec)) return rc;
  if (int rc = exchange_ready()) return rc;
  const ExStore store{shuffle_id, map_id, cached};
  return write_lane_run(wt, c, in, nullptr, RowIds::hash(spec.keys), &store, partition_family(codec), nullptr,
                        pass_through);
}

int b2s_partition_compress_rows_hash_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                                         uint32_t checksum_alg, uint32_t num_partitions, uint64_t n_records,
                                         const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
                                         uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
                                         const uint32_t* key_len, const int32_t* key_null_field, uint8_t* dst_base,
                                         uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                         uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{false, dev_index, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RecordSpec spec = hash_spec(n_keys, key_type, key_off, key_len, key_null_field);
  if (int rc = hash_args(c, in, spec)) return rc;
  return write_lane_run(wt, c, in, nullptr, RowIds::hash(spec.keys), nullptr, partition_family(codec), nullptr,
                        pass_through);
}

// ------------------------------------------------------------------------------------------------------------
// write side, partial aggregation: a map task's rows grouped by key, Spark's buffers folded, one partial row per key,
// then the hash call's partition + compress step over the partial rows
// ------------------------------------------------------------------------------------------------------------
// The buffers of the n_aggs functions (each function's in Spark's aggBufferAttributes order) as the device folds them,
// checked before the device: the function, its input type, the buffer count, the value slot and null bit.  A variance
// is one buffer (one merge entry) of three partial-row fields.
static int partial_agg_args(uint32_t n_aggs, const uint32_t* fn, const uint32_t* val_type, const uint32_t* val_off,
                            const int32_t* val_null, PartialAggSpec* out) {
  PartialAggSpec& s = *out;
  if (n_aggs > kMaxAggs) return fail(B2S_E_ARG, "n_aggs must be at most 16%s");
  if (n_aggs && (!fn || !val_type || !val_off || !val_null)) return fail(B2S_E_ARG, "null argument%s");
  auto add = [&](uint32_t op, uint32_t stage, uint32_t vt, uint32_t off, int32_t nf, bool to_double) {
    if (s.n_bufs == kMaxAggs) return false;
    const uint32_t k = s.n_bufs++;
    s.op[k] = op;
    s.stage[k] = stage;
    s.to_double[k] = to_double;
    s.vtype[k] = vt;
    s.voff[k] = off;
    s.vnull[k] = nf;
    if (agg_decimal_op(op)) s.wide[k] = s.n_dec++;
    if (op == B2S_AGG_VARIANCE) s.var[k] = s.n_var++;
    s.n_fields += op == B2S_AGG_VARIANCE ? 3 : 1;
    s.dsum |= op == B2S_AGG_SUM_FLOAT64;
    return true;
  };
  for (uint32_t a = 0; a < n_aggs; a++) {
    const uint32_t f = fn[a], vt = val_type[a], kind = vt & 0xff, p = (vt >> 8) & 0xff, sc = vt >> 16;
    if ((f < B2S_WINDOW_SUM || f > B2S_WINDOW_AVG) && f != B2S_WINDOW_VARIANCE)
      return fail(B2S_E_ARG, "unknown aggregate function%s");
    if (kind > B2S_WINDOW_VAL_BYTES || (kind != B2S_WINDOW_VAL_DECIMAL && (vt >> 8)) || (vt >> 24))
      return fail(B2S_E_ARG, "unknown val_type%s");
    if (kind == B2S_WINDOW_VAL_DECIMAL && (p < 1 || p > 38 || sc > p))
      return fail(B2S_E_ARG, "a decimal input needs 1 <= p <= 38 and s <= p%s");
    const bool none = kind == B2S_WINDOW_VAL_NONE, bytes = kind == B2S_WINDOW_VAL_BYTES;
    const bool dec = kind == B2S_WINDOW_VAL_DECIMAL, fp = kind == B2S_WINDOW_VAL_FLOAT32 || kind == B2S_WINDOW_VAL_FLOAT64;
    if ((none || bytes) && f != B2S_WINDOW_COUNT)
      return fail(B2S_E_ARG, "only COUNT takes B2S_WINDOW_VAL_NONE or B2S_WINDOW_VAL_BYTES%s");
    if (!none) {
      if (val_off[a] < 8 || val_off[a] % 8)
        return fail(B2S_E_ARG, "val_off must be a field's 8-byte slot (a multiple of 8, past the null words)%s");
      if (val_null[a] < -1 || val_null[a] >= 65536)
        return fail(B2S_E_ARG, "val_null_field must be -1 or a field ordinal below 65536%s");
    }
    const uint32_t off = none ? 0 : val_off[a];
    const int32_t nf = none ? -1 : val_null[a];
    bool ok = true;
    switch (f) {
      case B2S_WINDOW_SUM:
        if (dec) {
          if (p > 28) return fail(B2S_E_ARG, "a decimal SUM input needs p <= 28 (its buffer is decimal(p + 10))%s");
          ok = add(B2S_AGG_SUM_DECIMAL | (p + 10) << 8, kStageZero, vt, off, nf, false) &&
               add(B2S_AGG_MIN_INT32, kStageIsEmpty, vt, off, nf, false);
        } else {
          ok = add(fp ? B2S_AGG_SUM_FLOAT64 : B2S_AGG_SUM_INT64, kStageValue, vt, off, nf, false);
        }
        break;
      case B2S_WINDOW_COUNT:
        ok = add(B2S_AGG_SUM_INT64, kStageCount, vt, off, nf, false);
        break;
      case B2S_WINDOW_AVG:
        if (dec) {
          if (p > 27) return fail(B2S_E_ARG, "a decimal AVG input needs p <= 27 (Average adds with Add)%s");
          ok = add(B2S_AGG_SUM_DECIMAL | (p + 10) << 8, kStageZero, vt, off, nf, false);
        } else {
          ok = add(B2S_AGG_SUM_FLOAT64, kStageZero, vt, off, nf, true);
        }
        ok = ok && add(B2S_AGG_SUM_INT64, kStageCount, vt, off, nf, false);
        break;
      case B2S_WINDOW_VARIANCE:  // [n, avg, m2] over Cast(child, DoubleType)
        if (dec)
          return fail(B2S_E_ARG, "VARIANCE takes an int8 .. int64, float or double input (a decimal's cast to double "
                                 "is Decimal.toDouble)%s");
        ok = add(B2S_AGG_VARIANCE, kStageValue, vt, off, nf, true);
        break;
      default: {  // MIN, MAX
        const bool mx = f == B2S_WINDOW_MAX;
        uint32_t op;
        if (kind == B2S_WINDOW_VAL_INT32) op = mx ? B2S_AGG_MAX_INT32 : B2S_AGG_MIN_INT32;
        else if (kind == B2S_WINDOW_VAL_INT64 || (dec && p <= 18)) op = mx ? B2S_AGG_MAX_INT64 : B2S_AGG_MIN_INT64;
        else if (kind == B2S_WINDOW_VAL_FLOAT64) op = mx ? B2S_AGG_MAX_FLOAT64 : B2S_AGG_MIN_FLOAT64;
        else if (dec) op = mx ? B2S_AGG_MAX_DECIMAL : B2S_AGG_MIN_DECIMAL;
        else
          return fail(B2S_E_ARG, "MIN and MAX take an int, long, double or decimal input (the reduce side merges no "
                                 "other)%s");
        ok = add(op, kStageValue, vt, off, nf, false);
      }
    }
    if (!ok) return fail(B2S_E_ARG, "more than 16 aggregation buffers (the reduce-side merge's limit)%s");
  }
  return 0;
}

// The key columns as the partial rows hold them: column c is field c (slot 8 + 8 c, one null word), null bit c when the
// input's column is nullable
static KeySpec partial_row_keys(const KeySpec& in) {
  KeySpec k = in;
  for (uint32_t c = 0; c < in.n; c++) {
    k.off[c] = 8 + 8 * c;
    k.null_field[c] = in.null_field[c] >= 0 ? (int32_t)c : -1;
  }
  return k;
}

// The records' offsets (into the sort workspace ws, with key_bytes of key) and their checks (the verdict in paws' header,
// ids n u32 of scratch), one readback: a bad record or a wrong byte total fails the call with the record it names
static int partial_agg_checked(Slot& S, const PartialAggSpec& spec, uint64_t n, const uint8_t* d_rec,
                               uint64_t rec_bytes, const uint32_t* d_len, uint32_t key_bytes, uint8_t* ws,
                               uint8_t* paws, uint32_t* ids, uint64_t* launches) {
  cudaStream_t st = S.st;
  const KeySpec& ks = spec.keys;
  uint64_t* hdr = partial_agg_header(paws);
  uint64_t* rb = (uint64_t*)S.hmeta.p;
  launch_partial_agg_offsets(d_len, n, key_bytes, ws, paws, st, launches);
  launch_partial_agg_check(d_rec, rec_bytes, n, key_bytes, spec, ws, paws, ids, st, launches);
  CU(cudaMemcpyAsync(rb, hdr, 24, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if (rb[0] != ~0ull) {
    if ((rb[0] & 7) != kPaBadValue) return row_ids_verdict(RowIds::hash(ks), rb[0]);
    static const char* const why[] = {"", "its row does not hold a value slot", "its row does not hold a value's null word",
                                      "a decimal value's size is not 1..16 or it runs past its row"};
    char msg[256];
    snprintf(msg, sizeof msg, "record %llu is not a serialized row of the aggregated columns: %s",
             (unsigned long long)(rb[0] >> 3), why[rb[2] & 3]);
    return fail(B2S_E_ARG, "%s", msg);
  }
  if (rb[1] != rec_bytes) {
    char msg[256];
    const KeySortWs w = carve_key_sort_ws(ws, n, key_bytes);
    if (rb[1] > rec_bytes)
      snprintf(msg, sizeof msg, "rec_len sums to %llu bytes, rec_bytes is %llu: record %llu ends past rec_bytes",
               (unsigned long long)rb[1], (unsigned long long)rec_bytes,
               (unsigned long long)first_record_past(w.src_off, w.len, n, rec_bytes));
    else
      snprintf(msg, sizeof msg, "rec_len sums to %llu bytes, rec_bytes is %llu", (unsigned long long)rb[1],
               (unsigned long long)rec_bytes);
    return fail(B2S_E_ARG, "%s", msg);
  }
  return 0;
}

// the aggregation step's workspace in S.fws: the key sort's, the refinement rounds', the grouping's and its own
static size_t partial_agg_fws_bytes(uint64_t n, const PartialAggSpec& spec) {
  const uint32_t key_bytes = rows_key_bytes(spec.keys);
  return rows_sort_ws_bytes(n, key_bytes) + (rows_key_refines(spec.keys) ? rows_refine_ws_bytes(n, 1) : 0) +
         rows_aggregate_ws_bytes(n, 0, 0) + partial_agg_ws_bytes(n, spec);
}

// The key sort of n checked records (ranges: their one range's offset) and, for a key that refines (rws), its rounds,
// one readback each: the sorted record indices *idx and the head flags *heads (nullptr: where the key words differ)
static int sort_checked_rows(Slot& S, const KeySpec& ks, uint64_t n, const uint8_t* d_rec, const uint64_t* ranges,
                             uint8_t* ws, uint8_t* rws, const uint32_t** idx, const uint32_t** heads,
                             uint64_t* launches) {
  cudaStream_t st = S.st;
  uint64_t* rb = (uint64_t*)S.hmeta.p;
  *idx = launch_rows_order(d_rec, n, ks, ranges, 1, ws, rws, st, launches);
  *heads = nullptr;
  if (!rws) return 0;
  // the key columns were checked, so no round finds a bad string or decimal
  for (uint32_t d = kKeyPrefixBytes;; d += kKeyChunkBytes) {
    launch_rows_refine_mark(n, d, rws, 1, st, launches);
    CU(cudaMemcpyAsync(rb, rows_refine_readback(rws, n, 1), 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    const uint64_t tied = rb[0] & 0xffffffffull, runs = rb[0] >> 32;
    if (!tied) break;
    launch_rows_refine_round(d_rec, n, ks, tied, runs, d, ws, rws, 1, st, launches);
  }
  *idx = rows_refine_order(rws, n, 1);
  *heads = rows_refine_heads(rws, n, 1);
  return 0;
}

// The aggregation step on S over n device-resident records (d_rec, rec_bytes; d_len): offsets, checks
// (partial_agg_checked), the key sort and its refinement rounds, the grouping, the folds (one readback: groups,
// partial-row bytes) and the partial rows into S.aggrows, their record lengths at *row_len (in S.fws).  Marks G1, and G0
// unless the caller marked it before a step of its own.
static int partial_agg_rows(Slot& S, const PartialAggSpec& spec, uint64_t n, const uint8_t* d_rec, uint64_t rec_bytes,
                            const uint32_t* d_len, uint64_t* groups, uint64_t* out_bytes, const uint32_t** row_len,
                            uint64_t* launches, bool mark_g0 = true) {
  cudaStream_t st = S.st;
  const KeySpec& ks = spec.keys;
  const uint32_t key_bytes = rows_key_bytes(ks);
  const bool refine = rows_key_refines(ks);
  const size_t part[4] = {rows_sort_ws_bytes(n, key_bytes), refine ? rows_refine_ws_bytes(n, 1) : 0,
                          rows_aggregate_ws_bytes(n, 0, 0), partial_agg_ws_bytes(n, spec)};
  if (int rc = S.fws.ensure(partial_agg_fws_bytes(n, spec))) return rc;
  uint8_t* ws = (uint8_t*)S.fws.p;
  uint8_t *rws = refine ? ws + part[0] : nullptr, *gws = ws + part[0] + part[1], *paws = gws + part[2];
  uint64_t* hdr = partial_agg_header(paws);
  *row_len = partial_agg_row_len(paws, n, spec);
  if (int rc = S.hmeta.ensure(48)) return rc;
  uint64_t* rb = (uint64_t*)S.hmeta.p;
  if (mark_g0) CU(S.mark(G0, st, *launches));
  if (int rc = partial_agg_checked(S, spec, n, d_rec, rec_bytes, d_len, key_bytes, ws, paws,
                                   (uint32_t*)partial_agg_row_len(paws, n, spec), launches))
    return rc;
  *groups = *out_bytes = 0;
  if (!n) {
    CU(S.mark(G1, st, *launches));
    return 0;
  }
  const uint32_t *idx, *heads;
  if (int rc = sort_checked_rows(S, ks, n, d_rec, hdr + 3, ws, rws, &idx, &heads, launches)) return rc;
  launch_rows_group(d_rec, n, idx, heads, key_bytes, AggSpec{}, ws, gws, st, launches);
  launch_partial_agg_fold(d_rec, n, idx, key_bytes, spec, ws, gws, paws, st, launches);
  CU(cudaMemcpyAsync(rb, hdr + 4, 16, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *groups = rb[0];
  *out_bytes = rb[1];
  if (int rc = S.aggrows.ensure(rb[1] + 64)) return rc;
  launch_partial_agg_emit(d_rec, n, rb[0], idx, key_bytes, spec, ws, gws, paws, (uint8_t*)S.aggrows.p, st, launches);
  CU(S.mark(G1, st, *launches));
  return 0;
}

// b2s_aggregate_grouping_sets_partition_compress_rows_hash_*'s grouping sets: n_sets masks of key columns
struct GroupingSets {
  uint32_t n_sets;
  const uint32_t* mask;
};

// The grouping sets' rules, before the device: gid takes the 16th key column; every mask names key columns only, once
// (aggregate_partition_call checks that n_keys + 1 + the buffers' fields stay within one null word's 32)
static int grouping_sets_args(uint32_t n_keys, uint64_t n, const GroupingSets& g) {
  if (n_keys < 1 || n_keys >= kMaxKeys)
    return fail(B2S_E_ARG, "n_keys must be in [1, 15] with grouping sets (gid is the 16th key column)%s");
  if (!g.n_sets || !g.mask) return fail(B2S_E_ARG, "grouping sets need n_sets >= 1 and a set_mask array%s");
  if (n >= ((1ull << 32) + g.n_sets - 1) / g.n_sets)
    return fail(B2S_E_ARG, "n_records * n_sets must be below 2^32 (the projected records)%s");
  std::vector<uint8_t> seen(1u << n_keys);
  for (uint32_t k = 0; k < g.n_sets; k++) {
    const uint32_t m = g.mask[k];
    if (m >> n_keys) return fail(B2S_E_ARG, "a grouping set's mask names a column at or above n_keys%s");
    if (seen[m]++) return fail(B2S_E_ARG, "two grouping sets are equal (Spark adds _gen_grouping_pos for them)%s");
  }
  return 0;
}

// The aggregation over the projected records (rows_expand.cu): key columns c at slot 8 + 8 c with null bit c, gid an
// INT64 at slot 8 + 8 n_keys that is never null, aggregate input i at slot 8 + 8 (n_keys + 1 + i) with null bit
// n_keys + 1 + i when the caller's input has one; and the expansion's own spec
static int grouping_sets_spec(const KeySpec& ks, uint32_t n_aggs, const uint32_t* fn, const uint32_t* val_type,
                              const uint32_t* val_off, const int32_t* val_null, uint32_t n_sets, ExpandSpec* xs,
                              PartialAggSpec* out) {
  const uint32_t nk = ks.n;
  xs->keys = ks;
  xs->n_sets = n_sets;
  uint32_t ty[kMaxKeys], off[kMaxKeys], len[kMaxKeys];
  int32_t nul[kMaxKeys];
  for (uint32_t c = 0; c < nk; c++) {
    ty[c] = ks.type[c];
    off[c] = 8 + 8 * c;
    len[c] = ks.len[c];
    nul[c] = (int32_t)c;
  }
  ty[nk] = B2S_KEY_INT64;
  off[nk] = 8 + 8 * nk;
  len[nk] = 8;
  nul[nk] = -1;
  uint32_t poff[kMaxAggs] = {};
  int32_t pnull[kMaxAggs];
  for (uint32_t a = 0; a < n_aggs; a++) {
    pnull[a] = -1;
    if ((val_type[a] & 0xff) == B2S_WINDOW_VAL_NONE) continue;
    const uint32_t i = xs->n_in++, f = nk + 1 + i;
    xs->vtype[i] = val_type[a];
    xs->voff[i] = val_off[a];
    xs->vnull[i] = val_null[a];
    xs->reads[i] = fn[a] != B2S_WINDOW_COUNT;
    poff[a] = 8 + 8 * f;
    pnull[a] = val_null[a] >= 0 ? (int32_t)f : -1;
  }
  out->keys = keys_spec(nk + 1, ty, off, len, nul).keys;
  return partial_agg_args(n_aggs, fn, val_type, poff, pnull, out);
}

// Expand on S: the caller's n records checked once (partial_agg_checked: a bad record is named by its input index),
// then each projected once per grouping set into S.xrows (rows_expand.cu; one readback: the projected bytes) ->
// *x_rec, *x_bytes, *x_len, the aggregation step's records.  S.fws is sized once for this and for the aggregation step
// over the projected records (xagg).  After G0, which the caller marks.
static int expand_rows(Slot& S, const PartialAggSpec& spec, const PartialAggSpec& xagg, const ExpandSpec& xs,
                       const uint32_t* set_mask, uint64_t n, const uint8_t* d_rec, uint64_t rec_bytes,
                       const uint32_t* d_len, const uint8_t** x_rec, uint64_t* x_bytes, const uint32_t** x_len,
                       uint64_t* launches) {
  cudaStream_t st = S.st;
  const uint32_t key_bytes = rows_key_bytes(spec.keys);
  const size_t part[3] = {rows_sort_ws_bytes(n, key_bytes), 256 + align_up(n * 4, 256), expand_ws_bytes(n, xs.n_sets)};
  if (int rc = S.fws.ensure(std::max(part[0] + part[1] + part[2], partial_agg_fws_bytes(n * xs.n_sets, xagg))))
    return rc;
  if (int rc = S.hmeta.ensure(48)) return rc;
  uint8_t* ws = (uint8_t*)S.fws.p;
  uint8_t *paws = ws + part[0], *xws = paws + part[1];
  uint64_t* rb = (uint64_t*)S.hmeta.p;
  if (int rc = partial_agg_checked(S, spec, n, d_rec, rec_bytes, d_len, key_bytes, ws, paws, (uint32_t*)(paws + 256),
                                   launches))
    return rc;
  const uint64_t* rec_off = carve_key_sort_ws(ws, n, key_bytes).src_off;
  CU(cudaMemcpyAsync(expand_masks(xws, n, xs.n_sets), set_mask, (size_t)xs.n_sets * 4, cudaMemcpyHostToDevice, st));
  launch_expand_size(d_rec, rec_off, n, xs, xws, st, launches);
  CU(cudaMemcpyAsync(rb, expand_header(xws), 16, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if (rb[1] != ~0ull) {
    char msg[256];
    snprintf(msg, sizeof msg, "record %llu: its row projected for a grouping set passes UnsafeRow's 2^31 - 1 bytes",
             (unsigned long long)rb[1]);
    return fail(B2S_E_UNSUPPORTED, "%s", msg);
  }
  const uint64_t N = n * xs.n_sets, len_sz = align_up(N * 4, 256);
  *x_bytes = rb[0];
  if (int rc = S.xrows.ensure(len_sz + rb[0] + 64)) return rc;
  *x_len = (const uint32_t*)S.xrows.p;
  *x_rec = (const uint8_t*)S.xrows.p + len_sz;
  launch_expand_write(d_rec, rec_off, n, xs, xws, (uint32_t*)S.xrows.p, (uint8_t*)S.xrows.p + len_sz, st, launches);
  return 0;
}

// b2s_aggregate_partition_compress_rows_hash_* (gs null) and b2s_aggregate_grouping_sets_partition_compress_rows_hash_*:
// the checks before the device, then on the write lane (with grouping sets, the expansion first) the aggregation step
// and the partition + compress step over the partial rows
static int aggregate_partition_call(bool packed, uint32_t dev_index, uint32_t codec, int32_t level,
                                    uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
                                    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes,
                                    const uint32_t* rec_len, uint32_t n_keys, const uint32_t* key_type,
                                    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
                                    uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type,
                                    const uint32_t* val_off, const int32_t* val_null_field, uint8_t* dst_base,
                                    uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                    uint64_t* checksum_out, int32_t* status, uint64_t* n_groups,
                                    const GroupingSets* gs = nullptr) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  if (n_groups) *n_groups = 0;
  const MapCall c{packed, dev_index, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RecordSpec rspec = keys_spec(n_keys, key_type, key_off, key_len, key_null_field);
  PartialAggSpec spec;
  spec.keys = rspec.keys;
  if (!n_groups) return fail(B2S_E_ARG, "null argument%s");
  if (int rc = partial_agg_args(n_aggs, agg_fn, val_type, val_off, val_null_field, &spec)) return rc;
  if (spec.keys.n + (gs ? 1 : 0) + spec.n_fields > 32)
    return fail(B2S_E_ARG, gs ? "n_keys + 1 + the buffers' fields (3 per VARIANCE) must be at most 32 (one null word)%s"
                              : "n_keys + the buffers' fields (3 per VARIANCE) must be at most 32 (one null word)%s");
  if (gs)
    if (int rc = grouping_sets_args(n_keys, n_records, *gs)) return rc;
  if (int rc = hash_args(c, in, rspec)) return rc;
  PartialAggSpec xagg;  // with grouping sets, the aggregation over the projected records
  ExpandSpec xs;
  if (gs)
    if (int rc = grouping_sets_spec(spec.keys, n_aggs, agg_fn, val_type, val_off, val_null_field, gs->n_sets, &xs,
                                    &xagg))
      return rc;
  const PartialAggSpec& step = gs ? xagg : spec;
  if (!n_records && rec_bytes)
    return fail(B2S_E_ARG, "rec_len sums to 0 bytes, rec_bytes is %s", std::to_string(rec_bytes).c_str());
  auto aggregate = [&](Slot& S, const MapRows& d_in, MapRows* rows, uint64_t* launches) -> int {
    int rc;
    if (gs) {  // the aggregation step over the projected records; its span (G0, G1) takes in the expansion
      const uint8_t* x_rec = nullptr;
      const uint32_t* x_len = nullptr;
      uint64_t x_bytes = 0;
      CU(S.mark(G0, S.st, *launches));
      if ((rc = expand_rows(S, spec, xagg, xs, gs->mask, d_in.n, d_in.rec, d_in.bytes, d_in.len, &x_rec, &x_bytes,
                            &x_len, launches)))
        return rc;
      rc = partial_agg_rows(S, step, d_in.n * gs->n_sets, x_rec, x_bytes, x_len, &rows->n, &rows->bytes, &rows->len,
                            launches, false);
    } else {
      rc = partial_agg_rows(S, spec, d_in.n, d_in.rec, d_in.bytes, d_in.len, &rows->n, &rows->bytes, &rows->len,
                            launches);
    }
    rows->rec = (const uint8_t*)S.aggrows.p;
    return rc;
  };
  return write_lane_run(wt, c, in, nullptr, RowIds::hash(partial_row_keys(step.keys)), nullptr,
                        Family::kPartialAggregate, n_groups, aggregate);
}

int b2s_aggregate_partition_compress_rows_hash_packed(
    uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len, uint32_t n_keys,
    const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
    uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type, const uint32_t* val_off,
    const int32_t* val_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
    uint64_t* dst_total, uint64_t* checksum_out, int32_t* status, uint64_t* n_groups) {
  return aggregate_partition_call(true, 0, codec, level, codec_block_size, checksum_alg, num_partitions, n_records,
                                  rec_base, rec_bytes, rec_len, n_keys, key_type, key_off, key_len, key_null_field,
                                  n_aggs, agg_fn, val_type, val_off, val_null_field, dst_base, dst_cap, dst_off,
                                  dst_len, dst_total, checksum_out, status, n_groups);
}

int b2s_aggregate_partition_compress_rows_hash_dev(
    uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
    uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
    uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
    const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
    uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status, uint64_t* n_groups) {
  return aggregate_partition_call(false, dev_index, codec, level, codec_block_size, checksum_alg, num_partitions,
                                  n_records, rec_base, rec_bytes, rec_len, n_keys, key_type, key_off, key_len,
                                  key_null_field, n_aggs, agg_fn, val_type, val_off, val_null_field, dst_base, dst_cap,
                                  dst_off, dst_len, dst_total, checksum_out, status, n_groups);
}

int b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed(
    uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len, uint32_t n_keys,
    const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
    uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type, const uint32_t* val_off,
    const int32_t* val_null_field, uint32_t n_sets, const uint32_t* set_mask, uint8_t* dst_base, uint64_t dst_cap,
    uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status,
    uint64_t* n_groups) {
  const GroupingSets gs{n_sets, set_mask};
  return aggregate_partition_call(true, 0, codec, level, codec_block_size, checksum_alg, num_partitions, n_records,
                                  rec_base, rec_bytes, rec_len, n_keys, key_type, key_off, key_len, key_null_field,
                                  n_aggs, agg_fn, val_type, val_off, val_null_field, dst_base, dst_cap, dst_off,
                                  dst_len, dst_total, checksum_out, status, n_groups, &gs);
}

int b2s_aggregate_grouping_sets_partition_compress_rows_hash_dev(
    uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
    uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
    uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
    const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, uint32_t n_sets, const uint32_t* set_mask,
    uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
    uint64_t* checksum_out, int32_t* status, uint64_t* n_groups) {
  const GroupingSets gs{n_sets, set_mask};
  return aggregate_partition_call(false, dev_index, codec, level, codec_block_size, checksum_alg, num_partitions,
                                  n_records, rec_base, rec_bytes, rec_len, n_keys, key_type, key_off, key_len,
                                  key_null_field, n_aggs, agg_fn, val_type, val_off, val_null_field, dst_base, dst_cap,
                                  dst_off, dst_len, dst_total, checksum_out, status, n_groups, &gs);
}

// ------------------------------------------------------------------------------------------------------------
// write side, window group limit: a map task's rows sorted by the window key and cut to each partition's first rows
// by WindowGroupLimitExec(Partial)'s rule, then the hash call's partition + compress step over the kept rows
// ------------------------------------------------------------------------------------------------------------
// The limit's own rules, before the device: *n_out, the whole key as a composite key, the partition columns (no order
// flag, at least one order column after them), the limit, and SinglePartition (num_partitions 1) without partition
// columns
static int window_limit_args(const RecordSpec& spec, uint32_t n_partition_keys, uint32_t limit_fn, int32_t limit,
                             uint32_t num_partitions, const uint64_t* n_out) {
  if (!n_out) return fail(B2S_E_ARG, "null argument%s");
  if (int rc = key_columns_args(spec)) return rc;
  if (n_partition_keys >= spec.n_keys || n_partition_keys >= kMaxKeys)
    return fail(B2S_E_ARG, "n_partition_keys must be in [0, 15] and leave at least one ORDER BY column%s");
  for (uint32_t c = 0; c < n_partition_keys; c++)
    if (spec.keys.type[c] & ~kKeyTypeMask) return fail(B2S_E_ARG, "a partition column takes no order flag%s");
  if (limit_fn > B2S_WINDOW_DENSE_RANK || limit < 1)
    return fail(B2S_E_ARG, "limit_fn must be ROW_NUMBER, RANK or DENSE_RANK, with a limit of at least 1%s");
  if (!n_partition_keys && num_partitions != 1)
    return fail(B2S_E_ARG, "without partition columns the exchange is SinglePartition: num_partitions must be 1%s");
  return 0;
}

// The limit step on S over n device-resident records (d_rec, rec_bytes; d_len): offsets and checks (partial_agg_checked,
// every key column by the hash call's record checks), the key sort and its refinement rounds, the peer groups, the
// partitions and limit values (one readback: kept records, their bytes, a partition too large), then the kept records
// gathered in sorted order into S.aggrows: their lengths, then the records -> *kept, *kept_bytes, *kept_len,
// *kept_rec.  Marks G0, G1.
static int window_limit_rows(Slot& S, const KeySpec& ks, const WindowShape& shape, uint64_t n, const uint8_t* d_rec,
                             uint64_t rec_bytes, const uint32_t* d_len, uint64_t* kept, uint64_t* kept_bytes,
                             const uint32_t** kept_len, const uint8_t** kept_rec, uint64_t* launches) {
  cudaStream_t st = S.st;
  PartialAggSpec checks;  // no buffers; the key columns without their order flags, as the hash kernel reads them
  checks.keys = ks;
  for (uint32_t c = 0; c < ks.n; c++) checks.keys.type[c] &= kKeyTypeMask;
  const uint32_t key_bytes = rows_key_bytes(ks);
  const bool refine = rows_key_refines(ks);
  const size_t part[5] = {rows_sort_ws_bytes(n, key_bytes), refine ? rows_refine_ws_bytes(n, 1) : 0,
                          rows_aggregate_ws_bytes(n, 0, 0), partial_agg_ws_bytes(n, checks), window_ws_bytes(n, shape)};
  if (int rc = S.fws.ensure(part[0] + part[1] + part[2] + part[3] + part[4])) return rc;
  uint8_t* ws = (uint8_t*)S.fws.p;
  uint8_t *rws = refine ? ws + part[0] : nullptr, *gws = ws + part[0] + part[1], *paws = gws + part[2];
  uint8_t* wws = paws + part[3];
  if (int rc = S.hmeta.ensure(kWindowReadbackBytes)) return rc;
  uint64_t* rb = (uint64_t*)S.hmeta.p;
  CU(S.mark(G0, st, *launches));
  if (int rc = partial_agg_checked(S, checks, n, d_rec, rec_bytes, d_len, key_bytes, ws, paws,
                                   (uint32_t*)partial_agg_row_len(paws, n, checks), launches))
    return rc;
  *kept = *kept_bytes = 0;
  if (!n) {
    CU(S.mark(G1, st, *launches));
    return 0;
  }
  const uint32_t *idx, *heads;
  if (int rc = sort_checked_rows(S, ks, n, d_rec, partial_agg_header(paws) + 3, ws, rws, &idx, &heads, launches))
    return rc;
  launch_rows_group(d_rec, n, idx, heads, key_bytes, AggSpec{}, ws, gws, st, launches);
  launch_window_limit(d_rec, n, idx, shape, key_bytes, ws, gws, wws, st, launches);
  CU(cudaMemcpyAsync(rb, window_readback(wws, n, shape), kWindowReadbackBytes, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if (rb[3]) return fail(B2S_E_UNSUPPORTED, "a window partition holds more than 2^31 - 1 records%s");
  *kept = rb[0];
  *kept_bytes = rb[1];
  const uint64_t len_sz = align_up(rb[0] * 4, 256);
  if (int rc = S.aggrows.ensure(len_sz + rb[1] + 64)) return rc;
  *kept_len = (const uint32_t*)S.aggrows.p;
  *kept_rec = (const uint8_t*)S.aggrows.p + len_sz;
  launch_window_limit_gather(d_rec, n, idx, rb[0], key_bytes, shape, ws, wws, (uint32_t*)S.aggrows.p,
                             (uint8_t*)S.aggrows.p + len_sz, st, launches);
  CU(S.mark(G1, st, *launches));
  return 0;
}

// b2s_window_limit_partition_compress_rows_hash_*: the checks before the device, then on the write lane the limit step
// and the partition + compress step over the kept rows, hashed by the partition columns (none: SinglePartition)
static int window_limit_partition_call(bool packed, uint32_t dev_index, uint32_t codec, int32_t level,
                                       uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
                                       uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes,
                                       const uint32_t* rec_len, uint32_t n_partition_keys, uint32_t n_keys,
                                       const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                       const int32_t* key_null_field, uint32_t limit_fn, int32_t limit,
                                       uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                                       uint64_t* dst_total, uint64_t* checksum_out, int32_t* status,
                                       uint64_t* n_out_records) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  if (n_out_records) *n_out_records = 0;
  const MapCall c{packed, dev_index, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RecordSpec spec = keys_spec(n_keys, key_type, key_off, key_len, key_null_field);
  if (int rc = window_limit_args(spec, n_partition_keys, limit_fn, limit, num_partitions, n_out_records)) return rc;
  const RecordSpec pspec = keys_spec(n_partition_keys, key_type, key_off, key_len, key_null_field);
  const RowIds ids = n_partition_keys ? RowIds::hash(pspec.keys) : RowIds::single_partition(spec.keys);
  if (int rc = n_partition_keys ? hash_args(c, in, pspec) : partition_args(c, in, nullptr, ids)) return rc;
  if (!n_records && rec_bytes)
    return fail(B2S_E_ARG, "rec_len sums to 0 bytes, rec_bytes is %s", std::to_string(rec_bytes).c_str());
  WindowShape shape{};  // no functions: the limit and the partition columns only
  shape.limit_fn = limit_fn;
  shape.limit = limit;
  shape.part = pspec.keys;
  auto limit_step = [&](Slot& S, const MapRows& d_in, MapRows* rows, uint64_t* launches) {
    return window_limit_rows(S, spec.keys, shape, d_in.n, d_in.rec, d_in.bytes, d_in.len, &rows->n, &rows->bytes,
                             &rows->len, &rows->rec, launches);
  };
  return write_lane_run(wt, c, in, nullptr, ids, nullptr, Family::kPartialAggregate, n_out_records, limit_step);
}

int b2s_window_limit_partition_compress_rows_hash_packed(
    uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t num_partitions,
    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t limit_fn, int32_t limit, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out,
    int32_t* status, uint64_t* n_out_records) {
  return window_limit_partition_call(true, 0, codec, level, codec_block_size, checksum_alg, num_partitions, n_records,
                                     rec_base, rec_bytes, rec_len, n_partition_keys, n_keys, key_type, key_off,
                                     key_len, key_null_field, limit_fn, limit, dst_base, dst_cap, dst_off, dst_len,
                                     dst_total, checksum_out, status, n_out_records);
}

int b2s_window_limit_partition_compress_rows_hash_dev(
    uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
    uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t limit_fn, int32_t limit, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out,
    int32_t* status, uint64_t* n_out_records) {
  return window_limit_partition_call(false, dev_index, codec, level, codec_block_size, checksum_alg, num_partitions,
                                     n_records, rec_base, rec_bytes, rec_len, n_partition_keys, n_keys, key_type,
                                     key_off, key_len, key_null_field, limit_fn, limit, dst_base, dst_cap, dst_off,
                                     dst_len, dst_total, checksum_out, status, n_out_records);
}

// ------------------------------------------------------------------------------------------------------------
// write side, range-partitioned rows: Spark's RangePartitioner id of every row, then the partition + compress step
// ------------------------------------------------------------------------------------------------------------
// The composite calls' column rules (order flags allowed), the partition step's checks with n_bounds + 1 partitions,
// and the bound arrays'; a device is needed only after them, as for the hash call.
static int range_args(const MapCall& c, const MapRows& in, const RecordSpec& spec, const RowIds& ids) {
  if (ids.n_bounds > (1u << 24) - 1) return fail(B2S_E_ARG, "n_bounds must be at most 2^24 - 1%s");
  if (int rc = partition_args(c, in, nullptr, ids)) return rc;
  if (int rc = key_columns_args(spec)) return rc;
  if (ids.n_bounds && (!ids.bound_base || !ids.bound_len)) return fail(B2S_E_ARG, "null argument%s");
  uint64_t sum = 0;
  for (uint32_t j = 0; j < ids.n_bounds; j++) sum += ids.bound_len[j];
  if (sum != ids.bound_bytes) {
    char msg[128];
    snprintf(msg, sizeof msg, "bound_len sums to %llu bytes, bound_bytes is %llu", (unsigned long long)sum,
             (unsigned long long)ids.bound_bytes);
    return fail(B2S_E_ARG, "%s", msg);
  }
  return 0;
}

int b2s_partition_compress_rows_range_packed(uint32_t codec, int32_t level, uint32_t codec_block_size,
                                             uint32_t checksum_alg, uint64_t n_records, const uint8_t* rec_base,
                                             uint64_t rec_bytes, const uint32_t* rec_len, uint32_t n_keys,
                                             const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                             const int32_t* key_null_field, uint32_t n_bounds,
                                             const uint8_t* bound_base, uint64_t bound_bytes,
                                             const uint32_t* bound_len, uint8_t* dst_base, uint64_t dst_cap,
                                             uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                             uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{true, 0, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  n_bounds + 1, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RecordSpec spec = keys_spec(n_keys, key_type, key_off, key_len, key_null_field);
  const RowIds ids = RowIds::range(spec.keys, n_bounds, bound_base, bound_bytes, bound_len);
  if (int rc = range_args(c, in, spec, ids)) return rc;
  return write_lane_run(wt, c, in, nullptr, ids, nullptr, partition_family(codec), nullptr, pass_through);
}

int b2s_partition_compress_rows_range_cached_packed(int32_t shuffle_id, int64_t map_id, uint32_t codec, int32_t level,
                                                    uint32_t codec_block_size, uint32_t checksum_alg,
                                                    uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes,
                                                    const uint32_t* rec_len, uint32_t n_keys,
                                                    const uint32_t* key_type, const uint32_t* key_off,
                                                    const uint32_t* key_len, const int32_t* key_null_field,
                                                    uint32_t n_bounds, const uint8_t* bound_base,
                                                    uint64_t bound_bytes, const uint32_t* bound_len,
                                                    uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                                                    uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out,
                                                    int32_t* status, int32_t* cached) {
  const WallTimer wt = begin_call();
  if (int rc = cached_args(dst_total, cached)) return rc;
  const MapCall c{true, 0, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  n_bounds + 1, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RecordSpec spec = keys_spec(n_keys, key_type, key_off, key_len, key_null_field);
  const RowIds ids = RowIds::range(spec.keys, n_bounds, bound_base, bound_bytes, bound_len);
  if (int rc = range_args(c, in, spec, ids)) return rc;
  if (int rc = exchange_ready()) return rc;
  const ExStore store{shuffle_id, map_id, cached};
  return write_lane_run(wt, c, in, nullptr, ids, &store, partition_family(codec), nullptr, pass_through);
}

int b2s_partition_compress_rows_range_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                                          uint32_t checksum_alg, uint64_t n_records, const uint8_t* rec_base,
                                          uint64_t rec_bytes, const uint32_t* rec_len, uint32_t n_keys,
                                          const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                          const int32_t* key_null_field, uint32_t n_bounds, const uint8_t* bound_base,
                                          uint64_t bound_bytes, const uint32_t* bound_len, uint8_t* dst_base,
                                          uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                          uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{false, dev_index, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  n_bounds + 1, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  const RecordSpec spec = keys_spec(n_keys, key_type, key_off, key_len, key_null_field);
  const RowIds ids = RowIds::range(spec.keys, n_bounds, bound_base, bound_bytes, bound_len);
  if (int rc = range_args(c, in, spec, ids)) return rc;
  return write_lane_run(wt, c, in, nullptr, ids, nullptr, partition_family(codec), nullptr, pass_through);
}

// ------------------------------------------------------------------------------------------------------------
// write side, round-robin-partitioned rows: Spark's repartition(n) order and ids, then the partition + compress step
// ------------------------------------------------------------------------------------------------------------
// The partition step's checks, then the position and sort flag; a device is needed only after them, as for the hash
// call.  start + n past 2^31 - 1 is refused: Spark's Int position would wrap there.
static int round_robin_args(const MapCall& c, const MapRows& in, int32_t start, uint32_t sort) {
  if (int rc = partition_args(c, in, nullptr, RowIds::round_robin(start, sort))) return rc;
  if (start < 0 || (uint32_t)start >= c.R) return fail(B2S_E_ARG, "start_position must be in [0, num_partitions)%s");
  if (sort > 1) return fail(B2S_E_ARG, "sort_rows must be 0 or 1%s");
  if ((uint64_t)start + in.n > 0x7fffffffull)
    return fail(B2S_E_ARG, "start_position + n_records is past 2^31 - 1, where Spark's position wraps%s");
  return 0;
}

int b2s_partition_compress_rows_round_robin_packed(uint32_t codec, int32_t level, uint32_t codec_block_size,
                                                   uint32_t checksum_alg, uint32_t num_partitions,
                                                   int32_t start_position, uint32_t sort_rows, uint64_t n_records,
                                                   const uint8_t* rec_base, uint64_t rec_bytes,
                                                   const uint32_t* rec_len, uint8_t* dst_base, uint64_t dst_cap,
                                                   uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                                   uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{true, 0, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  if (int rc = round_robin_args(c, in, start_position, sort_rows)) return rc;
  return write_lane_run(wt, c, in, nullptr, RowIds::round_robin(start_position, sort_rows), nullptr,
                        partition_family(codec), nullptr, pass_through);
}

int b2s_partition_compress_rows_round_robin_cached_packed(int32_t shuffle_id, int64_t map_id, uint32_t codec,
                                                          int32_t level, uint32_t codec_block_size,
                                                          uint32_t checksum_alg, uint32_t num_partitions,
                                                          int32_t start_position, uint32_t sort_rows,
                                                          uint64_t n_records, const uint8_t* rec_base,
                                                          uint64_t rec_bytes, const uint32_t* rec_len,
                                                          uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                                                          uint64_t* dst_len, uint64_t* dst_total,
                                                          uint64_t* checksum_out, int32_t* status, int32_t* cached) {
  const WallTimer wt = begin_call();
  if (int rc = cached_args(dst_total, cached)) return rc;
  const MapCall c{true, 0, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  if (int rc = round_robin_args(c, in, start_position, sort_rows)) return rc;
  if (int rc = exchange_ready()) return rc;
  const ExStore store{shuffle_id, map_id, cached};
  return write_lane_run(wt, c, in, nullptr, RowIds::round_robin(start_position, sort_rows), &store,
                        partition_family(codec), nullptr, pass_through);
}

int b2s_partition_compress_rows_round_robin_dev(uint32_t dev_index, uint32_t codec, int32_t level,
                                                uint32_t codec_block_size, uint32_t checksum_alg,
                                                uint32_t num_partitions, int32_t start_position, uint32_t sort_rows,
                                                uint64_t n_records, const uint8_t* rec_base, uint64_t rec_bytes,
                                                const uint32_t* rec_len, uint8_t* dst_base, uint64_t dst_cap,
                                                uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                                                uint64_t* checksum_out, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  const MapCall c{false, dev_index, codec, level, block_size_or_default(codec_block_size), checksum_alg,
                  num_partitions, dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, status};
  const MapRows in{n_records, rec_base, rec_bytes, rec_len};
  if (int rc = round_robin_args(c, in, start_position, sort_rows)) return rc;
  return write_lane_run(wt, c, in, nullptr, RowIds::round_robin(start_position, sort_rows), nullptr,
                        partition_family(codec), nullptr, pass_through);
}

// The whole-task buffers of a sort call (read-lane slot 0: compressed blocks, decoded arena, sorted copy, sort
// workspace) only grow while they are in use.  When a call ends — whatever its result — every one of them above
// kSortKeepBytes is freed, so one oversized task does not keep several times its size of device memory for the rest
// of the process; buffers up to that size stay for the next call (a TeraSort reducer of 200 over 10 GiB needs ~55 MB).
struct SortBufferTrim {
  Slot& S;
  ~SortBufferTrim() {
    for (DevBuf* b : {&S.src, &S.dst, &S.parena, &S.pws, &S.fws})
      if (b->cap > kSortKeepBytes) b->release();
  }
};

// A source of an exchange-cache sorted read (b2s_exchange_read_sort_*): a cached range (records on the device, held by
// a reference for the call; status B2S_E_NOT_CACHED when it is not resident) or fetched block `block`.  A cached range
// of a row writer's entry has its record boundaries (marked): n_rec offsets at rec_off, numbered in the entry, whose
// first record is at entry offset first_off.
struct SortSource {
  bool cached = false;
  int32_t status = B2S_OK;
  const uint8_t* src = nullptr;
  uint64_t len = 0;
  uint32_t block = 0;
  bool marked = false;
  const uint64_t* rec_off = nullptr;
  uint64_t first_off = 0, n_rec = 0;
};

// A reduce task's sources once decoded (decode_task): their records back to back in source order in arena (source i:
// length[i] bytes at place[i]) and their statuses.  Only this struct tells a fetched block (its status is the decode
// job's) from an exchange read's cached range (mix: its SortSource's).  report() writes status[] and bad_slice[].
struct DecodedTask {
  std::vector<SortSource>* mix;
  int32_t *status_out, *bad_slice_out;  // bad_slice_out: nullptr when not wanted
  uint32_t n_src;
  std::vector<uint64_t> place, length;
  DecompressJob J;
  const uint8_t* arena = nullptr;
  uint64_t total = 0;
  bool failed = false;  // a source failed: the call ends with nothing sorted or written

  DecodedTask(std::vector<SortSource>* mix, uint32_t n, int32_t* status, int32_t* bad_slice)
      : mix(mix), status_out(status), bad_slice_out(bad_slice), n_src(mix ? (uint32_t)mix->size() : n), place(n_src),
        length(n_src) {}
  bool cached(uint32_t i) const { return mix && (*mix)[i].cached; }
  uint32_t block(uint32_t i) const { return mix ? (*mix)[i].block : i; }
  int32_t& status(uint32_t i) { return cached(i) ? (*mix)[i].status : J.h.status[block(i)]; }
  const SortSource* marked(uint32_t i) const { return cached(i) && (*mix)[i].marked ? &(*mix)[i] : nullptr; }
  // Source i fails with B2S_E_CORRUPT.  Only the call's first failed source is named in b2s_last_error ("block i" or
  // "cached source i", then what); a later one only gets its status.
  void fail_source(uint32_t i, const std::string& what) {
    status(i) = B2S_E_CORRUPT;
    if (!failed) fail(B2S_E_CORRUPT, cached(i) ? "cached source %s" : "block %s", (std::to_string(i) + what).c_str());
    failed = true;
  }
  void bad_row(uint32_t i, uint64_t byte, const char* why) {
    fail_source(i, ": bad row record at byte " + std::to_string(byte) + ": " + why);
  }
  // a value the device found bad in the record at arena byte at_byte: the source holding it (the last non-empty one
  // that starts at or before it) fails as for a framing verdict -> report()
  int fail_row_at(uint64_t at_byte, const char* why) {
    uint32_t i = 0;
    for (uint32_t k = 0; k < n_src; k++)
      if (place[k] <= at_byte && length[k]) i = k;
    bad_row(i, at_byte - place[i], why);
    return report();
  }
  int report() {  // -> 0, the result of a call that ends because a source failed (nothing is sorted or written)
    for (uint32_t i = 0; i < n_src; i++) {
      status_out[i] = status(i);
      if (bad_slice_out) bad_slice_out[i] = cached(i) ? -1 : J.h.bad[block(i)];
    }
    return 0;
  }
};

// Decodes the n blocks at d_src + src_dev_off[i] (src_contiguous: back to back) into T.  Phase A verifies and sizes
// them; a failed block, or (fixed-size records) a length that is not a multiple of record_bytes, fails the call.  Phase
// B decodes into S.dst (codec NONE: used in place, or copied there).  An exchange read (T.mix): the decoded offsets are
// shifted past the cached bytes before each block, and one gather moves the cached ranges (NONE: and blocks) around.
static int decode_task(Device* D, Slot& S, uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* d_src,
                       const uint64_t* src_dev_off, const uint64_t* src_len, bool src_contiguous,
                       const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_sum,
                       uint64_t srcb, const RecordSpec& spec, uint64_t out_cap, DecodedTask& T,
                       uint64_t* launches) {
  cudaStream_t st = S.st;
  DecompressJob& J = T.J;
  int rc;
  if (n) {
    rc = decompress_phase_a(S, D->tabs, codec, alg, n, src_dev_off, src_len, alg ? slice_base[n] : 0, slice_base,
                            slice_len, slice_sum, d_src, srcb, J, launches, true);
    if (rc) return rc;
    // the phase-A verdicts (checksums, stream headers) and decoded lengths, before anything is decoded
    CU(cudaMemcpyAsync(J.h.down, J.d.down, J.d.down_bytes, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
  } else {  // every source is cached
    CU(S.mark(K0, st));
  }
  uint64_t at = 0;
  for (uint32_t i = 0; i < T.n_src; i++) {
    const bool c = T.cached(i);
    const uint64_t len = c ? (*T.mix)[i].len : J.h.dst_len[T.block(i)];
    if (!c && T.status(i) == B2S_E_CORRUPT) T.fail_source(i, ": the compressed stream is corrupt");
    if (T.status(i) == B2S_OK && !spec.rows() && len % spec.record_bytes)
      T.fail_source(i, std::string(c ? " holds " : " decodes to ") + std::to_string(len) +
                           " bytes, not a multiple of record_bytes " + std::to_string(spec.record_bytes));
    T.failed |= T.status(i) != B2S_OK;
    T.place[i] = at;
    T.length[i] = len;
    at += len;
  }
  T.total = T.mix ? at : J.h.totals[1];
  if (T.failed) return T.report();
  if (!spec.rows() && T.total / spec.record_bytes > 0xffffffffull)
    return fail(B2S_E_ARG, "more than 2^32 - 1 records in one call (%s bytes)", std::to_string(T.total).c_str());
  // an aggregation's, join's or window's output is sized later
  if (!spec.aggregate && !spec.join && !spec.window && T.total > out_cap) {
    T.report();
    return fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s decoded bytes", std::to_string(T.total).c_str());
  }

  // the decoded arena: every source's records back to back in order; in S.dst unless codec NONE left them so
  T.arena = d_src;
  if (T.mix || codec != B2S_CODEC_NONE || (!src_contiguous && T.total)) {
    if ((rc = S.dst.ensure(T.total + 64))) return rc;
    T.arena = (const uint8_t*)S.dst.p;
  }
  if (T.mix) {
    std::vector<ExchangePiece> pieces;
    for (uint32_t i = 0; i < T.n_src; i++) {
      const SortSource& s = (*T.mix)[i];
      if (s.cached)
        exchange_add_pieces(pieces, s.src, T.place[i], s.len);
      else if (codec == B2S_CODEC_NONE)
        exchange_add_pieces(pieces, d_src + src_dev_off[s.block], T.place[i], src_len[s.block]);
      else
        J.h.dst_off[s.block] = T.place[i];
    }
    if (n && codec != B2S_CODEC_NONE)  // phase B decodes every block straight to its place among the cached ranges
      CU(cudaMemcpyAsync(J.d.dst_off, J.h.dst_off, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    if (!pieces.empty()) {
      if ((rc = S.xpieces.ensure(pieces.size() * sizeof(ExchangePiece)))) return rc;
      CU(cudaMemcpyAsync(S.xpieces.p, pieces.data(), pieces.size() * sizeof(ExchangePiece), cudaMemcpyHostToDevice,
                         st));
      launch_exchange_gather((const ExchangePiece*)S.xpieces.p, (uint32_t)pieces.size(), (uint8_t*)S.dst.p, st,
                             launches);
    }
  }
  if (codec != B2S_CODEC_NONE && n) {
    if ((rc = decompress_enqueue_b(S, J, d_src, (uint8_t*)S.dst.p, S.dst.cap, launches))) return rc;
    CU(cudaEventSynchronize(S.ev_b));
    CU(cudaGetLastError());
    for (uint32_t i = 0; i < T.n_src; i++)
      if (!T.cached(i) && T.status(i) != B2S_OK) T.fail_source(i, ": the compressed stream is corrupt");
  } else if (!T.mix && !src_contiguous) {
    for (uint32_t i = 0; i < n; i++)
      if (src_len[i])
        CU(cudaMemcpyAsync((uint8_t*)S.dst.p + J.h.dst_off[i], d_src + src_dev_off[i], src_len[i],
                           cudaMemcpyDeviceToDevice, st));
  }
  return T.report();
}

// a source whose row verdict v[i] (framing, or the key pass's string check) is not ~0 fails, the first one named
static void take_verdicts(DecodedTask& T, const RecordSpec& spec, const uint64_t* v) {
  const char* const why[] = {"", "the block ends inside a size prefix", "the size is negative",
                             "the record runs past the block end",
                             spec.join     ? "the row is shorter than its side's fixed region"
                             : spec.window ? "the row is shorter than its fixed region"
                                           : "the row is shorter than key_off + key_len",
                             "the row does not hold the null-bit word", "the row is shorter than an aggregate slot",
                             "a string key runs past the end of its row, or a decimal key's size "
                             "is not in [1, 16] or its bytes run past the end of its row"};
  for (uint32_t i = 0; i < T.n_src; i++)
    if (v[i] != ~0ull) T.bad_row(i, v[i] & ((1ull << 61) - 1), why[v[i] >> 61]);
}

// A window's output-row shape from its arguments (launch_window_values; the field list is the tail's)
static void window_shape(const RecordSpec& spec, WindowShape& shape) {
  const WindowSpec& ws = *spec.window;
  shape.n = ws.n_fields;
  shape.bw = bitset_words(ws.n_fields);
  shape.out_bw = bitset_words(ws.n_fields + ws.n_fns);
  shape.n_fns = ws.n_fns;
  for (uint32_t j = 0; j < ws.n_fns; j++) {
    shape.fn[j] = ws.fn[j];
    shape.arg[j] = (uint32_t)ws.fn_arg[j];
    shape.wide[j] = -1;
    shape.nn[j] = -1;
    if (ws.fn[j] < B2S_WINDOW_SUM) continue;
    const uint32_t vt = ws.val_type[j], p = (vt >> 8) & 0xff;
    shape.frame[j] = ws.frame[j];
    shape.vtype[j] = vt;
    shape.voff[j] = ws.val_off[j];
    shape.vnull[j] = ws.val_null[j];
    if (ws.fn[j] >= B2S_WINDOW_LAG) {  // an offset function: a non-null index when it skips nulls that can occur
      shape.flags[j] = ws.flags[j];
      shape.dflt[j] = ws.dflt[j];
      if ((ws.flags[j] & B2S_WINDOW_IGNORE_NULLS) && ws.val_null[j] >= 0) shape.nn[j] = (int32_t)shape.n_nn++;
      shape.n_off++;
      if ((vt & 0xff) == B2S_WINDOW_VAL_DECIMAL && p > 18) shape.n_wide_off++;
      continue;
    }
    shape.agg[j] = shape.n_agg++;
    const uint32_t rp = p + (ws.fn[j] == B2S_WINDOW_SUM ? 10 : ws.fn[j] == B2S_WINDOW_AVG ? 4 : 0);
    if ((vt & 0xff) == B2S_WINDOW_VAL_DECIMAL && ws.fn[j] != B2S_WINDOW_COUNT && rp > 18)
      shape.wide[j] = (int32_t)shape.n_wide++;
  }
  for (uint32_t j = 0; j < ws.n_fns; j++) {  // sliding frames: bounds sets, result states, the staged order column
    shape.bnd[j] = shape.res[j] = -1;
    if (!ws.frames || (ws.frame[j] != B2S_WINDOW_FRAME_ROWS && ws.frame[j] != B2S_WINDOW_FRAME_RANGE)) continue;
    const int64_t lo = ws.lower[j], hi = ws.upper[j];
    uint32_t b = 0;
    while (b < shape.n_bnd && !(shape.bkind[b] == ws.frame[j] && shape.blo[b] == lo && shape.bhi[b] == hi)) b++;
    if (b == shape.n_bnd) {
      shape.bkind[b] = ws.frame[j];
      shape.blo[b] = lo;
      shape.bhi[b] = hi;
      shape.n_bnd++;
    }
    shape.bnd[j] = (int32_t)b;
    const bool finite = [](int64_t k) {
      return k != 0 && k != B2S_WINDOW_UNBOUNDED_PRECEDING && k != B2S_WINDOW_UNBOUNDED_FOLLOWING;
    }(lo) || (hi != 0 && hi != B2S_WINDOW_UNBOUNDED_PRECEDING && hi != B2S_WINDOW_UNBOUNDED_FOLLOWING);
    if (ws.frame[j] == B2S_WINDOW_FRAME_RANGE && finite) {
      const uint32_t c = ws.n_partition_keys;
      shape.ord_staged = true;
      shape.ord_type = spec.keys.type[c];
      shape.ord_off = spec.keys.off[c];
      shape.ord_len = spec.keys.len[c];
      shape.ord_null = spec.keys.null_field[c];
    }
    const uint32_t fn = ws.fn[j], kind = ws.val_type[j] & 0xff;
    if (lo == B2S_WINDOW_UNBOUNDED_PRECEDING || fn < B2S_WINDOW_SUM || fn > B2S_WINDOW_AVG) continue;
    const bool dbl = (fn == B2S_WINDOW_SUM && (kind == B2S_WINDOW_VAL_FLOAT32 || kind == B2S_WINDOW_VAL_FLOAT64)) ||
                     (fn == B2S_WINDOW_AVG && kind != B2S_WINDOW_VAL_DECIMAL);
    if (!dbl && fn != B2S_WINDOW_MIN && fn != B2S_WINDOW_MAX) continue;  // sums and counts: prefix differences
    shape.res[j] = (int32_t)shape.n_res++;
    if (dbl) continue;
    const bool rows = ws.frame[j] == B2S_WINDOW_FRAME_ROWS && hi != B2S_WINDOW_UNBOUNDED_FOLLOWING;
    const uint64_t width = rows ? (uint64_t)(hi - lo + 1) : ~0ull;
    shape.rmq_width = std::max(shape.rmq_width, width);
  }
  shape.limit_fn = ws.limit_fn;
  shape.limit = ws.limit;
  shape.part.n = ws.n_partition_keys;
  for (uint32_t c = 0; c < ws.n_partition_keys; c++) {
    shape.part.type[c] = spec.keys.type[c];
    shape.part.off[c] = spec.keys.off[c];
    shape.part.len[c] = spec.keys.len[c];
    shape.part.null_field[c] = spec.keys.null_field[c];
  }
}

// A reduce task's rows in key order (order_rows): idx (nullptr: arena order), heads (nullptr: where key words differ),
// and S.pws's parts in order: sort, aggregation, refinement (nullptr unless the key refines), join or window grouping,
// join, window.
struct RowOrder {
  uint64_t records = 0;
  uint32_t key_bytes = 0;
  const uint32_t *idx = nullptr, *heads = nullptr;
  uint8_t *ws = nullptr, *aws = nullptr, *rws = nullptr, *gws = nullptr, *jws = nullptr, *wws = nullptr;
  void carve(uint8_t* base, const size_t (&bytes)[6]) {
    uint8_t** part[] = {&ws, &aws, &rws, &gws, &jws, &wws};
    for (int k = 0; k < 6; k++) {
      *part[k] = base;
      base += bytes[k];
    }
  }
};

// Orders T's rows by key into R: framing, one readback of the record count and the verdicts (a bad source fails the
// call), which sizes the workspace with the tail's parts (a join's n_join_fields), then emit, the first-pass sort and
// the refine rounds, one readback each.  jk: a join's keys per side as its kernels encode them; nullptr: spec.keys.
static int order_rows(Slot& S, const RecordSpec& spec, DecodedTask& T, const JoinKeys* jk, uint32_t n_join_fields,
                      RowOrder& R, uint64_t* launches) {
  cudaStream_t st = S.st;
  const KeySpec& ks = spec.keys;
  const uint32_t n_src = T.n_src;
  uint64_t min_key = 0, min_null = 0;
  for (uint32_t c = 0; c < ks.n && !jk; c++) {  // a join checks each side's rows in its key pass
    min_key = std::max<uint64_t>(min_key, (uint64_t)ks.off[c] + ks.len[c]);
    if (ks.null_field[c] >= 0) min_null = std::max<uint64_t>(min_null, null_word(ks.null_field[c]) + 8);
  }
  const WindowSpec* win = spec.window;  // a window's rows hold its whole fixed region, which holds every key slot
  if (win) min_key = 8ull * (bitset_words(win->n_fields) + win->n_fields);
  WindowShape wshape{};
  if (win) window_shape(spec, wshape);
  // a cached range with record boundaries is marked from them instead of walked (its walk is empty)
  std::vector<uint64_t> walk(T.length);
  std::vector<RowsMark> marks;
  for (uint32_t i = 0; i < n_src; i++) {
    const SortSource* s = T.marked(i);
    if (!s) continue;
    walk[i] = 0;
    marks.push_back(RowsMark{s->rec_off, T.place[i] - s->first_off, T.place[i],
                             marks.empty() ? 0 : marks.back().first + marks.back().count, s->n_rec, i});
  }
  int rc;
  if ((rc = S.fws.ensure(rows_frame_ws_bytes(T.total, n_src, (uint32_t)marks.size())))) return rc;
  uint8_t* fws = (uint8_t*)S.fws.p;
  CU(S.mark(P0, st));
  CU(S.mark(F0, st, *launches));
  launch_rows_frame(T.arena, T.total, T.place.data(), walk.data(), n_src, min_key, min_null, agg_min_row(spec), fws,
                    st, launches, marks.data(), (uint32_t)marks.size());
  CU(S.mark(F1, st, *launches));
  std::vector<uint64_t> rb(n_src + 1);
  CU(cudaMemcpyAsync(rb.data(), rows_frame_readback(fws, T.total, n_src), rows_frame_readback_bytes(n_src),
                     cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  for (const RowsMark& m : marks) rb[1 + m.range] = rows_mark_verdict(rb[1 + m.range]);
  take_verdicts(T, spec, rb.data() + 1);
  if (T.failed) return T.report();
  const uint64_t records = R.records = rb[0];
  if (records > 0xffffffffull)
    return fail(B2S_E_ARG, "more than 2^32 - 1 records in one call (%s records)", std::to_string(records).c_str());
  const KeySpec& encoded = jk ? jk->side[0] : ks;
  R.key_bytes = rows_key_bytes(encoded);
  const bool refine = rows_key_refines(encoded);
  const AggSpec agg = spec.aggregate ? agg_spec(spec) : AggSpec{};
  const size_t part[6] = {rows_sort_ws_bytes(records, R.key_bytes),
                          spec.aggregate ? rows_aggregate_ws_bytes(records, spec.n_aggs, agg.n_wide, agg.n_var) : 0,
                          refine ? rows_refine_ws_bytes(records, n_src) : 0,
                          jk || win ? rows_aggregate_ws_bytes(records, 0, 0) : 0,
                          jk ? join_ws_bytes(records, n_src, n_join_fields) : 0,
                          win ? window_ws_bytes(records, wshape) : 0};
  if ((records || jk) && (rc = S.pws.ensure(part[0] + part[1] + part[2] + part[3] + part[4] + part[5]))) return rc;
  R.carve((uint8_t*)S.pws.p, part);
  if (!refine) R.rws = nullptr;
  CU(S.mark(F2, st, *launches));
  launch_rows_emit(T.arena, T.total, n_src, fws, records, R.key_bytes, R.ws, st, launches);
  CU(S.mark(F3, st, *launches));
  const uint64_t* ranges = rows_frame_ranges(fws, T.total, n_src);
  R.idx = jk ? launch_rows_join_order(T.arena, records, *jk, ranges, n_src, join_readback(R.jws, records, n_src) + 4,
                                      R.ws, R.rws, st, launches)
             : launch_rows_order(T.arena, records, ks, ranges, n_src, R.ws, R.rws, st, launches);
  if (!refine || !records) return 0;
  // one readback per round: the tied records and their runs (the first also brings the string verdicts)
  std::vector<uint64_t> rrb(n_src + 1);
  for (uint32_t d = kKeyPrefixBytes, round = 0;; d += kKeyChunkBytes, round++) {
    launch_rows_refine_mark(records, d, R.rws, n_src, st, launches);
    CU(cudaMemcpyAsync(rrb.data(), rows_refine_readback(R.rws, records, n_src), (round ? 1 : rrb.size()) * 8,
                       cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    if (!round) {
      take_verdicts(T, spec, rrb.data() + 1);
      if (T.failed) return T.report();
    }
    const uint64_t tied = rrb[0] & 0xffffffffull, runs = rrb[0] >> 32;
    if (!tied) break;
    if (jk) launch_rows_join_refine_round(T.arena, records, *jk, tied, runs, d, R.ws, R.rws, st, launches);
    else launch_rows_refine_round(T.arena, records, ks, tied, runs, d, R.ws, R.rws, n_src, st, launches);
  }
  R.idx = rows_refine_order(R.rws, records, n_src);
  R.heads = rows_refine_heads(R.rws, records, n_src);
  return 0;
}

// The end of an aggregation: grouping, one readback of the group count, output bytes (*total, checked against out_cap)
// and decimal verdict, the heads' gather and the merge into d_out.  A bad out-of-line decimal (kAggBad*) fails its
// source and nothing is written.  The dominant step is this one (marks G0, G1).
static int aggregate_rows_tail(Slot& S, const RecordSpec& spec, DecodedTask& T, const RowOrder& R, uint8_t* d_out,
                               uint64_t out_cap, uint64_t* total, uint64_t* n_rec, uint64_t* n_groups,
                               uint64_t* launches) {
  cudaStream_t st = S.st;
  const AggSpec agg = agg_spec(spec);
  uint64_t rb[3] = {0, 0, ~0ull};  // groups, output bytes, decimal verdict
  CU(S.mark(G0, st, *launches));
  if (R.records) {
    launch_rows_group(T.arena, R.records, R.idx, R.heads, R.key_bytes, agg, R.ws, R.aws, st, launches);
    CU(cudaMemcpyAsync(rb, rows_aggregate_readback(R.aws, R.records, agg.n, agg.n_wide), (agg.n_wide ? 3 : 2) * 8,
                       cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
  }
  if (rb[2] != ~0ull) {
    static const char* const why[] = {"",
                                      "a decimal aggregate's size is not in [1, 16] or its bytes run past the end of "
                                      "its row",
                                      "a decimal aggregate's 16-byte region runs past the end of its row",
                                      "a decimal aggregate's 16-byte region starts before the end of a slot or null "
                                      "word in use"};
    return T.fail_row_at(rb[2] >> 2, why[rb[2] & 3]);
  }
  *total = rb[1];
  if (rb[1] > out_cap)
    return fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s output bytes", std::to_string(rb[1]).c_str());
  launch_rows_aggregate(T.arena, R.records, rb[0], R.key_bytes, agg, R.ws, R.aws, d_out, st, launches);
  CU(S.mark(G1, st, *launches));
  CU(S.mark(P1, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *n_rec = R.records;
  if (n_groups) *n_groups = rb[0];
  return 0;
}

// A join's key columns per side (JoinKeys: a plain column nullable on one side only takes kNullByteOnly on the other,
// so equal keys encode equal; a null-safe column encodes its trailing isnull byte on both sides whatever their null
// fields; split: the arena offset of the right side's first block) and its joined row's shape, whose key columns are
// those a null makes unmatchable (a null-safe column's null field is -1 there) and whose field lists (left VAR /
// DECIMAL_WIDE fields, right ones, right DECIMAL_WIDE ones, left DECIMAL_WIDE ones) go to fields.  An existence join's
// row is the left row and one boolean field: no right field list.
static void join_layout(const RecordSpec& spec, uint64_t split, JoinKeys& jk, JoinShape& shape,
                        std::vector<uint32_t>& fields) {
  const JoinSpec& js = *spec.join;
  jk.side[0] = spec.keys;
  jk.side[1] = js.right;
  shape.keys[0] = spec.keys;
  shape.keys[1] = js.right;
  for (uint32_t c = 0; c < spec.keys.n; c++) {
    if (spec.keys.type[c] & B2S_KEY_NULL_SAFE) {
      shape.keys[0].null_field[c] = shape.keys[1].null_field[c] = -1;
      continue;
    }
    int32_t& l = jk.side[0].null_field[c];
    int32_t& r = jk.side[1].null_field[c];
    if (l >= 0 && r < 0) r = kNullByteOnly;
    if (r >= 0 && l < 0) l = kNullByteOnly;
  }
  jk.split = split;
  shape.type = js.type;
  shape.split = split;
  for (uint32_t s = 0; s < 2; s++) {
    shape.n[s] = js.n_fields[s];
    shape.bw[s] = bitset_words(js.n_fields[s]);
    jk.fixed[s] = 8 * (shape.bw[s] + shape.n[s]);
  }
  const bool exists = js.type == B2S_JOIN_EXISTENCE;
  shape.out_bw = bitset_words(shape.n[0] + (exists ? 1 : shape.n[1]));
  fields.clear();
  const bool rows = !join_keeps_whole(js.type);  // a semi or anti join: no kinds
  for (uint32_t s = 0; s < 2; s++) {
    for (uint32_t f = 0; rows && !(exists && s) && f < shape.n[s]; f++)
      if (js.kind[s][f] != B2S_FIELD_FIXED) fields.push_back(f);
    shape.n_var[s] = (uint32_t)fields.size() - (s ? shape.n_var[0] : 0);
  }
  for (uint32_t s : {1u, 0u}) {  // the null side's wide decimals: the right side's, then the left side's
    const size_t before = fields.size();
    for (uint32_t f = 0; rows && !exists && f < shape.n[s]; f++)
      if (js.kind[s][f] == B2S_FIELD_DECIMAL_WIDE) fields.push_back(f);
    shape.n_wide[s] = (uint32_t)(fields.size() - before);
  }
}

// The end of a join: grouping, counts (one readback with the key pass's verdicts; *total = output bytes), the joined
// rows into *d_out (nullptr: into S.parena, returned there) and the per-side counts.  The dominant step (G0, G1).
static int join_rows_tail(Slot& S, const RecordSpec& spec, DecodedTask& T, const RowOrder& R, const JoinShape& shape,
                          const std::vector<uint32_t>& fields, uint8_t** d_out, uint64_t out_cap, uint64_t* total,
                          uint64_t* n_rec, uint64_t* launches) {
  cudaStream_t st = S.st;
  std::vector<uint64_t> jb(4 + T.n_src, ~0ull);
  jb[0] = jb[1] = jb[2] = jb[3] = 0;
  CU(S.mark(G0, st, *launches));
  if (R.records) {
    launch_rows_group(T.arena, R.records, R.idx, R.heads, R.key_bytes, AggSpec{}, R.ws, R.gws, st, launches);
    launch_join_count(T.arena, R.records, R.idx, shape, fields.data(), (uint32_t)fields.size(), R.key_bytes, R.ws,
                      R.gws, R.jws, T.n_src, st, launches);
    CU(cudaMemcpyAsync(jb.data(), join_readback(R.jws, R.records, T.n_src), join_readback_bytes(T.n_src),
                       cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
  }
  take_verdicts(T, spec, jb.data() + 4);
  if (T.failed) return T.report();
  if (jb[3]) return fail(B2S_E_UNSUPPORTED, "a joined row is longer than 2^31 - 1 bytes%s");
  *total = jb[1];
  if (jb[1] > out_cap)
    return fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s output bytes", std::to_string(jb[1]).c_str());
  if (!*d_out) {
    if (int rc = S.parena.ensure(jb[1] + 64)) return rc;
    *d_out = (uint8_t*)S.parena.p;
  }
  launch_join_emit(T.arena, R.records, R.idx, jb[0], R.key_bytes, spec.join->type, R.ws, R.jws, T.n_src, *d_out, st,
                   launches);
  CU(S.mark(G1, st, *launches));
  CU(S.mark(P1, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *n_rec = jb[0];
  *spec.join->n_side[0] = jb[2];
  *spec.join->n_side[1] = R.records - jb[2];
  return 0;
}

// The end of a window: grouping (the peer groups), then partitions, values and output bytes (one readback: *total =
// output bytes), the output rows into *d_out (nullptr: into S.parena, returned there) and the input record count.  The
// dominant step (G0, G1).
static int window_rows_tail(Slot& S, const RecordSpec& spec, DecodedTask& T, const RowOrder& R, uint8_t** d_out,
                            uint64_t out_cap, uint64_t* total, uint64_t* n_rec, uint64_t* launches) {
  cudaStream_t st = S.st;
  const WindowSpec& ws = *spec.window;
  WindowShape shape{};
  window_shape(spec, shape);
  std::vector<uint32_t> fields;  // the slots whose offsets move
  for (uint32_t f = 0; f < ws.n_fields; f++)
    if (ws.kind[f] != B2S_FIELD_FIXED) fields.push_back(f);
  shape.n_var = (uint32_t)fields.size();
  // output records, output bytes, a row too long, a partition too large, a bad decimal input, a frame bound wraps
  uint64_t wb[6] = {0, 0, 0, 0, ~0ull, 0};
  CU(S.mark(G0, st, *launches));
  if (R.records) {
    launch_rows_group(T.arena, R.records, R.idx, R.heads, R.key_bytes, AggSpec{}, R.ws, R.gws, st, launches);
    launch_window_values(T.arena, R.records, R.idx, shape, fields.data(), R.key_bytes, R.ws, R.gws, R.wws, st,
                         launches);
    CU(cudaMemcpyAsync(wb, window_readback(R.wws, R.records, shape), kWindowReadbackBytes, cudaMemcpyDeviceToHost,
                       st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
  }
  if (wb[4] != ~0ull)
    return T.fail_row_at(wb[4] >> 2, (wb[4] & 3) == kWindowBadBytes
                                         ? "a string input's bytes lie outside its row's variable-length region"
                                         : "a decimal input's size is not in [1, 16] or its bytes run past the end of "
                                           "its row");
  if (wb[3]) return fail(B2S_E_UNSUPPORTED, "a window partition holds more than 2^31 - 1 records%s");
  if (wb[5])
    return fail(B2S_E_UNSUPPORTED, "a sliding frame's bound wraps in Spark's int arithmetic (a partition's size plus "
                                   "a ROWS offset past 2^31 - 1, or a RANGE bound outside its column's type)%s");
  if (wb[2]) return fail(B2S_E_UNSUPPORTED, "an output row is longer than 2^31 - 1 bytes%s");
  *total = wb[1];
  if (wb[1] > out_cap)
    return fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s output bytes", std::to_string(wb[1]).c_str());
  if (!*d_out) {
    if (int rc = S.parena.ensure(wb[1] + 64)) return rc;
    *d_out = (uint8_t*)S.parena.p;
  }
  launch_window_emit(T.arena, R.records, R.idx, wb[0], R.key_bytes, shape, ws.limit_fn != B2S_WINDOW_NO_LIMIT,
                     R.ws, R.wws, *d_out, st, launches);
  CU(S.mark(G1, st, *launches));
  CU(S.mark(P1, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *n_rec = wb[0];
  *ws.n_in = R.records;
  return 0;
}

// After decode_task: the fixed-size records' key sort, or order_rows and the tail of the call's family (a row sort's:
// the gather), into *d_sorted (nullptr: into S.parena, returned there).  A failed source: 0, status[] set, *n_rec 0.
static int run_reduce_task(Slot& S, const RecordSpec& spec, DecodedTask& T, uint8_t** d_sorted, uint64_t out_cap,
                           uint64_t* total, uint64_t* n_rec, uint64_t* n_groups, uint64_t* launches) {
  int rc;
  if (!*d_sorted && !spec.join && !spec.window) {
    if ((rc = S.parena.ensure(T.total + 64))) return rc;
    *d_sorted = (uint8_t*)S.parena.p;
  }
  uint64_t records;
  if (!spec.rows()) {  // fixed-size records: their key sort
    records = T.total / spec.record_bytes;
    if (records && (rc = S.pws.ensure(key_sort_ws_bytes(records, spec.keys.len[0])))) return rc;
    CU(S.mark(P0, S.st));
    launch_key_sort(T.arena, records, spec.record_bytes, spec.keys.off[0], spec.keys.len[0], (uint8_t*)S.pws.p,
                    *d_sorted, S.st, launches);
  } else {
    // a join: its key columns per side as its kernels encode them (a column nullable on one side only takes a null
    // byte on both), which set the key's width for every step, and its joined row's shape
    std::vector<uint32_t> join_fields;
    JoinKeys jk;
    JoinShape shape{};
    if (spec.join)
      join_layout(spec, T.n_src > spec.join->n_left ? T.place[spec.join->n_left] : T.total, jk, shape, join_fields);
    RowOrder R;
    rc = order_rows(S, spec, T, spec.join ? &jk : nullptr, (uint32_t)join_fields.size(), R, launches);
    if (rc || T.failed) return rc;
    if (spec.join) return join_rows_tail(S, spec, T, R, shape, join_fields, d_sorted, out_cap, total, n_rec, launches);
    if (spec.window) return window_rows_tail(S, spec, T, R, d_sorted, out_cap, total, n_rec, launches);
    if (spec.aggregate) return aggregate_rows_tail(S, spec, T, R, *d_sorted, out_cap, total, n_rec, n_groups, launches);
    records = R.records;
    launch_rows_gather(T.arena, records, R.key_bytes, R.idx, R.ws, *d_sorted, S.st, launches);
  }
  CU(S.mark(P1, S.st));
  CU(cudaStreamSynchronize(S.st));
  CU(cudaGetLastError());
  *n_rec = records;
  return 0;
}

// A reduce task's n blocks at src_base + src_off[i], src_len[i] bytes each (*srcb in all), where its decode reads them:
// device blocks where they are, or (packed) host blocks in one upload back to back into S.src between marks H0 and H1
// (the whole task is resident at once: no chunking), blocks adjacent in host memory in one copy.  -> *base, *off.
static int task_blocks(Slot& S, bool packed, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
                       const uint64_t* src_len, std::vector<uint64_t>& dev_off, const uint8_t** base,
                       const uint64_t** off, uint64_t* srcb) {
  cudaStream_t st = S.st;
  *srcb = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (packed) dev_off.push_back(*srcb);
    *srcb += src_len[i];
  }
  *base = src_base;
  *off = src_off;
  if (!packed) return 0;
  if (int rc = S.src.ensure(*srcb + 64)) return rc;
  CU(S.mark(H0, st));
  for (uint32_t i = 0; i < n;) {
    uint32_t j = i + 1;
    while (j < n && src_off[j] == src_off[j - 1] + src_len[j - 1]) j++;
    const uint64_t bytes = dev_off[j - 1] + src_len[j - 1] - dev_off[i];
    if (bytes)
      CU(cudaMemcpyAsync((uint8_t*)S.src.p + dev_off[i], src_base + src_off[i], bytes, cudaMemcpyHostToDevice, st));
    i = j;
  }
  CU(S.mark(H1, st));
  *base = (const uint8_t*)S.src.p;
  *off = dev_off.data();
  return 0;
}

// A reduce task on the read lane of D (decode_task, run_reduce_task) over device blocks into device memory at dst_base,
// or (packed) over host blocks, with one upload before and one download into dst_base (host memory) after.
static int read_task_run(Device* D, bool packed, uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* src_base,
                         const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                         const uint64_t* slice_len, const uint64_t* slice_checksum, const RecordSpec& spec,
                         uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                         uint64_t* n_groups, int32_t* status, int32_t* bad_slice, const WallTimer& wt,
                         std::vector<SortSource>* mix) {
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  SortBufferTrim trim{S};
  cudaStream_t st = S.st;
  std::vector<uint64_t> dev_off;
  const uint8_t* blocks;
  const uint64_t* block_off;
  uint64_t srcb;
  int rc = task_blocks(S, packed, n, src_base, src_off, src_len, dev_off, &blocks, &block_off, &srcb);
  if (rc) return rc;
  uint8_t* out = packed ? nullptr : dst_base;
  uint64_t launches = 0;
  DecodedTask T(mix, n, status, bad_slice);
  rc = decode_task(D, S, codec, alg, n, blocks, block_off, src_len, packed, slice_base, slice_len, slice_checksum, srcb,
                   spec, dst_cap, T, &launches);
  *dst_total = T.failed ? 0 : T.total;  // a failed source: nothing is written
  *n_records = 0;
  if (!rc && !T.failed) rc = run_reduce_task(S, spec, T, &out, dst_cap, dst_total, n_records, n_groups, &launches);
  if (rc) return rc;
  const uint64_t down = packed && *n_records ? *dst_total : 0;
  if (packed) {
    CU(S.mark(D0, st));
    if (down) CU(cudaMemcpyAsync(dst_base, out, down, cudaMemcpyDeviceToHost, st));
    CU(S.mark(D1, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
  }
  end_call(wt, launches, CallBytes{srcb, *dst_total, packed ? srcb : 0, down}, &S, spec.family());
  return 0;
}

// The sources of an exchange sorted read: the fetched ones compacted in source order with their slices (what
// read_task_run takes as its blocks), and every source in order.
struct MixedSources {
  std::vector<SortSource> src;
  std::vector<uint64_t> off, len, slice_len, slice_sum;
  std::vector<uint32_t> slice_base{0};
};

static int exchange_sort_args(int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids, const uint8_t* cached,
                              uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* src_base,
                              const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                              const uint64_t* slice_len, const uint64_t* slice_checksum, const RecordSpec& spec,
                              const void* dst_base, uint64_t dst_cap,
                              const uint64_t* dst_total, const uint64_t* n_records, const int32_t* status,
                              MixedSources& M) {
  int rc = reduce_range_args(start_reduce, end_reduce);
  if (rc) return rc;
  if (n && (!map_ids || !cached || !status)) return fail(B2S_E_ARG, "null argument%s");
  M.src.resize(n);
  for (uint32_t i = 0; i < n; i++) {
    M.src[i].cached = cached[i] != 0;
    if (M.src[i].cached) continue;
    if (!src_off || !src_len) return fail(B2S_E_ARG, "null argument%s");
    if (alg && (!slice_base || !slice_len || !slice_checksum)) return fail(B2S_E_ARG, "slice arrays required%s");
    M.src[i].block = (uint32_t)M.off.size();
    M.off.push_back(src_off[i]);
    M.len.push_back(src_len[i]);
    if (alg) {
      if (slice_base[i + 1] < slice_base[i]) return fail(B2S_E_ARG, "slice_base must be non-decreasing%s");
      M.slice_len.insert(M.slice_len.end(), slice_len + slice_base[i], slice_len + slice_base[i + 1]);
      M.slice_sum.insert(M.slice_sum.end(), slice_checksum + slice_base[i], slice_checksum + slice_base[i + 1]);
      M.slice_base.push_back((uint32_t)M.slice_len.size());
    }
  }
  const uint32_t m = (uint32_t)M.off.size();
  return sort_args(codec, alg, m, M.off.data(), M.len.data(), M.slice_base.data(), M.slice_len.data(),
                   M.slice_sum.data(), spec, src_base, dst_base, dst_cap, dst_total, n_records, status);
}

// references the cached sources of M on device D and describes them; B2S_E_ARG when a range exceeds an entry
static int exchange_sort_sources(const ExRefs& refs, int32_t start_reduce, int32_t end_reduce, MixedSources& M) {
  if (int rc = refs.check_range(end_reduce)) return rc;
  for (uint32_t i = 0; i < (uint32_t)M.src.size(); i++) {
    SortSource& s = M.src[i];
    if (!s.cached) continue;
    if (refs.entry[i]) {
      s.src = refs.range(i, start_reduce, end_reduce, &s.len);
      s.marked = refs.bounds(i, start_reduce, end_reduce, &s.first_off, &s.rec_off, &s.n_rec);
    } else {
      s.status = B2S_E_NOT_CACHED;
    }
  }
  return 0;
}

// the exchange-cache key of a sorted read whose sources may be resident (b2s_exchange_read_sort_*)
struct ExchangeRead {
  int32_t shuffle, start_reduce, end_reduce;
  const int64_t* map_ids;
  const uint8_t* cached;
};

// The body of the sort calls: zero the outputs, check the arguments and take the device, then run on the read lane
// over device-resident blocks into device memory, or (packed) over host blocks into host memory.  x: an exchange read,
// whose sources are cached ranges or fetched blocks.  A plain sort checks the device before its arguments; an
// exchange read checks its arguments, then that the exchange cache can be used, then the device.
static int sort_call(uint32_t dev_index, bool packed, const ExchangeRead* x, uint32_t codec, uint32_t alg, uint32_t n,
                     const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                     const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                     const RecordSpec& spec, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
                     uint64_t* n_records, int32_t* status, int32_t* bad_slice, uint64_t* n_groups = nullptr) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  if (n_records) *n_records = 0;
  if (n_groups) *n_groups = 0;
  Device* D;
  MixedSources M;
  int rc;
  if (!x) {
    if ((rc = sort_device(dev_index, &D))) return rc;
    rc = sort_args(codec, alg, n, src_off, src_len, slice_base, slice_len, slice_checksum, spec, src_base, dst_base,
                   dst_cap, dst_total, n_records, status);
  } else if ((rc = exchange_sort_args(x->start_reduce, x->end_reduce, x->map_ids, x->cached, codec, alg, n, src_base,
                                      src_off, src_len, slice_base, slice_len, slice_checksum, spec, dst_base, dst_cap,
                                      dst_total, n_records, status, M)) ||
             (rc = exchange_ready())) {
    return rc;
  } else {
    rc = sort_device(dev_index, &D);
  }
  if (rc || !n) return rc;
  std::optional<ExRefs> refs;
  std::vector<SortSource>* mix = nullptr;
  if (x) {
    refs.emplace(D->ordinal, x->shuffle, n, x->map_ids, x->cached);
    if ((rc = exchange_sort_sources(*refs, x->start_reduce, x->end_reduce, M))) return rc;
    n = (uint32_t)M.off.size();
    src_off = M.off.data();
    src_len = M.len.data();
    slice_base = M.slice_base.data();
    slice_len = M.slice_len.data();
    slice_checksum = M.slice_sum.data();
    mix = &M.src;
  }
  return read_task_run(D, packed, codec, alg, n, src_base, src_off, src_len, slice_base, slice_len, slice_checksum,
                       spec, dst_base, dst_cap, dst_total, n_records, n_groups, status, bad_slice, wt, mix);
}

int b2s_decompress_sort_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                            const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                            const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                            uint32_t record_bytes, uint32_t key_off, uint32_t key_len, uint8_t* dst_base,
                            uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                            int32_t* bad_slice) {
  return sort_call(dev_index, false, nullptr, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, fixed_spec(record_bytes, key_off, key_len), dst_base, dst_cap, dst_total, n_records,
                   status, bad_slice);
}

int b2s_decompress_sort_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                               const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                               const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t record_bytes,
                               uint32_t key_off, uint32_t key_len, uint8_t* dst_base, uint64_t dst_cap,
                               uint64_t* dst_total, uint64_t* n_records, int32_t* status, int32_t* bad_slice) {
  return sort_call(t_device, true, nullptr, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, fixed_spec(record_bytes, key_off, key_len), dst_base, dst_cap, dst_total, n_records,
                   status, bad_slice);
}

int b2s_decompress_sort_rows_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                 const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                 const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                                 uint32_t key_type, uint32_t key_off, uint32_t key_len, int32_t null_field,
                                 uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                                 int32_t* status, int32_t* bad_slice) {
  return sort_call(dev_index, false, nullptr, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, rows_spec(key_type, key_off, key_len, null_field), dst_base, dst_cap, dst_total,
                   n_records, status, bad_slice);
}

int b2s_decompress_sort_rows_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                                    const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t key_type,
                                    uint32_t key_off, uint32_t key_len, int32_t null_field, uint8_t* dst_base,
                                    uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                                    int32_t* bad_slice) {
  return sort_call(t_device, true, nullptr, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, rows_spec(key_type, key_off, key_len, null_field), dst_base, dst_cap, dst_total,
                   n_records, status, bad_slice);
}

// the row sort's call with the aggregates; *dst_total is 0 when a block failed (nothing is written).  x: an exchange
// read, as for sort_call
static int aggregate_call(uint32_t dev_index, bool packed, uint32_t codec, uint32_t alg, uint32_t n,
                          const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                          const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                          const RecordSpec& spec, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
                          uint64_t* n_records, uint64_t* n_groups, int32_t* status, int32_t* bad_slice,
                          const ExchangeRead* x = nullptr) {
  if (!n_groups) {
    if (dst_total) *dst_total = 0;
    if (n_records) *n_records = 0;
    return fail(B2S_E_ARG, "null argument%s");
  }
  const int rc = sort_call(dev_index, packed, x, codec, alg, n, src_base, src_off, src_len, slice_base,
                           slice_len, slice_checksum, spec, dst_base, dst_cap, dst_total, n_records, status, bad_slice,
                           n_groups);
  if (!rc && !*n_records) *dst_total = 0;
  return rc;
}

int b2s_decompress_aggregate_rows_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                         const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                                         const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t key_type,
                                         uint32_t key_off, uint32_t key_len, int32_t null_field, uint32_t n_aggs,
                                         const uint32_t* agg_op, const uint32_t* agg_off, const int32_t* agg_null_field,
                                         uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                                         uint64_t* n_groups, int32_t* status, int32_t* bad_slice) {
  return aggregate_call(t_device, true, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                        slice_checksum,
                        aggregate_spec(key_type, key_off, key_len, null_field, n_aggs, agg_op, agg_off, agg_null_field),
                        dst_base, dst_cap, dst_total, n_records, n_groups, status, bad_slice);
}

int b2s_decompress_aggregate_rows_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                      const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                      const uint32_t* slice_base, const uint64_t* slice_len,
                                      const uint64_t* slice_checksum, uint32_t key_type, uint32_t key_off,
                                      uint32_t key_len, int32_t null_field, uint32_t n_aggs, const uint32_t* agg_op,
                                      const uint32_t* agg_off, const int32_t* agg_null_field, uint8_t* dst_base,
                                      uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_groups,
                                      int32_t* status, int32_t* bad_slice) {
  return aggregate_call(dev_index, false, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                        slice_checksum,
                        aggregate_spec(key_type, key_off, key_len, null_field, n_aggs, agg_op, agg_off, agg_null_field),
                        dst_base, dst_cap, dst_total, n_records, n_groups, status, bad_slice);
}

int b2s_decompress_sort_rows_keys_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                         const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                                         const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_keys,
                                         const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                         const int32_t* key_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                         uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                                         int32_t* bad_slice) {
  return sort_call(t_device, true, nullptr, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, keys_spec(n_keys, key_type, key_off, key_len, key_null_field), dst_base, dst_cap,
                   dst_total, n_records, status, bad_slice);
}

int b2s_decompress_sort_rows_keys_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                      const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                      const uint32_t* slice_base, const uint64_t* slice_len,
                                      const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type,
                                      const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
                                      uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                                      int32_t* status, int32_t* bad_slice) {
  return sort_call(dev_index, false, nullptr, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, keys_spec(n_keys, key_type, key_off, key_len, key_null_field), dst_base, dst_cap,
                   dst_total, n_records, status, bad_slice);
}

int b2s_decompress_aggregate_rows_keys_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                              const uint8_t* src_base, const uint64_t* src_off,
                                              const uint64_t* src_len, const uint32_t* slice_base,
                                              const uint64_t* slice_len, const uint64_t* slice_checksum,
                                              uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
                                              const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_aggs,
                                              const uint32_t* agg_op, const uint32_t* agg_off,
                                              const int32_t* agg_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                              uint64_t* dst_total, uint64_t* n_records, uint64_t* n_groups,
                                              int32_t* status, int32_t* bad_slice) {
  return aggregate_call(t_device, true, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                        slice_checksum,
                        with_aggregates(keys_spec(n_keys, key_type, key_off, key_len, key_null_field), n_aggs, agg_op,
                                        agg_off, agg_null_field),
                        dst_base, dst_cap, dst_total, n_records, n_groups, status, bad_slice);
}

int b2s_decompress_aggregate_rows_keys_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                           const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                           const uint32_t* slice_base, const uint64_t* slice_len,
                                           const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type,
                                           const uint32_t* key_off, const uint32_t* key_len,
                                           const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_op,
                                           const uint32_t* agg_off, const int32_t* agg_null_field, uint8_t* dst_base,
                                           uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
                                           uint64_t* n_groups, int32_t* status, int32_t* bad_slice) {
  return aggregate_call(dev_index, false, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                        slice_checksum,
                        with_aggregates(keys_spec(n_keys, key_type, key_off, key_len, key_null_field), n_aggs, agg_op,
                                        agg_off, agg_null_field),
                        dst_base, dst_cap, dst_total, n_records, n_groups, status, bad_slice);
}

// The join calls: the composite-key row sort's call over both sides, with the join's outputs zeroed first; every
// count and *dst_total are 0 when a block failed (nothing is written).
// ------------------------------------------------------------------------------------------------------------
// read + write, one DISTINCT group's middle stage: a reducer's (G ++ X, F) partial rows merged per (G, X) group as the
// aggregated read merges them (Spark's PartialMerge), then folded per G group (F's buffers merged, D's updated over the
// distinct column: HashAggregate(G, F: PartialMerge, D: Partial)), then hash-partitioned by G and compressed
// ------------------------------------------------------------------------------------------------------------
// The call's functions: the key columns (the first n_group_keys are G, the rest X), F as (fn, val_type) and D as
// (fn, val_type, column)
struct DistinctFns {
  uint32_t n_group_keys, n_keys;
  const uint32_t *key_type, *key_len;
  uint32_t n_aggs;
  const uint32_t *agg_fn, *val_type;
  uint32_t n_distinct;
  const uint32_t *distinct_fn, *distinct_val_type;
  const int32_t* distinct_column;
};

// What the arguments make of a call: the aggregated read's spec over the input rows (its arrays held here), the step's
// spec over the merged rows, and each output field's initial value (a global aggregate's row without input)
struct DistinctPlan {
  uint32_t key_off[kMaxKeys];
  int32_t key_nf[kMaxKeys];
  uint32_t op[kMaxAggs], off[kMaxAggs];
  int32_t nf[kMaxAggs];
  RecordSpec read;
  PartialAggSpec step;
  std::vector<int> init;  // per step buffer: 0 the value 0, 1 the value 1 (isEmpty), -1 null
};

// a key column's type agrees with a distinct function's val_type (the value the buffer reads from the column's slot)
static bool distinct_type_ok(uint32_t kt, uint32_t fn, uint32_t vt) {
  const uint32_t kind = vt & 0xff, p = (vt >> 8) & 0xff;
  switch (kt) {
    case B2S_KEY_INT8: return kind == B2S_WINDOW_VAL_INT8;
    case B2S_KEY_INT16: return kind == B2S_WINDOW_VAL_INT16;
    case B2S_KEY_INT32: return kind == B2S_WINDOW_VAL_INT32;
    case B2S_KEY_INT64: return kind == B2S_WINDOW_VAL_INT64 || (kind == B2S_WINDOW_VAL_DECIMAL && p <= 18);
    case B2S_KEY_FLOAT32: return kind == B2S_WINDOW_VAL_FLOAT32;
    case B2S_KEY_FLOAT64: return kind == B2S_WINDOW_VAL_FLOAT64;
    case kDecimalKey: return kind == B2S_WINDOW_VAL_DECIMAL && p > 18;
    default: return fn == B2S_WINDOW_COUNT && kind == B2S_WINDOW_VAL_BYTES;  // string, binary, boolean
  }
}

// the initial values of one function's buffers, in its buffers' order (Spark's initialValues)
static void distinct_inits(uint32_t fn, uint32_t vt, std::vector<int>& init) {
  const bool dec = (vt & 0xff) == B2S_WINDOW_VAL_DECIMAL;
  if (fn == B2S_WINDOW_SUM) {
    if (dec) init.insert(init.end(), {0, 1});
    else init.push_back(-1);
  } else if (fn == B2S_WINDOW_AVG) {
    init.insert(init.end(), {0, 0});
  } else if (fn == B2S_WINDOW_COUNT || fn == B2S_WINDOW_VARIANCE) {
    init.push_back(0);
  } else {
    init.push_back(-1);
  }
}

// Every rule of the call before the device (B2S_E_ARG): the key columns, F and D, the layouts' limits, and the merge
// entries over the input's buffers: each of F's buffers at its field (n_keys + its field ordinal)
static int distinct_plan(const DistinctFns& d, uint32_t num_partitions, DistinctPlan& P) {
  if (d.n_keys < 1 || d.n_keys > kMaxKeys || d.n_group_keys >= d.n_keys)
    return fail(B2S_E_ARG, "n_keys must be in [1, 16] and n_group_keys below it (at least one distinct column)%s");
  if (!d.key_type || !d.key_len) return fail(B2S_E_ARG, "null argument%s");
  if (d.n_aggs > kMaxAggs || d.n_distinct > kMaxAggs) return fail(B2S_E_ARG, "n_aggs and n_distinct must be at most 16%s");
  if ((d.n_aggs && (!d.agg_fn || !d.val_type)) ||
      (d.n_distinct && (!d.distinct_fn || !d.distinct_val_type || !d.distinct_column)))
    return fail(B2S_E_ARG, "null argument%s");
  if (!d.n_distinct) return fail(B2S_E_ARG, "n_distinct must be at least 1 (no DISTINCT function: use the "
                                            "aggregated read)%s");
  const uint32_t nk = d.n_keys;
  for (uint32_t c = 0; c < nk; c++) {
    P.key_off[c] = 8 + 8 * c;
    P.key_nf[c] = (int32_t)c;
  }
  P.read = keys_spec(nk, d.key_type, P.key_off, d.key_len, P.key_nf);
  if (int rc = key_columns_args(P.read)) return rc;
  for (uint32_t c = 0; c < nk; c++) {
    if (d.key_type[c] & ~kKeyTypeMask) return fail(B2S_E_ARG, "the key columns take no order flag%s");
    if (c < d.n_group_keys && d.key_type[c] == B2S_KEY_BYTES && d.key_len[c] != 1)
      return fail(B2S_E_ARG, "a hashed B2S_KEY_BYTES column is a boolean: key_len must be 1%s");
  }
  if (!d.n_group_keys && num_partitions != 1)
    return fail(B2S_E_ARG, "without grouping columns the exchange is SinglePartition: num_partitions must be 1%s");
  // F: its buffers as the map side lays them out, then a merge entry for each
  PartialAggSpec& st = P.step;
  st.merge = true;
  uint32_t field = nk, n_read = 0;
  for (uint32_t a = 0; a < d.n_aggs; a++) {
    PartialAggSpec f;
    const uint32_t off = 8, one_off[1] = {off};
    const int32_t one_nf[1] = {-1};
    if (int rc = partial_agg_args(1, d.agg_fn + a, d.val_type + a, one_off, one_nf, &f)) return rc;
    distinct_inits(d.agg_fn[a], d.val_type[a], P.init);
    for (uint32_t b = 0; b < f.n_bufs; b++) {
      if (st.n_bufs == kMaxAggs || n_read == kMaxAggs)
        return fail(B2S_E_ARG, "more than 16 aggregation buffers (the reduce-side merge's limit)%s");
      const uint32_t op = f.op[b], k = st.n_bufs++, slot = 8 + 8 * field;
      const bool var = op == B2S_AGG_VARIANCE;
      uint32_t vt = f.vtype[b];
      if (op == B2S_AGG_SUM_INT64) vt = B2S_WINDOW_VAL_INT64;
      else if (op == B2S_AGG_SUM_FLOAT64 || var) vt = B2S_WINDOW_VAL_FLOAT64;
      else if (op == B2S_AGG_MIN_INT32 && f.stage[b] == kStageIsEmpty) vt = B2S_WINDOW_VAL_INT32;
      else if (agg_base_op(op) == B2S_AGG_SUM_DECIMAL) vt = B2S_WINDOW_VAL_DECIMAL | agg_precision(op) << 8;
      st.op[k] = op;
      st.vtype[k] = vt;
      st.voff[k] = slot;
      st.vnull[k] = var ? -1 : (int32_t)field;
      st.stage[k] = var || agg_base_op(op) == B2S_AGG_SUM_DECIMAL ? kStageMerge : kStageValue;
      if (st.stage[k] == kStageMerge) (var ? st.n_merge_var : st.n_merge_dec)++;
      if (agg_decimal_op(op)) st.wide[k] = st.n_dec++;
      if (var) {
        st.wide[k] = st.n_dec;  // avg and m2 staged as two high words
        st.n_dec += 2;
        st.var[k] = st.n_var++;
      }
      st.dsum |= op == B2S_AGG_SUM_FLOAT64;
      st.n_fields += var ? 3 : 1;
      P.op[n_read] = op;
      P.off[n_read] = slot;
      P.nf[n_read] = var ? -1 : (int32_t)field;
      n_read++;
      field += var ? 3 : 1;
    }
  }
  if (field > 32) return fail(B2S_E_ARG, "n_keys + F's buffer fields (3 per VARIANCE) must be at most 32 (the input's "
                                         "one null word)%s");
  P.read = with_aggregates(P.read, n_read, P.op, P.off, P.nf);
  // D: each function's update over its distinct column, or count(DISTINCT every distinct column)
  uint32_t all_mask = 0;
  for (uint32_t c = d.n_group_keys; c < nk; c++) all_mask |= 1u << c;
  for (uint32_t a = 0; a < d.n_distinct; a++) {
    const uint32_t fn = d.distinct_fn[a], vt = d.distinct_val_type[a];
    const int32_t col = d.distinct_column[a];
    if (fn == B2S_WINDOW_MIN || fn == B2S_WINDOW_MAX)
      return fail(B2S_E_ARG, "MIN and MAX take no DISTINCT (Spark's optimizer drops it)%s");
    if (fn != B2S_WINDOW_SUM && fn != B2S_WINDOW_COUNT && fn != B2S_WINDOW_AVG && fn != B2S_WINDOW_VARIANCE)
      return fail(B2S_E_ARG, "a distinct function must be COUNT, SUM, AVG or VARIANCE%s");
    if (col == B2S_DISTINCT_ALL_COLUMNS) {
      if (fn != B2S_WINDOW_COUNT || vt != B2S_WINDOW_VAL_NONE)
        return fail(B2S_E_ARG, "B2S_DISTINCT_ALL_COLUMNS is count(DISTINCT every distinct column): COUNT with "
                               "B2S_WINDOW_VAL_NONE%s");
      if (st.n_bufs == kMaxAggs) return fail(B2S_E_ARG, "more than 16 aggregation buffers in the output%s");
      const uint32_t k = st.n_bufs++;
      st.op[k] = B2S_AGG_SUM_INT64;
      st.stage[k] = kStageCountAll;
      st.vtype[k] = B2S_WINDOW_VAL_NONE;
      st.voff[k] = all_mask;
      st.vnull[k] = -1;
      st.n_fields++;
      P.init.push_back(0);
      continue;
    }
    if (col < (int32_t)d.n_group_keys || col >= (int32_t)nk)
      return fail(B2S_E_ARG, "a distinct function's column must be a distinct column (in [n_group_keys, n_keys)) or "
                             "B2S_DISTINCT_ALL_COLUMNS%s");
    // one DISTINCT group: every distinct function's children are all of X, so with several X columns the only one is
    // count(DISTINCT x1, .., xn); over one of them a (G, X) row is not a distinct value of that column
    if (nk - d.n_group_keys > 1)
      return fail(B2S_E_ARG, "with several distinct columns a distinct function must take them all "
                             "(B2S_DISTINCT_ALL_COLUMNS)%s");
    if (!distinct_type_ok(d.key_type[col], fn, vt))
      return fail(B2S_E_ARG, "a distinct function's val_type does not agree with its column's key type%s");
    PartialAggSpec f;
    const uint32_t off[1] = {8 + 8 * (uint32_t)col};
    const int32_t nf[1] = {col};
    if (int rc = partial_agg_args(1, &fn, &vt, off, nf, &f)) return rc;
    distinct_inits(fn, vt, P.init);
    for (uint32_t b = 0; b < f.n_bufs; b++) {
      if (st.n_bufs == kMaxAggs) return fail(B2S_E_ARG, "more than 16 aggregation buffers in the output%s");
      const uint32_t k = st.n_bufs++, op = f.op[b];
      st.op[k] = op;
      st.stage[k] = f.stage[b];
      st.to_double[k] = f.to_double[b];
      st.vtype[k] = f.vtype[b];
      st.voff[k] = f.voff[b];
      st.vnull[k] = f.vnull[b];
      if (agg_decimal_op(op)) st.wide[k] = st.n_dec++;
      if (op == B2S_AGG_VARIANCE) st.var[k] = st.n_var++;
      st.dsum |= op == B2S_AGG_SUM_FLOAT64;
    }
    st.n_fields += f.n_fields;
  }
  if (d.n_group_keys + st.n_fields > 32)
    return fail(B2S_E_ARG, "n_group_keys + the output's buffer fields (3 per VARIANCE) must be at most 32 (one null "
                           "word)%s");
  st.keys = keys_spec(d.n_group_keys ? d.n_group_keys : 1, d.key_type, P.key_off, d.key_len, P.key_nf).keys;
  st.keys.n = d.n_group_keys;
  return 0;
}

// A global aggregate's one output row without input: HashAggregateExec's outputForEmptyGroupingKeyWithoutInput, the
// initial buffers as UnsafeProjection writes them ([size: int32 big-endian][row])
static std::vector<uint8_t> initial_row(const DistinctPlan& P) {
  const PartialAggSpec& st = P.step;
  const uint32_t nf = st.n_fields, fixed = 8 * (1 + nf);
  uint32_t wide = 0;
  for (uint32_t k = 0; k < st.n_bufs; k++) wide += agg_decimal_wide(st.op[k]) ? 1 : 0;
  std::vector<uint8_t> rec(4 + fixed + 16 * wide, 0);
  uint8_t* row = rec.data() + 4;
  uint64_t nulls = 0;
  uint32_t f = 0, var_at = fixed;
  for (uint32_t k = 0; k < st.n_bufs; k++) {
    const uint32_t op = st.op[k];
    uint64_t slot = P.init[k] > 0 ? 1 : 0;
    if (agg_decimal_wide(op)) {  // 16 bytes; 0 is BigInteger.toByteArray's one byte 00
      slot = ((uint64_t)var_at << 32) | (P.init[k] < 0 ? 0 : 1);
      var_at += 16;
    }
    if (P.init[k] < 0) nulls |= 1ull << f;
    memcpy(row + 8 + 8 * f, &slot, 8);
    f += op == B2S_AGG_VARIANCE ? 3 : 1;  // a variance's (0.0, 0.0, 0.0)
  }
  memcpy(row, &nulls, 8);
  const uint32_t size = (uint32_t)rec.size() - 4;
  for (int b = 0; b < 4; b++) rec[b] = (uint8_t)(size >> (24 - 8 * b));
  return rec;
}

// The whole call on the read lane's slot 0: decode, the aggregated read's order and merge by G ++ X (the merged rows
// into S.parena, their lengths in S.pws), the step over them in S.fws (no sort: heads where G's encoding changes) into
// S.aggrows, and the partition + compress step.  No step ensures a buffer that holds its own input: the partition step
// ensures S.pws, S.parena and (packed) S.dst, which hold only stage 2's inputs and outputs by then.
static int distinct_task_run(Device* D, const MapCall& c, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
                             const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
                             const uint64_t* slice_checksum, const DistinctPlan& P, uint64_t* counts, int32_t* status,
                             int32_t* bad_slice, const WallTimer& wt) {
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  const SortBufferTrim trim{S};
  const PartialAggTrim trim_step{S};
  cudaStream_t st = S.st;
  std::vector<uint64_t> dev_off;
  const uint8_t* blocks;
  const uint64_t* block_off;
  uint64_t srcb;
  int rc = task_blocks(S, c.packed, n, src_base, src_off, src_len, dev_off, &blocks, &block_off, &srcb);
  if (rc) return rc;
  uint64_t launches = 0;
  const RecordSpec& spec = P.read;
  const PartialAggSpec& step = P.step;
  DecodedTask T(nullptr, n, status, bad_slice);
  RowOrder R;
  if (n) {  // no blocks: an empty reducer, straight to the step
    rc = decode_task(D, S, c.codec, c.alg, n, blocks, block_off, src_len, c.packed, slice_base, slice_len,
                     slice_checksum, srcb, spec, ~0ull, T, &launches);
    if (rc) return rc;
    if (!T.failed) rc = order_rows(S, spec, T, nullptr, 0, R, &launches);
    if (rc) return rc;
  }
  // stage 2: the (G, X) groups merged into S.parena
  uint64_t merged_bytes = 0, n_in = 0, n_gx = 0;
  if (n && !T.failed) {
    if ((rc = S.parena.ensure(T.total + 64))) return rc;
    rc = aggregate_rows_tail(S, spec, T, R, (uint8_t*)S.parena.p, T.total, &merged_bytes, &n_in, &n_gx, &launches);
    if (rc) return rc;
  }
  if (T.failed) {  // nothing is written
    for (uint32_t p = 0; p < c.R; p++) {
      c.dst_off[p] = c.dst_len[p] = 0;
      if (c.checksum_out) c.checksum_out[p] = 0;
      c.status[p] = B2S_OK;
    }
    return 0;
  }
  const double read_ms = S.span(K0, G1);
  // stage 3 over the n_gx merged rows: offsets, G's heads, grouping, folds (one readback: rows, bytes), emit
  const uint8_t* merged = (const uint8_t*)S.parena.p;
  const uint32_t key_bytes = rows_key_bytes(step.keys);
  const size_t part[4] = {rows_sort_ws_bytes(n_gx, key_bytes), 256 + align_up(n_gx * 4, 256),
                          rows_aggregate_ws_bytes(n_gx, 0, 0), partial_agg_ws_bytes(n_gx, step)};
  if ((rc = S.fws.ensure(part[0] + part[1] + part[2] + part[3]))) return rc;
  uint8_t* ws = (uint8_t*)S.fws.p;
  uint32_t* heads = (uint32_t*)(ws + part[0] + 256);
  uint8_t *gws = ws + part[0] + part[1], *paws = gws + part[2];
  if ((rc = S.hmeta.ensure(48))) return rc;
  uint64_t* rb = (uint64_t*)S.hmeta.p;
  CU(S.mark(G0, st, launches));
  launch_partial_agg_offsets(rows_group_lengths(R.aws, R.records), n_gx, key_bytes, ws, paws, st, &launches);
  uint64_t rows = 0, rows_bytes = 0;
  const uint32_t* d_row_len = partial_agg_row_len(paws, n_gx, step);
  if (n_gx) {
    launch_partial_agg_heads(merged, n_gx, key_bytes, step.keys, ws, heads, st, &launches);
    launch_rows_group(merged, n_gx, nullptr, heads, key_bytes, AggSpec{}, ws, gws, st, &launches);
    launch_partial_agg_fold(merged, n_gx, nullptr, key_bytes, step, ws, gws, paws, st, &launches);
    CU(cudaMemcpyAsync(rb, partial_agg_header(paws) + 4, 16, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    rows = rb[0];
    rows_bytes = rb[1];
    if ((rc = S.aggrows.ensure(rows_bytes + 64))) return rc;
    launch_partial_agg_emit(merged, n_gx, rows, nullptr, key_bytes, step, ws, gws, paws, (uint8_t*)S.aggrows.p, st,
                            &launches);
  } else if (!step.keys.n) {  // a global aggregate without input: its initial row
    const std::vector<uint8_t> row = initial_row(P);
    const uint32_t len = (uint32_t)row.size();
    rows = 1;
    rows_bytes = len;
    if ((rc = S.aggrows.ensure(256 + len + 64))) return rc;
    CU(cudaMemcpyAsync((uint8_t*)S.aggrows.p + 256, row.data(), len, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(S.aggrows.p, &len, 4, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    d_row_len = (const uint32_t*)S.aggrows.p;
  }
  CU(S.mark(G1, st, launches));
  const uint8_t* d_rows = (const uint8_t*)S.aggrows.p + (n_gx || !rows ? 0 : 256);
  const KeySpec keys = partial_row_keys(step.keys);
  const RowIds ids = step.keys.n ? RowIds::hash(keys) : RowIds::single_partition(keys);
  uint64_t arena = 0, fit = 0;
  rc = partition_tail(D, S, c, MapRows{rows, d_rows, rows_bytes, d_row_len}, nullptr, ids, nullptr, &arena, &fit,
                      &launches);
  if (rc && rc != B2S_E_DST_TOO_SMALL) return rc;
  counts[0] = n_in;
  counts[1] = n_gx;
  counts[2] = rows;
  t_timing.kernel_ms += read_ms;
  end_call(wt, launches, CallBytes{srcb, arena, c.packed ? srcb : 0, fit}, &S, Family::kPartialAggregate);
  return rc;
}

// b2s_decompress_aggregate_distinct_partition_compress_rows_hash_*: zero the outputs, every check before the device,
// then the device (B2S_E_CUDA without one) and the run
static int distinct_call(bool packed, uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                         uint32_t alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
                         const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
                         const uint64_t* slice_checksum, const DistinctFns& fns, uint32_t num_partitions,
                         uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                         uint64_t* dst_total, uint64_t* checksum_out, int32_t* part_status, uint64_t* counts,
                         int32_t* status, int32_t* bad_slice) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  if (counts) counts[0] = counts[1] = counts[2] = 0;
  if (!counts || !dst_total) return fail(B2S_E_ARG, "null argument%s");
  DistinctPlan P;
  if (int rc = distinct_plan(fns, num_partitions, P)) return rc;
  uint64_t unused_total = 0, unused_records = 0;
  if (int rc = sort_args(codec, alg, n, src_off, src_len, slice_base, slice_len, slice_checksum, P.read, src_base,
                         nullptr, 0, &unused_total, &unused_records, status))
    return rc;
  const MapCall c{packed, dev_index, codec, level, block_size_or_default(codec_block_size), alg, num_partitions,
                  dst_base, dst_cap, dst_off, dst_len, dst_total, checksum_out, part_status};
  if (int rc = partition_args(c, MapRows{}, nullptr, RowIds::hash(P.step.keys))) return rc;
  if (dst_cap && !dst_base) return fail(B2S_E_ARG, "null argument%s");
  Device* D;
  if (int rc = sort_device(packed ? t_device : dev_index, &D)) return rc;
  return distinct_task_run(D, c, n, src_base, src_off, src_len, slice_base, slice_len, slice_checksum, P, counts,
                           status, bad_slice, wt);
}

int b2s_decompress_aggregate_distinct_partition_compress_rows_hash_packed(
    uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t n,
    const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
    const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_group_keys, uint32_t n_keys,
    const uint32_t* key_type, const uint32_t* key_len, uint32_t n_aggs, const uint32_t* agg_fn,
    const uint32_t* val_type, uint32_t n_distinct, const uint32_t* distinct_fn, const uint32_t* distinct_val_type,
    const int32_t* distinct_column, uint32_t num_partitions, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
    uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* part_status, uint64_t* counts,
    int32_t* status, int32_t* bad_slice) {
  const DistinctFns fns{n_group_keys, n_keys, key_type, key_len, n_aggs, agg_fn, val_type,
                        n_distinct, distinct_fn, distinct_val_type, distinct_column};
  return distinct_call(true, 0, codec, level, codec_block_size, checksum_alg, n, src_base, src_off, src_len,
                       slice_base, slice_len, slice_checksum, fns, num_partitions, dst_base, dst_cap, dst_off,
                       dst_len, dst_total, checksum_out, part_status, counts, status, bad_slice);
}

int b2s_decompress_aggregate_distinct_partition_compress_rows_hash_dev(
    uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg, uint32_t n,
    const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
    const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_group_keys, uint32_t n_keys,
    const uint32_t* key_type, const uint32_t* key_len, uint32_t n_aggs, const uint32_t* agg_fn,
    const uint32_t* val_type, uint32_t n_distinct, const uint32_t* distinct_fn, const uint32_t* distinct_val_type,
    const int32_t* distinct_column, uint32_t num_partitions, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
    uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* part_status, uint64_t* counts,
    int32_t* status, int32_t* bad_slice) {
  const DistinctFns fns{n_group_keys, n_keys, key_type, key_len, n_aggs, agg_fn, val_type,
                        n_distinct, distinct_fn, distinct_val_type, distinct_column};
  return distinct_call(false, dev_index, codec, level, codec_block_size, checksum_alg, n, src_base, src_off, src_len,
                       slice_base, slice_len, slice_checksum, fns, num_partitions, dst_base, dst_cap, dst_off,
                       dst_len, dst_total, checksum_out, part_status, counts, status, bad_slice);
}

static int join_call(uint32_t dev_index, bool packed, uint32_t join_type, uint32_t codec, uint32_t alg,
                     uint32_t n_left, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
                     const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
                     const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_len,
                     const uint32_t* left_key_off, const int32_t* left_key_null_field, const uint32_t* right_key_off,
                     const int32_t* right_key_null_field, uint32_t n_left_fields, const uint8_t* left_field_kind,
                     uint32_t n_right_fields, const uint8_t* right_field_kind, uint8_t* dst_base, uint64_t dst_cap,
                     uint64_t* dst_total, uint64_t* n_left_records, uint64_t* n_right_records,
                     uint64_t* n_out_records, int32_t* status, int32_t* bad_slice) {
  if (n_left_records) *n_left_records = 0;
  if (n_right_records) *n_right_records = 0;
  JoinSpec js;
  js.type = join_type;
  js.n_left = n_left;
  const RecordSpec right = keys_spec(n_keys, key_type, right_key_off, key_len, right_key_null_field);
  js.right = right.keys;
  js.right_arrays = right.key_arrays;
  js.n_fields[0] = n_left_fields;
  js.n_fields[1] = n_right_fields;
  js.kind[0] = left_field_kind;
  js.kind[1] = right_field_kind;
  js.n_side[0] = n_left_records;
  js.n_side[1] = n_right_records;
  RecordSpec spec = keys_spec(n_keys, key_type, left_key_off, key_len, left_key_null_field);
  spec.null_safe = true;
  spec.join = &js;
  const int rc = sort_call(dev_index, packed, nullptr, codec, alg, n, src_base, src_off, src_len, slice_base, slice_len,
                           slice_checksum, spec, dst_base, dst_cap, dst_total, n_out_records, status, bad_slice);
  if (!rc && !*n_out_records) *dst_total = 0;
  return rc;
}

int b2s_decompress_join_rows_keys_packed(
    uint32_t join_type, uint32_t codec, uint32_t checksum_alg, uint32_t n_left, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_len,
    const uint32_t* left_key_off, const int32_t* left_key_null_field, const uint32_t* right_key_off,
    const int32_t* right_key_null_field, uint32_t n_left_fields, const uint8_t* left_field_kind,
    uint32_t n_right_fields, const uint8_t* right_field_kind, uint8_t* dst_base, uint64_t dst_cap,
    uint64_t* dst_total, uint64_t* n_left_records, uint64_t* n_right_records, uint64_t* n_out_records, int32_t* status,
    int32_t* bad_slice) {
  return join_call(t_device, true, join_type, codec, checksum_alg, n_left, n, src_base, src_off, src_len, slice_base,
                   slice_len, slice_checksum, n_keys, key_type, key_len, left_key_off, left_key_null_field,
                   right_key_off, right_key_null_field, n_left_fields, left_field_kind, n_right_fields,
                   right_field_kind, dst_base, dst_cap, dst_total, n_left_records, n_right_records, n_out_records,
                   status, bad_slice);
}

int b2s_decompress_join_rows_keys_dev(
    uint32_t dev_index, uint32_t join_type, uint32_t codec, uint32_t checksum_alg, uint32_t n_left, uint32_t n,
    const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
    const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_len, const uint32_t* left_key_off, const int32_t* left_key_null_field,
    const uint32_t* right_key_off, const int32_t* right_key_null_field, uint32_t n_left_fields,
    const uint8_t* left_field_kind, uint32_t n_right_fields, const uint8_t* right_field_kind, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_left_records, uint64_t* n_right_records,
    uint64_t* n_out_records, int32_t* status, int32_t* bad_slice) {
  return join_call(dev_index, false, join_type, codec, checksum_alg, n_left, n, src_base, src_off, src_len, slice_base,
                   slice_len, slice_checksum, n_keys, key_type, key_len, left_key_off, left_key_null_field,
                   right_key_off, right_key_null_field, n_left_fields, left_field_kind, n_right_fields,
                   right_field_kind, dst_base, dst_cap, dst_total, n_left_records, n_right_records, n_out_records,
                   status, bad_slice);
}

// The window calls: the composite-key row sort's call with the window's arguments ws (its n_in the input count, zeroed
// first); every count and *dst_total are 0 when a block failed (nothing is written).  The aggregate and offset calls
// check their functions before the device.
static int window_call(uint32_t dev_index, bool packed, uint32_t codec, uint32_t alg, uint32_t n,
                       const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                       const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                       uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                       const int32_t* key_null_field, WindowSpec& ws, uint8_t* dst_base, uint64_t dst_cap,
                       uint64_t* dst_total, uint64_t* n_out_records, int32_t* status, int32_t* bad_slice) {
  if (ws.n_in) *ws.n_in = 0;
  if (ws.agg) {
    if (dst_total) *dst_total = 0;
    if (n_out_records) *n_out_records = 0;
    if (int rc = ws.frames   ? window_frame_fn_args(ws, n_keys, key_type)
                 : ws.offset ? window_offset_fn_args(ws)
                             : window_agg_fn_args(ws)) {
      begin_call();  // a new call, with an empty b2s_last_timing
      return rc;
    }
  }
  RecordSpec spec = keys_spec(n_keys, key_type, key_off, key_len, key_null_field);
  spec.window = &ws;
  const int rc = sort_call(dev_index, packed, nullptr, codec, alg, n, src_base, src_off, src_len, slice_base, slice_len,
                           slice_checksum, spec, dst_base, dst_cap, dst_total, n_out_records, status, bad_slice);
  if (!rc && !*n_out_records) *dst_total = 0;
  return rc;
}

static WindowSpec window_ranking_spec(uint32_t n_partition_keys, uint32_t n_fields, const uint8_t* field_kind,
                                      uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, uint32_t limit_fn,
                                      int32_t limit, uint64_t* n_records) {
  WindowSpec ws;
  ws.n_partition_keys = n_partition_keys;
  ws.n_fields = n_fields;
  ws.kind = field_kind;
  ws.n_fns = n_fns;
  ws.fn = fn;
  ws.fn_arg = fn_arg;
  ws.limit_fn = limit_fn;
  ws.limit = limit;
  ws.n_in = n_records;
  return ws;
}

static WindowSpec window_aggregate_spec(uint32_t n_partition_keys, uint32_t n_fields, const uint8_t* field_kind,
                                        uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg,
                                        const uint32_t* fn_frame, const uint32_t* val_type, const uint32_t* val_off,
                                        const int32_t* val_null_field, uint64_t* n_records) {
  WindowSpec ws = window_ranking_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, B2S_WINDOW_NO_LIMIT,
                                      0, n_records);
  ws.agg = true;
  ws.frame = fn_frame;
  ws.val_type = val_type;
  ws.val_off = val_off;
  ws.val_null = val_null_field;
  return ws;
}

static WindowSpec window_offset_spec(uint32_t n_partition_keys, uint32_t n_fields, const uint8_t* field_kind,
                                     uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame,
                                     const uint32_t* val_type, const uint32_t* val_off, const int32_t* val_null_field,
                                     const uint32_t* fn_flags, const uint64_t* fn_default, uint64_t* n_records) {
  WindowSpec ws = window_aggregate_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, fn_frame, val_type,
                                        val_off, val_null_field, n_records);
  ws.offset = true;
  ws.flags = fn_flags;
  ws.dflt = fn_default;
  return ws;
}

int b2s_decompress_window_rows_keys_packed(
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, uint32_t limit_fn, int32_t limit,
    uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_out_records,
    int32_t* status, int32_t* bad_slice) {
  WindowSpec ws =
      window_ranking_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, limit_fn, limit, n_records);
  return window_call(t_device, true, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                     slice_checksum, n_keys, key_type, key_off, key_len, key_null_field, ws, dst_base, dst_cap,
                     dst_total, n_out_records, status, bad_slice);
}

int b2s_decompress_window_rows_keys_dev(
    uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields,
    const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, uint32_t limit_fn,
    int32_t limit, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
    uint64_t* n_out_records, int32_t* status, int32_t* bad_slice) {
  WindowSpec ws =
      window_ranking_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, limit_fn, limit, n_records);
  return window_call(dev_index, false, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                     slice_checksum, n_keys, key_type, key_off, key_len, key_null_field, ws, dst_base, dst_cap,
                     dst_total, n_out_records, status, bad_slice);
}

int b2s_decompress_window_aggregate_rows_keys_packed(
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
    uint64_t* n_records, uint64_t* n_out_records, int32_t* status, int32_t* bad_slice) {
  WindowSpec ws = window_aggregate_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, fn_frame,
                                        val_type, val_off, val_null_field, n_records);
  return window_call(t_device, true, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                     slice_checksum, n_keys, key_type, key_off, key_len, key_null_field, ws, dst_base, dst_cap,
                     dst_total, n_out_records, status, bad_slice);
}

int b2s_decompress_window_aggregate_rows_keys_dev(
    uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields,
    const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame,
    const uint32_t* val_type, const uint32_t* val_off, const int32_t* val_null_field, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_out_records, int32_t* status,
    int32_t* bad_slice) {
  WindowSpec ws = window_aggregate_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, fn_frame,
                                        val_type, val_off, val_null_field, n_records);
  return window_call(dev_index, false, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                     slice_checksum, n_keys, key_type, key_off, key_len, key_null_field, ws, dst_base, dst_cap,
                     dst_total, n_out_records, status, bad_slice);
}

int b2s_decompress_window_offset_rows_keys_packed(
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, const uint32_t* fn_flags, const uint64_t* fn_default,
    uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_out_records,
    int32_t* status, int32_t* bad_slice) {
  WindowSpec ws = window_offset_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, fn_frame, val_type,
                                     val_off, val_null_field, fn_flags, fn_default, n_records);
  return window_call(t_device, true, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                     slice_checksum, n_keys, key_type, key_off, key_len, key_null_field, ws, dst_base, dst_cap,
                     dst_total, n_out_records, status, bad_slice);
}

int b2s_decompress_window_offset_rows_keys_dev(
    uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields,
    const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame,
    const uint32_t* val_type, const uint32_t* val_off, const int32_t* val_null_field, const uint32_t* fn_flags,
    const uint64_t* fn_default, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
    uint64_t* n_out_records, int32_t* status, int32_t* bad_slice) {
  WindowSpec ws = window_offset_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, fn_frame, val_type,
                                     val_off, val_null_field, fn_flags, fn_default, n_records);
  return window_call(dev_index, false, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                     slice_checksum, n_keys, key_type, key_off, key_len, key_null_field, ws, dst_base, dst_cap,
                     dst_total, n_out_records, status, bad_slice);
}

static WindowSpec window_frame_spec(uint32_t n_partition_keys, uint32_t n_fields, const uint8_t* field_kind,
                                    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame,
                                    const uint32_t* val_type, const uint32_t* val_off, const int32_t* val_null_field,
                                    const uint32_t* fn_flags, const uint64_t* fn_default, const int64_t* frame_lower,
                                    const int64_t* frame_upper, uint64_t* n_records) {
  WindowSpec ws = window_offset_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, fn_frame, val_type,
                                     val_off, val_null_field, fn_flags, fn_default, n_records);
  ws.frames = true;
  ws.lower = frame_lower;
  ws.upper = frame_upper;
  return ws;
}

int b2s_decompress_window_frame_rows_keys_packed(
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
    uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame, const uint32_t* val_type,
    const uint32_t* val_off, const int32_t* val_null_field, const uint32_t* fn_flags, const uint64_t* fn_default,
    const int64_t* frame_lower, const int64_t* frame_upper, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
    uint64_t* n_records, uint64_t* n_out_records, int32_t* status, int32_t* bad_slice) {
  WindowSpec ws = window_frame_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, fn_frame, val_type,
                                    val_off, val_null_field, fn_flags, fn_default, frame_lower, frame_upper, n_records);
  return window_call(t_device, true, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                     slice_checksum, n_keys, key_type, key_off, key_len, key_null_field, ws, dst_base, dst_cap,
                     dst_total, n_out_records, status, bad_slice);
}

int b2s_decompress_window_frame_rows_keys_dev(
    uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
    const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_fields,
    const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg, const uint32_t* fn_frame,
    const uint32_t* val_type, const uint32_t* val_off, const int32_t* val_null_field, const uint32_t* fn_flags,
    const uint64_t* fn_default, const int64_t* frame_lower, const int64_t* frame_upper, uint8_t* dst_base,
    uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, uint64_t* n_out_records, int32_t* status,
    int32_t* bad_slice) {
  WindowSpec ws = window_frame_spec(n_partition_keys, n_fields, field_kind, n_fns, fn, fn_arg, fn_frame, val_type,
                                    val_off, val_null_field, fn_flags, fn_default, frame_lower, frame_upper, n_records);
  return window_call(dev_index, false, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                     slice_checksum, n_keys, key_type, key_off, key_len, key_null_field, ws, dst_base, dst_cap,
                     dst_total, n_out_records, status, bad_slice);
}

// ------------------------------------------------------------------------------------------------------------
// exchange cache calls
// ------------------------------------------------------------------------------------------------------------
int b2s_exchange_set_budget(uint32_t dev_index, uint64_t bytes) {
  int rc = exchange_ready();
  if (rc) return rc;
  Device* D;
  if ((rc = get_device(dev_index, &D))) return rc;
  std::vector<ExEntry*> dead;
  {
    std::lock_guard<std::mutex> lk(g_ex.mtx);
    g_ex.budget[D->ordinal] = bytes;
    ex_make_room(D->ordinal, 0, dead, true);
    if (!bytes)  // off: every entry goes, a referenced one when its reader is done
      for (auto it = g_ex.by_key.begin(); it != g_ex.by_key.end();) {
        ExEntry* e = (it++)->second;
        if (e->ordinal == D->ordinal) ex_unlink(e, dead);
      }
  }
  ex_free(dead);
  return 0;
}

int b2s_exchange_remove(int32_t shuffle_id, int64_t map_id) {
  int rc = exchange_ready();
  if (rc) return rc;
  std::vector<ExEntry*> dead;
  int removed = 0;
  {
    std::lock_guard<std::mutex> lk(g_ex.mtx);
    for (auto it = g_ex.by_key.begin(); it != g_ex.by_key.end();) {
      ExEntry* e = (it++)->second;
      if (e->shuffle == shuffle_id && (map_id == -1 || e->map == map_id)) {
        ex_unlink(e, dead);  // a referenced entry is freed by its last reader
        removed++;
      }
    }
  }
  ex_free(dead);
  return removed;
}

int b2s_exchange_lookup(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, uint32_t n_maps,
                        const int64_t* map_ids, uint64_t* len) {
  int rc = reduce_range_args(start_reduce, end_reduce);
  if (rc) return rc;
  if (n_maps && (!map_ids || !len)) return fail(B2S_E_ARG, "null argument%s");
  if ((rc = exchange_ready())) return rc;
  Device* D;
  if ((rc = get_device(t_device, &D))) return rc;
  std::lock_guard<std::mutex> lk(g_ex.mtx);
  int hits = 0;
  for (uint32_t i = 0; i < n_maps; i++) {
    len[i] = UINT64_MAX;
    auto it = g_ex.by_key.find({shuffle_id, map_ids[i]});
    if (it == g_ex.by_key.end() || it->second->ordinal != D->ordinal) continue;
    const std::vector<uint64_t>& ps = it->second->part_start;
    if ((uint64_t)end_reduce + 1 > ps.size())
      return fail(B2S_E_ARG, "end_reduce exceeds the partitions of a cached map output%s");
    len[i] = ps[(size_t)end_reduce] - ps[(size_t)start_reduce];
    hits++;
  }
  return hits;
}

int b2s_exchange_read_packed(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, uint32_t n_maps,
                             const int64_t* map_ids, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                             uint64_t* dst_len, uint64_t* dst_total, int32_t* status) {
  const WallTimer wt = begin_call();
  if (dst_total) *dst_total = 0;
  int rc = reduce_range_args(start_reduce, end_reduce);
  if (rc) return rc;
  if (!dst_total || (n_maps && (!map_ids || !dst_off || !dst_len || !status)) || (dst_cap && !dst_base))
    return fail(B2S_E_ARG, "null argument%s");
  if ((rc = exchange_ready())) return rc;
  Device* D;
  if ((rc = get_device(t_device, &D))) return rc;
  ExRefs refs(D->ordinal, shuffle_id, n_maps, map_ids, nullptr);
  if ((rc = refs.check_range(end_reduce))) return rc;
  std::vector<ExchangePiece> pieces;
  uint64_t total = 0;
  for (uint32_t i = 0; i < n_maps; i++) {
    uint64_t len = 0;
    if (refs.entry[i]) {
      const uint8_t* src = refs.range(i, start_reduce, end_reduce, &len);
      exchange_add_pieces(pieces, src, total, len);
    }
    status[i] = refs.entry[i] ? B2S_OK : B2S_E_NOT_CACHED;
    dst_off[i] = total;
    dst_len[i] = len;
    total += len;
  }
  *dst_total = total;
  if (total > dst_cap) return fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s cached bytes", std::to_string(total).c_str());
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  SortBufferTrim trim{S};
  cudaStream_t st = S.st;
  uint64_t launches = 0;
  if ((rc = S.dst.ensure(total + 64)) || (rc = S.xpieces.ensure(pieces.size() * sizeof(ExchangePiece) + 64)))
    return rc;
  CU(S.mark(K0, st));
  CU(S.mark(T0, st));
  if (!pieces.empty()) {
    CU(cudaMemcpyAsync(S.xpieces.p, pieces.data(), pieces.size() * sizeof(ExchangePiece), cudaMemcpyHostToDevice, st));
    launch_exchange_gather((const ExchangePiece*)S.xpieces.p, (uint32_t)pieces.size(), (uint8_t*)S.dst.p, st,
                           &launches);
  }
  CU(S.mark(T1, st));
  CU(S.mark(K1, st));
  CU(S.mark(D0, st));
  if (total) CU(cudaMemcpyAsync(dst_base, S.dst.p, total, cudaMemcpyDeviceToHost, st));
  CU(S.mark(D1, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  end_call(wt, launches, CallBytes{total, total, 0, total}, &S);
  return 0;
}

int b2s_exchange_read_sort_packed(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids,
                                  const uint8_t* cached, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                  const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                  const uint32_t* slice_base, const uint64_t* slice_len,
                                  const uint64_t* slice_checksum, uint32_t record_bytes, uint32_t key_off,
                                  uint32_t key_len, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
                                  uint64_t* n_records, int32_t* status, int32_t* bad_slice) {
  const ExchangeRead x{shuffle_id, start_reduce, end_reduce, map_ids, cached};
  return sort_call(t_device, true, &x, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, fixed_spec(record_bytes, key_off, key_len), dst_base, dst_cap, dst_total, n_records,
                   status, bad_slice);
}

int b2s_exchange_read_sort_dev(uint32_t dev_index, int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce,
                               const int64_t* map_ids, const uint8_t* cached, uint32_t codec, uint32_t checksum_alg,
                               uint32_t n, const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                               const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                               uint32_t record_bytes, uint32_t key_off, uint32_t key_len, uint8_t* dst_base,
                               uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                               int32_t* bad_slice) {
  const ExchangeRead x{shuffle_id, start_reduce, end_reduce, map_ids, cached};
  return sort_call(dev_index, false, &x, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, fixed_spec(record_bytes, key_off, key_len), dst_base, dst_cap, dst_total, n_records,
                   status, bad_slice);
}

int b2s_decompressed_size_batch(uint32_t codec, uint32_t n, const uint8_t* const* src, const uint64_t* src_len,
                                uint64_t* out_len, int32_t* status) {
  if (n && (!src || !src_len || !out_len || !status)) return fail(B2S_E_ARG, "null argument%s");
  return decompress_host(codec, 0, n, src, src_len, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr,
                         out_len, nullptr, status, nullptr, true);
}

// ------------------------------------------------------------------------------------------------------------
// exchange cache, rows: the composite-key row sort and aggregation over cached and fetched sources
// ------------------------------------------------------------------------------------------------------------
int b2s_exchange_read_sort_rows_keys_packed(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce,
                                            const int64_t* map_ids, const uint8_t* cached, uint32_t codec,
                                            uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                            const uint64_t* src_off, const uint64_t* src_len,
                                            const uint32_t* slice_base, const uint64_t* slice_len,
                                            const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type,
                                            const uint32_t* key_off, const uint32_t* key_len,
                                            const int32_t* key_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                            uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                                            int32_t* bad_slice) {
  const ExchangeRead x{shuffle_id, start_reduce, end_reduce, map_ids, cached};
  return sort_call(t_device, true, &x, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, keys_spec(n_keys, key_type, key_off, key_len, key_null_field), dst_base, dst_cap,
                   dst_total, n_records, status, bad_slice);
}

int b2s_exchange_read_sort_rows_keys_dev(uint32_t dev_index, int32_t shuffle_id, int32_t start_reduce,
                                         int32_t end_reduce, const int64_t* map_ids, const uint8_t* cached,
                                         uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                                         const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                                         const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t n_keys,
                                         const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                         const int32_t* key_null_field, uint8_t* dst_base, uint64_t dst_cap,
                                         uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                                         int32_t* bad_slice) {
  const ExchangeRead x{shuffle_id, start_reduce, end_reduce, map_ids, cached};
  return sort_call(dev_index, false, &x, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                   slice_checksum, keys_spec(n_keys, key_type, key_off, key_len, key_null_field), dst_base, dst_cap,
                   dst_total, n_records, status, bad_slice);
}

int b2s_exchange_read_aggregate_rows_keys_packed(
    int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids, const uint8_t* cached,
    uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base, const uint64_t* src_off,
    const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
    uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
    const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_op, const uint32_t* agg_off,
    const int32_t* agg_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records,
    uint64_t* n_groups, int32_t* status, int32_t* bad_slice) {
  const ExchangeRead x{shuffle_id, start_reduce, end_reduce, map_ids, cached};
  return aggregate_call(t_device, true, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                        slice_checksum,
                        with_aggregates(keys_spec(n_keys, key_type, key_off, key_len, key_null_field), n_aggs, agg_op,
                                        agg_off, agg_null_field),
                        dst_base, dst_cap, dst_total, n_records, n_groups, status, bad_slice, &x);
}

int b2s_exchange_read_aggregate_rows_keys_dev(
    uint32_t dev_index, int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids,
    const uint8_t* cached, uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
    const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
    const uint64_t* slice_checksum, uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_off,
    const uint32_t* key_len, const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_op,
    const uint32_t* agg_off, const int32_t* agg_null_field, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
    uint64_t* n_records, uint64_t* n_groups, int32_t* status, int32_t* bad_slice) {
  const ExchangeRead x{shuffle_id, start_reduce, end_reduce, map_ids, cached};
  return aggregate_call(dev_index, false, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len,
                        slice_checksum,
                        with_aggregates(keys_spec(n_keys, key_type, key_off, key_len, key_null_field), n_aggs, agg_op,
                                        agg_off, agg_null_field),
                        dst_base, dst_cap, dst_total, n_records, n_groups, status, bad_slice, &x);
}

}  // extern "C"
