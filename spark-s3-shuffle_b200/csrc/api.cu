// api.cu — runtime + C ABI of libb200shuffle.so (see include/b200shuffle.h for the contract and the reference
// interfaces each entry point replaces).
//
// Structure: a process-wide context with one Device per selected GPU.  A Device owns NSLOT pipeline slots; a slot is
// a CUDA stream plus grow-only device buffers (staged source/destination arenas, descriptor "meta" block, codec
// scratch) and a pinned host block for descriptor traffic.  Host-pointer entry points cut a batch into chunks of
// ~64 MiB, and run H2D -> kernels -> (size readback) -> D2H per chunk on rotating slots so copies of one chunk
// overlap kernels of another.  "_dev" entry points run the same kernel sequence on caller-owned device arenas.
// There is no CPU fallback anywhere in this file: without a device every compute entry point fails with B2S_E_CUDA.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "kernels.h"

using namespace b2s;

namespace {

thread_local std::string t_last_error;
thread_local b2s_timing t_timing;
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
uint32_t g_lz4d_chunk_blocks = 65536;  // decode side: the token walk is latency bound, more blocks per launch = more loads in flight; B2S_LZ4D_CHUNK_BLOCKS
int g_lz4d_legacy = 0;
int g_trace = 0;  // B2S_TRACE=1: per-chunk timeline of the compress pipeline on stderr  // B2S_LZ4D_LEGACY=1: single-kernel tile decoder for every block size (A/B comparisons)

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int g_read_priority = 1;       // B2S_READ_PRIORITY=0: both lanes at the default stream priority
int g_read_lag = 1;            // B2S_READ_LAG: chunks between the stages of the read pipeline (upload+sizes | decode | download)
int g_overlap = 1;             // B2S_OVERLAP=0: match / token kernels on the main stream (no two-stream overlap); A/B runs
uint64_t g_copy_piece = 0;     // B2S_COPY_PIECE_MB: host<->device payload copies are issued in pieces of this size so the
                               // copy engines interleave the two lanes' transfers instead of draining one lane's queue
cudaError_t copy_async(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st) {
  if (!g_copy_piece || bytes <= g_copy_piece) return cudaMemcpyAsync(dst, src, bytes, kind, st);
  for (size_t at = 0; at < bytes; at += g_copy_piece) {
    const size_t k = std::min<size_t>(g_copy_piece, bytes - at);
    cudaError_t e = cudaMemcpyAsync((uint8_t*)dst + at, (const uint8_t*)src + at, k, kind, st);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

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

struct Slot {
  cudaStream_t st = nullptr;
  cudaStream_t st2 = nullptr;                               // side stream: match kernels of chunk k+1 overlap parse/emit of chunk k
  cudaEvent_t ev_fork = nullptr, ev_match[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;              // readback milestones
  cudaEvent_t ev_k0 = nullptr, ev_k1 = nullptr;            // kernel region
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;            // dominant kernel
  cudaEvent_t ev_h0 = nullptr, ev_h1 = nullptr, ev_d0 = nullptr, ev_d1 = nullptr;  // copies
  cudaEvent_t ev_p0 = nullptr, ev_p1 = nullptr;            // partition step (b2s_partition_compress_*)
  DevBuf meta, scratch, desc, src, dst, zmeta;
  DevBuf pws, parena;  // partition workspace (sort keys, offsets) and the partitioned arena in front of compression
  DevBuf xpieces;      // the copy pieces of an exchange-cache read (exchange.cu)
  PinBuf hmeta;
  // per-launch event pairs around the dominant kernel of a call (grow-only pool; `used` pairs are valid)
  std::vector<cudaEvent_t> ev_dom;
  std::vector<cudaEvent_t> trace;  // B2S_TRACE=1: (match0, match1, tail0, tail1) per compress chunk, printed by add_timing
  size_t dom_used = 0;
  int dom_pair(cudaEvent_t* a, cudaEvent_t* b) {
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

uint32_t block_size_or_default(uint32_t codec, uint32_t bs) {
  (void)codec;
  return bs ? bs : 32768u;
}

// pick the checksum work-item size: enough items to fill the machine, big enough to amortise the combine
uint32_t pick_tile_shift(uint64_t total_bytes) {
  uint32_t s = 20;  // 1 MiB
  const uint64_t want_items = (uint64_t)kSMs * 32 * 4;
  while (s > 14 && (total_bytes >> s) < want_items) s--;
  return s;
}

double ms_between(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0;
  if (cudaEventElapsedTime(&ms, a, b) != cudaSuccess) {
    (void)cudaGetLastError();  // unrecorded event: not an error of the call being timed
    return 0;
  }
  return ms;
}

struct WallTimer {
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  double ms() const { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
};

// --------------------------------------------------------------------------------------------------------------
// compress job: one chunk of n streams living in a device source arena
// --------------------------------------------------------------------------------------------------------------
// bytes every stream adds around its codec blocks: LZ4Block end mark (21) / xerial stream header (16)
inline uint64_t stream_overhead(uint32_t codec) {
  return codec == B2S_CODEC_SNAPPY_XERIAL ? 16ull : codec == B2S_CODEC_ZSTD ? 9ull : 21ull;  // + zstd: frame header 6 + end block 3
}

struct CompressJob {
  uint32_t n = 0, nb = 0, codec = 0;
  // pinned host mirror
  uint64_t *h_src_off = nullptr, *h_src_len = nullptr;
  uint32_t* h_blk_base = nullptr;
  uint64_t *h_dst_off = nullptr, *h_dst_len = nullptr, *h_cks = nullptr, *h_total = nullptr;
  int32_t* h_status = nullptr;
  size_t up_bytes = 0, down_bytes = 0;
  uint8_t *d_up = nullptr, *d_down = nullptr;
  uint8_t *h_up = nullptr, *h_down = nullptr;
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

// lays out pinned + device meta for a compress chunk; returns 0 or error
int compress_prepare(Slot& S, uint32_t codec, uint32_t bs, uint32_t n, const uint64_t* src_len, CompressJob& J) {
  if (int rc = check_codec_block(codec, bs)) return rc;
  J.n = n;
  J.codec = codec;
  uint64_t nb = 0;
  for (uint32_t i = 0; i < n; i++) nb += (src_len[i] + bs - 1) / bs;
  if (nb >= 0x7fffffffull) return fail(B2S_E_ARG, "too many codec blocks in one chunk%s");
  J.nb = (uint32_t)nb;
  // pinned: upload [src_off | src_len | blk_base], download [dst_off | dst_len | cks | total | status]
  size_t up = align_up(n * 8, 16) * 2 + align_up((n + 1) * 4, 16);
  size_t down = align_up(n * 8, 16) * 3 + 16 + align_up(n * 4, 16);
  int rc = S.hmeta.ensure(up + down + 64);
  if (rc) return rc;
  Carver hc(S.hmeta.p);
  J.h_up = (uint8_t*)hc.take<uint64_t>(0);
  J.h_src_off = hc.take<uint64_t>(n);
  J.h_src_len = hc.take<uint64_t>(n);
  J.h_blk_base = hc.take<uint32_t>(n + 1);
  hc.off = align_up(hc.off, 16);
  J.up_bytes = hc.off;
  J.h_down = (uint8_t*)hc.take<uint64_t>(0);
  size_t d0 = hc.off;
  J.h_dst_off = hc.take<uint64_t>(n);
  J.h_dst_len = hc.take<uint64_t>(n);
  J.h_cks = hc.take<uint64_t>(n);
  J.h_total = hc.take<uint64_t>(2);
  J.h_status = hc.take<int32_t>(n);
  hc.off = align_up(hc.off, 16);
  J.down_bytes = hc.off - d0;
  return 0;
}

struct CompressDevMeta {
  uint64_t *src_off, *src_len;
  uint32_t* blk_base;
  uint64_t *dst_off, *dst_len, *cks, *total;
  int32_t* status;
  uint32_t *csize, *hash, *nseq;
  uint64_t *sizes, *work_base, *ws;
  unsigned int* counter;
};

// Compression level.  LZ4Block and Snappy have none in the reference either (lz4-java's fast compressor, snappy-java);
// for Zstandard (spark.io.compression.zstd.level, codec chosen at storage/S3ShuffleReader.scala:57-60) the level sets the
// match finder's hash-table size: 1 -> 2^11 entries per block (fastest), 2 / unspecified -> 2^12, >= 3 -> 2^13 (more
// shared memory per warp, fewer resident warps, more matches found).
int hlog_for_level(uint32_t codec, int32_t level) {
  if (codec != B2S_CODEC_ZSTD || level <= 0) return 0;
  return level == 1 ? 11 : level == 2 ? 12 : 13;
}

int compress_enqueue(Context* C, Slot& S, const ChecksumTables& tabs, uint32_t bs, uint32_t alg, CompressJob& J,
                     const uint8_t* d_src, uint8_t* d_dst, uint64_t dst_cap, CompressDevMeta& M, uint64_t* launches,
                     int32_t level) {
  const uint32_t n = J.n, nb = J.nb;
  const uint32_t chunk = std::min<uint32_t>(nb ? nb : 1, g_lz4_chunk_blocks);
  size_t ws_elems = std::max(scan_ws_elems(nb + 1), checksum_ws_elems(n)) + 4;
  size_t need = J.up_bytes + J.down_bytes + align_up((size_t)nb * 4, 16) * 3 + align_up(((size_t)nb + 1) * 8, 16) +
                align_up(((size_t)n + 1) * 8, 16) + ws_elems * 8 + 256;
  int rc = S.meta.ensure(need);
  if (rc) return rc;
  const size_t ws_bytes = align_up(lz4_compress_ws_bytes(chunk, bs, J.codec), 256);
  rc = S.scratch.ensure(ws_bytes * (nb > chunk ? 2 : 1));
  if (rc) return rc;
  Carver dc(S.meta.p);
  J.d_up = (uint8_t*)dc.take<uint64_t>(0);
  M.src_off = dc.take<uint64_t>(n);
  M.src_len = dc.take<uint64_t>(n);
  M.blk_base = dc.take<uint32_t>(n + 1);
  dc.off = align_up(dc.off, 16);
  J.d_down = (uint8_t*)dc.take<uint64_t>(0);
  M.dst_off = dc.take<uint64_t>(n);
  M.dst_len = dc.take<uint64_t>(n);
  M.cks = dc.take<uint64_t>(n);
  M.total = dc.take<uint64_t>(2);
  M.status = dc.take<int32_t>(n);
  M.csize = dc.take<uint32_t>(nb);
  M.hash = dc.take<uint32_t>(nb);
  M.nseq = dc.take<uint32_t>(nb);
  M.sizes = dc.take<uint64_t>((size_t)nb + 1);
  M.work_base = dc.take<uint64_t>((size_t)n + 1);
  M.ws = dc.take<uint64_t>(ws_elems);
  M.counter = dc.take<unsigned int>(4);

  // blk_base prefix on the host
  uint64_t acc = 0;
  for (uint32_t i = 0; i < n; i++) {
    J.h_blk_base[i] = (uint32_t)acc;
    acc += (J.h_src_len[i] + bs - 1) / bs;
  }
  J.h_blk_base[n] = (uint32_t)acc;

  cudaStream_t st = S.st;
  CU(cudaMemcpyAsync(J.d_up, J.h_up, J.up_bytes, cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(J.d_down, 0, J.down_bytes, st));
  CU(cudaEventRecord(S.ev_k0, st));
  const uint32_t codec = J.codec;
  CU(cudaEventRecord(S.ev_t0, st));
  // Chunks of `chunk` codec blocks.  The match kernel (issue bound, shared-memory limited) of chunk k+1 runs on the
  // side stream while parse (latency bound, one thread per block), scan and emit of chunk k run on the main stream;
  // the two workspaces alternate.  The side stream forks BEFORE the per-block XXH32 pass (LZ4Block headers; only the
  // emit kernel needs it), so that pass runs beside the first chunk's match kernel instead of in front of it.
  cudaStream_t side = g_overlap ? S.st2 : st;
  CU(cudaEventRecord(S.ev_fork, st));
  CU(cudaStreamWaitEvent(side, S.ev_fork, 0));
  if (codec == B2S_CODEC_LZ4BLOCK)
    launch_xxh32_encode(d_src, M.src_off, M.src_len, M.blk_base, n, nb, bs, kXxhSeed, M.hash, st, launches);
  CU(cudaMemsetAsync(M.total, 0, 16, st));
  uint32_t k = 0;
  for (uint32_t b0 = 0; b0 < nb; b0 += chunk, k++) {
    const uint32_t m = std::min<uint32_t>(chunk, nb - b0);
    const int par = (int)(k & 1);
    uint8_t* ws = (uint8_t*)S.scratch.p + (size_t)par * ws_bytes;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    S.dom_pair(&e0, &e1);
    if (k >= 2) CU(cudaStreamWaitEvent(side, S.ev_free[par], 0));  // emit of chunk k-2 has released this workspace
    launch_lz4_match(d_src, M.src_off, M.src_len, M.blk_base, n, b0, m, bs, codec, ws, M.counter + par, side, launches,
                     e0, e1, hlog_for_level(codec, level));
    CU(cudaEventRecord(S.ev_match[par], side));
    CU(cudaStreamWaitEvent(st, S.ev_match[par], 0));
    cudaEvent_t t0 = nullptr, t1 = nullptr, tp = nullptr;
    if (g_trace && S.trace.size() < 4096) {
      cudaEventCreate(&t0);
      cudaEventCreate(&t1);
      cudaEventCreate(&tp);
      S.trace.push_back(e0); S.trace.push_back(e1); S.trace.push_back(t0); S.trace.push_back(t1); S.trace.push_back(tp);
      CU(cudaEventRecord(t0, st));
    }
    launch_lz4_parse_emit(d_src, M.src_off, M.src_len, M.blk_base, n, b0, m, bs, codec, ws, M.nseq, M.csize, M.hash,
                          M.sizes, M.total, M.ws, d_dst, dst_cap, st, launches, tp);
    if (t1) CU(cudaEventRecord(t1, st));
    CU(cudaEventRecord(S.ev_free[par], st));
  }
  CU(cudaEventRecord(S.ev_t1, st));
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
  CU(cudaEventRecord(S.ev_k1, st));
  CU(cudaMemcpyAsync(J.h_down, J.d_down, J.down_bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(S.ev_a, st));
  CU(cudaGetLastError());
  (void)C;
  return 0;
}

// --------------------------------------------------------------------------------------------------------------
// decompress job
// --------------------------------------------------------------------------------------------------------------
struct DecompressJob {
  uint32_t n = 0, n_slices = 0, codec = 0;
  uint64_t nb = 0, total_out = 0;
  uint64_t *h_src_off = nullptr, *h_src_len = nullptr;
  uint64_t *h_slice_off = nullptr, *h_slice_len = nullptr, *h_slice_sum = nullptr;
  uint32_t *h_slice_owner = nullptr, *h_slice_base = nullptr;
  uint64_t* h_totals = nullptr;  // [nb_total, olen_total]
  uint64_t *h_dst_off = nullptr, *h_dst_len = nullptr;
  int32_t *h_status = nullptr, *h_bad = nullptr;
  size_t up_bytes = 0, down_bytes = 0;
  uint8_t *h_up = nullptr, *h_down = nullptr, *d_up = nullptr, *d_down = nullptr;
  // device
  uint64_t *src_off = nullptr, *src_len = nullptr, *slice_off = nullptr, *slice_len = nullptr, *slice_sum = nullptr;
  uint32_t *slice_owner = nullptr, *slice_base = nullptr;
  uint64_t *nblk = nullptr, *olen = nullptr, *dst_off = nullptr, *totals = nullptr, *cks_got = nullptr,
           *work_base = nullptr, *ws = nullptr;
  int32_t *status = nullptr, *bad = nullptr;
  unsigned int* counter = nullptr;
  // zstd: per-stream counts / bases (blocks, sequences, literal bytes) and their totals
  uint64_t *zcnt = nullptr, *zbase = nullptr;
  uint64_t znb = 0, znseq = 0, zlit = 0;
  bool size_only = false;
};

// allow_none: codec NONE verifies the slices only and reports the stored lengths as decoded lengths in phase A (the
// key sort of uncompressed blocks); phase B is not run for it
int decompress_prepare(Slot& S, uint32_t codec, uint32_t alg, uint32_t n, uint32_t n_slices, DecompressJob& J,
                       bool allow_none = false) {
  if (codec != B2S_CODEC_LZ4BLOCK && codec != B2S_CODEC_SNAPPY_XERIAL && codec != B2S_CODEC_ZSTD &&
      !(allow_none && codec == B2S_CODEC_NONE))
    return fail(B2S_E_UNSUPPORTED, "codec %s not supported by this build", "");
  J.n = n;
  J.codec = codec;
  J.n_slices = alg ? n_slices : 0;
  const uint32_t s = J.n_slices;
  size_t up = align_up(n * 8, 16) * 2 + align_up((size_t)s * 8, 16) * 3 + align_up((size_t)s * 4, 16) +
              align_up(((size_t)n + 1) * 4, 16);
  size_t down = 32 + align_up(n * 8, 16) * 2 + align_up(n * 4, 16) * 2;
  int rc = S.hmeta.ensure(up + down + 128);
  if (rc) return rc;
  Carver hc(S.hmeta.p);
  J.h_up = (uint8_t*)hc.take<uint64_t>(0);
  J.h_src_off = hc.take<uint64_t>(n);
  J.h_src_len = hc.take<uint64_t>(n);
  J.h_slice_off = hc.take<uint64_t>(s);
  J.h_slice_len = hc.take<uint64_t>(s);
  J.h_slice_sum = hc.take<uint64_t>(s);
  J.h_slice_owner = hc.take<uint32_t>(s);
  J.h_slice_base = hc.take<uint32_t>((size_t)n + 1);
  hc.off = align_up(hc.off, 16);
  J.up_bytes = hc.off;
  J.h_down = (uint8_t*)hc.take<uint64_t>(0);
  size_t d0 = hc.off;
  J.h_totals = hc.take<uint64_t>(4);
  J.h_dst_off = hc.take<uint64_t>(n);
  J.h_dst_len = hc.take<uint64_t>(n);
  J.h_status = hc.take<int32_t>(n);
  J.h_bad = hc.take<int32_t>(n);
  hc.off = align_up(hc.off, 16);
  J.down_bytes = hc.off - d0;
  return 0;
}

// phase A: checksum verify + header count + scans + totals readback
int decompress_enqueue_a(Slot& S, const ChecksumTables& tabs, uint32_t alg, DecompressJob& J, const uint8_t* d_src,
                         uint64_t src_bytes, uint64_t* launches) {
  const uint32_t n = J.n, s = J.n_slices;
  size_t ws_elems = std::max(scan_ws_elems((size_t)n + 1), checksum_ws_elems(s)) + 4;
  size_t need = J.up_bytes + J.down_bytes + align_up((size_t)n * 8, 16) * 1 + align_up((size_t)s * 8, 16) +
                align_up(((size_t)s + 1) * 8, 16) + ws_elems * 8 + 256;
  int rc = S.meta.ensure(need);
  if (rc) return rc;
  Carver dc(S.meta.p);
  J.d_up = (uint8_t*)dc.take<uint64_t>(0);
  J.src_off = dc.take<uint64_t>(n);
  J.src_len = dc.take<uint64_t>(n);
  J.slice_off = dc.take<uint64_t>(s);
  J.slice_len = dc.take<uint64_t>(s);
  J.slice_sum = dc.take<uint64_t>(s);
  J.slice_owner = dc.take<uint32_t>(s);
  J.slice_base = dc.take<uint32_t>((size_t)n + 1);
  dc.off = align_up(dc.off, 16);
  J.d_down = (uint8_t*)dc.take<uint64_t>(0);
  J.totals = dc.take<uint64_t>(4);
  J.dst_off = dc.take<uint64_t>(n);
  J.olen = dc.take<uint64_t>(n);
  J.status = dc.take<int32_t>(n);
  J.bad = dc.take<int32_t>(n);
  J.nblk = dc.take<uint64_t>(n);
  J.cks_got = dc.take<uint64_t>(s);
  J.work_base = dc.take<uint64_t>((size_t)s + 1);
  J.ws = dc.take<uint64_t>(ws_elems);
  J.counter = dc.take<unsigned int>(4);

  cudaStream_t st = S.st;
  CU(cudaMemcpyAsync(J.d_up, J.h_up, J.up_bytes, cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(J.d_down, 0, J.down_bytes, st));
  CU(cudaMemsetAsync(J.bad, 0xff, (size_t)n * 4, st));
  CU(cudaEventRecord(S.ev_k0, st));
  if (alg != B2S_CHECKSUM_NONE && s) {
    launch_checksum(tabs, alg, d_src, J.slice_off, J.slice_len, s, pick_tile_shift(src_bytes), J.work_base, J.ws,
                    J.cks_got, st, launches);
    launch_checksum_compare(J.cks_got, J.slice_sum, J.slice_owner, J.slice_base, s, J.status, J.bad, st, launches);
  }
  if (J.codec == B2S_CODEC_ZSTD) {
    // walk (count) -> totals to the host -> walk (fill) -> entropy decode of every block in parallel -> stream sizes.
    // The one blocking readback sizes the descriptor array and the literal / sequence workspace (zstd_par.h).
    rc = S.zmeta.ensure(((size_t)n * 6 + 8) * 8);
    if (rc) return rc;
    J.zcnt = (uint64_t*)S.zmeta.p;
    J.zbase = J.zcnt + (size_t)n * 3;
    uint64_t* ztot = J.zbase + (size_t)n * 3;
    launch_zstd_count(d_src, J.src_off, J.src_len, n, J.zcnt, J.status, st, launches);
    CU(cudaMemcpyAsync(J.zbase, J.zcnt, (size_t)n * 24, cudaMemcpyDeviceToDevice, st));
    for (int k = 0; k < 3; k++) launch_exclusive_scan_u64(J.zbase + (size_t)n * k, n, ztot + k, J.ws, st, launches);
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
    launch_zstd_fill(d_src, J.src_off, J.src_len, n, J.zcnt, J.zbase, S.desc.p, J.status, st, launches);
    launch_zstd_entropy(J.size_only, d_src, S.desc.p, J.znb, (uint8_t*)S.scratch.p, J.zlit, J.znseq, J.status, st,
                        launches);
    launch_zstd_sum(S.desc.p, J.zcnt, J.zbase, n, J.olen, J.status, st, launches);
    CU(cudaMemsetAsync(J.nblk, 0, (size_t)n * 8, st));
  } else if (J.codec == B2S_CODEC_SNAPPY_XERIAL)
    launch_xerial_count(d_src, J.src_off, J.src_len, n, J.nblk, J.olen, J.totals + 2, J.status, st, launches);
  else if (J.codec == B2S_CODEC_NONE) {  // stored bytes: decoded length = block length, no codec blocks
    CU(cudaMemcpyAsync(J.olen, J.src_len, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
    CU(cudaMemsetAsync(J.nblk, 0, (size_t)n * 8, st));
  } else
    launch_lz4block_count(d_src, J.src_off, J.src_len, n, J.nblk, J.olen, J.totals + 2, J.status, st, launches);
  // dst_off = exclusive scan(olen) ; blk_base = exclusive scan(nblk) (in place)
  CU(cudaMemcpyAsync(J.dst_off, J.olen, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
  launch_exclusive_scan_u64(J.dst_off, n, J.totals + 1, J.ws, st, launches);
  launch_exclusive_scan_u64(J.nblk, n, J.totals + 0, J.ws, st, launches);
  CU(cudaMemcpyAsync(J.h_totals, J.totals, 32, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(S.ev_a, st));
  CU(cudaGetLastError());
  return 0;
}

// phase B (after ev_a): descriptors, decode, XXH32 verify, meta readback
int decompress_enqueue_b(Slot& S, DecompressJob& J, const uint8_t* d_src, uint8_t* d_dst, uint64_t dst_cap,
                         uint64_t* launches) {
  J.nb = J.h_totals[0];
  J.total_out = J.h_totals[1];
  if (J.codec == B2S_CODEC_ZSTD) {
    cudaStream_t zst = S.st;
    CU(cudaEventRecord(S.ev_t0, zst));
    launch_zstd_execute(d_src, S.desc.p, J.zcnt, J.zbase, J.n, (const uint8_t*)S.scratch.p, J.zlit, J.znseq, J.olen,
                        d_dst, J.dst_off, dst_cap, J.status, zst, launches);
    CU(cudaEventRecord(S.ev_t1, zst));
    CU(cudaEventRecord(S.ev_k1, zst));
    CU(cudaMemcpyAsync(J.h_down, J.d_down, J.down_bytes, cudaMemcpyDeviceToHost, zst));
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
    launch_xerial_fill(d_src, J.src_off, J.src_len, J.n, J.nblk, J.dst_off, J.olen, dst_cap, J.status, desc, st,
                       launches);
  else
    launch_lz4block_fill(d_src, J.src_off, J.src_len, J.n, J.nblk, J.dst_off, J.olen, dst_cap, J.status, desc, st,
                         launches);
  CU(cudaEventRecord(S.ev_t0, st));
  const uint64_t max_olen = J.h_totals[2], max_clen = J.h_totals[3];
  const bool small_blocks = max_olen <= 65536 && max_clen < 65536;
  if (J.codec == B2S_CODEC_SNAPPY_XERIAL && !small_blocks)
    return fail(B2S_E_UNSUPPORTED, "snappy chunks larger than 64 KiB are not supported%s");
  if (J.nb && small_blocks && (J.codec == B2S_CODEC_SNAPPY_XERIAL || !g_lz4d_legacy)) {
    // tokens (thread per block) + copy (lane per sequence), in chunks that bound the record workspace
    const uint32_t nb = (uint32_t)J.nb;
    const uint32_t rec_stride = lz4_decode_rec_stride(J.codec, (uint32_t)max_olen, (uint32_t)max_clen);
    const uint32_t chunk = std::min<uint32_t>(nb, g_lz4d_chunk_blocks);
    const size_t nrec_bytes = align_up((size_t)nb * 4, 256);
    const size_t ws_bytes = align_up(lz4_decode_ws_bytes(chunk, rec_stride), 256);
    rc = S.scratch.ensure(nrec_bytes + ws_bytes * (nb > chunk ? 2 : 1));
    if (rc) return rc;
    uint32_t* nrec = (uint32_t*)S.scratch.p;
    // token walk (thread per block, latency bound) of chunk k+1 on the side stream, copies of chunk k on the main one
    CU(cudaEventRecord(S.ev_fork, st));
    CU(cudaStreamWaitEvent(S.st2, S.ev_fork, 0));
    uint32_t k = 0;
    for (uint32_t b0 = 0; b0 < nb; b0 += chunk, k++) {
      const uint32_t m = std::min<uint32_t>(chunk, nb - b0);
      const int par = (int)(k & 1);
      uint8_t* ws = (uint8_t*)S.scratch.p + nrec_bytes + (size_t)par * ws_bytes;
      if (k >= 2) CU(cudaStreamWaitEvent(S.st2, S.ev_free[par], 0));
      cudaEvent_t q0 = nullptr, q1 = nullptr;
      if (g_trace && S.trace.size() < 4096) {
        cudaEventCreate(&q0);
        cudaEventCreate(&q1);
        CU(cudaEventRecord(q0, S.st2));
      }
      launch_lz4_tokens(J.codec, desc, b0, m, rec_stride, d_src, ws, nrec, J.status, S.st2, launches);
      if (q1) CU(cudaEventRecord(q1, S.st2));
      CU(cudaEventRecord(S.ev_match[par], S.st2));
      CU(cudaStreamWaitEvent(st, S.ev_match[par], 0));
      cudaEvent_t e0 = nullptr, e1 = nullptr;
      S.dom_pair(&e0, &e1);
      CU(cudaEventRecord(e0, st));
      launch_lz4_copy(desc, b0, m, rec_stride, d_src, d_dst, ws, nrec, st, launches);
      CU(cudaEventRecord(e1, st));
      if (q0) {  // trace rows: (tokens0, tokens1, copy0, copy1, copy1)
        S.trace.push_back(q0); S.trace.push_back(q1);
        cudaEvent_t c0 = nullptr, c1 = nullptr, c2 = nullptr;
        cudaEventCreate(&c0); cudaEventCreate(&c1); cudaEventCreate(&c2);
        // e0/e1 belong to the dom pool; re-record private copies right here (same stream position as e1)
        CU(cudaEventRecord(c1, st)); CU(cudaEventRecord(c2, st));
        S.trace.push_back(e0); S.trace.push_back(c1); S.trace.push_back(c2);
        cudaEventDestroy(c0);
      }
      CU(cudaEventRecord(S.ev_free[par], st));
    }
  } else if (J.nb) {
    launch_lz4_decompress(desc, (uint32_t)J.nb, d_src, d_dst, J.status, J.counter, st, launches);
  }
  CU(cudaEventRecord(S.ev_t1, st));
  // One XXH32 pass over all decoded blocks after the last chunk.  Queueing it chunk by chunk on the side stream (beside
  // the next chunk's copy kernel) was measured slower: both kernels are
  // memory-latency bound and take each other's L2 / DRAM queue slots.
  if (J.codec == B2S_CODEC_LZ4BLOCK)
    launch_xxh32_verify(desc, (uint32_t)J.nb, d_dst, kXxhSeed, 0x0FFFFFFFu, J.status, st, launches);
  CU(cudaEventRecord(S.ev_k1, st));
  CU(cudaMemcpyAsync(J.h_down, J.d_down, J.down_bytes, cudaMemcpyDeviceToHost, st));
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

void add_timing(Slot& S, bool copies) {
  t_timing.kernel_ms += ms_between(S.ev_k0, S.ev_k1);
  t_timing.top_kernel_ms += ms_between(S.ev_t0, S.ev_t1);
  for (size_t k = 0; k < S.dom_used; k++) {
    t_timing.dominant_ms += ms_between(S.ev_dom[2 * k], S.ev_dom[2 * k + 1]);
    t_timing.dominant_launches++;
  }
  if (g_trace && !S.trace.empty()) {
    cudaEvent_t base = S.trace[0];
    for (size_t k = 0; k + 4 < S.trace.size(); k += 5) {
      fprintf(stderr, "chunk %2zu: A(match|tokens) %7.3f..%7.3f  B(parse|copy) %7.3f..%7.3f  end %7.3f ms\n", k / 5,
              ms_between(base, S.trace[k]), ms_between(base, S.trace[k + 1]), ms_between(base, S.trace[k + 2]),
              ms_between(base, S.trace[k + 4]), ms_between(base, S.trace[k + 3]));
      // (events at k, k+1 [compress] / k+2 [decode] belong to the dominant-kernel pool or are leaked: tracing only)
      cudaEventDestroy(S.trace[k + 3]);
      cudaEventDestroy(S.trace[k + 4]);
    }
    S.trace.clear();
  }
  S.dom_used = 0;
  if (copies) t_timing.h2d_ms += ms_between(S.ev_h0, S.ev_h1);  // d2h is added once the payload copy has run
}

// groups streams [i0, i1) into chunks of ~g_host_chunk_bytes
void make_chunks(uint32_t n, const uint64_t* len, std::vector<uint32_t>& starts) {
  starts.clear();
  uint32_t i = 0;
  while (i < n) {
    starts.push_back(i);
    uint64_t bytes = 0;
    uint32_t cnt = 0;
    while (i < n && cnt < kChunkStreams && (cnt == 0 || bytes + len[i] <= g_host_chunk_bytes)) {
      bytes += len[i];
      i++;
      cnt++;
    }
  }
  starts.push_back(n);
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
  uint64_t bytes = 0;
  std::vector<uint64_t> part_start;  // R + 1 offsets of the partitions in buf
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
  g_ex.used[e->ordinal] -= e->bytes;
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
    if (kv.second->ordinal == ordinal && !kv.second->refs) idle += kv.second->bytes;
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
};

// Keeps `bytes` of partitioned records at d_rec (device memory of the current device `ordinal`, stream st) as the
// entry (shuffle, map): exact-size allocation, device-to-device copy.  Returns 1 when stored, 0 when it does not fit.
int ex_store(int ordinal, cudaStream_t st, int32_t shuffle, int64_t map, const uint8_t* d_rec, uint64_t bytes,
             std::vector<uint64_t>&& part_start) {
  std::vector<ExEntry*> dead;
  bool fits;
  {
    std::lock_guard<std::mutex> lk(g_ex.mtx);
    auto it = g_ex.by_key.find({shuffle, map});
    if (it != g_ex.by_key.end()) ex_unlink(it->second, dead);  // a stale output of this map is never served again
    fits = g_ex.budget[ordinal] > 0 && ex_make_room(ordinal, bytes, dead);
    if (fits) g_ex.used[ordinal] += bytes;  // reserved until the entry is linked
  }
  ex_free(dead);
  dead.clear();
  if (!fits) return 0;
  ExEntry* e = new ExEntry();
  e->shuffle = shuffle;
  e->map = map;
  e->ordinal = ordinal;
  e->bytes = bytes;
  e->part_start = std::move(part_start);
  bool ok = true;
  if (bytes) {
    ok = cudaMalloc(&e->buf, bytes) == cudaSuccess &&
         cudaMemcpyAsync(e->buf, d_rec, bytes, cudaMemcpyDeviceToDevice, st) == cudaSuccess &&
         cudaStreamSynchronize(st) == cudaSuccess;
    if (!ok) (void)cudaGetLastError();  // not stored; the call's own outputs are unaffected
  }
  {
    std::lock_guard<std::mutex> lk(g_ex.mtx);
    g_ex.used[ordinal] -= bytes;
    if (!ok) {
      dead.push_back(e);
    } else {
      auto it = g_ex.by_key.find({shuffle, map});
      if (it != g_ex.by_key.end()) ex_unlink(it->second, dead);  // stored by another thread meanwhile
      g_ex.used[ordinal] += bytes;
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
  int count = 0;
  const cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0)
    return fail(B2S_E_CUDA, "no CUDA device: %s", e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
  return fail(B2S_E_NOT_INIT, "b2s_init has not been called%s");
}

int reduce_range_args(int32_t start_reduce, int32_t end_reduce) {
  if (start_reduce < 0 || end_reduce < start_reduce || end_reduce > (1 << 24))
    return fail(B2S_E_ARG, "reduce range must satisfy 0 <= start_reduce <= end_reduce <= 2^24%s");
  return 0;
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
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0)
    return fail(B2S_E_CUDA, "no CUDA device: %s", e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
  g_lz4_hlog = env_int("B2S_LZ4_HLOG", g_lz4_hlog);
  g_lz4d_tile = env_int("B2S_LZ4D_TILE", g_lz4d_tile);
  g_lz4_pipe = env_int("B2S_LZ4_PIPE", g_lz4_pipe);
  g_lz4d_tokens = env_int("B2S_LZ4D_TOKENS", g_lz4d_tokens);
  g_lz4_chunk_blocks = (uint32_t)std::max(1, env_int("B2S_LZ4_CHUNK_BLOCKS", (int)g_lz4_chunk_blocks));
  g_lz4d_legacy = env_int("B2S_LZ4D_LEGACY", 0);
  g_trace = env_int("B2S_TRACE", 0);
  g_numa = env_int("B2S_NUMA", 1);
  g_overlap = env_int("B2S_OVERLAP", g_overlap);
  g_read_priority = env_int("B2S_READ_PRIORITY", g_read_priority);
  g_read_lag = std::max(1, env_int("B2S_READ_LAG", g_read_lag));
  g_copy_piece = (uint64_t)std::max(0, env_int("B2S_COPY_PIECE_MB", 0)) << 20;
  g_lz4d_chunk_blocks = (uint32_t)std::max(1, env_int("B2S_LZ4D_CHUNK_BLOCKS", (int)g_lz4d_chunk_blocks));
  g_host_chunk_bytes = (uint64_t)std::max(1, env_int("B2S_HOST_CHUNK_MB", (int)(g_host_chunk_bytes >> 20))) << 20;
  // streams_per_gpu: pipeline slots (stream pairs + staging) per lane, 0 = default; B2S_SLOTS overrides
  g_nslot = std::min(NSLOT, std::max(2, env_int("B2S_SLOTS", streams_per_gpu ? (int)streams_per_gpu : g_nslot)));
  Context* C = new Context();
  for (int d = 0; d < count && d < 32; d++) {
    if (gpu_mask && !(gpu_mask & (1u << d))) continue;
    CU(cudaSetDevice(d));
    Device* D = new Device();
    D->ordinal = d;
    char busid[32] = {0};
    if (g_numa && cudaDeviceGetPCIBusId(busid, sizeof busid, d) == cudaSuccess) D->numa_node = numa::node_of_pci(busid);
    (void)cudaGetLastError();
    t_numa_node = D->numa_node;
    for (int l = 0; l < kLanes; l++)
      for (int k = 0; k < g_nslot; k++) {
        Slot& S = D->lane[l].slot[k];
        // the read lane's kernels are short and latency bound (token walks, per-stream header walks, two host round
        // trips per chunk): they get the higher stream priority so they are not queued behind the write lane's grids
        int prio_lo = 0, prio_hi = 0;
        cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
        const int prio = (l == kLaneRead && g_read_priority) ? prio_hi : prio_lo;
        CU(cudaStreamCreateWithPriority(&S.st, cudaStreamNonBlocking, prio));
        CU(cudaStreamCreateWithPriority(&S.st2, cudaStreamNonBlocking, prio));
        cudaEvent_t* evs2[] = {&S.ev_fork, &S.ev_match[0], &S.ev_match[1], &S.ev_free[0], &S.ev_free[1]};
        for (auto p : evs2) CU(cudaEventCreateWithFlags(p, cudaEventDisableTiming));
        cudaEvent_t* evs[] = {&S.ev_a, &S.ev_b, &S.ev_k0, &S.ev_k1, &S.ev_t0, &S.ev_t1, &S.ev_h0, &S.ev_h1, &S.ev_d0, &S.ev_d1,
                              &S.ev_p0, &S.ev_p1};
        for (auto p : evs) CU(cudaEventCreate(p));
        // pinned_bytes_per_gpu: the library's own pinned descriptor blocks are sized up front (split over the slots)
        // instead of growing on first use; 0 = grow on demand.  Payload staging is the caller's (b2s_host_alloc).
        if (pinned_bytes_per_gpu) {
          const uint64_t per = std::min<uint64_t>(pinned_bytes_per_gpu / (uint64_t)(kLanes * g_nslot), 64ull << 20);
          if (per >= 4096 && S.hmeta.ensure(per)) return B2S_E_NOMEM;
        }
      }
    if (checksum_tables_create(&D->tabs)) return fail(B2S_E_CUDA, "checksum table upload failed%s");
    if (zstd_ctables_create(&D->zstd_ctables)) return fail(B2S_E_CUDA, "zstd table upload failed%s");
    zstd_set_ctables(d, D->zstd_ctables);
    CU(cudaEventCreate(&D->ev_mark[0]));
    CU(cudaEventCreate(&D->ev_mark[1]));
    C->devs.push_back(D);
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
  for (Device* D : g_ctx->devs) {
    cudaSetDevice(D->ordinal);
    cudaDeviceSynchronize();
    for (int l = 0; l < kLanes; l++)
    for (int k = 0; k < NSLOT; k++) {
      Slot& S = D->lane[l].slot[k];
      S.meta.release();
      S.scratch.release();
      S.desc.release();
      S.zmeta.release();
      S.src.release();
      S.dst.release();
      S.pws.release();
      S.parena.release();
      S.xpieces.release();
      S.hmeta.release();
      cudaEvent_t evs[] = {S.ev_a, S.ev_b, S.ev_k0, S.ev_k1, S.ev_t0, S.ev_t1, S.ev_h0, S.ev_h1, S.ev_d0, S.ev_d1,
                           S.ev_p0, S.ev_p1};
      for (auto ev : evs)
        if (ev) cudaEventDestroy(ev);
      for (auto ev : S.ev_dom) cudaEventDestroy(ev);
      S.ev_dom.clear();
      cudaEvent_t evs2[] = {S.ev_fork, S.ev_match[0], S.ev_match[1], S.ev_free[0], S.ev_free[1]};
      for (auto ev : evs2)
        if (ev) cudaEventDestroy(ev);
      if (S.st2) cudaStreamDestroy(S.st2);
      if (S.st) cudaStreamDestroy(S.st);
    }
    checksum_tables_destroy(&D->tabs);
    zstd_ctables_destroy(D->zstd_ctables);
    for (auto ev : D->ev_mark)
      if (ev) cudaEventDestroy(ev);
    delete D;
  }
  delete g_ctx;
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
  const uint64_t bs = block_size_or_default(codec, codec_block_size);
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
  CU(cudaEventRecord(S.ev_k0, st));
  CU(cudaEventRecord(S.ev_t0, st));
  launch_checksum(D->tabs, alg, d_base, d_off, d_len, n, pick_tile_shift(total_bytes), d_work, d_ws, d_out, st,
                  launches);
  CU(cudaEventRecord(S.ev_t1, st));
  CU(cudaEventRecord(S.ev_k1, st));
  CU(cudaMemcpyAsync(h_out, d_out, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  memcpy(out, h_out, (size_t)n * 8);
  return 0;
}

int b2s_checksum_dev(uint32_t dev_index, uint32_t alg, uint32_t n, const void* d_base, const uint64_t* off,
                     const uint64_t* len, uint64_t* out) {
  WallTimer wt;
  t_timing = b2s_timing{};
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
  add_timing(Ln.slot[0], false);
  t_timing.kernel_launches = launches;
  t_timing.src_bytes = total;
  t_timing.total_ms = wt.ms();
  g_ctx->launches += launches;
  return 0;
}

static int checksum_host(uint32_t alg, uint32_t n, const uint8_t* const* ptr, const uint64_t* len, uint64_t* out) {
  WallTimer wt;
  t_timing = b2s_timing{};
  Device* D;
  int rc = get_device(t_device, &D);
  if (rc) return rc;
  if (!n) return 0;
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  std::vector<uint32_t> starts;
  make_chunks(n, len, starts);
  std::vector<uint64_t> dev_off;
  std::vector<Run> runs;
  uint64_t launches = 0;
  for (size_t c = 0; c + 1 < starts.size(); c++) {
    Slot& S = Ln.slot[0];
    const uint32_t i0 = starts[c], cnt = starts[c + 1] - starts[c];
    dev_off.resize(cnt);
    uint64_t bytes = plan_runs(cnt, ptr + i0, len + i0, dev_off.data(), runs);
    rc = S.src.ensure(bytes + 64);
    if (rc) return rc;
    CU(cudaEventRecord(S.ev_h0, S.st));
    for (const Run& r : runs)
      CU(copy_async((uint8_t*)S.src.p + r.dev_off, r.host, r.bytes, cudaMemcpyHostToDevice, S.st));
    CU(cudaEventRecord(S.ev_h1, S.st));
    rc = checksum_chunk_dev(D, S, alg, cnt, (const uint8_t*)S.src.p, dev_off.data(), len + i0, out + i0, bytes,
                            &launches);
    if (rc) return rc;
    add_timing(S, false);
    t_timing.h2d_ms += ms_between(S.ev_h0, S.ev_h1);
    t_timing.h2d_bytes += bytes;
    t_timing.d2h_bytes += (uint64_t)cnt * 8;
    t_timing.src_bytes += bytes;
  }
  t_timing.kernel_launches = launches;
  t_timing.total_ms = wt.ms();
  g_ctx->launches += launches;
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
  WallTimer wt;
  t_timing = b2s_timing{};
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
  const uint32_t bs = block_size_or_default(codec, codec_block_size);
  CompressJob J;
  rc = compress_prepare(S, codec, bs, n, src_len, J);
  if (rc) return rc;
  memcpy(J.h_src_off, src_off, (size_t)n * 8);
  memcpy(J.h_src_len, src_len, (size_t)n * 8);
  CompressDevMeta M;
  uint64_t launches = 0;
  rc = compress_enqueue(g_ctx, S, D->tabs, bs, checksum_alg, J, (const uint8_t*)d_src_base, (uint8_t*)d_dst_base,
                        dst_cap, M, &launches, level);
  if (rc) return rc;
  CU(cudaEventSynchronize(S.ev_a));
  CU(cudaGetLastError());
  memcpy(dst_off, J.h_dst_off, (size_t)n * 8);
  memcpy(dst_len, J.h_dst_len, (size_t)n * 8);
  memcpy(status, J.h_status, (size_t)n * 4);
  if (checksum_out) {
    if (checksum_alg) memcpy(checksum_out, J.h_cks, (size_t)n * 8);
    else memset(checksum_out, 0, (size_t)n * 8);
  }
  uint64_t total = J.h_total[0] + stream_overhead(codec) * n, srcb = 0;
  for (uint32_t i = 0; i < n; i++) srcb += src_len[i];
  if (dst_total) *dst_total = total;
  add_timing(S, false);
  t_timing.kernel_launches = launches;
  t_timing.src_bytes = srcb;
  t_timing.dst_bytes = total;
  t_timing.total_ms = wt.ms();
  g_ctx->launches += launches;
  return 0;
}

// shared engine for the host-pointer write path.  packed_dst != nullptr: outputs back to back into that arena.
static int compress_host(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t alg, uint32_t n,
                         const uint8_t* const* src, const uint64_t* src_len, uint8_t* packed_dst, uint64_t packed_cap,
                         uint8_t* const* dst, const uint64_t* dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                         uint64_t* dst_total, uint64_t* checksum_out, int32_t* status) {
  WallTimer wt;
  t_timing = b2s_timing{};
  Device* D;
  int rc = get_device(t_device, &D);
  if (rc) return rc;
  if (alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (dst_total) *dst_total = 0;
  if (!n) return 0;
  Lane& Ln = D->lane[kLaneWrite];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  const uint32_t bs = block_size_or_default(codec, codec_block_size);
  std::vector<uint32_t> starts;
  make_chunks(n, src_len, starts);
  const size_t nchunks = starts.size() - 1;
  std::vector<CompressJob> jobs(nchunks);
  std::vector<std::vector<Run>> runs(g_nslot);
  uint64_t launches = 0, run_off = 0;

  auto finish = [&](size_t c) -> int {
    Slot& S = Ln.slot[c % g_nslot];
    CompressJob& J = jobs[c];
    const uint32_t i0 = starts[c];
    CU(cudaEventSynchronize(S.ev_a));
    add_timing(S, true);
    const uint64_t chunk_total = J.h_total[0] + stream_overhead(codec) * J.n;
    for (uint32_t k = 0; k < J.n; k++) {
      status[i0 + k] = J.h_status[k];
      dst_len[i0 + k] = J.h_dst_len[k];
      if (checksum_out) checksum_out[i0 + k] = alg ? J.h_cks[k] : 0;
    }
    CU(cudaEventRecord(S.ev_d0, S.st));
    if (packed_dst) {
      if (run_off + chunk_total > packed_cap) {
        for (uint32_t k = 0; k < J.n; k++) {
          dst_off[i0 + k] = run_off + J.h_dst_off[k];
          if (run_off + J.h_dst_off[k] + J.h_dst_len[k] > packed_cap) status[i0 + k] = B2S_E_DST_TOO_SMALL;
        }
        // copy what fits so that earlier streams of the chunk stay valid
        uint64_t fit = packed_cap > run_off ? packed_cap - run_off : 0;
        if (fit) CU(copy_async(packed_dst + run_off, S.dst.p, fit, cudaMemcpyDeviceToHost, S.st));
        t_timing.d2h_bytes += fit;
      } else {
        for (uint32_t k = 0; k < J.n; k++) dst_off[i0 + k] = run_off + J.h_dst_off[k];
        if (chunk_total)
          CU(copy_async(packed_dst + run_off, S.dst.p, chunk_total, cudaMemcpyDeviceToHost, S.st));
        t_timing.d2h_bytes += chunk_total;
      }
      run_off += chunk_total;
    } else {
      for (uint32_t k = 0; k < J.n; k++) {
        const uint32_t i = i0 + k;
        if (status[i] != 0) continue;
        if (J.h_dst_len[k] > dst_cap[i]) {
          status[i] = B2S_E_DST_TOO_SMALL;
          continue;
        }
        CU(cudaMemcpyAsync(dst[i], (uint8_t*)S.dst.p + J.h_dst_off[k], J.h_dst_len[k], cudaMemcpyDeviceToHost, S.st));
        t_timing.d2h_bytes += J.h_dst_len[k];
      }
      run_off += chunk_total;
    }
    CU(cudaEventRecord(S.ev_d1, S.st));
    t_timing.dst_bytes += chunk_total;
    return 0;
  };

  for (size_t c = 0; c < nchunks; c++) {
    Slot& S = Ln.slot[c % g_nslot];
    if (c >= (size_t)g_nslot) {
      rc = finish(c - g_nslot);
      if (rc) return rc;
      CU(cudaStreamSynchronize(S.st));  // payload of the slot's previous chunk has left the device
      t_timing.d2h_ms += ms_between(S.ev_d0, S.ev_d1);
    }
    const uint32_t i0 = starts[c], cnt = starts[c + 1] - starts[c];
    CompressJob& J = jobs[c];
    rc = compress_prepare(S, codec, bs, cnt, src_len + i0, J);
    if (rc) return rc;
    memcpy(J.h_src_len, src_len + i0, (size_t)cnt * 8);
    uint64_t bytes = plan_runs(cnt, src + i0, src_len + i0, J.h_src_off, runs[c % g_nslot]);
    rc = S.src.ensure(bytes + 64);
    if (rc) return rc;
    uint64_t bound = 0;
    for (uint32_t k = 0; k < cnt; k++) bound += b2s_compress_bound(codec, bs, src_len[i0 + k]);
    rc = S.dst.ensure(bound + 64);
    if (rc) return rc;
    CU(cudaEventRecord(S.ev_h0, S.st));
    for (const Run& r : runs[c % g_nslot])
      CU(copy_async((uint8_t*)S.src.p + r.dev_off, r.host, r.bytes, cudaMemcpyHostToDevice, S.st));
    CU(cudaEventRecord(S.ev_h1, S.st));
    t_timing.h2d_bytes += bytes;
    t_timing.src_bytes += bytes;
    CompressDevMeta M;
    rc = compress_enqueue(g_ctx, S, D->tabs, bs, alg, J, (const uint8_t*)S.src.p, (uint8_t*)S.dst.p, S.dst.cap, M,
                          &launches, level);
    if (rc) return rc;
  }
  for (size_t c = nchunks > (size_t)g_nslot ? nchunks - g_nslot : 0; c < nchunks; c++) {
    rc = finish(c);
    if (rc) return rc;
  }
  for (int k = 0; k < g_nslot; k++) {
    CU(cudaStreamSynchronize(Ln.slot[k].st));
    if ((size_t)k < nchunks) t_timing.d2h_ms += ms_between(Ln.slot[k].ev_d0, Ln.slot[k].ev_d1);
  }
  CU(cudaGetLastError());
  if (dst_total) *dst_total = run_off;
  t_timing.kernel_launches = launches;
  t_timing.total_ms = wt.ms();
  g_ctx->launches += launches;
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
  const uint64_t bs = block_size_or_default(codec, codec_block_size);
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

// The partition step and the compression of the non-empty partitions, on device-resident records.  d_dst receives the
// .data arena (dst_cap bytes); *arena_bytes the bytes it needs.  Returns B2S_E_DST_TOO_SMALL (status[] set for the
// partitions that do not fit) when dst_cap is short.  part_start (optional) receives the R + 1 partition offsets of the
// partitioned records, which are in d_dst (codec NONE) or S.parena.
static int partition_compress_run(Device* D, Slot& S, uint32_t codec, int32_t level, uint32_t bs, uint32_t alg,
                                  uint32_t R, uint64_t n, const uint8_t* d_rec, uint64_t rec_bytes,
                                  const uint32_t* d_len, const uint32_t* d_part, uint8_t* d_dst, uint64_t dst_cap,
                                  uint64_t* dst_off, uint64_t* dst_len, uint64_t* checksum_out, int32_t* status,
                                  uint64_t* arena_bytes, uint64_t* launches,
                                  std::vector<uint64_t>* part_start = nullptr) {
  cudaStream_t st = S.st;
  std::vector<uint64_t> pstart(R), plen(R);
  CU(cudaEventRecord(S.ev_p0, st));
  CU(cudaEventRecord(S.ev_k0, st));
  PartitionPlan P;
  if (n) {
    int rc = S.pws.ensure(partition_ws_bytes(n, R));
    if (rc) return rc;
    launch_partition(d_len, d_part, n, R, (uint8_t*)S.pws.p, &P, st, launches);
    // the one readback between the partition step and compression: [bad id, byte total, partition offsets]
    rc = S.hmeta.ensure(P.readback_bytes);
    if (rc) return rc;
    const uint64_t* rb = (const uint64_t*)S.hmeta.p;
    CU(cudaMemcpyAsync(S.hmeta.p, P.readback, P.readback_bytes, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    char msg[256];
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
  } else if (rec_bytes) {
    return fail(B2S_E_ARG, "rec_len sums to 0 bytes, rec_bytes is %s", std::to_string(rec_bytes).c_str());
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
    CU(cudaEventRecord(S.ev_p1, st));
    CU(cudaEventRecord(S.ev_t0, st));
    CU(cudaEventRecord(S.ev_t1, st));
    if (alg && rec_bytes) {  // over every partition, empty ones included
      size_t ws_elems = checksum_ws_elems(R) + 4;
      int rc = S.meta.ensure(align_up((size_t)R * 8, 16) * 3 + align_up(((size_t)R + 1) * 8, 16) + ws_elems * 8 + 128);
      if (rc) return rc;
      rc = S.hmeta.ensure(align_up((size_t)R * 8, 16) * 3 + 64);
      if (rc) return rc;
      Carver hc(S.hmeta.p), dc(S.meta.p);
      uint64_t* h_off = hc.take<uint64_t>(R);
      uint64_t* h_len = hc.take<uint64_t>(R);
      uint64_t* h_out = hc.take<uint64_t>(R);
      uint64_t* d_off = dc.take<uint64_t>(R);
      uint64_t* d_slen = dc.take<uint64_t>(R);
      uint64_t* d_out = dc.take<uint64_t>(R);
      uint64_t* d_work = dc.take<uint64_t>((size_t)R + 1);
      uint64_t* d_ws = dc.take<uint64_t>(ws_elems);
      memcpy(h_off, pstart.data(), (size_t)R * 8);
      memcpy(h_len, plen.data(), (size_t)R * 8);
      CU(cudaMemcpyAsync(d_off, h_off, (size_t)R * 8, cudaMemcpyHostToDevice, st));
      CU(cudaMemcpyAsync(d_slen, h_len, (size_t)R * 8, cudaMemcpyHostToDevice, st));
      launch_checksum(D->tabs, alg, d_dst, d_off, d_slen, R, pick_tile_shift(rec_bytes), d_work, d_ws, d_out, st,
                      launches);
      CU(cudaEventRecord(S.ev_k1, st));
      CU(cudaMemcpyAsync(h_out, d_out, (size_t)R * 8, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      memcpy(checksum_out, h_out, (size_t)R * 8);
    } else {
      CU(cudaEventRecord(S.ev_k1, st));
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
  std::vector<uint64_t> ne_len(m);
  for (uint32_t k = 0; k < m; k++) ne_len[k] = plen[ne[k]];
  CompressJob J;
  uint64_t total = 0;
  if (m) {
    int rc = S.parena.ensure(rec_bytes + 64);
    if (rc) return rc;
    launch_partition_gather(d_rec, d_len, n, P, (uint8_t*)S.parena.p, st, launches);
    CU(cudaEventRecord(S.ev_p1, st));
    rc = compress_prepare(S, codec, bs, m, ne_len.data(), J);
    if (rc) return rc;
    for (uint32_t k = 0; k < m; k++) {
      J.h_src_off[k] = pstart[ne[k]];
      J.h_src_len[k] = ne_len[k];
    }
    CompressDevMeta M;
    rc = compress_enqueue(g_ctx, S, D->tabs, bs, alg, J, (const uint8_t*)S.parena.p, d_dst, dst_cap, M, launches, level);
    if (rc) return rc;
    CU(cudaEventSynchronize(S.ev_a));
    CU(cudaGetLastError());
    total = J.h_total[0] + stream_overhead(codec) * m;
  } else {
    CU(cudaEventRecord(S.ev_p1, st));
    CU(cudaEventRecord(S.ev_k0, st));
    CU(cudaEventRecord(S.ev_t0, st));
    CU(cudaEventRecord(S.ev_t1, st));
    CU(cudaEventRecord(S.ev_k1, st));
    CU(cudaStreamSynchronize(st));
  }
  *arena_bytes = total;
  bool short_dst = false;
  uint64_t at = 0;  // an empty partition sits where the next non-empty one starts
  for (uint32_t p = 0, k = 0; p < R; p++) {
    if (k < m && ne[k] == p) {
      dst_off[p] = J.h_dst_off[k];
      dst_len[p] = J.h_dst_len[k];
      checksum_out[p] = alg ? J.h_cks[k] : 0;
      status[p] = J.h_status[k];
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

static int partition_args(uint32_t codec, uint32_t bs, uint32_t alg, uint32_t R, uint64_t n, const void* rec_base,
                          uint64_t rec_bytes, const uint32_t* rec_len, const uint32_t* rec_part, const void* dst_base,
                          const uint64_t* dst_off, const uint64_t* dst_len, const int32_t* status) {
  if (alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (codec != B2S_CODEC_NONE)
    if (int rc = check_codec_block(codec, bs)) return rc;
  if (R < 1 || R > (1u << 24)) return fail(B2S_E_ARG, "num_partitions must be in [1, 2^24]%s");
  if (n > 0xffffffffull) return fail(B2S_E_ARG, "more than 2^32 - 1 records in one call%s");
  if ((n && (!rec_len || !rec_part)) || (rec_bytes && !rec_base) || !dst_off || !dst_len || !status)
    return fail(B2S_E_ARG, "null argument%s");
  if (rec_bytes && !dst_base) return fail(B2S_E_ARG, "null argument%s");
  return 0;
}

static void partition_timing(Slot& S, uint32_t codec, uint64_t n_launches, uint64_t rec_bytes, uint64_t arena) {
  add_timing(S, false);
  // kernel_ms: partition step + compression; top_kernel_ms: the codec step, or the partition step for codec NONE
  t_timing.kernel_ms = ms_between(S.ev_p0, S.ev_k1);
  if (codec == B2S_CODEC_NONE) t_timing.top_kernel_ms = ms_between(S.ev_p0, S.ev_p1);
  t_timing.kernel_launches = n_launches;
  t_timing.src_bytes = rec_bytes;
  t_timing.dst_bytes = arena;
  g_ctx->launches += n_launches;
}

int b2s_partition_compress_dev(uint32_t dev_index, uint32_t codec, int32_t level, uint32_t codec_block_size,
                               uint32_t checksum_alg, uint32_t num_partitions, uint64_t n_records,
                               const uint8_t* rec_base, uint64_t rec_bytes, const uint32_t* rec_len,
                               const uint32_t* rec_part, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off,
                               uint64_t* dst_len, uint64_t* dst_total, uint64_t* checksum_out, int32_t* status) {
  WallTimer wt;
  t_timing = b2s_timing{};
  if (dst_total) *dst_total = 0;
  const uint32_t bs = block_size_or_default(codec, codec_block_size);
  int rc = partition_args(codec, bs, checksum_alg, num_partitions, n_records, rec_base, rec_bytes, rec_len, rec_part,
                          dst_base, dst_off, dst_len, status);
  if (rc) return rc;
  Device* D;
  rc = get_device(dev_index, &D);
  if (rc) return rc;
  Lane& Ln = D->lane[kLaneWrite];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  std::vector<uint64_t> cks(num_partitions);
  uint64_t launches = 0, arena = 0;
  rc = partition_compress_run(D, S, codec, level, bs, checksum_alg, num_partitions, n_records, rec_base, rec_bytes,
                              rec_len, rec_part, dst_base, dst_cap, dst_off, dst_len, cks.data(), status, &arena,
                              &launches);
  if (rc && rc != B2S_E_DST_TOO_SMALL) return rc;
  if (checksum_out) memcpy(checksum_out, cks.data(), (size_t)num_partitions * 8);
  if (dst_total) *dst_total = arena;
  partition_timing(S, codec, launches, rec_bytes, arena);
  t_timing.total_ms = wt.ms();
  return rc;
}

// what a cached store keeps: the exchange-cache key and where to report whether it was stored
struct ExStore {
  int32_t shuffle;
  int64_t map;
  int32_t* cached;
};

static int partition_compress_packed(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
                                     uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base,
                                     uint64_t rec_bytes, const uint32_t* rec_len, const uint32_t* rec_part,
                                     uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                                     uint64_t* dst_total, uint64_t* checksum_out, int32_t* status,
                                     const ExStore* store) {
  WallTimer wt;
  t_timing = b2s_timing{};
  if (dst_total) *dst_total = 0;
  const uint32_t bs = block_size_or_default(codec, codec_block_size);
  int rc = partition_args(codec, bs, checksum_alg, num_partitions, n_records, rec_base, rec_bytes, rec_len, rec_part,
                          dst_base, dst_off, dst_len, status);
  if (rc) return rc;
  Device* D;
  rc = get_device(t_device, &D);
  if (rc) return rc;
  Lane& Ln = D->lane[kLaneWrite];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  // one upload of [records | rec_len | rec_part]; the whole map output is partitioned at once, so there is no chunking
  const size_t rec_sz = align_up(rec_bytes, 16), len_sz = align_up(n_records * 4, 16);
  rc = S.src.ensure(rec_sz + 2 * len_sz + 64);
  if (rc) return rc;
  const uint64_t bound = b2s_partition_compress_bound(codec, bs, num_partitions, rec_bytes);
  rc = S.dst.ensure(bound + 64);
  if (rc) return rc;
  uint8_t* d_rec = (uint8_t*)S.src.p;
  uint32_t* d_len = (uint32_t*)(d_rec + rec_sz);
  uint32_t* d_part = (uint32_t*)(d_rec + rec_sz + len_sz);
  cudaStream_t st = S.st;
  CU(cudaEventRecord(S.ev_h0, st));
  if (rec_bytes) CU(copy_async(d_rec, rec_base, rec_bytes, cudaMemcpyHostToDevice, st));
  if (n_records) {
    CU(cudaMemcpyAsync(d_len, rec_len, n_records * 4, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_part, rec_part, n_records * 4, cudaMemcpyHostToDevice, st));
  }
  CU(cudaEventRecord(S.ev_h1, st));
  std::vector<uint64_t> cks(num_partitions), part_start;
  uint64_t launches = 0, arena = 0;
  rc = partition_compress_run(D, S, codec, level, bs, checksum_alg, num_partitions, n_records, d_rec, rec_bytes, d_len,
                              d_part, (uint8_t*)S.dst.p, S.dst.cap, dst_off, dst_len, cks.data(), status, &arena,
                              &launches, store ? &part_start : nullptr);
  if (rc) return rc;
  // the device arena is sized by the bound, so a short caller arena shows up here: copy what fits, flag the rest
  int result = 0;
  uint64_t fit = arena;
  if (arena > dst_cap) {
    fit = dst_cap;
    for (uint32_t p = 0; p < num_partitions; p++)
      if (dst_len[p] && dst_off[p] + dst_len[p] > dst_cap) status[p] = B2S_E_DST_TOO_SMALL;
    result = fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s bytes of the .data arena", std::to_string(arena).c_str());
  }
  CU(cudaEventRecord(S.ev_d0, st));
  if (fit) CU(copy_async(dst_base, S.dst.p, fit, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(S.ev_d1, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  if (checksum_out) memcpy(checksum_out, cks.data(), (size_t)num_partitions * 8);
  if (dst_total) *dst_total = arena;
  partition_timing(S, codec, launches, rec_bytes, arena);
  t_timing.h2d_ms = ms_between(S.ev_h0, S.ev_h1);
  t_timing.d2h_ms = ms_between(S.ev_d0, S.ev_d1);
  t_timing.h2d_bytes = rec_bytes + n_records * 8;
  t_timing.d2h_bytes = fit;
  if (store && !result) {
    // the partitioned records are still in this slot (the write lane is held): in front of compression, or the arena
    // itself for codec NONE
    const uint8_t* parts = (const uint8_t*)(codec == B2S_CODEC_NONE ? S.dst.p : S.parena.p);
    *store->cached = ex_store(D->ordinal, st, store->shuffle, store->map, parts, rec_bytes, std::move(part_start));
  }
  t_timing.total_ms = wt.ms();
  return result;
}

int b2s_partition_compress_packed(uint32_t codec, int32_t level, uint32_t codec_block_size, uint32_t checksum_alg,
                                  uint32_t num_partitions, uint64_t n_records, const uint8_t* rec_base,
                                  uint64_t rec_bytes, const uint32_t* rec_len, const uint32_t* rec_part,
                                  uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_off, uint64_t* dst_len,
                                  uint64_t* dst_total, uint64_t* checksum_out, int32_t* status) {
  return partition_compress_packed(codec, level, codec_block_size, checksum_alg, num_partitions, n_records, rec_base,
                                   rec_bytes, rec_len, rec_part, dst_base, dst_cap, dst_off, dst_len, dst_total,
                                   checksum_out, status, nullptr);
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
  const ExStore store{shuffle_id, map_id, cached};
  return partition_compress_packed(codec, level, codec_block_size, checksum_alg, num_partitions, n_records, rec_base,
                                   rec_bytes, rec_len, rec_part, dst_base, dst_cap, dst_off, dst_len, dst_total,
                                   checksum_out, status, &store);
}

// ------------------------------------------------------------------------------------------------------------
// read side
// ------------------------------------------------------------------------------------------------------------
// fills the slice arrays of a job for blocks [i0, i0+cnt); dev_off = device offsets of the blocks
static void fill_slices(DecompressJob& J, uint32_t i0, uint32_t cnt, const uint64_t* dev_off, const uint64_t* src_len,
                        const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_sum) {
  uint32_t s = 0;
  for (uint32_t k = 0; k < cnt; k++) {
    J.h_slice_base[k] = s;
    if (!J.n_slices) continue;
    uint64_t o = dev_off[k];
    for (uint32_t q = slice_base[i0 + k]; q < slice_base[i0 + k + 1]; q++) {
      J.h_slice_off[s] = o;
      J.h_slice_len[s] = slice_len[q];
      J.h_slice_sum[s] = slice_sum[q];
      J.h_slice_owner[s] = k;
      o += slice_len[q];
      s++;
    }
    (void)src_len;
  }
  J.h_slice_base[cnt] = s;
}

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
  WallTimer wt;
  t_timing = b2s_timing{};
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
  const uint32_t ns = checksum_alg ? slice_base[n] : 0;
  rc = decompress_prepare(S, codec, checksum_alg, n, ns, J);
  if (rc) return rc;
  memcpy(J.h_src_off, src_off, (size_t)n * 8);
  memcpy(J.h_src_len, src_len, (size_t)n * 8);
  fill_slices(J, 0, n, src_off, src_len, slice_base, slice_len, slice_checksum);
  uint64_t srcb = 0, launches = 0;
  for (uint32_t i = 0; i < n; i++) srcb += src_len[i];
  rc = decompress_enqueue_a(S, D->tabs, checksum_alg, J, (const uint8_t*)d_src_base, srcb, &launches);
  if (rc) return rc;
  CU(cudaEventSynchronize(S.ev_a));
  rc = decompress_enqueue_b(S, J, (const uint8_t*)d_src_base, (uint8_t*)d_dst_base, dst_cap, &launches);
  if (rc) return rc;
  CU(cudaEventSynchronize(S.ev_b));
  CU(cudaGetLastError());
  memcpy(dst_off, J.h_dst_off, (size_t)n * 8);
  memcpy(dst_len, J.h_dst_len, (size_t)n * 8);
  memcpy(status, J.h_status, (size_t)n * 4);
  if (bad_slice) memcpy(bad_slice, J.h_bad, (size_t)n * 4);
  if (dst_total) *dst_total = J.total_out;
  add_timing(S, false);
  t_timing.kernel_launches = launches;
  t_timing.src_bytes = srcb;
  t_timing.dst_bytes = J.total_out;
  t_timing.total_ms = wt.ms();
  g_ctx->launches += launches;
  return 0;
}

static int decompress_host(uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* const* src,
                           const uint64_t* src_len, const uint32_t* slice_base, const uint64_t* slice_len,
                           const uint64_t* slice_sum, uint8_t* packed_dst, uint64_t packed_cap, uint8_t* const* dst,
                           const uint64_t* dst_cap, uint64_t* dst_off, uint64_t* dst_len, uint64_t* dst_total,
                           int32_t* status, int32_t* bad_slice, bool size_only) {
  WallTimer wt;
  t_timing = b2s_timing{};
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
      const b2s_timing keep = t_timing;
      rc = m ? decompress_host(codec, alg, m, sp.data(), sl.data(), sb.data(), l.data(), c.data(), packed_dst, packed_cap,
                               dst ? dp.data() : nullptr, dst_cap ? dc.data() : nullptr, doff.data(), dl.data(), &total,
                               st.data(), bd.data(), size_only)
             : 0;
      if (!m) t_timing = keep;
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
  std::vector<uint32_t> starts;
  make_chunks(n, src_len, starts);
  const size_t nchunks = starts.size() - 1;
  std::vector<DecompressJob> jobs(nchunks);
  std::vector<uint64_t> chunk_src_bytes(nchunks);
  std::vector<std::vector<Run>> runs(g_nslot);
  uint64_t launches = 0, run_off = 0;

  auto stage_a = [&](size_t c) -> int {
    Slot& S = Ln.slot[c % g_nslot];
    if (c >= (size_t)g_nslot) {
      CU(cudaStreamSynchronize(S.st));
      t_timing.d2h_ms += ms_between(S.ev_d0, S.ev_d1);
    }
    const uint32_t i0 = starts[c], cnt = starts[c + 1] - starts[c];
    DecompressJob& J = jobs[c];
    const uint32_t ns = alg ? slice_base[i0 + cnt] - slice_base[i0] : 0;
    int r = decompress_prepare(S, codec, alg, cnt, ns, J);
    if (r) return r;
    J.size_only = size_only;
    memcpy(J.h_src_len, src_len + i0, (size_t)cnt * 8);
    uint64_t bytes = plan_runs(cnt, src + i0, src_len + i0, J.h_src_off, runs[c % g_nslot]);
    chunk_src_bytes[c] = bytes;
    fill_slices(J, i0, cnt, J.h_src_off, src_len, slice_base, slice_len, slice_sum);
    r = S.src.ensure(bytes + 64);
    if (r) return r;
    CU(cudaEventRecord(S.ev_h0, S.st));
    for (const Run& q : runs[c % g_nslot])
      CU(copy_async((uint8_t*)S.src.p + q.dev_off, q.host, q.bytes, cudaMemcpyHostToDevice, S.st));
    CU(cudaEventRecord(S.ev_h1, S.st));
    t_timing.h2d_bytes += bytes;
    t_timing.src_bytes += bytes;
    return decompress_enqueue_a(S, D->tabs, alg, J, (const uint8_t*)S.src.p, bytes, &launches);
  };
  auto stage_b = [&](size_t c) -> int {
    Slot& S = Ln.slot[c % g_nslot];
    DecompressJob& J = jobs[c];
    CU(cudaEventSynchronize(S.ev_a));
    if (size_only) {
      J.total_out = J.h_totals[1];
      CU(cudaMemcpyAsync(J.h_down, J.d_down, J.down_bytes, cudaMemcpyDeviceToHost, S.st));
      CU(cudaEventRecord(S.ev_b, S.st));
      return 0;
    }
    int r = S.dst.ensure(J.h_totals[1] + 64);
    if (r) return r;
    return decompress_enqueue_b(S, J, (const uint8_t*)S.src.p, (uint8_t*)S.dst.p, S.dst.cap, &launches);
  };
  auto stage_c = [&](size_t c) -> int {
    Slot& S = Ln.slot[c % g_nslot];
    DecompressJob& J = jobs[c];
    const uint32_t i0 = starts[c];
    CU(cudaEventSynchronize(S.ev_b));
    if (!size_only) add_timing(S, true);
    CU(cudaEventRecord(S.ev_d0, S.st));
    for (uint32_t k = 0; k < J.n; k++) {
      const uint32_t i = i0 + k;
      status[i] = J.h_status[k];
      dst_len[i] = size_only ? J.h_dst_len[k] : J.h_dst_len[k];
      if (bad_slice) bad_slice[i] = J.h_bad[k];
      if (dst_off) dst_off[i] = run_off + J.h_dst_off[k];
    }
    if (size_only) {
      // h_dst_len holds olen from phase A
    } else if (packed_dst) {
      uint64_t fit = J.total_out;
      if (run_off + J.total_out > packed_cap) {
        fit = packed_cap > run_off ? packed_cap - run_off : 0;
        for (uint32_t k = 0; k < J.n; k++)
          if (status[i0 + k] == 0 && run_off + J.h_dst_off[k] + J.h_dst_len[k] > packed_cap)
            status[i0 + k] = B2S_E_DST_TOO_SMALL;
      }
      if (fit) CU(copy_async(packed_dst + run_off, S.dst.p, fit, cudaMemcpyDeviceToHost, S.st));
      t_timing.d2h_bytes += fit;
    } else {
      for (uint32_t k = 0; k < J.n; k++) {
        const uint32_t i = i0 + k;
        if (status[i] != 0 || J.h_dst_len[k] == 0) continue;
        if (J.h_dst_len[k] > dst_cap[i]) {
          status[i] = B2S_E_DST_TOO_SMALL;
          continue;
        }
        CU(cudaMemcpyAsync(dst[i], (uint8_t*)S.dst.p + J.h_dst_off[k], J.h_dst_len[k], cudaMemcpyDeviceToHost, S.st));
        t_timing.d2h_bytes += J.h_dst_len[k];
      }
    }
    CU(cudaEventRecord(S.ev_d1, S.st));
    run_off += J.total_out;
    t_timing.dst_bytes += J.total_out;
    return 0;
  };

  // software pipeline over the chunks: enqueue chunk c's upload + phase A first (never blocks on younger work), then
  // phase B of chunk c-1 (waits for its sizes), then the download of chunk c-2 (waits for its decode)
  // (lag chunks between the stages, so that lag uploads / decodes are queued on the device while the host waits for one
  // chunk's sizes — the write lane keeps g_nslot chunks in flight and would otherwise own the copy queues; needs
  // 2 * lag + 1 <= g_nslot slots)
  const size_t lag = (size_t)std::max(1, std::min(g_read_lag, (g_nslot - 1) / 2));
  for (size_t c = 0; c < nchunks + 2 * lag; c++) {
    if (c < nchunks && (rc = stage_a(c))) return rc;
    if (c >= lag && c - lag < nchunks && (rc = stage_b(c - lag))) return rc;
    if (c >= 2 * lag && c - 2 * lag < nchunks && (rc = stage_c(c - 2 * lag))) return rc;
  }
  for (int k = 0; k < g_nslot; k++) {
    CU(cudaStreamSynchronize(Ln.slot[k].st));
    if ((size_t)k < nchunks) t_timing.d2h_ms += ms_between(Ln.slot[k].ev_d0, Ln.slot[k].ev_d1);
  }
  CU(cudaGetLastError());
  if (dst_total) *dst_total = run_off;
  t_timing.kernel_launches = launches;
  t_timing.total_ms = wt.ms();
  g_ctx->launches += launches;
  return 0;
}

// builds the flattened slice arrays used by the engine from the per-block pointer form
static int flatten_slices(uint32_t n, const uint32_t* n_slices, const uint64_t* const* slice_len,
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
  return 0;
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
// read side, key-sorted: verify + decode a reduce task's blocks, then sort its fixed-size records by key
// ------------------------------------------------------------------------------------------------------------
static int sort_args(uint32_t codec, uint32_t alg, uint32_t n, const uint64_t* src_off, const uint64_t* src_len,
                     const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                     uint32_t record_bytes, uint32_t key_off, uint32_t key_len, const void* src_base,
                     const void* dst_base, uint64_t dst_cap, const uint64_t* dst_total, const uint64_t* n_records,
                     const int32_t* status) {
  if (alg > B2S_CHECKSUM_CRC32C) return fail(B2S_E_UNSUPPORTED, "Unsupported shuffle checksum algorithm%s");
  if (codec > B2S_CODEC_ZSTD) return fail(B2S_E_UNSUPPORTED, "codec %s not supported by this build", "");
  if (record_bytes == 0) return fail(B2S_E_ARG, "record_bytes must be at least 1%s");
  if (key_len < 1 || key_len > 16) return fail(B2S_E_ARG, "key_len must be in [1, 16]%s");
  if ((uint64_t)key_off + key_len > record_bytes) return fail(B2S_E_ARG, "key_off + key_len exceeds record_bytes%s");
  if (!dst_total || !n_records) return fail(B2S_E_ARG, "null argument%s");
  if (n && (!src_base || !src_off || !src_len || !status)) return fail(B2S_E_ARG, "null argument%s");
  if (dst_cap && !dst_base) return fail(B2S_E_ARG, "null argument%s");
  if (alg && n && (!slice_base || !slice_len || !slice_checksum)) return fail(B2S_E_ARG, "slice arrays required%s");
  if (alg && n) return check_slices(n, src_len, slice_base, slice_len);
  return 0;
}

// without a usable device the sort calls report B2S_E_CUDA (b2s_init has failed for that reason), otherwise as get_device
static int sort_device(uint32_t dev_index, Device** out) {
  if (!g_ctx) {
    int count = 0;
    const cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0)
      return fail(B2S_E_CUDA, "no CUDA device: %s", e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
  }
  return get_device(dev_index, out);
}

// The whole-task buffers of a sort call (read-lane slot 0: compressed blocks, decoded arena, sorted copy, sort
// workspace) only grow while they are in use.  When a call ends — whatever its result — every one of them above
// kSortKeepBytes is freed, so one oversized task does not keep several times its size of device memory for the rest
// of the process; buffers up to that size stay for the next call (a TeraSort reducer of 200 over 10 GiB needs ~55 MB).
constexpr size_t kSortKeepBytes = 1ull << 30;
struct SortBufferTrim {
  Slot& S;
  ~SortBufferTrim() {
    for (DevBuf* b : {&S.src, &S.dst, &S.parena, &S.pws})
      if (b->cap > kSortKeepBytes) b->release();
  }
};

// A source of an exchange-cache sorted read (b2s_exchange_read_sort_*): a cached range (records on the device, held by
// a reference for the call; status B2S_E_NOT_CACHED when it is not resident) or fetched block `block`.
struct SortSource {
  bool cached = false;
  int32_t status = B2S_OK;
  const uint8_t* src = nullptr;
  uint64_t len = 0;
  uint32_t block = 0;
};

// The whole reduce task on the device: compressed blocks at d_src + src_dev_off[i] (src_contiguous: back to back from
// d_src in block order, no gaps).  Phase A verifies the slices and sizes every block; a failed block, or a decoded
// length that is not a multiple of record_bytes, ends the call with status[] set and *n_rec = 0 (nothing decoded or
// sorted).  Then the blocks are decoded into S.dst (codec NONE: used in place, or copied there), their records sorted
// into *d_sorted (nullptr: into S.parena, returned there).
// mix (exchange-cache reads): the call's sources in order, the n blocks being its fetched ones; status[] / bad_slice[]
// are per source.  Every source's records land at their source-order place in S.dst: phase A's decoded offsets are
// shifted past the cached bytes in front of each block before phase B decodes, and one gather moves the cached ranges
// (codec NONE: and the fetched blocks) around them.
static int decompress_sort_run(Device* D, Slot& S, uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* d_src,
                               const uint64_t* src_dev_off, const uint64_t* src_len, bool src_contiguous,
                               const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_sum,
                               uint32_t record_bytes, uint32_t key_off, uint32_t key_len, uint8_t** d_sorted,
                               uint64_t out_cap, uint64_t* total, uint64_t* n_rec, int32_t* status, int32_t* bad_slice,
                               uint64_t* launches, const std::vector<SortSource>* mix = nullptr) {
  cudaStream_t st = S.st;
  DecompressJob J;
  int rc;
  if (n) {
    const uint32_t ns = alg ? slice_base[n] : 0;
    rc = decompress_prepare(S, codec, alg, n, ns, J, true);
    if (rc) return rc;
    memcpy(J.h_src_off, src_dev_off, (size_t)n * 8);
    memcpy(J.h_src_len, src_len, (size_t)n * 8);
    fill_slices(J, 0, n, src_dev_off, src_len, slice_base, slice_len, slice_sum);
    uint64_t srcb = 0;
    for (uint32_t i = 0; i < n; i++) srcb += src_len[i];
    rc = decompress_enqueue_a(S, D->tabs, alg, J, d_src, srcb, launches);
    if (rc) return rc;
    // the phase-A verdicts (checksums, stream headers) and decoded lengths, before anything is decoded
    CU(cudaMemcpyAsync(J.h_down, J.d_down, J.down_bytes, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
  } else {  // every source is cached
    CU(cudaEventRecord(S.ev_k0, st));
  }
  const uint32_t n_src = mix ? (uint32_t)mix->size() : n;
  auto cached = [&](uint32_t i) { return mix && (*mix)[i].cached; };
  auto block = [&](uint32_t i) { return mix ? (*mix)[i].block : i; };
  std::vector<int32_t> cached_status(n_src, B2S_OK);
  std::vector<uint64_t> place(n_src);  // each source's offset in the decoded arena
  uint64_t at = 0;
  *n_rec = 0;
  bool failed = false;
  char msg[256];
  for (uint32_t i = 0; i < n_src; i++) {
    const bool c = cached(i);
    int32_t& s = c ? cached_status[i] : J.h_status[block(i)];
    const uint64_t len = c ? (*mix)[i].len : J.h_dst_len[block(i)];
    if (c) s = (*mix)[i].status;
    if (s == B2S_OK && len % record_bytes) {
      s = B2S_E_CORRUPT;
      if (!failed) {
        snprintf(msg, sizeof msg, "%s %u %s %llu bytes, not a multiple of record_bytes %u", c ? "cached source" : "block",
                 i, c ? "holds" : "decodes to", (unsigned long long)len, record_bytes);
        fail(B2S_E_CORRUPT, "%s", msg);
      }
    }
    failed |= s != B2S_OK;
    place[i] = at;
    at += len;
  }
  *total = mix ? at : J.h_totals[1];
  auto report = [&]() {
    for (uint32_t i = 0; i < n_src; i++) {
      status[i] = cached(i) ? cached_status[i] : J.h_status[block(i)];
      if (bad_slice) bad_slice[i] = cached(i) ? -1 : J.h_bad[block(i)];
    }
  };
  auto skip_events = [&](bool decode, bool sort) -> int {  // stand-ins for the steps a call does not run
    if (decode) {
      CU(cudaEventRecord(S.ev_t0, st));
      CU(cudaEventRecord(S.ev_t1, st));
      CU(cudaEventRecord(S.ev_k1, st));
    }
    if (sort) {
      CU(cudaEventRecord(S.ev_p0, st));
      CU(cudaEventRecord(S.ev_p1, st));
    }
    CU(cudaStreamSynchronize(st));
    return 0;
  };
  if (failed) {
    report();
    return skip_events(true, true);
  }
  const uint64_t records = *total / record_bytes;
  if (records > 0xffffffffull)
    return fail(B2S_E_ARG, "more than 2^32 - 1 records in one call (%s bytes)", std::to_string(*total).c_str());
  if (*total > out_cap) {
    report();
    return fail(B2S_E_DST_TOO_SMALL, "dst_cap is below the %s decoded bytes", std::to_string(*total).c_str());
  }

  // the decoded arena: every block's records back to back in block order
  const uint8_t* arena = d_src;
  if (mix) {
    if ((rc = S.dst.ensure(*total + 64))) return rc;
    arena = (const uint8_t*)S.dst.p;
    std::vector<ExchangePiece> pieces;
    for (uint32_t i = 0; i < n_src; i++) {
      const SortSource& s = (*mix)[i];
      if (s.cached)
        exchange_add_pieces(pieces, s.src, place[i], s.len);
      else if (codec == B2S_CODEC_NONE)
        exchange_add_pieces(pieces, d_src + src_dev_off[s.block], place[i], src_len[s.block]);
      else
        J.h_dst_off[s.block] = place[i];
    }
    if (n && codec != B2S_CODEC_NONE)  // phase B decodes every block straight to its place among the cached ranges
      CU(cudaMemcpyAsync(J.dst_off, J.h_dst_off, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    if (!pieces.empty()) {
      if ((rc = S.xpieces.ensure(pieces.size() * sizeof(ExchangePiece)))) return rc;
      CU(cudaMemcpyAsync(S.xpieces.p, pieces.data(), pieces.size() * sizeof(ExchangePiece), cudaMemcpyHostToDevice,
                         st));
      launch_exchange_gather((const ExchangePiece*)S.xpieces.p, (uint32_t)pieces.size(), (uint8_t*)S.dst.p, st,
                             launches);
    }
  }
  if (codec == B2S_CODEC_NONE || !n) {
    if (!mix && !src_contiguous && *total) {
      if ((rc = S.dst.ensure(*total + 64))) return rc;
      for (uint32_t i = 0; i < n; i++)
        if (src_len[i])
          CU(cudaMemcpyAsync((uint8_t*)S.dst.p + J.h_dst_off[i], d_src + src_dev_off[i], src_len[i],
                             cudaMemcpyDeviceToDevice, st));
      arena = (const uint8_t*)S.dst.p;
    }
    if ((rc = skip_events(true, false))) return rc;
  } else {
    if (!mix && (rc = S.dst.ensure(*total + 64))) return rc;
    rc = decompress_enqueue_b(S, J, d_src, (uint8_t*)S.dst.p, S.dst.cap, launches);
    if (rc) return rc;
    CU(cudaEventSynchronize(S.ev_b));
    CU(cudaGetLastError());
    for (uint32_t i = 0; i < n; i++) failed |= J.h_status[i] != B2S_OK;
    if (failed) {
      report();
      return skip_events(false, true);
    }
    arena = (const uint8_t*)S.dst.p;
  }
  report();

  if (!*d_sorted) {
    if ((rc = S.parena.ensure(*total + 64))) return rc;
    *d_sorted = (uint8_t*)S.parena.p;
  }
  if (records && (rc = S.pws.ensure(key_sort_ws_bytes(records, key_len)))) return rc;
  CU(cudaEventRecord(S.ev_p0, st));
  launch_key_sort(arena, records, record_bytes, key_off, key_len, (uint8_t*)S.pws.p, *d_sorted, st, launches);
  CU(cudaEventRecord(S.ev_p1, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  *n_rec = records;
  return 0;
}

// kernel_ms: verification + decode + sort; top_kernel_ms: the sort step
static void sort_timing(Slot& S, uint64_t n_launches, uint64_t src_bytes, uint64_t total) {
  add_timing(S, false);
  t_timing.kernel_ms = ms_between(S.ev_k0, S.ev_p1);
  t_timing.top_kernel_ms = ms_between(S.ev_p0, S.ev_p1);
  t_timing.kernel_launches = n_launches;
  t_timing.src_bytes = src_bytes;
  t_timing.dst_bytes = total;
  g_ctx->launches += n_launches;
}

// decompress_sort on the read lane of D over device-resident blocks, sorted into dst_base (device memory)
static int sort_dev_run(Device* D, uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* src_base,
                        const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                        const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t record_bytes,
                        uint32_t key_off, uint32_t key_len, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
                        uint64_t* n_records, int32_t* status, int32_t* bad_slice, const WallTimer& wt,
                        const std::vector<SortSource>* mix = nullptr) {
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  SortBufferTrim trim{S};
  uint64_t launches = 0, srcb = 0;
  for (uint32_t i = 0; i < n; i++) srcb += src_len[i];
  uint8_t* out = dst_base;
  int rc = decompress_sort_run(D, S, codec, alg, n, src_base, src_off, src_len, false, slice_base, slice_len,
                               slice_checksum, record_bytes, key_off, key_len, &out, dst_cap, dst_total, n_records,
                               status, bad_slice, &launches, mix);
  if (rc) return rc;
  sort_timing(S, launches, srcb, *dst_total);
  t_timing.total_ms = wt.ms();
  return 0;
}

// decompress_sort on the read lane of D over host blocks: one upload, the sort, one download into dst_base
static int sort_packed_run(Device* D, uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* src_base,
                           const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                           const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t record_bytes,
                           uint32_t key_off, uint32_t key_len, uint8_t* dst_base, uint64_t dst_cap,
                           uint64_t* dst_total, uint64_t* n_records, int32_t* status, int32_t* bad_slice,
                           const WallTimer& wt, const std::vector<SortSource>* mix = nullptr) {
  Lane& Ln = D->lane[kLaneRead];
  std::lock_guard<std::mutex> lk(Ln.mtx);
  Slot& S = Ln.slot[0];
  SortBufferTrim trim{S};
  // one upload of every block, back to back (the whole task is resident at once: no chunking)
  std::vector<uint64_t> dev_off(n);
  uint64_t srcb = 0;
  for (uint32_t i = 0; i < n; i++) {
    dev_off[i] = srcb;
    srcb += src_len[i];
  }
  int rc;
  if ((rc = S.src.ensure(srcb + 64))) return rc;
  cudaStream_t st = S.st;
  CU(cudaEventRecord(S.ev_h0, st));
  for (uint32_t i = 0; i < n;) {  // blocks adjacent in host memory go up in one copy
    uint32_t j = i + 1;
    while (j < n && src_off[j] == src_off[j - 1] + src_len[j - 1]) j++;
    const uint64_t bytes = dev_off[j - 1] + src_len[j - 1] - dev_off[i];
    if (bytes) CU(copy_async((uint8_t*)S.src.p + dev_off[i], src_base + src_off[i], bytes, cudaMemcpyHostToDevice, st));
    i = j;
  }
  CU(cudaEventRecord(S.ev_h1, st));
  uint64_t launches = 0;
  uint8_t* sorted = nullptr;
  rc = decompress_sort_run(D, S, codec, alg, n, (const uint8_t*)S.src.p, dev_off.data(), src_len, true, slice_base,
                           slice_len, slice_checksum, record_bytes, key_off, key_len, &sorted, dst_cap, dst_total,
                           n_records, status, bad_slice, &launches, mix);
  if (rc) return rc;
  const uint64_t down = *n_records ? *dst_total : 0;
  CU(cudaEventRecord(S.ev_d0, st));
  if (down) CU(copy_async(dst_base, sorted, down, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(S.ev_d1, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  sort_timing(S, launches, srcb, *dst_total);
  t_timing.h2d_ms = ms_between(S.ev_h0, S.ev_h1);
  t_timing.d2h_ms = ms_between(S.ev_d0, S.ev_d1);
  t_timing.h2d_bytes = srcb;
  t_timing.d2h_bytes = down;
  t_timing.total_ms = wt.ms();
  return 0;
}

int b2s_decompress_sort_dev(uint32_t dev_index, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                            const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                            const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                            uint32_t record_bytes, uint32_t key_off, uint32_t key_len, uint8_t* dst_base,
                            uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                            int32_t* bad_slice) {
  WallTimer wt;
  t_timing = b2s_timing{};
  if (dst_total) *dst_total = 0;
  if (n_records) *n_records = 0;
  Device* D;
  int rc = sort_device(dev_index, &D);
  if (rc) return rc;
  rc = sort_args(codec, checksum_alg, n, src_off, src_len, slice_base, slice_len, slice_checksum, record_bytes, key_off,
                 key_len, src_base, dst_base, dst_cap, dst_total, n_records, status);
  if (rc || !n) return rc;
  return sort_dev_run(D, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len, slice_checksum,
                      record_bytes, key_off, key_len, dst_base, dst_cap, dst_total, n_records, status, bad_slice, wt);
}

int b2s_decompress_sort_packed(uint32_t codec, uint32_t checksum_alg, uint32_t n, const uint8_t* src_base,
                               const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                               const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t record_bytes,
                               uint32_t key_off, uint32_t key_len, uint8_t* dst_base, uint64_t dst_cap,
                               uint64_t* dst_total, uint64_t* n_records, int32_t* status, int32_t* bad_slice) {
  WallTimer wt;
  t_timing = b2s_timing{};
  if (dst_total) *dst_total = 0;
  if (n_records) *n_records = 0;
  Device* D;
  int rc = sort_device(t_device, &D);
  if (rc) return rc;
  rc = sort_args(codec, checksum_alg, n, src_off, src_len, slice_base, slice_len, slice_checksum, record_bytes, key_off,
                 key_len, src_base, dst_base, dst_cap, dst_total, n_records, status);
  if (rc || !n) return rc;
  return sort_packed_run(D, codec, checksum_alg, n, src_base, src_off, src_len, slice_base, slice_len, slice_checksum,
                         record_bytes, key_off, key_len, dst_base, dst_cap, dst_total, n_records, status, bad_slice,
                         wt);
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
  WallTimer wt;
  t_timing = b2s_timing{};
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
  CU(cudaEventRecord(S.ev_k0, st));
  CU(cudaEventRecord(S.ev_t0, st));
  if (!pieces.empty()) {
    CU(cudaMemcpyAsync(S.xpieces.p, pieces.data(), pieces.size() * sizeof(ExchangePiece), cudaMemcpyHostToDevice, st));
    launch_exchange_gather((const ExchangePiece*)S.xpieces.p, (uint32_t)pieces.size(), (uint8_t*)S.dst.p, st,
                           &launches);
  }
  CU(cudaEventRecord(S.ev_t1, st));
  CU(cudaEventRecord(S.ev_k1, st));
  CU(cudaEventRecord(S.ev_d0, st));
  if (total) CU(copy_async(dst_base, S.dst.p, total, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(S.ev_d1, st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  add_timing(S, false);
  t_timing.d2h_ms = ms_between(S.ev_d0, S.ev_d1);
  t_timing.d2h_bytes = total;
  t_timing.kernel_launches = launches;
  t_timing.src_bytes = total;
  t_timing.dst_bytes = total;
  t_timing.total_ms = wt.ms();
  g_ctx->launches += launches;
  return 0;
}

// The sources of an exchange sorted read: the fetched ones compacted in source order with their slices (what
// decompress_sort_run takes as its blocks), and every source in order.
struct MixedSources {
  std::vector<SortSource> src;
  std::vector<uint64_t> off, len, slice_len, slice_sum;
  std::vector<uint32_t> slice_base{0};
};

static int exchange_sort_args(int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids, const uint8_t* cached,
                              uint32_t codec, uint32_t alg, uint32_t n, const uint8_t* src_base,
                              const uint64_t* src_off, const uint64_t* src_len, const uint32_t* slice_base,
                              const uint64_t* slice_len, const uint64_t* slice_checksum, uint32_t record_bytes,
                              uint32_t key_off, uint32_t key_len, const void* dst_base, uint64_t dst_cap,
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
                   M.slice_sum.data(), record_bytes, key_off, key_len, src_base, dst_base, dst_cap, dst_total,
                   n_records, status);
}

// references the cached sources of M on device D and describes them; B2S_E_ARG when a range exceeds an entry
static int exchange_sort_sources(const ExRefs& refs, int32_t start_reduce, int32_t end_reduce, MixedSources& M) {
  if (int rc = refs.check_range(end_reduce)) return rc;
  for (uint32_t i = 0; i < (uint32_t)M.src.size(); i++) {
    SortSource& s = M.src[i];
    if (!s.cached) continue;
    if (refs.entry[i]) s.src = refs.range(i, start_reduce, end_reduce, &s.len);
    else s.status = B2S_E_NOT_CACHED;
  }
  return 0;
}

int b2s_exchange_read_sort_packed(int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce, const int64_t* map_ids,
                                  const uint8_t* cached, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                  const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                                  const uint32_t* slice_base, const uint64_t* slice_len,
                                  const uint64_t* slice_checksum, uint32_t record_bytes, uint32_t key_off,
                                  uint32_t key_len, uint8_t* dst_base, uint64_t dst_cap, uint64_t* dst_total,
                                  uint64_t* n_records, int32_t* status, int32_t* bad_slice) {
  WallTimer wt;
  t_timing = b2s_timing{};
  if (dst_total) *dst_total = 0;
  if (n_records) *n_records = 0;
  MixedSources M;
  int rc = exchange_sort_args(start_reduce, end_reduce, map_ids, cached, codec, checksum_alg, n, src_base, src_off,
                              src_len, slice_base, slice_len, slice_checksum, record_bytes, key_off, key_len, dst_base,
                              dst_cap, dst_total, n_records, status, M);
  if (rc) return rc;
  if ((rc = exchange_ready())) return rc;
  Device* D;
  if ((rc = get_device(t_device, &D)) || !n) return rc;
  ExRefs refs(D->ordinal, shuffle_id, n, map_ids, cached);
  if ((rc = exchange_sort_sources(refs, start_reduce, end_reduce, M))) return rc;
  const uint32_t m = (uint32_t)M.off.size();
  return sort_packed_run(D, codec, checksum_alg, m, src_base, M.off.data(), M.len.data(), M.slice_base.data(),
                         M.slice_len.data(), M.slice_sum.data(), record_bytes, key_off, key_len, dst_base, dst_cap,
                         dst_total, n_records, status, bad_slice, wt, &M.src);
}

int b2s_exchange_read_sort_dev(uint32_t dev_index, int32_t shuffle_id, int32_t start_reduce, int32_t end_reduce,
                               const int64_t* map_ids, const uint8_t* cached, uint32_t codec, uint32_t checksum_alg,
                               uint32_t n, const uint8_t* src_base, const uint64_t* src_off, const uint64_t* src_len,
                               const uint32_t* slice_base, const uint64_t* slice_len, const uint64_t* slice_checksum,
                               uint32_t record_bytes, uint32_t key_off, uint32_t key_len, uint8_t* dst_base,
                               uint64_t dst_cap, uint64_t* dst_total, uint64_t* n_records, int32_t* status,
                               int32_t* bad_slice) {
  WallTimer wt;
  t_timing = b2s_timing{};
  if (dst_total) *dst_total = 0;
  if (n_records) *n_records = 0;
  MixedSources M;
  int rc = exchange_sort_args(start_reduce, end_reduce, map_ids, cached, codec, checksum_alg, n, src_base, src_off,
                              src_len, slice_base, slice_len, slice_checksum, record_bytes, key_off, key_len, dst_base,
                              dst_cap, dst_total, n_records, status, M);
  if (rc) return rc;
  if ((rc = exchange_ready())) return rc;
  Device* D;
  if ((rc = get_device(dev_index, &D)) || !n) return rc;
  ExRefs refs(D->ordinal, shuffle_id, n, map_ids, cached);
  if ((rc = exchange_sort_sources(refs, start_reduce, end_reduce, M))) return rc;
  const uint32_t m = (uint32_t)M.off.size();
  return sort_dev_run(D, codec, checksum_alg, m, src_base, M.off.data(), M.len.data(), M.slice_base.data(),
                      M.slice_len.data(), M.slice_sum.data(), record_bytes, key_off, key_len, dst_base, dst_cap,
                      dst_total, n_records, status, bad_slice, wt, &M.src);
}

int b2s_decompressed_size_batch(uint32_t codec, uint32_t n, const uint8_t* const* src, const uint64_t* src_len,
                                uint64_t* out_len, int32_t* status) {
  if (n && (!src || !src_len || !out_len || !status)) return fail(B2S_E_ARG, "null argument%s");
  return decompress_host(codec, 0, n, src, src_len, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr,
                         out_len, nullptr, status, nullptr, true);
}

}  // extern "C"
