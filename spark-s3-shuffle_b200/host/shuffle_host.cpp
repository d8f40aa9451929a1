// shuffle_host.cpp — host-side mirror (C++) of the reference's plugin classes on the codec path, above the C ABI.
// See include/b200shuffle_host.h for the class ↔ reference file:line map.  Only file:// roots; S3 I/O is out of scope.
#include "../../include/b200shuffle_host.h"

#include <sys/stat.h>
#include <unistd.h>

#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <map>
#include <memory>
#include <mutex>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/b200shuffle.h"

namespace b2s {
namespace host {

// ---- exception types named after what the reference throws -----------------------------------------------
struct RuntimeException : std::runtime_error { using std::runtime_error::runtime_error; };
struct IOException : std::runtime_error { using std::runtime_error::runtime_error; };
struct SparkException : std::runtime_error { using std::runtime_error::runtime_error; };
struct UnsupportedOperationException : std::runtime_error { using std::runtime_error::runtime_error; };
struct CodecException : std::runtime_error { using std::runtime_error::runtime_error; };

// ---- block ids (org.apache.spark.storage.BlockId names) ---------------------------------------------------
struct BlockId {
  enum Kind { Shuffle, ShuffleBatch, Data, Index, Checksum } kind;
  int32_t shuffleId;
  int64_t mapId;
  int32_t reduceId;     // start reduce id for ShuffleBatch
  int32_t endReduceId;  // ShuffleBatch only
  std::string name() const {
    std::ostringstream o;
    o << "shuffle_" << shuffleId << "_" << mapId << "_" << reduceId;
    switch (kind) {
      case ShuffleBatch: o << "_" << endReduceId; break;
      case Data: o << ".data"; break;
      case Index: o << ".index"; break;
      case Checksum: o << ".checksum"; break;
      default: break;
    }
    return o.str();
  }
};

// ---- pinned byte arena (what the JVM side wraps as a direct ByteBuffer) --------------------------------------
class PinnedArena {
 public:
  ~PinnedArena() { release(p_, pinned_); }
  uint8_t* data() { return p_; }
  uint64_t size() const { return n_; }
  uint64_t capacity() const { return cap_; }
  void clear() { n_ = 0; }
  void reserve(uint64_t cap) {
    if (cap <= cap_) return;
    uint64_t nc = cap_ ? cap_ : (1u << 20);
    while (nc < cap) nc *= 2;
    // Pinned when a CUDA device exists; plain heap otherwise so that pass-through mode (bytes already compressed
    // upstream, no codec call) still works on a GPU-less box.  This is memory only: compute has no CPU fallback.
    bool pinned = true;
    uint8_t* q = (uint8_t*)b2s_host_alloc(nc);
    if (!q) {
      pinned = false;
      q = (uint8_t*)malloc(nc);
      if (!q) throw CodecException("out of host memory");
    }
    if (n_) memcpy(q, p_, n_);
    release(p_, pinned_);
    p_ = q;
    pinned_ = pinned;
    cap_ = nc;
  }
  void append(const uint8_t* b, uint64_t n) {
    reserve(n_ + n);
    memcpy(p_ + n_, b, n);
    n_ += n;
  }
  void resize(uint64_t n) {
    reserve(n);
    n_ = n;
  }

 private:
  static void release(uint8_t* p, bool pinned) {
    if (!p) return;
    if (pinned) b2s_host_free(p); else free(p);
  }
  uint8_t* p_ = nullptr;
  uint64_t n_ = 0, cap_ = 0;
  bool pinned_ = false;
};

static void mkdirs(const std::string& dir) {
  std::string cur;
  for (size_t i = 0; i < dir.size(); i++) {
    cur.push_back(dir[i]);
    if (dir[i] == '/' || i + 1 == dir.size()) {
      if (cur.size() > 1 && mkdir(cur.c_str(), 0777) != 0 && errno != EEXIST)
        throw IOException("mkdir " + cur + ": " + strerror(errno));
    }
  }
}

}  // namespace host
}  // namespace b2s
#include "streams.h"
#include "codec_adapter.h"
#include "coalesce.h"
namespace b2s {
namespace host {

// ---- S3ShuffleDispatcher (helper/S3ShuffleDispatcher.scala) -------------------------------------------------
class S3ShuffleDispatcher {
 public:
  explicit S3ShuffleDispatcher(const std::string& conf_text) {
    std::istringstream in(conf_text);
    std::string line;
    while (std::getline(in, line)) {
      size_t eq = line.find('=');
      if (eq == std::string::npos) continue;
      conf_[line.substr(0, eq)] = line.substr(eq + 1);
    }
    appId = get("spark.app.id", "app-local");
    std::string rd = get("spark.shuffle.s3.rootDir", "sparkS3shuffle/");  // :50
    rootDir = (!rd.empty() && rd.back() == '/') ? rd : rd + "/";            // :51
    rootIsLocal = rootDir.rfind("file:", 0) == 0;                            // :52
    bufferSize = getInt("spark.shuffle.s3.bufferSize", 8 * 1024 * 1024);
    maxBufferSizeTask = getInt("spark.shuffle.s3.maxBufferSizeTask", 128 * 1024 * 1024);
    maxConcurrencyTask = getInt("spark.shuffle.s3.maxConcurrencyTask", 10);
    cachePartitionLengths = getBool("spark.shuffle.s3.cachePartitionLengths", true);
    cacheChecksums = getBool("spark.shuffle.s3.cacheChecksums", true);
    cleanupShuffleFiles = getBool("spark.shuffle.s3.cleanup", true);
    folderPrefixes = getInt("spark.shuffle.s3.folderPrefixes", 10);
    alwaysCreateIndex = getBool("spark.shuffle.s3.alwaysCreateIndex", false);
    forceBatchFetch = getBool("spark.shuffle.s3.forceBatchFetch", false);
    checksumAlgorithm = get("spark.shuffle.checksum.algorithm", "ADLER32");  // Spark 3.5 default [U]
    checksumEnabled = getBool("spark.shuffle.checksum.enabled", true);
    shuffleCompress = getBool("spark.shuffle.compress", true);
    codecName = get("spark.io.compression.codec", "lz4");
    lz4BlockSize = (uint32_t)getSize("spark.io.compression.lz4.blockSize", 32 * 1024);
    zstdLevel = getInt("spark.io.compression.zstd.level", 1);  // Spark's default [U]; reaches b2s_compress_* as `level`
    gpuEnabled = getBool("spark.shuffle.s3.gpu.enabled", true);  // additive key (SURVEY.md §5 config row)
    gpuCodecBufferSize = (uint64_t)getSize("spark.shuffle.s3.gpu.codecBufferSize", 64L * 1024 * 1024);  // additive
    gpuReadBatchBlocks = getInt("spark.shuffle.s3.gpu.readBatchBlocks", 0);  // additive; 0 = all completed blocks
    gpuCoalesce = getBool("spark.shuffle.s3.gpu.coalesce", false);  // additive: group-commit the calls of concurrent task threads
    // additive: per-device bytes of map outputs kept in HBM for reducers on the same device (INTEGRATION.md §3f); 0 = off
    gpuExchangeCacheBytes = (uint64_t)std::max(0L, getSize("spark.shuffle.s3.gpu.exchangeCacheBytes", 0));
    if (!rootIsLocal && rootDir.find("://") != std::string::npos)
      throw UnsupportedOperationException("only file:// roots are implemented by the host mirror: " + rootDir);
  }

  std::string localRoot() const { return rootIsLocal ? rootDir.substr(rootDir.find(':') + 1 + (rootDir.compare(5, 2, "//") == 0 ? 2 : 0)) : rootDir; }

  // :120-144  ${rootDir}${mapId % folderPrefixes}/${appId}/${shuffleId}/${blockId.name}
  std::string getPath(const BlockId& b) const {
    std::ostringstream o;
    o << localRoot() << (b.mapId % folderPrefixes) << "/" << appId << "/" << b.shuffleId << "/" << b.name();
    return o.str();
  }
  std::string shuffleDir(int64_t prefix, int32_t shuffleId) const {
    std::ostringstream o;
    o << localRoot() << prefix << "/" << appId << "/" << shuffleId;
    return o.str();
  }
  // :174-188 removeShuffle: every prefix folder
  void removeShuffle(int32_t shuffleId) const {
    // fs.delete(path, true) in the reference — no shell involved.  rootDir / app id come from user configuration: an
    // empty, relative or "/" root would aim a recursive delete at the working directory or the file system root.
    namespace fs = std::filesystem;
    const std::string root = localRoot();
    if (root.empty() || root[0] != '/' || fs::path(root).lexically_normal() == fs::path("/") || appId.empty() ||
        appId.find('/') != std::string::npos)
      return;
    for (int i = 0; i < folderPrefixes; i++) {
      std::error_code ec;
      fs::remove_all(fs::path(shuffleDir(i, shuffleId)), ec);  // like the reference: failures are only logged
    }
  }
  // the exchange-cache budget on every device, once the codec runtime is up (the writer stores, the reader looks up)
  void applyExchangeBudget() {
    std::call_once(exchangeBudgetSet_, [&] {
      const int n = b2s_device_count();
      for (int i = 0; i < n; i++) {
        const int rc = b2s_exchange_set_budget((uint32_t)i, gpuExchangeCacheBytes);
        if (rc != 0)
          throw CodecException(std::string("b2s_exchange_set_budget: ") + b2s_strerror(rc) + ": " + b2s_last_error());
      }
    });
  }
  int codecId() const {
    if (!shuffleCompress) return B2S_CODEC_NONE;
    if (codecName == "lz4" || codecName == "org.apache.spark.io.LZ4CompressionCodec") return B2S_CODEC_LZ4BLOCK;
    if (codecName == "snappy") return B2S_CODEC_SNAPPY_XERIAL;
    if (codecName == "zstd") return B2S_CODEC_ZSTD;
    throw UnsupportedOperationException("Unsupported compression codec: " + codecName);
  }

  std::string appId, rootDir, checksumAlgorithm, codecName;
  bool rootIsLocal = false, cachePartitionLengths = true, cacheChecksums = true, cleanupShuffleFiles = true,
       alwaysCreateIndex = false, forceBatchFetch = false, checksumEnabled = true, shuffleCompress = true,
       gpuEnabled = true;
  int bufferSize = 0, maxBufferSizeTask = 0, maxConcurrencyTask = 0, folderPrefixes = 10;
  uint32_t lz4BlockSize = 32768;
  int zstdLevel = 1;
  uint64_t gpuCodecBufferSize = 64ull << 20;
  int gpuReadBatchBlocks = 0;
  bool gpuCoalesce = false;
  uint64_t gpuExchangeCacheBytes = 0;
  CoalescingQueue queue;  // one per dispatcher = one per executor JVM (helper/S3ShuffleDispatcher.scala:240-254)

  // caches of S3ShuffleHelper (helper/S3ShuffleHelper.scala:15-16) live with the dispatcher instance here
  std::mutex cacheMutex;
  std::map<std::string, std::vector<int64_t>> cachedArrayLengths, cachedChecksums;

 private:
  std::string get(const std::string& k, const std::string& d) const {
    auto it = conf_.find(k);
    return it == conf_.end() ? d : it->second;
  }
  int getInt(const std::string& k, int d) const {
    auto it = conf_.find(k);
    return it == conf_.end() ? d : atoi(it->second.c_str());
  }
  long getSize(const std::string& k, long d) const {
    auto it = conf_.find(k);
    if (it == conf_.end()) return d;
    char* end = nullptr;
    long v = strtol(it->second.c_str(), &end, 10);
    if (end && (*end == 'k' || *end == 'K')) v *= 1024;
    if (end && (*end == 'm' || *end == 'M')) v *= 1024 * 1024;
    return v;
  }
  bool getBool(const std::string& k, bool d) const {
    auto it = conf_.find(k);
    return it == conf_.end() ? d : (it->second == "true" || it->second == "1");
  }
  std::map<std::string, std::string> conf_;
  std::once_flag exchangeBudgetSet_;
};

// ---- S3ShuffleHelper (helper/S3ShuffleHelper.scala) ---------------------------------------------------------
class S3ShuffleHelper {
 public:
  // :94-103 (+ "CRC32C", the case the Scala shim adds)
  static uint32_t createChecksumAlgorithm(const std::string& algorithm) {
    if (algorithm == "ADLER32") return B2S_CHECKSUM_ADLER32;
    if (algorithm == "CRC32") return B2S_CHECKSUM_CRC32;
    if (algorithm == "CRC32C") return B2S_CHECKSUM_CRC32C;
    throw UnsupportedOperationException("Unsupported shuffle checksum algorithm: " + algorithm + ".");
  }
  static int64_t emptyChecksum(uint32_t alg) { return alg == B2S_CHECKSUM_ADLER32 ? 1 : 0; }

  // :44-47  Array(0) ++ lengths.tail.scan(lengths.head)(_ + _)
  static void writePartitionLengths(S3ShuffleDispatcher& d, int32_t shuffleId, int64_t mapId,
                                    const std::vector<int64_t>& lengths) {
    std::vector<int64_t> acc(lengths.size() + 1, 0);
    for (size_t i = 0; i < lengths.size(); i++) acc[i + 1] = acc[i] + lengths[i];
    writeArrayAsBlock(d, BlockId{BlockId::Index, shuffleId, mapId, 0, 0}, acc);
  }
  // :49-51
  static void writeChecksum(S3ShuffleDispatcher& d, int32_t shuffleId, int64_t mapId,
                            const std::vector<int64_t>& checksums) {
    writeArrayAsBlock(d, BlockId{BlockId::Checksum, shuffleId, mapId, 0, 0}, checksums);
  }
  // :53-59 DataOutputStream.writeLong = big endian
  static void writeArrayAsBlock(S3ShuffleDispatcher& d, const BlockId& b, const std::vector<int64_t>& a) {
    std::string path = d.getPath(b);
    mkdirs(path.substr(0, path.rfind('/')));
    std::ofstream f(path, std::ios::binary | std::ios::trunc);
    if (!f) throw IOException("cannot create " + path);
    for (int64_t v : a) {
      unsigned char be[8];
      for (int k = 0; k < 8; k++) be[k] = (unsigned char)((uint64_t)v >> (56 - 8 * k));
      f.write((const char*)be, 8);
    }
  }
  // :105-121
  static std::vector<int64_t> readBlockAsArray(S3ShuffleDispatcher& d, const BlockId& b) {
    std::string path = d.getPath(b);
    std::ifstream f(path, std::ios::binary | std::ios::ate);
    if (!f) throw IOException("File does not exist: " + path);
    std::streamoff len = f.tellg();
    if (len % 8 != 0) throw SparkException("Unexpected file length when reading " + b.name());  // :112-114
    f.seekg(0);
    std::vector<int64_t> out((size_t)(len / 8));
    for (auto& v : out) {
      unsigned char be[8];
      f.read((char*)be, 8);
      uint64_t x = 0;
      for (int k = 0; k < 8; k++) x = (x << 8) | be[k];
      v = (int64_t)x;
    }
    return out;
  }
  // :67-92 cached readers
  static std::vector<int64_t> getPartitionLengths(S3ShuffleDispatcher& d, int32_t shuffleId, int64_t mapId) {
    BlockId b{BlockId::Index, shuffleId, mapId, 0, 0};
    if (!d.cachePartitionLengths) return readBlockAsArray(d, b);
    std::lock_guard<std::mutex> lk(d.cacheMutex);
    auto it = d.cachedArrayLengths.find(b.name());
    if (it == d.cachedArrayLengths.end()) it = d.cachedArrayLengths.emplace(b.name(), readBlockAsArray(d, b)).first;
    return it->second;
  }
  static std::vector<int64_t> getChecksums(S3ShuffleDispatcher& d, int32_t shuffleId, int64_t mapId) {
    BlockId b{BlockId::Checksum, shuffleId, mapId, 0, 0};
    if (!d.cacheChecksums) return readBlockAsArray(d, b);
    std::lock_guard<std::mutex> lk(d.cacheMutex);
    auto it = d.cachedChecksums.find(b.name());
    if (it == d.cachedChecksums.end()) it = d.cachedChecksums.emplace(b.name(), readBlockAsArray(d, b)).first;
    return it->second;
  }
  static void purgeCachedDataForShuffle(S3ShuffleDispatcher& d, int32_t shuffleId) {  // :22-31
    std::lock_guard<std::mutex> lk(d.cacheMutex);
    std::string pre = "shuffle_" + std::to_string(shuffleId) + "_";
    for (auto* m : {&d.cachedArrayLengths, &d.cachedChecksums})
      for (auto it = m->begin(); it != m->end();) it = (it->first.rfind(pre, 0) == 0) ? m->erase(it) : std::next(it);
  }
};

static void ensure_codec_runtime() {
  int rc = b2s_init(0, 0, 0);
  if (rc != 0) throw CodecException(std::string("b2s_init: ") + b2s_strerror(rc) + ": " + b2s_last_error());
}

static void submit_or_throw(CoalescingQueue& q, CodecRequest& r, const char* what) {
  const int rc = q.submit(r);
  if (rc != 0) throw CodecException(std::string(what) + ": " + b2s_strerror(rc) + ": " + r.error);
}

// The output half of commitAllPartitions (shuffle/S3ShuffleMapOutputWriter.scala:91-118): the .data object from
// `segments` (its bytes in order, data_len in all; created when createData), then .index and .checksum.
static void writeMapOutput(S3ShuffleDispatcher& d, int32_t shuffleId, int64_t mapId, bool createData,
                           const std::vector<std::pair<const uint8_t*, uint64_t>>& segments, uint64_t data_len,
                           const std::vector<int64_t>& partitionLengths, const std::vector<int64_t>& checksums,
                           std::unique_ptr<S3MeasureOutputStream>& measure) {
  int64_t sum = 0;
  for (int64_t v : partitionLengths) sum += v;
  if ((int64_t)data_len != sum)
    throw RuntimeException("S3ShuffleMapOutputWriter: Unexpected output length " + std::to_string(data_len) +
                           ", expected: " + std::to_string(sum) + ".");
  if (createData) {
    std::string path = d.getPath(BlockId{BlockId::Data, shuffleId, mapId, 0, 0});
    mkdirs(path.substr(0, path.rfind('/')));
    // initStream (:43-49): BufferedOutputStream(S3MeasureOutputStream(createBlock(shuffleBlock), name), bufferSize)
    measure.reset(new S3MeasureOutputStream(path, BlockId{BlockId::Data, shuffleId, mapId, 0, 0}.name(),
                                            (size_t)d.bufferSize));
    for (auto& sg : segments) measure->write(sg.first, sg.second);
    measure->flush();  // :102-107
    measure->close();
  }
  if (sum > 0 || d.alwaysCreateIndex) {  // :111
    S3ShuffleHelper::writePartitionLengths(d, shuffleId, mapId, partitionLengths);
    if (d.checksumEnabled) S3ShuffleHelper::writeChecksum(d, shuffleId, mapId, checksums);
  }
}

// ---- S3ShuffleMapOutputWriter (shuffle/S3ShuffleMapOutputWriter.scala) --------------------------------------
class S3ShuffleMapOutputWriter {
 public:
  S3ShuffleMapOutputWriter(S3ShuffleDispatcher& d, int32_t shuffleId, int64_t mapId, int32_t numPartitions)
      : d_(d), shuffleId_(shuffleId), mapId_(mapId), numPartitions_(numPartitions),
        partitionLengths_((size_t)numPartitions, 0), partOff_((size_t)numPartitions, 0) {
    gpu_ = d.gpuEnabled && d.codecId() != B2S_CODEC_NONE;
  }

  // :67-83
  void getPartitionWriter(int32_t reducePartitionId) {
    if (reducePartitionId <= lastPartitionWriterId_)
      throw RuntimeException("Precondition: Expect a monotonically increasing reducePartitionId.");
    if (reducePartitionId >= numPartitions_) throw RuntimeException("Precondition: Invalid partition id.");
    lastPartitionWriterId_ = reducePartitionId;
    current_ = reducePartitionId;
    byteCount_ = 0;
    streamOpen_ = true;
    partOff_[(size_t)current_] = (int64_t)buf_.size();
  }
  // :182-188
  void write(const uint8_t* b, uint64_t n) {
    if (!streamOpen_) throw IOException("S3ShuffleOutputStream is already closed.");
    buf_.append(b, n);
    byteCount_ += (int64_t)n;
  }
  // :197-201
  void closePartition() {
    if (current_ < 0) return;
    partitionLengths_[(size_t)current_] = byteCount_;
    totalBytesWritten_ += byteCount_;
    streamOpen_ = false;
  }

  // :91-118
  std::vector<int64_t> commitAllPartitions(const int64_t* checksums_in) {
    std::vector<int64_t> checksums((size_t)numPartitions_, 0);
    const uint8_t* data = buf_.data();
    uint64_t data_len = buf_.size();
    std::vector<std::pair<const uint8_t*, uint64_t>> segments{{data, data_len}};  // what goes into .data, in order
    if ((int64_t)data_len != totalBytesWritten_)
      throw RuntimeException("S3ShuffleMapOutputWriter: Unexpected output length " + std::to_string(data_len) +
                             ", expected: " + std::to_string(totalBytesWritten_) + ".");
    const uint32_t alg = d_.checksumEnabled ? S3ShuffleHelper::createChecksumAlgorithm(d_.checksumAlgorithm) : 0;
    if (gpu_) {
      // SURVEY.md §3.2 option B: upstream wrote serialized *uncompressed* bytes; compress + checksum every
      // non-empty partition in one batch.  Empty partitions stay 0 bytes long, as with Spark's own writers.
      ensure_codec_runtime();
      std::vector<uint64_t> off, len, doff, dlen, cks;
      std::vector<int32_t> status, idx;
      uint64_t bound = 0;
      for (int32_t p = 0; p < numPartitions_; p++) {
        if (partitionLengths_[(size_t)p] == 0) continue;
        idx.push_back(p);
        off.push_back((uint64_t)partOff_[(size_t)p]);
        len.push_back((uint64_t)partitionLengths_[(size_t)p]);
        bound += b2s_compress_bound((uint32_t)d_.codecId(), d_.lz4BlockSize, len.back());
      }
      const uint32_t n = (uint32_t)idx.size();
      doff.resize(n); dlen.resize(n); cks.resize(n); status.resize(n);
      out_.resize(bound);
      uint64_t total = 0;
      if (d_.gpuCoalesce) {
        // through the executor's group-commit queue: per-stream pointers, every output at its bound-sized slot
        std::vector<const uint8_t*> sp(n);
        std::vector<uint8_t*> dp(n);
        std::vector<uint64_t> cap(n);
        uint64_t o = 0;
        for (uint32_t k = 0; k < n; k++) {
          sp[k] = data + off[k];
          cap[k] = b2s_compress_bound((uint32_t)d_.codecId(), d_.lz4BlockSize, len[k]);
          dp[k] = out_.data() + o;
          doff[k] = o;
          o += cap[k];
        }
        CodecRequest r;
        r.op = 0;
        r.codec = (uint32_t)d_.codecId();
        r.block_size = d_.lz4BlockSize;
        r.level = d_.zstdLevel;
        r.checksum_alg = alg;
        r.n = n;
        r.src = sp.data();
        r.src_len = len.data();
        r.dst = dp.data();
        r.dst_cap = cap.data();
        r.dst_len = dlen.data();
        r.checksum_out = cks.data();
        r.status = status.data();
        submit_or_throw(d_.queue, r, "b2s_compress_batch");
        for (uint32_t k = 0; k < n; k++) total += dlen[k];
      } else {
        int rc = b2s_compress_packed((uint32_t)d_.codecId(), d_.zstdLevel, d_.lz4BlockSize, alg, n, data, off.data(), len.data(),
                                     out_.data(), bound, doff.data(), dlen.data(), &total, cks.data(), status.data());
        if (rc != 0) throw CodecException(std::string("b2s_compress_packed: ") + b2s_strerror(rc) + ": " + b2s_last_error());
      }
      for (uint32_t k = 0; k < n; k++)
        if (status[k] != 0) throw IOException(std::string("compress failed: ") + b2s_strerror(status[k]));
      std::fill(partitionLengths_.begin(), partitionLengths_.end(), 0);
      for (int32_t p = 0; p < numPartitions_; p++) checksums[(size_t)p] = alg ? S3ShuffleHelper::emptyChecksum(alg) : 0;
      for (uint32_t k = 0; k < n; k++) {
        partitionLengths_[(size_t)idx[k]] = (int64_t)dlen[k];
        checksums[(size_t)idx[k]] = (int64_t)cks[k];
      }
      data_len = total;
      segments.clear();  // partition k's stream sits at out_ + doff[k] (back to back in the packed form)
      for (uint32_t k = 0; k < n; k++) segments.push_back({out_.data() + doff[k], dlen[k]});
    } else if (checksums_in) {
      for (int32_t p = 0; p < numPartitions_; p++) checksums[(size_t)p] = checksums_in[p];
    }
    // the .data object exists as soon as a stream was opened (:43-49)
    writeMapOutput(d_, shuffleId_, mapId_, lastPartitionWriterId_ >= 0, segments, data_len, partitionLengths_,
                   checksums, measure_);
    return partitionLengths_;
  }
  void abort() {  // :120-134
    buf_.clear();
    streamOpen_ = false;
  }
  const S3MeasureOutputStream* measure() const { return measure_.get(); }

 private:
  S3ShuffleDispatcher& d_;
  int32_t shuffleId_;
  int64_t mapId_;
  int32_t numPartitions_;
  std::vector<int64_t> partitionLengths_, partOff_;
  int64_t totalBytesWritten_ = 0, byteCount_ = 0;
  int32_t lastPartitionWriterId_ = -1, current_ = -1;
  bool streamOpen_ = false, gpu_ = true;
  PinnedArena buf_, out_;
  std::unique_ptr<S3MeasureOutputStream> measure_;
};

// ---- GPU serialized writer: what UnsafeShuffleWriter + ShuffleExternalSorter do for a SerializedShuffleHandle -----
// insertRecord(record, partitionId) collects the serialized records back to back with their reduce ids, in any
// partition order (ShuffleExternalSorter.insertRecord).  commit() hands them to ONE b2s_partition_compress_packed call
// (stable partition by reduce id, then compress + checksum every partition on the GPU) and writes .data / .index /
// .checksum through the same code as S3ShuffleMapOutputWriter.commitAllPartitions.  The files are byte for byte what
// that writer produces when every partition is opened in order and fed its records in insertion order.
class S3SerializedShuffleWriter {
 public:
  S3SerializedShuffleWriter(S3ShuffleDispatcher& d, int32_t shuffleId, int64_t mapId, int32_t numPartitions)
      : d_(d), shuffleId_(shuffleId), mapId_(mapId), numPartitions_(numPartitions) {
    if (numPartitions < 1 || numPartitions > (1 << 24))  // PackedRecordPointer's 24-bit partition id
      throw RuntimeException("Precondition: numPartitions must be in [1, 2^24].");
    if (!d.gpuEnabled) throw UnsupportedOperationException("the serialized GPU writer needs spark.shuffle.s3.gpu.enabled");
  }
  // HashPartitioning by these key columns (b2s_partition_compress_rows_hash_packed): every later insert is one
  // serialized row whose partitionId is ignored, and commit() computes Spark's ids on the GPU
  void hashRows(uint32_t nKeys, const uint32_t* type, const uint32_t* off, const uint32_t* len, const int32_t* nullField) {
    if (!recLen_.empty()) throw RuntimeException("Precondition: hash_rows must come before the first insert.");
    if (nKeys < 1 || nKeys > 16) throw RuntimeException("Precondition: n_keys must be in [1, 16].");
    keyType_.assign(type, type + nKeys);
    keyOff_.assign(off, off + nKeys);
    keyLen_.assign(len, len + nKeys);
    keyNull_.assign(nullField, nullField + nKeys);
  }
  // RangePartitioning by these key columns over these bounds (b2s_partition_compress_rows_range_packed): as hashRows,
  // with Spark's RangePartitioner ids; the writer's numPartitions is the bounds' count + 1
  void rangeRows(uint32_t nKeys, const uint32_t* type, const uint32_t* off, const uint32_t* len, const int32_t* nullField,
                 uint32_t nBounds, const uint8_t* boundBase, uint64_t boundBytes, const uint32_t* boundLen) {
    if ((uint64_t)nBounds + 1 != (uint64_t)numPartitions_)
      throw RuntimeException("Precondition: range_rows needs n_bounds + 1 == numPartitions.");
    if (nBounds && (!boundBase || !boundLen)) throw RuntimeException("Precondition: null bound arrays.");
    hashRows(nKeys, type, off, len, nullField);
    range_ = true;
    boundRows_.assign(boundBase, boundBase + (nBounds ? boundBytes : 0));
    boundLen_.assign(boundLen, boundLen + nBounds);
  }
  // RoundRobinPartitioning (b2s_partition_compress_rows_round_robin_packed): every later insert is one serialized row
  // whose partitionId is ignored, and commit() sorts (sortRows) and deals the rows out on the GPU from startPosition
  void roundRobinRows(uint32_t numPartitions, int32_t startPosition, uint32_t sortRows) {
    if (!recLen_.empty()) throw RuntimeException("Precondition: round_robin_rows must come before the first insert.");
    if ((uint64_t)numPartitions != (uint64_t)numPartitions_)
      throw RuntimeException("Precondition: round_robin_rows needs num_partitions == numPartitions.");
    roundRobin_ = true;
    rrStart_ = startPosition;
    rrSort_ = sortRows;
  }
  // The partial aggregation of a grouped aggregation's map side (b2s_aggregate_partition_compress_rows_hash_packed):
  // after hashRows and before the first insert; commit() groups the rows by hashRows' key columns, folds these
  // functions' buffers and hash-partitions the partial rows on the GPU.  No cached form exists, so the call is the same
  // with the exchange cache on.
  void aggregateRows(uint32_t nAggs, const uint32_t* fn, const uint32_t* valType, const uint32_t* valOff,
                     const int32_t* valNull) {
    if (!recLen_.empty()) throw RuntimeException("Precondition: aggregate_rows must come before the first insert.");
    if (keyType_.empty() || range_ || roundRobin_ || windowLimit_)
      throw RuntimeException("Precondition: aggregate_rows needs hash_rows first.");
    if (nAggs > 16) throw RuntimeException("Precondition: n_aggs must be at most 16.");
    if (nAggs && (!fn || !valType || !valOff || !valNull)) throw RuntimeException("Precondition: null aggregate arrays.");
    aggregate_ = true;
    aggFn_.assign(fn, fn + nAggs);
    aggType_.assign(valType, valType + nAggs);
    aggOff_.assign(valOff, valOff + nAggs);
    aggNull_.assign(valNull, valNull + nAggs);
  }
  // The grouping sets of a ROLLUP, CUBE or GROUPING SETS aggregation's map side
  // (b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed): after aggregateRows and before the first insert;
  // commit() expands every row once per set (bit c of a mask: key column c is in the set), then aggregates and
  // hash-partitions the partial rows keyed by the grouping columns and spark_grouping_id on the GPU.
  void groupingSets(uint32_t nSets, const uint32_t* mask) {
    if (!recLen_.empty()) throw RuntimeException("Precondition: grouping_sets must come before the first insert.");
    if (!aggregate_) throw RuntimeException("Precondition: grouping_sets needs aggregate_rows first.");
    if (!nSets || !mask) throw RuntimeException("Precondition: grouping_sets needs at least one set.");
    setMask_.assign(mask, mask + nSets);
  }
  // The partial limit of a top-N-per-group window's map side (b2s_window_limit_partition_compress_rows_hash_packed), in
  // place of hashRows and before the first insert: commit() sorts the rows by these key columns (the first nPartKeys the
  // PARTITION BY columns, then the ORDER BY columns), keeps those whose limitFn value in their partition is at most
  // limit, and hash-partitions them by the partition columns on the GPU (none: SinglePartition).  No cached form exists,
  // so the call is the same with the exchange cache on.
  void windowLimit(uint32_t nPartKeys, uint32_t nKeys, const uint32_t* type, const uint32_t* off, const uint32_t* len,
                   const int32_t* nullField, uint32_t limitFn, int32_t limit) {
    if (!keyType_.empty() || roundRobin_)
      throw RuntimeException("Precondition: window_limit takes the place of hash_rows, range_rows and round_robin_rows.");
    if (nPartKeys >= nKeys) throw RuntimeException("Precondition: window_limit needs an ORDER BY column.");
    hashRows(nKeys, type, off, len, nullField);
    windowLimit_ = true;
    limitPartKeys_ = nPartKeys;
    limitFn_ = limitFn;
    limit_ = limit;
  }
  void insertRecord(int32_t partitionId, const uint8_t* b, uint64_t n) {
    const bool hashed = !keyType_.empty() || roundRobin_;
    if (!hashed && (partitionId < 0 || partitionId >= numPartitions_))
      throw RuntimeException("Precondition: Invalid partition id.");
    if (n > 0xffffffffull) throw RuntimeException("Precondition: record longer than 4 GiB.");
    records_.append(b, n);
    recLen_.push_back((uint32_t)n);
    if (!hashed) recPart_.push_back((uint32_t)partitionId);
  }
  std::vector<int64_t> commit() {
    ensure_codec_runtime();
    const uint32_t R = (uint32_t)numPartitions_;
    const uint32_t codec = (uint32_t)d_.codecId();
    const uint32_t alg = d_.checksumEnabled ? S3ShuffleHelper::createChecksumAlgorithm(d_.checksumAlgorithm) : 0;
    const uint64_t bound = b2s_partition_compress_bound(codec, d_.lz4BlockSize, R, records_.size());
    out_.resize(bound ? bound : 1);
    std::vector<uint64_t> doff(R), dlen(R), cks(R);
    std::vector<int32_t> status(R);
    uint64_t total = 0;
    int rc;
    const char* call = "b2s_partition_compress_packed";
    // With the exchange cache on, every form calls its cached one: the same outputs, and the partitioned records stay in
    // HBM for local reducers (a row writer's with its record boundaries)
    const bool cache = d_.gpuExchangeCacheBytes != 0;
    if (cache) d_.applyExchangeBudget();
    int32_t cached = 0;
    if (aggregate_) {
      // the partial rows' arena is not known before the call: the bound of the input's bytes first, then the exact
      // size the call reports when that is short
      const bool sets = !setMask_.empty();
      call = sets ? "b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed"
                  : "b2s_aggregate_partition_compress_rows_hash_packed";
      uint64_t groups = 0;
      for (int attempt = 0;; attempt++) {
        if (sets)
          rc = b2s_aggregate_grouping_sets_partition_compress_rows_hash_packed(
              codec, d_.zstdLevel, d_.lz4BlockSize, alg, R, recLen_.size(), records_.data(), records_.size(),
              recLen_.data(), (uint32_t)keyType_.size(), keyType_.data(), keyOff_.data(), keyLen_.data(),
              keyNull_.data(), (uint32_t)aggFn_.size(), aggFn_.data(), aggType_.data(), aggOff_.data(),
              aggNull_.data(), (uint32_t)setMask_.size(), setMask_.data(), out_.data(), out_.size(), doff.data(),
              dlen.data(), &total, cks.data(), status.data(), &groups);
        else
          rc = b2s_aggregate_partition_compress_rows_hash_packed(
              codec, d_.zstdLevel, d_.lz4BlockSize, alg, R, recLen_.size(), records_.data(), records_.size(),
              recLen_.data(), (uint32_t)keyType_.size(), keyType_.data(), keyOff_.data(), keyLen_.data(),
              keyNull_.data(), (uint32_t)aggFn_.size(), aggFn_.data(), aggType_.data(), aggOff_.data(),
              aggNull_.data(), out_.data(), out_.size(), doff.data(), dlen.data(), &total, cks.data(), status.data(),
              &groups);
        if (rc != B2S_E_DST_TOO_SMALL || attempt) break;
        out_.resize(total);
      }
    } else if (windowLimit_) {
      call = "b2s_window_limit_partition_compress_rows_hash_packed";
      uint64_t kept = 0;
      rc = b2s_window_limit_partition_compress_rows_hash_packed(
          codec, d_.zstdLevel, d_.lz4BlockSize, alg, R, recLen_.size(), records_.data(), records_.size(),
          recLen_.data(), limitPartKeys_, (uint32_t)keyType_.size(), keyType_.data(), keyOff_.data(), keyLen_.data(),
          keyNull_.data(), limitFn_, limit_, out_.data(), bound, doff.data(), dlen.data(), &total, cks.data(),
          status.data(), &kept);
    } else if (roundRobin_ && cache) {
      call = "b2s_partition_compress_rows_round_robin_cached_packed";
      rc = b2s_partition_compress_rows_round_robin_cached_packed(
          shuffleId_, mapId_, codec, d_.zstdLevel, d_.lz4BlockSize, alg, R, rrStart_, rrSort_, recLen_.size(),
          records_.data(), records_.size(), recLen_.data(), out_.data(), bound, doff.data(), dlen.data(), &total,
          cks.data(), status.data(), &cached);
    } else if (roundRobin_) {
      call = "b2s_partition_compress_rows_round_robin_packed";
      rc = b2s_partition_compress_rows_round_robin_packed(
          codec, d_.zstdLevel, d_.lz4BlockSize, alg, R, rrStart_, rrSort_, recLen_.size(), records_.data(),
          records_.size(), recLen_.data(), out_.data(), bound, doff.data(), dlen.data(), &total, cks.data(),
          status.data());
    } else if (range_ && cache) {
      call = "b2s_partition_compress_rows_range_cached_packed";
      rc = b2s_partition_compress_rows_range_cached_packed(
          shuffleId_, mapId_, codec, d_.zstdLevel, d_.lz4BlockSize, alg, recLen_.size(), records_.data(),
          records_.size(), recLen_.data(), (uint32_t)keyType_.size(), keyType_.data(), keyOff_.data(), keyLen_.data(),
          keyNull_.data(), (uint32_t)boundLen_.size(), boundRows_.data(), boundRows_.size(), boundLen_.data(),
          out_.data(), bound, doff.data(), dlen.data(), &total, cks.data(), status.data(), &cached);
    } else if (range_) {
      call = "b2s_partition_compress_rows_range_packed";
      rc = b2s_partition_compress_rows_range_packed(
          codec, d_.zstdLevel, d_.lz4BlockSize, alg, recLen_.size(), records_.data(), records_.size(), recLen_.data(),
          (uint32_t)keyType_.size(), keyType_.data(), keyOff_.data(), keyLen_.data(), keyNull_.data(),
          (uint32_t)boundLen_.size(), boundRows_.data(), boundRows_.size(), boundLen_.data(), out_.data(), bound,
          doff.data(), dlen.data(), &total, cks.data(), status.data());
    } else if (!keyType_.empty() && cache) {
      call = "b2s_partition_compress_rows_hash_cached_packed";
      rc = b2s_partition_compress_rows_hash_cached_packed(
          shuffleId_, mapId_, codec, d_.zstdLevel, d_.lz4BlockSize, alg, R, recLen_.size(), records_.data(),
          records_.size(), recLen_.data(), (uint32_t)keyType_.size(), keyType_.data(), keyOff_.data(), keyLen_.data(),
          keyNull_.data(), out_.data(), bound, doff.data(), dlen.data(), &total, cks.data(), status.data(), &cached);
    } else if (!keyType_.empty()) {
      call = "b2s_partition_compress_rows_hash_packed";
      rc = b2s_partition_compress_rows_hash_packed(
          codec, d_.zstdLevel, d_.lz4BlockSize, alg, R, recLen_.size(), records_.data(), records_.size(),
          recLen_.data(), (uint32_t)keyType_.size(), keyType_.data(), keyOff_.data(), keyLen_.data(), keyNull_.data(),
          out_.data(), bound, doff.data(), dlen.data(), &total, cks.data(), status.data());
    } else if (cache) {
      call = "b2s_partition_compress_cached_packed";
      rc = b2s_partition_compress_cached_packed(shuffleId_, mapId_, codec, d_.zstdLevel, d_.lz4BlockSize, alg, R,
                                                recLen_.size(), records_.data(), records_.size(), recLen_.data(),
                                                recPart_.data(), out_.data(), bound, doff.data(), dlen.data(), &total,
                                                cks.data(), status.data(), &cached);
    } else {
      rc = b2s_partition_compress_packed(codec, d_.zstdLevel, d_.lz4BlockSize, alg, R, recLen_.size(), records_.data(),
                                         records_.size(), recLen_.data(), recPart_.data(), out_.data(), bound,
                                         doff.data(), dlen.data(), &total, cks.data(), status.data());
    }
    if (rc != 0) throw CodecException(std::string(call) + ": " + b2s_strerror(rc) + ": " + b2s_last_error());
    std::vector<int64_t> lengths(R), checksums(R);
    for (uint32_t p = 0; p < R; p++) {
      if (status[p] != 0) throw IOException(std::string("compress failed: ") + b2s_strerror(status[p]));
      lengths[p] = (int64_t)dlen[p];
      checksums[p] = (int64_t)cks[p];
    }
    writeMapOutput(d_, shuffleId_, mapId_, true, {{out_.data(), total}}, total, lengths, checksums, measure_);
    return lengths;
  }
  const S3MeasureOutputStream* measure() const { return measure_.get(); }
  int32_t numPartitions() const { return numPartitions_; }
  // Commits a .data arena that another call writes in this writer's place (a reduce task that ends in this map
  // output, S3ShuffleReader::aggregateDistinctRows): partition(dst, cap, dst_off, dst_len, &total, checksums, status)
  // fills it like b2s_partition_compress_packed, retried once with the exact size on B2S_E_DST_TOO_SMALL; check() runs
  // after the call and throws to leave no files; then .data / .index / .checksum are written as commit() writes them.
  template <class Partition, class Check>
  std::vector<int64_t> commitFrom(const char* call, uint64_t guess, Partition&& partition, Check&& check) {
    if (!recLen_.empty() || !keyType_.empty() || roundRobin_)
      throw RuntimeException("Precondition: a writer committed by a reader takes no rows and no partitioning.");
    const uint32_t R = (uint32_t)numPartitions_;
    std::vector<uint64_t> doff(R), dlen(R), cks(R);
    std::vector<int32_t> status(R);
    uint64_t total = 0;
    int rc = B2S_E_DST_TOO_SMALL;
    for (int attempt = 0; attempt < 2 && rc == B2S_E_DST_TOO_SMALL; attempt++) {
      out_.resize(attempt ? (total ? total : 1) : (guess ? guess : 1));
      rc = partition(out_.data(), (uint64_t)out_.size(), doff.data(), dlen.data(), &total, cks.data(), status.data());
    }
    if (rc != 0) throw CodecException(std::string(call) + ": " + b2s_strerror(rc) + ": " + b2s_last_error());
    check();
    std::vector<int64_t> lengths(R), checksums(R);
    for (uint32_t p = 0; p < R; p++) {
      if (status[p] != 0) throw IOException(std::string("compress failed: ") + b2s_strerror(status[p]));
      lengths[p] = (int64_t)dlen[p];
      checksums[p] = (int64_t)cks[p];
    }
    writeMapOutput(d_, shuffleId_, mapId_, true, {{out_.data(), total}}, total, lengths, checksums, measure_);
    return lengths;
  }

 private:
  S3ShuffleDispatcher& d_;
  int32_t shuffleId_;
  int64_t mapId_;
  int32_t numPartitions_;
  PinnedArena records_, out_;
  std::vector<uint32_t> recLen_, recPart_;
  std::vector<uint32_t> keyType_, keyOff_, keyLen_;  // hashRows' key columns (empty: the caller's partition ids)
  std::vector<int32_t> keyNull_;
  bool range_ = false;  // rangeRows: the ids are RangePartitioner ids over these bounds
  std::vector<uint8_t> boundRows_;
  std::vector<uint32_t> boundLen_;
  bool aggregate_ = false;  // aggregateRows: the rows are aggregated by hashRows' key columns first
  std::vector<uint32_t> aggFn_, aggType_, aggOff_;
  std::vector<int32_t> aggNull_;
  std::vector<uint32_t> setMask_;  // groupingSets: the rows are expanded once per set before the aggregation
  bool windowLimit_ = false;  // windowLimit: hashRows' key columns are the window key, the first limitPartKeys_ hashed
  uint32_t limitPartKeys_ = 0, limitFn_ = 0;
  int32_t limit_ = 0;
  bool roundRobin_ = false;  // roundRobinRows: Spark's repartition(n) order and ids from rrStart_
  int32_t rrStart_ = 0;
  uint32_t rrSort_ = 0;
  std::unique_ptr<S3MeasureOutputStream> measure_;
};

// ---- S3SingleSpillShuffleMapOutputWriter (shuffle/S3SingleSpillShuffleMapOutputWriter.scala:24-64) ------------------
// UnsafeShuffleWriter's single-spill fast path: the spill file already holds the compressed, checksummed partition
// streams back to back; it is moved (local root: rename, copy when that fails across devices) to the .data object,
// then .checksum and .index are written — in that order, as the reference does.  SURVEY.md §8(f)-3: with
// verifyOnTransfer the per-partition checksums are recomputed over the file's bytes by the GPU (one packed batch) and
// compared with the ones handed in, which is the "checksum-on-the-fly" the copy loop at :54-58 has room for.
class S3SingleSpillShuffleMapOutputWriter {
 public:
  S3SingleSpillShuffleMapOutputWriter(S3ShuffleDispatcher& d, int32_t shuffleId, int64_t mapId)
      : d_(d), shuffleId_(shuffleId), mapId_(mapId) {}

  void transferMapSpillFile(const std::string& spillFile, const std::vector<int64_t>& partitionLengths,
                            const std::vector<int64_t>& checksums, bool verifyOnTransfer) {
    std::string path = d_.getPath(BlockId{BlockId::Data, shuffleId_, mapId_, 0, 0});
    mkdirs(path.substr(0, path.rfind('/')));
    if (verifyOnTransfer && d_.checksumEnabled) {
      const uint32_t alg = S3ShuffleHelper::createChecksumAlgorithm(d_.checksumAlgorithm);
      std::ifstream f(spillFile, std::ios::binary | std::ios::ate);
      if (!f) throw IOException("File does not exist: " + spillFile);
      const uint64_t len = (uint64_t)f.tellg();
      int64_t sum = 0;
      for (int64_t v : partitionLengths) sum += v;
      if ((int64_t)len != sum)
        throw RuntimeException("S3SingleSpillShuffleMapOutputWriter: Unexpected spill length " + std::to_string(len) +
                               ", expected: " + std::to_string(sum) + ".");
      ensure_codec_runtime();
      PinnedArena buf;
      buf.resize(len ? len : 1);
      f.seekg(0);
      f.read((char*)buf.data(), (std::streamsize)len);
      const uint32_t n = (uint32_t)partitionLengths.size();
      std::vector<uint64_t> off(n), ln(n), got(n);
      uint64_t o = 0;
      for (uint32_t i = 0; i < n; i++) {
        off[i] = o;
        ln[i] = (uint64_t)partitionLengths[i];
        o += ln[i];
      }
      int rc = b2s_checksum_packed(alg, n, buf.data(), off.data(), ln.data(), got.data());
      if (rc != 0) throw CodecException(std::string("b2s_checksum_packed: ") + b2s_strerror(rc) + ": " + b2s_last_error());
      for (uint32_t i = 0; i < n; i++)
        if ((int64_t)got[i] != checksums[i])
          throw SparkException("Invalid checksum detected for " +
                               BlockId{BlockId::Shuffle, shuffleId_, mapId_, (int32_t)i, 0}.name());
    }
    if (rename(spillFile.c_str(), path.c_str()) != 0) {  // Files.move; falls back to a copy across file systems
      std::ifstream in(spillFile, std::ios::binary);
      if (!in) throw IOException("File does not exist: " + spillFile);
      std::ofstream out(path, std::ios::binary | std::ios::trunc);
      if (!out) throw IOException("cannot create " + path);
      out << in.rdbuf();
      in.close();
      unlink(spillFile.c_str());
    }
    if (d_.checksumEnabled) S3ShuffleHelper::writeChecksum(d_, shuffleId_, mapId_, checksums);  // :60-62
    S3ShuffleHelper::writePartitionLengths(d_, shuffleId_, mapId_, partitionLengths);             // :63
  }

 private:
  S3ShuffleDispatcher& d_;
  int32_t shuffleId_;
  int64_t mapId_;
};

// ---- S3ShuffleReader (storage/S3ShuffleReader.scala + block iterator/stream + prefetcher + checksum validation) ---
// The slices of a block (one per reduce partition it covers) travel with it, so that the per-partition validation of
// S3ChecksumValidationStream (storage/S3ChecksumValidationStream.scala:54-86) runs on the GPU inside the same batch
// call that decodes the block: verify first, then decompress, the reference's order (:99-110).
struct ShuffleBlockInfo {
  BlockId id;
  uint32_t mapPos = 0;  // index of the block's map in the reader's map list
  std::vector<uint64_t> sliceLen, sliceSum;
};

// computeShuffleBlocks (storage/S3ShuffleReader.scala:160-197, file-listing variant) + S3ShuffleBlockIterator
// (storage/S3ShuffleBlockIterator.scala:36-43) + filterNot(maxBytes == 0) and the read metrics (:89-97).  want (may be
// nullptr = every map): the maps to fetch; the others are served from the exchange cache.
static std::deque<S3BufferedPrefetchIterator::Source> computeShuffleBlockStreams(
    S3ShuffleDispatcher& d, int32_t shuffleId, const std::vector<int64_t>& mapIds, int32_t start, int32_t end,
    bool batch, std::vector<ShuffleBlockInfo>& info, uint64_t& remoteBytesRead, uint64_t& remoteBlocksFetched,
    const std::vector<uint8_t>* want = nullptr) {
  std::deque<S3BufferedPrefetchIterator::Source> out;
  const bool verify = d.checksumEnabled;
  for (uint32_t pos = 0; pos < (uint32_t)mapIds.size(); pos++) {
    if (want && !(*want)[pos]) continue;
    const int64_t mapId = mapIds[pos];
    std::vector<int64_t> acc = S3ShuffleHelper::getPartitionLengths(d, shuffleId, mapId);
    if ((int)acc.size() < end + 1)
      throw SparkException("index of map " + std::to_string(mapId) + " has too few partitions");
    std::vector<int64_t> sums;
    if (verify) sums = S3ShuffleHelper::getChecksums(d, shuffleId, mapId);
    std::vector<std::pair<int32_t, int32_t>> ranges;
    if (batch && end - start > 1) ranges.push_back({start, end});
    else for (int32_t r = start; r < end; r++) ranges.push_back({r, r + 1});
    const std::string path = d.getPath(BlockId{BlockId::Data, shuffleId, mapId, 0, 0});
    for (auto [rs, re] : ranges) {
      const int64_t a = acc[(size_t)rs], b = acc[(size_t)re];
      if (b - a == 0) continue;                // filterNot(_._2.maxBytes == 0)  (:91)
      remoteBytesRead += (uint64_t)(b - a);    // incRemoteBytesRead (:94)
      remoteBlocksFetched += 1;                // incRemoteBlocksFetched (:95)
      ShuffleBlockInfo bi;
      bi.mapPos = pos;
      bi.id = (re - rs > 1) ? BlockId{BlockId::ShuffleBatch, shuffleId, mapId, rs, re}
                            : BlockId{BlockId::Shuffle, shuffleId, mapId, rs, re};
      if (verify && sums.size() < (size_t)re)  // a short or stale .checksum object (the reference: ArrayIndexOutOfBounds)
        throw SparkException("Checksum file of " + bi.id.name() + " holds fewer entries than the index");
      if (verify)
        for (int32_t r = rs; r < re; r++) {    // S3ChecksumValidationStream walks the .index differences (:68-86)
          bi.sliceLen.push_back((uint64_t)(acc[(size_t)r + 1] - acc[(size_t)r]));
          bi.sliceSum.push_back((uint64_t)sums[(size_t)r]);
        }
      S3BufferedPrefetchIterator::Source src;
      src.id = bi.id;
      src.stream.reset(new S3ShuffleBlockStream(path, a, b));
      src.tag = info.size();
      info.push_back(std::move(bi));
      out.push_back(std::move(src));
    }
  }
  return out;
}

// A block as a sorted read drains it from the prefetcher: (its tag, the whole compressed block).
using FetchedBlock = std::pair<uint64_t, std::vector<uint8_t>>;

// The sources of one sorted-read call, staged in the order given: their bytes back to back in one pinned arena, each
// source's offset and length there, and its checksum slices (source k's are [sliceBase[k], sliceBase[k + 1])).  A null
// source, the place of a map the exchange cache serves, stages as no bytes and no slices.
struct StagedBlocks {
  using Side = std::pair<const std::vector<ShuffleBlockInfo>*, const std::vector<const FetchedBlock*>*>;
  StagedBlocks(const std::vector<ShuffleBlockInfo>& info, const std::vector<const FetchedBlock*>& sources)
      : StagedBlocks({Side{&info, &sources}}) {}
  // the sources of several readers back to back, each with its reader's block info
  explicit StagedBlocks(std::initializer_list<Side> sides) {
    for (const Side& side : sides)
      for (const FetchedBlock* f : *side.second) {
        off.push_back(bytes);
        len.push_back(f ? f->second.size() : 0);
        bytes += len.back();
        if (f) {
          const ShuffleBlockInfo& bi = (*side.first)[f->first];
          sliceLen.insert(sliceLen.end(), bi.sliceLen.begin(), bi.sliceLen.end());
          sliceSum.insert(sliceSum.end(), bi.sliceSum.begin(), bi.sliceSum.end());
        }
        sliceBase.push_back((uint32_t)sliceLen.size());
      }
    src.resize(bytes ? bytes : 1);
    size_t k = 0;
    for (const Side& side : sides)
      for (const FetchedBlock* f : *side.second) {
        if (f) memcpy(src.data() + off[k], f->second.data(), (size_t)len[k]);
        k++;
      }
  }
  PinnedArena src;
  uint64_t bytes = 0;
  std::vector<uint64_t> off, len, sliceLen, sliceSum;
  std::vector<uint32_t> sliceBase{0};
};

// A block's status from a decode call, thrown as the reference reports it.
static void throwBlockStatus(int32_t status, const BlockId& id) {
  if (status == B2S_E_CHECKSUM)  // storage/S3ChecksumValidationStream.scala:72-74
    throw SparkException("Invalid checksum detected for " + id.name());
  if (status == B2S_E_CORRUPT) throw IOException("Stream is corrupted");
  if (status != 0) throw IOException(std::string("decompress failed: ") + b2s_strerror(status));
}

// Runs call(cap) with `out` reset to cap bytes.  A call that finds cap too small ends with the bytes it needs in
// `total`; it then runs once more with exactly that.
template <typename Call>
static int callWithRetry(std::unique_ptr<uint8_t[]>& out, uint64_t cap, const uint64_t& total, Call&& call) {
  int rc = B2S_E_DST_TOO_SMALL;
  for (int attempt = 0; attempt < 2 && rc == B2S_E_DST_TOO_SMALL; attempt++) {
    if (attempt) cap = total;
    out.reset(new uint8_t[(size_t)(cap ? cap : 1)]);
    rc = call(cap);
  }
  return rc;
}

class S3ShuffleReader {
 public:
  struct Block {
    BlockId id;
    const uint8_t* data = nullptr;
    uint64_t len = 0;
  };
  S3ShuffleReader(S3ShuffleDispatcher& d, int32_t shuffleId, std::vector<int64_t> mapIds, int32_t startPartition,
                  int32_t endPartition, bool doBatchFetch)
      : d_(d), shuffleId_(shuffleId), mapIds_(std::move(mapIds)), start_(startPartition), end_(endPartition),
        batch_(doBatchFetch || d.forceBatchFetch) {}
  ~S3ShuffleReader() { iter_.reset(); }

  // read(): storage/S3ShuffleReader.scala:77-110 — everything the task reads, drained batch by batch.  With the exchange
  // cache on (INTEGRATION.md §3f) the maps resident on this thread's device come from it first, one block per map
  // covering [start, end); only the others are fetched, and only their bytes count as remote bytes read.
  void read() {
    std::vector<uint8_t> fetch = cacheMisses();
    std::vector<Block> all;
    std::vector<std::unique_ptr<uint8_t[]>> bufs;
    if (d_.codecId() != B2S_CODEC_NONE) readCached(fetch, all, bufs);  // codec "none" is refused by start() below
    start(false, &fetch);
    while (nextBatch((size_t)d_.gpuReadBatchBlocks)) {
      all.insert(all.end(), blocks_.begin(), blocks_.end());
      for (auto& p : decoded_) bufs.push_back(std::move(p));
      decoded_.clear();
    }
    blocks_ = std::move(all);
    decoded_ = std::move(bufs);
  }

  void open() { start(false); }

  // One sorted-read call's sources, as readSources stages them for `call`
  struct Sources {
    uint32_t codec, alg, n;
    const int64_t* ids;      // the map of each source
    const uint8_t* cached;   // 1: the source is that map's cached range
    bool anyCached;          // false: every source is a fetched block (the plain calls apply)
    StagedBlocks& src;       // the fetched blocks, a cached source staged as no bytes
    const uint32_t* sb;      // their checksum slices (nullptr without checksums)
    const uint64_t* sl;
    const uint64_t* sc;
    int32_t* status;
    int32_t* bad;
  };
  // The body of readSorted and readRows: the task's blocks are fetched and staged in computeShuffleBlocks order (map,
  // then reduce id), except that with the exchange cache on a map resident on this thread's device is one cached source
  // in its place; then call(sources, cap, &total, &records, &groups, &name) runs the one read into sorted_ (cap bytes;
  // a call that finds cap too small ends with the bytes needed in total and is run once more with exactly that).  Maps
  // the cache no longer holds when the call runs (status B2S_E_NOT_CACHED) are fetched and the call repeated.
  template <typename Call>
  void readSources(Call&& call) {
    std::vector<uint8_t> fetch = cacheMisses();
    start(true, &fetch);
    std::vector<FetchedBlock> fetched;
    drainWhole(fetched);
    const uint32_t M = (uint32_t)mapIds_.size();
    const bool verify = d_.checksumEnabled;
    const uint32_t alg = verify ? S3ShuffleHelper::createChecksumAlgorithm(d_.checksumAlgorithm) : 0;
    ensure_codec_runtime();
    const uint32_t codec = (uint32_t)d_.codecId();
    while (true) {
      std::sort(fetched.begin(), fetched.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
      std::vector<std::vector<uint32_t>> ofMap(M);  // the fetched blocks of each map, in reduce-id order
      for (uint32_t k = 0; k < (uint32_t)fetched.size(); k++) ofMap[info_[fetched[k].first].mapPos].push_back(k);
      std::vector<int64_t> ids;
      std::vector<uint8_t> cached;
      std::vector<uint32_t> mapOf;
      std::vector<const FetchedBlock*> from;  // the source's entry of `fetched`, null for a cached source
      auto add = [&](uint32_t m, const FetchedBlock* f) {
        ids.push_back(mapIds_[m]);
        cached.push_back(f ? 0 : 1);
        from.push_back(f);
        mapOf.push_back(m);
      };
      for (uint32_t m = 0; m < M; m++) {
        if (!fetch[m]) add(m, nullptr);
        else for (uint32_t k : ofMap[m]) add(m, &fetched[k]);
      }
      const uint32_t n = (uint32_t)ids.size();
      StagedBlocks src(info_, from);
      const bool anyCached = std::find(cached.begin(), cached.end(), 1) != cached.end();
      uint64_t cachedBytes = 0;
      if (anyCached) {
        std::vector<uint64_t> hitLen(n);
        lookup(n, ids.data(), hitLen.data());
        for (uint32_t k = 0; k < n; k++)
          if (cached[k] && hitLen[k] != UINT64_MAX) cachedBytes += hitLen[k];
      }
      std::vector<int32_t> status(n), bad(n);
      const Sources x{codec, alg, n, ids.data(), cached.data(), anyCached, src,
                      verify ? src.sliceBase.data() : nullptr, verify ? src.sliceLen.data() : nullptr,
                      verify ? src.sliceSum.data() : nullptr, status.data(), bad.data()};
      uint64_t total = 0, records = 0, groups = 0;
      const char* name = "";
      // Output size: codec NONE decodes to the stored bytes.  For a codec, a first guess of 4x the compressed bytes (the
      // pages of the untouched tail are never faulted in); a call it is too small for ends after verification with the
      // bytes needed in `total`, and the one retry uses exactly that.
      const uint64_t guess = (codec == B2S_CODEC_NONE ? src.bytes : src.bytes * 4) + cachedBytes;
      const int rc = callWithRetry(sorted_, guess, total,
                                   [&](uint64_t cap) { return call(x, cap, &total, &records, &groups, &name); });
      if (rc != 0) throw CodecException(std::string(name) + ": " + b2s_strerror(rc) + ": " + b2s_last_error());
      std::vector<uint8_t> late(M, 0);  // maps evicted between the lookup and the call: fetch them, then read again
      for (uint32_t k = 0; k < n; k++)
        if (status[k] == B2S_E_NOT_CACHED) late[mapOf[k]] = fetch[mapOf[k]] = 1;
      if (std::find(late.begin(), late.end(), 1) != late.end()) {
        auto more = computeShuffleBlockStreams(d_, shuffleId_, mapIds_, start_, end_, batch_, info_, remoteBytesRead_,
                                               remoteBlocksFetched_, &late);
        iter_.reset(new S3BufferedPrefetchIterator(std::move(more), d_.maxBufferSizeTask, d_.maxConcurrencyTask));
        drainWhole(fetched);
        continue;
      }
      for (uint32_t k = 0; k < n; k++)
        throwBlockStatus(status[k], cached[k] ? cachedBlockId(ids[k]) : info_[from[k]->first].id);
      sortedLen_ = total;
      sortedRecords_ = records;
      sortedGroups_ = groups;
      return;
    }
  }

  // read() for a shuffle with a key ordering whose records are recordBytes long and order by the unsigned bytes
  // [keyOff, keyOff + keyLen) (INTEGRATION.md §3e): every non-empty block is fetched and staged, then ONE
  // b2s_decompress_sort_packed call verifies, decodes and key-sorts all of the task's records.  The blocks go in
  // computeShuffleBlocks order (map, then reduce id), so records with equal keys come out in that order whatever the
  // order the fetches completed in.  Codec NONE (spark.shuffle.compress=false) is verified and sorted only.  With the
  // exchange cache on, a map resident on this thread's device is one cached source in that order instead of its blocks
  // (b2s_exchange_read_sort_packed); maps the cache no longer holds when the call runs are fetched and the call repeated.
  void readSorted(uint32_t recordBytes, uint32_t keyOff, uint32_t keyLen) {
    readSources([&](const Sources& x, uint64_t cap, uint64_t* total, uint64_t* records, uint64_t*, const char** call) {
      *call = "b2s_decompress_sort_packed";
      if (!x.anyCached)
        return b2s_decompress_sort_packed(x.codec, x.alg, x.n, x.src.src.data(), x.src.off.data(), x.src.len.data(),
                                          x.sb, x.sl, x.sc, recordBytes, keyOff, keyLen, sorted_.get(), cap, total,
                                          records, x.status, x.bad);
      return b2s_exchange_read_sort_packed(shuffleId_, start_, end_, x.ids, x.cached, x.codec, x.alg, x.n,
                                           x.src.src.data(), x.src.off.data(), x.src.len.data(), x.sb, x.sl, x.sc,
                                           recordBytes, keyOff, keyLen, sorted_.get(), cap, total, records, x.status,
                                           x.bad);
    });
  }
  // The key columns of readRows: column c is type[c] (B2S_KEY_*, B2S_STRING_KEY or B2S_DECIMAL_KEY, with the order
  // flags B2S_KEY_DESCENDING / B2S_KEY_NULLS_LAST) at row offset off[c], len[c] bytes, null bit nullField[c].
  // composite: the *_rows_keys_* calls (up to 16 columns, strings, decimals and flags included), else the one-key
  // ones.
  struct RowKeys {
    uint32_t n;
    const uint32_t* type;
    const uint32_t* off;
    const uint32_t* len;
    const int32_t* nullField;
    bool composite;
  };
  // The aggregates of readRows: aggregate k is op[k] (B2S_AGG_*, B2S_AGG_SUM_DECIMAL with its precision in bits
  // 8..15) over the 8-byte slot at row offset off[k], null bit nullField[k] (-1 = never null).
  struct RowAggregates {
    uint32_t n;
    const uint32_t* op;
    const uint32_t* off;
    const int32_t* nullField;
  };
  // read() for a Spark SQL exchange whose rows the reducer sorts (aggs == nullptr, INTEGRATION.md §3g) or whose partial
  // aggregates it merges (INTEGRATION.md §3h) by one typed key or a composite one: every non-empty block is fetched and
  // staged, then ONE b2s_decompress_{sort,aggregate}_rows[_keys]_packed call verifies, decodes and sorts the task's
  // UnsafeRowSerializer records ([int32 big-endian size][row]) by the key, nulls first, or groups them and merges each
  // group into one row per key in that order.  Blocks go in computeShuffleBlocks order, so equal keys come out in map,
  // then reduce-id order.  Codec NONE is verified and sorted only.  With the exchange cache on, the maps resident on this
  // thread's device are cached sources in that order, as in readSorted, through the composite-key exchange reads
  // (b2s_exchange_read_{sort,aggregate}_rows_keys_packed; a one-key read is their n_keys = 1 case, INTEGRATION.md §3m).
  void readRows(const RowKeys& keys, const RowAggregates* aggs) {
    readSources([&](const Sources& x, uint64_t cap, uint64_t* total, uint64_t* records, uint64_t* groups,
                    const char** call) {
      const uint32_t codec = x.codec, alg = x.alg, n = x.n;
      const uint8_t* src = x.src.src.data();
      const uint64_t *off = x.src.off.data(), *len = x.src.len.data();
      if (x.anyCached && aggs) {
        *call = "b2s_exchange_read_aggregate_rows_keys_packed";
        return b2s_exchange_read_aggregate_rows_keys_packed(
            shuffleId_, start_, end_, x.ids, x.cached, codec, alg, n, src, off, len, x.sb, x.sl, x.sc, keys.n,
            keys.type, keys.off, keys.len, keys.nullField, aggs->n, aggs->op, aggs->off, aggs->nullField,
            sorted_.get(), cap, total, records, groups, x.status, x.bad);
      }
      if (x.anyCached) {
        *call = "b2s_exchange_read_sort_rows_keys_packed";
        return b2s_exchange_read_sort_rows_keys_packed(shuffleId_, start_, end_, x.ids, x.cached, codec, alg, n, src,
                                                       off, len, x.sb, x.sl, x.sc, keys.n, keys.type, keys.off,
                                                       keys.len, keys.nullField, sorted_.get(), cap, total, records,
                                                       x.status, x.bad);
      }
      if (aggs && keys.composite) {
        *call = "b2s_decompress_aggregate_rows_keys_packed";
        return b2s_decompress_aggregate_rows_keys_packed(codec, alg, n, src, off, len, x.sb, x.sl, x.sc, keys.n,
                                                         keys.type, keys.off, keys.len, keys.nullField, aggs->n,
                                                         aggs->op, aggs->off, aggs->nullField, sorted_.get(), cap,
                                                         total, records, groups, x.status, x.bad);
      }
      if (aggs) {
        *call = "b2s_decompress_aggregate_rows_packed";
        return b2s_decompress_aggregate_rows_packed(codec, alg, n, src, off, len, x.sb, x.sl, x.sc, keys.type[0],
                                                    keys.off[0], keys.len[0], keys.nullField[0], aggs->n, aggs->op,
                                                    aggs->off, aggs->nullField, sorted_.get(), cap, total, records,
                                                    groups, x.status, x.bad);
      }
      if (keys.composite) {
        *call = "b2s_decompress_sort_rows_keys_packed";
        return b2s_decompress_sort_rows_keys_packed(codec, alg, n, src, off, len, x.sb, x.sl, x.sc, keys.n, keys.type,
                                                    keys.off, keys.len, keys.nullField, sorted_.get(), cap, total,
                                                    records, x.status, x.bad);
      }
      *call = "b2s_decompress_sort_rows_packed";
      return b2s_decompress_sort_rows_packed(codec, alg, n, src, off, len, x.sb, x.sl, x.sc, keys.type[0], keys.off[0],
                                             keys.len[0], keys.nullField[0], sorted_.get(), cap, total, records,
                                             x.status, x.bad);
    });
  }
  // The join's arguments (b2s_decompress_join_rows_keys_packed): its type, the key columns' types and lengths, each
  // side's key slots and null bits, field counts and field kinds.
  struct JoinArgs {
    uint32_t type, nKeys;
    const uint32_t *keyType, *keyLen, *leftOff;
    const int32_t* leftNull;
    const uint32_t* rightOff;
    const int32_t* rightNull;
    uint32_t nLeftFields;
    const uint8_t* leftKind;
    uint32_t nRightFields;
    const uint8_t* rightKind;
  };
  // read() for the left (streamed) side of a sort-merge join whose right (buffered) side `right` reads
  // (INTEGRATION.md §3n): both readers' non-empty blocks are fetched (the exchange cache is not consulted), each in
  // computeShuffleBlocks order, and staged left first; then ONE b2s_decompress_join_rows_keys_packed call verifies,
  // decodes, sorts and joins them, retried once with the exact size when its first guess is too small.  The joined rows
  // stay in this reader as a sorted read's records do; sortedRecords() is the number of output rows.
  void readJoined(S3ShuffleReader& right, const JoinArgs& j, uint64_t* nLeft, uint64_t* nRight) {
    std::vector<FetchedBlock> lf, rf;
    fetchAll(lf);
    right.fetchAll(rf);
    std::vector<const FetchedBlock*> ls, rs;
    for (const auto& f : lf)
      if (!f.second.empty()) ls.push_back(&f);
    for (const auto& f : rf)
      if (!f.second.empty()) rs.push_back(&f);
    const uint32_t alg = d_.checksumEnabled ? S3ShuffleHelper::createChecksumAlgorithm(d_.checksumAlgorithm) : 0;
    ensure_codec_runtime();
    const uint32_t codec = (uint32_t)d_.codecId();
    StagedBlocks src({StagedBlocks::Side{&info_, &ls}, StagedBlocks::Side{&right.info_, &rs}});
    const uint32_t nl = (uint32_t)ls.size(), n = nl + (uint32_t)rs.size();
    std::vector<int32_t> status(n), bad(n);
    uint64_t total = 0, out = 0;
    const uint64_t guess = codec == B2S_CODEC_NONE ? src.bytes : src.bytes * 4;
    const int rc = callWithRetry(sorted_, guess, total, [&](uint64_t cap) {
      return b2s_decompress_join_rows_keys_packed(
          j.type, codec, alg, nl, n, src.src.data(), src.off.data(), src.len.data(), alg ? src.sliceBase.data() : 0,
          alg ? src.sliceLen.data() : 0, alg ? src.sliceSum.data() : 0, j.nKeys, j.keyType, j.keyLen, j.leftOff,
          j.leftNull, j.rightOff, j.rightNull, j.nLeftFields, j.leftKind, j.nRightFields, j.rightKind, sorted_.get(),
          cap, &total, nLeft, nRight, &out, status.data(), bad.data());
    });
    if (rc != 0)
      throw CodecException(std::string("b2s_decompress_join_rows_keys_packed: ") + b2s_strerror(rc) + ": " +
                           b2s_last_error());
    for (uint32_t k = 0; k < n; k++)
      throwBlockStatus(status[k], k < nl ? info_[ls[k]->first].id : right.info_[rs[k - nl]->first].id);
    sortedLen_ = total;
    sortedRecords_ = out;
  }
  // The window's arguments (b2s_decompress_window_rows_keys_packed): the key columns (the first nPartitionKeys of them
  // partition), the input's field count and kinds, the functions and their arguments, and the limit; with aggregate,
  // b2s_decompress_window_aggregate_rows_keys_packed's, whose functions also have frames and input columns (no limit);
  // with offset, b2s_decompress_window_offset_rows_keys_packed's, whose functions also have flags and defaults.
  struct WindowArgs {
    uint32_t nPartitionKeys, nKeys;
    const uint32_t *keyType, *keyOff, *keyLen;
    const int32_t* keyNull;
    uint32_t nFields;
    const uint8_t* kind;
    uint32_t nFns;
    const uint32_t* fn;
    const int32_t* fnArg;
    uint32_t limitFn;
    int32_t limit;
    const uint32_t* frame = nullptr;
    const uint32_t* valType = nullptr;
    const uint32_t* valOff = nullptr;
    const int32_t* valNull = nullptr;
    bool aggregate = false;
    const uint32_t* flags = nullptr;
    const uint64_t* dflt = nullptr;
    bool offset = false;
    const int64_t* lower = nullptr;  // with frames, b2s_decompress_window_frame_rows_keys_packed's bounds
    const int64_t* upper = nullptr;
    bool frames = false;
  };
  // read() for a Spark SQL window over this shuffle read (INTEGRATION.md §3o): every non-empty block is fetched (the
  // exchange cache is not consulted) in computeShuffleBlocks order, then ONE b2s_decompress_window_rows_keys_packed
  // call (or the aggregate one) verifies, decodes and sorts the rows and evaluates the functions, retried once with the
  // exact size
  // when its first guess is too small.  The output rows stay in this reader as a sorted read's records do;
  // sortedRecords() is the number of output rows, *nRecords the input's.
  void readWindowRows(const WindowArgs& w, uint64_t* nRecords) {
    std::vector<FetchedBlock> fetched;
    fetchAll(fetched);
    std::vector<const FetchedBlock*> sources;
    for (const auto& f : fetched)
      if (!f.second.empty()) sources.push_back(&f);
    const uint32_t alg = d_.checksumEnabled ? S3ShuffleHelper::createChecksumAlgorithm(d_.checksumAlgorithm) : 0;
    ensure_codec_runtime();
    const uint32_t codec = (uint32_t)d_.codecId();
    StagedBlocks src(info_, sources);
    const uint32_t n = (uint32_t)sources.size();
    std::vector<int32_t> status(n), bad(n);
    uint64_t total = 0, out = 0;
    const uint64_t guess = codec == B2S_CODEC_NONE ? src.bytes * 2 : src.bytes * 4;
    const int rc = callWithRetry(sorted_, guess, total, [&](uint64_t cap) {
      if (w.frames)
        return b2s_decompress_window_frame_rows_keys_packed(
            codec, alg, n, src.src.data(), src.off.data(), src.len.data(), alg ? src.sliceBase.data() : 0,
            alg ? src.sliceLen.data() : 0, alg ? src.sliceSum.data() : 0, w.nPartitionKeys, w.nKeys, w.keyType,
            w.keyOff, w.keyLen, w.keyNull, w.nFields, w.kind, w.nFns, w.fn, w.fnArg, w.frame, w.valType, w.valOff,
            w.valNull, w.flags, w.dflt, w.lower, w.upper, sorted_.get(), cap, &total, nRecords, &out, status.data(),
            bad.data());
      if (w.offset)
        return b2s_decompress_window_offset_rows_keys_packed(
            codec, alg, n, src.src.data(), src.off.data(), src.len.data(), alg ? src.sliceBase.data() : 0,
            alg ? src.sliceLen.data() : 0, alg ? src.sliceSum.data() : 0, w.nPartitionKeys, w.nKeys, w.keyType,
            w.keyOff, w.keyLen, w.keyNull, w.nFields, w.kind, w.nFns, w.fn, w.fnArg, w.frame, w.valType, w.valOff,
            w.valNull, w.flags, w.dflt, sorted_.get(), cap, &total, nRecords, &out, status.data(), bad.data());
      if (w.aggregate)
        return b2s_decompress_window_aggregate_rows_keys_packed(
            codec, alg, n, src.src.data(), src.off.data(), src.len.data(), alg ? src.sliceBase.data() : 0,
            alg ? src.sliceLen.data() : 0, alg ? src.sliceSum.data() : 0, w.nPartitionKeys, w.nKeys, w.keyType,
            w.keyOff, w.keyLen, w.keyNull, w.nFields, w.kind, w.nFns, w.fn, w.fnArg, w.frame, w.valType, w.valOff,
            w.valNull, sorted_.get(), cap, &total, nRecords, &out, status.data(), bad.data());
      return b2s_decompress_window_rows_keys_packed(
          codec, alg, n, src.src.data(), src.off.data(), src.len.data(), alg ? src.sliceBase.data() : 0,
          alg ? src.sliceLen.data() : 0, alg ? src.sliceSum.data() : 0, w.nPartitionKeys, w.nKeys, w.keyType,
          w.keyOff, w.keyLen, w.keyNull, w.nFields, w.kind, w.nFns, w.fn, w.fnArg, w.limitFn, w.limit, sorted_.get(),
          cap, &total, nRecords, &out, status.data(), bad.data());
    });
    if (rc != 0)
      throw CodecException(std::string(w.frames      ? "b2s_decompress_window_frame_rows_keys_packed: "
                                       : w.offset    ? "b2s_decompress_window_offset_rows_keys_packed: "
                                       : w.aggregate ? "b2s_decompress_window_aggregate_rows_keys_packed: "
                                                     : "b2s_decompress_window_rows_keys_packed: ") +
                           b2s_strerror(rc) + ": " + b2s_last_error());
    for (uint32_t k = 0; k < n; k++) throwBlockStatus(status[k], info_[sources[k]->first].id);
    sortedLen_ = total;
    sortedRecords_ = out;
  }
  // One DISTINCT group's middle stage (b2s_decompress_aggregate_distinct_partition_compress_rows_hash_packed): the key
  // columns G ++ X (the first nGroupKeys G), F as (fn, valType), D as (fn, valType, column).
  struct DistinctArgs {
    uint32_t nGroupKeys, nKeys;
    const uint32_t *keyType, *keyLen;
    uint32_t nAggs;
    const uint32_t *aggFn, *valType;
    uint32_t nDistinct;
    const uint32_t *distinctFn, *distinctValType;
    const int32_t* distinctColumn;
  };
  // A reduce task of the exchange by G ++ X that ends in the map output of the exchange by G (INTEGRATION.md §3s):
  // every non-empty block is fetched (the exchange cache is not consulted) in computeShuffleBlocks order, then ONE call
  // merges, folds and hash-partitions the rows into `out`'s arena, whose map id is this reduce task and whose
  // numPartitions the second exchange's; `out` then commits its .data / .index / .checksum as its own commit() lays
  // them out.  A corrupt block throws as the other reads do, and no file is written.  counts: the call's three.
  std::vector<int64_t> aggregateDistinctRows(S3SerializedShuffleWriter& out, const DistinctArgs& a, uint64_t* counts) {
    std::vector<FetchedBlock> fetched;
    fetchAll(fetched);
    std::vector<const FetchedBlock*> sources;
    for (const auto& f : fetched)
      if (!f.second.empty()) sources.push_back(&f);
    const uint32_t alg = d_.checksumEnabled ? S3ShuffleHelper::createChecksumAlgorithm(d_.checksumAlgorithm) : 0;
    ensure_codec_runtime();
    const uint32_t codec = (uint32_t)d_.codecId();
    StagedBlocks src(info_, sources);
    const uint32_t n = (uint32_t)sources.size(), R = (uint32_t)out.numPartitions();
    std::vector<int32_t> status(n ? n : 1), bad(n ? n : 1);
    // the output rows are at most the input's size plus a partial row per group; the exact size is reported if not
    const uint64_t guess = b2s_partition_compress_bound(codec, d_.lz4BlockSize, R, (src.bytes + 4096) * 4);
    return out.commitFrom(
        "b2s_decompress_aggregate_distinct_partition_compress_rows_hash_packed", guess,
        [&](uint8_t* dst, uint64_t cap, uint64_t* doff, uint64_t* dlen, uint64_t* total, uint64_t* cks, int32_t* st) {
          return b2s_decompress_aggregate_distinct_partition_compress_rows_hash_packed(
              codec, d_.zstdLevel, d_.lz4BlockSize, alg, n, n ? src.src.data() : nullptr, src.off.data(),
              src.len.data(), alg ? src.sliceBase.data() : 0, alg ? src.sliceLen.data() : 0,
              alg ? src.sliceSum.data() : 0, a.nGroupKeys, a.nKeys, a.keyType, a.keyLen, a.nAggs, a.aggFn, a.valType,
              a.nDistinct, a.distinctFn, a.distinctValType, a.distinctColumn, R, dst, cap, doff, dlen, total, cks, st,
              counts, status.data(), bad.data());
        },
        [&] {
          for (uint32_t k = 0; k < n; k++) throwBlockStatus(status[k], info_[sources[k]->first].id);
        });
  }
  // every block of the task, fetched whole, in computeShuffleBlocks order
  void fetchAll(std::vector<FetchedBlock>& fetched) {
    start(true);
    drainWhole(fetched);
    std::sort(fetched.begin(), fetched.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  }
  const uint8_t* sortedData() const { return sorted_.get(); }
  uint64_t sortedLen() const { return sortedLen_; }
  uint64_t sortedRecords() const { return sortedRecords_; }
  uint64_t sortedGroups() const { return sortedGroups_; }

  // want (nullptr = every map): the maps whose blocks are fetched
  void start(bool allowNone, const std::vector<uint8_t>* want = nullptr) {
    iter_.reset();
    info_.clear();
    blocks_.clear();
    decoded_.clear();
    sorted_.reset();
    sortedLen_ = sortedRecords_ = sortedGroups_ = 0;
    remoteBytesRead_ = remoteBlocksFetched_ = 0;
    batches_ = 0;
    if (!allowNone && d_.codecId() == B2S_CODEC_NONE)
      throw UnsupportedOperationException("spark.shuffle.compress=false is served by the stock reader path");
    auto src = computeShuffleBlockStreams(d_, shuffleId_, mapIds_, start_, end_, batch_, info_, remoteBytesRead_,
                                          remoteBlocksFetched_, want);
    iter_.reset(new S3BufferedPrefetchIterator(std::move(src), d_.maxBufferSizeTask, d_.maxConcurrencyTask));
  }

  // every block the prefetcher delivers, whole, appended to `fetched` as (tag, bytes)
  void drainWhole(std::vector<FetchedBlock>& fetched) {
    while (iter_->hasNext()) {
      for (auto& f : iter_->nextBatch(0)) {
        auto& st = *f.stream;
        // the whole block through the adaptor, from its first byte: the buffered head, then (a block larger than the
        // task's budget) the tail straight from the block stream
        std::vector<uint8_t> b((size_t)st.totalBytes());
        int64_t at = 0, r;
        while (at < st.totalBytes() && (r = st.read(b.data() + at, st.totalBytes() - at)) > 0) at += r;
        b.resize((size_t)at);
        fetched.emplace_back(f.tag, std::move(b));
        st.close();  // the budget goes back to the prefetcher before the next fetches are waited for
      }
      batches_++;
    }
    stats_ = iter_->statistics();
  }

  // 1 for each map to fetch: every map, or, with the exchange cache on, those not resident on this thread's device
  std::vector<uint8_t> cacheMisses() {
    std::vector<uint8_t> fetch(mapIds_.size(), 1);
    if (!d_.gpuExchangeCacheBytes || mapIds_.empty()) return fetch;
    ensure_codec_runtime();
    std::vector<uint64_t> len(mapIds_.size());
    lookup((uint32_t)mapIds_.size(), mapIds_.data(), len.data());
    for (size_t m = 0; m < len.size(); m++) fetch[m] = len[m] == UINT64_MAX;
    return fetch;
  }
  // b2s_exchange_lookup of the reader's range for n maps: len[k] is UINT64_MAX when ids[k] is not resident
  void lookup(uint32_t n, const int64_t* ids, uint64_t* len) {
    const int rc = b2s_exchange_lookup(shuffleId_, start_, end_, n, ids, len);
    if (rc < 0) throw CodecException(std::string("b2s_exchange_lookup: ") + b2s_strerror(rc) + ": " + b2s_last_error());
  }
  BlockId cachedBlockId(int64_t mapId) const {
    return end_ - start_ > 1 ? BlockId{BlockId::ShuffleBatch, shuffleId_, mapId, start_, end_}
                             : BlockId{BlockId::Shuffle, shuffleId_, mapId, start_, start_ + 1};
  }

  // the maps not in `fetch`, from the exchange cache in one b2s_exchange_read_packed call: one block per map covering
  // [start, end) (empty ones dropped, as the fetch path drops empty blocks).  Maps it no longer holds go back to `fetch`.
  void readCached(std::vector<uint8_t>& fetch, std::vector<Block>& all, std::vector<std::unique_ptr<uint8_t[]>>& bufs) {
    std::vector<int64_t> ids;
    std::vector<uint32_t> pos;
    for (uint32_t m = 0; m < (uint32_t)mapIds_.size(); m++)
      if (!fetch[m]) {
        ids.push_back(mapIds_[m]);
        pos.push_back(m);
      }
    if (ids.empty()) return;
    const uint32_t n = (uint32_t)ids.size();
    std::vector<uint64_t> off(n), len(n);
    std::vector<int32_t> status(n);
    lookup(n, ids.data(), len.data());
    uint64_t guess = 0, total = 0;
    for (uint64_t l : len) guess += l == UINT64_MAX ? 0 : l;
    std::unique_ptr<uint8_t[]> buf;
    const int rc = callWithRetry(buf, guess, total, [&](uint64_t cap) {  // an entry stored again may have grown
      return b2s_exchange_read_packed(shuffleId_, start_, end_, n, ids.data(), buf.get(), cap, off.data(), len.data(),
                                      &total, status.data());
    });
    if (rc != 0)
      throw CodecException(std::string("b2s_exchange_read_packed: ") + b2s_strerror(rc) + ": " + b2s_last_error());
    for (uint32_t k = 0; k < n; k++) {
      if (status[k] != B2S_OK) {
        fetch[pos[k]] = 1;
        continue;
      }
      if (!len[k]) continue;
      Block blk;
      blk.id = cachedBlockId(ids[k]);
      blk.data = buf.get() + off[k];
      blk.len = len[k];
      all.push_back(blk);
    }
    bufs.push_back(std::move(buf));
  }

  // SURVEY.md §8(f)-2: drain the blocks the prefetcher has completed, verify + decode them in ONE C-ABI batch, give
  // their buffers back to the prefetcher's budget.  Returns false when the task has no more blocks.
  bool nextBatch(size_t maxBlocks) {
    if (!iter_) throw RuntimeException("reader is not open");
    blocks_.clear();
    decoded_.clear();
    if (!iter_->hasNext()) {
      stats_ = iter_->statistics();
      return false;
    }
    std::vector<S3BufferedPrefetchIterator::Fetched> got = iter_->nextBatch(maxBlocks);
    const uint32_t n = (uint32_t)got.size();
    const bool verify = d_.checksumEnabled;
    const uint32_t alg = verify ? S3ShuffleHelper::createChecksumAlgorithm(d_.checksumAlgorithm) : 0;
    std::vector<const uint8_t*> src(n);
    std::vector<uint64_t> len(n), dlen(n), dcap(n);
    std::vector<uint32_t> nsl(n);
    std::vector<const uint64_t*> slen(n), ssum(n);
    std::vector<std::unique_ptr<uint8_t[]>> spill;  // blocks larger than the task's buffer budget
    for (uint32_t k = 0; k < n; k++) {
      auto& st = *got[k].stream;
      const ShuffleBlockInfo& bi = info_[got[k].tag];
      src[k] = st.buffered();
      len[k] = (uint64_t)st.bufferedBytes();
      if (st.totalBytes() > st.bufferSize()) {  // read the tail through the adaptor, as the JVM codec stream would
        std::unique_ptr<uint8_t[]> full(new uint8_t[(size_t)st.totalBytes()]);
        int64_t at = 0, r;
        while (at < st.totalBytes() && (r = st.read(full.get() + at, st.totalBytes() - at)) > 0) at += r;
        src[k] = full.get();
        len[k] = (uint64_t)at;
        spill.push_back(std::move(full));
      }
      nsl[k] = (uint32_t)bi.sliceLen.size();
      slen[k] = bi.sliceLen.data();
      ssum[k] = bi.sliceSum.data();
    }
    ensure_codec_runtime();
    const int codec = d_.codecId();
    std::vector<int32_t> status(n), bad(n);
    int rc = b2s_decompressed_size_batch((uint32_t)codec, n, src.data(), len.data(), dlen.data(), status.data());
    if (rc != 0) throw CodecException(std::string("b2s_decompressed_size_batch: ") + b2s_strerror(rc) + ": " + b2s_last_error());
    uint64_t cap = 0;
    for (uint32_t k = 0; k < n; k++) cap += dlen[k];
    std::unique_ptr<uint8_t[]> out(new uint8_t[(size_t)(cap ? cap : 1)]);
    std::vector<uint8_t*> dst(n);
    uint64_t o = 0;
    for (uint32_t k = 0; k < n; k++) {
      dst[k] = out.get() + o;
      dcap[k] = dlen[k];
      o += dlen[k];
    }
    std::string rcText;
    if (d_.gpuCoalesce) {
      CodecRequest r;
      r.op = 1;
      r.codec = (uint32_t)codec;
      r.checksum_alg = alg;
      r.n = n;
      r.src = src.data();
      r.src_len = len.data();
      r.dst = dst.data();
      r.dst_cap = dcap.data();
      r.dst_len = dlen.data();
      r.n_slices = verify ? nsl.data() : nullptr;
      r.slice_len = verify ? slen.data() : nullptr;
      r.slice_checksum = verify ? ssum.data() : nullptr;
      r.bad_slice = bad.data();
      r.status = status.data();
      rc = d_.queue.submit(r);
      rcText = r.error;
    } else {
      rc = b2s_decompress_batch((uint32_t)codec, alg, n, src.data(), len.data(), verify ? nsl.data() : nullptr,
                                verify ? slen.data() : nullptr, verify ? ssum.data() : nullptr, dst.data(), dcap.data(),
                                dlen.data(), status.data(), bad.data());
      if (rc != 0) rcText = b2s_last_error();
    }
    for (auto& f : got) f.stream->close();  // onClose(bufferSize): the budget goes back to the prefetcher
    if (rc != 0) throw CodecException(std::string("b2s_decompress_batch: ") + b2s_strerror(rc) + ": " + rcText);
    for (uint32_t k = 0; k < n; k++) {
      const BlockId& id = info_[got[k].tag].id;
      throwBlockStatus(status[k], id);
      Block blk;
      blk.id = id;
      blk.data = dst[k];
      blk.len = dlen[k];
      blocks_.push_back(blk);
    }
    decoded_.push_back(std::move(out));
    batches_++;
    return true;
  }
  const std::vector<Block>& blocks() const { return blocks_; }
  uint64_t remoteBytesRead() const { return remoteBytesRead_; }
  uint64_t remoteBlocksFetched() const { return remoteBlocksFetched_; }
  uint64_t batches() const { return batches_; }
  S3BufferedPrefetchIterator::Statistics statistics() { return iter_ ? iter_->statistics() : stats_; }

 private:
  S3ShuffleDispatcher& d_;
  int32_t shuffleId_;
  std::vector<int64_t> mapIds_;
  int32_t start_, end_;
  bool batch_;
  std::vector<ShuffleBlockInfo> info_;
  std::unique_ptr<S3BufferedPrefetchIterator> iter_;
  std::vector<Block> blocks_;
  std::vector<std::unique_ptr<uint8_t[]>> decoded_;
  std::unique_ptr<uint8_t[]> sorted_;  // readSorted(): the task's records in key order
  uint64_t sortedLen_ = 0, sortedRecords_ = 0, sortedGroups_ = 0;
  uint64_t remoteBytesRead_ = 0, remoteBlocksFetched_ = 0, batches_ = 0;
  S3BufferedPrefetchIterator::Statistics stats_;
};

// the prefetcher on its own (no codec), for the CPU-side tests and for callers that want the compressed blocks
class PrefetchHandle {
 public:
  PrefetchHandle(S3ShuffleDispatcher& d, int32_t shuffleId, const std::vector<int64_t>& mapIds, int32_t start,
                 int32_t end, bool batch, int64_t maxBufferSize, int maxThreads) {
    auto src = computeShuffleBlockStreams(d, shuffleId, mapIds, start, end, batch || d.forceBatchFetch, info, remoteBytes,
                                          remoteBlocks);
    iter.reset(new S3BufferedPrefetchIterator(std::move(src), maxBufferSize > 0 ? maxBufferSize : d.maxBufferSizeTask,
                                              maxThreads > 0 ? maxThreads : d.maxConcurrencyTask));
  }
  ~PrefetchHandle() {
    open.clear();   // close the streams the caller still holds before the iterator goes away
    iter.reset();
  }
  std::vector<ShuffleBlockInfo> info;
  uint64_t remoteBytes = 0, remoteBlocks = 0, nextHandle = 1;
  std::map<uint64_t, S3BufferedPrefetchIterator::Fetched> open;
  std::unique_ptr<S3BufferedPrefetchIterator> iter;
};

}  // namespace host
}  // namespace b2s

// =====================================================================================================
// C wrapper
// =====================================================================================================
using namespace b2s::host;

static thread_local std::string t_err;
struct b2sh_dispatcher { std::unique_ptr<S3ShuffleDispatcher> d; };
struct b2sh_writer { std::unique_ptr<S3ShuffleMapOutputWriter> w; int32_t n; };
struct b2sh_serialized_writer { std::unique_ptr<S3SerializedShuffleWriter> w; };
struct b2sh_reader { std::unique_ptr<S3ShuffleReader> r; };
struct b2sh_prefetch { std::unique_ptr<PrefetchHandle> p; };
struct b2sh_codec { std::unique_ptr<B200CompressionCodec> c; };
struct b2sh_ostream { std::unique_ptr<B200CompressedOutputStream> s; };
struct b2sh_istream { std::unique_ptr<B200CompressedInputStream> s; };

template <typename F>
static int guarded(F&& f) {
  try {
    f();
    t_err.clear();
    return B2SH_OK;
  } catch (const RuntimeException& e) { t_err = e.what(); return B2SH_E_RUNTIME;
  } catch (const IOException& e) { t_err = e.what(); return B2SH_E_IO;
  } catch (const SparkException& e) { t_err = e.what(); return B2SH_E_SPARK;
  } catch (const UnsupportedOperationException& e) { t_err = e.what(); return B2SH_E_UNSUPPORTED;
  } catch (const CodecException& e) { t_err = e.what(); return B2SH_E_CODEC;
  } catch (const std::exception& e) { t_err = e.what(); return B2SH_E_RUNTIME; }
}

extern "C" {

const char* b2sh_last_error(void) { return t_err.c_str(); }

int b2sh_dispatcher_create(const char* conf, b2sh_dispatcher** out) {
  return guarded([&] { *out = new b2sh_dispatcher{std::make_unique<S3ShuffleDispatcher>(conf ? conf : "")}; });
}
void b2sh_dispatcher_destroy(b2sh_dispatcher* d) { delete d; }
int b2sh_dispatcher_get_path(b2sh_dispatcher* d, int kind, int32_t shuffle_id, int64_t map_id, char* buf, uint32_t cap) {
  return guarded([&] {
    BlockId::Kind k = kind == 0 ? BlockId::Data : kind == 1 ? BlockId::Index : BlockId::Checksum;
    std::string p = d->d->getPath(BlockId{k, shuffle_id, map_id, 0, 0});
    if (p.size() + 1 > cap) throw RuntimeException("path buffer too small");
    memcpy(buf, p.c_str(), p.size() + 1);
  });
}
int b2sh_dispatcher_remove_shuffle(b2sh_dispatcher* d, int32_t shuffle_id) {
  return guarded([&] {
    d->d->removeShuffle(shuffle_id);
    S3ShuffleHelper::purgeCachedDataForShuffle(*d->d, shuffle_id);
    // the map outputs kept in HBM go too (without a device or before b2s_init nothing was cached: nothing to do)
    if (d->d->gpuExchangeCacheBytes) (void)b2s_exchange_remove(shuffle_id, -1);
  });
}
int b2sh_helper_checksum_algorithm(const char* name) {
  int id = 0;
  int rc = guarded([&] { id = (int)S3ShuffleHelper::createChecksumAlgorithm(name ? name : ""); });
  return rc ? rc : id;
}
static int copy_out(const std::vector<int64_t>& v, int64_t* out, uint32_t cap, uint32_t* count) {
  *count = (uint32_t)v.size();
  if (v.size() > cap) throw RuntimeException("output array too small");
  memcpy(out, v.data(), v.size() * 8);
  return 0;
}
int b2sh_helper_get_partition_lengths(b2sh_dispatcher* d, int32_t s, int64_t m, int64_t* out, uint32_t cap, uint32_t* count) {
  return guarded([&] { copy_out(S3ShuffleHelper::getPartitionLengths(*d->d, s, m), out, cap, count); });
}
int b2sh_helper_get_checksums(b2sh_dispatcher* d, int32_t s, int64_t m, int64_t* out, uint32_t cap, uint32_t* count) {
  return guarded([&] { copy_out(S3ShuffleHelper::getChecksums(*d->d, s, m), out, cap, count); });
}

int b2sh_writer_create(b2sh_dispatcher* d, int32_t shuffle_id, int64_t map_id, int32_t num_partitions, b2sh_writer** out) {
  return guarded([&] {
    *out = new b2sh_writer{std::make_unique<S3ShuffleMapOutputWriter>(*d->d, shuffle_id, map_id, num_partitions), num_partitions};
  });
}
int b2sh_writer_open_partition(b2sh_writer* w, int32_t reduce_id) { return guarded([&] { w->w->getPartitionWriter(reduce_id); }); }
int b2sh_writer_write(b2sh_writer* w, const uint8_t* bytes, uint64_t n) { return guarded([&] { w->w->write(bytes, n); }); }
int b2sh_writer_close_partition(b2sh_writer* w) { return guarded([&] { w->w->closePartition(); }); }
int b2sh_writer_commit_all_partitions(b2sh_writer* w, const int64_t* checksums_in, int64_t* partition_lengths_out) {
  return guarded([&] {
    std::vector<int64_t> l = w->w->commitAllPartitions(checksums_in);
    memcpy(partition_lengths_out, l.data(), l.size() * 8);
  });
}
int b2sh_writer_abort(b2sh_writer* w) { return guarded([&] { w->w->abort(); }); }
void b2sh_writer_destroy(b2sh_writer* w) { delete w; }

int b2sh_serialized_writer_create(b2sh_dispatcher* d, int32_t shuffle_id, int64_t map_id, int32_t num_partitions,
                                  b2sh_serialized_writer** out) {
  return guarded([&] {
    *out = new b2sh_serialized_writer{std::make_unique<S3SerializedShuffleWriter>(*d->d, shuffle_id, map_id, num_partitions)};
  });
}
int b2sh_serialized_writer_hash_rows(b2sh_serialized_writer* w, uint32_t n_keys, const uint32_t* key_type,
                                     const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field) {
  return guarded([&] { w->w->hashRows(n_keys, key_type, key_off, key_len, key_null_field); });
}
int b2sh_serialized_writer_range_rows(b2sh_serialized_writer* w, uint32_t n_keys, const uint32_t* key_type,
                                      const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
                                      uint32_t n_bounds, const uint8_t* bound_base, uint64_t bound_bytes,
                                      const uint32_t* bound_len) {
  return guarded([&] {
    w->w->rangeRows(n_keys, key_type, key_off, key_len, key_null_field, n_bounds, bound_base, bound_bytes, bound_len);
  });
}
int b2sh_serialized_writer_round_robin_rows(b2sh_serialized_writer* w, uint32_t num_partitions, int32_t start_position,
                                            uint32_t sort_rows) {
  return guarded([&] { w->w->roundRobinRows(num_partitions, start_position, sort_rows); });
}
int b2sh_serialized_writer_aggregate_rows(b2sh_serialized_writer* w, uint32_t n_aggs, const uint32_t* agg_fn,
                                          const uint32_t* val_type, const uint32_t* val_off,
                                          const int32_t* val_null_field) {
  return guarded([&] { w->w->aggregateRows(n_aggs, agg_fn, val_type, val_off, val_null_field); });
}
int b2sh_serialized_writer_grouping_sets(b2sh_serialized_writer* w, uint32_t n_sets, const uint32_t* set_mask) {
  return guarded([&] { w->w->groupingSets(n_sets, set_mask); });
}
int b2sh_serialized_writer_window_limit(b2sh_serialized_writer* w, uint32_t n_partition_keys, uint32_t n_keys,
                                        const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                        const int32_t* key_null_field, uint32_t limit_fn, int32_t limit) {
  return guarded([&] {
    w->w->windowLimit(n_partition_keys, n_keys, key_type, key_off, key_len, key_null_field, limit_fn, limit);
  });
}
int b2sh_serialized_writer_insert(b2sh_serialized_writer* w, int32_t partition_id, const uint8_t* bytes, uint64_t len) {
  return guarded([&] { w->w->insertRecord(partition_id, bytes, len); });
}
int b2sh_serialized_writer_commit(b2sh_serialized_writer* w, int64_t* partition_lengths_out) {
  return guarded([&] {
    std::vector<int64_t> l = w->w->commit();
    memcpy(partition_lengths_out, l.data(), l.size() * 8);
  });
}
void b2sh_serialized_writer_destroy(b2sh_serialized_writer* w) { delete w; }

int b2sh_single_spill_transfer(b2sh_dispatcher* d, int32_t shuffle_id, int64_t map_id, const char* spill_file,
                               const int64_t* partition_lengths, const int64_t* checksums, uint32_t num_partitions,
                               int verify_on_transfer) {
  return guarded([&] {
    S3SingleSpillShuffleMapOutputWriter w(*d->d, shuffle_id, map_id);
    std::vector<int64_t> l(partition_lengths, partition_lengths + num_partitions);
    std::vector<int64_t> c(num_partitions, 0);
    if (checksums) c.assign(checksums, checksums + num_partitions);
    w.transferMapSpillFile(spill_file ? spill_file : "", l, c, verify_on_transfer != 0);
  });
}

int b2sh_reader_create(b2sh_dispatcher* d, int32_t shuffle_id, const int64_t* map_ids, uint32_t n_maps, int32_t start_partition,
                       int32_t end_partition, int do_batch_fetch, b2sh_reader** out) {
  return guarded([&] {
    *out = new b2sh_reader{std::make_unique<S3ShuffleReader>(*d->d, shuffle_id, std::vector<int64_t>(map_ids, map_ids + n_maps),
                                                             start_partition, end_partition, do_batch_fetch != 0)};
  });
}
int b2sh_reader_read(b2sh_reader* r, uint32_t* n_blocks) {
  return guarded([&] {
    r->r->read();
    *n_blocks = (uint32_t)r->r->blocks().size();
  });
}
// a sorted read's result: its bytes, their length, the records read and (the aggregated reads) the groups
static void sorted_result(const S3ShuffleReader& r, const uint8_t** data, uint64_t* len, uint64_t* n_records,
                          uint64_t* n_groups = nullptr) {
  *data = r.sortedData();
  *len = r.sortedLen();
  *n_records = r.sortedRecords();
  if (n_groups) *n_groups = r.sortedGroups();
}
int b2sh_reader_read_sorted(b2sh_reader* r, uint32_t record_bytes, uint32_t key_off, uint32_t key_len,
                            const uint8_t** data, uint64_t* len, uint64_t* n_records) {
  return guarded([&] {
    r->r->readSorted(record_bytes, key_off, key_len);
    sorted_result(*r->r, data, len, n_records);
  });
}
int b2sh_reader_read_sorted_rows(b2sh_reader* r, uint32_t key_type, uint32_t key_off, uint32_t key_len,
                                 int32_t null_field, const uint8_t** data, uint64_t* len, uint64_t* n_records) {
  return guarded([&] {
    r->r->readRows(S3ShuffleReader::RowKeys{1, &key_type, &key_off, &key_len, &null_field, false}, nullptr);
    sorted_result(*r->r, data, len, n_records);
  });
}
int b2sh_reader_read_aggregated_rows(b2sh_reader* r, uint32_t key_type, uint32_t key_off, uint32_t key_len,
                                     int32_t null_field, uint32_t n_aggs, const uint32_t* agg_op,
                                     const uint32_t* agg_off, const int32_t* agg_null_field, const uint8_t** data,
                                     uint64_t* len, uint64_t* n_records, uint64_t* n_groups) {
  return guarded([&] {
    const S3ShuffleReader::RowAggregates aggs{n_aggs, agg_op, agg_off, agg_null_field};
    r->r->readRows(S3ShuffleReader::RowKeys{1, &key_type, &key_off, &key_len, &null_field, false}, &aggs);
    sorted_result(*r->r, data, len, n_records, n_groups);
  });
}
int b2sh_reader_read_sorted_rows_keys(b2sh_reader* r, uint32_t n_keys, const uint32_t* key_type,
                                      const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
                                      const uint8_t** data, uint64_t* len, uint64_t* n_records) {
  return guarded([&] {
    r->r->readRows(S3ShuffleReader::RowKeys{n_keys, key_type, key_off, key_len, key_null_field, true}, nullptr);
    sorted_result(*r->r, data, len, n_records);
  });
}
int b2sh_reader_read_aggregated_rows_keys(b2sh_reader* r, uint32_t n_keys, const uint32_t* key_type,
                                          const uint32_t* key_off, const uint32_t* key_len,
                                          const int32_t* key_null_field, uint32_t n_aggs, const uint32_t* agg_op,
                                          const uint32_t* agg_off, const int32_t* agg_null_field,
                                          const uint8_t** data, uint64_t* len, uint64_t* n_records,
                                          uint64_t* n_groups) {
  return guarded([&] {
    const S3ShuffleReader::RowAggregates aggs{n_aggs, agg_op, agg_off, agg_null_field};
    r->r->readRows(S3ShuffleReader::RowKeys{n_keys, key_type, key_off, key_len, key_null_field, true}, &aggs);
    sorted_result(*r->r, data, len, n_records, n_groups);
  });
}
int b2sh_reader_read_joined_rows(b2sh_reader* left, b2sh_reader* right, uint32_t join_type, uint32_t n_keys,
                                 const uint32_t* key_type, const uint32_t* key_len, const uint32_t* left_key_off,
                                 const int32_t* left_key_null_field, const uint32_t* right_key_off,
                                 const int32_t* right_key_null_field, uint32_t n_left_fields,
                                 const uint8_t* left_field_kind, uint32_t n_right_fields,
                                 const uint8_t* right_field_kind, const uint8_t** data, uint64_t* len,
                                 uint64_t* n_left_records, uint64_t* n_right_records, uint64_t* n_out_records) {
  return guarded([&] {
    const S3ShuffleReader::JoinArgs j{join_type,     n_keys,         key_type,        key_len,
                                      left_key_off,  left_key_null_field, right_key_off, right_key_null_field,
                                      n_left_fields, left_field_kind, n_right_fields,  right_field_kind};
    left->r->readJoined(*right->r, j, n_left_records, n_right_records);
    sorted_result(*left->r, data, len, n_out_records);
  });
}
int b2sh_reader_read_window_rows(b2sh_reader* r, uint32_t n_partition_keys, uint32_t n_keys, const uint32_t* key_type,
                                 const uint32_t* key_off, const uint32_t* key_len, const int32_t* key_null_field,
                                 uint32_t n_fields, const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn,
                                 const int32_t* fn_arg, uint32_t limit_fn, int32_t limit, const uint8_t** data,
                                 uint64_t* len, uint64_t* n_records, uint64_t* n_out_records) {
  return guarded([&] {
    const S3ShuffleReader::WindowArgs w{n_partition_keys, n_keys,     key_type, key_off, key_len,  key_null_field,
                                        n_fields,         field_kind, n_fns,    fn,      fn_arg,   limit_fn,
                                        limit};
    r->r->readWindowRows(w, n_records);
    sorted_result(*r->r, data, len, n_out_records);
  });
}
int b2sh_reader_read_window_aggregate_rows(b2sh_reader* r, uint32_t n_partition_keys, uint32_t n_keys,
                                           const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                           const int32_t* key_null_field, uint32_t n_fields,
                                           const uint8_t* field_kind, uint32_t n_fns, const uint32_t* fn,
                                           const int32_t* fn_arg, const uint32_t* fn_frame, const uint32_t* val_type,
                                           const uint32_t* val_off, const int32_t* val_null_field,
                                           const uint8_t** data, uint64_t* len, uint64_t* n_records,
                                           uint64_t* n_out_records) {
  return guarded([&] {
    const S3ShuffleReader::WindowArgs w{n_partition_keys, n_keys,   key_type,        key_off,          key_len,
                                        key_null_field,   n_fields, field_kind,      n_fns,            fn,
                                        fn_arg,           B2S_WINDOW_NO_LIMIT, 0,    fn_frame,         val_type,
                                        val_off,          val_null_field,      true};
    r->r->readWindowRows(w, n_records);
    sorted_result(*r->r, data, len, n_out_records);
  });
}
int b2sh_reader_read_window_offset_rows(b2sh_reader* r, uint32_t n_partition_keys, uint32_t n_keys,
                                        const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                        const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
                                        uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg,
                                        const uint32_t* fn_frame, const uint32_t* val_type, const uint32_t* val_off,
                                        const int32_t* val_null_field, const uint32_t* fn_flags,
                                        const uint64_t* fn_default, const uint8_t** data, uint64_t* len,
                                        uint64_t* n_records, uint64_t* n_out_records) {
  return guarded([&] {
    S3ShuffleReader::WindowArgs w{n_partition_keys, n_keys,   key_type,        key_off,          key_len,
                                  key_null_field,   n_fields, field_kind,      n_fns,            fn,
                                  fn_arg,           B2S_WINDOW_NO_LIMIT, 0,    fn_frame,         val_type,
                                  val_off,          val_null_field,      true};
    w.flags = fn_flags;
    w.dflt = fn_default;
    w.offset = true;
    r->r->readWindowRows(w, n_records);
    sorted_result(*r->r, data, len, n_out_records);
  });
}
int b2sh_reader_read_window_frame_rows(b2sh_reader* r, uint32_t n_partition_keys, uint32_t n_keys,
                                       const uint32_t* key_type, const uint32_t* key_off, const uint32_t* key_len,
                                       const int32_t* key_null_field, uint32_t n_fields, const uint8_t* field_kind,
                                       uint32_t n_fns, const uint32_t* fn, const int32_t* fn_arg,
                                       const uint32_t* fn_frame, const uint32_t* val_type, const uint32_t* val_off,
                                       const int32_t* val_null_field, const uint32_t* fn_flags,
                                       const uint64_t* fn_default, const int64_t* frame_lower,
                                       const int64_t* frame_upper, const uint8_t** data, uint64_t* len,
                                       uint64_t* n_records, uint64_t* n_out_records) {
  return guarded([&] {
    S3ShuffleReader::WindowArgs w{n_partition_keys, n_keys,   key_type,        key_off,          key_len,
                                  key_null_field,   n_fields, field_kind,      n_fns,            fn,
                                  fn_arg,           B2S_WINDOW_NO_LIMIT, 0,    fn_frame,         val_type,
                                  val_off,          val_null_field,      true};
    w.flags = fn_flags;
    w.dflt = fn_default;
    w.offset = true;
    w.lower = frame_lower;
    w.upper = frame_upper;
    w.frames = true;
    r->r->readWindowRows(w, n_records);
    sorted_result(*r->r, data, len, n_out_records);
  });
}
int b2sh_reader_aggregate_distinct_rows(b2sh_reader* r, b2sh_serialized_writer* w, uint32_t n_group_keys,
                                        uint32_t n_keys, const uint32_t* key_type, const uint32_t* key_len,
                                        uint32_t n_aggs, const uint32_t* agg_fn, const uint32_t* val_type,
                                        uint32_t n_distinct, const uint32_t* distinct_fn,
                                        const uint32_t* distinct_val_type, const int32_t* distinct_column,
                                        int64_t* partition_lengths_out, uint64_t* counts) {
  return guarded([&] {
    if (!w || !partition_lengths_out || !counts) throw RuntimeException("Precondition: null argument.");
    const S3ShuffleReader::DistinctArgs a{n_group_keys, n_keys, key_type, key_len, n_aggs, agg_fn, val_type,
                                          n_distinct, distinct_fn, distinct_val_type, distinct_column};
    const std::vector<int64_t> lengths = r->r->aggregateDistinctRows(*w->w, a, counts);
    std::copy(lengths.begin(), lengths.end(), partition_lengths_out);
  });
}
int b2sh_reader_block(b2sh_reader* r, uint32_t k, int64_t* map_id, int32_t* start_reduce, int32_t* end_reduce,
                      const uint8_t** data, uint64_t* len) {
  return guarded([&] {
    if (k >= r->r->blocks().size()) throw RuntimeException("block index out of range");
    const auto& b = r->r->blocks()[k];
    *map_id = b.id.mapId;
    *start_reduce = b.id.reduceId;
    *end_reduce = b.id.kind == BlockId::ShuffleBatch ? b.id.endReduceId : b.id.reduceId + 1;
    *data = b.data;
    *len = b.len;
  });
}
uint64_t b2sh_reader_remote_bytes_read(b2sh_reader* r) { return r->r->remoteBytesRead(); }
void b2sh_reader_destroy(b2sh_reader* r) { delete r; }

static void copy_line(const std::string& line, char* buf, uint32_t cap) {
  if (!buf || !cap) return;
  const size_t k = std::min<size_t>(line.size(), cap - 1);
  memcpy(buf, line.data(), k);
  buf[k] = 0;
}
static void fill_prefetch_stats(const S3BufferedPrefetchIterator::Statistics& s, uint64_t* out, char* line, uint32_t cap) {
  if (out) {
    out[0] = (uint64_t)s.bytesRead;
    out[1] = (uint64_t)s.numStreams;
    out[2] = (uint64_t)s.timeWaiting;
    out[3] = (uint64_t)s.timePrefetching;
    out[4] = (uint64_t)s.totalRuntime;
    out[5] = (uint64_t)s.activeThreads;
    out[6] = (uint64_t)s.peakMemoryUsage;
    out[7] = (uint64_t)s.peakThreads;
  }
  copy_line(s.line, line, cap);
}

int b2sh_writer_statistics(b2sh_writer* w, uint64_t* bytes, uint64_t* nanos, char* line, uint32_t cap) {
  return guarded([&] {
    const S3MeasureOutputStream* m = w->w->measure();
    if (!m) throw RuntimeException("no .data object was written");
    if (bytes) *bytes = (uint64_t)m->bytes();
    if (nanos) *nanos = (uint64_t)m->timings();
    copy_line(m->statistics(), line, cap);
  });
}

int b2sh_serialized_writer_statistics(b2sh_serialized_writer* w, uint64_t* bytes, uint64_t* nanos, char* line,
                                      uint32_t cap) {
  return guarded([&] {
    const S3MeasureOutputStream* m = w->w->measure();
    if (!m) throw RuntimeException("no .data object was written");
    if (bytes) *bytes = (uint64_t)m->bytes();
    if (nanos) *nanos = (uint64_t)m->timings();
    copy_line(m->statistics(), line, cap);
  });
}

int b2sh_reader_open(b2sh_reader* r) { return guarded([&] { r->r->open(); }); }
int b2sh_reader_next_batch(b2sh_reader* r, uint32_t max_blocks, uint32_t* n_blocks) {
  return guarded([&] {
    const bool more = r->r->nextBatch(max_blocks);
    *n_blocks = more ? (uint32_t)r->r->blocks().size() : 0;
  });
}
int b2sh_reader_statistics(b2sh_reader* r, uint64_t* out8, uint64_t* batches, char* line, uint32_t cap) {
  return guarded([&] {
    fill_prefetch_stats(r->r->statistics(), out8, line, cap);
    if (batches) *batches = r->r->batches();
  });
}

int b2sh_prefetch_create(b2sh_dispatcher* d, int32_t shuffle_id, const int64_t* map_ids, uint32_t n_maps,
                         int32_t start_partition, int32_t end_partition, int do_batch_fetch, int64_t max_buffer_size,
                         int32_t max_threads, b2sh_prefetch** out) {
  return guarded([&] {
    *out = new b2sh_prefetch{std::make_unique<PrefetchHandle>(*d->d, shuffle_id, std::vector<int64_t>(map_ids, map_ids + n_maps),
                                                              start_partition, end_partition, do_batch_fetch != 0,
                                                              max_buffer_size, max_threads)};
  });
}
int b2sh_prefetch_has_next(b2sh_prefetch* p) { return p->p->iter->hasNext() ? 1 : 0; }
int b2sh_prefetch_next(b2sh_prefetch* p, int64_t* map_id, int32_t* start_reduce, int32_t* end_reduce,
                       const uint8_t** data, uint64_t* len, uint64_t* stream) {
  return guarded([&] {
    S3BufferedPrefetchIterator::Fetched f = p->p->iter->next();
    *map_id = f.id.mapId;
    *start_reduce = f.id.reduceId;
    *end_reduce = f.id.kind == BlockId::ShuffleBatch ? f.id.endReduceId : f.id.reduceId + 1;
    *data = f.stream->buffered();
    *len = (uint64_t)f.stream->bufferedBytes();
    *stream = p->p->nextHandle++;
    p->p->open.emplace(*stream, std::move(f));
  });
}
int b2sh_prefetch_close_stream(b2sh_prefetch* p, uint64_t stream) {
  return guarded([&] {
    auto it = p->p->open.find(stream);
    if (it == p->p->open.end()) return;  // "Double close detected. Ignoring."
    it->second.stream->close();
    p->p->open.erase(it);
  });
}
int b2sh_prefetch_statistics(b2sh_prefetch* p, uint64_t* out8, char* line, uint32_t cap) {
  return guarded([&] { fill_prefetch_stats(p->p->iter->statistics(), out8, line, cap); });
}
void b2sh_prefetch_destroy(b2sh_prefetch* p) { delete p; }

int b2sh_dispatcher_queue_statistics(b2sh_dispatcher* d, uint64_t* out4) {
  return guarded([&] {
    const CoalescingQueue::Statistics st = d->d->queue.statistics();
    out4[0] = st.calls;
    out4[1] = st.batches;
    out4[2] = st.maxMerged;
    out4[3] = st.streams;
  });
}
int b2sh_dispatcher_queue_compress(b2sh_dispatcher* d, uint32_t codec, int32_t level, uint32_t codec_block_size,
                                   uint32_t checksum_alg, uint32_t n, const uint8_t* const* src, const uint64_t* src_len,
                                   uint8_t* const* dst, const uint64_t* dst_cap, uint64_t* dst_len,
                                   uint64_t* checksum_out, int32_t* status) {
  return guarded([&] {
    ensure_codec_runtime();
    CodecRequest r;
    r.op = 0;
    r.codec = codec;
    r.level = level;
    r.block_size = codec_block_size;
    r.checksum_alg = checksum_alg;
    r.n = n;
    r.src = src;
    r.src_len = src_len;
    r.dst = dst;
    r.dst_cap = dst_cap;
    r.dst_len = dst_len;
    r.checksum_out = checksum_out;
    r.status = status;
    submit_or_throw(d->d->queue, r, "b2s_compress_batch");
  });
}
int b2sh_dispatcher_queue_decompress(b2sh_dispatcher* d, uint32_t codec, uint32_t checksum_alg, uint32_t n,
                                     const uint8_t* const* src, const uint64_t* src_len, const uint32_t* n_slices,
                                     const uint64_t* const* slice_len, const uint64_t* const* slice_checksum,
                                     uint8_t* const* dst, const uint64_t* dst_cap, uint64_t* dst_len, int32_t* status,
                                     int32_t* bad_slice) {
  return guarded([&] {
    ensure_codec_runtime();
    CodecRequest r;
    r.op = 1;
    r.codec = codec;
    r.checksum_alg = checksum_alg;
    r.n = n;
    r.src = src;
    r.src_len = src_len;
    r.dst = dst;
    r.dst_cap = dst_cap;
    r.dst_len = dst_len;
    r.n_slices = n_slices;
    r.slice_len = slice_len;
    r.slice_checksum = slice_checksum;
    r.bad_slice = bad_slice;
    r.status = status;
    submit_or_throw(d->d->queue, r, "b2s_decompress_batch");
  });
}

int b2sh_codec_create(b2sh_dispatcher* d, b2sh_codec** out) {
  return guarded([&] {
    *out = new b2sh_codec{std::make_unique<B200CompressionCodec>(d->d->codecId(), d->d->lz4BlockSize, d->d->gpuCodecBufferSize)};
  });
}
int b2sh_codec_supports_concatenation(b2sh_codec* c) {
  return B200CompressionCodec::supportsConcatenationOfSerializedStreams(c->c->codecId()) ? 1 : 0;
}
void b2sh_codec_destroy(b2sh_codec* c) { delete c; }
int b2sh_codec_output_stream(b2sh_codec* c, b2sh_sink_fn sink, void* ctx, b2sh_ostream** out) {
  return guarded([&] {
    if (!sink) throw RuntimeException("sink is null");
    *out = new b2sh_ostream{std::make_unique<B200CompressedOutputStream>(*c->c, [sink, ctx](const uint8_t* b, uint64_t n) {
      if (sink(ctx, b, n) < 0) throw IOException("the sink rejected the write");
    })};
  });
}
int b2sh_ostream_write(b2sh_ostream* s, const uint8_t* bytes, uint64_t n) { return guarded([&] { s->s->write(bytes, n); }); }
int b2sh_ostream_flush(b2sh_ostream* s) { return guarded([&] { s->s->flush(); }); }
int b2sh_ostream_close(b2sh_ostream* s, uint64_t* bytes_in, uint64_t* bytes_out, uint32_t* streams) {
  return guarded([&] {
    s->s->close();
    if (bytes_in) *bytes_in = s->s->bytesIn();
    if (bytes_out) *bytes_out = s->s->bytesOut();
    if (streams) *streams = s->s->streamsEmitted();
  });
}
void b2sh_ostream_destroy(b2sh_ostream* s) { delete s; }
int b2sh_codec_input_stream(b2sh_codec* c, b2sh_source_fn source, void* ctx, b2sh_istream** out) {
  return guarded([&] {
    if (!source) throw RuntimeException("source is null");
    *out = new b2sh_istream{std::make_unique<B200CompressedInputStream>(*c->c, [source, ctx](uint8_t* b, uint64_t cap) {
      return source(ctx, b, cap);
    })};
  });
}
int b2sh_istream_read(b2sh_istream* s, uint8_t* buf, uint64_t cap, int64_t* got) {
  return guarded([&] { *got = s->s->read(buf, cap); });
}
int b2sh_istream_close(b2sh_istream* s) { return guarded([&] { s->s->close(); }); }
void b2sh_istream_destroy(b2sh_istream* s) { delete s; }

}  // extern "C"
