// Host build of spark-s3-shuffle_b200/csrc/crc_gf.h for tests/test_crc_gf.py: the GF(2) power tables and the shift the
// CRC kernels of checksum.cu apply to partial CRCs, compiled by g++ so they can be checked without a GPU.
// Test infrastructure only — the C ABI never runs this.
#include "../../spark-s3-shuffle_b200/csrc/crc_gf.h"

namespace {
const uint32_t kPolys[2] = {0xEDB88320u, 0x82F63B78u};  // CRC32, CRC32C

struct Tables {
  uint32_t rows[16 * 256];
  uint32_t misc[b2s::kMiscWords];
};
const Tables& tables(int which) {
  static Tables t[2];
  static bool built[2] = {false, false};
  if (!built[which]) {
    b2s::build_crc_tables(kPolys[which], t[which].rows, t[which].misc);
    built[which] = true;
  }
  return t[which];
}
}  // namespace

extern "C" {
int cg_misc_words() { return b2s::kMiscWords; }
int cg_pow_bits() { return b2s::kPowBits; }
// the misc table of polynomial `which` (0 CRC32, 1 CRC32C), kMiscWords words
void cg_misc(int which, uint32_t* out) {
  for (int i = 0; i < b2s::kMiscWords; i++) out[i] = tables(which).misc[i];
}
// x^(8e) mod P (inverse: x^(-8e)), reflected, as the kernels compute it
uint32_t cg_xpow8(int which, unsigned long long e, int inverse) {
  const Tables& t = tables(which);
  return b2s::gf_xpow8(e, t.misc + (inverse ? b2s::kMiscXInv : b2s::kMiscXPow), kPolys[which]);
}
uint32_t cg_mul(int which, uint32_t a, uint32_t b) { return b2s::gf_mul(a, b, kPolys[which]); }
}
