// Host build of spark-s3-shuffle_b200/csrc/decimal128.h for tests/test_decimal128.py: the 128-bit add, range check,
// signed order and minimal encoding of the Decimal aggregate kernels, compiled by g++ so they can be checked without a
// GPU.  Test infrastructure only — the C ABI never runs this.
#include "../../spark-s3-shuffle_b200/csrc/decimal128.h"

extern "C" {
// s = a + b modulo 2^128 (lo, hi); returns 1 when the signed sum overflows 128 bits
int dc_add(uint64_t alo, uint64_t ahi, uint64_t blo, uint64_t bhi, uint64_t* s) {
  bool ovf;
  const b2s::Dec128 r = b2s::dec_add({alo, ahi}, {blo, bhi}, &ovf);
  s[0] = r.lo;
  s[1] = r.hi;
  return ovf ? 1 : 0;
}
int dc_fits(uint64_t lo, uint64_t hi, uint32_t p) { return b2s::dec_fits({lo, hi}, p) ? 1 : 0; }
int dc_less(uint64_t alo, uint64_t ahi, uint64_t blo, uint64_t bhi) {
  return b2s::dec_less({alo, ahi}, {blo, bhi}) ? 1 : 0;
}
// the minimal length, and out[0..15] = the bytes dec_encode stores
uint32_t dc_encode(uint64_t lo, uint64_t hi, uint8_t* out) {
  const b2s::Dec128 x{lo, hi};
  const uint32_t len = b2s::dec_bytes(x);
  uint64_t m0, m1;
  b2s::dec_encode(x, len, &m0, &m1);
  for (int i = 0; i < 8; i++) {
    out[i] = (uint8_t)(m0 >> (8 * i));
    out[8 + i] = (uint8_t)(m1 >> (8 * i));
  }
  return len;
}
void dc_of_long(uint64_t v, uint64_t* out) {
  const b2s::Dec128 r = b2s::dec_of_long(v);
  out[0] = r.lo;
  out[1] = r.hi;
}
}
