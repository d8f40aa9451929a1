// Runs the host build of the Zstandard decoder core over a corpus of frames and prints one verdict line per frame:
// "<single-pass result> <block-parallel result> <fnv-1a of the decoded bytes>".  Built once plainly and once with
// -fsanitize=address,undefined, so that a corpus can be screened for memory errors before it reaches the device.
// Corpus file: per frame, u64 output capacity, u64 frame length, the frame's bytes (little-endian).
#include "zstd_core_host.cpp"

#include <stdio.h>

static unsigned long long fnv(const unsigned char* p, long long n) {
  unsigned long long h = 1469598103934665603ull;
  for (long long i = 0; i < n; i++) h = (h ^ p[i]) * 1099511628211ull;
  return h;
}

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  unsigned long long hdr[2];
  while (fread(hdr, 8, 2, f) == 2) {
    std::vector<unsigned char> frame(hdr[1] ? hdr[1] : 1), a(hdr[0] ? hdr[0] : 1), b(hdr[0] ? hdr[0] : 1);
    if (fread(frame.data(), 1, hdr[1], f) != hdr[1]) return 2;
    const long long r = zc_decode(frame.data(), hdr[1], a.data(), hdr[0]);
    const long long r2 = zc_decode_par(frame.data(), hdr[1], b.data(), hdr[0], 0);
    printf("%lld %lld %llx %llx\n", r, r2, fnv(a.data(), r), fnv(b.data(), r2));
  }
  fclose(f);
  return 0;
}
