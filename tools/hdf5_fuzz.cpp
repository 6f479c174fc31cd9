// AddressSanitizer / UBSan harness for the HDF5 reader (csrc/hdf5io.cpp), host only:
//   g++ -std=c++17 -g -O1 -fsanitize=address,undefined -I/usr/local/cuda/include tools/hdf5_fuzz.cpp tnc_b200/csrc/hdf5io.cpp -lz -o /tmp/hdf5_fuzz
//   /tmp/hdf5_fuzz seed.h5 20000
// Mutates the seed file (byte flips, truncations, wild 8-byte words) and drives open / shape / attr / read on every
// mutant; any out-of-bounds access aborts.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>
#include "../include/tncb.h"

namespace tncb {
static std::string g_err;
void set_error(const std::string& m) { g_err = m; }
int fail(int status, const std::string& m) { g_err = m; return status; }
}

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: %s seed.h5 trials [group]\n", argv[0]); return 2; }
  const char* group = argc > 3 ? argv[3] : nullptr;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<uint8_t> seed;
  for (int c; (c = std::fgetc(f)) != EOF;) seed.push_back((uint8_t)c);
  std::fclose(f);
  std::mt19937_64 rng(12345);
  const std::string tmp = std::string(argv[1]) + ".mut";
  long ok = 0, rejected = 0, status_count[16] = {0};
  for (long t = 0; t < std::atol(argv[2]); t++) {
    std::vector<uint8_t> b = seed;
    const size_t span = std::min<size_t>(b.size(), 8192);
    switch (t % 4) {
      case 0: for (int k = 0, n = 1 + rng() % 6; k < n; k++) b[rng() % span] = (uint8_t)rng(); break;
      case 1: b.resize(rng() % b.size()); break;
      case 2: { size_t i = rng() % (span - 8); uint64_t v = rng() >> (rng() % 64); for (int q = 0; q < 8; q++) b[i + q] = (uint8_t)(v >> (8 * q)); break; }
      default: { size_t i = rng() % span; b[i] ^= (uint8_t)(1u << (rng() % 8)); break; }
    }
    f = std::fopen(tmp.c_str(), "wb");
    std::fwrite(b.data(), 1, b.size(), f);
    std::fclose(f);
    tncb_h5file* h = nullptr;
    int rc = tncb_hdf5_open(tmp.c_str(), group, &h);
    if (rc) { rejected++; status_count[-rc & 15]++; continue; }
    bool any_bad = false;
    for (size_t i = 0; i < tncb_hdf5_count(h); i++) {
      int rank; uint64_t dims[32], elems;
      tncb_hdf5_shape(h, i, &rank, dims, &elems);
      (void)tncb_hdf5_name(h, i);
      int64_t a[64]; size_t n;
      if (tncb_hdf5_attr(h, i, "bids", 64, a, &n)) any_bad = true;
      if (elems < (1u << 22)) {
        std::vector<double> out(2 * elems + 2);
        if ((rc = tncb_hdf5_read(h, i, out.data()))) { any_bad = true; status_count[-rc & 15]++; }
      }
    }
    tncb_hdf5_close(h);
    (any_bad ? rejected : ok)++;
  }
  std::printf("mutants read cleanly: %ld, rejected with a status: %ld (by status 1..10:", ok, rejected);
  for (int s = 1; s <= 10; s++) std::printf(" %ld", status_count[s]);
  std::printf(")\n");
  std::remove(tmp.c_str());
  return 0;
}
