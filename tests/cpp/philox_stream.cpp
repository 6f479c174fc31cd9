// The sampling random stream (tnc_b200/csrc/philox.h) compiled for the host, for tests/test_sampling_host.py.
// Each input line "key c0 c1 c2 c3" prints the Philox4x64-10 block of that key and 256-bit counter; each line
// "cand seed i" prints candidate i's block, then the bits of u and v as the kernels form them.  Numbers in decimal.
#include <cstdio>
#include <cstring>
#include "philox.h"

int main() {
  char tag[16];
  while (std::scanf("%15s", tag) == 1) {
    unsigned long long a[5] = {0, 0, 0, 0, 0};
    tncb::philox::Block b;
    if (std::strcmp(tag, "key") == 0) {
      for (int i = 0; i < 5; i++) if (std::scanf("%llu", &a[i]) != 1) return 2;
      b = tncb::philox::philox4x64_10(tncb::philox::Block{{a[1], a[2], a[3], a[4]}}, a[0], 0);
    } else {
      if (std::scanf("%llu %llu", &a[0], &a[1]) != 2) return 2;
      b = tncb::philox::candidate(a[0], a[1]);
    }
    std::printf("%llu %llu %llu %llu", (unsigned long long)b.w[0], (unsigned long long)b.w[1], (unsigned long long)b.w[2],
                (unsigned long long)b.w[3]);
    if (std::strcmp(tag, "cand") == 0) {
      const double u = tncb::philox::unit53(b.w[1]), v = tncb::philox::unit53(b.w[2]);
      unsigned long long ub, vb;
      std::memcpy(&ub, &u, 8);
      std::memcpy(&vb, &v, 8);
      std::printf(" %llu %llu", ub, vb);
    }
    std::printf("\n");
  }
  return 0;
}
