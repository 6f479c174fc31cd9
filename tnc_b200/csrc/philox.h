// Philox4x64-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC'11) with the constants of
// Random123 and numpy's np.random.Philox, for the host (tests) and the device (sample.cu) alike, so that the random
// stream of tncb_plan_sample has one definition.  Block `ctr` of key `key` is four 64-bit words; numpy's generator
// returns the same block for Philox(key=key, counter=ctr - 1).random_raw(4), because it increments its counter first.
#pragma once
#include <stdint.h>

#ifndef TNCB_HD
#ifdef __CUDACC__
#define TNCB_HD __host__ __device__ __forceinline__
#else
#define TNCB_HD inline
#endif
#endif

namespace tncb {
namespace philox {

struct Block { uint64_t w[4]; };

TNCB_HD void mulhilo(uint64_t a, uint64_t b, uint64_t* hi, uint64_t* lo) {
#ifdef __CUDA_ARCH__
  *lo = a * b;
  *hi = __umul64hi(a, b);
#else
  const unsigned __int128 p = (unsigned __int128)a * b;
  *lo = (uint64_t)p;
  *hi = (uint64_t)(p >> 64);
#endif
}

// ten rounds; the key is bumped by the Weyl constants between rounds
TNCB_HD Block philox4x64_10(Block c, uint64_t k0, uint64_t k1) {
  for (int r = 0; r < 10; r++) {
    uint64_t hi0, lo0, hi1, lo1;
    mulhilo(0xD2E7470EE14C6C93ull, c.w[0], &hi0, &lo0);
    mulhilo(0xCA5A826395121157ull, c.w[2], &hi1, &lo1);
    c = Block{{hi1 ^ c.w[1] ^ k0, lo1, hi0 ^ c.w[3] ^ k1, lo0}};
    k0 += 0x9E3779B97F4A7C15ull;
    k1 += 0xBB67AE8584CAA73Bull;
  }
  return c;
}

// candidate i of seed s: the block at counter (i, 0, 0, 0) of key (s, 0)
TNCB_HD Block candidate(uint64_t seed, uint64_t i) { return philox4x64_10(Block{{i, 0, 0, 0}}, seed, 0); }

// the top 53 bits of w as a double in [0, 1)
TNCB_HD double unit53(uint64_t w) { return (double)(w >> 11) * 0x1.0p-53; }

}  // namespace philox
}  // namespace tncb
