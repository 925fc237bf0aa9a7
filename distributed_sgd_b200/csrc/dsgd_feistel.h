/* dsgd_feistel.h -- `Random.shuffle(indices) take batchSize` (core/Slave.scala:86-88) without a shuffle: B distinct positions
 * in random order are pi(0), ..., pi(B - 1) of a keyed pseudo-random PERMUTATION pi of [0, n) -- a 4-round Feistel network on
 * the next even power of two, walked until the image falls inside [0, n) (a bijection restricted to its cycles through
 * [0, n) stays a bijection).  Distinct by construction, O(1) per position, every lane of a warp draws its own positions.
 * Plain C, compiled by nvcc into the async worker (dsgd_async.cuh) and the sampled evaluation's draw (k_draw_rows,
 * dsgd_kernels.cuh), and by gcc into libdsgd_host.so (dsgd_feistel_pos), where
 * tests/test_host_logic.py checks the permutation property on the very same source. */
#ifndef DSGD_FEISTEL_H
#define DSGD_FEISTEL_H
#include <stdint.h>

#ifdef __CUDACC__
#define DSGD_HD __host__ __device__ __forceinline__
#else
#define DSGD_HD static inline
#endif

/* smallest h with 4^h >= n */
DSGD_HD int dsgd_feistel_half_bits(uint64_t n) {
  int h = 1;
  while ((1ull << (2 * h)) < n) ++h;
  return h;
}

DSGD_HD uint32_t dsgd_feistel(uint32_t x, int half_bits, uint64_t key, uint32_t n) {
  const uint32_t mask = (1u << half_bits) - 1u;
  do {
    uint32_t L = x >> half_bits, R = x & mask;
    for (int r = 0; r < 4; ++r) {
      uint64_t z = key + 0x9E3779B97F4A7C15ull * (uint64_t)(r + 1) + (uint64_t)R * 0xD1342543DE82EF95ull;
      z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
      z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
      const uint32_t F = (uint32_t)(z >> 33) & mask;
      const uint32_t t = L ^ F;
      L = R;
      R = t;
    }
    x = (L << half_bits) | R;
  } while (x >= n);
  return x;
}
#endif
