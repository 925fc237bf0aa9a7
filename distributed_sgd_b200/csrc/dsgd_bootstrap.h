/* dsgd_bootstrap.h -- the Poisson(1) draw of the bootstrap calls (dsgd_eval_*bootstrap, DESIGN.md §4.19).  Replicate b gives
 * position i of a request the multiplicity m = #{k in 0..19 : u >= T_k}, u = H(key, b, i), T_k = floor(F(k) 2^64) with F the
 * Poisson(1) CDF: P(m = k) = F(k) - F(k - 1) to within 2^-64, m <= 20, and the tail beyond 19 (about 1.6e-19) goes to 20.
 * H is two rounds of splitmix64's finaliser: the replicate's stream z_b = mix(key + phi (b + 1)), then u = mix(z_b + phi
 * (i + 1)).  Each draw is a pure function of (key, b, i): the same on every grid, rank and row order.
 * Plain C, compiled by nvcc into the bootstrap kernels (dsgd_bootstrap.cuh) and by gcc into libdsgd_host.so
 * (dsgd_bootstrap_draw), where tests/test_oracle_bootstrap.py checks it against the Python restatement in oracle/bootstrap.py,
 * which also rebuilds the T_k exactly. */
#ifndef DSGD_BOOTSTRAP_H
#define DSGD_BOOTSTRAP_H
#include <stdint.h>

#ifdef __CUDACC__
#define DSGD_BOOT_HD __host__ __device__ __forceinline__
#else
#define DSGD_BOOT_HD static inline
#endif

#define DSGD_BOOT_MAX_M 20   /* the largest multiplicity */

DSGD_BOOT_HD uint64_t dsgd_boot_mix(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

/* the stream of replicate b */
DSGD_BOOT_HD uint64_t dsgd_boot_stream(uint64_t key, uint64_t b) { return dsgd_boot_mix(key + 0x9E3779B97F4A7C15ull * (b + 1)); }

/* m of position i in the replicate whose stream is zb */
DSGD_BOOT_HD int dsgd_boot_m(uint64_t zb, uint64_t i) {
  const uint64_t u = dsgd_boot_mix(zb + 0x9E3779B97F4A7C15ull * (i + 1));
  /* T_k = floor(F(k) 2^64), F(k) = e^-1 sum_{j <= k} 1 / j! */
  const uint64_t t[DSGD_BOOT_MAX_M] = {
      0x5E2D58D8B3BCDF1Aull, 0xBC5AB1B16779BE35ull, 0xEB715E1DC1582DC2ull, 0xFB23979734A252F1ull, 0xFF1025F59174DC3Dull,
      0xFFD90F3BA4055E19ull, 0xFFFA8B71FC72C913ull, 0xFFFF540C0914B3C9ull, 0xFFFFED1F4AA8F120ull, 0xFFFFFE216E641462ull,
      0xFFFFFFD4D85D3183ull, 0xFFFFFFFC6DA262B4ull, 0xFFFFFFFFBA12D178ull, 0xFFFFFFFFFB07C64Cull, 0xFFFFFFFFFFAB8EA5ull,
      0xFFFFFFFFFFFABE22ull, 0xFFFFFFFFFFFFB11Aull, 0xFFFFFFFFFFFFFBA1ull, 0xFFFFFFFFFFFFFFC5ull, 0xFFFFFFFFFFFFFFFDull};
  int m = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int k = 0; k < DSGD_BOOT_MAX_M; ++k) m += u >= t[k];
  return m;
}
#endif
