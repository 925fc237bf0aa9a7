// dsgd_fixed.cuh -- order-free exact sums: doubles cut into fixed-point limbs and added as 64-bit integers.
// Used by the persistent sync kernel (its per-CTA partials of W.d and ||W||^2, dsgd_persistent.cuh) and by the logistic row
// kernel (the per-sample logistic losses of a batch or an evaluation pass, dsgd_kernels.cuh).  The loss sum, at the end of
// this file: resolution 2^-160 per value, within one ulp of the exact sum (exact when that is a double) for any pass of values
// in [0, 2^52) the ABI accepts, NaN if a value is NaN, infinite or 2^52 or more.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dsgd {

// A double v with |v| < 2^52 is cut into five integers: |v| = l4 + l3 * 2^-40 + l2 * 2^-80 + l1 * 2^-120 + l0 * 2^-160,
// l3..l0 in [0, 2^40] (l0 rounded: resolution 2^-160), every cut exact in fp64 arithmetic; negative v contribute the
// negated limbs.  The limbs of all CTAs are added with 64-bit integer REDs (no overflow while CTAs < 2^8: 2^8 * 2^40 = 2^48)
// and converted back once.  Five limbs rather than three: at 2^-80 a partial ||W||^2 of weights around 1e-12 lost most of its
// digits and one of weights around 1e-13 read 0, while the k_update<true> path of larger batches sums in fp64 -- the same
// weights reported different losses at batch 32 G and 32 G + 1.  2^-160 keeps the relative error of ||W||^2 below 1e-15
// down to weights around 1e-16.  Zero limbs are not sent, so small partials cost no more REDs than before.
// One accumulator = 11 x u64 = 88 bytes {sd.l0..l4, sn.l0..l4, overflow count} on its own 128-byte line: every CTA adds ONE
// partial per step (one same-address RED per CTA and non-zero limb, tools/microbench.cu) and reads the 96 bytes from the
// line's start back with ONE coalesced request.  (First cut: 8 striped copies read with 16-byte loads = 2 368 requests on
// 4 lines after every barrier: c arrived later.)
constexpr int kAccStride = 16;   // u64 words between the three rotating accumulators (128 bytes)
constexpr int kAccLimbs = 5;
constexpr int kAccWords = 2 * kAccLimbs + 1;   // 11: {sd limbs, sn limbs, overflow}
static_assert(kAccWords + 1 <= kAccStride, "acc_read loads the accumulator and one pad word");
__device__ __forceinline__ void red_add_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// The limbs of a = |v| < 2^52: put(k, limb k) for k = 4, 3, 2, 1, 0, limb k worth 2^(40 k - 160).  F_i = floor(a * 2^(40 i)):
// scaling by a power of two and floor are exact.  Limb 4 - i is F_i - 2^40 F_(i-1), an integer below 2^40 and therefore exact
// too; the lowest limb rounds, at 2^-160.  The limbs are cut side by side rather than one from the remainder of the other: in
// the persistent kernel this runs just before the CTA's arrival at the grid barrier.
template <class Put>
__device__ __forceinline__ void acc_cut(double a, Put &&put) {
  double F[kAccLimbs - 1];
#pragma unroll
  for (int i = 0; i < kAccLimbs - 1; ++i) F[i] = floor(a * __longlong_as_double((1023ll + 40 * i) << 52));
  put(kAccLimbs - 1, F[0]);
#pragma unroll
  for (int i = 1; i < kAccLimbs - 1; ++i) put(kAccLimbs - 1 - i, F[i] - F[i - 1] * 0x1p40);
  put(0, rint(a * 0x1p160) - F[kAccLimbs - 2] * 0x1p40);   // [0, 2^40]
}
__device__ __forceinline__ void acc_push_one(unsigned long long *limbs, unsigned long long *ovf, double v) {
  if (!(fabs(v) < 4503599627370496.0)) {   // 2^52; also NaN / inf: the sum is reported as NaN
    red_add_u64(ovf, 1ull);
    return;
  }
  const bool neg = v < 0.0;                // negative values add the negated limbs (two's complement wraps)
  acc_cut(fabs(v), [&](int k, double limb) {
    if (limb != 0.0) {
      const unsigned long long u = (unsigned long long)(long long)limb;
      red_add_u64(limbs + k, neg ? (0ull - u) : u);
    }
  });
}
__device__ __forceinline__ void acc_push(unsigned long long *acc, double sd, double sn) {
  acc_push_one(acc, acc + 2 * kAccLimbs, sd);
  acc_push_one(acc + kAccLimbs, acc + 2 * kAccLimbs, sn);
}
// Limb sum q of limb k as a double (exact while |q| < 2^53)
__device__ __forceinline__ double acc_limb(unsigned long long q, int k) {
  return (double)(long long)q * __longlong_as_double((long long)(1023 - 160 + 40 * (k % kAccLimbs)) << 52);
}
// acc_read in two halves, so that a caller can put other loads into the same round trip: acc_load requests the words,
// acc_sum waits for them and sums.
__device__ __forceinline__ void acc_load(const unsigned long long *acc, int lane, unsigned long long &q0, unsigned long long &q1) {
  q0 = 0; q1 = 0;
  if (lane < (kAccWords + 1) / 2)   // 6 lanes x 16 bytes = the 88-byte accumulator (and a pad word) in one request
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(q0), "=l"(q1) : "l"(acc + 2 * lane) : "memory");
}
__device__ __forceinline__ void acc_sum(unsigned long long q0, unsigned long long q1, int lane, double &sd, double &sn) {
  // Word k = 2 lane + h is limb k % 5 of sd (k < 5) or of sn (5 <= k < 10), worth 2^(40 (k % 5) - 160); every limb sum is
  // below 2^48 in magnitude, so its conversion and scaling are exact.  Each lane adds its own two words first, so the
  // sums take six shuffles: sd = (limbs 0+1 + limbs 2+3) + limb 4, sn = (limb 0 + limbs 1+2) + limbs 3+4.  Word 10 counts
  // the partials that could not be summed.
  const double lo = acc_limb(q0, 2 * lane), hi = acc_limb(q1, 2 * lane + 1), pair = lo + hi;
  const double s01 = __shfl_sync(0xffffffffu, pair, 0), s23 = __shfl_sync(0xffffffffu, pair, 1);
  const double s4 = __shfl_sync(0xffffffffu, lo, 2), n0 = __shfl_sync(0xffffffffu, hi, 2);
  const double n12 = __shfl_sync(0xffffffffu, pair, 3), n34 = __shfl_sync(0xffffffffu, pair, 4);
  sd = (s01 + s23) + s4;
  sn = (n0 + n12) + n34;
  if (__any_sync(0xffffffffu, lane == kAccWords / 2 && q0 != 0)) {
    sd = __longlong_as_double(0x7ff8000000000000ll);
    sn = sd;
  }
}
// Called by a whole warp; all lanes return the two sums (identical in every CTA: integer additions commute).
__device__ __forceinline__ void acc_read(const unsigned long long *acc, int lane, double &sd, double &sn) {
  unsigned long long q0, q1;
  acc_load(acc, lane, q0, q1);
  acc_sum(q0, q1, lane, sd, sn);
}
// The persistent kernel's L1 form (kL1) keeps a third value in words kAccWords .. kAccWords + 4 of the same accumulator line,
// its overflows counted in word 2 * kAccLimbs with the other two.  Split like acc_read: acc_load_l1 requests, acc_sum_l1 sums.
__device__ __forceinline__ void acc_load_l1(const unsigned long long *acc, int lane, unsigned long long &q, unsigned long long &o) {
  q = 0; o = 0;
  if (lane < kAccLimbs) asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(q) : "l"(acc + kAccWords + lane) : "memory");
  if (lane == 0) asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(o) : "l"(acc + 2 * kAccLimbs) : "memory");
}
__device__ __forceinline__ double acc_sum_l1(unsigned long long q, unsigned long long o, int lane) {
  const double v = acc_limb(q, lane);
  const double v0 = __shfl_sync(0xffffffffu, v, 0), v1 = __shfl_sync(0xffffffffu, v, 1), v2 = __shfl_sync(0xffffffffu, v, 2);
  const double v3 = __shfl_sync(0xffffffffu, v, 3), v4 = __shfl_sync(0xffffffffu, v, 4);
  const double a = (((v4 + v3) + v2) + v1) + v0;   // from the top limb down
  return __shfl_sync(0xffffffffu, o, 0) != 0ull ? __longlong_as_double(0x7ff8000000000000ll) : a;
}
// Called by a whole warp; all lanes return the sum.
__device__ __forceinline__ double acc_read_l1(const unsigned long long *acc, int lane) {
  unsigned long long q, o;
  acc_load_l1(acc, lane, q, o);
  return acc_sum_l1(q, o, lane);
}

// ---- one sum of many non-negative values (the logistic losses of a pass) -------------------------------------------------
// Each value v in [0, 2^52) contributes R(v) = rint(v * 2^160) * 2^-160 (acc_cut's limbs, resolution 2^-160: a value below
// 2^-161 adds exactly 0); NaN, inf and values >= 2^52 are counted instead and the sum reads NaN.  Six limb words, limb k
// worth 2^(40 k - 160): limbs 0..3 as acc_cut cuts them, the integer part split into limb 4 (its low 40 bits) and limb 5; then
// one overflow count.  A thread adds its values' limbs in registers (acc_add_local) and propagates the carries after every
// value, so that limbs 0..4 stay below 2^40 and limb 5 grows by at most 2^13 per value; it pushes them once
// (acc_flush_local).  The words then hold below warps * 2^40 (limbs 0..4) and n * 2^13 (limb 5): no u64 wraps for any grid
// of fewer than 2^24 warps and any n below 2^50, far beyond what fits on a device.  Integer additions commute, so the sum has
// the same bits whatever the grid, the work split or the order of arrival; acc_value propagates the carries once more and
// converts the limbs from the top down: the result is within one ulp of the exact sum of the R(v), and equal to it whenever
// that sum is a double (every partial sum is then a prefix of its bits).
constexpr int kLossLimbs = kAccLimbs + 1;
constexpr int kLossAccWords = kLossLimbs + 1;   // 7: {limbs 0..5, overflow}
constexpr unsigned long long kLimbMask = (1ull << 40) - 1;
__device__ __forceinline__ void acc_carry(unsigned long long (&q)[kLossLimbs]) {
#pragma unroll
  for (int i = 0; i < kLossLimbs - 1; ++i) {   // limbs 0..4 into [0, 2^40)
    q[i + 1] += q[i] >> 40;
    q[i] &= kLimbMask;
  }
}
__device__ __forceinline__ void acc_add_local(unsigned long long (&lim)[kLossLimbs], unsigned long long &ovf, double v) {
  if (!(v >= 0.0 && v < 4503599627370496.0)) { ++ovf; return; }   // NaN, inf, >= 2^52 (or negative): reported as NaN
  // limbs 0..3 below 2^40 + 1, limb 4 (the integer part) below 2^52: no register passes 2^53 before the carries
  acc_cut(v, [&](int k, double limb) { lim[k] += (unsigned long long)(long long)limb; });
  acc_carry(lim);
}
__device__ __forceinline__ void acc_flush_local(unsigned long long *acc, const unsigned long long (&lim)[kLossLimbs],
                                                unsigned long long ovf) {
#pragma unroll
  for (int i = 0; i < kLossLimbs; ++i)
    if (lim[i]) red_add_u64(acc + i, lim[i]);
  if (ovf) red_add_u64(acc + kLossLimbs, ovf);
}
// One thread: the value of a kLossAccWords accumulator.
__device__ __forceinline__ double acc_value(const unsigned long long *acc) {
  if (acc[kLossLimbs] != 0ull) return __longlong_as_double(0x7ff8000000000000ll);
  unsigned long long q[kLossLimbs];
#pragma unroll
  for (int i = 0; i < kLossLimbs; ++i) q[i] = acc[i];
  acc_carry(q);
  double s = (double)q[kLossLimbs - 1] * 0x1p40;   // exact while the sum is below 2^93
#pragma unroll
  for (int i = kLossLimbs - 2; i >= 0; --i) s += (double)q[i] * __longlong_as_double((long long)(1023 - 160 + 40 * i) << 52);
  return s;
}

}  // namespace dsgd
