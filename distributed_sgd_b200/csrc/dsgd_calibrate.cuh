// dsgd_calibrate.cuh -- sm_90a kernels of the calibration calls (dsgd_calibrate*, dsgd_calibrated_probabilities,
// dsgd_eval_calibration*; DESIGN.md §4.11).
//
// A calibration is a pair (A, B): P(y = +1 | x) = 1 / (1 + exp(A f + B)) = sigmoid(-(A f + B)) with f = x . w as
// dsgd_margins returns it.  A fit is two launches on the ctx's stream:
//   1. k_calib_score: f of every position (row_margin, the one row fold) and its label into the score buffers, and the
//      counts N+, N- and NaN rows, which the host reads: they give the targets and the start point.
//   2. k_calib_fit: the whole Newton iteration of Lin, Lin and Weng's statement of Platt scaling in ONE cooperative
//      launch.  Every evaluation of a point adds its six sums in signed fixed-point limbs (dsgd_fixed.cuh's cut), so they
//      have the same bits for any grid, work split or row order; every CTA reads the same bits after a grid barrier and
//      runs the same scalar fp64 code, so all CTAs take the same decisions and (A, B, F, iterations) are order-free too.
// The fit is one kernel template, k_calib_fit<kW>, over counted rows (kW = false) and weighted rows (kW = true).
// k_calib_eval<kIso, kSmem> (dsgd_isotonic.cuh, beside the maps it applies) is the quality pass at a given (A, B) or
// isotonic map: Brier and log-loss sums in the same limbs, and M equal-width bins, into the CalibEvalWord block below.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dsgd_metrics.cuh"
#include "dsgd_persistent.cuh"

namespace dsgd {

// ---- signed six-limb sums ----------------------------------------------------------------------------------------
// The six-limb form of the loss sum (dsgd_fixed.cuh) for values of either sign: a negative value subtracts its limbs, and
// the carry is an arithmetic shift, so limbs 0..4 stay in [0, 2^40) and limb 5 carries the sign (two's complement: a limb
// of -3 becomes 2^40 - 3 and borrows 1 from the limb above).  The words are added as u64 and wrap like the integers they
// are; a sum is below 2^57 in magnitude for any grid of fewer than 2^17 threads, far from a wrap.
__device__ __forceinline__ void cal_carry(long long (&q)[kLossLimbs]) {
#pragma unroll
  for (int i = 0; i < kLossLimbs - 1; ++i) {
    q[i + 1] += q[i] >> 40;   // arithmetic: floor division
    q[i] &= (long long)kLimbMask;
  }
}
__device__ __forceinline__ void cal_add(long long (&lim)[kLossLimbs], unsigned long long &ovf, double v) {
  if (!(fabs(v) < 4503599627370496.0)) { ++ovf; return; }   // NaN, inf, |v| >= 2^52: the sum reads NaN
  const bool neg = v < 0.0;
  acc_cut(fabs(v), [&](int k, double limb) {
    const long long u = (long long)limb;
    lim[k] += neg ? -u : u;
  });
  cal_carry(lim);
}
// One thread: the value of six limb words.  Carries first; a negative sum (limb 5 below zero) is negated, carried again
// and converted as a positive one, so both signs convert from the top limb down through non-negative terms: within one ulp
// of the exact sum of the rounded values, and equal to it when that is a double.
__device__ __forceinline__ double cal_value(const unsigned long long *words) {
  long long q[kLossLimbs];
#pragma unroll
  for (int i = 0; i < kLossLimbs; ++i) q[i] = (long long)words[i];
  cal_carry(q);
  const bool neg = q[kLossLimbs - 1] < 0;
  if (neg) {
#pragma unroll
    for (int i = 0; i < kLossLimbs; ++i) q[i] = -q[i];
    cal_carry(q);
  }
  double s = (double)q[kLossLimbs - 1] * 0x1p40;
#pragma unroll
  for (int i = kLossLimbs - 2; i >= 0; --i) s += (double)q[i] * __longlong_as_double((long long)(1023 - 160 + 40 * i) << 52);
  return neg ? -s : s;
}

// ---- k_calib_prob ------------------------------------------------------------------------------------------------
// out[i] = sigmoid(-(a f + b)) for row samples[i], f = x . w (kIcpt: the score with the intercept, row_score): the
// calibrated probability under either model.  With
// (a, b) = (1, 0) the argument is -f exactly, i.e. k_margins<true>'s value bit for bit.  One warp per row.
template <bool kIcpt>
__global__ void __launch_bounds__(256) k_calib_prob(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                    const int32_t *__restrict__ samples, int64_t n,
                                                    const double *__restrict__ w, double a, double b,
                                                    double *__restrict__ out, const double *__restrict__ icpt) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = warp0; i < n; i += nwarps) {
    const double dot = row_score<kIcpt>(rp16, pairs, w, (int64_t)samples[i], lane, icpt);
    if (lane == 0) out[i] = sigmoid(-(a * dot + b));
  }
}

// ---- k_calib_score -----------------------------------------------------------------------------------------------
enum CalibWord : int { kCalPos = 0, kCalNeg = 1, kCalNan = 2, kCalCntWords = 4 };

// The weighted fit's three exact sums of R(c_i), each a kLossAccWords block: non-NaN positives, non-NaN negatives, NaN rows
enum CalibWeightWord : int { kCalWPos = 0, kCalWNeg = kLossAccWords, kCalWNan = 2 * kLossAccWords, kCalWWords = 3 * kLossAccWords };

// score[i] = x . w and lab[i] = the label of position i of the row set (samples == nullptr: rows [row_begin, row_begin + n)),
// and the counts of non-NaN positives, non-NaN negatives and NaN rows, the positions taken by warp_scores; the counts are
// flushed once per warp.
// kW (the weighted fit, DESIGN.md §4.17): cw[i] = c_i (row_weight), and R(c_i) added to the three CalibWeightWord sums at
// wacc; each warp adds its lanes' carried limbs with shuffles (below 2^45 each) and flushes them once.
template <bool kW, bool kIcpt>
__global__ void __launch_bounds__(256) k_calib_score(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                     const int8_t *__restrict__ label, const int32_t *__restrict__ samples,
                                                     int64_t row_begin, int64_t n, const double *__restrict__ w,
                                                     double *__restrict__ score, int8_t *__restrict__ lab,
                                                     unsigned long long *__restrict__ cnt, double w_pos, double w_neg,
                                                     const double *__restrict__ sw, double *__restrict__ cw,
                                                     unsigned long long *__restrict__ wacc, const double *__restrict__ icpt) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  unsigned c_pos = 0, c_neg = 0, c_nan = 0;
  unsigned long long l_pos[kLossLimbs] = {0, 0, 0, 0, 0, 0}, l_neg[kLossLimbs] = {0, 0, 0, 0, 0, 0};
  unsigned long long l_nan[kLossLimbs] = {0, 0, 0, 0, 0, 0}, o_pos = 0, o_neg = 0, o_nan = 0;
  warp_scores<kIcpt>(rp16, pairs, samples, row_begin, n, w, icpt, [&](int64_t i, int64_t r, double dot, bool mine) {
    if (!mine) return;
    const bool pos = label[r] > 0, nan = isnan(dot);
    score[i] = dot;
    lab[i] = pos ? 1 : -1;
    c_nan += nan;
    c_pos += pos && !nan;
    c_neg += !pos && !nan;
    if constexpr (kW) {
      const double ci = row_weight(pos, w_pos, w_neg, sw, r);
      cw[i] = ci;
      if (nan) acc_add_local(l_nan, o_nan, ci);
      else if (pos) acc_add_local(l_pos, o_pos, ci);
      else acc_add_local(l_neg, o_neg, ci);
    }
  });
  c_pos = __reduce_add_sync(full, c_pos);
  c_neg = __reduce_add_sync(full, c_neg);
  c_nan = __reduce_add_sync(full, c_nan);
  if constexpr (kW) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      o_pos += __shfl_xor_sync(full, o_pos, o);
      o_neg += __shfl_xor_sync(full, o_neg, o);
      o_nan += __shfl_xor_sync(full, o_nan, o);
#pragma unroll
      for (int k = 0; k < kLossLimbs; ++k) {
        l_pos[k] += __shfl_xor_sync(full, l_pos[k], o);
        l_neg[k] += __shfl_xor_sync(full, l_neg[k], o);
        l_nan[k] += __shfl_xor_sync(full, l_nan[k], o);
      }
    }
    if (lane == 0) {
      acc_flush_local(wacc + kCalWPos, l_pos, o_pos);
      acc_flush_local(wacc + kCalWNeg, l_neg, o_neg);
      acc_flush_local(wacc + kCalWNan, l_nan, o_nan);
    }
  }
  if (lane == 0) {
    if (c_pos) atomicAdd(&cnt[kCalPos], (unsigned long long)c_pos);
    if (c_neg) atomicAdd(&cnt[kCalNeg], (unsigned long long)c_neg);
    if (c_nan) atomicAdd(&cnt[kCalNan], (unsigned long long)c_nan);
  }
}

// ---- k_calib_fit -------------------------------------------------------------------------------------------------
constexpr int kCalSums = 6;                                  // F, dF/dA, dF/dB, H_AA, H_AB, H_BB
constexpr int kCalLineWords = kCalSums * kLossLimbs + 1;     // 37: six sums of six limbs, one overflow count
constexpr int kCalLineStride = 48;                           // u64 words between the three rotating lines (384 bytes)
constexpr int kCalThreads = 256;
constexpr int kCalMaxIter = 100;
enum CalibStatus : int { kCalConverged = 0, kCalIterLimit = 1, kCalLineSearch = 2, kCalNonFinite = 3 };
enum CalibOut : int { kCalOutA = 0, kCalOutB = 1, kCalOutF = 2, kCalOutIter = 3, kCalOutStatus = 4, kCalOutEvals = 5, kCalOutWords = 8 };

struct CalibFitParams {
  const double *score;        // n scores (NaN: the row is left out)
  const int8_t *lab;          // n labels, +1 / -1
  int64_t n;
  double t_pos, t_neg, b0;    // the targets and the start point B (A starts at 0), from the counts
  unsigned long long *acc;    // three lines of kCalLineStride words, zero at the launch
  unsigned *bar;              // grid barrier counter, zero at the launch
  int *abort_flag;
  long long timeout_cycles;
  unsigned long long *out;    // CalibOut words (A, B, F as the bits of doubles)
  int smem_cap;               // scores a CTA keeps in shared memory; the rest of its slice stays in global memory
  const double *cw;           // the weighted fit: n row weights c_i beside the scores (nullptr in the unweighted one)
};

__device__ __forceinline__ unsigned long long ld_relaxed_gpu_u64(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_gpu_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// One launch = one fit.  Each CTA owns a contiguous slice of the scores, copied to shared memory once.  One evaluation of a
// point (A, B): every thread folds the six terms of its scores into register limbs, the warps add them (shuffles, then
// shared atomics), the CTA adds its partial to the evaluation's accumulator line with one RED per non-zero word, and the
// grid meets at a barrier.  Then EVERY CTA reads the line, and its thread 0 converts the sums and runs the Newton and
// line-search arithmetic.  Every trial point of the line search gets all six sums, so an accepted point needs no second pass.
//
// INVARIANT (what keeps the barrier from hanging): whether the loop goes on, and to which point, depends ONLY on values
// read from the accumulator line after the barrier -- never on a CTA's own scores.  All CTAs read the same bits and run the
// same instructions on them, so all of them leave the loop after the same evaluation and none waits for a CTA that left.
// (The watchdog is the other exit: a CTA that gives up sets the abort flag, which every other CTA's wait polls.)
//
// The three lines rotate: evaluation e uses line e % 3.  After barrier e every CTA has finished reading line e - 1 (it read
// it before it arrived), so block 0 zeroes that line then, for evaluation e + 2; its arrival at barrier e + 1 (release)
// orders the zeroes before any CTA's REDs of evaluation e + 2.
//
// kW: the weighted fit (DESIGN.md §4.17).  A CTA keeps f, c and y of each score in shared memory (17 bytes instead of 9, so
// its cap is smaller); a row with R(c) = 0 is skipped before any term is formed; and each of the six terms is added as
// R(fl(c term)).  The weights change only what a CTA adds to the line, never what it reads from it, so the invariant above
// holds for both forms.
template <bool kW>
__global__ void __launch_bounds__(kCalThreads, 1) k_calib_fit(const CalibFitParams p) {
  extern __shared__ __align__(16) unsigned char cal_smem[];
  double *s_f = reinterpret_cast<double *>(cal_smem);
  double *s_c = s_f + p.smem_cap;
  int8_t *s_y = reinterpret_cast<int8_t *>(kW ? s_c + p.smem_cap : s_c);
  __shared__ unsigned long long s_red[kCalLineWords];    // the CTA's partial of one evaluation
  __shared__ unsigned long long s_line[kCalLineWords];   // the accumulator line as read after the barrier
  __shared__ double s_pt[2];                             // the point to evaluate next
  __shared__ int s_done;                                 // 1: the fit ended; -1: the watchdog fired

  const unsigned full = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t G = gridDim.x, slice = (p.n + G - 1) / G;
  const int64_t b = min(p.n, (int64_t)blockIdx.x * slice), e = min(p.n, b + slice);
  const int m = (int)(e - b), in_smem = min(m, p.smem_cap);
  for (int i = tid; i < in_smem; i += kCalThreads) {
    s_f[i] = p.score[b + i];
    if constexpr (kW) s_c[i] = p.cw[b + i];
    s_y[i] = p.lab[b + i];
  }
  if (tid < kCalLineWords) s_red[tid] = 0ull;
  if (tid == 0) {
    s_pt[0] = 0.0;
    s_pt[1] = p.b0;
    s_done = 0;
  }
  __syncthreads();

  // thread 0's state: the accepted point, its objective, the Newton direction from it and the line search's step
  double A = 0.0, B = 0.0, F = 0.0, dA = 0.0, dB = 0.0, gd = 0.0, step = 1.0;
  int iter = 0, status = kCalConverged;
  for (unsigned ev = 0;; ++ev) {
    const double pa = s_pt[0], pb = s_pt[1];
    long long lim[kCalSums][kLossLimbs];
#pragma unroll
    for (int s = 0; s < kCalSums; ++s)
#pragma unroll
      for (int k = 0; k < kLossLimbs; ++k) lim[s][k] = 0;
    unsigned long long ovf = 0;
    for (int i = tid; i < m; i += kCalThreads) {
      const double f = i < in_smem ? s_f[i] : __ldcg(p.score + b + i);
      const int8_t y = i < in_smem ? s_y[i] : __ldcg(p.lab + b + i);
      if (isnan(f)) continue;
      double c = 1.0;
      if constexpr (kW) {
        c = i < in_smem ? s_c[i] : __ldcg(p.cw + b + i);
        if (rint(c * 0x1p160) == 0.0) continue;   // R(c) = 0: the row adds exactly 0 to every sum
      }
      auto cw = [&](double v) {   // a term as it is added: c v in the weighted fit
        if constexpr (kW) return c * v;
        else return v;
      };
      const double t = y > 0 ? p.t_pos : p.t_neg;
      const double z = pa * f + pb;
      double term, pr, qr;   // pr = 1 / (1 + exp(z)) = P(y = +1), qr = 1 - pr, each from the half that does not cancel
      if (z >= 0.0) {
        const double ex = exp(-z), den = 1.0 + ex;
        term = t * z + log1p(ex);
        pr = ex / den;
        qr = 1.0 / den;
      } else {
        const double ex = exp(z), den = 1.0 + ex;
        term = (t - 1.0) * z + log1p(ex);
        pr = 1.0 / den;
        qr = ex / den;
      }
      const double d1 = t - pr, d2 = pr * qr;
      cal_add(lim[0], ovf, cw(term));
      cal_add(lim[1], ovf, cw(f * d1));
      cal_add(lim[2], ovf, cw(d1));
      cal_add(lim[3], ovf, cw((f * f) * d2));
      cal_add(lim[4], ovf, cw(f * d2));
      cal_add(lim[5], ovf, cw(d2));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ovf += __shfl_xor_sync(full, ovf, o);
#pragma unroll
      for (int s = 0; s < kCalSums; ++s)
#pragma unroll
        for (int k = 0; k < kLossLimbs; ++k) lim[s][k] += __shfl_xor_sync(full, lim[s][k], o);   // below 2^45: no carry lost
    }
    if (lane == 0) {
#pragma unroll
      for (int s = 0; s < kCalSums; ++s)
#pragma unroll
        for (int k = 0; k < kLossLimbs; ++k)
          if (lim[s][k]) atomicAdd(&s_red[s * kLossLimbs + k], (unsigned long long)lim[s][k]);
      if (ovf) atomicAdd(&s_red[kCalLineWords - 1], ovf);
    }
    __syncthreads();
    unsigned long long *line = p.acc + (ev % 3u) * kCalLineStride;
    if (tid < kCalLineWords) {
      const unsigned long long v = s_red[tid];
      if (v) red_add_u64(line + tid, v);
      s_red[tid] = 0ull;
    }
    __syncthreads();
    if (tid == 0 && !grid_barrier_arrive_wait(p.bar, (ev + 1u) * (unsigned)G, p.abort_flag, p.timeout_cycles)) s_done = -1;
    __syncthreads();
    if (s_done < 0) return;
    if (tid < kCalLineWords) {
      s_line[tid] = ld_relaxed_gpu_u64(line + tid);
      if (blockIdx.x == 0) st_relaxed_gpu_u64(p.acc + ((ev + 2u) % 3u) * kCalLineStride + tid, 0ull);
    }
    __syncthreads();
    if (tid == 0) {
      double S[kCalSums];
      bool finite = s_line[kCalLineWords - 1] == 0ull;
#pragma unroll
      for (int s = 0; s < kCalSums; ++s) S[s] = cal_value(s_line + s * kLossLimbs);
      bool accept = false, done = false;
      if (!finite) {
        status = kCalNonFinite;
        A = B = F = __longlong_as_double(0x7ff8000000000000ll);
        done = true;
      } else if (ev == 0) {
        accept = true;
      } else if (S[0] < F + 1e-4 * step * gd) {
        accept = true;
        ++iter;
      } else {
        step = step / 2.0;
        if (step < 1e-10) {
          status = kCalLineSearch;
          done = true;
        }
      }
      if (accept) {
        A = pa; B = pb; F = S[0];
        const double g1 = S[1], g2 = S[2], h11 = S[3] + 1e-12, h21 = S[4], h22 = S[5] + 1e-12;
        if (fabs(g1) < 1e-5 && fabs(g2) < 1e-5) {
          status = kCalConverged;
          done = true;
        } else if (iter >= kCalMaxIter) {
          status = kCalIterLimit;
          done = true;
        } else {
          const double det = h11 * h22 - h21 * h21;
          dA = -(h22 * g1 - h21 * g2) / det;
          dB = -(h11 * g2 - h21 * g1) / det;
          gd = g1 * dA + g2 * dB;
          step = 1.0;
        }
      }
      if (done) {
        s_done = 1;
      } else {
        s_pt[0] = A + step * dA;
        s_pt[1] = B + step * dB;
      }
    }
    __syncthreads();
    if (s_done) {
      if (blockIdx.x == 0 && tid == 0) {
        p.out[kCalOutA] = (unsigned long long)__double_as_longlong(A);
        p.out[kCalOutB] = (unsigned long long)__double_as_longlong(B);
        p.out[kCalOutF] = (unsigned long long)__double_as_longlong(F);
        p.out[kCalOutIter] = (unsigned long long)iter;
        p.out[kCalOutStatus] = (unsigned long long)status;
        p.out[kCalOutEvals] = (unsigned long long)ev + 1ull;
      }
      return;
    }
  }
}

// ---- the quality pass's block (k_calib_eval, dsgd_isotonic.cuh) ---------------------------------------------------
constexpr int kCalMaxBins = 64;
// Words of the quality pass's block
enum CalibEvalWord : int {
  kCevBrier = 0,                                   // [0, 7): limbs and overflow count of sum (p - o)^2
  kCevLog = kLossAccWords,                         // [7, 14): of the finite log-loss terms
  kCevRows = 2 * kLossAccWords,                    // rows used
  kCevNan = kCevRows + 1,                          // rows left out (their argument is NaN)
  kCevBinRows = 16,                                // [16, 80)
  kCevBinPos = kCevBinRows + kCalMaxBins,          // [80, 144)
  kCevBinLimbs = kCevBinPos + kCalMaxBins,         // [144, 528): six limbs of sum p per bin
  kCevOutSums = kCevBinLimbs + kCalMaxBins * kLossLimbs,   // [528, 530): Brier and log-loss sums as the bits of doubles
  kCevOutPsum = kCevOutSums + 2,                   // [530, 594): sum p per bin, likewise (k_calib_eval_finish)
  kCevInf = kCevOutPsum + kCalMaxBins,             // 594: rows whose log-loss term is infinite (an isotonic map only)
  kCevWords = 640
};

// The sums of a quality pass as doubles: thread 0 the Brier and log-loss sums, thread i sum p of bin i.
__global__ void k_calib_eval_finish(unsigned long long *__restrict__ blk, int n_bins) {
  const int i = threadIdx.x;
  if (i == 0) {
    blk[kCevOutSums] = (unsigned long long)__double_as_longlong(acc_value(blk + kCevBrier));
    blk[kCevOutSums + 1] = (unsigned long long)__double_as_longlong(acc_value(blk + kCevLog));
  }
  if (i < n_bins) {
    unsigned long long q[kLossAccWords];
#pragma unroll
    for (int k = 0; k < kLossLimbs; ++k) q[k] = blk[kCevBinLimbs + i * kLossLimbs + k];
    q[kLossLimbs] = 0ull;   // p is in [0, 1]: nothing to overflow
    blk[kCevOutPsum + i] = (unsigned long long)__double_as_longlong(acc_value(q));
  }
}

}  // namespace dsgd
