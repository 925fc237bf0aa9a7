// dsgd_metrics.cuh -- sm_90a kernels of the scoring and ranking-metric calls (dsgd_margins, dsgd_probabilities, the
// dsgd_eval_*metrics calls; DESIGN.md §4.8) and of the curve calls (dsgd_eval_*curve; §4.9, at the end of this file).
//
// A metrics pass is three steps on the ctx's stream:
//   1. k_metrics_score: x . w of every row in fp64 (row_margin, the body dsgd_margins runs too), the confusion counts, and
//      the row's score s = -(x . w) as an order-preserving u64 key -- positives from the front of one key array, negatives
//      from its back.  NaN scores are counted and not written.
//   2. cub::DeviceRadixSort::SortKeys on each of the two runs (the host reads their lengths in between).
//   3. k_auc_count: one thread per positive key, lower_bound / upper_bound in the sorted negatives, U2 in integers.
// Every word is an integer sum, so the result does not depend on the grid or on the order in which warps take rows.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dsgd_kernels.cuh"

namespace dsgd {

// Words of dsgd_eval_*metrics (include/dsgd.h) and the two slot counters that follow them in the ctx's counter block
enum MetricWord : int {
  kMetTp = 0, kMetFn = 1, kMetPosNone = 2,   // y = +1: pred +1, pred -1, no +-1 prediction (x.w == 0 or NaN)
  kMetFp = 3, kMetTn = 4, kMetNegNone = 5,   // y = -1: pred +1, pred -1, no +-1 prediction
  kMetU2 = 6,                                // sum over (positive, negative) pairs of 2*[s_pos > s_neg] + [s_pos == s_neg]
  kMetNan = 7,                               // rows whose score is NaN
  kMetPosSlots = 8, kMetNegSlots = 9,        // keys written so far to the positive run / the negative run
  kMetWords = 16,
  // a weighted pass (k_metrics_score<kSampleWeighted>) also sums R(c_i) of the NaN-score positives and negatives here
  kMetNanPos = 16, kMetNanNeg = kMetNanPos + kLossAccWords,
  kMetWWords = 32
};
static_assert(kMetNanNeg + kLossAccWords <= kMetWWords, "the weighted block holds both NaN sums");

// x . w of row r for one warp, every lane gets it: the row fold (dsgd_kernels.cuh) that decides the row on every other
// path.  dsgd_margins and the metrics pass both call this, so a metrics pass ranks exactly the values dsgd_margins returns
// for the same rows, and its confusion counts are the predictions of every dsgd_eval_* call.
__device__ __forceinline__ double row_margin(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                             const double *__restrict__ w, int64_t r, int lane) {
  const int64_t b = (int64_t)rp16[r] * 2, e = (int64_t)rp16[r + 1] * 2;
  return row_fold(pairs, b, e, lane, [&](uint32_t c) { return w[c]; });
}

// The score of row r: x . w, or on an intercept ctx (kIcpt) fl(x . w + filt(*icpt)), the score of every other reader
// (k_rows<..., kIcpt>, k_margins<..., kIcpt>).  Otherwise icpt is not read.
template <bool kIcpt>
__device__ __forceinline__ double row_score(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                            const double *__restrict__ w, int64_t r, int lane, const double *__restrict__ icpt) {
  const double dot = row_margin(rp16, pairs, w, r, lane);
  if constexpr (kIcpt) return dot + filt(__ldg(icpt));
  return dot;
}

// The positions of an evaluation pass over rows samples[0..n) (samples == nullptr: rows [row_begin, row_begin + n)).  A
// warp takes 32 consecutive positions at a time: lane j resolves position j to its row, the warp scores the 32 rows one
// after the other (row_score) and lane j keeps the j-th score.  Then f(i, r, s, mine) runs on every lane of the warp, so
// that f may use warp-wide intrinsics: position i, its row r and score s; mine is false past n, where r = 0 and s = 0.
// Every pass that scores rows in groups takes them here, so a curve, a calibration, a quality pass and a bootstrap rank
// exactly the scores of dsgd_margins.
template <bool kIcpt, class F>
__device__ __forceinline__ void warp_scores(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                            const int32_t *__restrict__ samples, int64_t row_begin, int64_t n,
                                            const double *__restrict__ w, const double *__restrict__ icpt, F f) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t g = warp0 * 32; g < n; g += nwarps * 32) {
    const int64_t i = g + lane;
    const bool mine = i < n;
    const int64_t r_own = mine ? (samples ? (int64_t)samples[i] : row_begin + i) : 0;
    const int m = (int)(n - g < 32 ? n - g : 32);
    double dot_own = 0.0;
    for (int j = 0; j < m; ++j) {
      const int64_t r = __shfl_sync(full, r_own, j);
      const double dot = row_score<kIcpt>(rp16, pairs, w, r, lane, icpt);
      if (lane == j) dot_own = dot;
    }
    f(i, r_own, dot_own, mine);
  }
}

// c_r = fl(w_y * s_r), the weight of row r in a weighted evaluation: its class weight (w_pos or w_neg by its label) times
// its sample weight (sw == nullptr: every s_r is 1).  The training side forms the same value in k_rows<..., kSampleWeighted,
// ...> and k_sync_persistent, each with its own expression.
__device__ __forceinline__ double row_weight(bool pos, double w_pos, double w_neg, const double *__restrict__ sw, int64_t r) {
  return (pos ? w_pos : w_neg) * (sw ? __ldg(&sw[r]) : 1.0);
}

// Order-preserving key of a score: +0 and -0 are one key, and key(a) < key(b) exactly when a < b (for non-NaN scores)
__device__ __forceinline__ unsigned long long score_key(double s) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(s == 0.0 ? 0.0 : s);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// ---------------------------------------------------------------------------------------------------
// k_margins: out[i] = x . w of row samples[i] (kProb: P(y = +1 | x), the model's probability: SparseLogistic's
// sigmoid(-x . w), with the `sigmoid` of the logistic gradient, or with kHuber SparseModifiedHuber's
// (clip(-x . w, -1, 1) + 1) / 2, scikit-learn's predict_proba for that loss, NaN for a NaN margin).  One warp per row, in sample order.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ double huber_prob(double dot) {
  double m = -dot;
  m = m < -1.0 ? -1.0 : (m > 1.0 ? 1.0 : m);
  return (m + 1.0) / 2.0;
}
// kIcpt (an intercept ctx): the score is fl(x . w + filt(*icpt)), as in k_rows<..., kIcpt>; otherwise icpt is not read.
template <bool kProb, bool kHuber, bool kIcpt>
__global__ void __launch_bounds__(256) k_margins(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                 const int32_t *__restrict__ samples, int64_t n,
                                                 const double *__restrict__ w, double *__restrict__ out,
                                                 const double *__restrict__ icpt) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  double beta = 0.0;
  if constexpr (kIcpt) beta = filt(__ldg(icpt));
  for (int64_t i = warp0; i < n; i += nwarps) {
    double dot = row_margin(rp16, pairs, w, (int64_t)samples[i], lane);
    if constexpr (kIcpt) dot = dot + beta;
    if (lane == 0) out[i] = !kProb ? dot : (kHuber ? huber_prob(dot) : sigmoid(-dot));
  }
}

// ---------------------------------------------------------------------------------------------------
// k_metrics_score: the scoring step of a metrics pass over rows samples[0..n) (samples == nullptr: rows [row_begin,
// row_begin + n)), its positions taken by warp_scores.  Each lane counts its rows in registers; the counts are flushed once
// per warp.  The keys go to keys[0..) (y = +1) and keys[..n) backwards (y = -1), their slots claimed with one atomic per
// warp and class for 32 rows.
// kSampleWeighted (the weighted curve pass): each key's row weight c_i (row_weight) goes to vals[] in the key's slot, and
// the NaN rows add R(c_i) to the kMetNanPos / kMetNanNeg limbs (each lane flushes its own once).  The weighted confusion
// sums need nothing more: pred follows the sign of s, so they are read from the runs' prefix sums at the key of +0
// (k_curve_sum).
// ---------------------------------------------------------------------------------------------------
template <int kWeight, bool kIcpt>
__global__ void __launch_bounds__(256) k_metrics_score(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                       const int8_t *__restrict__ label, const int32_t *__restrict__ samples,
                                                       int64_t row_begin, int64_t n, const double *__restrict__ w,
                                                       unsigned long long *__restrict__ keys,
                                                       unsigned long long *__restrict__ cnt, double w_pos, double w_neg,
                                                       const double *__restrict__ sw, double *__restrict__ vals,
                                                       const double *__restrict__ icpt) {
  static_assert(kWeight == kUnweighted || kWeight == kSampleWeighted, "a metrics pass counts rows or weighs them by c_i");
  constexpr bool kW = kWeight == kSampleWeighted;
  unsigned long long lim_np[kLossLimbs] = {0, 0, 0, 0, 0, 0}, lim_nn[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_np = 0, ovf_nn = 0;
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  unsigned c[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // this lane's rows, by MetricWord (kMetU2 unused)
  warp_scores<kIcpt>(rp16, pairs, samples, row_begin, n, w, icpt, [&](int64_t, int64_t r, double dot, bool mine) {
    const bool pos = mine && label[r] > 0, neg = mine && !pos;
    const bool nan = mine && isnan(dot);
    const int p = pred_of(dot);   // dsgd_forward's prediction; NaN -> 0
    c[kMetTp] += pos && p == 1;
    c[kMetFn] += pos && p == -1;
    c[kMetPosNone] += pos && p == 0;
    c[kMetFp] += neg && p == 1;
    c[kMetTn] += neg && p == -1;
    c[kMetNegNone] += neg && p == 0;
    c[kMetNan] += nan;
    const bool put_pos = pos && !nan, put_neg = neg && !nan;
    const unsigned bp = __ballot_sync(full, put_pos), bn = __ballot_sync(full, put_neg);
    unsigned long long base_p = 0, base_n = 0;
    if (lane == 0) {
      if (bp) base_p = atomicAdd(&cnt[kMetPosSlots], (unsigned long long)__popc(bp));
      if (bn) base_n = atomicAdd(&cnt[kMetNegSlots], (unsigned long long)__popc(bn));
    }
    base_p = __shfl_sync(full, base_p, 0);
    base_n = __shfl_sync(full, base_n, 0);
    const unsigned below = (1u << lane) - 1u;
    if (put_pos) keys[base_p + __popc(bp & below)] = score_key(-dot);
    if (put_neg) keys[n - 1 - (int64_t)(base_n + __popc(bn & below))] = score_key(-dot);
    if constexpr (kW) {
      const double ci = mine ? row_weight(pos, w_pos, w_neg, sw, r) : 0.0;
      if (put_pos) vals[base_p + __popc(bp & below)] = ci;
      if (put_neg) vals[n - 1 - (int64_t)(base_n + __popc(bn & below))] = ci;
      if (nan && pos) acc_add_local(lim_np, ovf_np, ci);
      if (nan && neg) acc_add_local(lim_nn, ovf_nn, ci);
    }
  });
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k == kMetU2) continue;
    const unsigned s = __reduce_add_sync(full, c[k]);
    if (lane == 0 && s) atomicAdd(&cnt[k], (unsigned long long)s);
  }
  if constexpr (kW) {
    acc_flush_local(cnt + kMetNanPos, lim_np, ovf_np);
    acc_flush_local(cnt + kMetNanNeg, lim_nn, ovf_nn);
  }
}

// ---------------------------------------------------------------------------------------------------
// k_auc_count: U2 = sum over the positive keys of 2 * #{negative keys below} + #{negative keys equal}, i.e. of
// lower_bound + upper_bound in the sorted negatives.  One thread per positive key, the sum in a register, one atomic per
// warp: integer additions, the same bits in any order.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_auc_count(const unsigned long long *__restrict__ pos, int64_t n_pos,
                                                   const unsigned long long *__restrict__ neg, int64_t n_neg,
                                                   unsigned long long *__restrict__ u2) {
  unsigned long long acc = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_pos; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = pos[i];
    int64_t lo = 0, hi = n_neg;   // lower_bound: first negative >= key
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (neg[mid] < key) lo = mid + 1; else hi = mid;
    }
    int64_t up = lo, top = n_neg;   // upper_bound: first negative > key, at or after lower_bound
    while (up < top) {
      const int64_t mid = (up + top) >> 1;
      if (neg[mid] <= key) up = mid + 1; else top = mid;
    }
    acc += (unsigned long long)(lo + up);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(u2, acc);
}

// ---------------------------------------------------------------------------------------------------
// Curves and average precision (the dsgd_eval_*curve calls; DESIGN.md §4.9).  A curve pass scores and sorts as a metrics
// pass does (both runs sorted even when the other class is empty), then:
//   4. k_curve_count: one thread per sorted key.  A positive adds U2 as k_auc_count does and v_i = tp_i / (tp_i + fp_i), the
//      precision at its own score, to fixed-point limbs (dsgd_fixed.cuh); every key that ends a tie group of the union of
//      the two runs counts one point.
//   5. k_curve_sum: S = sum of the v_i as a double.
//   6. (curve wanted) cub::DeviceMerge::MergeKeys of the two runs, cub::DeviceScan::ExclusiveSum of tie_end over the merged
//      keys, and k_curve_emit: the last key of every tie group writes its point, highest score first.
// Every count is an integer and S is an order-free fixed-point sum: the result does not depend on the grid.
// The weighted pass (§4.14) runs the same steps in their kSampleWeighted forms, with (key, c) pairs sorted and each run's
// prefix sums of R(c) scanned between steps 2 and 4 (limb_sum, below).
// ---------------------------------------------------------------------------------------------------

// Words of a curve pass's own counter block (after the MetricWord block, which holds U2)
enum CurveWord : int {
  kCurAcc = 0,                   // [0, kLossAccWords): the limbs of S and their overflow count (acc_add_local); S_ap when weighted
  kCurPoints = kLossAccWords,    // m: distinct scores among the non-NaN rows
  kCurSum = kLossAccWords + 1,   // S as the bits of a double (k_curve_sum)
  kCurWords = 16,
  // a weighted curve pass (DESIGN.md §4.14): the limbs of U2w, then the DSGD_WCURVE_WORDS results as the bits of doubles
  kCurU2w = 16,
  kCurOut = kCurU2w + kLossAccWords + 1,
  kCurWWords = kCurOut + 13 + 3
};

// ---------------------------------------------------------------------------------------------------
// The weighted curve pass (dsgd_eval_*weighted_curve; DESIGN.md §4.14).  k_metrics_score<kSampleWeighted> puts c_i beside
// every key and the runs are sorted as (key, c) pairs; an inclusive scan of R(c) over each sorted run then gives exact
// prefix sums, limb_sum values carried after every addition: integer arithmetic, so any scan order gives the same limbs.
// Every weight of the pass -- W+(>= t), W-(< t), the confusion sums -- is read() of a difference of two prefixes, with
// the same bits whatever the order, the grid or the scan's tiling.  The obvious layout: 56 bytes per row.
// ---------------------------------------------------------------------------------------------------
struct limb_sum {
  unsigned long long l[kLossLimbs];   // limb k worth 2^(40 k - 160), limbs 0..4 carried into [0, 2^40)
  unsigned long long ovf;             // values that could not be cut: 2^52 or more, inf or NaN
};
// R(c) as a limb_sum (the scan's input)
struct limb_of {
  __device__ __forceinline__ limb_sum operator()(double c) const {
    limb_sum s = {{0, 0, 0, 0, 0, 0}, 0};
    acc_add_local(s.l, s.ovf, c);
    return s;
  }
};
// a + b, carried (the scan's operator); sub: a - b, its limbs in two's complement until limb_read carries them
__device__ __forceinline__ limb_sum limb_add(const limb_sum &a, const limb_sum &b, bool sub = false) {
  limb_sum r;
#pragma unroll
  for (int k = 0; k < kLossLimbs; ++k) r.l[k] = sub ? a.l[k] - b.l[k] : a.l[k] + b.l[k];
  r.ovf = sub ? a.ovf - b.ovf : a.ovf + b.ovf;
  return r;
}
struct limb_plus {
  __device__ __forceinline__ limb_sum operator()(const limb_sum &a, const limb_sum &b) const {
    limb_sum r = limb_add(a, b);
    acc_carry(r.l);
    return r;
  }
};
// read(): the value of an exact limb sum whose limbs may be negative (a difference of prefixes, never negative in total).
// A signed carry makes the limbs canonical -- limbs 0..4 in [0, 2^40) -- so the result depends only on the exact value, and
// acc_value converts it as it converts every other fixed-point sum: the same bits as k_sw_fold's for the same value.
__device__ __forceinline__ double limb_read(limb_sum v) {
  unsigned long long q[kLossAccWords];
#pragma unroll
  for (int k = 0; k < kLossLimbs - 1; ++k) {
    v.l[k + 1] += (unsigned long long)((long long)v.l[k] >> 40);
    v.l[k] &= kLimbMask;
  }
#pragma unroll
  for (int k = 0; k < kLossLimbs; ++k) q[k] = v.l[k];
  q[kLossLimbs] = v.ovf;
  return acc_value(q);
}
// the exclusive prefix k of a run from its inclusive scan: the sum of R(c) over the run's first k keys
__device__ __forceinline__ limb_sum limb_prefix(const limb_sum *__restrict__ pre, int64_t k) {
  if (k == 0) return limb_sum{{0, 0, 0, 0, 0, 0}, 0};
  return pre[k - 1];
}
// an accumulator block (kLossAccWords words) as a limb_sum
__device__ __forceinline__ limb_sum limb_load(const unsigned long long *acc) {
  limb_sum s;
#pragma unroll
  for (int k = 0; k < kLossLimbs; ++k) s.l[k] = acc[k];
  s.ovf = acc[kLossLimbs];
  return s;
}

// first index in a[0, n) whose key is >= key
__device__ __forceinline__ int64_t key_lower_bound(const unsigned long long *__restrict__ a, int64_t n,
                                                   unsigned long long key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The score of a key: the inverse of score_key (a zero score comes back as +0)
__device__ __forceinline__ double key_score(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// Thread i < n_pos takes positive key i, thread n_pos + j negative key j.  For a positive at score s: fp = negatives with a
// score >= s = n_neg - lower_bound(neg, key), tp = positives with a score >= s = n_pos - lower_bound(pos, key) (its own key
// included, so tp >= 1), v = fl(tp / (tp + fp)) in [1/n, 1].  A key ends a tie group of the union when the next key of its
// own run differs and, for a positive, no negative has its key (a group shared by both runs ends in the negatives).
// The counts, U2 and the limbs are reduced over the warp in registers and added once per warp.
// kSampleWeighted: pos_c[i] = c_i of positive key i, pre_pos / pre_neg the inclusive scans of R(c) over the runs.  A positive
// adds R(fl(c_i B_i)), B_i = read(W-(< s_i) + W-(<= s_i)) = read(2 W-(< s_i) + W-(= s_i)), to U2w (cur + kCurU2w), and when
// c_i > 0 R(fl(c_i fl(T_i / (T_i + F_i)))), T_i = W+(>= s_i), F_i = W-(>= s_i), to S_ap in place of v_i; a zero-weight row's
// precision is never formed.  U2 and the points are counted as in the unweighted form.
template <int kWeight>
__global__ void __launch_bounds__(256) k_curve_count(const unsigned long long *__restrict__ pos, int64_t n_pos,
                                                     const unsigned long long *__restrict__ neg, int64_t n_neg,
                                                     unsigned long long *__restrict__ u2,
                                                     unsigned long long *__restrict__ cur,
                                                     const double *__restrict__ pos_c = nullptr,
                                                     const limb_sum *__restrict__ pre_pos = nullptr,
                                                     const limb_sum *__restrict__ pre_neg = nullptr) {
  static_assert(kWeight == kUnweighted || kWeight == kSampleWeighted, "a curve pass counts rows or weighs them by c_i");
  constexpr bool kW = kWeight == kSampleWeighted;
  const unsigned full = 0xffffffffu;
  unsigned long long lim[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf = 0, pairs = 0, points = 0;
  unsigned long long lim2[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf2 = 0;   // kW: U2w
  const int64_t total = n_pos + n_neg;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < n_pos) {
      const unsigned long long key = pos[i];
      const int64_t lo = key_lower_bound(neg, n_neg, key);
      int64_t up = lo, top = n_neg;   // upper_bound: first negative > key
      while (up < top) {
        const int64_t mid = (up + top) >> 1;
        if (neg[mid] <= key) up = mid + 1; else top = mid;
      }
      pairs += (unsigned long long)(lo + up);
      const int64_t lp = key_lower_bound(pos, i, key);
      if constexpr (kW) {
        const double ci = pos_c[i];
        const limb_sum below = limb_prefix(pre_neg, lo);
        acc_add_local(lim2, ovf2, ci * limb_read(limb_add(below, limb_prefix(pre_neg, up))));
        if (ci > 0.0) {
          const double t = limb_read(limb_add(limb_prefix(pre_pos, n_pos), limb_prefix(pre_pos, lp), true));
          const double f = limb_read(limb_add(limb_prefix(pre_neg, n_neg), below, true));
          acc_add_local(lim, ovf, ci * (t / (t + f)));
        }
      } else {
        const int64_t tp = n_pos - lp, fp = n_neg - lo;
        acc_add_local(lim, ovf, (double)tp / (double)(tp + fp));
      }
      points += (i + 1 == n_pos || pos[i + 1] != key) && up == lo;
    } else {
      const int64_t j = i - n_pos;
      points += j + 1 == n_neg || neg[j + 1] != neg[j];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    pairs += __shfl_xor_sync(full, pairs, o);
    points += __shfl_xor_sync(full, points, o);
    ovf += __shfl_xor_sync(full, ovf, o);
#pragma unroll
    for (int k = 0; k < kLossLimbs; ++k) lim[k] += __shfl_xor_sync(full, lim[k], o);   // each below 2^45: no carry lost
    if constexpr (kW) {
      ovf2 += __shfl_xor_sync(full, ovf2, o);
#pragma unroll
      for (int k = 0; k < kLossLimbs; ++k) lim2[k] += __shfl_xor_sync(full, lim2[k], o);
    }
  }
  if ((threadIdx.x & 31) == 0) {
    if (pairs) atomicAdd(u2, pairs);
    if (points) atomicAdd(cur + kCurPoints, points);
    acc_flush_local(cur + kCurAcc, lim, ovf);
    if constexpr (kW) acc_flush_local(cur + kCurU2w, lim2, ovf2);
  }
}

// One thread: S (NaN if a value could not be summed, which no v_i in [2^-31, 1] is).
// kSampleWeighted: the DSGD_WCURVE_WORDS words, each one read() of one exact sum, as the bits of doubles at cur + kCurOut.
// The confusion sums come from the runs' prefixes at the key of +0 (s < 0: below its lower bound, s > 0: from its upper
// bound on), and the NaN rows' weights from the kMetNanPos / kMetNanNeg blocks of the metric words met.
template <int kWeight>
__global__ void k_curve_sum(unsigned long long *__restrict__ cur, const unsigned long long *__restrict__ pos = nullptr,
                            int64_t n_pos = 0, const unsigned long long *__restrict__ neg = nullptr, int64_t n_neg = 0,
                            const limb_sum *__restrict__ pre_pos = nullptr, const limb_sum *__restrict__ pre_neg = nullptr,
                            const unsigned long long *__restrict__ met = nullptr) {
  if constexpr (kWeight == kUnweighted) {
    cur[kCurSum] = (unsigned long long)__double_as_longlong(acc_value(cur + kCurAcc));
  } else {
    const unsigned long long zero = score_key(0.0);
    const limb_sum p_lo = limb_prefix(pre_pos, key_lower_bound(pos, n_pos, zero));
    const limb_sum p_up = limb_prefix(pre_pos, key_lower_bound(pos, n_pos, zero + 1));
    const limb_sum n_lo = limb_prefix(pre_neg, key_lower_bound(neg, n_neg, zero));
    const limb_sum n_up = limb_prefix(pre_neg, key_lower_bound(neg, n_neg, zero + 1));
    const limb_sum p_all = limb_prefix(pre_pos, n_pos), n_all = limb_prefix(pre_neg, n_neg);
    const limb_sum p_nan = limb_load(met + kMetNanPos), n_nan = limb_load(met + kMetNanNeg);
    const limb_sum tp = limb_add(p_all, p_up, true), tn = n_lo;
    const limb_sum w_pos = limb_add(p_all, p_nan), w_neg = limb_add(n_all, n_nan);
    const double out[13] = {
        limb_read(tp), limb_read(p_lo), limb_read(limb_add(limb_add(p_up, p_lo, true), p_nan)),
        limb_read(limb_add(n_all, n_up, true)), limb_read(tn), limb_read(limb_add(limb_add(n_up, n_lo, true), n_nan)),
        limb_read(limb_load(cur + kCurU2w)), limb_read(limb_add(p_nan, n_nan)), limb_read(limb_load(cur + kCurAcc)),
        limb_read(limb_add(tp, tn)), limb_read(limb_add(w_pos, w_neg)), limb_read(w_pos), limb_read(w_neg)};
#pragma unroll
    for (int k = 0; k < 13; ++k) cur[kCurOut + k] = (unsigned long long)__double_as_longlong(out[k]);
  }
}

// 1 when merged key i is the last of its tie group (the scan's input)
struct tie_end {
  const unsigned long long *keys;
  int n;
  __device__ __forceinline__ int operator()(int i) const { return i + 1 == n || keys[i] != keys[i + 1]; }
};

// The last key i of every tie group of the merged runs writes point m - 1 - excl[i] (excl: exclusive scan of tie_end, so
// the highest score takes point 0): its score, and tp / fp = the keys at or above it in each run.
// kSampleWeighted: tp / fp receive the bits of the doubles W+(>= t_k) and W-(>= t_k), read from the runs' prefixes.
template <int kWeight>
__global__ void __launch_bounds__(256) k_curve_emit(const unsigned long long *__restrict__ merged, int64_t n_all,
                                                    const int *__restrict__ excl,
                                                    const unsigned long long *__restrict__ pos, int64_t n_pos,
                                                    const unsigned long long *__restrict__ neg, int64_t n_neg,
                                                    const unsigned long long *__restrict__ cur, double *__restrict__ thr,
                                                    long long *__restrict__ tp, long long *__restrict__ fp,
                                                    const limb_sum *__restrict__ pre_pos = nullptr,
                                                    const limb_sum *__restrict__ pre_neg = nullptr) {
  const int64_t m = (int64_t)cur[kCurPoints];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = merged[i];
    if (i + 1 < n_all && merged[i + 1] == key) continue;
    const int64_t k = m - 1 - excl[i];
    thr[k] = key_score(key);
    if constexpr (kWeight == kSampleWeighted) {
      const limb_sum p = limb_add(limb_prefix(pre_pos, n_pos), limb_prefix(pre_pos, key_lower_bound(pos, n_pos, key)), true);
      const limb_sum q = limb_add(limb_prefix(pre_neg, n_neg), limb_prefix(pre_neg, key_lower_bound(neg, n_neg, key)), true);
      tp[k] = __double_as_longlong(limb_read(p));
      fp[k] = __double_as_longlong(limb_read(q));
    } else {
      tp[k] = n_pos - key_lower_bound(pos, n_pos, key);
      fp[k] = n_neg - key_lower_bound(neg, n_neg, key);
    }
  }
}

}  // namespace dsgd
