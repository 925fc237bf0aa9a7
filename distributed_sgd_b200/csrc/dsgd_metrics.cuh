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
  kMetWords = 16
};

// x . w of row r for one warp, every lane gets it: the row fold (dsgd_kernels.cuh) that decides the row on every other
// path.  dsgd_margins and the metrics pass both call this, so a metrics pass ranks exactly the values dsgd_margins returns
// for the same rows, and its confusion counts are the predictions of every dsgd_eval_* call.
__device__ __forceinline__ double row_margin(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                             const double *__restrict__ w, int64_t r, int lane) {
  const int64_t b = (int64_t)rp16[r] * 2, e = (int64_t)rp16[r + 1] * 2;
  return row_fold(pairs, b, e, lane, [&](uint32_t c) { return w[c]; });
}

// Order-preserving key of a score: +0 and -0 are one key, and key(a) < key(b) exactly when a < b (for non-NaN scores)
__device__ __forceinline__ unsigned long long score_key(double s) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(s == 0.0 ? 0.0 : s);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// ---------------------------------------------------------------------------------------------------
// k_margins: out[i] = x . w of row samples[i] (kProb: P(y = +1 | x) = sigmoid(-x . w), the model's probability, with the
// `sigmoid` of the logistic gradient).  One warp per row, in sample order.
// ---------------------------------------------------------------------------------------------------
template <bool kProb>
__global__ void __launch_bounds__(256) k_margins(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                 const int32_t *__restrict__ samples, int64_t n,
                                                 const double *__restrict__ w, double *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = warp0; i < n; i += nwarps) {
    const double dot = row_margin(rp16, pairs, w, (int64_t)samples[i], lane);
    if (lane == 0) out[i] = kProb ? sigmoid(-dot) : dot;
  }
}

// ---------------------------------------------------------------------------------------------------
// k_metrics_score: the scoring step of a metrics pass over rows samples[0..n) (samples == nullptr: rows [row_begin,
// row_begin + n)).  A warp takes 32 consecutive positions at a time: lane j loads the id and label of position j, the warp
// computes the 32 dots one after the other and lane j keeps the j-th.  Each lane counts its rows in registers; the counts
// are flushed once per warp.  The keys go to keys[0..) (y = +1) and keys[..n) backwards (y = -1), their slots claimed with
// one atomic per warp and class for 32 rows.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_metrics_score(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                       const int8_t *__restrict__ label, const int32_t *__restrict__ samples,
                                                       int64_t row_begin, int64_t n, const double *__restrict__ w,
                                                       unsigned long long *__restrict__ keys,
                                                       unsigned long long *__restrict__ cnt) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  unsigned c[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // this lane's rows, by MetricWord (kMetU2 unused)
  for (int64_t g = warp0 * 32; g < n; g += nwarps * 32) {
    const int64_t i = g + lane;
    const bool mine = i < n;
    const int64_t r_own = mine ? (samples ? (int64_t)samples[i] : row_begin + i) : 0;
    const int m = (int)(n - g < 32 ? n - g : 32);
    double dot_own = 0.0;
    for (int j = 0; j < m; ++j) {
      const int64_t r = __shfl_sync(full, r_own, j);
      const double dot = row_margin(rp16, pairs, w, r, lane);
      if (lane == j) dot_own = dot;
    }
    const bool pos = mine && label[r_own] > 0, neg = mine && !pos;
    const bool nan = mine && isnan(dot_own);
    const int p = pred_of(dot_own);   // dsgd_forward's prediction; NaN -> 0
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
    if (put_pos) keys[base_p + __popc(bp & below)] = score_key(-dot_own);
    if (put_neg) keys[n - 1 - (int64_t)(base_n + __popc(bn & below))] = score_key(-dot_own);
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k == kMetU2) continue;
    const unsigned s = __reduce_add_sync(full, c[k]);
    if (lane == 0 && s) atomicAdd(&cnt[k], (unsigned long long)s);
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
// ---------------------------------------------------------------------------------------------------

// Words of a curve pass's own counter block (after the MetricWord block, which holds U2)
enum CurveWord : int {
  kCurAcc = 0,                   // [0, kLossAccWords): the limbs of S and their overflow count (acc_add_local)
  kCurPoints = kLossAccWords,    // m: distinct scores among the non-NaN rows
  kCurSum = kLossAccWords + 1,   // S as the bits of a double (k_curve_sum)
  kCurWords = 16
};

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
__global__ void __launch_bounds__(256) k_curve_count(const unsigned long long *__restrict__ pos, int64_t n_pos,
                                                     const unsigned long long *__restrict__ neg, int64_t n_neg,
                                                     unsigned long long *__restrict__ u2,
                                                     unsigned long long *__restrict__ cur) {
  const unsigned full = 0xffffffffu;
  unsigned long long lim[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf = 0, pairs = 0, points = 0;
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
      const int64_t tp = n_pos - key_lower_bound(pos, i, key), fp = n_neg - lo;
      acc_add_local(lim, ovf, (double)tp / (double)(tp + fp));
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
  }
  if ((threadIdx.x & 31) == 0) {
    if (pairs) atomicAdd(u2, pairs);
    if (points) atomicAdd(cur + kCurPoints, points);
    acc_flush_local(cur + kCurAcc, lim, ovf);
  }
}

// One thread: S (NaN if a value could not be summed, which no v_i in [2^-31, 1] is)
__global__ void k_curve_sum(unsigned long long *__restrict__ cur) {
  cur[kCurSum] = (unsigned long long)__double_as_longlong(acc_value(cur + kCurAcc));
}

// 1 when merged key i is the last of its tie group (the scan's input)
struct tie_end {
  const unsigned long long *keys;
  int n;
  __device__ __forceinline__ int operator()(int i) const { return i + 1 == n || keys[i] != keys[i + 1]; }
};

// The last key i of every tie group of the merged runs writes point m - 1 - excl[i] (excl: exclusive scan of tie_end, so
// the highest score takes point 0): its score, and tp / fp = the keys at or above it in each run.
__global__ void __launch_bounds__(256) k_curve_emit(const unsigned long long *__restrict__ merged, int64_t n_all,
                                                    const int *__restrict__ excl,
                                                    const unsigned long long *__restrict__ pos, int64_t n_pos,
                                                    const unsigned long long *__restrict__ neg, int64_t n_neg,
                                                    const unsigned long long *__restrict__ cur, double *__restrict__ thr,
                                                    long long *__restrict__ tp, long long *__restrict__ fp) {
  const int64_t m = (int64_t)cur[kCurPoints];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = merged[i];
    if (i + 1 < n_all && merged[i + 1] == key) continue;
    const int64_t k = m - 1 - excl[i];
    thr[k] = key_score(key);
    tp[k] = n_pos - key_lower_bound(pos, n_pos, key);
    fp[k] = n_neg - key_lower_bound(neg, n_neg, key);
  }
}

}  // namespace dsgd
