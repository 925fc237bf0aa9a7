// dsgd_topics.cuh -- sm_90a kernels of the topic calls (dsgd_select_topic, dsgd_eval_*topics; DESIGN.md §4.21).
//
// A ctx with topics keeps, beside its rows, each row's topic ids (a CSR, ascending within a row) and a copy of the labels
// dsgd_load_csr loaded.
//   * k_topic_select rewrites the binary labels as "has topic t" (t = -1: the loaded labels), and the sign of yabs with them.
//   * k_topic_eval scores every row against all T weight vectors in one pass and counts, per topic, the eight words of
//     dsgd_eval_metrics (U2 left 0), then the row words that need every topic of a row at once.
// Every word is an integer sum, so the result does not depend on the grid, the row order or the work split.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dsgd_kernels.cuh"
#include "dsgd_metrics.cuh"

namespace dsgd {

constexpr int kMaxTopics = 1024;   // DSGD_MAX_TOPICS
constexpr int kTopicWords = 8;     // words per topic, then kTopicWords row words (DSGD_TOPIC_WORDS(T) = 8 T + 8)
// the row words after the per-topic blocks
enum TopicRowWord : int {
  kTopRows = 0,      // rows
  kTopExact = 1,     // rows whose decision is right for every topic (p_t = y_t for all t; p = 0 is never right)
  kTopTop1 = 2,      // rows with a topic whose top-scored topic is one of theirs
  kTopNoTopic = 3,   // rows with no topic
  kTopNoScore = 4    // rows with no non-NaN score
};

// first index in ids[b, e) whose id is >= t
__device__ __forceinline__ int64_t topic_lower_bound(const int32_t *__restrict__ ids, int64_t b, int64_t e, int32_t t) {
  while (b < e) {
    const int64_t mid = (b + e) >> 1;
    if (ids[mid] < t) b = mid + 1; else e = mid;
  }
  return b;
}

// ---------------------------------------------------------------------------------------------------
// k_topic_select: one thread per row.  label[r] = +1 when row r has topic t and -1 otherwise (t < 0: label0[r], the labels
// dsgd_load_csr loaded); yabs[r] keeps its magnitude and takes the sign of the label, which is what k_repack writes for that
// label (a row with sum |x| = 0 included: -0.0f for y = -1).
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_topic_select(const int64_t *__restrict__ tptr, const int32_t *__restrict__ tids,
                                                      const int8_t *__restrict__ label0, int64_t n_rows, int32_t t,
                                                      int8_t *__restrict__ label, float *__restrict__ yabs) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  int8_t y;
  if (t < 0) {
    y = label0[r];
  } else {
    const int64_t b = tptr[r], e = tptr[r + 1];
    const int64_t k = topic_lower_bound(tids, b, e, t);
    y = (k < e && tids[k] == t) ? 1 : -1;
  }
  label[r] = y;
  yabs[r] = copysignf(fabsf(yabs[r]), y < 0 ? -1.0f : 1.0f);
}

// ---------------------------------------------------------------------------------------------------
// k_topic_eval: rows samples[0..n) (samples == nullptr: rows [row_begin, row_begin + n)) against the T weight vectors
// W[t * wdim, t * wdim + wdim) (on an intercept ctx the intercept is the last entry).
//   * A warp takes 32 consecutive positions at a time, as warp_scores does, and walks their rows one after the other.
//   * Of each row it loads chunk 0 of the row fold (the first kFoldPairs pairs, 4 per lane) into registers once, then folds
//     it T times: chunk 0 from the registers, the chunks past it from memory with row_fold_from.  That is the async
//     worker's split of the fold: the same terms in the same order as row_fold, so score_t has the bits dsgd_margins returns
//     for W_t (and k_metrics_score ranks for it).  kIcpt: score_t = fl(x . W_t + filt(beta_t)), as row_score.
//   * y_t comes from the row's ascending topic list, walked alongside t.
//   * Per-topic counts in shared memory (u32, one atomic per row and topic by lane 0), flushed once per CTA with u64
//     atomics into cnt[8 t + k].  Row words in lane 0's registers, flushed once per warp into cnt[8 T + k].
// Dynamic shared memory: 8 T u32 words.
// ---------------------------------------------------------------------------------------------------
template <bool kIcpt>
__global__ void __launch_bounds__(256) k_topic_eval(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                    const int64_t *__restrict__ tptr, const int32_t *__restrict__ tids,
                                                    const int32_t *__restrict__ samples, int64_t row_begin, int64_t n,
                                                    const double *__restrict__ W, int32_t T, int32_t dim,
                                                    unsigned long long *__restrict__ cnt) {
  extern __shared__ unsigned s_cnt[];   // [T][kTopicWords]
  for (int k = threadIdx.x; k < T * kTopicWords; k += blockDim.x) s_cnt[k] = 0u;
  __syncthreads();
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int64_t wdim = (int64_t)dim + (kIcpt ? 1 : 0);
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  unsigned long long rw[5] = {0, 0, 0, 0, 0};   // row words (lane 0's count)
  for (int64_t g = warp0 * 32; g < n; g += nwarps * 32) {
    const int64_t i = g + lane;
    const int64_t r_own = i < n ? (samples ? (int64_t)samples[i] : row_begin + i) : 0;
    const int m = (int)(n - g < 32 ? n - g : 32);
    for (int j = 0; j < m; ++j) {
      const int64_t r = __shfl_sync(full, r_own, j);
      const int64_t b = (int64_t)rp16[r] * 2, e = (int64_t)rp16[r + 1] * 2;
      uint2 pre[4];   // chunk 0: pair b + lane + 32 u, a zero pair past the window
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t k = b + lane + 32 * u;
        pre[u] = k < e ? __ldg(&pairs[k]) : make_uint2(0u, 0u);
      }
      const int64_t tb = tptr[r], te = tptr[r + 1];
      int64_t tk = tb;           // the row's next topic id at or after t
      bool exact = true;         // every decision so far right
      int best = -1;             // the top-scored topic so far (lowest x . W_t; ties: the lowest t)
      double best_dot = 0.0;
      bool best_has = false;
      for (int32_t t = 0; t < T; ++t) {
        const double *__restrict__ w = W + (int64_t)t * wdim;
        double acc = 0.0;
#pragma unroll
        for (int u = 0; u < 4; ++u)
          acc += filt(filt((double)__uint_as_float(pre[u].y)) * (pre[u].y << 1 ? __ldg(&w[pre[u].x]) : 0.0));
        double s = row_fold_from(pairs, b + kFoldPairs, e, lane, warp_sum(acc), [&](uint32_t c) { return __ldg(&w[c]); });
        if constexpr (kIcpt) s = s + filt(__ldg(&w[dim]));
        const bool has = tk < te && tids[tk] == t;
        tk += has;
        const int p = pred_of(s);
        exact = exact && p == (has ? 1 : -1);
        const bool nan = isnan(s);
        if (!nan && (best < 0 || s < best_dot)) { best = t; best_dot = s; best_has = has; }
        if (lane == 0) {
          unsigned *c = s_cnt + t * kTopicWords;
          atomicAdd(&c[(has ? kMetTp : kMetFp) + (p == 1 ? 0 : p == -1 ? 1 : 2)], 1u);
          if (nan) atomicAdd(&c[kMetNan], 1u);
        }
      }
      rw[kTopRows] += 1;
      rw[kTopExact] += exact;
      rw[kTopTop1] += te > tb && best_has;
      rw[kTopNoTopic] += te == tb;
      rw[kTopNoScore] += best < 0;
    }
  }
  if (lane == 0) {
    unsigned long long *rc = cnt + (int64_t)T * kTopicWords;
#pragma unroll
    for (int k = 0; k < 5; ++k)
      if (rw[k]) atomicAdd(&rc[k], rw[k]);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < T * kTopicWords; k += blockDim.x)
    if (s_cnt[k]) atomicAdd(&cnt[k], (unsigned long long)s_cnt[k]);
}

}  // namespace dsgd
