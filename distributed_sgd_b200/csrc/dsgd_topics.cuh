// dsgd_topics.cuh -- sm_90a kernels of the topic calls (dsgd_select_topic, dsgd_eval_*topics; DESIGN.md §4.21; the
// ranking calls dsgd_eval_*topic_ranking and dsgd_topics_topk, §4.22).
//
// A ctx with topics keeps, beside its rows, each row's topic ids (a CSR, ascending within a row) and a copy of the labels
// dsgd_load_csr loaded.
//   * k_topic_select rewrites the binary labels as "has topic t" (t = -1: the loaded labels), and the sign of yabs with them.
//   * k_topic_eval scores every row against all T weight vectors in one pass and counts, per topic, the eight words of
//     dsgd_eval_metrics (U2 left 0), then the row words that need every topic of a row at once.
//   * k_topic_rank ranks every row's topics by the same scores: the top k, or the multi-label ranking words and sums.
//   * k_topic_keys, a segmented sort and k_topic_tune place each topic's F1-optimal threshold (§4.23), which k_topic_eval's
//     thresholded form then applies.
// Every word is an integer sum (the ranking's fractions exact fixed-point sums), so the result does not depend on the grid,
// the row order or the work split.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "dsgd_fixed.cuh"
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

// The score of one row for one weight vector w, by the whole warp (every lane gets it): chunk 0 of the row fold from the
// registers pre (pair b + lane + 32 u, a zero pair past the window), the chunks past it from memory with row_fold_from.
// That is the async worker's split of the fold: the same terms in the same order as row_fold, so the score has the bits
// dsgd_margins returns for w.  kIcpt: fl(x . w + filt(w[dim])), as row_score.
template <bool kIcpt>
__device__ __forceinline__ double topic_score(const uint2 *__restrict__ pairs, const uint2 (&pre)[4], int64_t b, int64_t e,
                                              int lane, const double *__restrict__ w, int32_t dim) {
  double acc = 0.0;
#pragma unroll
  for (int u = 0; u < 4; ++u)
    acc += filt(filt((double)__uint_as_float(pre[u].y)) * (pre[u].y << 1 ? __ldg(&w[pre[u].x]) : 0.0));
  double s = row_fold_from(pairs, b + kFoldPairs, e, lane, warp_sum(acc), [&](uint32_t c) { return __ldg(&w[c]); });
  if constexpr (kIcpt) s = s + filt(__ldg(&w[dim]));
  return s;
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

// The thresholded rule of dsgd_eval*_thresholded_topics: present (+1) below tau, absent (-1) above it, none (0) at tau or
// for a NaN margin.  At tau = +-0 it is pred_of.
__device__ __forceinline__ int pred_at(double m, double tau) { return m < tau ? 1 : (m > tau ? -1 : 0); }

// ---------------------------------------------------------------------------------------------------
// k_topic_eval: rows samples[0..n) (samples == nullptr: rows [row_begin, row_begin + n)) against the T weight vectors
// W[t * wdim, t * wdim + wdim) (on an intercept ctx the intercept is the last entry).
//   * A warp takes 32 consecutive positions at a time, as warp_scores does, and walks their rows one after the other.
//   * Of each row it loads chunk 0 of the row fold (the first kFoldPairs pairs, 4 per lane) into registers once, then folds
//     it T times with topic_score, so score_t has the bits dsgd_margins returns for W_t (and k_metrics_score ranks for it).
//   * y_t comes from the row's ascending topic list, walked alongside t.
//   * p_t is pred_of(score_t); kThr: pred_at(score_t, thr[t]) (dsgd_eval*_thresholded_topics).  The top-1 word ranks the
//     raw scores either way.
//   * Per-topic counts in shared memory (u32, one atomic per row and topic by lane 0), flushed once per CTA with u64
//     atomics into cnt[8 t + k].  Row words in lane 0's registers, flushed once per warp into cnt[8 T + k].
// Dynamic shared memory: 8 T u32 words.
// ---------------------------------------------------------------------------------------------------
template <bool kIcpt, bool kThr = false>
__global__ void __launch_bounds__(256) k_topic_eval(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                    const int64_t *__restrict__ tptr, const int32_t *__restrict__ tids,
                                                    const int32_t *__restrict__ samples, int64_t row_begin, int64_t n,
                                                    const double *__restrict__ W, int32_t T, int32_t dim,
                                                    unsigned long long *__restrict__ cnt,
                                                    const double *__restrict__ thr = nullptr) {
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
        const double s = topic_score<kIcpt>(pairs, pre, b, e, lane, W + (int64_t)t * wdim, dim);
        const bool has = tk < te && tids[tk] == t;
        tk += has;
        int p;
        if constexpr (kThr) p = pred_at(s, __ldg(&thr[t]));
        else p = pred_of(s);
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

// ---------------------------------------------------------------------------------------------------
// Ranking a row's topics (dsgd_eval_*topic_ranking, dsgd_topics_topk; DESIGN.md §4.22).  The score of topic t is -m_t, m_t
// the margin topic_score gives; a higher score ranks first, so the order is the margins ascending, ties to the lower t
// (+0 and -0 compare equal).  A warp keeps its row's T margins in shared memory, topic t at sc[t]; lane l owns the topics
// l + 32 q, q < ceil(T / 32), and keeps one bit per owned topic in a 32-bit mask (T <= 1024).
// ---------------------------------------------------------------------------------------------------
constexpr int kRankMaxK = 32;   // DSGD_TOPIC_RANK_MAX_K
constexpr int kRankWarps = 4;   // warps per CTA of k_topic_rank: 4 T doubles of shared memory, at most 32 KB
constexpr int kRankWords = 8;   // integer row words before the k hit words (DSGD_TOPIC_RANK_WORDS(k) = 8 + k + 7 (2 + k))
enum TopicRankWord : int {
  kRkRows = 0,      // rows
  kRkRanked = 1,    // ranked rows (a topic, no NaN score)
  kRkNan = 2,       // rows with a NaN score
  kRkNoTopic = 3,   // rows with no topic and no NaN score
  kRkAll = 4,       // ranked rows with every topic
  kRkCoverage = 5,  // sum of max over l in Y of rank_l
  kRkMisorder = 6   // sum over l in Y of rank_l - L_l
};

// The first topic of the order among the topics not yet taken (bit q of `taken`: topic lane + 32 q) whose margin is not
// NaN: its margin into m and its id into t, on every lane; t = -1 when there is none.  Each lane walks its topics in
// ascending t with a strict <, then the xor butterfly keeps the lower (m, t) pair: a total order, so every lane ends with
// the same pair.
__device__ __forceinline__ void warp_first_topic(const double *sc, int32_t T, int nq, int lane, unsigned taken, double &m,
                                                 int &t) {
  double bm = 0.0;
  int bt = -1;
  for (int q = 0; q < nq; ++q) {
    const int u = lane + 32 * q;
    if (u < T && !((taken >> q) & 1u)) {
      const double v = sc[u];
      if (!isnan(v) && (bt < 0 || v < bm)) { bm = v; bt = u; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double om = __shfl_xor_sync(0xffffffffu, bm, o);
    const int ot = __shfl_xor_sync(0xffffffffu, bt, o);
    if (ot >= 0 && (bt < 0 || om < bm || (om == bm && ot < bt))) { bm = om; bt = ot; }
  }
  m = bm;
  t = bt;
}

// ---------------------------------------------------------------------------------------------------
// k_topic_rank: rows samples[0..n) (samples == nullptr: rows [row_begin, row_begin + n)) against the T weight vectors W, with
// the warp-per-row walk of k_topic_eval and topic_score for every margin.  After a row's T margins are in sc:
//   kTopk: k rounds of warp_first_topic, each taking its topic out; lane 0 writes round j's id and margin to
//     ids[i k + j], top[i k + j] (i the row's position; -1 and NaN once the non-NaN margins are used up).
//   else: the ranking words of DSGD_TOPIC_RANK_WORDS(k) into cnt.  A row is ranked when it has a topic (Y, from the loaded
//     topics) and no NaN margin.  For each l in Y, one pass over the warp's topics counts rank_l = #{u : m_u <= m_l} and
//     L_l = #{u in Y : m_u <= m_l} (packed in one u32 per lane, added with __reduce_add_sync): n_Y T / 32 shared loads per
//     lane.  The top-k is k rounds of warp_first_topic; round j's hit comes from the owner lane's Y mask.
//     Integer words: 0..6 in lane 0's registers, word 8 + j (hits in the first j + 1) in lane j's; flushed once per warp.
//     Fixed-point sums (acc_add_local, flushed once per warp with acc_flush_local): lane 0 holds A, lane 1 holds B, lane j
//     holds C_(j+1).  Every term is one IEEE division of two exact integers.
// Dynamic shared memory: kRankWarps T doubles.
// ---------------------------------------------------------------------------------------------------
template <bool kIcpt, bool kTopk>
__global__ void __launch_bounds__(32 * kRankWarps) k_topic_rank(const uint32_t *__restrict__ rp16,
                                                               const uint2 *__restrict__ pairs,
                                                               const int64_t *__restrict__ tptr,
                                                               const int32_t *__restrict__ tids,
                                                               const int32_t *__restrict__ samples, int64_t row_begin,
                                                               int64_t n, const double *__restrict__ W, int32_t T,
                                                               int32_t dim, int32_t k, unsigned long long *__restrict__ cnt,
                                                               int32_t *__restrict__ ids, double *__restrict__ top) {
  extern __shared__ double s_sc[];   // [kRankWarps][T]
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  double *sc = s_sc + (int64_t)(threadIdx.x >> 5) * T;
  const int nq = (T + 31) >> 5;
  const int64_t wdim = (int64_t)dim + (kIcpt ? 1 : 0);
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  unsigned long long rw[7] = {0, 0, 0, 0, 0, 0, 0};   // words 0..6 (lane 0's count)
  unsigned long long hits = 0;                        // word 8 + lane (lane < k)
  unsigned long long lim_ab[kLossLimbs] = {}, ovf_ab = 0;   // lane 0: A, lane 1: B
  unsigned long long lim_c[kLossLimbs] = {}, ovf_c = 0;     // lane j < k: C_(j+1)
  for (int64_t g = warp0 * 32; g < n; g += nwarps * 32) {
    const int64_t i_own = g + lane;
    const int64_t r_own = i_own < n ? (samples ? (int64_t)samples[i_own] : row_begin + i_own) : 0;
    const int m = (int)(n - g < 32 ? n - g : 32);
    for (int j = 0; j < m; ++j) {
      const int64_t r = __shfl_sync(full, r_own, j);
      const int64_t b = (int64_t)rp16[r] * 2, e = (int64_t)rp16[r + 1] * 2;
      uint2 pre[4];   // chunk 0: pair b + lane + 32 u, a zero pair past the window
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t c = b + lane + 32 * u;
        pre[u] = c < e ? __ldg(&pairs[c]) : make_uint2(0u, 0u);
      }
      for (int32_t t = 0; t < T; ++t) {
        const double s = topic_score<kIcpt>(pairs, pre, b, e, lane, W + (int64_t)t * wdim, dim);
        if (lane == (t & 31)) sc[t] = s;
      }
      __syncwarp();
      if constexpr (kTopk) {
        const int64_t i = g + j;
        unsigned taken = 0;
        for (int q = 0; q < k; ++q) {
          double bm;
          int bt;
          warp_first_topic(sc, T, nq, lane, taken, bm, bt);
          if (bt >= 0 && lane == (bt & 31)) taken |= 1u << (bt >> 5);
          if (lane == 0) {
            ids[i * k + q] = bt;
            top[i * k + q] = bt >= 0 ? bm : __longlong_as_double(0x7ff8000000000000ll);
          }
        }
      } else {
        const int64_t tb = tptr[r], te = tptr[r + 1];
        const int nY = (int)(te - tb);
        bool nan = false;
        for (int q = 0; q < nq; ++q) {
          const int u = lane + 32 * q;
          nan = nan || (u < T && isnan(sc[u]));
        }
        nan = __any_sync(full, nan);
        rw[kRkRows] += 1;
        if (nan) {
          rw[kRkNan] += 1;
        } else if (nY == 0) {
          rw[kRkNoTopic] += 1;
        } else {
          unsigned inY = 0;   // bit q: topic lane + 32 q is one of the row's
          for (int64_t c = tb; c < te; ++c) {
            const int32_t id = tids[c];
            if ((id & 31) == lane) inY |= 1u << (id >> 5);
          }
          rw[kRkRanked] += 1;
          rw[kRkAll] += nY == T;
          int cov = 0;
          int64_t mis = 0;
          for (int64_t c = tb; c < te; ++c) {
            const double ml = sc[tids[c]];
            unsigned cl = 0;   // low 16 bits: u with m_u <= m_l; high: those in Y
            for (int q = 0; q < nq; ++q) {
              const int u = lane + 32 * q;
              if (u < T && sc[u] <= ml) cl += 1u + (((inY >> q) & 1u) << 16);
            }
            cl = __reduce_add_sync(full, cl);
            const int rank = (int)(cl & 0xffffu), L = (int)(cl >> 16);
            cov = max(cov, rank);
            mis += rank - L;
            if (lane == 0) acc_add_local(lim_ab, ovf_ab, (double)L / (double)(rank * nY));
          }
          rw[kRkCoverage] += cov;
          rw[kRkMisorder] += mis;
          if (lane == 1 && nY < T) acc_add_local(lim_ab, ovf_ab, (double)mis / (double)((int64_t)nY * (T - nY)));
          unsigned taken = 0;
          int h = 0;
          for (int q = 0; q < k; ++q) {
            double bm;
            int bt;
            warp_first_topic(sc, T, nq, lane, taken, bm, bt);   // bt >= 0: no NaN and k <= T
            const int owner = bt & 31, bit = bt >> 5;
            h += (__shfl_sync(full, inY, owner) >> bit) & 1u;
            if (lane == owner) taken |= 1u << bit;
            if (lane == q) {
              hits += h;
              acc_add_local(lim_c, ovf_c, (double)h / (double)nY);
            }
          }
        }
      }
      __syncwarp();   // every lane is done with sc before the next row's margins go in
    }
  }
  if constexpr (!kTopk) {
    if (lane == 0) {
#pragma unroll
      for (int w = 0; w < 7; ++w)
        if (rw[w]) atomicAdd(&cnt[w], rw[w]);
    }
    if (lane < k && hits) atomicAdd(&cnt[kRankWords + lane], hits);
    unsigned long long *sums = cnt + kRankWords + k;   // A, B, C_1 .. C_k: kLossAccWords words each
    if (lane < 2) acc_flush_local(sums + lane * kLossAccWords, lim_ab, ovf_ab);
    if (lane < k) acc_flush_local(sums + (2 + lane) * kLossAccWords, lim_c, ovf_c);
  }
}

// ---------------------------------------------------------------------------------------------------
// Tuning each topic's threshold (dsgd_tune_topic_thresholds*; DESIGN.md §4.23).  The topics go in groups of G; a group's
// workspace is a [G][n] array of margin keys and a [G][n] array of has-topic bytes, n the request's positions.
//   1. k_topic_keys scores every position against the group's weight vectors with topic_score (the bits of dsgd_margins)
//      and writes score_key(m) (kKeyNaN for a NaN margin: it sorts last) and "row has topic t" at [t - t0][i].
//   2. A segmented radix sort orders each topic's keys, the bytes with them.
//   3. k_topic_tune scans one topic's sorted segment per CTA and writes its threshold and its DSGD_TOPIC_TUNE_WORDS.
// ---------------------------------------------------------------------------------------------------
constexpr unsigned long long kKeyNaN = ~0ull;   // the key of a NaN margin, above score_key of every other margin
constexpr int kTuneThreads = 256;               // threads of k_topic_tune
constexpr int kTuneItems = 8;                   // consecutive positions per thread and tile of k_topic_tune
enum TopicTuneWord : int {
  kTuRows = 0, kTuPos = 1, kTuNan = 2, kTuDistinct = 3, kTuTp = 4, kTuPred = 5, kTuStatus = 6, kTuCand = 7
};
enum TopicTuneStatus : int { kTuned = 0, kNoPositive = 1, kBelowFbr = 2, kNoMargin = 3 };

// k_topic_keys: positions [0, n) of the rows (samples, or rows [row_begin, row_begin + n)) against topics [t0, t0 + G),
// walked as k_topic_eval walks them; lane 0 writes position i's key and byte of topic t0 + g at g n + i.
template <bool kIcpt>
__global__ void __launch_bounds__(256) k_topic_keys(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                    const int64_t *__restrict__ tptr, const int32_t *__restrict__ tids,
                                                    const int32_t *__restrict__ samples, int64_t row_begin, int64_t n,
                                                    const double *__restrict__ W, int32_t t0, int32_t G, int32_t dim,
                                                    unsigned long long *__restrict__ keys, uint8_t *__restrict__ has) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int64_t wdim = (int64_t)dim + (kIcpt ? 1 : 0);
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t g0 = warp0 * 32; g0 < n; g0 += nwarps * 32) {
    const int64_t i_own = g0 + lane;
    const int64_t r_own = i_own < n ? (samples ? (int64_t)samples[i_own] : row_begin + i_own) : 0;
    const int m = (int)(n - g0 < 32 ? n - g0 : 32);
    for (int j = 0; j < m; ++j) {
      const int64_t r = __shfl_sync(full, r_own, j), i = g0 + j;
      const int64_t b = (int64_t)rp16[r] * 2, e = (int64_t)rp16[r + 1] * 2;
      uint2 pre[4];   // chunk 0: pair b + lane + 32 u, a zero pair past the window
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t k = b + lane + 32 * u;
        pre[u] = k < e ? __ldg(&pairs[k]) : make_uint2(0u, 0u);
      }
      const int64_t te = tptr[r + 1];
      int64_t tk = topic_lower_bound(tids, tptr[r], te, t0);   // the row's next topic id at or after t
      for (int32_t g = 0; g < G; ++g) {
        const int32_t t = t0 + g;
        const double s = topic_score<kIcpt>(pairs, pre, b, e, lane, W + (int64_t)t * wdim, dim);
        const bool y = tk < te && tids[tk] == t;
        tk += y;
        if (lane == 0) {
          keys[(int64_t)g * n + i] = isnan(s) ? kKeyNaN : score_key(s);
          has[(int64_t)g * n + i] = y;
        }
      }
    }
  }
}

// One candidate of a topic: tp and pp = rows with m <= c_j (one past c_j's last position in the sorted segment); j < 0: none
struct tune_cand {
  unsigned long long tp, pp;
  long long j;
};

// The better of two candidates: the higher F1 = 2 tp / (P + pp), compared exactly by cross-multiplication in 128 bits, and
// of equal F1 the lower j (the one predicting fewer rows).  A total order on the candidates, so the block's reduction
// picks the same one in any order.
__device__ __forceinline__ tune_cand tune_pick(const tune_cand &a, const tune_cand &b, unsigned long long P) {
  if (b.j < 0) return a;
  if (a.j < 0) return b;
  const unsigned __int128 fa = (unsigned __int128)a.tp * (P + b.pp), fb = (unsigned __int128)b.tp * (P + a.pp);
  if (fa != fb) return fa > fb ? a : b;
  return a.j < b.j ? a : b;
}

// ---------------------------------------------------------------------------------------------------
// k_topic_tune: CTA s scans the sorted segment s (keys and has-topic bytes at s n .. s n + n) of topic t = t0 + s.
//   * P: a block sum of the bytes (NaN positions included).
//   * Tiles of kTuneThreads x kTuneItems positions, each thread kTuneItems consecutive ones.  A position ends a group when
//     its key is not kKeyNaN and the next key (kKeyNaN past the end) differs.  One block scan of (ends << 32 | bytes) gives
//     at each group end j = ends - 1 and tp_j; pp_j is the position + 1.
//   * Each thread keeps its best candidate (tune_pick), and remembers candidate 0 and the group end just before the key
//     of +inf; a block reduction picks the best.
//   * Thread 0 applies the status rules, places tau (the midpoint rule, +inf for the last candidate) and writes thr[t] and
//     words[8 t .. 8 t + 8).  The counts at tau = 0 (statuses 1 and 3) are the lower bound of score_key(0.0), P = 0 or no
//     non-NaN margin making tp 0; a last candidate at +inf counts at tau = +inf the rows below it.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTuneThreads) k_topic_tune(const unsigned long long *__restrict__ keys,
                                                             const uint8_t *__restrict__ has, int64_t n, int32_t t0,
                                                             double fbr, double *__restrict__ thr,
                                                             long long *__restrict__ words) {
  using Scan = cub::BlockScan<unsigned long long, kTuneThreads>;
  using Sum = cub::BlockReduce<unsigned long long, kTuneThreads>;
  using Best = cub::BlockReduce<tune_cand, kTuneThreads>;
  __shared__ union {
    typename Scan::TempStorage scan;
    typename Sum::TempStorage sum;
    typename Best::TempStorage best;
  } tmp;
  __shared__ unsigned long long s_P, s_c0[2], s_inf[2];   // P; candidate 0's (tp, pp); the counts below +inf
  const unsigned long long *k = keys + (int64_t)blockIdx.x * n;
  const uint8_t *h = has + (int64_t)blockIdx.x * n;
  const unsigned long long kInf = score_key(__longlong_as_double(0x7ff0000000000000ll));
  const unsigned long long lo32 = 0xffffffffull;
  unsigned long long p = 0;
  for (int64_t i = threadIdx.x; i < n; i += kTuneThreads) p += h[i];
  p = Sum(tmp.sum).Sum(p);
  if (threadIdx.x == 0) {
    s_P = p;
    s_c0[0] = s_c0[1] = s_inf[0] = s_inf[1] = 0;
  }
  __syncthreads();
  const unsigned long long P = s_P;
  tune_cand best{0, 0, -1};
  unsigned long long carry = 0;   // (ends << 32) | positives before the tile
  for (int64_t base = 0; base < n; base += (int64_t)kTuneThreads * kTuneItems) {
    const int64_t i0 = base + (int64_t)threadIdx.x * kTuneItems;
    unsigned long long kk[kTuneItems + 1], add[kTuneItems], tot = 0;
#pragma unroll
    for (int u = 0; u <= kTuneItems; ++u) kk[u] = i0 + u < n ? k[i0 + u] : kKeyNaN;
#pragma unroll
    for (int u = 0; u < kTuneItems; ++u) {
      const bool end = kk[u] != kKeyNaN && kk[u + 1] != kk[u];
      add[u] = (i0 + u < n ? (unsigned long long)h[i0 + u] : 0ull) + ((unsigned long long)end << 32);
      tot += add[u];
    }
    unsigned long long excl, agg;
    Scan(tmp.scan).ExclusiveSum(tot, excl, agg);
    __syncthreads();   // tmp is the next tile's
    unsigned long long run = carry + excl;
#pragma unroll
    for (int u = 0; u < kTuneItems; ++u) {
      run += add[u];
      if (add[u] >> 32) {
        const tune_cand c{run & lo32, (unsigned long long)(i0 + u + 1), (long long)(run >> 32) - 1};
        best = tune_pick(best, c, P);
        if (c.j == 0) { s_c0[0] = c.tp; s_c0[1] = c.pp; }
        if (kk[u + 1] == kInf) { s_inf[0] = c.tp; s_inf[1] = c.pp; }
      }
    }
    carry += agg;
  }
  best = Best(tmp.best).Reduce(best, [P](const tune_cand &a, const tune_cand &b) { return tune_pick(a, b, P); });
  __syncthreads();   // s_c0 and s_inf are written
  if (threadIdx.x != 0) return;
  const long long D = (long long)(carry >> 32);
  long long status, j = -1;
  unsigned long long tp, pp;
  double tau = 0.0;
  if (D == 0 || P == 0) {
    status = D == 0 ? kNoMargin : kNoPositive;
    tp = 0;
    pp = (unsigned long long)key_lower_bound(k, n, score_key(0.0));
  } else {
    status = (double)(2 * best.tp) / (double)(P + best.pp) < fbr ? kBelowFbr : kTuned;
    j = status == kBelowFbr ? 0 : best.j;
    tp = status == kBelowFbr ? s_c0[0] : best.tp;
    pp = status == kBelowFbr ? s_c0[1] : best.pp;
    const unsigned long long kc = k[pp - 1];   // c_j's key
    if (j == D - 1) {
      tau = __longlong_as_double(0x7ff0000000000000ll);
      if (kc == kInf) { tp = s_inf[0]; pp = s_inf[1]; }   // the rows at +inf get no prediction at tau = +inf
    } else {
      const double c = key_score(kc), c1 = key_score(k[pp]);
      const double mid = c / 2.0 + c1 / 2.0;
      tau = c < mid && mid <= c1 ? mid : c1;
    }
  }
  const int32_t t = t0 + (int32_t)blockIdx.x;
  long long *w = words + (int64_t)t * 8;
  w[kTuRows] = n;
  w[kTuPos] = (long long)P;
  w[kTuNan] = n - key_lower_bound(k, n, kKeyNaN);
  w[kTuDistinct] = D;
  w[kTuTp] = (long long)tp;
  w[kTuPred] = (long long)pp;
  w[kTuStatus] = status;
  w[kTuCand] = j;
  thr[t] = tau;
}

}  // namespace dsgd
