/*
 * TEST INFRASTRUCTURE ONLY -- CPU restatement of the per-topic threshold tuning of include/dsgd.h
 * (dsgd_tune_topic_thresholds*), the checker of tests/test_gpu_topic_thresholds.py.  Rows are the oracle's CSR
 * (dsgd_oracle.h).  The walk is not the device's: each topic's (margin, has-topic) pairs are sorted with qsort by margin
 * and scanned in order, candidates compared by 128-bit cross-multiplication.
 */
#include <math.h>
#include <stdlib.h>

#include "dsgd_oracle_common.h"   /* row_dot */

typedef struct {
  double m;
  int y;
} thresh_pair;

static int by_margin(const void *a, const void *b) {
  const double x = ((const thresh_pair *)a)->m, y = ((const thresh_pair *)b)->m;
  return (x > y) - (x < y);
}

/* thresholds[0 .. T) and words[0 .. 8 T) of dsgd_tune_topic_thresholds over rows idx[0..n) (idx == NULL: rows
 * [begin, begin + n)).  Row r has topics tids[tptr[r] .. tptr[r + 1]).  margins == NULL: topic t's margin of position i is
 * this library's left-fold dot of its row with W + t * a->dim; else margins[t * n + i].
 * Returns 0, -1 (allocation), -2 (a row outside the data or a topic outside [0, T)), -3 (n < 0, T < 1 or fbr outside
 * [0, 1]). */
int dsgd_oracle_topic_thresh(const dsgd_oracle_csr *a, const double *W, int32_t T, const int64_t *tptr,
                             const int32_t *tids, const int32_t *idx, int64_t begin, int64_t n, const double *margins,
                             double fbr, double *thresholds, int64_t *words) {
  if (n < 0 || T < 1 || !(fbr >= 0.0 && fbr <= 1.0)) return -3;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    if (r < 0 || r >= a->n_rows) return -2;
    for (int64_t c = tptr[r]; c < tptr[r + 1]; ++c)
      if (tids[c] < 0 || tids[c] >= T) return -2;
  }
  thresh_pair *v = malloc(sizeof(thresh_pair) * (size_t)(n > 0 ? n : 1));
  if (!v) return -1;
  for (int32_t t = 0; t < T; ++t) {
    int64_t P = 0, nn = 0, nan = 0;
    for (int64_t i = 0; i < n; ++i) {
      const int64_t r = idx ? idx[i] : begin + i;
      const double m = margins ? margins[(int64_t)t * n + i] : row_dot(a, r, W + (int64_t)t * a->dim);
      int y = 0;
      for (int64_t c = tptr[r]; c < tptr[r + 1]; ++c) y |= tids[c] == t;
      P += y;
      if (isnan(m)) { ++nan; continue; }
      v[nn].m = m == 0.0 ? 0.0 : m;
      v[nn].y = y;
      ++nn;
    }
    qsort(v, (size_t)nn, sizeof(thresh_pair), by_margin);
    /* one pass: the candidates at the group ends, the best (F1 higher, ties to lower j), candidate 0, and the counts below
     * +inf */
    int64_t D = 0, tp = 0, best_j = -1, best_tp = 0, best_pp = 0, c0_tp = 0, c0_pp = 0, inf_tp = 0, inf_pp = 0;
    for (int64_t i = 0; i < nn; ++i) {
      tp += v[i].y;
      if (i + 1 < nn && v[i + 1].m == v[i].m) continue;
      const int64_t j = D++, pp = i + 1;
      if (j == 0) { c0_tp = tp; c0_pp = pp; }
      if (i + 1 < nn && isinf(v[i + 1].m) && v[i + 1].m > 0) { inf_tp = tp; inf_pp = pp; }
      if (best_j < 0 || (unsigned __int128)tp * (uint64_t)(P + best_pp) > (unsigned __int128)best_tp * (uint64_t)(P + pp)) {
        best_j = j; best_tp = tp; best_pp = pp;
      }
    }
    int64_t status, j = -1, wtp = 0, wpp = 0;
    double tau = 0.0;
    if (D == 0 || P == 0) {
      status = D == 0 ? 3 : 1;
      for (int64_t i = 0; i < nn; ++i) wpp += v[i].m < 0.0;
    } else {
      const int below = (double)(2 * best_tp) / (double)(P + best_pp) < fbr;
      status = below ? 2 : 0;
      j = below ? 0 : best_j;
      wtp = below ? c0_tp : best_tp;
      wpp = below ? c0_pp : best_pp;
      const double c = v[wpp - 1].m;
      if (j == D - 1) {
        tau = INFINITY;
        if (isinf(c) && c > 0) { wtp = inf_tp; wpp = inf_pp; }
      } else {
        const double c1 = v[wpp].m, mid = c / 2.0 + c1 / 2.0;
        tau = c < mid && mid <= c1 ? mid : c1;
      }
    }
    thresholds[t] = tau;
    int64_t *w = words + (int64_t)t * 8;
    w[0] = n; w[1] = P; w[2] = nan; w[3] = D; w[4] = wtp; w[5] = wpp; w[6] = status; w[7] = j;
  }
  free(v);
  return 0;
}
