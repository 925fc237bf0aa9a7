/*
 * TEST INFRASTRUCTURE ONLY -- CPU restatement of the topic ranking of include/dsgd.h (dsgd_eval_*topic_ranking), the
 * checker of tests/test_gpu_topic_ranking.py.  Rows are the oracle's CSR (dsgd_oracle.h).  The walk is not the device's:
 * each row's topics are sorted by (margin, t) once, the ranks come from counting over every pair, and the top j is a prefix
 * of the sorted order.  The fixed-point sums are dsgd_oracle_common.h's fxsum.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "dsgd_oracle_common.h"   /* row_dot, fxsum */

/* the order of a row: margins ascending (the scores -m descending), ties to the lower topic; +0 and -0 compare equal */
static const double *g_m;
static int by_margin(const void *a, const void *b) {
  const int32_t x = *(const int32_t *)a, y = *(const int32_t *)b;
  if (g_m[x] < g_m[y]) return -1;
  if (g_m[x] > g_m[y]) return 1;
  return (x > y) - (x < y);
}

/* words[0 .. 8 + k + 7 (2 + k)) and sums[0 .. 2 + k) of dsgd_eval_topic_ranking over rows idx[0..n) (idx == NULL: rows
 * [begin, begin + n)).  Row r has topics tids[tptr[r] .. tptr[r + 1]) (ascending).  margins == NULL: topic t's margin of
 * position i is this library's left-fold dot of its row with W + t * a->dim; else margins[t * n + i].
 * Returns 0, -1 (allocation), -2 (a row outside the data or a topic outside [0, T)), -3 (n <= 0 or a bad k). */
int dsgd_oracle_topic_rank(const dsgd_oracle_csr *a, const double *W, int32_t T, int32_t k, const int64_t *tptr,
                           const int32_t *tids, const int32_t *idx, int64_t begin, int64_t n, const double *margins,
                           int64_t *words, double *sums) {
  if (n <= 0 || T < 1 || k < 1 || k > T || k > 32) return -3;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    if (r < 0 || r >= a->n_rows) return -2;
    for (int64_t c = tptr[r]; c < tptr[r + 1]; ++c)
      if (tids[c] < 0 || tids[c] >= T) return -2;
  }
  double *m = malloc(sizeof(double) * (size_t)T);
  int32_t *order = malloc(sizeof(int32_t) * (size_t)T);
  char *inY = malloc((size_t)T);
  fxsum *fx = calloc((size_t)(2 + k), sizeof(fxsum));   /* A, B, C_1 .. C_k */
  if (!m || !order || !inY || !fx) { free(m); free(order); free(inY); free(fx); return -1; }
  memset(words, 0, sizeof(int64_t) * (size_t)(8 + k));
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    int nan = 0;
    for (int32_t t = 0; t < T; ++t) {
      m[t] = margins ? margins[(int64_t)t * n + i] : row_dot(a, r, W + (int64_t)t * a->dim);
      nan |= isnan(m[t]);
      inY[t] = 0;
    }
    const int64_t nY = tptr[r + 1] - tptr[r];
    for (int64_t c = tptr[r]; c < tptr[r + 1]; ++c) inY[tids[c]] = 1;
    words[0] += 1;
    if (nan) { words[2] += 1; continue; }
    if (nY == 0) { words[3] += 1; continue; }
    words[1] += 1;
    words[4] += nY == T;
    int64_t cov = 0, p = 0;
    for (int32_t l = 0; l < T; ++l) {
      if (!inY[l]) continue;
      int64_t rank = 0, L = 0;   /* s_u >= s_l  <=>  m_u <= m_l */
      for (int32_t u = 0; u < T; ++u)
        if (m[u] <= m[l]) { ++rank; L += inY[u]; }
      if (rank > cov) cov = rank;
      p += rank - L;
      fx_add(&fx[0], (double)L / (double)(rank * nY));
    }
    words[5] += cov;
    words[6] += p;
    if (nY < T) fx_add(&fx[1], (double)p / (double)(nY * (T - nY)));
    for (int32_t t = 0; t < T; ++t) order[t] = t;
    g_m = m;
    qsort(order, (size_t)T, sizeof(int32_t), by_margin);
    int64_t h = 0;
    for (int32_t j = 0; j < k; ++j) {
      h += inY[order[j]];
      words[8 + j] += h;
      fx_add(&fx[2 + j], (double)h / (double)nY);
    }
  }
  for (int s = 0; s < 2 + k; ++s) {
    fxsum q = fx[s];
    fx_carry(&q);
    int64_t *blk = words + 8 + k + 7 * s;
    for (int l = 0; l < 6; ++l) blk[l] = (int64_t)q.l[l];
    blk[6] = (int64_t)q.ovf;
    sums[s] = fx_read(fx[s]);
  }
  free(m); free(order); free(inY); free(fx);
  return 0;
}
