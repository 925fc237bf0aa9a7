/*
 * TEST INFRASTRUCTURE ONLY -- CPU restatement of the one-pass topic evaluation of include/dsgd.h (dsgd_eval_*topics), the
 * checker of tests/test_gpu_topics.py.  It is T calls of the metrics checker (dsgd_oracle_metrics.c), each over the labels
 * "has topic t", plus the row words.  Rows are the oracle's CSR (dsgd_oracle.h).
 */
#include <stdlib.h>
#include <string.h>

#include "dsgd_oracle_common.h"   /* row_dot */

int dsgd_oracle_metrics(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t begin, int64_t n,
                        const double *margins, int64_t out[8]);

/* out[0 .. 8 T + 8): the words of dsgd_eval_topics over rows idx[0..n) (idx == NULL: rows [begin, begin + n)).  Row r has
 * topics tids[tptr[r] .. tptr[r + 1]) (ascending).  margins == NULL: topic t's margin of position i is this library's
 * left-fold dot of its row with W + t * a->dim; else margins[t * n + i] (e.g. the device's own, which carry the intercept).
 * Returns 0, -1 (allocation), -2 (a row outside the data), -3 (n <= 0). */
int dsgd_oracle_topics(const dsgd_oracle_csr *a, const double *W, int32_t T, const int64_t *tptr, const int32_t *tids,
                       const int32_t *idx, int64_t begin, int64_t n, const double *margins, int64_t *out) {
  if (n <= 0) return -3;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    if (r < 0 || r >= a->n_rows) return -2;
  }
  int8_t *lab = malloc((size_t)a->n_rows);
  double *m = malloc(sizeof(double) * (size_t)n * (size_t)T);
  if (!lab || !m) { free(lab); free(m); return -1; }
  for (int64_t t = 0; t < T; ++t)
    for (int64_t i = 0; i < n; ++i)
      m[t * n + i] = margins ? margins[t * n + i] : row_dot(a, idx ? idx[i] : begin + i, W + t * a->dim);
  memset(out, 0, sizeof(int64_t) * (size_t)(8 * T + 8));
  dsgd_oracle_csr at = *a;
  at.label = lab;
  int rc = 0;
  for (int32_t t = 0; t < T && rc == 0; ++t) {   /* the metrics checker over the labels "has topic t" */
    for (int64_t r = 0; r < a->n_rows; ++r) {
      int has = 0;
      for (int64_t k = tptr[r]; k < tptr[r + 1]; ++k) has |= tids[k] == t;
      lab[r] = has ? 1 : -1;
    }
    rc = dsgd_oracle_metrics(&at, NULL, idx, begin, n, m + (int64_t)t * n, out + 8 * (int64_t)t);
    out[8 * (int64_t)t + 6] = 0;
  }
  int64_t *rw = out + 8 * (int64_t)T;
  for (int64_t i = 0; i < n && rc == 0; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    int exact = 1, best = -1, best_has = 0;
    double best_m = 0.0;
    for (int32_t t = 0; t < T; ++t) {
      int has = 0;
      for (int64_t k = tptr[r]; k < tptr[r + 1]; ++k) has |= tids[k] == t;
      const double mt = m[(int64_t)t * n + i];
      const int p = mt < 0.0 ? 1 : (mt > 0.0 ? -1 : 0);   /* -signum(margin); none for 0 and NaN */
      exact &= p == (has ? 1 : -1);
      if (mt == mt && (best < 0 || mt < best_m)) { best = t; best_m = mt; best_has = has; }
    }
    rw[0] += 1;
    rw[1] += exact;
    rw[2] += tptr[r + 1] > tptr[r] && best_has;
    rw[3] += tptr[r + 1] == tptr[r];
    rw[4] += best < 0;
  }
  free(lab);
  free(m);
  return rc;
}
