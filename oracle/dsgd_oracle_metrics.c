/*
 * TEST INFRASTRUCTURE ONLY -- fp64 CPU restatement of the scores and ranking metrics of include/dsgd.h (dsgd_margins,
 * dsgd_eval_*metrics), the checker of tests/test_gpu_metrics.py.  Rows are the oracle's CSR (dsgd_oracle.h); the dot is
 * the oracle's left fold (dsgd_oracle.c: row_dot), restated here.
 */
#include <stdlib.h>

#include "dsgd_oracle_common.h"   /* row_dot */

static int rows_ok(const dsgd_oracle_csr *a, const int32_t *idx, int64_t begin, int64_t n) {
  if (!idx) return (begin < 0 || begin + n > a->n_rows) ? -2 : 0;
  for (int64_t i = 0; i < n; ++i)
    if (idx[i] < 0 || idx[i] >= a->n_rows) return -2;
  return 0;
}

/* margins[i] = x_r . w of row r = idx[i], or r = begin + i when idx == NULL. */
int dsgd_oracle_margins(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t begin, int64_t n,
                        double *margins) {
  if (rows_ok(a, idx, begin, n)) return -2;
  for (int64_t i = 0; i < n; ++i) margins[i] = row_dot(a, idx ? idx[i] : begin + i, w);
  return 0;
}

static int cmp_double(const void *x, const void *y) {
  const double a = *(const double *)x, b = *(const double *)y;
  return (a > b) - (a < b); /* -0 == +0: one score */
}

/* The eight words of dsgd_eval_metrics over rows idx[0..n) (idx == NULL: rows [begin, begin + n)): TP, FN, positives with no
 * +-1 prediction, FP, TN, negatives with none, U2 = sum over (positive, negative) pairs of 2*[s_pos > s_neg] + [s_pos == s_neg]
 * with s = -margin, and the rows whose margin is NaN (left out of U2).  margins == NULL: this file's left-fold dots; else
 * margins[i] is row i's margin (e.g. the device's own), so a test can check the counting apart from the dot.  The negatives'
 * scores are sorted with qsort and each positive is placed by binary search.  Returns 0, -1 (allocation), -2 (a row outside
 * the data) or -3 (n <= 0). */
int dsgd_oracle_metrics(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t begin, int64_t n,
                        const double *margins, int64_t out[8]) {
  if (n <= 0) return -3;
  if (rows_ok(a, idx, begin, n)) return -2;
  double *pos = malloc(sizeof(double) * (size_t)n), *neg = malloc(sizeof(double) * (size_t)n);
  if (!pos || !neg) { free(pos); free(neg); return -1; }
  int64_t np = 0, nn = 0;
  for (int k = 0; k < 8; ++k) out[k] = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    const double m = margins ? margins[i] : row_dot(a, r, w);
    const int y_pos = a->label[r] > 0;
    /* prediction -signum(m) (SparseSVM.scala:14): +1 when m < 0, -1 when m > 0, none when m is 0 or NaN */
    out[(y_pos ? 0 : 3) + (m < 0.0 ? 0 : (m > 0.0 ? 1 : 2))] += 1;
    if (m != m) { out[7] += 1; continue; }
    if (y_pos) pos[np++] = -m; else neg[nn++] = -m;
  }
  qsort(neg, (size_t)nn, sizeof(double), cmp_double);
  int64_t u2 = 0;
  for (int64_t i = 0; i < np; ++i) {
    int64_t lo = 0, hi = nn; /* first negative >= s */
    while (lo < hi) { int64_t mid = (lo + hi) / 2; if (neg[mid] < pos[i]) lo = mid + 1; else hi = mid; }
    int64_t up = lo, top = nn; /* first negative > s */
    while (up < top) { int64_t mid = (up + top) / 2; if (neg[mid] <= pos[i]) up = mid + 1; else top = mid; }
    u2 += lo + up; /* 2 * #{below} + #{equal} */
  }
  out[6] = u2;
  free(pos);
  free(neg);
  return 0;
}
