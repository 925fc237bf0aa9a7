/*
 * TEST INFRASTRUCTURE ONLY -- fp64 CPU restatement of the curves and average precision of include/dsgd.h
 * (dsgd_eval_*curve), the checker of tests/test_gpu_curve.py.  When the caller passes no margins it uses the left-fold dots
 * of dsgd_oracle_metrics.c (dsgd_oracle_margins).
 */
#include <stdlib.h>

#include "dsgd_oracle.h"

int dsgd_oracle_margins(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t begin, int64_t n,
                        double *margins);

typedef struct {
  double s;
  int pos;
} scored;

static int cmp_desc(const void *x, const void *y) {
  const double a = ((const scored *)x)->s, b = ((const scored *)y)->s;
  return (a < b) - (a > b); /* highest score first; -0 == +0: one score */
}

/* The points of the curve over rows idx[0..n) (idx == NULL: rows [begin, begin + n)), with s = -margin: one per distinct
 * non-NaN score t_k, highest first -- thr[k] = t_k (a zero score as +0), tp[k] / fp[k] = positive / negative rows with
 * s >= t_k -- and *n_points of them; v[i] = tp_i / (tp_i + fp_i) of every non-NaN positive row, counted at its own score, in
 * the order of the walk, and *n_v of them; *n_nan = rows whose margin is NaN.  margins == NULL: the left-fold dots of
 * dsgd_oracle_margins; else margins[i] is row i's margin.  The scores are sorted with qsort and walked once, a tie group at a
 * time.  Every output array holds n entries.  Returns 0, -1 (allocation), -2 (a row outside the data) or -3 (n <= 0). */
int dsgd_oracle_curve(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t begin, int64_t n,
                      const double *margins, int64_t *n_points, double *thr, int64_t *tp, int64_t *fp, double *v,
                      int64_t *n_v, int64_t *n_nan) {
  if (n <= 0) return -3;
  double *m = malloc(sizeof(double) * (size_t)n);
  scored *r = malloc(sizeof(scored) * (size_t)n);
  if (!m || !r) { free(m); free(r); return -1; }
  int rc = margins ? 0 : dsgd_oracle_margins(a, w, idx, begin, n, m);
  if (!rc)
    for (int64_t i = 0; i < n; ++i) {
      const int64_t row = idx ? idx[i] : begin + i;
      if (row < 0 || row >= a->n_rows) { rc = -2; break; }
    }
  if (rc) { free(m); free(r); return rc; }
  int64_t k = 0, nan = 0;
  for (int64_t i = 0; i < n; ++i) {
    const double mi = margins ? margins[i] : m[i];
    if (mi != mi) { ++nan; continue; }
    r[k].s = mi == 0.0 ? 0.0 : -mi;
    r[k].pos = a->label[idx ? idx[i] : begin + i] > 0;
    ++k;
  }
  qsort(r, (size_t)k, sizeof(scored), cmp_desc);
  int64_t ctp = 0, cfp = 0, pts = 0, nv = 0;
  for (int64_t i = 0; i < k;) {
    int64_t j = i, gp = 0;
    for (; j < k && r[j].s == r[i].s; ++j) gp += r[j].pos;
    ctp += gp;
    cfp += (j - i) - gp;
    thr[pts] = r[i].s;
    tp[pts] = ctp;
    fp[pts] = cfp;
    ++pts;
    for (int64_t g = 0; g < gp; ++g) v[nv++] = (double)ctp / (double)(ctp + cfp);
    i = j;
  }
  *n_points = pts;
  *n_v = nv;
  *n_nan = nan;
  free(m);
  free(r);
  return 0;
}
