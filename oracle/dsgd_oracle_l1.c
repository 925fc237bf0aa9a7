/*
 * TEST INFRASTRUCTURE ONLY -- see dsgd_oracle_l1.h.  The array restatement of dsgd_oracle.c and dsgd_oracle_logistic.c (whose
 * arithmetic it leaves alone), with the proximal L1 step after every update.
 */
#include "dsgd_oracle_l1.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#define EPS 1e-20 /* math/Sparse.scala:104 */

static inline double filt(double v) { return fabs(v) > EPS ? v : 0.0; }

/* (x * w).sum: products filtered, then folded in index order */
static double row_dot(const dsgd_oracle_csr *a, int64_t r, const double *w) {
  double s = 0.0;
  for (int64_t p = a->row_ptr[r]; p < a->row_ptr[r + 1]; ++p) s += filt(filt((double)a->val[p]) * w[a->col[p]]);
  return s;
}

static inline double softplus(double z) { return (z > 0.0 ? z : 0.0) + log1p(exp(-fabs(z))); }
static inline double sigmoid(double t) {
  if (t >= 0.0) return 1.0 / (1.0 + exp(-t));
  const double e = exp(t);
  return e / (1.0 + e);
}

double dsgd_oracle_l1_prox(double u, double tau) {
  if (!(tau > 0.0)) return u;
  return u > tau ? filt(u - tau) : (u < -tau ? filt(u + tau) : 0.0);
}

double dsgd_oracle_l1_norm(const double *w, int32_t dim, int64_t *nnz_out) {
  double s = 0.0, comp = 0.0;   /* Neumaier's compensated sum of non-negative terms */
  int64_t nnz = 0;
  for (int32_t j = 0; j < dim; ++j) {
    const double v = fabs(w[j]), t = s + v;
    comp += s >= v ? (s - t) + v : (v - t) + s;
    s = t;
    nnz += (w[j] != 0.0);
  }
  if (nnz_out) *nnz_out = nnz;
  return s + comp;
}

/* One worker's reply into g (dense, zero on entry), regularized with c on the keys that survived; returns its loss sum */
static double worker_gradient(const dsgd_oracle_csr *a, int32_t logistic, double c, const double *w, const int32_t *idx,
                              int64_t n, double *g) {
  double h = 0.0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx[i];
    const double y = (double)a->label[r], dot = row_dot(a, r, w);
    double s;   /* the row's gradient is x * s */
    if (logistic) {
      h += softplus(y * dot);
      s = y * sigmoid(y * dot);
    } else {
      const double p = -(double)((dot > 0.0) - (dot < 0.0)), l = 1.0 - y * p;   /* SparseSVM.scala:14-16 */
      h += l > 0.0 ? l : 0.0;
      if (y * dot < 0.0) continue;                                               /* SparseSVM.scala:28 */
      s = y;
    }
    for (int64_t p = a->row_ptr[r]; p < a->row_ptr[r + 1]; ++p) {
      const double gv = filt(filt((double)a->val[p]) * s);
      if (gv != 0.0) g[a->col[p]] = filt(g[a->col[p]] + gv);
    }
  }
  if (c != 0.0 && fabs(c) > EPS)
    for (int32_t j = 0; j < a->dim; ++j)
      if (g[j] != 0.0) g[j] = filt(g[j] + c);
  return h;
}

int dsgd_oracle_l1_sync_steps(const dsgd_oracle_csr *a, int32_t logistic, double lambda, double lambda1, const double *d,
                              double *w, const int32_t *idx, const int32_t *counts, int32_t n_workers, const double *lrs,
                              int64_t n_steps, double *losses_out, double *avg_sum) {
  if (n_workers <= 0) return -3;
  int64_t per_step = 0;
  for (int32_t k = 0; k < n_workers; ++k) {
    if (counts[k] <= 0) return -3;
    per_step += counts[k];
  }
  for (int64_t i = 0; i < per_step * n_steps; ++i)
    if (idx[i] < 0 || idx[i] >= a->n_rows) return -2;
  const int32_t dim = a->dim;
  double *g = (double *)malloc(sizeof(double) * (size_t)dim);
  double *sum = (double *)malloc(sizeof(double) * (size_t)dim);
  if (!g || !sum) { free(g); free(sum); return -1; }
  for (int64_t t = 0; t < n_steps; ++t) {
    const int32_t *step = idx + t * per_step;
    const double lr = lrs[t];
    double sd = 0.0, sn = 0.0;
    for (int32_t j = 0; j < dim; ++j) {
      sd += filt(w[j] * d[j]);
      sn += w[j] * w[j];
    }
    const double c = lambda * 2.0 * sd;   /* every request carries the same weights */
    memset(sum, 0, sizeof(double) * (size_t)dim);
    double h = 0.0;
    int64_t off = 0;
    for (int32_t k = 0; k < n_workers; ++k) {
      memset(g, 0, sizeof(double) * (size_t)dim);
      h += worker_gradient(a, logistic, c, w, step + off, counts[k], g);
      off += counts[k];
      for (int32_t j = 0; j < dim; ++j)   /* Vec.mean: left fold over workers, filter after every + */
        if (g[j] != 0.0) sum[j] = filt(sum[j] + g[j]);
    }
    if (losses_out) losses_out[t] = lambda * sn + lambda1 * dsgd_oracle_l1_norm(w, dim, NULL) + h / (double)per_step;
    const double tau = lr * lambda1;
    for (int32_t j = 0; j < dim; ++j) {
      double u = w[j];
      if (sum[j] != 0.0) {
        const double mean = filt(sum[j] / (double)n_workers);
        u = filt(u - filt(mean * lr));
      }
      w[j] = dsgd_oracle_l1_prox(u, tau);
      if (avg_sum) avg_sum[j] += w[j];
    }
  }
  free(g);
  free(sum);
  return 0;
}
