/*
 * TEST INFRASTRUCTURE ONLY -- see dsgd_oracle_logistic.h.  The same array restatement as dsgd_oracle.c (whose SVM arithmetic
 * it leaves alone), with the logistic loss and backward.
 */
#include "dsgd_oracle_logistic.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#define EPS 1e-20 /* math/Sparse.scala:104 */

static inline double filt(double v) { return fabs(v) > EPS ? v : 0.0; }

/* (x * w).sum: products filtered, then folded in index order (dsgd_oracle.c: row_dot) */
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

static int check_rows(const dsgd_oracle_csr *a, const int32_t *idx, int64_t begin, int64_t n) {
  if (!idx) return (begin < 0 || begin + n > a->n_rows) ? -2 : 0;
  for (int64_t i = 0; i < n; ++i)
    if (idx[i] < 0 || idx[i] >= a->n_rows) return -2;
  return 0;
}

static double norm_squared(const double *w, int32_t dim) {
  double s = 0.0;
  for (int32_t j = 0; j < dim; ++j) s += w[j] * w[j];
  return s;
}

static double reg_scalar(double lambda, const double *w, const double *d, int32_t dim) {
  double s = 0.0;
  for (int32_t j = 0; j < dim; ++j) s += filt(w[j] * d[j]);
  return lambda * 2.0 * s;
}

int dsgd_oracle_logistic_sample_losses(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t begin,
                                       int64_t n, double *losses) {
  if (check_rows(a, idx, begin, n)) return -2;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    losses[i] = softplus((double)a->label[r] * row_dot(a, r, w));
  }
  return 0;
}

int dsgd_oracle_logistic_loss_acc(const dsgd_oracle_csr *a, double lambda, const double *w, const int32_t *idx,
                                  int64_t begin, int64_t n, double *loss, double *acc) {
  if (n <= 0) return -3;
  if (check_rows(a, idx, begin, n)) return -2;
  double total = 0.0;
  int64_t correct = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    const double dot = row_dot(a, r, w), y = (double)a->label[r];
    total += softplus(y * dot);
    correct += ((double)((dot < 0.0) - (dot > 0.0)) == y);   /* -signum(x . w) == y */
  }
  if (loss) *loss = lambda * norm_squared(w, a->dim) + total / (double)n;
  if (acc) *acc = (double)correct / (double)n;
  return 0;
}

/* One worker's reply into g (dense, zero on entry): sum_i x_i * (y_i * sigmoid(z_i)) folded with the filter after every
 * addition, then regularize (c on the keys that survived).  Returns the batch's loss sum (a left fold). */
static double worker_gradient(const dsgd_oracle_csr *a, double c, const double *w, const int32_t *idx, int64_t n, double *g) {
  double h = 0.0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx[i];
    const double y = (double)a->label[r];
    const double z = y * row_dot(a, r, w);
    h += softplus(z);
    const double s = y * sigmoid(z);
    for (int64_t p = a->row_ptr[r]; p < a->row_ptr[r + 1]; ++p) {
      const double gv = filt(filt((double)a->val[p]) * s);   /* x * s: mapValues + constructor filter */
      if (gv != 0.0) g[a->col[p]] = filt(g[a->col[p]] + gv);
    }
  }
  if (c != 0.0 && fabs(c) > EPS)
    for (int32_t j = 0; j < a->dim; ++j)
      if (g[j] != 0.0) g[j] = filt(g[j] + c);
  return h;
}

int dsgd_oracle_logistic_gradient(const dsgd_oracle_csr *a, double lambda, const double *d, const double *w,
                                  const int32_t *idx, int64_t n, double *r_out, double *c_out) {
  if (n <= 0) return -3;
  if (check_rows(a, idx, 0, n)) return -2;
  const double c = reg_scalar(lambda, w, d, a->dim);
  memset(r_out, 0, sizeof(double) * (size_t)a->dim);
  worker_gradient(a, c, w, idx, n, r_out);
  if (c_out) *c_out = c;
  return 0;
}

int dsgd_oracle_logistic_sync_steps(const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                                    const int32_t *idx, const int32_t *counts, int32_t n_workers, double lr,
                                    int64_t n_steps, double *losses_out) {
  if (n_workers <= 0) return -3;
  int64_t per_step = 0;
  for (int32_t k = 0; k < n_workers; ++k) {
    if (counts[k] <= 0) return -3;
    per_step += counts[k];
  }
  if (check_rows(a, idx, 0, per_step * n_steps)) return -2;
  double *g = (double *)malloc(sizeof(double) * (size_t)a->dim);
  double *sum = (double *)malloc(sizeof(double) * (size_t)a->dim);
  if (!g || !sum) { free(g); free(sum); return -1; }
  for (int64_t s = 0; s < n_steps; ++s) {
    const int32_t *step = idx + s * per_step;
    const double c = reg_scalar(lambda, w, d, a->dim);   /* every request carries the same weights */
    memset(sum, 0, sizeof(double) * (size_t)a->dim);
    double h = 0.0;
    int64_t off = 0;
    for (int32_t k = 0; k < n_workers; ++k) {
      memset(g, 0, sizeof(double) * (size_t)a->dim);
      h += worker_gradient(a, c, w, step + off, counts[k], g);
      off += counts[k];
      for (int32_t j = 0; j < a->dim; ++j)   /* Vec.mean: left fold over workers, filter after every + */
        if (g[j] != 0.0) sum[j] = filt(sum[j] + g[j]);
    }
    if (losses_out) losses_out[s] = lambda * norm_squared(w, a->dim) + h / (double)per_step;
    for (int32_t j = 0; j < a->dim; ++j) {
      if (sum[j] == 0.0) continue;
      const double mean = filt(sum[j] / (double)n_workers);
      const double st = filt(mean * lr);
      w[j] = filt(w[j] - st);
    }
  }
  free(g);
  free(sum);
  return 0;
}
