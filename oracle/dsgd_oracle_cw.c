/*
 * TEST INFRASTRUCTURE ONLY -- see dsgd_oracle_cw.h.  The array restatement of the gradient, the evaluation and the sync step
 * with one weight per class; at weights (1, 1) its arithmetic is that of dsgd_oracle.c, dsgd_oracle_logistic.c and
 * dsgd_oracle_l1.c, which it leaves alone.
 */
#include "dsgd_oracle_cw.h"

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

/* Neumaier's compensated sum of non-negative terms */
typedef struct { double s, comp; } csum;
static inline void csum_add(csum *c, double v) {
  const double t = c->s + v;
  c->comp += c->s >= v ? (c->s - t) + v : (v - t) + c->s;
  c->s = t;
}

static double l1_norm(const double *w, int32_t dim) {
  csum c = {0.0, 0.0};
  for (int32_t j = 0; j < dim; ++j) csum_add(&c, fabs(w[j]));
  return c.s + c.comp;
}

/* The per-sample pass over n rows: per-class loss sums and counts; with g != NULL also the weighted gradient sum into g
 * (dense, zero on entry). */
static void rows_pass(const dsgd_oracle_csr *a, int32_t logistic, const double *w, const int32_t *idx, int64_t n, double w_pos,
                      double w_neg, double *g, double sums[2], int64_t counts[4]) {
  csum l[2] = {{0.0, 0.0}, {0.0, 0.0}};
  memset(counts, 0, sizeof(int64_t) * 4);
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx[i];
    const double y = (double)a->label[r], dot = row_dot(a, r, w);
    const int cls = y > 0.0 ? 0 : 1;
    const double wy = cls == 0 ? w_pos : w_neg;
    const double p = -(double)((dot > 0.0) - (dot < 0.0));   /* SparseSVM.scala:14 */
    counts[2 + cls] += 1;
    counts[cls] += (p == y);
    double s;   /* the row's gradient is x * s */
    if (logistic) {
      csum_add(&l[cls], softplus(y * dot));
      s = (y * sigmoid(y * dot)) * wy;
    } else {
      const double h = 1.0 - y * p;
      csum_add(&l[cls], h > 0.0 ? h : 0.0);
      if (y * dot < 0.0) continue;   /* SparseSVM.scala:28 */
      s = y * wy;
    }
    if (!g) continue;
    for (int64_t q = a->row_ptr[r]; q < a->row_ptr[r + 1]; ++q) {
      const double gv = filt(filt((double)a->val[q]) * s);
      if (gv != 0.0) g[a->col[q]] = filt(g[a->col[q]] + gv);
    }
  }
  sums[0] = l[0].s + l[0].comp;
  sums[1] = l[1].s + l[1].comp;
}

static int ids_ok(const dsgd_oracle_csr *a, const int32_t *idx, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (idx[i] < 0 || idx[i] >= a->n_rows) return 0;
  return 1;
}

static void regularize(double *g, int32_t dim, double c) {
  if (c != 0.0 && fabs(c) > EPS)
    for (int32_t j = 0; j < dim; ++j)
      if (g[j] != 0.0) g[j] = filt(g[j] + c);
}

static void scalars(const double *w, const double *d, int32_t dim, double lambda, double *c, double *nrm2) {
  double sd = 0.0, sn = 0.0;
  for (int32_t j = 0; j < dim; ++j) {
    sd += filt(w[j] * d[j]);
    sn += w[j] * w[j];
  }
  *c = lambda * 2.0 * sd;
  *nrm2 = sn;
}

int dsgd_oracle_cw_eval(const dsgd_oracle_csr *a, int32_t logistic, const double *w, const int32_t *idx, int64_t n,
                        double *sums_out, int64_t *counts_out) {
  if (n <= 0) return -3;
  if (!ids_ok(a, idx, n)) return -2;
  rows_pass(a, logistic, w, idx, n, 1.0, 1.0, NULL, sums_out, counts_out);
  return 0;
}

int dsgd_oracle_cw_gradient(const dsgd_oracle_csr *a, int32_t logistic, double lambda, const double *d, const double *w,
                            const int32_t *idx, int64_t n, double w_pos, double w_neg, int32_t do_regularize, double *grad_out,
                            double *loss_out, double *sums_out) {
  if (n <= 0) return -3;
  if (!ids_ok(a, idx, n)) return -2;
  double c, nrm2, sums[2];
  int64_t counts[4];
  scalars(w, d, a->dim, lambda, &c, &nrm2);
  memset(grad_out, 0, sizeof(double) * (size_t)a->dim);
  rows_pass(a, logistic, w, idx, n, w_pos, w_neg, grad_out, sums, counts);
  if (do_regularize) regularize(grad_out, a->dim, c);
  const double hp = w_pos * sums[0], hn = w_neg * sums[1];
  if (loss_out) *loss_out = lambda * nrm2 + (hp + hn) / (double)n;
  if (sums_out) { sums_out[0] = sums[0]; sums_out[1] = sums[1]; }
  return 0;
}

int dsgd_oracle_cw_sync_steps(const dsgd_oracle_csr *a, int32_t logistic, double lambda, double lambda1, const double *d,
                              double *w, const int32_t *idx, const int32_t *counts, int32_t n_workers, const double *lrs,
                              int64_t n_steps, double w_pos, double w_neg, double *losses_out, double *avg_sum) {
  if (n_workers <= 0) return -3;
  int64_t per_step = 0;
  for (int32_t k = 0; k < n_workers; ++k) {
    if (counts[k] <= 0) return -3;
    per_step += counts[k];
  }
  if (!ids_ok(a, idx, per_step * n_steps)) return -2;
  const int32_t dim = a->dim;
  double *g = (double *)malloc(sizeof(double) * (size_t)dim);
  double *sum = (double *)malloc(sizeof(double) * (size_t)dim);
  if (!g || !sum) { free(g); free(sum); return -1; }
  for (int64_t t = 0; t < n_steps; ++t) {
    const int32_t *step = idx + t * per_step;
    const double lr = lrs[t];
    double c, nrm2;
    scalars(w, d, dim, lambda, &c, &nrm2);   /* every request carries the same weights */
    memset(sum, 0, sizeof(double) * (size_t)dim);
    double h = 0.0;
    int64_t off = 0;
    for (int32_t k = 0; k < n_workers; ++k) {
      double sums[2];
      int64_t cn[4];
      memset(g, 0, sizeof(double) * (size_t)dim);
      rows_pass(a, logistic, w, step + off, counts[k], w_pos, w_neg, g, sums, cn);
      regularize(g, dim, c);
      const double hp = w_pos * sums[0], hn = w_neg * sums[1], hk = hp + hn;
      h = k == 0 ? hk : h + hk;
      off += counts[k];
      for (int32_t j = 0; j < dim; ++j)   /* Vec.mean: left fold over workers, filter after every + */
        if (g[j] != 0.0) sum[j] = filt(sum[j] + g[j]);
    }
    if (losses_out) {
      losses_out[t] = lambda1 > 0.0 ? lambda * nrm2 + lambda1 * l1_norm(w, dim) + h / (double)per_step
                                    : lambda * nrm2 + h / (double)per_step;
    }
    const double tau = lr * lambda1;
    for (int32_t j = 0; j < dim; ++j) {
      double u = w[j];
      if (sum[j] != 0.0) {
        const double mean = filt(sum[j] / (double)n_workers);
        u = filt(u - filt(mean * lr));
      }
      if (tau > 0.0) u = u > tau ? filt(u - tau) : (u < -tau ? filt(u + tau) : 0.0);
      w[j] = u;
      if (avg_sum) avg_sum[j] += w[j];
    }
  }
  free(g);
  free(sum);
  return 0;
}
