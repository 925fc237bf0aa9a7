/*
 * TEST INFRASTRUCTURE ONLY -- see dsgd_oracle_sw.h.  The array restatement of the gradient, the evaluation and the sync step
 * with one weight per row; it leaves the other checkers alone.
 */
#include "dsgd_oracle_sw.h"

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

/* The fixed-point sum of non-negative terms: limbs k = 0..5 worth 2^(40 k - 160), limbs 0..4 kept below 2^40 */
typedef struct { uint64_t q[6]; int bad; } fxsum;
#define LIMB_MASK ((1ull << 40) - 1)
static void fx_carry(uint64_t q[6]) {
  for (int i = 0; i < 5; ++i) {
    q[i + 1] += q[i] >> 40;
    q[i] &= LIMB_MASK;
  }
}
static void fx_add(fxsum *f, double v) {
  if (!(v >= 0.0 && v < 4503599627370496.0)) { f->bad = 1; return; }   /* NaN, inf, >= 2^52 */
  double F[4];   /* F_i = floor(v * 2^(40 i)), exact */
  for (int i = 0; i < 4; ++i) F[i] = floor(ldexp(v, 40 * i));
  f->q[4] += (uint64_t)F[0];
  for (int i = 1; i < 4; ++i) f->q[4 - i] += (uint64_t)(F[i] - F[i - 1] * 0x1p40);
  f->q[0] += (uint64_t)(rint(ldexp(v, 160)) - F[3] * 0x1p40);   /* the one rounding: to 2^-160, ties to even */
  fx_carry(f->q);
}
static double fx_value(const fxsum *f) {
  if (f->bad) return NAN;
  uint64_t q[6];
  memcpy(q, f->q, sizeof q);
  fx_carry(q);
  double s = (double)q[5] * 0x1p40;
  for (int i = 4; i >= 0; --i) s += (double)q[i] * ldexp(1.0, 40 * i - 160);
  return s;
}

static double l1_norm(const double *w, int32_t dim) {   /* Neumaier's compensated sum, as dsgd_oracle_cw.c */
  double s = 0.0, comp = 0.0;
  for (int32_t j = 0; j < dim; ++j) {
    const double v = fabs(w[j]), t = s + v;
    comp += s >= v ? (s - t) + v : (v - t) + s;
    s = t;
  }
  return s + comp;
}

/* The per-sample pass over n rows: S, the weight of the correct rows and the weight sum, and the correct count; with
 * g != NULL also the weighted gradient sum into g (dense, zero on entry). */
static void rows_pass(const dsgd_oracle_csr *a, int32_t logistic, const double *w, const int32_t *idx, int64_t n, double w_pos,
                      double w_neg, const double *sw, double *g, double sums[3], int64_t *correct) {
  fxsum fs, fok, fw;
  memset(&fs, 0, sizeof fs); memset(&fok, 0, sizeof fok); memset(&fw, 0, sizeof fw);
  *correct = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx[i];
    const double y = (double)a->label[r], dot = row_dot(a, r, w);
    const double ci = (y > 0.0 ? w_pos : w_neg) * (sw ? sw[r] : 1.0);
    const double p = -(double)((dot > 0.0) - (dot < 0.0));   /* SparseSVM.scala:14 */
    const int ok = p == y;
    *correct += ok;
    fx_add(&fok, ok ? ci : 0.0);
    fx_add(&fw, ci);
    double s;   /* the row's gradient is x * s */
    if (logistic) {
      fx_add(&fs, ci * softplus(y * dot));
      s = (y * sigmoid(y * dot)) * ci;
    } else {
      fx_add(&fs, ci * (1.0 - y * p));
      if (y * dot < 0.0) continue;   /* SparseSVM.scala:28 */
      s = y > 0.0 ? ci : -ci;
    }
    if (!g) continue;
    for (int64_t q = a->row_ptr[r]; q < a->row_ptr[r + 1]; ++q) {
      const double gv = filt(filt((double)a->val[q]) * s);
      if (gv != 0.0) g[a->col[q]] = filt(g[a->col[q]] + gv);
    }
  }
  sums[0] = fx_value(&fs);
  sums[1] = fx_value(&fok);
  sums[2] = fx_value(&fw);
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

int dsgd_oracle_sw_eval(const dsgd_oracle_csr *a, int32_t logistic, const double *w, const int32_t *idx, int64_t n,
                        double w_pos, double w_neg, const double *sw, double *sums_out, int64_t *counts_out) {
  if (n <= 0) return -3;
  if (!ids_ok(a, idx, n)) return -2;
  rows_pass(a, logistic, w, idx, n, w_pos, w_neg, sw, NULL, sums_out, counts_out + 1);
  counts_out[0] = n;
  return 0;
}

int dsgd_oracle_sw_gradient(const dsgd_oracle_csr *a, int32_t logistic, double lambda, const double *d, const double *w,
                            const int32_t *idx, int64_t n, double w_pos, double w_neg, const double *sw, int32_t do_regularize,
                            double *grad_out, double *loss_out, double *s_out) {
  if (n <= 0) return -3;
  if (!ids_ok(a, idx, n)) return -2;
  double c, nrm2, sums[3];
  int64_t correct;
  scalars(w, d, a->dim, lambda, &c, &nrm2);
  memset(grad_out, 0, sizeof(double) * (size_t)a->dim);
  rows_pass(a, logistic, w, idx, n, w_pos, w_neg, sw, grad_out, sums, &correct);
  if (do_regularize) regularize(grad_out, a->dim, c);
  if (loss_out) *loss_out = lambda * nrm2 + sums[0] / (double)n;
  if (s_out) *s_out = sums[0];
  return 0;
}

int dsgd_oracle_sw_sync_steps(const dsgd_oracle_csr *a, int32_t logistic, double lambda, double lambda1, const double *d,
                              double *w, const int32_t *idx, const int32_t *counts, int32_t n_workers, const double *lrs,
                              int64_t n_steps, double w_pos, double w_neg, const double *sw, double *losses_out,
                              double *avg_sum) {
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
      double sums[3];
      int64_t correct;
      memset(g, 0, sizeof(double) * (size_t)dim);
      rows_pass(a, logistic, w, step + off, counts[k], w_pos, w_neg, sw, g, sums, &correct);
      regularize(g, dim, c);
      h = k == 0 ? sums[0] : h + sums[0];
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
