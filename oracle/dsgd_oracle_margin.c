/*
 * TEST INFRASTRUCTURE ONLY -- see dsgd_oracle_margin.h.  The array restatement of the gradient, the evaluations and the sync
 * step of the margin models, in every weighting; it leaves the other checkers alone.
 */
#include "dsgd_oracle_margin.h"

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

int dsgd_oracle_margin_row(int32_t model, double z, double *loss_out, double *scale_out) {
  const double t = 1.0 + z;
  double l, s;
  switch (model) {
    case 1: l = softplus(z); s = sigmoid(z); break;
    case 2: l = z <= -1.0 ? 0.0 : t * t; s = z <= -1.0 ? 0.0 : 2.0 * t; break;
    case 3:
      l = z <= -1.0 ? 0.0 : (z <= 1.0 ? t * t : 4.0 * z);
      s = z <= -1.0 ? 0.0 : (z <= 1.0 ? 2.0 * t : 4.0);
      break;
    default: return -3;
  }
  if (loss_out) *loss_out = l;
  if (scale_out) *scale_out = s;
  return 0;
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

static double l1_norm(const double *w, int32_t dim) {   /* the device's fixed-point sum: every |w_j| > 1e-20 is exact in it */
  fxsum f;
  memset(&f, 0, sizeof f);
  for (int32_t j = 0; j < dim; ++j) fx_add(&f, fabs(w[j]));
  return fx_value(&f);
}

/* The totals of one pass (pass_rows) */
typedef struct {
  double s;          /* the pass's loss sum in its weighting (header) */
  double cls[2];     /* weighting 1: the unweighted loss sums of the y = +1 and y = -1 rows */
  double ok_w, all_w;   /* weighting 2: sum c_i [correct], sum c_i */
  int64_t correct, cls_ok[2], cls_n[2];
} pass_totals;

/* The per-sample pass over the listed rows (idx == NULL: rows [begin, begin + n)); with g != NULL also the gradient sum in
 * the weighting into g (dense, zero on entry), filtered after every addition. */
static void pass_rows(const dsgd_oracle_csr *a, int32_t model, int32_t weighting, const double *w, const int32_t *idx,
                      int64_t begin, int64_t n, double w_pos, double w_neg, const double *sw, double *g, pass_totals *o) {
  fxsum fs, fok, fw, fc[2];
  memset(&fs, 0, sizeof fs); memset(&fok, 0, sizeof fok); memset(&fw, 0, sizeof fw); memset(fc, 0, sizeof fc);
  memset(o, 0, sizeof *o);
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    const double y = (double)a->label[r], dot = row_dot(a, r, w), z = y * dot;
    const int cls = y > 0.0 ? 0 : 1;
    const double wy = cls == 0 ? w_pos : w_neg;
    const double c = weighting == 2 ? wy * (sw ? sw[r] : 1.0) : weighting == 1 ? wy : 1.0;
    const double p = -(double)((dot > 0.0) - (dot < 0.0));   /* SparseSVM.scala:14 */
    const int ok = p == y;
    double l, sc = 0.0;
    if (model == 0) l = 1.0 - y * p;
    else dsgd_oracle_margin_row(model, z, &l, &sc);
    o->correct += ok;
    o->cls_ok[cls] += ok;
    o->cls_n[cls] += 1;
    if (weighting == 2) {
      fx_add(&fs, c * l);
      fx_add(&fok, ok ? c : 0.0);
      fx_add(&fw, c);
    } else if (weighting == 1) {
      fx_add(&fc[cls], l);
    } else {
      fx_add(&fs, l);
    }
    if (!g) continue;
    double v;   /* the row's gradient is x * v */
    if (model == 0) {
      if (z < 0.0) continue;   /* SparseSVM.scala:28 */
      v = weighting == 0 ? y : (y > 0.0 ? c : -c);
    } else {
      v = weighting == 0 ? y * sc : (y * sc) * c;
    }
    for (int64_t q = a->row_ptr[r]; q < a->row_ptr[r + 1]; ++q) {
      const double gv = filt(filt((double)a->val[q]) * v);
      if (gv != 0.0) g[a->col[q]] = filt(g[a->col[q]] + gv);
    }
  }
  o->cls[0] = fx_value(&fc[0]);
  o->cls[1] = fx_value(&fc[1]);
  if (weighting == 1) {
    const double hp = w_pos * o->cls[0], hn = w_neg * o->cls[1];
    o->s = hp + hn;
  } else {
    o->s = fx_value(&fs);
  }
  o->ok_w = fx_value(&fok);
  o->all_w = fx_value(&fw);
}

static int bad_args(const dsgd_oracle_csr *a, int32_t model, int32_t weighting, const int32_t *idx, int64_t begin, int64_t n) {
  if (model < 0 || model > 3 || weighting < 0 || weighting > 2 || n <= 0) return -3;
  if (!idx) return (begin < 0 || begin + n > a->n_rows) ? -2 : 0;
  for (int64_t i = 0; i < n; ++i)
    if (idx[i] < 0 || idx[i] >= a->n_rows) return -2;
  return 0;
}

static void regularize(double *g, int32_t dim, double c) {
  if (c != 0.0 && fabs(c) > EPS)
    for (int32_t j = 0; j < dim; ++j)
      if (g[j] != 0.0) g[j] = filt(g[j] + c);
}

static void scalars(const double *w, const double *d, int32_t dim, double lambda, double *c, double *nrm2) {
  double sd = 0.0, sn = 0.0;
  for (int32_t j = 0; j < dim; ++j) {
    if (d) sd += filt(w[j] * d[j]);
    sn += w[j] * w[j];
  }
  *c = lambda * 2.0 * sd;
  *nrm2 = sn;
}

int dsgd_oracle_margin_sample_losses(const dsgd_oracle_csr *a, int32_t model, const double *w, const int32_t *idx,
                                     int64_t begin, int64_t n, double *losses) {
  int rc = bad_args(a, model, 0, idx, begin, n);
  if (rc) return rc;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = idx ? idx[i] : begin + i;
    const double y = (double)a->label[r], dot = row_dot(a, r, w);
    if (model == 0) losses[i] = 1.0 - y * -(double)((dot > 0.0) - (dot < 0.0));
    else dsgd_oracle_margin_row(model, y * dot, &losses[i], NULL);
  }
  return 0;
}

int dsgd_oracle_margin_loss_acc(const dsgd_oracle_csr *a, int32_t model, double lambda, const double *w, const int32_t *idx,
                                int64_t begin, int64_t n, double *loss_out, double *acc_out, double *s_out,
                                int64_t *correct_out) {
  int rc = bad_args(a, model, 0, idx, begin, n);
  if (rc) return rc;
  pass_totals o;
  double c, nrm2;
  pass_rows(a, model, 0, w, idx, begin, n, 1.0, 1.0, NULL, NULL, &o);
  scalars(w, NULL, a->dim, lambda, &c, &nrm2);
  if (loss_out) *loss_out = lambda * nrm2 + o.s / (double)n;
  if (acc_out) *acc_out = (double)o.correct / (double)n;
  if (s_out) *s_out = o.s;
  if (correct_out) *correct_out = o.correct;
  return 0;
}

int dsgd_oracle_margin_gradient(const dsgd_oracle_csr *a, int32_t model, int32_t weighting, double lambda, const double *d,
                                const double *w, const int32_t *idx, int64_t n, double w_pos, double w_neg, const double *sw,
                                int32_t do_regularize, double *grad_out, double *loss_out, double *s_out) {
  int rc = bad_args(a, model, weighting, idx, 0, n);
  if (rc || !idx) return rc ? rc : -3;
  double c, nrm2;
  pass_totals o;
  scalars(w, d, a->dim, lambda, &c, &nrm2);
  memset(grad_out, 0, sizeof(double) * (size_t)a->dim);
  pass_rows(a, model, weighting, w, idx, 0, n, w_pos, w_neg, sw, grad_out, &o);
  if (do_regularize) regularize(grad_out, a->dim, c);
  if (loss_out) *loss_out = lambda * nrm2 + o.s / (double)n;
  if (s_out) *s_out = o.s;
  return 0;
}

int dsgd_oracle_margin_eval(const dsgd_oracle_csr *a, int32_t model, int32_t weighting, const double *w, const int32_t *idx,
                            int64_t n, double w_pos, double w_neg, const double *sw, double *sums_out, int64_t *counts_out) {
  int rc = bad_args(a, model, weighting, idx, 0, n);
  if (rc || !idx || weighting == 0) return rc ? rc : -3;
  pass_totals o;
  pass_rows(a, model, weighting, w, idx, 0, n, w_pos, w_neg, sw, NULL, &o);
  if (weighting == 1) {
    sums_out[0] = o.cls[0]; sums_out[1] = o.cls[1];
    counts_out[0] = o.cls_ok[0]; counts_out[1] = o.cls_ok[1]; counts_out[2] = o.cls_n[0]; counts_out[3] = o.cls_n[1];
  } else {
    sums_out[0] = o.s; sums_out[1] = o.ok_w; sums_out[2] = o.all_w;
    counts_out[0] = n; counts_out[1] = o.correct;
  }
  return 0;
}

int dsgd_oracle_margin_sync_steps(const dsgd_oracle_csr *a, int32_t model, int32_t weighting, double lambda, double lambda1,
                                  const double *d, double *w, const int32_t *idx, const int32_t *counts, int32_t n_workers,
                                  const double *lrs, int64_t n_steps, double w_pos, double w_neg, const double *sw,
                                  double *losses_out, double *avg_sum) {
  if (n_workers <= 0) return -3;
  int64_t per_step = 0;
  for (int32_t k = 0; k < n_workers; ++k) {
    if (counts[k] <= 0) return -3;
    per_step += counts[k];
  }
  int rc = bad_args(a, model, weighting, idx, 0, per_step * n_steps);
  if (rc) return rc;
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
      pass_totals o;
      memset(g, 0, sizeof(double) * (size_t)dim);
      pass_rows(a, model, weighting, w, step + off, 0, counts[k], w_pos, w_neg, sw, g, &o);
      regularize(g, dim, c);
      h = k == 0 ? o.s : h + o.s;
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
