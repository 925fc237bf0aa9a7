/*
 * TEST INFRASTRUCTURE ONLY -- fp64 CPU restatement of the calibration calls of include/dsgd.h (dsgd_calibrate*,
 * dsgd_eval_calibration*) over an array of scores f = x . w and labels: Platt scaling as Lin, Lin and Weng (2007) state it,
 * and the quality sums and bins.  Written from the paper and from DESIGN.md §4.11; it shares no code with the library.
 * Every term is computed in fp64 with libm's exp / log1p; every sum over the rows is a Neumaier-compensated sum carried in
 * long double (64-bit significand on x86-64), which is math.fsum quality for these sizes: the error of a sum is far below one
 * ulp of a double before the final rounding.  Rows whose score is NaN are skipped.
 */
#include "dsgd_oracle_common.h"   /* sigmoid, softplus, ksum */

/* out6 = {F, dF/dA, dF/dB, H_AA, H_AB, H_BB} at (a, b), without the ridge */
void dsgd_oracle_calib_sums(const double *f, const int8_t *y, int64_t n, double t_pos, double t_neg, double a, double b,
                            double *out6) {
  ksum k[6] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int64_t i = 0; i < n; ++i) {
    if (isnan(f[i])) continue;
    const double t = y[i] > 0 ? t_pos : t_neg, z = a * f[i] + b;
    double term, p, q;
    if (z >= 0.0) {
      const double e = exp(-z), den = 1.0 + e;
      term = t * z + log1p(e);
      p = e / den;
      q = 1.0 / den;
    } else {
      const double e = exp(z), den = 1.0 + e;
      term = (t - 1.0) * z + log1p(e);
      p = 1.0 / den;
      q = e / den;
    }
    const double d1 = t - p, d2 = p * q;
    k_add(&k[0], term);
    k_add(&k[1], f[i] * d1);
    k_add(&k[2], d1);
    k_add(&k[3], (f[i] * f[i]) * d2);
    k_add(&k[4], f[i] * d2);
    k_add(&k[5], d2);
  }
  for (int j = 0; j < 6; ++j) out6[j] = k_val(&k[j]);
}

static int all_finite(const double *S) {
  int ok = 1;
  for (int j = 0; j < 6; ++j) ok &= isfinite(S[j]) != 0;
  return ok;
}

/* The fit.  ab_out = {A, B}; info_out = {iterations, status, rows used, NaN rows, points evaluated}; returns 0, or -9 when a
 * class is missing among the rows with a score (DSGD_ERR_EMPTY). */
int dsgd_oracle_calib_fit(const double *f, const int8_t *y, int64_t n, double *ab_out, double *objective_out, int64_t *info_out) {
  int64_t n_pos = 0, n_neg = 0, n_nan = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (isnan(f[i])) ++n_nan;
    else if (y[i] > 0) ++n_pos;
    else ++n_neg;
  }
  if (n_pos == 0 || n_neg == 0) return -9;
  const double t_pos = ((double)n_pos + 1.0) / ((double)n_pos + 2.0), t_neg = 1.0 / ((double)n_neg + 2.0);
  double A = 0.0, B = log(((double)n_neg + 1.0) / ((double)n_pos + 1.0)), F, S[6];
  int64_t iter = 0, status = 0, evals = 1;
  dsgd_oracle_calib_sums(f, y, n, t_pos, t_neg, A, B, S);
  F = S[0];
  for (;;) {
    if (!all_finite(S)) { status = 3; A = B = F = NAN; break; }
    const double g1 = S[1], g2 = S[2], h11 = S[3] + 1e-12, h21 = S[4], h22 = S[5] + 1e-12;
    if (fabs(g1) < 1e-5 && fabs(g2) < 1e-5) { status = 0; break; }
    if (iter >= 100) { status = 1; break; }
    const double det = h11 * h22 - h21 * h21;
    const double dA = -(h22 * g1 - h21 * g2) / det, dB = -(h11 * g2 - h21 * g1) / det, gd = g1 * dA + g2 * dB;
    double step = 1.0;
    int moved = 0;
    while (step >= 1e-10) {
      const double na = A + step * dA, nb = B + step * dB;
      dsgd_oracle_calib_sums(f, y, n, t_pos, t_neg, na, nb, S);
      ++evals;
      if (!all_finite(S)) break;                          /* the outer test reports it */
      if (S[0] < F + 1e-4 * step * gd) { A = na; B = nb; F = S[0]; moved = 1; break; }
      step = step / 2.0;
    }
    if (!moved) {
      if (all_finite(S)) { status = 2; break; }
      continue;                                          /* non-finite: S is tested at the loop's head */
    }
    ++iter;
  }
  ab_out[0] = A; ab_out[1] = B; *objective_out = F;
  info_out[0] = iter; info_out[1] = status; info_out[2] = n_pos + n_neg; info_out[3] = n_nan; info_out[4] = evals;
  return 0;
}

/* p_out[i] = sigmoid(-(a f_i + b)) (NaN for a NaN z) */
void dsgd_oracle_calib_probs(const double *f, int64_t n, double a, double b, double *p_out) {
  for (int64_t i = 0; i < n; ++i) p_out[i] = sigmoid(-(a * f[i] + b));
}

/* The quality pass: sums_out = {Brier sum, log-loss sum}; per bin rows, positives and sum p; words_out = {rows used, rows
 * left out}; *edge_rows_out = rows whose p * n_bins lies within 4 ulp of an integer (a different exp could bin them
 * elsewhere). */
void dsgd_oracle_calib_quality(const double *f, const int8_t *y, int64_t n, double a, double b, int32_t n_bins, double *sums_out,
                               int64_t *bin_rows, int64_t *bin_pos, double *bin_psum, int64_t *words_out, int64_t *edge_rows_out) {
  ksum brier = {0, 0, 0}, ll = {0, 0, 0}, ps[64];
  for (int k = 0; k < n_bins; ++k) { bin_rows[k] = bin_pos[k] = 0; ps[k].s = ps[k].c = 0; ps[k].bad = 0; }
  int64_t used = 0, out = 0, edge = 0;
  for (int64_t i = 0; i < n; ++i) {
    const double z = a * f[i] + b;
    if (isnan(z)) { ++out; continue; }
    const int pos = y[i] > 0;
    const double p = sigmoid(-z), d = p - (pos ? 1.0 : 0.0), s = p * (double)n_bins;
    ++used;
    k_add(&brier, d * d);
    k_add(&ll, softplus(pos ? z : -z));
    int k = (int)floor(s);
    if (k > n_bins - 1) k = n_bins - 1;
    const double r = rint(s);
    if (r >= 1.0 && r <= (double)(n_bins - 1) && fabs(s - r) <= 4.0 * 0x1p-52 * r) ++edge;
    ++bin_rows[k];
    bin_pos[k] += pos;
    k_add(&ps[k], p);
  }
  sums_out[0] = k_val(&brier); sums_out[1] = k_val(&ll);
  for (int k = 0; k < n_bins; ++k) bin_psum[k] = k_val(&ps[k]);
  words_out[0] = used; words_out[1] = out;
  *edge_rows_out = edge;
}
