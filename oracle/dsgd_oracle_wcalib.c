/*
 * TEST INFRASTRUCTURE ONLY -- fp64 CPU restatement of the weighted calibration calls of include/dsgd.h
 * (dsgd_calibrate_weighted*, dsgd_eval_*weighted_calibration) over an array of scores f = x . w, labels and row weights c:
 * Platt scaling with every row counted by its weight, and the weighted quality sums and bins.  Written from DESIGN.md §4.17
 * and §4.14; it shares no code with the library.
 *   - R(v) = rint(v 2^160) 2^-160 and read() are restated here: an exact sum of R values is kept as one integer in six
 *     40-bit limbs (the top one unbounded) and converted from the top limb down, so every weighted total -- W+, W-, the NaN
 *     rows' weight and every quality sum -- has the library's bits.
 *   - The six sums of the fit are Neumaier-compensated sums of fl(c term) carried in long double (as the unweighted checker
 *     sums its terms), so the fit agrees with the library to the fit's tolerances, not bit for bit.
 * A row with R(c) = 0 adds nothing and forms no term; a NaN score leaves the row out.
 */
#include <math.h>
#include <stdint.h>

/* ---- exact sums of R(v), v in [0, 2^52) ------------------------------------------------------------------------------- */
typedef struct { uint64_t l[6]; uint64_t ovf; } rsum;
static const uint64_t kMask = (1ull << 40) - 1;
static void r_carry(uint64_t *q) {
  for (int i = 0; i < 5; ++i) { q[i + 1] += q[i] >> 40; q[i] &= kMask; }
}
static void r_add(rsum *s, double v) {
  if (!(v >= 0.0 && v < 0x1p52)) { ++s->ovf; return; }
  double F[4];
  for (int i = 0; i < 4; ++i) F[i] = floor(v * ldexp(1.0, 40 * i));
  s->l[4] += (uint64_t)F[0];
  for (int i = 1; i < 4; ++i) s->l[4 - i] += (uint64_t)(F[i] - F[i - 1] * 0x1p40);
  s->l[0] += (uint64_t)(rint(v * 0x1p160) - F[3] * 0x1p40);
  r_carry(s->l);
}
static double r_read(const rsum *s) {
  if (s->ovf) return NAN;
  uint64_t q[6];
  for (int i = 0; i < 6; ++i) q[i] = s->l[i];
  r_carry(q);
  double x = (double)q[5] * 0x1p40;
  for (int i = 4; i >= 0; --i) x += (double)q[i] * ldexp(1.0, 40 * i - 160);
  return x;
}
static int r_zero(double c) { return rint(c * 0x1p160) == 0.0; }

/* ---- Neumaier sums in long double -------------------------------------------------------------------------------------- */
typedef struct { long double s, c; int bad; } ksum;
static void k_add(ksum *k, double v) {
  if (!(fabs(v) < 0x1p52)) { k->bad = 1; return; }
  const long double x = (long double)v, t = k->s + x;
  if (fabsl(k->s) >= fabsl(x)) k->c += (k->s - t) + x;
  else k->c += (x - t) + k->s;
  k->s = t;
}
static double k_val(const ksum *k) { return k->bad ? NAN : (double)(k->s + k->c); }

/* out6 = {F, dF/dA, dF/dB, H_AA, H_AB, H_BB} at (a, b), each a sum of fl(c term), without the ridge */
void dsgd_oracle_wcalib_sums(const double *f, const int8_t *y, const double *c, int64_t n, double t_pos, double t_neg,
                             double a, double b, double *out6) {
  ksum k[6] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int64_t i = 0; i < n; ++i) {
    if (isnan(f[i]) || r_zero(c[i])) continue;
    const double t = y[i] > 0 ? t_pos : t_neg, z = a * f[i] + b, ci = c[i];
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
    k_add(&k[0], ci * term);
    k_add(&k[1], ci * (f[i] * d1));
    k_add(&k[2], ci * d1);
    k_add(&k[3], ci * ((f[i] * f[i]) * d2));
    k_add(&k[4], ci * (f[i] * d2));
    k_add(&k[5], ci * d2);
  }
  for (int j = 0; j < 6; ++j) out6[j] = k_val(&k[j]);
}

/* wsums_out = {W+, W-, NaN rows' weight}; targets_out = {t+, t-, B0} */
void dsgd_oracle_wcalib_targets(const double *f, const int8_t *y, const double *c, int64_t n, double *wsums_out,
                                double *targets_out) {
  rsum wp = {{0}, 0}, wn = {{0}, 0}, wnan = {{0}, 0};
  for (int64_t i = 0; i < n; ++i) r_add(isnan(f[i]) ? &wnan : y[i] > 0 ? &wp : &wn, c[i]);
  const double p = r_read(&wp), q = r_read(&wn);
  wsums_out[0] = p; wsums_out[1] = q; wsums_out[2] = r_read(&wnan);
  targets_out[0] = (p + 1.0) / (p + 2.0);
  targets_out[1] = 1.0 / (q + 2.0);
  targets_out[2] = log((q + 1.0) / (p + 1.0));
}

static int all_finite(const double *S) {
  int ok = 1;
  for (int j = 0; j < 6; ++j) ok &= isfinite(S[j]) != 0;
  return ok;
}

/* The weighted fit.  ab_out = {A, B}; info_out = {iterations, status, rows used, NaN rows, points evaluated};
 * wsums_out = {W+, W-, NaN rows' weight}.  Returns 0, or -3 (DSGD_ERR_EMPTY) when W+ or W- is 0 (wsums_out set). */
int dsgd_oracle_wcalib_fit(const double *f, const int8_t *y, const double *c, int64_t n, double *ab_out, double *objective_out,
                           int64_t *info_out, double *wsums_out) {
  double tg[3], S[6];
  dsgd_oracle_wcalib_targets(f, y, c, n, wsums_out, tg);
  if (wsums_out[0] == 0.0 || wsums_out[1] == 0.0) return -3;
  int64_t n_rows = 0, n_nan = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (isnan(f[i])) ++n_nan;
    else ++n_rows;
  }
  const double t_pos = tg[0], t_neg = tg[1];
  double A = 0.0, B = tg[2], F;
  int64_t iter = 0, status = 0, evals = 1;
  dsgd_oracle_wcalib_sums(f, y, c, n, t_pos, t_neg, A, B, S);
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
      dsgd_oracle_wcalib_sums(f, y, c, n, t_pos, t_neg, na, nb, S);
      ++evals;
      if (!all_finite(S)) break;
      if (S[0] < F + 1e-4 * step * gd) { A = na; B = nb; F = S[0]; moved = 1; break; }
      step = step / 2.0;
    }
    if (!moved) {
      if (all_finite(S)) { status = 2; break; }
      continue;
    }
    ++iter;
  }
  ab_out[0] = A; ab_out[1] = B; *objective_out = F;
  info_out[0] = iter; info_out[1] = status; info_out[2] = n_rows; info_out[3] = n_nan; info_out[4] = evals;
  return 0;
}

static double sigmoid(double t) {
  if (t >= 0.0) return 1.0 / (1.0 + exp(-t));
  const double e = exp(t);
  return e / (1.0 + e);
}
static double softplus(double z) { return (z > 0.0 ? z : 0.0) + log1p(exp(-fabs(z))); }

/* The weighted quality pass: sums_out = {sum R(c (p - o)^2), sum R(c l), sum R(c), 0}; per bin sum R(c), the same over the
 * positives and sum R(c p) (a bin value of 2^52 or more makes that bin's three sums NaN); words_out = {rows used, rows left
 * out}; *edge_rows_out = rows of positive weight whose p * n_bins lies within 4 ulp of an integer. */
void dsgd_oracle_wcalib_quality(const double *f, const int8_t *y, const double *c, int64_t n, double a, double b,
                                int32_t n_bins, double *sums_out, double *bin_weight, double *bin_pos_weight,
                                double *bin_psum, int64_t *words_out, int64_t *edge_rows_out) {
  rsum brier = {{0}, 0}, ll = {{0}, 0}, wt = {{0}, 0}, bw[64], bp[64], bs[64];
  for (int k = 0; k < n_bins; ++k) {
    bw[k] = (rsum){{0}, 0};
    bp[k] = (rsum){{0}, 0};
    bs[k] = (rsum){{0}, 0};
  }
  int64_t used = 0, out = 0, edge = 0;
  for (int64_t i = 0; i < n; ++i) {
    const double z = a * f[i] + b;
    if (isnan(z)) { ++out; continue; }
    ++used;
    const double ci = c[i];
    if (r_zero(ci)) continue;
    const int pos = y[i] > 0;
    const double p = sigmoid(-z), d = p - (pos ? 1.0 : 0.0), s = p * (double)n_bins;
    r_add(&brier, ci * (d * d));
    r_add(&ll, ci * softplus(pos ? z : -z));
    r_add(&wt, ci);
    int k = (int)floor(s);
    if (k > n_bins - 1) k = n_bins - 1;
    const double r = rint(s);
    if (r >= 1.0 && r <= (double)(n_bins - 1) && fabs(s - r) <= 4.0 * 0x1p-52 * r) ++edge;
    const double vs[3] = {ci, ci, ci * p};
    int bad = 0;
    for (int j = 0; j < 3; ++j) bad |= !(vs[j] < 0x1p52);
    if (bad) { ++bw[k].ovf; ++bp[k].ovf; ++bs[k].ovf; continue; }
    r_add(&bw[k], ci);
    if (pos) r_add(&bp[k], ci);
    r_add(&bs[k], ci * p);
  }
  sums_out[0] = r_read(&brier); sums_out[1] = r_read(&ll); sums_out[2] = r_read(&wt); sums_out[3] = 0.0;
  for (int k = 0; k < n_bins; ++k) {
    bin_weight[k] = r_read(&bw[k]);
    bin_pos_weight[k] = r_read(&bp[k]);
    bin_psum[k] = r_read(&bs[k]);
  }
  words_out[0] = used; words_out[1] = out;
  *edge_rows_out = edge;
}
