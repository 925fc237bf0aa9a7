/*
 * TEST INFRASTRUCTURE ONLY -- fp64 CPU restatement of the isotonic calibration calls of include/dsgd.h
 * (dsgd_calibrate_isotonic*, dsgd_isotonic_probabilities, dsgd_eval_isotonic_calibration*) over an array of margins
 * f = x . w and labels.  Written from the header and DESIGN.md §4.16; it shares no code with the library.
 * The fit is the sequential algorithm: qsort of the scores s = -f, one pass over the distinct scores for the points, and
 * Andrew's monotone chain over them in int64.  Apply is numpy.interp's arithmetic.  The quality pass cuts every Brier term
 * and every p into the library's fixed-point limbs (resolution 2^-160) and converts the integer sums from the top limb
 * down, so those sums are the library's bit for bit; the log-loss sum is Neumaier-compensated in long double.
 */
#include <stdlib.h>

#include "dsgd_oracle_common.h"   /* fxsum, ksum */

typedef struct { double s; int8_t y; } srow;

/* descending score; +0 and -0 compare equal */
static int by_score_desc(const void *a, const void *b) {
  const double x = ((const srow *)a)->s, z = ((const srow *)b)->s;
  return (x < z) - (x > z);
}

static int64_t cross(int64_t ox, int64_t oy, int64_t ax, int64_t ay, int64_t bx, int64_t by) {
  return (ax - ox) * (by - oy) - (ay - oy) * (bx - ox);
}

/* The fit.  Outputs as the library's: X, Y ascending (n_points_out entries), block rows / positives ascending,
 * info = {blocks, points, rows used, NaN rows, distinct scores}.  Returns 0, or -3 when no row has a non-NaN score. */
int dsgd_oracle_iso_fit(const double *f, const int8_t *y, int64_t n, int64_t *n_points_out, double *X, double *Y,
                        int64_t *rows_out, int64_t *pos_out, int64_t *info) {
  srow *r = malloc(sizeof(srow) * (size_t)(n > 0 ? n : 1));
  int64_t used = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (isnan(f[i])) continue;
    const double s = -f[i];
    r[used].s = s == 0.0 ? 0.0 : s;
    r[used].y = y[i] > 0;
    ++used;
  }
  if (used == 0) { free(r); return -3; }
  qsort(r, (size_t)used, sizeof(srow), by_score_desc);
  /* point i: the origin (i = 0) or distinct score i - 1 with the rows at or above it */
  double *thr = malloc(sizeof(double) * (size_t)used);
  int64_t *px = malloc(sizeof(int64_t) * (size_t)(used + 1)), *py = malloc(sizeof(int64_t) * (size_t)(used + 1));
  int64_t m = 0, tp = 0, all = 0;
  px[0] = py[0] = 0;
  for (int64_t i = 0; i < used; ++i) {
    tp += r[i].y;
    ++all;
    if (i + 1 == used || r[i + 1].s != r[i].s) {
      thr[m] = r[i].s;
      ++m;
      px[m] = all;
      py[m] = tp;
    }
  }
  int64_t *h = malloc(sizeof(int64_t) * (size_t)(m + 1)), top = 0;
  for (int64_t i = 0; i <= m; ++i) {
    while (top >= 2 && cross(px[h[top - 2]], py[h[top - 2]], px[h[top - 1]], py[h[top - 1]], px[i], py[i]) >= 0) --top;
    h[top++] = i;
  }
  const int64_t B = top - 1;
  int64_t k = 0;
  for (int64_t o = 0; o < B; ++o) {   /* ascending score: the hull's segments from the last */
    const int64_t b = B - 1 - o, i0 = h[b], i1 = h[b + 1];
    const int64_t rows = px[i1] - px[i0], pos = py[i1] - py[i0];
    const double p = (double)pos / (double)rows;
    rows_out[o] = rows;
    pos_out[o] = pos;
    X[k] = thr[i1 - 1];
    Y[k++] = p;
    if (i1 - i0 >= 2) {
      X[k] = thr[i0];
      Y[k++] = p;
    }
  }
  *n_points_out = k;
  info[0] = B;
  info[1] = k;
  info[2] = used;
  info[3] = n - used;
  info[4] = m;
  free(h); free(px); free(py); free(thr); free(r);
  return 0;
}

/* numpy.interp(s, X, Y) for k >= 2, and the header's NaN rule for every k */
static double interp(double s, const double *X, const double *Y, int64_t k) {
  if (isnan(s)) return s;
  if (s <= X[0]) return Y[0];
  if (s >= X[k - 1]) return Y[k - 1];
  int64_t lo = 0, hi = k - 1;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) / 2;
    if (X[mid] <= s) lo = mid; else hi = mid;
  }
  if (X[lo] == s) return Y[lo];
  const double slope = (Y[lo + 1] - Y[lo]) / (X[lo + 1] - X[lo]);
  double v = slope * (s - X[lo]) + Y[lo];
  if (isnan(v)) {
    v = slope * (s - X[lo + 1]) + Y[lo + 1];
    if (isnan(v) && Y[lo] == Y[lo + 1]) v = Y[lo];
  }
  return v;
}

/* out[i] = interp(-f[i]) */
void dsgd_oracle_iso_probs(const double *f, int64_t n, const double *X, const double *Y, int64_t k, double *out) {
  for (int64_t i = 0; i < n; ++i) out[i] = interp(-f[i], X, Y, k);
}

/* The quality pass: sums_out = {Brier sum, log-loss sum over the finite terms}; per bin rows, positives and sum p;
 * words_out = {rows used, rows left out, rows with an infinite term}. */
void dsgd_oracle_iso_quality(const double *f, const int8_t *y, int64_t n, const double *X, const double *Y, int64_t k,
                             int32_t n_bins, double *sums_out, int64_t *bin_rows, int64_t *bin_pos, double *bin_psum,
                             int64_t *words_out) {
  fxsum brier = {{0}, 0}, ps[64];
  ksum ll = {0, 0, 0};
  for (int b = 0; b < n_bins; ++b) { bin_rows[b] = bin_pos[b] = 0; ps[b] = brier; }
  int64_t used = 0, out = 0, inf = 0;
  for (int64_t i = 0; i < n; ++i) {
    const double s = -f[i];
    if (isnan(s)) { ++out; continue; }
    const int pos = y[i] > 0;
    const double p = interp(s, X, Y, k), o = pos ? 1.0 : 0.0, d = p - o;
    ++used;
    fx_add(&brier, d * d);
    const double term = pos ? -log(p) : -log1p(-p);
    if (isinf(term)) ++inf; else k_add(&ll, term);
    int b = (int)floor(p * (double)n_bins);
    b = b < n_bins - 1 ? b : n_bins - 1;
    ++bin_rows[b];
    bin_pos[b] += pos;
    fx_add(&ps[b], p);
  }
  sums_out[0] = fx_read(brier);
  sums_out[1] = k_val(&ll);
  for (int b = 0; b < n_bins; ++b) bin_psum[b] = fx_read(ps[b]);
  words_out[0] = used;
  words_out[1] = out;
  words_out[2] = inf;
}
