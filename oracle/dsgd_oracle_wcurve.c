/*
 * TEST INFRASTRUCTURE ONLY -- fp64 CPU restatement of the weighted curves of include/dsgd.h (dsgd_eval_*weighted_curve),
 * the checker of tests/test_gpu_weighted_curve.py.  It takes the rows' margins (the device's own, from dsgd_margins), their
 * labels and their weights c_i, and returns the metrics words, the DSGD_WCURVE_WORDS weighted words and the points.
 *
 * Every weight is an exact sum of R(c) = rint(c * 2^160) * 2^-160, kept in six 40-bit limbs and an overflow count as the
 * device keeps it (csrc/dsgd_fixed.cuh), and read() converts an exact sum as acc_value does: limbs carried, then converted
 * from the top limb down.  The walk is not the device's: the rows are sorted by score, highest first, and walked one tie
 * group at a time with running sums of the groups above (as dsgd_oracle_curve.c walks), so W+(>= t) and W-(>= t) are
 * running totals here where the device reads them as differences of prefix sums.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define LIMBS 6
#define LIMB_MASK ((1ull << 40) - 1)

typedef struct {
  uint64_t l[LIMBS];
  uint64_t ovf;
} lsum;

/* the limbs are carried into [0, 2^40) for limbs 0..4, signed: a difference of two sums may hold negative limbs */
static void carry(lsum *s) {
  for (int k = 0; k < LIMBS - 1; ++k) {
    s->l[k + 1] += (uint64_t)((int64_t)s->l[k] >> 40);
    s->l[k] &= LIMB_MASK;
  }
}

/* s += R(v): the cut of acc_cut (limbs 4..1 from floors of v * 2^(40 i), limb 0 rounded at 2^-160); v NaN, infinite,
 * negative or 2^52 or more is counted in ovf and the sum reads NaN */
static void add_r(lsum *s, double v) {
  if (!(v >= 0.0 && v < 4503599627370496.0)) { ++s->ovf; return; }
  double F[4];
  for (int i = 0; i < 4; ++i) F[i] = floor(v * ldexp(1.0, 40 * i));
  s->l[4] += (uint64_t)(int64_t)F[0];
  for (int i = 1; i < 4; ++i) s->l[4 - i] += (uint64_t)(int64_t)(F[i] - F[i - 1] * 0x1p40);
  s->l[0] += (uint64_t)(int64_t)(rint(v * 0x1p160) - F[3] * 0x1p40);
  carry(s);
}

static lsum plus(lsum a, lsum b) {
  for (int k = 0; k < LIMBS; ++k) a.l[k] += b.l[k];
  a.ovf += b.ovf;
  carry(&a);
  return a;
}

static lsum minus(lsum a, lsum b) {
  for (int k = 0; k < LIMBS; ++k) a.l[k] -= b.l[k];
  a.ovf -= b.ovf;
  carry(&a);
  return a;
}

/* read(): acc_value of the carried limbs */
static double read_sum(lsum s) {
  if (s.ovf) return NAN;
  carry(&s);
  double r = (double)s.l[LIMBS - 1] * 0x1p40;
  for (int k = LIMBS - 2; k >= 0; --k) r += (double)s.l[k] * ldexp(1.0, 40 * k - 160);
  return r;
}

/* read() of the exact sum of R(v[i]) over i < n: the reader the device's acc_value computes */
double dsgd_oracle_wcurve_read(const double *v, int64_t n) {
  lsum s;
  memset(&s, 0, sizeof s);
  for (int64_t i = 0; i < n; ++i) add_r(&s, v[i]);
  return read_sum(s);
}

typedef struct {
  double s, c;
  int pos;
} wrow;

static int cmp_desc(const void *x, const void *y) {
  const double a = ((const wrow *)x)->s, b = ((const wrow *)y)->s;
  return (a < b) - (a > b); /* highest score first; -0 == +0: one score */
}

/* Rows i < n with margin margins[i], label label[i] (> 0: positive) and weight c[i]; s = -margin.  words[0..7]: the
 * metrics words of dsgd_eval_metrics (counts and U2); wsums[0..12]: the DSGD_WCURVE_WORDS words of include/dsgd.h; the
 * points thr[k] (a zero score as +0), tpw[k] = W+(>= thr[k]), fpw[k] = W-(>= thr[k]), highest score first, and
 * *n_points of them (thr == NULL: no points).  Every output array of points holds n entries.  Returns 0, -1 (allocation)
 * or -3 (n <= 0). */
int dsgd_oracle_wcurve(const double *margins, const int8_t *label, const double *c, int64_t n, int64_t *words,
                       double *wsums, int64_t *n_points, double *thr, double *tpw, double *fpw) {
  if (n <= 0) return -3;
  wrow *r = malloc(sizeof(wrow) * (size_t)n);
  if (!r) return -1;
  lsum z, tp, fn, pnone, fp, tn, nnone, nan_w, correct, all, wp, wn, u2w, sap, tot_n;
  memset(&z, 0, sizeof z);
  tp = fn = pnone = fp = tn = nnone = nan_w = correct = all = wp = wn = u2w = sap = tot_n = z;
  int64_t cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0}, k = 0;
  /* the confusion words, row by row: pred +1 when x.w < 0 (s > 0), -1 when x.w > 0, none when x.w is 0 or NaN */
  for (int64_t i = 0; i < n; ++i) {
    const double m = margins[i], ci = c[i];
    const int pos = label[i] > 0, nan = m != m;
    const int pred = m < 0.0 ? 1 : m > 0.0 ? -1 : 0;
    lsum *cell = pos ? (pred == 1 ? &tp : pred == -1 ? &fn : &pnone) : (pred == 1 ? &fp : pred == -1 ? &tn : &nnone);
    ++cnt[pos ? (pred == 1 ? 0 : pred == -1 ? 1 : 2) : (pred == 1 ? 3 : pred == -1 ? 4 : 5)];
    add_r(cell, ci);
    add_r(&all, ci);
    add_r(pos ? &wp : &wn, ci);
    if ((pos && pred == 1) || (!pos && pred == -1)) add_r(&correct, ci);
    if (nan) {
      ++cnt[7];
      add_r(&nan_w, ci);
      continue;
    }
    if (!pos) add_r(&tot_n, ci);
    r[k].s = m == 0.0 ? 0.0 : -m;
    r[k].c = ci;
    r[k].pos = pos;
    ++k;
  }
  qsort(r, (size_t)k, sizeof(wrow), cmp_desc);
  /* one tie group at a time, highest score first; above_p / above_n: W+(> t), W-(> t); n_above: negatives above (counts) */
  lsum above_p = z, above_n = z;
  int64_t pts = 0, n_above = 0, n_neg = 0, u2 = 0;
  for (int64_t i = 0; i < k; ++i) n_neg += !r[i].pos;
  for (int64_t i = 0; i < k;) {
    int64_t j = i, gneg = 0;
    lsum gp = z, gn = z;
    for (; j < k && r[j].s == r[i].s; ++j) {
      add_r(r[j].pos ? &gp : &gn, r[j].c);
      gneg += !r[j].pos;
    }
    const lsum t_sum = plus(above_p, gp), f_sum = plus(above_n, gn);
    const lsum below_n = minus(tot_n, f_sum);   /* W-(< t) */
    const double b = read_sum(plus(plus(below_n, below_n), gn));
    const double t = read_sum(t_sum), f = read_sum(f_sum);
    const int64_t n_below = n_neg - n_above - gneg;
    for (int64_t g = i; g < j; ++g) {
      if (!r[g].pos) continue;
      u2 += 2 * n_below + gneg;
      add_r(&u2w, r[g].c * b);
      if (r[g].c > 0.0) add_r(&sap, r[g].c * (t / (t + f)));
    }
    if (thr) {
      thr[pts] = r[i].s;
      tpw[pts] = t;
      fpw[pts] = f;
    }
    ++pts;
    above_p = t_sum;
    above_n = f_sum;
    n_above += gneg;
    i = j;
  }
  for (int w = 0; w < 8; ++w) words[w] = cnt[w];
  words[6] = u2;
  const lsum w_out[13] = {tp, fn, pnone, fp, tn, nnone, u2w, nan_w, sap, correct, all, wp, wn};
  for (int w = 0; w < 13; ++w) wsums[w] = read_sum(w_out[w]);
  *n_points = pts;
  free(r);
  return 0;
}
