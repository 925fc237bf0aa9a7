/*
 * TEST INFRASTRUCTURE ONLY -- the primitives every checker of libdsgd_oracle.so shares, written once: the reference's 1e-20
 * filter, the row dot, the logistic loss and its derivative, the device's fixed-point sum and a compensated long-double sum.
 * Everything here is static inline; the header exports nothing.
 */
#ifndef DSGD_ORACLE_COMMON_H
#define DSGD_ORACLE_COMMON_H

#include <math.h>
#include <stdint.h>

#include "dsgd_oracle.h"

#define EPS 1e-20 /* math/Sparse.scala:104 */

static inline double filt(double v) { return fabs(v) > EPS ? v : 0.0; }

/* x . w  = (x * w).sum  (math/Vec.scala:58; math/Sparse.scala:46,20-31): the product map is built first, which drops
 * products with |x_j w_j| <= 1e-20, then folded; the row itself is a Sparse, so its tiny entries are absent.  Fold order
 * here is index order (the reference's is HashMap order, not reproducible without a JVM -- SURVEY.md 2.3). */
static inline double row_dot(const dsgd_oracle_csr *a, int64_t r, const double *w) {
  double s = 0.0;
  for (int64_t p = a->row_ptr[r]; p < a->row_ptr[r + 1]; ++p) s += filt(filt((double)a->val[p]) * w[a->col[p]]);
  return s;
}

/* softplus(z) = log(1 + e^z) and sigmoid(t) = 1 / (1 + e^-t), in their stable forms */
static inline double softplus(double z) { return (z > 0.0 ? z : 0.0) + log1p(exp(-fabs(z))); }
static inline double sigmoid(double t) {
  if (t >= 0.0) return 1.0 / (1.0 + exp(-t));
  const double e = exp(t);
  return e / (1.0 + e);
}

/* The device's fixed-point sum (csrc/dsgd_fixed.cuh): every term v is rounded to R(v) = rint(v 2^160) 2^-160 and added
 * exactly as an integer in six 40-bit limbs, limb k worth 2^(40 k - 160), limbs 0..4 carried into [0, 2^40), the top one
 * unbounded.  A term that is NaN, infinite, negative or 2^52 or more is counted in ovf, and the sum then reads NaN.  The
 * carry shifts arithmetically, so a difference of two sums carries its negative limbs too. */
typedef struct {
  uint64_t l[6];
  uint64_t ovf;
} fxsum;

static inline void fx_carry(fxsum *s) {
  for (int k = 0; k < 5; ++k) {
    s->l[k + 1] += (uint64_t)((int64_t)s->l[k] >> 40);
    s->l[k] &= (1ull << 40) - 1;
  }
}

static inline void fx_add(fxsum *s, double v) {
  if (!(v >= 0.0 && v < 0x1p52)) { ++s->ovf; return; }
  double F[4];   /* F_i = floor(v 2^(40 i)), exact */
  for (int i = 0; i < 4; ++i) F[i] = floor(ldexp(v, 40 * i));
  s->l[4] += (uint64_t)F[0];
  for (int i = 1; i < 4; ++i) s->l[4 - i] += (uint64_t)(F[i] - F[i - 1] * 0x1p40);
  s->l[0] += (uint64_t)(rint(ldexp(v, 160)) - F[3] * 0x1p40);   /* the one rounding: to 2^-160, ties to even */
  fx_carry(s);
}

/* read(): the carried limbs converted from the top limb down, as the device's acc_value */
static inline double fx_read(fxsum s) {
  if (s.ovf) return NAN;
  fx_carry(&s);
  double r = (double)s.l[5] * 0x1p40;
  for (int k = 4; k >= 0; --k) r += (double)s.l[k] * ldexp(1.0, 40 * k - 160);
  return r;
}

/* Neumaier's compensated sum carried in long double (64-bit significand on x86-64): math.fsum quality for these sizes, the
 * error far below one ulp of a double before the final rounding.  A term that is NaN, infinite or of magnitude 2^52 or more
 * makes the sum read NaN. */
typedef struct {
  long double s, c;
  int bad;
} ksum;

static inline void k_add(ksum *k, double v) {
  if (!(fabs(v) < 0x1p52)) { k->bad = 1; return; }
  const long double x = (long double)v, t = k->s + x;
  if (fabsl(k->s) >= fabsl(x)) k->c += (k->s - t) + x;
  else k->c += (x - t) + k->s;
  k->s = t;
}

static inline double k_val(const ksum *k) { return k->bad ? NAN : (double)(k->s + k->c); }

#endif
