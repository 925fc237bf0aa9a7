/*
 * TEST INFRASTRUCTURE ONLY -- fp64, array-based CPU restatement of the sample-weighted gradient, evaluation and sync step
 * (DESIGN.md section 4.13), for SparseSVM and SparseLogistic.  Conventions are those of dsgd_oracle.h (same CSR struct, dense
 * vectors with 0.0 for "key absent", the 1e-20 filter wherever the reference builds a new Sparse).  It is validated against
 * the literal restatement in oracle/sw.py and against oracle/dsgd_oracle_cw.c at sample weights 1.
 *
 * Row i of label y has the combined weight c_i = fl(w_y * s_i) (w_pos for y = +1, w_neg for y = -1; s_i its sample weight,
 * 1 for every row when sw == NULL).  backward: SVM, where !(y * (x.w) < 0), adds filt(filt(x_j) * s) with s = y * c_i;
 * logistic s = (y * sigmoid(z)) * c_i.  The loss of n rows is lambda ||w||^2 (+ lambda1 ||w||_1) + S / n with
 * S = sum_i R(fl(c_i * L_i)), L_i the unweighted per-sample loss, summed as the device sums it: each term cut into 40-bit
 * fixed-point limbs of resolution 2^-160, the limbs added as integers, converted once from the top limb down (NaN if a term
 * is NaN, infinite or 2^52 or more).  With several workers each worker forms its S and the sums are added in worker order.
 */
#ifndef DSGD_ORACLE_SW_H
#define DSGD_ORACLE_SW_H

#include <stdint.h>

#include "dsgd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Weighted totals over the n listed rows at w: sums_out[0..2] = S, sum c_i [pred_i == y_i], sum c_i (each a fixed-point
 * sum); counts_out[0..1] = rows, correct. */
int dsgd_oracle_sw_eval(const dsgd_oracle_csr *a, int32_t logistic, const double *w, const int32_t *idx, int64_t n,
                        double w_pos, double w_neg, const double *sw, double *sums_out, int64_t *counts_out);

/* One request: the weighted gradient sum of the listed rows into grad_out (dim values), regularized with c = 2 lambda (w.d)
 * on its support when `regularize`; *loss_out (optional) = lambda ||w||^2 + S / n; *s_out (optional) = S. */
int dsgd_oracle_sw_gradient(const dsgd_oracle_csr *a, int32_t logistic, double lambda, const double *d, const double *w,
                            const int32_t *idx, int64_t n, double w_pos, double w_neg, const double *sw, int32_t regularize,
                            double *grad_out, double *loss_out, double *s_out);

/* n_steps sync steps as dsgd_oracle_cw_sync_steps (K workers, a rate per step, lambda1 >= 0) with the sample weights. */
int dsgd_oracle_sw_sync_steps(const dsgd_oracle_csr *a, int32_t logistic, double lambda, double lambda1, const double *d,
                              double *w, const int32_t *idx, const int32_t *counts, int32_t n_workers, const double *lrs,
                              int64_t n_steps, double w_pos, double w_neg, const double *sw, double *losses_out,
                              double *avg_sum);

#ifdef __cplusplus
}
#endif
#endif
