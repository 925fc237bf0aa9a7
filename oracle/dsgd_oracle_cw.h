/*
 * TEST INFRASTRUCTURE ONLY -- fp64, array-based CPU restatement of the class-weighted gradient, evaluation and sync step
 * (DESIGN.md section 4.12), for SparseSVM and SparseLogistic.  Conventions are those of dsgd_oracle.h (same CSR struct, dense
 * vectors with 0.0 for "key absent", the 1e-20 filter wherever the reference builds a new Sparse).  It is validated against
 * the literal restatement in oracle/cw.py.
 *
 * A row of label y has the weight w_y (w_pos for y = +1, w_neg for y = -1).  backward: SVM, where !(y * (x.w) < 0), adds
 * filt(filt(x_j) * s) with s = y * w_y; logistic s = (y * sigmoid(z)) * w_y.  The loss of n rows is
 * lambda ||w||^2 (+ lambda1 ||w||_1) + (fl(w_pos * L_pos) + fl(w_neg * L_neg)) / n, L_pos and L_neg the per-class sums of the
 * unweighted per-sample losses (the logistic ones summed with compensation); with several workers each worker forms its
 * weighted sum and the sums are added in worker order.
 */
#ifndef DSGD_ORACLE_CW_H
#define DSGD_ORACLE_CW_H

#include <stdint.h>

#include "dsgd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Per-class totals over the n listed rows at w: sums_out[0..1] = L_pos, L_neg; counts_out[0..3] = correct_pos, correct_neg,
 * n_pos, n_neg. */
int dsgd_oracle_cw_eval(const dsgd_oracle_csr *a, int32_t logistic, const double *w, const int32_t *idx, int64_t n,
                        double *sums_out, int64_t *counts_out);

/* One request: the weighted gradient sum of the listed rows into grad_out (dim values), regularized with c = 2 lambda (w.d)
 * on its support when `regularize`; *loss_out (optional) = lambda ||w||^2 + weighted loss sum / n; sums_out (optional) =
 * L_pos, L_neg. */
int dsgd_oracle_cw_gradient(const dsgd_oracle_csr *a, int32_t logistic, double lambda, const double *d, const double *w,
                            const int32_t *idx, int64_t n, double w_pos, double w_neg, int32_t regularize, double *grad_out,
                            double *loss_out, double *sums_out);

/* n_steps sync steps as dsgd_oracle_l1_sync_steps (K workers, a rate per step, lambda1 >= 0) with the class weights. */
int dsgd_oracle_cw_sync_steps(const dsgd_oracle_csr *a, int32_t logistic, double lambda, double lambda1, const double *d,
                              double *w, const int32_t *idx, const int32_t *counts, int32_t n_workers, const double *lrs,
                              int64_t n_steps, double w_pos, double w_neg, double *losses_out, double *avg_sum);

#ifdef __cplusplus
}
#endif
#endif
