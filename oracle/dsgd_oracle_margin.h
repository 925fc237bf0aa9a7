/*
 * TEST INFRASTRUCTURE ONLY -- fp64, array-based CPU restatement of the gradient, the evaluations and the sync step of every
 * model, with the model as an argument: 0 SparseSVM, 1 SparseLogistic (DESIGN.md section 4.5), 2 SparseSquaredHinge,
 * 3 SparseModifiedHuber (section 4.15); in every weighting, with the L1 step (section 4.10), per-step rates and the averaging
 * sum.  It is the checker of record of the sync path for every model and option.  Conventions are those of dsgd_oracle.h
 * (same CSR struct, dense vectors with 0.0 for "key absent", the 1e-20 filter wherever the reference builds a new Sparse).
 * It is validated against the literal restatements in oracle/scala_semantics_margin.py, cw.py, sw.py and l1.py, and its
 * unweighted SVM against dsgd_oracle.c.
 *
 * One sample, z = y * (x . w) and t = fl(1 + z), evaluated in this order (the kernel's, dsgd_kernels.cuh):
 *   squared hinge    z <= -1: L = 0, s = 0;   else L = t * t, s = 2 * t
 *   modified Huber   z <= -1: L = 0, s = 0;   -1 < z <= 1: L = t * t, s = 2 * t;   z > 1: L = 4 * z, s = 4
 * backward adds filt(filt(x_j) * v) for v = y * s (unweighted) or (y * s) * c (weighted, c = w_y or c_i = fl(w_y * s_i)).
 * The SVM adds v = y (weighted: +-c) where !(z < 0) and has the loss 1 - y * pred; the logistic model has
 * L = softplus(z) = max(z, 0) + log1p(exp(-|z|)) and s = sigmoid(z), e / (1 + e) with e = exp(z) below 0.
 *
 * Weighting (`weighting`): 0 none; 1 class weights (w_pos, w_neg); 2 sample weights (c_i = fl(w_y * s_i), every s_i = 1
 * when sw == NULL).  Loss sums are the device's: every non-integer sum is the fixed-point sum of dsgd_fixed.cuh (terms
 * rounded to 2^-160, limbs added as integers, converted once from the top limb down), so it has the device's bits.
 *   weighting 0: S = sum R(L_i);  1: S = fl(fl(w_pos * sum_pos R(L_i)) + fl(w_neg * sum_neg R(L_i)));  2: S = sum R(fl(c_i L_i)).
 * A request's loss is lambda ||w||^2 + S / n; a sync step's is lambda ||w||^2 (+ lambda1 ||w||_1) + (S_1 + S_2 + ...) / batch
 * with the workers' S added in worker order and ||w||_1 a fixed-point sum, at the weights before the step.
 * The L1 step at rate lr_t, tau = lr_t * lambda1, after the update on every column:
 *   w_j = u_j > tau ? filt(u_j - tau) : (u_j < -tau ? filt(u_j + tau) : 0)        (tau <= 0: w_j = u_j).
 */
#ifndef DSGD_ORACLE_MARGIN_H
#define DSGD_ORACLE_MARGIN_H

#include <stdint.h>

#include "dsgd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* L(z) and s(z) of one sample of model 1, 2 or 3 (-3 for another model). */
int dsgd_oracle_margin_row(int32_t model, double z, double *loss_out, double *scale_out);

/* The L1 proximal step of one value at threshold tau (above); the sync step applies it to every column. */
double dsgd_oracle_margin_prox(double u, double tau);

/* ||w||_1 as the device sums it (the fixed-point sum of the |w_j|), and #{w_j != 0} into *nnz_out (optional). */
double dsgd_oracle_margin_l1_norm(const double *w, int32_t dim, int64_t *nnz_out);

/* The per-sample losses L_i (without lambda ||w||^2) of the listed rows, or of rows [begin, begin + n) with idx == NULL. */
int dsgd_oracle_margin_sample_losses(const dsgd_oracle_csr *a, int32_t model, const double *w, const int32_t *idx,
                                     int64_t begin, int64_t n, double *losses);

/* Unweighted evaluation of the listed rows (idx == NULL: rows [begin, begin + n)): *s_out = S, *correct_out,
 * *loss_out = lambda ||w||^2 + S / n, *acc_out = correct / n (each optional). */
int dsgd_oracle_margin_loss_acc(const dsgd_oracle_csr *a, int32_t model, double lambda, const double *w, const int32_t *idx,
                                int64_t begin, int64_t n, double *loss_out, double *acc_out, double *s_out,
                                int64_t *correct_out);

/* One request: the gradient sum of the listed rows in `weighting` into grad_out (dim values), regularized with
 * c = 2 lambda (w . d) on its support when `regularize`; *loss_out (optional) = lambda ||w||^2 + S / n; *s_out (optional) = S;
 * *c_out (optional) = c. */
int dsgd_oracle_margin_gradient(const dsgd_oracle_csr *a, int32_t model, int32_t weighting, double lambda, const double *d,
                                const double *w, const int32_t *idx, int64_t n, double w_pos, double w_neg, const double *sw,
                                int32_t regularize, double *grad_out, double *loss_out, double *s_out, double *c_out);

/* A weighted evaluation of the listed rows: weighting 1 (dsgd_eval*_class): sums_out[0..1] = the unweighted loss sums of the
 * y = +1 and y = -1 rows, counts_out[0..3] = correct+, correct-, rows+, rows-;  weighting 2 (dsgd_eval*_weighted):
 * sums_out[0..2] = S, sum c_i [correct], sum c_i, counts_out[0..1] = rows, correct. */
int dsgd_oracle_margin_eval(const dsgd_oracle_csr *a, int32_t model, int32_t weighting, const double *w, const int32_t *idx,
                            int64_t n, double w_pos, double w_neg, const double *sw, double *sums_out, int64_t *counts_out);

/* n_steps sync steps: per step K requests (worker k takes counts[k] ids) at the same weights, each regularized, their mean
 * filtered after each addition, w_j <- dsgd_oracle_margin_prox(filt(w_j - filt(filt(mean_j / K) * lrs[t])), lrs[t] * lambda1)
 * on every column.
 * losses_out (optional) as above; avg_sum (optional) += the weights after every step. */
int dsgd_oracle_margin_sync_steps(const dsgd_oracle_csr *a, int32_t model, int32_t weighting, double lambda, double lambda1,
                                  const double *d, double *w, const int32_t *idx, const int32_t *counts, int32_t n_workers,
                                  const double *lrs, int64_t n_steps, double w_pos, double w_neg, const double *sw,
                                  double *losses_out, double *avg_sum);

#ifdef __cplusplus
}
#endif
#endif
