/*
 * TEST INFRASTRUCTURE ONLY -- fp64, array-based CPU restatement of the sync step with an L1 penalty (DESIGN.md section 4.10),
 * for SparseSVM and SparseLogistic, one step at a time.  Conventions are those of dsgd_oracle.h (same CSR struct, dense
 * vectors with 0.0 for "key absent", the 1e-20 filter wherever the reference builds a new Sparse).  It is validated against
 * the literal restatement in oracle/l1.py.
 *
 * Step t at rate lr_t: the step of dsgd_oracle_sync_steps / dsgd_oracle_logistic_sync_steps gives u (u_j = w_j on the columns
 * the step did not touch); then on every column, with tau = lr_t * lambda1,
 *   w_j = u_j > tau ? filt(u_j - tau) : (u_j < -tau ? filt(u_j + tau) : 0)        (tau == 0: w_j = u_j).
 * The step's loss is lambda ||w||^2 + lambda1 ||w||_1 + loss sum / batch at the weights before the step, added in that
 * order; ||w||_1 is summed with compensation (exact whenever the sum of |w_j| is a double, as for dyadic weights).
 */
#ifndef DSGD_ORACLE_L1_H
#define DSGD_ORACLE_L1_H

#include <stdint.h>

#include "dsgd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The proximal step of lambda1 * ||w||_1 at threshold tau (above), for one value. */
double dsgd_oracle_l1_prox(double u, double tau);

/* sum_j |w_j| (compensated) and #{w_j != 0}. */
double dsgd_oracle_l1_norm(const double *w, int32_t dim, int64_t *nnz_out);

/* n_steps sync steps of `logistic` (0: SparseSVM, 1: SparseLogistic): per step K requests (worker k takes counts[k] ids), mean
 * over workers filtered after each addition, w <- prox(w - lrs[t] * mean, lrs[t] * lambda1).  losses_out (optional) as
 * above; avg_sum (optional) += the weights after every step, column by column. */
int dsgd_oracle_l1_sync_steps(const dsgd_oracle_csr *a, int32_t logistic, double lambda, double lambda1, const double *d,
                              double *w, const int32_t *idx, const int32_t *counts, int32_t n_workers, const double *lrs,
                              int64_t n_steps, double *losses_out, double *avg_sum);

#ifdef __cplusplus
}
#endif
#endif
