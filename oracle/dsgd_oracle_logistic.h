/*
 * TEST INFRASTRUCTURE ONLY -- fp64, array-based CPU restatement of SparseLogistic, the logistic-loss model beside SparseSVM
 * (DESIGN.md section 4.5).  Conventions are those of dsgd_oracle.h (same CSR struct, dense vectors with 0.0 for "key absent",
 * the 1e-20 filter wherever the reference builds a new Sparse).  It is validated against the literal map-based restatement in
 * oracle/scala_semantics_logistic.py.  The model-independent parts (forward, dimSparsity) are dsgd_oracle.c's.
 *
 * For one sample z = y * (x . w):  loss softplus(z) = max(z, 0) + log1p(exp(-|z|));  backward x * (y * sigmoid(z)),
 * sigmoid(t) = t >= 0 ? 1 / (1 + exp(-t)) : e / (1 + e), e = exp(t);  regularize and the sync step are the SVM's.
 */
#ifndef DSGD_ORACLE_LOGISTIC_H
#define DSGD_ORACLE_LOGISTIC_H

#include <stdint.h>

#include "dsgd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* loss = lambda*||w||^2 + mean_i softplus(z_i) (a left fold), acc = #{-signum(x_i . w) == y_i}/n.  idx == NULL: rows
 * [begin, begin + n). */
int dsgd_oracle_logistic_loss_acc(const dsgd_oracle_csr *a, double lambda, const double *w, const int32_t *idx,
                                  int64_t begin, int64_t n, double *loss, double *acc);
/* The per-sample losses softplus(z_i), for sums taken elsewhere (math.fsum). */
int dsgd_oracle_logistic_sample_losses(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t begin,
                                       int64_t n, double *losses);
/* r = regularize(sum_i backward(w, x_i, y_i), w); c_out (optional) = 2*lambda*(w . d). */
int dsgd_oracle_logistic_gradient(const dsgd_oracle_csr *a, double lambda, const double *d, const double *w,
                                  const int32_t *idx, int64_t n, double *r_out, double *c_out);
/* n_steps sync steps: per step K requests (worker k takes counts[k] ids), mean over workers filtered after each addition,
 * w <- w - lr * mean; losses_out (optional) = loss(w_before, all samples of the step). */
int dsgd_oracle_logistic_sync_steps(const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                                    const int32_t *idx, const int32_t *counts, int32_t n_workers, double lr,
                                    int64_t n_steps, double *losses_out);

#ifdef __cplusplus
}
#endif
#endif
