/*
 * TEST INFRASTRUCTURE ONLY -- fp64, array-based CPU restatement of the reference's SGD hot path.
 *
 * The reference (zifeo/distributed-sgd, Scala) cannot run in this image (no JVM), so this is the
 * checker the CUDA path is compared against, and the "port" CPU baseline bench.py times.  It is
 * validated against the literal map-based restatement in oracle/scala_semantics.py, which in turn is
 * pinned against the reference's VecTests known answers.  PARITY STATUS: unpinned for SparseSVM /
 * Slave / Master (the reference holds no tests or golden vectors there -- SURVEY.md 8c).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may link
 * or load this library.  The product (distributed_sgd_b200/) never does.
 *
 * Conventions: rows are CSR (int64 row_ptr, int32 0-based col, fp32 val promoted to double exactly,
 * int8 label in {-1,+1}); weights / gradients / dimSparsity are dense double[dim] where 0.0 means
 * "key absent from the reference's Map".  CSR column c stands for the reference's 1-based feature
 * key c+1; dimSparsity is passed already shifted into the weight index space (see
 * dsgd_oracle_dim_sparsity).  Citations are path:line under
 * src/main/scala/epfl/distributed/ of the reference repository.
 */
#ifndef DSGD_ORACLE_H
#define DSGD_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int64_t n_rows;
  int32_t dim;
  const int64_t *row_ptr; /* n_rows + 1 */
  const int32_t *col;     /* nnz, 0-based */
  const float *val;       /* nnz */
  const int8_t *label;    /* n_rows, +1 / -1 */
} dsgd_oracle_csr;

/* SparseSVM.forward for each listed row: p = -signum(x . w)  (core/ml/SparseSVM.scala:14; core/Slave.scala:129-140). */
int dsgd_oracle_forward(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t n, double *preds);

/* SparseSVM.loss(w, samples) = lambda*||w||^2 + mean_i max(0, 1 - y_i p_i)  (SparseSVM.scala:16,20-23), and
 * accuracy = #{p_i == y_i}/n (core/Master.scala:100-103).  idx == NULL means rows [begin, begin+n). */
int dsgd_oracle_loss_acc(const dsgd_oracle_csr *a, double lambda, const double *w, const int32_t *idx,
                         int64_t begin, int64_t n, double *loss, double *acc);

/* Slave gradient request: r = regularize(sum_i backward(w, x_i, y_i), w)  (core/Slave.scala:142-157;
 * SparseSVM.scala:26-31; math/Vec.scala:65-75,128-131).  r_out is dense[dim]; c_out (optional) receives
 * c = 2*lambda*(w . d). */
int dsgd_oracle_gradient(const dsgd_oracle_csr *a, double lambda, const double *d, const double *w,
                         const int32_t *idx, int64_t n, double *r_out, double *c_out);

/* One synchronous step: K gradient requests (worker k gets idx[off_k .. off_k + counts[k])), mean over
 * workers, w <- w - lr*mean  (core/Master.scala:184-197).  loss_out (optional) = SparseSVM.loss(w_before,
 * all samples of the step) -- our definition of "per-step loss" (SURVEY.md F5).
 * threads: 1 = serial; K = one thread per logical worker (what the reference does, core/Slave.scala:142). */
int dsgd_oracle_sync_step(const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                          const int32_t *idx, const int32_t *counts, int32_t n_workers, double lr,
                          double *loss_out, int32_t threads);

/* n_steps consecutive sync steps; idx holds n_steps * sum(counts) indices, step-major then worker-major. */
int dsgd_oracle_sync_steps(const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                           const int32_t *idx, const int32_t *counts, int32_t n_workers, double lr,
                           int64_t n_steps, double *losses_out, int32_t threads);

/* ALL-CORES CONTEXT: one logical worker, its batch split over `threads` threads (rows in parallel, shared accumulator).
 * NOT the reference's parallelism (one thread per gradient request, core/Slave.scala:142); agrees with the serial form
 * to rounding.  bench.py reports it beside the one-thread-per-worker baseline. */
int dsgd_oracle_sync_steps_allcores(const dsgd_oracle_csr *a, double lambda, const double *d, double *w, const int32_t *idx,
                                    int64_t batch, double lr, int64_t n_steps, double *losses_out, int32_t threads);

/* Async worker iteration: delta = lr * regularize(mean_i backward(w_snapshot, x_i, y_i), w_snapshot)
 * (core/Slave.scala:92-99).  delta_out dense[dim]. The caller applies w -= delta to every replica
 * (core/Slave.scala:101-105,177-185; core/ml/GradState.scala:8). */
int dsgd_oracle_async_delta(const dsgd_oracle_csr *a, double lambda, const double *d, const double *w_snapshot,
                            const int32_t *idx, int64_t n, double lr, double *delta_out);

/* Sequential async run of one worker with concurrency 1: for each of n_updates iterations take `batch`
 * indices, compute delta against the current weights, apply it (w -= delta).  Deterministic single-
 * replica Hogwild (the K=1 case of core/Slave.scala:79-111). */
int dsgd_oracle_async_run(const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                          const int32_t *idx, int32_t batch, int64_t n_updates, double lr);

/* dimSparsity (Main.scala:54-65) over rows [0, n_train): reference key (c+1)-1 = c  ->  1/(df_c + 1) for df_c > 0,
 * then expressed in the WEIGHT index space: the reference dots w (keys c+1) with d (keys c), so weight column c
 * meets the entry of column c+1 (quirk Q3).  d_out[c] = 1/(df_{c+1}+1) if c+1 < dim and df_{c+1} > 0 else 0. */
int dsgd_oracle_dim_sparsity(const dsgd_oracle_csr *a, int64_t n_train, double *d_out);

#ifdef __cplusplus
}
#endif
#endif
