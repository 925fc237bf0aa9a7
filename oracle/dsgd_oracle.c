/*
 * TEST INFRASTRUCTURE ONLY -- see dsgd_oracle.h for the role of this file and the parity status.
 *
 * fp64 array-based restatement of the reference's sync / async SGD arithmetic.  The reference keeps
 * every vector as an immutable Map[Int, Number] whose constructor drops entries with |v| <= 1e-20
 * (math/Sparse.scala:108-118); here a dense double[dim] plays the map and "v == 0.0" plays "key absent",
 * and the filter is re-applied wherever the reference builds a new Sparse.
 */
#include "dsgd_oracle.h"

#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "dsgd_oracle_common.h"   /* EPS, filt, row_dot */

static inline double signum(double v) { return (double)((v > 0.0) - (v < 0.0)); }

static int check_idx(const dsgd_oracle_csr *a, const int32_t *idx, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (idx[i] < 0 || idx[i] >= a->n_rows) return -2;
  return 0;
}

int dsgd_oracle_forward(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t n, double *preds) {
  if (check_idx(a, idx, n)) return -2;
  for (int64_t i = 0; i < n; ++i) preds[i] = signum(row_dot(a, idx[i], w)) * -1.0; /* SparseSVM.scala:14 */
  return 0;
}

static double norm_squared(const double *w, int32_t dim) { /* math/Vec.scala:55 */
  double s = 0.0;
  for (int32_t j = 0; j < dim; ++j) s += w[j] * w[j];
  return s;
}

int dsgd_oracle_loss_acc(const dsgd_oracle_csr *a, double lambda, const double *w, const int32_t *idx,
                         int64_t begin, int64_t n, double *loss, double *acc) {
  if (n <= 0) return -3; /* reduce on an empty collection throws in the reference */
  if (idx && check_idx(a, idx, n)) return -2;
  if (!idx && (begin < 0 || begin + n > a->n_rows)) return -2;
  double total = 0.0;
  int64_t correct = 0;
  for (int64_t i = 0; i < n; ++i) {
    int64_t r = idx ? idx[i] : begin + i;
    double p = signum(row_dot(a, r, w)) * -1.0;    /* SparseSVM.scala:14 */
    double y = (double)a->label[r];
    double l = 1.0 - y * p;                        /* SparseSVM.scala:16 */
    total += l > 0.0 ? l : 0.0;
    correct += (p == y);                           /* core/Master.scala:102 */
  }
  if (loss) *loss = lambda * norm_squared(w, a->dim) + total / (double)n; /* SparseSVM.scala:20-23 */
  if (acc) *acc = (double)correct / (double)n;
  return 0;
}

/* c = lambda * 2.0 * w.dot(dimSparsity)  (SparseSVM.scala:31) */
static double reg_scalar(double lambda, const double *w, const double *d, int32_t dim) {
  double s = 0.0;
  for (int32_t j = 0; j < dim; ++j) s += filt(w[j] * d[j]);
  return lambda * 2.0 * s;
}

/* Accumulate sum_i backward(w, x_i, y_i) into g (dense, caller-zeroed), recording first-touch columns in
 * `touched` (capacity dim).  Returns via *hinge the sum of per-sample losses of the batch.
 * Vec.sum is a left fold of `+`, each of which re-filters its result (math/Vec.scala:128-131;
 * math/Sparse.scala:33,108-118). */
static void accumulate_batch(const dsgd_oracle_csr *a, const double *w, const int32_t *idx, int64_t n, double *g,
                             int32_t *touched, int32_t *n_touched, uint8_t *mark, double *hinge) {
  double h = 0.0;
  for (int64_t i = 0; i < n; ++i) {
    int64_t r = idx[i];
    double y = (double)a->label[r];
    double dot = row_dot(a, r, w);
    double p = signum(dot) * -1.0;
    double l = 1.0 - y * p;
    h += l > 0.0 ? l : 0.0;
    double activity = y * dot;         /* SparseSVM.scala:27 */
    if (activity < 0.0) continue;      /* SparseSVM.scala:28: zerosLike, adds nothing */
    for (int64_t p2 = a->row_ptr[r]; p2 < a->row_ptr[r + 1]; ++p2) {
      int32_t j = a->col[p2];
      double gv = filt(filt((double)a->val[p2]) * y); /* x * y: mapValues + constructor filter */
      if (gv == 0.0) continue;
      if (!mark[j]) { mark[j] = 1; touched[(*n_touched)++] = j; }
      g[j] = filt(g[j] + gv);
    }
  }
  if (hinge) *hinge = h;
}

typedef struct {
  int32_t *touched;
  uint8_t *mark;
  double *g;
} scratch_t;

static int scratch_init(scratch_t *s, int32_t dim) {
  s->touched = (int32_t *)malloc(sizeof(int32_t) * (size_t)dim);
  s->mark = (uint8_t *)calloc((size_t)dim, 1);
  s->g = (double *)calloc((size_t)dim, sizeof(double));
  return (s->touched && s->mark && s->g) ? 0 : -1;
}
static void scratch_free(scratch_t *s) { free(s->touched); free(s->mark); free(s->g); }

/* Worker request body on scratch: leaves r = regularize(sum, w) in s->g on the touched set. */
static void worker_gradient(const dsgd_oracle_csr *a, double c, const double *w, const int32_t *idx, int64_t n,
                            scratch_t *s, int32_t *n_touched, double *hinge) {
  *n_touched = 0;
  accumulate_batch(a, w, idx, n, s->g, s->touched, n_touched, s->mark, hinge);
  /* regularize: grad + grad.valueLike(c): c lands on the keys that SURVIVED the filter (Vec.scala:65-75) */
  if (c != 0.0 && fabs(c) > EPS) {
    for (int32_t t = 0; t < *n_touched; ++t) {
      int32_t j = s->touched[t];
      if (s->g[j] != 0.0) s->g[j] = filt(s->g[j] + c);
    }
  }
}

static void scratch_reset(scratch_t *s, int32_t n_touched) {
  for (int32_t t = 0; t < n_touched; ++t) { s->g[s->touched[t]] = 0.0; s->mark[s->touched[t]] = 0; }
}

int dsgd_oracle_gradient(const dsgd_oracle_csr *a, double lambda, const double *d, const double *w,
                         const int32_t *idx, int64_t n, double *r_out, double *c_out) {
  if (n <= 0) return -3; /* Vec.sum on an empty list throws (math/Vec.scala:129, quirk Q7) */
  if (check_idx(a, idx, n)) return -2;
  scratch_t s;
  if (scratch_init(&s, a->dim)) return -1;
  double c = reg_scalar(lambda, w, d, a->dim);
  int32_t nt = 0;
  worker_gradient(a, c, w, idx, n, &s, &nt, NULL);
  memcpy(r_out, s.g, sizeof(double) * (size_t)a->dim);
  if (c_out) *c_out = c;
  scratch_free(&s);
  return 0;
}

/* ---- synchronous step(s) ------------------------------------------------------------------------- */

typedef struct {
  const dsgd_oracle_csr *a;
  const double *w;
  double c;
  const int32_t *idx;
  int64_t n;
  scratch_t *s;
  int32_t n_touched;
  double hinge;
} worker_job;

static void *worker_thread(void *p) {
  worker_job *j = (worker_job *)p;
  worker_gradient(j->a, j->c, j->w, j->idx, j->n, j->s, &j->n_touched, &j->hinge);
  return NULL;
}

typedef struct {
  int32_t K;
  scratch_t *ws;      /* per worker */
  scratch_t sum;      /* cross-worker sum, touched union */
  worker_job *jobs;
  pthread_t *tids;
} step_ctx;

static int step_ctx_init(step_ctx *sc, int32_t K, int32_t dim) {
  sc->K = K;
  sc->ws = (scratch_t *)calloc((size_t)K, sizeof(scratch_t));
  sc->jobs = (worker_job *)calloc((size_t)K, sizeof(worker_job));
  sc->tids = (pthread_t *)calloc((size_t)K, sizeof(pthread_t));
  if (!sc->ws || !sc->jobs || !sc->tids) return -1;
  for (int32_t k = 0; k < K; ++k)
    if (scratch_init(&sc->ws[k], dim)) return -1;
  return scratch_init(&sc->sum, dim);
}
static void step_ctx_free(step_ctx *sc) {
  for (int32_t k = 0; k < sc->K; ++k) scratch_free(&sc->ws[k]);
  scratch_free(&sc->sum);
  free(sc->ws); free(sc->jobs); free(sc->tids);
}

static int one_sync_step(step_ctx *sc, const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                         const int32_t *idx, const int32_t *counts, double lr, double *loss_out, int32_t threads) {
  const int32_t K = sc->K;
  /* every request carries the same weights, so c is the same for every worker (Master.scala:186-188) */
  const double c = reg_scalar(lambda, w, d, a->dim);
  int64_t off = 0, total = 0;
  for (int32_t k = 0; k < K; ++k) {
    if (counts[k] <= 0) return -3; /* empty slice => Vec.sum throws => fit fails (quirk Q7) */
    worker_job *j = &sc->jobs[k];
    j->a = a; j->w = w; j->c = c; j->idx = idx + off; j->n = counts[k]; j->s = &sc->ws[k];
    off += counts[k]; total += counts[k];
  }
  if (threads > 1 && K > 1) {
    for (int32_t k = 1; k < K; ++k) pthread_create(&sc->tids[k], NULL, worker_thread, &sc->jobs[k]);
    worker_thread(&sc->jobs[0]);
    for (int32_t k = 1; k < K; ++k) pthread_join(sc->tids[k], NULL);
  } else {
    for (int32_t k = 0; k < K; ++k) worker_thread(&sc->jobs[k]);
  }
  if (loss_out) {
    double h = 0.0;
    for (int32_t k = 0; k < K; ++k) h += sc->jobs[k].hinge;
    *loss_out = lambda * norm_squared(w, a->dim) + h / (double)total; /* SparseSVM.scala:20-23 on w_before */
  }
  /* Vec.mean(res) = (r_0 + r_1 + ... ) / K  -- left fold in worker order, filter after every + (Master.scala:194) */
  scratch_t *S = &sc->sum;
  int32_t nts = 0;
  for (int32_t k = 0; k < K; ++k) {
    scratch_t *s = &sc->ws[k];
    for (int32_t t = 0; t < sc->jobs[k].n_touched; ++t) {
      int32_t j = s->touched[t];
      if (s->g[j] == 0.0) continue;
      if (!S->mark[j]) { S->mark[j] = 1; S->touched[nts++] = j; }
      S->g[j] = filt(S->g[j] + s->g[j]);
    }
    scratch_reset(s, sc->jobs[k].n_touched);
  }
  /* w - learningRate * grad  (Master.scala:197): (sum / K) filtered, * lr filtered, subtraction filtered */
  for (int32_t t = 0; t < nts; ++t) {
    int32_t j = S->touched[t];
    double mean = filt(S->g[j] / (double)K);
    double step = filt(mean * lr);
    w[j] = filt(w[j] - step);
  }
  scratch_reset(S, nts);
  return 0;
}

/* Threaded form: K persistent worker threads (the reference serves its gradient requests from a fixed thread pool,
 * utils/Pool.scala:13), two barriers per step; thread 0 plays the master between them. */
typedef struct {
  step_ctx *sc;
  const dsgd_oracle_csr *a;
  double lambda, lr;
  const double *d;
  double *w;
  const int32_t *idx;
  const int32_t *counts;
  int64_t n_steps, per_step;
  double *losses_out;
  pthread_barrier_t *bar;
  int32_t k;
  int *rc;
} pool_arg;

static void aggregate_and_update(step_ctx *sc, const dsgd_oracle_csr *a, double lambda, double *w, double lr,
                                 double *loss_out, int64_t total) {
  const int32_t K = sc->K;
  if (loss_out) {
    double h = 0.0;
    for (int32_t k = 0; k < K; ++k) h += sc->jobs[k].hinge;
    *loss_out = lambda * norm_squared(w, a->dim) + h / (double)total;
  }
  scratch_t *S = &sc->sum;
  int32_t nts = 0;
  for (int32_t k = 0; k < K; ++k) {
    scratch_t *s = &sc->ws[k];
    for (int32_t t = 0; t < sc->jobs[k].n_touched; ++t) {
      int32_t j = s->touched[t];
      if (s->g[j] == 0.0) continue;
      if (!S->mark[j]) { S->mark[j] = 1; S->touched[nts++] = j; }
      S->g[j] = filt(S->g[j] + s->g[j]);
    }
    scratch_reset(s, sc->jobs[k].n_touched);
  }
  for (int32_t t = 0; t < nts; ++t) {
    int32_t j = S->touched[t];
    double mean = filt(S->g[j] / (double)K);
    double step = filt(mean * lr);
    w[j] = filt(w[j] - step);
  }
  scratch_reset(S, nts);
}

static void *pool_thread(void *p) {
  pool_arg *g = (pool_arg *)p;
  step_ctx *sc = g->sc;
  for (int64_t s = 0; s < g->n_steps; ++s) {
    if (g->k == 0) {  /* the master prepares the K requests: same weights, hence the same c, for everybody */
      const double c = reg_scalar(g->lambda, g->w, g->d, g->a->dim);
      int64_t off = 0;
      for (int32_t k = 0; k < sc->K; ++k) {
        worker_job *j = &sc->jobs[k];
        j->a = g->a; j->w = g->w; j->c = c; j->idx = g->idx + s * g->per_step + off; j->n = g->counts[k]; j->s = &sc->ws[k];
        off += g->counts[k];
      }
    }
    pthread_barrier_wait(g->bar);
    worker_thread(&sc->jobs[g->k]);
    pthread_barrier_wait(g->bar);
    if (g->k == 0)
      aggregate_and_update(sc, g->a, g->lambda, g->w, g->lr, g->losses_out ? g->losses_out + s : NULL, g->per_step);
  }
  return NULL;
}

int dsgd_oracle_sync_steps(const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                           const int32_t *idx, const int32_t *counts, int32_t n_workers, double lr,
                           int64_t n_steps, double *losses_out, int32_t threads) {
  if (n_workers <= 0) return -3;
  int64_t per_step = 0;
  for (int32_t k = 0; k < n_workers; ++k) {
    if (counts[k] <= 0) return -3; /* empty slice => Vec.sum throws => fit fails (quirk Q7) */
    per_step += counts[k];
  }
  if (check_idx(a, idx, per_step * n_steps)) return -2;
  step_ctx sc;
  if (step_ctx_init(&sc, n_workers, a->dim)) return -1;
  int rc = 0;
  if (threads > 1 && n_workers > 1 && n_steps > 0) {
    pthread_barrier_t bar;
    pthread_barrier_init(&bar, NULL, (unsigned)n_workers);
    pool_arg *args = (pool_arg *)calloc((size_t)n_workers, sizeof(pool_arg));
    for (int32_t k = 0; k < n_workers; ++k) {
      pool_arg g = {&sc, a, lambda, lr, d, w, idx, counts, n_steps, per_step, losses_out, &bar, k, &rc};
      args[k] = g;
    }
    for (int32_t k = 1; k < n_workers; ++k) pthread_create(&sc.tids[k], NULL, pool_thread, &args[k]);
    pool_thread(&args[0]);
    for (int32_t k = 1; k < n_workers; ++k) pthread_join(sc.tids[k], NULL);
    pthread_barrier_destroy(&bar);
    free(args);
  } else {
    for (int64_t s = 0; s < n_steps && rc == 0; ++s)
      rc = one_sync_step(&sc, a, lambda, d, w, idx + s * per_step, counts, lr, losses_out ? losses_out + s : NULL, 1);
  }
  step_ctx_free(&sc);
  return rc;
}

int dsgd_oracle_sync_step(const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                          const int32_t *idx, const int32_t *counts, int32_t n_workers, double lr,
                          double *loss_out, int32_t threads) {
  return dsgd_oracle_sync_steps(a, lambda, d, w, idx, counts, n_workers, lr, 1, loss_out, threads);
}

/* ---- asynchronous worker ------------------------------------------------------------------------- */

/* delta on scratch: lr * regularize(mean, w_snapshot); returns touched count (core/Slave.scala:92-99). */
static void async_delta_scratch(const dsgd_oracle_csr *a, double lambda, const double *d, const double *w,
                                const int32_t *idx, int64_t n, double lr, scratch_t *s, int32_t *nt) {
  *nt = 0;
  accumulate_batch(a, w, idx, n, s->g, s->touched, nt, s->mark, NULL);
  const double c = reg_scalar(lambda, w, d, a->dim);
  const int add_c = (c != 0.0 && fabs(c) > EPS);
  for (int32_t t = 0; t < *nt; ++t) {
    int32_t j = s->touched[t];
    double m = filt(s->g[j] / (double)n);       /* Vec.mean = sum / size (math/Vec.scala:139) */
    if (m != 0.0 && add_c) m = filt(m + c);     /* regularize on the surviving keys */
    s->g[j] = filt(m * lr);                     /* learningRate * (...) */
  }
}

int dsgd_oracle_async_delta(const dsgd_oracle_csr *a, double lambda, const double *d, const double *w_snapshot,
                            const int32_t *idx, int64_t n, double lr, double *delta_out) {
  if (n <= 0) return -3;
  if (check_idx(a, idx, n)) return -2;
  scratch_t s;
  if (scratch_init(&s, a->dim)) return -1;
  int32_t nt = 0;
  async_delta_scratch(a, lambda, d, w_snapshot, idx, n, lr, &s, &nt);
  memcpy(delta_out, s.g, sizeof(double) * (size_t)a->dim);
  scratch_free(&s);
  return 0;
}

int dsgd_oracle_async_run(const dsgd_oracle_csr *a, double lambda, const double *d, double *w,
                          const int32_t *idx, int32_t batch, int64_t n_updates, double lr) {
  if (batch <= 0) return -3;
  if (check_idx(a, idx, (int64_t)batch * n_updates)) return -2;
  scratch_t s;
  if (scratch_init(&s, a->dim)) return -1;
  for (int64_t u = 0; u < n_updates; ++u) {
    int32_t nt = 0;
    async_delta_scratch(a, lambda, d, w, idx + u * batch, batch, lr, &s, &nt);
    for (int32_t t = 0; t < nt; ++t) {          /* weights.transform(_ - gradUpdate)  (Slave.scala:101) */
      int32_t j = s.touched[t];
      w[j] = filt(w[j] - s.g[j]);
    }
    scratch_reset(&s, nt);
  }
  scratch_free(&s);
  return 0;
}

/* ---- dimSparsity ---------------------------------------------------------------------------------- */

int dsgd_oracle_dim_sparsity(const dsgd_oracle_csr *a, int64_t n_train, double *d_out) {
  if (n_train < 0 || n_train > a->n_rows) return -2;
  int64_t *df = (int64_t *)calloc((size_t)a->dim, sizeof(int64_t));
  if (!df) return -1;
  for (int64_t p = a->row_ptr[0]; p < a->row_ptr[n_train]; ++p)
    if (fabs((double)a->val[p]) > EPS) df[a->col[p]] += 1; /* keys of the row's map (Main.scala:57-60) */
  for (int32_t c = 0; c < a->dim; ++c) {
    /* reference d key c holds 1/(df_c + 1) (Main.scala:61-63); weight column c carries reference key c+1,
     * so in the dot product it meets d key c+1 (quirk Q3). */
    int32_t src = c + 1;
    d_out[c] = (src < a->dim && df[src] != 0) ? 1.0 / ((double)df[src] + 1.0) : 0.0;
  }
  free(df);
  return 0;
}

/* ---------------------------------------------------------------------------------------------------------------------
 * ALL-CORES CONTEXT (not the reference's parallelism: the reference serves one gradient request on ONE pool thread,
 * core/Slave.scala:142).  One logical worker whose batch is split over T threads, to show what the same arithmetic does
 * when a CPU box throws every core at a single worker's step: rows in parallel (each thread adds its y*x entries to a
 * shared accumulator with compare-and-swap, filter after every addition), c and ||w||^2 as per-thread partial sums combined
 * in thread order, the update applied by whichever thread touched a column first; three spin barriers per step.
 * Summation order inside a batch differs from the serial left fold, so results agree with dsgd_oracle_sync_steps to
 * rounding (tests/test_oracle_c_vs_literal.py), not to the bit.  Used by bench.py for the `all_cores` context figure only.
 * ------------------------------------------------------------------------------------------------------------------- */
typedef struct {
  volatile int count;
  volatile int sense;
  int n;
} spin_barrier;

static void spin_wait(spin_barrier *b, int *local_sense) {
  *local_sense = !*local_sense;
  if (__atomic_add_fetch(&b->count, 1, __ATOMIC_ACQ_REL) == b->n) {
    b->count = 0;
    __atomic_store_n(&b->sense, *local_sense, __ATOMIC_RELEASE);
  } else {
    while (__atomic_load_n(&b->sense, __ATOMIC_ACQUIRE) != *local_sense) __builtin_ia32_pause();
  }
}

typedef struct {
  const dsgd_oracle_csr *a;
  double lambda, lr;
  const double *d;
  double *w;
  const int32_t *idx;
  int64_t n_steps, batch;
  double *losses_out;
  double *g;              /* shared accumulator, dense */
  uint8_t *mark;          /* shared first-touch marks */
  double *part;           /* [T][4]: partial w.d, partial ||w||^2, partial hinge, pad */
  spin_barrier *bar;
  int32_t *touched;       /* this thread's first-touched columns (capacity dim) */
  int T, t;
} mt_arg;

static inline void atomic_add_filt(double *p, double v) {
  uint64_t *q = (uint64_t *)p;
  uint64_t old = __atomic_load_n(q, __ATOMIC_RELAXED);
  for (;;) {
    double o, nv;
    memcpy(&o, &old, 8);
    nv = filt(o + v);
    uint64_t nb;
    memcpy(&nb, &nv, 8);
    if (__atomic_compare_exchange_n(q, &old, nb, 1, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) return;
  }
}

static void *mt_thread(void *p) {
  mt_arg *g = (mt_arg *)p;
  const dsgd_oracle_csr *a = g->a;
  const int T = g->T, t = g->t;
  const int32_t dim = a->dim;
  const int32_t j0 = (int32_t)((int64_t)dim * t / T), j1 = (int32_t)((int64_t)dim * (t + 1) / T);
  const int64_t r0 = g->batch * t / T, r1 = g->batch * (t + 1) / T;
  int sense = 0;
  for (int64_t s = 0; s < g->n_steps; ++s) {
    /* partial sums over this thread's column range: c = 2 lambda (w . d), ||w||^2 */
    double sd = 0.0, sn = 0.0;
    for (int32_t j = j0; j < j1; ++j) { sd += filt(g->w[j] * g->d[j]); sn += g->w[j] * g->w[j]; }
    g->part[4 * t + 0] = sd; g->part[4 * t + 1] = sn;
    spin_wait(g->bar, &sense);
    double wd = 0.0, nrm = 0.0;
    for (int k = 0; k < T; ++k) { wd += g->part[4 * k + 0]; nrm += g->part[4 * k + 1]; }
    const double c = g->lambda * 2.0 * wd;
    /* this thread's rows of the batch */
    const int32_t *idx = g->idx + s * g->batch;
    int32_t nt = 0;
    double h = 0.0;
    for (int64_t i = r0; i < r1; ++i) {
      const int64_t r = idx[i];
      const double y = (double)a->label[r];
      const double dot = row_dot(a, r, g->w);
      const double pr = signum(dot) * -1.0;
      const double l = 1.0 - y * pr;
      h += l > 0.0 ? l : 0.0;
      if (y * dot < 0.0) continue;
      for (int64_t p2 = a->row_ptr[r]; p2 < a->row_ptr[r + 1]; ++p2) {
        const int32_t j = a->col[p2];
        const double gv = filt(filt((double)a->val[p2]) * y);
        if (gv == 0.0) continue;
        if (!__atomic_exchange_n(&g->mark[j], 1, __ATOMIC_RELAXED)) g->touched[nt++] = j;
        atomic_add_filt(&g->g[j], gv);
      }
    }
    g->part[4 * t + 2] = h;
    spin_wait(g->bar, &sense);   /* the batch sum is complete; w is still w_before */
    if (t == 0 && g->losses_out) {
      double hs = 0.0;
      for (int k = 0; k < T; ++k) hs += g->part[4 * k + 2];
      g->losses_out[s] = g->lambda * nrm + hs / (double)g->batch;
    }
    /* regularize on the support, mean over the (one) worker, update -- for the columns this thread touched first */
    const int add_c = (c != 0.0 && fabs(c) > EPS);
    for (int32_t q = 0; q < nt; ++q) {
      const int32_t j = g->touched[q];
      double v = g->g[j];
      if (v != 0.0 && add_c) v = filt(v + c);
      const double step = filt(filt(v / 1.0) * g->lr);
      g->w[j] = filt(g->w[j] - step);
      g->g[j] = 0.0;
      g->mark[j] = 0;
    }
    spin_wait(g->bar, &sense);   /* w_after is complete before anybody reads it */
  }
  return NULL;
}

int dsgd_oracle_sync_steps_allcores(const dsgd_oracle_csr *a, double lambda, const double *d, double *w, const int32_t *idx,
                                    int64_t batch, double lr, int64_t n_steps, double *losses_out, int32_t threads) {
  if (batch <= 0 || threads <= 0) return -3;
  if (check_idx(a, idx, batch * n_steps)) return -2;
  const int T = threads;
  spin_barrier bar = {0, 0, T};
  double *g = (double *)calloc((size_t)a->dim, sizeof(double));
  uint8_t *mark = (uint8_t *)calloc((size_t)a->dim, 1);
  double *part = (double *)calloc((size_t)T * 4, sizeof(double));
  mt_arg *args = (mt_arg *)calloc((size_t)T, sizeof(mt_arg));
  pthread_t *tids = (pthread_t *)calloc((size_t)T, sizeof(pthread_t));
  int rc = (g && mark && part && args && tids) ? 0 : -1;
  for (int t = 0; t < T && rc == 0; ++t) {
    mt_arg m = {a, lambda, lr, d, w, idx, n_steps, batch, losses_out, g, mark, part, &bar, NULL, T, t};
    m.touched = (int32_t *)malloc(sizeof(int32_t) * (size_t)a->dim);
    if (!m.touched) rc = -1;
    args[t] = m;
  }
  if (rc == 0) {
    for (int t = 1; t < T; ++t) pthread_create(&tids[t], NULL, mt_thread, &args[t]);
    mt_thread(&args[0]);
    for (int t = 1; t < T; ++t) pthread_join(tids[t], NULL);
  }
  for (int t = 0; t < T; ++t)
    if (args) free(args[t].touched);
  free(g); free(mark); free(part); free(args); free(tids);
  return rc;
}
