/*
 * dsgd.h -- C ABI of the H100-native (sm_90a) data-parallel SGD hot path (libdsgd.so).
 *
 * This is the drop-in boundary for zifeo/distributed-sgd's hot path.  The reference has no FFI of its
 * own (it is 100 % Scala over gRPC, SURVEY.md F1/F2); the seams this ABI sits behind are the handlers of
 * its gRPC `Slave` service and the step body of `Master.fit`.  Every entry point names the reference
 * interface it replaces (path:line under the reference repository's src/main/).  INTEGRATION.md shows the JNI /
 * Scala binding a maintainer would add; distributed_sgd_b200/ is the Python host that mirrors the
 * reference's Slave / Master / SparseSVM surface over this ABI.
 *
 * Conventions
 *  - One opaque dsgd_ctx per GPU == one reference Slave (+ its SparseSVM).  In sync mode every ctx also
 *    carries the Master's weight vector (weights stay resident on the device; the reference's per-request
 *    weight broadcast, core/Master.scala:186-188, disappears).
 *  - Every call returns 0 (DSGD_OK) or a negative DSGD_ERR_*; dsgd_last_error() gives the message.  No
 *    exception crosses the ABI.  The caller owns all host buffers; they are consumed before the call
 *    returns.  The ctx owns all device memory.
 *  - Vectors (weights, gradients, dimSparsity) are dense double[dim]; 0.0 stands for "key absent from the
 *    reference's Map[Int, Number]".  The reference's wire type is double (protobuf/proto.proto:28-31).
 *  - Rows are CSR with 0-based int32 columns and fp32 values; CSR column c stands for the reference's
 *    1-based feature key c+1 (utils/Dataset.scala:30).  Sample indices are row ids into what
 *    dsgd_load_csr received (the reference addresses a slave by global row id, core/Slave.scala:149).
 *  - Arithmetic: values fp32 (exactly promoted), every accumulation and all state in fp64, like the
 *    reference's spire.math.Number over Double.
 *  - Every fp64 row dot x . w on the device is the row fold: the row window cut into 128-pair chunks from its start, in
 *    chunk c lane l sums the filtered products of pairs 128 c + l + 32 u (u = 0..3, in order, from +0.0), an xor
 *    butterfly per chunk, then 0.0 + the chunk partials in order.  Every request, evaluation, metrics, sync and async
 *    path uses it (the fp32 streaming pass decides only rows whose sign the fold cannot change), so a row's margin,
 *    prediction and gate depend on the row and w alone: not on the request size, the grid or the other rows of a step.
 *    The reference sums in HashMap order; the oracle's index-order fold can differ in the last bits, and in sign where
 *    the products cancel to within fp64 rounding.
 *  - Threading: calls on one ctx are serialised by the caller, except dsgd_update_grad,
 *    dsgd_get_weights, dsgd_async_updates and dsgd_stop_async, which are safe while the async loop runs
 *    (the reference serves them from its 8-thread pool concurrently with asyncTask, core/Slave.scala:24-30).
 *    dsgd_update_grad may also be called from several threads at once: the calls take a lock of the ctx and
 *    each delta is applied exactly once.
 *    From dsgd_start_async until dsgd_stop_async, every call that takes a list of row ids (dsgd_forward,
 *    dsgd_gradient, dsgd_margins, dsgd_probabilities, dsgd_eval_samples_*) refuses a list of more ids than
 *    loaded rows with DSGD_ERR_STATE: its buffers would have to grow, and growing one waits for every kernel on
 *    the device, the running loop included.
 */
#ifndef DSGD_H
#define DSGD_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSGD_OK 0
#define DSGD_ERR_INVALID (-1) /* bad argument; the reference's require(...) / IllegalArgumentException        */
#define DSGD_ERR_STATE (-2)   /* wrong mode or state: "slave is in synchronous mode", "already running"        */
#define DSGD_ERR_EMPTY (-3)   /* empty batch: Vec.sum on an empty list throws (math/Vec.scala:129, quirk Q7)   */
#define DSGD_ERR_RANGE (-4)   /* sample index outside the loaded rows (ArrayIndexOutOfBounds in the reference)  */
#define DSGD_ERR_CUDA (-5)    /* CUDA runtime error, or no usable GPU (there is no CPU fallback)                */
#define DSGD_ERR_NCCL (-6)    /* NCCL error                                                                     */
#define DSGD_ERR_NOMEM (-7)
#define DSGD_ERR_TIMEOUT (-8) /* a device-side wait (peer flag, grid barrier) hit its watchdog                  */

#define DSGD_UNIQUE_ID_BYTES 128
#define DSGD_IPC_HANDLE_BYTES 64

/* dsgd_create flags */
#define DSGD_FLAG_ASYNC 1u /* the `async` constructor argument of Slave / Master (core/Slave.scala:20) */
/* The model is SparseLogistic instead of SparseSVM: per-sample loss softplus(z) = log(1 + e^z) and gradient
 * x * (y * sigmoid(z)), z = y * (x . w); prediction, regularize() and the sync step are the SVM's.  Every call that depends
 * on the model follows it: dsgd_gradient, dsgd_eval, the dsgd_eval_*_sums calls, the sync steps and their losses.  A logistic
 * ctx takes the per-step sync path (never the persistent or fused kernel), so world > 1 needs dsgd_comm_init.  Combined with
 * DSGD_FLAG_ASYNC, dsgd_create fails with DSGD_ERR_INVALID (async mode supports the SVM model only). */
#define DSGD_FLAG_LOGISTIC 2u
/* The margin models beside it, z = y * (x . w), t = fl(1 + z) (DESIGN.md section 4.15):
 *   DSGD_FLAG_SQUARED_HINGE   SparseSquaredHinge, the L2-loss SVM: per-sample loss 0 for z <= -1, else t * t; gradient
 *                             x * (y * s) with s = 0 for z <= -1, else 2 * t.
 *   DSGD_FLAG_MODIFIED_HUBER  SparseModifiedHuber: loss 0 for z <= -1, t * t for -1 < z <= 1, 4 * z above; s = 0, 2 * t, 4.
 * Like DSGD_FLAG_LOGISTIC they keep the SVM's prediction, regularize() and sync step, follow it in every call that depends
 * on the model, add their losses in the fixed-point limbs of the logistic loss sum, are refused by the *_counts calls
 * (DSGD_ERR_STATE) and take the per-step sync path.  dsgd_probabilities serves SparseModifiedHuber, not
 * SparseSquaredHinge.  dsgd_create fails with DSGD_ERR_INVALID on more than one model flag, and on any model flag with
 * DSGD_FLAG_ASYNC.
 * Loss sums and the 2^52 limit: a summed value of 2^52 or more, infinite or NaN makes its sum NaN (the squared hinge
 * reaches 2^52 at z = 2^26 - 1, modified Huber at z = 2^50; their losses pass it long before the logistic loss does).  The
 * next pass or step starts from a clean sum.  The unweighted and per-class evaluations sum L_i; a class-weighted gradient or
 * step sums L_i per class and then takes fl(w_pos * S+) + fl(w_neg * S-); the weighted evaluations (dsgd_eval*_weighted)
 * and a sample-weighted gradient or step sum fl(c_i * L_i).  So with class weights (2, 1/2) and a row of L in
 * [2^51, 2^52), the class-weighted loss is finite and the weighted evaluation NaN; with a class weight of 0 and a row of
 * finite L >= 2^52 in that class, the class-weighted loss is NaN (0 * NaN) and the weighted evaluation adds an exact 0.
 * At a NaN z the squared hinge's scale is NaN, which the 1e-20 filter drops (no gradient), and modified Huber's is 4 (both
 * branch tests are false). */
#define DSGD_FLAG_SQUARED_HINGE 4u
#define DSGD_FLAG_MODIFIED_HUBER 8u
/* An unregularised intercept beta, combinable with any one model flag (DESIGN.md section 4.18): the weight of a virtual
 * column whose value is 1 in every row.  Every score x . w becomes fl(x . w + filt(beta)), beta added once after the row
 * fold; row i adds filt(s_i) (what it scatters onto a column with x = 1) to beta's gradient; the step is
 * beta <- filt(beta - filt(filt(g_b / K) * lr)); averaging averages beta too.  beta is in no penalty: not in
 * lambda * ||w||^2, not in c = 2 lambda (w . d), not in the L1 step, ||w||_1 or its non-zero count.
 * Lengths: on an intercept ctx every weight vector the ABI reads or writes is dim + 1 doubles, beta last -- dsgd_set_weights,
 * dsgd_get_weights, the `w` of every request and evaluation, dsgd_average_weights' output, and dsgd_gradient's grad_out
 * (beta's gradient at [dim]).  d (dsgd_set_dim_sparsity) stays dim long.
 * Paths: an intercept ctx takes the per-step sync path (never the persistent or fused kernel, so world > 1 needs
 * dsgd_comm_init; a rank wired with the peer exchange only fails with DSGD_ERR_STATE before any launch) and the fp64 row
 * kernel for every request (never the fp32 streaming pass).  Every reader scores with beta: dsgd_margins,
 * dsgd_probabilities, the metrics and curve calls, the Platt, isotonic and weighted calibrations and their probabilities and
 * quality passes.  dsgd_info reports "intercept": true.  Combined with
 * DSGD_FLAG_ASYNC, dsgd_create fails with DSGD_ERR_INVALID before it looks for a device. */
#define DSGD_FLAG_INTERCEPT 16u

typedef struct dsgd_ctx dsgd_ctx;

/* ---- lifecycle: `new Slave(node, master, data, model, async)` + `new SparseSVM(lambda, dimSparsity)`
 *      (Main.scala:68,138,149; core/Slave.scala:20; core/ml/SparseSVM.scala:11) ------------------------ */
int dsgd_create(dsgd_ctx **out, int device, int32_t dim, double lambda, int rank, int world, uint32_t flags);
int dsgd_destroy(dsgd_ctx *ctx);
/* Message of the last failing call on ctx (ctx == NULL: last failing dsgd_create on this thread). */
const char *dsgd_last_error(const dsgd_ctx *ctx);
/* Build / device facts as a JSON string (SM count, arch, kernels compiled). */
const char *dsgd_info(const dsgd_ctx *ctx);
/* Use the caller's CUDA stream (a cudaStream_t) for everything the ctx launches; NULL restores the
 * ctx's own stream.  Lets a host time the ctx's kernels with its own events. */
int dsgd_set_stream(dsgd_ctx *ctx, void *cuda_stream);
int dsgd_synchronize(dsgd_ctx *ctx);
/* CUDA-event stopwatch on the ctx's launch stream (what bench.py times kernels with). */
int dsgd_timer_start(dsgd_ctx *ctx);
int dsgd_timer_stop(dsgd_ctx *ctx, float *elapsed_ms);
/* Number of kernels this ctx has launched so far (bench.py's gpu_launches). */
int dsgd_launch_count(const dsgd_ctx *ctx, int64_t *count);

/* Kernel stopwatch for the roofline figure: between begin and end, every sample_every-th launch of the
 * gradient kernel (the dominant kernel of a step) is bracketed by CUDA events on the launch stream; end
 * returns their mean duration and how many launches were sampled. */
int dsgd_profile_begin(dsgd_ctx *ctx, int32_t sample_every);
int dsgd_profile_end(dsgd_ctx *ctx, float *mean_ms, int64_t *n_sampled);
/* Optional: allocate every device buffer the sync path needs for calls of up to n_samples sample ids and n_steps steps
 * now (staging, per-step losses and learning rates, the persistent kernel's buffers, the exchange's weight words) instead of on first
 * use.  cudaMalloc synchronises the whole device: a host that drives several contexts on ONE GPU from several threads
 * must reserve before the first fused step, or a rank allocating late waits for a rank that already runs and waits for
 * it.  (One context per GPU never needs this.) */
int dsgd_reserve(dsgd_ctx *ctx, int64_t n_samples, int64_t n_steps);
/* CTAs of the persistent sync kernel (0 = one per SM, the default and the fastest).  The kernel is cooperative and its
 * ranks wait for each other, so K contexts that share ONE GPU (the K-rank tests on a single-GPU box: tests/
 * test_gpu_fused_one_gpu.py) must each take at most 1/K of the SMs. */
int dsgd_set_grid_limit(dsgd_ctx *ctx, int32_t n_ctas);
/* Developer aid (tools/timeline.py): with the environment variable DSGD_PERSIST_TIMELINE set, the persistent sync kernel
 * stamps clock64 per phase (CTA 0, 256 steps x 16 slots) and, for steps 100..103, {barrier arrival ns, barrier exit ns,
 * pairs of the CTA's rows, chunks of the rows | (rows of more than one chunk << 32)} per CTA; this copies the last launch's DSGD_TIMELINE_WORDS int64 words out. */
#define DSGD_TIMELINE_WORDS (256 * 16 + 4 * 160 * 4)
int dsgd_debug_timeline(dsgd_ctx *ctx, long long *out);
/* Diagnostic: rows the streaming pass (forward / gradient / eval / sampled eval of 2048 rows or more) recomputed in fp64
 * because the sign of their fp32 dot product was inside the rounding band; cumulative since dsgd_create, every streaming
 * pass counted. */
int dsgd_stream_exact_rows(dsgd_ctx *ctx, int64_t *rows);

/* ---- data: the `data: Array[(Vec, Int)]` constructor argument (core/Slave.scala:20; Main.scala:138,149).
 *      Rows are repacked on the device into 16-byte aligned (col, val) windows.  label in {-1, +1}.  A row is
 *      a Map in the reference: a column repeated within one row (in any order) is DSGD_ERR_INVALID; columns
 *      need not be sorted.  A reload drops a staged sample stream (dsgd_stage_samples): its ids named the previous
 *      rows, so stage again before dsgd_sync_steps_staged. ------------------------------------------------------ */
int dsgd_load_csr(dsgd_ctx *ctx, int64_t n_rows, int64_t nnz, const int64_t *row_ptr, const int32_t *col,
                  const float *val, const int8_t *label);

/* ---- model: SparseSVM.dimSparsity (core/ml/SparseSVM.scala:11).  d is given in the WEIGHT index space. */
int dsgd_set_dim_sparsity(dsgd_ctx *ctx, const double *d);
/* Main.scala:54-65 on the device: inverse (document frequency + 1) over rows [0, n_train), including the
 * reference's off-by-one key shift (quirk Q3).  Installs the result; d_out (optional) receives a copy. */
int dsgd_compute_dim_sparsity(dsgd_ctx *ctx, int64_t n_train, double *d_out);

/* ---- resident weights: GradState.grad on the master (core/ml/GradState.scala:6), `weights` Ref on an
 *      async slave (core/Slave.scala:30).  w == NULL in a request below (forward, gradient, every evaluation) reads
 *      the resident weights.  On a DSGD_FLAG_ASYNC ctx it reads a snapshot of the replica taken when the call starts,
 *      exactly as if that snapshot had been passed as w: dsgd_update_grad, a peer's pushes and a loop that ended by
 *      itself on max_updates change the replica between calls. ---------------------------------------------- */
int dsgd_set_weights(dsgd_ctx *ctx, const double *w);
int dsgd_get_weights(dsgd_ctx *ctx, double *w);

/* ---- SlaveImpl.forward (core/Slave.scala:129-140; SparseSVM.scala:14): preds[i] = -signum(x_i . w).
 *      w == NULL: use the resident weights.  The ids go to a buffer of their own, as those of every request do: a
 *      sample stream staged with dsgd_stage_samples is left intact (this holds for dsgd_gradient too). ---------- */
int dsgd_forward(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *preds_out);

/* ---- SlaveImpl.gradient (core/Slave.scala:142-157; SparseSVM.scala:26-31): grad_out[dim] =
 *      regularize(sum_i backward(w, x_i, y_i), w).  loss_out (optional) = SparseSVM.loss(w, these samples)
 *      (SparseSVM.scala:20-23).  w == NULL: resident weights.  n == 0 -> DSGD_ERR_EMPTY. -------------------- */
int dsgd_gradient(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *grad_out,
                  double *loss_out);

/* ---- Master.localLoss / localAccuracy over rows [row_begin, row_end) (core/Master.scala:100-107): one
 *      streaming pass; loss = lambda*||w||^2 + mean hinge, acc = #{pred == y} / n. ------------------------- */
int dsgd_eval(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *loss_out,
              double *acc_out);

/* Sharded form of the same pass: the exact integer sums (hinge losses are 0, 1 or 2 per sample) and
 * ||w||^2, so that a host can combine row shards evaluated on different GPUs without rounding. */
int dsgd_eval_counts(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *hinge_sum,
                     int64_t *correct, double *norm_squared);

/* ---- Master.localSampledLoss / localSampledAccuracy (core/Master.scala:109-118) on a sample drawn on the device:
 *      position i of the draw is row row_begin + dsgd_feistel(i, half_bits(n), key, n), n = row_end - row_begin, a keyed
 *      permutation of the range (`Random.shuffle(indices) take k` without a shuffle, dsgd_feistel.h).  Evaluates positions
 *      [pos_begin, pos_end), so ranks that draw with the same key can split one sample between them; returns the same
 *      exact counters as dsgd_eval_counts.  w == NULL: resident weights.  The drawn ids go to a buffer of their own: a
 *      sample stream staged with dsgd_stage_samples is left intact.  Errors: no rows loaded -> DSGD_ERR_STATE; range
 *      outside the loaded rows -> DSGD_ERR_RANGE; n == 0 or pos_end <= pos_begin -> DSGD_ERR_EMPTY; pos_begin < 0,
 *      pos_end > n, or n >= 2^32 -> DSGD_ERR_INVALID. */
int dsgd_eval_sampled_counts(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                             int64_t pos_begin, int64_t pos_end, int64_t *hinge_sum, int64_t *correct,
                             double *norm_squared);
/* The same counters over a caller's list of n row ids; repeats are allowed and every occurrence counts.  For a host that
 * draws the sample itself (the JVM-exact draw, or a JVM master using its own Random).  n == 0 -> DSGD_ERR_EMPTY; an id
 * outside the loaded rows -> DSGD_ERR_RANGE before anything is launched.  The staged sample stream is left intact. */
int dsgd_eval_samples_counts(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, int64_t *hinge_sum,
                             int64_t *correct, double *norm_squared);
/* The three *_counts calls above report the hinge sum as an integer, which only the SVM has: on a ctx of any other model they
 * fail with DSGD_ERR_STATE.  The *_sums forms take the same arguments and report the sum of the per-sample losses as a double
 * instead, for either model (for the SVM, the hinge sum: an exact integer held in a double).  The logistic sum is added in
 * fixed point on the device, so a pass returns the same bits whatever the order in which its rows are taken. */
int dsgd_eval_sums(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *loss_sum, int64_t *correct,
                   double *norm_squared);
int dsgd_eval_sampled_sums(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                           int64_t pos_begin, int64_t pos_end, double *loss_sum, int64_t *correct, double *norm_squared);
int dsgd_eval_samples_sums(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *loss_sum,
                           int64_t *correct, double *norm_squared);

/* ---- scores and ranking metrics, for either model.  The conventions of the evaluations above: w == NULL reads the resident
 *      weights (on an async ctx, a snapshot taken when the call starts); the ids go to a buffer of their own, so a staged
 *      sample stream is left intact; no rows loaded -> DSGD_ERR_STATE; an id or a range outside the loaded rows ->
 *      DSGD_ERR_RANGE, before anything is launched; n == 0 (an empty range, no positions) -> DSGD_ERR_EMPTY; a NULL output
 *      -> DSGD_ERR_INVALID.  The dot product x_i . w is the row fold (Conventions), the one that decides the row on every
 *      other path, and the metrics rank exactly the values dsgd_margins returns for the same rows. ---- */
/* margins_out[i] = x_i . w in fp64 (the value whose -signum dsgd_forward reports) */
int dsgd_margins(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *margins_out);
/* SparseLogistic: probs_out[i] = P(y = +1 | x_i) = sigmoid(-x_i . w), with the sigmoid of the logistic gradient;
 * SparseModifiedHuber: (clip(-x_i . w, -1, 1) + 1) / 2.  An SVM or squared-hinge ctx -> DSGD_ERR_STATE (its margins are not
 * probabilities). */
int dsgd_probabilities(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *probs_out);

#define DSGD_METRICS_WORDS 8
/* out[0] TP  (y=+1, pred=+1)   out[1] FN (y=+1, pred=-1)   out[2] y=+1 with no +-1 prediction (x.w == 0 or NaN)
 * out[3] FP  (y=-1, pred=+1)   out[4] TN (y=-1, pred=-1)   out[5] y=-1 with no +-1 prediction
 * out[6] U2 = sum over (positive, negative) pairs of 2*[s_pos > s_neg] + [s_pos == s_neg], s = -x.w, NaN rows left out
 * out[7] rows whose score is NaN
 * pred is dsgd_forward's prediction, so out[0] + out[4] is the `correct` of dsgd_eval_* over the same rows.  A NaN row has no
 * prediction: it counts in out[2] or out[5] and in out[7].  +0 and -0 are one score.  Every word is an exact integer, whatever
 * the grid or the row order.  ROC AUC = U2 / (2 P N), P = out[0] + out[1] + out[2] positive rows, N = out[3] + out[4] + out[5]
 * negative rows; it is undefined (NaN) when out[7] > 0 or P or N is 0.
 * The sampled form draws as dsgd_eval_sampled_counts (its further errors are that call's); the list form counts a repeated id
 * every time and takes at most 2^31 - 1 ids (DSGD_ERR_INVALID), so U2 <= 2 (n/2)^2 fits in int64.  A pass sorts the scores: it
 * grows its buffers (two 8-byte keys per row and the sort's storage) on first use, like the other requests. */
int dsgd_eval_metrics(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *out);
int dsgd_eval_sampled_metrics(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                              int64_t pos_begin, int64_t pos_end, int64_t *out);
int dsgd_eval_samples_metrics(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, int64_t *out);

/* ---- Topics: one-vs-rest labels of a multi-label data set (DESIGN.md §4.21).  Sync mode only.
 *      dsgd_load_topics: the topics of every loaded row as a CSR: row r has the ids topic_id[topic_ptr[r] .. topic_ptr[r+1]),
 *      strictly ascending, each in [0, n_topics); topic_ptr holds n_rows + 1 entries, topic_ptr[0] = 0, and topic_ptr[n_rows]
 *      is the id count.  Everything is checked on the host before anything changes on the device: a topic_ptr that is not
 *      monotone or does not start at 0, an id outside [0, n_topics), ids of a row not strictly ascending, or n_topics outside
 *      [1, DSGD_MAX_TOPICS] -> DSGD_ERR_INVALID; no rows loaded or an async ctx -> DSGD_ERR_STATE.  The ctx keeps a copy of
 *      the labels dsgd_load_csr loaded; loading topics again first restores them.  dsgd_load_csr drops the topics.
 *      dsgd_select_topic(t): label(r) = +1 when row r has topic t, else -1, for every row, and the streaming pass's
 *      per-row word follows (its sign is the label).  t = -1: the labels dsgd_load_csr loaded.  Every training and
 *      evaluation path reads the labels when it launches, so after the call every one of them sees exactly the labels a
 *      ctx freshly loaded with them would.  No topics loaded or an async ctx -> DSGD_ERR_STATE; t outside [-1, T) ->
 *      DSGD_ERR_INVALID.
 *      dsgd_eval*_topics: W holds n_topics weight vectors of the weight length (dim, or dim + 1 with the intercept last),
 *      W_t = W[t * wlen .. (t + 1) * wlen), each the w a caller would pass to dsgd_margins.  Over the rows of the request
 *      (the three row forms of the metrics calls, with their errors), with y_t = +1 when the row has topic t (from the
 *      loaded topics, never from the current labels) and p_t the prediction of dsgd_forward for W_t:
 *        out[8 t .. 8 t + 8)  the DSGD_METRICS_WORDS of dsgd_eval_metrics for the labels y_t and the weights W_t, except
 *                             out[8 t + 6] (U2), which is 0
 *        out[8 T + 0]         rows
 *        out[8 T + 1]         rows with p_t = y_t for every t (p = 0 is never right)
 *        out[8 T + 2]         rows with a topic whose top-scored topic is one of theirs: the top-scored topic has the lowest
 *                             x . W_t among the non-NaN scores (the highest score -x . W_t), ties to the lowest t
 *        out[8 T + 3]         rows with no topic
 *        out[8 T + 4]         rows with no non-NaN score
 *        out[8 T + 5 .. 8)    0
 *      Every word is an exact integer, the same whatever the grid or the row order.  n_topics other than the loaded T or a
 *      NULL W or out -> DSGD_ERR_INVALID; no topics loaded or an async ctx -> DSGD_ERR_STATE; all before anything is
 *      launched.  A call copies T * wlen doubles to the device. */
#define DSGD_MAX_TOPICS 1024
#define DSGD_TOPIC_WORDS(T) (8 * (int64_t)(T) + 8)
int dsgd_load_topics(dsgd_ctx *ctx, int32_t n_topics, const int64_t *topic_ptr, const int32_t *topic_id);
int dsgd_select_topic(dsgd_ctx *ctx, int32_t topic);
int dsgd_eval_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, int64_t row_begin, int64_t row_end, int64_t *out);
int dsgd_eval_sampled_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, int64_t row_begin, int64_t row_end,
                             uint64_t key, int64_t pos_begin, int64_t pos_end, int64_t *out);
int dsgd_eval_samples_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, const int32_t *samples, int64_t n,
                             int64_t *out);

/* ---- Per-topic decision thresholds (DESIGN.md §4.23).  Sync mode only.  For a row and topic t, m_t is the margin
 *      dsgd_margins returns for W_t, bit for bit (fl(x . W_t + filt(beta_t)) on an intercept ctx).  The thresholded rule at
 *      tau_t: p_t = +1 (present) when m_t < tau_t, -1 when m_t > tau_t, and 0 (no prediction) when m_t == tau_t or m_t is
 *      NaN; at tau = +-0 it is dsgd_forward's prediction.
 *      dsgd_tune_topic_thresholds*: SCut, the F1-optimal threshold of every topic over the rows of the request (the three
 *      row forms of the metrics calls; a list counts repeats every time).  For topic t, P = rows with topic t (from the
 *      loaded topics, never the current labels; NaN-margin rows included) and c_0 < ... < c_(D-1) its distinct non-NaN
 *      margins (+0 and -0 are one).  Candidate j predicts present the pp_j rows with m <= c_j, tp_j of them with the topic;
 *      its threshold is tau_j = mid = fl(c_j / 2 + c_(j+1) / 2) when c_j < mid <= c_(j+1), else c_(j+1), and tau_(D-1) =
 *      +inf.  The best candidate has the highest F1_j = 2 tp_j / (P + pp_j), compared exactly, ties to the lowest j.
 *      Status (word 6) and thresholds_out[t]:
 *        0 tuned          tau of the best candidate
 *        1 no positive    P = 0 (and D > 0): tau = 0, j = -1
 *        2 below fbr      fl(2 tp / (P + pp)) < fbr for the best candidate: tau_0 (SCutFBR.1), j = 0
 *        3 no margin      D = 0 (no non-NaN margin, or no row): tau = 0, j = -1
 *      words_out holds DSGD_TOPIC_TUNE_WORDS(T) int64 words, eight per topic at 8 t: rows, P, rows with a NaN margin, D, then
 *      tp and rows predicted present by the thresholded rule at thresholds_out[t] over the same rows, the status and j.  At
 *      tau_j the rule predicts candidate j's rows, except a last candidate at c = +inf, whose rows at +inf sit at tau = +inf
 *      and get no prediction.  Every output has the same bits for a multiset of rows whatever the grid, the row order, the
 *      form or the topic grouping.  The errors of dsgd_eval*_topics, a NULL output, and fbr NaN or outside [0, 1] ->
 *      DSGD_ERR_INVALID, all before anything is launched or grown.  Rows are replicated on every rank, and a call tunes over
 *      its whole request.  The topics go in groups of G = max(1, min(T, floor(2^27 / n))) over n positions: the call keeps
 *      18 G n bytes of device workspace.
 *      dsgd_eval*_thresholded_topics: the words of dsgd_eval*_topics with p_t by the thresholded rule at thresholds[t]; the
 *      exact-match word (8 T + 1) uses these p_t, the top-1 word (8 T + 2) still ranks the raw margins.  Its errors, a NULL
 *      thresholds or a NaN threshold (+-inf are allowed) -> DSGD_ERR_INVALID, all before anything is launched. */
#define DSGD_TOPIC_TUNE_WORDS(T) (8 * (int64_t)(T))
int dsgd_tune_topic_thresholds(dsgd_ctx *ctx, const double *W, int32_t n_topics, double fbr, int64_t row_begin,
                               int64_t row_end, double *thresholds_out, int64_t *words_out);
int dsgd_tune_topic_thresholds_sampled(dsgd_ctx *ctx, const double *W, int32_t n_topics, double fbr, int64_t row_begin,
                                       int64_t row_end, uint64_t key, int64_t pos_begin, int64_t pos_end,
                                       double *thresholds_out, int64_t *words_out);
int dsgd_tune_topic_thresholds_samples(dsgd_ctx *ctx, const double *W, int32_t n_topics, double fbr,
                                       const int32_t *samples, int64_t n, double *thresholds_out, int64_t *words_out);
int dsgd_eval_thresholded_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, const double *thresholds,
                                 int64_t row_begin, int64_t row_end, int64_t *out);
int dsgd_eval_sampled_thresholded_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, const double *thresholds,
                                         int64_t row_begin, int64_t row_end, uint64_t key, int64_t pos_begin,
                                         int64_t pos_end, int64_t *out);
int dsgd_eval_samples_thresholded_topics(dsgd_ctx *ctx, const double *W, int32_t n_topics, const double *thresholds,
                                         const int32_t *samples, int64_t n, int64_t *out);

/* ---- Ranking a row's topics (DESIGN.md §4.22).  Sync mode only.  For a row and topic t, m_t is the margin dsgd_margins
 *      returns for W_t, bit for bit (fl(x . W_t + filt(beta_t)) on an intercept ctx), and its score is s_t = -m_t: a higher
 *      score ranks first, and +0 and -0 are one score.  Y is the row's loaded topics (never the current labels), n_Y = |Y|.
 *      The order is the topics sorted by s descending, ties to the lower t; top_j is its first j topics.
 *      rank_l = #{u : s_u >= s_l} (ties count against the row) and L_l = #{u in Y : s_u >= s_l}.  A row is ranked when
 *      n_Y >= 1 and none of its T scores is NaN.
 *      dsgd_eval*_topic_ranking: W and n_topics as dsgd_eval*_topics, 1 <= k <= min(T, DSGD_TOPIC_RANK_MAX_K), the rows in
 *      the three forms of the metrics calls.  words_out holds DSGD_TOPIC_RANK_WORDS(k) int64 words:
 *        words[0]              rows
 *        words[1]              ranked rows, N
 *        words[2]              rows with a NaN score
 *        words[3]              rows with no topic and no NaN score (words[0] = words[1] + words[2] + words[3])
 *        words[4]              ranked rows with n_Y = T (they have no ranking-loss pair)
 *        words[5]              sum over ranked rows of max over l in Y of rank_l (coverage)
 *        words[6]              sum over ranked rows and l in Y of rank_l - L_l: mis-ordered (own, other) pairs, ties counted
 *        words[7]              0
 *        words[8 + j - 1]      sum over ranked rows of |top_j intersect Y|, j = 1 .. k
 *      then 2 + k fixed-point sums in blocks of 7 words each (limbs 0..5, limb i worth
 *      2^(40 i - 160), the carries propagated so that limbs 0..4 lie in [0, 2^40), then an overflow count), in the order
 *        A    over ranked rows and l in Y: fl(L_l / (rank_l n_Y))
 *        B    over ranked rows with n_Y < T: fl(p_r / (n_Y (T - n_Y))), p_r the row's share of words[6]
 *        C_j  for j = 1 .. k, over ranked rows: fl(|top_j intersect Y| / n_Y)
 *      Each term is one IEEE division of two exact integers, summed exactly at a resolution of 2^-160 as the logistic loss
 *      sum is; sums_out[2 + k] holds each block's value, converted as that sum's reader converts it.  Every output has the
 *      same bits for any grid, row order or split, and limbs added over several calls (as float64 too: every limb is below
 *      2^40) give, once the carries are propagated, the limbs of one call over all their rows.  The errors of
 *      dsgd_eval*_topics, and a k outside [1, min(T, DSGD_TOPIC_RANK_MAX_K)] -> DSGD_ERR_INVALID, before any launch.
 *      dsgd_topics_topk: for the listed rows (no topics need be loaded: a model can rank new rows), ids_out[i k .. i k + k)
 *      holds the first k topics of the order over row samples[i]'s non-NaN scores and margins_out their margins, with the
 *      bits of dsgd_margins; slots past the non-NaN count hold -1 and NaN.  n_topics outside [1, DSGD_MAX_TOPICS], a bad k
 *      or a NULL array -> DSGD_ERR_INVALID; an async ctx -> DSGD_ERR_STATE; the list's errors as dsgd_margins; all before
 *      any launch. */
#define DSGD_TOPIC_RANK_MAX_K 32
#define DSGD_TOPIC_RANK_WORDS(k) (8 + (int64_t)(k) + 7 * (2 + (int64_t)(k)))
int dsgd_eval_topic_ranking(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k, int64_t row_begin, int64_t row_end,
                            int64_t *words_out, double *sums_out);
int dsgd_eval_sampled_topic_ranking(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k, int64_t row_begin,
                                    int64_t row_end, uint64_t key, int64_t pos_begin, int64_t pos_end, int64_t *words_out,
                                    double *sums_out);
int dsgd_eval_samples_topic_ranking(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k, const int32_t *samples,
                                    int64_t n, int64_t *words_out, double *sums_out);
int dsgd_topics_topk(dsgd_ctx *ctx, const double *W, int32_t n_topics, int32_t k, const int32_t *samples, int64_t n,
                     int32_t *ids_out, double *margins_out);

/* ---- ROC and precision-recall curves and average precision over the same three row forms, with the conventions and errors
 *      of the metrics calls above.  Over the non-NaN rows, let t_0 > t_1 > ... > t_(m-1) be the distinct scores s = -x.w
 *      (+0 and -0 are one score).  Point k: thr_out[k] = t_k (a zero score as +0), tp_out[k] = positive rows with s >= t_k,
 *      fp_out[k] = negative rows with s >= t_k; the last point counts every non-NaN positive and negative.  ROC is
 *      (fp / N, tp / P), precision-recall is (tp / (tp + fp), tp / P).  *n_points_out = m <= n, the rows of the request.
 *      words_out receives the DSGD_METRICS_WORDS words of the metrics call over the same rows, bit for bit.
 *      *ap_out = average precision, the step-wise sum of (R_k - R_(k-1)) Prec_k: every non-NaN positive row i adds
 *      v_i = tp_i / (tp_i + fp_i), one IEEE division of the counts at its own score; the v_i are added exactly in fixed point
 *      (the result is within one ulp of the exact sum, and equal to it when that is a double), and AP = S / P.  AP is NaN when
 *      a score is NaN or P = 0, and 1 when N = 0.  So AP has the same bits whatever the row order or the grid.
 *      thr_out, tp_out and fp_out hold at least n entries each, or are all NULL: then only the words, AP and m are computed,
 *      and nothing of size n is copied back.  Any other mix, or a NULL words_out, ap_out or n_points_out ->
 *      DSGD_ERR_INVALID.  The list form takes at most 2^31 - 1 ids.  A pass grows its buffers (about 52 bytes per row and the
 *      sort's, merge's and scan's storage) on first use, except on an async ctx, whose first loop start sizes them. */
int dsgd_eval_curve(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *words_out, double *ap_out,
                    int64_t *n_points_out, double *thr_out, int64_t *tp_out, int64_t *fp_out);
int dsgd_eval_sampled_curve(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                            int64_t pos_begin, int64_t pos_end, int64_t *words_out, double *ap_out, int64_t *n_points_out,
                            double *thr_out, int64_t *tp_out, int64_t *fp_out);
int dsgd_eval_samples_curve(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, int64_t *words_out,
                            double *ap_out, int64_t *n_points_out, double *thr_out, int64_t *tp_out, int64_t *fp_out);

/* ---- Poisson bootstrap of the test metrics over the same three row forms (DESIGN.md §4.19).  Position i of a request is
 *      r - row_begin (range), the index p - pos_begin of draw position p (sampled) or the list index (list): two calls over the
 *      same rows with the same bkey resample them identically, whatever weights they score.  Replicate b gives position i the
 *      multiplicity m_i(b) = #{k in 0..19 : u >= T_k}, u = H(bkey, b, i), T_k = floor(F(k) 2^64), F the Poisson(1) CDF (m <=
 *      20; the draw and the T_k are in distributed_sgd_b200/csrc/dsgd_bootstrap.h).  Replicate b is defined as the unweighted
 *      evaluation of the expanded list -- the request's ids with position i repeated m_i(b) times, in position order -- and
 *      for each b in [b_begin, b_end), at index j = b - b_begin:
 *        words_out[9 j + 0 .. 7]  the DSGD_METRICS_WORDS of dsgd_eval_samples_metrics over the expanded list, bit for bit
 *        words_out[9 j + 8]       sum of m_i(b), the replicate's size
 *        ap_out[j]                *ap_out of dsgd_eval_samples_curve over the expanded list, bit for bit (NaN when a score
 *                                 is NaN or the replicate has no positive)
 *        loss_out[j]              the loss sum of dsgd_eval_samples_sums over the expanded list, bit for bit (the SVM's
 *                                 integer hinge sum; the fixed-point sum of the other models, NaN as there)
 *      A replicate's bits do not depend on the grid, the row order or which other replicates the call computes.  The pass is
 *      unweighted: class and sample weights are not read.  All four models, with or without an intercept; the scores are
 *      those dsgd_margins returns.  Errors: a NULL output, b_begin < 0, or a request of more than 2^26 rows ->
 *      DSGD_ERR_INVALID; b_end <= b_begin -> DSGD_ERR_EMPTY; an async ctx while its loop runs -> DSGD_ERR_STATE; all before
 *      anything is launched.  Otherwise the errors and the w == NULL convention are those of the metrics calls.  A pass grows
 *      its buffers (about 36 bytes per row, 52 for the models other than the SVM, and the sort's storage) on first use. */
#define DSGD_BOOTSTRAP_WORDS 9
int dsgd_eval_bootstrap(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t bkey, int64_t b_begin,
                        int64_t b_end, int64_t *words_out, double *ap_out, double *loss_out);
int dsgd_eval_sampled_bootstrap(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                int64_t pos_begin, int64_t pos_end, uint64_t bkey, int64_t b_begin, int64_t b_end,
                                int64_t *words_out, double *ap_out, double *loss_out);
int dsgd_eval_samples_bootstrap(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, uint64_t bkey,
                                int64_t b_begin, int64_t b_end, int64_t *words_out, double *ap_out, double *loss_out);

/* ---- weighted curves: the curve calls above with every row counted by its weight, on any sync ctx and for either model.
 *      Rows, the three row forms, s = -x.w, NaN handling, ties and the m points are exactly those of dsgd_eval_curve.  Row
 *      i's weight is c_i = fl(w_y * s_i), the class weight of its label times its sample weight (dsgd_set_class_weights,
 *      dsgd_set_sample_weights): without sample weights c_i = w_y, and with class weights (1, 1) as well c_i = 1.
 *      R(v) is the fixed-point cut of the loss sums (resolution 2^-160; a value of 2^52 or more, or a NaN, makes its sum
 *      NaN), and read() converts an exact sum of R values to a double: it depends only on the exact value, so every word has
 *      the same bits whatever the row order, the grid or the rank.  W+(>= t) = read(sum R(c_i)) over the non-NaN positive
 *      rows with s >= t; W+(< t), W+(= t) and the W- forms over the negative rows likewise.
 *      wsums_out[0..12] (DSGD_WCURVE_WORDS), each one read() of one exact sum:
 *        0 TP weight (positives, s > 0: pred +1)   1 FN weight (s < 0)   2 positives with no prediction (s = +-0 or NaN)
 *        3 FP weight   4 TN weight   5 negatives with no prediction
 *        6 U2w = sum over the non-NaN positives of R(fl(c_i B_i)), B_i = read(2 W-(< s_i) + W-(= s_i))
 *        7 weight of the NaN-score rows
 *        8 S_ap = sum over the non-NaN positives with c_i > 0 of R(fl(c_i fl(T_i / (T_i + F_i)))), T_i = W+(>= s_i),
 *          F_i = W-(>= s_i); a zero-weight row adds exactly 0 to every sum and its precision is never formed
 *        9 weight of the correct rows (TP and TN as one sum)   10 sum of c_i over all rows
 *        11 W+ and 12 W-: the weight of all positive and of all negative rows, NaN scores included
 *      Weighted ROC AUC = U2w / (2 W+ W-), NaN when a score is NaN or W+ or W- is 0; weighted AP = S_ap / W+, NaN when a score
 *      is NaN or W+ = 0, and 1 when W- = 0.  Range: a product term of 2^52 or more makes its word NaN; U2w is finite while
 *      max c * 2 W- < 2^52.
 *      words_out receives the DSGD_METRICS_WORDS words of the metrics call over the same rows, bit for bit (counts, not
 *      weights).  *n_points_out = m; point k: thr_out[k] bit for bit that of dsgd_eval_curve (zero-weight rows still define
 *      points), tpw_out[k] = W+(>= t_k), fpw_out[k] = W-(>= t_k).  Recent scikit-learn versions drop zero-weight rows before
 *      they choose thresholds, so their curves can have fewer points; the areas agree.
 *      At c = 1: words 0..7 are the curve call's words as doubles (U2w = U2), S_ap has the limbs of its S (AP bit for bit)
 *      and tpw / fpw equal tp / fp.  With integer weights whose products stay below 2^53, U2w is the U2 of the id list in
 *      which row i appears c_i times.  Words 9 and 10 are dsgd_eval_weighted's sums_out[1] and sums_out[2], bit for bit.
 *      thr_out, tpw_out and fpw_out hold at least n entries each, or are all NULL (then only the words are computed).  The
 *      errors are those of dsgd_eval_curve; an async ctx -> DSGD_ERR_STATE before anything is launched.  A pass grows its
 *      buffers (the curve call's and 72 bytes more per row: c, its sort alternate and the prefix sums) on first use. */
#define DSGD_WCURVE_WORDS 13
int dsgd_eval_weighted_curve(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *words_out,
                             double *wsums_out, int64_t *n_points_out, double *thr_out, double *tpw_out, double *fpw_out);
int dsgd_eval_sampled_weighted_curve(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                     int64_t pos_begin, int64_t pos_end, int64_t *words_out, double *wsums_out,
                                     int64_t *n_points_out, double *thr_out, double *tpw_out, double *fpw_out);
int dsgd_eval_samples_weighted_curve(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, int64_t *words_out,
                                     double *wsums_out, int64_t *n_points_out, double *thr_out, double *tpw_out,
                                     double *fpw_out);

/* ---- weighted bootstrap: the Poisson bootstrap above with every row counted by its weight c_i = fl(w_y * s_i), the weight
 *      of the weighted curves (DESIGN.md §4.20).  The rows, positions, multiplicities m_i(b) and expanded lists are those of
 *      dsgd_eval*_bootstrap: a weighted and an unweighted call with the same bkey resample the same rows.  Replicate b is
 *      defined as the weighted calls over its expanded list, every copy of row i weighing c_i; for each b in [b_begin, b_end),
 *      at index j = b - b_begin:
 *        words_out[2 j]             sum of m_i(b), the rows of the expanded list (the weighted loss's divisor)
 *        words_out[2 j + 1]         its NaN-score rows (word 7 of dsgd_eval_samples_metrics over it)
 *        wsums_out[13 j + 0 .. 12]  the DSGD_WCURVE_WORDS of dsgd_eval_samples_weighted_curve over it, bit for bit
 *        loss_out[j]                sums_out[0] of dsgd_eval_samples_weighted over it, S = sum R(fl(c_i L_i)), bit for bit
 *      NaN follows those calls: a term of 2^52 or more, inf or NaN makes its word NaN.  With c = 1 the words 0..7, AP and the
 *      loss are the unweighted replicate's bit for bit, and words_out[2 j] is its size.  A replicate's bits do not depend on
 *      the grid, the row order or which other replicates the call computes.  All four models, with or without an intercept.
 *      Errors: a NULL output, b_begin < 0, or a request of more than 2^26 rows -> DSGD_ERR_INVALID; b_end <= b_begin ->
 *      DSGD_ERR_EMPTY; an async ctx -> DSGD_ERR_STATE; all before anything is launched.  Otherwise the errors and the
 *      w == NULL convention are those of the metrics calls.  A pass grows its buffers (about 48 bytes per row, 56 for the
 *      models other than the SVM, and the sort's storage) on first use. */
int dsgd_eval_weighted_bootstrap(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t bkey,
                                 int64_t b_begin, int64_t b_end, int64_t *words_out, double *wsums_out, double *loss_out);
int dsgd_eval_sampled_weighted_bootstrap(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                         int64_t pos_begin, int64_t pos_end, uint64_t bkey, int64_t b_begin, int64_t b_end,
                                         int64_t *words_out, double *wsums_out, double *loss_out);
int dsgd_eval_samples_weighted_bootstrap(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, uint64_t bkey,
                                         int64_t b_begin, int64_t b_end, int64_t *words_out, double *wsums_out,
                                         double *loss_out);

/* ---- calibration: scores into probabilities, for either model, over the same three row forms and with the conventions and
 *      errors of the metrics calls above.  With f = x_i . w exactly as dsgd_margins returns it, a calibration is a pair (A, B)
 *      and P(y = +1 | x_i) = 1 / (1 + exp(A f + B)), computed as sigmoid(-(A f + B)) with the sigmoid of the logistic gradient.
 *      A positive row has a negative x . w here, so a fitted A is normally positive, and the SparseLogistic model's own
 *      probability is the calibration (1, 0) bit for bit.
 *      dsgd_calibrate* fit (A, B) by Platt scaling as Lin, Lin and Weng (2007) state it: rows whose f is NaN are left out and
 *      counted; with N+ / N- the remaining positive / negative rows the targets are t = (N+ + 1) / (N+ + 2) and 1 / (N- + 2);
 *      Newton's method from (0, log((N- + 1) / (N+ + 1))) with a ridge of 1e-12 on the Hessian's diagonal, at most 100
 *      iterations, a backtracking line search (step 1 halved down to 1e-10, sufficient decrease 1e-4), stopping when both
 *      gradient components are below 1e-5.  The whole iteration is one cooperative kernel launch.  Every sum over the rows
 *      is added exactly in fixed point, so ab_out = {A, B}, *objective_out = F(A, B) and the iteration count have the same
 *      bits for a range, the same ids in any order, any grid limit and either model flag.
 *      info_out[0] Newton iterations (accepted steps)   info_out[1] status: 0 converged, 1 iteration limit, 2 the line search
 *      failed (A, B are the last accepted point), 3 a sum was not finite (a term NaN, infinite or >= 2^52: A, B and F are NaN)
 *      info_out[2] rows used   info_out[3] NaN rows left out   info_out[4] points evaluated (one grid barrier each)
 *      No positive or no negative row with a score -> DSGD_ERR_EMPTY.  While an async loop runs -> DSGD_ERR_STATE (a
 *      cooperative grid cannot share the device with a kernel that never ends); after dsgd_stop_async, or once the loop has
 *      ended by itself, the calls work.  A barrier that hits its watchdog -> DSGD_ERR_TIMEOUT. ---- */
#define DSGD_CALIBRATION_INFO_WORDS 5
int dsgd_calibrate(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *ab_out, double *objective_out,
                   int64_t *info_out);
int dsgd_calibrate_sampled(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key, int64_t pos_begin,
                           int64_t pos_end, double *ab_out, double *objective_out, int64_t *info_out);
int dsgd_calibrate_samples(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *ab_out,
                           double *objective_out, int64_t *info_out);
/* probs_out[i] = sigmoid(-(a x_i . w + b)); a or b not finite -> DSGD_ERR_INVALID.  On a SparseLogistic ctx (1, 0) returns
 * the bits of dsgd_probabilities.  Works beside a running async loop, like dsgd_margins. */
int dsgd_calibrated_probabilities(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double a, double b,
                                  double *probs_out);
/* Calibration quality at (a, b) over the rows whose z = a f + b is not NaN, with p = sigmoid(-z) and o = 1 for a positive row,
 * 0 otherwise:  sums_out[0] = sum (p - o)^2 (Brier)   sums_out[1] = sum of -log p (o = 1) or -log(1 - p) (o = 0), as the
 * stable softplus of the logistic loss;  n_bins (1 .. DSGD_CALIBRATION_MAX_BINS, else DSGD_ERR_INVALID) equal-width bins on
 * [0, 1], bin = min(n_bins - 1, floor(p n_bins)): bin_rows[k] rows, bin_pos[k] positive rows, bin_psum[k] = sum p (n_bins
 * entries each);  words_out[0] rows used, words_out[1] rows left out.  The counts are exact and the sums are added in fixed
 * point: the same bits in any row order.  Works beside a running async loop. */
#define DSGD_CALIBRATION_MAX_BINS 64
int dsgd_eval_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double a, double b,
                          int32_t n_bins, double *sums_out, int64_t *bin_rows, int64_t *bin_pos, double *bin_psum,
                          int64_t *words_out);
int dsgd_eval_sampled_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                  int64_t pos_begin, int64_t pos_end, double a, double b, int32_t n_bins, double *sums_out,
                                  int64_t *bin_rows, int64_t *bin_pos, double *bin_psum, int64_t *words_out);
int dsgd_eval_samples_calibration(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double a, double b,
                                  int32_t n_bins, double *sums_out, int64_t *bin_rows, int64_t *bin_pos, double *bin_psum,
                                  int64_t *words_out);

/* ---- weighted calibration: the Platt fit and its quality pass with every row counted by its weight (DESIGN.md §4.17), on
 *      any sync ctx and for any model.  Row i's weight is c_i = fl(w_y * s_i), exactly that of the weighted curves: without
 *      sample weights c_i = w_y, and with class weights (1, 1) as well c_i = 1.  To calibrate on sample weights alone after
 *      training with class weights, call dsgd_set_class_weights(ctx, 1, 1) first.  R(v) and read() are those of the weighted
 *      curves; every weighted total below is read() of one exact sum, so it has the same bits whatever the row order, the
 *      grid or the model flag.  A row has zero weight when R(c_i) = 0 (every c_i of 2^-161 or less): it adds exactly 0 to
 *      every sum, and no term of it is formed.
 *      dsgd_calibrate_weighted*: the fit of dsgd_calibrate* with W+ and W-, the weights of the positive and negative rows
 *      whose f is not NaN, in place of N+ and N-: targets (W+ + 1) / (W+ + 2) and 1 / (W- + 2), start (0, log((W- + 1) /
 *      (W+ + 1))) -- scikit-learn's weighted priors -- and each of the six sums over the rows adds R(fl(c_i term_i)).  A
 *      weighted term of 2^52 or more makes its sum non-finite (status 3), and so does a W+ or W- that is not finite.  The
 *      Newton, ridge, line-search and stop rules are those of dsgd_calibrate; the gradient bound stays 1e-5 in absolute
 *      terms, so large weights make status 2 likelier.  ab_out, objective_out and info_out as there (info_out[2] and [3]
 *      count rows, not weights); wsums_out[0..2] = {W+, W-, the weight of the NaN rows}.  W+ = 0 or W- = 0 ->
 *      DSGD_ERR_EMPTY (wsums_out is set).  An async ctx -> DSGD_ERR_STATE before anything is launched; a NULL output ->
 *      DSGD_ERR_INVALID.  A fit grows 8 bytes per row more than dsgd_calibrate's.  At c = 1 every output equals
 *      dsgd_calibrate's bit for bit. */
#define DSGD_CALIBRATION_WSUMS 3
int dsgd_calibrate_weighted(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *ab_out,
                            double *objective_out, int64_t *info_out, double *wsums_out);
int dsgd_calibrate_weighted_sampled(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                    int64_t pos_begin, int64_t pos_end, double *ab_out, double *objective_out,
                                    int64_t *info_out, double *wsums_out);
int dsgd_calibrate_weighted_samples(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *ab_out,
                                    double *objective_out, int64_t *info_out, double *wsums_out);
/* Weighted quality at (a, b), over the rows of dsgd_eval_calibration with its p, o, bins and arguments:
 *   sums_out[0] = sum R(fl(c (p - o)^2)) (Brier)   sums_out[1] = sum R(fl(c l)), l the log-loss term of dsgd_eval_calibration
 *   sums_out[2] = sum R(c) over the rows used       sums_out[3] = 0 (a sigmoid's term is never infinite)
 *   bin_weight[k] = sum R(c), bin_pos_weight[k] = the same over the positive rows, bin_psum[k] = sum R(fl(c p)), n_bins
 *   doubles each; a bin value of 2^52 or more makes that bin's three sums NaN, one elsewhere makes its sum NaN.
 *   words_out[0] rows used, words_out[1] rows left out: counts, as dsgd_eval_calibration's.
 * At c = 1 the sums and bin_psum equal dsgd_eval_calibration's bit for bit, and the bin weights its bin counts.  Errors are
 * those of dsgd_eval_calibration; an async ctx -> DSGD_ERR_STATE before anything is launched. */
#define DSGD_WCALIBRATION_SUMS 4
int dsgd_eval_weighted_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double a, double b,
                                   int32_t n_bins, double *sums_out, double *bin_weight, double *bin_pos_weight,
                                   double *bin_psum, int64_t *words_out);
int dsgd_eval_sampled_weighted_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                           int64_t pos_begin, int64_t pos_end, double a, double b, int32_t n_bins,
                                           double *sums_out, double *bin_weight, double *bin_pos_weight, double *bin_psum,
                                           int64_t *words_out);
int dsgd_eval_samples_weighted_calibration(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double a,
                                           double b, int32_t n_bins, double *sums_out, double *bin_weight,
                                           double *bin_pos_weight, double *bin_psum, int64_t *words_out);

/* ---- isotonic calibration: a non-parametric map from the score to a probability, for any model (DESIGN.md §4.16).  The
 *      rows, the three row forms, the score s = -x . w (f = x . w exactly as dsgd_margins returns it), NaN handling and the
 *      +0 / -0 rule are those of dsgd_eval_curve.
 *      Fit: the m distinct non-NaN scores t_0 > ... > t_(m-1) give the points P_k = (n_k, tp_k), n_k = tp_k + fp_k the rows
 *      with s >= t_k and tp_k the positive ones, and P_-1 = (0, 0).  The blocks are the segments of the upper concave hull of
 *      P_-1 .. P_(m-1); a hull vertex lies STRICTLY above the chord of its hull neighbours, so collinear points are not
 *      vertices, two adjacent blocks never have the same exact value, and the block list is unique.  A block is one hull
 *      segment and spans the distinct scores of the points after its left vertex up to its right one; its value is
 *      p_b = fl(positives / rows) of its rows, one IEEE division of two exact counts.  p_b does not increase as the score decreases: this is scikit-learn's
 *      IsotonicRegression(increasing=True, out_of_bounds="clip") fitted on (s, y in {0, 1}).  Every coordinate is an integer
 *      below 2^31 and every hull test an exact int64 cross product, so the outputs have one bit pattern for a multiset of
 *      rows, whatever the row form, the row order, the grid limit or the model flag.
 *      Outputs, ascending in s (scikit-learn's X_thresholds_ / y_thresholds_):  x_out: the lowest and the highest distinct
 *      score of every block (once when they are the same score; a zero score as +0);  y_out: the block's p_b at each;
 *      *n_points_out = k, their number (k <= m);  rows_out[j] / pos_out[j]: the rows and positive rows of block j
 *      (j ascending in s), so that p_j = fl(pos_out[j] / rows_out[j]).  Every output array holds at least n entries.
 *      info_out (DSGD_ISOTONIC_INFO_WORDS): [0] blocks  [1] points k  [2] rows used  [3] NaN rows left out  [4] distinct
 *      scores m.  A set of one class is valid (one block, p = 0 or 1); only "no row with a non-NaN score" ->
 *      DSGD_ERR_EMPTY.  A NULL output -> DSGD_ERR_INVALID.  The list form takes at most 2^31 - 1 ids.  The fit is a curve
 *      pass that leaves its points on the device, then the hull in parallel: tiles of DSGD_ISOTONIC_TILE points (an
 *      environment variable, 1 .. 2048, default 2048; the result does not depend on it) and ceil(log2 tiles) merge rounds.
 *      It grows the curve pass's buffers and about 52 bytes more per row on first use, except on an async ctx, whose first
 *      loop start sizes them; the launches count in dsgd_launch_count (the scans' own kernels do not). */
#define DSGD_ISOTONIC_INFO_WORDS 5
int dsgd_calibrate_isotonic(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *n_points_out,
                            double *x_out, double *y_out, int64_t *rows_out, int64_t *pos_out, int64_t *info_out);
int dsgd_calibrate_isotonic_sampled(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                    int64_t pos_begin, int64_t pos_end, int64_t *n_points_out, double *x_out, double *y_out,
                                    int64_t *rows_out, int64_t *pos_out, int64_t *info_out);
int dsgd_calibrate_isotonic_samples(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, int64_t *n_points_out,
                                    double *x_out, double *y_out, int64_t *rows_out, int64_t *pos_out, int64_t *info_out);
/* Apply: probs_out[i] = numpy.interp(s_i, X, Y) with s_i = -x_i . w and numpy's own arithmetic: a NaN s gives NaN; s <= X_0
 * gives Y_0 and s >= X_(k-1) gives Y_(k-1) (clip); else j with X_j <= s < X_(j+1) by binary search, s == X_j gives Y_j, and
 * otherwise slope (s - X_j) + Y_j with slope = (Y_(j+1) - Y_j) / (X_(j+1) - X_j); if that is NaN, slope (s - X_(j+1)) +
 * Y_(j+1); if that is NaN too and Y_j == Y_(j+1), Y_j.  The library is built without contraction, so this is numpy's
 * result bit for bit (numpy itself returns Y_0 for a NaN s when k == 1).  X must be finite and strictly increasing, Y in
 * [0, 1], k >= 1, else DSGD_ERR_INVALID.  Maps of up to 6144 points are held in shared memory, larger ones read through L2.
 * Works beside a running async loop once a map of k points or more has been applied on the ctx (else DSGD_ERR_STATE). */
int dsgd_isotonic_probabilities(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, const double *X,
                                const double *Y, int64_t k, double *probs_out);
/* Quality at the map (X, Y), with p = the value dsgd_isotonic_probabilities gives and o = 1 for a positive row, 0 otherwise,
 * over the rows whose s is not NaN: the outputs of dsgd_eval_calibration -- sums_out[0] the Brier sum, the bins as there --
 * with sums_out[1] = the sum of -log p (o = 1) or -log1p(-p) (o = 0) over the rows whose term is finite.  words_out
 * (DSGD_ISOTONIC_EVAL_WORDS): [0] rows used  [1] rows left out (NaN s)  [2] rows whose term is infinite (p = 0 with o = 1,
 * or p = 1 with o = 0): any such row makes the log loss +inf.  The map's checks are those of dsgd_isotonic_probabilities. */
#define DSGD_ISOTONIC_EVAL_WORDS 3
int dsgd_eval_isotonic_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, const double *X,
                                   const double *Y, int64_t k, int32_t n_bins, double *sums_out, int64_t *bin_rows,
                                   int64_t *bin_pos, double *bin_psum, int64_t *words_out);
int dsgd_eval_sampled_isotonic_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                           int64_t pos_begin, int64_t pos_end, const double *X, const double *Y, int64_t k,
                                           int32_t n_bins, double *sums_out, int64_t *bin_rows, int64_t *bin_pos,
                                           double *bin_psum, int64_t *words_out);
int dsgd_eval_samples_isotonic_calibration(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, const double *X,
                                           const double *Y, int64_t k, int32_t n_bins, double *sums_out, int64_t *bin_rows,
                                           int64_t *bin_pos, double *bin_psum, int64_t *words_out);

/* ---- weighted isotonic calibration: the isotonic fit and its quality pass with every row counted by its weight c_i, the
 *      weight of the weighted calibration calls above (DESIGN.md §4.17); on any sync ctx and for any model.
 *      Fit: the points are the distinct non-NaN scores t_0 > ... > t_(m-1) with the exact sums X_k = W(>= t_k) and
 *      Y_k = W+(>= t_k) of the weighted curve pass, and P_-1 = (0, 0).  A point whose weight increment X_k - X_(k-1) is
 *      exactly zero (only zero-weight rows at its score) is dropped before the hull, as scikit-learn drops zero-weight rows,
 *      so its score never enters X.  The blocks are the segments of the upper concave hull of the rest, with strict
 *      vertices as in dsgd_calibrate_isotonic; every coordinate is an integer in units of 2^-160 and every turn test an
 *      exact 512-bit comparison, so the outputs have one bit pattern for a multiset of (row, weight) whatever the row form,
 *      the row order, the grid limit, the tile size or the model flag.  A block's value is p_b = fl(read(dY) / read(dX));
 *      at c = 1 this is dsgd_calibrate_isotonic's fl(pos / rows) bit for bit, and every output equals that call's.
 *      Outputs as dsgd_calibrate_isotonic's, except: wrows_out[j] / wpos_out[j] the block's weight and positive weight (as
 *      doubles, read() of exact sums); info_out[2] the non-NaN rows of positive weight; info_out[4] the distinct scores
 *      among them (the points kept); wsums_out[0..1] = {W+, W-} of the non-NaN rows.  The turn test is exact while the total
 *      weight of the non-NaN rows is below 2^96 (2^64 and far more are accepted): 2^96 or more, or a c_i of 2^52 or more,
 *      -> DSGD_ERR_RANGE before the hull.  No non-NaN row of positive weight -> DSGD_ERR_EMPTY (one class is valid).  An
 *      async ctx -> DSGD_ERR_STATE before anything is launched; a NULL output -> DSGD_ERR_INVALID.  DSGD_ISOTONIC_TILE
 *      applies (the result does not depend on it).  A fit grows about 150 bytes per row more than the weighted curve pass.
 *      X and Y feed dsgd_isotonic_probabilities unchanged. */
int dsgd_calibrate_isotonic_weighted(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, int64_t *n_points_out,
                                     double *x_out, double *y_out, double *wrows_out, double *wpos_out, int64_t *info_out,
                                     double *wsums_out);
int dsgd_calibrate_isotonic_weighted_sampled(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                                             int64_t pos_begin, int64_t pos_end, int64_t *n_points_out, double *x_out,
                                             double *y_out, double *wrows_out, double *wpos_out, int64_t *info_out,
                                             double *wsums_out);
int dsgd_calibrate_isotonic_weighted_samples(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                             int64_t *n_points_out, double *x_out, double *y_out, double *wrows_out,
                                             double *wpos_out, int64_t *info_out, double *wsums_out);
/* Weighted quality at the map (X, Y): dsgd_eval_weighted_calibration's outputs with p and the log-loss term of
 * dsgd_eval_isotonic_calibration: sums_out[1] adds R(fl(c l)) over the finite terms, sums_out[3] = sum R(c) over the rows of
 * positive weight whose term is infinite (any such row makes the weighted log loss +inf), words_out
 * (DSGD_ISOTONIC_EVAL_WORDS) [2] = their number.  The map's checks are those of dsgd_isotonic_probabilities; an async ctx
 * -> DSGD_ERR_STATE. */
int dsgd_eval_weighted_isotonic_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, const double *X,
                                            const double *Y, int64_t k, int32_t n_bins, double *sums_out, double *bin_weight,
                                            double *bin_pos_weight, double *bin_psum, int64_t *words_out);
int dsgd_eval_sampled_weighted_isotonic_calibration(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end,
                                                    uint64_t key, int64_t pos_begin, int64_t pos_end, const double *X,
                                                    const double *Y, int64_t k, int32_t n_bins, double *sums_out,
                                                    double *bin_weight, double *bin_pos_weight, double *bin_psum,
                                                    int64_t *words_out);
int dsgd_eval_samples_weighted_isotonic_calibration(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n,
                                                    const double *X, const double *Y, int64_t k, int32_t n_bins,
                                                    double *sums_out, double *bin_weight, double *bin_pos_weight,
                                                    double *bin_psum, int64_t *words_out);

/* ---- communicator for sync mode: replaces the gRPC channels between master and slaves
 *      (core/package.scala:16-21; core/Master.scala:222-243).  Rank 0 makes an id, the host transports it
 *      (its own RPC), every rank calls dsgd_comm_init.  world == 1 needs neither. -------------------------- */
int dsgd_comm_unique_id(uint8_t id[DSGD_UNIQUE_ID_BYTES]);
int dsgd_comm_init(dsgd_ctx *ctx, const uint8_t id[DSGD_UNIQUE_ID_BYTES]);

/* Peer exchange for the FUSED multi-GPU step: each rank exports its receive area, the host transports the handles, every rank imports every other rank's.  Once all world-1 peers
 * are attached, sync steps with one worker per GPU run as one persistent kernel per call that sums the workers'
 * replies directly out of peer memory over NVLink (no NCCL call, no launch per step; only the non-zero entries of a
 * reply travel); otherwise the NCCL allreduce path is used, which needs dsgd_comm_init: without a communicator, a step
 * the fused kernel cannot take (batch above 32 x CTAs per rank, dim + 1 above 448 x CTAs, several workers on a rank)
 * fails with DSGD_ERR_STATE before anything is launched.  Up to 8 ranks (one NVSwitch box).  dsgd_xchg_attach is
 * the same-process form. */
int dsgd_xchg_export(dsgd_ctx *ctx, uint8_t handle[DSGD_IPC_HANDLE_BYTES]);
int dsgd_xchg_import(dsgd_ctx *ctx, int peer_rank, const uint8_t handle[DSGD_IPC_HANDLE_BYTES]);
int dsgd_xchg_attach(dsgd_ctx *ctx, int peer_rank, dsgd_ctx *peer);
/* Traffic of the fused step so far, for the NVLink figures of the bench: words this rank has stored into EACH peer's
 * receive area (a value word is 16 bytes on the wire -- one non-zero gradient entry --, a bitmap word 8 bytes -- which of
 * 32 columns were sent) and the SGD steps of those launches.  Any pointer may be NULL. */
int dsgd_xchg_stats(dsgd_ctx *ctx, int64_t *value_words, int64_t *bitmap_words, int64_t *steps);

/* ---- logical workers of a sync step.  Default: this ctx is ONE worker (its whole slice is one
 *      GradientRequest) and the master averages over `world` results.  With n_local > 1 the slice of every
 *      following step is cut into n_local consecutive requests of counts[v] samples, each with its own batch
 *      sum and its own regularize() support, exactly as if n_local slaves had answered (core/Slave.scala:
 *      147-155); k_total is the number of results the master averages (Vec.mean divisor, core/Master.scala:194
 *      -- the reference zips workers with split groups, so it can be smaller than the node count).
 *      n_local == 0: this rank only joins the exchange (a slave without a split group). ---------------- */
int dsgd_set_workers(dsgd_ctx *ctx, int32_t n_local, const int32_t *counts, int32_t k_total);

/* ---- one synchronous step of Master.fit (core/Master.scala:184-197): this rank's worker computes its
 *      regularized batch-sum gradient on `samples`, gradients are summed over ranks (allreduce over NVLink
 *      instead of K gRPC replies), and every rank applies w <- w - lr * (sum / world).  All ranks call it with
 *      their own slice.  loss_out (optional) = SparseSVM.loss(w_before, all samples of the step). ------------ */
int dsgd_sync_step(dsgd_ctx *ctx, const int32_t *samples, int64_t n, double lr, double *loss_out);
/* n_steps consecutive steps (the inner loop of an epoch, core/Master.scala:179): samples holds
 * n_steps * n_per_step indices, step-major.  losses_out (optional) holds n_steps values. */
int dsgd_sync_steps(dsgd_ctx *ctx, const int32_t *samples, int64_t n_per_step, int64_t n_steps, double lr,
                    double *losses_out);
/* The same with one learning rate per step (a decaying schedule inside one call): `lrs` holds n_steps rates in host
 * memory and step s uses lrs[s].  One call gives exactly what n_steps calls of dsgd_sync_steps would, each taking one
 * step with its scalar lrs[s]: weights, losses, the resident state and the averaging sum and count, bit for bit.  The
 * arguments are checked as in dsgd_sync_steps; lrs == NULL with n_steps > 0 -> DSGD_ERR_INVALID, an async ctx ->
 * DSGD_ERR_STATE; the rates themselves are not checked (nor is a scalar lr).  Every rank of a multi-rank step passes
 * the same table, as every rank passes the same scalar lr to dsgd_sync_steps.  The table is copied to the device on
 * the ctx's stream into a buffer that dsgd_reserve(.., n_steps) sizes in advance (K contexts sharing ONE GPU reserve
 * before their threads start stepping, as for the per-step losses). */
int dsgd_sync_steps_lr(dsgd_ctx *ctx, const int32_t *samples, int64_t n_per_step, int64_t n_steps, const double *lrs,
                       double *losses_out);
/* The same split in three, so a host can keep the index stream resident: stage = H2D of the sample slices
 * (the `samples` field of GradientRequest, protobuf/proto.proto:60-63); run = device only; read = D2H.  The stream stays
 * until the next dsgd_stage_samples, dsgd_sync_step or dsgd_sync_steps (which stage their own samples and so replace it)
 * or dsgd_load_csr (which drops it); the requests (forward, gradient, the evaluations) leave it intact. */
int dsgd_stage_samples(dsgd_ctx *ctx, const int32_t *samples, int64_t n);
int dsgd_sync_steps_staged(dsgd_ctx *ctx, int64_t first, int64_t n_per_step, int64_t n_steps, double lr,
                           int want_losses);
int dsgd_read_losses(dsgd_ctx *ctx, double *losses_out, int64_t n_steps);

/* ---- averaged SGD (Polyak-Ruppert) on the device, sync mode.  dsgd_average_begin zeroes a per-column fp64 sum A[dim] and
 *      a step count n; every sync step that runs after it, on any path (persistent, fused K-rank, per-step, logistic),
 *      then adds the weights after the step to A -- every column, whether the step changed it or not -- and 1 to n.  The
 *      starting weights of a call are not added.  Per column the additions happen in step order in plain fp64, so the sum
 *      does not depend on which path ran a step or on how the steps are split into calls.  dsgd_average_end stops the
 *      accumulation and keeps A and n.  dsgd_set_weights leaves both alone; a call of zero steps adds nothing.
 *      dsgd_average_weights: avg_out[j] = A[j] / n, with the 1e-20 filter of a new Sparse; n_steps_out = n; either
 *      pointer may be NULL.  Errors: an async ctx -> DSGD_ERR_STATE (every call); dsgd_average_weights before any
 *      dsgd_average_begin -> DSGD_ERR_STATE, with n == 0 -> DSGD_ERR_EMPTY.
 *      The first dsgd_average_begin allocates A with cudaMalloc, which synchronises the whole device: K contexts that
 *      share ONE GPU call it before their threads start stepping (see dsgd_reserve). ---------------------------------- */
int dsgd_average_begin(dsgd_ctx *ctx);   /* zero the sum and the count; average every following sync step */
int dsgd_average_end(dsgd_ctx *ctx);     /* stop averaging; the sum and the count stay readable */
int dsgd_average_weights(dsgd_ctx *ctx, double *avg_out, int64_t *n_steps_out);

/* ---- L1 penalty (lasso / elastic net) of the sync steps.  dsgd_set_l1 sets lambda1 >= 0 (0 at creation: every call then
 *      runs the kernels it ran without this option).  With lambda1 > 0 every sync step, on every path and for both models,
 *      first does what it does without the penalty -- u_j = filt(w_j - filt(mean_j * lr_t)) on the columns the step touched,
 *      u_j = w_j elsewhere -- and then takes the proximal step of lambda1 * ||w||_1 on EVERY column with tau = fl(lr_t *
 *      lambda1) (lr_t the scalar rate or lrs[t]):  w_j = u_j > tau ? filt(u_j - tau) : (u_j < -tau ? filt(u_j + tau) : 0),
 *      the 1e-20 filter of a new Sparse.  tau == 0 leaves u as it is.  c = 2 lambda (w . d), the averaging sum and the next
 *      step see the thresholded weights; the step's loss is lambda ||W||^2 + lambda1 ||W||_1 + loss sum / batch at the
 *      weights the gradient was taken at.  dsgd_gradient and every dsgd_eval_* call are unchanged (the penalty belongs to
 *      the step).  One worker on one GPU takes the persistent kernel's L1 form up to 32 rows per CTA, the per-step path
 *      above; the fused K-rank peer exchange has no L1 form, so with world > 1 a ctx with lambda1 > 0 needs dsgd_comm_init
 *      (a rank wired with the peer exchange only fails with DSGD_ERR_STATE before anything is launched).  The per-step
 *      path reads ||w||_1 of the weights it starts from off the device: dsgd_set_l1 (turning the penalty on),
 *      dsgd_set_weights and every step of an L1 ctx keep it.
 *      dsgd_weights_l1: *l1_out = ||w||_1 (summed in fixed-point limbs: exact before one final rounding, the same bits in any
 *      order and on every rank) and *nnz_out = #{w_j != 0}, of `w` (dim host values) or with w == NULL of the resident
 *      weights; either output may be NULL.
 *      Errors: lambda1 < 0 or not finite -> DSGD_ERR_INVALID; either call on an async ctx -> DSGD_ERR_STATE. ---------------- */
int dsgd_set_l1(dsgd_ctx *ctx, double lambda1);
/* *dim_out = the dim the ctx was created with (for bindings that check an array's length before passing it in). */
int dsgd_dim(const dsgd_ctx *ctx, int32_t *dim_out);
int dsgd_weights_l1(dsgd_ctx *ctx, const double *w, double *l1_out, int64_t *nnz_out);

/* ---- class weights (sync mode): one weight per label, (w_pos, w_neg) for y = +1 and y = -1, both finite and >= 0, (1, 1)
 *      when the ctx is created.  Write w_y for the weight of a row's label.  The model's backward and loss follow them:
 *        SVM       the gate !(y * (x.w) < 0) is unchanged; a row that passes adds filt(filt(x_j) * s), s = y * w_y
 *        logistic  s = (y * sigmoid(z)) * w_y
 *        loss      of n rows: lambda ||w||^2 (+ lambda1 ||w||_1) + (w_pos * L_pos + w_neg * L_neg) / n, L_pos and L_neg the
 *                  per-class sums of the UNWEIGHTED per-sample losses (SVM: integers; logistic: fixed-point sums), each
 *                  product rounded, then their sum: the divisor is the row count, not the sum of the weights.
 *      They act in every sync step (per-step losses included) and in dsgd_gradient (grad_out and loss_out).  Predictions,
 *      margins, probabilities, metrics, curves, calibration and every dsgd_eval* call do not depend on them, and neither do
 *      regularize, the update, the L1 step, averaging or the rate table, which act on the summed gradient.  At (1, 1) every
 *      call launches exactly the kernels it launches without this call.  With other weights one worker on one GPU takes the
 *      persistent kernel's weighted form up to 32 rows per CTA (with averaging, a rate table and L1 as without weights), the
 *      per-step path above, and large SVM requests the streaming pass's per-class form.  The fused K-rank peer exchange has
 *      no weighted form: with world > 1 a weighted ctx takes the NCCL path and needs dsgd_comm_init, and a rank wired with
 *      the peer exchange only fails with DSGD_ERR_STATE before anything is launched.
 *      Errors: a weight negative, NaN or infinite -> DSGD_ERR_INVALID; the setter on an async ctx -> DSGD_ERR_STATE. -------- */
int dsgd_set_class_weights(dsgd_ctx *ctx, double w_pos, double w_neg);
int dsgd_get_class_weights(const dsgd_ctx *ctx, double *w_pos_out, double *w_neg_out);
/* Per-class evaluation, for either model and whatever the class weights are; rows and weights as in dsgd_eval,
 * dsgd_eval_sampled_counts and dsgd_eval_samples_counts.  *norm_squared = ||w||^2; loss_sums_out[0..1] = the unweighted loss
 * sums of the y = +1 and of the y = -1 rows (SVM: exact integers held in doubles; logistic: fixed-point sums, the same bits in
 * any row order); counts_out[0..3] = correct_pos, correct_neg, n_pos, n_neg.  Any output may be NULL.  The two classes add up
 * to what dsgd_eval_counts / dsgd_eval_sums report for the same rows (integers exactly), and correct_c / n_c is the recall of
 * class c. */
int dsgd_eval_class(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *norm_squared,
                    double *loss_sums_out, int64_t *counts_out);
int dsgd_eval_sampled_class(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                            int64_t pos_begin, int64_t pos_end, double *norm_squared, double *loss_sums_out,
                            int64_t *counts_out);
int dsgd_eval_samples_class(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *norm_squared,
                            double *loss_sums_out, int64_t *counts_out);

/* ---- sample weights (sync mode): one weight s_i per loaded row, finite and >= 0, held on the device in fp64.  Without them
 *      every s_i is 1.  The class weights still apply: row i's combined weight is c_i = fl(w_y * s_i), so s_i = 1 gives
 *      c_i = w_y exactly.  The model's backward and loss follow c_i:
 *        SVM       the gate !(y * (x.w) < 0) is unchanged; a row that passes adds filt(filt(x_j) * s), s = y * c_i
 *        logistic  s = (y * sigmoid(z)) * c_i
 *        loss      of n rows: lambda ||w||^2 (+ lambda1 ||w||_1) + S / n, S = sum_i R(fl(c_i * L_i)) with L_i the unweighted
 *                  per-sample loss, added in the fixed-point limbs of the logistic loss sum (the same bits in any row order,
 *                  grid or rank split; NaN if a term is 2^52 or more).  The divisor is the row count.
 *      A row of c_i = 0 scatters nothing and still counts in n.  With s = 1 and class weights (1, 1) S is the integer hinge
 *      sum or the logistic loss sum, so every loss has the bits of the unweighted call.  They act in every sync step and in
 *      dsgd_gradient; regularize, the update, the L1 step, averaging, the rate table, predictions, margins, metrics, curves,
 *      calibration and every other dsgd_eval* call do not depend on them.  Loading weights, all ones included, selects the
 *      sample-weighted kernels: one worker on one GPU takes the persistent kernel's sample-weighted form up to 32 rows per
 *      CTA (with averaging, a rate table and L1 as without weights), the per-step path above, and dsgd_gradient the fp64
 *      row kernel at any size (the streaming pass has no sample-weighted form).  The fused K-rank peer exchange has no
 *      weighted form: with
 *      world > 1 a weighted ctx needs dsgd_comm_init, and a rank wired with the peer exchange only fails with DSGD_ERR_STATE
 *      before anything is launched.  dsgd_load_csr drops the weights (they named the previous rows).
 *      dsgd_set_sample_weights: n == the loaded rows; sw == NULL with n == 0 clears the weights.  The first call allocates
 *      the weights with cudaMalloc, which synchronises the whole device, and so does the first persistent run with weights
 *      loaded (its per-step hinge codes): K contexts that share ONE GPU call it, then dsgd_reserve, before their threads
 *      start stepping.
 *      Errors: a weight negative, NaN or infinite, or a length other than the loaded rows -> DSGD_ERR_INVALID (checked on the
 *      host before anything changes); an async ctx or no rows loaded -> DSGD_ERR_STATE. ------------------------------------ */
int dsgd_set_sample_weights(dsgd_ctx *ctx, const double *sw, int64_t n);
/* Weighted evaluation, for either model; rows and weights as in dsgd_eval_class and its siblings.  An async ctx has no
 * class or sample weights, so there every c_i is 1; w == NULL reads a snapshot of the replica taken when the call starts,
 * as every other request does there.
 * *norm_squared = ||w||^2; sums_out[0..2] = S = sum c_i L_i, sum c_i [pred_i == y_i] and sum c_i, each a fixed-point sum (the
 * same bits in any row order); counts_out[0..1] = rows, correct.  Any output may be NULL.  Without sample weights c_i = w_y;
 * with class weights (1, 1) as well, S has the bits of dsgd_eval_sums' loss sum and the counts equal dsgd_eval_counts'. */
int dsgd_eval_weighted(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, double *norm_squared,
                       double *sums_out, int64_t *counts_out);
int dsgd_eval_sampled_weighted(dsgd_ctx *ctx, const double *w, int64_t row_begin, int64_t row_end, uint64_t key,
                               int64_t pos_begin, int64_t pos_end, double *norm_squared, double *sums_out,
                               int64_t *counts_out);
int dsgd_eval_samples_weighted(dsgd_ctx *ctx, const double *w, const int32_t *samples, int64_t n, double *norm_squared,
                               double *sums_out, int64_t *counts_out);

/* ---- async (Hogwild) mode.  Every worker keeps its own weight replica (core/Slave.scala:30) and pushes each
 *      delta to every peer replica and to the master's replica (core/Slave.scala:101-105).  Here replicas are
 *      reached by ADDRESS over NVLink: a rank exports its replica, the host transports the handle, peers import
 *      it and the device loop issues system-scope fp64 reductions (red.add) straight into peer memory.
 *      Replaces the slave<->slave and slave->master channels (core/Slave.scala:23,26; core/Master.scala:
 *      229-233).  `which`: DSGD_REPLICA_SELF = this worker's replica; DSGD_REPLICA_MASTER = the master's replica
 *      (GradState.grad + the update counter, core/MasterAsync.scala:66,164-177), hosted by the ctx that calls
 *      dsgd_async_host_master.  peer_rank in dsgd_ipc_import: 0..world-1, or `world` for the master replica.
 *      A worker's delta goes to at most 17 replicas (its own, 15 peers and the master; an outbox takes one of them), so
 *      dsgd_create with DSGD_FLAG_ASYNC refuses world > 16 with DSGD_ERR_INVALID (sync mode has no such bound).  A running
 *      loop keeps the replica table it started with: dsgd_ipc_import and dsgd_peer_attach fail with DSGD_ERR_STATE while
 *      it runs. */
#define DSGD_REPLICA_SELF 0
#define DSGD_REPLICA_MASTER 1
int dsgd_async_host_master(dsgd_ctx *ctx, const double *w0);
int dsgd_ipc_export(dsgd_ctx *ctx, int which, uint8_t handle[DSGD_IPC_HANDLE_BYTES]);
int dsgd_ipc_import(dsgd_ctx *ctx, int peer_rank, const uint8_t handle[DSGD_IPC_HANDLE_BYTES]);
/* Same-process peers (several ctxs in one host process, e.g. a JVM driving all GPUs of a box): attach by ctx. */
int dsgd_peer_attach(dsgd_ctx *ctx, int peer_rank, dsgd_ctx *peer, int which);
/* SlaveImpl.startAsync (core/Slave.scala:159-175): weights := w0, then the worker loop (asyncTask,
 * core/Slave.scala:79-111) runs on the device until dsgd_stop_async or until this worker has made max_updates
 * updates (0: unbounded).  concurrency = Hogwild lanes on this GPU (warps running the loop body concurrently on
 * the shared replica; 1 = the reference's strictly sequential loop).  seed drives the device-side sampling of
 * `assigned` (core/Slave.scala:84,87; batch > 1 indexes rows by POSITION like the reference, quirk Q6).
 * w0 == NULL keeps the resident replica: initialise every replica with dsgd_set_weights first, then start the
 * loops, and no delta a faster peer pushes early is overwritten (the reference has that start-up race).
 * Returns immediately; the loop runs on its own stream.  The first async loop on a device (this call or dsgd_async_replay)
 * first loads every kernel of the library, so that no later call waits for the running loop to load one (CUDA loads kernels
 * lazily by default); that needs a driver for CUDA 12.4 or later, else DSGD_ERR_CUDA. */
int dsgd_start_async(dsgd_ctx *ctx, const double *w0, const int32_t *assigned, int64_t n_assigned, int32_t batch,
                     double lr, int32_t concurrency, int64_t max_updates, uint64_t seed);
/* The same loop body over a RECORDED sampling sequence (n_updates * batch row ids), one lane, blocking: the
 * deterministic K = 1 case of core/Slave.scala:79-111, used to replay a reference run and by the parity tests. */
int dsgd_async_replay(dsgd_ctx *ctx, const double *w0, const int32_t *samples, int32_t batch, int64_t n_updates,
                      double lr);
/* SlaveImpl.stopAsync (core/Slave.scala:187-195): raises the stop flag and waits for the loop to drain. */
int dsgd_stop_async(dsgd_ctx *ctx);
/* 1 while the device loop is running (it also ends by itself after max_updates). */
int dsgd_async_running(dsgd_ctx *ctx, int *running);
/* Device time of the last finished async loop (CUDA events on the loop's stream), for benchmarks. */
int dsgd_async_elapsed_ms(dsgd_ctx *ctx, float *elapsed_ms);
/* SlaveImpl.updateGrad / AsyncMasterGrpcImpl.updateGrad (core/Slave.scala:177-185; core/MasterAsync.scala:
 * 164-177): weights -= delta for a sparse delta given as (idx, val) pairs, applied to this context's own replica (a host-side
 * sender -- e.g. a gRPC colleague -- uses it; GPU peers write the replica directly over NVLink).  Like the reference's new Sparse,
 * an entry whose result is |w - v| <= 1e-20 becomes exactly 0.  Safe from several threads at once (see Threading). */
int dsgd_update_grad(dsgd_ctx *ctx, const int32_t *idx, const double *val, int64_t nnz);
/* GradState.updates (core/ml/GradState.scala:8; core/MasterAsync.scala:165): updates the master replica has
 * received if this ctx hosts or has imported it, else the updates this worker has made. */
int dsgd_async_updates(dsgd_ctx *ctx, int64_t *count);
/* Snapshot of the master replica (gradState.single().grad, core/MasterAsync.scala:109). */
int dsgd_async_master_weights(dsgd_ctx *ctx, double *w_out);
/* Colleagues that are NOT GPU peers (reference JVM slaves or a JVM master reached over gRPC, core/Slave.scala:104-105): the
 * worker loop adds every -delta it applies to one more replica-shaped accumulator, the OUTBOX.  The host reads it while the
 * loop runs and forwards the difference since its last read as ONE updateGrad message (w -= sum of the deltas of the period:
 * the reference sends one message per iteration; Hogwild's additions commute).  Enable before dsgd_start_async (zeroes the
 * accumulator); acc_out[dim] = sum of -delta since then.  dsgd_async_outbox_read is safe while the loop runs. */
int dsgd_async_outbox_enable(dsgd_ctx *ctx);
int dsgd_async_outbox_read(dsgd_ctx *ctx, double *acc_out);

#ifdef __cplusplus
}
#endif
#endif /* DSGD_H */
