/* JNI shim between epfl.distributed.nativ.DsgdNative (Scala, see DsgdNative.scala) and the C ABI of
 * include/dsgd.h.  Compile-gated: the build image has no JDK (no jni.h); on a box with one:
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../../include \
 *       -o libdsgd_jni.so dsgd_jni.c -L.. -ldsgd
 *
 * Every C-ABI call that touches the GPU BLOCKS (it synchronises a CUDA stream; a fused multi-GPU step even waits for
 * the other ranks' threads to launch), so no array is ever pinned across one: inputs are copied out with
 * Get<Type>ArrayRegion before the call and outputs copied back with Set<Type>ArrayRegion after it.  (JNI forbids
 * blocking inside a GetPrimitiveArrayCritical region -- it stalls the collector for the whole JVM, and with several
 * contexts driven from several JVM threads it can deadlock: rank A's kernel waits for rank B's launch while B's thread
 * waits for the collector that A's critical region holds off.)  A NULL array is passed on as NULL / length 0.
 *
 * The library reads and writes the full length the header names through raw pointers, so every array is checked against
 * that length before the call: a wrong length is DSGD_ERR_INVALID, with nothing launched and nothing copied back.
 *
 * tests/test_abi_surface.py compiles this file against a minimal stand-in jni.h (tests/jni_mock/) and checks that the
 * facade covers the header; tests/test_gpu_jni.py runs it against the library through a stand-in JNIEnv. */
#ifdef DSGD_HAVE_JNI
#include <jni.h>
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "dsgd.h"

#define CTX(h) ((dsgd_ctx *)(intptr_t)(h))
#define FN(name) JNIEXPORT jint JNICALL Java_epfl_distributed_nativ_DsgdNative_00024_##name

/* copy of a Java array in C memory (in), or a C buffer of the array's length to be copied back (out) */
typedef struct { void *p; jsize n; int bad; } buf_t;
#define DEF_BUF(Name, JT, CT)                                                                                  \
  static __attribute__((unused)) buf_t in_##Name(JNIEnv *env, JT##Array a) {                                                             \
    buf_t b = {NULL, 0, 0};                                                                                      \
    if (!a) return b;                                                                                            \
    b.n = (*env)->GetArrayLength(env, a);                                                                        \
    b.p = malloc(sizeof(CT) * (size_t)(b.n > 0 ? b.n : 1));                                                      \
    if (!b.p) { b.bad = 1; return b; }                                                                           \
    if (b.n > 0) (*env)->Get##Name##ArrayRegion(env, a, 0, b.n, (JT *)b.p);                                      \
    return b;                                                                                                    \
  }                                                                                                              \
  static __attribute__((unused)) buf_t out_##Name(JNIEnv *env, JT##Array a) {                                                            \
    buf_t b = {NULL, 0, 0};                                                                                      \
    if (!a) return b;                                                                                            \
    b.n = (*env)->GetArrayLength(env, a);                                                                        \
    b.p = calloc((size_t)(b.n > 0 ? b.n : 1), sizeof(CT));                                                       \
    if (!b.p) b.bad = 1;                                                                                         \
    return b;                                                                                                    \
  }                                                                                                              \
  static __attribute__((unused)) void back_##Name(JNIEnv *env, JT##Array a, buf_t b, int rc) {                                           \
    if (a && b.p && rc == DSGD_OK && b.n > 0) (*env)->Set##Name##ArrayRegion(env, a, 0, b.n, (const JT *)b.p);   \
    free(b.p);                                                                                                   \
  }
DEF_BUF(Int, jint, int32_t)
DEF_BUF(Long, jlong, int64_t)
DEF_BUF(Float, jfloat, float)
DEF_BUF(Double, jdouble, double)
DEF_BUF(Byte, jbyte, int8_t)

/* rc, or else DSGD_ERR_NOMEM when a copy failed, or else DSGD_ERR_INVALID when an array is too short */
static int checked(int rc, int bad, int invalid) {
  return rc != DSGD_OK ? rc : bad ? DSGD_ERR_NOMEM : invalid ? DSGD_ERR_INVALID : DSGD_OK;
}
/* a non-null array shorter than n */
static int short_of(const buf_t *b, jlong n) { return b->p && b->n < n; }

/* The length of a weight vector of the ctx: dim, or dim + 1 on a ctx created with DSGD_FLAG_INTERCEPT, which dsgd_info
 * names.  dsgd_info rewrites a string the ctx owns, and getWeights may run on several threads at once while the async loop
 * runs (include/dsgd.h, Threading); the shim is the only caller of dsgd_info and holds info_lock from the call until it has
 * read the string. */
static pthread_mutex_t info_lock = PTHREAD_MUTEX_INITIALIZER;
static int weight_len(jlong h, int32_t *n) {
  int rc = dsgd_dim(CTX(h), n);
  if (rc != DSGD_OK) return rc;
  pthread_mutex_lock(&info_lock);
  if (strstr(dsgd_info(CTX(h)), "\"intercept\": true")) ++*n;
  pthread_mutex_unlock(&info_lock);
  return rc;
}
enum { DIM, WEIGHTS };         /* what an array's length is measured against: dim, or the weight length */
enum { AT_LEAST, EXACTLY };
/* DSGD_OK when b is null or holds exactly / at least the ctx's dim or weight length values */
static int sized(jlong h, const buf_t *b, int what, int how) {
  int32_t n = 0;
  int rc = b->bad ? DSGD_ERR_NOMEM : !b->p ? DSGD_OK : what == WEIGHTS ? weight_len(h, &n) : dsgd_dim(CTX(h), &n);
  return checked(rc, 0, b->p && (how == EXACTLY ? b->n != n : b->n < n));
}

/* The rows a request names: a range [rowBegin, rowEnd), positions [posBegin, posEnd) of the sample drawn on the device
 * from the range with `key`, or a list of row ids (copied into `ids` when the request opens). */
typedef struct {
  enum { RANGE, DRAWN, LIST } form;
  jlong rowBegin, rowEnd, key, posBegin, posEnd;
  jintArray samples;
  buf_t ids;
} rows_t;
static rows_t range_rows(jlong rowBegin, jlong rowEnd) { return (rows_t){RANGE, rowBegin, rowEnd, 0, 0, 0, NULL, {0}}; }
static rows_t drawn_rows(jlong rowBegin, jlong rowEnd, jlong key, jlong posBegin, jlong posEnd) {
  return (rows_t){DRAWN, rowBegin, rowEnd, key, posBegin, posEnd, NULL, {0}};
}
static rows_t list_rows(jintArray samples) { return (rows_t){LIST, 0, 0, 0, 0, 0, samples, {0}}; }
/* the rows of a call that takes weights and names no rows (setWeights, weightsL1) */
static rows_t no_rows(void) { return range_rows(0, 0); }

/* One request: the weights w (null: the resident ones, else exactly the weight length) and its rows, copied in. */
typedef struct { buf_t w; rows_t r; } req_t;
static int req_open(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, req_t *q) {
  q->w = in_Double(env, w);
  q->r = r;
  q->r.ids = in_Int(env, r.samples);
  return checked(sized(h, &q->w, WEIGHTS, EXACTLY), q->r.ids.bad, 0);
}
static void req_close(req_t *q) { free(q->w.p); free(q->r.ids.p); }
/* the number of rows a request names */
static jlong rows_n(const req_t *q) {
  return q->r.form == RANGE ? q->r.rowEnd - q->r.rowBegin : q->r.form == DRAWN ? q->r.posEnd - q->r.posBegin : q->r.ids.n;
}
/* the call of one evaluation family in the request's row form: fn, fn_sampled or fn_samples, the outputs after the rows */
#define ROW_CALL(h, q, fn, fn_sampled, fn_samples, ...)                                                                   \
  ((q).r.form == RANGE   ? fn(CTX(h), (q).w.p, (q).r.rowBegin, (q).r.rowEnd, __VA_ARGS__)                                \
   : (q).r.form == DRAWN ? fn_sampled(CTX(h), (q).w.p, (q).r.rowBegin, (q).r.rowEnd, (uint64_t)(q).r.key, (q).r.posBegin, \
                                      (q).r.posEnd, __VA_ARGS__)                                                          \
                         : fn_samples(CTX(h), (q).w.p, (q).r.ids.p, (q).r.ids.n, __VA_ARGS__))

/* ---- lifecycle ---- */
JNIEXPORT jlong JNICALL Java_epfl_distributed_nativ_DsgdNative_00024_create(JNIEnv *env, jobject self, jint device, jint dim,
                                                                          jdouble lambda, jint rank, jint world, jint flags) {
  dsgd_ctx *ctx = NULL;
  int rc = dsgd_create(&ctx, device, dim, lambda, rank, world, (uint32_t)flags);   /* new Slave(...) + SparseSVM(lambda, .) */
  return rc == DSGD_OK ? (jlong)(intptr_t)ctx : (jlong)rc; /* negative = error code */
}
FN(destroy)(JNIEnv *env, jobject self, jlong h) { return dsgd_destroy(CTX(h)); }
JNIEXPORT jstring JNICALL Java_epfl_distributed_nativ_DsgdNative_00024_lastError(JNIEnv *env, jobject self, jlong h) {
  return (*env)->NewStringUTF(env, dsgd_last_error(CTX(h)));
}

/* ---- data / model ---- */
FN(loadCsr)(JNIEnv *env, jobject self, jlong h, jlongArray rowPtr, jintArray col, jfloatArray value, jbyteArray label) {
  buf_t rp = in_Long(env, rowPtr), c = in_Int(env, col), v = in_Float(env, value), l = in_Byte(env, label);
  int rc = checked(DSGD_OK, rp.bad | c.bad | v.bad | l.bad, rp.n < 1 || l.n != rp.n - 1 || v.n != c.n);
  if (rc == DSGD_OK) rc = dsgd_load_csr(CTX(h), rp.n - 1, c.n, rp.p, c.p, v.p, l.p);   /* Dataset.rcv1 rows as CSR (utils/Dataset.scala:23-47) */
  free(rp.p); free(c.p); free(v.p); free(l.p);
  return rc;
}
FN(setDimSparsity)(JNIEnv *env, jobject self, jlong h, jdoubleArray d) {
  buf_t b = in_Double(env, d);
  int rc = sized(h, &b, DIM, EXACTLY);
  if (rc == DSGD_OK) rc = dsgd_set_dim_sparsity(CTX(h), b.p);            /* SparseSVM.dimSparsity */
  free(b.p);
  return rc;
}
FN(computeDimSparsity)(JNIEnv *env, jobject self, jlong h, jlong nTrain, jdoubleArray out) {
  buf_t o = out_Double(env, out);
  int rc = sized(h, &o, DIM, AT_LEAST);
  if (rc == DSGD_OK) rc = dsgd_compute_dim_sparsity(CTX(h), nTrain, o.p); /* Main.scala:54-65 */
  back_Double(env, out, o, rc);
  return rc;
}
FN(setWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray w) {
  req_t q;
  int rc = req_open(env, h, w, no_rows(), &q);
  if (rc == DSGD_OK) rc = dsgd_set_weights(CTX(h), q.w.p);
  req_close(&q);
  return rc;
}
FN(getWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray w) {
  buf_t o = out_Double(env, w);
  int rc = sized(h, &o, WEIGHTS, AT_LEAST);
  if (rc == DSGD_OK) rc = dsgd_get_weights(CTX(h), o.p);
  back_Double(env, w, o, rc);
  return rc;
}

/* ---- requests ---- */
/* the calls that give one double per listed row; out at least as long as samples */
typedef int (*per_row_fn)(dsgd_ctx *, const double *, const int32_t *, int64_t, double *);
static int per_row(JNIEnv *env, jlong h, jdoubleArray w, jintArray samples, jdoubleArray out, per_row_fn fn) {
  req_t q;
  buf_t o = out_Double(env, out);
  int rc = req_open(env, h, w, list_rows(samples), &q);
  rc = checked(rc, o.bad, o.n < q.r.ids.n);
  if (rc == DSGD_OK) rc = fn(CTX(h), q.w.p, q.r.ids.p, q.r.ids.n, o.p);
  back_Double(env, out, o, rc);
  req_close(&q);
  return rc;
}
FN(gradient)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray grad) {
  req_t q;
  buf_t g = out_Double(env, grad);
  int rc = req_open(env, h, w, list_rows(samples), &q);
  if (rc == DSGD_OK) rc = sized(h, &g, WEIGHTS, AT_LEAST);
  if (rc == DSGD_OK) rc = dsgd_gradient(CTX(h), q.w.p, q.r.ids.p, q.r.ids.n, g.p, NULL);  /* core/Slave.scala:142-157 */
  back_Double(env, grad, g, rc);
  req_close(&q);
  return rc;
}
FN(forward)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray preds) {
  return per_row(env, h, w, samples, preds, dsgd_forward);                                 /* core/Slave.scala:129-140 */
}
FN(eval)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray lossAcc) {
  req_t q;
  buf_t o = out_Double(env, lossAcc);                                   /* lossAcc(0) = loss, lossAcc(1) = accuracy */
  int rc = checked(req_open(env, h, w, range_rows(rowBegin, rowEnd), &q), o.bad, o.n < 2);
  if (rc == DSGD_OK) rc = dsgd_eval(CTX(h), q.w.p, rowBegin, rowEnd, (double *)o.p, (double *)o.p + 1);  /* core/Master.scala:100-107 */
  back_Double(env, lossAcc, o, rc);
  req_close(&q);
  return rc;
}

/* exact shardable form: hingeCorrect(0) = hinge sum, (1) = #correct; the sampled form is core/Master.scala:109-118 with
 * the sample drawn on the device (positions [posBegin, posEnd)), the list form the row ids the JVM drew with its own Random */
static int req_counts(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jlongArray hingeCorrect, jdoubleArray normSquared) {
  req_t q;
  buf_t c = out_Long(env, hingeCorrect), n = out_Double(env, normSquared);
  int rc = checked(req_open(env, h, w, r, &q), c.bad | n.bad, c.n < 2 || n.n < 1);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_counts, dsgd_eval_sampled_counts, dsgd_eval_samples_counts, (int64_t *)c.p,
                  (int64_t *)c.p + 1, n.p);
  back_Long(env, hingeCorrect, c, rc);
  back_Double(env, normSquared, n, rc);
  req_close(&q);
  return rc;
}
FN(evalCounts)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray hingeCorrect,
               jdoubleArray normSquared) {
  return req_counts(env, h, w, range_rows(rowBegin, rowEnd), hingeCorrect, normSquared);
}
FN(evalSampledCounts)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                      jlong posBegin, jlong posEnd, jlongArray hingeCorrect, jdoubleArray normSquared) {
  return req_counts(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), hingeCorrect, normSquared);
}
FN(evalSamplesCounts)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray hingeCorrect,
                      jdoubleArray normSquared) {
  return req_counts(env, h, w, list_rows(samples), hingeCorrect, normSquared);
}
/* The *Sums forms serve either model (the *Counts forms refuse a logistic ctx): lossSumNormSquared(0) = sum of the per-sample
 * losses, (1) = ||w||^2; correct(0) = #correct. */
static int req_sums(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdoubleArray lossSumNormSquared, jlongArray correct) {
  req_t q;
  buf_t s = out_Double(env, lossSumNormSquared), c = out_Long(env, correct);
  int rc = checked(req_open(env, h, w, r, &q), s.bad | c.bad, s.n < 2 || c.n < 1);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_sums, dsgd_eval_sampled_sums, dsgd_eval_samples_sums, (double *)s.p, (int64_t *)c.p,
                  (double *)s.p + 1);
  back_Double(env, lossSumNormSquared, s, rc);
  back_Long(env, correct, c, rc);
  req_close(&q);
  return rc;
}
FN(evalSums)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray lossSumNormSquared,
             jlongArray correct) {
  return req_sums(env, h, w, range_rows(rowBegin, rowEnd), lossSumNormSquared, correct);
}
FN(evalSampledSums)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                    jlong posBegin, jlong posEnd, jdoubleArray lossSumNormSquared, jlongArray correct) {
  return req_sums(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), lossSumNormSquared, correct);
}
FN(evalSamplesSums)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray lossSumNormSquared,
                    jlongArray correct) {
  return req_sums(env, h, w, list_rows(samples), lossSumNormSquared, correct);
}
/* scores and ranking metrics, either model: out(i) = x_i . w (margins) or P(y = +1 | x_i) (probabilities, SparseLogistic
 * only); metrics(0..7) = the DSGD_METRICS_WORDS counts of dsgd_eval_metrics.  An output shorter than that is DSGD_ERR_INVALID. */
FN(margins)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray out) {
  return per_row(env, h, w, samples, out, dsgd_margins);
}
FN(probabilities)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray out) {
  return per_row(env, h, w, samples, out, dsgd_probabilities);
}
static int req_metrics(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jlongArray metrics) {
  req_t q;
  buf_t m = out_Long(env, metrics);
  int rc = checked(req_open(env, h, w, r, &q), m.bad, m.n < DSGD_METRICS_WORDS);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_metrics, dsgd_eval_sampled_metrics, dsgd_eval_samples_metrics, (int64_t *)m.p);
  back_Long(env, metrics, m, rc);
  req_close(&q);
  return rc;
}
FN(evalMetrics)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray metrics) {
  return req_metrics(env, h, w, range_rows(rowBegin, rowEnd), metrics);
}
FN(evalSampledMetrics)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                       jlong posBegin, jlong posEnd, jlongArray metrics) {
  return req_metrics(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), metrics);
}
FN(evalSamplesMetrics)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray metrics) {
  return req_metrics(env, h, w, list_rows(samples), metrics);
}
/* curves and average precision: metrics(0..7) as above, ap(0) = average precision, nPoints(0) = m, and thr / tp / fp (0 until
 * m) the points, highest score first -- all three null for average precision alone, else each at least as long as the
 * request's rows (n = rowEnd - rowBegin, posEnd - posBegin or samples.length).  A shorter array is DSGD_ERR_INVALID. */
static int req_curve(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jlongArray metrics, jdoubleArray ap,
                     jlongArray nPoints, jdoubleArray thr, jlongArray tp, jlongArray fp) {
  req_t q;
  buf_t m = out_Long(env, metrics), a = out_Double(env, ap), k = out_Long(env, nPoints), t = out_Double(env, thr),
        bt = out_Long(env, tp), bf = out_Long(env, fp);
  int rc = req_open(env, h, w, r, &q);
  const jlong n = rows_n(&q);
  rc = checked(rc, m.bad | a.bad | k.bad | t.bad | bt.bad | bf.bad,
               m.n < DSGD_METRICS_WORDS || a.n < 1 || k.n < 1 || short_of(&t, n) || short_of(&bt, n) || short_of(&bf, n));
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_curve, dsgd_eval_sampled_curve, dsgd_eval_samples_curve, (int64_t *)m.p, (double *)a.p,
                  (int64_t *)k.p, (double *)t.p, (int64_t *)bt.p, (int64_t *)bf.p);
  back_Long(env, metrics, m, rc);
  back_Double(env, ap, a, rc);
  back_Long(env, nPoints, k, rc);
  back_Double(env, thr, t, rc);
  back_Long(env, tp, bt, rc);
  back_Long(env, fp, bf, rc);
  req_close(&q);
  return rc;
}
FN(evalCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray metrics,
              jdoubleArray ap, jlongArray nPoints, jdoubleArray thr, jlongArray tp, jlongArray fp) {
  return req_curve(env, h, w, range_rows(rowBegin, rowEnd), metrics, ap, nPoints, thr, tp, fp);
}
FN(evalSampledCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                     jlong posBegin, jlong posEnd, jlongArray metrics, jdoubleArray ap, jlongArray nPoints, jdoubleArray thr,
                     jlongArray tp, jlongArray fp) {
  return req_curve(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), metrics, ap, nPoints, thr, tp, fp);
}
FN(evalSamplesCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray metrics,
                     jdoubleArray ap, jlongArray nPoints, jdoubleArray thr, jlongArray tp, jlongArray fp) {
  return req_curve(env, h, w, list_rows(samples), metrics, ap, nPoints, thr, tp, fp);
}

/* Poisson bootstrap: replicates [bBegin, bEnd) with key bKey; words(9 j .. 9 j + 8) = the DSGD_BOOTSTRAP_WORDS words of
 * replicate bBegin + j, ap(j) its average precision, loss(j) its loss sum.  An output shorter than the replicates is
 * DSGD_ERR_INVALID. */
static int req_boot(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jlong bKey, jlong bBegin, jlong bEnd, jlongArray words,
                    jdoubleArray ap, jdoubleArray loss) {
  req_t q;
  buf_t m = out_Long(env, words), a = out_Double(env, ap), l = out_Double(env, loss);
  const jlong k = bEnd > bBegin ? bEnd - bBegin : 0;
  int rc = checked(req_open(env, h, w, r, &q), m.bad | a.bad | l.bad, m.n < k * DSGD_BOOTSTRAP_WORDS || a.n < k || l.n < k);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_bootstrap, dsgd_eval_sampled_bootstrap, dsgd_eval_samples_bootstrap, (uint64_t)bKey, bBegin,
                  bEnd, (int64_t *)m.p, (double *)a.p, (double *)l.p);
  back_Long(env, words, m, rc);
  back_Double(env, ap, a, rc);
  back_Double(env, loss, l, rc);
  req_close(&q);
  return rc;
}
FN(evalBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong bKey, jlong bBegin,
                  jlong bEnd, jlongArray words, jdoubleArray ap, jdoubleArray loss) {
  return req_boot(env, h, w, range_rows(rowBegin, rowEnd), bKey, bBegin, bEnd, words, ap, loss);
}
FN(evalSampledBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                         jlong posBegin, jlong posEnd, jlong bKey, jlong bBegin, jlong bEnd, jlongArray words,
                         jdoubleArray ap, jdoubleArray loss) {
  return req_boot(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), bKey, bBegin, bEnd, words, ap, loss);
}
FN(evalSamplesBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlong bKey, jlong bBegin,
                         jlong bEnd, jlongArray words, jdoubleArray ap, jdoubleArray loss) {
  return req_boot(env, h, w, list_rows(samples), bKey, bBegin, bEnd, words, ap, loss);
}

/* weighted Poisson bootstrap: replicates [bBegin, bEnd) with key bKey; words(2 j), words(2 j + 1) = the size and the NaN-score
 * rows of replicate bBegin + j, wsums(13 j .. 13 j + 12) its DSGD_WCURVE_WORDS, loss(j) its weighted loss sum.  An output
 * shorter than the replicates is DSGD_ERR_INVALID. */
static int req_wboot(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jlong bKey, jlong bBegin, jlong bEnd, jlongArray words,
                     jdoubleArray wsums, jdoubleArray loss) {
  req_t q;
  buf_t m = out_Long(env, words), s = out_Double(env, wsums), l = out_Double(env, loss);
  const jlong k = bEnd > bBegin ? bEnd - bBegin : 0;
  int rc = checked(req_open(env, h, w, r, &q), m.bad | s.bad | l.bad, m.n < k * 2 || s.n < k * DSGD_WCURVE_WORDS || l.n < k);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_weighted_bootstrap, dsgd_eval_sampled_weighted_bootstrap,
                  dsgd_eval_samples_weighted_bootstrap, (uint64_t)bKey, bBegin, bEnd, (int64_t *)m.p, (double *)s.p,
                  (double *)l.p);
  back_Long(env, words, m, rc);
  back_Double(env, wsums, s, rc);
  back_Double(env, loss, l, rc);
  req_close(&q);
  return rc;
}
FN(evalWeightedBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong bKey,
                          jlong bBegin, jlong bEnd, jlongArray words, jdoubleArray wsums, jdoubleArray loss) {
  return req_wboot(env, h, w, range_rows(rowBegin, rowEnd), bKey, bBegin, bEnd, words, wsums, loss);
}
FN(evalSampledWeightedBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                                 jlong posBegin, jlong posEnd, jlong bKey, jlong bBegin, jlong bEnd, jlongArray words,
                                 jdoubleArray wsums, jdoubleArray loss) {
  return req_wboot(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), bKey, bBegin, bEnd, words, wsums, loss);
}
FN(evalSamplesWeightedBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlong bKey,
                                 jlong bBegin, jlong bEnd, jlongArray words, jdoubleArray wsums, jdoubleArray loss) {
  return req_wboot(env, h, w, list_rows(samples), bKey, bBegin, bEnd, words, wsums, loss);
}

/* calibration: ab(0..1) = (A, B), objective(0) = F(A, B), info(0..4) = the DSGD_CALIBRATION_INFO_WORDS words; probabilities:
 * out(i) = sigmoid(-(a x_i . w + b)); quality: sums(0..1) = Brier and log-loss sums, binRows / binPos / binPsum at least nBins
 * long, words(0..1) = rows used and left out.  A shorter array is DSGD_ERR_INVALID.  nBins outside
 * 1 .. DSGD_CALIBRATION_MAX_BINS is the library's DSGD_ERR_INVALID: only the lengths are checked here. */
static jlong bins_n(jint nBins) { return nBins > 0 ? nBins : 0; }
static int req_calib(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdoubleArray ab, jdoubleArray objective,
                     jlongArray info) {
  req_t q;
  buf_t a = out_Double(env, ab), f = out_Double(env, objective), i = out_Long(env, info);
  int rc = checked(req_open(env, h, w, r, &q), a.bad | f.bad | i.bad,
                   a.n < 2 || f.n < 1 || i.n < DSGD_CALIBRATION_INFO_WORDS);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_calibrate, dsgd_calibrate_sampled, dsgd_calibrate_samples, (double *)a.p, (double *)f.p,
                  (int64_t *)i.p);
  back_Double(env, ab, a, rc);
  back_Double(env, objective, f, rc);
  back_Long(env, info, i, rc);
  req_close(&q);
  return rc;
}
FN(calibrate)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray ab,
              jdoubleArray objective, jlongArray info) {
  return req_calib(env, h, w, range_rows(rowBegin, rowEnd), ab, objective, info);
}
FN(calibrateSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                     jlong posBegin, jlong posEnd, jdoubleArray ab, jdoubleArray objective, jlongArray info) {
  return req_calib(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), ab, objective, info);
}
FN(calibrateSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray ab,
                     jdoubleArray objective, jlongArray info) {
  return req_calib(env, h, w, list_rows(samples), ab, objective, info);
}
FN(calibratedProbabilities)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdouble a, jdouble b,
                            jdoubleArray out) {
  req_t q;
  buf_t o = out_Double(env, out);
  int rc = req_open(env, h, w, list_rows(samples), &q);
  rc = checked(rc, o.bad, o.n < q.r.ids.n);
  if (rc == DSGD_OK) rc = dsgd_calibrated_probabilities(CTX(h), q.w.p, q.r.ids.p, q.r.ids.n, a, b, o.p);
  back_Double(env, out, o, rc);
  req_close(&q);
  return rc;
}
static int req_quality(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdouble a, jdouble b, jint nBins, jdoubleArray sums,
                       jlongArray binRows, jlongArray binPos, jdoubleArray binPsum, jlongArray words) {
  req_t q;
  buf_t s = out_Double(env, sums), br = out_Long(env, binRows), bp = out_Long(env, binPos), ps = out_Double(env, binPsum),
        wd = out_Long(env, words);
  const jlong m = bins_n(nBins);
  int rc = checked(req_open(env, h, w, r, &q), s.bad | br.bad | bp.bad | ps.bad | wd.bad,
                   s.n < 2 || wd.n < 2 || br.n < m || bp.n < m || ps.n < m);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_calibration, dsgd_eval_sampled_calibration, dsgd_eval_samples_calibration, a, b, nBins,
                  (double *)s.p, (int64_t *)br.p, (int64_t *)bp.p, (double *)ps.p, (int64_t *)wd.p);
  back_Double(env, sums, s, rc);
  back_Long(env, binRows, br, rc);
  back_Long(env, binPos, bp, rc);
  back_Double(env, binPsum, ps, rc);
  back_Long(env, words, wd, rc);
  req_close(&q);
  return rc;
}
FN(evalCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdouble a, jdouble b,
                    jint nBins, jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum,
                    jlongArray words) {
  return req_quality(env, h, w, range_rows(rowBegin, rowEnd), a, b, nBins, sums, binRows, binPos, binPsum, words);
}
FN(evalSampledCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                           jlong posBegin, jlong posEnd, jdouble a, jdouble b, jint nBins, jdoubleArray sums,
                           jlongArray binRows, jlongArray binPos, jdoubleArray binPsum, jlongArray words) {
  return req_quality(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), a, b, nBins, sums, binRows, binPos,
                     binPsum, words);
}
FN(evalSamplesCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdouble a, jdouble b,
                           jint nBins, jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum,
                           jlongArray words) {
  return req_quality(env, h, w, list_rows(samples), a, b, nBins, sums, binRows, binPos, binPsum, words);
}

/* weighted calibration: the calibration natives with wsums(0..2) = W+, W- and the NaN rows' weight added to a fit; quality:
 * sums(0..3) = weighted Brier and log-loss sums, the weight used and the infinite-term weight, binWeight / binPosWeight /
 * binPsum at least nBins long (doubles), words(0..1) as there.  A shorter array is DSGD_ERR_INVALID. */
static int req_wcalib(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdoubleArray ab, jdoubleArray objective,
                      jlongArray info, jdoubleArray wsums) {
  req_t q;
  buf_t a = out_Double(env, ab), f = out_Double(env, objective), i = out_Long(env, info), s = out_Double(env, wsums);
  int rc = checked(req_open(env, h, w, r, &q), a.bad | f.bad | i.bad | s.bad,
                   a.n < 2 || f.n < 1 || i.n < DSGD_CALIBRATION_INFO_WORDS || s.n < DSGD_CALIBRATION_WSUMS);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_calibrate_weighted, dsgd_calibrate_weighted_sampled, dsgd_calibrate_weighted_samples,
                  (double *)a.p, (double *)f.p, (int64_t *)i.p, (double *)s.p);
  back_Double(env, ab, a, rc);
  back_Double(env, objective, f, rc);
  back_Long(env, info, i, rc);
  back_Double(env, wsums, s, rc);
  req_close(&q);
  return rc;
}
FN(calibrateWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray ab,
                      jdoubleArray objective, jlongArray info, jdoubleArray wsums) {
  return req_wcalib(env, h, w, range_rows(rowBegin, rowEnd), ab, objective, info, wsums);
}
FN(calibrateWeightedSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                             jlong posBegin, jlong posEnd, jdoubleArray ab, jdoubleArray objective, jlongArray info,
                             jdoubleArray wsums) {
  return req_wcalib(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), ab, objective, info, wsums);
}
FN(calibrateWeightedSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray ab,
                             jdoubleArray objective, jlongArray info, jdoubleArray wsums) {
  return req_wcalib(env, h, w, list_rows(samples), ab, objective, info, wsums);
}
static int req_wquality(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdouble a, jdouble b, jint nBins, jdoubleArray sums,
                        jdoubleArray binWeight, jdoubleArray binPosWeight, jdoubleArray binPsum, jlongArray words) {
  req_t q;
  buf_t s = out_Double(env, sums), bw = out_Double(env, binWeight), bp = out_Double(env, binPosWeight),
        ps = out_Double(env, binPsum), wd = out_Long(env, words);
  const jlong m = bins_n(nBins);
  int rc = checked(req_open(env, h, w, r, &q), s.bad | bw.bad | bp.bad | ps.bad | wd.bad,
                   s.n < DSGD_WCALIBRATION_SUMS || wd.n < 2 || bw.n < m || bp.n < m || ps.n < m);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_weighted_calibration, dsgd_eval_sampled_weighted_calibration,
                  dsgd_eval_samples_weighted_calibration, a, b, nBins, (double *)s.p, (double *)bw.p, (double *)bp.p,
                  (double *)ps.p, (int64_t *)wd.p);
  back_Double(env, sums, s, rc);
  back_Double(env, binWeight, bw, rc);
  back_Double(env, binPosWeight, bp, rc);
  back_Double(env, binPsum, ps, rc);
  back_Long(env, words, wd, rc);
  req_close(&q);
  return rc;
}
FN(evalWeightedCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdouble a,
                            jdouble b, jint nBins, jdoubleArray sums, jdoubleArray binWeight, jdoubleArray binPosWeight,
                            jdoubleArray binPsum, jlongArray words) {
  return req_wquality(env, h, w, range_rows(rowBegin, rowEnd), a, b, nBins, sums, binWeight, binPosWeight, binPsum, words);
}
FN(evalSampledWeightedCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                   jlong key, jlong posBegin, jlong posEnd, jdouble a, jdouble b, jint nBins,
                                   jdoubleArray sums, jdoubleArray binWeight, jdoubleArray binPosWeight,
                                   jdoubleArray binPsum, jlongArray words) {
  return req_wquality(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), a, b, nBins, sums, binWeight,
                      binPosWeight, binPsum, words);
}
FN(evalSamplesWeightedCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdouble a,
                                   jdouble b, jint nBins, jdoubleArray sums, jdoubleArray binWeight,
                                   jdoubleArray binPosWeight, jdoubleArray binPsum, jlongArray words) {
  return req_wquality(env, h, w, list_rows(samples), a, b, nBins, sums, binWeight, binPosWeight, binPsum, words);
}

/* isotonic calibration: nPoints(0) = k, x / y(0 until k) the thresholds and their values, blockRows / blockPos(0 until
 * blocks), info(0..4) = the DSGD_ISOTONIC_INFO_WORDS words; x, y, blockRows and blockPos at least as long as the request's
 * rows.  Probabilities and quality at the map (x, y): x and y of one length k >= 1; out at least as long as samples; the
 * quality arrays as for evalCalibration, words(0..2) = rows used, rows left out and rows with an infinite log-loss term.
 * A shorter array is DSGD_ERR_INVALID. */
static int req_iso(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jlongArray nPoints, jdoubleArray x, jdoubleArray y,
                   jlongArray blockRows, jlongArray blockPos, jlongArray info) {
  req_t q;
  buf_t k = out_Long(env, nPoints), bx = out_Double(env, x), by = out_Double(env, y), br = out_Long(env, blockRows),
        bp = out_Long(env, blockPos), i = out_Long(env, info);
  int rc = req_open(env, h, w, r, &q);
  const jlong n = rows_n(&q);
  rc = checked(rc, k.bad | bx.bad | by.bad | br.bad | bp.bad | i.bad,
               k.n < 1 || i.n < DSGD_ISOTONIC_INFO_WORDS || bx.n < n || by.n < n || br.n < n || bp.n < n);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_calibrate_isotonic, dsgd_calibrate_isotonic_sampled, dsgd_calibrate_isotonic_samples,
                  (int64_t *)k.p, (double *)bx.p, (double *)by.p, (int64_t *)br.p, (int64_t *)bp.p, (int64_t *)i.p);
  back_Long(env, nPoints, k, rc);
  back_Double(env, x, bx, rc);
  back_Double(env, y, by, rc);
  back_Long(env, blockRows, br, rc);
  back_Long(env, blockPos, bp, rc);
  back_Long(env, info, i, rc);
  req_close(&q);
  return rc;
}
FN(calibrateIsotonic)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray nPoints,
                      jdoubleArray x, jdoubleArray y, jlongArray blockRows, jlongArray blockPos, jlongArray info) {
  return req_iso(env, h, w, range_rows(rowBegin, rowEnd), nPoints, x, y, blockRows, blockPos, info);
}
FN(calibrateIsotonicSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                             jlong posBegin, jlong posEnd, jlongArray nPoints, jdoubleArray x, jdoubleArray y,
                             jlongArray blockRows, jlongArray blockPos, jlongArray info) {
  return req_iso(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), nPoints, x, y, blockRows, blockPos, info);
}
FN(calibrateIsotonicSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray nPoints,
                             jdoubleArray x, jdoubleArray y, jlongArray blockRows, jlongArray blockPos, jlongArray info) {
  return req_iso(env, h, w, list_rows(samples), nPoints, x, y, blockRows, blockPos, info);
}
FN(isotonicProbabilities)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray x,
                          jdoubleArray y, jdoubleArray out) {
  req_t q;
  buf_t bx = in_Double(env, x), by = in_Double(env, y), o = out_Double(env, out);
  int rc = req_open(env, h, w, list_rows(samples), &q);
  rc = checked(rc, bx.bad | by.bad | o.bad, o.n < q.r.ids.n || bx.n != by.n);
  if (rc == DSGD_OK) rc = dsgd_isotonic_probabilities(CTX(h), q.w.p, q.r.ids.p, q.r.ids.n, bx.p, by.p, bx.n, o.p);
  back_Double(env, out, o, rc);
  req_close(&q);
  free(bx.p); free(by.p);
  return rc;
}
static int req_iso_quality(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdoubleArray x, jdoubleArray y, jint nBins,
                           jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum, jlongArray words) {
  req_t q;
  buf_t bx = in_Double(env, x), by = in_Double(env, y), s = out_Double(env, sums), br = out_Long(env, binRows),
        bp = out_Long(env, binPos), ps = out_Double(env, binPsum), wd = out_Long(env, words);
  const jlong m = bins_n(nBins);
  int rc = checked(req_open(env, h, w, r, &q), bx.bad | by.bad | s.bad | br.bad | bp.bad | ps.bad | wd.bad,
                   s.n < 2 || wd.n < DSGD_ISOTONIC_EVAL_WORDS || br.n < m || bp.n < m || ps.n < m || bx.n != by.n);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_isotonic_calibration, dsgd_eval_sampled_isotonic_calibration,
                  dsgd_eval_samples_isotonic_calibration, bx.p, by.p, bx.n, nBins, (double *)s.p, (int64_t *)br.p,
                  (int64_t *)bp.p, (double *)ps.p, (int64_t *)wd.p);
  back_Double(env, sums, s, rc);
  back_Long(env, binRows, br, rc);
  back_Long(env, binPos, bp, rc);
  back_Double(env, binPsum, ps, rc);
  back_Long(env, words, wd, rc);
  req_close(&q);
  free(bx.p); free(by.p);
  return rc;
}
FN(evalIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray x,
                            jdoubleArray y, jint nBins, jdoubleArray sums, jlongArray binRows, jlongArray binPos,
                            jdoubleArray binPsum, jlongArray words) {
  return req_iso_quality(env, h, w, range_rows(rowBegin, rowEnd), x, y, nBins, sums, binRows, binPos, binPsum, words);
}
FN(evalSampledIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                   jlong key, jlong posBegin, jlong posEnd, jdoubleArray x, jdoubleArray y, jint nBins,
                                   jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum,
                                   jlongArray words) {
  return req_iso_quality(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), x, y, nBins, sums, binRows, binPos,
                         binPsum, words);
}
FN(evalSamplesIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray x,
                                   jdoubleArray y, jint nBins, jdoubleArray sums, jlongArray binRows, jlongArray binPos,
                                   jdoubleArray binPsum, jlongArray words) {
  return req_iso_quality(env, h, w, list_rows(samples), x, y, nBins, sums, binRows, binPos, binPsum, words);
}

/* weighted isotonic calibration: the isotonic natives with blockWeight / blockPosWeight (doubles) in place of the block counts
 * and wsums(0..1) = W+, W- added to a fit; weighted quality at (x, y): the weighted quality arrays with words(0..2) as for
 * evalIsotonicCalibration.  A shorter array is DSGD_ERR_INVALID. */
static int req_wiso(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jlongArray nPoints, jdoubleArray x, jdoubleArray y,
                    jdoubleArray blockWeight, jdoubleArray blockPosWeight, jlongArray info, jdoubleArray wsums) {
  req_t q;
  buf_t k = out_Long(env, nPoints), bx = out_Double(env, x), by = out_Double(env, y), bw = out_Double(env, blockWeight),
        bp = out_Double(env, blockPosWeight), i = out_Long(env, info), s = out_Double(env, wsums);
  int rc = req_open(env, h, w, r, &q);
  const jlong n = rows_n(&q);
  rc = checked(rc, k.bad | bx.bad | by.bad | bw.bad | bp.bad | i.bad | s.bad,
               k.n < 1 || i.n < DSGD_ISOTONIC_INFO_WORDS || s.n < 2 || bx.n < n || by.n < n || bw.n < n || bp.n < n);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_calibrate_isotonic_weighted, dsgd_calibrate_isotonic_weighted_sampled,
                  dsgd_calibrate_isotonic_weighted_samples, (int64_t *)k.p, (double *)bx.p, (double *)by.p, (double *)bw.p,
                  (double *)bp.p, (int64_t *)i.p, (double *)s.p);
  back_Long(env, nPoints, k, rc);
  back_Double(env, x, bx, rc);
  back_Double(env, y, by, rc);
  back_Double(env, blockWeight, bw, rc);
  back_Double(env, blockPosWeight, bp, rc);
  back_Long(env, info, i, rc);
  back_Double(env, wsums, s, rc);
  req_close(&q);
  return rc;
}
FN(calibrateIsotonicWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                              jlongArray nPoints, jdoubleArray x, jdoubleArray y, jdoubleArray blockWeight,
                              jdoubleArray blockPosWeight, jlongArray info, jdoubleArray wsums) {
  return req_wiso(env, h, w, range_rows(rowBegin, rowEnd), nPoints, x, y, blockWeight, blockPosWeight, info, wsums);
}
FN(calibrateIsotonicWeightedSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                     jlong key, jlong posBegin, jlong posEnd, jlongArray nPoints, jdoubleArray x,
                                     jdoubleArray y, jdoubleArray blockWeight, jdoubleArray blockPosWeight, jlongArray info,
                                     jdoubleArray wsums) {
  return req_wiso(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), nPoints, x, y, blockWeight, blockPosWeight,
                  info, wsums);
}
FN(calibrateIsotonicWeightedSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples,
                                     jlongArray nPoints, jdoubleArray x, jdoubleArray y, jdoubleArray blockWeight,
                                     jdoubleArray blockPosWeight, jlongArray info, jdoubleArray wsums) {
  return req_wiso(env, h, w, list_rows(samples), nPoints, x, y, blockWeight, blockPosWeight, info, wsums);
}
static int req_wiso_quality(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdoubleArray x, jdoubleArray y, jint nBins,
                            jdoubleArray sums, jdoubleArray binWeight, jdoubleArray binPosWeight, jdoubleArray binPsum,
                            jlongArray words) {
  req_t q;
  buf_t bx = in_Double(env, x), by = in_Double(env, y), s = out_Double(env, sums), bw = out_Double(env, binWeight),
        bp = out_Double(env, binPosWeight), ps = out_Double(env, binPsum), wd = out_Long(env, words);
  const jlong m = bins_n(nBins);
  int rc = checked(req_open(env, h, w, r, &q), bx.bad | by.bad | s.bad | bw.bad | bp.bad | ps.bad | wd.bad,
                   s.n < DSGD_WCALIBRATION_SUMS || wd.n < DSGD_ISOTONIC_EVAL_WORDS || bw.n < m || bp.n < m || ps.n < m ||
                       bx.n != by.n);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_weighted_isotonic_calibration, dsgd_eval_sampled_weighted_isotonic_calibration,
                  dsgd_eval_samples_weighted_isotonic_calibration, bx.p, by.p, bx.n, nBins, (double *)s.p, (double *)bw.p,
                  (double *)bp.p, (double *)ps.p, (int64_t *)wd.p);
  back_Double(env, sums, s, rc);
  back_Double(env, binWeight, bw, rc);
  back_Double(env, binPosWeight, bp, rc);
  back_Double(env, binPsum, ps, rc);
  back_Long(env, words, wd, rc);
  req_close(&q);
  free(bx.p); free(by.p);
  return rc;
}
FN(evalWeightedIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                    jdoubleArray x, jdoubleArray y, jint nBins, jdoubleArray sums, jdoubleArray binWeight,
                                    jdoubleArray binPosWeight, jdoubleArray binPsum, jlongArray words) {
  return req_wiso_quality(env, h, w, range_rows(rowBegin, rowEnd), x, y, nBins, sums, binWeight, binPosWeight, binPsum,
                          words);
}
FN(evalSampledWeightedIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                           jlong key, jlong posBegin, jlong posEnd, jdoubleArray x, jdoubleArray y,
                                           jint nBins, jdoubleArray sums, jdoubleArray binWeight,
                                           jdoubleArray binPosWeight, jdoubleArray binPsum, jlongArray words) {
  return req_wiso_quality(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), x, y, nBins, sums, binWeight,
                          binPosWeight, binPsum, words);
}
FN(evalSamplesWeightedIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples,
                                           jdoubleArray x, jdoubleArray y, jint nBins, jdoubleArray sums,
                                           jdoubleArray binWeight, jdoubleArray binPosWeight, jdoubleArray binPsum,
                                           jlongArray words) {
  return req_wiso_quality(env, h, w, list_rows(samples), x, y, nBins, sums, binWeight, binPosWeight, binPsum, words);
}

/* ---- sync mode ---- */
FN(commUniqueId)(JNIEnv *env, jobject self, jbyteArray id) {
  buf_t b = out_Byte(env, id);
  int rc = b.bad ? DSGD_ERR_NOMEM : (b.n < DSGD_UNIQUE_ID_BYTES ? DSGD_ERR_INVALID : dsgd_comm_unique_id((uint8_t *)b.p));
  back_Byte(env, id, b, rc);
  return rc;
}
FN(commInit)(JNIEnv *env, jobject self, jlong h, jbyteArray id) {
  buf_t b = in_Byte(env, id);
  int rc = b.bad ? DSGD_ERR_NOMEM : (b.n < DSGD_UNIQUE_ID_BYTES ? DSGD_ERR_INVALID : dsgd_comm_init(CTX(h), (const uint8_t *)b.p));
  free(b.p);
  return rc;
}
FN(xchgExport)(JNIEnv *env, jobject self, jlong h, jbyteArray handle) {
  buf_t b = out_Byte(env, handle);
  int rc = b.bad ? DSGD_ERR_NOMEM : (b.n < DSGD_IPC_HANDLE_BYTES ? DSGD_ERR_INVALID : dsgd_xchg_export(CTX(h), (uint8_t *)b.p));
  back_Byte(env, handle, b, rc);
  return rc;
}
FN(xchgImport)(JNIEnv *env, jobject self, jlong h, jint peerRank, jbyteArray handle) {
  buf_t b = in_Byte(env, handle);
  int rc = b.bad ? DSGD_ERR_NOMEM
                 : (b.n < DSGD_IPC_HANDLE_BYTES ? DSGD_ERR_INVALID : dsgd_xchg_import(CTX(h), peerRank, (const uint8_t *)b.p));
  free(b.p);
  return rc;
}
/* one JVM driving all GPUs of the box: the Master's slave list (core/Master.scala:222-243) becomes attach calls */
FN(xchgAttach)(JNIEnv *env, jobject self, jlong h, jint peerRank, jlong peer) { return dsgd_xchg_attach(CTX(h), peerRank, CTX(peer)); }
FN(xchgStats)(JNIEnv *env, jobject self, jlong h, jlongArray out) {   /* out(0) value words, (1) bitmap words, (2) steps */
  buf_t b = out_Long(env, out);
  int rc = b.bad ? DSGD_ERR_NOMEM
                 : (b.n < 3 ? DSGD_ERR_INVALID : dsgd_xchg_stats(CTX(h), (int64_t *)b.p, (int64_t *)b.p + 1, (int64_t *)b.p + 2));
  back_Long(env, out, b, rc);
  return rc;
}
FN(streamExactRows)(JNIEnv *env, jobject self, jlong h, jlongArray out) {   /* rows the streaming pass recomputed in fp64 */
  buf_t b = out_Long(env, out);
  int rc = b.bad ? DSGD_ERR_NOMEM : (b.n < 1 ? DSGD_ERR_INVALID : dsgd_stream_exact_rows(CTX(h), (int64_t *)b.p));
  back_Long(env, out, b, rc);
  return rc;
}
FN(setWorkers)(JNIEnv *env, jobject self, jlong h, jintArray counts, jint kTotal) {
  buf_t b = in_Int(env, counts);
  int rc = b.bad ? DSGD_ERR_NOMEM : dsgd_set_workers(CTX(h), b.n, b.p, kTotal);
  free(b.p);
  return rc;
}
FN(syncSteps)(JNIEnv *env, jobject self, jlong h, jintArray samples, jlong n_per_step, jlong n_steps, jdouble lr,
              jdoubleArray losses) {
  buf_t bs = in_Int(env, samples), bl = out_Double(env, losses);
  int rc = DSGD_ERR_NOMEM;
  if (!(bs.bad | bl.bad)) {
    if ((jlong)bs.n < n_per_step * n_steps || (bl.p && (jlong)bl.n < n_steps)) rc = DSGD_ERR_INVALID;
    else rc = dsgd_sync_steps(CTX(h), bs.p, n_per_step, n_steps, lr, bl.p);   /* Master.fit's batch loop, core/Master.scala:179-198 */
  }
  back_Double(env, losses, bl, rc);
  free(bs.p);
  return rc;
}
/* the same with a learning rate per step: lrs(s) for step s (a decaying schedule inside one call) */
FN(syncStepsLr)(JNIEnv *env, jobject self, jlong h, jintArray samples, jlong n_per_step, jlong n_steps, jdoubleArray lrs,
                jdoubleArray losses) {
  buf_t bs = in_Int(env, samples), br = in_Double(env, lrs), bl = out_Double(env, losses);
  int rc = DSGD_ERR_NOMEM;
  if (!(bs.bad | br.bad | bl.bad)) {
    if ((jlong)bs.n < n_per_step * n_steps || (jlong)br.n < n_steps || (bl.p && (jlong)bl.n < n_steps)) rc = DSGD_ERR_INVALID;
    else rc = dsgd_sync_steps_lr(CTX(h), bs.p, n_per_step, n_steps, br.p, bl.p);
  }
  back_Double(env, losses, bl, rc);
  free(bs.p); free(br.p);
  return rc;
}
/* averaged SGD: begin zeroes the device-side sum, every following sync step adds its new weights; avg(dim) = the mean,
 * nSteps(0) = the number of steps averaged (either array may be null) */
FN(averageBegin)(JNIEnv *env, jobject self, jlong h) { return dsgd_average_begin(CTX(h)); }
FN(averageEnd)(JNIEnv *env, jobject self, jlong h) { return dsgd_average_end(CTX(h)); }
FN(averageWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray avg, jlongArray nSteps) {
  buf_t ba = out_Double(env, avg), bn = out_Long(env, nSteps);
  int rc = checked(sized(h, &ba, WEIGHTS, AT_LEAST), bn.bad, short_of(&bn, 1));
  if (rc == DSGD_OK) rc = dsgd_average_weights(CTX(h), (double *)ba.p, (int64_t *)bn.p);
  back_Double(env, avg, ba, rc);
  back_Long(env, nSteps, bn, rc);
  return rc;
}
/* L1 penalty of the sync steps: setL1(lambda1 >= 0); weightsL1: l1(0) = ||w||_1 and nnz(0) = the non-zero weights of w (dim
 * values, dim + 1 with an intercept, which the norm leaves out), or of the resident weights when w is null.  A w of another
 * length, or an empty output array, is DSGD_ERR_INVALID. */
FN(setL1)(JNIEnv *env, jobject self, jlong h, jdouble lambda1) { return dsgd_set_l1(CTX(h), lambda1); }
FN(weightsL1)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jdoubleArray l1, jlongArray nnz) {
  req_t q;
  buf_t bl = out_Double(env, l1), bn = out_Long(env, nnz);
  int rc = checked(req_open(env, h, w, no_rows(), &q), bl.bad | bn.bad, short_of(&bl, 1) || short_of(&bn, 1));
  if (rc == DSGD_OK) rc = dsgd_weights_l1(CTX(h), (const double *)q.w.p, (double *)bl.p, (int64_t *)bn.p);
  back_Double(env, l1, bl, rc);
  back_Long(env, nnz, bn, rc);
  req_close(&q);
  return rc;
}
/* Class weights of the sync steps and of gradient: setClassWeights(wPos, wNeg), both finite and >= 0; getClassWeights:
 * out(0) = wPos, out(1) = wNeg.  The per-class evaluations, either model: sums(0) = ||w||^2, sums(1..2) = the unweighted loss
 * sums of the y = +1 and y = -1 rows; counts(0..3) = correct+, correct-, n+, n-.  A shorter output is DSGD_ERR_INVALID. */
FN(setClassWeights)(JNIEnv *env, jobject self, jlong h, jdouble wPos, jdouble wNeg) {
  return dsgd_set_class_weights(CTX(h), wPos, wNeg);
}
FN(getClassWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray out) {
  buf_t bo = out_Double(env, out);
  int rc = DSGD_ERR_NOMEM;
  if (!bo.bad) rc = bo.n < 2 ? DSGD_ERR_INVALID : dsgd_get_class_weights(CTX(h), (double *)bo.p, (double *)bo.p + 1);
  back_Double(env, out, bo, rc);
  return rc;
}
static int req_class(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdoubleArray sums, jlongArray counts) {
  req_t q;
  buf_t s = out_Double(env, sums), c = out_Long(env, counts);
  int rc = checked(req_open(env, h, w, r, &q), s.bad | c.bad, s.n < 3 || c.n < 4);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_class, dsgd_eval_sampled_class, dsgd_eval_samples_class, (double *)s.p, (double *)s.p + 1,
                  (int64_t *)c.p);
  back_Double(env, sums, s, rc);
  back_Long(env, counts, c, rc);
  req_close(&q);
  return rc;
}
FN(evalClass)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray sums,
              jlongArray counts) {
  return req_class(env, h, w, range_rows(rowBegin, rowEnd), sums, counts);
}
FN(evalSampledClass)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                     jlong posBegin, jlong posEnd, jdoubleArray sums, jlongArray counts) {
  return req_class(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), sums, counts);
}
FN(evalSamplesClass)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray sums,
                     jlongArray counts) {
  return req_class(env, h, w, list_rows(samples), sums, counts);
}

/* Sample weights of the sync steps, of gradient and of the weighted evaluations: setSampleWeights(sw), one weight per loaded
 * row (finite and >= 0; the library checks the length against the rows), null clears them.  The weighted evaluations, either
 * model: sums(0) = ||w||^2, sums(1..3) = S = sum c_i L_i, sum c_i [correct], sum c_i; counts(0..1) = rows, correct.  A
 * shorter output is DSGD_ERR_INVALID. */
FN(setSampleWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray sw) {
  buf_t b = in_Double(env, sw);
  int rc = b.bad ? DSGD_ERR_NOMEM : dsgd_set_sample_weights(CTX(h), (const double *)b.p, b.p ? (int64_t)b.n : 0);
  free(b.p);
  return rc;
}
/* ---- topics (sync mode) ---- */
/* the rows loaded on the ctx, which dsgd_info names (read under info_lock, as weight_len reads it) */
static int loaded_rows(jlong h, jlong *n) {
  int32_t dim = 0;
  int rc = dsgd_dim(CTX(h), &dim);
  if (rc != DSGD_OK) return rc;
  pthread_mutex_lock(&info_lock);
  const char *s = strstr(dsgd_info(CTX(h)), "\"n_rows\": ");
  *n = s ? strtoll(s + strlen("\"n_rows\": "), NULL, 10) : -1;
  pthread_mutex_unlock(&info_lock);
  return *n < 0 ? DSGD_ERR_INVALID : DSGD_OK;
}
/* topicPtr exactly rows + 1 long, and topicId exactly topicPtr(rows) */
FN(loadTopics)(JNIEnv *env, jobject self, jlong h, jint nTopics, jlongArray topicPtr, jintArray topicId) {
  buf_t p = in_Long(env, topicPtr), t = in_Int(env, topicId);
  jlong n = 0;
  int rc = checked(loaded_rows(h, &n), p.bad | t.bad, 0);
  if (rc == DSGD_OK) rc = checked(DSGD_OK, 0, !p.p || p.n != n + 1 || ((const int64_t *)p.p)[n] != (int64_t)t.n);
  if (rc == DSGD_OK) rc = dsgd_load_topics(CTX(h), nTopics, (const int64_t *)p.p, (const int32_t *)t.p);
  free(p.p); free(t.p);
  return rc;
}
FN(selectTopic)(JNIEnv *env, jobject self, jlong h, jint topic) { return dsgd_select_topic(CTX(h), topic); }
/* W exactly nTopics weight vectors long (null: refused by the library), out at least DSGD_TOPIC_WORDS(nTopics) */
static int req_topics(JNIEnv *env, jlong h, jdoubleArray W, jint nTopics, rows_t r, jlongArray out) {
  buf_t bw = in_Double(env, W), o = out_Long(env, out);
  r.ids = in_Int(env, r.samples);
  int32_t wl = 0;
  int rc = checked(weight_len(h, &wl), bw.bad | o.bad | r.ids.bad, 0);
  if (rc == DSGD_OK)
    rc = checked(DSGD_OK, 0, nTopics < 1 || (bw.p && bw.n != (jlong)nTopics * wl) || o.n < DSGD_TOPIC_WORDS(nTopics));
  if (rc == DSGD_OK)
    rc = r.form == RANGE ? dsgd_eval_topics(CTX(h), bw.p, nTopics, r.rowBegin, r.rowEnd, o.p)
         : r.form == DRAWN ? dsgd_eval_sampled_topics(CTX(h), bw.p, nTopics, r.rowBegin, r.rowEnd, (uint64_t)r.key, r.posBegin,
                                                      r.posEnd, o.p)
                           : dsgd_eval_samples_topics(CTX(h), bw.p, nTopics, r.ids.p, r.ids.n, o.p);
  back_Long(env, out, o, rc);
  free(bw.p); free(r.ids.p);
  return rc;
}
FN(evalTopics)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jlong rowBegin, jlong rowEnd,
               jlongArray out) {
  return req_topics(env, h, W, nTopics, range_rows(rowBegin, rowEnd), out);
}
FN(evalSampledTopics)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jlong rowBegin, jlong rowEnd,
                      jlong key, jlong posBegin, jlong posEnd, jlongArray out) {
  return req_topics(env, h, W, nTopics, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), out);
}
FN(evalSamplesTopics)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jintArray samples, jlongArray out) {
  return req_topics(env, h, W, nTopics, list_rows(samples), out);
}
/* W exactly nTopics weight vectors long (null: refused by the library), thresholds at least nTopics long (null: refused by
 * the library), out at least DSGD_TOPIC_WORDS(nTopics) */
static int req_thresholded_topics(JNIEnv *env, jlong h, jdoubleArray W, jint nTopics, jdoubleArray thresholds, rows_t r,
                                  jlongArray out) {
  buf_t bw = in_Double(env, W), bt = in_Double(env, thresholds), o = out_Long(env, out);
  r.ids = in_Int(env, r.samples);
  int32_t wl = 0;
  int rc = checked(weight_len(h, &wl), bw.bad | bt.bad | o.bad | r.ids.bad, 0);
  if (rc == DSGD_OK)
    rc = checked(DSGD_OK, 0, nTopics < 1 || (bw.p && bw.n != (jlong)nTopics * wl) || (bt.p && bt.n < (jlong)nTopics) ||
                                 o.n < DSGD_TOPIC_WORDS(nTopics));
  if (rc == DSGD_OK)
    rc = r.form == RANGE ? dsgd_eval_thresholded_topics(CTX(h), bw.p, nTopics, bt.p, r.rowBegin, r.rowEnd, o.p)
         : r.form == DRAWN ? dsgd_eval_sampled_thresholded_topics(CTX(h), bw.p, nTopics, bt.p, r.rowBegin, r.rowEnd,
                                                                  (uint64_t)r.key, r.posBegin, r.posEnd, o.p)
                           : dsgd_eval_samples_thresholded_topics(CTX(h), bw.p, nTopics, bt.p, r.ids.p, r.ids.n, o.p);
  back_Long(env, out, o, rc);
  free(bw.p); free(bt.p); free(r.ids.p);
  return rc;
}
FN(evalThresholdedTopics)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jdoubleArray thresholds,
                          jlong rowBegin, jlong rowEnd, jlongArray out) {
  return req_thresholded_topics(env, h, W, nTopics, thresholds, range_rows(rowBegin, rowEnd), out);
}
FN(evalSampledThresholdedTopics)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jdoubleArray thresholds,
                                 jlong rowBegin, jlong rowEnd, jlong key, jlong posBegin, jlong posEnd, jlongArray out) {
  return req_thresholded_topics(env, h, W, nTopics, thresholds, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), out);
}
FN(evalSamplesThresholdedTopics)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jdoubleArray thresholds,
                                 jintArray samples, jlongArray out) {
  return req_thresholded_topics(env, h, W, nTopics, thresholds, list_rows(samples), out);
}
/* W exactly nTopics weight vectors long (null: refused by the library), thresholds at least nTopics and words at least
 * DSGD_TOPIC_TUNE_WORDS(nTopics) long */
static int req_tune_topic_thresholds(JNIEnv *env, jlong h, jdoubleArray W, jint nTopics, jdouble fbr, rows_t r,
                                     jdoubleArray thresholds, jlongArray words) {
  buf_t bw = in_Double(env, W), t = out_Double(env, thresholds), o = out_Long(env, words);
  r.ids = in_Int(env, r.samples);
  int32_t wl = 0;
  int rc = checked(weight_len(h, &wl), bw.bad | t.bad | o.bad | r.ids.bad, 0);
  if (rc == DSGD_OK)
    rc = checked(DSGD_OK, 0, nTopics < 1 || (bw.p && bw.n != (jlong)nTopics * wl) || t.n < (jlong)nTopics ||
                                 o.n < DSGD_TOPIC_TUNE_WORDS(nTopics));
  if (rc == DSGD_OK)
    rc = r.form == RANGE ? dsgd_tune_topic_thresholds(CTX(h), bw.p, nTopics, fbr, r.rowBegin, r.rowEnd, t.p, o.p)
         : r.form == DRAWN ? dsgd_tune_topic_thresholds_sampled(CTX(h), bw.p, nTopics, fbr, r.rowBegin, r.rowEnd,
                                                                (uint64_t)r.key, r.posBegin, r.posEnd, t.p, o.p)
                           : dsgd_tune_topic_thresholds_samples(CTX(h), bw.p, nTopics, fbr, r.ids.p, r.ids.n, t.p, o.p);
  back_Double(env, thresholds, t, rc);
  back_Long(env, words, o, rc);
  free(bw.p); free(r.ids.p);
  return rc;
}
FN(tuneTopicThresholds)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jdouble fbr, jlong rowBegin,
                        jlong rowEnd, jdoubleArray thresholds, jlongArray words) {
  return req_tune_topic_thresholds(env, h, W, nTopics, fbr, range_rows(rowBegin, rowEnd), thresholds, words);
}
FN(tuneTopicThresholdsSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jdouble fbr,
                               jlong rowBegin, jlong rowEnd, jlong key, jlong posBegin, jlong posEnd,
                               jdoubleArray thresholds, jlongArray words) {
  return req_tune_topic_thresholds(env, h, W, nTopics, fbr, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd),
                                   thresholds, words);
}
FN(tuneTopicThresholdsSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jdouble fbr,
                               jintArray samples, jdoubleArray thresholds, jlongArray words) {
  return req_tune_topic_thresholds(env, h, W, nTopics, fbr, list_rows(samples), thresholds, words);
}
/* W exactly nTopics weight vectors long (null: refused by the library), words at least DSGD_TOPIC_RANK_WORDS(k) and sums
 * at least 2 + k (k itself is checked by the library) */
static int req_topic_ranking(JNIEnv *env, jlong h, jdoubleArray W, jint nTopics, jint k, rows_t r, jlongArray words,
                             jdoubleArray sums) {
  buf_t bw = in_Double(env, W), o = out_Long(env, words), s = out_Double(env, sums);
  r.ids = in_Int(env, r.samples);
  int32_t wl = 0;
  int rc = checked(weight_len(h, &wl), bw.bad | o.bad | s.bad | r.ids.bad, 0);
  if (rc == DSGD_OK)
    rc = checked(DSGD_OK, 0, nTopics < 1 || k < 1 || k > DSGD_TOPIC_RANK_MAX_K || (bw.p && bw.n != (jlong)nTopics * wl) ||
                                 o.n < DSGD_TOPIC_RANK_WORDS(k) || s.n < 2 + (jlong)k);
  if (rc == DSGD_OK)
    rc = r.form == RANGE ? dsgd_eval_topic_ranking(CTX(h), bw.p, nTopics, k, r.rowBegin, r.rowEnd, o.p, s.p)
         : r.form == DRAWN ? dsgd_eval_sampled_topic_ranking(CTX(h), bw.p, nTopics, k, r.rowBegin, r.rowEnd, (uint64_t)r.key,
                                                             r.posBegin, r.posEnd, o.p, s.p)
                           : dsgd_eval_samples_topic_ranking(CTX(h), bw.p, nTopics, k, r.ids.p, r.ids.n, o.p, s.p);
  back_Long(env, words, o, rc);
  back_Double(env, sums, s, rc);
  free(bw.p); free(r.ids.p);
  return rc;
}
FN(evalTopicRanking)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jint k, jlong rowBegin, jlong rowEnd,
                     jlongArray words, jdoubleArray sums) {
  return req_topic_ranking(env, h, W, nTopics, k, range_rows(rowBegin, rowEnd), words, sums);
}
FN(evalSampledTopicRanking)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jint k, jlong rowBegin,
                            jlong rowEnd, jlong key, jlong posBegin, jlong posEnd, jlongArray words, jdoubleArray sums) {
  return req_topic_ranking(env, h, W, nTopics, k, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), words, sums);
}
FN(evalSamplesTopicRanking)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jint k, jintArray samples,
                            jlongArray words, jdoubleArray sums) {
  return req_topic_ranking(env, h, W, nTopics, k, list_rows(samples), words, sums);
}
/* W exactly nTopics weight vectors long, ids and margins at least samples.length * k */
FN(topicsTopk)(JNIEnv *env, jobject self, jlong h, jdoubleArray W, jint nTopics, jint k, jintArray samples, jintArray ids,
               jdoubleArray margins) {
  buf_t bw = in_Double(env, W), sm = in_Int(env, samples), oi = out_Int(env, ids), om = out_Double(env, margins);
  int32_t wl = 0;
  int rc = checked(weight_len(h, &wl), bw.bad | sm.bad | oi.bad | om.bad, 0);
  const jlong nk = (jlong)sm.n * (k > 0 ? k : 0);
  if (rc == DSGD_OK)
    rc = checked(DSGD_OK, 0, nTopics < 1 || k < 1 || k > DSGD_TOPIC_RANK_MAX_K || (bw.p && bw.n != (jlong)nTopics * wl) ||
                                 !oi.p || !om.p || oi.n < nk || om.n < nk);
  if (rc == DSGD_OK) rc = dsgd_topics_topk(CTX(h), bw.p, nTopics, k, sm.p, sm.n, oi.p, om.p);
  back_Int(env, ids, oi, rc);
  back_Double(env, margins, om, rc);
  free(bw.p); free(sm.p);
  return rc;
}
static int req_weighted(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jdoubleArray sums, jlongArray counts) {
  req_t q;
  buf_t s = out_Double(env, sums), c = out_Long(env, counts);
  int rc = checked(req_open(env, h, w, r, &q), s.bad | c.bad, s.n < 4 || c.n < 2);
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_weighted, dsgd_eval_sampled_weighted, dsgd_eval_samples_weighted, (double *)s.p,
                  (double *)s.p + 1, (int64_t *)c.p);
  back_Double(env, sums, s, rc);
  back_Long(env, counts, c, rc);
  req_close(&q);
  return rc;
}
FN(evalWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray sums,
                 jlongArray counts) {
  return req_weighted(env, h, w, range_rows(rowBegin, rowEnd), sums, counts);
}
FN(evalSampledWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                        jlong posBegin, jlong posEnd, jdoubleArray sums, jlongArray counts) {
  return req_weighted(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), sums, counts);
}
FN(evalSamplesWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray sums,
                        jlongArray counts) {
  return req_weighted(env, h, w, list_rows(samples), sums, counts);
}

/* weighted curves: metrics(0..7) as the curve calls', wsums(0 until DSGD_WCURVE_WORDS) the weighted words, nPoints(0) = m, and
 * thr / tpw / fpw (0 until m) the points -- all three null for the words alone, else each at least as long as the request's
 * rows.  A shorter array is DSGD_ERR_INVALID, checked before the call. */
static int req_wcurve(JNIEnv *env, jlong h, jdoubleArray w, rows_t r, jlongArray metrics, jdoubleArray wsums,
                      jlongArray nPoints, jdoubleArray thr, jdoubleArray tpw, jdoubleArray fpw) {
  req_t q;
  buf_t m = out_Long(env, metrics), s = out_Double(env, wsums), k = out_Long(env, nPoints), t = out_Double(env, thr),
        bt = out_Double(env, tpw), bf = out_Double(env, fpw);
  int rc = req_open(env, h, w, r, &q);
  const jlong n = rows_n(&q);
  rc = checked(rc, m.bad | s.bad | k.bad | t.bad | bt.bad | bf.bad,
               m.n < DSGD_METRICS_WORDS || s.n < DSGD_WCURVE_WORDS || k.n < 1 || short_of(&t, n) || short_of(&bt, n) ||
                   short_of(&bf, n));
  if (rc == DSGD_OK)
    rc = ROW_CALL(h, q, dsgd_eval_weighted_curve, dsgd_eval_sampled_weighted_curve, dsgd_eval_samples_weighted_curve,
                  (int64_t *)m.p, (double *)s.p, (int64_t *)k.p, (double *)t.p, (double *)bt.p, (double *)bf.p);
  back_Long(env, metrics, m, rc);
  back_Double(env, wsums, s, rc);
  back_Long(env, nPoints, k, rc);
  back_Double(env, thr, t, rc);
  back_Double(env, tpw, bt, rc);
  back_Double(env, fpw, bf, rc);
  req_close(&q);
  return rc;
}
FN(evalWeightedCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray metrics,
                      jdoubleArray wsums, jlongArray nPoints, jdoubleArray thr, jdoubleArray tpw, jdoubleArray fpw) {
  return req_wcurve(env, h, w, range_rows(rowBegin, rowEnd), metrics, wsums, nPoints, thr, tpw, fpw);
}
FN(evalSampledWeightedCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                             jlong posBegin, jlong posEnd, jlongArray metrics, jdoubleArray wsums, jlongArray nPoints,
                             jdoubleArray thr, jdoubleArray tpw, jdoubleArray fpw) {
  return req_wcurve(env, h, w, drawn_rows(rowBegin, rowEnd, key, posBegin, posEnd), metrics, wsums, nPoints, thr, tpw, fpw);
}
FN(evalSamplesWeightedCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray metrics,
                             jdoubleArray wsums, jlongArray nPoints, jdoubleArray thr, jdoubleArray tpw, jdoubleArray fpw) {
  return req_wcurve(env, h, w, list_rows(samples), metrics, wsums, nPoints, thr, tpw, fpw);
}

/* ---- async (Hogwild) mode ---- */
FN(asyncHostMaster)(JNIEnv *env, jobject self, jlong h, jdoubleArray w0) {
  buf_t b = in_Double(env, w0);
  int rc = sized(h, &b, DIM, EXACTLY);
  if (rc == DSGD_OK) rc = dsgd_async_host_master(CTX(h), b.p);   /* GradState of MasterAsync, core/MasterAsync.scala:66 */
  free(b.p);
  return rc;
}
FN(ipcExport)(JNIEnv *env, jobject self, jlong h, jint which, jbyteArray handle) {
  buf_t b = out_Byte(env, handle);
  int rc = b.bad ? DSGD_ERR_NOMEM : (b.n < DSGD_IPC_HANDLE_BYTES ? DSGD_ERR_INVALID : dsgd_ipc_export(CTX(h), which, (uint8_t *)b.p));
  back_Byte(env, handle, b, rc);
  return rc;
}
FN(ipcImport)(JNIEnv *env, jobject self, jlong h, jint peerRank, jbyteArray handle) {
  buf_t b = in_Byte(env, handle);
  int rc = b.bad ? DSGD_ERR_NOMEM
                 : (b.n < DSGD_IPC_HANDLE_BYTES ? DSGD_ERR_INVALID : dsgd_ipc_import(CTX(h), peerRank, (const uint8_t *)b.p));
  free(b.p);
  return rc;
}
FN(peerAttach)(JNIEnv *env, jobject self, jlong h, jint peerRank, jlong peer, jint which) {
  return dsgd_peer_attach(CTX(h), peerRank, CTX(peer), which);             /* the slave<->slave channels, core/Slave.scala:23,26 */
}
FN(startAsync)(JNIEnv *env, jobject self, jlong h, jdoubleArray w0, jintArray assigned, jint batch, jdouble lr,
               jint concurrency, jlong maxUpdates, jlong seed) {
  buf_t bw = in_Double(env, w0), ba = in_Int(env, assigned);
  int rc = checked(sized(h, &bw, DIM, EXACTLY), ba.bad, 0);
  if (rc == DSGD_OK)
    rc = dsgd_start_async(CTX(h), bw.p, ba.p, ba.n, batch, lr, concurrency, maxUpdates, (uint64_t)seed);  /* core/Slave.scala:159-175 */
  free(bw.p); free(ba.p);
  return rc;
}
FN(stopAsync)(JNIEnv *env, jobject self, jlong h) { return dsgd_stop_async(CTX(h)); }   /* core/Slave.scala:187-195 */
FN(asyncRunning)(JNIEnv *env, jobject self, jlong h, jintArray out) {
  buf_t b = out_Int(env, out);
  int rc = b.bad ? DSGD_ERR_NOMEM : (b.n < 1 ? DSGD_ERR_INVALID : dsgd_async_running(CTX(h), (int *)b.p));
  back_Int(env, out, b, rc);
  return rc;
}
FN(updateGrad)(JNIEnv *env, jobject self, jlong h, jintArray idx, jdoubleArray value) {
  buf_t bi = in_Int(env, idx), bv = in_Double(env, value);
  int rc = DSGD_ERR_NOMEM;
  if (!(bi.bad | bv.bad)) rc = bi.n != bv.n ? DSGD_ERR_INVALID : dsgd_update_grad(CTX(h), bi.p, bv.p, bi.n);  /* core/Slave.scala:177-185 */
  free(bi.p); free(bv.p);
  return rc;
}
FN(asyncUpdates)(JNIEnv *env, jobject self, jlong h, jlongArray out) {
  buf_t b = out_Long(env, out);
  int rc = b.bad ? DSGD_ERR_NOMEM : (b.n < 1 ? DSGD_ERR_INVALID : dsgd_async_updates(CTX(h), (int64_t *)b.p));  /* GradState.updates */
  back_Long(env, out, b, rc);
  return rc;
}
FN(asyncMasterWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray out) {
  buf_t b = out_Double(env, out);
  int rc = sized(h, &b, DIM, AT_LEAST);
  if (rc == DSGD_OK) rc = dsgd_async_master_weights(CTX(h), b.p);   /* gradState.single().grad, core/MasterAsync.scala:109 */
  back_Double(env, out, b, rc);
  return rc;
}
FN(asyncOutboxEnable)(JNIEnv *env, jobject self, jlong h) {
  (void)env; (void)self;
  return dsgd_async_outbox_enable(CTX(h));            /* deltas for colleagues reached over gRPC, core/Slave.scala:104-105 */
}
FN(asyncOutboxRead)(JNIEnv *env, jobject self, jlong h, jdoubleArray out) {
  buf_t b = out_Double(env, out);
  int rc = sized(h, &b, DIM, AT_LEAST);
  if (rc == DSGD_OK) rc = dsgd_async_outbox_read(CTX(h), b.p);
  back_Double(env, out, b, rc);
  return rc;
}
#endif /* DSGD_HAVE_JNI */
