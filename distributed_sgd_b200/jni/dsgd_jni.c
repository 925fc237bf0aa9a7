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
 * tests/test_abi_surface.py compiles this file against a minimal stand-in jni.h (tests/jni_mock/) -- a syntax and type
 * check against include/dsgd.h, not a run under a JVM -- and checks that the facade covers the header. */
#ifdef DSGD_HAVE_JNI
#include <jni.h>
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
  int rc = DSGD_ERR_NOMEM;                               /* Dataset.rcv1 rows as CSR (utils/Dataset.scala:23-47) */
  if (!(rp.bad | c.bad | v.bad | l.bad))
    rc = rp.n < 1 ? DSGD_ERR_INVALID : dsgd_load_csr(CTX(h), rp.n - 1, c.n, rp.p, c.p, v.p, l.p);
  free(rp.p); free(c.p); free(v.p); free(l.p);
  return rc;
}
FN(setDimSparsity)(JNIEnv *env, jobject self, jlong h, jdoubleArray d) {
  buf_t b = in_Double(env, d);
  int rc = b.bad ? DSGD_ERR_NOMEM : dsgd_set_dim_sparsity(CTX(h), b.p);            /* SparseSVM.dimSparsity */
  free(b.p);
  return rc;
}
FN(computeDimSparsity)(JNIEnv *env, jobject self, jlong h, jlong nTrain, jdoubleArray out) {
  buf_t o = out_Double(env, out);
  int rc = o.bad ? DSGD_ERR_NOMEM : dsgd_compute_dim_sparsity(CTX(h), nTrain, o.p); /* Main.scala:54-65 */
  back_Double(env, out, o, rc);
  return rc;
}
FN(setWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray w) {
  buf_t b = in_Double(env, w);
  int rc = b.bad ? DSGD_ERR_NOMEM : dsgd_set_weights(CTX(h), b.p);
  free(b.p);
  return rc;
}
FN(getWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray w) {
  buf_t o = out_Double(env, w);
  int rc = o.bad ? DSGD_ERR_NOMEM : dsgd_get_weights(CTX(h), o.p);
  back_Double(env, w, o, rc);
  return rc;
}

/* ---- requests ---- */
FN(gradient)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray grad) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bg = out_Double(env, grad);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bg.bad)) rc = dsgd_gradient(CTX(h), bw.p, bs.p, bs.n, bg.p, NULL);  /* core/Slave.scala:142-157 */
  back_Double(env, grad, bg, rc);
  free(bw.p); free(bs.p);
  return rc;
}
FN(forward)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray preds) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bp = out_Double(env, preds);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bp.bad)) rc = dsgd_forward(CTX(h), bw.p, bs.p, bs.n, bp.p);          /* core/Slave.scala:129-140 */
  back_Double(env, preds, bp, rc);
  free(bw.p); free(bs.p);
  return rc;
}
FN(eval)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray lossAcc) {
  buf_t bw = in_Double(env, w), bo = out_Double(env, lossAcc);          /* lossAcc(0) = loss, lossAcc(1) = accuracy */
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bo.bad))
    rc = bo.n < 2 ? DSGD_ERR_INVALID
                  : dsgd_eval(CTX(h), bw.p, rowBegin, rowEnd, (double *)bo.p, (double *)bo.p + 1);  /* core/Master.scala:100-107 */
  back_Double(env, lossAcc, bo, rc);
  free(bw.p);
  return rc;
}
FN(evalCounts)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray hingeCorrect,
               jdoubleArray normSquared) {
  buf_t bw = in_Double(env, w), bc = out_Long(env, hingeCorrect), bn = out_Double(env, normSquared);
  int rc = DSGD_ERR_NOMEM;               /* exact shardable form: hingeCorrect(0) = hinge sum, (1) = #correct */
  if (!(bw.bad | bc.bad | bn.bad))
    rc = (bc.n < 2 || bn.n < 1) ? DSGD_ERR_INVALID
                                : dsgd_eval_counts(CTX(h), bw.p, rowBegin, rowEnd, (int64_t *)bc.p, (int64_t *)bc.p + 1, bn.p);
  back_Long(env, hingeCorrect, bc, rc);
  back_Double(env, normSquared, bn, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledCounts)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                      jlong posBegin, jlong posEnd, jlongArray hingeCorrect, jdoubleArray normSquared) {
  buf_t bw = in_Double(env, w), bc = out_Long(env, hingeCorrect), bn = out_Double(env, normSquared);
  int rc = DSGD_ERR_NOMEM;               /* core/Master.scala:109-118, sample drawn on the device: positions [posBegin, posEnd) */
  if (!(bw.bad | bc.bad | bn.bad))
    rc = (bc.n < 2 || bn.n < 1) ? DSGD_ERR_INVALID
                                : dsgd_eval_sampled_counts(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd,
                                                           (int64_t *)bc.p, (int64_t *)bc.p + 1, bn.p);
  back_Long(env, hingeCorrect, bc, rc);
  back_Double(env, normSquared, bn, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesCounts)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray hingeCorrect,
                      jdoubleArray normSquared) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bc = out_Long(env, hingeCorrect), bn = out_Double(env, normSquared);
  int rc = DSGD_ERR_NOMEM;               /* the same counters over row ids the JVM drew with its own Random */
  if (!(bw.bad | bs.bad | bc.bad | bn.bad))
    rc = (bc.n < 2 || bn.n < 1) ? DSGD_ERR_INVALID
                                : dsgd_eval_samples_counts(CTX(h), bw.p, bs.p, bs.n, (int64_t *)bc.p, (int64_t *)bc.p + 1, bn.p);
  back_Long(env, hingeCorrect, bc, rc);
  back_Double(env, normSquared, bn, rc);
  free(bw.p); free(bs.p);
  return rc;
}
/* The *Sums forms serve either model (the *Counts forms refuse a logistic ctx): lossSumNormSquared(0) = sum of the per-sample
 * losses, (1) = ||w||^2; correct(0) = #correct. */
FN(evalSums)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray lossSumNormSquared,
             jlongArray correct) {
  buf_t bw = in_Double(env, w), bs = out_Double(env, lossSumNormSquared), bc = out_Long(env, correct);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bc.bad))
    rc = (bs.n < 2 || bc.n < 1) ? DSGD_ERR_INVALID
                                : dsgd_eval_sums(CTX(h), bw.p, rowBegin, rowEnd, (double *)bs.p, (int64_t *)bc.p, (double *)bs.p + 1);
  back_Double(env, lossSumNormSquared, bs, rc);
  back_Long(env, correct, bc, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledSums)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                    jlong posBegin, jlong posEnd, jdoubleArray lossSumNormSquared, jlongArray correct) {
  buf_t bw = in_Double(env, w), bs = out_Double(env, lossSumNormSquared), bc = out_Long(env, correct);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bc.bad))
    rc = (bs.n < 2 || bc.n < 1) ? DSGD_ERR_INVALID
                                : dsgd_eval_sampled_sums(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd,
                                                         (double *)bs.p, (int64_t *)bc.p, (double *)bs.p + 1);
  back_Double(env, lossSumNormSquared, bs, rc);
  back_Long(env, correct, bc, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesSums)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray lossSumNormSquared,
                    jlongArray correct) {
  buf_t bw = in_Double(env, w), bi = in_Int(env, samples), bs = out_Double(env, lossSumNormSquared),
        bc = out_Long(env, correct);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bi.bad | bs.bad | bc.bad))
    rc = (bs.n < 2 || bc.n < 1) ? DSGD_ERR_INVALID
                                : dsgd_eval_samples_sums(CTX(h), bw.p, bi.p, bi.n, (double *)bs.p, (int64_t *)bc.p,
                                                         (double *)bs.p + 1);
  back_Double(env, lossSumNormSquared, bs, rc);
  back_Long(env, correct, bc, rc);
  free(bw.p); free(bi.p);
  return rc;
}
/* scores and ranking metrics, either model: out(i) = x_i . w (margins) or P(y = +1 | x_i) (probabilities, SparseLogistic
 * only); metrics(0..7) = the DSGD_METRICS_WORDS counts of dsgd_eval_metrics.  An output shorter than that is DSGD_ERR_INVALID. */
FN(margins)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray out) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bo = out_Double(env, out);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bo.bad)) rc = bo.n < bs.n ? DSGD_ERR_INVALID : dsgd_margins(CTX(h), bw.p, bs.p, bs.n, bo.p);
  back_Double(env, out, bo, rc);
  free(bw.p); free(bs.p);
  return rc;
}
FN(probabilities)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray out) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bo = out_Double(env, out);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bo.bad)) rc = bo.n < bs.n ? DSGD_ERR_INVALID : dsgd_probabilities(CTX(h), bw.p, bs.p, bs.n, bo.p);
  back_Double(env, out, bo, rc);
  free(bw.p); free(bs.p);
  return rc;
}
FN(evalMetrics)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray metrics) {
  buf_t bw = in_Double(env, w), bm = out_Long(env, metrics);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bm.bad))
    rc = bm.n < DSGD_METRICS_WORDS ? DSGD_ERR_INVALID : dsgd_eval_metrics(CTX(h), bw.p, rowBegin, rowEnd, (int64_t *)bm.p);
  back_Long(env, metrics, bm, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledMetrics)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                       jlong posBegin, jlong posEnd, jlongArray metrics) {
  buf_t bw = in_Double(env, w), bm = out_Long(env, metrics);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bm.bad))
    rc = bm.n < DSGD_METRICS_WORDS ? DSGD_ERR_INVALID
                                   : dsgd_eval_sampled_metrics(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd,
                                                               (int64_t *)bm.p);
  back_Long(env, metrics, bm, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesMetrics)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray metrics) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bm = out_Long(env, metrics);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bm.bad))
    rc = bm.n < DSGD_METRICS_WORDS ? DSGD_ERR_INVALID : dsgd_eval_samples_metrics(CTX(h), bw.p, bs.p, bs.n, (int64_t *)bm.p);
  back_Long(env, metrics, bm, rc);
  free(bw.p); free(bs.p);
  return rc;
}
/* curves and average precision: metrics(0..7) as above, ap(0) = average precision, nPoints(0) = m, and thr / tp / fp (0 until
 * m) the points, highest score first -- all three null for average precision alone, else each at least as long as the
 * request's rows (n = rowEnd - rowBegin, posEnd - posBegin or samples.length).  A shorter array is DSGD_ERR_INVALID. */
typedef struct { buf_t m, a, k, t, tp, fp; } curve_bufs;
static curve_bufs curve_out(JNIEnv *env, jlongArray metrics, jdoubleArray ap, jlongArray nPoints, jdoubleArray thr,
                            jlongArray tp, jlongArray fp) {
  curve_bufs c = {out_Long(env, metrics), out_Double(env, ap), out_Long(env, nPoints), out_Double(env, thr),
                  out_Long(env, tp), out_Long(env, fp)};
  return c;
}
static int curve_bad(const curve_bufs *c) { return c->m.bad | c->a.bad | c->k.bad | c->t.bad | c->tp.bad | c->fp.bad; }
static int curve_short(const curve_bufs *c, jlong n) {
  if (c->m.n < DSGD_METRICS_WORDS || c->a.n < 1 || c->k.n < 1) return 1;
  return (c->t.p && c->t.n < n) || (c->tp.p && c->tp.n < n) || (c->fp.p && c->fp.n < n);
}
static void curve_back(JNIEnv *env, jlongArray metrics, jdoubleArray ap, jlongArray nPoints, jdoubleArray thr, jlongArray tp,
                       jlongArray fp, curve_bufs *c, int rc) {
  back_Long(env, metrics, c->m, rc);
  back_Double(env, ap, c->a, rc);
  back_Long(env, nPoints, c->k, rc);
  back_Double(env, thr, c->t, rc);
  back_Long(env, tp, c->tp, rc);
  back_Long(env, fp, c->fp, rc);
}
FN(evalCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray metrics,
              jdoubleArray ap, jlongArray nPoints, jdoubleArray thr, jlongArray tp, jlongArray fp) {
  buf_t bw = in_Double(env, w);
  curve_bufs c = curve_out(env, metrics, ap, nPoints, thr, tp, fp);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | curve_bad(&c)))
    rc = curve_short(&c, rowEnd - rowBegin)
             ? DSGD_ERR_INVALID
             : dsgd_eval_curve(CTX(h), bw.p, rowBegin, rowEnd, (int64_t *)c.m.p, (double *)c.a.p, (int64_t *)c.k.p,
                               (double *)c.t.p, (int64_t *)c.tp.p, (int64_t *)c.fp.p);
  curve_back(env, metrics, ap, nPoints, thr, tp, fp, &c, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                     jlong posBegin, jlong posEnd, jlongArray metrics, jdoubleArray ap, jlongArray nPoints, jdoubleArray thr,
                     jlongArray tp, jlongArray fp) {
  buf_t bw = in_Double(env, w);
  curve_bufs c = curve_out(env, metrics, ap, nPoints, thr, tp, fp);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | curve_bad(&c)))
    rc = curve_short(&c, posEnd - posBegin)
             ? DSGD_ERR_INVALID
             : dsgd_eval_sampled_curve(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd, (int64_t *)c.m.p,
                                       (double *)c.a.p, (int64_t *)c.k.p, (double *)c.t.p, (int64_t *)c.tp.p,
                                       (int64_t *)c.fp.p);
  curve_back(env, metrics, ap, nPoints, thr, tp, fp, &c, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray metrics,
                     jdoubleArray ap, jlongArray nPoints, jdoubleArray thr, jlongArray tp, jlongArray fp) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples);
  curve_bufs c = curve_out(env, metrics, ap, nPoints, thr, tp, fp);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | curve_bad(&c)))
    rc = curve_short(&c, bs.n)
             ? DSGD_ERR_INVALID
             : dsgd_eval_samples_curve(CTX(h), bw.p, bs.p, bs.n, (int64_t *)c.m.p, (double *)c.a.p, (int64_t *)c.k.p,
                                       (double *)c.t.p, (int64_t *)c.tp.p, (int64_t *)c.fp.p);
  curve_back(env, metrics, ap, nPoints, thr, tp, fp, &c, rc);
  free(bw.p); free(bs.p);
  return rc;
}

/* Poisson bootstrap: replicates [bBegin, bEnd) with key bKey; words(9 j .. 9 j + 8) = the DSGD_BOOTSTRAP_WORDS words of
 * replicate bBegin + j, ap(j) its average precision, loss(j) its loss sum.  An output shorter than the replicates is
 * DSGD_ERR_INVALID. */
typedef struct { buf_t m, a, l; } boot_bufs;
static boot_bufs boot_out(JNIEnv *env, jlongArray words, jdoubleArray ap, jdoubleArray loss) {
  boot_bufs c = {out_Long(env, words), out_Double(env, ap), out_Double(env, loss)};
  return c;
}
static int boot_bad(const boot_bufs *c) { return c->m.bad | c->a.bad | c->l.bad; }
static int boot_short(const boot_bufs *c, jlong bBegin, jlong bEnd) {
  const jlong k = bEnd > bBegin ? bEnd - bBegin : 0;
  return c->m.n < k * DSGD_BOOTSTRAP_WORDS || c->a.n < k || c->l.n < k;
}
static void boot_back(JNIEnv *env, jlongArray words, jdoubleArray ap, jdoubleArray loss, boot_bufs *c, int rc) {
  back_Long(env, words, c->m, rc);
  back_Double(env, ap, c->a, rc);
  back_Double(env, loss, c->l, rc);
}
FN(evalBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong bKey, jlong bBegin,
                  jlong bEnd, jlongArray words, jdoubleArray ap, jdoubleArray loss) {
  buf_t bw = in_Double(env, w);
  boot_bufs c = boot_out(env, words, ap, loss);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | boot_bad(&c)))
    rc = boot_short(&c, bBegin, bEnd) ? DSGD_ERR_INVALID
                                      : dsgd_eval_bootstrap(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)bKey, bBegin, bEnd,
                                                            (int64_t *)c.m.p, (double *)c.a.p, (double *)c.l.p);
  boot_back(env, words, ap, loss, &c, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                         jlong posBegin, jlong posEnd, jlong bKey, jlong bBegin, jlong bEnd, jlongArray words,
                         jdoubleArray ap, jdoubleArray loss) {
  buf_t bw = in_Double(env, w);
  boot_bufs c = boot_out(env, words, ap, loss);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | boot_bad(&c)))
    rc = boot_short(&c, bBegin, bEnd)
             ? DSGD_ERR_INVALID
             : dsgd_eval_sampled_bootstrap(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd, (uint64_t)bKey,
                                           bBegin, bEnd, (int64_t *)c.m.p, (double *)c.a.p, (double *)c.l.p);
  boot_back(env, words, ap, loss, &c, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlong bKey, jlong bBegin,
                         jlong bEnd, jlongArray words, jdoubleArray ap, jdoubleArray loss) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples);
  boot_bufs c = boot_out(env, words, ap, loss);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | boot_bad(&c)))
    rc = boot_short(&c, bBegin, bEnd) ? DSGD_ERR_INVALID
                                      : dsgd_eval_samples_bootstrap(CTX(h), bw.p, bs.p, bs.n, (uint64_t)bKey, bBegin, bEnd,
                                                                    (int64_t *)c.m.p, (double *)c.a.p, (double *)c.l.p);
  boot_back(env, words, ap, loss, &c, rc);
  free(bw.p); free(bs.p);
  return rc;
}

/* weighted Poisson bootstrap: replicates [bBegin, bEnd) with key bKey; words(2 j), words(2 j + 1) = the size and the NaN-score
 * rows of replicate bBegin + j, wsums(13 j .. 13 j + 12) its DSGD_WCURVE_WORDS, loss(j) its weighted loss sum.  The buffers
 * are those of the unweighted bootstrap, with wsums in ap's place.  An output shorter than the replicates is
 * DSGD_ERR_INVALID. */
static int wboot_short(const boot_bufs *c, jlong bBegin, jlong bEnd) {
  const jlong k = bEnd > bBegin ? bEnd - bBegin : 0;
  return c->m.n < k * 2 || c->a.n < k * DSGD_WCURVE_WORDS || c->l.n < k;
}
FN(evalWeightedBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong bKey,
                          jlong bBegin, jlong bEnd, jlongArray words, jdoubleArray wsums, jdoubleArray loss) {
  buf_t bw = in_Double(env, w);
  boot_bufs c = boot_out(env, words, wsums, loss);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | boot_bad(&c)))
    rc = wboot_short(&c, bBegin, bEnd)
             ? DSGD_ERR_INVALID
             : dsgd_eval_weighted_bootstrap(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)bKey, bBegin, bEnd, (int64_t *)c.m.p,
                                            (double *)c.a.p, (double *)c.l.p);
  boot_back(env, words, wsums, loss, &c, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledWeightedBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                                 jlong posBegin, jlong posEnd, jlong bKey, jlong bBegin, jlong bEnd, jlongArray words,
                                 jdoubleArray wsums, jdoubleArray loss) {
  buf_t bw = in_Double(env, w);
  boot_bufs c = boot_out(env, words, wsums, loss);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | boot_bad(&c)))
    rc = wboot_short(&c, bBegin, bEnd)
             ? DSGD_ERR_INVALID
             : dsgd_eval_sampled_weighted_bootstrap(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd,
                                                    (uint64_t)bKey, bBegin, bEnd, (int64_t *)c.m.p, (double *)c.a.p,
                                                    (double *)c.l.p);
  boot_back(env, words, wsums, loss, &c, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesWeightedBootstrap)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlong bKey,
                                 jlong bBegin, jlong bEnd, jlongArray words, jdoubleArray wsums, jdoubleArray loss) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples);
  boot_bufs c = boot_out(env, words, wsums, loss);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | boot_bad(&c)))
    rc = wboot_short(&c, bBegin, bEnd)
             ? DSGD_ERR_INVALID
             : dsgd_eval_samples_weighted_bootstrap(CTX(h), bw.p, bs.p, bs.n, (uint64_t)bKey, bBegin, bEnd, (int64_t *)c.m.p,
                                                    (double *)c.a.p, (double *)c.l.p);
  boot_back(env, words, wsums, loss, &c, rc);
  free(bw.p); free(bs.p);
  return rc;
}

/* calibration: ab(0..1) = (A, B), objective(0) = F(A, B), info(0..4) = the DSGD_CALIBRATION_INFO_WORDS words; probabilities:
 * out(i) = sigmoid(-(a x_i . w + b)); quality: sums(0..1) = Brier and log-loss sums, binRows / binPos / binPsum at least nBins
 * long, words(0..1) = rows used and left out.  A shorter array is DSGD_ERR_INVALID. */
typedef struct { buf_t ab, f, info; } calib_bufs;
static calib_bufs calib_out(JNIEnv *env, jdoubleArray ab, jdoubleArray objective, jlongArray info) {
  calib_bufs c = {out_Double(env, ab), out_Double(env, objective), out_Long(env, info)};
  return c;
}
static int calib_bad(const calib_bufs *c) { return c->ab.bad | c->f.bad | c->info.bad; }
static int calib_short(const calib_bufs *c) { return c->ab.n < 2 || c->f.n < 1 || c->info.n < DSGD_CALIBRATION_INFO_WORDS; }
static void calib_back(JNIEnv *env, jdoubleArray ab, jdoubleArray objective, jlongArray info, calib_bufs *c, int rc) {
  back_Double(env, ab, c->ab, rc);
  back_Double(env, objective, c->f, rc);
  back_Long(env, info, c->info, rc);
}
FN(calibrate)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray ab,
              jdoubleArray objective, jlongArray info) {
  buf_t bw = in_Double(env, w);
  calib_bufs c = calib_out(env, ab, objective, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | calib_bad(&c)))
    rc = calib_short(&c) ? DSGD_ERR_INVALID
                         : dsgd_calibrate(CTX(h), bw.p, rowBegin, rowEnd, (double *)c.ab.p, (double *)c.f.p, (int64_t *)c.info.p);
  calib_back(env, ab, objective, info, &c, rc);
  free(bw.p);
  return rc;
}
FN(calibrateSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                     jlong posBegin, jlong posEnd, jdoubleArray ab, jdoubleArray objective, jlongArray info) {
  buf_t bw = in_Double(env, w);
  calib_bufs c = calib_out(env, ab, objective, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | calib_bad(&c)))
    rc = calib_short(&c) ? DSGD_ERR_INVALID
                         : dsgd_calibrate_sampled(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd,
                                                  (double *)c.ab.p, (double *)c.f.p, (int64_t *)c.info.p);
  calib_back(env, ab, objective, info, &c, rc);
  free(bw.p);
  return rc;
}
FN(calibrateSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray ab,
                     jdoubleArray objective, jlongArray info) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples);
  calib_bufs c = calib_out(env, ab, objective, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | calib_bad(&c)))
    rc = calib_short(&c) ? DSGD_ERR_INVALID
                         : dsgd_calibrate_samples(CTX(h), bw.p, bs.p, bs.n, (double *)c.ab.p, (double *)c.f.p, (int64_t *)c.info.p);
  calib_back(env, ab, objective, info, &c, rc);
  free(bw.p); free(bs.p);
  return rc;
}
FN(calibratedProbabilities)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdouble a, jdouble b,
                            jdoubleArray out) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bo = out_Double(env, out);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bo.bad))
    rc = bo.n < bs.n ? DSGD_ERR_INVALID : dsgd_calibrated_probabilities(CTX(h), bw.p, bs.p, bs.n, a, b, bo.p);
  back_Double(env, out, bo, rc);
  free(bw.p); free(bs.p);
  return rc;
}
typedef struct { buf_t s, r, p, ps, wd; } quality_bufs;
static quality_bufs quality_out(JNIEnv *env, jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum,
                                jlongArray words) {
  quality_bufs q = {out_Double(env, sums), out_Long(env, binRows), out_Long(env, binPos), out_Double(env, binPsum),
                    out_Long(env, words)};
  return q;
}
static int quality_bad(const quality_bufs *q) { return q->s.bad | q->r.bad | q->p.bad | q->ps.bad | q->wd.bad; }
/* nBins outside 1 .. DSGD_CALIBRATION_MAX_BINS is the library's DSGD_ERR_INVALID: only the lengths are checked here */
static int quality_short(const quality_bufs *q, jint nBins) {
  const jlong m = nBins > 0 ? nBins : 0;
  return q->s.n < 2 || q->wd.n < 2 || q->r.n < m || q->p.n < m || q->ps.n < m;
}
static void quality_back(JNIEnv *env, jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum,
                         jlongArray words, quality_bufs *q, int rc) {
  back_Double(env, sums, q->s, rc);
  back_Long(env, binRows, q->r, rc);
  back_Long(env, binPos, q->p, rc);
  back_Double(env, binPsum, q->ps, rc);
  back_Long(env, words, q->wd, rc);
}
FN(evalCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdouble a, jdouble b,
                    jint nBins, jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum,
                    jlongArray words) {
  buf_t bw = in_Double(env, w);
  quality_bufs q = quality_out(env, sums, binRows, binPos, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | quality_bad(&q)))
    rc = quality_short(&q, nBins)
             ? DSGD_ERR_INVALID
             : dsgd_eval_calibration(CTX(h), bw.p, rowBegin, rowEnd, a, b, nBins, (double *)q.s.p, (int64_t *)q.r.p,
                                     (int64_t *)q.p.p, (double *)q.ps.p, (int64_t *)q.wd.p);
  quality_back(env, sums, binRows, binPos, binPsum, words, &q, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                           jlong posBegin, jlong posEnd, jdouble a, jdouble b, jint nBins, jdoubleArray sums,
                           jlongArray binRows, jlongArray binPos, jdoubleArray binPsum, jlongArray words) {
  buf_t bw = in_Double(env, w);
  quality_bufs q = quality_out(env, sums, binRows, binPos, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | quality_bad(&q)))
    rc = quality_short(&q, nBins)
             ? DSGD_ERR_INVALID
             : dsgd_eval_sampled_calibration(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd, a, b, nBins,
                                             (double *)q.s.p, (int64_t *)q.r.p, (int64_t *)q.p.p, (double *)q.ps.p,
                                             (int64_t *)q.wd.p);
  quality_back(env, sums, binRows, binPos, binPsum, words, &q, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdouble a, jdouble b,
                           jint nBins, jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum,
                           jlongArray words) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples);
  quality_bufs q = quality_out(env, sums, binRows, binPos, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | quality_bad(&q)))
    rc = quality_short(&q, nBins)
             ? DSGD_ERR_INVALID
             : dsgd_eval_samples_calibration(CTX(h), bw.p, bs.p, bs.n, a, b, nBins, (double *)q.s.p, (int64_t *)q.r.p,
                                             (int64_t *)q.p.p, (double *)q.ps.p, (int64_t *)q.wd.p);
  quality_back(env, sums, binRows, binPos, binPsum, words, &q, rc);
  free(bw.p); free(bs.p);
  return rc;
}

/* weighted calibration: the calibration natives with wsums(0..2) = W+, W- and the NaN rows' weight added to a fit; quality:
 * sums(0..3) = weighted Brier and log-loss sums, the weight used and the infinite-term weight, binWeight / binPosWeight /
 * binPsum at least nBins long (doubles), words(0..1) as there.  A shorter array is DSGD_ERR_INVALID. */
static int wcalib_short(const calib_bufs *c, const buf_t *ws) { return calib_short(c) || ws->n < DSGD_CALIBRATION_WSUMS; }
FN(calibrateWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray ab,
                      jdoubleArray objective, jlongArray info, jdoubleArray wsums) {
  buf_t bw = in_Double(env, w), ws = out_Double(env, wsums);
  calib_bufs c = calib_out(env, ab, objective, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | ws.bad | calib_bad(&c)))
    rc = wcalib_short(&c, &ws) ? DSGD_ERR_INVALID
                               : dsgd_calibrate_weighted(CTX(h), bw.p, rowBegin, rowEnd, (double *)c.ab.p, (double *)c.f.p,
                                                         (int64_t *)c.info.p, ws.p);
  calib_back(env, ab, objective, info, &c, rc);
  back_Double(env, wsums, ws, rc);
  free(bw.p);
  return rc;
}
FN(calibrateWeightedSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                             jlong posBegin, jlong posEnd, jdoubleArray ab, jdoubleArray objective, jlongArray info,
                             jdoubleArray wsums) {
  buf_t bw = in_Double(env, w), ws = out_Double(env, wsums);
  calib_bufs c = calib_out(env, ab, objective, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | ws.bad | calib_bad(&c)))
    rc = wcalib_short(&c, &ws) ? DSGD_ERR_INVALID
                               : dsgd_calibrate_weighted_sampled(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin,
                                                                 posEnd, (double *)c.ab.p, (double *)c.f.p,
                                                                 (int64_t *)c.info.p, ws.p);
  calib_back(env, ab, objective, info, &c, rc);
  back_Double(env, wsums, ws, rc);
  free(bw.p);
  return rc;
}
FN(calibrateWeightedSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray ab,
                             jdoubleArray objective, jlongArray info, jdoubleArray wsums) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), ws = out_Double(env, wsums);
  calib_bufs c = calib_out(env, ab, objective, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | ws.bad | calib_bad(&c)))
    rc = wcalib_short(&c, &ws) ? DSGD_ERR_INVALID
                               : dsgd_calibrate_weighted_samples(CTX(h), bw.p, bs.p, bs.n, (double *)c.ab.p, (double *)c.f.p,
                                                                 (int64_t *)c.info.p, ws.p);
  calib_back(env, ab, objective, info, &c, rc);
  back_Double(env, wsums, ws, rc);
  free(bw.p); free(bs.p);
  return rc;
}
typedef struct { buf_t s, wt, pw, ps, wd; } wquality_bufs;
static wquality_bufs wquality_out(JNIEnv *env, jdoubleArray sums, jdoubleArray binWeight, jdoubleArray binPosWeight,
                                  jdoubleArray binPsum, jlongArray words) {
  wquality_bufs q = {out_Double(env, sums), out_Double(env, binWeight), out_Double(env, binPosWeight),
                     out_Double(env, binPsum), out_Long(env, words)};
  return q;
}
static int wquality_bad(const wquality_bufs *q) { return q->s.bad | q->wt.bad | q->pw.bad | q->ps.bad | q->wd.bad; }
static int wquality_short(const wquality_bufs *q, jint nBins) {
  const jlong m = nBins > 0 ? nBins : 0;
  return q->s.n < DSGD_WCALIBRATION_SUMS || q->wd.n < 2 || q->wt.n < m || q->pw.n < m || q->ps.n < m;
}
static void wquality_back(JNIEnv *env, jdoubleArray sums, jdoubleArray binWeight, jdoubleArray binPosWeight,
                          jdoubleArray binPsum, jlongArray words, wquality_bufs *q, int rc) {
  back_Double(env, sums, q->s, rc);
  back_Double(env, binWeight, q->wt, rc);
  back_Double(env, binPosWeight, q->pw, rc);
  back_Double(env, binPsum, q->ps, rc);
  back_Long(env, words, q->wd, rc);
}
FN(evalWeightedCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdouble a,
                            jdouble b, jint nBins, jdoubleArray sums, jdoubleArray binWeight, jdoubleArray binPosWeight,
                            jdoubleArray binPsum, jlongArray words) {
  buf_t bw = in_Double(env, w);
  wquality_bufs q = wquality_out(env, sums, binWeight, binPosWeight, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | wquality_bad(&q)))
    rc = wquality_short(&q, nBins)
             ? DSGD_ERR_INVALID
             : dsgd_eval_weighted_calibration(CTX(h), bw.p, rowBegin, rowEnd, a, b, nBins, q.s.p, q.wt.p, q.pw.p, q.ps.p,
                                              (int64_t *)q.wd.p);
  wquality_back(env, sums, binWeight, binPosWeight, binPsum, words, &q, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledWeightedCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                   jlong key, jlong posBegin, jlong posEnd, jdouble a, jdouble b, jint nBins,
                                   jdoubleArray sums, jdoubleArray binWeight, jdoubleArray binPosWeight,
                                   jdoubleArray binPsum, jlongArray words) {
  buf_t bw = in_Double(env, w);
  wquality_bufs q = wquality_out(env, sums, binWeight, binPosWeight, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | wquality_bad(&q)))
    rc = wquality_short(&q, nBins)
             ? DSGD_ERR_INVALID
             : dsgd_eval_sampled_weighted_calibration(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd, a, b,
                                                      nBins, q.s.p, q.wt.p, q.pw.p, q.ps.p, (int64_t *)q.wd.p);
  wquality_back(env, sums, binWeight, binPosWeight, binPsum, words, &q, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesWeightedCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdouble a,
                                   jdouble b, jint nBins, jdoubleArray sums, jdoubleArray binWeight,
                                   jdoubleArray binPosWeight, jdoubleArray binPsum, jlongArray words) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples);
  wquality_bufs q = wquality_out(env, sums, binWeight, binPosWeight, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | wquality_bad(&q)))
    rc = wquality_short(&q, nBins)
             ? DSGD_ERR_INVALID
             : dsgd_eval_samples_weighted_calibration(CTX(h), bw.p, bs.p, bs.n, a, b, nBins, q.s.p, q.wt.p, q.pw.p, q.ps.p,
                                                      (int64_t *)q.wd.p);
  wquality_back(env, sums, binWeight, binPosWeight, binPsum, words, &q, rc);
  free(bw.p); free(bs.p);
  return rc;
}

/* isotonic calibration: nPoints(0) = k, x / y(0 until k) the thresholds and their values, blockRows / blockPos(0 until
 * blocks), info(0..4) = the DSGD_ISOTONIC_INFO_WORDS words; x, y, blockRows and blockPos at least as long as the request's
 * rows.  Probabilities and quality at the map (x, y): x and y of one length k >= 1; out at least as long as samples; the
 * quality arrays as for evalCalibration, words(0..2) = rows used, rows left out and rows with an infinite log-loss term.
 * A shorter array is DSGD_ERR_INVALID. */
typedef struct { buf_t k, x, y, r, p, info; } iso_bufs;
static iso_bufs iso_out(JNIEnv *env, jlongArray nPoints, jdoubleArray x, jdoubleArray y, jlongArray blockRows,
                        jlongArray blockPos, jlongArray info) {
  iso_bufs c = {out_Long(env, nPoints), out_Double(env, x), out_Double(env, y), out_Long(env, blockRows),
                out_Long(env, blockPos), out_Long(env, info)};
  return c;
}
static int iso_bad(const iso_bufs *c) { return c->k.bad | c->x.bad | c->y.bad | c->r.bad | c->p.bad | c->info.bad; }
static int iso_short(const iso_bufs *c, jlong n) {
  return c->k.n < 1 || c->info.n < DSGD_ISOTONIC_INFO_WORDS || c->x.n < n || c->y.n < n || c->r.n < n || c->p.n < n;
}
static void iso_back(JNIEnv *env, jlongArray nPoints, jdoubleArray x, jdoubleArray y, jlongArray blockRows,
                     jlongArray blockPos, jlongArray info, iso_bufs *c, int rc) {
  back_Long(env, nPoints, c->k, rc);
  back_Double(env, x, c->x, rc);
  back_Double(env, y, c->y, rc);
  back_Long(env, blockRows, c->r, rc);
  back_Long(env, blockPos, c->p, rc);
  back_Long(env, info, c->info, rc);
}
FN(calibrateIsotonic)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray nPoints,
                      jdoubleArray x, jdoubleArray y, jlongArray blockRows, jlongArray blockPos, jlongArray info) {
  buf_t bw = in_Double(env, w);
  iso_bufs c = iso_out(env, nPoints, x, y, blockRows, blockPos, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | iso_bad(&c)))
    rc = iso_short(&c, rowEnd - rowBegin)
             ? DSGD_ERR_INVALID
             : dsgd_calibrate_isotonic(CTX(h), bw.p, rowBegin, rowEnd, (int64_t *)c.k.p, (double *)c.x.p, (double *)c.y.p,
                                       (int64_t *)c.r.p, (int64_t *)c.p.p, (int64_t *)c.info.p);
  iso_back(env, nPoints, x, y, blockRows, blockPos, info, &c, rc);
  free(bw.p);
  return rc;
}
FN(calibrateIsotonicSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                             jlong posBegin, jlong posEnd, jlongArray nPoints, jdoubleArray x, jdoubleArray y,
                             jlongArray blockRows, jlongArray blockPos, jlongArray info) {
  buf_t bw = in_Double(env, w);
  iso_bufs c = iso_out(env, nPoints, x, y, blockRows, blockPos, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | iso_bad(&c)))
    rc = iso_short(&c, posEnd - posBegin)
             ? DSGD_ERR_INVALID
             : dsgd_calibrate_isotonic_sampled(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd,
                                               (int64_t *)c.k.p, (double *)c.x.p, (double *)c.y.p, (int64_t *)c.r.p,
                                               (int64_t *)c.p.p, (int64_t *)c.info.p);
  iso_back(env, nPoints, x, y, blockRows, blockPos, info, &c, rc);
  free(bw.p);
  return rc;
}
FN(calibrateIsotonicSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray nPoints,
                             jdoubleArray x, jdoubleArray y, jlongArray blockRows, jlongArray blockPos, jlongArray info) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples);
  iso_bufs c = iso_out(env, nPoints, x, y, blockRows, blockPos, info);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | iso_bad(&c)))
    rc = iso_short(&c, bs.n)
             ? DSGD_ERR_INVALID
             : dsgd_calibrate_isotonic_samples(CTX(h), bw.p, bs.p, bs.n, (int64_t *)c.k.p, (double *)c.x.p, (double *)c.y.p,
                                               (int64_t *)c.r.p, (int64_t *)c.p.p, (int64_t *)c.info.p);
  iso_back(env, nPoints, x, y, blockRows, blockPos, info, &c, rc);
  free(bw.p); free(bs.p);
  return rc;
}
FN(isotonicProbabilities)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray x,
                          jdoubleArray y, jdoubleArray out) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bx = in_Double(env, x), by = in_Double(env, y),
        bo = out_Double(env, out);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bx.bad | by.bad | bo.bad))
    rc = bo.n < bs.n || bx.n != by.n ? DSGD_ERR_INVALID
                                     : dsgd_isotonic_probabilities(CTX(h), bw.p, bs.p, bs.n, bx.p, by.p, bx.n, bo.p);
  back_Double(env, out, bo, rc);
  free(bw.p); free(bs.p); free(bx.p); free(by.p);
  return rc;
}
static int iso_quality_short(const quality_bufs *q, jint nBins, const buf_t *bx, const buf_t *by) {
  return quality_short(q, nBins) || q->wd.n < DSGD_ISOTONIC_EVAL_WORDS || bx->n != by->n;
}
FN(evalIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray x,
                            jdoubleArray y, jint nBins, jdoubleArray sums, jlongArray binRows, jlongArray binPos,
                            jdoubleArray binPsum, jlongArray words) {
  buf_t bw = in_Double(env, w), bx = in_Double(env, x), by = in_Double(env, y);
  quality_bufs q = quality_out(env, sums, binRows, binPos, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bx.bad | by.bad | quality_bad(&q)))
    rc = iso_quality_short(&q, nBins, &bx, &by)
             ? DSGD_ERR_INVALID
             : dsgd_eval_isotonic_calibration(CTX(h), bw.p, rowBegin, rowEnd, bx.p, by.p, bx.n, nBins, (double *)q.s.p,
                                              (int64_t *)q.r.p, (int64_t *)q.p.p, (double *)q.ps.p, (int64_t *)q.wd.p);
  quality_back(env, sums, binRows, binPos, binPsum, words, &q, rc);
  free(bw.p); free(bx.p); free(by.p);
  return rc;
}
FN(evalSampledIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                   jlong key, jlong posBegin, jlong posEnd, jdoubleArray x, jdoubleArray y, jint nBins,
                                   jdoubleArray sums, jlongArray binRows, jlongArray binPos, jdoubleArray binPsum,
                                   jlongArray words) {
  buf_t bw = in_Double(env, w), bx = in_Double(env, x), by = in_Double(env, y);
  quality_bufs q = quality_out(env, sums, binRows, binPos, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bx.bad | by.bad | quality_bad(&q)))
    rc = iso_quality_short(&q, nBins, &bx, &by)
             ? DSGD_ERR_INVALID
             : dsgd_eval_sampled_isotonic_calibration(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd, bx.p,
                                                      by.p, bx.n, nBins, (double *)q.s.p, (int64_t *)q.r.p, (int64_t *)q.p.p,
                                                      (double *)q.ps.p, (int64_t *)q.wd.p);
  quality_back(env, sums, binRows, binPos, binPsum, words, &q, rc);
  free(bw.p); free(bx.p); free(by.p);
  return rc;
}
FN(evalSamplesIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray x,
                                   jdoubleArray y, jint nBins, jdoubleArray sums, jlongArray binRows, jlongArray binPos,
                                   jdoubleArray binPsum, jlongArray words) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bx = in_Double(env, x), by = in_Double(env, y);
  quality_bufs q = quality_out(env, sums, binRows, binPos, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bx.bad | by.bad | quality_bad(&q)))
    rc = iso_quality_short(&q, nBins, &bx, &by)
             ? DSGD_ERR_INVALID
             : dsgd_eval_samples_isotonic_calibration(CTX(h), bw.p, bs.p, bs.n, bx.p, by.p, bx.n, nBins, (double *)q.s.p,
                                                      (int64_t *)q.r.p, (int64_t *)q.p.p, (double *)q.ps.p,
                                                      (int64_t *)q.wd.p);
  quality_back(env, sums, binRows, binPos, binPsum, words, &q, rc);
  free(bw.p); free(bs.p); free(bx.p); free(by.p);
  return rc;
}

/* weighted isotonic calibration: the isotonic natives with blockWeight / blockPosWeight (doubles) in place of the block counts
 * and wsums(0..1) = W+, W- added to a fit; weighted quality at (x, y): the weighted quality arrays with words(0..2) as for
 * evalIsotonicCalibration.  A shorter array is DSGD_ERR_INVALID. */
typedef struct { buf_t k, x, y, r, p, info, ws; } wiso_bufs;
static wiso_bufs wiso_out(JNIEnv *env, jlongArray nPoints, jdoubleArray x, jdoubleArray y, jdoubleArray blockWeight,
                          jdoubleArray blockPosWeight, jlongArray info, jdoubleArray wsums) {
  wiso_bufs c = {out_Long(env, nPoints), out_Double(env, x), out_Double(env, y), out_Double(env, blockWeight),
                 out_Double(env, blockPosWeight), out_Long(env, info), out_Double(env, wsums)};
  return c;
}
static int wiso_bad(const wiso_bufs *c) {
  return c->k.bad | c->x.bad | c->y.bad | c->r.bad | c->p.bad | c->info.bad | c->ws.bad;
}
static int wiso_short(const wiso_bufs *c, jlong n) {
  return c->k.n < 1 || c->info.n < DSGD_ISOTONIC_INFO_WORDS || c->ws.n < 2 || c->x.n < n || c->y.n < n || c->r.n < n ||
         c->p.n < n;
}
static void wiso_back(JNIEnv *env, jlongArray nPoints, jdoubleArray x, jdoubleArray y, jdoubleArray blockWeight,
                      jdoubleArray blockPosWeight, jlongArray info, jdoubleArray wsums, wiso_bufs *c, int rc) {
  back_Long(env, nPoints, c->k, rc);
  back_Double(env, x, c->x, rc);
  back_Double(env, y, c->y, rc);
  back_Double(env, blockWeight, c->r, rc);
  back_Double(env, blockPosWeight, c->p, rc);
  back_Long(env, info, c->info, rc);
  back_Double(env, wsums, c->ws, rc);
}
FN(calibrateIsotonicWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                              jlongArray nPoints, jdoubleArray x, jdoubleArray y, jdoubleArray blockWeight,
                              jdoubleArray blockPosWeight, jlongArray info, jdoubleArray wsums) {
  buf_t bw = in_Double(env, w);
  wiso_bufs c = wiso_out(env, nPoints, x, y, blockWeight, blockPosWeight, info, wsums);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | wiso_bad(&c)))
    rc = wiso_short(&c, rowEnd - rowBegin)
             ? DSGD_ERR_INVALID
             : dsgd_calibrate_isotonic_weighted(CTX(h), bw.p, rowBegin, rowEnd, (int64_t *)c.k.p, c.x.p, c.y.p, c.r.p, c.p.p,
                                                (int64_t *)c.info.p, c.ws.p);
  wiso_back(env, nPoints, x, y, blockWeight, blockPosWeight, info, wsums, &c, rc);
  free(bw.p);
  return rc;
}
FN(calibrateIsotonicWeightedSampled)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                     jlong key, jlong posBegin, jlong posEnd, jlongArray nPoints, jdoubleArray x,
                                     jdoubleArray y, jdoubleArray blockWeight, jdoubleArray blockPosWeight, jlongArray info,
                                     jdoubleArray wsums) {
  buf_t bw = in_Double(env, w);
  wiso_bufs c = wiso_out(env, nPoints, x, y, blockWeight, blockPosWeight, info, wsums);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | wiso_bad(&c)))
    rc = wiso_short(&c, posEnd - posBegin)
             ? DSGD_ERR_INVALID
             : dsgd_calibrate_isotonic_weighted_sampled(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd,
                                                        (int64_t *)c.k.p, c.x.p, c.y.p, c.r.p, c.p.p, (int64_t *)c.info.p,
                                                        c.ws.p);
  wiso_back(env, nPoints, x, y, blockWeight, blockPosWeight, info, wsums, &c, rc);
  free(bw.p);
  return rc;
}
FN(calibrateIsotonicWeightedSamples)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples,
                                     jlongArray nPoints, jdoubleArray x, jdoubleArray y, jdoubleArray blockWeight,
                                     jdoubleArray blockPosWeight, jlongArray info, jdoubleArray wsums) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples);
  wiso_bufs c = wiso_out(env, nPoints, x, y, blockWeight, blockPosWeight, info, wsums);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | wiso_bad(&c)))
    rc = wiso_short(&c, bs.n)
             ? DSGD_ERR_INVALID
             : dsgd_calibrate_isotonic_weighted_samples(CTX(h), bw.p, bs.p, bs.n, (int64_t *)c.k.p, c.x.p, c.y.p, c.r.p,
                                                        c.p.p, (int64_t *)c.info.p, c.ws.p);
  wiso_back(env, nPoints, x, y, blockWeight, blockPosWeight, info, wsums, &c, rc);
  free(bw.p); free(bs.p);
  return rc;
}
static int wiso_quality_short(const wquality_bufs *q, jint nBins, const buf_t *bx, const buf_t *by) {
  return wquality_short(q, nBins) || q->wd.n < DSGD_ISOTONIC_EVAL_WORDS || bx->n != by->n;
}
FN(evalWeightedIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                    jdoubleArray x, jdoubleArray y, jint nBins, jdoubleArray sums, jdoubleArray binWeight,
                                    jdoubleArray binPosWeight, jdoubleArray binPsum, jlongArray words) {
  buf_t bw = in_Double(env, w), bx = in_Double(env, x), by = in_Double(env, y);
  wquality_bufs q = wquality_out(env, sums, binWeight, binPosWeight, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bx.bad | by.bad | wquality_bad(&q)))
    rc = wiso_quality_short(&q, nBins, &bx, &by)
             ? DSGD_ERR_INVALID
             : dsgd_eval_weighted_isotonic_calibration(CTX(h), bw.p, rowBegin, rowEnd, bx.p, by.p, bx.n, nBins, q.s.p, q.wt.p,
                                                       q.pw.p, q.ps.p, (int64_t *)q.wd.p);
  wquality_back(env, sums, binWeight, binPosWeight, binPsum, words, &q, rc);
  free(bw.p); free(bx.p); free(by.p);
  return rc;
}
FN(evalSampledWeightedIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd,
                                           jlong key, jlong posBegin, jlong posEnd, jdoubleArray x, jdoubleArray y,
                                           jint nBins, jdoubleArray sums, jdoubleArray binWeight,
                                           jdoubleArray binPosWeight, jdoubleArray binPsum, jlongArray words) {
  buf_t bw = in_Double(env, w), bx = in_Double(env, x), by = in_Double(env, y);
  wquality_bufs q = wquality_out(env, sums, binWeight, binPosWeight, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bx.bad | by.bad | wquality_bad(&q)))
    rc = wiso_quality_short(&q, nBins, &bx, &by)
             ? DSGD_ERR_INVALID
             : dsgd_eval_sampled_weighted_isotonic_calibration(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin,
                                                               posEnd, bx.p, by.p, bx.n, nBins, q.s.p, q.wt.p, q.pw.p,
                                                               q.ps.p, (int64_t *)q.wd.p);
  wquality_back(env, sums, binWeight, binPosWeight, binPsum, words, &q, rc);
  free(bw.p); free(bx.p); free(by.p);
  return rc;
}
FN(evalSamplesWeightedIsotonicCalibration)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples,
                                           jdoubleArray x, jdoubleArray y, jint nBins, jdoubleArray sums,
                                           jdoubleArray binWeight, jdoubleArray binPosWeight, jdoubleArray binPsum,
                                           jlongArray words) {
  buf_t bw = in_Double(env, w), bs = in_Int(env, samples), bx = in_Double(env, x), by = in_Double(env, y);
  wquality_bufs q = wquality_out(env, sums, binWeight, binPosWeight, binPsum, words);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bx.bad | by.bad | wquality_bad(&q)))
    rc = wiso_quality_short(&q, nBins, &bx, &by)
             ? DSGD_ERR_INVALID
             : dsgd_eval_samples_weighted_isotonic_calibration(CTX(h), bw.p, bs.p, bs.n, bx.p, by.p, bx.n, nBins, q.s.p,
                                                               q.wt.p, q.pw.p, q.ps.p, (int64_t *)q.wd.p);
  wquality_back(env, sums, binWeight, binPosWeight, binPsum, words, &q, rc);
  free(bw.p); free(bs.p); free(bx.p); free(by.p);
  return rc;
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
  int rc = DSGD_ERR_NOMEM;
  if (!(ba.bad | bn.bad))
    rc = (bn.p && bn.n < 1) ? DSGD_ERR_INVALID : dsgd_average_weights(CTX(h), (double *)ba.p, (int64_t *)bn.p);
  back_Double(env, avg, ba, rc);
  back_Long(env, nSteps, bn, rc);
  return rc;
}
/* The length of a weight vector of the ctx: dim, or dim + 1 on a ctx created with DSGD_FLAG_INTERCEPT (dsgd_info names it) */
static int weight_len(jlong h, int32_t *n) {
  int rc = dsgd_dim(CTX(h), n);
  if (rc == DSGD_OK && strstr(dsgd_info(CTX(h)), "\"intercept\": true")) ++*n;
  return rc;
}
/* L1 penalty of the sync steps: setL1(lambda1 >= 0); weightsL1: l1(0) = ||w||_1 and nnz(0) = the non-zero weights of w (dim
 * values, dim + 1 with an intercept, which the norm leaves out), or of the resident weights when w is null.  A w of another
 * length, or an empty output array, is DSGD_ERR_INVALID. */
FN(setL1)(JNIEnv *env, jobject self, jlong h, jdouble lambda1) { return dsgd_set_l1(CTX(h), lambda1); }
FN(weightsL1)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jdoubleArray l1, jlongArray nnz) {
  buf_t bw = in_Double(env, w), bl = out_Double(env, l1), bn = out_Long(env, nnz);
  int rc = DSGD_ERR_NOMEM;
  int32_t dim = 0;
  if (!(bw.bad | bl.bad | bn.bad) && (rc = weight_len(h, &dim)) == DSGD_OK)
    rc = (bw.p && (int32_t)bw.n != dim) || (bl.p && bl.n < 1) || (bn.p && bn.n < 1)
             ? DSGD_ERR_INVALID
             : dsgd_weights_l1(CTX(h), (const double *)bw.p, (double *)bl.p, (int64_t *)bn.p);
  back_Double(env, l1, bl, rc);
  back_Long(env, nnz, bn, rc);
  free(bw.p);
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
FN(evalClass)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray sums,
              jlongArray counts) {
  buf_t bw = in_Double(env, w), bs = out_Double(env, sums), bc = out_Long(env, counts);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bc.bad))
    rc = (bs.n < 3 || bc.n < 4) ? DSGD_ERR_INVALID
                                : dsgd_eval_class(CTX(h), bw.p, rowBegin, rowEnd, (double *)bs.p, (double *)bs.p + 1, (int64_t *)bc.p);
  back_Double(env, sums, bs, rc);
  back_Long(env, counts, bc, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledClass)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                     jlong posBegin, jlong posEnd, jdoubleArray sums, jlongArray counts) {
  buf_t bw = in_Double(env, w), bs = out_Double(env, sums), bc = out_Long(env, counts);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bc.bad))
    rc = (bs.n < 3 || bc.n < 4) ? DSGD_ERR_INVALID
                                : dsgd_eval_sampled_class(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd,
                                                          (double *)bs.p, (double *)bs.p + 1, (int64_t *)bc.p);
  back_Double(env, sums, bs, rc);
  back_Long(env, counts, bc, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesClass)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray sums,
                     jlongArray counts) {
  buf_t bw = in_Double(env, w), bi = in_Int(env, samples), bs = out_Double(env, sums), bc = out_Long(env, counts);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bi.bad | bs.bad | bc.bad))
    rc = (bs.n < 3 || bc.n < 4) ? DSGD_ERR_INVALID
                                : dsgd_eval_samples_class(CTX(h), bw.p, bi.p, bi.n, (double *)bs.p, (double *)bs.p + 1,
                                                          (int64_t *)bc.p);
  back_Double(env, sums, bs, rc);
  back_Long(env, counts, bc, rc);
  free(bw.p); free(bi.p);
  return rc;
}

/* Sample weights of the sync steps, of gradient and of the weighted evaluations: setSampleWeights(sw), one weight per loaded
 * row (finite and >= 0; the library checks the length against the rows), null clears them.  The weighted evaluations, either
 * model: sums(0) = ||w||^2, sums(1..3) = S = sum c_i L_i, sum c_i [correct], sum c_i; counts(0..1) = rows, correct.  A w
 * whose length is not dim, or a shorter output, is DSGD_ERR_INVALID. */
FN(setSampleWeights)(JNIEnv *env, jobject self, jlong h, jdoubleArray sw) {
  buf_t b = in_Double(env, sw);
  int rc = b.bad ? DSGD_ERR_NOMEM : dsgd_set_sample_weights(CTX(h), (const double *)b.p, b.p ? (int64_t)b.n : 0);
  free(b.p);
  return rc;
}
/* DSGD_OK when w is null or holds a weight vector (weight_len values) and the outputs are long enough */
static int weighted_args(jlong h, const buf_t *bw, const buf_t *bs, const buf_t *bc) {
  int32_t dim = 0;
  int rc = weight_len(h, &dim);
  if (rc) return rc;
  return ((bw->p && (int32_t)bw->n != dim) || bs->n < 4 || bc->n < 2) ? DSGD_ERR_INVALID : DSGD_OK;
}
FN(evalWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jdoubleArray sums,
                 jlongArray counts) {
  buf_t bw = in_Double(env, w), bs = out_Double(env, sums), bc = out_Long(env, counts);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bc.bad) && (rc = weighted_args(h, &bw, &bs, &bc)) == DSGD_OK)
    rc = dsgd_eval_weighted(CTX(h), bw.p, rowBegin, rowEnd, (double *)bs.p, (double *)bs.p + 1, (int64_t *)bc.p);
  back_Double(env, sums, bs, rc);
  back_Long(env, counts, bc, rc);
  free(bw.p);
  return rc;
}
FN(evalSampledWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                        jlong posBegin, jlong posEnd, jdoubleArray sums, jlongArray counts) {
  buf_t bw = in_Double(env, w), bs = out_Double(env, sums), bc = out_Long(env, counts);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bs.bad | bc.bad) && (rc = weighted_args(h, &bw, &bs, &bc)) == DSGD_OK)
    rc = dsgd_eval_sampled_weighted(CTX(h), bw.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd, (double *)bs.p,
                                    (double *)bs.p + 1, (int64_t *)bc.p);
  back_Double(env, sums, bs, rc);
  back_Long(env, counts, bc, rc);
  free(bw.p);
  return rc;
}
FN(evalSamplesWeighted)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jdoubleArray sums,
                        jlongArray counts) {
  buf_t bw = in_Double(env, w), bi = in_Int(env, samples), bs = out_Double(env, sums), bc = out_Long(env, counts);
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | bi.bad | bs.bad | bc.bad) && (rc = weighted_args(h, &bw, &bs, &bc)) == DSGD_OK)
    rc = dsgd_eval_samples_weighted(CTX(h), bw.p, bi.p, bi.n, (double *)bs.p, (double *)bs.p + 1, (int64_t *)bc.p);
  back_Double(env, sums, bs, rc);
  back_Long(env, counts, bc, rc);
  free(bw.p); free(bi.p);
  return rc;
}

/* weighted curves: metrics(0..7) as the curve calls', wsums(0 until DSGD_WCURVE_WORDS) the weighted words, nPoints(0) = m, and
 * thr / tpw / fpw (0 until m) the points -- all three null for the words alone, else each at least as long as the request's
 * rows.  w is null or holds dim values.  A shorter array is DSGD_ERR_INVALID, checked before the call. */
typedef struct { buf_t w, m, s, k, t, tp, fp; } wcurve_bufs;
static wcurve_bufs wcurve_in(JNIEnv *env, jdoubleArray w, jlongArray metrics, jdoubleArray wsums, jlongArray nPoints,
                             jdoubleArray thr, jdoubleArray tpw, jdoubleArray fpw) {
  wcurve_bufs c = {in_Double(env, w),      out_Long(env, metrics), out_Double(env, wsums), out_Long(env, nPoints),
                   out_Double(env, thr),   out_Double(env, tpw),   out_Double(env, fpw)};
  return c;
}
static int wcurve_bad(const wcurve_bufs *c) { return c->w.bad | c->m.bad | c->s.bad | c->k.bad | c->t.bad | c->tp.bad | c->fp.bad; }
static int wcurve_args(jlong h, const wcurve_bufs *c, jlong n) {
  int32_t dim = 0;
  int rc = weight_len(h, &dim);
  if (rc) return rc;
  if ((c->w.p && (int32_t)c->w.n != dim) || c->m.n < DSGD_METRICS_WORDS || c->s.n < DSGD_WCURVE_WORDS || c->k.n < 1)
    return DSGD_ERR_INVALID;
  return ((c->t.p && c->t.n < n) || (c->tp.p && c->tp.n < n) || (c->fp.p && c->fp.n < n)) ? DSGD_ERR_INVALID : DSGD_OK;
}
static void wcurve_back(JNIEnv *env, jlongArray metrics, jdoubleArray wsums, jlongArray nPoints, jdoubleArray thr,
                        jdoubleArray tpw, jdoubleArray fpw, wcurve_bufs *c, int rc) {
  back_Long(env, metrics, c->m, rc);
  back_Double(env, wsums, c->s, rc);
  back_Long(env, nPoints, c->k, rc);
  back_Double(env, thr, c->t, rc);
  back_Double(env, tpw, c->tp, rc);
  back_Double(env, fpw, c->fp, rc);
  free(c->w.p);
}
FN(evalWeightedCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlongArray metrics,
                      jdoubleArray wsums, jlongArray nPoints, jdoubleArray thr, jdoubleArray tpw, jdoubleArray fpw) {
  wcurve_bufs c = wcurve_in(env, w, metrics, wsums, nPoints, thr, tpw, fpw);
  int rc = DSGD_ERR_NOMEM;
  if (!wcurve_bad(&c) && (rc = wcurve_args(h, &c, rowEnd - rowBegin)) == DSGD_OK)
    rc = dsgd_eval_weighted_curve(CTX(h), c.w.p, rowBegin, rowEnd, (int64_t *)c.m.p, (double *)c.s.p, (int64_t *)c.k.p,
                                  (double *)c.t.p, (double *)c.tp.p, (double *)c.fp.p);
  wcurve_back(env, metrics, wsums, nPoints, thr, tpw, fpw, &c, rc);
  return rc;
}
FN(evalSampledWeightedCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jlong rowBegin, jlong rowEnd, jlong key,
                             jlong posBegin, jlong posEnd, jlongArray metrics, jdoubleArray wsums, jlongArray nPoints,
                             jdoubleArray thr, jdoubleArray tpw, jdoubleArray fpw) {
  wcurve_bufs c = wcurve_in(env, w, metrics, wsums, nPoints, thr, tpw, fpw);
  int rc = DSGD_ERR_NOMEM;
  if (!wcurve_bad(&c) && (rc = wcurve_args(h, &c, posEnd - posBegin)) == DSGD_OK)
    rc = dsgd_eval_sampled_weighted_curve(CTX(h), c.w.p, rowBegin, rowEnd, (uint64_t)key, posBegin, posEnd, (int64_t *)c.m.p,
                                          (double *)c.s.p, (int64_t *)c.k.p, (double *)c.t.p, (double *)c.tp.p,
                                          (double *)c.fp.p);
  wcurve_back(env, metrics, wsums, nPoints, thr, tpw, fpw, &c, rc);
  return rc;
}
FN(evalSamplesWeightedCurve)(JNIEnv *env, jobject self, jlong h, jdoubleArray w, jintArray samples, jlongArray metrics,
                             jdoubleArray wsums, jlongArray nPoints, jdoubleArray thr, jdoubleArray tpw, jdoubleArray fpw) {
  buf_t bi = in_Int(env, samples);
  wcurve_bufs c = wcurve_in(env, w, metrics, wsums, nPoints, thr, tpw, fpw);
  int rc = DSGD_ERR_NOMEM;
  if (!(bi.bad | wcurve_bad(&c)) && (rc = wcurve_args(h, &c, bi.n)) == DSGD_OK)
    rc = dsgd_eval_samples_weighted_curve(CTX(h), c.w.p, bi.p, bi.n, (int64_t *)c.m.p, (double *)c.s.p, (int64_t *)c.k.p,
                                          (double *)c.t.p, (double *)c.tp.p, (double *)c.fp.p);
  wcurve_back(env, metrics, wsums, nPoints, thr, tpw, fpw, &c, rc);
  free(bi.p);
  return rc;
}

/* ---- async (Hogwild) mode ---- */
FN(asyncHostMaster)(JNIEnv *env, jobject self, jlong h, jdoubleArray w0) {
  buf_t b = in_Double(env, w0);
  int rc = b.bad ? DSGD_ERR_NOMEM : dsgd_async_host_master(CTX(h), b.p);   /* GradState of MasterAsync, core/MasterAsync.scala:66 */
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
  int rc = DSGD_ERR_NOMEM;
  if (!(bw.bad | ba.bad))
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
  int rc = b.bad ? DSGD_ERR_NOMEM : dsgd_async_master_weights(CTX(h), b.p);   /* gradState.single().grad, core/MasterAsync.scala:109 */
  back_Double(env, out, b, rc);
  return rc;
}
FN(asyncOutboxEnable)(JNIEnv *env, jobject self, jlong h) {
  (void)env; (void)self;
  return dsgd_async_outbox_enable(CTX(h));            /* deltas for colleagues reached over gRPC, core/Slave.scala:104-105 */
}
FN(asyncOutboxRead)(JNIEnv *env, jobject self, jlong h, jdoubleArray out) {
  buf_t b = out_Double(env, out);
  int rc = b.bad ? DSGD_ERR_NOMEM : (b.n < 1 ? DSGD_ERR_INVALID : dsgd_async_outbox_read(CTX(h), b.p));
  back_Double(env, out, b, rc);
  return rc;
}
#endif /* DSGD_HAVE_JNI */
