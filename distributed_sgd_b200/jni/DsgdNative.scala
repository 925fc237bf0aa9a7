// Scala facade over libdsgd_jni.so -> libdsgd.so (include/dsgd.h).  NOT compiled in this repository: the build
// image has no JVM toolchain (no javac / scalac / sbt / jni.h).  It is the binding a maintainer of
// zifeo/distributed-sgd would add under src/main/scala/epfl/distributed/nativ/.
package epfl.distributed.nativ

import epfl.distributed.math.Vec

object DsgdNative {
  System.loadLibrary("dsgd_jni") // links against libdsgd.so

  // every native returns the C ABI's status code; 0 = OK, negative = DSGD_ERR_*  (include/dsgd.h).  Arrays are copied in
  // before and out after the call (Get/Set<Type>ArrayRegion): nothing is pinned while a call blocks on the GPU.
  // flags: FlagAsync | one model flag (DSGD_FLAG_*); FlagLogistic, FlagSquaredHinge or FlagModifiedHuber selects
  // SparseLogistic, SparseSquaredHinge or SparseModifiedHuber instead of SparseSVM (sync mode only, at most one of them)
  final val FlagAsync = 1
  final val FlagLogistic = 2
  final val FlagSquaredHinge = 4
  final val FlagModifiedHuber = 8
  // FlagIntercept (with any one model flag, sync mode only): an unregularised intercept.  Every weight array in or out --
  // setWeights, getWeights, each request's w, gradient's grad (the intercept's gradient last), averageWeights -- is then
  // dim + 1 long, the intercept last; d stays dim long.  The shim checks every array against the length the library
  // reads or writes (a request's w: null or exactly that length), and returns DSGD_ERR_INVALID before the call otherwise.
  final val FlagIntercept = 16
  @native def create(device: Int, dim: Int, lambda: Double, rank: Int, world: Int, flags: Int): Long
  @native def destroy(ctx: Long): Int
  @native def lastError(ctx: Long): String
  // data / model
  @native def loadCsr(ctx: Long, rowPtr: Array[Long], col: Array[Int], value: Array[Float], label: Array[Byte]): Int
  @native def setDimSparsity(ctx: Long, d: Array[Double]): Int
  @native def computeDimSparsity(ctx: Long, nTrain: Long, out: Array[Double]): Int
  @native def setWeights(ctx: Long, w: Array[Double]): Int
  @native def getWeights(ctx: Long, w: Array[Double]): Int
  // SlaveImpl.forward / gradient, Master.localLoss / localAccuracy (w == null: the resident weights)
  @native def forward(ctx: Long, w: Array[Double], samples: Array[Int], preds: Array[Double]): Int
  @native def gradient(ctx: Long, w: Array[Double], samples: Array[Int], grad: Array[Double]): Int
  @native def eval(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, lossAcc: Array[Double]): Int
  @native def evalCounts(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, hingeCorrect: Array[Long],
                         normSquared: Array[Double]): Int
  // Master.localSampledLoss / localSampledAccuracy: positions [posBegin, posEnd) of a sample of rows [rowBegin, rowEnd)
  // drawn on the device with `key`, or a list of row ids the JVM drew itself (its own Random); same counters as evalCounts
  @native def evalSampledCounts(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                                posEnd: Long, hingeCorrect: Array[Long], normSquared: Array[Double]): Int
  @native def evalSamplesCounts(ctx: Long, w: Array[Double], samples: Array[Int], hingeCorrect: Array[Long],
                                normSquared: Array[Double]): Int
  // the same passes for every model (the *Counts forms refuse a ctx of any model but the SVM): lossSumNormSquared = {sum of the per-sample
  // losses, ||w||^2}, correct = {#correct}
  @native def evalSums(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, lossSumNormSquared: Array[Double],
                       correct: Array[Long]): Int
  @native def evalSampledSums(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                              posEnd: Long, lossSumNormSquared: Array[Double], correct: Array[Long]): Int
  @native def evalSamplesSums(ctx: Long, w: Array[Double], samples: Array[Int], lossSumNormSquared: Array[Double],
                              correct: Array[Long]): Int
  // scores (out.length >= samples.length): the margins x.w, or P(y = +1 | x) on a FlagLogistic or FlagModifiedHuber context; ranking metrics
  // (metrics.length >= MetricsWords): TP, FN, positives without a prediction, FP, TN, negatives without one, U2, NaN rows --
  // AUC = U2 / (2 P N)
  final val MetricsWords = 8
  @native def margins(ctx: Long, w: Array[Double], samples: Array[Int], out: Array[Double]): Int
  @native def probabilities(ctx: Long, w: Array[Double], samples: Array[Int], out: Array[Double]): Int
  @native def evalMetrics(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, metrics: Array[Long]): Int
  @native def evalSampledMetrics(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                                 posEnd: Long, metrics: Array[Long]): Int
  @native def evalSamplesMetrics(ctx: Long, w: Array[Double], samples: Array[Int], metrics: Array[Long]): Int
  // ROC / precision-recall curves: metrics as above, ap(0) = average precision, nPoints(0) = m, and thr / tp / fp(0 until m)
  // one point per distinct score, highest first.  thr, tp and fp are all null (average precision only) or each at least as
  // long as the request's rows.
  @native def evalCurve(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, metrics: Array[Long], ap: Array[Double],
                        nPoints: Array[Long], thr: Array[Double], tp: Array[Long], fp: Array[Long]): Int
  @native def evalSampledCurve(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                               posEnd: Long, metrics: Array[Long], ap: Array[Double], nPoints: Array[Long],
                               thr: Array[Double], tp: Array[Long], fp: Array[Long]): Int
  @native def evalSamplesCurve(ctx: Long, w: Array[Double], samples: Array[Int], metrics: Array[Long], ap: Array[Double],
                               nPoints: Array[Long], thr: Array[Double], tp: Array[Long], fp: Array[Long]): Int
  // Poisson bootstrap, either model: replicates [bBegin, bEnd) with key bKey; words(9 j until 9 j + 9) = the metrics words and
  // the size of replicate bBegin + j, ap(j) its average precision, loss(j) its loss sum.  Each array holds at least the
  // replicates' entries.
  @native def evalBootstrap(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, bKey: Long, bBegin: Long, bEnd: Long,
                            words: Array[Long], ap: Array[Double], loss: Array[Double]): Int
  @native def evalSampledBootstrap(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                                   posEnd: Long, bKey: Long, bBegin: Long, bEnd: Long, words: Array[Long],
                                   ap: Array[Double], loss: Array[Double]): Int
  @native def evalSamplesBootstrap(ctx: Long, w: Array[Double], samples: Array[Int], bKey: Long, bBegin: Long, bEnd: Long,
                                   words: Array[Long], ap: Array[Double], loss: Array[Double]): Int
  // weighted Poisson bootstrap, every row counted by c_i = class weight x sample weight: words(2 j) and words(2 j + 1) = the
  // size and the NaN-score rows of replicate bBegin + j, wsums(13 j until 13 j + 13) its weighted curve words, loss(j) its
  // weighted loss sum.  Each array holds at least the replicates' entries.
  @native def evalWeightedBootstrap(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, bKey: Long, bBegin: Long,
                                    bEnd: Long, words: Array[Long], wsums: Array[Double], loss: Array[Double]): Int
  @native def evalSampledWeightedBootstrap(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long,
                                           posBegin: Long, posEnd: Long, bKey: Long, bBegin: Long, bEnd: Long,
                                           words: Array[Long], wsums: Array[Double], loss: Array[Double]): Int
  @native def evalSamplesWeightedBootstrap(ctx: Long, w: Array[Double], samples: Array[Int], bKey: Long, bBegin: Long,
                                           bEnd: Long, words: Array[Long], wsums: Array[Double], loss: Array[Double]): Int
  // calibration (Platt scaling): ab(0..1) = (A, B) of P(y = +1 | x) = 1 / (1 + exp(A x.w + B)), objective(0) = F(A, B),
  // info(0..4) = iterations, status (0 converged, 1 iteration limit, 2 line search failed, 3 non-finite sum), rows used, NaN
  // rows, points evaluated.  Quality at (a, b): sums(0..1) = Brier and log-loss sums, binRows / binPos / binPsum(0 until
  // nBins), words(0..1) = rows used and left out.
  @native def calibrate(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, ab: Array[Double], objective: Array[Double],
                        info: Array[Long]): Int
  @native def calibrateSampled(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                               posEnd: Long, ab: Array[Double], objective: Array[Double], info: Array[Long]): Int
  @native def calibrateSamples(ctx: Long, w: Array[Double], samples: Array[Int], ab: Array[Double], objective: Array[Double],
                               info: Array[Long]): Int
  @native def calibratedProbabilities(ctx: Long, w: Array[Double], samples: Array[Int], a: Double, b: Double,
                                      out: Array[Double]): Int
  @native def evalCalibration(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, a: Double, b: Double, nBins: Int,
                              sums: Array[Double], binRows: Array[Long], binPos: Array[Long], binPsum: Array[Double],
                              words: Array[Long]): Int
  @native def evalSampledCalibration(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                                     posEnd: Long, a: Double, b: Double, nBins: Int, sums: Array[Double],
                                     binRows: Array[Long], binPos: Array[Long], binPsum: Array[Double],
                                     words: Array[Long]): Int
  @native def evalSamplesCalibration(ctx: Long, w: Array[Double], samples: Array[Int], a: Double, b: Double, nBins: Int,
                                     sums: Array[Double], binRows: Array[Long], binPos: Array[Long], binPsum: Array[Double],
                                     words: Array[Long]): Int
  // weighted calibration (every row counted by its weight c_i): the calls above with wsums(0..2) = W+, W- and the NaN rows'
  // weight added to a fit; weighted quality: sums(0..3) = Brier and log-loss sums, weight used, infinite-term weight (0),
  // binWeight / binPosWeight / binPsum(0 until nBins), words(0..1) = rows used and left out.
  @native def calibrateWeighted(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, ab: Array[Double],
                                objective: Array[Double], info: Array[Long], wsums: Array[Double]): Int
  @native def calibrateWeightedSampled(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                                       posEnd: Long, ab: Array[Double], objective: Array[Double], info: Array[Long],
                                       wsums: Array[Double]): Int
  @native def calibrateWeightedSamples(ctx: Long, w: Array[Double], samples: Array[Int], ab: Array[Double],
                                       objective: Array[Double], info: Array[Long], wsums: Array[Double]): Int
  @native def evalWeightedCalibration(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, a: Double, b: Double,
                                      nBins: Int, sums: Array[Double], binWeight: Array[Double],
                                      binPosWeight: Array[Double], binPsum: Array[Double], words: Array[Long]): Int
  @native def evalSampledWeightedCalibration(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long,
                                             posBegin: Long, posEnd: Long, a: Double, b: Double, nBins: Int,
                                             sums: Array[Double], binWeight: Array[Double], binPosWeight: Array[Double],
                                             binPsum: Array[Double], words: Array[Long]): Int
  @native def evalSamplesWeightedCalibration(ctx: Long, w: Array[Double], samples: Array[Int], a: Double, b: Double,
                                             nBins: Int, sums: Array[Double], binWeight: Array[Double],
                                             binPosWeight: Array[Double], binPsum: Array[Double], words: Array[Long]): Int
  // isotonic calibration: nPoints(0) = k, x / y(0 until k) the thresholds ascending in s = -x.w and their probabilities,
  // blockRows / blockPos(0 until blocks), info(0..4) = blocks, points, rows used, NaN rows, distinct scores; x, y, blockRows
  // and blockPos at least as long as the request's rows.  P(y = +1 | x) = numpy.interp(s, x, y).  Quality at the map (x, y):
  // as evalCalibration, words(0..2) = rows used, rows left out, rows with an infinite log-loss term.
  @native def calibrateIsotonic(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, nPoints: Array[Long],
                                x: Array[Double], y: Array[Double], blockRows: Array[Long], blockPos: Array[Long],
                                info: Array[Long]): Int
  @native def calibrateIsotonicSampled(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                                       posEnd: Long, nPoints: Array[Long], x: Array[Double], y: Array[Double],
                                       blockRows: Array[Long], blockPos: Array[Long], info: Array[Long]): Int
  @native def calibrateIsotonicSamples(ctx: Long, w: Array[Double], samples: Array[Int], nPoints: Array[Long],
                                       x: Array[Double], y: Array[Double], blockRows: Array[Long], blockPos: Array[Long],
                                       info: Array[Long]): Int
  @native def isotonicProbabilities(ctx: Long, w: Array[Double], samples: Array[Int], x: Array[Double], y: Array[Double],
                                    out: Array[Double]): Int
  @native def evalIsotonicCalibration(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, x: Array[Double],
                                      y: Array[Double], nBins: Int, sums: Array[Double], binRows: Array[Long],
                                      binPos: Array[Long], binPsum: Array[Double], words: Array[Long]): Int
  @native def evalSampledIsotonicCalibration(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long,
                                             posBegin: Long, posEnd: Long, x: Array[Double], y: Array[Double], nBins: Int,
                                             sums: Array[Double], binRows: Array[Long], binPos: Array[Long],
                                             binPsum: Array[Double], words: Array[Long]): Int
  @native def evalSamplesIsotonicCalibration(ctx: Long, w: Array[Double], samples: Array[Int], x: Array[Double],
                                             y: Array[Double], nBins: Int, sums: Array[Double], binRows: Array[Long],
                                             binPos: Array[Long], binPsum: Array[Double], words: Array[Long]): Int
  // weighted isotonic calibration: blockWeight / blockPosWeight in place of the block counts, wsums(0..1) = W+, W-; weighted
  // quality at (x, y): sums(0..3), binWeight / binPosWeight / binPsum, words(0..2) as for evalIsotonicCalibration.
  @native def calibrateIsotonicWeighted(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, nPoints: Array[Long],
                                        x: Array[Double], y: Array[Double], blockWeight: Array[Double],
                                        blockPosWeight: Array[Double], info: Array[Long], wsums: Array[Double]): Int
  @native def calibrateIsotonicWeightedSampled(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long,
                                               posBegin: Long, posEnd: Long, nPoints: Array[Long], x: Array[Double],
                                               y: Array[Double], blockWeight: Array[Double], blockPosWeight: Array[Double],
                                               info: Array[Long], wsums: Array[Double]): Int
  @native def calibrateIsotonicWeightedSamples(ctx: Long, w: Array[Double], samples: Array[Int], nPoints: Array[Long],
                                               x: Array[Double], y: Array[Double], blockWeight: Array[Double],
                                               blockPosWeight: Array[Double], info: Array[Long], wsums: Array[Double]): Int
  @native def evalWeightedIsotonicCalibration(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, x: Array[Double],
                                              y: Array[Double], nBins: Int, sums: Array[Double], binWeight: Array[Double],
                                              binPosWeight: Array[Double], binPsum: Array[Double], words: Array[Long]): Int
  @native def evalSampledWeightedIsotonicCalibration(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long,
                                                     posBegin: Long, posEnd: Long, x: Array[Double], y: Array[Double],
                                                     nBins: Int, sums: Array[Double], binWeight: Array[Double],
                                                     binPosWeight: Array[Double], binPsum: Array[Double],
                                                     words: Array[Long]): Int
  @native def evalSamplesWeightedIsotonicCalibration(ctx: Long, w: Array[Double], samples: Array[Int], x: Array[Double],
                                                     y: Array[Double], nBins: Int, sums: Array[Double],
                                                     binWeight: Array[Double], binPosWeight: Array[Double],
                                                     binPsum: Array[Double], words: Array[Long]): Int
  // sync mode: cluster membership (core/Master.scala:222-243) becomes attach / import calls; the step loop one call
  @native def commUniqueId(id: Array[Byte]): Int                       // 128 bytes; rank 0 makes it, every rank commInit()s it
  @native def commInit(ctx: Long, id: Array[Byte]): Int
  @native def xchgExport(ctx: Long, handle: Array[Byte]): Int          // 64 bytes; one JVM per GPU: ship it over the node's gRPC
  @native def xchgImport(ctx: Long, peerRank: Int, handle: Array[Byte]): Int
  @native def xchgAttach(ctx: Long, peerRank: Int, peerCtx: Long): Int // one JVM driving all GPUs of the box
  @native def xchgStats(ctx: Long, out: Array[Long]): Int
  @native def streamExactRows(ctx: Long, out: Array[Long]): Int // diagnostic: rows of streaming passes recomputed in fp64
  @native def setWorkers(ctx: Long, counts: Array[Int], kTotal: Int): Int
  @native def syncSteps(ctx: Long, samples: Array[Int], nPerStep: Long, nSteps: Long, lr: Double, losses: Array[Double]): Int
  // the same with one learning rate per step: step s uses lrs(s) (every rank passes the same table)
  @native def syncStepsLr(ctx: Long, samples: Array[Int], nPerStep: Long, nSteps: Long, lrs: Array[Double],
                          losses: Array[Double]): Int
  // averaged SGD (sync mode): every sync step after averageBegin adds its new weights to a device-side sum until averageEnd;
  // averageWeights: avg = the mean of those weights, nSteps(0) = how many (either may be null)
  @native def averageBegin(ctx: Long): Int
  @native def averageEnd(ctx: Long): Int
  @native def averageWeights(ctx: Long, avg: Array[Double], nSteps: Array[Long]): Int
  // L1 penalty of the sync steps (elastic net with lambda): every step soft-thresholds every weight at lr * lambda1;
  // weightsL1: l1(0) = ||w||_1, nnz(0) = the non-zero weights, of w or (w null) of the resident weights
  @native def setL1(ctx: Long, lambda1: Double): Int
  @native def weightsL1(ctx: Long, w: Array[Double], l1: Array[Double], nnz: Array[Long]): Int
  // class weights of the sync steps and of gradient (both finite and >= 0; (1, 1) by default); out = {wPos, wNeg}.  The
  // per-class evaluations, either model: sums = {||w||^2, loss sum of the y = +1 rows, of the y = -1 rows} (unweighted),
  // counts = {correct+, correct-, n+, n-}
  @native def setClassWeights(ctx: Long, wPos: Double, wNeg: Double): Int
  @native def getClassWeights(ctx: Long, out: Array[Double]): Int
  @native def evalClass(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, sums: Array[Double],
                        counts: Array[Long]): Int
  @native def evalSampledClass(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                               posEnd: Long, sums: Array[Double], counts: Array[Long]): Int
  @native def evalSamplesClass(ctx: Long, w: Array[Double], samples: Array[Int], sums: Array[Double],
                               counts: Array[Long]): Int
  // sample weights of the sync steps, of gradient and of the weighted evaluations: one per loaded row (finite and >= 0), null
  // clears them.  The weighted evaluations, either model: sums = {||w||^2, S = sum c_i L_i, sum c_i [correct], sum c_i},
  // counts = {rows, correct}
  @native def setSampleWeights(ctx: Long, sw: Array[Double]): Int
  @native def evalWeighted(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, sums: Array[Double],
                           counts: Array[Long]): Int
  @native def evalSampledWeighted(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                                  posEnd: Long, sums: Array[Double], counts: Array[Long]): Int
  @native def evalSamplesWeighted(ctx: Long, w: Array[Double], samples: Array[Int], sums: Array[Double],
                                  counts: Array[Long]): Int
  // weighted curves, either model: metrics as evalCurve's, wsums(0 until 13) the DSGD_WCURVE_WORDS weighted words, nPoints(0)
  // = m, thr / tpw / fpw(0 until m) the points (W+ and W- at or above each score); all three null for the words alone, else
  // each at least as long as the request's rows.  An async ctx is refused.
  @native def evalWeightedCurve(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, metrics: Array[Long],
                                wsums: Array[Double], nPoints: Array[Long], thr: Array[Double], tpw: Array[Double],
                                fpw: Array[Double]): Int
  @native def evalSampledWeightedCurve(ctx: Long, w: Array[Double], rowBegin: Long, rowEnd: Long, key: Long, posBegin: Long,
                                       posEnd: Long, metrics: Array[Long], wsums: Array[Double], nPoints: Array[Long],
                                       thr: Array[Double], tpw: Array[Double], fpw: Array[Double]): Int
  @native def evalSamplesWeightedCurve(ctx: Long, w: Array[Double], samples: Array[Int], metrics: Array[Long],
                                       wsums: Array[Double], nPoints: Array[Long], thr: Array[Double], tpw: Array[Double],
                                       fpw: Array[Double]): Int
  // async (Hogwild) mode
  @native def asyncHostMaster(ctx: Long, w0: Array[Double]): Int
  @native def ipcExport(ctx: Long, which: Int, handle: Array[Byte]): Int
  @native def ipcImport(ctx: Long, peerRank: Int, handle: Array[Byte]): Int
  @native def peerAttach(ctx: Long, peerRank: Int, peerCtx: Long, which: Int): Int
  @native def startAsync(ctx: Long, w0: Array[Double], assigned: Array[Int], batch: Int, lr: Double,
                         concurrency: Int, maxUpdates: Long, seed: Long): Int
  @native def stopAsync(ctx: Long): Int
  @native def asyncRunning(ctx: Long, out: Array[Int]): Int
  @native def updateGrad(ctx: Long, idx: Array[Int], value: Array[Double]): Int
  @native def asyncUpdates(ctx: Long, out: Array[Long]): Int
  @native def asyncMasterWeights(ctx: Long, out: Array[Double]): Int
  @native def asyncOutboxEnable(ctx: Long): Int
  @native def asyncOutboxRead(ctx: Long, out: Array[Double]): Int

  /** Vec (keys are the reference's 1-based feature ids) -> dense array in the ABI's 0-based column space. */
  def densify(v: Vec, dim: Int): Array[Double] = {
    val a = new Array[Double](dim)
    v.map.foreach { case (k, x) => a(k - 1) = x.toDouble }
    a
  }

  def sparsify(a: Array[Double], dim: Int): Vec =
    Vec(a.iterator.zipWithIndex.collect { case (x, i) if x != 0.0 => (i + 1) -> spire.math.Number(x) }.toMap, dim)

  def check(ctx: Long, rc: Int): Unit = rc match {
    case 0            => ()
    case -1 | -3      => throw new IllegalArgumentException(lastError(ctx)) // require(...) / Vec.sum(empty)
    case -4           => throw new IndexOutOfBoundsException(lastError(ctx))
    case _            => throw new IllegalStateException(lastError(ctx))
  }
}
