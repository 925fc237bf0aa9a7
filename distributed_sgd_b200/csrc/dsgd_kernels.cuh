// dsgd_kernels.cuh -- sm_90a kernels of the SGD hot path (see DESIGN.md for the layout and rooflines).
//
// Device layout of the rows ("row windows"): one array of 8-byte (col:int32, val:fp32) pairs, each row
// padded with (col = last col, val = 0) pairs to a multiple of 2 pairs so that every row window starts on
// a 16-byte boundary and is a multiple of 16 bytes long (what cp.async.bulk / 128-bit loads need).
// rp16[r] is the window start in 16-byte units.  A val == 0 pair is arithmetically inert everywhere:
// it adds 0 to the dot product and is skipped by the scatter.
//
// State vectors (w, g, d) are fp64 and live in L2 (3 x 378 KB on a 50 MB L2); the HBM stream is the
// row windows only.  All reference arithmetic cited as path:line under
// src/main/scala/epfl/distributed/ of the reference repository.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dsgd_feistel.h"
#include "dsgd_fixed.cuh"

namespace dsgd {

constexpr double kEps = 1e-20;  // math/Sparse.scala:104

// Slots of the per-ctx scalar block (double[kNumScal]) kept on the device.
enum Scal : int {
  kScalC = 0,      // c = 2*lambda*(w . d) of the CURRENT resident weights (SparseSVM.scala:31)
  kScalNrm2 = 1,   // ||w||^2 of the current resident weights (SparseSVM.scala:21)
  kScalReqC = 2,   // same two for a request-supplied weight vector (GradientRequest.weights)
  kScalReqNrm2 = 3,
  kScalL1 = 4,     // ||w||_1 of the current resident weights: refreshed by every sync call of an L1 ctx (k_l1_norm), then
                   // kept by its update kernels (k_update<..., kL1>)
  kNumScal = 8
};
// Slots of the per-ctx counter block (unsigned long long[kNumCnt]).
enum Cnt : int {
  kCntHinge = 0,    // sum of per-sample hinge losses of the running batch (integers: 0, 1 or 2 each)
  kCntCorrect = 1,  // #{pred == y}
  kCntTicket = 2,   // last-block ticket of k_update
  kCntWLoss = 3,    // class-weighted batch: the bits of the double w_pos * L_pos + w_neg * L_neg (k_class_fold), which the
                    // weighted tails (kCw) read instead of kCntHinge / kCntLoss
  kCntLoss = 8,     // every model but the SVM: fixed-point sum of the batch's per-sample losses (kLossAccWords words, dsgd_fixed.cuh)
  kCntL1 = 16,      // fixed-point sum of |w_j| (kLossAccWords words): k_update<..., kL1>, k_l1_norm; zero between launches
  kCntNnz = 23,     // #{w_j != 0} of k_l1_norm; zero between launches
  // per-class counters of k_rows<..., kClassWeighted, ...>, cleared by k_class_fold: index 0 is the class y = +1, index 1 the
  // class y = -1
  kCntClassN = 24,        // rows
  kCntClassCorrect = 26,  // #{pred == y}
  kCntClassHinge = 28,    // SVM: hinge sums (integers)
  kCntClassLoss = 32,     // not the SVM: two fixed-point sums of the unweighted losses, kLossAccWords words each
  // fixed-point sums of k_rows<..., kSampleWeighted, ...> (kLossAccWords words each), taken by k_sw_fold: S = sum R(c_i L_i),
  // and for an evaluation sum R(c_i [pred_i == y_i]) and sum R(c_i)
  kCntSwLoss = 48,
  kCntSwCorrect = 56,
  kCntSwWeight = 64,
  // an intercept ctx (kIcpt): the intercept's gradient of the running pass, its positive and its negative parts as two
  // fixed-point sums (kLossAccWords words each) of k_rows<..., kIcpt>, taken by k_finish, k_finish_acc or k_update
  kCntIcpt = 72,
  kNumCnt = 88
};
static_assert(kCntLoss + kLossAccWords <= kCntL1 && kCntL1 + kLossAccWords <= kCntNnz && kCntNnz < kCntClassN &&
                  kCntClassLoss + 2 * kLossAccWords <= kCntSwLoss && kCntSwLoss + kLossAccWords <= kCntSwCorrect &&
                  kCntSwCorrect + kLossAccWords <= kCntSwWeight && kCntSwWeight + kLossAccWords <= kCntIcpt &&
                  kCntIcpt + 2 * kLossAccWords <= kNumCnt,
              "counter block");
// Slot of the intercept's gradient in the gradient buffer g and the workers' sum gsum of an intercept ctx: after the loss sum
// ([dim]) and the batch size ([dim + 1]), which keep their places, so that a plain ctx's buffers do not change.
constexpr int kIcptSlot = 2;

// Model of a ctx, a compile-time parameter of the kernels whose arithmetic depends on it.
constexpr int kSvm = 0;        // SparseSVM: hinge loss, integer per-sample losses (SparseSVM.scala:11-33)
constexpr int kLogistic = 1;   // SparseLogistic: softplus loss, gradient x * (y * sigmoid(y * x.w))
constexpr int kSquaredHinge = 2;    // SparseSquaredHinge: the L2-loss SVM, loss (1 + z)^2 above z = -1
constexpr int kModifiedHuber = 3;   // SparseModifiedHuber: (1 + z)^2 on (-1, 1], 4 z above
// Every model but the SVM has non-integer per-sample losses: they are added in the fixed-point limbs of dsgd_fixed.cuh
// Weighting of a sync pass, a compile-time parameter of the row pass and of the persistent kernel.
constexpr int kUnweighted = 0;
constexpr int kClassWeighted = 1;    // dsgd_set_class_weights: row i counts w_y (w_pos or w_neg by its label)
constexpr int kSampleWeighted = 2;   // dsgd_set_sample_weights: row i counts c_i = fl(w_y * s_i), the class weights included

// Sum of the per-sample losses of the running batch or pass, and its reset.  kCw: the class-weighted sum of k_class_fold.
template <int kModel, bool kCw = false>
__device__ __forceinline__ double batch_loss_sum(const unsigned long long *cnt) {
  if (kCw) return __longlong_as_double((long long)cnt[kCntWLoss]);
  return kModel != kSvm ? acc_value(cnt + kCntLoss) : (double)cnt[kCntHinge];
}
template <int kModel, bool kCw = false>
__device__ __forceinline__ void clear_batch_loss(unsigned long long *cnt) {
  if (kCw) {
    cnt[kCntWLoss] = 0ull;
    return;
  }
  cnt[kCntHinge] = 0ull;
  if (kModel != kSvm)
#pragma unroll
    for (int i = 0; i < kLossAccWords; ++i) cnt[kCntLoss + i] = 0ull;
}

__device__ __forceinline__ double filt(double v) { return fabs(v) > kEps ? v : 0.0; }  // Sparse.scala:108-118

// The proximal step of the L1 penalty at threshold tau = lr * lambda1: u shrunk towards 0 by tau, 0 where |u| <= tau, with the
// 1e-20 filter of a new Sparse.  tau == 0 (lambda1 == 0, or a zero rate) returns u itself: the step without the penalty.
__device__ __forceinline__ double soft_threshold(double u, double tau) {
  if (!(tau > 0.0)) return u;
  return u > tau ? filt(u - tau) : (u < -tau ? filt(u + tau) : 0.0);
}

// Adds R(a) of every thread of the block (a in [0, 2^52), dsgd_fixed.cuh) to the kLossAccWords accumulator acc: the limbs are
// summed in registers, over the warp and over the block, carried once and pushed by thread 0 with one RED per non-zero word,
// then fenced, so that a ticket thread 0 takes afterwards orders them.  Called by all kThreads threads.
template <int kThreads>
__device__ __forceinline__ void acc_push_block(double a, unsigned long long *__restrict__ acc) {
  __shared__ unsigned long long sh[kThreads / 32][kLossAccWords];
  unsigned long long lim[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf = 0;
  acc_add_local(lim, ovf, a);   // limbs 0..4 below 2^40, limb 5 below 2^13: a block's sums stay below 2^48
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int i = 0; i < kLossLimbs; ++i) lim[i] += __shfl_xor_sync(0xffffffffu, lim[i], o);
    ovf += __shfl_xor_sync(0xffffffffu, ovf, o);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kLossLimbs; ++i) sh[wid][i] = lim[i];
    sh[wid][kLossLimbs] = ovf;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < kLossLimbs; ++i) lim[i] = 0;
    ovf = 0;
    for (int w = 0; w < kThreads / 32; ++w) {
#pragma unroll
      for (int i = 0; i < kLossLimbs; ++i) lim[i] += sh[w][i];
      ovf += sh[w][kLossLimbs];
    }
    acc_carry(lim);   // limbs 0..4 below 2^40 again: the words of 2^24 blocks cannot wrap
    acc_flush_local(acc, lim, ovf);
    __threadfence();
  }
}
// One thread, after every push has landed: the value of the accumulator, which is left zeroed
__device__ __forceinline__ double acc_take(unsigned long long *acc) {
  unsigned long long q[kLossAccWords];
#pragma unroll
  for (int i = 0; i < kLossAccWords; ++i) {
    q[i] = __ldcg(acc + i);
    acc[i] = 0ull;
  }
  return acc_value(q);
}
// One thread, after a scattering pass of an intercept ctx: the intercept's gradient g_b = filt(P - N) from the two sums of
// kCntIcpt (both left zeroed), as regularize() leaves an entry that c is never added to
__device__ __forceinline__ double icpt_take(unsigned long long *cnt) {
  const double p = acc_take(cnt + kCntIcpt);
  const double n = acc_take(cnt + kCntIcpt + kLossAccWords);
  return filt(p - n);
}

// Gradient scatter: a reduction WITHOUT a return value.  Written as PTX `red` because nvcc 12.9 compiles atomicAdd(double *)
// with an unused result to ATOMG (result discarded, but the response still travels back: ncu counted 1.9 M returned sectors
// per 300 steps) inside the large persistent kernels, and to REDG only in small ones.
__device__ __forceinline__ void red_add_f64(double *p, double v) {
  asm volatile("red.relaxed.gpu.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ void red_add_f64_sys(double *p, double v) {   // peer replicas over NVLink
  asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ void red_add_u64_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// prediction = -signum(x . w)  (core/ml/SparseSVM.scala:14)
__device__ __forceinline__ int pred_of(double dot) { return (dot > 0.0) ? -1 : ((dot < 0.0) ? 1 : 0); }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------------
// The row fold: the one fp64 summation order of x . w for a row window on the device, so that a row's margin, prediction
// and gate are a function of the row and w alone, whichever kernel takes the row and whatever else is in the request.
//   * The window of L pairs (padding included) is cut into kFoldPairs-pair chunks from its start.
//   * In chunk c, lane l sums filt(filt(x) * w) over the pairs 128 c + l + 32 u, u = 0 .. 3 in order, from +0.0.
//   * The xor butterfly 16, 8, 4, 2, 1 reduces the lanes to the chunk partial.
//   * The dot is 0.0 + part_0 + part_1 + ..., in chunk order.  No partial is -0 (every lane sum starts at +0.0 and filt
//     never returns -0), so a one-chunk window's dot is its partial.
// The listed chunks of the persistent sync step (consume_stage, dsgd_persistent.cuh) are this fold with the chunks spread
// over warps.  row_fold_from continues a fold whose chunks before pair c have been added to dot already (the async workers
// hold chunk 0 in registers); wt(col) is the weight of column col.  Called by the whole warp; every lane gets the dot.
// ---------------------------------------------------------------------------------------------------
constexpr int kFoldPairs = 128;
template <class Wt>
__device__ __forceinline__ double row_fold_from(const uint2 *__restrict__ pairs, int64_t c, int64_t e, int lane, double dot,
                                                Wt &&wt) {
  const uint2 *__restrict__ src = pairs + c;
  const int len = (int)(e - c);   // a row window is far below 2^31 pairs
  for (int c0 = 0; c0 < len; c0 += kFoldPairs) {
    const int ce = min(c0 + kFoldPairs, len);
    double acc = 0.0;
    for (int k = c0 + lane; k < ce; k += 32) {
      const uint2 pr = __ldg(&src[k]);
      acc += filt(filt((double)__uint_as_float(pr.y)) * wt(pr.x));  // (x * w).sum  (math/Vec.scala:58; math/Sparse.scala:46)
    }
    dot += warp_sum(acc);
  }
  return dot;
}
template <class Wt>
__device__ __forceinline__ double row_fold(const uint2 *__restrict__ pairs, int64_t b, int64_t e, int lane, Wt &&wt) {
  return row_fold_from(pairs, b, e, lane, 0.0, wt);
}

// Block-wide sum in a fixed order (deterministic run to run). Result valid in thread 0.
template <int kThreads>
__device__ __forceinline__ double block_sum(double v, double *smem /* kThreads/32 */) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < kThreads / 32; ++i) s += smem[i];
  }
  __syncthreads();
  return s;
}

// ---------------------------------------------------------------------------------------------------
// k_prepare: c = lambda*2*(w . d) and ||w||^2 for a weight vector (SparseSVM.scala:31,21).  One block,
// fixed-order reduction.  47 236 elements: ~2 us; only used when the host installs weights -- in the
// step loop k_update produces both numbers for the next step.
// ---------------------------------------------------------------------------------------------------
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_prepare(const double *__restrict__ w, const double *__restrict__ d,
                                                      int dim, double lambda, double *__restrict__ scal_c,
                                                      double *__restrict__ scal_nrm2) {
  __shared__ double red[kThreads / 32];
  double sd = 0.0, sn = 0.0;
  for (int j = threadIdx.x; j < dim; j += kThreads) {
    const double wj = w[j];
    sd += filt(wj * d[j]);  // (w * d).sum: products below 1e-20 are dropped by the Sparse constructor
    sn += wj * wj;
  }
  sd = block_sum<kThreads>(sd, red);
  sn = block_sum<kThreads>(sn, red);
  if (threadIdx.x == 0) {
    *scal_c = lambda * 2.0 * sd;
    *scal_nrm2 = sn;
  }
}

// ---------------------------------------------------------------------------------------------------
// SparseLogistic, one sample with z = y * (x . w):  loss softplus(z) = max(z, 0) + log1p(exp(-|z|)),
// backward x * (y * sigmoid(z)).  Both stable for any z; fp64 exp / log1p (no fast-math intrinsics), the formulas of the
// oracle.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ double softplus(double z) { return (z > 0.0 ? z : 0.0) + log1p(exp(-fabs(z))); }
__device__ __forceinline__ double sigmoid(double t) {
  if (t >= 0.0) return 1.0 / (1.0 + exp(-t));
  const double e = exp(t);
  return e / (1.0 + e);
}

// ---------------------------------------------------------------------------------------------------
// SparseSquaredHinge and SparseModifiedHuber, one sample with z = y * (x . w) and t = fl(1 + z).  The classifier's margin
// is -z (the prediction is -signum(x . w)), so both losses vanish for z <= -1.  Per-sample loss L and backward scale s
// (backward x * (y * s), weighted (y * s) * c), each a short chain of correctly rounded fp64 operations in this order:
//   squared hinge    z <= -1: L = 0, s = 0;   else L = t * t, s = 2 * t
//   modified Huber   z <= -1: L = 0, s = 0;   -1 < z <= 1: L = t * t, s = 2 * t;   z > 1: L = 4 * z, s = 4
// The modified Huber loss is continuous at z = 1 (t * t = 4 = 4 * z, 2 * t = 4).  With --fmad=false nothing is contracted,
// so the C oracle (oracle/dsgd_oracle_margin.c) gives the same bits.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ double sq_hinge_loss(double z) {
  const double t = 1.0 + z;
  return z <= -1.0 ? 0.0 : t * t;
}
__device__ __forceinline__ double sq_hinge_scale(double z) { return z <= -1.0 ? 0.0 : 2.0 * (1.0 + z); }
__device__ __forceinline__ double mod_huber_loss(double z) {
  const double t = 1.0 + z;
  return z <= -1.0 ? 0.0 : (z <= 1.0 ? t * t : 4.0 * z);
}
__device__ __forceinline__ double mod_huber_scale(double z) { return z <= -1.0 ? 0.0 : (z <= 1.0 ? 2.0 * (1.0 + z) : 4.0); }

// The per-sample loss L(z) and backward scale s(z) of a model other than the SVM (whose loss is an integer of the
// prediction and whose gate is a branch of k_rows)
template <int kModel>
__device__ __forceinline__ double row_loss(double z) {
  static_assert(kModel != kSvm, "the SVM's loss is the integer hinge of its prediction");
  if constexpr (kModel == kLogistic) return softplus(z);
  else if constexpr (kModel == kSquaredHinge) return sq_hinge_loss(z);
  else return mod_huber_loss(z);
}
template <int kModel>
__device__ __forceinline__ double row_scale(double z) {
  static_assert(kModel != kSvm, "the SVM's scale is its label");
  if constexpr (kModel == kLogistic) return sigmoid(z);
  else if constexpr (kModel == kSquaredHinge) return sq_hinge_scale(z);
  else return mod_huber_scale(z);
}

// ---------------------------------------------------------------------------------------------------
// k_rows: the per-sample body of SlaveImpl.gradient / SlaveImpl.forward (core/Slave.scala:129-157) for every model and
// weighting: one warp per row window; fp64 dot with the L2-resident weights (every loss but the SVM's needs the dot's
// value, not only its sign: the fp32 streaming pass of dsgd_stream.cuh is SVM-only); prediction, per-sample loss and gate;
// scatter into the dense gradient with fp64 reductions at L2 (no return value -> RED, not ATOM).
//   kScatter: accumulate backward() into g            (SparseSVM.scala:26-29)
//   kPreds:   write p = -signum(x.w) per sample       (SparseSVM.scala:14); the unweighted SVM pass only
// samples == nullptr walks rows [row_begin, row_begin + n).
// The scatter value s of a row, then filt(filt(x_j) * s) per entry, so a zero weight adds nothing:
//   SVM       s = y, weighted y * c  (an exact sign flip of c),  added where !(y * dot < 0)
//   logistic  s = y * sigmoid(z), weighted (y * sigmoid(z)) * c,  added for every row
//   squared hinge, modified Huber  s = y * s(z), weighted (y * s(z)) * c (row_scale),  added where z > -1 (s(z) = 0 below)
// where c is the row's weight: w_y with class weights, c_i = fl(w_y * s_i) with sample weights (sw == nullptr, an
// evaluation of a ctx without sample weights: every s_i is 1).  The unweighted passes do not read w_pos, w_neg or sw, and
// kScatter = false with class weights is the pass of dsgd_eval*_class, which does not read the weights.
// Lane 0's tally, the same in any row order or grid (integer counters, or R(.) added to fixed-point limbs in registers
// and pushed once per warp, dsgd_fixed.cuh):
//   unweighted      SVM: the hinge sum and the correct count (hinge losses are integers: y, p in {-1,0,1});
//                   other models: the correct count and the limbs of L(z) (row_loss)
//   class weights   rows, correct predictions and the unweighted loss per class (SVM: integer hinge sums; others: two
//                   limb blocks, a row adds its loss to its class's block and an exact 0 to the other); k_class_fold
//                   applies the weights
//   sample weights  R(fl(c_i * L_i)) into one limb block (S, kCntSwLoss) and the correct count; an evaluation (kScatter =
//                   false) also R(c_i) of the correct rows (kCntSwCorrect) and of every row (kCntSwWeight).  With s = 1
//                   and w = (1, 1) the SVM's S is the integer hinge sum and any other model's S the unweighted limb sum.
// The counters are plain locals of every form, each form using its own: held in a struct, nvcc orders the loop's
// registers differently, and the forms would no longer compile to the instructions of the separate kernels they replaced.
// kIcpt (an intercept ctx, DESIGN.md 4.18): beta = *icpt is the weight of a virtual column of value 1 in every row.  The
// score is fl(fold + filt(beta)) (the fold's dot, then beta once), and a scattering pass adds each row's filt(s), the value
// it scatters onto a column with x = 1, to beta's gradient: lane 0 keeps the positive and the negative values in two limb
// blocks and pushes them once per warp to kCntIcpt (the same bits in any row order or grid).  Otherwise icpt is not read.
// ---------------------------------------------------------------------------------------------------
template <int kModel, int kWeight, bool kScatter, bool kPreds = false, bool kIcpt = false>
__global__ void __launch_bounds__(256) k_rows(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                              const int8_t *__restrict__ label, const int32_t *__restrict__ samples,
                                              int64_t row_begin, int64_t n, const double *__restrict__ w,
                                              double *__restrict__ g, double *__restrict__ preds,
                                              unsigned long long *__restrict__ cnt, double w_pos, double w_neg,
                                              const double *__restrict__ sw, const double *__restrict__ icpt = nullptr) {
  static_assert(!kPreds || (kModel == kSvm && kWeight == kUnweighted), "only the unweighted SVM pass writes predictions");
  constexpr bool kCls = kWeight == kClassWeighted, kSw = kWeight == kSampleWeighted;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  // lane 0 only
  unsigned hinge = 0, correct = 0;
  unsigned long long lim[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf = 0;
  unsigned long long lim_ok[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_ok = 0;
  unsigned long long lim_w[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_w = 0;
  unsigned n_pos = 0, n_neg = 0, ok_pos = 0, ok_neg = 0, h_pos = 0, h_neg = 0;
  unsigned long long lim_pos[kLossLimbs] = {0, 0, 0, 0, 0, 0}, lim_neg[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_pos = 0, ovf_neg = 0;
  unsigned long long lim_bp[kLossLimbs] = {0, 0, 0, 0, 0, 0}, lim_bn[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_bp = 0, ovf_bn = 0;
  double beta = 0.0;
  if constexpr (kIcpt) beta = filt(__ldg(icpt));
  for (int64_t i = warp0; i < n; i += nwarps) {
    const int64_t r = samples ? (int64_t)samples[i] : row_begin + i;
    const int64_t b = (int64_t)rp16[r] * 2, e = (int64_t)rp16[r + 1] * 2;
    double dot = row_fold(pairs, b, e, lane, [&](uint32_t c) { return w[c]; });
    if constexpr (kIcpt) dot = dot + beta;
    const double y = (double)label[r];
    const int yi = (int)label[r];
    const bool pos = yi > 0;
    const double z = y * dot;
    const double ci = kSw ? (pos ? w_pos : w_neg) * (sw ? __ldg(&sw[r]) : 1.0) : 1.0;
    if (lane == 0) {
      if constexpr (kSw) {
        const int p = pred_of(dot);
        const bool ok = p == yi;
        correct += (unsigned)ok;
        double l;
        if constexpr (kModel != kSvm) l = row_loss<kModel>(z);
        else l = (double)(1 - yi * p);
        acc_add_local(lim, ovf, ci * l);
        if (!kScatter) {
          acc_add_local(lim_ok, ovf_ok, ok ? ci : 0.0);
          acc_add_local(lim_w, ovf_w, ci);
        }
      } else if constexpr (kCls) {
        const int p = pred_of(dot);
        const unsigned ok = (unsigned)(p == yi);
        if (pos) { ++n_pos; ok_pos += ok; } else { ++n_neg; ok_neg += ok; }
        if constexpr (kModel != kSvm) {
          const double l = row_loss<kModel>(z);
          acc_add_local(lim_pos, ovf_pos, pos ? l : 0.0);
          acc_add_local(lim_neg, ovf_neg, pos ? 0.0 : l);
        } else {
          const unsigned l = (unsigned)(1 - yi * p);
          if (pos) h_pos += l; else h_neg += l;
        }
      } else if constexpr (kModel != kSvm) {
        correct += (unsigned)(pred_of(dot) == (int)y);
        acc_add_local(lim, ovf, row_loss<kModel>(z));
      } else {
        const int p = pred_of(dot);
        const int yv = (int)y;
        hinge += (unsigned)(1 - yv * p);  // max(0, 1 - y*p), never negative for y,p in {-1,0,1}
        correct += (unsigned)(p == yv);
        if (kPreds) preds[i] = (double)p;
      }
    }
    if (kScatter) {
      const double c = kCls ? (pos ? w_pos : w_neg) : ci;   // the row's weight
      double s;
      if constexpr (kModel != kSvm) {
        if (kModel != kLogistic && z <= -1.0) continue;   // s = 0: the row scatters nothing
        s = kWeight == kUnweighted ? y * row_scale<kModel>(z) : (y * row_scale<kModel>(z)) * c;
      } else {
        if (z < 0.0) continue;  // SparseSVM.scala:28: gradient unless activity < 0
        s = kWeight == kUnweighted ? y : (pos ? c : -c);
      }
      if constexpr (kIcpt) {
        const double sb = filt(s);   // filt(filt(1) * s)
        if (lane == 0) {
          if (sb > 0.0) acc_add_local(lim_bp, ovf_bp, sb);
          else if (sb < 0.0) acc_add_local(lim_bn, ovf_bn, -sb);
        }
      }
      for (int64_t k = b + lane; k < e; k += 32) {
        const uint2 pr = pairs[k];
        const double gv = filt(filt((double)__uint_as_float(pr.y)) * s);  // x * s: mapValues + constructor filter
        if (gv == 0.0) continue;
        // the unweighted SVM's atomicAdd compiles to the same RED; red_add_f64 here would reorder the kernel's registers
        if (kModel == kSvm && kWeight == kUnweighted) atomicAdd(&g[pr.x], gv);
        else red_add_f64(&g[pr.x], gv);
      }
    }
  }
  if (lane == 0) {
    if constexpr (kCls) {
      if (n_pos) atomicAdd(&cnt[kCntClassN], (unsigned long long)n_pos);
      if (n_neg) atomicAdd(&cnt[kCntClassN + 1], (unsigned long long)n_neg);
      if (ok_pos) atomicAdd(&cnt[kCntClassCorrect], (unsigned long long)ok_pos);
      if (ok_neg) atomicAdd(&cnt[kCntClassCorrect + 1], (unsigned long long)ok_neg);
      if (kModel != kSvm) {
        acc_flush_local(cnt + kCntClassLoss, lim_pos, ovf_pos);
        acc_flush_local(cnt + kCntClassLoss + kLossAccWords, lim_neg, ovf_neg);
      } else {
        if (h_pos) atomicAdd(&cnt[kCntClassHinge], (unsigned long long)h_pos);
        if (h_neg) atomicAdd(&cnt[kCntClassHinge + 1], (unsigned long long)h_neg);
      }
    } else if (kSw || kModel != kSvm) {
      if (correct) atomicAdd(&cnt[kCntCorrect], (unsigned long long)correct);
      acc_flush_local(cnt + (kSw ? kCntSwLoss : kCntLoss), lim, ovf);
      if (kSw && !kScatter) {
        acc_flush_local(cnt + kCntSwCorrect, lim_ok, ovf_ok);
        acc_flush_local(cnt + kCntSwWeight, lim_w, ovf_w);
      }
    } else if (hinge | correct) {
      atomicAdd(&cnt[kCntHinge], (unsigned long long)hinge);
      atomicAdd(&cnt[kCntCorrect], (unsigned long long)correct);
    }
    if constexpr (kIcpt && kScatter) {
      acc_flush_local(cnt + kCntIcpt, lim_bp, ovf_bp);
      acc_flush_local(cnt + kCntIcpt + kLossAccWords, lim_bn, ovf_bn);
    }
  }
}

// k_sw_fold, one thread after a sample-weighted pass: S's bits into cnt[kCntWLoss] for the weighted tails (out == nullptr;
// the correct count stays in kCntCorrect), or {||w||^2, S, sum c_i [correct], sum c_i, correct} into out[0..4] (an
// evaluation).  The limb blocks, and in an evaluation the correct count, are cleared either way.
__global__ void k_sw_fold(unsigned long long *__restrict__ cnt, const double *__restrict__ scal_nrm2, double *__restrict__ out) {
  const double s = acc_take(cnt + kCntSwLoss);
  if (out) {
    out[0] = *scal_nrm2;
    out[1] = s;
    out[2] = acc_take(cnt + kCntSwCorrect);
    out[3] = acc_take(cnt + kCntSwWeight);
    out[4] = (double)cnt[kCntCorrect];
    cnt[kCntCorrect] = 0ull;
  } else {
    cnt[kCntWLoss] = (unsigned long long)__double_as_longlong(s);
  }
}

// k_class_fold, one thread after a class-weighted pass: L = fl(fl(w_pos * L_pos) + fl(w_neg * L_neg)) into cnt[kCntWLoss]
// and the correct total into cnt[kCntCorrect] for the weighted tails (out == nullptr), or the per-class totals and ||w||^2
// into out[0..6] (an evaluation); the per-class words are cleared either way.
template <int kModel>
__global__ void k_class_fold(unsigned long long *__restrict__ cnt, double w_pos, double w_neg,
                             const double *__restrict__ scal_nrm2, double *__restrict__ out) {
  double l_pos, l_neg;
  if (kModel != kSvm) {
    l_pos = acc_take(cnt + kCntClassLoss);
    l_neg = acc_take(cnt + kCntClassLoss + kLossAccWords);
  } else {
    l_pos = (double)cnt[kCntClassHinge];   // exact: counts are far below 2^53
    l_neg = (double)cnt[kCntClassHinge + 1];
    cnt[kCntClassHinge] = 0ull;
    cnt[kCntClassHinge + 1] = 0ull;
  }
  const unsigned long long ok_pos = cnt[kCntClassCorrect], ok_neg = cnt[kCntClassCorrect + 1];
  if (out) {
    out[0] = *scal_nrm2;
    out[1] = l_pos;
    out[2] = l_neg;
    out[3] = (double)ok_pos;
    out[4] = (double)ok_neg;
    out[5] = (double)cnt[kCntClassN];
    out[6] = (double)cnt[kCntClassN + 1];
  } else {
    const double a = w_pos * l_pos, b = w_neg * l_neg;
    cnt[kCntWLoss] = (unsigned long long)__double_as_longlong(a + b);
    cnt[kCntCorrect] = ok_pos + ok_neg;
  }
  cnt[kCntClassN] = 0ull;
  cnt[kCntClassN + 1] = 0ull;
  cnt[kCntClassCorrect] = 0ull;
  cnt[kCntClassCorrect + 1] = 0ull;
}

// ---------------------------------------------------------------------------------------------------
// k_finish: regularize in place -- r_j = g_j + c on the keys that survived the 1e-20 filter
// (SparseSVM.scala:31; math/Vec.scala:65-75).  Also publishes the batch's hinge sum and size in
// g[dim], g[dim+1] so that they ride along in the gradient allreduce.
//   kModel, kCw: where the batch's loss sum comes from (batch_loss_sum; kCw after k_class_fold).
//   kIcpt: also the intercept's gradient (icpt_take, never regularized) into g[dim + kIcptSlot].
// ---------------------------------------------------------------------------------------------------
template <int kModel, bool kCw, bool kIcpt = false>
__global__ void __launch_bounds__(256) k_finish(double *__restrict__ g, int dim, const double *__restrict__ scal_c,
                                                const unsigned long long *__restrict__ cnt, double n_samples) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const double c = *scal_c;
  const bool add_c = (c != 0.0) && (fabs(c) > kEps);
  if (j < dim) {
    double v = filt(g[j]);
    if (v != 0.0 && add_c) v = filt(v + c);
    g[j] = v;
  } else if (j == dim) {
    g[dim] = batch_loss_sum<kModel, kCw>(cnt);
    g[dim + 1] = n_samples;
    if constexpr (kIcpt)   // the request clears the two sums afterwards, with g
      g[dim + kIcptSlot] = filt(acc_value(cnt + kCntIcpt) - acc_value(cnt + kCntIcpt + kLossAccWords));
  }
}

// ---------------------------------------------------------------------------------------------------
// k_finish_acc: one logical worker's reply folded into the master's running sum.  r = regularize(g) on the
// worker's own support (SparseSVM.scala:31), then sum <- sum + r with the constructor filter after the
// addition (Vec.sum is a left fold of `+`, math/Vec.scala:128-131), g cleared for the next worker.
// Slots [dim], [dim+1] of `sum` carry the loss total (kCw: the weighted one) and the sample count of the step.
// kIcpt: slot [dim + kIcptSlot] folds the intercept's gradients like any other entry (icpt_take, never regularized).
// ---------------------------------------------------------------------------------------------------
template <int kModel, bool kCw, bool kIcpt = false>
__global__ void __launch_bounds__(256) k_finish_acc(double *__restrict__ g, double *__restrict__ sum, int dim,
                                                    const double *__restrict__ scal_c,
                                                    unsigned long long *__restrict__ cnt, double n_samples, int first) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const double c = *scal_c;
  const bool add_c = (c != 0.0) && (fabs(c) > kEps);
  if (j < dim) {
    const double raw = g[j];
    double v = filt(raw);
    if (v != 0.0 && add_c) v = filt(v + c);
    if (raw != 0.0) g[j] = 0.0;
    sum[j] = first ? v : filt(sum[j] + v);
  } else if (j == dim) {
    const double h = batch_loss_sum<kModel, kCw>(cnt);
    sum[dim] = first ? h : sum[dim] + h;
    sum[dim + 1] = first ? n_samples : sum[dim + 1] + n_samples;
    if constexpr (kIcpt) {
      const double v = icpt_take(cnt);
      sum[dim + kIcptSlot] = first ? v : filt(sum[dim + kIcptSlot] + v);
    }
    clear_batch_loss<kModel, kCw>(cnt);
    cnt[kCntCorrect] = 0ull;
  }
}

// ---------------------------------------------------------------------------------------------------
// k_update: the master's aggregate + SGD update (core/Master.scala:194,197) fused with the bookkeeping
// for the next step:  w_j <- w_j - lr * (sum_j / K);  gradient buffer zeroed;  c and ||w||^2 of the NEW
// weights reduced (fixed order: per-block partial -> last block sums the slots in index order) so that the
// next step needs no separate reduction; per-step loss = lambda*||w_before||^2 + hinge/total written.
//   kFuseRegularize: the buffer holds the raw local sum (single worker): apply regularize() here.
//   otherwise it holds sum_k r^(k) (already regularized per worker, then allreduced).
//   kModel: where the batch's loss sum comes from (batch_loss_sum).
//   kAvg: also avg_j <- avg_j + w_j of the NEW weights, every column (averaged SGD, dsgd_average_begin); otherwise avg is
//   nullptr.
//   kL1: after the update, the proximal step of the L1 penalty lambda1 * ||w||_1 on EVERY column,
//   w_j <- soft_threshold(u_j, lr * lambda1); c, ||w||^2, ||w||_1 and the averaging sum then see the thresholded weights, and
//   the step's loss adds lambda1 * ||w_before||_1 (scal[kScalL1]).  ||w||_1 is summed in fixed-point limbs (acc_push_block),
//   so it has the same bits as k_l1_norm over the same weights.  Otherwise lambda1 is not read.
//   kCw: the batch's loss sum is the class-weighted one of k_class_fold (batch_loss_sum<kModel, true>).
//   kIcpt: the last block's thread 0 also steps the intercept beta = w[dim] on its gradient g_b (icpt_take with
//   kFuseRegularize, else g[dim + kIcptSlot]): beta <- filt(beta - filt(filt(g_b / K) * lr)), the other entries' chain
//   without c and without the L1 step; averaging adds beta to avg[dim].  beta is in neither c, ||w||^2 nor ||w||_1.
// ---------------------------------------------------------------------------------------------------
template <bool kFuseRegularize, int kModel, bool kAvg, bool kL1, bool kCw, bool kIcpt = false>
__global__ void __launch_bounds__(256) k_update(double *__restrict__ w, float *__restrict__ w32, double *__restrict__ g,
                                                const double *__restrict__ d, int dim, double lambda, double lr,
                                                double inv_k_den, double *__restrict__ scal,
                                                unsigned long long *__restrict__ cnt, double *__restrict__ partial,
                                                double n_samples_local, double *__restrict__ loss_out,
                                                double *__restrict__ avg, double lambda1) {
  __shared__ double red[8];
  __shared__ bool is_last;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const double c = scal[kScalC];
  const bool add_c = (c != 0.0) && (fabs(c) > kEps);
  double pd = 0.0, pn = 0.0, pa = 0.0;
  if (j < dim) {
    const double raw = g[j];
    double v = raw;
    if (kFuseRegularize) {
      v = filt(v);
      if (v != 0.0 && add_c) v = filt(v + c);
    }
    double wn = w[j];
    const double w_before = wn;
    if (raw != 0.0) g[j] = 0.0;
    if (v != 0.0) {
      const double mean = filt(v / inv_k_den);  // Vec.mean: sum / K
      const double step = filt(mean * lr);      // learningRate * grad
      wn = filt(wn - step);                     // batchWeights - ...
      if (!kL1) {
        w[j] = wn;
        w32[j] = (float)wn;
      }
    }
    if (kL1) {
      wn = soft_threshold(wn, lr * lambda1);
      if (__double_as_longlong(wn) != __double_as_longlong(w_before)) {
        w[j] = wn;
        w32[j] = (float)wn;
      }
      pa = fabs(wn);
    }
    if (kAvg) avg[j] = avg[j] + wn;
    pd = filt(wn * d[j]);
    pn = wn * wn;
  }
  if (kL1) acc_push_block<256>(pa, cnt + kCntL1);
  pd = block_sum<256>(pd, red);
  pn = block_sum<256>(pn, red);
  if (threadIdx.x == 0) {
    partial[2 * blockIdx.x] = pd;
    partial[2 * blockIdx.x + 1] = pn;
    __threadfence();
    const unsigned long long t = atomicAdd(&cnt[kCntTicket], 1ull);
    is_last = (t == (unsigned long long)gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    double sd = 0.0, sn = 0.0;
    if (threadIdx.x == 0) {
      for (unsigned b = 0; b < gridDim.x; ++b) {
        sd += __ldcg(&partial[2 * b]);
        sn += __ldcg(&partial[2 * b + 1]);
      }
      // per-step loss on the weights the gradient was taken at (SparseSVM.scala:20-23; SURVEY.md F5)
      double hinge, total;
      if (kFuseRegularize) {
        hinge = batch_loss_sum<kModel, kCw>(cnt);
        total = n_samples_local;
      } else {
        hinge = g[dim];
        total = g[dim + 1];
        g[dim] = 0.0;
        g[dim + 1] = 0.0;
      }
      if (kL1) {
        if (loss_out) *loss_out = lambda * scal[kScalNrm2] + lambda1 * scal[kScalL1] + hinge / total;
        scal[kScalL1] = acc_take(cnt + kCntL1);
      } else if (loss_out) {
        *loss_out = lambda * scal[kScalNrm2] + hinge / total;
      }
      scal[kScalC] = lambda * 2.0 * sd;
      scal[kScalNrm2] = sn;
      if constexpr (kIcpt) {
        double gb;
        if (kFuseRegularize) {
          gb = icpt_take(cnt);
        } else {
          gb = g[dim + kIcptSlot];
          g[dim + kIcptSlot] = 0.0;
        }
        double beta = w[dim];
        if (gb != 0.0) {
          beta = filt(beta - filt(filt(gb / inv_k_den) * lr));
          w[dim] = beta;
          w32[dim] = (float)beta;
        }
        if (kAvg) avg[dim] = avg[dim] + beta;
      }
      clear_batch_loss<kModel, kCw>(cnt);
      cnt[kCntCorrect] = 0ull;
      cnt[kCntTicket] = 0ull;
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// k_l1_norm + k_l1_finish: ||w||_1 = sum_j |w_j| in the fixed-point limbs (exact in any order: every |w_j| > 1e-20 is a
// multiple of 2^-160) and #{w_j != 0}, over one column per thread; k_l1_finish converts the sum once, writes it to *l1_out
// and the count to *nnz_out (if not null), and clears the counter words for the next pass.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_l1_norm(const double *__restrict__ w, int dim, unsigned long long *__restrict__ cnt) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const double wj = j < dim ? w[j] : 0.0;
  acc_push_block<256>(fabs(wj), cnt + kCntL1);
  const int nz = __syncthreads_count(wj != 0.0);
  if (threadIdx.x == 0 && nz) atomicAdd(&cnt[kCntNnz], (unsigned long long)nz);
}
__global__ void k_l1_finish(unsigned long long *__restrict__ cnt, double *__restrict__ l1_out, long long *__restrict__ nnz_out) {
  *l1_out = acc_take(cnt + kCntL1);
  if (nnz_out) *nnz_out = (long long)cnt[kCntNnz];
  cnt[kCntNnz] = 0ull;
}

// ---------------------------------------------------------------------------------------------------
// k_loss_scalar: loss = lambda*||w||^2 + loss sum/n, acc = correct/n from the counters (SVM: hinge sum, an integer;
// other models: the fixed-point sum of their per-sample losses; kCw: the class-weighted sum of k_class_fold).
// ---------------------------------------------------------------------------------------------------
template <int kModel, bool kCw>
__global__ void k_loss_scalar(const double *__restrict__ scal_nrm2, unsigned long long *__restrict__ cnt, double lambda,
                              double n, double *__restrict__ out2) {
  out2[0] = lambda * (*scal_nrm2) + batch_loss_sum<kModel, kCw>(cnt) / n;
  out2[1] = (double)cnt[kCntCorrect] / n;
  out2[2] = batch_loss_sum<kModel, kCw>(cnt);   // SVM: exact, counts are far below 2^53
  out2[3] = (double)cnt[kCntCorrect];
  out2[4] = *scal_nrm2;
  clear_batch_loss<kModel, kCw>(cnt);
  cnt[kCntCorrect] = 0ull;
}

// ---------------------------------------------------------------------------------------------------
// K0: document frequencies and dimSparsity (Main.scala:54-65).
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_col_hist(const uint2 *__restrict__ pairs, int64_t n_pairs,
                                                  unsigned *__restrict__ df) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_pairs; k += (int64_t)gridDim.x * blockDim.x) {
    const uint2 pr = pairs[k];
    if (fabs((double)__uint_as_float(pr.y)) > kEps) atomicAdd(&df[pr.x], 1u);  // padding pairs have val == 0
  }
}
__global__ void __launch_bounds__(256) k_dim_sparsity(const unsigned *__restrict__ df, int dim, double *__restrict__ d) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < dim) {
    // reference key c of d holds 1/(df_c + 1); weight column c is reference key c+1, so it meets d key c+1 (Q3)
    const int src = c + 1;
    d[c] = (src < dim && df[src] != 0u) ? 1.0 / ((double)df[src] + 1.0) : 0.0;
  }
}

// ---------------------------------------------------------------------------------------------------
// Repack: host CSR (row_ptr int64, col, val) -> aligned pair windows.  One thread per destination pair.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_repack(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ col,
                                                const float *__restrict__ val, const uint32_t *__restrict__ rp16,
                                                const int8_t *__restrict__ label, int64_t n_rows, uint2 *__restrict__ pairs,
                                                float *__restrict__ yabs) {
  // one warp per row keeps the writes coalesced
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = warp0; r < n_rows; r += nwarps) {
    const int64_t sb = row_ptr[r], se = row_ptr[r + 1];
    const int64_t db = (int64_t)rp16[r] * 2, de = (int64_t)rp16[r + 1] * 2;
    const int64_t len = se - sb;
    double asum = 0.0;
    for (int64_t k = lane; k < de - db; k += 32) {
      uint2 pr;
      if (k < len) {
        // |v| <= 1e-20 is absent from the reference's row (Sparse.scala:108-118) and every kernel filters it out: stored as
        // 0, so that the streaming pass's fp32 dot and yabs see the live values only
        const float v = val[sb + k];
        const float vf = fabs((double)v) > kEps ? v : 0.f;
        pr.x = (uint32_t)col[sb + k];
        pr.y = __float_as_uint(vf);
        asum += fabs((double)vf);
      } else {
        pr.x = len > 0 ? (uint32_t)col[se - 1] : 0u;
        pr.y = 0u;
      }
      pairs[db + k] = pr;
    }
    // yabs[r] = label * sum_j |x_j| rounded UP to fp32 (the sign bit carries the label, also on a zero sum): the streaming
    // pass reads the label and the rounding-band scale of a row with one 4-byte load
    asum = warp_sum(asum);
    if (lane == 0) {
      const float a = __double2float_ru(asum);
      yabs[r] = label[r] < 0 ? -a : a;
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// k_draw_rows: positions [pos_begin, pos_begin + n_pos) of a keyed permutation of [0, n) as row ids (Master.scala:
// 109-118: `Random.shuffle(workingData.indices) take samplesCount`, dsgd_feistel.h).  One thread per position.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_draw_rows(int32_t *__restrict__ ids, int64_t n_pos, uint32_t pos_begin,
                                                   int half_bits, uint64_t key, uint32_t n, int64_t row_begin) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_pos) ids[i] = (int32_t)(row_begin + (int64_t)dsgd_feistel(pos_begin + (uint32_t)i, half_bits, key, n));
}

__global__ void __launch_bounds__(256) k_to_f32(const double *__restrict__ src, float *__restrict__ dst, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) dst[j] = (float)src[j];
}

}  // namespace dsgd
