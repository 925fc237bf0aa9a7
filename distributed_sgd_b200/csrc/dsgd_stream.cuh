// dsgd_stream.cuh -- streaming pass over many row windows: Master.localLoss/localAccuracy (core/Master.scala:
// 100-107), SlaveImpl.forward (core/Slave.scala:129-140) and large-batch SlaveImpl.gradient (142-157).
//
// This is the HBM-bound form of the hot path (roofline: 8*nnz + 16 bytes per sample, SURVEY.md 8d).
//   * The weight vector is staged ONCE per CTA into shared memory as fp32 (47 236 x 4 B = 189 KB of the 227 KB),
//     so the ~94 gathers per row hit shared-memory banks, not 32-byte L2 sectors.  One persistent CTA per SM.
//   * FLAT STREAM.  A warp owns blocks of 32 rows and walks their 16-byte units (2 pairs) as ONE virtual
//     stream: unit v of the block belongs to the row whose prefix-sum interval contains v, found with one ballot
//     and one or-reduction per 32 units -- every lane loads a useful unit whatever the row lengths are (round 1
//     walked a row per 16-lane group: 47 of 64 load slots used on the mean row, long rows serialised), kUnroll
//     128-bit loads per lane are in flight before the first is used (64 KB per SM), and consecutive rows of an
//     evaluation pass make every warp load one contiguous 512-byte request.
//   * The dot is needed for its SIGN only (prediction, gate: SparseSVM.scala:14,28), so it is accumulated with fp32
//     FMAs against the fp32 weights -- no fp32->fp64 conversions (ncu, round 1: the XU pipe they run on was 46 %
//     busy).  A lane accumulates its units of the open row; the warp reduces once per ROW END (one 5-step butterfly
//     of ONE float), not per load, and the row's lane just keeps the sum: predictions, counters and gates of the 32
//     rows are worked out by 32 lanes in parallel after the block's stream.  The kernel is ISSUE-bound before it is
//     HBM-bound (fewer warp instructions per 64 pairs made the evaluation
//     pass faster at every step), so every per-slot instruction counts: groups that lie inside the block
//     carry no bounds predicates (only a block's last group does), a slot without a row end adds its products with one
//     FADD, and a pass over CONSECUTIVE rows (kContig: evaluation) needs no row lookup for its loads at all -- the windows
//     are back to back in the pair array -- so its four loads leave before the row-end masks are even computed.
//   * Blocks are dealt dynamically (one atomic per block, requested a block ahead); the last fifth of a pass goes out in
//     blocks of half the size so the warps run dry together.
//   * Exactness against the fp64 arithmetic of the reference.  Let W = max(max|w32|, 2^-126) over the staged weights and
//     u = 2^-24.  If the fp32 dot is FINITE, no operation of its chain overflowed (an overflow gives +-inf, and inf + x is
//     inf or NaN), and no weight the row reads is infinite or NaN (0 * inf and x * NaN are NaN).  Then every rounding is
//     relative with at most u, or absolute: (float)w is within max(u |w|, 2^-150) <= u W of w, and a product or fma that
//     lands in fp32's subnormal range is within 2^-150 (sums of fp32 values are exact there).  So the fp32 result differs
//     from x.w by at most
//       (D + 1) * u * W * sum|x| + 2 * 2^-150 per unit,   D = units/32 + 9 roundings on the longest add chain
//     (product, fma, at most units/32 + 1 lane additions, 5 butterfly steps), + 1 for rounding w (first-order bound,
//     1.5x slack).  sum|x| per row is computed once when the rows are loaded (k_repack, rounded up -- to inf when it
//     exceeds FLT_MAX -- and stored with the label in its sign bit: one 4-byte load per row).  The reference also drops
//     every value and every product with magnitude <= 1e-20 (the Sparse constructor, filt): k_repack stores such values
//     as 0, and the products the fp32 dot keeps are bounded by 1e-20 per pair, so the band gets 2 * 1e-20 per unit on top
//     (which also covers the subnormal 2^-150 terms).  The band is formed in fp64 from W, which is at least 2^-126, so it
//     neither underflows (a band of 0 would decide every row of subnormal weights from its fp32 sign) nor overflows.  Rows
//     whose fp32 dot is not finite or whose |dot| is inside the band are recomputed after the block's stream with the fp64
//     weights from L2, by the row fold (dsgd_kernels.cuh) that decides the row on every other path
//     (tests/test_gpu_streaming.py, test_gpu_stream_range.py, test_gpu_row_fold.py; tests/stream_band_model.py restates
//     this decision on the CPU; dsgd_stream_exact_rows counts the recomputed rows).  Outside the band the fp32 sign is the
//     row fold's sign: there |exact x.w| >= band / 3, far above the difference between any two fp64 summation orders
//     (every fp64 product is finite: |x| and |w| are at most FLT_MAX), so every prediction and gate decision of the
//     pass is that of the row fold.  An infinite weight anywhere makes W, hence every band, infinite (or NaN on a row
//     whose values were all filtered): the whole pass is recomputed.
//   * Scatter (gradient): rows that pass the gate are re-walked after the block's stream (their units are in
//     L1/L2) and y*x goes to g with fp64 REDs.  On trained weights few rows pass (the misclassified ones) and the pass
//     runs at the streaming rate; on untrained weights every row passes and the fp64 RED rate at L2 bounds it
//     (tools/microbench.cu).  Per-CTA fixed-point accumulators in shared memory for the most frequent columns were
//     measured and dropped (no net gain).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dsgd_kernels.cuh"

namespace dsgd {

struct TrueTag { static constexpr bool value = true; };
struct FalseTag { static constexpr bool value = false; };

constexpr int kStreamThreads = 1024;
constexpr int kStreamUnroll = 4;

struct StreamParams {
  const uint32_t *rp16;
  const uint4 *units;      // the pair array viewed as 16-byte units (2 pairs)
  const float *yabs;       // per row: label * sum_j |x_j| (rounded up); the sign bit is the label
  const int32_t *samples;  // nullptr: rows [row_begin, row_begin + n)
  int64_t row_begin, n;
  const double *w;         // fp64 weights (exact fallback, L2)
  const float *w32;        // fp32 shadow of the same weights
  int dim;
  double *g;               // scatter target (fp64, L2) or nullptr
  double *preds;           // per-sample predictions or nullptr
  unsigned long long *cnt; // kCntHinge / kCntCorrect
  unsigned long long *n_exact;     // rows that took the exact fallback (diagnostic)
  unsigned long long *next_block;  // work counter (zero on entry): blocks beyond the first wave are claimed dynamically
  int rows_log2;               // rows per block = 1 << rows_log2 (5, 4 or 3): the host picks it so that every warp gets
                               // several blocks (a block is the unit of the dynamic work distribution)
  int64_t n_big;               // blocks [0, n_big) have 1 << rows_log2 rows, the blocks after them 1 << tail_log2: the
  int tail_log2;               // last part of a pass is dealt in smaller pieces, so the warps run dry together
  // ---- class weights (kCls); last, so that the parameter offsets of the other instantiations stay where they were ----
  double w_pos, w_neg;         // a row of label y that passes the gate scatters x * (y * w_y)
};

__host__ __device__ constexpr size_t stream_smem_bytes(int dim) { return (((size_t)dim + 3) & ~(size_t)3) * sizeof(float); }

// kContig: the rows of the pass are consecutive (samples == nullptr), hence so are their windows in the pair array: unit v
// of a block sits at (first window) + v and the loads need no row lookup (5 instructions per slot less, and the row-end
// masks are worked out while the loads are in flight).
// kCls: the per-class form (dsgd_set_class_weights, dsgd_eval*_class).  Every thread keeps the hinge and correct counts of
// the y = -1 rows and the rows of each class apart (six counters instead of two), reduced and flushed like the two, into the
// kCntClass* words that k_class_fold reads; the scatter value is x * (y * w_y).  The rounding band and the fp64
// recomputation are unchanged: the weight never touches the dot.
template <bool kScatter, bool kPreds, bool kContig, bool kCls = false>
__global__ void __launch_bounds__(kStreamThreads, 1) k_stream_rows(const StreamParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float *ws = reinterpret_cast<float *>(smem_raw);
  __shared__ float s_wmax[kStreamThreads / 32];
  constexpr bool kRows = kCls && !kScatter;   // a gradient reports neither rows nor correct predictions: its per-class form
                                              // counts the two hinge sums only (1024 threads leave 64 registers each)
  constexpr int kCounters = kRows ? 6 : (kCls ? 4 : 2);
  __shared__ unsigned long long s_cnt[kCounters];
  unsigned hinge_neg = 0, correct_neg = 0, n_pos = 0, n_neg = 0;   // kCls only; hinge and correct then count the y = +1 rows

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int rlog = p.rows_log2, tlog = p.tail_log2;
  const int64_t tail_row0 = p.n_big << rlog;   // first row of the smaller tail blocks
  const int64_t n_blocks = p.n_big + ((p.n - tail_row0 + (1 << tlog) - 1) >> tlog);
  const int64_t warp_global = (int64_t)blockIdx.x * (kStreamThreads / 32) + warp;
  const int64_t n_warps = (int64_t)gridDim.x * (kStreamThreads / 32);
  unsigned hinge = 0, correct = 0, n_exact = 0;

  // bounds of the block being processed / the next one: lane l holds row l of the block
  auto load_block = [&](int64_t blk, int64_t &first, uint32_t &b, uint32_t &e, float &ya, bool &valid) {
    const bool big = blk < p.n_big;
    first = big ? (blk << rlog) : tail_row0 + ((blk - p.n_big) << tlog);
    const int64_t i = first + lane;
    b = 0u; e = 0u; ya = 0.f;
    valid = blk < n_blocks && lane < (1 << (big ? rlog : tlog)) && i < p.n;
    if (valid) {
      const int64_t rid = (!kContig && p.samples) ? (int64_t)__ldg(&p.samples[i]) : p.row_begin + i;
      b = __ldg(&p.rp16[rid]);
      e = __ldg(&p.rp16[rid + 1]);
      ya = __ldg(&p.yabs[rid]);
    }
  };
  // Work distribution: the first wave is static (block = warp id), later blocks are claimed from a global counter one
  // step ahead; the ticket (an atomic with a return value) is requested when a block starts and read when it ends, the
  // next block's bounds were prefetched a block earlier.
  unsigned long long ticket = 0;   // lane 0: the pending claim
  auto claim_issue = [&]() {
    if (lane == 0) ticket = atomicAdd(p.next_block, 1ull);
  };
  auto claim_get = [&]() -> int64_t { return (int64_t)__shfl_sync(0xffffffffu, ticket, 0) + n_warps; };
  uint32_t nb, ne; float nya; bool nvalid; int64_t nfirst;
  int64_t blk = warp_global;
  int64_t blk_next = n_blocks;
  if (blk < n_blocks) claim_issue();
  load_block(blk, nfirst, nb, ne, nya, nvalid);   // (requested before the weights are staged: latency off the path)

  // ---- stage the fp32 weights, find max|w| ----
  float wmax = 0.f;
  {
    const float4 *src = reinterpret_cast<const float4 *>(p.w32);
    float4 *dst = reinterpret_cast<float4 *>(ws);
    const int n4 = p.dim >> 2;
    for (int i = threadIdx.x; i < n4; i += kStreamThreads) {
      const float4 v = __ldg(&src[i]);
      dst[i] = v;
      wmax = fmaxf(wmax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
    for (int i = (n4 << 2) + threadIdx.x; i < p.dim; i += kStreamThreads) {
      const float v = __ldg(&p.w32[i]);
      ws[i] = v;
      wmax = fmaxf(wmax, fabsf(v));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = fmaxf(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) s_wmax[warp] = wmax;
    if (threadIdx.x < kCounters) s_cnt[threadIdx.x] = 0ull;
    __syncthreads();
    wmax = 0.f;
#pragma unroll
    for (int i = 0; i < kStreamThreads / 32; ++i) wmax = fmaxf(wmax, s_wmax[i]);
  }
  // one gradient entry (SparseSVM.scala:26-29): a reduction without a return value
  auto scatter_one = [&](uint32_t col, double gv) {
    if (gv != 0.0) red_add_f64(&p.g[col], gv);
  };

  if (blk < n_blocks) blk_next = claim_get();
  for (; blk < n_blocks;) {
    uint32_t b = nb;
    int len = (int)(ne - nb);   // units
    float ya = nya;
    bool valid = nvalid;
    const int64_t first = nfirst;   // first row (position in the pass) of this block
    load_block(blk_next, nfirst, nb, ne, nya, nvalid);
    if (blk_next < n_blocks) claim_issue();   // for the block after next: read at the end of this block
    int opos = lane;            // position of this lane's row inside the block (before compaction)
    // empty rows: dot 0 -> prediction 0, hinge 1, never correct, nothing to scatter (SparseSVM.scala:14-16)
    if (valid && len == 0) {
      if (kCls && (__float_as_uint(ya) >> 31)) { hinge_neg += 1u; if (kRows) ++n_neg; }
      else { hinge += 1u; if (kRows) ++n_pos; }
      if (kPreds) p.preds[first + lane] = 0.0;
    }
    const unsigned ne_mask = __ballot_sync(0xffffffffu, valid && len > 0);
    if (ne_mask != 0xffffffffu) {   // compact the non-empty rows to lanes 0 .. n-1 (order kept)
      const unsigned src = __fns(ne_mask, 0, lane + 1);
      const bool has = src < 32u;
      const int sl = has ? (int)src : 0;
      b = __shfl_sync(0xffffffffu, b, sl);
      len = __shfl_sync(0xffffffffu, len, sl);
      ya = __shfl_sync(0xffffffffu, ya, sl);
      opos = sl;
      valid = has;
      if (!has) len = 0;
    } else {
      valid = true;
    }
    const int y = (__float_as_uint(ya) >> 31) ? -1 : 1;
    // P = inclusive prefix sum of the row lengths: row l covers virtual units [P - len, P)
    int P = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, P, o);
      if (lane >= o) P += a;
    }
    const int total = __shfl_sync(0xffffffffu, P, 31);
    const uint32_t base = b - (uint32_t)(P - len);   // unit address of virtual unit v of this row = base + v (mod 2^32)
    const uint32_t base0 = __shfl_sync(0xffffffffu, base, 0);   // kContig: the same for every row of the block
    const int my_end = len > 0 ? P - 1 : -1;          // virtual position of this row's LAST unit
    float acc_p = 0.f;                                // this lane's share of the OPEN row: sum x*w
    float dot_mine = 0.f;                             // this lane's row: x.w in fp32 once the row is closed
    int row0 = 0;                                     // rows closed so far (warp-uniform)

    // One GROUP = kStreamUnroll slots of 32 units: where rows end inside the group (one or-reduction per slot), hence the
    // row of each lane's unit, then the 128-bit loads -- all issued before the first is used (64 KB in flight per SM).
    // Groups that lie entirely inside the block (kFull) carry no bounds predicates; the block's last group does.
    // (A software-prefetched form -- group g + 1 fetched before group g is processed, 768 threads x 80 registers -- was
    // measured SLOWER per evaluation pass: the lost warps cost more
    // latency hiding than the deeper queue bought.)
    auto do_group = [&](auto full_tag, const int v0) {
      constexpr bool kFull = decltype(full_tag)::value;
      uint4 q[kStreamUnroll];
      unsigned ends[kStreamUnroll];   // bit j: a row's LAST unit sits at lane j of this slot
      const unsigned pos = (unsigned)(my_end - v0);          // < 32 * kStreamUnroll iff the row ends in this group
      const unsigned bit = 1u << (pos & 31u);
      if constexpr (kContig) {
#pragma unroll
        for (int i = 0; i < kStreamUnroll; ++i) {
          if (kFull || v0 + 32 * i + lane < total) q[i] = __ldg(&p.units[base0 + (uint32_t)(v0 + 32 * i + lane)]);
          else q[i] = make_uint4(0u, 0u, 0u, 0u);  // col 0, val +0.0f
        }
#pragma unroll
        for (int i = 0; i < kStreamUnroll; ++i)
          ends[i] = __reduce_or_sync(0xffffffffu, (pos >> 5) == (unsigned)i ? bit : 0u);
      } else {
        int r0 = row0;
#pragma unroll
        for (int i = 0; i < kStreamUnroll; ++i) {
          ends[i] = __reduce_or_sync(0xffffffffu, (pos >> 5) == (unsigned)i ? bit : 0u);
          const int rmy = r0 + __popc(ends[i] & lt_mask);      // row of this lane's unit
          r0 += __popc(ends[i]);
          const uint32_t bs = __shfl_sync(0xffffffffu, base, rmy & 31);
          if (kFull || v0 + 32 * i + lane < total) q[i] = __ldg(&p.units[bs + (uint32_t)(v0 + 32 * i + lane)]);
          else q[i] = make_uint4(0u, 0u, 0u, 0u);
        }
      }
#pragma unroll
      for (int i = 0; i < kStreamUnroll; ++i) {
        float pp = __fmaf_rn(__uint_as_float(q[i].w), ws[q[i].z], __uint_as_float(q[i].y) * ws[q[i].x]);
        if (!kFull && !(v0 + 32 * i + lane < total)) pp = 0.f;   // a masked unit reads ws[0]: keep a NaN / inf weight out
        unsigned m = ends[i];
        if (m == 0u) {   // warp-uniform: no row ends inside this slot
          acc_p += pp;
        } else {
          const int rmy = row0 + __popc(m & lt_mask);           // row0 == rows closed before this slot
          do {   // close the rows that end inside this slot, in order
            m &= m - 1u;
            float sp = acc_p + (rmy == row0 ? pp : 0.f);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sp += __shfl_xor_sync(0xffffffffu, sp, o);
            if (lane == row0) dot_mine = sp;
            acc_p = 0.f;
            ++row0;
          } while (m);
          acc_p = (rmy == row0) ? pp : 0.f;
        }
      }
    };
    {
      int v0 = 0;
      for (; v0 + 32 * kStreamUnroll <= total; v0 += 32 * kStreamUnroll) do_group(TrueTag{}, v0);
      if (v0 < total) do_group(FalseTag{}, v0);
    }
    // ---- 32 rows decided by 32 lanes: inside the rounding band -> exact recomputation; else the sign is certain ----
    bool need_exact = false, do_scatter = false;
    int pred_mine = 0;
    // prediction known for this lane's row: counters and the gate (y * dot < 0  <=>  pred == y)
    auto finalize = [&](int pr) {
      pred_mine = pr;
      if (kCls && y < 0) {
        hinge_neg += (unsigned)(1 - y * pr);
        if (kRows) { correct_neg += (unsigned)(pr == y); ++n_neg; }
      } else {
        hinge += (unsigned)(1 - y * pr);
        if (!kCls || kRows) correct += (unsigned)(pr == y);
        if (kRows) ++n_pos;
      }
      do_scatter = kScatter && (pr != y);
    };
    if (valid) {
      // rounding band + the products the reference drops (|x_j w_j| <= 1e-20, filt) but the fp32 dot keeps: one per pair.
      // In fp64, so that neither the band nor its product with yabs underflows or overflows; a dot that is not finite (an
      // fp32 overflow somewhere in the chain, an inf or NaN weight) says nothing about the fp64 sign.
      // 1.5 * 2^-24 * max(max|w|, 2^-126): 2^-24 * 2^-126 bounds the rounding of a subnormal weight (formed per row, so
      // that the stream loop keeps one fp32 register for it, as before)
      const double band_scale = 1.5 * 5.9604644775390625e-8 * fmax((double)wmax, 1.1754943508222875e-38);
      const double thresh = band_scale * (double)fabsf(ya) * (double)((len >> 5) + 10) + 2e-20 * (double)len;
      const float adot = fabsf(dot_mine);
      if (!(adot <= 3.40282347e38f && (double)adot > thresh)) need_exact = true;   // also catches NaN
      else finalize(dot_mine > 0.f ? -1 : 1);
    }
    // ---- exact recomputation of the rows the fp32 sign could not decide ----
    unsigned ex = __ballot_sync(0xffffffffu, need_exact);
    while (ex) {
      const int r = __ffs(ex) - 1;
      ex &= ex - 1u;
      const uint32_t rb = __shfl_sync(0xffffffffu, b, r);
      const int rl = __shfl_sync(0xffffffffu, len, r);
      const int64_t pb = 2 * (int64_t)rb;   // the window in pairs
      const double dot = row_fold(reinterpret_cast<const uint2 *>(p.units), pb, pb + 2 * (int64_t)rl, lane,
                                  [&](uint32_t c) { return __ldcg(&p.w[c]); });
      if (lane == r) {
        finalize(pred_of(dot));
        ++n_exact;
      }
    }
    if (kPreds) {
      if (valid) p.preds[first + opos] = (double)pred_mine;
    }
    // ---- scatter y*x of the rows that passed the gate (SparseSVM.scala:28) ----
    if (kScatter) {
      unsigned sc = __ballot_sync(0xffffffffu, do_scatter);
      while (sc) {
        const int r = __ffs(sc) - 1;
        sc &= sc - 1u;
        const uint32_t rb = __shfl_sync(0xffffffffu, b, r);
        const int rl = __shfl_sync(0xffffffffu, len, r);
        const int yr = __shfl_sync(0xffffffffu, y, r);
        const double yy = kCls ? (yr > 0 ? p.w_pos : -p.w_neg) : (double)yr;
        for (int u = lane; u < rl; u += 32) {
          const uint4 qq = __ldg(&p.units[rb + (uint32_t)u]);
          scatter_one(qq.x, filt(filt((double)__uint_as_float(qq.y)) * yy));
          scatter_one(qq.z, filt(filt((double)__uint_as_float(qq.w)) * yy));
        }
      }
    }
    blk = blk_next;
    if (blk < n_blocks) blk_next = claim_get();
  }
  // ---- counters: lane -> warp -> CTA -> one atomic per CTA ----
  hinge = __reduce_add_sync(0xffffffffu, hinge);
  correct = __reduce_add_sync(0xffffffffu, correct);
  n_exact = __reduce_add_sync(0xffffffffu, n_exact);
  if (kCls) {
    hinge_neg = __reduce_add_sync(0xffffffffu, hinge_neg);
    correct_neg = __reduce_add_sync(0xffffffffu, correct_neg);
    if (lane == 0) {
      atomicAdd(&s_cnt[kCounters > 2 ? 2 : 0], (unsigned long long)hinge_neg);
      atomicAdd(&s_cnt[kCounters > 3 ? 3 : 0], (unsigned long long)correct_neg);
    }
    if (kRows) {
      n_pos = __reduce_add_sync(0xffffffffu, n_pos);
      n_neg = __reduce_add_sync(0xffffffffu, n_neg);
      if (lane == 0) {
        atomicAdd(&s_cnt[kCounters - 2], (unsigned long long)n_pos);
        atomicAdd(&s_cnt[kCounters - 1], (unsigned long long)n_neg);
      }
    }
  }
  if (lane == 0) {
    atomicAdd(&s_cnt[0], (unsigned long long)hinge);
    atomicAdd(&s_cnt[1], (unsigned long long)correct);
    if (p.n_exact && n_exact) atomicAdd(p.n_exact, (unsigned long long)n_exact);
  }
  __syncthreads();
  if (kCls) {
    // s_cnt: hinge+, correct+, hinge-, correct-, rows+, rows-
    const int t = threadIdx.x;
    const int word = t < 4 ? ((t & 1) ? kCntClassCorrect : kCntClassHinge) + (t >> 1) : kCntClassN + (t - 4);
    if (t < kCounters && s_cnt[t]) atomicAdd(&p.cnt[word], s_cnt[t]);
    return;
  }
  if (threadIdx.x == 0) {
    if (s_cnt[0]) atomicAdd(&p.cnt[kCntHinge], s_cnt[0]);
    if (s_cnt[1]) atomicAdd(&p.cnt[kCntCorrect], s_cnt[1]);
  }
}

}  // namespace dsgd
