// dsgd_bootstrap.cuh -- sm_90a kernels of the bootstrap calls (dsgd_eval_*bootstrap; DESIGN.md §4.19) and of the weighted
// bootstrap calls (dsgd_eval_*weighted_bootstrap; §4.20, at the end of this file).
//
// Replicate b of a request of n rows is the unweighted evaluation of its expanded list: position i repeated m_i(b) times,
// m_i(b) the Poisson(1) draw of dsgd_bootstrap.h.  Scoring and sorting do not depend on b, so a bootstrap pass does them once:
//   1. k_boot_score: the score of every position, taken by warp_scores as every scoring pass takes it (the same fold,
//      the same intercept), its sort key ~score_key(s) (s = -(x . w): highest score first; a NaN score takes the largest
//      key, ~0, and sorts last) and a 32-bit tag: the position, its confusion word (kMetTp .. kMetNegNone), its SVM hinge
//      1 - y p in {0, 1, 2} and a NaN bit.  Every model but the SVM also keeps the row's loss L (row_loss), by position.
//   2. cub::DeviceRadixSort::SortPairs of (key, tag) over all n positions.
//   3. k_boot_arrange: in sorted order, the last element of every tie group of non-NaN scores records the index of its
//      group's first element (-1 elsewhere), and L is gathered into sorted order.
//   4. k_boot_rep: one CTA per replicate, tile by tile over the sorted elements.  Each element draws its m from its position;
//      a block scan carries the (positive, negative) mass, packed as P << 32 | N, above and through every element.  At the end
//      of a group, with A the mass above it and E the mass through it (P_g = E.P - A.P, N_g = E.N - A.N):
//        U2 += N_g (2 A.P + P_g)               -- 2 per (positive above, negative) pair, 1 per tied pair
//        S  += P_g R(E.P / (E.P + E.N))        -- when P_g > 0: the precision at the group's score, once per positive copy
//      and every element adds m to its confusion word, its NaN word and the replicate's size, and m copies of its loss.
// Every sum is an integer or an order-free fixed-point sum (dsgd_fixed.cuh): a replicate has the same bits on any grid, and
// they are those of dsgd_eval_samples_metrics / _curve / _sums over the expanded list (tests/test_gpu_bootstrap.py).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/block/block_scan.cuh>

#include "dsgd_bootstrap.h"
#include "dsgd_kernels.cuh"
#include "dsgd_metrics.cuh"

namespace dsgd {

constexpr int64_t kBootMaxRows = 1ll << 26;   // with m <= 20: sum m < 2^31 and U2 < 2^61, every word an exact int64
constexpr uint32_t kBootPosMask = (1u << 26) - 1u;
constexpr int kBootThreads = 256, kBootItems = 4, kBootTile = kBootThreads * kBootItems;
// a replicate's output: the DSGD_BOOTSTRAP_WORDS words, then S (the AP sum) and the loss sum as the bits of doubles
enum BootWord : int { kBootSize = 8, kBootS = 9, kBootLoss = 10, kBootOutWords = 11 };
static_assert(kMetTp == 0 && kMetNegNone == 5 && kMetU2 == 6 && kMetNan == 7, "a tag's confusion word is a word index");

// ---------------------------------------------------------------------------------------------------
// k_boot_score: the positions taken by warp_scores; every position's key and tag go to its own slot, and (kModel != kSvm)
// loss[i] = L(y (x . w)), the per-row loss of k_rows.
// ---------------------------------------------------------------------------------------------------
template <int kModel, bool kIcpt>
__global__ void __launch_bounds__(256) k_boot_score(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                    const int8_t *__restrict__ label, const int32_t *__restrict__ samples,
                                                    int64_t row_begin, int64_t n, const double *__restrict__ w,
                                                    unsigned long long *__restrict__ keys, uint32_t *__restrict__ tags,
                                                    double *__restrict__ loss, const double *__restrict__ icpt) {
  warp_scores<kIcpt>(rp16, pairs, samples, row_begin, n, w, icpt, [&](int64_t i, int64_t r, double dot, bool mine) {
    if (!mine) return;
    const int y = (int)label[r];
    const bool pos = y > 0, nan = isnan(dot);
    const int p = pred_of(dot);
    const uint32_t word = pos ? (p == 1 ? kMetTp : p == -1 ? kMetFn : kMetPosNone) : (p == 1 ? kMetFp : p == -1 ? kMetTn : kMetNegNone);
    keys[i] = nan ? ~0ull : ~score_key(-dot);
    tags[i] = (uint32_t)i | word << 26 | (uint32_t)(1 - y * p) << 29 | (uint32_t)nan << 31;
    if constexpr (kModel != kSvm) loss[i] = row_loss<kModel>((double)y * dot);
  });
}

// k_boot_arrange: gs[j] = the first index of element j's tie group when j ends a group of non-NaN scores, else -1; kLoss:
// eloss[j] = loss of element j's position
template <bool kLoss>
__global__ void __launch_bounds__(256) k_boot_arrange(const unsigned long long *__restrict__ keys,
                                                      const uint32_t *__restrict__ tags, int64_t n,
                                                      const double *__restrict__ loss, int *__restrict__ gs,
                                                      double *__restrict__ eloss) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = keys[j];
    const bool end = key != ~0ull && (j + 1 == n || keys[j + 1] != key);
    gs[j] = end ? (int)key_lower_bound(keys, j + 1, key) : -1;
    if constexpr (kLoss) eloss[j] = loss[tags[j] & kBootPosMask];
  }
}

// lim += m R(v) (v in [0, 2^52), not NaN), carried: limbs 0..3 of R(v) are below 2^40 + 1, so each product is split at bit 40
// into its limb and the next.  Limb 4, R(v)'s integer part, is added whole: callers keep m v below 2^63 (v <= 1 for S, m <= 20
// for a loss).
__device__ __forceinline__ void acc_add_times(unsigned long long (&lim)[kLossLimbs], double v, unsigned long long m) {
  acc_cut(v, [&](int k, double limb) {
    const unsigned long long q = (unsigned long long)(long long)limb, lo = q * m;
    if (k == kLossLimbs - 2) {
      lim[k] += lo;
      return;
    }
    lim[k] += lo & kLimbMask;
    lim[k + 1] += (lo >> 40) | (__umul64hi(q, m) << 24);
  });
  acc_carry(lim);
}

// ---------------------------------------------------------------------------------------------------
// k_boot_rep: replicate b0 + blockIdx.x over the n sorted elements; out[kBootOutWords * blockIdx.x ..] its words.  Thread t
// takes elements 4 t .. 4 t + 3 of each 1024-element tile; incl[] holds the tile's inclusive masses, and a_open the mass
// through the last group end of the tiles before, which is the mass above any group that began before this tile.
// ---------------------------------------------------------------------------------------------------
template <bool kLoss>
__global__ void __launch_bounds__(kBootThreads) k_boot_rep(const uint32_t *__restrict__ tags, const int *__restrict__ gs,
                                                           const double *__restrict__ eloss, int64_t n, uint64_t bkey,
                                                           int64_t b0, unsigned long long *__restrict__ out) {
  using Scan = cub::BlockScan<unsigned long long, kBootThreads>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ unsigned long long incl[kBootTile];
  __shared__ long long last_end;
  __shared__ unsigned long long red[kBootThreads / 32][24];
  const uint64_t zb = dsgd_boot_stream(bkey, (uint64_t)(b0 + blockIdx.x));
  const unsigned long long lo32 = 0xffffffffull;
  unsigned c[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // the six confusion words, then NaN and size
  unsigned long long u2 = 0, hinge = 0, carry = 0, a_open = 0;
  unsigned long long lim_s[kLossLimbs] = {0, 0, 0, 0, 0, 0}, lim_l[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_l = 0;
  for (int64_t t0 = 0; t0 < n; t0 += kBootTile) {
    const int base = threadIdx.x * kBootItems;
    uint32_t tag[kBootItems];
    int g[kBootItems];
    unsigned m[kBootItems];
    unsigned long long pn[kBootItems], sum = 0;
#pragma unroll
    for (int k = 0; k < kBootItems; ++k) {
      const int64_t j = t0 + base + k;
      tag[k] = j < n ? tags[j] : 0u;
      g[k] = j < n ? gs[j] : -1;
      m[k] = j < n ? (unsigned)dsgd_boot_m(zb, tag[k] & kBootPosMask) : 0u;
      pn[k] = ((tag[k] >> 26) & 7u) < 3u ? (unsigned long long)m[k] << 32 : (unsigned long long)m[k];
      sum += pn[k];
    }
    if (threadIdx.x == 0) last_end = -1;
    unsigned long long excl, total;
    Scan(scan_tmp).ExclusiveSum(sum, excl, total);
    unsigned long long run = carry + excl;
#pragma unroll
    for (int k = 0; k < kBootItems; ++k) {
      run += pn[k];
      incl[base + k] = run;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kBootItems; ++k) {
      if (m[k]) {
        c[(tag[k] >> 26) & 7u] += m[k];
        c[6] += (tag[k] >> 31) * m[k];
        c[7] += m[k];
        if constexpr (kLoss) {
          const double l = eloss[t0 + base + k];
          if (!(l >= 0.0 && l < 4503599627370496.0)) ovf_l += m[k];   // NaN, inf, >= 2^52: the sum reads NaN
          else acc_add_times(lim_l, l, m[k]);
        } else {
          hinge += (unsigned long long)((tag[k] >> 29) & 3u) * m[k];
        }
      }
      if (g[k] >= 0) {
        const unsigned long long E = incl[base + k];
        const unsigned long long A = g[k] > t0 ? incl[g[k] - 1 - t0] : a_open;
        const unsigned long long Pa = A >> 32, Pt = E >> 32, Nt = E & lo32;
        const unsigned long long Pg = Pt - Pa, Ng = Nt - (A & lo32);
        u2 += Ng * (2 * Pa + Pg);
        if (Pg) acc_add_times(lim_s, (double)Pt / (double)(Pt + Nt), Pg);
        atomicMax(&last_end, (long long)(t0 + base + k));
      }
    }
    __syncthreads();
    if (last_end >= 0) a_open = incl[last_end - t0];
    carry += total;
    __syncthreads();
  }
  // block sums: 8 counts, U2, the hinge sum, S's and the loss's limbs and the loss's overflow count
  unsigned long long v[24];
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = c[k];
  v[8] = u2;
  v[9] = hinge;
#pragma unroll
  for (int k = 0; k < kLossLimbs; ++k) {
    v[10 + k] = lim_s[k];
    v[16 + k] = lim_l[k];
  }
  v[22] = ovf_l;
  v[23] = 0;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 23; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (lane == 0) red[wid][k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t[24];
    for (int k = 0; k < 23; ++k) {
      t[k] = 0;
      for (int q = 0; q < kBootThreads / 32; ++q) t[k] += red[q][k];
    }
    unsigned long long *o = out + (int64_t)kBootOutWords * blockIdx.x;
    for (int k = 0; k < 6; ++k) o[k] = t[k];
    o[kMetU2] = t[8];
    o[kMetNan] = t[6];
    o[kBootSize] = t[7];
    unsigned long long s[kLossAccWords], l[kLossAccWords];
    for (int k = 0; k < kLossLimbs; ++k) {
      s[k] = t[10 + k];
      l[k] = t[16 + k];
    }
    s[kLossLimbs] = 0;
    l[kLossLimbs] = t[22];
    o[kBootS] = (unsigned long long)__double_as_longlong(acc_value(s));
    o[kBootLoss] = (unsigned long long)__double_as_longlong(kLoss ? acc_value(l) : (double)t[9]);
  }
}

// ---------------------------------------------------------------------------------------------------
// The weighted bootstrap (dsgd_eval_*weighted_bootstrap; DESIGN.md §4.20).  Replicate b is the weighted curve and the weighted
// evaluation of the expanded list, every copy of row i weighing c_i = fl(w_y s_i).  Every weighted word is read() of an exact
// sum and m copies of a term add exactly m R(term), so the pass scores and sorts as the unweighted one does (k_boot_score,
// one SortPairs) and then:
//   3. k_wboot_arrange: in sorted order, each element's tie group [gf, gl] (-1 for a NaN score), its c and fl(c L).
//   4. k_wboot_rep: one CTA per replicate.  Sweep 1, order-free: the size, the NaN rows, the loss limbs and W-, the weight
//      of the non-NaN negatives.  Sweep 2, highest score first, one element per thread and tile: a block scan of the
//      (positive, negative) masses sum m R(c) as limb_sums.  A group's end, with E the mass through it and A- the negative
//      mass above it, forms T = read(E+), F = read(E-) and B = read(2 (W- - E-) + (E- - A-)) = read(2 W-(< s) + W-(= s)); every
//      non-NaN positive copy of the group then adds R(fl(c B)) to U2w and, when c > 0, R(fl(c fl(T / (T + F)))) to S_ap --
//      k_curve_count<kSampleWeighted>'s expressions.  A group that began in an earlier tile is re-walked from its first
//      element when it ends (at most one per tile, so at most 2 n element visits); m is a pure function of the position.
//      The confusion, NaN and class weights are the scan's values at the first s <= 0, s < 0 and NaN elements and at n.
// ---------------------------------------------------------------------------------------------------
constexpr int kWbThreads = 256;
// a replicate's output: sum m, the NaN-score rows, the DSGD_WCURVE_WORDS words and the loss sum S as the bits of doubles
enum WBootWord : int { kWbSize = 0, kWbNan = 1, kWbSums = 2, kWbLoss = kWbSums + 13, kWbOutWords = 16 };

// k_wboot_arrange: gf[j] / gl[j] the first / last index of element j's tie group (-1: a NaN score), ec[j] = c of its row
// (row_weight) and ecl[j] = fl(c L), the term of
// k_rows<..., kSampleWeighted, ...>: L the loss by position (kLoss) or the SVM's hinge 1 - y p from the tag.
template <bool kLoss>
__global__ void __launch_bounds__(256) k_wboot_arrange(const unsigned long long *__restrict__ keys,
                                                       const uint32_t *__restrict__ tags, int64_t n,
                                                       const int32_t *__restrict__ samples, int64_t row_begin, double w_pos,
                                                       double w_neg, const double *__restrict__ sw,
                                                       const double *__restrict__ loss, int *__restrict__ gf,
                                                       int *__restrict__ gl, double *__restrict__ ec,
                                                       double *__restrict__ ecl) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = keys[j];
    const uint32_t tag = tags[j];
    const bool nan = key == ~0ull;
    gf[j] = nan ? -1 : (int)key_lower_bound(keys, j + 1, key);
    gl[j] = nan ? -1 : (int)(j + key_lower_bound(keys + j, n - j, key + 1) - 1);
    const int64_t p = tag & kBootPosMask, r = samples ? (int64_t)samples[p] : row_begin + p;
    const bool pos = ((tag >> 26) & 7u) < 3u;
    const double ci = row_weight(pos, w_pos, w_neg, sw, r);
    const double l = kLoss ? loss[p] : (double)((tag >> 29) & 3u);
    ec[j] = ci;
    ecl[j] = ci * l;
  }
}

// the (positive, negative) masses of the scan
struct limb_pair {
  limb_sum p, n;
};
struct limb_pair_plus {
  __device__ __forceinline__ limb_pair operator()(const limb_pair &a, const limb_pair &b) const {
    return limb_pair{limb_plus()(a.p, b.p), limb_plus()(a.n, b.n)};
  }
};
// m R(v) as a limb_sum, v outside [0, 2^52) counted m times as an overflow
__device__ __forceinline__ limb_sum limb_times(double v, unsigned m) {
  limb_sum s = {{0, 0, 0, 0, 0, 0}, 0};
  if (!(v >= 0.0 && v < 4503599627370496.0)) s.ovf = m;
  else if (m) acc_add_times(s.l, v, m);
  return s;
}
// lim += m R(v), ovf += m when v is outside [0, 2^52)
__device__ __forceinline__ void acc_add_local_times(unsigned long long (&lim)[kLossLimbs], unsigned long long &ovf, double v,
                                                    unsigned m) {
  if (!(v >= 0.0 && v < 4503599627370496.0)) ovf += m;
  else acc_add_times(lim, v, m);
}
// The sum of v over the CTA into thread 0's v (the others' v are partial); red: kWbThreads / 32 rows of K words
template <int K>
__device__ __forceinline__ void wb_block_sum(unsigned long long (&v)[K], unsigned long long (*red)[K]) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (lane == 0) red[wid][k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      v[k] = 0;
      for (int q = 0; q < kWbThreads / 32; ++q) v[k] += red[q][k];
    }
  }
  __syncthreads();
}
// the group-end values a positive's terms need
struct wb_group {
  double t, f, b;
};

// ---------------------------------------------------------------------------------------------------
// k_wboot_rep: replicate b0 + blockIdx.x over the n sorted elements (keys: the sorted keys); out[kWbOutWords * blockIdx.x ..]
// its words.  Thread t takes element t0 + t of each tile.  Two CTAs per SM (at most 128 registers, a few hundred bytes
// spilled): at 1 000 replicates 17 % faster than one CTA at 255 registers (DESIGN.md §4.20).
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kWbThreads, 2) k_wboot_rep(const unsigned long long *__restrict__ keys,
                                                           const uint32_t *__restrict__ tags, const int *__restrict__ gf,
                                                           const int *__restrict__ gl, const double *__restrict__ ec,
                                                           const double *__restrict__ ecl, int64_t n, uint64_t bkey,
                                                           int64_t b0, unsigned long long *__restrict__ out) {
  using Scan = cub::BlockScan<limb_pair, kWbThreads, cub::BLOCK_SCAN_WARP_SCANS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ limb_pair carry;               // the masses of the tiles before
  __shared__ limb_sum a_neg[kWbThreads];   // at a group's first element: the negative mass above the group
  __shared__ wb_group grp[kWbThreads];      // at a group's last element: its T, F and B
  __shared__ limb_pair bnd[3];              // the masses above the first s <= 0, s < 0 and NaN elements
  __shared__ limb_sum w_neg, a_open;        // W-; the negative mass above the group open at the tile's start
  __shared__ wb_group rw;                   // the group that ends in this tile and began before it
  __shared__ int64_t edge[3];
  __shared__ unsigned long long red[kWbThreads / 32][kLossAccWords * 2 + 2];
  const uint64_t zb = dsgd_boot_stream(bkey, (uint64_t)(b0 + blockIdx.x));
  const limb_sum zero = {{0, 0, 0, 0, 0, 0}, 0};
  if (threadIdx.x == 0) {
    const unsigned long long k0 = ~score_key(0.0);   // s > 0 sorts before k0, s < 0 after it, NaN (~0) last
    edge[0] = key_lower_bound(keys, n, k0);
    edge[1] = key_lower_bound(keys, n, k0 + 1);
    edge[2] = key_lower_bound(keys, n, ~0ull);
    for (int k = 0; k < 3; ++k) bnd[k] = limb_pair{zero, zero};
    a_open = zero;
    carry = limb_pair{zero, zero};
  }
  // sweep 1: the size, the NaN rows, the loss limbs and W-
  {
    unsigned long long size = 0, nan_rows = 0, lim_l[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_l = 0;
    unsigned long long lim_w[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_w = 0;
    for (int64_t j = threadIdx.x; j < n; j += kWbThreads) {
      const uint32_t tag = tags[j];
      const unsigned m = (unsigned)dsgd_boot_m(zb, tag & kBootPosMask);
      if (!m) continue;
      size += m;
      nan_rows += (tag >> 31) * m;
      acc_add_local_times(lim_l, ovf_l, ecl[j], m);
      if (!(tag >> 31) && ((tag >> 26) & 7u) >= 3u) acc_add_local_times(lim_w, ovf_w, ec[j], m);
    }
    unsigned long long v[kLossAccWords * 2 + 2];
#pragma unroll
    for (int k = 0; k < kLossLimbs; ++k) {
      v[k] = lim_l[k];
      v[kLossAccWords + k] = lim_w[k];
    }
    v[kLossLimbs] = ovf_l;
    v[kLossAccWords + kLossLimbs] = ovf_w;
    v[2 * kLossAccWords] = size;
    v[2 * kLossAccWords + 1] = nan_rows;
    wb_block_sum(v, red);
    if (threadIdx.x == 0) {
      unsigned long long *o = out + (int64_t)kWbOutWords * blockIdx.x;
      o[kWbSize] = v[2 * kLossAccWords];
      o[kWbNan] = v[2 * kLossAccWords + 1];
      o[kWbLoss] = (unsigned long long)__double_as_longlong(acc_value(&v[0]));
      limb_sum wn = limb_load(&v[kLossAccWords]);
      acc_carry(wn.l);
      w_neg = wn;
    }
    __syncthreads();
  }
  // sweep 2
  unsigned long long lim_u[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_u = 0, lim_s[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_s = 0;
  const int64_t e0 = edge[0], e1 = edge[1], e2 = edge[2];
  for (int64_t t0 = 0; t0 < n; t0 += kWbThreads) {
    const int64_t j = t0 + threadIdx.x;
    const bool in = j < n;
    const uint32_t tag = in ? tags[j] : 0u;
    const unsigned m = in ? (unsigned)dsgd_boot_m(zb, tag & kBootPosMask) : 0u;
    const bool pos = ((tag >> 26) & 7u) < 3u, nan = (tag >> 31) != 0u;
    const double c = in ? ec[j] : 0.0;
    const int g0 = in ? gf[j] : -1, g1 = in ? gl[j] : -1;
    const limb_sum x = limb_times(c, m);
    limb_pair excl, agg;
    Scan(scan_tmp).ExclusiveScan(limb_pair{pos ? x : zero, pos ? zero : x}, excl, limb_pair{zero, zero}, limb_pair_plus(),
                                 agg);
    excl = limb_pair_plus()(carry, excl);
    if (in) {
      if (g0 == j) a_neg[threadIdx.x] = excl.n;
      if (j + 1 == e0) bnd[0] = limb_pair_plus()(excl, limb_pair{pos ? x : zero, pos ? zero : x});
      if (j + 1 == e1) bnd[1] = limb_pair_plus()(excl, limb_pair{pos ? x : zero, pos ? zero : x});
      if (j + 1 == e2) bnd[2] = limb_pair_plus()(excl, limb_pair{pos ? x : zero, pos ? zero : x});
    }
    __syncthreads();
    if (threadIdx.x == 0) carry = limb_pair_plus()(carry, agg);   // every thread has read it above
    if (in && g1 == j) {   // a group's end: its T, F and B
      const limb_pair e = limb_pair_plus()(excl, limb_pair{pos ? x : zero, pos ? zero : x});
      const limb_sum an = g0 >= t0 ? a_neg[g0 - t0] : a_open;
      limb_sum bs;
#pragma unroll
      for (int k = 0; k < kLossLimbs; ++k) bs.l[k] = 2 * w_neg.l[k] - e.n.l[k] - an.l[k];
      bs.ovf = 2 * w_neg.ovf - e.n.ovf - an.ovf;
      const wb_group gv{limb_read(e.p), limb_read(e.n), limb_read(bs)};
      grp[threadIdx.x] = gv;
      if (g0 < t0) rw = gv;
    }
    __syncthreads();
    const int64_t t1 = t0 + kWbThreads;
    if (in && pos && !nan && m && g1 < t1) {
      const wb_group gv = grp[g1 - t0];
      acc_add_local_times(lim_u, ovf_u, c * gv.b, m);
      if (c > 0.0) acc_add_local_times(lim_s, ovf_s, c * (gv.t / (gv.t + gv.f)), m);
    }
    // the group that ends here and began before this tile: its elements of the earlier tiles
    const int64_t first = (t0 > 0 && gl[t0 - 1] >= t0 && gl[t0 - 1] < t1) ? gf[t0 - 1] : t0;
    if (first < t0) {
      const wb_group gv = rw;
      for (int64_t k = first + threadIdx.x; k < t0; k += kWbThreads) {
        const uint32_t tk = tags[k];
        if (((tk >> 26) & 7u) >= 3u) continue;
        const unsigned mk = (unsigned)dsgd_boot_m(zb, tk & kBootPosMask);
        if (!mk) continue;
        const double ck = ec[k];
        acc_add_local_times(lim_u, ovf_u, ck * gv.b, mk);
        if (ck > 0.0) acc_add_local_times(lim_s, ovf_s, ck * (gv.t / (gv.t + gv.f)), mk);
      }
    }
    // the negative mass above the group still open at the tile's end
    if (threadIdx.x == kWbThreads - 1 && in && g1 >= t1) a_open = g0 >= t0 ? a_neg[g0 - t0] : a_open;
    __syncthreads();
  }
  // block sums of U2w's and S_ap's limbs
  unsigned long long v[kLossAccWords * 2 + 2] = {};
#pragma unroll
  for (int k = 0; k < kLossLimbs; ++k) {
    v[k] = lim_u[k];
    v[kLossAccWords + k] = lim_s[k];
  }
  v[kLossLimbs] = ovf_u;
  v[kLossAccWords + kLossLimbs] = ovf_s;
  wb_block_sum(v, red);
  if (threadIdx.x == 0) {
    // the masses at the three edges and at n: tp = P(e0), fn = P(e2) - P(e1), no prediction = P(e1) - P(e0) + P(n) - P(e2)
    const limb_pair p0 = bnd[0], p1 = bnd[1], p2 = bnd[2], pn = carry;
    const limb_sum p_nan = limb_add(pn.p, p2.p, true), n_nan = limb_add(pn.n, p2.n, true);
    const limb_sum tp = p0.p, tn = limb_add(p2.n, p1.n, true);
    const double w[13] = {limb_read(tp), limb_read(limb_add(p2.p, p1.p, true)),
                          limb_read(limb_add(limb_add(p1.p, p0.p, true), p_nan)), limb_read(p0.n), limb_read(tn),
                          limb_read(limb_add(limb_add(p1.n, p0.n, true), n_nan)), limb_read(limb_load(&v[0])),
                          limb_read(limb_add(p_nan, n_nan)), limb_read(limb_load(&v[kLossAccWords])),
                          limb_read(limb_add(tp, tn)), limb_read(limb_add(pn.p, pn.n)), limb_read(pn.p), limb_read(pn.n)};
    unsigned long long *o = out + (int64_t)kWbOutWords * blockIdx.x;
#pragma unroll
    for (int k = 0; k < 13; ++k) o[kWbSums + k] = (unsigned long long)__double_as_longlong(w[k]);
  }
}

}  // namespace dsgd
