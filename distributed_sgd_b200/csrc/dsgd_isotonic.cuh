// dsgd_isotonic.cuh -- sm_90a kernels of the isotonic calibration calls (dsgd_calibrate_isotonic*,
// dsgd_isotonic_probabilities, dsgd_eval_isotonic_calibration*; DESIGN.md §4.16).
//
// Isotonic regression of 0/1 labels on the score s = -x . w is the upper concave hull of the curve's points: with the m
// distinct scores t_0 > t_1 > ... > t_(m-1) that a curve pass leaves in c_thr, and tp_k / fp_k the rows with s >= t_k, the
// points are P_-1 = (0, 0) and P_k = (n_k, tp_k), n_k = tp_k + fp_k.  Here point i of the hull kernels is P_(i-1): point 0 is
// the origin.  Every coordinate is an integer below 2^31, so the turn test is an int64 cross product and exact, and the hull
// (vertices strictly above the chord of their neighbours) is one set whatever the algorithm that builds it.  The fit:
//   1. k_iso_tile: each CTA takes a tile of S consecutive points into shared memory and its thread 0 runs the monotone chain.
//   2. ceil(log2 tiles) rounds of k_iso_merge: each CTA merges two adjacent hulls -- the bridge (upper common tangent) by a
//      binary search over the left hull with a binary search over the right one inside it, then the surviving vertices
//      compacted into the other of two ping-pong buffers.
//   3. an exclusive scan of every block's X count (1 or 2) and k_iso_emit: X, Y and the block counts, ascending in s.
// The three hull kernels are templates over a point set: k_iso_tile<P>, k_iso_merge<P> and k_iso_emit<P> with P = IsoCounts
// here, or IsoWeights for the weighted fit (DESIGN.md §4.17).  k_iso_prob<kSmem> applies a map (X, Y) to rows as
// numpy.interp does, and k_calib_eval<kIso, kSmem> is the quality pass at a sigmoid or at a map.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dsgd_calibrate.cuh"
#include "dsgd_metrics.cuh"

namespace dsgd {

constexpr int kIsoTileMax = 2048;    // points of a tile in shared memory: 16 bytes of coordinates and 4 of stack each (40 KB)
constexpr int kIsoThreads = 256;
constexpr int kIsoSmemPoints = 6144; // (X, Y) pairs k_iso_prob / k_calib_eval keep in shared memory (96 KB); more stay in L2

// ---- point sets ----------------------------------------------------------------------------------------------------
// The hull kernels are templates over a point set P: IsoCounts here (the fit over counted rows) or IsoWeights below (the
// fit over weighted rows).  A kernel takes P's two arrays and P gives
//   point(i, x, y): the coordinates of point i (point 0 is the origin), of type P::Coord;
//   P::Ref: how the hull passes a coordinate it already holds (an int64 by value, a u256 by reference: a copy spills);
//   turn(o, a, b): a value > 0 when b lies strictly above the line from o through a, 0 when the three are collinear and
//   < 0 below, for o before a and b along the curve;
//   above(v, u, r): a value > 0 when u lies strictly above the line from v through r, for v before u and r (the bridge's
//   test: the sign of (r - v) x (u - v));
//   block(x0, y0, x1, y1, rows, pos): the values k_iso_emit writes for the hull segment from (x0, y0) to (x1, y1), of type
//   P::Block, and it returns the segment's probability p.

// Point i: the origin, or (tp + fp, tp) of curve point i - 1.  A block's values are its rows and positives,
// p = fl(pos / rows).
struct IsoCounts {
  using Coord = long long;
  using Ref = long long;
  using Block = long long;
  const long long *__restrict__ tp, *__restrict__ fp;
  __device__ __forceinline__ void point(int i, long long &x, long long &y) const {
    if (i == 0) { x = 0; y = 0; return; }
    y = tp[i - 1];
    x = y + fp[i - 1];
  }
  // (a - o) x (b - o).  Every coordinate is below 2^31, so each product is below 2^62 and the difference is exact.
  __device__ __forceinline__ static long long turn(Ref ox, Ref oy, Ref ax, Ref ay, Ref bx, Ref by) {
    return (ax - ox) * (by - oy) - (ay - oy) * (bx - ox);
  }
  __device__ __forceinline__ static long long above(Ref vx, Ref vy, Ref ux, Ref uy, Ref rx, Ref ry) {
    return turn(vx, vy, rx, ry, ux, uy);   // (r - v) x (u - v)
  }
  __device__ __forceinline__ static double block(Ref x0, Ref y0, Ref x1, Ref y1, Block &rows, Block &pos) {
    rows = x1 - x0;
    pos = y1 - y0;
    return (double)pos / (double)rows;
  }
};

// ---- the hull ------------------------------------------------------------------------------------------------------
// Every hull kernel takes the point set's two arrays (c0, c1): (tp, fp) of IsoCounts or (qx, qy) of IsoWeights.
// Tile t of S points [t S, min(M, (t + 1) S)): its upper hull by the monotone chain (a point is popped when it lies on or
// below the chord of its neighbours), vertex indices into hv[t S ..) and their count into hc[t].  Grid-stride over tiles.
// Shared memory: S (2 sizeof(P::Coord) + 4) bytes.
template <class P>
__global__ void __launch_bounds__(kIsoThreads) k_iso_tile(const typename P::Coord *__restrict__ c0,
                                                          const typename P::Coord *__restrict__ c1, int M, int S,
                                                          int *__restrict__ hv, int *__restrict__ hc) {
  using Coord = typename P::Coord;
  const P pts{c0, c1};
  extern __shared__ __align__(16) unsigned char iso_smem[];
  Coord *sx = reinterpret_cast<Coord *>(iso_smem), *sy = sx + S;
  int *st = reinterpret_cast<int *>(sy + S);
  __shared__ int s_top;
  const int T = (M + S - 1) / S;
  for (int t = blockIdx.x; t < T; t += gridDim.x) {
    const int b = t * S, len = min(S, M - b);
    for (int j = threadIdx.x; j < len; j += blockDim.x) pts.point(b + j, sx[j], sy[j]);
    __syncthreads();
    if (threadIdx.x == 0) {
      int top = 0;
      for (int j = 0; j < len; ++j) {
        typename P::Ref x = sx[j], y = sy[j];
        while (top >= 2 && P::turn(sx[st[top - 2]], sy[st[top - 2]], sx[st[top - 1]], sy[st[top - 1]], x, y) >= 0) --top;
        st[top++] = j;
      }
      s_top = top;
      hc[t] = top;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < s_top; j += blockDim.x) hv[b + j] = b + st[j];
    __syncthreads();
  }
}

// One merge round over hulls of width W points (hull g at hv_in[g W ..), hc_in[g] vertices): pair p merges hulls 2p and
// 2p + 1 into hull p of width 2W at hv_out[2p W ..); an odd last hull is copied.  L = l_0 .. l_(a-1), R = r_0 .. r_(b-1),
// every x of L below every x of R, each strictly concave.  j(v), the tangent point from a vertex v of L on R: the first j
// with r_(j+1) strictly below the line v -> r_j (the last of two collinear tangent points).  The bridge's left end: the
// first i with l_(i+1) not strictly above the line l_i -> r_(j(l_i)), which holds for every i after it and for none before
// it; the merged hull is l_0 .. l_i, r_(j(l_i)) .. r_(b-1).
template <class P>
__global__ void __launch_bounds__(kIsoThreads) k_iso_merge(const typename P::Coord *__restrict__ c0,
                                                           const typename P::Coord *__restrict__ c1, int n_hulls, int W,
                                                           const int *__restrict__ hv_in, const int *__restrict__ hc_in,
                                                           int *__restrict__ hv_out, int *__restrict__ hc_out) {
  using Coord = typename P::Coord;
  const P pts{c0, c1};
  __shared__ int s_br[2];
  const int pairs = (n_hulls + 1) / 2;
  for (int p = blockIdx.x; p < pairs; p += gridDim.x) {
    const int *L = hv_in + (int64_t)2 * p * W;
    const int a = hc_in[2 * p];
    const bool single = 2 * p + 1 >= n_hulls;
    const int *R = L + W;
    const int b = single ? 0 : hc_in[2 * p + 1];
    if (threadIdx.x == 0) {
      int i_end = a - 1, j_end = 0;
      if (!single) {
        auto tangent = [&](typename P::Ref vx, typename P::Ref vy) {
          int lo = 0, hi = b - 1;
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            Coord x0, y0, x1, y1;
            pts.point(R[mid], x0, y0);
            pts.point(R[mid + 1], x1, y1);
            if (P::turn(vx, vy, x0, y0, x1, y1) >= 0) lo = mid + 1; else hi = mid;
          }
          return lo;
        };
        int lo = 0, hi = a - 1;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          Coord vx, vy, ux, uy, rx, ry;
          pts.point(L[mid], vx, vy);
          pts.point(L[mid + 1], ux, uy);
          pts.point(R[tangent(vx, vy)], rx, ry);
          if (P::above(vx, vy, ux, uy, rx, ry) > 0) lo = mid + 1; else hi = mid;
        }
        Coord vx, vy;
        pts.point(L[lo], vx, vy);
        i_end = lo;
        j_end = tangent(vx, vy);
      }
      s_br[0] = i_end;
      s_br[1] = j_end;
      hc_out[p] = i_end + 1 + (single ? 0 : b - j_end);
    }
    __syncthreads();
    const int i_end = s_br[0], j_end = s_br[1];
    int *out = hv_out + (int64_t)2 * p * W;
    for (int k = threadIdx.x; k <= i_end; k += blockDim.x) out[k] = L[k];
    if (!single)
      for (int k = threadIdx.x; k < b - j_end; k += blockDim.x) out[i_end + 1 + k] = R[j_end + k];
    __syncthreads();
  }
}

// X entries of block o (ascending score) of the final hull h_0 .. h_B: 2 when it spans two or more distinct scores, else 1
struct iso_x_count {
  const int *h;
  int B;
  __device__ __forceinline__ int operator()(int o) const {
    const int b = B - 1 - o;
    return 1 + (h[b + 1] - h[b] >= 2);
  }
};

// Block o (ascending score) is hull segment b = B - 1 - o, from vertex h_b to h_(b+1): points h_b .. h_(b+1) - 1 of thr, its
// highest score thr[h_b] and its lowest thr[h_(b+1) - 1]; P::block gives its p and the values blk_rows[o] and blk_pos[o].
// excl: the exclusive scan of iso_x_count; the last block writes the number of X entries to *n_x.
template <class P>
__global__ void __launch_bounds__(256) k_iso_emit(const int *__restrict__ h, int B, const int *__restrict__ excl,
                                                  const double *__restrict__ thr, const typename P::Coord *__restrict__ c0,
                                                  const typename P::Coord *__restrict__ c1, double *__restrict__ X,
                                                  double *__restrict__ Y, typename P::Block *__restrict__ blk_rows,
                                                  typename P::Block *__restrict__ blk_pos,
                                                  unsigned long long *__restrict__ n_x) {
  const P pts{c0, c1};
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < B; o += gridDim.x * blockDim.x) {
    const int b = B - 1 - o, i0 = h[b], i1 = h[b + 1];
    typename P::Coord x0, y0, x1, y1;
    pts.point(i0, x0, y0);
    pts.point(i1, x1, y1);
    typename P::Block rows, pos;
    const double p = P::block(x0, y0, x1, y1, rows, pos);
    blk_rows[o] = rows;
    blk_pos[o] = pos;
    const int at = excl[o];
    const bool two = i1 - i0 >= 2;
    X[at] = thr[i1 - 1];
    Y[at] = p;
    if (two) {
      X[at + 1] = thr[i0];
      Y[at + 1] = p;
    }
    if (o == B - 1) *n_x = (unsigned long long)(at + 1 + two);
  }
}

// ---- applying a map ----------------------------------------------------------------------------------------------------
// numpy.interp(s, X, Y) for k >= 1 points, X strictly increasing: NaN for a NaN s, the end values outside [X_0, X_(k-1)],
// Y_j at s == X_j, and else slope (s - X_j) + Y_j with slope = (Y_(j+1) - Y_j) / (X_(j+1) - X_j), X_j <= s < X_(j+1); a NaN
// there retries from the right end, and a NaN again between equal Y gives Y_j.  No contraction (--fmad=false).
__device__ __forceinline__ double iso_interp(double s, const double *X, const double *Y, int k) {
  if (isnan(s)) return s;
  if (s <= X[0]) return Y[0];
  if (s >= X[k - 1]) return Y[k - 1];
  int lo = 0, hi = k - 1;   // X[lo] <= s < X[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (X[mid] <= s) lo = mid; else hi = mid;
  }
  if (X[lo] == s) return Y[lo];
  const double slope = (Y[lo + 1] - Y[lo]) / (X[lo + 1] - X[lo]);
  double v = slope * (s - X[lo]) + Y[lo];
  if (isnan(v)) {
    v = slope * (s - X[lo + 1]) + Y[lo + 1];
    if (isnan(v) && Y[lo] == Y[lo + 1]) v = Y[lo];
  }
  return v;
}

// The map in shared memory (kSmem: k <= kIsoSmemPoints) or read through L2
template <bool kSmem>
__device__ __forceinline__ void iso_stage(const double *__restrict__ X, const double *__restrict__ Y, int k,
                                          const double *&xs, const double *&ys) {
  if constexpr (kSmem) {
    extern __shared__ __align__(16) unsigned char iso_map[];
    double *sx = reinterpret_cast<double *>(iso_map), *sy = sx + k;
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
      sx[i] = X[i];
      sy[i] = Y[i];
    }
    __syncthreads();
    xs = sx;
    ys = sy;
  } else {
    xs = X;
    ys = Y;
  }
}

// out[i] = interp(-(x . w)) for row samples[i], x . w the row fold of dsgd_margins.  One warp per row.
template <bool kSmem, bool kIcpt>
__global__ void __launch_bounds__(256) k_iso_prob(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                  const int32_t *__restrict__ samples, int64_t n,
                                                  const double *__restrict__ w, const double *__restrict__ X,
                                                  const double *__restrict__ Y, int k, double *__restrict__ out,
                                                  const double *__restrict__ icpt) {
  const double *xs, *ys;
  iso_stage<kSmem>(X, Y, k, xs, ys);
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = warp0; i < n; i += nwarps) {
    const double dot = row_score<kIcpt>(rp16, pairs, w, (int64_t)samples[i], lane, icpt);
    if (lane == 0) out[i] = iso_interp(-dot, xs, ys, k);
  }
}

// ---- the quality pass (dsgd_eval_calibration*, dsgd_eval_isotonic_calibration*) --------------------------------------
// The quality pass over rows samples[0..n) (samples == nullptr: rows [row_begin, row_begin + n)) with n_bins equal-width
// bins into the CalibEvalWord block: bin = min(n_bins - 1, floor(p n_bins)).  At a sigmoid (kIso = false): z = a f + b,
// p = sigmoid(-z) and the log-loss term softplus(+-z); a NaN z leaves the row out.  At the map (X, Y) (kIso): p = interp(s),
// s = -f, and the term -log p (o = 1) or -log1p(-p) (o = 0); a NaN s leaves the row out, and a row whose term is infinite
// (p = 0 with o = 1, p = 1 with o = 0) is counted in kCevInf and adds nothing to the sum.  Positions are taken by
// warp_scores.  The two sums go to register limbs; the bins to shared memory: rows and positives as integers, sum p as
// limb words added with shared u64 atomics (p <= 1: each limb adds at most 2^40, so a CTA's words hold 2^24 rows without a
// wrap, and a grid of 8 CTAs per SM leaves a CTA fewer than that for any 32-bit row count).  The CTA propagates each bin's
// carries and adds its words to the block with REDs.
template <bool kIso, bool kSmem, bool kIcpt>
__global__ void __launch_bounds__(256) k_calib_eval(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                                    const int8_t *__restrict__ label, const int32_t *__restrict__ samples,
                                                    int64_t row_begin, int64_t n, const double *__restrict__ w, double a,
                                                    double b, const double *__restrict__ X, const double *__restrict__ Y,
                                                    int k, int n_bins, unsigned long long *__restrict__ blk,
                                                    const double *__restrict__ icpt) {
  __shared__ unsigned long long s_rows[kCalMaxBins], s_pos[kCalMaxBins], s_lim[kCalMaxBins][kLossLimbs];
  const double *xs, *ys;
  iso_stage<kSmem>(X, Y, k, xs, ys);
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kCalMaxBins; i += blockDim.x) {
    s_rows[i] = 0ull;
    s_pos[i] = 0ull;
#pragma unroll
    for (int q = 0; q < kLossLimbs; ++q) s_lim[i][q] = 0ull;
  }
  __syncthreads();
  unsigned long long lb[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ll[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_b = 0, ovf_l = 0;
  unsigned c_rows = 0, c_nan = 0, c_inf = 0;
  warp_scores<kIcpt>(rp16, pairs, samples, row_begin, n, w, icpt, [&](int64_t, int64_t r, double dot, bool mine) {
    if (!mine) return;
    const double z = kIso ? -dot : a * dot + b;   // kIso: the score s
    if (isnan(z)) { ++c_nan; return; }
    const bool pos = label[r] > 0;
    const double pr = kIso ? iso_interp(z, xs, ys, k) : sigmoid(-z), o = pos ? 1.0 : 0.0, dlt = pr - o;
    ++c_rows;
    acc_add_local(lb, ovf_b, dlt * dlt);
    const double term = kIso ? (pos ? -log(pr) : -log1p(-pr)) : softplus(pos ? z : -z);
    if (kIso && isinf(term)) ++c_inf;
    else acc_add_local(ll, ovf_l, term);
    int bin = (int)floor(pr * (double)n_bins);
    bin = bin < n_bins - 1 ? bin : n_bins - 1;
    atomicAdd(&s_rows[bin], 1ull);
    if (pos) atomicAdd(&s_pos[bin], 1ull);
    acc_cut(pr, [&](int q, double limb) {
      if (limb != 0.0) atomicAdd(&s_lim[bin][q], (unsigned long long)(long long)limb);
    });
  });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ovf_b += __shfl_xor_sync(full, ovf_b, o);
    ovf_l += __shfl_xor_sync(full, ovf_l, o);
#pragma unroll
    for (int q = 0; q < kLossLimbs; ++q) {
      lb[q] += __shfl_xor_sync(full, lb[q], o);
      ll[q] += __shfl_xor_sync(full, ll[q], o);
    }
  }
  c_rows = __reduce_add_sync(full, c_rows);
  c_nan = __reduce_add_sync(full, c_nan);
  if constexpr (kIso) c_inf = __reduce_add_sync(full, c_inf);
  if (lane == 0) {
    acc_flush_local(blk + kCevBrier, lb, ovf_b);
    acc_flush_local(blk + kCevLog, ll, ovf_l);
    if (c_rows) atomicAdd(&blk[kCevRows], (unsigned long long)c_rows);
    if (c_nan) atomicAdd(&blk[kCevNan], (unsigned long long)c_nan);
    if (kIso && c_inf) atomicAdd(&blk[kCevInf], (unsigned long long)c_inf);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_bins; i += blockDim.x) {
    if (!s_rows[i]) continue;
    red_add_u64(blk + kCevBinRows + i, s_rows[i]);
    if (s_pos[i]) red_add_u64(blk + kCevBinPos + i, s_pos[i]);
    unsigned long long q[kLossLimbs];
#pragma unroll
    for (int t = 0; t < kLossLimbs; ++t) q[t] = s_lim[i][t];
    acc_carry(q);
#pragma unroll
    for (int t = 0; t < kLossLimbs; ++t)
      if (q[t]) red_add_u64(blk + kCevBinLimbs + i * kLossLimbs + t, q[t]);
  }
}

// ---- the weighted fit (dsgd_calibrate_isotonic_weighted*; DESIGN.md §4.17) ----------------------------------------------
// A point's coordinates are the exact sums X = W(>= t) and Y = W+(>= t) of the weighted curve pass, integers in units of
// 2^-160 held in four u64 words (u256).  The hull needs them below 2^256, i.e. a total weight below 2^96; the host refuses
// more before the hull.  After the zero-weight points are dropped X strictly increases and Y does not decrease along the
// points, so every difference the turn test forms is >= 0 and the cross product is the comparison of two unsigned 512-bit
// products: exact.
struct u256 { unsigned long long w[4]; };
__device__ __forceinline__ u256 u256_sub(const u256 &a, const u256 &b) {   // a - b, a >= b
  u256 r;
  unsigned long long borrow = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const unsigned long long d = a.w[i] - b.w[i], d2 = d - borrow;
    borrow = (a.w[i] < b.w[i]) | (d < borrow);
    r.w[i] = d2;
  }
  return r;
}
__device__ __forceinline__ bool u256_eq(const u256 &a, const u256 &b) {
  return a.w[0] == b.w[0] && a.w[1] == b.w[1] && a.w[2] == b.w[2] && a.w[3] == b.w[3];
}
// a * b as eight words, least significant first
__device__ __forceinline__ void u256_mul(const u256 &a, const u256 &b, unsigned long long (&r)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) r[i] = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    unsigned long long carry = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned long long lo = a.w[i] * b.w[j], hi = __umul64hi(a.w[i], b.w[j]);
      const unsigned long long s1 = r[i + j] + lo, c1 = s1 < lo;
      const unsigned long long s2 = s1 + carry, c2 = s2 < carry;
      r[i + j] = s2;
      carry = hi + c1 + c2;   // below 2^64: hi <= 2^64 - 2
    }
    r[i + 4] = carry;
  }
}
// read() of an exact sum given as a u256 in units of 2^-160: its six 40-bit limbs converted as acc_value converts them
__device__ __forceinline__ double u256_read(const u256 &v) {
  unsigned long long q[kLossAccWords];
#pragma unroll
  for (int k = 0; k < kLossLimbs - 1; ++k) {
    const int b = 40 * k, wi = b >> 6, sh = b & 63;
    unsigned long long x = v.w[wi] >> sh;
    if (sh > 24 && wi < 3) x |= v.w[wi + 1] << (64 - sh);
    q[k] = x & kLimbMask;
  }
  q[kLossLimbs - 1] = (v.w[3] >> 8);   // bits 200 .. 255
  q[kLossLimbs] = 0;
  return acc_value(q);
}
// A canonical non-negative limb_sum as a u256 (limbs 0..4 in [0, 2^40), limb 5 below 2^56)
__device__ __forceinline__ u256 u256_of(limb_sum v) {
#pragma unroll
  for (int k = 0; k < kLossLimbs - 1; ++k) {
    v.l[k + 1] += (unsigned long long)((long long)v.l[k] >> 40);
    v.l[k] &= kLimbMask;
  }
  u256 r = {{0, 0, 0, 0}};
#pragma unroll
  for (int k = 0; k < kLossLimbs; ++k) {
    const int b = 40 * k, wi = b >> 6, sh = b & 63;
    r.w[wi] |= v.l[k] << sh;
    if (sh > 24 && wi < 3) r.w[wi + 1] |= v.l[k] >> (64 - sh);
  }
  return r;
}

// Point k of the weighted curve pass (thr[k], highest score first): X_k and Y_k from the runs' prefix sums, and keep[k] = 1
// when its weight increment X_k - X_(k-1) is not zero (X_(-1) = 0).  Also counts the rows of positive weight (R(c) > 0)
// among the runs' keys into *n_wrows.
__global__ void __launch_bounds__(256) k_iso_wpoint(const double *__restrict__ thr, int64_t m,
                                                    const unsigned long long *__restrict__ pos, int64_t n_pos,
                                                    const unsigned long long *__restrict__ neg, int64_t n_neg,
                                                    const limb_sum *__restrict__ pre_pos, const limb_sum *__restrict__ pre_neg,
                                                    const double *__restrict__ pos_c, const double *__restrict__ neg_c,
                                                    u256 *__restrict__ px, u256 *__restrict__ py, int *__restrict__ keep,
                                                    unsigned long long *__restrict__ n_wrows) {
  const limb_sum p_all = limb_prefix(pre_pos, n_pos), n_all = limb_prefix(pre_neg, n_neg);
  auto at = [&](int64_t k, u256 &x, u256 &y) {
    const unsigned long long key = score_key(thr[k]);
    const limb_sum p = limb_add(p_all, limb_prefix(pre_pos, key_lower_bound(pos, n_pos, key)), true);
    const limb_sum q = limb_add(n_all, limb_prefix(pre_neg, key_lower_bound(neg, n_neg, key)), true);
    y = u256_of(p);
    x = u256_of(limb_add(p, q));
  };
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += stride) {
    u256 x, y, x0 = {{0, 0, 0, 0}}, y0;
    at(k, x, y);
    if (k > 0) at(k - 1, x0, y0);
    px[k] = x;
    py[k] = y;
    keep[k] = !u256_eq(x, x0);
  }
  unsigned long long c = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_pos + n_neg; i += stride) {
    const double ci = i < n_pos ? pos_c[i] : neg_c[i - n_pos];
    c += rint(ci * 0x1p160) != 0.0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(n_wrows, c);
}
// The kept points packed: point excl[k] of (qx, qy, qthr) is point k; the last thread writes the kept count
__global__ void __launch_bounds__(256) k_iso_wpack(int64_t m, const int *__restrict__ keep, const int *__restrict__ excl,
                                                   const u256 *__restrict__ px, const u256 *__restrict__ py,
                                                   const double *__restrict__ thr, u256 *__restrict__ qx,
                                                   u256 *__restrict__ qy, double *__restrict__ qthr,
                                                   unsigned long long *__restrict__ n_kept) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += (int64_t)gridDim.x * blockDim.x) {
    if (keep[k]) {
      const int j = excl[k];
      qx[j] = px[k];
      qy[j] = py[k];
      qthr[j] = thr[k];
    }
    if (k == m - 1) *n_kept = (unsigned long long)(excl[k] + keep[k]);
  }
}
// The weighted fit's point set for the hull kernels: point i is the origin, or kept point i - 1 of (qx, qy).  A block's
// values are its weight and positive weight, read() of exact differences, p = fl(read(dY) / read(dX)).
struct IsoWeights {
  using Coord = u256;
  using Ref = const u256 &;
  using Block = double;
  const u256 *__restrict__ qx, *__restrict__ qy;
  __device__ __forceinline__ void point(int i, u256 &x, u256 &y) const {
    if (i == 0) { x = u256{{0, 0, 0, 0}}; y = x; return; }
    x = qx[i - 1];
    y = qy[i - 1];
  }
  // The sign of (a - o) x (b - o): o comes before a and b, so every difference is >= 0 and the cross product is the
  // comparison of two unsigned 512-bit products.
  __device__ __forceinline__ static int turn(Ref ox, Ref oy, Ref ax, Ref ay, Ref bx, Ref by) {
    unsigned long long p[8], q[8];
    u256_mul(u256_sub(ax, ox), u256_sub(by, oy), p);
    u256_mul(u256_sub(ay, oy), u256_sub(bx, ox), q);
#pragma unroll
    for (int i = 7; i >= 0; --i)
      if (p[i] != q[i]) return p[i] > q[i] ? 1 : -1;
    return 0;
  }
  __device__ __forceinline__ static int above(Ref vx, Ref vy, Ref ux, Ref uy, Ref rx, Ref ry) {
    return -turn(vx, vy, ux, uy, rx, ry);   // (r - v) x (u - v) = -((u - v) x (r - v))
  }
  __device__ __forceinline__ static double block(Ref x0, Ref y0, Ref x1, Ref y1, Block &w, Block &pw) {
    w = u256_read(u256_sub(x1, x0));
    pw = u256_read(u256_sub(y1, y0));
    return pw / w;
  }
};

// ---- the weighted quality pass (dsgd_eval_*weighted_calibration, dsgd_eval_*weighted_isotonic_calibration) -----------
// kIso: p = interp(s) at the map (X, Y) and the log-loss term -log p or -log1p(-p); else p = sigmoid(-z), z = a f + b, and
// the term softplus(+-z); each as k_calib_eval<kIso, kSmem>, its positions taken by warp_scores.  c_i is row_weight.  A
// row with R(c) = 0 is counted in kCwvRows and adds nothing else.  The sums add R(fl(c (p - o)^2)), R(fl(c l)) over the finite
// terms, R(c) over the rows used and R(c) over the rows whose term is infinite (counted in kCwvInf too); bin k adds R(c),
// R(c) of the positives and R(fl(c p)) to its three limb blocks in shared memory.  A bin value of 2^52 or more is counted
// in the bin's overflow word; the integer part of a value is split at 2^40 between limbs 4 and 5, so every shared word
// grows by at most 2^40 per row, as in the unweighted bins.  The host reads every sum with read().
enum CalibWEvalWord : int {
  kCwvBrier = 0,                                   // [0, 7): limbs and overflow count of sum R(c (p - o)^2)
  kCwvLog = kLossAccWords,                         // [7, 14): of sum R(c l), finite terms
  kCwvW = 2 * kLossAccWords,                       // [14, 21): of sum R(c) over the rows used
  kCwvInfW = 3 * kLossAccWords,                    // [21, 28): of sum R(c) over the rows whose term is infinite
  kCwvRows = 4 * kLossAccWords,                    // rows used
  kCwvNan = kCwvRows + 1,                          // rows left out
  kCwvInf = kCwvRows + 2,                          // rows of positive weight whose term is infinite
  kCwvBins = 32,                                   // per bin: kCwvBinStride words {weight, positive weight, sum c p, overflow}
  kCwvBinStride = 3 * kLossLimbs + 1,
  kCwvWords = kCwvBins + kCalMaxBins * kCwvBinStride
};
// v >= 0 into a bin's limb block in shared memory (limbs 0..5), its overflow counted at *ovf
__device__ __forceinline__ void cal_bin_add(unsigned long long *lim, unsigned long long *ovf, double v) {
  if (!(v < 4503599627370496.0)) { atomicAdd(ovf, 1ull); return; }
  acc_cut(v, [&](int k, double limb) {
    if (limb == 0.0) return;
    const unsigned long long u = (unsigned long long)(long long)limb;
    if (k == kLossLimbs - 2) {
      if (u & kLimbMask) atomicAdd(&lim[k], u & kLimbMask);
      if (u >> 40) atomicAdd(&lim[k + 1], u >> 40);
    } else {
      atomicAdd(&lim[k], u);
    }
  });
}
template <bool kIso, bool kSmem, bool kIcpt>
__global__ void __launch_bounds__(256) k_weval(const uint32_t *__restrict__ rp16, const uint2 *__restrict__ pairs,
                                               const int8_t *__restrict__ label, const int32_t *__restrict__ samples,
                                               int64_t row_begin, int64_t n, const double *__restrict__ w, double a, double b,
                                               const double *__restrict__ X, const double *__restrict__ Y, int k, int n_bins,
                                               unsigned long long *__restrict__ blk, double w_pos, double w_neg,
                                               const double *__restrict__ sw, const double *__restrict__ icpt) {
  __shared__ unsigned long long s_bins[kCalMaxBins * kCwvBinStride];
  const double *xs = nullptr, *ys = nullptr;
  if constexpr (kIso) iso_stage<kSmem>(X, Y, k, xs, ys);
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kCalMaxBins * kCwvBinStride; i += blockDim.x) s_bins[i] = 0ull;
  __syncthreads();
  unsigned long long lb[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ll[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_b = 0, ovf_l = 0;
  unsigned long long lw[kLossLimbs] = {0, 0, 0, 0, 0, 0}, li[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf_w = 0, ovf_i = 0;
  unsigned c_rows = 0, c_nan = 0, c_inf = 0;
  warp_scores<kIcpt>(rp16, pairs, samples, row_begin, n, w, icpt, [&](int64_t, int64_t r, double dot, bool mine) {
    if (!mine) return;
    const double z = kIso ? -dot : a * dot + b;   // kIso: the score s
    if (isnan(z)) { ++c_nan; return; }
    ++c_rows;
    const bool pos = label[r] > 0;
    const double c = row_weight(pos, w_pos, w_neg, sw, r);
    if (rint(c * 0x1p160) == 0.0) return;   // R(c) = 0: the row adds exactly 0 to every sum
    const double pr = kIso ? iso_interp(z, xs, ys, k) : sigmoid(-z), o = pos ? 1.0 : 0.0, dlt = pr - o;
    const double term = kIso ? (pos ? -log(pr) : -log1p(-pr)) : softplus(pos ? z : -z);
    acc_add_local(lb, ovf_b, c * (dlt * dlt));
    if (kIso && isinf(term)) {
      ++c_inf;
      acc_add_local(li, ovf_i, c);
    } else {
      acc_add_local(ll, ovf_l, c * term);
    }
    acc_add_local(lw, ovf_w, c);
    int bin = (int)floor(pr * (double)n_bins);
    bin = bin < n_bins - 1 ? bin : n_bins - 1;
    unsigned long long *bl = s_bins + bin * kCwvBinStride, *bo = bl + 3 * kLossLimbs;
    cal_bin_add(bl, bo, c);
    if (pos) cal_bin_add(bl + kLossLimbs, bo, c);
    cal_bin_add(bl + 2 * kLossLimbs, bo, c * pr);
  });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ovf_b += __shfl_xor_sync(full, ovf_b, o);
    ovf_l += __shfl_xor_sync(full, ovf_l, o);
    ovf_w += __shfl_xor_sync(full, ovf_w, o);
    ovf_i += __shfl_xor_sync(full, ovf_i, o);
#pragma unroll
    for (int q = 0; q < kLossLimbs; ++q) {
      lb[q] += __shfl_xor_sync(full, lb[q], o);
      ll[q] += __shfl_xor_sync(full, ll[q], o);
      lw[q] += __shfl_xor_sync(full, lw[q], o);
      li[q] += __shfl_xor_sync(full, li[q], o);
    }
  }
  c_rows = __reduce_add_sync(full, c_rows);
  c_nan = __reduce_add_sync(full, c_nan);
  c_inf = __reduce_add_sync(full, c_inf);
  if (lane == 0) {
    acc_flush_local(blk + kCwvBrier, lb, ovf_b);
    acc_flush_local(blk + kCwvLog, ll, ovf_l);
    acc_flush_local(blk + kCwvW, lw, ovf_w);
    acc_flush_local(blk + kCwvInfW, li, ovf_i);
    if (c_rows) atomicAdd(&blk[kCwvRows], (unsigned long long)c_rows);
    if (c_nan) atomicAdd(&blk[kCwvNan], (unsigned long long)c_nan);
    if (c_inf) atomicAdd(&blk[kCwvInf], (unsigned long long)c_inf);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_bins * 3; i += blockDim.x) {
    const int bin = i / 3, s = i % 3;
    unsigned long long q[kLossLimbs];
#pragma unroll
    for (int t = 0; t < kLossLimbs; ++t) q[t] = s_bins[bin * kCwvBinStride + s * kLossLimbs + t];
    acc_carry(q);
    unsigned long long *dst = blk + kCwvBins + bin * kCwvBinStride;
#pragma unroll
    for (int t = 0; t < kLossLimbs; ++t)
      if (q[t]) red_add_u64(dst + s * kLossLimbs + t, q[t]);
    const unsigned long long ov = s_bins[bin * kCwvBinStride + 3 * kLossLimbs];
    if (s == 0 && ov) red_add_u64(dst + 3 * kLossLimbs, ov);
  }
}

}  // namespace dsgd
