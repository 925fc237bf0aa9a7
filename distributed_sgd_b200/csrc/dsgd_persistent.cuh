// dsgd_persistent.cuh -- the synchronous SGD loop as ONE persistent, warp-specialised cooperative kernel.
//
// Replaces, for a whole run of consecutive steps, the body of Master.fit's batch loop
// (core/Master.scala:179-198) together with the slave's gradient request (core/Slave.scala:142-157):
// no launch, no host round trip and exactly ONE grid-wide barrier per SGD step -- on one GPU and on K GPUs.
//
// Latencies this design answers (tools/microbench.cu measures them): an L2 hit and a gpu-scope grid barrier each cost
// hundreds to thousands of cycles; the step is a chain of dependent latencies, so the
// kernel removes links from the chain:
//   * PRODUCER warp (one per CTA): row windows do not depend on the weights, so it walks the sample ids
//     kStages steps ahead -- ids -> row pointers -> one TMA bulk copy (cp.async.bulk, mbarrier
//     complete_tx) per row into the stage's shared-memory partition, plus a chunk list.
//   * CONSUMER warps: the CTA's rows of a step are cut into 128-pair chunks dealt round-robin to the
//     warps.  A row that is ONE chunk (85 % of them) is finished by the warp that holds it in registers: dot,
//     gate, RED of y*x into g.  Longer rows: partial dots per chunk (fixed order), then gate + scatter per chunk -- by the
//     row's own warps after a named barrier of the row's when the stage is at most one chunk per warp, else in a second pass.
//   * UPDATE warps: weights are double-buffered and gradients triple-buffered in L2 so the update of step
//     t-1 and the gradient of step t share one barrier interval.
//   * c_t = 2*lambda*(W_t . d) (SparseSVM.scala:31) is a dot over the whole weight vector that the NEXT interval needs
//     first thing, and it must be the same bits in every CTA and on every GPU.  Each CTA adds its partial {W.d, ||W||^2}
//     to a small EXACT fixed-point accumulator (five 40-bit limbs per value, 64-bit integer REDs, one 128-byte line)
//     before it arrives at the grid barrier: integer sums do not depend on the order of arrival, so there is nothing to
//     sort out afterwards -- update warp 0 of every CTA reads the 96 bytes after the barrier (one L2 round trip,
//     overlapped with the consumers' first gathers) and has c.  (Summing fp64 partials from a shared area after the
//     barrier, a second counter barrier among the update warps and an all-to-all flag barrier were all slower.)
//   * GRID BARRIER: one release arrival on a counter, relaxed polling.  Its cost is fences and L2 round trips, not
//     contention (tools/microbench.cu); the acquire fence is not needed here (see grid_barrier_arrive_wait).  The barrier is
//     still the largest single item of a step.
//
// One GPU (kMulti == false), interval I_t between grid barrier t-1 and t, W_t = weights step t differentiates at:
//   consumers: x.W_t with W_t[col] = update(W_{t-1}[col], g_{t-1}[col], c_{t-1}) applied on the fly; gate; RED into g_t
//   updaters : W_t buffer <- update(W_{t-1}, g_{t-1}, c_{t-1}); zero g_{t+1}'s buffer; c_t, ||W_t||^2
//   W and g of a column sit side by side in one 16-byte record {W, g} (three rotating record arrays): a consumer needs
//   ONE 128-bit gather per non-zero -- the scattered 8-byte accesses of a CTA's non-zeros are what its time grows with
//   (two gathers and one RED per pair were measured slower).
//
// K GPUs (kMulti == true; one process or ctx per GPU, every rank's receive area mapped into every peer over
// NVLink), interval I_T:
//   everybody : push the NON-ZERO entries of this CTA's column slice of g_{T-1} to every peer as "LL" words
//               (16-byte {data, tag} stores: valid as soon as the tag matches -- no fence, no flag, one one-way
//               hop) plus one 8-byte LL word per 32 columns carrying the bitmap of which entries were sent.
//               A batch-256 gradient touches ~10 % of the 47 236 columns: ~0.15 MB per peer and step instead of
//               the 0.76 MB of the dense exchange of round 1.
//   column threads (one column per barrier-synchronised thread): the K replies of step T-1 (own from local
//               g_{T-1}, the peers' bitmap word and, where its bit is set, the value word), each regularized on
//               its own support and folded in rank order (Vec.mean's left fold, core/Master.scala:194;
//               SURVEY.md H4), W_T = W_{T-1} - lr*sum/K published as a local LL word (tag T+1)
//   consumers : ONE 16-byte gather per non-zero -- the LL word of W_T[col], spinning on its tag
//   Every rank computes the full update itself in the same order: replicas stay bit-identical, nothing is
//   broadcast, there is no collective call.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "dsgd_fixed.cuh"
#include "dsgd_kernels.cuh"

namespace dsgd {

constexpr int kMaxWorld = 8;  // ranks of the fused exchange: the GPUs of one NVSwitch box

struct PersistParams {
  const uint32_t *rp16;
  const uint2 *pairs;
  const int8_t *label;
  const int32_t *samples;  // n_steps * batch ids, step-major
  int64_t n_steps;
  int32_t batch;
  int32_t dim;
  double *wbuf[2];  // K GPUs: on entry wbuf[0] holds the initial weights
  double *gbuf[3];  // K GPUs: gradient buffers, all zero on entry and on exit
  double2 *rec[3];  // one GPU: rotating records {W, g} per column; on entry all three = {W_init, 0}
  const double *d;
  unsigned long long *acc;  // [3 rotating][kAccStride]: fixed-point accumulators of {W.d, ||W||^2}; zero on entry
  unsigned *hinge;  // one GPU: [n_steps][gridDim.x], the hinge count of every step and CTA (every slot is stored)
  double *losses;   // [n_steps] or nullptr
  double *w_out;    // resident weights after the last step
  float *w32_out;
  double *scal;     // kScalC / kScalNrm2 of the resident weights
  unsigned *bar;    // grid barrier: arrival counter, zero on entry
  int *abort_flag;  // set to 1 if a wait hit the watchdog
  double lambda, lr, k_den;
  long long timeout_cycles;
  long long *tl;    // debug timeline (dsgd_debug_timeline) or nullptr
  // ---- K GPUs ----
  int world, rank;
  int64_t step_base;                      // global step number of this launch's first step (same on all ranks)
  unsigned long long *xval[kMaxWorld];    // value words of rank k's receive area: [sender][parity][xstride] x 16 B; [rank] is local
  unsigned long long *xbm[kMaxWorld];     // bitmap words of rank k's receive area: [sender][parity][xwords] x 8 B
  int xstride, xwords;
  unsigned long long *llw[2];             // this rank's weights as LL words, double-buffered by step parity
  unsigned long long *xstats;             // [0] value words, [1] bitmap words this rank pushed to ONE peer (diagnostic)
  // ---- averaged SGD (kAvg); last, so that the parameter offsets of the other instantiations stay where they were ----
  double *avg;                            // [dim] running sum of W_t over the averaged steps: read at launch, written at exit
  // ---- per-step learning rates (kLrTable); last for the same reason ----
  const double *lrs;                      // [n_steps]: step s of this launch uses lrs[s] instead of lr
  // ---- L1 penalty (kL1, one GPU); last for the same reason ----
  double lambda1;                         // every update is followed by soft_threshold(., lr * lambda1) on every column
  // ---- one GPU with losses; last for the same reason ----
  double *loss_nrm;                       // [2][n_steps]: ||W_t||^2, then (kL1) ||W_t||_1, of every step t of the launch
  // ---- class weights (kClassWeighted, one GPU); last for the same reason ----
  double w_pos, w_neg;                    // a row of label y scatters x * (y * w_y); the step's loss is (w_pos H+ + w_neg H-) / batch
  // ---- sample weights (kSampleWeighted, one GPU); last for the same reason ----
  const double *sw;                       // [rows]: row i scatters x * (y * c_i), c_i = w_y * sw[i]
  unsigned long long *hcode;              // [n_steps][gridDim.x]: the 2-bit hinge codes of every step's rows of every CTA
};
static_assert(sizeof(PersistParams) <= 4000, "kernel parameter space is 4 KB");

// ---- PTX helpers: mbarrier + TMA bulk copy -------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *b, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, uint64_t *b) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(b))
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *b, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(b)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: if the phase does not complete within `timeout` cycles (or somebody already raised the abort
// flag) the flag is raised and the caller carries on -- results are then garbage, but nothing deadlocks and the
// host turns the flag into DSGD_ERR_TIMEOUT.
__device__ __forceinline__ void mbar_wait(uint64_t *b, unsigned parity, int *abort_flag, long long timeout) {
  if (mbar_try_wait(b, parity)) return;
  const long long t0 = clock64();
  unsigned spins = 0;
  while (!mbar_try_wait(b, parity)) {
    if ((++spins & 255u) == 0u && (clock64() - t0 > timeout || *(volatile int *)abort_flag)) {
      *(volatile int *)abort_flag = 1;
      return;
    }
  }
}
__device__ __forceinline__ unsigned ld_relaxed_gpu(const unsigned *p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(unsigned *p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned atom_acq_rel_gpu_add(unsigned *p, unsigned v) {
  unsigned old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ void st_relaxed_gpu(unsigned *p, unsigned v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int n_threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int n_threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}
__device__ __forceinline__ long long global_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// "LL" element of the cross-GPU exchange: a double travels as two 8-byte words {low 32 bits, tag} and
// {high 32 bits, tag}.  An aligned 8-byte store is single-copy atomic, so a word whose tag matches carries valid
// data: no fence, no separate flag, one one-way NVLink store per word (the scheme of NCCL's LL protocol).
__device__ __forceinline__ void ll_store(unsigned long long *dst, double v, unsigned tag) {
  const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
  const unsigned long long w0 = (bits & 0xffffffffull) | ((unsigned long long)tag << 32);
  const unsigned long long w1 = (bits >> 32) | ((unsigned long long)tag << 32);
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(w0), "l"(w1) : "memory");
}
__device__ __forceinline__ bool ll_try_load(const unsigned long long *src, unsigned tag, double &v) {
  unsigned long long w0, w1;
  asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(src) : "memory");
  if ((unsigned)(w0 >> 32) != tag || (unsigned)(w1 >> 32) != tag) return false;
  v = __longlong_as_double((long long)((w0 & 0xffffffffull) | (w1 << 32)));
  return true;
}
// 32 payload bits + tag in ONE 8-byte word (the bitmap of a 32-column group)
__device__ __forceinline__ void ll_store32(unsigned long long *dst, unsigned v, unsigned tag) {
  const unsigned long long w = (unsigned long long)v | ((unsigned long long)tag << 32);
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(w) : "memory");
}
__device__ __forceinline__ bool ll_try_load32(const unsigned long long *src, unsigned tag, unsigned &v) {
  unsigned long long w;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(src) : "memory");
  v = (unsigned)w;
  return (unsigned)(w >> 32) == tag;
}

// w_j after one SGD update given the raw gradient-sum entry (same arithmetic as k_update<true>):
// regularize on the surviving key (SparseSVM.scala:31), mean over workers, times lr, subtract, each with the
// Sparse constructor's 1e-20 filter (core/Master.scala:194,197; math/Sparse.scala:108-118).
__device__ __forceinline__ double apply_update(double wv, double graw, double c, bool add_c, double k_den, double lr) {
  double v = filt(graw);
  if (v != 0.0) {
    if (add_c) v = filt(v + c);
    if (v != 0.0) {
      const double mean = (k_den == 1.0) ? v : filt(v / k_den);  // x / 1.0 == x exactly
      const double step = filt(mean * lr);
      wv = filt(wv - step);
    }
  }
  return wv;
}

// ---- grid barrier among the barrier-synchronised warps of every CTA (the producer warp stays out) -------------------
// Called by one thread between two CTA-level barriers: one RELEASE arrival on a counter, relaxed polling.
// There is no acquire fence after the poll.  What follows the barrier reads mutable global data only with instructions
// that are served by L2 -- ld.global.cg / ld.relaxed.gpu / red / the LL words' ld.relaxed.sys -- never through L1, and a
// thread cannot issue them before the branch on the polled value resolves, so they reach L2 after the arrival they
// observed, which every peer performed after its own writes (release).  Leaving the fence out shortens every barrier; the trajectories are checked
// against the oracle to 1e-12 over hundreds of steps in the tests and in every bench run (`parity`).
// Returns false if the watchdog fired.
__device__ __forceinline__ bool grid_barrier_arrive_wait(unsigned *bar, unsigned target, int *abort_flag, long long timeout) {
  red_release_gpu_add(bar, 1u);
  const long long t0 = clock64();
  unsigned spins = 0;
  bool ok = true;
  while ((int)(ld_relaxed_gpu(bar) - target) < 0) {
    if ((++spins & 1023u) == 0u && (clock64() - t0 > timeout || *(volatile int *)abort_flag)) {
      *(volatile int *)abort_flag = 1;
      ok = false;
      break;
    }
  }
  return ok;
}

constexpr int kChunkPairs = 128;             // 4 pairs per lane per chunk
static_assert(kChunkPairs == kFoldPairs, "a listed row's chunks are the chunks of the row fold");
constexpr uint32_t kChunkGlobal = 1u << 31;  // chunk offset flag: read from global, the row did not fit the stage
constexpr int kMaxRowsPerCta = 32;           // rows of one step per CTA (one producer lane each)
// Hardware named barriers of the rows of several chunks that their own warps finish (consume_stage): ids 5..15.  0 is
// __syncthreads, 2 the consumers' second pass, 3 and 4 the CTA's barriers around the grid barrier.
constexpr int kRowBarFirst = 5, kRowBars = 11;

template <int kMaxChunks>
struct StageMeta {
  int n_rows;
  int n_chunks;
  int n_multi;                       // listed rows of more than one chunk
  int two_pass;                      // 1: the rows of several chunks take the second pass after a barrier of all consumers
  int n_pairs;                       // pairs of the CTA's rows in this stage (diagnostic)
  int row_y[kMaxRowsPerCta];
  uint32_t row_b[kMaxRowsPerCta];    // window start (16-byte units) -- for rows that missed the chunk list
  int row_len[kMaxRowsPerCta];       // pairs, padding included
  short row_first[kMaxRowsPerCta];   // first chunk of the row
  short row_nch[kMaxRowsPerCta];     // chunks of the row; -1: not in the chunk list (whole-row slow path)
  signed char row_bar[kMaxRowsPerCta];   // named barrier of a row of several chunks finished by its own warps, or -1
  uint32_t ch_off[kMaxChunks];       // pair offset inside the stage partition, or kChunkGlobal | global pair index
  short ch_n[kMaxChunks];            // pairs in the chunk (<= kChunkPairs)
  short ch_row[kMaxChunks];          // local row
  double part[kMaxChunks];           // pass-1 partial dot of the chunk
};

// kSampleWeighted: shared memory past the end of PersistSmem (the other forms launch without it) -- the combined weight c_i of
// every row of every stage, written by the producer with the stage's metadata, and the 2-bit hinge codes of the CTA's rows of
// the step
template <int kStages>
struct PersistSwSmem {
  double row_c[kStages][kMaxRowsPerCta];
  unsigned long long code;
};

template <int kCons, int kUpd, int kStages, int kStagePairs, int kMaxChunks>
struct PersistSmem {
  uint2 ring[kStages][kStagePairs];
  StageMeta<kMaxChunks> meta[kStages];
  uint64_t full[kStages];
  uint64_t empty[kStages];
  uint64_t c_bar[2];    // c of the weights interval t updates from
  uint64_t u_bar;       // every warp that owns columns has published its share of {W_T . d, ||W_T||^2} in red[]
  double red[kCons + kUpd][2];
  double c_val[2];
  double nrm_val[2];
  unsigned hinge_acc;
  int ok;
  long long tl_warp[kCons + kUpd];   // debug timeline: when each warp reached the CTA barrier
};

#define DSGD_TL(slot_)                                                                        \
  do {                                                                                        \
    if (p.tl && blockIdx.x == 0 && lane == 0 && t < 256) p.tl[t * 16 + (slot_)] = clock64(); \
  } while (0)
// per-CTA records of steps 100..103: {barrier arrival ns, barrier exit ns, pairs of the CTA's rows, chunks | multi-chunk rows << 32}
constexpr int kTlSteps = 4, kTlFirst = 100, kTlCtas = 160, kTlPerCta = 4;
constexpr int kTlWords = 256 * 16 + kTlSteps * kTlCtas * kTlPerCta;

// ---- weight fetch of the consumers: W_t[col] -----------------------------------------------------------------
// One GPU: the update of step t-1 applied on the fly to (W_{t-1}[col], g_{t-1}[col]); c_{t-1} arrives through an
// mbarrier (completed during the previous interval, so the wait normally falls through).
// kL1: the update is followed by the proximal step of the L1 penalty, soft_threshold(., tau), on every column the consumers
// read -- also on those whose g_{t-1} is 0.
template <bool kL1 = false>
struct FetchLocal {
  const double2 *R;   // records {W_{t-1}, g_{t-1}}
  uint64_t *cbar;
  unsigned cpar;
  const double *cval;
  int *abort_flag;
  long long timeout;
  double k_den, lr;
  double tau = 0.0;   // kL1 only
  double c = 0.0;
  bool add_c = false, have_c = false, good = true;
  __device__ __forceinline__ void need_c() {
    if (!have_c) {
      mbar_wait(cbar, cpar, abort_flag, timeout);
      c = *(volatile const double *)cval;
      add_c = (c != 0.0) && (fabs(c) > kEps);
      have_c = true;
    }
  }
  __device__ __forceinline__ void get4(const uint2 (&pr)[4], double (&wv)[4]) {
    double2 r[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      r[u] = make_double2(0.0, 0.0);
      if (pr[u].y << 1) r[u] = __ldcg(&R[pr[u].x]);  // val != +-0: a zero value contributes filt(0 * w) == 0 whatever the weight
    }
    need_c();
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      wv[u] = apply_update(r[u].x, r[u].y, c, add_c, k_den, lr);
      if constexpr (kL1) wv[u] = soft_threshold(wv[u], tau);
    }
  }
  __device__ __forceinline__ double get1(uint32_t col) {
    need_c();
    const double2 r = __ldcg(&R[col]);
    const double wv = apply_update(r.x, r.y, c, add_c, k_den, lr);
    if constexpr (kL1) return soft_threshold(wv, tau);
    return wv;
  }
};
// K GPUs: the LL word of W_T[col] published by the column's thread of this GPU, spinning on its tag.
struct FetchLL {
  const unsigned long long *LW;
  unsigned tag;
  int *abort_flag;
  long long timeout;
  bool good = true;
  __device__ __forceinline__ void spin(const unsigned long long *src, double &v) {
    unsigned spins = 0;
    const long long t0 = clock64();
    while (!ll_try_load(src, tag, v)) {
      if ((++spins & 255u) == 0u && (clock64() - t0 > timeout || *(volatile int *)abort_flag)) {
        *(volatile int *)abort_flag = 1;
        good = false;
        v = 0.0;
        break;
      }
    }
  }
  // All pending words are REQUESTED before any is looked at (a request and its check written together compile into
  // one dependent round trip per word: nvcc reuses the destination registers).
  __device__ __forceinline__ void get4(const uint2 (&pr)[4], double (&wv)[4]) {
    unsigned pend = 0;   // bit u: word of pair u not published yet; all pending words are re-requested together
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      wv[u] = 0.0;
      if (pr[u].y << 1) pend |= 1u << u;
    }
    unsigned spins = 0;
    const long long t0 = clock64();
    while (pend) {
      unsigned long long w0[4], w1[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        w0[u] = 0ull; w1[u] = 0ull;
        if (pend & (1u << u))
          asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0[u]), "=l"(w1[u]) : "l"(LW + 2 * (size_t)pr[u].x) : "memory");
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if ((pend & (1u << u)) && (unsigned)(w0[u] >> 32) == tag && (unsigned)(w1[u] >> 32) == tag) {
          wv[u] = __longlong_as_double((long long)((w0[u] & 0xffffffffull) | (w1[u] << 32)));
          pend &= ~(1u << u);
        }
      if (pend && (++spins & 63u) == 0u && (clock64() - t0 > timeout || *(volatile int *)abort_flag)) {
        *(volatile int *)abort_flag = 1;
        good = false;
        pend = 0;
      }
    }
  }
  __device__ __forceinline__ double get1(uint32_t col) {
    double v;
    spin(LW + 2 * (size_t)col, v);
    return v;
  }
};

// The pairs of chunk c, 4 per lane (val 0 past the chunk's end: inert).
template <int kMaxChunks>
__device__ __forceinline__ void chunk_pairs(const StageMeta<kMaxChunks> &mt, const uint2 *ring, const uint2 *pairs, int c, int lane,
                                            uint2 (&pr)[4]) {
  const uint32_t off = mt.ch_off[c];
  const int n = mt.ch_n[c];
  const uint2 *src = (off & kChunkGlobal) ? (pairs + (off & ~kChunkGlobal)) : (ring + off);
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int k = u * 32 + lane;
    pr[u] = (k < n) ? src[k] : make_uint2(0u, 0u);
  }
}

// ---- the consumer warps' work on one stage: SlaveImpl.gradient's per-sample body (core/Slave.scala:147-153) ----
// x.W per row (math/Vec.scala:58), prediction and hinge loss (SparseSVM.scala:14-16), gate (SparseSVM.scala:28),
// RED of y*x into g (entry of column c at gbase + gstride * c).  A row that is ONE chunk (85 % of them) is gated and
// scattered by the warp that computed its dot, from the registers that still hold its pairs.  A row of several chunks:
//   * per row (the stage lists every row in at most kCons chunks, so a warp holds at most one chunk): the row's warps leave
//     their partials in part[], meet on the row's own named barrier (row_bar, nch * 32 threads), each sums the row's partials
//     in chunk order and gates and scatters its own chunk from its registers; the warp of the row's first chunk counts the
//     hinge.  No warp waits for a row it does not hold, and a warp waits on one barrier at most.
//   * otherwise (two_pass): a second pass after a barrier among all consumer warps re-reads each chunk's pairs.
// Both sum the same partials in the same order and issue the same REDs.
// pre (optional): the pairs of the warp's first chunk, already loaded with chunk_pairs
// kWeight == kClassWeighted: a row of label y scatters x * s with s = y * w_y instead of x * y, at all three scatter sites,
// and its hinge loss is counted in the low 16 bits of the returned word for y = +1 and in the high 16 bits for y = -1.  A
// CTA holds at most kMaxRowsPerCta = 32 rows of hinge <= 2 per step, so a half holds at most 64 and never carries into the
// other.
// kWeight == kSampleWeighted: row m of the stage scatters x * s with s = y * row_c[m] (row_c: the stage's combined
// weights), and its hinge loss l in {0, 1, 2} is returned as the code l << 2 m of a 64-bit word: 32 rows x 2 bits, no
// carries.
template <int kCons, int kMaxChunks, int kWeight = kUnweighted, class Fetch>
__device__ __forceinline__ std::conditional_t<kWeight == kSampleWeighted, unsigned long long, unsigned> consume_stage(
    StageMeta<kMaxChunks> &mt, const uint2 *ring, const uint2 *pairs, double *gbase, const int gstride, Fetch &fetch, int warp,
    int lane, long long *tl, const uint2 (*pre)[4] = nullptr, double w_pos = 1.0, double w_neg = 1.0,
    const double *row_c = nullptr) {
  using Hinge = std::conditional_t<kWeight == kSampleWeighted, unsigned long long, unsigned>;
  const int n_ch = mt.n_chunks;
  Hinge hinge = 0;  // lane 0 only
  // the scatter scalar of row m, and its hinge loss in its class's half (class weights) or its code (sample weights)
  auto scale_of = [&](int yi, double y, int m) {
    if constexpr (kWeight == kSampleWeighted) return yi > 0 ? row_c[m] : -row_c[m];
    return kWeight == kClassWeighted ? (yi > 0 ? w_pos : -w_neg) : y;
  };
  auto hinge_of = [&](int yi, unsigned l, int m) -> Hinge {
    if constexpr (kWeight == kSampleWeighted) return (Hinge)l << (2 * m);
    return kWeight == kClassWeighted ? l << (yi > 0 ? 0 : 16) : l;
  };
  // ---- pass 1: dots of this warp's chunks ----
  for (int c = warp; c < n_ch; c += kCons) {
    uint2 pr[4];
    double wv[4];
    if (pre && c == warp) {
#pragma unroll
      for (int u = 0; u < 4; ++u) pr[u] = (*pre)[u];
    } else {
      chunk_pairs(mt, ring, pairs, c, lane, pr);
    }
    fetch.get4(pr, wv);
    double acc = 0.0;
#pragma unroll
    for (int u = 0; u < 4; ++u) acc += filt(filt((double)__uint_as_float(pr[u].y)) * wv[u]);  // (x * w).sum
    if (tl && lane == 0 && c == warp) tl[2] = clock64();   // first chunk: weights arrived, products done
    acc = warp_sum(acc);
    if (tl && lane == 0 && c == warp) tl[4] = clock64();   // ... dot reduced
    {
      const int row1 = mt.ch_row[c];
      const int nch1 = mt.row_nch[row1];
      int first1 = c;
      if (nch1 > 1) {   // the row's dot: its chunks' partials in chunk order, once every warp of the row has left its own
        if (lane == 0) mt.part[c] = acc;
        const int bar = mt.row_bar[row1];
        if (bar < 0) continue;   // two_pass
        named_bar_sync(bar, nch1 * 32);
        first1 = mt.row_first[row1];
        acc = 0.0;
        for (int i = 0; i < nch1; ++i) acc += mt.part[first1 + i];
      }
      {
        const int yi = mt.row_y[row1];
        const double y = (double)yi;
        if (c == first1 && lane == 0) hinge += hinge_of(yi, (unsigned)(1 - yi * pred_of(acc)), row1);
        if (!(y * acc < 0.0)) {  // SparseSVM.scala:28
          const double sc = scale_of(yi, y, row1);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const double gvv = filt(filt((double)__uint_as_float(pr[u].y)) * sc);
            if (gvv != 0.0) red_add_f64(gbase + (size_t)gstride * pr[u].x, gvv);
          }
        }
      }
    }
  }
  // ---- pass 2 (two_pass: rows of several chunks): row dot = chunk partials in order, prediction, gate, scatter ----
  if (mt.two_pass) {
    named_bar_sync(2, kCons * 32);
    for (int c = warp; c < n_ch; c += kCons) {
      const int row = mt.ch_row[c];
      const int first = mt.row_first[row], nch = mt.row_nch[row];
      if (nch == 1) continue;
      double dot = 0.0;
      for (int i = 0; i < nch; ++i) dot += mt.part[first + i];
      const int yi = mt.row_y[row];
      const double y = (double)yi;
      if (c == first && lane == 0) hinge += hinge_of(yi, (unsigned)(1 - yi * pred_of(dot)), row);
      if (!(y * dot < 0.0)) {
        const double sc = scale_of(yi, y, row);
        const uint32_t off = mt.ch_off[c];
        const int n = mt.ch_n[c];
        const uint2 *src = (off & kChunkGlobal) ? (pairs + (off & ~kChunkGlobal)) : (ring + off);
        for (int k = lane; k < n; k += 32) {
          const uint2 pr = src[k];
          const double gvv = filt(filt((double)__uint_as_float(pr.y)) * sc);
          if (gvv != 0.0) red_add_f64(gbase + (size_t)gstride * pr.x, gvv);
        }
      }
    }
  }
  // rows outside the chunk list: empty rows (dot 0 -> prediction 0, hinge 1, nothing to scatter) and, if a step
  // ever overflows the chunk list, whole rows straight from global memory, one warp per row
  for (int m = warp; m < mt.n_rows; m += kCons) {
    const int nch = mt.row_nch[m];
    if (nch == 0) {
      if (lane == 0) hinge += hinge_of(mt.row_y[m], 1u, m);
    } else if (nch < 0) {
      const uint2 *grow = pairs + (size_t)mt.row_b[m] * 2;
      const int len = mt.row_len[m];
      // the row fold (dsgd_kernels.cuh): the dot pass 2 gives the same row when it is listed
      const double dot = row_fold(grow, 0, len, lane, [&](uint32_t c) { return fetch.get1(c); });
      const int yi = mt.row_y[m];
      const double y = (double)yi;
      if (lane == 0) hinge += hinge_of(yi, (unsigned)(1 - yi * pred_of(dot)), m);
      if (!(y * dot < 0.0))
        for (int k = lane; k < len; k += 32) {
          const uint2 pr = __ldg(&grow[k]);
          const double gvv = filt(filt((double)__uint_as_float(pr.y)) * scale_of(yi, y, m));
          if (gvv != 0.0) red_add_f64(gbase + (size_t)gstride * pr.x, gvv);
        }
    }
  }
  return hinge;
}

// kAvg: averaged SGD -- every column's p.avg[j] += W_t[j] for t = 1 .. S (W_0, the launch's starting weights, is not
// added), in step order, in plain fp64.  One GPU: the update threads keep the sums of their register columns in registers
// (loaded at launch start, stored in the epilogue); the columns past the register ones read-modify-write p.avg every step.
// K GPUs: the column thread keeps its column's sum in a register.
// kLrTable: step s of the launch takes the rate p.lrs[s] instead of p.lr.  Interval t applies the update of step t-1 (the
// consumers' on-the-fly fetch, the update warps, the K-GPU column threads), so all of them use lrs[t-1]; interval 0
// applies no update.
// kL1 (one GPU only): the update of step t-1 is followed by the proximal step of the L1 penalty on EVERY column, tau =
// lr * lambda1 with the same lr, in both places that apply it (the consumers' FetchLocal and the update warps); interval 0
// applies none.  A register column whose value changed is stored into the next three record buffers (ttl), as after a
// gradient update.  ||W_T||_1 travels like W_T . d and ||W_T||^2: fp64 per-warp partials in sm.red[warp - kCons][0] (the
// consumers' slots, unused on one GPU), summed per CTA by update warp 0 and pushed as fixed-point limbs into words 11..15
// of the step's accumulator (overflow word 10 shared).  The loss of step t-1 adds lambda1 * ||W_{t-1}||_1.
// kWeight == kClassWeighted (one GPU only): class weights -- consume_stage scales every scatter by the weight of the row's
// label and packs the CTA's hinge counts of the two classes into the halves of the word it already accumulates in
// sm.hinge_acc and stores in its hinge[t * G + CTA] slot (no new buffer, nothing new on the barrier path); the epilogue's
// per-step warp splits the halves, sums each over the G slots in integers and forms (w_pos * H+ + w_neg * H-) / batch once.
// kWeight == kSampleWeighted (one GPU only): sample weights -- the producer lane that loads row m's label also loads its
// sample weight and puts the combined weight c = w_y * sw[id] beside the stage's metadata (PersistSwSmem, past the end of
// PersistSmem); consume_stage scales every scatter by it and returns the rows' 2-bit hinge codes, which the consumer warps
// OR into one shared word.  The thread that arrives at the grid barrier stores that word into hcode[t * G + CTA] and clears
// it after the barrier has passed (nothing new before the arrival); the epilogue's per-step warp re-forms S = sum R(c_i *
// code_i) of the step in fixed-point limbs from the codes, p.samples, the labels and the weights.  Includes the class
// weights.
template <int kCons, int kUpd, int kStages, int kStagePairs, int kMaxChunks, bool kMulti, bool kAvg, bool kLrTable,
          bool kL1 = false, int kWeight = kUnweighted>
__global__ void __launch_bounds__((kCons + kUpd + 1) * 32, 1) k_sync_persistent(const PersistParams p) {
  using Smem = PersistSmem<kCons, kUpd, kStages, kStagePairs, kMaxChunks>;
  static_assert(!kL1 || (!kMulti && kUpd <= kCons), "the L1 form is one-GPU only and keeps its partials in the consumers' slots");
  static_assert(kWeight == kUnweighted || !kMulti, "the weighted forms are one-GPU only");
  static_assert(2 * kMaxRowsPerCta <= 64, "a CTA's hinge codes of one step fit one 64-bit word");
  static_assert(2 * kMaxRowsPerCta < (1 << 16), "a CTA's hinge count of one class fits a 16-bit half");
  static_assert(kAccWords + kAccLimbs <= kAccStride, "the L1 limbs follow the accumulator's overflow word");
  static_assert(kCons / 2 <= kRowBars, "every row of several chunks in a stage of at most kCons chunks has a named barrier");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
  using SwSmem = PersistSwSmem<kStages>;
  SwSmem &swm = *reinterpret_cast<SwSmem *>(smem_raw + sizeof(Smem));   // sample-weighted only: launched with the larger size

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const bool is_cons = warp < kCons;
  const bool is_upd = warp >= kCons && warp < kCons + kUpd;
  const int G = gridDim.x;
  const int B = p.batch;
  const int64_t S = p.n_steps;
  constexpr int kSyncThreads = (kCons + kUpd) * 32;
  // rows of a step owned by this CTA: i = blockIdx.x + m * G  (a small batch is spread over all CTAs); <= 32
  const int n_r = (B > (int)blockIdx.x) ? (B - 1 - (int)blockIdx.x) / G + 1 : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&sm.full[s], 1u);
      mbar_init(&sm.empty[s], (unsigned)kCons);
    }
    mbar_init(&sm.c_bar[0], 1u);
    mbar_init(&sm.c_bar[1], 1u);
    mbar_init(&sm.u_bar, (unsigned)(kMulti ? kCons + kUpd : kUpd));
    sm.c_val[0] = 0.0;   // interval 0 has no pending update (g_{-1} == 0): its c is never used
    sm.nrm_val[0] = 0.0;
    sm.hinge_acc = 0u;
    if constexpr (kWeight == kSampleWeighted) swm.code = 0ull;
    sm.ok = 1;
  }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) mbar_arrive(&sm.c_bar[0]);

  // =========================================================================================================
  // PRODUCER warp: runs ahead of everybody else, bounded only by the empty[] barriers.  Lane m owns row m.
  // =========================================================================================================
  if (!is_cons && !is_upd) {
    auto load_id = [&](int64_t t) -> int32_t {
      return (t < S && lane < n_r) ? __ldg(&p.samples[t * B + blockIdx.x + lane * G]) : -1;
    };
    uint32_t b0 = 0, e0 = 0, b1 = 0, e1 = 0;
    int y0 = 0, y1 = 0;
    double s0 = 0.0, s1 = 0.0;   // sample-weighted: the sample weights of the two windows
    auto load_win = [&](int32_t id, uint32_t &b, uint32_t &e, int &y, double &sw) {
      b = 0u; e = 0u; y = 0;
      if constexpr (kWeight == kSampleWeighted) sw = 0.0;
      if (id >= 0) {
        b = __ldg(&p.rp16[id]);
        e = __ldg(&p.rp16[id + 1]);
        y = (int)__ldg(&p.label[id]);
        if constexpr (kWeight == kSampleWeighted) sw = __ldg(&p.sw[id]);
      }
    };
    load_win(load_id(0), b0, e0, y0, s0);   // window of step t      (stage C input)
    load_win(load_id(1), b1, e1, y1, s1);   // window of step t + 1  (stage B)
    int32_t id_next = load_id(2);       // sample id of step t + 2 (stage A)
    for (int64_t t = 0; t < S; ++t) {
      const int st = (int)t & (kStages - 1);
      if (t >= kStages) {
        mbar_wait(&sm.empty[st], (unsigned)(((t / kStages) - 1) & 1), p.abort_flag, p.timeout_cycles);
        if (*(volatile int *)p.abort_flag) return;  // the barrier-synchronised warps gave up (watchdog)
      }
      auto &mt = sm.meta[st];
      // lay the rows out: exclusive scans over the CTA's rows of pairs and chunks
      const int len = (lane < n_r) ? (int)(e0 - b0) * 2 : 0;
      const int nch = (len + kChunkPairs - 1) / kChunkPairs;
      int ps = len, cs = nch;  // inclusive warp scans
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, ps, o), c2 = __shfl_up_sync(0xffffffffu, cs, o);
        if (lane >= o) { ps += a; cs += c2; }
      }
      const int my_pair = ps - len, my_chunk = cs - nch;
      const bool listed = (my_chunk + nch) <= kMaxChunks;           // prefix property: later rows miss too
      const bool in_ring = listed && (my_pair + len) <= kStagePairs;
      if (lane < n_r) {
        mt.row_y[lane] = y0;
        if constexpr (kWeight == kSampleWeighted) swm.row_c[st][lane] = (y0 > 0 ? p.w_pos : p.w_neg) * s0;
        mt.row_b[lane] = b0;
        mt.row_len[lane] = len;
        mt.row_first[lane] = (short)my_chunk;
        mt.row_nch[lane] = (short)(listed ? nch : -1);
        if (listed) {
          for (int c = 0; c < nch; ++c) {
            const int n = min(kChunkPairs, len - c * kChunkPairs);
            mt.ch_off[my_chunk + c] = in_ring ? (uint32_t)(my_pair + c * kChunkPairs)
                                              : (kChunkGlobal | (b0 * 2u + (uint32_t)(c * kChunkPairs)));
            mt.ch_n[my_chunk + c] = (short)n;
            mt.ch_row[my_chunk + c] = (short)lane;
          }
        }
      }
      const unsigned my_bytes = (lane < n_r && in_ring) ? (unsigned)len * 8u : 0u;
      const unsigned ring_bytes = __reduce_add_sync(0xffffffffu, my_bytes);
      // chunks actually written to the list: everything up to the first row that did not fit it
      const int listed_chunks = __reduce_max_sync(0xffffffffu, (lane < n_r && listed) ? (my_chunk + nch) : 0);
      const unsigned multi = __ballot_sync(0xffffffffu, lane < n_r && listed && nch > 1);
      // the rows of several chunks are finished by their own warps when every row is listed and every consumer warp holds
      // at most one chunk; each such row gets a named barrier of its own (kCons chunks hold at most kCons / 2 of them)
      const bool per_row = __all_sync(0xffffffffu, lane >= n_r || listed) && listed_chunks <= kCons;
      if (lane < n_r)
        mt.row_bar[lane] = (signed char)((per_row && nch > 1) ? kRowBarFirst + __popc(multi & ((1u << lane) - 1u)) : -1);
      if (lane == 31) mt.n_pairs = ps;
      if (lane == 0) {
        mt.n_rows = n_r;
        mt.n_chunks = listed_chunks;
        mt.n_multi = __popc(multi);
        mt.two_pass = (multi != 0u && !per_row) ? 1 : 0;
      }
      __syncwarp();  // every lane's metadata is written before lane 0 arrives on the full barrier
      if (lane == 0) {
        if (ring_bytes) mbar_expect_tx(&sm.full[st], ring_bytes);
        else mbar_arrive(&sm.full[st]);  // metadata only: complete the phase
      }
      __syncwarp();
      if (my_bytes) bulk_g2s(&sm.ring[st][my_pair], p.pairs + (size_t)b0 * 2, my_bytes, &sm.full[st]);
      // advance the register pipeline
      b0 = b1; e0 = e1; y0 = y1;
      if constexpr (kWeight == kSampleWeighted) s0 = s1;
      load_win(id_next, b1, e1, y1, s1);
      id_next = load_id(t + 3);
    }
    return;
  }

  // =========================================================================================================
  // barrier-synchronised warps (consumers + updaters)
  // =========================================================================================================
  double lr = p.lr;   // kLrTable: the rate of the update this interval applies (installed after the barrier that opens it)
  const int64_t base = kMulti ? p.step_base : 0;
  unsigned phase = 0;
  // one GPU: the update threads of all CTAs stride over the columns
  const int n_upd = G * kUpd * 32;
  const int u0 = blockIdx.x * kUpd * 32 + ((int)threadIdx.x - kCons * 32);
  // K GPUs: one column per barrier-synchronised thread; slices are multiples of 32 columns so that a warp's columns
  // share one bitmap word.  Slot [dim] is the packed counter of the step: hinge + 2^32 * samples.
  const int K = p.world, me = p.rank;
  const int slice = ((p.dim + 1 + G - 1) / G + 31) & ~31;
  const int j_col = blockIdx.x * slice + (int)threadIdx.x;
  const bool col_act = kMulti && (int)threadIdx.x < slice && j_col <= p.dim;
  const int col_word = j_col >> 5;
  unsigned long long st_val = 0, st_bm = 0;
  // one GPU, update threads: the columns this thread owns for the whole launch (W_{t-1}[j], d[j], buffers still to refresh,
  // "the g half seen last interval was non-zero"); K GPUs, column threads: W_{T-1}[j_col] and d[j_col]
  constexpr int kUpdCols = 2;
  double wreg[kUpdCols], dreg[kUpdCols];
  double areg[kUpdCols];   // kAvg: running sums of the same columns
  int ttl[kUpdCols];
  bool gnz[kUpdCols];
#pragma unroll
  for (int i = 0; i < kUpdCols; ++i) {
    wreg[i] = dreg[i] = 0.0;
    areg[i] = 0.0;
    ttl[i] = 0;
    gnz[i] = false;
    if constexpr (!kMulti) {
      const int j = u0 + i * n_upd;
      if (is_upd && j < p.dim) {
        wreg[i] = __ldcg(&p.rec[2][j].x);
        dreg[i] = __ldg(&p.d[j]);
        if constexpr (kAvg) areg[i] = p.avg[j];
      }
    }
  }
  if constexpr (kMulti) {
    if (col_act && j_col < p.dim) {
      wreg[0] = __ldcg(&p.wbuf[0][j_col]);
      dreg[0] = __ldg(&p.d[j_col]);
      if constexpr (kAvg) areg[0] = p.avg[j_col];
    }
  }

  // one GPU, consumer warps: the pairs of the warp's first chunk of the next step, loaded from the stage while the grid barrier
  // is still pending (the stage does not depend on the weights), so that the interval starts with the gathers
  uint2 pre[4];
  auto prefetch = [&](int64_t tn) {
    const int st = (int)tn & (kStages - 1);
    const auto &mt = sm.meta[st];
    mbar_wait(&sm.full[st], (unsigned)(((unsigned)tn / kStages) & 1u), p.abort_flag, p.timeout_cycles);
#pragma unroll
    for (int u = 0; u < 4; ++u) pre[u] = make_uint2(0u, 0u);
    if (warp < mt.n_chunks) chunk_pairs(mt, &sm.ring[st][0], p.pairs, warp, lane, pre);
  };
  if (!kMulti && is_cons && S > 0) prefetch(0);

  // rotating buffer indices kept as small integers (64-bit % 3 per warp and step is ~100 instructions on the critical path)
  int gi_prev = (int)((base + 2) % 3), gi_cur = (int)(base % 3), gi_next = (int)((base + 1) % 3);   // K GPUs: by global step
  int ti_prev = 2, ti_cur = 0, ti_next = 1;                                                          // by step of this launch
  for (int64_t T = base; T <= base + S; ++T) {
    const int64_t t = T - base;
    const bool first = (t == 0), last = (t == S);
    const double *Gprev = p.gbuf[gi_prev];   // g_{T-1}
    double *Gcur = p.gbuf[gi_cur];
    double *Gzero = p.gbuf[gi_next];
    const unsigned long long *acc_prev = p.acc + (size_t)ti_prev * kAccStride;   // partials of W_{T-1}: complete at barrier t-1
    unsigned long long *acc_cur = p.acc + (size_t)ti_cur * kAccStride;           // partials of W_T: added before barrier t
    unsigned long long *acc_next = p.acc + (size_t)ti_next * kAccStride;         // read during interval t-1: zeroed now
    const double2 *Rprev = p.rec[ti_prev];   // one GPU: {W_{t-1}, g_{t-1}}
    double2 *Rcur = p.rec[ti_cur];           //          {W_t (written by the updaters), g_t (RED by the consumers)}
    double2 *Rnext = p.rec[ti_next];         //          its g half is zeroed for step t+1
    const unsigned c_par = (unsigned)((t >> 1) & 1);
    const bool tl_cta = p.tl && t >= kTlFirst && t < kTlFirst + kTlSteps && blockIdx.x < kTlCtas;
    long long *tl_rec = tl_cta ? p.tl + 256 * 16 + ((t - kTlFirst) * kTlCtas + blockIdx.x) * kTlPerCta : nullptr;
    long long *tl_row = (p.tl && blockIdx.x == 0 && t < 256) ? p.tl + t * 16 : nullptr;
    bool ok = true;
    // kLrTable: the rate of step t, which interval t+1 applies, requested now, a whole interval before it is needed, and
    // installed after this interval's barrier.  The load completes while the interval works, so neither the barrier
    // (whose release arrival orders the thread's earlier memory operations) nor the next interval's update, which is on
    // the critical path, waits for it.
    double lr_next = lr;
    if constexpr (kLrTable) {
      if (!last) lr_next = __ldg(&p.lrs[t]);
    }
    if (warp == 0) DSGD_TL(0);

    // one GPU, update threads: g_{t-1} of the register columns, requested before anything else.  Update warp 0 then waits
    // for these loads and the accumulator's below in ONE round trip (the accumulator's asm loads, "memory" clobbers, would
    // otherwise hold them back until the accumulator had arrived: a second round trip before the CTA's partial is pushed).
    double gv[kUpdCols];
#pragma unroll
    for (int i = 0; i < kUpdCols; ++i) {
      const int j = u0 + i * n_upd;
      gv[i] = (!kMulti && is_upd && j < p.dim) ? __ldcg(&Rprev[j].y) : 0.0;
    }

    // ---- update warp 0, first thing: c_{T-1} and ||W_{T-1}||^2 from the partials the last barrier delivered ----
    if (warp == kCons && !first) {
      double c_prev, nrm_prev, l1_prev = 0.0;
      if (kMulti && t == 1) {
        c_prev = p.scal[kScalC];                              // W_base came from the host: k_prepare / previous launch
        nrm_prev = p.scal[kScalNrm2];
      } else {
        unsigned long long q0, q1, ql = 0, ol = 0;
        acc_load(acc_prev, lane, q0, q1);
        if constexpr (kL1) acc_load_l1(acc_prev, lane, ql, ol);   // in the same round trip
        double sd, sn;
        acc_sum(q0, q1, lane, sd, sn);
        c_prev = p.lambda * 2.0 * sd;
        nrm_prev = sn;
        if constexpr (kL1) l1_prev = acc_sum_l1(ql, ol, lane);
      }
      if (blockIdx.x == 0 && lane < (kL1 ? kAccStride : kAccWords)) acc_next[lane] = 0ull;
      if (lane == 0) {
        sm.c_val[t & 1] = c_prev;
        sm.nrm_val[t & 1] = nrm_prev;
        mbar_arrive(&sm.c_bar[t & 1]);
        // one GPU: the norms of the loss of step t-1, which is formed after the last step (epilogue)
        if (!kMulti && p.losses && blockIdx.x == 0) {
          p.loss_nrm[t - 1] = nrm_prev;
          if constexpr (kL1) p.loss_nrm[S + t - 1] = l1_prev;
        }
      }
      __syncwarp();
      DSGD_TL(9);
    }
    double pd = 0.0, pn = 0.0;   // this thread's share of W_T . d and ||W_T||^2
    double pa = 0.0;             // kL1: its share of ||W_T||_1
    const double tau = (kL1 && !first) ? lr * p.lambda1 : 0.0;   // interval 0 applies no update and no threshold
    // The CTA's partial {W_T . d, ||W_T||^2}: every warp that owns columns leaves its share in shared memory as soon as its
    // columns are done (no waiting); update warp 0 -- idle until the barrier anyway -- sums them in warp order and adds
    // ONE fixed-point value per CTA to the step's accumulator, well before the arrival.
    auto publish_partial = [&]() {
      pd = warp_sum(pd);
      pn = warp_sum(pn);
      if constexpr (kL1) pa = warp_sum(pa);
      if (lane == 0) {
        sm.red[warp][0] = pd;
        sm.red[warp][1] = pn;
        if constexpr (kL1) sm.red[warp - kCons][0] = pa;
        mbar_arrive(&sm.u_bar);
      }
      if (warp == kCons) {
        mbar_wait(&sm.u_bar, (unsigned)(t & 1), p.abort_flag, p.timeout_cycles);
        if (lane == 0) {
          double sd = 0.0, sn = 0.0;
#pragma unroll
          for (int i = kMulti ? 0 : kCons; i < kCons + kUpd; ++i) { sd += sm.red[i][0]; sn += sm.red[i][1]; }
          if (sd != 0.0 || sn != 0.0) acc_push(acc_cur, sd, sn);
          if constexpr (kL1) {
            double sa = 0.0;
#pragma unroll
            for (int i = 0; i < kUpd; ++i) sa += sm.red[i][0];
            if (sa != 0.0) acc_push_one(acc_cur + kAccWords, acc_cur + 2 * kAccLimbs, sa);
          }
        }
        __syncwarp();
      }
    };

    if constexpr (kMulti) {
      // ---------------------------------------------------------------------------------------------------
      // push g_{T-1} (sparse) and update this thread's column
      // ---------------------------------------------------------------------------------------------------
      unsigned long long *LWcur = p.llw[T & 1];               // LL words of W_T, tag T+1
      const int parp = (int)((T + 1) & 1);                    // receive parity of step T-1
      const unsigned gtag = (unsigned)T;                      // words of step T-1 carry tag T
      const unsigned wtag = (unsigned)(T + 1);                // W_T words carry tag T+1
      if ((int)threadIdx.x < slice) {                         // whole warps: slice is a multiple of 32
        if (first) {
          // W_base arrives as plain doubles from the host (wbuf[0]): publish it in LL form, no update pending
          if (col_act) {
            if (j_col < p.dim) ll_store(LWcur + 2 * (size_t)j_col, wreg[0], wtag);
            Gzero[j_col] = 0.0;
          }
        } else {
          double own = 0.0;
          if (col_act) {
            own = __ldcg(&Gprev[j_col]);
            if (j_col < p.dim) own = filt(own);               // a filtered-out entry is an absent key: not sent
          }
          const unsigned my_bits = __ballot_sync(0xffffffffu, own != 0.0);
          const bool warp_act = blockIdx.x * slice + (warp << 5) <= p.dim;   // the warp's first column exists
          if (warp_act) {
            const size_t vslot = 2 * (((size_t)me * 2 + parp) * p.xstride + (size_t)j_col);
            const size_t bslot = ((size_t)me * 2 + parp) * p.xwords + (size_t)col_word;
            for (int k = 0; k < K; ++k) {
              if (k == me) continue;
              if (lane == 0) ll_store32(p.xbm[k] + bslot, my_bits, gtag);
              if (own != 0.0) ll_store(p.xval[k] + vslot, own, gtag);
            }
            if (lane == 0) { st_bm += 1; st_val += (unsigned)__popc(my_bits); }
          }
          if (warp == 0) DSGD_TL(11);
          if (warp_act) {
            // bitmap words of the K-1 peers for this warp's 32 columns (one broadcast load each), then the value words
            // whose bit is set: everything requested before anything is waited for -- c_{T-1} included
            double raw[kMaxWorld];
            unsigned need = 0;   // bit k: value word of peer k still to be waited for
            double wn = wreg[0];                 // W_{T-1}[j_col]: this thread computed it one interval ago
            const unsigned long long *bm0 = p.xbm[me] + (size_t)parp * p.xwords + (size_t)col_word;
            const unsigned long long *vl0 = p.xval[me] + 2 * ((size_t)parp * p.xstride + (size_t)j_col);
            // All K-1 bitmap words are requested together and re-requested together until every one carries this step's
            // tag: the wait is the LATEST peer plus one poll, not a poll per peer in turn (polling one peer after the
            // other costs a round trip per peer).  Polling HARDER does not pay:
            // a second request set half a round trip behind the first made the 2-GPU step 8.6 -> 13.5 us, and requesting
            // every thread's value word along with the bitmap word (66 000 more requests per round) 8.5 -> 8.6 us --
            // the polled lines are the ones the NVLink writes are landing in.
            unsigned bits[kMaxWorld];
            unsigned pend = 0;   // bit k: bitmap word of peer k not here yet
#pragma unroll
            for (int k = 0; k < kMaxWorld; ++k) {
              raw[k] = (k == me) ? own : 0.0;
              bits[k] = 0u;
              if (k < K && k != me) pend |= 1u << k;
            }
            {
              unsigned spins = 0;
              const long long t0 = clock64();
              while (pend) {
#pragma unroll
                for (int k = 0; k < kMaxWorld; ++k)
                  if (pend & (1u << k)) {
                    if (ll_try_load32(bm0 + (size_t)k * 2 * p.xwords, gtag, bits[k])) pend &= ~(1u << k);
                  }
                if (pend && (++spins & 63u) == 0u && (clock64() - t0 > p.timeout_cycles || *(volatile int *)p.abort_flag)) {
                  *(volatile int *)p.abort_flag = 1;
                  ok = false;
#pragma unroll
                  for (int k = 0; k < kMaxWorld; ++k)
                    if (pend & (1u << k)) bits[k] = 0u;
                  pend = 0;
                }
              }
            }
#pragma unroll
            for (int k = 0; k < kMaxWorld; ++k)
              if (k < K && k != me && ((bits[k] >> lane) & 1u)) need |= 1u << k;
            // the value words of every peer that sent this column: requested together, looked at together
            auto poll_values = [&]() {
              unsigned long long v0[kMaxWorld], v1[kMaxWorld];
#pragma unroll
              for (int k = 0; k < kMaxWorld; ++k) {
                v0[k] = 0ull; v1[k] = 0ull;
                if (need & (1u << k))
                  asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];"
                               : "=l"(v0[k]), "=l"(v1[k]) : "l"(vl0 + 2 * (size_t)k * 2 * p.xstride) : "memory");
              }
#pragma unroll
              for (int k = 0; k < kMaxWorld; ++k)
                if ((need & (1u << k)) && (unsigned)(v0[k] >> 32) == gtag && (unsigned)(v1[k] >> 32) == gtag) {
                  raw[k] = __longlong_as_double((long long)((v0[k] & 0xffffffffull) | (v1[k] << 32)));
                  need &= ~(1u << k);
                }
            };
            if (need) poll_values();
            mbar_wait(&sm.c_bar[t & 1], c_par, p.abort_flag, p.timeout_cycles);
            const double c_prev = *(volatile double *)&sm.c_val[t & 1];
            const bool add_c = (c_prev != 0.0) && (fabs(c_prev) > kEps);
            if (col_act) {
              {
                unsigned spins = 0;
                const long long t0 = clock64();
                while (need) {
                  poll_values();
                  if (need && (++spins & 63u) == 0u && (clock64() - t0 > p.timeout_cycles || *(volatile int *)p.abort_flag)) {
                    *(volatile int *)p.abort_flag = 1;
                    ok = false;
                    need = 0;
                  }
                }
              }
              double s = 0.0;
#pragma unroll
              for (int k = 0; k < kMaxWorld; ++k) {
                if (k < K) {
                  if (j_col == p.dim) {
                    s += raw[k];                                // packed counters: plain sum
                  } else {
                    double v = filt(raw[k]);
                    if (v != 0.0 && add_c) v = filt(v + c_prev);  // regularize on this worker's own support
                    s = (k == 0) ? v : filt(s + v);               // Vec.sum: left fold over the replies
                  }
                }
              }
              if (j_col == p.dim) {
                if (p.losses) {  // loss of step T-1 on W_{T-1}: lambda*||W||^2 + (all ranks' hinge) / (all ranks' samples)
                  const double ns = floor(s / 4294967296.0);
                  p.losses[t - 1] = p.lambda * *(volatile double *)&sm.nrm_val[t & 1] + (s - ns * 4294967296.0) / ns;
                }
              } else {
                if (s != 0.0) {
                  const double mean = filt(s / (double)K);
                  const double step = filt(mean * lr);
                  wn = filt(wn - step);
                }
                wreg[0] = wn;
                if constexpr (kAvg) areg[0] = areg[0] + wn;   // W_T, T >= base + 1
                ll_store(LWcur + 2 * (size_t)j_col, wn, wtag);
                pd = filt(wn * dreg[0]);
                pn = wn * wn;
              }
              Gzero[j_col] = 0.0;
            }
          }
        }
      }
      if (warp == 0) DSGD_TL(12);
      publish_partial();
      if (is_cons && !last) {
        const int st = (int)t & (kStages - 1);
        auto &mt = sm.meta[st];
        mbar_wait(&sm.full[st], (unsigned)(((unsigned)t / kStages) & 1u), p.abort_flag, p.timeout_cycles);
        if (warp == 0) DSGD_TL(1);
        FetchLL fetch{LWcur, wtag, p.abort_flag, p.timeout_cycles};
        const unsigned hinge = consume_stage<kCons, kMaxChunks>(mt, &sm.ring[st][0], p.pairs, Gcur, 1, fetch, warp, lane,
                                                                          warp == 0 ? tl_row : nullptr);
        ok = ok && fetch.good;
        if (lane == 0 && hinge) atomicAdd(&sm.hinge_acc, hinge);
        if (tl_rec && warp == 0 && lane == 0) {
          tl_rec[2] = mt.n_pairs;
          tl_rec[3] = (long long)mt.n_chunks | ((long long)mt.n_multi << 32);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[st]);
        if (warp == 0) DSGD_TL(3);
      }
    } else {
      // ---------------------------------------------------------------------------------------------------
      // one GPU
      // ---------------------------------------------------------------------------------------------------
      if (is_cons) {
        if (!last) {
          const int st = (int)t & (kStages - 1);
          auto &mt = sm.meta[st];   // full: waited for by prefetch(t)
          FetchLocal<kL1> fetch{Rprev, &sm.c_bar[t & 1], c_par, &sm.c_val[t & 1], p.abort_flag, p.timeout_cycles, p.k_den, lr};
          if constexpr (kL1) fetch.tau = tau;
          const auto hinge = consume_stage<kCons, kMaxChunks, kWeight>(mt, &sm.ring[st][0], p.pairs, &Rcur[0].y, 2, fetch, warp,
                                                                       lane, warp == 0 ? tl_row : nullptr, &pre, p.w_pos, p.w_neg,
                                                                       kWeight == kSampleWeighted ? swm.row_c[st] : nullptr);
          if constexpr (kWeight == kSampleWeighted) {
            if (lane == 0 && hinge) atomicOr(&swm.code, hinge);
          } else {
            if (lane == 0 && hinge) atomicAdd(&sm.hinge_acc, hinge);
          }
          if (tl_rec && warp == 0 && lane == 0) {
            tl_rec[2] = mt.n_pairs;
            tl_rec[3] = (long long)mt.n_chunks | ((long long)mt.n_multi << 32);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.empty[st]);
          if (warp == 0) DSGD_TL(3);
        }
      } else {
        // ---- update warps: W_t <- update(W_{t-1}, g_{t-1}, c_{t-1}).  A thread owns the same (up to kUpdCols) columns for
        //      the whole launch: their W and d stay in registers, only g_{t-1} is read (requested before c is waited
        //      for), and W_t is stored only into the record buffers that do not hold it yet (the three buffers after a
        //      change), a g half is zeroed only if it was non-zero: most columns of a step cost one 8-byte load (gv,
        //      requested at the top of the interval) ----
        mbar_wait(&sm.c_bar[t & 1], c_par, p.abort_flag, p.timeout_cycles);
        const double c_prev = *(volatile double *)&sm.c_val[t & 1];
        const bool add_c = (c_prev != 0.0) && (fabs(c_prev) > kEps);
#pragma unroll
        for (int i = 0; i < kUpdCols; ++i) {
          const int j = u0 + i * n_upd;
          if (j < p.dim) {
            if (gv[i] != 0.0) {
              wreg[i] = apply_update(wreg[i], gv[i], c_prev, add_c, p.k_den, lr);
              ttl[i] = 3;
            }
            if constexpr (kL1) {
              const double wt = soft_threshold(wreg[i], tau);
              if (__double_as_longlong(wt) != __double_as_longlong(wreg[i])) { wreg[i] = wt; ttl[i] = 3; }
              pa += fabs(wreg[i]);
            }
            if (ttl[i] > 0) { Rcur[j].x = wreg[i]; --ttl[i]; }
            if (gnz[i]) Rnext[j].y = 0.0;          // held g_{t-2}, read for the last time during interval t-1
            gnz[i] = gv[i] != 0.0;
            if constexpr (kAvg) if (!first) areg[i] = areg[i] + wreg[i];   // W_t, t >= 1
            pd += filt(wreg[i] * dreg[i]);
            pn += wreg[i] * wreg[i];
          }
        }
        for (int j = u0 + kUpdCols * n_upd; j < p.dim; j += n_upd) {   // more columns than kUpdCols per update thread
          const double2 r = __ldcg(&Rprev[j]);
          double wn = apply_update(r.x, r.y, c_prev, add_c, p.k_den, lr);
          if constexpr (kL1) {
            wn = soft_threshold(wn, tau);
            pa += fabs(wn);
          }
          Rcur[j].x = wn;
          Rnext[j].y = 0.0;
          if constexpr (kAvg) if (!first) p.avg[j] = p.avg[j] + wn;
          pd += filt(wn * __ldg(&p.d[j]));
          pn += wn * wn;
        }
        if (warp == kCons) DSGD_TL(10);
        publish_partial();
      }
    }

    if (!ok) *(volatile int *)&sm.ok = 0;
    if (tl_row && lane == 0) sm.tl_warp[warp] = clock64();
    // Barrier 3: the CTA's work of the interval is done; only the thread that arrives at the grid barrier waits for it (one GPU:
    // the consumers arrive and load the next step's first chunk meanwhile).  Barrier 4: the grid barrier has passed.
    if (!kMulti && is_cons) {
      named_bar_arrive(3, kSyncThreads);
      if (t + 1 < S) prefetch(t + 1);
    } else {
      named_bar_sync(3, kSyncThreads);
    }
    ++phase;
    if (threadIdx.x == kCons * 32) {   // update warp 0, lane 0
      if (tl_row) {   // when the slowest consumer warp / update warp of CTA 0 reached the CTA barrier
        long long mc = 0, mu = 0;
        for (int i = 0; i < kCons; ++i) mc = max(mc, sm.tl_warp[i]);
        for (int i = kCons; i < kCons + kUpd; ++i) mu = max(mu, sm.tl_warp[i]);
        tl_row[13] = mc;
        tl_row[14] = mu;
      }
      unsigned h = 0;
      if (!last) {   // the CTA's hinge total; K GPUs add it and the step's sample count to the counter column before arriving
        h = sm.hinge_acc;
        if constexpr (kMulti) {
          if (h) red_add_f64(&Gcur[p.dim], (double)h);
          if (blockIdx.x == 0) red_add_f64(&Gcur[p.dim], (double)B * 4294967296.0);
        }
        sm.hinge_acc = 0u;
      }
      if (tl_rec) tl_rec[0] = global_ns();
      else if (tl_row) tl_row[6] = clock64();
      bool bar_ok = grid_barrier_arrive_wait(p.bar, phase * (unsigned)G, p.abort_flag, p.timeout_cycles);
      if (*(volatile int *)&sm.ok == 0) { *(volatile int *)p.abort_flag = 1; bar_ok = false; }
      sm.ok = bar_ok ? 1 : 0;
      if (tl_rec) tl_rec[1] = global_ns();
      else if (tl_row) tl_row[7] = clock64();
      // one GPU: the CTA's hinge count of step t into its own slot, zero included.  A plain store after the barrier: the
      // release of this arrival does not wait for it (a count shared by all CTAs was one same-address atomic per CTA in front
      // of every arrival), and the next one finds it long done.  Nothing reads it before the epilogue.
      if (!kMulti && !last && p.losses) p.hinge[(size_t)t * G + blockIdx.x] = h;
      // sample-weighted: the rows' hinge codes of step t, the same way.  Every consumer warp OR'd its codes in before
      // barrier 3, and the consumers of step t + 1 start after barrier 4: the word is read and cleared in between.
      if constexpr (kWeight == kSampleWeighted) {
        if (!last) {
          if (p.losses) p.hcode[(size_t)t * G + blockIdx.x] = swm.code;
          swm.code = 0ull;
        }
      }
    }
    named_bar_sync(4, kSyncThreads);
    if (*(volatile int *)&sm.ok == 0) return;
    if constexpr (kLrTable) lr = lr_next;
    { const int a = gi_prev; gi_prev = gi_cur; gi_cur = gi_next; gi_next = a; }
    { const int a = ti_prev; ti_prev = ti_cur; ti_cur = ti_next; ti_next = a; }
  }

  // ---- epilogue: publish W_{base+S} as the resident weights ----------------------------------------------------
  if (blockIdx.x == 0 && warp == kCons && S > 0) {
    double sd, sn;
    acc_read(p.acc + (size_t)ti_prev * kAccStride, lane, sd, sn);   // partials of W_S: complete at the last barrier
    double l1 = 0.0;
    if constexpr (kL1) l1 = acc_read_l1(p.acc + (size_t)ti_prev * kAccStride, lane);
    if (lane == 0) {
      p.scal[kScalC] = p.lambda * 2.0 * sd;
      p.scal[kScalNrm2] = sn;
      if constexpr (kL1) p.scal[kScalL1] = l1;
    }
  }
  // one GPU: loss of step s = lambda*||W_s||^2 (+ lambda1*||W_s||_1) + hinge_s/batch (SparseSVM.scala:20-23; SURVEY.md F5), one
  // warp per step.  The hinge count is the integer sum of the CTAs' slots, the same in any order.  Every slot and norm was
  // stored before the last barrier's arrivals, and is read through L2 (see grid_barrier_arrive_wait).
  if constexpr (!kMulti && kWeight != kSampleWeighted) {
    if (p.losses) {
      for (int64_t s = (int64_t)blockIdx.x * (kCons + kUpd) + warp; s < S; s += (int64_t)G * (kCons + kUpd)) {
        unsigned h = 0;
        if constexpr (kWeight == kClassWeighted) {   // the halves are summed apart: G slots of at most 64 each
          unsigned hn = 0;
          for (int b = lane; b < G; b += 32) {
            const unsigned v = __ldcg(&p.hinge[s * G + b]);
            h += v & 0xffffu;
            hn += v >> 16;
          }
          h = __reduce_add_sync(0xffffffffu, h);
          hn = __reduce_add_sync(0xffffffffu, hn);
          if (lane == 0) {
            const double hp_w = p.w_pos * (double)h, hn_w = p.w_neg * (double)hn;
            double pen = p.lambda * __ldcg(&p.loss_nrm[s]);
            if constexpr (kL1) pen = pen + p.lambda1 * __ldcg(&p.loss_nrm[S + s]);
            p.losses[s] = pen + (hp_w + hn_w) / (double)B;
          }
        } else {
          for (int b = lane; b < G; b += 32) h += __ldcg(&p.hinge[s * G + b]);
          h = __reduce_add_sync(0xffffffffu, h);
          if (lane == 0) {
            if constexpr (kL1)
              p.losses[s] = p.lambda * __ldcg(&p.loss_nrm[s]) + p.lambda1 * __ldcg(&p.loss_nrm[S + s]) + (double)h / (double)B;
            else
              p.losses[s] = p.lambda * __ldcg(&p.loss_nrm[s]) + (double)h / (double)B;
          }
        }
      }
    }
  }
  if constexpr (kMulti) {
    const unsigned long long *LW = p.llw[(base + S) & 1];
    const unsigned wtag = (unsigned)(base + S + 1);
    const int n_all = G * kSyncThreads;
    for (int j = blockIdx.x * kSyncThreads + threadIdx.x; j < p.dim; j += n_all) {
      double wv = 0.0;
      ll_try_load(LW + 2 * (size_t)j, wtag, wv);             // complete: written before the last grid barrier
      p.w_out[j] = wv;
      p.w32_out[j] = (float)wv;
    }
    if (p.xstats && lane == 0 && (st_val | st_bm)) {
      atomicAdd(&p.xstats[0], st_val);
      atomicAdd(&p.xstats[1], st_bm);
    }
    if constexpr (kAvg) {
      if (col_act && j_col < p.dim) p.avg[j_col] = areg[0];
    }
  } else if (is_upd) {
    const double2 *Rfin = p.rec[ti_prev];
#pragma unroll
    for (int i = 0; i < kUpdCols; ++i) {
      const int j = u0 + i * n_upd;
      if (j < p.dim) {
        p.w_out[j] = wreg[i];
        p.w32_out[j] = (float)wreg[i];
        if constexpr (kAvg) p.avg[j] = areg[i];
      }
    }
    for (int j = u0 + kUpdCols * n_upd; j < p.dim; j += n_upd) {
      const double wv = __ldcg(&Rfin[j]).x;
      p.w_out[j] = wv;
      p.w32_out[j] = (float)wv;
    }
  }
  // sample-weighted: the loss of step s = lambda*||W_s||^2 (+ lambda1*||W_s||_1) + S_s / batch, S_s = sum R(c_i * code_i)
  // over the step's rows (row i of the step is row i / G of CTA i % G), summed in fixed-point limbs: the same bits in any
  // order.  After the weights are stored, so that the limbs do not share the registers that hold them.
  if constexpr (kWeight == kSampleWeighted) {
    if (p.losses) {
      for (int64_t s = (int64_t)blockIdx.x * (kCons + kUpd) + warp; s < S; s += (int64_t)G * (kCons + kUpd)) {
        unsigned long long lim[kLossLimbs] = {0, 0, 0, 0, 0, 0}, ovf = 0;
        for (int i = lane; i < B; i += 32) {
          const int b = i % G, m = i / G;
          const unsigned code = (unsigned)(__ldcg(&p.hcode[s * G + b]) >> (2 * m)) & 3u;
          const int32_t id = __ldg(&p.samples[s * B + i]);
          const double c = (__ldg(&p.label[id]) > 0 ? p.w_pos : p.w_neg) * __ldg(&p.sw[id]);
          acc_add_local(lim, ovf, c * (double)code);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {   // limbs 0..4 below 2^40 per lane: the warp's sums stay below 2^45
#pragma unroll
          for (int k = 0; k < kLossLimbs; ++k) lim[k] += __shfl_xor_sync(0xffffffffu, lim[k], o);
          ovf += __shfl_xor_sync(0xffffffffu, ovf, o);
        }
        if (lane == 0) {
          unsigned long long q[kLossAccWords];
#pragma unroll
          for (int k = 0; k < kLossLimbs; ++k) q[k] = lim[k];
          q[kLossLimbs] = ovf;
          double pen = p.lambda * __ldcg(&p.loss_nrm[s]);
          if constexpr (kL1) pen = pen + p.lambda1 * __ldcg(&p.loss_nrm[S + s]);
          p.losses[s] = pen + acc_value(q) / (double)B;
        }
      }
    }
  }
}

// One GPU: the records a launch starts from -- all three buffers = {W, 0}.
__global__ void __launch_bounds__(256) k_rec_init(const double *__restrict__ w, int dim, double2 *__restrict__ rec0,
                                                  double2 *__restrict__ rec1, double2 *__restrict__ rec2) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < dim) {
    const double2 r = make_double2(w[j], 0.0);
    rec0[j] = r;
    rec1[j] = r;
    rec2[j] = r;
  }
}

}  // namespace dsgd
