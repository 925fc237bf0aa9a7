// dsgd_async.cuh -- asynchronous (Hogwild) worker loop as a persistent kernel with lock-free peer writes.
//
// Reference: Slave.asyncTask (core/Slave.scala:79-111) + SlaveImpl.updateGrad (177-185) +
// AsyncMasterGrpcImpl.updateGrad (core/MasterAsync.scala:164-177).  Per iteration the reference worker
//   samples a batch, snapshots its weights, computes  delta = lr * regularize(mean_i backward(w, x_i, y_i), w),
//   applies  w_self -= delta, and sends the SAME sparse delta to every peer slave and to the master, which each
//   apply  w -= delta  (the master also counts updates).
// Here every replica (peers' and the master's) is mapped into this GPU's address space over NVLink and the
// "send" is a system-scope fp64 reduction (red.add of -delta_j) straight into peer memory: no message, no
// lock, uniform cost to every peer through the NVSwitch.
//
// One Hogwild LANE is one warp running the loop body; `concurrency` lanes share this GPU's replica (1 lane ==
// the reference's strictly sequential loop).  c = 2*lambda*(w . d) needs the whole weight vector every iteration
// in the reference; each replica instead carries S = w . d in a control slot, and whoever applies a delta to a
// replica also applies  S -= sum_j delta_j d_j  to it -- O(nnz) instead of O(dim), same value up to fp64 rounding.
//
// Every replica update of the reference builds a new Sparse (`weights.single.transform(_ - gradUpdate)`, core/Slave.scala:
// 101, 180; `grad - gradUpdate`, core/ml/GradState.scala:8), so an entry with |w - delta| <= 1e-20 leaves the map.  A red.add
// cannot filter its result; instead the lane checks its snapshot wv of the entry after sending -delta: when wv - delta is tiny
// and nonzero it sends that residual as well, so the entry lands on exactly 0 (async_apply_key).  Every replica, the outbox
// and S receive the same amounts.  The check follows the red.adds, so the common case waits for nothing new.  With one lane the
// snapshot is the entry, so this is the reference's arithmetic exactly; with concurrent lanes another lane may move the entry
// between the snapshot and the red.add (DESIGN.md 4.4).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dsgd_feistel.h"
#include "dsgd_kernels.cuh"

namespace dsgd {

constexpr int kMaxReplicas = 17;  // 16 workers + the master replica
// control slots that follow the dim weights (and two spare doubles) of every replica block
constexpr int kCtlS = 2;        // double: S = w . d of this replica
constexpr int kCtlUpdates = 3;  // unsigned long long: updates applied to this replica's owner (the master's counter)
constexpr int kReplicaPad = 8;  // doubles after the weights

struct AsyncParams {
  const uint32_t *rp16;
  const uint2 *pairs;
  const int8_t *label;
  const double *d;
  int dim;
  const int32_t *assigned;  // row ids this worker may sample (StartAsyncRequest.samples)
  int64_t n_assigned;
  const int32_t *replay;    // explicit sequence of max_updates * batch row ids, or nullptr (sample on the device)
  int batch;
  double lr, lambda;
  double *replica[kMaxReplicas];  // [0] = own replica; then peers; the master last if present
  int n_replicas;
  int master_slot;          // index into replica[] of the master replica, or -1
  double *scratch;          // [n_lanes][dim] zero on entry and exit: per-lane batch accumulator
  int32_t *batch_rows;      // [n_lanes][batch]
  int n_lanes;
  long long max_updates;    // total over lanes; <= 0: until stopped
  unsigned long long seed;
  volatile int *stop;       // raised by dsgd_stop_async
  unsigned long long *claimed;  // next iteration number to claim (lanes race for iterations)
  unsigned long long *done;     // iterations finished by this worker
};

// w -= delta on key j of every replica, the result filtered against the snapshot wv (math/Sparse.scala:108-118); sd += the
// amount times d_j
__device__ __forceinline__ void async_apply_key(const AsyncParams &p, int j, double wv, double delta, double dj, double &sd) {
  for (int q = 0; q < p.n_replicas; ++q) red_add_f64_sys(&p.replica[q][j], -delta);
  sd += delta * dj;
  const double nw = wv - delta;
  if (nw != 0.0 && fabs(nw) <= kEps) {   // the entry would keep a residual the reference's new Sparse drops
    for (int q = 0; q < p.n_replicas; ++q) red_add_f64_sys(&p.replica[q][j], -nw);
    sd += nw * dj;
  }
}

__device__ __forceinline__ unsigned long long mix64(unsigned long long &s) {
  unsigned long long z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// `Random.shuffle(indices) take batchSize` (core/Slave.scala:86-88): the first B images of a keyed pseudo-random permutation
// of [0, n) (dsgd_feistel.h).  The rejection loop of round 1 compared each candidate with all earlier ones on one lane:
// milliseconds per batch of 256 or 1024.
// One row of a batch, requested one row ahead of its use: window bounds, label and the first 128 pairs.
struct AsyncBatchRow {
  int64_t s0, s1;
  double y;
  uint2 pre[4];
};
__device__ __forceinline__ AsyncBatchRow async_fetch_batch_row(const AsyncParams &p, const int32_t *rows, int b, int B, int lane) {
  AsyncBatchRow row;
  row.s0 = row.s1 = 0;
  row.y = 0.0;
#pragma unroll
  for (int u = 0; u < 4; ++u) row.pre[u] = make_uint2(0u, 0u);
  if (b >= B) return row;
  const int32_t r = rows[b];
  row.s0 = (int64_t)__ldg(&p.rp16[r]) * 2;
  row.s1 = (int64_t)__ldg(&p.rp16[r + 1]) * 2;
  row.y = (double)__ldg(&p.label[r]);
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int64_t k = row.s0 + lane + 32 * u;
    if (k < row.s1) row.pre[u] = __ldg(&p.pairs[k]);
  }
  return row;
}

__global__ void __launch_bounds__(128) k_async_worker(const AsyncParams p) {
  const int lane = threadIdx.x & 31;
  const int lane_id = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);  // Hogwild lane
  if (lane_id >= p.n_lanes) return;
  double *w = p.replica[0];
  double *scratch = p.scratch + (size_t)lane_id * p.dim;
  int32_t *rows = p.batch_rows + (size_t)lane_id * p.batch;
  const int B = p.batch;
  unsigned long long rng = p.seed * 0xD1342543DE82EF95ull + 0x632BE59BD9B4E019ull * (unsigned long long)(lane_id + 1);
  const int half_bits = dsgd_feistel_half_bits((uint64_t)p.n_assigned);

  for (;;) {
    if (*p.stop) break;
    // claim the next iteration (keeps the total bounded and, with a replay sequence, deals the recorded batches)
    unsigned long long it = 0;
    if (lane == 0) it = atomicAdd(p.claimed, 1ull);
    it = __shfl_sync(0xffffffffu, it, 0);
    if (p.max_updates > 0 && it >= (unsigned long long)p.max_updates) break;

    // ---- 1. the batch (core/Slave.scala:83-88) ----
    if (p.replay) {
      for (int b = lane; b < B; b += 32) rows[b] = p.replay[it * (unsigned long long)B + b];
    } else if (B == 1) {
      // data(assignedSamples(Random.nextInt(size)))
      if (lane == 0) rows[0] = p.assigned[mix64(rng) % (unsigned long long)p.n_assigned];
    } else {
      // Random.shuffle(assignedSamples.indices) take batchSize map data: POSITIONS 0..n-1 index `data` directly
      // (quirk Q6), drawn without replacement: the first B images of this iteration's permutation
      unsigned long long key = 0;
      if (lane == 0) key = mix64(rng);
      key = __shfl_sync(0xffffffffu, key, 0);
      for (int b = lane; b < B; b += 32) rows[b] = (int32_t)dsgd_feistel((uint32_t)b, half_bits, key, (uint32_t)p.n_assigned);
    }
    __syncwarp();

    // ---- 2. c from the replica's running S = w . d (SparseSVM.scala:31) ----
    const double S = *(volatile double *)&w[p.dim + kCtlS];
    const double c = p.lambda * 2.0 * S;
    const bool add_c = (c != 0.0) && (fabs(c) > kEps);

    // ---- 3. backward per sample against the current replica, summed into the lane's scratch.  Row b + 1 (bounds, label,
    //         first 128 pairs: nothing that depends on the weights) is requested before row b is worked on ----
    {
      AsyncBatchRow cur = async_fetch_batch_row(p, rows, 0, B, lane);
      for (int b = 0; b < B; ++b) {
        const AsyncBatchRow nxt = async_fetch_batch_row(p, rows, b + 1, B, lane);
        double wv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) wv[u] = (cur.pre[u].y << 1) ? __ldcg(&w[cur.pre[u].x]) : 0.0;
        double acc = 0.0;   // the row fold (dsgd_kernels.cuh): chunk 0 from the registers, the chunks past it from memory
#pragma unroll
        for (int u = 0; u < 4; ++u) acc += filt(filt((double)__uint_as_float(cur.pre[u].y)) * wv[u]);
        const double dot = row_fold_from(p.pairs, cur.s0 + kFoldPairs, cur.s1, lane, warp_sum(acc),
                                         [&](uint32_t c) { return __ldcg(&w[c]); });
        if (!(cur.y * dot < 0.0)) {  // SparseSVM.scala:28
          // Vec.sum: left fold in batch order, filter after each +.  A column occurs once per row (dsgd_load_csr rejects
          // repeated keys), so the lane's four read-modify-writes are independent -- all four scratch entries are requested
          // before the first is used (one L2 round trip instead of four dependent ones)
          double gv[4], sv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            gv[u] = (cur.s0 + lane + 32 * u < cur.s1) ? filt(filt((double)__uint_as_float(cur.pre[u].y)) * cur.y) : 0.0;
            sv[u] = (gv[u] != 0.0) ? scratch[cur.pre[u].x] : 0.0;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u)
            if (gv[u] != 0.0) scratch[cur.pre[u].x] = filt(sv[u] + gv[u]);
          for (int64_t k = cur.s0 + 128 + lane; k < cur.s1; k += 32) {
            const uint2 pr = p.pairs[k];
            const double g = filt(filt((double)__uint_as_float(pr.y)) * cur.y);
            if (g != 0.0) scratch[pr.x] = filt(scratch[pr.x] + g);
          }
        }
        __syncwarp();
        cur = nxt;
      }
    }

    // ---- 4. delta = lr * regularize(sum / B, w) on the summed support; apply to every replica ----
    double sd = 0.0;  // sum_j delta_j * d_j
    {
      AsyncBatchRow cur = async_fetch_batch_row(p, rows, 0, B, lane);
      for (int b = 0; b < B; ++b) {
        const AsyncBatchRow nxt = async_fetch_batch_row(p, rows, b + 1, B, lane);
        // the key's summed value v, its dimSparsity factor and the replica's snapshot wv of it -> delta applied to every
        // replica; the first row of the batch that holds the key claims it (the next rows see 0)
        auto apply_key = [&](const int j, const double v, const double dj, const double wv) {
          scratch[j] = 0.0;                           // claim the key
          double m = filt(v / (double)B);             // Vec.mean = sum / size (math/Vec.scala:139)
          if (m != 0.0 && add_c) m = filt(m + c);     // regularize on the surviving keys
          const double delta = filt(m * p.lr);        // learningRate * (...)
          if (delta != 0.0) async_apply_key(p, j, wv, delta, dj, sd);
        };
        double v4[4], d4[4], w4[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {   // the lane's four entries, their dimSparsity factors and weights: requested together
          // a padding pair repeats the row's last column with val == 0: only the real pair may claim the key
          const bool live = (cur.s0 + lane + 32 * u < cur.s1) && filt((double)__uint_as_float(cur.pre[u].y)) != 0.0;
          v4[u] = live ? scratch[cur.pre[u].x] : 0.0;
          d4[u] = live ? __ldg(&p.d[cur.pre[u].x]) : 0.0;
          w4[u] = live ? __ldcg(&w[cur.pre[u].x]) : 0.0;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (v4[u] != 0.0) apply_key(cur.pre[u].x, v4[u], d4[u], w4[u]);
        for (int64_t k = cur.s0 + 128 + lane; k < cur.s1; k += 32) {
          const uint2 pr = p.pairs[k];
          if (filt((double)__uint_as_float(pr.y)) == 0.0) continue;
          const double v = scratch[pr.x];
          if (v != 0.0) apply_key(pr.x, v, p.d[pr.x], __ldcg(&w[pr.x]));
        }
        __syncwarp();
        cur = nxt;
      }
    }
    sd = warp_sum(sd);
    if (lane == 0) {
      if (sd != 0.0)
        for (int q = 0; q < p.n_replicas; ++q) red_add_f64_sys(&p.replica[q][p.dim + kCtlS], -sd);
      if (p.master_slot >= 0)
        red_add_u64_sys(reinterpret_cast<unsigned long long *>(&p.replica[p.master_slot][p.dim + kCtlUpdates]), 1ull);
      __threadfence_system();
      atomicAdd(p.done, 1ull);
    }
    __syncwarp();
  }
}

// Batch 1 on rows with unique columns (dsgd_load_csr checks; the reference's rows are Maps): the loop body of
// BASELINE.json configs[3] -- one sample per update -- without the per-lane scratch vector.  With one sample the batch sum IS
// the row's backward (sum = 0 + y*x, mean = sum / 1.0), so the delta of every non-zero is formed straight from the pair.
// An update is a chain of dependent latencies (sample id -> row pointers -> row window from HBM -> weight gathers from
// L2 -> reduce -> REDs), and with `concurrency` = 1 (the reference's one sequential loop per slave, core/Slave.scala:79-111)
// throughput is 1 / chain.  What does not depend on the weights leaves the chain: the NEXT iteration's sample id, row
// pointers, label and the first 128 pairs of its window are fetched while the current iteration computes; the deltas go
// out as fire-and-forget REDs (the reference's updateGrad futures are not awaited either, core/Slave.scala:104-105) and
// are fenced once, when the loop ends; the stop flag is looked at every 32 iterations.
constexpr int kAsyncPre = 4;   // pairs per lane held in registers for the next row
static_assert(32 * kAsyncPre == kFoldPairs, "the registers hold chunk 0 of the row fold");
struct AsyncRow {
  int64_t s0, s1;
  double y;
  uint2 pre[kAsyncPre];
  bool valid;
};
__device__ __forceinline__ AsyncRow async_fetch_row(const AsyncParams &p, bool have, unsigned long long it, unsigned long long &rng,
                                                    int lane) {
  AsyncRow row;
  row.valid = have;
  row.s0 = row.s1 = 0;
  row.y = 0.0;
#pragma unroll
  for (int u = 0; u < kAsyncPre; ++u) row.pre[u] = make_uint2(0u, 0u);
  if (!have) return row;
  int32_t r = 0;
  if (lane == 0)   // data(assignedSamples(Random.nextInt(size)))  (core/Slave.scala:84)
    r = p.replay ? __ldg(&p.replay[it]) : __ldg(&p.assigned[mix64(rng) % (unsigned long long)p.n_assigned]);
  r = __shfl_sync(0xffffffffu, r, 0);
  row.s0 = (int64_t)__ldg(&p.rp16[r]) * 2;
  row.s1 = (int64_t)__ldg(&p.rp16[r + 1]) * 2;
  row.y = (double)__ldg(&p.label[r]);
#pragma unroll
  for (int u = 0; u < kAsyncPre; ++u) {
    const int64_t k = row.s0 + lane + 32 * u;
    if (k < row.s1) row.pre[u] = __ldg(&p.pairs[k]);
  }
  return row;
}

__global__ void __launch_bounds__(128) k_async_worker_b1(const AsyncParams p) {
  const int lane = threadIdx.x & 31;
  const int lane_id = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (lane_id >= p.n_lanes) return;
  double *w = p.replica[0];
  unsigned long long rng = p.seed * 0xD1342543DE82EF95ull + 0x632BE59BD9B4E019ull * (unsigned long long)(lane_id + 1);
  // iterations are claimed from a shared counter (keeps the total bounded and deals a replay sequence in order); a
  // single lane just counts
  unsigned long long local_it = 0;
  auto claim = [&](unsigned long long &it) -> bool {
    if (p.n_lanes == 1) {
      it = local_it++;
    } else {
      unsigned long long v = 0;
      if (lane == 0) v = atomicAdd(p.claimed, 1ull);
      it = __shfl_sync(0xffffffffu, v, 0);
    }
    return !(p.max_updates > 0 && it >= (unsigned long long)p.max_updates);
  };
  unsigned long long it = 0, it_next = 0;
  bool have = claim(it);
  AsyncRow cur = async_fetch_row(p, have, it, rng, lane);
  unsigned n_done = 0;
  while (cur.valid) {
    bool stop = false;
    if ((n_done & 31u) == 0u) stop = (*p.stop != 0);
    const bool have_next = !stop && claim(it_next);
    const AsyncRow nxt = async_fetch_row(p, have_next, it_next, rng, lane);   // in flight while this iteration computes

    // ---- c from the replica's running S = w . d (SparseSVM.scala:31) ----
    const double S = *(volatile double *)&w[p.dim + kCtlS];
    const double c = p.lambda * 2.0 * S;
    const bool add_c = (c != 0.0) && (fabs(c) > kEps);
    const double y = cur.y;

    // ---- backward against the current replica: x . w, gate (SparseSVM.scala:26-29) ----
    double wv[kAsyncPre];
#pragma unroll
    for (int u = 0; u < kAsyncPre; ++u) wv[u] = (cur.pre[u].y << 1) ? __ldcg(&w[cur.pre[u].x]) : 0.0;
    double acc = 0.0;   // the row fold (dsgd_kernels.cuh): chunk 0 from the registers, the chunks past it from memory
#pragma unroll
    for (int u = 0; u < kAsyncPre; ++u) acc += filt(filt((double)__uint_as_float(cur.pre[u].y)) * wv[u]);
    const double dot = row_fold_from(p.pairs, cur.s0 + kFoldPairs, cur.s1, lane, warp_sum(acc),
                                     [&](uint32_t c) { return __ldcg(&w[c]); });

    // ---- delta = lr * regularize(y * x / 1, w); apply to every replica (core/Slave.scala:92-105) ----
    double sd = 0.0;
    if (!(y * dot < 0.0)) {
      // wv: the snapshot of the entry the dot product used (reloaded for the pairs past the first 128)
      auto push = [&](uint2 pr, double wv) {
        const double xv = filt((double)__uint_as_float(pr.y));
        if (xv == 0.0) return;                          // padding pair (or an explicit zero): no key
        double m = filt(filt(xv * y) / 1.0);            // Vec.sum of one vector, Vec.mean = sum / size
        if (m != 0.0 && add_c) m = filt(m + c);
        const double delta = filt(m * p.lr);
        if (delta != 0.0) async_apply_key(p, pr.x, wv, delta, __ldg(&p.d[pr.x]), sd);
      };
#pragma unroll
      for (int u = 0; u < kAsyncPre; ++u) push(cur.pre[u], wv[u]);
      for (int64_t k = cur.s0 + lane + 32 * kAsyncPre; k < cur.s1; k += 32) {
        const uint2 pr = __ldg(&p.pairs[k]);
        push(pr, __ldcg(&w[pr.x]));
      }
    }
    sd = warp_sum(sd);
    if (lane == 0) {
      if (sd != 0.0)
        for (int q = 0; q < p.n_replicas; ++q) red_add_f64_sys(&p.replica[q][p.dim + kCtlS], -sd);
      if (p.master_slot >= 0)
        red_add_u64_sys(reinterpret_cast<unsigned long long *>(&p.replica[p.master_slot][p.dim + kCtlUpdates]), 1ull);
      atomicAdd(p.done, 1ull);
    }
    __syncwarp();
    ++n_done;
    cur = nxt;
  }
  __threadfence_system();   // every delta of this lane is visible in every replica before the kernel reports completion
}

// weights -= delta for a sparse delta, keeping S in step (core/Slave.scala:177-185; core/ml/GradState.scala:8)
__global__ void __launch_bounds__(256) k_async_apply_delta(double *__restrict__ w, int dim, const double *__restrict__ d,
                                                           const int32_t *__restrict__ idx,
                                                           const double *__restrict__ val, int64_t nnz, int count_update) {
  __shared__ double red[8];
  double sd = 0.0;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
    const double v = filt(val[k]);
    if (v != 0.0) {
      // w - v, filtered: a tiny nonzero result is taken out as well, so the entry lands on exactly 0
      const double nw = atomicAdd_system(&w[idx[k]], -v) - v;
      sd += v * d[idx[k]];
      if (nw != 0.0 && fabs(nw) <= kEps) {
        atomicAdd_system(&w[idx[k]], -nw);
        sd += nw * d[idx[k]];
      }
    }
  }
  sd = block_sum<256>(sd, red);
  if (threadIdx.x == 0) {
    if (sd != 0.0) atomicAdd_system(&w[dim + kCtlS], -sd);
    if (count_update && blockIdx.x == 0)
      atomicAdd_system(reinterpret_cast<unsigned long long *>(&w[dim + kCtlUpdates]), 1ull);
  }
}

// S = w . d into the replica's control slot (fixed order), used when weights are installed
template <int kThreads>
__global__ void __launch_bounds__(kThreads) k_async_init_ctl(double *__restrict__ w, const double *__restrict__ d, int dim) {
  __shared__ double red[kThreads / 32];
  double s = 0.0;
  for (int j = threadIdx.x; j < dim; j += kThreads) s += filt(w[j] * d[j]);
  s = block_sum<kThreads>(s, red);
  if (threadIdx.x == 0) {
    w[dim + kCtlS] = s;
    reinterpret_cast<unsigned long long *>(w)[dim + kCtlUpdates] = 0ull;
  }
}

}  // namespace dsgd
