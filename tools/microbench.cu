// Dev microbenchmarks for the latency model of the persistent SGD kernel (sm_90a).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench microbench.cu && ./microbench
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>
namespace cg = cooperative_groups;
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1);} } while (0)

__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned *p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_relaxed_gpu(const unsigned *p) { unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void red_release_gpu_add(unsigned *p, unsigned v) { asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red_relaxed_gpu_add(unsigned *p, unsigned v) { asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// 1. pointer chase: latency of dependent loads (.cg = L2, default = L1 allowed)
template <int MODE>
__global__ void k_chase(const unsigned *chain, int hops, long long *out, unsigned *sink) {
  unsigned i = 0;
  long long t0 = clock64();
  for (int h = 0; h < hops; ++h) {
    if (MODE == 0) i = __ldcg(&chain[i]);
    else if (MODE == 1) i = chain[i];
    else i = ld_relaxed_gpu(&chain[i]);
  }
  long long t1 = clock64();
  *out = (t1 - t0) / hops;
  *sink = i;
}

// 2. grid barrier cost: G CTAs, each interval does nothing but the barrier
template <int MODE>
__global__ void k_barrier(unsigned *bar, int iters, long long *out) {
  __shared__ int dummy;
  long long t0 = clock64();
  for (int it = 1; it <= iters; ++it) {
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned target = (unsigned)it * gridDim.x;
      if (MODE == 0) { red_release_gpu_add(bar, 1u); while (ld_acquire_gpu(bar) < target) {} }
      else if (MODE == 1) { __threadfence(); atomicAdd(bar, 1u); while (*(volatile unsigned *)bar < target) {} __threadfence(); }
      else { red_relaxed_gpu_add(bar, 1u); while (ld_relaxed_gpu(bar) < target) {} }
      dummy = it;
    }
    __syncthreads();
  }
  long long t1 = clock64();
  if (blockIdx.x == 0 && threadIdx.x == 0) *out = (t1 - t0) / iters;
}
__global__ void k_cg_barrier(int iters, long long *out) {
  cg::grid_group g = cg::this_grid();
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) g.sync();
  long long t1 = clock64();
  if (blockIdx.x == 0 && threadIdx.x == 0) *out = (t1 - t0) / iters;
}

// 3. RED throughput: each of nthreads does `reps` REDs; addresses either all distinct-ish or a few hot ones
template <typename T>
__global__ void k_red(T *buf, int n_addr, int reps, long long *out) {
  const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
  long long t0 = clock64();
  unsigned a = tid * 2654435761u;
  for (int r = 0; r < reps; ++r) { a = a * 1664525u + 1013904223u; atomicAdd(&buf[(a >> 8) % n_addr], (T)1); }
  __threadfence();
  long long t1 = clock64();
  if (tid == 0) *out = (t1 - t0);
}

// 4. store -> release -> observe latency: CTA 0 writes a flag, CTA 1 polls it; round trip ping-pong
__global__ void k_pingpong(unsigned *flags, int iters, long long *out) {
  if (threadIdx.x != 0) return;
  long long t0 = clock64();
  if (blockIdx.x == 0) {
    for (int it = 1; it <= iters; ++it) { red_release_gpu_add(&flags[0], 1u); while (ld_acquire_gpu(&flags[32]) < (unsigned)it) {} }
    *out = (clock64() - t0) / iters;
  } else {
    for (int it = 1; it <= iters; ++it) { while (ld_acquire_gpu(&flags[0]) < (unsigned)it) {} red_release_gpu_add(&flags[32], 1u); }
  }
}


// 5. the flag barrier of dsgd_persistent.cuh (kOpt & 1): arrivals on a counter nobody polls, last arriver raises one
//    flag per group of GROUP CTAs.  PRE_RED: every thread issues one fp64 RED before arriving (what a step does).
__device__ __forceinline__ unsigned atom_acq_rel_gpu_add(unsigned *p, unsigned v) {
  unsigned old; asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory"); return old;
}
template <int GROUP, bool PRE_RED, bool FLAGS>
__global__ void k_barrier2(unsigned *bar, unsigned *flags, double *buf, int iters, long long *out) {
  __shared__ int dummy;
  unsigned a = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
  long long t0 = clock64();
  for (int it = 1; it <= iters; ++it) {
    if (PRE_RED) { a = a * 1664525u + 1013904223u; atomicAdd(&buf[(a >> 8) % 47236], 1.0); }
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned target = (unsigned)it * gridDim.x;
      if (FLAGS) {
        const unsigned old = atom_acq_rel_gpu_add(bar, 1u);
        if (old + 1u == target) {
          asm volatile("fence.acq_rel.gpu;" ::: "memory");
          for (unsigned g = 0; g < (gridDim.x + GROUP - 1) / GROUP; ++g)
            asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(flags + g * 32), "r"((unsigned)it) : "memory");
        } else {
          const unsigned *f = flags + (blockIdx.x / GROUP) * 32;
          while ((int)(ld_relaxed_gpu(f) - (unsigned)it) < 0) {}
          asm volatile("fence.acq_rel.gpu;" ::: "memory");
        }
      } else {
        red_release_gpu_add(bar, 1u);
        while (ld_relaxed_gpu(bar) < target) {}
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
      }
      dummy = it;
    }
    __syncthreads();
  }
  long long t1 = clock64();
  if (blockIdx.x == 0 && threadIdx.x == 0) *out = (t1 - t0) / iters;
}

// 6. scattered 8-byte gathers from an L2-resident vector (the weight gathers of a step): loads per SM-cycle
__global__ void k_gather(const double *buf, int n_addr, int reps, long long *out, double *sink) {
  const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned a = tid * 2654435761u;
  double acc = 0.0;
  long long t0 = clock64();
  for (int r = 0; r < reps; r += 4) {
    double v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) { a = a * 1664525u + 1013904223u; v[u] = __ldcg(&buf[(a >> 8) % n_addr]); }
    acc += (v[0] + v[1]) + (v[2] + v[3]);
  }
  long long t1 = clock64();
  if (acc == 12345.678) *sink = acc;
  if (tid == 0) *out = (t1 - t0);
}

// 7. hardware cluster barrier (one cluster; release/acquire vs relaxed arrive)
template <bool RELAXED>
__global__ void k_cluster_barrier(int iters, long long *out) {
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
    if (RELAXED) asm volatile("barrier.cluster.arrive.relaxed.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
    else asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  }
  long long t1 = clock64();
  if (blockIdx.x == 0 && threadIdx.x == 0) *out = (t1 - t0) / iters;
}

// 8. latency of the first scattered loads AFTER a grid barrier (what a step's consumers do): every warp of the first
//    n_warps warps issues LOADS independent 16-byte ld.cg gathers per lane from an L2-resident vector and waits for them.
//    BAR: 0 = no barrier, 1 = release/acquire counter barrier (as shipped), 2 = relaxed barrier, 3 = barrier + every thread
//    issued one fp64 RED before it
template <int BAR, int LOADS>
__global__ void k_post_barrier_load(unsigned *bar, const double2 *buf, double *redbuf, int n_addr, int n_warps, int iters,
                                    long long *out, double *sink) {
  __shared__ int dummy;
  const int warp = threadIdx.x >> 5;
  unsigned a = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
  long long tot = 0;
  double acc = 0.0;
  for (int it = 1; it <= iters; ++it) {
    if (BAR == 3) { a = a * 1664525u + 1013904223u; atomicAdd(&redbuf[(a >> 8) % n_addr], 1.0); }
    __syncthreads();
    if (BAR != 0 && threadIdx.x == 0) {
      const unsigned target = (unsigned)it * gridDim.x;
      if (BAR == 2) { red_relaxed_gpu_add(bar, 1u); while (ld_relaxed_gpu(bar) < target) {} }
      else { red_release_gpu_add(bar, 1u); while (ld_relaxed_gpu(bar) < target) {} asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
      dummy = it;
    }
    __syncthreads();
    if (warp < n_warps) {
      const long long t0 = clock64();
      double2 v[LOADS];
#pragma unroll
      for (int u = 0; u < LOADS; ++u) { a = a * 1664525u + 1013904223u; v[u] = __ldcg(&buf[(a >> 8) % n_addr]); }
#pragma unroll
      for (int u = 0; u < LOADS; ++u) acc += v[u].x + v[u].y;
      if (acc == 12345.678) *sink = acc;     // forces the wait
      const long long t1 = clock64();
      tot += t1 - t0;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *out = tot / iters;
}

// 9. does it matter that the gathered vector was WRITTEN (REDs / partial stores from all SMs) just before the barrier?
//    WR: 0 = read only, 1 = every thread REDs 4 entries before the barrier, 2 = every thread stores 8 bytes into 4 entries
template <int WR>
__global__ void k_rw_then_gather(unsigned *bar, double2 *buf, int n_addr, int iters, long long *out, double *sink) {
  __shared__ int dummy;
  unsigned a = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
  long long tot = 0;
  double acc = 0.0;
  for (int it = 1; it <= iters; ++it) {
    if (WR) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        a = a * 1664525u + 1013904223u;
        double *q = &buf[(a >> 8) % n_addr].y;
        if (WR == 1) asm volatile("red.relaxed.gpu.global.add.f64 [%0], %1;" ::"l"(q), "d"(1.0) : "memory");
        else *(volatile double *)q = 1.0;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned target = (unsigned)it * gridDim.x;
      red_release_gpu_add(bar, 1u); while (ld_relaxed_gpu(bar) < target) {} asm volatile("fence.acq_rel.gpu;" ::: "memory");
      dummy = it;
    }
    __syncthreads();
    if (threadIdx.x < 256) {   // 8 warps x 1 gather per lane
      const long long t0 = clock64();
      a = a * 1664525u + 1013904223u;
      const double2 v = __ldcg(&buf[(a >> 8) % n_addr]);
      acc += v.x + v.y;
      if (acc == 12345.678) *sink = acc;
      tot += clock64() - t0;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *out = tot / iters;
}

// 10. variants of 9: WHO wrote, WHERE, how long ago, and how the gather is issued.
//   WR 1: all SMs RED before the barrier; 3: only CTA 0 REDs (4 x 448 entries); 4: all SMs RED into the OTHER half of the
//   vector (gathers go to the half nobody wrote)
//   RD 0: ld.cg   1: ld.relaxed.gpu   2: atom.add.f64 of 0.0 (performed at L2)   3: ld.cg after spinning 6000 cycles
template <int WR, int RD>
__global__ void k_rw_variants(unsigned *bar, double2 *buf, int n_addr, int iters, long long *out, double *sink) {
  __shared__ int dummy;
  unsigned a = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
  long long tot = 0;
  double acc = 0.0;
  const int half = n_addr / 2;
  for (int it = 1; it <= iters; ++it) {
    if (WR == 1 || WR == 4 || (WR == 3 && blockIdx.x == 0)) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        a = a * 1664525u + 1013904223u;
        const int idx = (WR == 4) ? half + (int)((a >> 8) % half) : (int)((a >> 8) % half);
        asm volatile("red.relaxed.gpu.global.add.f64 [%0], %1;" ::"l"(&buf[idx].y), "d"(1.0) : "memory");
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned target = (unsigned)it * gridDim.x;
      red_release_gpu_add(bar, 1u); while (ld_relaxed_gpu(bar) < target) {} asm volatile("fence.acq_rel.gpu;" ::: "memory");
      dummy = it;
    }
    __syncthreads();
    if (RD == 3) { const long long w0 = clock64(); while (clock64() - w0 < 6000) {} }
    if (threadIdx.x < 256) {
      const long long t0 = clock64();
      a = a * 1664525u + 1013904223u;
      const double2 *q = &buf[(a >> 8) % half];
      double2 v;
      if (RD == 1) asm volatile("ld.relaxed.gpu.global.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(q) : "memory");
      else if (RD == 2) { asm volatile("atom.relaxed.gpu.global.add.f64 %0, [%1], %2;" : "=d"(v.x) : "l"(&q->x), "d"(0.0) : "memory"); v.y = 0.0; }
      else v = __ldcg(q);
      acc += v.x + v.y;
      if (acc == 12345.678) *sink = acc;
      tot += clock64() - t0;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *out = tot / iters;
}

// 11. how the WRITER stores decides what the readers pay?  ST 0: st.volatile (as 9/WR 2)  1: st.global.cg  2: st.relaxed.gpu
//     3: st.global.wt  4: atom.exch.b64  5: red.global.add.f64 (reference)  6: st.relaxed.sys.v2 16 bytes (the LL word)
template <int ST>
__global__ void k_store_kinds(unsigned *bar, double2 *buf, int n_addr, int iters, long long *out, double *sink) {
  __shared__ int dummy;
  unsigned a = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u;
  long long tot = 0;
  double acc = 0.0;
  for (int it = 1; it <= iters; ++it) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      a = a * 1664525u + 1013904223u;
      double *q = &buf[(a >> 8) % n_addr].y;
      const double v = (double)it;
      if (ST == 0) *(volatile double *)q = v;
      else if (ST == 1) asm volatile("st.global.cg.f64 [%0], %1;" ::"l"(q), "d"(v) : "memory");
      else if (ST == 2) asm volatile("st.relaxed.gpu.global.f64 [%0], %1;" ::"l"(q), "d"(v) : "memory");
      else if (ST == 3) asm volatile("st.global.wt.f64 [%0], %1;" ::"l"(q), "d"(v) : "memory");
      else if (ST == 4) { unsigned long long o; asm volatile("atom.relaxed.gpu.global.exch.b64 %0, [%1], %2;" : "=l"(o) : "l"(q), "l"(__double_as_longlong(v)) : "memory"); if (o == 12345ull) *sink = 1.0; }
      else if (ST == 5) asm volatile("red.relaxed.gpu.global.add.f64 [%0], %1;" ::"l"(q), "d"(1.0) : "memory");
      else asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(q - 1), "l"((unsigned long long)it), "l"((unsigned long long)it) : "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned target = (unsigned)it * gridDim.x;
      red_release_gpu_add(bar, 1u); while (ld_relaxed_gpu(bar) < target) {}
      dummy = it;
    }
    __syncthreads();
    if (threadIdx.x < 256) {
      const long long t0 = clock64();
      a = a * 1664525u + 1013904223u;
      const double2 v = __ldcg(&buf[(a >> 8) % n_addr]);
      acc += v.x + v.y;
      if (acc == 12345.678) *sink = acc;
      tot += clock64() - t0;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *out = tot / iters;
}

int main() {
  int dev = 0; CK(cudaSetDevice(dev));
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, dev));
  printf("%s, %d SMs, clock %d kHz\n", prop.name, prop.multiProcessorCount, prop.clockRate);
  long long *out; CK(cudaMallocManaged(&out, 8)); unsigned *sink; CK(cudaMalloc(&sink, 4));
  // chase over 64 KB (L2 resident after first pass) and over 1 GB (DRAM)
  for (size_t bytes : {size_t(64) << 10, size_t(8) << 20, size_t(1) << 30}) {
    size_t n = bytes / 4; std::vector<unsigned> h(n);
    // random single cycle with stride >= 128 B granularity
    size_t lines = n / 32; std::vector<unsigned> perm(lines); for (size_t i = 0; i < lines; ++i) perm[i] = i;
    for (size_t i = lines - 1; i > 0; --i) { size_t j = rand() % (i + 1); std::swap(perm[i], perm[j]); }
    for (size_t i = 0; i < lines; ++i) h[perm[i] * 32] = perm[(i + 1) % lines] * 32;
    unsigned *d; CK(cudaMalloc(&d, bytes)); CK(cudaMemcpy(d, h.data(), bytes, cudaMemcpyHostToDevice));
    int hops = 20000;
    for (int rep = 0; rep < 2; ++rep) {
      k_chase<0><<<1, 1>>>(d, hops, out, sink); CK(cudaDeviceSynchronize()); long long a = *out;
      k_chase<1><<<1, 1>>>(d, hops, out, sink); CK(cudaDeviceSynchronize()); long long b = *out;
      k_chase<2><<<1, 1>>>(d, hops, out, sink); CK(cudaDeviceSynchronize()); long long c = *out;
      if (rep) printf("chase %8zu KB: ld.cg %lld cyc/hop, ld (L1) %lld, ld.relaxed.gpu %lld\n", bytes >> 10, a, b, c);
    }
    CK(cudaFree(d));
  }
  unsigned *bar; CK(cudaMalloc(&bar, 1024));
  for (int G : {2, 8, 32, 64, 132}) {
    long long r[4];
    for (int mode = 0; mode < 3; ++mode) {
      CK(cudaMemset(bar, 0, 1024));
      int iters = 2000; void *args[] = {&bar, &iters, &out};
      void *fn = mode == 0 ? (void *)k_barrier<0> : mode == 1 ? (void *)k_barrier<1> : (void *)k_barrier<2>;
      CK(cudaLaunchCooperativeKernel(fn, dim3(G), dim3(512), args, 0, 0)); CK(cudaDeviceSynchronize()); r[mode] = *out;
    }
    { int iters = 2000; void *args[] = {&iters, &out};
      CK(cudaLaunchCooperativeKernel((void *)k_cg_barrier, dim3(G), dim3(512), args, 0, 0)); CK(cudaDeviceSynchronize()); r[3] = *out; }
    printf("grid barrier G=%3d x512thr: red.release/ld.acquire %lld cyc, fence+atomic+volatile %lld, relaxed %lld, cg::grid.sync %lld\n", G, r[0], r[1], r[2], r[3]);
  }
  { CK(cudaMemset(bar, 0, 1024)); int iters = 2000; k_pingpong<<<2, 32>>>(bar, iters, out); CK(cudaDeviceSynchronize());
    printf("ping-pong round trip (release add -> acquire poll, two CTAs): %lld cyc\n", *out); }
  double *bd; float *bf; CK(cudaMalloc(&bd, 8 << 20)); CK(cudaMalloc(&bf, 4 << 20)); CK(cudaMemset(bd, 0, 8 << 20)); CK(cudaMemset(bf, 0, 4 << 20));
  for (int n_addr : {1, 16, 1024, 47236, 1 << 20}) {
    for (int blocks : {32, 132}) {
      int reps = 64;
      k_red<double><<<blocks, 256>>>(bd, n_addr, reps, out); CK(cudaDeviceSynchronize()); long long a = *out;
      k_red<float><<<blocks, 256>>>(bf, n_addr, reps, out); CK(cudaDeviceSynchronize()); long long b = *out;
      double total = (double)blocks * 256 * reps;
      printf("RED n_addr=%7d blocks=%3d: f64 %lld cyc (%.3f cyc/op chip-wide), f32 %lld cyc (%.3f)\n", n_addr, blocks, a, a / total, b, b / total);
    }
  }
  // ---- round-2 questions ----
  unsigned *flags; CK(cudaMalloc(&flags, 32 * 4 * 256));
  {
    const int G = prop.multiProcessorCount; int iters = 2000;
    auto run = [&](void *fn, const char *name) {
      CK(cudaMemset(bar, 0, 1024)); CK(cudaMemset(flags, 0, 32 * 4 * 256));
      void *args[] = {&bar, &flags, &bd, &iters, &out};
      CK(cudaLaunchCooperativeKernel(fn, dim3(G), dim3(448), args, 0, 0)); CK(cudaDeviceSynchronize());
      printf("barrier2 G=%d x448thr %-44s %lld cyc\n", G, name, *out);
    };
    run((void *)k_barrier2<8, false, false>, "counter polled by all (as shipped):");
    run((void *)k_barrier2<1, false, true>, "flags, one per CTA:");
    run((void *)k_barrier2<8, false, true>, "flags, one per 8 CTAs:");
    run((void *)k_barrier2<32, false, true>, "flags, one per 32 CTAs:");
    run((void *)k_barrier2<8, true, false>, "counter polled by all + 1 RED/thread:");
    run((void *)k_barrier2<8, true, true>, "flags per 8 CTAs + 1 RED/thread:");
  }
  for (int threads : {256, 1024})
    for (int blocks : {8, 16, 32, 66, 132}) {
      int reps = 64, n_addr = 47236;
      k_red<double><<<blocks, threads>>>(bd, n_addr, reps, out); CK(cudaDeviceSynchronize()); long long a = *out;
      k_gather<<<blocks, threads>>>(bd, n_addr, reps, out, bd + n_addr); CK(cudaDeviceSynchronize()); long long b = *out;
      const double per_sm = (double)threads * reps;
      printf("scattered 8 B over 47236 doubles, %3d CTAs x %4d thr: RED.f64 %.3f /SM-cycle, ld.cg %.3f /SM-cycle\n", blocks, threads,
             per_sm / a, per_sm / b);
    }
  {
    const int G = prop.multiProcessorCount; int iters = 1000, n_addr = 47236;
    double2 *rb; CK(cudaMalloc(&rb, sizeof(double2) * n_addr)); CK(cudaMemset(rb, 0, sizeof(double2) * n_addr));
    auto run = [&](void *fn, int n_warps, const char *name) {
      CK(cudaMemset(bar, 0, 1024));
      void *args[] = {&bar, &rb, &bd, &n_addr, &n_warps, &iters, &out, &bd};
      CK(cudaLaunchCooperativeKernel(fn, dim3(G), dim3(448), args, 0, 0)); CK(cudaDeviceSynchronize());
      printf("post-barrier gathers, %2d warps/SM x %-28s %lld cyc until the loads are back\n", n_warps, name, *out);
    };
    for (int nw : {1, 8, 14}) {
      run((void *)k_post_barrier_load<0, 1>, nw, "1 load/lane, no barrier:");
      run((void *)k_post_barrier_load<1, 1>, nw, "1 load/lane, rel/acq barrier:");
      run((void *)k_post_barrier_load<2, 1>, nw, "1 load/lane, relaxed barrier:");
      run((void *)k_post_barrier_load<0, 4>, nw, "4 loads/lane, no barrier:");
      run((void *)k_post_barrier_load<1, 4>, nw, "4 loads/lane, rel/acq barrier:");
      run((void *)k_post_barrier_load<3, 4>, nw, "4 loads/lane, RED + barrier:");
    }
  }
  {
    const int G = prop.multiProcessorCount; int iters = 1000, n_addr = 47236;
    double2 *rb; CK(cudaMalloc(&rb, sizeof(double2) * n_addr)); CK(cudaMemset(rb, 0, sizeof(double2) * n_addr));
    auto run = [&](void *fn, const char *name) {
      CK(cudaMemset(bar, 0, 1024));
      void *args[] = {&bar, &rb, &n_addr, &iters, &out, &bd};
      CK(cudaLaunchCooperativeKernel(fn, dim3(G), dim3(448), args, 0, 0)); CK(cudaDeviceSynchronize());
      printf("gather (8 warps x 1 per lane) after the barrier, vector %-36s %lld cyc\n", name, *out);
    };
    run((void *)k_rw_then_gather<0>, "read-only:");
    run((void *)k_rw_then_gather<1>, "RED into by every thread before:");
    run((void *)k_rw_then_gather<2>, "stored into by every thread before:");
    run((void *)k_store_kinds<0>, "st.volatile by all:");
    run((void *)k_store_kinds<1>, "st.global.cg by all:");
    run((void *)k_store_kinds<2>, "st.relaxed.gpu by all:");
    run((void *)k_store_kinds<3>, "st.global.wt by all:");
    run((void *)k_store_kinds<4>, "atom.exch.b64 by all:");
    run((void *)k_store_kinds<5>, "red.add.f64 by all:");
    run((void *)k_store_kinds<6>, "st.relaxed.sys.v2 (LL word) by all:");
    run((void *)k_rw_variants<1, 0>, "[half] RED by all, ld.cg:");
    run((void *)k_rw_variants<3, 0>, "[half] RED by CTA 0 only, ld.cg:");
    run((void *)k_rw_variants<4, 0>, "[half] RED by all into the OTHER half:");
    run((void *)k_rw_variants<1, 1>, "[half] RED by all, ld.relaxed.gpu:");
    run((void *)k_rw_variants<1, 2>, "[half] RED by all, atom.add 0.0:");
    run((void *)k_rw_variants<1, 3>, "[half] RED by all, 6000 cycles later:");
  }
  for (int csz : {8, 16}) {
    for (int relaxed = 0; relaxed < 2; ++relaxed) {
      void *fn = relaxed ? (void *)k_cluster_barrier<true> : (void *)k_cluster_barrier<false>;
      if (csz > 8 && cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) { cudaGetLastError(); continue; }
      cudaLaunchConfig_t cfg = {}; cfg.gridDim = dim3(csz); cfg.blockDim = dim3(448);
      cudaLaunchAttribute at; at.id = cudaLaunchAttributeClusterDimension; at.val.clusterDim.x = csz; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
      cfg.attrs = &at; cfg.numAttrs = 1;
      int iters = 2000;
      cudaError_t e = relaxed ? cudaLaunchKernelEx(&cfg, k_cluster_barrier<true>, iters, out) : cudaLaunchKernelEx(&cfg, k_cluster_barrier<false>, iters, out);
      if (e != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) { printf("cluster barrier size %d: %s\n", csz, cudaGetErrorString(cudaGetLastError())); continue; }
      printf("cluster barrier, 1 cluster of %2d CTAs x448thr, %s: %lld cyc\n", csz, relaxed ? "relaxed" : "release/acquire", *out);
    }
  }
  return 0;
}
