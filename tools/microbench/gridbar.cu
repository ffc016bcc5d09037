// Microbenchmark: cost of one grid-wide barrier in a cooperative kernel on an H100 - cooperative_groups grid.sync() against
// hand-written counter barriers (the small-model equalization pays ~7 of them per sweep, 49 sweeps on MobileNetV2).
// build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/microbench/gridbar tools/microbench/gridbar.cu
#include <cooperative_groups.h>
#include <cstdio>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
  unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void red_release(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_relaxed(unsigned* p, unsigned v) {
  asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// mode 0: cg grid.sync; 1: release-add + acquire-poll by thread 0; 2: fence + relaxed add + relaxed poll + fence;
// 3: like 1, but the poll is done by one lane while the CTA waits on bar.sync (same as 1) and the payload check is skipped
template <int MODE>
__global__ void k_bar(unsigned* ctr, unsigned* payload, int iters, unsigned long long* out_ns, int* bad) {
  cg::grid_group grid = cg::this_grid();
  const unsigned nb = gridDim.x;
  unsigned target = 0;
  unsigned long long t0 = 0;
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  int nbad = 0;
  for (int it = 0; it < iters; ++it) {
    // payload: every CTA publishes its iteration stamp, after the barrier it checks a far neighbour's
    if (threadIdx.x == 32) payload[blockIdx.x * 32] = (unsigned)(it + 1);
    if (MODE == 0) {
      grid.sync();
    } else {
      __syncthreads();
      if (threadIdx.x == 0) {
        target += nb;
        if (MODE == 1 || MODE == 3) {
          red_release(ctr, 1u);
          while ((int)(ld_acquire(ctr) - target) < 0) { }
        } else {
          __threadfence();
          red_relaxed(ctr, 1u);
          while ((int)(ld_relaxed(ctr) - target) < 0) { }
          __threadfence();
        }
      }
      __syncthreads();
    }
    if (threadIdx.x == 64) {
      const unsigned other = (blockIdx.x + nb / 2 + 1) % nb;
      const unsigned v = *((volatile unsigned*)&payload[other * 32]);
      if (v != (unsigned)(it + 1) && v != (unsigned)(it + 2)) nbad++;
    }
  }
  if (nbad) atomicAdd(bad, nbad);
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned long long t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    *out_ns = t1 - t0;
  }
}

template <int MODE>
static void run(int blocks, int threads, int iters) {
  unsigned *ctr, *payload; unsigned long long* ns; int* bad;
  cudaMalloc(&ctr, 256); cudaMemset(ctr, 0, 256);
  cudaMalloc(&payload, 4 * 32 * 1024); cudaMemset(payload, 0, 4 * 32 * 1024);
  cudaMalloc(&ns, 8); cudaMalloc(&bad, 4); cudaMemset(bad, 0, 4);
  void* args[] = {&ctr, &payload, &iters, &ns, &bad};
  for (int rep = 0; rep < 3; ++rep) {
    cudaMemset(ctr, 0, 256);
    cudaError_t e = cudaLaunchCooperativeKernel((void*)k_bar<MODE>, dim3(blocks), dim3(threads), args, 0, 0);
    if (e != cudaSuccess) { printf("mode %d blocks %d: launch failed: %s\n", MODE, blocks, cudaGetErrorString(e)); return; }
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("mode %d blocks %d: %s\n", MODE, blocks, cudaGetErrorString(e)); return; }
  }
  unsigned long long h; int hb;
  cudaMemcpy(&h, ns, 8, cudaMemcpyDeviceToHost); cudaMemcpy(&hb, bad, 4, cudaMemcpyDeviceToHost);
  printf("mode %d  %4d CTAs x %3d thr: %7.3f us per barrier  (stale reads %d)\n", MODE, blocks, threads, (double)h * 1e-3 / iters, hb);
  cudaFree(ctr); cudaFree(payload); cudaFree(ns); cudaFree(bad);
}

int main() {
  const int iters = 2000;
  for (int blocks : {148, 296, 444}) {
    run<0>(blocks, 256, iters);
    run<1>(blocks, 256, iters);
    run<2>(blocks, 256, iters);
  }
  return 0;
}
