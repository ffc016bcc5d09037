// Microbenchmark: the copy ceilings the streaming weight passes are measured against, on one GPU.
//   read     a read-only TMA stream: bulk loads of 18 KB stages into a per-SM ring, consumer warps hand every stage
//            straight back (the shape of the fold's read-only scan)
//   rw       read -> bulk store in place: the consumer warp that takes a stage issues its bulk store and hands the stage
//            back once the store has READ it (the shape of k_cle_stack's pass, minus the arithmetic)
// One CTA per SM, a producer warp + N consumer warps, S stages; sequence numbers are dealt modulo N as in bc_stream.cuh.
// Also two non-TMA references: an ld.global.v4 read-only sweep and a cudaMemcpy device-to-device copy.
// Bytes: read = buffer size; rw and memcpy = 2 x buffer size.  Each configuration is timed with CUDA events, best of 5.
// build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/microbench/hbm_ceiling tools/microbench/hbm_ceiling.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int kStageBytes = 4608 * 4;   // one [512,3,3] fp32 row
constexpr long long kTileBlock = 64;    // block-cyclic tile ownership, as TileCursor

__device__ __forceinline__ uint32_t su32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(su32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(su32(b)) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t n) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(su32(b)), "r"(n) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  asm volatile("{\n\t.reg .pred P1;\n\tW:\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t@P1 bra D;\n\tbra W;\n\tD:\n\t}"
               ::"r"(su32(b)), "r"(parity), "r"(0x989680u) : "memory");
}
__device__ __forceinline__ void g2s(void* dst, const void* src, uint32_t n, uint64_t* b) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(su32(dst)), "l"(src), "r"(n), "r"(su32(b)) : "memory");
}
__device__ __forceinline__ void s2g(void* dst, const void* src, uint32_t n) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(su32(src)), "r"(n) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

// STORE = false: read-only stream; true: read -> bulk store in place.
template <bool STORE>
__global__ void __launch_bounds__(256, 1) k_ring(float* buf, long long tiles, int S, int N) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = (uint64_t*)(smem + (size_t)S * kStageBytes);
  uint64_t* empty = full + S;
  int* seq = (int*)(empty + S);            // sequence number of the item in each stage
  int* kind = seq + S;                      // 0 tile, 1 padding, 2 end
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < S; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 1); seq[i] = -1; kind[i] = 0; }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const long long G = gridDim.x, b = blockIdx.x;
  const long long mine = (((tiles + kTileBlock - 1) / kTileBlock + G - 1 - b) / G) * kTileBlock;   // upper bound; tiles past the end are skipped
  if (warp == N) {                         // producer
    if (lane != 0) return;
    unsigned long long n = 0;
    for (long long k = 0; k < mine; ++k) {
      const long long t = ((k / kTileBlock) * G + b) * kTileBlock + k % kTileBlock;
      if (t >= tiles) break;
      const int s = (int)(n % S);
      if (n >= (unsigned long long)S) mbar_wait(empty + s, (uint32_t)(((n / S) - 1) & 1));
      seq[s] = (int)n; kind[s] = 0;
      mbar_expect(full + s, kStageBytes);
      g2s(smem + (size_t)s * kStageBytes, buf + t * (kStageBytes / 4), kStageBytes, full + s);
      ++n;
    }
    while (n % N) {                        // padding so that every consumer ends on its own END
      const int s = (int)(n % S);
      if (n >= (unsigned long long)S) mbar_wait(empty + s, (uint32_t)(((n / S) - 1) & 1));
      seq[s] = (int)n; kind[s] = 1; mbar_arrive(full + s); ++n;
    }
    for (int i = 0; i < N; ++i) {
      const int s = (int)(n % S);
      if (n >= (unsigned long long)S) mbar_wait(empty + s, (uint32_t)(((n / S) - 1) & 1));
      seq[s] = (int)n; kind[s] = 2; mbar_arrive(full + s); ++n;
    }
    return;
  }
  if (warp > N) return;
  // consumers: item n = warp (mod N); the stamp check of bc_take (a parity wait alone can see the previous phase)
  for (unsigned long long n = warp;; n += N) {
    const int s = (int)(n % S);
    const uint32_t par = (uint32_t)((n / S) & 1);
    const volatile int* vs = seq + s;
    for (;;) {
      mbar_wait(full + s, par);
      if (*vs == (int)n) break;
      __nanosleep(64);
    }
    mbar_wait(full + s, par);
    const int v = ((const volatile int*)kind)[s];
    if (v == 2) { __syncwarp(); if (lane == 0) mbar_arrive(empty + s); break; }
    if (STORE && v == 0 && lane == 0) {
      const long long k = (long long)n;      // item k is the producer's k-th tile
      const long long t = ((k / kTileBlock) * G + b) * kTileBlock + k % kTileBlock;
      s2g(buf + t * (kStageBytes / 4), smem + (size_t)s * kStageBytes, kStageBytes);
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + s);
  }
  if (STORE && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

__global__ void __launch_bounds__(512) k_ldg(const float4* __restrict__ p, long long n4, float* sink) {
  float acc = 0.f;
  const long long st = (long long)gridDim.x * blockDim.x;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * st < n4; i += 4 * st) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[u].x), "=f"(v[u].y), "=f"(v[u].z), "=f"(v[u].w) : "l"(p + i + u * st));
#pragma unroll
    for (int u = 0; u < 4; ++u) acc += v[u].x + v[u].y + v[u].z + v[u].w;
  }
  for (; i < n4; i += st) { const float4 v = p[i]; acc += v.x + v.y + v.z + v.w; }
  if (acc == 12345.678f) *sink = acc;
}

template <typename F>
static float best_ms(F launch) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  launch();                                   // warm-up
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < 5; ++r) {
    CK(cudaEventRecord(a));
    launch();
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b));
    if (ms < best) best = ms;
  }
  CK(cudaGetLastError());
  cudaEventDestroy(a); cudaEventDestroy(b);
  return best;
}

int main(int argc, char** argv) {
  const double gb = argc > 1 ? atof(argv[1]) : 12.0;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s, %d SMs\n", prop.name, prop.multiProcessorCount);
  fflush(stdout);
  if (FILE* f = popen("nvidia-smi --query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem --format=csv,noheader", "r")) {
    char line[256];
    while (fgets(line, sizeof line, f)) printf("nvidia-smi: %s", line);
    pclose(f);
  }
  const long long tiles = (long long)(gb * 1e9) / kStageBytes;
  const size_t bytes = (size_t)tiles * kStageBytes;
  float* buf; float* sink;
  CK(cudaMalloc(&buf, bytes));
  CK(cudaMalloc(&sink, 4));
  CK(cudaMemset(buf, 0, bytes));
  printf("buffer: %.2f GB (%lld tiles of %d B)\n", bytes * 1e-9, tiles, kStageBytes);
  const int G = prop.multiProcessorCount;

  const float ms_ldg = best_ms([&] { k_ldg<<<G * 4, 512>>>((const float4*)buf, (long long)(bytes / 16), sink); });
  printf("ldg.v4 read-only          : %7.3f ms  %6.3f TB/s\n", ms_ldg, bytes / (ms_ldg * 1e-3) / 1e12);
  const size_t half = bytes / 2;
  const float ms_cpy = best_ms([&] { CK(cudaMemcpyAsync(buf + half / 4, buf, half, cudaMemcpyDeviceToDevice)); });
  printf("cudaMemcpy d2d (rd+wr)    : %7.3f ms  %6.3f TB/s\n", ms_cpy, 2.0 * half / (ms_cpy * 1e-3) / 1e12);

  const int stage_counts[] = {4, 6, 8, 9, 10, 11, 12};
  const int consumer_counts[] = {1, 2, 3, 4, 5, 6, 7};
  for (int store = 0; store < 2; ++store) {
    printf("%s ring (TB/s counts %s):\n", store ? "read -> bulk store" : "read-only TMA", store ? "read + write" : "read");
    printf("  stages \\ consumers");
    for (int N : consumer_counts) printf("  %5d", N);
    printf("\n");
    for (int S : stage_counts) {
      printf("  %18d", S);
      const size_t smem = (size_t)S * kStageBytes + 16 * S + 8 * S + 64;
      for (int N : consumer_counts) {
        const void* kern = store ? (const void*)k_ring<true> : (const void*)k_ring<false>;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const float ms = best_ms([&] {
          if (store) k_ring<true><<<G, (N + 1) * 32, smem>>>(buf, tiles, S, N);
          else k_ring<false><<<G, (N + 1) * 32, smem>>>(buf, tiles, S, N);
        });
        printf("  %5.3f", (store ? 2.0 : 1.0) * bytes / (ms * 1e-3) / 1e12);
        fflush(stdout);
      }
      printf("\n");
    }
  }
  CK(cudaFree(buf)); CK(cudaFree(sink));
  return 0;
}
