// RowPipe: a per-CTA ring of shared-memory stages fed by the TMA unit (bulk async copies, no tensor map).
//
// Every arena pass of this library streams contiguous chunks of rows ("tiles") of fp32 weight matrices: read a tile,
// reduce / rescale it, write it back.  The HBM pipeline is decoupled from the threads:
//
//   producer (one elected thread)   cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes   gmem -> stage
//   consumers (all threads)         mbarrier.try_wait.parity  ->  work on the tile in shared memory, in place
//   write-back (elected thread)     fence.proxy.async + cp.async.bulk.global.shared::cta.bulk_group    stage -> gmem
//   stage reuse                     cp.async.bulk.wait_group.read  (the store has finished READING the stage)
//
// With S stages the loads of tiles k+1 .. k+S-1 are in flight while tile k is processed, independent of register
// pressure or occupancy: bytes in flight per SM = CTAs/SM x (S-1) x stage size.  SASS: UBLKCP / SYNCS.
//
// Tiles that cannot be moved by a bulk copy (base or size not a multiple of 16 bytes) take the same path with
// cooperative ld/st.global.cg instead; tiles larger than a stage are "direct" (the consumer works on global memory).
#pragma once
#include "common.cuh"

namespace dfq {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

enum TileKind { TK_BULK = 0, TK_PLAIN = 1, TK_DIRECT = 2 };

struct TileDesc {
  float* gptr;     // first float of the tile in the arena
  int task;        // index into the phase's task list (layer)
  int row0, nrows;
  int floats;      // nrows * row_len
  int kind;
  int seq;         // BcRing: sequence number of the item that occupies the stage (see bc_take)
};

#ifndef DFQ_PIPE_STAGES
#define DFQ_PIPE_STAGES 3
#endif
#ifndef DFQ_CTAS
#define DFQ_CTAS 3
#endif
constexpr int kPipeStages = DFQ_PIPE_STAGES;   // stages per CTA
constexpr int kPipeCtas = DFQ_CTAS;             // co-resident CTAs per SM the kernels are compiled for
constexpr int kStageFloats = 4608;                 // 18 KB: one [512,3,3] row, 8 rows of 576, 512 depthwise rows ...
constexpr int kStageBytes = kStageFloats * 4;
#ifndef DFQ_PIPE_MAX_ROWS
#define DFQ_PIPE_MAX_ROWS 32
#endif
constexpr int kPipeMaxRows = DFQ_PIPE_MAX_ROWS;                   // rows per tile at most: spreads layers of short rows (depthwise) over the grid

// rows per tile for a matrix of `row_len`-float rows (host and device must agree)
__host__ __device__ inline int pipe_rows_per_tile(int row_len) {
  if (row_len > kStageFloats) return 1;            // direct
  int r = kStageFloats / row_len;
  if (r > kPipeMaxRows) r = kPipeMaxRows;          // short rows: more, smaller tiles (small models are latency-bound, not bandwidth-bound)
  if (row_len % 4 != 0 && r >= 4) r &= ~3;         // keep every full tile a multiple of 16 bytes
  return r < 1 ? 1 : r;
}
__host__ __device__ inline int pipe_tiles(int rows, int row_len) {
  const int r = pipe_rows_per_tile(row_len);
  return (rows + r - 1) / r;
}

struct RowPipe {
  float* stage[kPipeStages];
  uint64_t* full;          // [kPipeStages]
  TileDesc* desc;          // [kPipeStages]
  unsigned long long head; // tiles issued   (meaningful in the producer thread only)
  unsigned long long tail; // tiles consumed (identical in all threads)

  // smem: kPipeStages*kStageBytes (128-aligned) + barriers + descriptors, carved by the caller
  __device__ void init(unsigned char* smem) {
    for (int i = 0; i < kPipeStages; ++i) stage[i] = (float*)(smem + (size_t)i * kStageBytes);
    full = (uint64_t*)(smem + (size_t)kPipeStages * kStageBytes);
    desc = (TileDesc*)(smem + (size_t)kPipeStages * kStageBytes + 64);
    head = tail = 0;
    if (threadIdx.x == 0) {
      for (int i = 0; i < kPipeStages; ++i) mbar_init(full + i, 1);
      mbar_fence_init();
    }
    __syncthreads();
  }
  static constexpr size_t smem_bytes() { return (size_t)kPipeStages * kStageBytes + 64 + kPipeStages * sizeof(TileDesc) + 64; }

  // Producer side (thread 0): make tile `d` available in the next stage.
  __device__ __forceinline__ void issue(const TileDesc& d) {
    const int s = (int)(head % kPipeStages);
    desc[s] = d;
    if (d.kind == TK_BULK) {
      mbar_arrive_expect_tx(full + s, (uint32_t)d.floats * 4u);
      bulk_g2s(stage[s], d.gptr, (uint32_t)d.floats * 4u, full + s);
    } else {
      mbar_arrive(full + s);     // nothing to wait for: consumers fetch (plain) or work in place (direct)
    }
    head++;
  }

  // Consumer side (all threads): wait for the tile at the tail; returns its stage index.
  __device__ __forceinline__ int acquire() {
    const int s = (int)(tail % kPipeStages);
    mbar_wait(full + s, (uint32_t)((tail / kPipeStages) & 1));
    const TileDesc d = desc[s];
    if (d.kind == TK_PLAIN) {     // cooperative fetch of a tile the TMA unit cannot move
      for (int i = threadIdx.x; i < d.floats; i += blockDim.x) stage[s][i] = ldg_stream1(d.gptr + i);
      __syncthreads();
    }
    return s;
  }

  // All threads, after the tile was modified in place in shared memory: write it back and free the stage.
  // `more` = the producer still has tiles to issue in this phase (next = its descriptor, valid in thread 0).
  template <bool STORE>
  __device__ __forceinline__ void release(int s, bool more, const TileDesc& next) {
    const TileDesc d = desc[s];
    if (STORE && d.kind == TK_BULK) fence_proxy_async_smem();   // my generic-proxy writes -> visible to the async proxy
    __syncthreads();
    if (STORE && d.kind == TK_PLAIN) {
      for (int i = threadIdx.x; i < d.floats; i += blockDim.x) stg_stream1(d.gptr + i, stage[s][i]);
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      if (STORE && d.kind == TK_BULK) { bulk_s2g(d.gptr, stage[s], (uint32_t)d.floats * 4u); bulk_commit(); }
      if (more) {
        // the stage to refill held tile tail-1... no: it is stage (head % S); its store was committed at least one
        // release ago whenever S >= 2 tiles are in flight, so allow only the newest store group to be pending
        if (STORE) bulk_wait_read<1>();
        // the newest group may be the store of the very stage we refill when S-1 == 1 lookahead; S = 3 keeps them apart
        issue(next);
      }
    }
    tail++;
  }

  // End of a phase, before a grid barrier: every store of this CTA has landed in global memory.
  __device__ __forceinline__ void drain() {
    if (threadIdx.x == 0) {
      bulk_wait_all();
      fence_proxy_async_all();
      __threadfence();
    }
    __syncthreads();
  }
};

// Walks this CTA's tiles (block-cyclic, TileCursor) over a list of matrices.  Geo(q, base, rows, row_len) describes task q.
// CACHE: keep the geometry of the task in hand in the iterator (the streaming kernels' single producer lane; costs four
// registers per iterator, which the 80-register RowPipe kernels do not have: k_bn_fold ran slower with it).
template <typename Geo, bool CACHE = false>
struct MatIter {
  const long long* ptr;
  int q, q_end;
  TileCursor cur;
  Geo geo;
  // geometry of task `gq`, fetched once per task: geo() chases two dependent global loads (task -> layer -> shape), and the
  // single producer lane of a streaming kernel would otherwise pay that latency for EVERY tile it issues
  int gq;
  float* g_base; int g_rows, g_row_len;
  __device__ __forceinline__ void start(const long long* p, int q_begin, int q_end_, Geo g) {
    ptr = p; q_end = q_end_; geo = g; gq = -1; g_base = nullptr; g_rows = g_row_len = 0;
    cur.init(p[q_begin], p[q_end_]);
    q = cur.valid() ? find_task(p, q_begin, q_end_, cur.t) : q_begin;
  }
  __device__ __forceinline__ bool valid() const { return cur.valid(); }
  __device__ __forceinline__ void next() {
    cur.next();
    while (q + 1 < q_end && ptr[q + 1] <= cur.t) ++q;
  }
  __device__ __forceinline__ void fill(TileDesc& d) {
    float* base; int rows, row_len;
    if (CACHE) {
      if (q != gq) { geo(q, g_base, g_rows, g_row_len); gq = q; }
      base = g_base; rows = g_rows; row_len = g_row_len;
    } else {
      geo(q, base, rows, row_len);
    }
    const int rpt = pipe_rows_per_tile(row_len);
    d.task = q;
    d.row0 = (int)(cur.t - ptr[q]) * rpt;
    d.nrows = min(rpt, rows - d.row0);
    d.floats = d.nrows * row_len;
    d.gptr = base + (size_t)d.row0 * row_len;
    if (row_len > kStageFloats) d.kind = TK_DIRECT;
    else d.kind = (((((uintptr_t)d.gptr) & 15) == 0) && ((d.floats & 3) == 0)) ? TK_BULK : TK_PLAIN;
  }
};

}  // namespace dfq
