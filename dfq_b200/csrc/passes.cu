// Batched arena passes other than equalization: BN fold, bias correction, weight/bias fake-quant.
//
//   dfq_bn_fold           utils/layer_transform.py:231-276  (merge_batchnorm)
//   dfq_bias_correct      dfq.py:173-293                    (bias_correction)
//   dfq_quantize_tensors  utils/layer_transform.py:279-296  (quantize_targ_layer)
#include <cooperative_groups.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "rowpipe.cuh"
#include "colscan.cuh"
#include "bc_stream.cuh"

namespace cg = cooperative_groups;

namespace dfq {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunk = kThreads * 16;   // floats per flat tile

// round-robin tile ownership shared by all batched kernels: tiles are numbered consecutively over the
// task list; CTA b owns global tile indices congruent to b modulo gridDim.x
__device__ __forceinline__ int first_tile(long long base) {
  int f = (int)(((long long)blockIdx.x - base) % (long long)gridDim.x);
  return f < 0 ? f + gridDim.x : f;
}

// ------------------------------------------------------------------------------------------------
// BN fold
// ------------------------------------------------------------------------------------------------
struct FoldGeo {
  float* arena; const DfqLayer* L; const DfqFold* F;
  __device__ __forceinline__ void operator()(int q, float*& base, int& rows, int& row_len) const {
    const DfqLayer l = L[F[q].layer];
    base = arena + l.w_off; rows = l.rows; row_len = l.cols * l.kk;
  }
};

// One output row: W[o,:] *= gamma/sqrt(var+eps) in place (shared memory or, for rows larger than a stage, global).
template <int TPR, bool GLOBAL>
__device__ __forceinline__ void fold_row(float* arena, const DfqLayer& l, const DfqFold& f, float* row, int o, int lane) {
  const int n = l.cols * l.kk;
  // layer_transform.py:251: gamma / sqrt(var + eps) formed first, then multiplied in
  const float gamma = arena[f.gamma_off + o], var = arena[f.var_off + o];
  const float den = __fsqrt_rn(__fadd_rn(var, f.bn_eps));
  const float fac = __fdiv_rn(gamma, den);
  if (!GLOBAL && (n & 3) == 0) {
    float4* r4 = (float4*)row;
    for (int i = lane; i < (n >> 2); i += TPR) {
      float4 v = r4[i];
      v.x = __fmul_rn(v.x, fac); v.y = __fmul_rn(v.y, fac); v.z = __fmul_rn(v.z, fac); v.w = __fmul_rn(v.w, fac);
      r4[i] = v;
    }
  } else if (GLOBAL) {
    for (int i = lane; i < n; i += TPR) stg_stream1(row + i, __fmul_rn(ldg_stream1(row + i), fac));
  } else {
    for (int i = lane; i < n; i += TPR) row[i] = __fmul_rn(row[i], fac);
  }
  if (lane == 0) {
    // layer_transform.py:260-261: b*f + (beta - (gamma*mean)/sqrt(var+eps))
    const float beta = arena[f.beta_off + o], mean = arena[f.mean_off + o];
    const float b = arena[l.bias_off + o];
    const float shift = __fsub_rn(beta, __fdiv_rn(__fmul_rn(gamma, mean), den));
    arena[l.bias_off + o] = __fadd_rn(__fmul_rn(b, fac), shift);
    arena[f.fake_w_off + o] = fabsf(gamma);   // :264
    arena[f.fake_b_off + o] = beta;           // :265
  }
}

constexpr int kFoldScanCols = 1024;   // columns whose extrema a CTA accumulates in shared memory (more: global atomics)

// buffer 0 of the column-extrema arrays of every fold that scans: +inf / -inf
__global__ void k_fold_reset_cols(float* arena, const DfqLayer* __restrict__ L, const DfqFold* __restrict__ F, int nF) {
  for (int q = blockIdx.x; q < nF; q += gridDim.x) {
    const DfqFold f = F[q];
    if (f.scan_go <= 0) continue;
    const DfqLayer l = L[f.layer];
    const int nch = (l.rows / f.scan_go) * f.scan_gi;
    for (int j = threadIdx.x; j < nch; j += blockDim.x) { arena[l.cmin_off + j] = DFQ_INF; arena[l.cmax_off + j] = -DFQ_INF; }
  }
}

__global__ void __launch_bounds__(kThreads, kPipeCtas)
k_bn_fold(float* arena, const DfqLayer* __restrict__ L, const DfqFold* __restrict__ F, int nF,
          const long long* __restrict__ tptr) {
  extern __shared__ __align__(128) unsigned char pipe_smem[];
  __shared__ float s_cmin[kFoldScanCols], s_cmax[kFoldScanCols];
  RowPipe pipe;
  pipe.init(pipe_smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  MatIter<FoldGeo> it;
  it.start(tptr, 0, nF, FoldGeo{arena, L, F});
  MatIter<FoldGeo> ahead = it;
  TileDesc nd;
  if (threadIdx.x == 0)
    for (int i = 0; i < kPipeStages - 1 && ahead.valid(); ++i) { ahead.fill(nd); pipe.issue(nd); ahead.next(); }
  // column scan of the folded rows (DfqFold.scan_go > 0): partial extrema per CTA and layer, flushed when the layer changes
  for (int j = threadIdx.x; j < kFoldScanCols; j += kThreads) { s_cmin[j] = DFQ_INF; s_cmax[j] = -DFQ_INF; }
  int cur = -1, nch = 0;
  bool scanning = false, use_smem = false;
  float *dmin = nullptr, *dmax = nullptr;
  auto flush = [&]() {
    if (!scanning || !use_smem) return;
    __syncthreads();
    colscan_flush<kThreads>(threadIdx.x, nch, s_cmin, s_cmax, dmin, dmax);
    __syncthreads();
  };
  while (it.valid()) {
    const int sidx = pipe.acquire();
    const TileDesc d = pipe.desc[sidx];
    const DfqFold f = F[d.task];
    const DfqLayer l = L[f.layer];
    const int row_len = l.cols * l.kk;
    if (d.task != cur) {
      flush();
      cur = d.task;
      scanning = f.scan_go > 0;
      if (scanning) {
        nch = (l.rows / f.scan_go) * f.scan_gi;
        use_smem = nch <= kFoldScanCols;
        dmin = arena + l.cmin_off; dmax = arena + l.cmax_off;    // buffer 0
      }
    }
    if (d.kind == TK_DIRECT) {
      for (int r = 0; r < d.nrows; ++r)
        fold_row<kThreads, true>(arena, l, f, d.gptr + (size_t)r * row_len, d.row0 + r, threadIdx.x);
    } else if (d.nrows == 1) {
      fold_row<kThreads, false>(arena, l, f, pipe.stage[sidx], d.row0, threadIdx.x);
    } else {
      for (int r = warp; r < d.nrows; r += kWarps)
        fold_row<32, false>(arena, l, f, pipe.stage[sidx] + (size_t)r * row_len, d.row0 + r, lane);
    }
    if (scanning) {
      __syncthreads();     // the tile's rows are final
      const bool single = (f.scan_go == l.rows), own = (pipe_rows_per_tile(row_len) == 1);
      if (d.kind == TK_DIRECT)
        colscan_tile<kThreads, true>(d.gptr, threadIdx.x, d.row0, d.nrows, l.cols, l.kk, f.scan_go, f.scan_gi, single, own,
                                     use_smem, s_cmin, s_cmax, dmin, dmax);
      else
        colscan_tile<kThreads, false>(pipe.stage[sidx], threadIdx.x, d.row0, d.nrows, l.cols, l.kk, f.scan_go, f.scan_gi, single,
                                      own, use_smem, s_cmin, s_cmax, dmin, dmax);
    }
    bool more = false;
    if (threadIdx.x == 0) {
      more = ahead.valid();
      if (more) { ahead.fill(nd); ahead.next(); }
    }
    pipe.release<true>(sidx, more, nd);
    it.next();
  }
  flush();
  pipe.drain();
}

// ------------------------------------------------------------------------------------------------
// per-tensor min/max over a task list (flat tiles), then in-place fake quantization
// ------------------------------------------------------------------------------------------------
struct FlatTask { int64_t off; int64_t n; int64_t minmax_off; int32_t num_bits; int32_t symmetric; };

__device__ __forceinline__ void cta_minmax_atomic(float mn, float mx, float* dst2, float* red) {
  mn = warp_min(mn); mx = warp_max(mx);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) { red[w] = mn; red[kWarps + w] = mx; }
  __syncthreads();
  if (w == 0) {
    float a = red[l & (kWarps - 1)], b = red[kWarps + (l & (kWarps - 1))];
#pragma unroll
    for (int o = kWarps / 2; o > 0; o >>= 1) {
      a = fminf(a, __shfl_xor_sync(0xffffffffu, a, o));
      b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
    }
    if (l == 0) { atomic_min_f(dst2, a); atomic_max_f(dst2 + 1, b); }
  }
}

__device__ __forceinline__ void tile_minmax(const float* x, int64_t n, int64_t t, float& mn, float& mx) {
  const int64_t lo = t * kChunk;
  const int64_t hi = min(lo + (int64_t)kChunk, n);
  if ((((uintptr_t)x) & 15) == 0) {
    const float4* x4 = (const float4*)x;
    const int64_t lo4 = lo >> 2, hi4 = hi >> 2;
    for (int64_t i = lo4 + threadIdx.x; i < hi4; i += kThreads) {
      const float4 v = ldg_stream(x4 + i);
      mn = fminf(mn, fminf(fminf(v.x, v.y), fminf(v.z, v.w)));
      mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
    }
    for (int64_t i = (hi4 << 2) + threadIdx.x; i < hi; i += kThreads) {
      const float v = ldg_stream1(x + i); mn = fminf(mn, v); mx = fmaxf(mx, v);
    }
  } else {
    for (int64_t i = lo + threadIdx.x; i < hi; i += kThreads) {
      const float v = ldg_stream1(x + i); mn = fminf(mn, v); mx = fmaxf(mx, v);
    }
  }
}

__global__ void k_minmax_init(float* arena, const FlatTask* __restrict__ T, int nT) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nT; i += gridDim.x * blockDim.x) {
    arena[T[i].minmax_off] = DFQ_INF;
    arena[T[i].minmax_off + 1] = -DFQ_INF;
  }
}

__global__ void __launch_bounds__(kThreads)
k_minmax_tasks(float* arena, const FlatTask* __restrict__ T, int nT, const long long* __restrict__ tptr) {
  __shared__ float red[2 * kWarps];
  const TileSpan sp = tile_span(tptr, 0, nT);
  for (int ti = sp.q; ti < nT && tptr[ti] < sp.hi; ++ti) {
    const FlatTask t = T[ti];
    const long long base = tptr[ti];
    const long long k0 = max(sp.lo, base) - base, k1 = min(sp.hi, tptr[ti + 1]) - base;
    if (k1 <= k0) continue;
    float mn = DFQ_INF, mx = -DFQ_INF;
    for (long long k = k0; k < k1; ++k) tile_minmax(arena + t.off, t.n, k, mn, mx);
    cta_minmax_atomic(mn, mx, arena + t.minmax_off, red);
  }
}

template <bool RECIP>
__global__ void __launch_bounds__(kThreads)
k_quant_tasks(float* arena, const FlatTask* __restrict__ T, int nT, const long long* __restrict__ tptr) {
  const TileSpan sp = tile_span(tptr, 0, nT);
  for (int ti = sp.q; ti < nT && tptr[ti] < sp.hi; ++ti) {
    const FlatTask t = T[ti];
    const long long base = tptr[ti];
    const long long k0 = max(sp.lo, base) - base, k1 = min(sp.hi, tptr[ti + 1]) - base;
    if (k1 > k0) {
      // float(param.min()), float(param.max()) -> Python doubles (layer_transform.py:289,294)
      const QuantScalars q = quant_scalars((double)__ldcg(arena + t.minmax_off), (double)__ldcg(arena + t.minmax_off + 1),
                                           t.num_bits, t.symmetric);
      float* x = arena + t.off;
      for (long long k = k0; k < k1; ++k) {
        const int64_t lo = k * kChunk, hi = min(lo + (int64_t)kChunk, t.n);
        if ((t.off & 3) == 0) {
          float4* x4 = (float4*)x;
          const int64_t lo4 = lo >> 2, hi4 = hi >> 2;
          for (int64_t i = lo4 + threadIdx.x; i < hi4; i += kThreads) {
            float4 v = ldg_stream(x4 + i);
            v.x = fake_quant<RECIP>(v.x, q); v.y = fake_quant<RECIP>(v.y, q);
            v.z = fake_quant<RECIP>(v.z, q); v.w = fake_quant<RECIP>(v.w, q);
            stg_stream(x4 + i, v);
          }
          for (int64_t i = (hi4 << 2) + threadIdx.x; i < hi; i += kThreads) stg_stream1(x + i, fake_quant<RECIP>(ldg_stream1(x + i), q));
        } else {
          for (int64_t i = lo + threadIdx.x; i < hi; i += kThreads) stg_stream1(x + i, fake_quant<RECIP>(ldg_stream1(x + i), q));
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// bias correction engine (persistent cooperative kernel)
// ------------------------------------------------------------------------------------------------
// scipy.stats.norm.pdf / cdf in float64 on an fp32 argument, rounded to fp32 (dfq.py:182-183)
__device__ __forceinline__ float std_pdf(float x32) {
  const double x = (double)x32;
  return (float)(exp(-x * x / 2.0) / 2.5066282746310002);   // sqrt(2*pi)
}
__device__ __forceinline__ float std_cdf(float x32) {
  // scipy.special.ndtr (cephes)
  const double x = (double)x32 * 0.70710678118654752440;
  const double z = fabs(x);
  double y;
  if (z < 0.70710678118654752440) y = 0.5 + 0.5 * erf(x);
  else { y = 0.5 * erfc(z); if (x > 0) y = 1.0 - y; }
  return (float)y;
}
// dfq.py:184 calculate_mean + :240 clamp; every op an individually rounded fp32 op as in eager PyTorch
__device__ __forceinline__ float relu_gauss_mean(float g, float b) {
  const float q = __fdiv_rn(-b, g);
  const float t1 = __fmul_rn(g, std_pdf(q));
  const float t2 = __fmul_rn(b, __fsub_rn(1.0f, std_cdf(q)));
  const float e = __fadd_rn(t1, t2);
  return e < 0.f ? 0.f : e;      // NaN stays NaN (expect[expect < 0] = 0)
}

struct BcGeo {
  float* arena; const DfqLayer* L; const DfqBcLayer* B;
  __device__ __forceinline__ void operator()(int q, float*& base, int& rows, int& row_len) const {
    const DfqLayer l = L[B[q].layer];
    base = arena + l.w_off; rows = l.rows; row_len = l.cols * l.kk;
  }
};

constexpr int kExpectCache = 2048;

// eps . E[x] of one output row held in shared (or, for rows larger than a stage, global) memory.
// Returns the row's dot product in every thread of the row's group.
template <int TPR, bool RAW>
__device__ __forceinline__ double bc_row(const float* __restrict__ row, int cols, int kk, const float* __restrict__ ex,
                                         const QuantScalars& q, int lane) {
  double acc = 0.0;
  for (int j = lane; j < cols; j += TPR) {
    const float* p = row + (size_t)j * kk;
    float E = 0.f;
    if (RAW) {                     // bias absorption: sum_k W (dfq.py:150-153)
      for (int k = 0; k < kk; ++k) E = __fadd_rn(E, p[k]);
    } else if (kk == 9) {
#pragma unroll
      for (int k = 0; k < 9; ++k) { const float w = p[k]; E = __fadd_rn(E, __fsub_rn(fake_quant<false>(w, q), w)); }
    } else {
      for (int k = 0; k < kk; ++k) { const float w = p[k]; E = __fadd_rn(E, __fsub_rn(fake_quant<false>(w, q), w)); }
    }
    acc += (double)E * (double)ex[j];
  }
  return warp_sum(acc);
}

__global__ void __launch_bounds__(kThreads, kPipeCtas)
k_bc_engine(float* arena, const DfqLayer* __restrict__ L, const DfqBcLayer* __restrict__ B, int nB,
            const DfqExpectTerm* __restrict__ T, const int* __restrict__ level_ptr, int n_levels, int num_bits,
            const long long* __restrict__ row_ptr, const long long* __restrict__ mm_ptr, const int* __restrict__ level_local) {
  cg::grid_group grid = cg::this_grid();
  __shared__ float red[2 * kWarps];
  __shared__ double dred[kWarps];
  __shared__ __align__(16) float s_ex[kExpectCache];
  extern __shared__ __align__(128) unsigned char pipe_smem[];
  RowPipe pipe;
  pipe.init(pipe_smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  TileDesc nd;

  // ---- per-tensor min/max of every corrected weight (dfq.py:14 via :218), streamed through the pipe ----------
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < nB; i += gridDim.x * kThreads) {
    __stcg(arena + B[i].minmax_off, DFQ_INF);
    __stcg(arena + B[i].minmax_off + 1, -DFQ_INF);
  }
  grid.sync();
  // layers whose column extrema the caller vouches for (DfqBcLayer.n_col > 0): reduce those, do not stream the weights
  for (int bi = blockIdx.x; bi < nB; bi += gridDim.x) {
    const DfqBcLayer b = B[bi];
    if (b.n_col <= 0) continue;
    float mn = DFQ_INF, mx = -DFQ_INF;
    for (int j = threadIdx.x; j < b.n_col; j += kThreads) {
      mn = fminf(mn, __ldcg(arena + b.colmin_off + j)); mx = fmaxf(mx, __ldcg(arena + b.colmax_off + j));
    }
    cta_minmax_atomic(mn, mx, arena + b.minmax_off, red);
  }
  {
    MatIter<BcGeo> it;
    it.start(mm_ptr, 0, nB, BcGeo{arena, L, B});   // mm_ptr: tile prefix with zero tiles for those layers
    MatIter<BcGeo> ahead = it;
    if (threadIdx.x == 0)
      for (int i = 0; i < kPipeStages - 1 && ahead.valid(); ++i) { ahead.fill(nd); pipe.issue(nd); ahead.next(); }
    int cur = -1;
    float mn = DFQ_INF, mx = -DFQ_INF;
    while (it.valid()) {
      const int sidx = pipe.acquire();
      const TileDesc d = pipe.desc[sidx];
      if (d.task != cur) {
        if (cur >= 0) cta_minmax_atomic(mn, mx, arena + B[cur].minmax_off, red);
        cur = d.task; mn = DFQ_INF; mx = -DFQ_INF;
      }
      if (d.kind == TK_DIRECT) {
        for (int i = threadIdx.x; i < d.floats; i += kThreads) { const float v = ldg_stream1(d.gptr + i); mn = fminf(mn, v); mx = fmaxf(mx, v); }
      } else if ((d.floats & 3) == 0) {
        const float4* b4 = (const float4*)pipe.stage[sidx];
        for (int i = threadIdx.x; i < (d.floats >> 2); i += kThreads) {
          const float4 v = b4[i];
          mn = fminf(mn, fminf(fminf(v.x, v.y), fminf(v.z, v.w)));
          mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
        }
      } else {
        const float* bf = pipe.stage[sidx];
        for (int i = threadIdx.x; i < d.floats; i += kThreads) { mn = fminf(mn, bf[i]); mx = fmaxf(mx, bf[i]); }
      }
      bool more = false;
      if (threadIdx.x == 0) { more = ahead.valid(); if (more) { ahead.fill(nd); ahead.next(); } }
      pipe.release<false>(sidx, more, nd);
      it.next();
    }
    if (cur >= 0) cta_minmax_atomic(mn, mx, arena + B[cur].minmax_off, red);
  }
  grid.sync();

  for (int lev = 0; lev < n_levels; ++lev) {
    // ---- E[x] of every layer of this level (dfq.py:228-278); one CTA per layer, terms in order ----
    // A level of a few small layers (level_local: a serial model, one layer per level) skips this phase and its grid barrier:
    // every CTA evaluates the recipe itself, straight into its shared-memory copy, when it reaches the layer below.
    const bool local = level_local[lev] != 0;
    if (!local) {
    for (int bi = level_ptr[lev] + blockIdx.x; bi < level_ptr[lev + 1]; bi += gridDim.x) {
      const DfqBcLayer b = B[bi];
      float* ex = arena + b.expect_off;
      for (int ti = b.term_begin; ti < b.term_end; ++ti) {
        const DfqExpectTerm t = T[ti];
        for (int ch = threadIdx.x; ch < t.n; ch += kThreads) {
          const float fb = __ldcg(arena + t.bn_b_off + ch);
          const float v = t.relu ? relu_gauss_mean(__ldcg(arena + t.bn_w_off + ch), fb) : fb;
          float* d = ex + t.dst_off + ch;
          __stcg(d, t.accumulate ? __fadd_rn(__ldcg(d), v) : v);
        }
        __syncthreads();
      }
    }
    grid.sync();
    }
    // ---- eps . E[x] per output row (dfq.py:216-219,281-293): rows streamed through the pipe, read only ---------
    MatIter<BcGeo> it;
    it.start(row_ptr, level_ptr[lev], level_ptr[lev + 1], BcGeo{arena, L, B});
    MatIter<BcGeo> ahead = it;
    if (threadIdx.x == 0)
      for (int i = 0; i < kPipeStages - 1 && ahead.valid(); ++i) { ahead.fill(nd); pipe.issue(nd); ahead.next(); }
    int cur = -1;
    DfqBcLayer b; DfqLayer l; QuantScalars q; int so = 1, ex_cached = 0;
    while (it.valid()) {
      const int sidx = pipe.acquire();
      const TileDesc d = pipe.desc[sidx];
      if (d.task != cur) {
        cur = d.task;
        b = B[cur]; l = L[b.layer];
        q = quant_scalars((double)__ldcg(arena + b.minmax_off), (double)__ldcg(arena + b.minmax_off + 1), num_bits, b.signed_mode);
        so = l.rows / (b.expect_len / l.cols);
        ex_cached = (b.expect_len <= kExpectCache);
        __syncthreads();
        if (local) {             // host guarantees expect_len <= kExpectCache for every layer of a local level
          for (int ti = b.term_begin; ti < b.term_end; ++ti) {
            const DfqExpectTerm t = T[ti];
            for (int ch = threadIdx.x; ch < t.n; ch += kThreads) {
              const float fb = __ldcg(arena + t.bn_b_off + ch);
              const float v = t.relu ? relu_gauss_mean(__ldcg(arena + t.bn_w_off + ch), fb) : fb;
              float* dst = s_ex + t.dst_off + ch;
              *dst = t.accumulate ? __fadd_rn(*dst, v) : v;
            }
            __syncthreads();
          }
        } else if (ex_cached) {
          for (int j = threadIdx.x; j < b.expect_len; j += kThreads) s_ex[j] = __ldcg(arena + b.expect_off + j);
          __syncthreads();
        }
      }
      const int row_len = l.cols * l.kk;
      const bool raw = (b.flags & 1) != 0;
      if (d.nrows == 1) {
        const int o = d.row0;
        const float* row = (d.kind == TK_DIRECT) ? d.gptr : pipe.stage[sidx];
        const float* ex = (ex_cached ? s_ex : arena + b.expect_off) + (size_t)(o / so) * l.cols;
        // the leader's read-modify-write operands are requested before the row is processed: their latency is hidden
        float old_bias = 0.f, old_next = 0.f;
        if (threadIdx.x == 0) {
          old_bias = __ldcg(arena + l.bias_off + o);
          if (b.next_bn_b_off >= 0) old_next = __ldcg(arena + b.next_bn_b_off + o);
        }
        double acc = raw ? bc_row<kThreads, true>(row, l.cols, l.kk, ex, q, threadIdx.x)
                         : bc_row<kThreads, false>(row, l.cols, l.kk, ex, q, threadIdx.x);
        if (lane == 0) dred[warp] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
          acc = 0.0;
#pragma unroll
          for (int i = 0; i < kWarps; ++i) acc += dred[i];
          const float dl = (float)acc;
          __stcg(arena + b.delta_off + o, dl);
          __stcg(arena + l.bias_off + o, __fadd_rn(old_bias, (b.flags & 2) ? dl : -dl));              // dfq.py:292 / :164
          if (b.next_bn_b_off >= 0) __stcg(arena + b.next_bn_b_off + o, __fadd_rn(old_next, -dl));   // dfq.py:204-206,293
        }
      } else {
        // a warp per row, 32 rows per batch: lane j requests row j's read-modify-write operands before the batch and
        // writes row j's results after it (two global-memory latencies per batch instead of two per row)
        const int mine = (d.nrows - warp + kWarps - 1) / kWarps;
        for (int base = 0; base < mine; base += 32) {
          const int il = base + lane;
          const int ol = d.row0 + warp + il * kWarps;
          float old_bias = 0.f, old_next = 0.f, dl = 0.f;
          if (il < mine) {
            old_bias = __ldcg(arena + l.bias_off + ol);
            if (b.next_bn_b_off >= 0) old_next = __ldcg(arena + b.next_bn_b_off + ol);
          }
          const int nb = min(32, mine - base);
          for (int j = 0; j < nb; ++j) {
            const int r = warp + (base + j) * kWarps;
            const int o = d.row0 + r;
            const float* row = pipe.stage[sidx] + (size_t)r * row_len;
            const float* ex = (ex_cached ? s_ex : arena + b.expect_off) + (size_t)(o / so) * l.cols;
            const double acc = raw ? bc_row<32, true>(row, l.cols, l.kk, ex, q, lane) : bc_row<32, false>(row, l.cols, l.kk, ex, q, lane);
            if (lane == j) dl = (float)acc;
          }
          if (il < mine) {
            __stcg(arena + b.delta_off + ol, dl);
            __stcg(arena + l.bias_off + ol, __fadd_rn(old_bias, (b.flags & 2) ? dl : -dl));              // dfq.py:292 / :164
            if (b.next_bn_b_off >= 0) __stcg(arena + b.next_bn_b_off + ol, __fadd_rn(old_next, -dl));   // dfq.py:204-206,293
          }
        }
      }
      bool more = false;
      if (threadIdx.x == 0) { more = ahead.valid(); if (more) { ahead.fill(nd); ahead.next(); } }
      pipe.release<false>(sidx, more, nd);
      it.next();
    }
    grid.sync();
  }
}


// ------------------------------------------------------------------------------------------------
// bias correction, streaming variant (bc_stream.cuh): warp-autonomous consumers, no CTA barrier per tile
// ------------------------------------------------------------------------------------------------
static_assert(kPipeMaxRows <= 32, "a consumer warp retires one row per lane");

// Producer side of one ring phase: this CTA's tiles of tasks [q_begin, q_end) in block-cyclic order, then SKIP items up to
// a multiple of kBcConsumers, then one END per consumer.  Called by lane 0 of the producer warp only.
__device__ __forceinline__ void bc_feed(BcRing& ring, unsigned long long& n, const long long* ptr, int q_begin, int q_end,
                                        const BcGeo& geo) {
  TileDesc d;
#ifndef DFQ_BC_FEED_CACHE
#define DFQ_BC_FEED_CACHE 1
#endif
  MatIter<BcGeo, DFQ_BC_FEED_CACHE != 0> it;
  it.start(ptr, q_begin, q_end, geo);
  while (it.valid()) { it.fill(d); bc_produce(ring, n++, d); it.next(); }
  d.gptr = nullptr; d.task = -1; d.row0 = d.nrows = d.floats = 0;
  d.kind = BTK_SKIP;
  while (n % kBcConsumers) bc_produce(ring, n++, d);
  d.kind = BTK_END;
  for (int i = 0; i < kBcConsumers; ++i) bc_produce(ring, n++, d);
}

__global__ void __launch_bounds__(kBcThreads, 1)
k_bc_stream(float* arena, const DfqLayer* __restrict__ L, const DfqBcLayer* __restrict__ B, int nB,
            const DfqExpectTerm* __restrict__ T, const int* __restrict__ level_ptr, int n_levels, int num_bits,
            const long long* __restrict__ row_ptr, const long long* __restrict__ mm_ptr) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(128) unsigned char ring_smem[];
  BcRing ring;
  ring.init(ring_smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool producer = (warp == kBcConsumers);
  unsigned long long n = producer ? 0 : (unsigned long long)warp;     // producer: next sequence number; consumer: my next item
  const BcGeo geo{arena, L, B};

  // ---- per-tensor min/max of every corrected weight (dfq.py:14 via :218) --------------------------------------
  for (int i = blockIdx.x * kBcThreads + threadIdx.x; i < nB; i += gridDim.x * kBcThreads) {
    __stcg(arena + B[i].minmax_off, DFQ_INF);
    __stcg(arena + B[i].minmax_off + 1, -DFQ_INF);
  }
  grid.sync();
  // caller-vouched column extrema (DfqBcLayer.n_col > 0): a warp per layer reduces them
  for (int bi = blockIdx.x * (kBcThreads / 32) + warp; bi < nB; bi += gridDim.x * (kBcThreads / 32)) {
    const DfqBcLayer b = B[bi];
    if (b.n_col <= 0) continue;
    float mn = DFQ_INF, mx = -DFQ_INF;
    for (int j = lane; j < b.n_col; j += 32) {
      mn = fminf(mn, __ldcg(arena + b.colmin_off + j)); mx = fmaxf(mx, __ldcg(arena + b.colmax_off + j));
    }
    mn = warp_min(mn); mx = warp_max(mx);
    if (lane == 0) { atomic_min_f(arena + b.minmax_off, mn); atomic_max_f(arena + b.minmax_off + 1, mx); }
  }
  if (mm_ptr[nB] > 0) {          // the others: streamed through the ring, one min/max pair per tile
    if (producer) {
      if (lane == 0) bc_feed(ring, n, mm_ptr, 0, nB, geo);
    } else {
      for (;; n += kBcConsumers) {
        const int s = bc_take(ring, n);
        const TileDesc d = ring.desc[s];
        if (d.kind == BTK_END) { bc_give_back(ring, s, lane); n += kBcConsumers; break; }
        if (d.kind != BTK_SKIP) {
          float mn = DFQ_INF, mx = -DFQ_INF;
          if (d.kind == TK_BULK && (d.floats & 3) == 0) {
            const float4* b4 = (const float4*)ring.stage(s);
            for (int i = lane; i < (d.floats >> 2); i += 32) {
              const float4 v = b4[i];
              mn = fminf(mn, fminf(fminf(v.x, v.y), fminf(v.z, v.w)));
              mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
            }
          } else if (d.kind == TK_BULK) {
            for (int i = lane; i < d.floats; i += 32) { const float v = ring.stage(s)[i]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
          } else {
            for (int i = lane; i < d.floats; i += 32) { const float v = ldg_stream1(d.gptr + i); mn = fminf(mn, v); mx = fmaxf(mx, v); }
          }
          mn = warp_min(mn); mx = warp_max(mx);
          if (lane == 0) { atomic_min_f(arena + B[d.task].minmax_off, mn); atomic_max_f(arena + B[d.task].minmax_off + 1, mx); }
        }
        bc_give_back(ring, s, lane);
      }
    }
  }
  grid.sync();

  for (int lev = 0; lev < n_levels; ++lev) {
    // ---- E[x] of every layer of this level (dfq.py:228-278); one CTA per layer, terms in order ----
    for (int bi = level_ptr[lev] + blockIdx.x; bi < level_ptr[lev + 1]; bi += gridDim.x) {
      const DfqBcLayer b = B[bi];
      float* ex = arena + b.expect_off;
      for (int ti = b.term_begin; ti < b.term_end; ++ti) {
        const DfqExpectTerm t = T[ti];
        for (int ch = threadIdx.x; ch < t.n; ch += kBcThreads) {
          const float fb = __ldcg(arena + t.bn_b_off + ch);
          const float v = t.relu ? relu_gauss_mean(__ldcg(arena + t.bn_w_off + ch), fb) : fb;
          float* d = ex + t.dst_off + ch;
          __stcg(d, t.accumulate ? __fadd_rn(__ldcg(d), v) : v);
        }
        __syncthreads();
      }
    }
    grid.sync();
    // ---- eps . E[x] per output row (dfq.py:216-219,281-293) ---------------------------------------------------
    if (producer) {
      if (lane == 0) bc_feed(ring, n, row_ptr, level_ptr[lev], level_ptr[lev + 1], geo);
    } else {
      int cur = -1, cur_group = -1, so = 1;
      DfqBcLayer b; DfqLayer l; BcFastQuant f;
      int mode = 1;                                  // 0: XU-free arithmetic, 1: IEEE chain, 2: raw sums (bias absorption)
      bool excached = false;
      float* exs = ring.ex_cache(warp);
      for (;; n += kBcConsumers) {
        const int s = bc_take(ring, n);
        const TileDesc d = ring.desc[s];
        if (d.kind == BTK_END) { bc_give_back(ring, s, lane); n += kBcConsumers; break; }
        if (d.kind == BTK_SKIP) { bc_give_back(ring, s, lane); continue; }
        if (d.task != cur) {
          cur = d.task; cur_group = -1;
          b = B[cur]; l = L[b.layer];
          f = bc_fast_quant(quant_scalars((double)__ldcg(arena + b.minmax_off), (double)__ldcg(arena + b.minmax_off + 1),
                                          num_bits, b.signed_mode), num_bits);
          so = l.rows / (b.expect_len / l.cols);
          mode = (b.flags & 1) ? 2 : (f.ok ? 0 : 1);
          excached = l.cols <= kBcExCols;
        }
        const int row_len = l.cols * l.kk;
        if (d.kind == TK_PLAIN) {       // a tile the TMA unit cannot move: the warp fetches it itself
          for (int i = lane; i < d.floats; i += 32) ring.stage(s)[i] = ldg_stream1(d.gptr + i);
          __syncwarp();
        }
        // lane r requests row r's read-modify-write operands before the tile and retires them after it
        float old_bias = 0.f, old_next = 0.f, dl = 0.f;
        if (lane < d.nrows) {
          old_bias = __ldcg(arena + l.bias_off + d.row0 + lane);
          if (b.next_bn_b_off >= 0) old_next = __ldcg(arena + b.next_bn_b_off + d.row0 + lane);
        }
        const uint32_t sbase = smem_u32(ring.stage(s));
        // (Tried: copying a [512,3,3] row to registers - 144 per lane, 224 registers per thread - and handing the stage back
        // BEFORE the arithmetic, so that the whole ring is loading.  The straight-line code that needs (16 columns x 9 taps
        // fully unrolled, ~1900 instructions, every warp at a different place in it) misses the instruction cache like the very
        // first version of this kernel did, and was slower.  The rolled shared-memory loop stays.)
        for (int r = 0; r < d.nrows; ++r) {
          const int g = (d.row0 + r) / so;
          const float* ex = arena + b.expect_off + (size_t)g * l.cols;
          if (excached && g != cur_group) {
            cur_group = g;
            __syncwarp();
            for (int j = lane; j < l.cols; j += 32) exs[j] = __ldcg(ex + j);
            __syncwarp();
          }
          double acc;
          if (d.kind == TK_DIRECT) {
            const float* row = d.gptr + (size_t)r * row_len;
            acc = mode == 0 ? bc_stream_row_gmem<0>(row, l.cols, l.kk, ex, f, lane)
                : mode == 1 ? bc_stream_row_gmem<1>(row, l.cols, l.kk, ex, f, lane)
                            : bc_stream_row_gmem<2>(row, l.cols, l.kk, ex, f, lane);
          } else {
            const uint32_t srow = sbase + (uint32_t)r * (uint32_t)row_len * 4u;
            const float* xs = excached ? exs : nullptr;
            if (mode == 0) {
              acc = l.kk == 9 ? bc_stream_row_smem<0, 9>(srow, l.cols, 9, xs, ex, f, lane)
                  : l.kk == 1 ? bc_stream_row_smem<0, 1>(srow, l.cols, 1, xs, ex, f, lane)
                              : bc_stream_row_smem<0, 0>(srow, l.cols, l.kk, xs, ex, f, lane);
            } else if (mode == 1) {
              acc = bc_stream_row_smem<1, 0>(srow, l.cols, l.kk, xs, ex, f, lane);
            } else {
              acc = bc_stream_row_smem<2, 0>(srow, l.cols, l.kk, xs, ex, f, lane);
            }
          }
          if (lane == r) dl = (float)acc;
        }
        if (lane < d.nrows) {
          const int ol = d.row0 + lane;
          __stcg(arena + b.delta_off + ol, dl);
          __stcg(arena + l.bias_off + ol, __fadd_rn(old_bias, (b.flags & 2) ? dl : -dl));              // dfq.py:292 / :164
          if (b.next_bn_b_off >= 0) __stcg(arena + b.next_bn_b_off + ol, __fadd_rn(old_next, -dl));   // dfq.py:204-206,293
        }
        bc_give_back(ring, s, lane);
      }
    }
    grid.sync();
  }
}

// Library self-test hook: the element-wise quantization error Q(w) - w of one tensor computed with the streaming kernel's
// XU-free arithmetic (eps_fast) and with the plain IEEE chain of quantize.py:70-74 (eps_div); *ok = the per-tensor guard.
__global__ void k_bc_selftest(const float* __restrict__ w, float* eps_fast, float* eps_div, int64_t n,
                              const float* __restrict__ minmax2, int num_bits, int symmetric, int* ok) {
  const QuantScalars q = quant_scalars((double)minmax2[0], (double)minmax2[1], num_bits, symmetric);
  const BcFastQuant f = bc_fast_quant(q, num_bits);
  if (blockIdx.x == 0 && threadIdx.x == 0) *ok = f.ok;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x = w[i];
    eps_fast[i] = bc_qerr_own_range(x, f);
    eps_div[i] = __fsub_rn(fake_quant<false>(x, q), x);
  }
}

}  // namespace dfq

using namespace dfq;

static int pick_grid(const void* kernel, int64_t max_tiles, int* grid, size_t dyn_smem = 0) {
  int dev = 0, sms = 0, per_sm = 0;
  DFQ_CUDA(cudaGetDevice(&dev));
  DFQ_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  DFQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, dyn_smem));
  if (per_sm < 1) { set_error("kernel does not fit on an SM"); return DFQ_E_NOT_COOPERATIVE; }
  *grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)sms * per_sm, max_tiles));
  return 0;
}

extern "C" int dfq_bn_fold(float* arena, int64_t arena_floats, const DfqLayer* layers, int32_t n_layers,
                           const DfqFold* folds, int32_t n_folds, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(arena && layers && folds, "null argument");
  if (n_folds <= 0) return 0;
  std::vector<long long> tptr(n_folds + 1, 0);
  bool any_scan = false;
  for (int i = 0; i < n_folds; ++i) {
    DFQ_REQUIRE(folds[i].layer >= 0 && folds[i].layer < n_layers, "fold layer index");
    const DfqLayer& l = layers[folds[i].layer];
    DFQ_REQUIRE(l.w_off >= 0 && l.w_off + (int64_t)l.rows * l.cols * l.kk <= arena_floats, "weight outside arena");
    tptr[i + 1] = tptr[i] + pipe_tiles(l.rows, l.cols * l.kk);
    if (folds[i].scan_go > 0) {
      const DfqFold& f = folds[i];
      DFQ_REQUIRE(f.scan_gi > 0 && l.rows % f.scan_go == 0 && f.scan_gi == l.cols, "fold scan geometry (DfqRelation.go / .gi of the layer's rel_in)");
      const int64_t nch = (int64_t)(l.rows / f.scan_go) * f.scan_gi;
      DFQ_REQUIRE(l.cmin_off >= 0 && l.cmax_off >= 0 && l.cmin_off + 2 * nch <= arena_floats && l.cmax_off + 2 * nch <= arena_floats,
                  "fold scan needs the layer's column range scratch");
      any_scan = true;
    }
  }
  int grid, rc;
  const size_t dyn = RowPipe::smem_bytes();
  DFQ_CUDA(cudaFuncSetAttribute(k_bn_fold, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
  if ((rc = pick_grid((const void*)k_bn_fold, tptr[n_folds], &grid, dyn))) return rc;
  TablePack tp;
  const int iL = tp.add(layers, n_layers), iF = tp.add(folds, n_folds), iP = tp.add(tptr.data(), n_folds + 1);
  if ((rc = tp.upload(st))) return rc;
  if (any_scan) k_fold_reset_cols<<<std::min(n_folds, 4096), 128, 0, st>>>(arena, tp.ptr<DfqLayer>(iL), tp.ptr<DfqFold>(iF), n_folds);
  k_bn_fold<<<grid, kThreads, dyn, st>>>(arena, tp.ptr<DfqLayer>(iL), tp.ptr<DfqFold>(iF), n_folds, tp.ptr<long long>(iP));
  DFQ_CUDA(cudaGetLastError());
  tp.release(st);
  return 0;
}

extern "C" int dfq_quantize_tensors(float* arena, int64_t arena_floats, const DfqQuantTask* tasks, int32_t n_tasks,
                                    int div_mode, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(arena && tasks, "null argument");
  if (n_tasks <= 0) return 0;
  std::vector<FlatTask> ft(n_tasks);
  std::vector<long long> tptr(n_tasks + 1, 0);
  for (int i = 0; i < n_tasks; ++i) {
    DFQ_REQUIRE(tasks[i].off >= 0 && tasks[i].n > 0 && tasks[i].off + tasks[i].n <= arena_floats, "tensor outside arena");
    DFQ_REQUIRE(tasks[i].minmax_off >= 0 && tasks[i].minmax_off + 2 <= arena_floats, "minmax scratch outside arena");
    DFQ_REQUIRE(tasks[i].num_bits >= 1 && tasks[i].num_bits <= 32, "num_bits");
    ft[i] = {tasks[i].off, tasks[i].n, tasks[i].minmax_off, tasks[i].num_bits, tasks[i].symmetric};
    tptr[i + 1] = tptr[i] + (tasks[i].n + kChunk - 1) / kChunk;
  }
  int grid, rc;
  if ((rc = pick_grid((const void*)k_minmax_tasks, tptr[n_tasks], &grid))) return rc;
  TablePack tp;
  const int iT = tp.add(ft.data(), n_tasks), iP = tp.add(tptr.data(), n_tasks + 1);
  if ((rc = tp.upload(st))) return rc;
  FlatTask* dT = tp.ptr<FlatTask>(iT); long long* dP = tp.ptr<long long>(iP);
  k_minmax_init<<<std::min(std::max(1, sm_count()), (n_tasks + 255) / 256), 256, 0, st>>>(arena, dT, n_tasks);
  k_minmax_tasks<<<grid, kThreads, 0, st>>>(arena, dT, n_tasks, dP);
  if (div_mode) k_quant_tasks<true><<<grid, kThreads, 0, st>>>(arena, dT, n_tasks, dP);
  else          k_quant_tasks<false><<<grid, kThreads, 0, st>>>(arena, dT, n_tasks, dP);
  DFQ_CUDA(cudaGetLastError());
  tp.release(st);
  return 0;
}

extern "C" int dfq_bias_correct(float* arena, int64_t arena_floats, const DfqLayer* layers, int32_t n_layers,
                                const DfqBcLayer* bc, int32_t n_bc, const DfqExpectTerm* terms, int32_t n_terms,
                                const int32_t* level_ptr, int32_t n_levels, int32_t num_bits, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool trace = getenv("DFQ_TRACE") != nullptr;
  const auto h0 = std::chrono::steady_clock::now();
  auto ms_since = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - h0).count(); };
  DFQ_REQUIRE(arena && layers && bc && terms && level_ptr, "null argument");
  if (n_bc <= 0 || n_levels <= 0) return 0;
  DFQ_REQUIRE(level_ptr[0] == 0 && level_ptr[n_levels] == n_bc, "levels must partition the layer list");
  int64_t max_tiles = 1;
  std::vector<long long> row_ptr(n_bc + 1, 0), mm_ptr(n_bc + 1, 0);
  for (int i = 0; i < n_bc; ++i) {
    const DfqBcLayer& b = bc[i];
    DFQ_REQUIRE(b.layer >= 0 && b.layer < n_layers, "bc layer index");
    const DfqLayer& l = layers[b.layer];
    DFQ_REQUIRE(b.expect_len > 0 && b.expect_len % l.cols == 0, "expectation length must be groups*cols");
    DFQ_REQUIRE(l.rows % (b.expect_len / l.cols) == 0, "rows not divisible by groups");
    DFQ_REQUIRE(b.term_begin >= 0 && b.term_end <= n_terms && b.term_begin <= b.term_end, "term range");
    for (int t = b.term_begin; t < b.term_end; ++t)
      DFQ_REQUIRE(terms[t].dst_off >= 0 && terms[t].dst_off + terms[t].n <= b.expect_len, "term outside expectation vector");
    DFQ_REQUIRE(b.expect_off >= 0 && b.expect_off + b.expect_len <= arena_floats, "expect scratch outside arena");
    row_ptr[i + 1] = row_ptr[i] + pipe_tiles(l.rows, l.cols * l.kk);
    if (b.n_col > 0)
      DFQ_REQUIRE(b.colmin_off >= 0 && b.colmax_off >= 0 && b.colmin_off + b.n_col <= arena_floats && b.colmax_off + b.n_col <= arena_floats,
                  "column-extrema hint outside arena");
    mm_ptr[i + 1] = mm_ptr[i] + (b.n_col > 0 ? 0 : pipe_tiles(l.rows, l.cols * l.kk));
  }
  max_tiles = std::max<int64_t>(max_tiles, row_ptr[n_bc]);
  std::vector<int32_t> level_local(n_levels, 0);
  for (int lv = 0; lv < n_levels; ++lv) {
    bool ok = (level_ptr[lv + 1] - level_ptr[lv]) <= 4;
    for (int i = level_ptr[lv]; ok && i < level_ptr[lv + 1]; ++i) ok = bc[i].expect_len <= kExpectCache;
    level_local[lv] = ok ? 1 : 0;
  }
  int grid, rc;
  // Large phases (bandwidth-bound: many tiles per CTA and level) take the streaming kernel, small models (latency-bound:
  // a few tiles per level, level_local shortcuts) the per-CTA engine.  DFQ_BC_STREAM=0/1 forces one of them.
  const int sms = std::max(1, sm_count());
  bool stream_variant = row_ptr[n_bc] >= (long long)16 * sms * n_levels;
  if (const char* e = getenv("DFQ_BC_STREAM")) stream_variant = atoi(e) != 0;
  if (stream_variant) {
    const size_t dyn_s = BcRing::smem_bytes();
    DFQ_CUDA(cudaFuncSetAttribute(k_bc_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_s));
    int per_sm = 0;
    DFQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_bc_stream, kBcThreads, dyn_s));
    if (per_sm < 1) { set_error("k_bc_stream does not fit on an SM"); return DFQ_E_NOT_COOPERATIVE; }
    grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)sms * per_sm, max_tiles));
    TablePack tp;
    const int iL = tp.add(layers, n_layers), iB = tp.add(bc, n_bc), iT = tp.add(terms, n_terms);
    const int iLP = tp.add(level_ptr, n_levels + 1), iRP = tp.add(row_ptr.data(), n_bc + 1), iMP = tp.add(mm_ptr.data(), n_bc + 1);
    if ((rc = tp.upload(st))) return rc;
    DfqLayer* dL = tp.ptr<DfqLayer>(iL); DfqBcLayer* dB = tp.ptr<DfqBcLayer>(iB); DfqExpectTerm* dT = tp.ptr<DfqExpectTerm>(iT);
    int32_t* dLP = tp.ptr<int32_t>(iLP); long long* dRP = tp.ptr<long long>(iRP); long long* dMP = tp.ptr<long long>(iMP);
    void* args[] = {&arena, &dL, &dB, (void*)&n_bc, &dT, &dLP, (void*)&n_levels, (void*)&num_bits, &dRP, &dMP};
    DFQ_CUDA(cudaLaunchCooperativeKernel((void*)k_bc_stream, dim3(grid), dim3(kBcThreads), args, dyn_s, st));
    tp.release(st);
    if (trace) fprintf(stderr, "[dfq_bias_correct] streaming variant, grid %d, host ms %.3f\n", grid, ms_since());
    return 0;
  }
  const size_t dyn = RowPipe::smem_bytes();
  DFQ_CUDA(cudaFuncSetAttribute(k_bc_engine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
  if ((rc = pick_grid((const void*)k_bc_engine, max_tiles, &grid, dyn))) return rc;
  TablePack tp;
  const int iL = tp.add(layers, n_layers), iB = tp.add(bc, n_bc), iT = tp.add(terms, n_terms);
  const int iLP = tp.add(level_ptr, n_levels + 1), iRP = tp.add(row_ptr.data(), n_bc + 1), iMP = tp.add(mm_ptr.data(), n_bc + 1);
  const int iLL = tp.add(level_local.data(), n_levels);
  if ((rc = tp.upload(st))) return rc;
  DfqLayer* dL = tp.ptr<DfqLayer>(iL); DfqBcLayer* dB = tp.ptr<DfqBcLayer>(iB); DfqExpectTerm* dT = tp.ptr<DfqExpectTerm>(iT);
  int32_t* dLP = tp.ptr<int32_t>(iLP); long long* dRP = tp.ptr<long long>(iRP); long long* dMP = tp.ptr<long long>(iMP);
  int32_t* dLL = tp.ptr<int32_t>(iLL);
  void* args[] = {&arena, &dL, &dB, (void*)&n_bc, &dT, &dLP, (void*)&n_levels, (void*)&num_bits, &dRP, &dMP, &dLL};
  const double h_prep = ms_since();
  DFQ_CUDA(cudaLaunchCooperativeKernel((void*)k_bc_engine, dim3(grid), dim3(kThreads), args, dyn, st));
  tp.release(st);
  if (trace) fprintf(stderr, "[dfq_bias_correct] host ms: tables+upload %.3f, launch returned %.3f\n", h_prep, ms_since());
  return 0;
}

extern "C" int dfq_selftest_bc_arithmetic(const float* w, float* eps_fast, float* eps_div, int64_t n, const float* minmax2,
                                          int num_bits, int symmetric, int* ok_dev, void* stream) {
  DFQ_REQUIRE(w && eps_fast && eps_div && minmax2 && ok_dev && n > 0, "bad argument");
  k_bc_selftest<<<(int)std::min<int64_t>((int64_t)std::max(1, sm_count()) * 8, (n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, eps_fast, eps_div, n, minmax2,
                                                                                                   num_bits, symmetric, ok_dev);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}
