// BN-statistics matching loss of the distilled-data generation (ZeroQ/distill_data.py:171-196), fused.
//
// The reference evaluates, per BatchNorm layer and per Adam iteration, on the layer's INPUT x [N, C, H, W]:
//     m[n,c] = mean_hw x                              (:176-178)
//     s[n,c] = std_hw (x + eps)   (unbiased)          (:179-182)
//     L_mean = sum_{n,c} (mu[c] - m[n,c])^2 / C       own_loss, :41-46
//     L_std  = sum_{n,c} (sigma[c] - s[n,c])^2 / C
// with a dozen eager ops and several full-size temporaries, and autograd replays them backwards.  Here:
//   forward  ONE pass over x: a warp (short rows) or a CTA (long rows) per (n, c) row accumulates sum(y), sum(y^2), y = x + eps,
//            in float64; m, s are kept for the backward pass, the two losses are accumulated with one atomicAdd(double) pair
//            per CTA;
//   backward ONE pass: dL/dx[n,c,i] = gm * 2 (m - mu_c) / (C*HW)  +  gs * 2 (s - sigma_c) / C * (y_i - mean(y)) / ((HW-1) * s)
//            ACCUMULATED into the gradient buffer (the layer's input also receives the gradient of the network path).
// HBM-bound: 4 B/element forward, 8-12 B/element backward.
#include <cstdint>

#include "common.cuh"

namespace dfq {

constexpr int kDThreads = 256;
// dfq_bnstat_loss_fwd: rows of at least this many elements get a CTA each, shorter ones a warp
constexpr int kBnstatCtaRow = 2048;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// rows = N*C rows of hw floats.  CTA_ROW: one CTA per row (hw large), else one warp per row.
template <bool CTA_ROW>
__global__ void __launch_bounds__(kDThreads)
k_bnstat_fwd(const float* __restrict__ x, int64_t rows, int64_t hw, int C, const float* __restrict__ mu,
             const float* __restrict__ sigma, float eps, float* __restrict__ m_out, float* __restrict__ s_out, double* loss2) {
  __shared__ double red[3][kDThreads / 32];
  __shared__ float redf[2][kDThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double lm = 0.0, ls = 0.0;
  const int64_t step = CTA_ROW ? gridDim.x : (int64_t)gridDim.x * (kDThreads / 32);
  for (int64_t r = CTA_ROW ? blockIdx.x : blockIdx.x * (int64_t)(kDThreads / 32) + warp; r < rows; r += step) {
    const float* p = x + r * hw;
    double a = 0.0, b = 0.0, sx = 0.0;       // sum(y), sum(y^2) with y = x + eps, and sum(x)
    float ylo = DFQ_INF, yhi = -DFQ_INF;     // extrema of y: a constant row gets s = 0 exactly
    const int tid = CTA_ROW ? threadIdx.x : lane, nt = CTA_ROW ? kDThreads : 32;
    if ((hw & 3) == 0 && ((((uintptr_t)p) & 15) == 0)) {
      const float4* p4 = (const float4*)p;
      for (int64_t i = tid; i < (hw >> 2); i += nt) {
        const float4 v = __ldg(p4 + i);
        const float y0 = __fadd_rn(v.x, eps), y1 = __fadd_rn(v.y, eps), y2 = __fadd_rn(v.z, eps), y3 = __fadd_rn(v.w, eps);
        a += ((double)y0 + (double)y1) + ((double)y2 + (double)y3);
        b += ((double)y0 * y0 + (double)y1 * y1) + ((double)y2 * y2 + (double)y3 * y3);
        sx += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w);
        ylo = fminf(ylo, fminf(fminf(y0, y1), fminf(y2, y3))); yhi = fmaxf(yhi, fmaxf(fmaxf(y0, y1), fmaxf(y2, y3)));
      }
    } else {
      for (int64_t i = tid; i < hw; i += nt) {
        const float v = __ldg(p + i), y = __fadd_rn(v, eps);
        a += (double)y; b += (double)y * y; sx += (double)v;
        ylo = fminf(ylo, y); yhi = fmaxf(yhi, y);
      }
    }
    a = warp_sum_d(a); b = warp_sum_d(b); sx = warp_sum_d(sx);
    ylo = warp_min(ylo); yhi = warp_max(yhi);
    if (CTA_ROW) {
      __syncthreads();
      if (lane == 0) { red[0][warp] = a; red[1][warp] = b; red[2][warp] = sx; redf[0][warp] = ylo; redf[1][warp] = yhi; }
      __syncthreads();
      a = 0.0; b = 0.0; sx = 0.0;
      for (int i = 0; i < kDThreads / 32; ++i) {
        a += red[0][i]; b += red[1][i]; sx += red[2][i]; ylo = fminf(ylo, redf[0][i]); yhi = fmaxf(yhi, redf[1][i]);
      }
    }
    if (tid == 0) {
      const double n = (double)hw;
      const double mean_y = a / n;
      double var = (b - a * mean_y) / (n - 1.0);       // unbiased; hw == 1 -> 0/0 = NaN like torch.std
      // the single-pass variance of a constant row rounds to a tiny value of either sign instead of 0 (a NaN stays)
      if (var < 0.0 || (var > 0.0 && ylo == yhi)) var = 0.0;
      const float m = (float)(sx / n), s = (float)sqrt(var);
      m_out[r] = m; s_out[r] = s;
      const int c = (int)(r % C);
      const double dm = (double)mu[c] - (double)m, dsd = (double)sigma[c] - (double)s;
      lm += dm * dm; ls += dsd * dsd;
    }
  }
  // one atomic pair per CTA
  lm = warp_sum_d(lm); ls = warp_sum_d(ls);
  __syncthreads();
  if (lane == 0) { red[0][warp] = lm; red[1][warp] = ls; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double A = 0.0, B = 0.0;
    for (int i = 0; i < kDThreads / 32; ++i) { A += red[0][i]; B += red[1][i]; }
    if (A != 0.0 || B != 0.0) { atomicAdd(loss2, A / (double)C); atomicAdd(loss2 + 1, B / (double)C); }
  }
}

// dL/dm per element of a row, and the coefficient of (y_i - mean(y)) in dL/ds per element.  A zero-variance row (a dead
// channel) has no std gradient: torch's std backward masks std == 0 to 0, where 1/s would give inf (or NaN for x == 0).
__device__ __forceinline__ double bnstat_mean_coef(double gm, float m, float mu, double inv_c, int64_t hw) {
  return gm * 2.0 * ((double)m - (double)mu) * inv_c / (double)hw;
}
__device__ __forceinline__ double bnstat_std_coef(double gs, float s, float sigma, double inv_c, int64_t hw) {
  if (s == 0.f) return 0.0;
  return gs * 2.0 * ((double)s - (double)sigma) * inv_c / ((double)(hw - 1) * (double)s);
}

__global__ void __launch_bounds__(kDThreads)
k_bnstat_bwd(const float* __restrict__ x, float* __restrict__ gx, int64_t rows, int64_t hw, int C, const float* __restrict__ mu,
             const float* __restrict__ sigma, float eps, const float* __restrict__ m_in, const float* __restrict__ s_in,
             const float* __restrict__ g2, int accumulate) {
  const double gm = (double)g2[0], gs = (double)g2[1];
  const int64_t n = rows * hw;
  const double inv_c = 1.0 / (double)C;
  for (int64_t i = (blockIdx.x * (int64_t)kDThreads + threadIdx.x) * 4; i < n; i += (int64_t)gridDim.x * kDThreads * 4) {
    // four consecutive elements; a row boundary may fall inside when hw % 4 != 0: handle element-wise
    float out[4];
    const int lim = (int)min((int64_t)4, n - i);
    int64_t r = i / hw;
    int64_t off = i - r * hw;
    float m = m_in[r], s = s_in[r];
    int c = (int)(r % C);
    double ka = bnstat_mean_coef(gm, m, mu[c], inv_c, hw);
    double kb = bnstat_std_coef(gs, s, sigma[c], inv_c, hw);
    for (int k = 0; k < lim; ++k) {
      if (off == hw) {
        ++r; off = 0;
        m = m_in[r]; s = s_in[r]; c = (int)(r % C);
        ka = bnstat_mean_coef(gm, m, mu[c], inv_c, hw);
        kb = bnstat_std_coef(gs, s, sigma[c], inv_c, hw);
      }
      const float y = __fadd_rn(x[i + k], eps);
      const double g = ka + kb * ((double)y - ((double)m + (double)eps));
      out[k] = (float)g;
      ++off;
    }
    for (int k = 0; k < lim; ++k) gx[i + k] = accumulate ? gx[i + k] + out[k] : out[k];
  }
}

}  // namespace dfq

using namespace dfq;

extern "C" int dfq_bnstat_loss_fwd(const float* x, int64_t n, int64_t c, int64_t hw, const float* bn_mean, const float* bn_std,
                                   float eps, float* mean_out, float* std_out, double* loss2, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(x && bn_mean && bn_std && mean_out && std_out && loss2 && n > 0 && c > 0 && hw > 0, "bad argument");
  DFQ_REQUIRE(c <= 0x7fffffff, "too many channels");
  DFQ_CUDA(cudaMemsetAsync(loss2, 0, 2 * sizeof(double), st));
  const int64_t rows = n * c;
  const int sms = std::max(1, sm_count());
  if (hw >= kBnstatCtaRow) {
    const int grid = (int)std::min<int64_t>(rows, (int64_t)sms * 8);
    k_bnstat_fwd<true><<<grid, kDThreads, 0, st>>>(x, rows, hw, (int)c, bn_mean, bn_std, eps, mean_out, std_out, loss2);
  } else {
    const int grid = (int)std::min<int64_t>((rows + 7) / 8, (int64_t)sms * 8);
    k_bnstat_fwd<false><<<grid, kDThreads, 0, st>>>(x, rows, hw, (int)c, bn_mean, bn_std, eps, mean_out, std_out, loss2);
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_bnstat_loss_bwd(const float* x, float* grad_x, int64_t n, int64_t c, int64_t hw, const float* bn_mean,
                                   const float* bn_std, float eps, const float* mean_in, const float* std_in,
                                   const float* grad_loss2, int accumulate, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(x && grad_x && bn_mean && bn_std && mean_in && std_in && grad_loss2 && n > 0 && c > 0 && hw > 0, "bad argument");
  const int64_t total = n * c * hw;
  const int sms = std::max(1, sm_count());
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((total + kDThreads * 4 - 1) / (kDThreads * 4), (int64_t)sms * 16));
  k_bnstat_bwd<<<grid, kDThreads, 0, st>>>(x, grad_x, n * c, hw, (int)c, bn_mean, bn_std, eps, mean_in, std_in, grad_loss2, accumulate);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}
