// Int8 execution of calibrated Conv2d / Linear layers: ncnn's dequantizing int8 convolution (the scheme of the int8
// table convert_ncnn.py:178-201 writes) on the H100.  Symmetric codes q(v, s) = clamp(round_half_away(v * s), -127, 127)
// for activations (one scale per tensor) and weights (one scale per output channel), an exact int32 accumulation and the
// epilogue  y = fp32(fp32_rn(acc) * dq[o]) + bias[o]  with dq[o] = fp32(1 / fp32(a * w_s[o])) supplied by the caller.
//
//   k_i8_quantize_nhwc   fp32 NCHW -> int8 NHWC, channels padded to Cpad (multiple of 16) with zero bytes
//   k_i8_pack_dense      fp32 [O, C, kh, kw] -> int8 [O][kh][kw][Cpad]: GEMM K = (tap, channel) contiguous
//   k_i8_pack_dw         fp32 [C, 1, kh, kw] -> int8 [kh*kw][Cpad] (channels last)
//   k_i8_conv_mma        groups == 1: implicit GEMM on the tensor cores (mma.sync m16n8k32 s8), M = N*OH*OW pixels,
//                        N = O, K = kh*kw*Cpad; a cp.async ring gathers the im2col rows 16 channels (16 B) at a time
//   k_i8_conv_dw         groups == C == O: int32 MACs on the CUDA cores over the NHWC codes
// Both convolutions have three epilogues on one main loop (template parameter Out): fp32 NCHW (dfq_i8_conv); the next layer's
// int8 NHWC codes after the activation clamp (dfq_i8_conv_requant), which keeps activations in int8 between chained layers;
// and the residual epilogue (dfq_i8_conv_fused): clamp, fp32 residual add, clamp, then fp32 NCHW and / or the codes, so a
// residual block's add and an output with several consumers need no separate pass over an fp32 tensor.  The code stores of
// the last two can target a channel slice of a wider tensor (dfq_i8_conv_slice), so the producers of a channel
// concatenation write the consumer's input directly; k_i8_maxpool pools codes, or fp32 to fp32 and / or codes.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace dfq {
namespace {

__device__ __forceinline__ int8_t q8(float v, float s) {
  const float p = roundf(__fmul_rn(v, s));              // roundf: half away from zero
  return (int8_t)(int)fminf(fmaxf(p, -127.f), 127.f);
}

__device__ __forceinline__ float dequant(int32_t acc, float dq, float b) {
  return __fadd_rn(__fmul_rn(__int2float_rn(acc), dq), b);
}

// Where the epilogue puts its result.  F32: fp32 NCHW y (and optionally the int32 sums).  I8: the codes of the next layer,
// int8 NHWC yq[N, OH, OW, cpad] (cpad = O rounded up to 16, pad channels 0), requantized at the next layer's scale after
// the activation clamp [lo, hi].
// FUSED: Fused below.
// Both code-writing epilogues store pixel m's chunks [0, cpad) at yq + m * cstride: cstride = cpad for a tensor of its own,
// wider for a channel slice of a concatenation (yq then points at the slice's first channel, dfq_i8_conv_slice).
enum class Out { F32, I8, FUSED };
struct Requant {
  int8_t* yq;
  float scale, lo, hi;
  int cpad, cstride;
};

// What the per-layer path computes between two layers, in its order: dequant(), the activation (relu / relu6 / hardtanh,
// composed into one clamp that keeps NaN as torch does), q8() at the next layer's scale.
__device__ __forceinline__ int8_t requant(int32_t acc, float dq, float b, const Requant& rq) {
  float v = dequant(acc, dq, b);
  v = v < rq.lo ? rq.lo : (v > rq.hi ? rq.hi : v);
  return q8(v, rq.scale);
}

// requant()'s clamp (NaN stays NaN) as a function.  requant() keeps its own copy: written through this function, nvcc emits
// a different (smaller, two registers wider) schedule for the I8 kernels.
__device__ __forceinline__ float clamp_keep_nan(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

// The residual epilogue (DfqI8Epilogue): y = fp32 NCHW [N, O, OH, OW] and / or yq = int8 NHWC [N, OH, OW, cpad] codes at
// `scale`, either one NULL; r = fp32 NCHW residual of y's shape, or NULL.  yq and cpad come first, as in Requant, so the
// code store below serves both.
struct Fused {
  int8_t* yq;
  float scale, pre_lo, pre_hi;
  int cpad, cstride;
  const float* r;
  float* y;
  float post_lo, post_hi;
};
template <Out OUT> struct EpiOf { using type = Requant; };
template <> struct EpiOf<Out::FUSED> { using type = Fused; };

// What the per-layer path computes from the convolution to the tensor after a residual block's add, in its order: the
// pass-throughs before the add as one clamp, the fp32 add (rv = r[n, o, p], ignored without a residual), the ones after it.
__device__ __forceinline__ float fused_value(int32_t acc, float dq, float b, float rv, const Fused& e) {
  float v = clamp_keep_nan(dequant(acc, dq, b), e.pre_lo, e.pre_hi);
  if (e.r) v = __fadd_rn(v, rv);
  return clamp_keep_nan(v, e.post_lo, e.post_hi);
}

// ------------------------------------------------------------------------------------------------------------------
// quantizer and packers
// ------------------------------------------------------------------------------------------------------------------

// One thread per (n, 16-channel chunk, pixel); pixels fastest so the NCHW reads of each channel are coalesced.
__global__ void k_i8_quantize_nhwc(const float* __restrict__ x, int8_t* __restrict__ q, int C, int HW, int Cpad, int64_t total,
                                   float s) {
  const int chunks = Cpad / 16;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i % HW;
    const int64_t t = i / HW;
    const int ch = (int)(t % chunks);
    const int64_t n = t / chunks;
    alignas(16) int8_t v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = ch * 16 + j;
      v[j] = c < C ? q8(x[(n * C + c) * HW + p], s) : (int8_t)0;
    }
    *reinterpret_cast<int4*>(q + (n * HW + p) * Cpad + ch * 16) = *reinterpret_cast<const int4*>(v);
  }
}

__global__ void k_i8_pack_dense(const float* __restrict__ w, const float* __restrict__ ws, int8_t* __restrict__ out, int C,
                                int taps, int Cpad, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int64_t t = i / Cpad;
    const int tap = (int)(t % taps);
    const int64_t o = t / taps;
    out[i] = c < C ? q8(w[(o * C + c) * taps + tap], ws[o]) : (int8_t)0;
  }
}

__global__ void k_i8_pack_dw(const float* __restrict__ w, const float* __restrict__ ws, int8_t* __restrict__ out, int C,
                             int taps, int Cpad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= taps * Cpad) return;
  const int c = i % Cpad, tap = i / Cpad;
  out[i] = c < C ? q8(w[c * taps + tap], ws[c]) : (int8_t)0;
}

// ------------------------------------------------------------------------------------------------------------------
// dense implicit GEMM on the tensor cores
// ------------------------------------------------------------------------------------------------------------------
constexpr int BM = 128, BN = 64, BK = 64, STAGES = 3, THREADS = 128;
constexpr int A_BYTES = BM * BK, B_BYTES = BN * BK, STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int EPI_LD = BM + 4;                                  // int32 words per staged output-channel row
static_assert(BN * EPI_LD * 4 <= STAGES * STAGE_BYTES, "epilogue staging must fit in the pipeline's shared memory");

// Rows are 64 B = four 16-byte chunks; chunk c of row r lives at chunk c ^ ((r >> 1) & 3), which keeps the eight rows an
// ldmatrix phase reads (and the cp.async stores) on eight distinct 16-byte bank groups.
__device__ __forceinline__ int swz(int row, int chunk) { return row * BK + ((chunk ^ ((row >> 1) & 3)) << 4); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int n = valid ? 16 : 0;                                 // src-size 0: the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(n));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

__device__ __forceinline__ void mma_s8(int32_t* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 4 warps as 2 (M) x 2 (N); each warp owns a 64 x 32 tile = 4 x 4 mma tiles.
template <Out OUT>
__global__ void __launch_bounds__(THREADS) k_i8_conv_mma(const int8_t* __restrict__ xq, const int8_t* __restrict__ wq,
                                                         const float* __restrict__ dq, const float* __restrict__ bias,
                                                         float* __restrict__ y, int32_t* __restrict__ acc_out, DfqI8Conv g,
                                                         typename EpiOf<OUT>::type rq) {
  __shared__ __align__(128) unsigned char smem[STAGES * STAGE_BYTES];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1;
  const int64_t M = (int64_t)g.N * g.OH * g.OW;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int o0 = blockIdx.y * BN;
  const int K = g.kh * g.kw * g.Cpad;
  const int KT = (K + BK - 1) / BK;
  const int OHW = g.OH * g.OW;

  // this thread's gather slots: rows tid/4 + 32 i of the A tile and of the B tile, chunk tid % 4 of each
  const int chunk = tid & 3;
  const int8_t* a_img[4];
  int a_ih[4], a_iw[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + (tid >> 2) + 32 * i;
    if (m < M) {
      const int n = (int)(m / OHW), p = (int)(m % OHW);
      a_img[i] = xq + (int64_t)n * g.H * g.W * g.Cpad;
      a_ih[i] = (p / g.OW) * g.stride_h - g.pad_h;
      a_iw[i] = (p % g.OW) * g.stride_w - g.pad_w;
    } else {
      a_img[i] = xq;
      a_ih[i] = -(1 << 29);                                     // never inside the image
      a_iw[i] = 0;
    }
  }
  const uint32_t s_base = (uint32_t)__cvta_generic_to_shared(smem);

  auto load_tile = [&](int kt, int stage) {
    const uint32_t sa = s_base + stage * STAGE_BYTES, sb = sa + A_BYTES;
    const int k = (kt * 4 + chunk) * 16;                        // first of the 16 channels of this chunk
    const bool k_ok = k < K;
    const int tap = k / g.Cpad, c0 = k - tap * g.Cpad;
    const int dr = (tap / g.kw) * g.dil_h, ds = (tap % g.kw) * g.dil_w;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int ih = a_ih[i] + dr, iw = a_iw[i] + ds;
      const bool ok = k_ok && (unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W;
      const int8_t* src = ok ? a_img[i] + ((int64_t)ih * g.W + iw) * g.Cpad + c0 : xq;
      cp_async16(sa + swz((tid >> 2) + 32 * i, chunk), src, ok);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int o = o0 + (tid >> 2) + 32 * i;
      const bool ok = k_ok && o < g.O;
      const int8_t* src = ok ? wq + (int64_t)o * K + k : wq;
      cp_async16(sb + swz((tid >> 2) + 32 * i, chunk), src, ok);
    }
  };

  int32_t acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < KT) load_tile(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();                                            // tile kt landed; everyone is done with tile kt - 1
    if (kt + STAGES - 1 < KT) load_tile(kt + STAGES - 1, (kt + STAGES - 1) % STAGES);
    cp_async_commit();
    const uint32_t sa = s_base + (kt % STAGES) * STAGE_BYTES, sb = sa + A_BYTES;
#pragma unroll
    for (int ks = 0; ks < BK / 32; ++ks) {
      uint32_t a[4][4], b[4][2];
#pragma unroll
      for (int i = 0; i < 4; ++i) {                             // matrices: rows 0-7 / 8-15 x k bytes 0-15 / 16-31
        const int row = wm * 64 + i * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        ldmatrix_x4(sa + swz(row, ks * 2 + (lane >> 4)), a[i][0], a[i][1], a[i][2], a[i][3]);
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {                             // matrices: n 0-7 x k 0-15 / 16-31, then n 8-15
        const int row = wn * 32 + j * 16 + (lane & 7) + (lane >> 4) * 8;
        ldmatrix_x4(sb + swz(row, ks * 2 + ((lane >> 3) & 1)), b[2 * j][0], b[2 * j][1], b[2 * j + 1][0], b[2 * j + 1][1]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_s8(acc[i][j], a[i], b[j][0], b[j][1]);
    }
  }
  cp_async_wait<0>();
  __syncthreads();

  if constexpr (OUT == Out::FUSED) {
    // Straight from the accumulator layout: for one register, a warp holds 8 consecutive pixels (m) of 4 channels, so the
    // residual reads and the fp32 stores run in 32-byte pieces along the pixels of one channel.  A piece is one 32-byte
    // sector when OH * OW is a multiple of 8; otherwise (7x7, 14x14 maps) it can straddle two sectors or two images.
    // The codes are staged pixel-major as in the I8 epilogue and stored below.
    float d[4][2], b[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = o0 + wn * 32 + j * 8 + (lane & 3) * 2 + h;
        d[j][h] = o < g.O ? dq[o] : 0.f;
        b[j][h] = o < g.O && bias ? bias[o] : 0.f;
      }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int ml = wm * 64 + i * 16 + (lane >> 2) + rr * 8;
        const int64_t m = m0 + ml;
        const int64_t pix = m < M ? (m / OHW) * g.O * OHW + m % OHW : 0;   // NCHW offset of (n, channel 0, p)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int ol = wn * 32 + j * 8 + (lane & 3) * 2;
          uint8_t c[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int o = o0 + ol + h;
            c[h] = 0;
            if (m < M && o < g.O) {
              const int64_t idx = pix + (int64_t)o * OHW;
              const float v = fused_value(acc[i][j][2 * rr + h], d[j][h], b[j][h], rq.r ? rq.r[idx] : 0.f, rq);
              if (rq.y) rq.y[idx] = v;
              c[h] = (uint8_t)q8(v, rq.scale);
            }
          }
          if (rq.yq) *reinterpret_cast<uint16_t*>(smem + swz(ml, ol >> 4) + (ol & 15)) = (uint16_t)(c[0] | (c[1] << 8));
        }
      }
    if (!rq.yq) return;
  }
  if constexpr (OUT == Out::I8) {
    // requantize in registers and stage the codes pixel-major, [m][64 channels] with the A tile's swizzle: the 2-byte stores
    // of a warp (8 pixels x 4 channel pairs) and the 16-byte reads of a quarter warp (2 pixels x 4 chunks) are conflict-free.
    // Channels O .. o0 + 63 stage as 0, so the last tile writes the zero pad of yq.
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ol = wn * 32 + j * 8 + (lane & 3) * 2;          // this thread's channel pair ol, ol + 1
      float d[2], b[2];
      bool ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = o0 + ol + h;
        ok[h] = o < g.O;
        d[h] = ok[h] ? dq[o] : 0.f;
        b[h] = ok[h] && bias ? bias[o] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int m = wm * 64 + i * 16 + (lane >> 2) + rr * 8;
          const uint8_t c0 = ok[0] ? (uint8_t)requant(acc[i][j][2 * rr], d[0], b[0], rq) : 0;
          const uint8_t c1 = ok[1] ? (uint8_t)requant(acc[i][j][2 * rr + 1], d[1], b[1], rq) : 0;
          *reinterpret_cast<uint16_t*>(smem + swz(m, ol >> 4) + (ol & 15)) = (uint16_t)(c0 | (c1 << 8));
        }
    }
  }
  if constexpr (OUT != Out::F32) {
    __syncthreads();
    // one 16-byte chunk = 16 channels of one pixel; chunks at or past cpad (= O rounded up to 16) are not written
    for (int e = tid; e < BM * (BN / 16); e += THREADS) {
      const int ml = e >> 2, c = e & 3;
      const int64_t m = m0 + ml;
      const int o = o0 + c * 16;
      if (m >= M || o >= rq.cpad) continue;
      *reinterpret_cast<int4*>(rq.yq + m * rq.cstride + o) = *reinterpret_cast<const int4*>(smem + swz(ml, c));
    }
    return;
  }

  // stage the tile as [o][m] so the NCHW stores run along the pixels
  int32_t* st = reinterpret_cast<int32_t*>(smem);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int m = wm * 64 + i * 16 + (lane >> 2) + (r >> 1) * 8;
        const int o = wn * 32 + j * 8 + (lane & 3) * 2 + (r & 1);
        st[o * EPI_LD + m] = acc[i][j][r];
      }
  __syncthreads();
  for (int e = tid; e < BM * BN; e += THREADS) {
    const int ml = e % BM, ol = e / BM;
    const int64_t m = m0 + ml;
    const int o = o0 + ol;
    if (m >= M || o >= g.O) continue;
    const int32_t v = st[ol * EPI_LD + ml];
    const int64_t n = m / OHW, p = m % OHW;
    const int64_t idx = (n * g.O + o) * OHW + p;
    y[idx] = dequant(v, dq[o], bias ? bias[o] : 0.f);
    if (acc_out) acc_out[idx] = v;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// depthwise on the CUDA cores: one thread per (n, 16 channels, output pixel), pixels fastest
// ------------------------------------------------------------------------------------------------------------------
template <Out OUT>
__global__ void k_i8_conv_dw(const int8_t* __restrict__ xq, const int8_t* __restrict__ wq, const float* __restrict__ dq,
                             const float* __restrict__ bias, float* __restrict__ y, int32_t* __restrict__ acc_out, DfqI8Conv g,
                             int64_t total, typename EpiOf<OUT>::type rq) {
  const int chunks = g.Cpad / 16, OHW = g.OH * g.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int p = (int)(i % OHW);
    const int64_t t = i / OHW;
    const int ch = (int)(t % chunks);
    const int64_t n = t / chunks;
    if constexpr (OUT != Out::F32) {
      // the input's Cpad may be wider than yq's cpad = round_up(O, 16): chunks past it hold only pad channels, and yq has
      // no room for them
      if (ch * 16 >= rq.cpad) continue;
    }
    const int oh = p / g.OW, ow = p % g.OW;
    int32_t acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0;
    const int8_t* img = xq + n * g.H * g.W * g.Cpad + ch * 16;
    for (int r = 0; r < g.kh; ++r) {
      const int ih = oh * g.stride_h - g.pad_h + r * g.dil_h;
      if ((unsigned)ih >= (unsigned)g.H) continue;
      for (int s = 0; s < g.kw; ++s) {
        const int iw = ow * g.stride_w - g.pad_w + s * g.dil_w;
        if ((unsigned)iw >= (unsigned)g.W) continue;
        const int4 xv = __ldg(reinterpret_cast<const int4*>(img + ((int64_t)ih * g.W + iw) * g.Cpad));
        const int4 wv = __ldg(reinterpret_cast<const int4*>(wq + (r * g.kw + s) * g.Cpad + ch * 16));
        const int8_t* xb = reinterpret_cast<const int8_t*>(&xv);
        const int8_t* wb = reinterpret_cast<const int8_t*>(&wv);
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[j] += (int32_t)xb[j] * (int32_t)wb[j];
      }
    }
    if constexpr (OUT == Out::FUSED) {                          // r and y along the pixels, as the F32 stores
      alignas(16) int8_t v[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = ch * 16 + j;
        v[j] = 0;
        if (c < g.C) {
          const int64_t idx = (n * g.C + c) * OHW + p;
          const float f = fused_value(acc[j], dq[c], bias ? bias[c] : 0.f, rq.r ? rq.r[idx] : 0.f, rq);
          if (rq.y) rq.y[idx] = f;
          v[j] = q8(f, rq.scale);
        }
      }
      if (rq.yq) *reinterpret_cast<int4*>(rq.yq + (n * OHW + p) * rq.cstride + ch * 16) = *reinterpret_cast<const int4*>(v);
      continue;
    }
    if constexpr (OUT == Out::I8) {                             // the 16 channels of this pixel in one store
      alignas(16) int8_t v[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = ch * 16 + j;
        v[j] = c < g.C ? requant(acc[j], dq[c], bias ? bias[c] : 0.f, rq) : (int8_t)0;
      }
      *reinterpret_cast<int4*>(rq.yq + (n * OHW + p) * rq.cstride + ch * 16) = *reinterpret_cast<const int4*>(v);
      continue;
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = ch * 16 + j;
      if (c >= g.C) break;
      const int64_t idx = (n * g.C + c) * OHW + p;
      y[idx] = dequant(acc[j], dq[c], bias ? bias[c] : 0.f);
      if (acc_out) acc_out[idx] = acc[j];
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// max pooling: one thread per (n, 16 channels, output pixel), pixels fastest, as k_i8_conv_dw
// ------------------------------------------------------------------------------------------------------------------
// CODES: xq int8 NHWC [N, H, W, Cpad] -> yq int8 NHWC [N, OH, OW, Cpad], a byte-wise signed max of 16-byte taps.  q8() is
// monotone non-decreasing for a scale >= 0, so the max of the codes is the code of the max for any window without NaN.
// A window with no tap inside the input (possible with dilation) is -inf in torch, whose code is -127; pad channels 0.
// !CODES: x fp32 NCHW [N, C, H, W] -> y fp32 NCHW [N, C, OH, OW] and / or yq int8 NHWC at `scale`, with torch's CUDA rule:
// from -inf, taps row-major, the running max replaced when v > m or v is NaN (so the first of tied values is kept).
template <bool CODES>
__global__ void k_i8_maxpool(const int8_t* __restrict__ xq, const float* __restrict__ x, float* __restrict__ y,
                             int8_t* __restrict__ yq, float scale, DfqI8Pool g, int64_t total) {
  const int chunks = g.Cpad / 16, OHW = g.OH * g.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int p = (int)(i % OHW);
    const int64_t t = i / OHW;
    const int ch = (int)(t % chunks);
    const int64_t n = t / chunks;
    const int h0 = (p / g.OW) * g.stride_h - g.pad_h, w0 = (p % g.OW) * g.stride_w - g.pad_w;
    alignas(16) int8_t v[16];
    if constexpr (CODES) {
      const int8_t* img = xq + n * g.H * g.W * g.Cpad + ch * 16;
      int m[4] = {(int)0x81818181, (int)0x81818181, (int)0x81818181, (int)0x81818181};
      bool any = false;
      for (int r = 0; r < g.kh; ++r) {
        const int ih = h0 + r * g.dil_h;
        if ((unsigned)ih >= (unsigned)g.H) continue;
        for (int s = 0; s < g.kw; ++s) {
          const int iw = w0 + s * g.dil_w;
          if ((unsigned)iw >= (unsigned)g.W) continue;
          const int4 q = __ldg(reinterpret_cast<const int4*>(img + ((int64_t)ih * g.W + iw) * g.Cpad));
          m[0] = __vmaxs4(m[0], q.x), m[1] = __vmaxs4(m[1], q.y), m[2] = __vmaxs4(m[2], q.z), m[3] = __vmaxs4(m[3], q.w);
          any = true;
        }
      }
      *reinterpret_cast<int4*>(v) = make_int4(m[0], m[1], m[2], m[3]);
      if (!any) {
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = ch * 16 + j < g.C ? (int8_t)-127 : (int8_t)0;
      }
    } else {
#pragma unroll 1
      for (int j = 0; j < 16; ++j) {
        const int c = ch * 16 + j;
        v[j] = 0;
        if (c >= g.C) continue;
        const float* img = x + (n * g.C + c) * g.H * g.W;
        float mx = -INFINITY;
        for (int r = 0; r < g.kh; ++r) {
          const int ih = h0 + r * g.dil_h;
          if ((unsigned)ih >= (unsigned)g.H) continue;
          for (int s = 0; s < g.kw; ++s) {
            const int iw = w0 + s * g.dil_w;
            if ((unsigned)iw >= (unsigned)g.W) continue;
            const float f = __ldg(img + (int64_t)ih * g.W + iw);
            if (f > mx || isnan(f)) mx = f;
          }
        }
        if (y) y[(n * g.C + c) * OHW + p] = mx;
        v[j] = q8(mx, scale);
      }
      if (!yq) continue;
    }
    *reinterpret_cast<int4*>(yq + (n * OHW + p) * g.Cpad + ch * 16) = *reinterpret_cast<const int4*>(v);
  }
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// [a, a + na) and [b, b + nb) share a byte; a NULL range shares none
inline bool overlap(const void* a, int64_t na, const void* b, int64_t nb) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return a && b && x < y + (uintptr_t)nb && y < x + (uintptr_t)na;
}

inline bool ordered(float lo, float hi) { return !std::isnan(lo) && !std::isnan(hi) && lo <= hi; }

int check_geometry(const DfqI8Conv* g) {
  DFQ_REQUIRE(g != nullptr, "dfq_i8: null geometry");
  DFQ_REQUIRE(g->N > 0 && g->C > 0 && g->H > 0 && g->W > 0 && g->O > 0 && g->kh > 0 && g->kw > 0, "dfq_i8: empty dimension");
  DFQ_REQUIRE(g->stride_h > 0 && g->stride_w > 0 && g->dil_h > 0 && g->dil_w > 0 && g->pad_h >= 0 && g->pad_w >= 0,
              "dfq_i8: bad stride / padding / dilation");
  DFQ_REQUIRE(g->Cpad >= g->C && g->Cpad % 16 == 0, "dfq_i8: Cpad must be a multiple of 16 that holds C");
  DFQ_REQUIRE(g->OH == (g->H + 2 * g->pad_h - g->dil_h * (g->kh - 1) - 1) / g->stride_h + 1 &&
                  g->OW == (g->W + 2 * g->pad_w - g->dil_w * (g->kw - 1) - 1) / g->stride_w + 1 && g->OH > 0 && g->OW > 0,
              "dfq_i8: OH / OW do not follow from the geometry");
  if (g->groups != 1 && !(g->groups == g->C && g->O == g->C)) {
    set_error("dfq_i8: unsupported grouping: groups=%d C=%d O=%d (needs groups == 1, or groups == C == O)", g->groups, g->C,
              g->O);
    return DFQ_E_UNSUPPORTED;
  }
  return 0;
}

// torch's pooling_output_shape: floor division, and in ceil mode the last window starts inside the input or its left pad
int pool_extent(int in, int k, int pad, int stride, int dil, bool ceil_mode) {
  const int64_t num = (int64_t)in + 2 * pad - (int64_t)dil * (k - 1) - 1 + (ceil_mode ? stride - 1 : 0);
  int64_t out = (num >= 0 ? num / stride : -((-num + stride - 1) / stride)) + 1;
  if (ceil_mode && (out - 1) * stride >= (int64_t)in + pad) --out;
  return (int)out;
}

int grid_for(int64_t total, int threads) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((total + threads - 1) / threads, (int64_t)sm_count() * 32));
}

}  // namespace
}  // namespace dfq

using namespace dfq;

extern "C" int dfq_i8_quantize_nhwc(const float* x, int8_t* q, int32_t N, int32_t C, int32_t H, int32_t W, int32_t Cpad,
                                    float scale, void* stream) {
  DFQ_REQUIRE(x && q && N > 0 && C > 0 && H > 0 && W > 0, "dfq_i8_quantize_nhwc: bad arguments");
  DFQ_REQUIRE(Cpad >= C && Cpad % 16 == 0, "dfq_i8_quantize_nhwc: Cpad must be a multiple of 16 that holds C");
  DFQ_REQUIRE(aligned16(q), "dfq_i8_quantize_nhwc: q must be 16-byte aligned");
  const int64_t total = (int64_t)N * (Cpad / 16) * H * W;
  k_i8_quantize_nhwc<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(x, q, C, H * W, Cpad, total, scale);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_pack_weights(const float* w, const float* w_scale, int8_t* packed, const DfqI8Conv* g, void* stream) {
  if (int rc = check_geometry(g)) return rc;
  DFQ_REQUIRE(w && w_scale && packed, "dfq_i8_pack_weights: null pointer");
  const int taps = g->kh * g->kw;
  cudaStream_t st = (cudaStream_t)stream;
  if (g->groups == 1) {
    const int64_t total = (int64_t)g->O * taps * g->Cpad;
    k_i8_pack_dense<<<grid_for(total, 256), 256, 0, st>>>(w, w_scale, packed, g->C, taps, g->Cpad, total);
  } else {
    k_i8_pack_dw<<<(taps * g->Cpad + 255) / 256, 256, 0, st>>>(w, w_scale, packed, g->C, taps, g->Cpad);
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_conv(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, float* y, int32_t* acc_out,
                           const DfqI8Conv* g, void* stream) {
  if (int rc = check_geometry(g)) return rc;
  DFQ_REQUIRE(xq && wq && dq && y, "dfq_i8_conv: null pointer");
  DFQ_REQUIRE(aligned16(xq) && aligned16(wq), "dfq_i8_conv: codes must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (g->groups == 1) {
    const int64_t M = (int64_t)g->N * g->OH * g->OW;
    DFQ_REQUIRE((M + BM - 1) / BM < (1LL << 31), "dfq_i8_conv: too many output pixels");
    const dim3 grid((unsigned)((M + BM - 1) / BM), (unsigned)((g->O + BN - 1) / BN));
    k_i8_conv_mma<Out::F32><<<grid, THREADS, 0, st>>>(xq, wq, dq, bias, y, acc_out, *g, Requant{});
  } else {
    const int64_t total = (int64_t)g->N * (g->Cpad / 16) * g->OH * g->OW;
    k_i8_conv_dw<Out::F32><<<grid_for(total, 256), 256, 0, st>>>(xq, wq, dq, bias, y, acc_out, *g, total, Requant{});
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_conv_requant(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, int8_t* yq,
                                   float out_scale, float act_lo, float act_hi, const DfqI8Conv* g, void* stream) {
  if (int rc = check_geometry(g)) return rc;
  DFQ_REQUIRE(xq && wq && dq && yq, "dfq_i8_conv_requant: null pointer");
  DFQ_REQUIRE(aligned16(xq) && aligned16(wq), "dfq_i8_conv_requant: codes must be 16-byte aligned");
  DFQ_REQUIRE(aligned16(yq), "dfq_i8_conv_requant: yq must be 16-byte aligned");
  DFQ_REQUIRE(!std::isnan(act_lo) && !std::isnan(act_hi) && act_lo <= act_hi,
              "dfq_i8_conv_requant: activation bounds must be ordered and not NaN");
  DFQ_REQUIRE(std::isfinite(out_scale) && out_scale >= 0.f, "dfq_i8_conv_requant: out_scale must be finite and non-negative");
  const int cpad = (g->O + 15) / 16 * 16;
  const Requant rq{yq, out_scale, act_lo, act_hi, cpad, cpad};
  cudaStream_t st = (cudaStream_t)stream;
  if (g->groups == 1) {
    const int64_t M = (int64_t)g->N * g->OH * g->OW;
    DFQ_REQUIRE((M + BM - 1) / BM < (1LL << 31), "dfq_i8_conv_requant: too many output pixels");
    const dim3 grid((unsigned)((M + BM - 1) / BM), (unsigned)((g->O + BN - 1) / BN));
    k_i8_conv_mma<Out::I8><<<grid, THREADS, 0, st>>>(xq, wq, dq, bias, nullptr, nullptr, *g, rq);
  } else {
    const int64_t total = (int64_t)g->N * (g->Cpad / 16) * g->OH * g->OW;
    k_i8_conv_dw<Out::I8><<<grid_for(total, 256), 256, 0, st>>>(xq, wq, dq, bias, nullptr, nullptr, *g, total, rq);
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_conv_fused(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, const DfqI8Epilogue* e,
                                 const DfqI8Conv* g, void* stream) {
  if (int rc = check_geometry(g)) return rc;
  DFQ_REQUIRE(xq && wq && dq && e, "dfq_i8_conv_fused: null pointer");
  DFQ_REQUIRE(aligned16(xq) && aligned16(wq), "dfq_i8_conv_fused: codes must be 16-byte aligned");
  DFQ_REQUIRE(e->y || e->yq, "dfq_i8_conv_fused: no output requested (y and yq are both NULL)");
  DFQ_REQUIRE(aligned16(e->yq), "dfq_i8_conv_fused: yq must be 16-byte aligned");
  DFQ_REQUIRE(((uintptr_t)e->residual & 3) == 0 && ((uintptr_t)e->y & 3) == 0,
              "dfq_i8_conv_fused: residual and y must be 4-byte aligned");
  DFQ_REQUIRE(ordered(e->pre_lo, e->pre_hi) && ordered(e->post_lo, e->post_hi),
              "dfq_i8_conv_fused: pre / post clamp bounds must be ordered and not NaN");
  DFQ_REQUIRE(!e->yq || (std::isfinite(e->out_scale) && e->out_scale >= 0.f),
              "dfq_i8_conv_fused: out_scale must be finite and non-negative when yq is written");
  const int cpad = (g->O + 15) / 16 * 16;
  const int64_t pixels = (int64_t)g->N * g->OH * g->OW;
  const int64_t y_bytes = pixels * g->O * (int64_t)sizeof(float), yq_bytes = pixels * cpad;
  DFQ_REQUIRE(!overlap(e->residual, y_bytes, e->y, y_bytes) && !overlap(e->residual, y_bytes, e->yq, yq_bytes),
              "dfq_i8_conv_fused: residual overlaps y or yq");
  DFQ_REQUIRE(!overlap(e->y, y_bytes, e->yq, yq_bytes), "dfq_i8_conv_fused: y overlaps yq");
  const Fused ep{e->yq, e->out_scale, e->pre_lo, e->pre_hi, cpad, cpad, e->residual, e->y, e->post_lo, e->post_hi};
  cudaStream_t st = (cudaStream_t)stream;
  if (g->groups == 1) {
    DFQ_REQUIRE((pixels + BM - 1) / BM < (1LL << 31), "dfq_i8_conv_fused: too many output pixels");
    const dim3 grid((unsigned)((pixels + BM - 1) / BM), (unsigned)((g->O + BN - 1) / BN));
    k_i8_conv_mma<Out::FUSED><<<grid, THREADS, 0, st>>>(xq, wq, dq, bias, nullptr, nullptr, *g, ep);
  } else {
    const int64_t total = (int64_t)g->N * (g->Cpad / 16) * g->OH * g->OW;
    k_i8_conv_dw<Out::FUSED><<<grid_for(total, 256), 256, 0, st>>>(xq, wq, dq, bias, nullptr, nullptr, *g, total, ep);
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_conv_slice(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, const DfqI8Epilogue* e,
                                 int32_t coff, int32_t cstride, const DfqI8Conv* g, void* stream) {
  if (int rc = check_geometry(g)) return rc;
  DFQ_REQUIRE(xq && wq && dq && e, "dfq_i8_conv_slice: null pointer");
  DFQ_REQUIRE(aligned16(xq) && aligned16(wq), "dfq_i8_conv_slice: codes must be 16-byte aligned");
  DFQ_REQUIRE(e->yq, "dfq_i8_conv_slice: no codes requested (yq is NULL)");
  DFQ_REQUIRE(aligned16(e->yq), "dfq_i8_conv_slice: yq must be 16-byte aligned");
  DFQ_REQUIRE(((uintptr_t)e->residual & 3) == 0 && ((uintptr_t)e->y & 3) == 0,
              "dfq_i8_conv_slice: residual and y must be 4-byte aligned");
  DFQ_REQUIRE(ordered(e->pre_lo, e->pre_hi) && ordered(e->post_lo, e->post_hi),
              "dfq_i8_conv_slice: pre / post clamp bounds must be ordered and not NaN");
  DFQ_REQUIRE(std::isfinite(e->out_scale) && e->out_scale >= 0.f, "dfq_i8_conv_slice: out_scale must be finite and non-negative");
  const int cpad = (g->O + 15) / 16 * 16;
  DFQ_REQUIRE(coff >= 0 && cstride > 0 && coff % 16 == 0 && cstride % 16 == 0,
              "dfq_i8_conv_slice: coff and cstride must be non-negative multiples of 16");
  DFQ_REQUIRE((int64_t)coff + cpad <= cstride, "dfq_i8_conv_slice: the slice coff + round_up(O, 16) exceeds cstride");
  const int64_t pixels = (int64_t)g->N * g->OH * g->OW;
  const int64_t y_bytes = pixels * g->O * (int64_t)sizeof(float);
  int8_t* yq = e->yq + coff;
  const int64_t slice_bytes = (pixels - 1) * cstride + cpad;          // first to last byte the slice's chunks cover
  DFQ_REQUIRE(!overlap(e->residual, y_bytes, yq, slice_bytes), "dfq_i8_conv_slice: residual overlaps the slice");
  DFQ_REQUIRE(!overlap(e->y, y_bytes, yq, slice_bytes), "dfq_i8_conv_slice: y overlaps the slice");
  DFQ_REQUIRE(!overlap(e->residual, y_bytes, e->y, y_bytes), "dfq_i8_conv_slice: residual overlaps y");
  cudaStream_t st = (cudaStream_t)stream;
  const bool dense = g->groups == 1;
  DFQ_REQUIRE(!dense || (pixels + BM - 1) / BM < (1LL << 31), "dfq_i8_conv_slice: too many output pixels");
  const dim3 grid((unsigned)((pixels + BM - 1) / BM), (unsigned)((g->O + BN - 1) / BN));
  const int64_t total = (int64_t)g->N * (g->Cpad / 16) * g->OH * g->OW;
  if (!e->residual && !e->y && e->post_lo == -INFINITY && e->post_hi == INFINITY) {
    // codes only after one clamp: the requantizing epilogue
    const Requant rq{yq, e->out_scale, e->pre_lo, e->pre_hi, cpad, cstride};
    if (dense) k_i8_conv_mma<Out::I8><<<grid, THREADS, 0, st>>>(xq, wq, dq, bias, nullptr, nullptr, *g, rq);
    else k_i8_conv_dw<Out::I8><<<grid_for(total, 256), 256, 0, st>>>(xq, wq, dq, bias, nullptr, nullptr, *g, total, rq);
  } else {
    const Fused ep{yq, e->out_scale, e->pre_lo, e->pre_hi, cpad, cstride, e->residual, e->y, e->post_lo, e->post_hi};
    if (dense) k_i8_conv_mma<Out::FUSED><<<grid, THREADS, 0, st>>>(xq, wq, dq, bias, nullptr, nullptr, *g, ep);
    else k_i8_conv_dw<Out::FUSED><<<grid_for(total, 256), 256, 0, st>>>(xq, wq, dq, bias, nullptr, nullptr, *g, total, ep);
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_maxpool(const int8_t* xq, const float* x, float* y, int8_t* yq, float out_scale, const DfqI8Pool* g,
                              void* stream) {
  DFQ_REQUIRE(g != nullptr, "dfq_i8_maxpool: null geometry");
  DFQ_REQUIRE(g->N > 0 && g->C > 0 && g->H > 0 && g->W > 0 && g->kh > 0 && g->kw > 0, "dfq_i8_maxpool: empty dimension");
  DFQ_REQUIRE(g->stride_h > 0 && g->stride_w > 0 && g->dil_h > 0 && g->dil_w > 0 && g->pad_h >= 0 && g->pad_w >= 0 &&
                  (g->ceil_mode == 0 || g->ceil_mode == 1),
              "dfq_i8_maxpool: bad stride / padding / dilation / ceil_mode");
  DFQ_REQUIRE(g->pad_h <= g->kh / 2 && g->pad_w <= g->kw / 2 && g->pad_h <= (g->dil_h * (g->kh - 1) + 1) / 2 &&
                  g->pad_w <= (g->dil_w * (g->kw - 1) + 1) / 2,
              "dfq_i8_maxpool: padding must be at most half of the kernel and of the effective kernel");
  DFQ_REQUIRE(g->Cpad >= g->C && g->Cpad % 16 == 0, "dfq_i8_maxpool: Cpad must be a multiple of 16 that holds C");
  DFQ_REQUIRE(g->OH == pool_extent(g->H, g->kh, g->pad_h, g->stride_h, g->dil_h, g->ceil_mode) &&
                  g->OW == pool_extent(g->W, g->kw, g->pad_w, g->stride_w, g->dil_w, g->ceil_mode) && g->OH > 0 && g->OW > 0,
              "dfq_i8_maxpool: OH / OW do not follow from the geometry");
  DFQ_REQUIRE((xq != nullptr) != (x != nullptr), "dfq_i8_maxpool: give exactly one input, codes xq or fp32 x");
  const int64_t in_px = (int64_t)g->N * g->H * g->W, out_px = (int64_t)g->N * g->OH * g->OW;
  const int64_t total = out_px * (g->Cpad / 16);
  cudaStream_t st = (cudaStream_t)stream;
  if (xq) {
    DFQ_REQUIRE(yq && !y, "dfq_i8_maxpool: codes in give codes out only (yq, no y)");
    DFQ_REQUIRE(aligned16(xq) && aligned16(yq), "dfq_i8_maxpool: xq and yq must be 16-byte aligned");
    DFQ_REQUIRE(!overlap(xq, in_px * g->Cpad, yq, out_px * g->Cpad), "dfq_i8_maxpool: yq overlaps xq");
    k_i8_maxpool<true><<<grid_for(total, 256), 256, 0, st>>>(xq, nullptr, nullptr, yq, 0.f, *g, total);
  } else {
    DFQ_REQUIRE(y || yq, "dfq_i8_maxpool: no output requested (y and yq are both NULL)");
    DFQ_REQUIRE(aligned16(yq), "dfq_i8_maxpool: yq must be 16-byte aligned");
    DFQ_REQUIRE(((uintptr_t)x & 3) == 0 && ((uintptr_t)y & 3) == 0, "dfq_i8_maxpool: x and y must be 4-byte aligned");
    DFQ_REQUIRE(!yq || (std::isfinite(out_scale) && out_scale >= 0.f),
                "dfq_i8_maxpool: out_scale must be finite and non-negative when yq is written");
    const int64_t x_bytes = in_px * g->C * 4, y_bytes = out_px * g->C * 4, yq_bytes = out_px * g->Cpad;
    DFQ_REQUIRE(!overlap(x, x_bytes, y, y_bytes) && !overlap(x, x_bytes, yq, yq_bytes) && !overlap(y, y_bytes, yq, yq_bytes),
                "dfq_i8_maxpool: x, y and yq overlap");
    k_i8_maxpool<false><<<grid_for(total, 256), 256, 0, st>>>(nullptr, x, y, yq, out_scale, *g, total);
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}
