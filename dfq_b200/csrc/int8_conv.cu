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
// concatenation write the consumer's input directly; k_i8_maxpool pools codes, or fp32 to fp32 and / or codes;
// k_i8_upsample_bilinear resizes fp32 as torch does, to fp32 and / or codes in such a channel slice.
// A fourth epilogue writes the fp32 output pixel-major into a slice of a detection head's [N, R, k] concatenation
// (dfq_i8_conv_nhwc), so the permute / contiguous / cat of SSD's heads need no copies.
//
// A second integer scheme runs on the same main loops: the reference's asymmetric per-tensor min / max quantization
// (QuantMeasure for activations, quantize_targ_layer for weights).  Codes q in [0, 2^b - 1] are stored shifted,
// q' = q - 128, so the s8 x s8 tensor-core path and every layout stay as they are; the shift moves into the offsets.
//   k_i8_quantize_affine   fp32 NCHW -> int8 NHWC q' (pad channels 0) and S[n, h, w] = sum of q' over the real channels
//   k_i8_pack_affine       already fake-quantized fp32 weights -> their codes q' in the dense or depthwise layout, counting
//                          the weights the round trip fp32(fp32(q fw) + mw) does not reproduce bit for bit
//   k_i8_affine_table      dense: per output channel, the (kh+1) x (kw+1) prefix table of the tap sums of q'
//   Out::AFFINE            y = fp32(kP P + kA A + kW Wv + kN Nv) + bias[o] in double (dfq_i8_affine_conv): P the int32
//                          sum, A the sum of q' over the in-image taps (dense: of S; depthwise: per channel in the main
//                          loop), Wv the sum of q' of the weights over the same taps, Nv their count times C / groups
//   Out::AFFINE_FUSED      the same value through the clamps and residual add of Out::FUSED, then fp32 NCHW and / or the
//                          NEXT layer's shifted codes and their per-pixel sums S (dfq_i8_affine_conv_fused), which keeps
//                          affine activations in int8 between chained layers
//   Out::AFFINE_OBSERVED   Out::AFFINE_FUSED with QuantMeasure's fake quantization (fake_quant<true>) on the value after the
//                          first clamp and / or on the residual, each when its observer is on (dfq_i8_affine_conv_observed):
//                          the observers the reference's replace_op() puts on a residual add's operands run in the epilogue
//   Out::AFFINE_LAYOUT     Out::AFFINE_OBSERVED (either observer optional) whose codes go to a channel slice of a wider
//                          tensor and whose S adds into a sum the concatenation's writers share, and whose out-of-image taps
//                          may read a pad code z' instead of being left out (dfq_i8_affine_conv_layout): a zero F.pad folded
//                          into the convolution.  Dense layers correct P, A, Wv and Nv in the epilogue; the depthwise main
//                          loop reads z' (k_i8_conv_dw<..., true>).
//   k_i8_affine_upsample   torch's bilinear upsample (k_i8_upsample_bilinear's value) through clamp, observer, clamp to the
//                          consumer's codes in a channel slice, S added (dfq_i8_affine_upsample_bilinear)
//   Out::AFFINE_ROWS       Out::AFFINE's value through clamp, QuantMeasure's fake quantization (either optional), clamp and a
//                          second fake quantization, written pixel-major into a slice of a detection head's [N, R, k]
//                          concatenation (dfq_i8_affine_conv_rows), as Out::ROWS
//   k_i8_maxpool<., true>  k_i8_maxpool on shifted codes, or fp32 to fp32 and / or the consumer's shifted codes, with their
//                          per-pixel sums S (dfq_i8_affine_maxpool)
#include <algorithm>
#include <cmath>

#include "bilinear.cuh"
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
// FUSED: Fused below.  ROWS: Rows below.
// Both code-writing epilogues store pixel m's chunks [0, cpad) at yq + m * cstride: cstride = cpad for a tensor of its own,
// wider for a channel slice of a concatenation (yq then points at the slice's first channel, dfq_i8_conv_slice).
enum class Out { F32, I8, FUSED, ROWS, AFFINE, AFFINE_FUSED, AFFINE_OBSERVED, AFFINE_LAYOUT, AFFINE_ROWS };
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
// The pixel-major fp32 epilogue (dfq_i8_conv_nhwc): v = clamp(clamp(dequant, pre), post) goes to
// y[n * img_stride + off + p * O + o], the permute(0, 2, 3, 1) of the NCHW output placed at `off` inside each image's
// img_stride floats (a slice along dim 1 of a detection head's [N, R, k] concatenation).
struct Rows {
  float* y;
  int64_t off, img_stride;
  float pre_lo, pre_hi, post_lo, post_hi;
};
// The affine epilogue (dfq_i8_affine_conv): S and table are the dense layer's per-pixel code sums and per-output-channel
// prefix tables (unused by the depthwise kernel), k the constants of DfqI8Affine.
struct Affine {
  const int32_t* S;
  const int32_t* table;
  double kP, kA, kW, kN;
};
// The affine residual epilogue (DfqI8AffineEpilogue): Affine's value, clamp(pre), + r (NULL: none), clamp(post), then y
// (kernel argument, NULL: none) and / or yq = int8 NHWC [N, OH, OW, cpad] codes at the consumer's scalars (neg_min,
// inv_scale, qmax) and S_out[n, p] = their sum over the real channels (NULL: none; atomicAdd into a zeroed S_out when
// several launches' tiles or threads share a pixel, S_atomic).
struct AffineFused : Affine {
  const float* r;
  int8_t* yq;
  int32_t* S_out;
  float neg_min, inv_scale, qmax;
  float pre_lo, pre_hi, post_lo, post_hi;
  int cpad;
  bool S_atomic;
};
// The observed affine epilogue (DfqI8AffineObserve): AffineFused's, with the fake quantization of `obs` on the value after
// the pre clamp (obs_on) and of `res` on the residual (res_on).
struct AffineObserved : AffineFused {
  QuantScalars obs, res;
  bool obs_on, res_on;
};
// The layout epilogue (DfqI8AffineLayout): AffineObserved's, the codes of pixel m at yq + m * cstride (yq at the slice's
// first channel), and with pad_on every out-of-image tap reading the shifted code pad_code over the C real channels.
struct AffineLayout : AffineObserved {
  int cstride, pad_code;
  bool pad_on;
};
// The affine rows epilogue (DfqI8AffineRows): Affine's value, clamp(pre), fq(obs) (obs_on), clamp(post), fq(tail)
// (tail_on), stored as Rows stores it.
struct AffineRows : Affine {
  float* y;
  int64_t off, img_stride;
  float pre_lo, pre_hi, post_lo, post_hi;
  QuantScalars obs, tail;
  bool obs_on, tail_on;
};
template <Out OUT> struct EpiOf { using type = Requant; };
template <> struct EpiOf<Out::FUSED> { using type = Fused; };
template <> struct EpiOf<Out::ROWS> { using type = Rows; };
template <> struct EpiOf<Out::AFFINE> { using type = Affine; };
template <> struct EpiOf<Out::AFFINE_FUSED> { using type = AffineFused; };
template <> struct EpiOf<Out::AFFINE_OBSERVED> { using type = AffineObserved; };
template <> struct EpiOf<Out::AFFINE_LAYOUT> { using type = AffineLayout; };
template <> struct EpiOf<Out::AFFINE_ROWS> { using type = AffineRows; };
__host__ __device__ constexpr bool affine_out(Out o) {
  return o == Out::AFFINE || o == Out::AFFINE_FUSED || o == Out::AFFINE_OBSERVED || o == Out::AFFINE_LAYOUT ||
         o == Out::AFFINE_ROWS;
}
__host__ __device__ constexpr bool affine_epilogue(Out o) {
  return o == Out::AFFINE_FUSED || o == Out::AFFINE_OBSERVED || o == Out::AFFINE_LAYOUT;
}
__host__ __device__ constexpr bool observed(Out o) { return o == Out::AFFINE_OBSERVED || o == Out::AFFINE_LAYOUT; }

// the int8 elements between two pixels' codes in yq: a tensor of its own (cpad), or a concatenation's (cstride)
template <Out OUT>
__device__ __forceinline__ int64_t code_stride(const typename EpiOf<OUT>::type& e) {
  if constexpr (OUT == Out::AFFINE_LAYOUT) return e.cstride;
  else return e.cpad;
}

// fp32(kP P + kA A + kW Wv + kN Nv) + b: each product and sum a separately rounded double op, in this order
__device__ __forceinline__ float affine_value(int32_t P, int32_t A, int32_t Wv, int32_t Nv, float b, const Affine& e) {
  double t = __dmul_rn(e.kP, (double)P);
  t = __dadd_rn(t, __dmul_rn(e.kA, (double)A));
  t = __dadd_rn(t, __dmul_rn(e.kW, (double)Wv));
  t = __dadd_rn(t, __dmul_rn(e.kN, (double)Nv));
  return __fadd_rn(__double2float_rn(t), b);
}

// The taps r in [lo, hi) of one axis whose input coordinate o * stride - pad + r * dil lies in [0, in): a range, since the
// coordinate grows with r.  lo == hi when none does.
__device__ __forceinline__ int2 tap_range(int o, int stride, int pad, int dil, int k, int in) {
  const int base = o * stride - pad;
  const int lo = base >= 0 ? 0 : min(k, (-base + dil - 1) / dil);
  const int hi = base > in - 1 ? 0 : min(k, (in - 1 - base) / dil + 1);
  return make_int2(lo, max(lo, hi));
}

// The activation code of the affine scheme, shifted: q = rint(clamp(fp32(fp32(v + neg_min) * inv_scale), 0, qmax)) - 128,
// the ops of the fake quantization (common.cuh fake_quant<true>), so fp32(fp32((q' + 128) * scale) + min) is its output.
// NaN has no code there; fmaxf turns it into 0 here (code -128).
__device__ __forceinline__ int8_t affine_code(float v, float neg_min, float inv_scale, float qmax) {
  const float t = fminf(fmaxf(__fmul_rn(__fadd_rn(v, neg_min), inv_scale), 0.f), qmax);
  return (int8_t)((int)rintf(t) - 128);
}

// What the per-layer path computes from the convolution to the tensor after a residual block's add, in its order: the
// pass-throughs before the add as one clamp, the fp32 add (rv = r[n, o, p], ignored without a residual), the ones after it.
__device__ __forceinline__ float fused_value(int32_t acc, float dq, float b, float rv, const Fused& e) {
  float v = clamp_keep_nan(dequant(acc, dq, b), e.pre_lo, e.pre_hi);
  if (e.r) v = __fadd_rn(v, rv);
  return clamp_keep_nan(v, e.post_lo, e.post_hi);
}

// The observed add of Out::AFFINE_OBSERVED after the pre clamp: QuantMeasure's eval-mode output (common.cuh fake_quant, the
// reciprocal multiply of CUDA tensors) of v and of the residual r[idx], each when its observer is on, then the fp32 add.
__device__ __forceinline__ float observed_add(float v, int64_t idx, const AffineObserved& e) {
  if (e.obs_on) v = fake_quant<true>(v, e.obs);
  if (e.r) {
    float rv = e.r[idx];
    if (e.res_on) rv = fake_quant<true>(rv, e.res);
    v = __fadd_rn(v, rv);
  }
  return v;
}

// fused_value without a residual, for the Rows epilogue
__device__ __forceinline__ float rows_value(int32_t acc, float dq, float b, const Rows& e) {
  return clamp_keep_nan(clamp_keep_nan(dequant(acc, dq, b), e.pre_lo, e.pre_hi), e.post_lo, e.post_hi);
}

// What the per-layer path computes from the affine layer's value to a detection head's concatenation, in its order: the
// pass-throughs, the cat operand's observer, the cat tail's pass-throughs, the observer of the cat's single user (an
// elementwise op, so per slice)
__device__ __forceinline__ float affine_rows_value(float v, const AffineRows& e) {
  v = clamp_keep_nan(v, e.pre_lo, e.pre_hi);
  if (e.obs_on) v = fake_quant<true>(v, e.obs);
  v = clamp_keep_nan(v, e.post_lo, e.post_hi);
  if (e.tail_on) v = fake_quant<true>(v, e.tail);
  return v;
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

// One thread per (n, pixel): its Cpad / 16 chunks of shifted codes and their sum over the real channels, S[n, h, w].
__global__ void k_i8_quantize_affine(const float* __restrict__ x, int8_t* __restrict__ q, int32_t* __restrict__ S, int C,
                                     int HW, int Cpad, int64_t total, float neg_min, float inv_scale, float qmax) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i % HW, n = i / HW;
    int32_t sum = 0;
    for (int ch = 0; ch < Cpad / 16; ++ch) {
      alignas(16) int8_t v[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = ch * 16 + j;
        v[j] = c < C ? affine_code(x[(n * C + c) * HW + p], neg_min, inv_scale, qmax) : (int8_t)0;
        sum += v[j];
      }
      *reinterpret_cast<int4*>(q + i * Cpad + ch * 16) = *reinterpret_cast<const int4*>(v);
    }
    S[i] = sum;
  }
}

// Weight codes of an already fake-quantized tensor: q = clamp(rint(fp32(fp32(w - w_min) / w_scale)), 0, qmax), stored as
// q - 128 in the layout of k_i8_pack_dense (dense) or k_i8_pack_dw (depthwise, element i = (tap, c)).  *n_bad counts the
// weights with fp32(fp32(q * w_scale) + w_min) != w, bit for bit.
__global__ void k_i8_pack_affine(const float* __restrict__ w, int8_t* __restrict__ out, int32_t* __restrict__ n_bad, int C,
                                 int taps, int Cpad, bool dense, int64_t total, float w_min, float w_scale, float qmax) {
  int32_t bad = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int64_t t = i / Cpad;
    int8_t code = 0;
    if (c < C) {
      const float v = dense ? w[((t / taps) * C + c) * taps + t % taps] : w[(int64_t)c * taps + t];
      const float q = fminf(fmaxf(rintf(__fdiv_rn(__fsub_rn(v, w_min), w_scale)), 0.f), qmax);
      bad += __float_as_uint(__fadd_rn(__fmul_rn(q, w_scale), w_min)) != __float_as_uint(v);
      code = (int8_t)((int)q - 128);
    }
    out[i] = code;
  }
  if (bad) atomicAdd(n_bad, bad);
}

// One thread per output channel o of a dense layer: T[r][s] = sum of its codes over taps (r' < r, s' < s) and all channels,
// table + o * (kh + 1) * (kw + 1), row-major.  The in-image taps of any output pixel form a rectangle [r0, r1) x [s0, s1)
// (tap_range), whose sum is T[r1][s1] - T[r0][s1] - T[r1][s0] + T[r0][s0].
__global__ void k_i8_affine_table(const int8_t* __restrict__ wq, int32_t* __restrict__ table, int O, int kh, int kw,
                                  int Cpad) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= O) return;
  const int tw = kw + 1;
  int32_t* T = table + (int64_t)o * (kh + 1) * tw;
  for (int s = 0; s <= kw; ++s) T[s] = 0;
  for (int r = 0; r < kh; ++r) {
    T[(r + 1) * tw] = 0;
    int32_t row = 0;
    for (int s = 0; s < kw; ++s) {
      const int4* src = reinterpret_cast<const int4*>(wq + ((int64_t)o * kh * kw + r * kw + s) * Cpad);
      for (int ch = 0; ch < Cpad / 16; ++ch) {
        const int4 v = src[ch];
        row = __dp4a(v.x, 0x01010101, row), row = __dp4a(v.y, 0x01010101, row);
        row = __dp4a(v.z, 0x01010101, row), row = __dp4a(v.w, 0x01010101, row);
      }
      T[(r + 1) * tw + s + 1] = T[r * tw + s + 1] + row;
    }
  }
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

  if constexpr (affine_out(OUT)) {
    // Past the [o][m] staging below: per pixel of the tile (THREADS == BM, one each) A = the sum of S over its in-image
    // taps and the tap rectangle (r0 | r1 << 16, s0 | s1 << 16).
    static_assert(THREADS == BM && BN * EPI_LD * 4 + BM * 12 <= STAGES * STAGE_BYTES, "affine epilogue staging");
    int32_t* sA = reinterpret_cast<int32_t*>(smem + BN * EPI_LD * 4);
    uint32_t* sR = reinterpret_cast<uint32_t*>(sA + BM);
    {
      const int64_t m = m0 + tid;
      int32_t a = 0;
      int2 rr = make_int2(0, 0), ss = make_int2(0, 0);
      if (m < M) {
        const int n = (int)(m / OHW), p = (int)(m % OHW), oh = p / g.OW, ow = p % g.OW;
        rr = tap_range(oh, g.stride_h, g.pad_h, g.dil_h, g.kh, g.H);
        ss = tap_range(ow, g.stride_w, g.pad_w, g.dil_w, g.kw, g.W);
        const int32_t* img = rq.S + (int64_t)n * g.H * g.W;
        for (int r = rr.x; r < rr.y; ++r) {
          const int32_t* row = img + (int64_t)(oh * g.stride_h - g.pad_h + r * g.dil_h) * g.W;
          for (int s = ss.x; s < ss.y; ++s) a += row[ow * g.stride_w - g.pad_w + s * g.dil_w];
        }
      }
      sA[tid] = a;
      sR[2 * tid] = (uint32_t)rr.x | ((uint32_t)rr.y << 16);
      sR[2 * tid + 1] = (uint32_t)ss.x | ((uint32_t)ss.y << 16);
    }
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
    const int tw = g.kw + 1, tsize = (g.kh + 1) * tw;
    if constexpr (OUT == Out::AFFINE_ROWS) {
      // channels fastest, so the stores run along each pixel's row of the pixel-major output
      for (int e = tid; e < BM * BN; e += THREADS) {
        const int ol = e % BN, ml = e / BN;
        const int64_t m = m0 + ml;
        const int o = o0 + ol;
        if (m >= M || o >= g.O) continue;
        const int32_t P = st[ol * EPI_LD + ml];
        const uint32_t rh = sR[2 * ml], rw = sR[2 * ml + 1];
        const int r0 = rh & 0xffff, r1 = rh >> 16, s0 = rw & 0xffff, s1 = rw >> 16;
        const int32_t* T = rq.table + (int64_t)o * tsize;
        const int32_t Wv = T[r1 * tw + s1] - T[r0 * tw + s1] - T[r1 * tw + s0] + T[r0 * tw + s0];
        const float v = affine_value(P, sA[ml], Wv, (r1 - r0) * (s1 - s0) * g.C, bias ? bias[o] : 0.f, rq);
        rq.y[(m / OHW) * rq.img_stride + rq.off + (m % OHW) * g.O + o] = affine_rows_value(v, rq);
      }
      return;
    } else if constexpr (OUT == Out::AFFINE) {
      for (int e = tid; e < BM * BN; e += THREADS) {
        const int ml = e % BM, ol = e / BM;
        const int64_t m = m0 + ml;
        const int o = o0 + ol;
        if (m >= M || o >= g.O) continue;
        const int32_t P = st[ol * EPI_LD + ml];
        const uint32_t rh = sR[2 * ml], rw = sR[2 * ml + 1];
        const int r0 = rh & 0xffff, r1 = rh >> 16, s0 = rw & 0xffff, s1 = rw >> 16;
        const int32_t* T = rq.table + (int64_t)o * tsize;
        const int32_t Wv = T[r1 * tw + s1] - T[r0 * tw + s1] - T[r1 * tw + s0] + T[r0 * tw + s0];
        const int64_t idx = ((m / OHW) * g.O + o) * OHW + m % OHW;
        y[idx] = affine_value(P, sA[ml], Wv, (r1 - r0) * (s1 - s0) * g.C, bias ? bias[o] : 0.f, rq);
        if (acc_out) acc_out[idx] = P;
      }
      return;
    } else {
      // Each element's code replaces its sum in the staging (the same thread reads and writes the word; channels O ..
      // o0 + 63 stage code 0, the pad of yq); then one thread per pixel gathers its 64 codes, stores its chunks below
      // cpad and sums them into S.  The residual reads and the y stores run along the pixels of one channel, as the F32
      // epilogue's.
      for (int e = tid; e < BM * BN; e += THREADS) {
        const int ml = e % BM, ol = e / BM;
        const int64_t m = m0 + ml;
        const int o = o0 + ol;
        if (m >= M) continue;
        int32_t code = 0;
        if (o < g.O) {
          int32_t P = st[ol * EPI_LD + ml];
          const uint32_t rh = sR[2 * ml], rw = sR[2 * ml + 1];
          const int r0 = rh & 0xffff, r1 = rh >> 16, s0 = rw & 0xffff, s1 = rw >> 16;
          const int32_t* T = rq.table + (int64_t)o * tsize;
          int32_t Wv = T[r1 * tw + s1] - T[r0 * tw + s1] - T[r1 * tw + s0] + T[r0 * tw + s0];
          const int64_t idx = ((m / OHW) * g.O + o) * OHW + m % OHW;
          int32_t A = sA[ml], Nv = (r1 - r0) * (s1 - s0) * g.C;
          if constexpr (OUT == Out::AFFINE_LAYOUT) {
            // the out-of-image taps loaded 0; with a pad code they hold z' over the C real channels, which adds
            // z' (Wtot - Win) to P and z' C (taps - in-image taps) to A; Wv and Nv then cover every tap
            if (rq.pad_on) {
              const int32_t Wt = T[g.kh * tw + g.kw];
              P += rq.pad_code * (Wt - Wv);
              A += rq.pad_code * (g.kh * g.kw * g.C - Nv);
              Wv = Wt, Nv = g.kh * g.kw * g.C;
            }
          }
          float v = affine_value(P, A, Wv, Nv, bias ? bias[o] : 0.f, rq);
          v = clamp_keep_nan(v, rq.pre_lo, rq.pre_hi);
          if constexpr (observed(OUT)) {
            v = observed_add(v, idx, rq);
          } else {
            if (rq.r) v = __fadd_rn(v, rq.r[idx]);
          }
          v = clamp_keep_nan(v, rq.post_lo, rq.post_hi);
          if (y) y[idx] = v;
          code = affine_code(v, rq.neg_min, rq.inv_scale, rq.qmax);
        }
        st[ol * EPI_LD + ml] = code;
      }
      if (!rq.yq) return;
      __syncthreads();
      const int64_t m = m0 + tid;
      if (m >= M) return;
      int32_t sum = 0;
#pragma unroll
      for (int c = 0; c < BN / 16; ++c) {
        alignas(16) int8_t v[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          v[j] = (int8_t)st[(c * 16 + j) * EPI_LD + tid];
          sum += v[j];
        }
        if (o0 + c * 16 < rq.cpad)
          *reinterpret_cast<int4*>(rq.yq + m * code_stride<OUT>(rq) + o0 + c * 16) = *reinterpret_cast<const int4*>(v);
      }
      if (rq.S_out) {
        if (rq.S_atomic) atomicAdd(rq.S_out + m, sum);
        else rq.S_out[m] = sum;
      }
      return;
    }
  }
  if constexpr (OUT == Out::ROWS) {
    // Straight from the accumulator layout: for one register pair (h = 0, 1), a warp holds 8 pixels x 8 consecutive
    // channels, so the stores run in 32-byte pieces along the channels of each pixel's row.  4-byte stores: off and O are
    // arbitrary, so a row may start at any float.
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
        const int64_t m = m0 + wm * 64 + i * 16 + (lane >> 2) + rr * 8;
        if (m >= M) continue;
        float* row = rq.y + (m / OHW) * rq.img_stride + rq.off + (m % OHW) * g.O;
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int o = o0 + wn * 32 + j * 8 + (lane & 3) * 2 + h;
            if (o < g.O) row[o] = rows_value(acc[i][j][2 * rr + h], d[j][h], b[j][h], rq);
          }
      }
    return;
  }
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
  if constexpr (OUT == Out::I8 || OUT == Out::FUSED) {
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
// PAD (Out::AFFINE_LAYOUT with a pad code): every tap counts, the out-of-image ones reading the code rq.pad_code.
template <Out OUT, bool PAD = false>
__global__ void k_i8_conv_dw(const int8_t* __restrict__ xq, const int8_t* __restrict__ wq, const float* __restrict__ dq,
                             const float* __restrict__ bias, float* __restrict__ y, int32_t* __restrict__ acc_out, DfqI8Conv g,
                             int64_t total, typename EpiOf<OUT>::type rq) {
  static_assert(!PAD || OUT == Out::AFFINE_LAYOUT, "a pad code is the layout epilogue's");
  const int chunks = g.Cpad / 16, OHW = g.OH * g.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int p = (int)(i % OHW);
    const int64_t t = i / OHW;
    const int ch = (int)(t % chunks);
    const int64_t n = t / chunks;
    constexpr bool affine = affine_out(OUT);
    if constexpr (OUT == Out::I8 || OUT == Out::FUSED || affine_epilogue(OUT)) {
      // the input's Cpad may be wider than yq's cpad = round_up(O, 16): chunks past it hold only pad channels, and yq has
      // no room for them
      if (ch * 16 >= rq.cpad) continue;
    }
    const int oh = p / g.OW, ow = p % g.OW;
    int32_t acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0;
    int32_t xsum[16], wsum[16], ntaps = 0;                      // affine: A, Wv per channel, the in-image taps
    if constexpr (affine) {
#pragma unroll
      for (int j = 0; j < 16; ++j) xsum[j] = wsum[j] = 0;
    }
    const int8_t* img = xq + n * g.H * g.W * g.Cpad + ch * 16;
    auto mac = [&](const int4& xv, int r, int s) {
      const int4 wv = __ldg(reinterpret_cast<const int4*>(wq + (r * g.kw + s) * g.Cpad + ch * 16));
      const int8_t* xb = reinterpret_cast<const int8_t*>(&xv);
      const int8_t* wb = reinterpret_cast<const int8_t*>(&wv);
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] += (int32_t)xb[j] * (int32_t)wb[j];
      if constexpr (affine) {
#pragma unroll
        for (int j = 0; j < 16; ++j) xsum[j] += xb[j], wsum[j] += wb[j];
        ++ntaps;
      }
    };
    if constexpr (PAD) {
      const int z = (int)(uint8_t)rq.pad_code * 0x01010101;    // z' in every byte (pad channels: weights 0)
      const int4 zv = make_int4(z, z, z, z);
      for (int r = 0; r < g.kh; ++r) {
        const int ih = oh * g.stride_h - g.pad_h + r * g.dil_h;
        const bool row = (unsigned)ih < (unsigned)g.H;
        for (int s = 0; s < g.kw; ++s) {
          const int iw = ow * g.stride_w - g.pad_w + s * g.dil_w;
          mac(row && (unsigned)iw < (unsigned)g.W
                  ? __ldg(reinterpret_cast<const int4*>(img + ((int64_t)ih * g.W + iw) * g.Cpad)) : zv, r, s);
        }
      }
    } else {
      for (int r = 0; r < g.kh; ++r) {
        const int ih = oh * g.stride_h - g.pad_h + r * g.dil_h;
        if ((unsigned)ih >= (unsigned)g.H) continue;
        for (int s = 0; s < g.kw; ++s) {
          const int iw = ow * g.stride_w - g.pad_w + s * g.dil_w;
          if ((unsigned)iw >= (unsigned)g.W) continue;
          mac(__ldg(reinterpret_cast<const int4*>(img + ((int64_t)ih * g.W + iw) * g.Cpad)), r, s);
        }
      }
    }
    if constexpr (OUT == Out::AFFINE_ROWS) {                    // this pixel's 16 channels of its row
      float* row = rq.y + n * rq.img_stride + rq.off + (int64_t)p * g.C + ch * 16;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = ch * 16 + j;
        if (c < g.C) row[j] = affine_rows_value(affine_value(acc[j], xsum[j], wsum[j], ntaps, bias ? bias[c] : 0.f, rq), rq);
      }
      continue;
    }
    if constexpr (OUT == Out::AFFINE) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = ch * 16 + j;
        if (c >= g.C) break;
        const int64_t idx = (n * g.C + c) * OHW + p;
        y[idx] = affine_value(acc[j], xsum[j], wsum[j], ntaps, bias ? bias[c] : 0.f, rq);
        if (acc_out) acc_out[idx] = acc[j];
      }
      continue;
    }
    if constexpr (affine_epilogue(OUT)) {                       // as Out::FUSED; the pixel's sum shared by its chunks
      alignas(16) int8_t v[16];
      int32_t sum = 0;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = ch * 16 + j;
        v[j] = 0;
        if (c < g.C) {
          const int64_t idx = (n * g.C + c) * OHW + p;
          float f = affine_value(acc[j], xsum[j], wsum[j], ntaps, bias ? bias[c] : 0.f, rq);
          f = clamp_keep_nan(f, rq.pre_lo, rq.pre_hi);
          if constexpr (observed(OUT)) {
            f = observed_add(f, idx, rq);
          } else {
            if (rq.r) f = __fadd_rn(f, rq.r[idx]);
          }
          f = clamp_keep_nan(f, rq.post_lo, rq.post_hi);
          if (y) y[idx] = f;
          v[j] = affine_code(f, rq.neg_min, rq.inv_scale, rq.qmax);
          sum += v[j];
        }
      }
      if (rq.yq) {
        *reinterpret_cast<int4*>(rq.yq + (n * OHW + p) * code_stride<OUT>(rq) + ch * 16) = *reinterpret_cast<const int4*>(v);
        if (rq.S_out) {
          if (rq.S_atomic) atomicAdd(rq.S_out + n * OHW + p, sum);
          else rq.S_out[n * OHW + p] = sum;
        }
      }
      continue;
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
    if constexpr (OUT == Out::ROWS) {                           // this pixel's 16 channels of its row
      float* row = rq.y + n * rq.img_stride + rq.off + (int64_t)p * g.C + ch * 16;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = ch * 16 + j;
        if (c < g.C) row[j] = rows_value(acc[j], dq[c], bias ? bias[c] : 0.f, rq);
      }
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
// A window with no tap inside the input (possible with dilation) is -inf in torch, whose code is -127 (AFFINE: -128, below);
// pad channels 0.
// !CODES: x fp32 NCHW [N, C, H, W] -> y fp32 NCHW [N, C, OH, OW] and / or yq int8 NHWC at `scale`, with torch's CUDA rule:
// from -inf, taps row-major, the running max replaced when v > m or v is NaN (so the first of tied values is kept).
// AFFINE (dfq_i8_affine_maxpool): the codes are the affine scheme's shifted codes, in [-128, 127].  affine_code is monotone
// non-decreasing too (a positive inv_scale), the empty window's -inf has code -128, the !CODES codes are the consumer's
// (a.neg_min, a.inv_scale, a.qmax) and, with a.S, S[n, p] += the sum of the pooled codes over the real channels.
struct AffinePool {
  int32_t* S;
  float neg_min, inv_scale, qmax;
};

template <bool CODES, bool AFFINE = false>
__global__ void k_i8_maxpool(const int8_t* __restrict__ xq, const float* __restrict__ x, float* __restrict__ y,
                             int8_t* __restrict__ yq, float scale, DfqI8Pool g, int64_t total, AffinePool a) {
  constexpr int lowest = AFFINE ? (int)0x80808080 : (int)0x81818181;   // the smallest code in every byte
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
      int m[4] = {lowest, lowest, lowest, lowest};
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
        for (int j = 0; j < 16; ++j) v[j] = ch * 16 + j < g.C ? (int8_t)lowest : (int8_t)0;
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
        if constexpr (AFFINE) {
          if (yq) v[j] = affine_code(mx, a.neg_min, a.inv_scale, a.qmax);
        } else {
          v[j] = q8(mx, scale);
        }
      }
      if (!yq) continue;
    }
    if constexpr (AFFINE) {
      if (a.S) {
        int32_t sum = 0;
#pragma unroll
        for (int j = 0; j < 16; ++j) sum += ch * 16 + j < g.C ? v[j] : 0;
        atomicAdd(a.S + n * OHW + p, sum);
      }
    }
    *reinterpret_cast<int4*>(yq + (n * OHW + p) * g.Cpad + ch * 16) = *reinterpret_cast<const int4*>(v);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// bilinear upsampling: one thread per (n, 16 channels, output pixel), pixels fastest, as k_i8_conv_dw
// ------------------------------------------------------------------------------------------------------------------
// x fp32 NCHW [N, C, H, W] -> y fp32 NCHW [N, C, OH, OW] and / or the codes q8(clamp(y, lo, hi), out_scale) into channels
// [coff, coff + round_up(C, 16)) of int8 NHWC yq [N, OH, OW, cstride] (one 16-byte store per thread, pad channels 0).
// y is bit for bit torch's CUDA upsample_bilinear2d_out_frame<float, float> (bilinear.cuh).
__global__ void k_i8_upsample_bilinear(const float* __restrict__ x, float* __restrict__ y, int8_t* __restrict__ yq,
                                       DfqI8Resize g, float scale_h, float scale_w, int64_t total) {
  const int chunks = (g.C + 15) / 16;
  const int64_t HW = (int64_t)g.H * g.W, OHW = (int64_t)g.OH * g.OW;    // a plane may exceed 2^31 pixels
  const bool copy = g.H == g.OH && g.W == g.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i % OHW;
    const int64_t t = i / OHW;
    const int ch = (int)(t % chunks);
    const int64_t n = t / chunks;
    const int oh = (int)(p / g.OW), ow = (int)(p % g.OW);
    const BilinearTap th = bilinear_tap(oh, scale_h, g.align_corners, g.H);
    const BilinearTap tw = bilinear_tap(ow, scale_w, g.align_corners, g.W);
    alignas(16) int8_t v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = ch * 16 + j;
      v[j] = 0;
      if (c >= g.C) continue;
      const float f = bilinear_value(x + (n * g.C + c) * HW, g.W, oh, ow, th, tw, copy);
      if (y) y[(n * g.C + c) * OHW + p] = f;
      v[j] = q8(clamp_keep_nan(f, g.lo, g.hi), g.out_scale);
    }
    if (yq)
      *reinterpret_cast<int4*>(yq + (n * OHW + p) * g.cstride + g.coff + ch * 16) = *reinterpret_cast<const int4*>(v);
  }
}

// The affine scheme's scalars of dfq_i8_affine_upsample_bilinear: the observer (obs_on) and the consumer's quantizer.
struct AffineResize {
  QuantScalars obs;
  float neg_min, inv_scale, qmax;
  float pre_lo, pre_hi, post_lo, post_hi;
  bool obs_on;
};

// k_i8_upsample_bilinear's thread layout and value v, then clamp(pre), the observer, clamp(post) and the consumer's shifted
// code into channels [coff, coff + round_up(C, 16)) of yq [N, OH, OW, cstride], the 16 codes' sum added to S[n, p].
__global__ void k_i8_affine_upsample(const float* __restrict__ x, int8_t* __restrict__ yq, int32_t* __restrict__ S,
                                     DfqI8AffineResize g, AffineResize a, float scale_h, float scale_w, int64_t total) {
  const int chunks = (g.C + 15) / 16;
  const int64_t HW = (int64_t)g.H * g.W, OHW = (int64_t)g.OH * g.OW;
  const bool copy = g.H == g.OH && g.W == g.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i % OHW;
    const int64_t t = i / OHW;
    const int ch = (int)(t % chunks);
    const int64_t n = t / chunks;
    const int oh = (int)(p / g.OW), ow = (int)(p % g.OW);
    const BilinearTap th = bilinear_tap(oh, scale_h, g.align_corners, g.H);
    const BilinearTap tw = bilinear_tap(ow, scale_w, g.align_corners, g.W);
    alignas(16) int8_t v[16];
    int32_t sum = 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = ch * 16 + j;
      v[j] = 0;
      if (c >= g.C) continue;
      float f = clamp_keep_nan(bilinear_value(x + (n * g.C + c) * HW, g.W, oh, ow, th, tw, copy), a.pre_lo, a.pre_hi);
      if (a.obs_on) f = fake_quant<true>(f, a.obs);
      f = clamp_keep_nan(f, a.post_lo, a.post_hi);
      v[j] = affine_code(f, a.neg_min, a.inv_scale, a.qmax);
      sum += v[j];
    }
    *reinterpret_cast<int4*>(yq + (n * OHW + p) * g.cstride + g.coff + ch * 16) = *reinterpret_cast<const int4*>(v);
    if (S) atomicAdd(S + n * OHW + p, sum);
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

#define DFQ_REQUIRE_WHO(cond, msg)                                         \
  do {                                                                     \
    if (!(cond)) {                                                         \
      ::dfq::set_error("%s: %s (%s)", who, msg, #cond);                    \
      return DFQ_E_ARG;                                                    \
    }                                                                      \
  } while (0)

// The convolution of output mode OUT on g with epilogue ep: the tensor-core main loop for groups == 1, else the depthwise
// one (PAD: its variant that reads the pad code on out-of-image taps)
template <Out OUT, bool PAD = false>
int launch_conv(const char* who, const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, float* y,
                int32_t* acc_out, const DfqI8Conv* g, const typename EpiOf<OUT>::type& ep, cudaStream_t st) {
  if (g->groups == 1) {
    const int64_t M = (int64_t)g->N * g->OH * g->OW;
    DFQ_REQUIRE_WHO((M + BM - 1) / BM < (1LL << 31), "too many output pixels");
    const dim3 grid((unsigned)((M + BM - 1) / BM), (unsigned)((g->O + BN - 1) / BN));
    k_i8_conv_mma<OUT><<<grid, THREADS, 0, st>>>(xq, wq, dq, bias, y, acc_out, *g, ep);
  } else {
    const int64_t total = (int64_t)g->N * (g->Cpad / 16) * g->OH * g->OW;
    k_i8_conv_dw<OUT, PAD><<<grid_for(total, 256), 256, 0, st>>>(xq, wq, dq, bias, y, acc_out, *g, total, ep);
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

// A slice of a concatenation's codes: channels [coff, coff + cpad) of rows of cstride codes, 16-aligned inside the row;
// `channels` names the dimension cpad rounds up (O or C)
int check_slice(const char* who, int64_t coff, int64_t cstride, int cpad, char channels) {
  DFQ_REQUIRE_WHO(coff >= 0 && cstride > 0 && coff % 16 == 0 && cstride % 16 == 0,
                  "coff and cstride must be non-negative multiples of 16");
  if (coff + cpad > cstride) {
    set_error("%s: the slice coff + round_up(%c, 16) exceeds cstride (coff + cpad <= cstride)", who, channels);
    return DFQ_E_ARG;
  }
  return 0;
}

// A max pool's geometry: torch's max_pool2d (padding at most half the kernel, OH / OW as torch forms them) on codes of
// Cpad channels; exactly one input, codes xq or fp32 x
int check_pool(const char* who, const DfqI8Pool* g, const void* xq, const void* x) {
  DFQ_REQUIRE_WHO(g != nullptr, "null geometry");
  DFQ_REQUIRE_WHO(g->N > 0 && g->C > 0 && g->H > 0 && g->W > 0 && g->kh > 0 && g->kw > 0, "empty dimension");
  DFQ_REQUIRE_WHO(g->stride_h > 0 && g->stride_w > 0 && g->dil_h > 0 && g->dil_w > 0 && g->pad_h >= 0 && g->pad_w >= 0 &&
                      (g->ceil_mode == 0 || g->ceil_mode == 1),
                  "bad stride / padding / dilation / ceil_mode");
  DFQ_REQUIRE_WHO(g->pad_h <= g->kh / 2 && g->pad_w <= g->kw / 2 && g->pad_h <= (g->dil_h * (g->kh - 1) + 1) / 2 &&
                      g->pad_w <= (g->dil_w * (g->kw - 1) + 1) / 2,
                  "padding must be at most half of the kernel and of the effective kernel");
  DFQ_REQUIRE_WHO(g->Cpad >= g->C && g->Cpad % 16 == 0, "Cpad must be a multiple of 16 that holds C");
  DFQ_REQUIRE_WHO(g->OH == pool_extent(g->H, g->kh, g->pad_h, g->stride_h, g->dil_h, g->ceil_mode) &&
                      g->OW == pool_extent(g->W, g->kw, g->pad_w, g->stride_w, g->dil_w, g->ceil_mode) && g->OH > 0 &&
                      g->OW > 0,
                  "OH / OW do not follow from the geometry");
  DFQ_REQUIRE_WHO((xq != nullptr) != (x != nullptr), "give exactly one input, codes xq or fp32 x");
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// ncnn model files: weight codes verbatim, and ncnn's plane mean
// ------------------------------------------------------------------------------------------------------------------

// Element (o, c, tap) of ncnn's codes [O][C/g][kh][kw] -> its index in the packed layout of k_i8_pack_dense (groups == 1:
// [O][taps][Cpad]) or k_i8_pack_dw (depthwise, c == 0: [taps][Cpad] with channel o)
__device__ __forceinline__ int64_t packed_index(int64_t o, int c, int tap, int taps, int Cpad, bool dense) {
  return dense ? (o * taps + tap) * Cpad + c : (int64_t)tap * Cpad + o;
}

// One thread per packed byte: the code it holds, or 0 in a pad channel
__global__ void k_i8_pack_codes(const int8_t* __restrict__ codes, int8_t* __restrict__ out, int C, int taps, int Cpad,
                                bool dense, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cpad);
    const int64_t t = i / Cpad;
    if (dense) {
      const int tap = (int)(t % taps);
      const int64_t o = t / taps;
      out[i] = c < C ? codes[(o * C + c) * taps + tap] : (int8_t)0;
    } else {
      out[i] = c < C ? codes[(int64_t)c * taps + t] : (int8_t)0;
    }
  }
}

// One thread per code of ncnn's layout, read back from the packed layout
__global__ void k_i8_unpack_codes(const int8_t* __restrict__ packed, int8_t* __restrict__ codes, int Cg, int taps, int Cpad,
                                  bool dense, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int tap = (int)(i % taps);
    const int64_t t = i / taps;
    codes[i] = packed[packed_index(t / Cg, (int)(t % Cg), tap, taps, Cpad, dense)];
  }
}

// ncnn's mean of each (image, channel) plane of x [N, C, P]: sum = 0.f, then sum += x[p] for p = 0 .. P - 1 in order (fp32,
// each add rounded), then sum * k (Reduction MEAN: k = fp32(1 / P)) or sum / P (Pooling global average, divide).  Row r
// of the output walks [N, cols): cols = Cpad when the codes are written (r past C: a pad channel, code 0), else C.
// Each warp owns 32 consecutive rows.  It stages them 32 columns at a time through shared memory - one coalesced 128-byte
// load per plane - and lane i then adds row i's 32 values in plane order, so the order is the sequential one.
constexpr int PM_WARPS = 8;

__global__ void __launch_bounds__(PM_WARPS * 32) k_i8_plane_mean(const float* __restrict__ x, float* __restrict__ y,
                                                                 int8_t* __restrict__ yq, int C, int cols, int64_t P,
                                                                 int64_t rows, bool divide, float k, float out_scale) {
  __shared__ float tile[PM_WARPS][32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float(*s)[33] = tile[warp];
  for (int64_t base = ((int64_t)blockIdx.x * PM_WARPS + warp) * 32; base < rows;
       base += (int64_t)gridDim.x * PM_WARPS * 32) {
    const int64_t r = base + lane;
    const int64_t n = r / cols;
    const int c = (int)(r - n * cols);
    const bool real = r < rows && c < C;
    const int64_t off = real ? (n * C + c) * P : -1;        // this lane's plane, broadcast to the warp below
    float sum = 0.f;
    for (int64_t j0 = 0; j0 < P; j0 += 32) {
      const bool col = j0 + lane < P;
#pragma unroll 8
      for (int i = 0; i < 32; ++i) {
        const int64_t o = __shfl_sync(0xffffffffu, off, i);
        if (o >= 0 && col) s[i][lane] = __ldg(x + o + j0 + lane);
      }
      __syncwarp();
      const int m = P - j0 < 32 ? (int)(P - j0) : 32;
      for (int j = 0; j < m; ++j) sum = __fadd_rn(sum, s[lane][j]);
      __syncwarp();
    }
    if (r >= rows) continue;
    const float v = divide ? __fdiv_rn(sum, (float)P) : __fmul_rn(sum, k);
    if (real && y) y[n * C + c] = v;
    if (yq) yq[r] = real ? q8(v, out_scale) : (int8_t)0;
  }
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
  return launch_conv<Out::F32>("dfq_i8_conv", xq, wq, dq, bias, y, acc_out, g, Requant{}, (cudaStream_t)stream);
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
  return launch_conv<Out::I8>("dfq_i8_conv_requant", xq, wq, dq, bias, nullptr, nullptr, g, rq, (cudaStream_t)stream);
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
  return launch_conv<Out::FUSED>("dfq_i8_conv_fused", xq, wq, dq, bias, nullptr, nullptr, g, ep, (cudaStream_t)stream);
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
  if (int rc = check_slice("dfq_i8_conv_slice", coff, cstride, cpad, 'O')) return rc;
  const int64_t pixels = (int64_t)g->N * g->OH * g->OW;
  const int64_t y_bytes = pixels * g->O * (int64_t)sizeof(float);
  int8_t* yq = e->yq + coff;
  const int64_t slice_bytes = (pixels - 1) * cstride + cpad;          // first to last byte the slice's chunks cover
  DFQ_REQUIRE(!overlap(e->residual, y_bytes, yq, slice_bytes), "dfq_i8_conv_slice: residual overlaps the slice");
  DFQ_REQUIRE(!overlap(e->y, y_bytes, yq, slice_bytes), "dfq_i8_conv_slice: y overlaps the slice");
  DFQ_REQUIRE(!overlap(e->residual, y_bytes, e->y, y_bytes), "dfq_i8_conv_slice: residual overlaps y");
  cudaStream_t st = (cudaStream_t)stream;
  if (!e->residual && !e->y && e->post_lo == -INFINITY && e->post_hi == INFINITY) {
    // codes only after one clamp: the requantizing epilogue
    const Requant rq{yq, e->out_scale, e->pre_lo, e->pre_hi, cpad, cstride};
    return launch_conv<Out::I8>("dfq_i8_conv_slice", xq, wq, dq, bias, nullptr, nullptr, g, rq, st);
  }
  const Fused ep{yq, e->out_scale, e->pre_lo, e->pre_hi, cpad, cstride, e->residual, e->y, e->post_lo, e->post_hi};
  return launch_conv<Out::FUSED>("dfq_i8_conv_slice", xq, wq, dq, bias, nullptr, nullptr, g, ep, st);
}

extern "C" int dfq_i8_conv_nhwc(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, const DfqI8Epilogue* e,
                                int64_t off, int64_t img_stride, const DfqI8Conv* g, void* stream) {
  if (int rc = check_geometry(g)) return rc;
  DFQ_REQUIRE(xq && wq && dq && e, "dfq_i8_conv_nhwc: null pointer");
  DFQ_REQUIRE(aligned16(xq) && aligned16(wq), "dfq_i8_conv_nhwc: codes must be 16-byte aligned");
  DFQ_REQUIRE(e->y, "dfq_i8_conv_nhwc: no output (y is NULL)");
  DFQ_REQUIRE(((uintptr_t)e->y & 3) == 0, "dfq_i8_conv_nhwc: y must be 4-byte aligned");
  DFQ_REQUIRE(!e->residual && !e->yq, "dfq_i8_conv_nhwc: residual and yq must be NULL (fp32 rows only)");
  DFQ_REQUIRE(ordered(e->pre_lo, e->pre_hi) && ordered(e->post_lo, e->post_hi),
              "dfq_i8_conv_nhwc: pre / post clamp bounds must be ordered and not NaN");
  const int64_t extent = (int64_t)g->OH * g->OW * g->O;              // floats of one image's rows
  DFQ_REQUIRE(off >= 0, "dfq_i8_conv_nhwc: off must be non-negative");
  DFQ_REQUIRE(img_stride >= off + extent, "dfq_i8_conv_nhwc: img_stride must be at least off + OH * OW * O");
  const int64_t x_bytes = (int64_t)g->N * g->H * g->W * g->Cpad;
  const int64_t y_bytes = ((g->N - 1) * img_stride + extent) * (int64_t)sizeof(float);   // first to last row written
  DFQ_REQUIRE(!overlap(xq, x_bytes, e->y + off, y_bytes), "dfq_i8_conv_nhwc: y overlaps xq");
  const Rows ep{e->y, off, img_stride, e->pre_lo, e->pre_hi, e->post_lo, e->post_hi};
  return launch_conv<Out::ROWS>("dfq_i8_conv_nhwc", xq, wq, dq, bias, nullptr, nullptr, g, ep, (cudaStream_t)stream);
}

extern "C" int dfq_i8_maxpool(const int8_t* xq, const float* x, float* y, int8_t* yq, float out_scale, const DfqI8Pool* g,
                              void* stream) {
  if (int rc = check_pool("dfq_i8_maxpool", g, xq, x)) return rc;
  const int64_t in_px = (int64_t)g->N * g->H * g->W, out_px = (int64_t)g->N * g->OH * g->OW;
  const int64_t total = out_px * (g->Cpad / 16);
  cudaStream_t st = (cudaStream_t)stream;
  if (xq) {
    DFQ_REQUIRE(yq && !y, "dfq_i8_maxpool: codes in give codes out only (yq, no y)");
    DFQ_REQUIRE(aligned16(xq) && aligned16(yq), "dfq_i8_maxpool: xq and yq must be 16-byte aligned");
    DFQ_REQUIRE(!overlap(xq, in_px * g->Cpad, yq, out_px * g->Cpad), "dfq_i8_maxpool: yq overlaps xq");
    k_i8_maxpool<true><<<grid_for(total, 256), 256, 0, st>>>(xq, nullptr, nullptr, yq, 0.f, *g, total, AffinePool{});
  } else {
    DFQ_REQUIRE(y || yq, "dfq_i8_maxpool: no output requested (y and yq are both NULL)");
    DFQ_REQUIRE(aligned16(yq), "dfq_i8_maxpool: yq must be 16-byte aligned");
    DFQ_REQUIRE(((uintptr_t)x & 3) == 0 && ((uintptr_t)y & 3) == 0, "dfq_i8_maxpool: x and y must be 4-byte aligned");
    DFQ_REQUIRE(!yq || (std::isfinite(out_scale) && out_scale >= 0.f),
                "dfq_i8_maxpool: out_scale must be finite and non-negative when yq is written");
    const int64_t x_bytes = in_px * g->C * 4, y_bytes = out_px * g->C * 4, yq_bytes = out_px * g->Cpad;
    DFQ_REQUIRE(!overlap(x, x_bytes, y, y_bytes) && !overlap(x, x_bytes, yq, yq_bytes) && !overlap(y, y_bytes, yq, yq_bytes),
                "dfq_i8_maxpool: x, y and yq overlap");
    k_i8_maxpool<false><<<grid_for(total, 256), 256, 0, st>>>(nullptr, x, y, yq, out_scale, *g, total, AffinePool{});
  }
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_upsample_bilinear(const float* x, float* y, int8_t* yq, const DfqI8Resize* g, void* stream) {
  DFQ_REQUIRE(g != nullptr, "dfq_i8_upsample_bilinear: null geometry");
  DFQ_REQUIRE(x != nullptr, "dfq_i8_upsample_bilinear: null input");
  DFQ_REQUIRE(g->N > 0 && g->C > 0 && g->H > 0 && g->W > 0 && g->OH > 0 && g->OW > 0,
              "dfq_i8_upsample_bilinear: empty dimension (every size must be positive)");
  DFQ_REQUIRE(g->align_corners == 0 || g->align_corners == 1, "dfq_i8_upsample_bilinear: align_corners must be 0 or 1");
  const int cpad = (g->C + 15) / 16 * 16;
  if (int rc = check_slice("dfq_i8_upsample_bilinear", g->coff, g->cstride, cpad, 'C')) return rc;
  DFQ_REQUIRE(y || yq, "dfq_i8_upsample_bilinear: no output requested (y and yq are both NULL)");
  DFQ_REQUIRE(aligned16(yq), "dfq_i8_upsample_bilinear: yq must be 16-byte aligned");
  DFQ_REQUIRE(((uintptr_t)x & 3) == 0 && ((uintptr_t)y & 3) == 0, "dfq_i8_upsample_bilinear: x and y must be 4-byte aligned");
  DFQ_REQUIRE(!yq || (std::isfinite(g->out_scale) && g->out_scale >= 0.f),
              "dfq_i8_upsample_bilinear: out_scale must be finite and non-negative when yq is written");
  DFQ_REQUIRE(ordered(g->lo, g->hi), "dfq_i8_upsample_bilinear: clamp bounds must be ordered and not NaN");
  const int64_t in_px = (int64_t)g->N * g->H * g->W, out_px = (int64_t)g->N * g->OH * g->OW;
  const int64_t x_bytes = in_px * g->C * 4, y_bytes = out_px * g->C * 4;
  const int8_t* slice = yq ? yq + g->coff : nullptr;
  const int64_t slice_bytes = (out_px - 1) * g->cstride + cpad;       // first to last byte the slice's chunks cover
  DFQ_REQUIRE(!overlap(x, x_bytes, y, y_bytes) && !overlap(x, x_bytes, slice, slice_bytes),
              "dfq_i8_upsample_bilinear: x overlaps y or the slice");
  DFQ_REQUIRE(!overlap(y, y_bytes, slice, slice_bytes), "dfq_i8_upsample_bilinear: y overlaps the slice");
  const int64_t total = out_px * (cpad / 16);
  const bool ac = g->align_corners == 1;
  k_i8_upsample_bilinear<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      x, y, yq, *g, bilinear_scale(g->H, g->OH, ac), bilinear_scale(g->W, g->OW, ac), total);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

// ---- the affine scheme -------------------------------------------------------------------------------------------------
namespace dfq {
namespace {

// codes of 1..8 bits; K = kh * kw * C / groups below 2^17, so that |P| <= K * 128 * 128 < 2^31 (codes of -128 reach the
// main loop)
int check_affine(const DfqI8Conv* g, int num_bits, const char* who) {
  if (int rc = check_geometry(g)) return rc;
  if (num_bits > 8) {
    set_error("%s: %d-bit codes do not fit in int8 (at most 8 bits)", who, num_bits);
    return DFQ_E_UNSUPPORTED;
  }
  if (num_bits < 1) {
    set_error("%s: num_bits must be at least 1, got %d", who, num_bits);
    return DFQ_E_ARG;
  }
  const int64_t K = (int64_t)g->kh * g->kw * (g->C / g->groups);
  if (K >= (1 << 17)) {
    set_error("%s: K = kh * kw * C / groups = %lld reaches 131072, where K * 128 * 128 overflows the int32 sums", who,
              (long long)K);
    return DFQ_E_UNSUPPORTED;
  }
  return 0;
}

// QuantMeasure's scalars of a quantizer with 1..8 bits (`bits_name` in the error) and a finite range whose scale and
// inverse are finite fp32 numbers (`range_name` in the error)
int quantizer(const char* who, const char* bits_name, const char* range_name, float lo, float hi, int32_t bits,
              QuantScalars* q) {
  if (bits < 1 || bits > 8) {
    set_error("%s: %s must be in [1, 8], got %d", who, bits_name, bits);
    return bits > 8 ? DFQ_E_UNSUPPORTED : DFQ_E_ARG;
  }
  *q = quant_scalars((double)lo, (double)hi, bits, 0);
  if (!(std::isfinite(lo) && std::isfinite(hi) && std::isfinite(q->scale) && std::isfinite(q->inv_scale))) {
    set_error("%s: %s [%g, %g] is not finite or gives a scale that is not a finite fp32 number", who, range_name, lo, hi);
    return DFQ_E_ARG;
  }
  return 0;
}

// What every affine convolution entry checks of its geometry, codes, weights and constants; out: its output (y or the
// epilogue)
int check_affine_conv(const char* who, const DfqI8Conv* g, const int8_t* xq, const int32_t* S, const int8_t* wq,
                      const int32_t* table, const DfqI8Affine* k, const void* out) {
  if (int rc = check_affine(g, 8, who)) return rc;
  DFQ_REQUIRE_WHO(xq && wq && k && out, "null pointer");
  DFQ_REQUIRE_WHO(g->groups != 1 || (S && table), "a dense layer needs S and its prefix table");
  DFQ_REQUIRE_WHO(aligned16(xq) && aligned16(wq), "codes must be 16-byte aligned");
  if (!(std::isfinite(k->kP) && std::isfinite(k->kA) && std::isfinite(k->kW) && std::isfinite(k->kN))) {
    set_error("%s: the constants kP, kA, kW, kN must be finite, got %g, %g, %g, %g", who, k->kP, k->kA, k->kW, k->kN);
    return DFQ_E_ARG;
  }
  return 0;
}

}  // namespace
}  // namespace dfq

extern "C" int dfq_i8_affine_quantize(const float* x, int8_t* q, int32_t* S, int32_t N, int32_t C, int32_t H, int32_t W,
                                      int32_t Cpad, float act_min, float act_max, int32_t num_bits, void* stream) {
  DFQ_REQUIRE(x && q && S && N > 0 && C > 0 && H > 0 && W > 0, "dfq_i8_affine_quantize: bad arguments");
  DFQ_REQUIRE(Cpad >= C && Cpad % 16 == 0, "dfq_i8_affine_quantize: Cpad must be a multiple of 16 that holds C");
  DFQ_REQUIRE(aligned16(q), "dfq_i8_affine_quantize: q must be 16-byte aligned");
  QuantScalars qs;
  if (int rc = quantizer("dfq_i8_affine_quantize", "num_bits", "the range", act_min, act_max, num_bits, &qs)) return rc;
  const int64_t total = (int64_t)N * H * W;
  k_i8_quantize_affine<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(x, q, S, C, H * W, Cpad, total, qs.neg_min,
                                                                                qs.inv_scale, qs.qmax);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_affine_pack(const float* w, float w_min, float w_scale, int32_t num_bits, int8_t* packed,
                                  int32_t* table, int32_t* n_bad, const DfqI8Conv* g, void* stream) {
  if (int rc = check_affine(g, num_bits, "dfq_i8_affine_pack")) return rc;
  DFQ_REQUIRE(w && packed && n_bad, "dfq_i8_affine_pack: null pointer");
  DFQ_REQUIRE(g->groups != 1 || table, "dfq_i8_affine_pack: a dense layer needs its prefix table");
  DFQ_REQUIRE(aligned16(packed), "dfq_i8_affine_pack: packed must be 16-byte aligned");
  if (!(std::isfinite(w_min) && std::isfinite(w_scale) && w_scale > 0.f)) {
    set_error("dfq_i8_affine_pack: w_min must be finite and w_scale finite and positive, got %g and %g", w_min, w_scale);
    return DFQ_E_ARG;
  }
  const int taps = g->kh * g->kw;
  const bool dense = g->groups == 1;
  const int64_t total = (dense ? (int64_t)g->O : 1) * taps * g->Cpad;
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_CUDA(cudaMemsetAsync(n_bad, 0, sizeof(int32_t), st));
  k_i8_pack_affine<<<grid_for(total, 256), 256, 0, st>>>(w, packed, n_bad, g->C, taps, g->Cpad, dense, total, w_min, w_scale,
                                                         (float)(ldexp(1.0, num_bits) - 1.0));
  DFQ_CUDA(cudaGetLastError());
  if (dense) {
    k_i8_affine_table<<<(g->O + 127) / 128, 128, 0, st>>>(packed, table, g->O, g->kh, g->kw, g->Cpad);
    DFQ_CUDA(cudaGetLastError());
  }
  return 0;
}

extern "C" int dfq_i8_affine_conv(const int8_t* xq, const int32_t* S, const int8_t* wq, const int32_t* table,
                                  const DfqI8Affine* k, const float* bias, float* y, int32_t* acc_out, const DfqI8Conv* g,
                                  void* stream) {
  const char* who = "dfq_i8_affine_conv";
  if (int rc = check_affine_conv(who, g, xq, S, wq, table, k, y)) return rc;
  const Affine ep{S, table, k->kP, k->kA, k->kW, k->kN};
  return launch_conv<Out::AFFINE>(who, xq, wq, nullptr, bias, y, acc_out, g, ep, (cudaStream_t)stream);
}

namespace dfq {
namespace {

// An observer of DfqI8AffineObserve: off (bits 0), or QuantMeasure's scalars of a finite range with 1..8 bits.
int observer_scalars(const char* who, const char* which, float lo, float hi, int32_t bits, QuantScalars* q, bool* on) {
  *on = bits > 0;
  if (bits < 0) {
    set_error("%s: %s_bits must be 0 (off) or in [1, 8], got %d", who, which, bits);
    return DFQ_E_ARG;
  }
  if (bits > 8) {
    set_error("%s: %s_bits = %d: the epilogue's observers have at most 8 bits", who, which, bits);
    return DFQ_E_UNSUPPORTED;
  }
  if (!*on) return 0;
  char range[32];
  std::snprintf(range, sizeof range, "the %s observer's range", which);
  return quantizer(who, which, range, lo, hi, bits, q);
}

// dfq_i8_affine_conv_fused (o == NULL, Out::AFFINE_FUSED), dfq_i8_affine_conv_observed (Out::AFFINE_OBSERVED) and
// dfq_i8_affine_conv_layout (Out::AFFINE_LAYOUT: o NULL or observed's, the layout l)
template <Out OUT>
int affine_conv_epilogue(const char* who, const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                         const DfqI8Affine* k, const float* bias, const DfqI8AffineEpilogue* e, const DfqI8AffineObserve* o,
                         const DfqI8AffineLayout* l, const DfqI8Conv* g, void* stream) {
  if (int rc = check_affine_conv(who, g, xq, S_in, wq, table, k, e)) return rc;
  DFQ_REQUIRE_WHO(e->y || e->yq, "no output requested (y and yq are both NULL)");
  DFQ_REQUIRE_WHO(!e->S || e->yq, "S is the sum of the codes; it needs yq");
  DFQ_REQUIRE_WHO(aligned16(e->yq), "yq must be 16-byte aligned");
  DFQ_REQUIRE_WHO(((uintptr_t)e->residual & 3) == 0 && ((uintptr_t)e->y & 3) == 0 && ((uintptr_t)e->S & 3) == 0,
                  "residual, y and S must be 4-byte aligned");
  DFQ_REQUIRE_WHO(ordered(e->pre_lo, e->pre_hi) && ordered(e->post_lo, e->post_hi),
                  "pre / post clamp bounds must be ordered and not NaN");
  QuantScalars qs{};
  if (e->yq) {                                                  // the consumer's quantizer, as dfq_i8_affine_quantize
    if (int rc = quantizer(who, "out_bits", "the output range", e->out_min, e->out_max, e->out_bits, &qs)) return rc;
  }
  const int cpad = (g->O + 15) / 16 * 16;
  const int64_t pixels = (int64_t)g->N * g->OH * g->OW;
  int64_t coff = 0, cstride = cpad;
  bool accumulate = false;
  if constexpr (OUT == Out::AFFINE_LAYOUT) {
    DFQ_REQUIRE_WHO(l != nullptr, "null layout descriptor");
    if (int rc = check_slice(who, l->coff, l->cstride, cpad, 'O')) return rc;
    DFQ_REQUIRE_WHO((l->S_accumulate == 0 || l->S_accumulate == 1) && (l->pad_code_on == 0 || l->pad_code_on == 1),
                    "S_accumulate and pad_code_on must be 0 or 1");
    DFQ_REQUIRE_WHO(!l->pad_code_on || (l->pad_code >= -128 && l->pad_code <= 127), "the pad code must be in [-128, 127]");
    coff = l->coff, cstride = l->cstride, accumulate = l->S_accumulate == 1;
  }
  int8_t* yq = e->yq ? e->yq + coff : nullptr;
  const int64_t y_bytes = pixels * g->O * (int64_t)sizeof(float), yq_bytes = (pixels - 1) * cstride + cpad;
  const int64_t s_bytes = pixels * 4;
  DFQ_REQUIRE_WHO(!overlap(e->residual, y_bytes, e->y, y_bytes) && !overlap(e->residual, y_bytes, yq, yq_bytes) &&
                      !overlap(e->residual, y_bytes, e->S, s_bytes),
                  "residual overlaps y, yq or S");
  DFQ_REQUIRE_WHO(!overlap(e->y, y_bytes, yq, yq_bytes) && !overlap(e->y, y_bytes, e->S, s_bytes) &&
                      !overlap(yq, yq_bytes, e->S, s_bytes),
                  "y, yq and S overlap");
  const bool dense = g->groups == 1;
  typename EpiOf<OUT>::type ep{};
  if constexpr (observed(OUT)) {
    DFQ_REQUIRE_WHO(OUT == Out::AFFINE_LAYOUT || o != nullptr, "null observer descriptor");
    if (o) {
      if (int rc = observer_scalars(who, "obs", o->obs_min, o->obs_max, o->obs_bits, &ep.obs, &ep.obs_on)) return rc;
      if (int rc = observer_scalars(who, "res", o->res_min, o->res_max, o->res_bits, &ep.res, &ep.res_on)) return rc;
      DFQ_REQUIRE_WHO(!ep.res_on || e->residual, "the residual's observer is on but there is no residual");
      DFQ_REQUIRE_WHO(ep.obs_on || ep.res_on, "both observers are off (dfq_i8_affine_conv_fused computes that)");
    }
  }
  // one writer per pixel of S: a dense layer whose 64-channel tile covers O, a depthwise one with one 16-channel chunk;
  // a concatenation's writers add into the S its caller zeroed
  const bool atomic = e->S && (accumulate || (dense ? g->O > BN : cpad > 16));
  cudaStream_t st = (cudaStream_t)stream;
  if (atomic && !accumulate) DFQ_CUDA(cudaMemsetAsync(e->S, 0, s_bytes, st));
  static_cast<Affine&>(ep) = Affine{S_in, table, k->kP, k->kA, k->kW, k->kN};
  ep.r = e->residual, ep.yq = yq, ep.S_out = e->S;
  ep.neg_min = qs.neg_min, ep.inv_scale = qs.inv_scale, ep.qmax = qs.qmax;
  ep.pre_lo = e->pre_lo, ep.pre_hi = e->pre_hi, ep.post_lo = e->post_lo, ep.post_hi = e->post_hi;
  ep.cpad = cpad, ep.S_atomic = atomic;
  if constexpr (OUT == Out::AFFINE_LAYOUT) {
    ep.cstride = (int)cstride, ep.pad_code = l->pad_code, ep.pad_on = l->pad_code_on;
    if (ep.pad_on) return launch_conv<OUT, true>(who, xq, wq, nullptr, bias, e->y, nullptr, g, ep, st);
  }
  return launch_conv<OUT>(who, xq, wq, nullptr, bias, e->y, nullptr, g, ep, st);
}

}  // namespace
}  // namespace dfq

extern "C" int dfq_i8_affine_conv_fused(const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                                        const DfqI8Affine* k, const float* bias, const DfqI8AffineEpilogue* e,
                                        const DfqI8Conv* g, void* stream) {
  return affine_conv_epilogue<Out::AFFINE_FUSED>("dfq_i8_affine_conv_fused", xq, S_in, wq, table, k, bias, e, nullptr,
                                                 nullptr, g, stream);
}

extern "C" int dfq_i8_affine_conv_observed(const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                                           const DfqI8Affine* k, const float* bias, const DfqI8AffineEpilogue* e,
                                           const DfqI8AffineObserve* o, const DfqI8Conv* g, void* stream) {
  return affine_conv_epilogue<Out::AFFINE_OBSERVED>("dfq_i8_affine_conv_observed", xq, S_in, wq, table, k, bias, e, o,
                                                    nullptr, g, stream);
}

extern "C" int dfq_i8_affine_conv_layout(const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                                         const DfqI8Affine* k, const float* bias, const DfqI8AffineEpilogue* e,
                                         const DfqI8AffineObserve* o, const DfqI8AffineLayout* l, const DfqI8Conv* g,
                                         void* stream) {
  return affine_conv_epilogue<Out::AFFINE_LAYOUT>("dfq_i8_affine_conv_layout", xq, S_in, wq, table, k, bias, e, o, l, g,
                                                  stream);
}

extern "C" int dfq_i8_affine_upsample_bilinear(const float* x, int8_t* yq, int32_t* S, const DfqI8AffineResize* g,
                                               void* stream) {
  const char* who = "dfq_i8_affine_upsample_bilinear";
  DFQ_REQUIRE(g != nullptr, "dfq_i8_affine_upsample_bilinear: null geometry");
  DFQ_REQUIRE(x != nullptr && yq != nullptr, "dfq_i8_affine_upsample_bilinear: null input or codes");
  DFQ_REQUIRE(g->N > 0 && g->C > 0 && g->H > 0 && g->W > 0 && g->OH > 0 && g->OW > 0,
              "dfq_i8_affine_upsample_bilinear: empty dimension (every size must be positive)");
  DFQ_REQUIRE(g->align_corners == 0 || g->align_corners == 1,
              "dfq_i8_affine_upsample_bilinear: align_corners must be 0 or 1");
  const int cpad = (g->C + 15) / 16 * 16;
  if (int rc = check_slice(who, g->coff, g->cstride, cpad, 'C')) return rc;
  DFQ_REQUIRE(aligned16(yq) && ((uintptr_t)x & 3) == 0 && ((uintptr_t)S & 3) == 0,
              "dfq_i8_affine_upsample_bilinear: yq must be 16-byte aligned, x and S 4-byte aligned");
  DFQ_REQUIRE(ordered(g->pre_lo, g->pre_hi) && ordered(g->post_lo, g->post_hi),
              "dfq_i8_affine_upsample_bilinear: pre / post clamp bounds must be ordered and not NaN");
  AffineResize a{};
  if (int rc = observer_scalars(who, "obs", g->obs_min, g->obs_max, g->obs_bits, &a.obs, &a.obs_on)) return rc;
  QuantScalars qs;
  if (int rc = quantizer(who, "out_bits", "the output range", g->out_min, g->out_max, g->out_bits, &qs)) return rc;
  const int64_t in_px = (int64_t)g->N * g->H * g->W, out_px = (int64_t)g->N * g->OH * g->OW;
  const int8_t* slice = yq + g->coff;
  const int64_t x_bytes = in_px * g->C * 4, slice_bytes = (out_px - 1) * g->cstride + cpad, s_bytes = out_px * 4;
  DFQ_REQUIRE(!overlap(x, x_bytes, slice, slice_bytes) && !overlap(x, x_bytes, S, s_bytes) &&
                  !overlap(slice, slice_bytes, S, s_bytes),
              "dfq_i8_affine_upsample_bilinear: x, the slice and S overlap");
  a.neg_min = qs.neg_min, a.inv_scale = qs.inv_scale, a.qmax = qs.qmax;
  a.pre_lo = g->pre_lo, a.pre_hi = g->pre_hi, a.post_lo = g->post_lo, a.post_hi = g->post_hi;
  const int64_t total = out_px * (cpad / 16);
  const bool ac = g->align_corners == 1;
  k_i8_affine_upsample<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      x, yq, S, *g, a, bilinear_scale(g->H, g->OH, ac), bilinear_scale(g->W, g->OW, ac), total);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_affine_maxpool(const int8_t* xq, const float* x, float* y, int8_t* yq, int32_t* S, float out_min,
                                     float out_max, int32_t out_bits, const DfqI8Pool* g, void* stream) {
  const char* who = "dfq_i8_affine_maxpool";
  if (int rc = check_pool(who, g, xq, x)) return rc;
  DFQ_REQUIRE_WHO(!S || yq, "S is the sum of the codes; it needs yq");
  DFQ_REQUIRE_WHO(((uintptr_t)S & 3) == 0, "S must be 4-byte aligned");
  const int64_t in_px = (int64_t)g->N * g->H * g->W, out_px = (int64_t)g->N * g->OH * g->OW;
  const int64_t yq_bytes = out_px * g->Cpad, s_bytes = out_px * 4;
  AffinePool a{S, 0.f, 0.f, 0.f};
  if (xq) {
    DFQ_REQUIRE_WHO(yq && !y, "codes in give codes out only (yq, no y)");
    DFQ_REQUIRE_WHO(aligned16(xq) && aligned16(yq), "xq and yq must be 16-byte aligned");
    const int64_t xq_bytes = in_px * g->Cpad;
    DFQ_REQUIRE_WHO(!overlap(xq, xq_bytes, yq, yq_bytes) && !overlap(xq, xq_bytes, S, s_bytes) &&
                        !overlap(yq, yq_bytes, S, s_bytes),
                    "xq, yq and S overlap");
  } else {
    DFQ_REQUIRE_WHO(y || yq, "no output requested (y and yq are both NULL)");
    DFQ_REQUIRE_WHO(aligned16(yq), "yq must be 16-byte aligned");
    DFQ_REQUIRE_WHO(((uintptr_t)x & 3) == 0 && ((uintptr_t)y & 3) == 0, "x and y must be 4-byte aligned");
    if (yq) {                                                   // the consumer's quantizer, as dfq_i8_affine_quantize
      QuantScalars qs;
      if (int rc = quantizer(who, "out_bits", "the output range", out_min, out_max, out_bits, &qs)) return rc;
      a.neg_min = qs.neg_min, a.inv_scale = qs.inv_scale, a.qmax = qs.qmax;
    }
    const int64_t x_bytes = in_px * g->C * 4, y_bytes = out_px * g->C * 4;
    DFQ_REQUIRE_WHO(!overlap(x, x_bytes, y, y_bytes) && !overlap(x, x_bytes, yq, yq_bytes) &&
                        !overlap(x, x_bytes, S, s_bytes) && !overlap(y, y_bytes, yq, yq_bytes) &&
                        !overlap(y, y_bytes, S, s_bytes) && !overlap(yq, yq_bytes, S, s_bytes),
                    "x, y, yq and S overlap");
  }
  const int64_t total = out_px * (g->Cpad / 16);
  cudaStream_t st = (cudaStream_t)stream;
  if (S) DFQ_CUDA(cudaMemsetAsync(S, 0, s_bytes, st));       // the chunks of a pixel add their sums
  if (xq) k_i8_maxpool<true, true><<<grid_for(total, 256), 256, 0, st>>>(xq, nullptr, nullptr, yq, 0.f, *g, total, a);
  else k_i8_maxpool<false, true><<<grid_for(total, 256), 256, 0, st>>>(nullptr, x, y, yq, 0.f, *g, total, a);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_affine_conv_rows(const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                                       const DfqI8Affine* k, const float* bias, const DfqI8AffineRows* r, const DfqI8Conv* g,
                                       void* stream) {
  const char* who = "dfq_i8_affine_conv_rows";
  if (int rc = check_affine_conv(who, g, xq, S_in, wq, table, k, r)) return rc;
  DFQ_REQUIRE_WHO(r->y, "no output (y is NULL)");
  DFQ_REQUIRE_WHO(((uintptr_t)r->y & 3) == 0, "y must be 4-byte aligned");
  DFQ_REQUIRE_WHO(ordered(r->pre_lo, r->pre_hi) && ordered(r->post_lo, r->post_hi),
                  "pre / post clamp bounds must be ordered and not NaN");
  const int64_t extent = (int64_t)g->OH * g->OW * g->O;                // floats of one image's rows
  DFQ_REQUIRE_WHO(r->off >= 0, "off must be non-negative");
  DFQ_REQUIRE_WHO(r->img_stride >= r->off + extent, "img_stride must be at least off + OH * OW * O");
  const int64_t x_bytes = (int64_t)g->N * g->H * g->W * g->Cpad, s_bytes = (int64_t)g->N * g->H * g->W * 4;
  const int64_t y_bytes = ((g->N - 1) * r->img_stride + extent) * (int64_t)sizeof(float);   // first to last row written
  DFQ_REQUIRE_WHO(!overlap(xq, x_bytes, r->y + r->off, y_bytes) && !overlap(S_in, s_bytes, r->y + r->off, y_bytes),
                  "y overlaps xq or S");
  AffineRows ep{};
  if (int rc = observer_scalars(who, "obs", r->obs_min, r->obs_max, r->obs_bits, &ep.obs, &ep.obs_on)) return rc;
  if (int rc = observer_scalars(who, "tail", r->tail_min, r->tail_max, r->tail_bits, &ep.tail, &ep.tail_on)) return rc;
  static_cast<Affine&>(ep) = Affine{S_in, table, k->kP, k->kA, k->kW, k->kN};
  ep.y = r->y, ep.off = r->off, ep.img_stride = r->img_stride;
  ep.pre_lo = r->pre_lo, ep.pre_hi = r->pre_hi, ep.post_lo = r->post_lo, ep.post_hi = r->post_hi;
  return launch_conv<Out::AFFINE_ROWS>(who, xq, wq, nullptr, bias, nullptr, nullptr, g, ep, (cudaStream_t)stream);
}

// The packed layout's geometry: a dense or depthwise layer of g (the packers read O, C, kh, kw, groups and Cpad)
static int check_codes(const char* who, const DfqI8Conv* g, const int8_t* a, const int8_t* b) {
  if (int rc = check_geometry(g)) return rc;
  DFQ_REQUIRE_WHO(a && b, "null pointer");
  const int64_t n_codes = (int64_t)g->O * (g->C / g->groups) * g->kh * g->kw;
  const int64_t n_packed = (int64_t)(g->groups == 1 ? g->O : 1) * g->kh * g->kw * g->Cpad;
  DFQ_REQUIRE_WHO(!overlap(a, n_codes, b, n_packed), "codes and packed overlap");
  return 0;
}

extern "C" int dfq_i8_pack_codes(const int8_t* codes, int8_t* packed, const DfqI8Conv* g, void* stream) {
  if (int rc = check_codes("dfq_i8_pack_codes", g, codes, packed)) return rc;
  const int taps = g->kh * g->kw;
  const bool dense = g->groups == 1;
  const int64_t total = (int64_t)(dense ? g->O : 1) * taps * g->Cpad;
  k_i8_pack_codes<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(codes, packed, g->C, taps, g->Cpad, dense, total);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_unpack_codes(const int8_t* packed, int8_t* codes, const DfqI8Conv* g, void* stream) {
  if (int rc = check_codes("dfq_i8_unpack_codes", g, codes, packed)) return rc;
  const int taps = g->kh * g->kw;
  const bool dense = g->groups == 1;
  const int64_t total = (int64_t)g->O * (g->C / g->groups) * taps;
  k_i8_unpack_codes<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(packed, codes, g->C / g->groups, taps, g->Cpad,
                                                                            dense, total);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_i8_plane_mean(const float* x, float* y, int8_t* yq, int64_t N, int32_t C, int64_t P, int32_t divide,
                                 float out_scale, void* stream) {
  const char* who = "dfq_i8_plane_mean";
  DFQ_REQUIRE_WHO(x != nullptr, "null input");
  DFQ_REQUIRE_WHO(y || yq, "no output requested (y and yq are both NULL)");
  DFQ_REQUIRE_WHO(N > 0 && C > 0 && P > 0, "empty dimension");
  DFQ_REQUIRE_WHO(divide == 0 || divide == 1, "divide must be 0 (multiply by fp32(1 / P)) or 1 (divide by P)");
  DFQ_REQUIRE_WHO(((uintptr_t)x & 3) == 0 && ((uintptr_t)y & 3) == 0, "x and y must be 4-byte aligned");
  DFQ_REQUIRE_WHO(aligned16(yq), "yq must be 16-byte aligned");
  DFQ_REQUIRE_WHO(!yq || (std::isfinite(out_scale) && out_scale >= 0.f),
                  "out_scale must be finite and non-negative when yq is written");
  DFQ_REQUIRE_WHO(N <= INT64_MAX / C / P / 4, "x is too large");
  const int cpad = (C + 15) / 16 * 16;
  const int64_t x_bytes = N * C * P * 4, y_bytes = N * C * 4, yq_bytes = N * cpad;
  DFQ_REQUIRE_WHO(!overlap(x, x_bytes, y, y_bytes) && !overlap(x, x_bytes, yq, yq_bytes) && !overlap(y, y_bytes, yq, yq_bytes),
                  "x, y and yq overlap");
  const int cols = yq ? cpad : C;
  const int64_t rows = N * cols;
  const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>((rows + PM_WARPS * 32 - 1) / (PM_WARPS * 32),
                                                                (int64_t)sm_count() * 8));
  k_i8_plane_mean<<<(unsigned)blocks, PM_WARPS * 32, 0, (cudaStream_t)stream>>>(x, y, yq, C, cols, P, rows, divide != 0,
                                                                                1.f / (float)P, out_scale);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}
