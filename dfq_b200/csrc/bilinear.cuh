// torch's CUDA bilinear resize (upsample_bilinear2d_out_frame<float, float>) for one output element, shared by the int8
// upsample kernels (int8_conv.cu) and the segmentation argmax (segment.cu).
#pragma once
#include "common.cuh"

namespace dfq {

// torch compiles upsample_bilinear2d_out_frame with contraction on; its sm_90 SASS (torch 2.11) is, per axis and per
// element:
//   src = align_corners ? FMUL(dst, scale) : FFMA(FADD(dst, 0.5), scale, -0.5), then src < 0 ? 0 : src (NaN kept)
//   i   = F2I.TRUNC(src), l1 = FADD(src, -i), l0 = FADD(1, -l1), i + 1 only while i < in - 1
//   row = FFMA(w_l0, x[h][w_i], FMUL(w_l1, x[h][w_i + w_p]))             for h = h_i and h_i + h_p
//   y   = FFMA(h_l0, row(h_i), FMUL(h_l1, row(h_i + h_p)))
// The library builds with --fmad=false, so the same operations are spelled out with __fmaf_rn / __fmul_rn / __fadd_rn.
// An unchanged size is torch's plain copy (0 * inf and -0.0 + 0.0 would make the formula differ from x).
struct BilinearTap {
  int i0, i1;
  float l0, l1;
};

__device__ __forceinline__ BilinearTap bilinear_tap(int dst, float scale, bool align_corners, int in) {
  float src = align_corners ? __fmul_rn((float)dst, scale) : __fmaf_rn(__fadd_rn((float)dst, 0.5f), scale, -0.5f);
  if (!align_corners) src = src < 0.f ? 0.f : src;
  BilinearTap t;
  t.i0 = (int)src;
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  t.l1 = __fadd_rn(src, -(float)t.i0);
  t.l0 = __fadd_rn(1.f, -t.l1);
  return t;
}

// torch's output at (oh, ow) of one channel plane img [H, W] (copy: the size does not change)
__device__ __forceinline__ float bilinear_value(const float* img, int W, int oh, int ow, const BilinearTap& th,
                                                const BilinearTap& tw, bool copy) {
  if (copy) return __ldg(img + (int64_t)oh * W + ow);
  const float* r0 = img + (int64_t)th.i0 * W;
  const float* r1 = img + (int64_t)th.i1 * W;
  const float a = __fmaf_rn(tw.l0, __ldg(r0 + tw.i0), __fmul_rn(tw.l1, __ldg(r0 + tw.i1)));
  const float b = __fmaf_rn(tw.l0, __ldg(r1 + tw.i0), __fmul_rn(tw.l1, __ldg(r1 + tw.i1)));
  return __fmaf_rn(th.l0, a, __fmul_rn(th.l1, b));
}

// torch's area_pixel_compute_scale<float> without a scale_factor, formed on the host as torch forms it
inline float bilinear_scale(int in, int out, bool align_corners) {
  if (align_corners) return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
  return (float)in / (float)out;
}

}  // namespace dfq
