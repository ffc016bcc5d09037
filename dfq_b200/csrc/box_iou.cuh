// box_utils.iou_of (utils/detection/box_utils.py) for one pair of corner-form boxes, in the reference's fp32 op order.
// Shared by the SSD post-processing (detect.cu) and the VOC average precision (detect_map.cu).
#pragma once
#include <cuda_runtime.h>

namespace dfq {

// torch.maximum / torch.minimum / clamp(min=0): NaN in, NaN out
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }
__device__ __forceinline__ float nan_min(float a, float b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ float clamp0(float a) { return a < 0.f ? 0.f : a; }

// box_utils.iou_of(r, c) for one pair, in the reference's op order: r's area first in the denominator
__device__ __forceinline__ float iou_of(const float4 r, const float4 c) {
  const float ow = clamp0(nan_min(r.z, c.z) - nan_max(r.x, c.x));
  const float oh = clamp0(nan_min(r.w, c.w) - nan_max(r.y, c.y));
  const float ov = ow * oh;
  const float a0 = clamp0(r.z - r.x) * clamp0(r.w - r.y);
  const float a1 = clamp0(c.z - c.x) * clamp0(c.w - c.y);
  return ov / (((a0 + a1) - ov) + 1e-5f);
}

}  // namespace dfq
