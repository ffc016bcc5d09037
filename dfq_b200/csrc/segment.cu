// Segmentation predictions and confusion counts on the device, fused with the final bilinear resize: the label map of
// torch.max(F.interpolate(logits, (OH, OW), mode="bilinear", align_corners=...), 1)[1] and the confusion matrix the
// reference's Evaluator (utils/metrics.py) builds from it, in one pass over the labels.  The full-resolution logits are
// never written: each output pixel reads the low-resolution planes through its two bilinear taps.
//
//   k_seg_argmax   one thread per output pixel (n, oh, ow), pixels fastest: the C resized values (bilinear.cuh), their
//                  argmax under torch's CUDA max(dim) rule, optionally the int64 prediction and, optionally, the pixel
//                  added to count[label][pred] in a per-CTA shared histogram of C * C uint32 that is flushed into the
//                  uint64 matrix with one 64-bit atomicAdd per non-zero bin.
#include <algorithm>

#include "bilinear.cuh"
#include "common.cuh"

namespace dfq {
namespace {

constexpr int kSegThreads = 256;
constexpr int kSegMaxClasses = 160;                  // C * C uint32 bins = 100 KB of shared memory
constexpr int64_t kSegMaxPixelsPerCta = 1ll << 31;   // a uint32 bin of one CTA cannot overflow

// The label of one pixel as the reference's Evaluator sees it after forward_all's astype(np.uint8), or -1 when the mask
// (0 <= gt < C) drops it.  uint8 / int64: the value itself.  float32: truncated toward zero (astype's cast) when
// -1 < v < 256, where numpy's cast is defined; NaN and every other value are dropped.
template <int LT>
__device__ __forceinline__ int seg_label(const void* labels, int64_t i, int C) {
  if (LT == DFQ_SEG_LABEL_U8) {
    const int v = __ldg((const uint8_t*)labels + i);
    return v < C ? v : -1;
  } else if (LT == DFQ_SEG_LABEL_I64) {
    const int64_t v = __ldg((const long long*)labels + i);
    return v >= 0 && v < C ? (int)v : -1;
  } else {
    const float v = __ldg((const float*)labels + i);
    if (!(v > -1.f && v < 256.f)) return -1;
    const int t = (int)v;
    return t < C ? t : -1;
  }
}

// torch's CUDA max(dim) (GreaterOrNan, ATen/native/SharedReduceOps.h) as a scan over c ascending: the first NaN wins over
// everything, otherwise a strictly larger value replaces the best, so equal values (-0.0 and +0.0 included) keep the lower
// index.
template <int LT, bool PRED, bool COUNT>
__global__ void __launch_bounds__(kSegThreads) k_seg_argmax(const float* __restrict__ x, const void* __restrict__ labels,
                                                            int64_t* __restrict__ pred,
                                                            unsigned long long* __restrict__ count, DfqSegArgmax d,
                                                            float scale_h, float scale_w, int64_t total) {
  extern __shared__ uint32_t hist[];
  const int C = d.C;
  if (COUNT) {
    for (int b = threadIdx.x; b < C * C; b += blockDim.x) hist[b] = 0;
    __syncthreads();
  }
  const int64_t HW = (int64_t)d.H * d.W, OHW = (int64_t)d.OH * d.OW;
  const bool copy = d.H == d.OH && d.W == d.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / OHW, p = i - n * OHW;
    const int oh = (int)(p / d.OW), ow = (int)(p - (int64_t)oh * d.OW);
    const BilinearTap th = bilinear_tap(oh, scale_h, d.align_corners, d.H);
    const BilinearTap tw = bilinear_tap(ow, scale_w, d.align_corners, d.W);
    const float* img = x + n * C * HW;
    float best = bilinear_value(img, d.W, oh, ow, th, tw, copy);
    int arg = 0;
    for (int c = 1; c < C; ++c) {
      const float v = bilinear_value(img + c * HW, d.W, oh, ow, th, tw, copy);
      if (best == best && (v != v || v > best)) {
        best = v;
        arg = c;
      }
    }
    if (PRED) pred[i] = arg;
    if (COUNT) {
      const int gt = seg_label<LT>(labels, i, C);
      if (gt >= 0) atomicAdd(&hist[gt * C + arg], 1u);
    }
  }
  if (COUNT) {
    __syncthreads();
    for (int b = threadIdx.x; b < C * C; b += blockDim.x)
      if (hist[b]) atomicAdd(count + b, (unsigned long long)hist[b]);
  }
}

// [a, a + na) and [b, b + nb) share a byte; a NULL range shares none
bool overlap(const void* a, int64_t na, const void* b, int64_t nb) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return a && b && x < y + (uintptr_t)nb && y < x + (uintptr_t)na;
}

// a * b * c when it is below 2^62, else -1
int64_t product(int64_t a, int64_t b, int64_t c) {
  const double p = (double)a * (double)b * (double)c;
  return p < 4.6e18 ? a * b * c : -1;
}

template <int LT, bool PRED, bool COUNT>
int launch(const float* x, const void* labels, int64_t* pred, uint64_t* count, const DfqSegArgmax& d, int64_t total,
           cudaStream_t st) {
  auto kern = k_seg_argmax<LT, PRED, COUNT>;
  const size_t smem = COUNT ? sizeof(uint32_t) * d.C * d.C : 0;
  int per_sm = 1;
  if (smem > 48 * 1024) DFQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  DFQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kSegThreads, smem));
  // a grid the device holds at once (each CTA zeroes and flushes its histogram once), but enough CTAs that none handles
  // more than kSegMaxPixelsPerCta pixels
  const int64_t want = (total + kSegThreads - 1) / kSegThreads;
  int64_t grid = std::min<int64_t>(want, (int64_t)sm_count() * std::max(per_sm, 1));
  const int64_t per_cta = kSegMaxPixelsPerCta / kSegThreads * kSegThreads;
  grid = std::max<int64_t>(grid, (total + per_cta - 1) / per_cta);
  if (grid > INT32_MAX) {
    set_error("dfq_seg_argmax: %lld pixels need more than 2^31 - 1 CTAs", (long long)total);
    return DFQ_E_UNSUPPORTED;
  }
  const bool ac = d.align_corners != 0;
  kern<<<(int)grid, kSegThreads, smem, st>>>(x, labels, pred, (unsigned long long*)count, d,
                                             bilinear_scale(d.H, d.OH, ac), bilinear_scale(d.W, d.OW, ac), total);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

template <bool PRED>
int launch_counted(const float* x, const void* labels, int64_t* pred, uint64_t* count, const DfqSegArgmax& d,
                   int64_t total, cudaStream_t st) {
  switch (d.label_type) {
    case DFQ_SEG_LABEL_U8: return launch<DFQ_SEG_LABEL_U8, PRED, true>(x, labels, pred, count, d, total, st);
    case DFQ_SEG_LABEL_I64: return launch<DFQ_SEG_LABEL_I64, PRED, true>(x, labels, pred, count, d, total, st);
    default: return launch<DFQ_SEG_LABEL_F32, PRED, true>(x, labels, pred, count, d, total, st);
  }
}

}  // namespace
}  // namespace dfq

using namespace dfq;

extern "C" int dfq_seg_argmax(const float* logits, const void* labels, int64_t* pred, uint64_t* count,
                              const DfqSegArgmax* d, void* stream) {
  const char* who = "dfq_seg_argmax";
  if (!d) { set_error("%s: descriptor is NULL", who); return DFQ_E_ARG; }
  if (d->N < 1 || d->C < 1 || d->H < 1 || d->W < 1 || d->OH < 1 || d->OW < 1) {
    set_error("%s: N, C, H, W, OH and OW must be positive, got %d, %d, %d, %d, %d, %d", who, d->N, d->C, d->H, d->W,
              d->OH, d->OW);
    return DFQ_E_ARG;
  }
  if (d->align_corners != 0 && d->align_corners != 1) {
    set_error("%s: align_corners must be 0 or 1, got %d", who, d->align_corners);
    return DFQ_E_ARG;
  }
  if (d->label_type != DFQ_SEG_LABEL_U8 && d->label_type != DFQ_SEG_LABEL_I64 && d->label_type != DFQ_SEG_LABEL_F32) {
    set_error("%s: unknown label_type %d", who, d->label_type);
    return DFQ_E_ARG;
  }
  if (d->C > kSegMaxClasses) {
    set_error("%s: C = %d is above the limit %d", who, d->C, kSegMaxClasses);
    return DFQ_E_UNSUPPORTED;
  }
  const int64_t total = product(d->N, d->OH, d->OW), in = product((int64_t)d->N * d->C, d->H, d->W);
  if (total < 0 || in < 0) { set_error("%s: the tensors have 2^62 elements or more", who); return DFQ_E_UNSUPPORTED; }
  if (!logits) { set_error("%s: logits is NULL", who); return DFQ_E_ARG; }
  if ((labels == nullptr) != (count == nullptr)) {
    set_error("%s: labels and count must both be given or both be NULL", who);
    return DFQ_E_ARG;
  }
  if (!pred && !count) { set_error("%s: neither pred nor count is given", who); return DFQ_E_ARG; }
  const int lsize = d->label_type == DFQ_SEG_LABEL_U8 ? 1 : d->label_type == DFQ_SEG_LABEL_I64 ? 8 : 4;
  if (((uintptr_t)logits & 3) || ((uintptr_t)pred & 7) || ((uintptr_t)count & 7) ||
      ((uintptr_t)labels & (lsize - 1))) {
    set_error("%s: misaligned pointer (logits 4, pred 8, count 8, labels %d bytes)", who, lsize);
    return DFQ_E_ARG;
  }
  const int64_t nx = 4 * in, nl = labels ? lsize * total : 0, np = pred ? 8 * total : 0, nc = 8ll * d->C * d->C;
  if (overlap(count, nc, logits, nx) || overlap(count, nc, labels, nl) || overlap(count, nc, pred, np) ||
      overlap(pred, np, logits, nx) || overlap(pred, np, labels, nl)) {
    set_error("%s: count and pred must not overlap the other buffers", who);
    return DFQ_E_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (!count) return launch<DFQ_SEG_LABEL_U8, true, false>(logits, nullptr, pred, nullptr, *d, total, st);
  return pred ? launch_counted<true>(logits, labels, pred, count, *d, total, st)
              : launch_counted<false>(logits, labels, nullptr, count, *d, total, st);
}
