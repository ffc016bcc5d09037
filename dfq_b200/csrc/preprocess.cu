// Evaluation preprocessing on the device: the reference's resize, crop and normalisation of decoded uint8 RGB images, bit
// for bit Pillow's BILINEAR / NEAREST resize (classification and segmentation) and OpenCV's INTER_LINEAR (SSD), for a batch
// of images of mixed sizes in one launch.
//
//   k_pre_resample   one CTA per (image, tile of kTileH x kTileW output pixels after the crop): pixels that are cropped
//                    away are never computed.  The source rows the tile's row taps reach are taken kChunk at a time; the
//                    horizontal pass of a chunk (every row x the tile's columns x 3 channels) goes into shared memory, and
//                    each thread adds the chunk's share of its pixel's vertical taps to three integer accumulators.  Both
//                    libraries' vertical steps are a sum of one term per tap, so the chunking changes no result.  The
//                    normalised value is written NCHW float32, and the label plane, when there is one, by the same thread.
//
// The tap tables (per output coordinate: K {source index, weight} pairs) are built on the host and travel in the batch
// blob with the pixels.  Horizontal taps read the source through the read-only cache: neighbouring output columns share
// all but one or two of their taps, so the tile's source bytes come from DRAM once.
#include <algorithm>

#include "common.cuh"

namespace dfq {
namespace {

constexpr int kTileW = 32;                 // one warp per output row: coalesced NCHW stores
constexpr int kTileH = 8;
constexpr int kPreThreads = kTileW * kTileH;
constexpr int kChunk = 32;                 // source rows of the horizontal pass held in shared memory at once
constexpr int kMaxTaps = 4096;

// Pillow's ImagingResampleHorizontal/Vertical_8bpc: ss = 1 << 21 + sum, clip8(ss >> 22).  OpenCV's HResizeLinear keeps
// the int32 sum.
template <int F>
__device__ __forceinline__ int h_pass(const uint8_t* __restrict__ row, const int2* __restrict__ taps, int K, int c) {
  int s = F == DFQ_PRE_PIL_BILINEAR ? 1 << 21 : 0;
  for (int k = 0; k < K; ++k) {
    const int2 t = __ldg(taps + k);
    s += (int)__ldg(row + 3 * t.x + c) * t.y;
  }
  return F == DFQ_PRE_PIL_BILINEAR ? min(max(s >> 22, 0), 255) : s;
}

// One vertical tap.  Pillow: the product, with the 1 << 21 start and >> 22 at the end.  OpenCV's VResizeLinearVec_32s8u:
// v_mul_hi of (S >> 4) and the int16 coefficient, summed, then (sum + 2) >> 2 saturated.
template <int F>
__device__ __forceinline__ int v_term(int s, int w) {
  return F == DFQ_PRE_PIL_BILINEAR ? s * w : ((s >> 4) * w) >> 16;
}

template <int F>
__device__ __forceinline__ float v_final(int acc) {
  return (float)(F == DFQ_PRE_PIL_BILINEAR ? min(max((acc + (1 << 21)) >> 22, 0), 255) : min(max((acc + 2) >> 2, 0), 255));
}

__device__ __forceinline__ float normalise(float u, int c, const DfqPreResample& d) {
  if (d.norm == DFQ_PRE_NORM_F32) return __fdiv_rn(__fsub_rn(__fdiv_rn(u, 255.f), d.mean[c]), d.std[c]);
  if (d.norm == DFQ_PRE_NORM_F64) {
    const float t = __fdiv_rn(u, 255.f);
    const float m = __double2float_rn(__dsub_rn((double)t, d.mean64[c]));
    return __double2float_rn(__ddiv_rn((double)m, d.std64[c]));
  }
  return __fdiv_rn(__fsub_rn(u, d.mean[c]), d.std[c]);
}

template <int F>
__global__ void __launch_bounds__(kPreThreads) k_pre_resample(const DfqPreResample d, const DfqPreImage* __restrict__ imgs,
                                                              const uint8_t* __restrict__ blob, float* __restrict__ out,
                                                              float* __restrict__ labels) {
  __shared__ int inter[kChunk][kTileW][3];
  const DfqPreImage im = imgs[blockIdx.y];
  const int tiles_x = (d.out_w + kTileW - 1) / kTileW;
  const int x0 = (blockIdx.x % tiles_x) * kTileW, y0 = (blockIdx.x / tiles_x) * kTileH;
  const int tx = threadIdx.x % kTileW, ty = threadIdx.x / kTileW;
  const int x = x0 + tx, y = y0 + ty;
  const bool live = x < d.out_w && y < d.out_h;
  const int xe = min(kTileW, d.out_w - x0);                       // live columns of the tile
  const int ylast = min(y0 + kTileH, d.out_h) - 1;
  const uint8_t* src = blob + im.src;
  const int2* xt = (const int2*)(blob + im.xtap);
  const int2* yt = (const int2*)(blob + im.ytap);
  // the source rows the tile's row taps reach: ascending within and across coordinates
  const int r_lo = __ldg(yt + (int64_t)y0 * im.yk).x, r_hi = __ldg(yt + (int64_t)ylast * im.yk + im.yk - 1).x + 1;
  const int2* my_taps = yt + (int64_t)min(y, d.out_h - 1) * im.yk;
  int acc[3] = {0, 0, 0};
  for (int r0 = r_lo; r0 < r_hi; r0 += kChunk) {
    const int rows = min(kChunk, r_hi - r0);
    for (int i = threadIdx.x; i < rows * xe; i += kPreThreads) {
      const int r = i / xe, cx = i % xe;
      const uint8_t* row = src + (int64_t)(r0 + r) * im.W * 3;
      const int2* taps = xt + (int64_t)(x0 + cx) * im.xk;
#pragma unroll
      for (int c = 0; c < 3; ++c) inter[r][cx][c] = h_pass<F>(row, taps, im.xk, c);
    }
    __syncthreads();
    if (live) {
      for (int k = 0; k < im.yk; ++k) {
        const int2 t = __ldg(my_taps + k);
        const int r = t.x - r0;
        if (r < 0 || r >= rows) continue;
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += v_term<F>(inter[r][tx][c], t.y);
      }
    }
    __syncthreads();
  }
  if (!live) return;
  const int64_t plane = (int64_t)d.out_h * d.out_w, pix = (int64_t)y * d.out_w + x;
  float* o = out + (int64_t)blockIdx.y * 3 * plane + pix;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * plane] = normalise(v_final<F>(acc[c]), c, d);
  if (im.label >= 0) {
    const int sy = __ldg((const int*)(blob + im.ynear) + y), sx = __ldg((const int*)(blob + im.xnear) + x);
    labels[(int64_t)blockIdx.y * plane + pix] = (float)__ldg(blob + im.label + (int64_t)sy * im.W + sx);
  }
}

// A table of `count` elements of `elem` bytes at byte offset `off`, inside the blob and aligned to `align`.
bool in_blob(int64_t off, int64_t count, int64_t elem, int64_t align, int64_t bytes) {
  return off >= 0 && off % align == 0 && count >= 0 && count <= (bytes - off) / elem;
}

}  // namespace
}  // namespace dfq

using namespace dfq;

extern "C" int dfq_pre_resample(const DfqPreResample* d, const DfqPreImage* images, const void* blob, float* out,
                                float* labels, void* stream) {
  if (!d || !images || !blob || !out) {
    set_error("dfq_pre_resample: d, images, blob and out must be non-NULL");
    return DFQ_E_ARG;
  }
  if (d->n < 1 || d->n > 65535 || d->out_h < 1 || d->out_w < 1 || d->blob_bytes < 1 ||
      (d->filter != DFQ_PRE_PIL_BILINEAR && d->filter != DFQ_PRE_CV_LINEAR) || d->norm < DFQ_PRE_NORM_F32 ||
      d->norm > DFQ_PRE_NORM_SUB_DIV) {
    set_error("dfq_pre_resample: n must be in 1 .. 65535, out_h, out_w and blob_bytes at least 1, filter and norm known "
              "(n %d, out %d x %d, blob %lld, filter %d, norm %d)", d->n, d->out_h, d->out_w, (long long)d->blob_bytes,
              d->filter, d->norm);
    return DFQ_E_ARG;
  }
  for (int c = 0; c < 3; ++c)
    if (d->norm == DFQ_PRE_NORM_F64 ? d->std64[c] == 0.0 : d->std[c] == 0.f) {
      set_error("dfq_pre_resample: std[%d] is zero", c);
      return DFQ_E_ARG;
    }
  const int64_t B = d->blob_bytes;
  int with_label = 0;
  for (int i = 0; i < d->n; ++i) {
    const DfqPreImage& m = images[i];
    const bool ok = m.H >= 1 && m.W >= 1 && m.xk >= 1 && m.xk <= kMaxTaps && m.yk >= 1 && m.yk <= kMaxTaps &&
                    in_blob(m.src, (int64_t)m.H * m.W * 3, 1, 1, B) &&
                    in_blob(m.xtap, (int64_t)d->out_w * m.xk, 8, 8, B) && in_blob(m.ytap, (int64_t)d->out_h * m.yk, 8, 8, B) &&
                    (m.label < 0 ? m.xnear < 0 && m.ynear < 0
                                 : in_blob(m.label, (int64_t)m.H * m.W, 1, 1, B) && in_blob(m.xnear, d->out_w, 4, 4, B) &&
                                       in_blob(m.ynear, d->out_h, 4, 4, B));
    if (!ok) {
      set_error("dfq_pre_resample: image %d: size %d x %d, taps %d / %d (1 .. %d), or a table outside the %lld-byte blob "
                "or misaligned", i, m.H, m.W, m.xk, m.yk, kMaxTaps, (long long)B);
      return DFQ_E_ARG;
    }
    with_label += m.label >= 0;
  }
  if (!(with_label == 0 && !labels) && !(with_label == d->n && labels)) {
    set_error("dfq_pre_resample: %d of %d images have a label, labels pointer %s", with_label, d->n,
              labels ? "given" : "NULL");
    return DFQ_E_ARG;
  }
  if ((uintptr_t)blob % 8 || (uintptr_t)out % 4 || (uintptr_t)labels % 4) {
    set_error("dfq_pre_resample: blob must be 8-byte aligned, out and labels 4-byte aligned");
    return DFQ_E_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  TablePack tp;
  const int iI = tp.add(images, d->n);
  if (int rc = tp.upload(st)) return rc;
  const dim3 grid(((d->out_w + kTileW - 1) / kTileW) * ((d->out_h + kTileH - 1) / kTileH), d->n);
  if (d->filter == DFQ_PRE_PIL_BILINEAR)
    k_pre_resample<DFQ_PRE_PIL_BILINEAR><<<grid, kPreThreads, 0, st>>>(*d, tp.ptr<DfqPreImage>(iI), (const uint8_t*)blob,
                                                                        out, labels);
  else
    k_pre_resample<DFQ_PRE_CV_LINEAR><<<grid, kPreThreads, 0, st>>>(*d, tp.ptr<DfqPreImage>(iI), (const uint8_t*)blob, out,
                                                                     labels);
  DFQ_CUDA(cudaGetLastError());
  tp.release(st);
  return 0;
}
