// SSD post-processing on the device: box decoding, per-class hard NMS and the flat per-image output of the reference's
// Predictor.predict (modeling/detection/predictor.py, utils/detection/box_utils.py), for a whole batch at once.
//
//   k_ssd_decode    one thread per (image, prior): convert_locations_to_boxes + center_form_to_corner_form, each fp32 op
//                   separately rounded in the reference's order (the library builds with --fmad=false; expf compiles to
//                   the same instructions with and without contraction, so it is torch's CUDA exp).
//   k_ssd_nms       one CTA per (image, foreground class): radix select of the candidate_size best candidates, bitonic
//                   sort, the suppression bitmask from the decoded boxes, then the greedy scan in one warp.
//   k_ssd_scan      one CTA: exclusive scan of the per-(image, class) pick counts.
//   k_ssd_compact   one CTA per (image, class): the picks into the flat outputs, scaled by the image sizes, with labels.
#include <algorithm>

#include <cub/block/block_scan.cuh>

#include "box_iou.cuh"
#include "common.cuh"

namespace dfq {
namespace {

constexpr int kNmsThreads = 256;
constexpr int kMaxCandidates = 1024;   // the greedy scan keeps one 32-bit word of the removed set per lane
constexpr int kScanThreads = 256;

__global__ void __launch_bounds__(256) k_ssd_decode(const float4* __restrict__ loc, const float4* __restrict__ priors,
                                                    float4* __restrict__ boxes, int64_t N, int64_t P, int prior_batch,
                                                    float cv, float sv) {
  const int64_t total = N * P;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 l = loc[i];
    const float4 p = priors[prior_batch == 1 ? i % P : i];
    const float cx = (l.x * cv) * p.z + p.x;
    const float cy = (l.y * cv) * p.w + p.y;
    const float w = expf(l.z * sv) * p.z;
    const float h = expf(l.w * sv) * p.w;
    const float hw = w * 0.5f, hh = h * 0.5f;   // torch divides by a CPU scalar as a multiply by its reciprocal
    boxes[i] = make_float4(cx - hw, cy - hh, cx + hw, cy + hh);
  }
}

// Order key of a candidate: the score's bits made unsigned-orderable (-0.0 folded onto +0.0), then P-1-index so that among
// equal scores the lower prior index is the larger key.  Keys are unique and never 0 (NaN is never a candidate).
__device__ __forceinline__ bool cand_key(float v, float thr, int64_t i, int64_t P, uint64_t* key) {
  if (!(v > thr)) return false;
  uint32_t u = __float_as_uint(v);
  if (u == 0x80000000u) u = 0;
  const uint32_t ord = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  *key = ((uint64_t)ord << 32) | (uint32_t)(P - 1 - i);
  return true;
}

// Dynamic shared memory of k_ssd_nms for K candidates: keys (a power of two, at least 2 so that the boxes after them are
// 16-byte aligned), boxes, mask rows of ceil(K/32) words.
__host__ __device__ inline int pow2_at_least(int k) {
  int p = 2;
  while (p < k) p <<= 1;
  return p;
}
inline size_t nms_smem(int K) {
  return sizeof(uint64_t) * pow2_at_least(K) + sizeof(float4) * K + sizeof(uint32_t) * (size_t)K * ((K + 31) / 32);
}

__global__ void __launch_bounds__(kNmsThreads) k_ssd_nms(const float* __restrict__ scores, const float4* __restrict__ boxes,
                                                        float4* __restrict__ slot_boxes, float* __restrict__ slot_probs,
                                                        int32_t* __restrict__ counts, int64_t P, int C, float thr,
                                                        float iou_thr, int K, int top_k) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int Kp = pow2_at_least(K);
  uint64_t* keys = (uint64_t*)smem;
  float4* bx = (float4*)(keys + Kp);
  uint32_t* mask = (uint32_t*)(bx + K);
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_count, s_digit, s_need, s_done;

  const int seg = blockIdx.x;                       // n * (C - 1) + (c - 1)
  const int64_t n = seg / (C - 1);
  const int c = seg % (C - 1) + 1;
  const float* s = scores + n * P * C + c;
  const int tid = threadIdx.x;

  if (tid == 0) s_count = 0;
  __syncthreads();
  uint32_t mine = 0;
  for (int64_t i = tid; i < P; i += blockDim.x) {
    uint64_t key;
    mine += cand_key(s[i * C], thr, i, P, &key);
  }
  atomicAdd(&s_count, mine);
  __syncthreads();
  const uint32_t n_cand = s_count;

  // MSB-first radix select over the 64-bit keys: afterwards the candidates kept are those whose key, shifted right by
  // `shift`, is at least prefix >> shift - exactly min(n_cand, K) of them.
  uint64_t prefix = 0;
  int shift = 64;
  if (n_cand > (uint32_t)K) {
    if (tid == 0) s_need = K;
    while (true) {
      shift -= 8;
      for (int d = tid; d < 256; d += blockDim.x) hist[d] = 0;
      __syncthreads();
      for (int64_t i = tid; i < P; i += blockDim.x) {
        uint64_t key;
        if (cand_key(s[i * C], thr, i, P, &key) && (shift == 56 || ((key ^ prefix) >> (shift + 8)) == 0))
          atomicAdd(&hist[(key >> shift) & 255], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        uint32_t need = s_need, above = 0;
        int d = 255;
        for (; d > 0 && above + hist[d] < need; --d) above += hist[d];
        s_digit = d;
        s_need = need - above;
        s_done = hist[d] == need - above;
      }
      __syncthreads();
      prefix |= (uint64_t)s_digit << shift;
      if (s_done) break;
      __syncthreads();
    }
  }
  if (tid == 0) s_count = 0;
  __syncthreads();
  for (int64_t i = tid; i < P; i += blockDim.x) {
    uint64_t key;
    if (cand_key(s[i * C], thr, i, P, &key) && (shift == 64 || (key >> shift) >= (prefix >> shift)))
      keys[atomicAdd(&s_count, 1u)] = key;
  }
  __syncthreads();
  const int m = (int)s_count;
  for (int i = m + tid; i < Kp; i += blockDim.x) keys[i] = 0;

  // bitonic sort, descending
  for (int k = 2; k <= Kp; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int i = tid; i < Kp; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const uint64_t a = keys[i], b = keys[l];
          if (((i & k) == 0) == (a < b)) { keys[i] = b; keys[l] = a; }
        }
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < m; i += blockDim.x) bx[i] = boxes[n * P + (P - 1 - (int64_t)(uint32_t)keys[i])];
  __syncthreads();

  // mask[i][w] bit b: candidate 32w + b (> i) is dropped when i is picked, i.e. !(iou_of(it, i) <= iou_thr)
  const int W = (m + 31) / 32;
  for (int t = tid; t < m * W; t += blockDim.x) {
    const int i = t / W, w = t % W;
    uint32_t bits = 0;
    if (32 * w + 31 > i) {
      const float4 cur = bx[i];
      const int j1 = min(32 * w + 32, m);
      for (int j = max(32 * w, i + 1); j < j1; ++j)
        if (!(iou_of(bx[j], cur) <= iou_thr)) bits |= 1u << (j - 32 * w);
    }
    mask[t] = bits;
  }
  __syncthreads();

  // greedy scan: lane l holds word l of the removed set
  if (tid < 32) {
    uint32_t removed = 0;
    int picked = 0;
    const int64_t slot0 = (int64_t)seg * K;
    for (int i = 0; i < m; ++i) {
      const uint32_t word = __shfl_sync(0xffffffffu, removed, i >> 5);
      if ((word >> (i & 31)) & 1u) continue;
      if (tid == 0) {
        slot_boxes[slot0 + picked] = bx[i];
        slot_probs[slot0 + picked] = s[(P - 1 - (int64_t)(uint32_t)keys[i]) * C];
      }
      ++picked;
      if (top_k > 0 && picked == top_k) break;
      if (tid < W) removed |= mask[i * W + tid];
    }
    if (tid == 0) counts[seg] = picked;
  }
}

__global__ void __launch_bounds__(kScanThreads) k_ssd_scan(const int32_t* __restrict__ counts, int64_t* __restrict__ offs,
                                                          int S) {
  using Scan = cub::BlockScan<long long, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const int per = (S + kScanThreads - 1) / kScanThreads;
  const int b = threadIdx.x * per, e = min(b + per, S);
  long long sum = 0;
  for (int i = b; i < e; ++i) sum += counts[i];
  long long run, total;
  Scan(tmp).ExclusiveSum(sum, run, total);
  for (int i = b; i < e; ++i) {
    offs[i] = run;
    run += counts[i];
  }
  if (threadIdx.x == 0) offs[S] = total;
}

__global__ void __launch_bounds__(128) k_ssd_compact(const float4* __restrict__ slot_boxes,
                                                    const float* __restrict__ slot_probs,
                                                    const int32_t* __restrict__ counts, const int64_t* __restrict__ offs,
                                                    const float* __restrict__ sizes, float4* __restrict__ out_boxes,
                                                    int64_t* __restrict__ out_labels, float* __restrict__ out_probs,
                                                    int C, int K) {
  const int seg = blockIdx.x;
  const int n = seg / (C - 1);
  const int64_t label = seg % (C - 1) + 1;
  const int cnt = counts[seg];
  const int64_t dst = offs[seg];
  for (int k = threadIdx.x; k < cnt; k += blockDim.x) {
    float4 b = slot_boxes[(int64_t)seg * K + k];
    if (sizes) {
      const float w = sizes[2 * n], h = sizes[2 * n + 1];
      b = make_float4(b.x * w, b.y * h, b.z * w, b.w * h);
    }
    out_boxes[dst + k] = b;
    out_labels[dst + k] = label;
    out_probs[dst + k] = slot_probs[(int64_t)seg * K + k];
  }
}

int check_desc(const DfqSsdNms* d, const char* who) {
  if (!d) { set_error("%s: descriptor is NULL", who); return DFQ_E_ARG; }
  if (d->N < 1 || d->P < 1) { set_error("%s: N and P must be positive, got %d and %d", who, d->N, d->P); return DFQ_E_ARG; }
  if (d->prior_batch != 1 && d->prior_batch != d->N) {
    set_error("%s: prior_batch must be 1 or N = %d, got %d", who, d->N, d->prior_batch);
    return DFQ_E_ARG;
  }
  return 0;
}

int check_nms(const DfqSsdNms* d, const char* who) {
  if (int rc = check_desc(d, who)) return rc;
  if (d->C < 2) { set_error("%s: C must be at least 2 (background and one class), got %d", who, d->C); return DFQ_E_ARG; }
  if (d->candidate_size < 1) { set_error("%s: candidate_size must be at least 1, got %d", who, d->candidate_size); return DFQ_E_ARG; }
  if (d->candidate_size > kMaxCandidates) {
    set_error("%s: candidate_size %d is above the limit %d", who, d->candidate_size, kMaxCandidates);
    return DFQ_E_UNSUPPORTED;
  }
  if ((int64_t)d->N * (d->C - 1) > INT32_MAX) { set_error("%s: N * (C - 1) does not fit in int32", who); return DFQ_E_UNSUPPORTED; }
  return 0;
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace
}  // namespace dfq

using namespace dfq;

extern "C" int dfq_ssd_decode(const float* locations, const float* priors, float* boxes, const DfqSsdNms* d, void* stream) {
  if (int rc = check_desc(d, "dfq_ssd_decode")) return rc;
  if (!locations || !priors || !boxes || !aligned16(locations) || !aligned16(priors) || !aligned16(boxes)) {
    set_error("dfq_ssd_decode: locations, priors and boxes must be non-NULL and 16-byte aligned");
    return DFQ_E_ARG;
  }
  const int64_t total = (int64_t)d->N * d->P;
  const int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)sm_count() * 16);
  k_ssd_decode<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)locations, (const float4*)priors, (float4*)boxes,
                                                       d->N, d->P, d->prior_batch, d->center_variance, d->size_variance);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_ssd_nms(const float* scores, const float* boxes, float* slot_boxes, float* slot_probs, int32_t* counts,
                           int64_t* offsets, const DfqSsdNms* d, void* stream) {
  if (int rc = check_nms(d, "dfq_ssd_nms")) return rc;
  if (!scores || !boxes || !slot_boxes || !slot_probs || !counts || !offsets || !aligned16(boxes) ||
      !aligned16(slot_boxes)) {
    set_error("dfq_ssd_nms: every pointer must be non-NULL, boxes and slot_boxes 16-byte aligned");
    return DFQ_E_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int S = d->N * (d->C - 1), K = d->candidate_size;
  const size_t smem = nms_smem(K);
  DFQ_CUDA(cudaFuncSetAttribute(k_ssd_nms, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_ssd_nms<<<S, kNmsThreads, smem, st>>>(scores, (const float4*)boxes, (float4*)slot_boxes, slot_probs, counts, d->P,
                                          d->C, d->prob_threshold, d->iou_threshold, K, d->top_k);
  DFQ_CUDA(cudaGetLastError());
  k_ssd_scan<<<1, kScanThreads, 0, st>>>(counts, offsets, S);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_ssd_compact(const float* slot_boxes, const float* slot_probs, const int32_t* counts,
                               const int64_t* offsets, const float* image_sizes, float* out_boxes, int64_t* out_labels,
                               float* out_probs, const DfqSsdNms* d, void* stream) {
  if (int rc = check_nms(d, "dfq_ssd_compact")) return rc;
  if (!slot_boxes || !slot_probs || !counts || !offsets || !out_boxes || !out_labels || !out_probs ||
      !aligned16(slot_boxes) || !aligned16(out_boxes)) {
    set_error("dfq_ssd_compact: every pointer but image_sizes must be non-NULL, slot_boxes and out_boxes 16-byte aligned");
    return DFQ_E_ARG;
  }
  k_ssd_compact<<<d->N * (d->C - 1), 128, 0, (cudaStream_t)stream>>>(
      (const float4*)slot_boxes, slot_probs, counts, offsets, image_sizes, (float4*)out_boxes, out_labels, out_probs, d->C,
      d->candidate_size);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}
