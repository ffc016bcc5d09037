// Classification accuracy on the device: the argmax of each row of the logits, bit for bit torch.max(logits, 1)[1] on
// CUDA, compared with the row's label and counted, without the predictions ever leaving the device.
//
//   k_cls_count   one warp per row (rows grid-strided over the warps of the grid): lane l scans the columns l, l + 32, ...
//                 ascending under torch's CUDA max(dim) rule, the 32 candidates are merged by butterfly shuffles under the
//                 same rule (a total order, so the merge order does not matter), lane 0 writes the int64 prediction and
//                 counts the row when its label equals it.  Each CTA adds its count to the uint64 counter with one 64-bit
//                 atomicAdd.
#include <algorithm>

#include "common.cuh"

namespace dfq {
namespace {

constexpr int kClsThreads = 256;
constexpr int kClsWarps = kClsThreads / 32;
constexpr int kClsNone = INT32_MAX;        // the index of a lane that holds no column (C < 32)

// torch's CUDA max(dim) combine (GreaterOrNan, ATen/native/SharedReduceOps.h): does (a, ia) win over (b, ib)?  A NaN wins
// over every number and the lower index wins between two NaNs; otherwise the larger value wins, and on equal values
// (-0.0 equal to +0.0) the lower index.  A total order on the (value, index) pairs.
__device__ __forceinline__ bool cls_wins(float a, int ia, float b, int ib) {
  if (ia == kClsNone) return false;
  if (ib == kClsNone) return true;
  if (a != a) return b == b || ia < ib;
  if (b != b) return false;
  return a == b ? ia < ib : a > b;
}

template <bool PRED, bool COUNT>
__global__ void __launch_bounds__(kClsThreads) k_cls_count(const float* __restrict__ x, const long long* __restrict__ labels,
                                                           long long* __restrict__ pred,
                                                           unsigned long long* __restrict__ correct, int64_t N, int C) {
  __shared__ unsigned long long warp_count[kClsWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long mine = 0;
  for (int64_t row = (int64_t)blockIdx.x * kClsWarps + warp; row < N; row += (int64_t)gridDim.x * kClsWarps) {
    const float* r = x + row * C;
    float best = 0.f;
    int arg = kClsNone;
    if (lane < C) {
      best = __ldg(r + lane);
      arg = lane;
      // the scan over this lane's columns, ascending: a strictly larger value or a NaN replaces a non-NaN best
      for (int c = lane + 32; c < C; c += 32) {
        const float v = __ldg(r + c);
        if (best == best && (v != v || v > best)) {
          best = v;
          arg = c;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
      if (cls_wins(ob, oa, best, arg)) {
        best = ob;
        arg = oa;
      }
    }
    if (lane == 0) {
      if (PRED) pred[row] = arg;
      if (COUNT) mine += __ldg(labels + row) == (long long)arg;
    }
  }
  if (COUNT) {
    if (lane == 0) warp_count[warp] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long s = 0;
#pragma unroll
      for (int w = 0; w < kClsWarps; ++w) s += warp_count[w];
      if (s) atomicAdd(correct, s);
    }
  }
}

// [a, a + na) and [b, b + nb) share a byte; a NULL range shares none
bool overlap(const void* a, int64_t na, const void* b, int64_t nb) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return a && b && x < y + (uintptr_t)nb && y < x + (uintptr_t)na;
}

template <bool PRED, bool COUNT>
int launch(const float* x, const int64_t* labels, int64_t* pred, uint64_t* correct, int64_t N, int C, cudaStream_t st) {
  auto kern = k_cls_count<PRED, COUNT>;
  int per_sm = 1;
  DFQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kClsThreads, 0));
  // enough CTAs to fill the device once; larger batches walk their rows grid-strided
  const int64_t want = (N + kClsWarps - 1) / kClsWarps;
  const int grid = (int)std::min<int64_t>(want, (int64_t)sm_count() * std::max(per_sm, 1));
  kern<<<grid, kClsThreads, 0, st>>>(x, (const long long*)labels, (long long*)pred, (unsigned long long*)correct, N, C);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace
}  // namespace dfq

using namespace dfq;

extern "C" int dfq_cls_count(const float* logits, const int64_t* labels, int64_t* pred, uint64_t* correct, int64_t N,
                             int32_t C, void* stream) {
  const char* who = "dfq_cls_count";
  if (N < 1 || C < 1) {
    set_error("%s: N and C must be positive, got %lld and %d", who, (long long)N, C);
    return DFQ_E_ARG;
  }
  if ((double)N * (double)C >= 1.15e18) {
    set_error("%s: the logits have 2^60 elements or more", who);
    return DFQ_E_UNSUPPORTED;
  }
  if (!logits) { set_error("%s: logits is NULL", who); return DFQ_E_ARG; }
  if ((labels == nullptr) != (correct == nullptr)) {
    set_error("%s: labels and correct must both be given or both be NULL", who);
    return DFQ_E_ARG;
  }
  if (!pred && !correct) { set_error("%s: neither pred nor correct is given", who); return DFQ_E_ARG; }
  if (((uintptr_t)logits & 3) || ((uintptr_t)labels & 7) || ((uintptr_t)pred & 7) || ((uintptr_t)correct & 7)) {
    set_error("%s: misaligned pointer (logits 4, labels, pred and correct 8 bytes)", who);
    return DFQ_E_ARG;
  }
  const int64_t nx = 4 * N * C, nl = labels ? 8 * N : 0, np = pred ? 8 * N : 0;
  if (overlap(correct, 8, logits, nx) || overlap(correct, 8, labels, nl) || overlap(correct, 8, pred, np) ||
      overlap(pred, np, logits, nx) || overlap(pred, np, labels, nl)) {
    set_error("%s: correct and pred must not overlap the other buffers", who);
    return DFQ_E_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (!correct) return launch<true, false>(logits, nullptr, pred, nullptr, N, C, st);
  return pred ? launch<true, true>(logits, labels, pred, correct, N, C, st)
              : launch<false, true>(logits, labels, nullptr, correct, N, C, st);
}
