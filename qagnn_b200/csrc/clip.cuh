// The gradient norm's body and launch packing, shared by clip_grad_norm_ (clip.cu) and the captured optimiser tail's first
// pass (tail.cu).  clip.cu states the summation order and the coefficient's rounding.
#pragma once

#include "multi_tensor.cuh"

namespace qagnn {

namespace {

using mt::kChunk;
using mt::kMaxTensors;
using mt::kThreads;

struct GradList {
  float* g[kMaxTensors];
  int64_t numel[kMaxTensors];
  int32_t chunk_end[kMaxTensors];  // inclusive prefix sum of the tensors' chunk counts
  int32_t n;
};

struct NormArgs {
  GradList l;
  double* slots;       // one per chunk of every launch
  int64_t base;        // the global index of this launch's first chunk
  int64_t total;       // chunks over every launch
  int32_t* counter;    // the last launch's arrival counter; null in the others
  float max_norm;
  float* total_norm;
  float* coef;
};

struct ScaleArgs {
  GradList l;
  const float* coef;
};

// [start, start + n) of tensor i for chunk c of a launch
__device__ __forceinline__ float* chunk_span(const GradList& l, int32_t c, int& n) {
  const int i = mt::chunk_owner(l.chunk_end, l.n, c);
  const int64_t c0 = (int64_t)(c - (i ? l.chunk_end[i - 1] : 0)) * kChunk;
  n = (int)min(kChunk, l.numel[i] - c0);
  return l.g[i] + c0;
}

__device__ __forceinline__ double add_square(double acc, float x) { return __fma_rn((double)x, (double)x, acc); }

// Step 2's tree: thread 0 returns the CTA's sum.  Every thread must call it.
__device__ __forceinline__ double block_sum(double v) {
  __shared__ double warp_sums[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x < 32) {
    s = threadIdx.x < kThreads / 32 ? warp_sums[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = kThreads / 64; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  }
  __syncthreads();  // warp_sums is free for the next call
  return s;
}

// clip_norm_kernel's body.  value(x) maps each gradient element to the value whose square is summed, and max_norm() gives the
// threshold to the last CTA.
template <class Value, class MaxNorm>
__device__ __forceinline__ void norm_body(const NormArgs& a, Value value, MaxNorm max_norm) {
  const int32_t chunks = a.l.n ? a.l.chunk_end[a.l.n - 1] : 0;
  for (int32_t c = blockIdx.x; c < chunks; c += gridDim.x) {
    int n;
    const float* g = chunk_span(a.l, c, n);
    const int n4 = n >> 2;
    double acc = 0.0;
    if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
#pragma unroll 8
      for (int j = threadIdx.x; j < n4; j += kThreads) {
        const float4 v = reinterpret_cast<const float4*>(g)[j];
        acc = add_square(add_square(add_square(add_square(acc, value(v.x)), value(v.y)), value(v.z)), value(v.w));
      }
    } else {
      for (int j = threadIdx.x; j < n4; j += kThreads)
        acc = add_square(add_square(add_square(add_square(acc, value(g[4 * j])), value(g[4 * j + 1])), value(g[4 * j + 2])),
                           value(g[4 * j + 3]));
    }
    if (4 * n4 + (int)threadIdx.x < n) acc = add_square(acc, value(g[4 * n4 + threadIdx.x]));
    acc = block_sum(acc);
    if (threadIdx.x == 0) a.slots[a.base + c] = acc;
  }
  if (a.counter == nullptr || !mt::last_to_arrive(a.counter)) return;
  double acc = 0.0;
  for (int64_t s = threadIdx.x; s < a.total; s += kThreads) acc += __ldcg(a.slots + s);
  acc = block_sum(acc);
  if (threadIdx.x == 0) {
    const float norm = __double2float_rn(__dsqrt_rn(acc));
    const float c = __fmul_rn(max_norm(), __frcp_rn(__fadd_rn(norm, (float)1e-6)));
    *a.total_norm = norm;
    *a.coef = c > 1.0f ? 1.0f : c;  // clamp(max=1): NaN > 1 is false, so a NaN stays
    *a.counter = 0;
  }
}


// Packs the tensors into launches (kMaxTensors and an int32 chunk prefix each) and calls launch(list, first chunk, is last)
// for every launch in order; at least one launch, empty when n_tensors is 0.
template <typename F>
int32_t for_each_launch(int32_t n_tensors, void* const* grads, const int64_t* numels, F launch) {
  static thread_local GradList l;  // 10 KB: kept off the stack
  l.n = 0;
  int64_t chunks = 0, base = 0;
  for (int32_t i = 0; i < n_tensors; ++i) {
    const int64_t nc = mt::chunk_count(numels[i]);
    if (mt::launch_full(l.n, chunks, nc)) {
      QAGNN_RETURN_IF(launch(l, base, false));
      base += chunks;
      l.n = 0;
      chunks = 0;
    }
    const int32_t j = l.n++;
    l.g[j] = (float*)grads[i];
    l.numel[j] = numels[i];
    chunks += nc;
    l.chunk_end[j] = (int32_t)chunks;
  }
  return launch(l, base, true);
}

int64_t slot_count(int32_t n_tensors, const int64_t* numels) {
  if (n_tensors < 0 || (n_tensors > 0 && !numels)) return -1;
  int64_t slots = 0;
  for (int32_t i = 0; i < n_tensors; ++i) {
    if (numels[i] < 0 || mt::chunk_count(numels[i]) > INT32_MAX) return -1;
    slots += mt::chunk_count(numels[i]);
  }
  return slots;
}

}  // namespace

}  // namespace qagnn
