// The multi-tensor launch scheme the optimiser steps (optim.cu) and the gradient clip (clip.cu) share.  Every tensor of a
// device is cut into chunks of kChunk elements; a launch carries up to kMaxTensors tensors' pointers in its __grid_constant__
// parameter block with an inclusive int32 prefix of their chunk counts, and a grid-stride loop hands chunks to CTAs, each
// finding its chunk's tensor by binary search over that prefix.  More tensors, or a prefix past INT32_MAX, go out as more
// launches.  A grid-wide arrival counter, zero between launches, elects the last CTA to finish.
#pragma once

#include "common.cuh"

namespace qagnn {

namespace mt {

constexpr int kThreads = 256;
constexpr int64_t kChunk = 8192;    // elements per chunk: 8 float4 per thread
constexpr int kMaxTensors = 512;    // per launch: the optimiser's parameter block stays under sm_90's 32764 bytes

inline int64_t chunk_count(int64_t numel) { return (numel + kChunk - 1) / kChunk; }

// True when a launch holding n tensors and `chunks` chunks has no room for a tensor of nc more chunks
inline bool launch_full(int32_t n, int64_t chunks, int64_t nc) { return n == kMaxTensors || chunks + nc > INT32_MAX; }

// One CTA per chunk up to 8 per SM, at least one
inline unsigned launch_blocks(int64_t chunks) { return (unsigned)max(min(chunks, (int64_t)kNumSMs * 8), (int64_t)1); }

// The tensor of chunk c: the first i < n whose chunk_end[i] exceeds c
__device__ __forceinline__ int chunk_owner(const int32_t* chunk_end, int n, int32_t c) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (chunk_end[mid] > c) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// Every thread of every CTA calls it once, after its last global write: true in the last CTA to arrive, which then sees
// every other CTA's writes.  That CTA owns *counter afterwards and must reset it to zero.
__device__ __forceinline__ bool last_to_arrive(int32_t* counter) {
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(counter, 1) == (int32_t)gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return false;
  __threadfence();
  return true;
}

}  // namespace mt

}  // namespace qagnn
