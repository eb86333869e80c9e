// The ordered sum of per-micro-batch gradient slots into .grad (qagnn_ordered_grad_sum;
// qagnn_b200.distributed.ordered_grad_sum_), the reduction of data-parallel training: every rank holds the gathered slots
// [M, ld] of one optimiser batch, micro-batch j's gradient of tensor i in row j from column cols[i], and writes
//   g  = init_from_grad[i] ? g + slot 0 : slot 0,   then   g = g + slot j   for j = 1 ... n_valid - 1, in that order,
// each add one fp32 __fadd_rn.  That is the sequence of adds one GPU performs when it accumulates the micro-batches into .grad
// one after another, so .grad comes out bit for bit.  Every element is owned by one thread, which walks the slots in order:
// the result does not depend on the grid, the launch split or the alignment, and there are no atomics.
#include "multi_tensor.cuh"

namespace qagnn {

namespace {

using mt::kChunk;
using mt::kMaxTensors;
using mt::kThreads;

struct SumList {
  float* g[kMaxTensors];
  int64_t numel[kMaxTensors];
  int64_t col[kMaxTensors];        // the tensor's first column in a slot row
  int32_t chunk_end[kMaxTensors];  // inclusive prefix sum of the tensors' chunk counts
  uint8_t init[kMaxTensors];       // nonzero: the sum starts from g
  int32_t n;
};

struct SumArgs {
  SumList l;
  const float* slots;
  int64_t ld;  // elements between consecutive slot rows
  int32_t n_valid;
};

template <typename T>
__device__ __forceinline__ T add4(T a, T b) {
  return T{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w)};
}

// Slot rows are read once: keep them out of L1 and mark them evict-first in L2, the .grad lines are what gets rewritten
__global__ void __launch_bounds__(kThreads) ordered_grad_sum_kernel(const __grid_constant__ SumArgs a) {
  const int32_t chunks = a.l.n ? a.l.chunk_end[a.l.n - 1] : 0;
  const int32_t nv = a.n_valid;
  for (int32_t c = blockIdx.x; c < chunks; c += gridDim.x) {
    const int i = mt::chunk_owner(a.l.chunk_end, a.l.n, c);
    const int64_t c0 = (int64_t)(c - (i ? a.l.chunk_end[i - 1] : 0)) * kChunk;
    const int n = (int)min(kChunk, a.l.numel[i] - c0);
    float* g = a.l.g[i] + c0;
    const float* s = a.slots + a.l.col[i] + c0;
    const bool init = a.l.init[i] != 0;
    int done = 0;
    if ((((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(s)) & 15) | (a.ld & 3)) == 0) {
      const int n4 = n >> 2;
      for (int j = threadIdx.x; j < n4; j += kThreads) {
        const float4* sj = reinterpret_cast<const float4*>(s) + j;
        float4 acc = __ldcs(sj);
        if (init) acc = add4(reinterpret_cast<const float4*>(g)[j], acc);
#pragma unroll 8
        for (int32_t k = 1; k < nv; ++k) acc = add4(acc, __ldcs(sj + k * (a.ld >> 2)));
        reinterpret_cast<float4*>(g)[j] = acc;
      }
      done = n4 << 2;
    }
    for (int j = done + threadIdx.x; j < n; j += kThreads) {
      float acc = __ldcs(s + j);
      if (init) acc = __fadd_rn(g[j], acc);
#pragma unroll 8
      for (int32_t k = 1; k < nv; ++k) acc = __fadd_rn(acc, __ldcs(s + j + k * a.ld));
      g[j] = acc;
    }
  }
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_ordered_grad_sum(int32_t n_tensors, void* const* grads, const int64_t* numels, const int64_t* cols,
                                          const int32_t* init_from_grad, const float* slots, int64_t ld, int32_t n_valid,
                                          void* stream) {
  if (n_tensors < 0 || n_valid < 1 || ld < 0 || (n_tensors > 0 && (!grads || !numels || !cols || !init_from_grad)))
    return QAGNN_ERR_INVALID_ARGUMENT;
  for (int32_t i = 0; i < n_tensors; ++i) {
    if (numels[i] < 0 || cols[i] < 0 || mt::chunk_count(numels[i]) > INT32_MAX) return QAGNN_ERR_INVALID_ARGUMENT;
    if (numels[i] > 0 && (!grads[i] || !slots || cols[i] + numels[i] > ld)) return QAGNN_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t st = (cudaStream_t)stream;
  static thread_local SumArgs sa;  // 15 KB: kept off the stack
  sa.slots = slots;
  sa.ld = ld;
  sa.n_valid = n_valid;
  SumList& l = sa.l;
  int64_t chunks = 0;
  auto launch = [&]() -> int32_t {
    if (chunks == 0) return QAGNN_OK;
    ordered_grad_sum_kernel<<<mt::launch_blocks(chunks), kThreads, 0, st>>>(sa);
    QAGNN_CHECK_LAUNCH();
    return QAGNN_OK;
  };
  l.n = 0;
  for (int32_t i = 0; i < n_tensors; ++i) {
    const int64_t nc = mt::chunk_count(numels[i]);
    if (nc == 0) continue;
    if (mt::launch_full(l.n, chunks, nc)) {
      QAGNN_RETURN_IF(launch());
      l.n = 0;
      chunks = 0;
    }
    const int32_t j = l.n++;
    l.g[j] = (float*)grads[i];
    l.numel[j] = numels[i];
    l.col[j] = cols[i];
    l.init[j] = init_from_grad[i] != 0;
    chunks += nc;
    l.chunk_end[j] = (int32_t)chunks;
  }
  return launch();
}
