// torch.nn.utils.clip_grad_norm_ (L2) over every fp32 gradient of one device in two multi-tensor launches
// (qagnn_clip_grad_norm; qagnn_b200.optim.clip_grad_norm_), with no host read and no floating-point atomics.
//
// clip_norm_kernel: S = sum of g^2 over every element of every tensor, in fp64.  Each square (double)g * (double)g is exact,
// so each accumulation step is one fp64 rounding (a DFMA).  The summation order depends only on the tensors' sizes and their
// order in the list, never on the grid, the SM count, the launch split or a pointer's alignment:
//   1. within a thread: chunk c of a tensor (multi_tensor.cuh: kChunk elements) has n elements and n4 = n / 4 quads; thread t
//      adds quads t, t + 256, t + 512, ... in that order, each quad's four elements in order, then element 4 n4 + t if it is
//      below n, into an fp64 partial that starts at +0;
//   2. the block tree: each warp sums its 32 partials with __shfl_down_sync at offsets 16, 8, 4, 2, 1, and warp 0 sums the
//      8 warp sums at offsets 4, 2, 1;
//   3. the result goes to slot number (chunk c's index in the concatenation of every tensor's chunks), written once;
//   4. across slots: the last CTA to arrive in the last launch has thread t add slots t, t + 256, ... in order from +0, then
//      sums the 256 partials with the tree of step 2.
// That CTA then writes total_norm = (float)sqrt_rn(S) (one rounding of the fp64 root) and the clip coefficient as torch's
// clip_grad_norm_ forms it from its fp32 total, one fp32 operation each: c = (float)max_norm * (1 / (total_norm + (float)1e-6))
// (Tensor.__rtruediv__ is reciprocal() * other), then clamp(c, max=1), which keeps a NaN.
//
// clip_scale_kernel: g = g * c in place, torch._foreach_mul_'s one fp32 multiply.  Every CTA reads c first and returns when
// it is 1.0f: x * 1.0f == x, so a batch that is not clipped reads each gradient once (4 bytes per element), not three times.
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

__global__ void __launch_bounds__(kThreads) clip_norm_kernel(const __grid_constant__ NormArgs a) {
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
        acc = add_square(add_square(add_square(add_square(acc, v.x), v.y), v.z), v.w);
      }
    } else {
      for (int j = threadIdx.x; j < n4; j += kThreads)
        acc = add_square(add_square(add_square(add_square(acc, g[4 * j]), g[4 * j + 1]), g[4 * j + 2]), g[4 * j + 3]);
    }
    if (4 * n4 + (int)threadIdx.x < n) acc = add_square(acc, g[4 * n4 + threadIdx.x]);
    acc = block_sum(acc);
    if (threadIdx.x == 0) a.slots[a.base + c] = acc;
  }
  if (a.counter == nullptr || !mt::last_to_arrive(a.counter)) return;
  double acc = 0.0;
  for (int64_t s = threadIdx.x; s < a.total; s += kThreads) acc += __ldcg(a.slots + s);
  acc = block_sum(acc);
  if (threadIdx.x == 0) {
    const float norm = __double2float_rn(__dsqrt_rn(acc));
    const float c = __fmul_rn(a.max_norm, __frcp_rn(__fadd_rn(norm, (float)1e-6)));
    *a.total_norm = norm;
    *a.coef = c > 1.0f ? 1.0f : c;  // clamp(max=1): NaN > 1 is false, so a NaN stays
    *a.counter = 0;
  }
}

__global__ void __launch_bounds__(kThreads) clip_scale_kernel(const __grid_constant__ ScaleArgs a) {
  const float k = *a.coef;
  if (k == 1.0f) return;
  const int32_t chunks = a.l.n ? a.l.chunk_end[a.l.n - 1] : 0;
  for (int32_t c = blockIdx.x; c < chunks; c += gridDim.x) {
    int n;
    float* g = chunk_span(a.l, c, n);
    int done = 0;
    if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
      const int n4 = n >> 2;
      for (int j = threadIdx.x; j < n4; j += kThreads) {
        float4 v = reinterpret_cast<float4*>(g)[j];
        v.x = __fmul_rn(v.x, k);
        v.y = __fmul_rn(v.y, k);
        v.z = __fmul_rn(v.z, k);
        v.w = __fmul_rn(v.w, k);
        reinterpret_cast<float4*>(g)[j] = v;
      }
      done = n4 << 2;
    }
    for (int j = done + threadIdx.x; j < n; j += kThreads) g[j] = __fmul_rn(g[j], k);
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

using namespace qagnn;

extern "C" int64_t qagnn_clip_grad_norm_slots(int32_t n_tensors, const int64_t* numels) { return slot_count(n_tensors, numels); }

extern "C" int32_t qagnn_clip_grad_norm(int32_t n_tensors, void* const* grads, const int64_t* numels, double max_norm,
                                        double* slots, int64_t n_slots, int32_t* counter, float* total_norm, float* coef,
                                        void* stream) {
  const int64_t need = slot_count(n_tensors, numels);
  if (need < 0 || (n_tensors > 0 && !grads) || (need > 0 && !slots) || !counter || !total_norm || !coef)
    return QAGNN_ERR_INVALID_ARGUMENT;
  for (int32_t i = 0; i < n_tensors; ++i)
    if (numels[i] > 0 && !grads[i]) return QAGNN_ERR_INVALID_ARGUMENT;
  if (n_slots < need) return QAGNN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  static thread_local NormArgs na;
  na.slots = slots;
  na.total = need;
  na.max_norm = (float)max_norm;
  na.total_norm = total_norm;
  na.coef = coef;
  QAGNN_RETURN_IF(for_each_launch(n_tensors, grads, numels, [&](const GradList& l, int64_t base, bool last) -> int32_t {
    na.l = l;
    na.base = base;
    na.counter = last ? counter : nullptr;
    clip_norm_kernel<<<mt::launch_blocks(l.n ? l.chunk_end[l.n - 1] : 0), kThreads, 0, st>>>(na);
    QAGNN_CHECK_LAUNCH();
    return QAGNN_OK;
  }));
  static thread_local ScaleArgs sa;
  sa.coef = coef;
  return for_each_launch(n_tensors, grads, numels, [&](const GradList& l, int64_t, bool) -> int32_t {
    sa.l = l;
    clip_scale_kernel<<<mt::launch_blocks(l.n ? l.chunk_end[l.n - 1] : 0), kThreads, 0, st>>>(sa);
    QAGNN_CHECK_LAUNCH();
    return QAGNN_OK;
  });
}
