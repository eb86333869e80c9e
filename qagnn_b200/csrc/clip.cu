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
#include "clip.cuh"

namespace qagnn {

namespace {

__global__ void __launch_bounds__(kThreads) clip_norm_kernel(const __grid_constant__ NormArgs a) {
  norm_body(a, [](float x) { return x; }, [&] { return a.max_norm; });
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
