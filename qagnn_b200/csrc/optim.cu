// RAdam step (qagnn_radam_step): the update of the reference's RAdam (utils/optimization_utils.py) over every fp32 tensor of
// one device in one launch, with GradScaler's inf skip and unscale taken on the device.
//
// Per element, t = the tensor's step + 1, each line one fp32 operation in the order the eager torch ops apply them, with the
// contractions PyTorch's CUDA kernels compile to (addcmul_ / add_(alpha) / addcdiv_ are `a + alpha * x`, one FMA):
//   [unscale]  g = g * inv_scale                                  (GradScaler.unscale_; written back to .grad)
//   mul_, addcmul_        v = fma(1 - b2, g * g, v * b2)
//   mul_, add_(alpha)     m = fma(g, 1 - b1, m * b1)
//   rectified (rho_t >= 5):   [wd != 0] p = fma(p, -wd*lr, p) ;  p = fma(-s*lr, m / (sqrt(v) + eps), p)
//   degenerated to SGD:       [wd != 0] p = fma(p, -wd*lr, p) ;  p = fma(m, -s*lr, p)
//   otherwise p is left as it is (m, v and the step still advance).
// The host-double scalars (1 - b2, -wd*lr, eps, ...) are rounded to fp32 as torch rounds them; s and the branch come from a
// per-(b1, b2) fp64 table built on the host with the reference's formula and indexed by the device step, and -s*lr is formed
// in fp64 before its rounding, as the reference forms it in Python.
//
// Work split: each tensor is cut into chunks of kChunk elements and a grid-stride loop hands chunks to CTAs; a CTA finds its
// chunk's tensor by binary search over the per-tensor chunk prefix held in the kernel parameters.  Every CTA reads the step
// counters, so they are advanced only by the last CTA to finish (a grid-wide arrival counter that the last CTA resets).  A
// nonzero found_inf leaves p, m, v and every step as they are.
#include "common.cuh"

namespace qagnn {

namespace {

constexpr int kThreads = 256;
constexpr int64_t kChunk = 8192;    // elements per chunk: 8 float4 per thread
constexpr int kMaxTensors = 512;    // per launch: the parameter block below stays under sm_90's 32764 bytes
constexpr int kMaxGroups = 16;      // distinct param groups per launch

enum : int32_t { kKindNone = 0, kKindSgd = 1, kKindRect = 2 };
enum : int32_t { kFlagDecay = 1, kFlagDegenerated = 2 };

struct RAdamGroup {
  const double* table;  // [table_len, 2]: (1.0 if rho_t >= 5 else 0.0, step size s) for t = row
  double lr;
  float beta1, om_beta1, beta2, om_beta2, eps, decay;  // fp32 of b1, 1 - b1, b2, 1 - b2, eps, -wd*lr
  int32_t flags;
};

struct RAdamArgs {
  float* p[kMaxTensors];
  float* g[kMaxTensors];
  float* m[kMaxTensors];
  float* v[kMaxTensors];
  int64_t* step[kMaxTensors];
  int64_t numel[kMaxTensors];
  int32_t chunk_end[kMaxTensors];  // inclusive prefix sum of the tensors' chunk counts
  uint8_t group[kMaxTensors];
  RAdamGroup groups[kMaxGroups];
  int64_t table_len;
  const float* found_inf;
  const float* grad_scale;
  int32_t* counter;
  int32_t n;
};
static_assert(sizeof(RAdamArgs) <= 32764, "RAdam kernel parameters exceed the 32764 bytes sm_90 accepts");

struct Coef {
  float inv, b1, om_b1, b2, om_b2, eps, decay, step;
  int32_t kind;
  bool unscale, has_decay, skip;
};

__device__ __forceinline__ void radam_elem(float& p, float& g, float& m, float& v, const Coef& k) {
  if (k.unscale) g = __fmul_rn(g, k.inv);
  if (k.skip) return;
  v = __fmaf_rn(k.om_b2, __fmul_rn(g, g), __fmul_rn(v, k.b2));
  m = __fmaf_rn(g, k.om_b1, __fmul_rn(m, k.b1));
  if (k.kind == kKindNone) return;
  if (k.has_decay) p = __fmaf_rn(p, k.decay, p);
  if (k.kind == kKindRect)
    p = __fmaf_rn(k.step, __fdiv_rn(m, __fadd_rn(__fsqrt_rn(v), k.eps)), p);
  else
    p = __fmaf_rn(m, k.step, p);
}

__device__ __forceinline__ void radam_scalar(float* p, float* g, float* m, float* v, int64_t j, const Coef& k) {
  float pp = p[j], gg = g[j], mm = m[j], vv = v[j];
  radam_elem(pp, gg, mm, vv, k);
  if (k.unscale) g[j] = gg;
  if (k.skip) return;
  m[j] = mm;
  v[j] = vv;
  if (k.kind != kKindNone) p[j] = pp;
}

__global__ void __launch_bounds__(kThreads) radam_kernel(const __grid_constant__ RAdamArgs a) {
  Coef k;
  k.skip = a.found_inf != nullptr && *a.found_inf != 0.f;
  k.unscale = a.grad_scale != nullptr;
  // GradScaler.unscale_: inv_scale = scale.double().reciprocal().float()
  k.inv = k.unscale ? __double2float_rn(__drcp_rn((double)*a.grad_scale)) : 1.f;
  const int32_t total = a.chunk_end[a.n - 1];
  for (int32_t c = blockIdx.x; c < total; c += gridDim.x) {
    int lo = 0, hi = a.n - 1;  // the first tensor whose chunk_end exceeds c
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (a.chunk_end[mid] > c) hi = mid; else lo = mid + 1;
    }
    const int i = lo;
    const int64_t c0 = (int64_t)(c - (i ? a.chunk_end[i - 1] : 0)) * kChunk;
    const int64_t n = min(kChunk, a.numel[i] - c0);
    const RAdamGroup& gr = a.groups[a.group[i]];
    k.b1 = gr.beta1; k.om_b1 = gr.om_beta1; k.b2 = gr.beta2; k.om_b2 = gr.om_beta2; k.eps = gr.eps; k.decay = gr.decay;
    k.kind = kKindNone;
    k.step = 0.f;
    if (!k.skip) {
      const int64_t t = min(max(*a.step[i] + 1, (int64_t)0), a.table_len - 1);
      const double rect = gr.table[2 * t], s = gr.table[2 * t + 1];
      k.kind = rect != 0.0 ? kKindRect : (gr.flags & kFlagDegenerated) ? kKindSgd : kKindNone;
      k.step = __double2float_rn(__dmul_rn(-s, gr.lr));
    }
    k.has_decay = (gr.flags & kFlagDecay) != 0;
    if (k.skip && !k.unscale) continue;
    float* p = a.p[i] + c0;
    float* g = a.g[i] + c0;
    float* m = a.m[i] + c0;
    float* v = a.v[i] + c0;
    const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                           reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    int64_t done = 0;
    if (aligned) {
      const int64_t n4 = n >> 2;
      for (int64_t j = threadIdx.x; j < n4; j += kThreads) {
        float4 pp = reinterpret_cast<float4*>(p)[j], gg = reinterpret_cast<float4*>(g)[j];
        float4 mm = reinterpret_cast<float4*>(m)[j], vv = reinterpret_cast<float4*>(v)[j];
        radam_elem(pp.x, gg.x, mm.x, vv.x, k);
        radam_elem(pp.y, gg.y, mm.y, vv.y, k);
        radam_elem(pp.z, gg.z, mm.z, vv.z, k);
        radam_elem(pp.w, gg.w, mm.w, vv.w, k);
        if (k.unscale) reinterpret_cast<float4*>(g)[j] = gg;
        if (k.skip) continue;
        reinterpret_cast<float4*>(m)[j] = mm;
        reinterpret_cast<float4*>(v)[j] = vv;
        if (k.kind != kKindNone) reinterpret_cast<float4*>(p)[j] = pp;
      }
      done = n4 << 2;
    }
    for (int64_t j = done + threadIdx.x; j < n; j += kThreads) radam_scalar(p, g, m, v, j, k);
  }
  // the last CTA to arrive advances the step counters: every CTA has read them by then
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(a.counter, 1) == (int32_t)gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (!k.skip)
    for (int i = threadIdx.x; i < a.n; i += kThreads) *a.step[i] += 1;
  if (threadIdx.x == 0) *a.counter = 0;
}

// Fills the per-launch copy of a group from the host doubles, rounding each scalar as torch rounds a Python float
void fill_group(RAdamGroup& gr, double lr, double wd, double b1, double b2, double eps, int32_t degenerated, const double* table) {
  gr.table = table;
  gr.lr = lr;
  gr.beta1 = (float)b1;
  gr.om_beta1 = (float)(1.0 - b1);
  gr.beta2 = (float)b2;
  gr.om_beta2 = (float)(1.0 - b2);
  gr.eps = (float)eps;
  gr.decay = (float)(-wd * lr);
  gr.flags = (wd != 0.0 ? kFlagDecay : 0) | (degenerated ? kFlagDegenerated : 0);
}

int32_t launch(const RAdamArgs& a, cudaStream_t st) {
  const int64_t chunks = a.chunk_end[a.n - 1];
  const unsigned blocks = (unsigned)max(min(chunks, (int64_t)kNumSMs * 8), (int64_t)1);
  radam_kernel<<<blocks, kThreads, 0, st>>>(a);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_radam_step(int32_t n_tensors, void* const* params, void* const* grads, void* const* exp_avgs,
                                    void* const* exp_avg_sqs, void* const* steps, const int64_t* numels,
                                    const int32_t* group_index, int32_t n_groups, const double* lr, const double* weight_decay,
                                    const double* beta1, const double* beta2, const double* eps,
                                    const int32_t* degenerated_to_sgd, void* const* step_tables, int64_t table_len,
                                    const float* found_inf, const float* grad_scale, int32_t* counter, void* stream) {
  if (n_tensors < 0 || n_groups < 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (n_tensors == 0) return QAGNN_OK;
  if (!params || !grads || !exp_avgs || !exp_avg_sqs || !steps || !numels || !group_index || n_groups == 0 || !lr ||
      !weight_decay || !beta1 || !beta2 || !eps || !degenerated_to_sgd || !step_tables || table_len < 2 || !counter)
    return QAGNN_ERR_INVALID_ARGUMENT;
  for (int32_t i = 0; i < n_tensors; ++i) {
    const int32_t gi = group_index[i];
    if (gi < 0 || gi >= n_groups || !steps[i] || numels[i] < 0 ||
        (numels[i] + kChunk - 1) / kChunk > INT32_MAX) return QAGNN_ERR_INVALID_ARGUMENT;
    if (numels[i] > 0 && (!params[i] || !grads[i] || !exp_avgs[i] || !exp_avg_sqs[i])) return QAGNN_ERR_INVALID_ARGUMENT;
    if (!step_tables[gi] || !(beta1[gi] >= 0.0 && beta1[gi] < 1.0) || !(beta2[gi] >= 0.0 && beta2[gi] < 1.0))
      return QAGNN_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t st = (cudaStream_t)stream;
  static thread_local RAdamArgs a;  // 28 KB: kept off the stack
  int32_t slot_of[kMaxGroups];      // global group of each per-launch slot
  int32_t n_slots = 0;
  a.n = 0;
  a.table_len = table_len;
  a.found_inf = found_inf;
  a.grad_scale = grad_scale;
  a.counter = counter;
  int64_t chunks = 0;
  for (int32_t i = 0; i < n_tensors; ++i) {
    const int32_t gi = group_index[i];
    const int64_t nc = (numels[i] + kChunk - 1) / kChunk;
    int32_t slot = -1;
    for (int32_t s = 0; s < n_slots; ++s)
      if (slot_of[s] == gi) slot = s;
    // a full launch (tensors, groups or the int32 chunk prefix) goes out first
    if (a.n == kMaxTensors || (slot < 0 && n_slots == kMaxGroups) || chunks + nc > INT32_MAX) {
      QAGNN_RETURN_IF(launch(a, st));
      a.n = 0;
      n_slots = 0;
      chunks = 0;
      slot = -1;
    }
    if (slot < 0) {
      slot = n_slots++;
      slot_of[slot] = gi;
      fill_group(a.groups[slot], lr[gi], weight_decay[gi], beta1[gi], beta2[gi], eps[gi], degenerated_to_sgd[gi],
                 (const double*)step_tables[gi]);
    }
    const int32_t j = a.n++;
    a.p[j] = (float*)params[i];
    a.g[j] = (float*)grads[i];
    a.m[j] = (float*)exp_avgs[i];
    a.v[j] = (float*)exp_avg_sqs[i];
    a.step[j] = (int64_t*)steps[i];
    a.numel[j] = numels[i];
    a.group[j] = (uint8_t)slot;
    chunks += nc;
    a.chunk_end[j] = (int32_t)chunks;
  }
  return launch(a, st);
}
