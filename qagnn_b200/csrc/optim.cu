// Multi-tensor optimiser steps over every fp32 tensor of one device in one launch, with GradScaler's inf skip and unscale taken
// on the device (qagnn_optim_step): the reference's RAdam (utils/optimization_utils.py), transformers' AdamW (3.4.0, the
// version the reference pins), and torch.optim.Adam and SGD as torch 2.11 steps them by default on CUDA (the foreach
// implementation, _multi_tensor_adam / _multi_tensor_sgd).  One kernel body serves all four, the update rule a template
// parameter.
//
// Per element, t = the tensor's step + 1, each line one fp32 operation in the order the eager torch ops apply them, with the
// contractions PyTorch's CUDA kernels compile to (addcmul_ / add_(alpha) / addcdiv_ are `a + alpha * x`, one FMA):
//   [unscale]  g = g * inv_scale                                  (GradScaler.unscale_; written back to .grad)
// RAdam:
//   mul_, addcmul_        v = fma(1 - b2, g * g, v * b2)
//   mul_, add_(alpha)     m = fma(g, 1 - b1, m * b1)
//   rectified (rho_t >= 5):   [wd != 0] p = fma(p, -wd*lr, p) ;  p = fma(-s*lr, m / (sqrt(v) + eps), p)
//   degenerated to SGD:       [wd != 0] p = fma(p, -wd*lr, p) ;  p = fma(m, -s*lr, p)
//   otherwise p is left as it is (m, v and the step still advance).
//   s and the branch come from a per-(b1, b2) fp64 table built on the host with the reference's formula, and -s*lr is formed
//   in fp64 before its rounding, as the reference forms it in Python.
// AdamW (exp_avg first, as transformers updates it):
//   mul_, add_(alpha)     m = fma(g, 1 - b1, m * b1)
//   mul_, addcmul_        v = fma(1 - b2, g * g, v * b2)
//   sqrt, add_            d = sqrt(v) + eps                          (two roundings: eps outside any bias correction)
//   addcdiv_              p = fma(-step_size, m / d, p)
//   [wd > 0] add_(alpha)  p = fma(p, -lr*wd, p)                      (after the update, on the new p)
//   step_size = lr * sqrt(1 - b2^t) / (1 - b1^t) with correct_bias, else lr.  The per-(b1, b2) fp64 table holds
//   (sqrt(1 - b2^t), 1 - b1^t) from Python's libm pow, and the kernel forms -((lr * sq) / bc1) in IEEE fp64 (the bits Python
//   computes) before its rounding.
// The host-double scalars (1 - b2, -wd*lr, eps, ...) are rounded to fp32 as torch rounds them.
//
// Adam and SGD follow torch's foreach ops in torch's order.  Established on the H100 against those ops: `a + alpha * x`
// (add(alpha), addcmul, addcdiv) and both branches of at::lerp are one FMA each, sqrt is correctly rounded, and the division
// by a scalar list (bias_correction2_sqrt) is a true fp32 division, not a multiply by a reciprocal.  The GPU tests compare
// every state tensor with torch's CUDA step bit for bit.
// Adam (amsgrad, maximize and decoupled_weight_decay off):
//   [wd != 0] _foreach_add(alpha)   d = fma(wd, p, g)             (a new tensor: .grad keeps g); else d = g
//   _foreach_lerp_                  m = lerp(m, d, 1 - b1)        (|w| < 0.5: fma(w, d - m, m); else fma(-(d - m), 1 - w, d))
//   _foreach_mul_, _foreach_addcmul_  v = fma(1 - b2, d * d, v * b2)
//   _foreach_sqrt, div_, add_       q = sqrt(v) / bc2_sqrt + eps  (three roundings)
//   _foreach_addcdiv_               p = fma(step_size, m / q, p)
//   step_size = (lr / (1 - b1^t)) * -1 and bc2_sqrt = (1 - b2^t) ** 0.5 are Python doubles that torch rounds to fp32.  The
//   per-(b1, b2) fp64 table holds ((1 - b2^t) ** 0.5, 1 - b1^t) as Python computes them; the kernel forms -(lr / bc1) in
//   IEEE fp64 from the group's lr, so a scheduler's lr is never frozen into a captured launch.
// SGD (maximize off):
//   [wd != 0] _foreach_add(alpha)   d = fma(wd, p, g)             (a new tensor); else d = g
//   [momentum != 0] first step      buf = d                        (torch's clone; first = the device step is 0)
//                   later steps     buf = fma(1 - dampening, d, buf * momentum)
//                   nesterov        d = fma(momentum, buf, d)      (in place on .grad when wd == 0, as torch does)
//                   else            d = buf
//   _foreach_add_(alpha=-lr)        p = fma(-lr, d, p)
//   SGD's StepGroup: beta1 = momentum, om_beta1 = 1 - dampening, decay = wd, flags: decay, nesterov (bit 2), momentum (4).
//   Every SGD tensor has a device step so that "the buffer is set" survives a skipped step; its buffer starts as zeros.
//
// The body and the packing live in optim.cuh, which the captured optimiser tail (tail.cu) shares.
// Work split: multi_tensor.cuh's chunks, launches and arrival counter.  Every CTA reads the step counters, so they are
// advanced only by the last CTA to finish.  A nonzero found_inf leaves p, the state and every step as they are.
#include "optim.cuh"

namespace qagnn {

namespace {

// one named kernel per rule, so profiles and SASS dumps tell them apart
__global__ void __launch_bounds__(kThreads) radam_kernel(const __grid_constant__ StepArgs a) { step_body<Rule::kRAdam>(a); }
__global__ void __launch_bounds__(kThreads) adamw_kernel(const __grid_constant__ StepArgs a) { step_body<Rule::kAdamW>(a); }
__global__ void __launch_bounds__(kThreads) adam_kernel(const __grid_constant__ StepArgs a) { step_body<Rule::kAdam>(a); }
__global__ void __launch_bounds__(kThreads) sgd_kernel(const __grid_constant__ StepArgs a) { step_body<Rule::kSgd>(a); }

template <Rule R>
int32_t launch(const StepArgs& a, cudaStream_t st) {
  const unsigned blocks = mt::launch_blocks(a.chunk_end[a.n - 1]);
  if constexpr (R == Rule::kRAdam)
    radam_kernel<<<blocks, kThreads, 0, st>>>(a);
  else if constexpr (R == Rule::kAdamW)
    adamw_kernel<<<blocks, kThreads, 0, st>>>(a);
  else if constexpr (R == Rule::kAdam)
    adam_kernel<<<blocks, kThreads, 0, st>>>(a);
  else
    sgd_kernel<<<blocks, kThreads, 0, st>>>(a);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

// The host side of qagnn_optim_step: validation, per-launch packing (512 tensors, 16 groups, an int32 chunk prefix) and the
// launches.  Only the groups the tensors use are checked.
template <Rule R>
int32_t step_all(int32_t n_tensors, void* const* params, void* const* grads, void* const* exp_avgs, void* const* exp_avg_sqs,
                 void* const* steps, const int64_t* numels, const int32_t* group_index, int32_t n_groups,
                 const GroupColumns& c, const float* found_inf, const float* grad_scale, int32_t* counter, cudaStream_t st) {
  if (n_tensors < 0 || n_groups < 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (n_tensors == 0) return QAGNN_OK;
  if (!tensors_valid<R>(n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index, n_groups) || !counter)
    return QAGNN_ERR_INVALID_ARGUMENT;
  for (int32_t i = 0; i < n_tensors; ++i) {
    const int32_t gi = group_index[i];
    if (!c.valid<R>(gi)) return QAGNN_ERR_INVALID_ARGUMENT;
    // SGD with momentum needs its buffer
    if (R == Rule::kSgd && numels[i] > 0 && c.beta1[gi] != 0.0 && !exp_avgs[i]) return QAGNN_ERR_INVALID_ARGUMENT;
  }
  static thread_local StepArgs a;  // 28 KB: kept off the stack
  a.table_len = c.table_len;
  a.found_inf = found_inf;
  a.grad_scale = grad_scale;
  a.counter = counter;
  return pack_launches(
      a, n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index,
      [&](int32_t slot, int32_t gi) { c.fill<R>(a.groups[slot], gi); }, [&](bool) { return launch<R>(a, st); });
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_optim_step(int32_t rule, int32_t n_tensors, void* const* params, void* const* grads,
                                    void* const* exp_avgs, void* const* exp_avg_sqs, void* const* steps, const int64_t* numels,
                                    const int32_t* group_index, int32_t n_groups, const double* lr, const double* weight_decay,
                                    const double* beta1, const double* beta2, const double* eps, const int32_t* rule_flag,
                                    void* const* step_tables, int64_t table_len, const float* found_inf,
                                    const float* grad_scale, int32_t* counter, void* stream) {
  const GroupColumns c{lr, weight_decay, beta1, beta2, eps, rule_flag, step_tables, table_len};
  return with_rule(rule, [&](auto r) {
    return step_all<decltype(r)::value>(n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index, n_groups,
                                        c, found_inf, grad_scale, counter, (cudaStream_t)stream);
  });
}
