// Multi-tensor optimiser steps over every fp32 tensor of one device in one launch, with GradScaler's inf skip and unscale taken
// on the device: the reference's RAdam (utils/optimization_utils.py; qagnn_radam_step) and transformers' AdamW (3.4.0, the
// version the reference pins; qagnn_adamw_step).  One kernel body serves both, the update rule a template parameter.
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
// torch.optim.Adam and SGD (Rule::kAdam, kSgd) run on the same body; optim_torch.cu states their rules and rounding.
//
// The body, the packing and the entries' host side live in optim.cuh, which torch's Adam and SGD (optim_torch.cu) and the
// captured optimiser tail (tail.cu) share.
// Work split: multi_tensor.cuh's chunks, launches and arrival counter.  Every CTA reads the step counters, so they are
// advanced only by the last CTA to finish.  A nonzero found_inf leaves p, m, v and every step as they are.
#include "optim.cuh"

namespace qagnn {

namespace {

// one named kernel per rule, so profiles and SASS dumps tell them apart
__global__ void __launch_bounds__(kThreads) radam_kernel(const __grid_constant__ StepArgs a) { step_body<Rule::kRAdam>(a); }
__global__ void __launch_bounds__(kThreads) adamw_kernel(const __grid_constant__ StepArgs a) { step_body<Rule::kAdamW>(a); }

template <Rule R>
int32_t launch(const StepArgs& a, cudaStream_t st) {
  const unsigned blocks = mt::launch_blocks(a.chunk_end[a.n - 1]);
  if constexpr (R == Rule::kRAdam)
    radam_kernel<<<blocks, kThreads, 0, st>>>(a);
  else
    adamw_kernel<<<blocks, kThreads, 0, st>>>(a);
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
  return step_all<Rule::kRAdam>(n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index, n_groups, lr,
                                weight_decay, beta1, beta2, eps, degenerated_to_sgd, step_tables, table_len, found_inf,
                                grad_scale, counter,
                                [&](const StepArgs& a) { return launch<Rule::kRAdam>(a, (cudaStream_t)stream); });
}

extern "C" int32_t qagnn_adamw_step(int32_t n_tensors, void* const* params, void* const* grads, void* const* exp_avgs,
                                    void* const* exp_avg_sqs, void* const* steps, const int64_t* numels,
                                    const int32_t* group_index, int32_t n_groups, const double* lr, const double* weight_decay,
                                    const double* beta1, const double* beta2, const double* eps, const int32_t* correct_bias,
                                    void* const* step_tables, int64_t table_len, const float* found_inf,
                                    const float* grad_scale, int32_t* counter, void* stream) {
  return step_all<Rule::kAdamW>(n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index, n_groups, lr,
                                weight_decay, beta1, beta2, eps, correct_bias, step_tables, table_len, found_inf,
                                grad_scale, counter,
                                [&](const StepArgs& a) { return launch<Rule::kAdamW>(a, (cudaStream_t)stream); });
}
