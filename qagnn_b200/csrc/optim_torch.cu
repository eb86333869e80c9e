// torch.optim.Adam and torch.optim.SGD as torch 2.11 steps them by default on CUDA (the foreach implementation,
// _multi_tensor_adam / _multi_tensor_sgd), over every fp32 tensor of one device in one launch, with GradScaler's inf skip
// and unscale taken on the device (qagnn_adam_step, qagnn_sgd_step; qagnn_b200.optim.Adam / SGD).  optim.cuh's body runs
// them, as it runs RAdam and AdamW (optim.cu), and this file also holds their pass 2 of the captured tail (tail.cu).
//
// Per element, t = the tensor's step + 1, each line one fp32 operation in torch's order.  Established on the H100 against
// torch's own foreach ops: `a + alpha * x` (add(alpha), addcmul, addcdiv) and both branches of at::lerp are one FMA each,
// sqrt is correctly rounded, and the division by a scalar list (bias_correction2_sqrt) is a true fp32 division, not a
// multiply by a reciprocal.  The GPU tests compare every state tensor with torch's CUDA step bit for bit.
//   [unscale]  g = g * inv_scale                                  (GradScaler.unscale_; written back to .grad)
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
// A nonzero found_inf leaves p, the state and every step as they are.
#include "optim.cuh"

namespace qagnn {

namespace {

__global__ void __launch_bounds__(kThreads) adam_kernel(const __grid_constant__ StepArgs a) { step_body<Rule::kAdam>(a); }
__global__ void __launch_bounds__(kThreads) sgd_kernel(const __grid_constant__ StepArgs a) { step_body<Rule::kSgd>(a); }
__global__ void __launch_bounds__(kThreads) tail_adam_kernel(const __grid_constant__ TailArgs a) { step_body<Rule::kAdam>(a); }
__global__ void __launch_bounds__(kThreads) tail_sgd_kernel(const __grid_constant__ TailArgs a) { step_body<Rule::kSgd>(a); }

template <Rule R>
int32_t launch(const StepArgs& a, cudaStream_t st) {
  const unsigned blocks = mt::launch_blocks(a.chunk_end[a.n - 1]);
  if constexpr (R == Rule::kAdam)
    adam_kernel<<<blocks, kThreads, 0, st>>>(a);
  else
    sgd_kernel<<<blocks, kThreads, 0, st>>>(a);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

}  // namespace

int32_t launch_torch_tail_step(Rule rule, const TailArgs& a, cudaStream_t st) {
  const unsigned blocks = mt::launch_blocks(a.chunk_end[a.n - 1]);
  if (rule == Rule::kAdam)
    tail_adam_kernel<<<blocks, kThreads, 0, st>>>(a);
  else if (rule == Rule::kSgd)
    tail_sgd_kernel<<<blocks, kThreads, 0, st>>>(a);
  else
    return QAGNN_ERR_INVALID_ARGUMENT;
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_adam_step(int32_t n_tensors, void* const* params, void* const* grads, void* const* exp_avgs,
                                   void* const* exp_avg_sqs, void* const* steps, const int64_t* numels,
                                   const int32_t* group_index, int32_t n_groups, const double* lr, const double* weight_decay,
                                   const double* beta1, const double* beta2, const double* eps, const int32_t* rule_flag,
                                   void* const* step_tables, int64_t table_len, const float* found_inf,
                                   const float* grad_scale, int32_t* counter, void* stream) {
  return step_all<Rule::kAdam>(n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index, n_groups, lr,
                               weight_decay, beta1, beta2, eps, rule_flag, step_tables, table_len, found_inf, grad_scale,
                               counter, [&](const StepArgs& a) { return launch<Rule::kAdam>(a, (cudaStream_t)stream); });
}

extern "C" int32_t qagnn_sgd_step(int32_t n_tensors, void* const* params, void* const* grads, void* const* momentum_buffers,
                                  void* const* exp_avg_sqs, void* const* steps, const int64_t* numels,
                                  const int32_t* group_index, int32_t n_groups, const double* lr, const double* weight_decay,
                                  const double* momentum, const double* dampening, const double* eps,
                                  const int32_t* nesterov, void* const* step_tables, int64_t table_len,
                                  const float* found_inf, const float* grad_scale, int32_t* counter, void* stream) {
  return step_all<Rule::kSgd>(n_tensors, params, grads, momentum_buffers, exp_avg_sqs, steps, numels, group_index, n_groups,
                              lr, weight_decay, momentum, dampening, eps, nesterov, step_tables, table_len, found_inf,
                              grad_scale, counter,
                              [&](const StepArgs& a) { return launch<Rule::kSgd>(a, (cudaStream_t)stream); });
}
