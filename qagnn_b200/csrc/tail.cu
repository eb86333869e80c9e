// The recipe's optimiser tail, `scaler.unscale_(opt); clip_grad_norm_(...); scheduler.step(); scaler.step(opt);
// scaler.update()`, in two passes over the gradients that a CUDA graph can replay (qagnn_step_tail;
// qagnn_b200.optim.CapturedTail).  What a replay must not freeze (each group's lr, -wd*lr, eps, betas and step table, the clip
// threshold, GradScaler's factors) lives in a device block the host rewrites before every replay (qagnn_step_tail_fill).
//
// tail_norm_kernel (pass 1) is clip_norm_kernel's body over u = g * inv_scale, inv_scale = (float)(1 / (double)scale) as
// GradScaler.unscale_ forms it, with its summation order, total_norm and coefficient.  Any non-finite g (the scaled value,
// as torch._amp_foreach_non_finite_check_and_unscale_ tests it) sets found_inf to 1.  Without a clip the reference does not
// call unscale_, and the pass is GradScaler._check_inf_per_device: inv_scale 1 and no norm.  It writes nothing per element.
//
// tail_{radam,adamw,adam,sgd}_kernel (pass 2) are optim.cuh's step body with the groups read from the block.  Each element
// takes c = (g * inv) * coef, the same two fp32 multiplies as unscale_ then clip_scale_kernel, each left out at a factor of 1 as
// they leave it; c goes back to .grad when either factor applies, found_inf or not.  Without a clip the step unscales as the
// eager step does under GradScaler.step.  The last CTA of the call's last launch then applies torch._amp_update_scale_ to
// the scaler's own tensors and clears found_inf.
//
// Traffic per fp32 parameter when clipping under a scaler: pass 1 reads g (4 bytes); pass 2 reads p, g, m, v and writes
// them (32).  The eager tail moves 48: unscale 8, norm 4, clip scale 8, step 28.
#include "clip.cuh"
#include "optim.cuh"

namespace qagnn {

namespace {

struct TailNormArgs {
  NormArgs a;
  const TailBlock* block;
  const float* grad_scale;  // null: inv_scale = 1
  float* found_inf;         // null: no check
};

__global__ void __launch_bounds__(kThreads) tail_norm_kernel(const __grid_constant__ TailNormArgs t) {
  const float inv = t.grad_scale != nullptr ? __double2float_rn(__drcp_rn((double)*t.grad_scale)) : 1.f;
  bool bad = false;
  norm_body(
      t.a,
      [&](float x) {
        bad |= !isfinite(x);
        return __fmul_rn(x, inv);
      },
      [&] { return t.block->max_norm; });
  if (bad && t.found_inf != nullptr) *t.found_inf = 1.f;  // every writer stores the same value
}

__global__ void __launch_bounds__(kThreads) tail_radam_kernel(const __grid_constant__ TailArgs a) { step_body<Rule::kRAdam>(a); }
__global__ void __launch_bounds__(kThreads) tail_adamw_kernel(const __grid_constant__ TailArgs a) { step_body<Rule::kAdamW>(a); }
__global__ void __launch_bounds__(kThreads) tail_adam_kernel(const __grid_constant__ TailArgs a) { step_body<Rule::kAdam>(a); }
__global__ void __launch_bounds__(kThreads) tail_sgd_kernel(const __grid_constant__ TailArgs a) { step_body<Rule::kSgd>(a); }

int64_t block_bytes(int32_t n_groups) {
  return n_groups <= 0 ? -1 : (int64_t)sizeof(TailBlock) + (int64_t)n_groups * (int64_t)sizeof(StepGroup);
}

template <Rule R>
int32_t launch_step(const TailArgs& a, cudaStream_t st) {
  const unsigned blocks = mt::launch_blocks(a.chunk_end[a.n - 1]);
  if constexpr (R == Rule::kRAdam)
    tail_radam_kernel<<<blocks, kThreads, 0, st>>>(a);
  else if constexpr (R == Rule::kAdamW)
    tail_adamw_kernel<<<blocks, kThreads, 0, st>>>(a);
  else if constexpr (R == Rule::kAdam)
    tail_adam_kernel<<<blocks, kThreads, 0, st>>>(a);
  else
    tail_sgd_kernel<<<blocks, kThreads, 0, st>>>(a);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

template <Rule R>
int32_t tail_all(int32_t n_tensors, void* const* params, void* const* grads, void* const* exp_avgs, void* const* exp_avg_sqs,
                 void* const* steps, const int64_t* numels, const int32_t* group_index, int32_t n_groups, int32_t n_norm,
                 void* const* norm_grads, const int64_t* norm_numels, int32_t clip, const void* block, double* slots,
                 int64_t n_slots, int32_t* counter, float* total_norm, float* coef, float* found_inf, float* scale,
                 int32_t* growth_tracker, void* stream) {
  if (n_tensors <= 0 || !block || !counter ||
      !tensors_valid<R>(n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index, n_groups))
    return QAGNN_ERR_INVALID_ARGUMENT;
  if ((scale != nullptr) != (growth_tracker != nullptr) || (scale != nullptr && found_inf == nullptr))
    return QAGNN_ERR_INVALID_ARGUMENT;
  cudaStream_t st = (cudaStream_t)stream;
  const TailBlock* blk = (const TailBlock*)block;
  if (clip || scale) {
    const int64_t need = slot_count(n_norm, norm_numels);
    if (need < 0 || (n_norm > 0 && !norm_grads) || (need > 0 && !slots) || (clip && (!total_norm || !coef)))
      return QAGNN_ERR_INVALID_ARGUMENT;
    for (int32_t i = 0; i < n_norm; ++i)
      if (norm_numels[i] > 0 && !norm_grads[i]) return QAGNN_ERR_INVALID_ARGUMENT;
    if (n_slots < need) return QAGNN_ERR_WORKSPACE;
    static thread_local TailNormArgs na;
    na.a.slots = slots;
    na.a.total = need;
    na.a.max_norm = 0.f;  // read from the block
    na.a.total_norm = total_norm;
    na.a.coef = coef;
    na.block = blk;
    na.grad_scale = clip ? scale : nullptr;
    na.found_inf = scale ? found_inf : nullptr;
    QAGNN_RETURN_IF(for_each_launch(n_norm, norm_grads, norm_numels, [&](const GradList& l, int64_t base, bool last) -> int32_t {
      na.a.l = l;
      na.a.base = base;
      na.a.counter = clip && last ? counter : nullptr;
      tail_norm_kernel<<<mt::launch_blocks(l.n ? l.chunk_end[l.n - 1] : 0), kThreads, 0, st>>>(na);
      QAGNN_CHECK_LAUNCH();
      return QAGNN_OK;
    }));
  }
  static thread_local TailArgs a;  // 28 KB: kept off the stack
  a.block = blk;
  a.found_inf = scale ? found_inf : nullptr;
  a.scale = scale;
  a.growth_tracker = growth_tracker;
  a.coef = clip ? coef : nullptr;
  a.counter = counter;
  return pack_launches(
      a, n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index,
      [&](int32_t slot, int32_t gi) { a.slot_group[slot] = gi; },
      [&](bool last) {
        a.last = last;
        return launch_step<R>(a, st);
      });
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" int64_t qagnn_step_tail_block_bytes(int32_t n_groups) { return block_bytes(n_groups); }

extern "C" int32_t qagnn_step_tail_fill(int32_t rule, int32_t n_groups, const double* lr, const double* weight_decay,
                                        const double* beta1, const double* beta2, const double* eps, const int32_t* rule_flag,
                                        void* const* step_tables, int64_t table_len, double max_norm, double growth_factor,
                                        double backoff_factor, int32_t growth_interval, void* block, int64_t n_bytes) {
  const GroupColumns c{lr, weight_decay, beta1, beta2, eps, rule_flag, step_tables, table_len};
  return with_rule(rule, [&](auto r) {
    constexpr Rule R = decltype(r)::value;
    if (n_groups <= 0 || !block) return QAGNN_ERR_INVALID_ARGUMENT;
    for (int32_t gi = 0; gi < n_groups; ++gi)
      if (!c.valid<R>(gi)) return QAGNN_ERR_INVALID_ARGUMENT;
    if (n_bytes < block_bytes(n_groups)) return QAGNN_ERR_WORKSPACE;
    TailBlock& b = *(TailBlock*)block;
    b.growth_factor = growth_factor;
    b.backoff_factor = backoff_factor;
    b.table_len = table_len;
    b.max_norm = (float)max_norm;
    b.growth_interval = growth_interval;
    b.n_groups = n_groups;
    b.pad = 0;
    StepGroup* groups = const_cast<StepGroup*>(block_groups(&b));
    for (int32_t gi = 0; gi < n_groups; ++gi) c.fill<R>(groups[gi], gi);
    return QAGNN_OK;
  });
}

extern "C" int32_t qagnn_step_tail(int32_t rule, int32_t n_tensors, void* const* params, void* const* grads,
                                   void* const* exp_avgs, void* const* exp_avg_sqs, void* const* steps, const int64_t* numels,
                                   const int32_t* group_index, int32_t n_groups, int32_t n_norm, void* const* norm_grads,
                                   const int64_t* norm_numels, int32_t clip, const void* block, double* slots, int64_t n_slots,
                                   int32_t* counter, float* total_norm, float* coef, float* found_inf, float* scale,
                                   int32_t* growth_tracker, void* stream) {
  return with_rule(rule, [&](auto r) {
    return tail_all<decltype(r)::value>(n_tensors, params, grads, exp_avgs, exp_avg_sqs, steps, numels, group_index, n_groups,
                                        n_norm, norm_grads, norm_numels, clip, block, slots, n_slots, counter, total_norm, coef,
                                        found_inf, scale, growth_tracker, stream);
  });
}
