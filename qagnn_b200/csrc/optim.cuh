// The optimiser step's kernel body and launch packing, shared by the eager step (optim.cu) and the captured optimiser tail
// (tail.cu).  optim.cu states the update rules and their rounding.
#pragma once

#include <type_traits>

#include "multi_tensor.cuh"

namespace qagnn {

using mt::kChunk;
using mt::kMaxTensors;
using mt::kThreads;
constexpr int kMaxGroups = 16;  // distinct param groups per launch

// kAdam and kSgd are torch.optim.Adam's and SGD's default CUDA (foreach) updates
enum class Rule { kRAdam, kAdamW, kAdam, kSgd };
enum : int32_t { kKindNone = 0, kKindSgd = 1, kKindRect = 2 };
// bit 2 is the rule's own: RAdam's degenerated_to_sgd, AdamW's correct_bias, SGD's nesterov; bit 4 is SGD's momentum != 0
enum : int32_t { kFlagDecay = 1, kFlagDegenerated = 2, kFlagCorrectBias = 2, kFlagNesterov = 2, kFlagMomentum = 4 };

// Adam and SGD take their weight decay as torch's `grads + wd * params`, on the gradient before the update
constexpr bool decays_gradient(Rule r) { return r == Rule::kAdam || r == Rule::kSgd; }

struct StepGroup {
  // [table_len, 2] for t = row.  RAdam: (1.0 if rho_t >= 5 else 0.0, step size s); AdamW: (sqrt(1 - b2^t), 1 - b1^t);
  // Adam: ((1 - b2^t) ** 0.5, 1 - b1^t); SGD: none (null)
  const double* table;
  double lr;
  // fp32 of b1, 1 - b1, b2, 1 - b2, eps, -wd*lr; Adam's decay is wd.  SGD: beta1 = momentum, om_beta1 = 1 - dampening,
  // decay = wd, and beta2, om_beta2 and eps unused
  float beta1, om_beta1, beta2, om_beta2, eps, decay;
  int32_t flags;
};

struct StepArgs {
  float* p[kMaxTensors];
  float* g[kMaxTensors];
  float* m[kMaxTensors];
  float* v[kMaxTensors];
  int64_t* step[kMaxTensors];
  int64_t numel[kMaxTensors];
  int32_t chunk_end[kMaxTensors];  // inclusive prefix sum of the tensors' chunk counts
  uint8_t group[kMaxTensors];
  StepGroup groups[kMaxGroups];
  int64_t table_len;
  const float* found_inf;
  const float* grad_scale;
  int32_t* counter;
  int32_t n;
};
static_assert(sizeof(StepArgs) <= 32764, "optimiser kernel parameters exceed the 32764 bytes sm_90 accepts");

// The captured tail's per-call block in device memory: what a graph replay must not freeze.  The host writes it before every
// replay (qagnn_step_tail_fill); n_groups StepGroup follow it.
struct TailBlock {
  double growth_factor, backoff_factor;  // GradScaler's, as torch._amp_update_scale_ takes them
  int64_t table_len;
  float max_norm;                        // the clip threshold, rounded to fp32 as clip_grad_norm_ rounds it
  int32_t growth_interval;
  int32_t n_groups;
  int32_t pad;
};
static_assert(sizeof(TailBlock) % alignof(StepGroup) == 0, "the groups follow the block header");

__host__ __device__ __forceinline__ const StepGroup* block_groups(const TailBlock* b) {
  return reinterpret_cast<const StepGroup*>(b + 1);
}

// The tail's step (pass 2): StepArgs with the groups read from the block and the clip, the scale update and found_inf's reset
struct TailArgs {
  float* p[kMaxTensors];
  float* g[kMaxTensors];
  float* m[kMaxTensors];
  float* v[kMaxTensors];
  int64_t* step[kMaxTensors];
  int64_t numel[kMaxTensors];
  int32_t chunk_end[kMaxTensors];
  uint8_t group[kMaxTensors];
  int32_t slot_group[kMaxGroups];  // the block's group of each per-launch slot
  const TailBlock* block;
  float* found_inf;        // pass 1's inf check, null without a scaler: the last launch's last CTA clears it
  float* scale;            // GradScaler's _scale and _growth_tracker, null without a scaler
  int32_t* growth_tracker;
  const float* coef;       // pass 1's clip coefficient, null without a clip
  int32_t* counter;
  int32_t n;
  int32_t last;            // the call's last launch: it updates the scale
};
static_assert(sizeof(TailArgs) <= 32764, "tail kernel parameters exceed the 32764 bytes sm_90 accepts");

namespace {

struct Coef {
  float inv, coef, b1, om_b1, b2, om_b2, eps, decay, step;
  float bc2;     // Adam: (float)bias_correction2_sqrt
  int32_t kind;  // AdamW, Adam and SGD always write p: kKindRect
  bool unscale, clip, write_g, has_decay, skip;
  bool momentum, nesterov, first;  // SGD: momentum != 0, nesterov, the momentum buffer not yet set (device step 0)
};

// at::lerp as torch's CUDA kernels compile it, fp32 weight w: self + w * (end - self) for |w| < 0.5, else
// end - (end - self) * (1 - w), each one FMA
__device__ __forceinline__ float torch_lerp(float self, float end, float w) {
  const float diff = __fsub_rn(end, self);
  return fabsf(w) < 0.5f ? __fmaf_rn(w, diff, self) : __fmaf_rn(-diff, __fsub_rn(1.f, w), end);
}

template <Rule R>
__device__ __forceinline__ void step_elem(float& p, float& g, float& m, float& v, const Coef& k) {
  if (k.unscale) g = __fmul_rn(g, k.inv);
  if (k.clip) g = __fmul_rn(g, k.coef);
  if (k.skip) return;
  if constexpr (R == Rule::kRAdam) {
    v = __fmaf_rn(k.om_b2, __fmul_rn(g, g), __fmul_rn(v, k.b2));
    m = __fmaf_rn(g, k.om_b1, __fmul_rn(m, k.b1));
    if (k.kind == kKindNone) return;
    if (k.has_decay) p = __fmaf_rn(p, k.decay, p);
    if (k.kind == kKindRect)
      p = __fmaf_rn(k.step, __fdiv_rn(m, __fadd_rn(__fsqrt_rn(v), k.eps)), p);
    else
      p = __fmaf_rn(m, k.step, p);
  } else if constexpr (R == Rule::kAdamW) {
    m = __fmaf_rn(g, k.om_b1, __fmul_rn(m, k.b1));
    v = __fmaf_rn(k.om_b2, __fmul_rn(g, g), __fmul_rn(v, k.b2));
    p = __fmaf_rn(k.step, __fdiv_rn(m, __fadd_rn(__fsqrt_rn(v), k.eps)), p);
    if (k.has_decay) p = __fmaf_rn(p, k.decay, p);
  } else if constexpr (R == Rule::kAdam) {
    const float d = k.has_decay ? __fmaf_rn(k.decay, p, g) : g;  // a new tensor: .grad keeps g
    m = torch_lerp(m, d, k.om_b1);
    v = __fmaf_rn(k.om_b2, __fmul_rn(d, d), __fmul_rn(v, k.b2));
    p = __fmaf_rn(k.step, __fdiv_rn(m, __fadd_rn(__fdiv_rn(__fsqrt_rn(v), k.bc2), k.eps)), p);
  } else {
    float d = k.has_decay ? __fmaf_rn(k.decay, p, g) : g;
    if (k.momentum) {
      m = k.first ? d : __fmaf_rn(k.om_b1, d, __fmul_rn(m, k.b1));
      if (k.nesterov) {
        d = __fmaf_rn(k.b1, m, d);
        if (!k.has_decay) g = d;  // torch adds into .grad itself when nothing decayed it into a new tensor
      } else {
        d = m;
      }
    }
    p = __fmaf_rn(k.step, d, p);
  }
}

template <Rule R>
__device__ __forceinline__ void step_scalar(float* p, float* g, float* m, float* v, int64_t j, const Coef& k) {
  if constexpr (R == Rule::kSgd) {  // no second moment, and a momentum buffer only with momentum != 0
    float pp = p[j], gg = g[j], mm = k.momentum ? m[j] : 0.f, vv = 0.f;
    step_elem<R>(pp, gg, mm, vv, k);
    if (k.write_g) g[j] = gg;
    if (k.skip) return;
    if (k.momentum) m[j] = mm;
    p[j] = pp;
  } else {
    float pp = p[j], gg = g[j], mm = m[j], vv = v[j];
    step_elem<R>(pp, gg, mm, vv, k);
    if (k.write_g) g[j] = gg;
    if (k.skip) return;
    m[j] = mm;
    v[j] = vv;
    if (k.kind != kKindNone) p[j] = pp;
  }
}

__device__ __forceinline__ const StepGroup& group_of(const StepArgs& a, int i) { return a.groups[a.group[i]]; }
__device__ __forceinline__ const StepGroup& group_of(const TailArgs& a, int i) {
  return block_groups(a.block)[a.slot_group[a.group[i]]];
}
__device__ __forceinline__ int64_t table_len_of(const StepArgs& a) { return a.table_len; }
__device__ __forceinline__ int64_t table_len_of(const TailArgs& a) { return a.block->table_len; }

// torch._amp_update_scale_: one call's scale update from its inf check
__device__ __forceinline__ void update_scale(float* scale, int32_t* growth_tracker, bool found_inf, const TailBlock& b) {
  if (found_inf) {
    *scale = __double2float_rn(__dmul_rn((double)*scale, b.backoff_factor));
    *growth_tracker = 0;
    return;
  }
  const int32_t successful = *growth_tracker + 1;
  if (successful == b.growth_interval) {
    const float grown = __double2float_rn(__dmul_rn((double)*scale, b.growth_factor));
    if (isfinite(grown)) *scale = grown;  // never grows past fp32 to inf
    *growth_tracker = 0;
  } else {
    *growth_tracker = successful;
  }
}

template <Rule R, class A>
__device__ __forceinline__ void step_body(const A& a) {
  constexpr bool kTail = std::is_same<A, TailArgs>::value;
  Coef k;
  k.skip = a.found_inf != nullptr && *a.found_inf != 0.f;
  if constexpr (kTail) {
    k.inv = a.scale != nullptr ? __double2float_rn(__drcp_rn((double)*a.scale)) : 1.f;
    // Under a clip as GradScaler.unscale_ then the clip's scale, each of which leaves g alone at a factor of 1; without a
    // clip as the eager step's unscale, which always multiplies.
    k.unscale = a.scale != nullptr && (a.coef == nullptr || k.inv != 1.f);
    k.coef = a.coef != nullptr ? *a.coef : 1.f;
    k.clip = k.coef != 1.f;  // a NaN coefficient multiplies, as in clip_scale_kernel
  } else {
    k.unscale = a.grad_scale != nullptr;
    // GradScaler.unscale_: inv_scale = scale.double().reciprocal().float()
    k.inv = k.unscale ? __double2float_rn(__drcp_rn((double)*a.grad_scale)) : 1.f;
    k.coef = 1.f;
    k.clip = false;
  }
  k.write_g = k.unscale || k.clip;
  const bool unscale_or_clip = k.write_g;
  const int32_t total = a.chunk_end[a.n - 1];
  for (int32_t c = blockIdx.x; c < total; c += gridDim.x) {
    const int i = mt::chunk_owner(a.chunk_end, a.n, c);
    const int64_t c0 = (int64_t)(c - (i ? a.chunk_end[i - 1] : 0)) * kChunk;
    const int64_t n = min(kChunk, a.numel[i] - c0);
    const StepGroup& gr = group_of(a, i);
    k.b1 = gr.beta1; k.om_b1 = gr.om_beta1; k.b2 = gr.beta2; k.om_b2 = gr.om_beta2; k.eps = gr.eps; k.decay = gr.decay;
    k.kind = kKindNone;
    k.step = 0.f;
    if constexpr (R == Rule::kSgd) {
      k.kind = kKindRect;
      k.step = __double2float_rn(-gr.lr);  // add_(grads, alpha=-lr)
      k.momentum = (gr.flags & kFlagMomentum) != 0;
      k.nesterov = (gr.flags & kFlagNesterov) != 0;
      k.first = !k.skip && *a.step[i] <= 0;
      k.write_g = unscale_or_clip || (!k.skip && k.momentum && k.nesterov && (gr.flags & kFlagDecay) == 0);
    } else if (!k.skip) {
      const int64_t t = min(max(*a.step[i] + 1, (int64_t)0), table_len_of(a) - 1);
      const double t0 = gr.table[2 * t], t1 = gr.table[2 * t + 1];
      if constexpr (R == Rule::kRAdam) {
        k.kind = t0 != 0.0 ? kKindRect : (gr.flags & kFlagDegenerated) ? kKindSgd : kKindNone;
        k.step = __double2float_rn(__dmul_rn(-t1, gr.lr));
      } else if constexpr (R == Rule::kAdamW) {
        // value=-step_size with step_size = lr * math.sqrt(bias_correction2) / bias_correction1, or lr
        k.kind = kKindRect;
        k.step = __double2float_rn(-((gr.flags & kFlagCorrectBias) ? __ddiv_rn(__dmul_rn(gr.lr, t0), t1) : gr.lr));
      } else {
        // step_size = (lr / bias_correction1) * -1 in Python doubles; addcdiv_ and div_ round it and bias_correction2_sqrt
        k.kind = kKindRect;
        k.step = __double2float_rn(-__ddiv_rn(gr.lr, t1));
        k.bc2 = __double2float_rn(t0);
      }
    }
    k.has_decay = (gr.flags & kFlagDecay) != 0;
    if (k.skip && !k.write_g) continue;
    float* p = a.p[i] + c0;
    float* g = a.g[i] + c0;
    float* m = a.m[i] + c0;  // SGD's v, and m without momentum, are null: offset here but never dereferenced
    float* v = a.v[i] + c0;
    const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                           reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    int64_t done = 0;
    if (aligned) {
      const int64_t n4 = n >> 2;
      for (int64_t j = threadIdx.x; j < n4; j += kThreads) {
        float4 pp = reinterpret_cast<float4*>(p)[j], gg = reinterpret_cast<float4*>(g)[j];
        float4 mm, vv;
        if constexpr (R == Rule::kSgd) {
          mm = k.momentum ? reinterpret_cast<float4*>(m)[j] : make_float4(0.f, 0.f, 0.f, 0.f);
          vv = mm;  // unused
        } else {
          mm = reinterpret_cast<float4*>(m)[j], vv = reinterpret_cast<float4*>(v)[j];
        }
        step_elem<R>(pp.x, gg.x, mm.x, vv.x, k);
        step_elem<R>(pp.y, gg.y, mm.y, vv.y, k);
        step_elem<R>(pp.z, gg.z, mm.z, vv.z, k);
        step_elem<R>(pp.w, gg.w, mm.w, vv.w, k);
        if (k.write_g) reinterpret_cast<float4*>(g)[j] = gg;
        if (k.skip) continue;
        if constexpr (R == Rule::kSgd) {
          if (k.momentum) reinterpret_cast<float4*>(m)[j] = mm;
        } else {
          reinterpret_cast<float4*>(m)[j] = mm;
          reinterpret_cast<float4*>(v)[j] = vv;
        }
        if (k.kind != kKindNone) reinterpret_cast<float4*>(p)[j] = pp;
      }
      done = n4 << 2;
    }
    for (int64_t j = done + threadIdx.x; j < n; j += kThreads) step_scalar<R>(p, g, m, v, j, k);
  }
  // the last CTA to arrive advances the step counters: every CTA has read them by then
  if (!mt::last_to_arrive(a.counter)) return;
  if (!k.skip)
    for (int i = threadIdx.x; i < a.n; i += kThreads) *a.step[i] += 1;
  if constexpr (kTail) {
    // every CTA of every launch of this call has read the scale and found_inf by now
    if (a.last && a.scale != nullptr && threadIdx.x == 0) {
      update_scale(a.scale, a.growth_tracker, k.skip, *a.block);
      *a.found_inf = 0.f;
    }
  }
  if (threadIdx.x == 0) *a.counter = 0;
}

// Fills the per-launch copy of a group from the host doubles, rounding each scalar as torch rounds a Python float.  SGD
// passes momentum as b1 and dampening as b2.
template <Rule R>
void fill_group(StepGroup& gr, double lr, double wd, double b1, double b2, double eps, int32_t flags, const double* table) {
  gr.table = table;
  gr.lr = lr;
  gr.beta1 = (float)b1;
  gr.om_beta1 = (float)(1.0 - (R == Rule::kSgd ? b2 : b1));
  gr.beta2 = (float)b2;
  gr.om_beta2 = (float)(1.0 - b2);
  gr.eps = (float)eps;
  gr.decay = (float)(decays_gradient(R) ? wd : -wd * lr);
  gr.flags = flags;
}

// A group's flags: RAdam, Adam and SGD decay when wd != 0 (before their update), AdamW when wd > 0 (after); rule_flag is
// RAdam's degenerated_to_sgd, AdamW's correct_bias or SGD's nesterov (Adam has none); b1 is SGD's momentum
template <Rule R>
int32_t group_flags(double wd, int32_t rule_flag, double b1) {
  const int32_t decay = (R == Rule::kAdamW ? wd > 0.0 : wd != 0.0) ? kFlagDecay : 0;
  if constexpr (R == Rule::kAdam) return decay;
  if constexpr (R == Rule::kSgd) return decay | (rule_flag ? kFlagNesterov : 0) | (b1 != 0.0 ? kFlagMomentum : 0);
  return decay | (rule_flag ? (R == Rule::kRAdam ? kFlagDegenerated : kFlagCorrectBias) : 0);
}

// One call's per-group hyperparameter columns as qagnn_optim_step and qagnn_step_tail_fill take them: the Python doubles, the
// rule's per-group flag (group_flags) and the device step tables of table_len rows, which SGD does without
struct GroupColumns {
  const double *lr, *weight_decay, *beta1, *beta2, *eps;
  const int32_t* rule_flag;
  void* const* step_tables;
  int64_t table_len;

  // Group gi as the rule accepts it: every column given, and betas in [0, 1) with a step table of two rows or more, or for
  // SGD a finite momentum >= 0 and a finite dampening
  template <Rule R>
  bool valid(int32_t gi) const {
    if (!lr || !weight_decay || !beta1 || !beta2 || !eps || !rule_flag) return false;
    const double b1 = beta1[gi], b2 = beta2[gi];
    if constexpr (R == Rule::kSgd) return b1 >= 0.0 && b1 < INFINITY && b2 > -INFINITY && b2 < INFINITY;
    return step_tables && table_len >= 2 && step_tables[gi] && b1 >= 0.0 && b1 < 1.0 && b2 >= 0.0 && b2 < 1.0;
  }

  // Fills the per-launch copy of group gi
  template <Rule R>
  void fill(StepGroup& gr, int32_t gi) const {
    fill_group<R>(gr, lr[gi], weight_decay[gi], beta1[gi], beta2[gi], eps[gi],
                  group_flags<R>(weight_decay[gi], rule_flag[gi], beta1[gi]),
                  R == Rule::kSgd ? nullptr : (const double*)step_tables[gi]);
  }
};

// Checks one step's tensor list: group indices in range, a step counter per tensor, data pointers for non-empty tensors.
// SGD has no exp_avg_sqs, and exp_avgs[i] (its momentum buffer) may be null; where it must not be, its caller checks.
template <Rule R>
bool tensors_valid(int32_t n_tensors, void* const* params, void* const* grads, void* const* exp_avgs, void* const* exp_avg_sqs,
                   void* const* steps, const int64_t* numels, const int32_t* group_index, int32_t n_groups) {
  constexpr bool kSgd = R == Rule::kSgd;
  if (!params || !grads || !exp_avgs || (!kSgd && !exp_avg_sqs) || !steps || !numels || !group_index || n_groups <= 0)
    return false;
  for (int32_t i = 0; i < n_tensors; ++i) {
    const int32_t gi = group_index[i];
    if (gi < 0 || gi >= n_groups || !steps[i] || numels[i] < 0 || mt::chunk_count(numels[i]) > INT32_MAX) return false;
    if (numels[i] > 0 && (!params[i] || !grads[i] || (!kSgd && (!exp_avgs[i] || !exp_avg_sqs[i])))) return false;
  }
  return true;
}

// Packs the tensors into launches of a (512 tensors, 16 groups, an int32 chunk prefix).  slot(s, gi) fills per-launch slot
// s for group gi; launch(last) sends a full launch, and the final one with last = true.
template <class A, class Slot, class Launch>
int32_t pack_launches(A& a, int32_t n_tensors, void* const* params, void* const* grads, void* const* exp_avgs,
                      void* const* exp_avg_sqs, void* const* steps, const int64_t* numels, const int32_t* group_index,
                      Slot slot_fill, Launch launch) {
  int32_t slot_of[kMaxGroups];  // global group of each per-launch slot
  int32_t n_slots = 0;
  a.n = 0;
  int64_t chunks = 0;
  for (int32_t i = 0; i < n_tensors; ++i) {
    const int32_t gi = group_index[i];
    const int64_t nc = mt::chunk_count(numels[i]);
    int32_t slot = -1;
    for (int32_t s = 0; s < n_slots; ++s)
      if (slot_of[s] == gi) slot = s;
    // a full launch (tensors, groups or the int32 chunk prefix) goes out first
    if (mt::launch_full(a.n, chunks, nc) || (slot < 0 && n_slots == kMaxGroups)) {
      QAGNN_RETURN_IF(launch(false));
      a.n = 0;
      n_slots = 0;
      chunks = 0;
      slot = -1;
    }
    if (slot < 0) {
      slot = n_slots++;
      slot_of[slot] = gi;
      slot_fill(slot, gi);
    }
    const int32_t j = a.n++;
    a.p[j] = (float*)params[i];
    a.g[j] = (float*)grads[i];
    a.m[j] = (float*)exp_avgs[i];
    a.v[j] = exp_avg_sqs ? (float*)exp_avg_sqs[i] : nullptr;
    a.step[j] = (int64_t*)steps[i];
    a.numel[j] = numels[i];
    a.group[j] = (uint8_t)slot;
    chunks += nc;
    a.chunk_end[j] = (int32_t)chunks;
  }
  return launch(true);
}

// Calls f(std::integral_constant<Rule, R>()) for the Rule of a QAGNN_RULE_* value; QAGNN_ERR_INVALID_ARGUMENT for any other
template <class F>
int32_t with_rule(int32_t rule, F f) {
  switch (rule) {
    case QAGNN_RULE_RADAM: return f(std::integral_constant<Rule, Rule::kRAdam>());
    case QAGNN_RULE_ADAMW: return f(std::integral_constant<Rule, Rule::kAdamW>());
    case QAGNN_RULE_ADAM: return f(std::integral_constant<Rule, Rule::kAdam>());
    case QAGNN_RULE_SGD: return f(std::integral_constant<Rule, Rule::kSgd>());
    default: return QAGNN_ERR_INVALID_ARGUMENT;
  }
}

}  // namespace

}  // namespace qagnn
