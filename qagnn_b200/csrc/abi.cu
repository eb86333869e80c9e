// extern "C" entry points declared in include/qagnn_b200.h: the forward orchestration of
// GATConvE (modeling/modeling_qagnn.py:411-484) and QAGNN_Message_Passing (modeling_qagnn.py:53-95).
#include <atomic>
#include <mutex>
#include <cuda_bf16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace qagnn {

static std::atomic<long long> g_launches{0};
static thread_local char g_cuda_err[256] = "";

void note_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int32_t cuda_fail(cudaError_t e, const char* file, int line) {
  const char* base = strrchr(file, '/');
  snprintf(g_cuda_err, sizeof(g_cuda_err), "%s (%s:%d)", cudaGetErrorString(e), base ? base + 1 : file, line);
  return QAGNN_ERR_CUDA;
}

// ---- stage timing -----------------------------------------------------------------------------------
namespace {
constexpr int kProfMax = 8192;
struct ProfState {
  bool on = false;
  int n = 0;                       // recorded intervals
  cudaEvent_t ev[kProfMax][2];
  int created = 0;
  int stage[kProfMax];
  int open_idx[QAGNN_PROF_STAGES];
  std::mutex mu;  // the stage timers are process-wide diagnostics: calls from several host threads serialise here
} g_prof;
}  // namespace

void prof_begin(int stage, cudaStream_t st) {
  if (!g_prof.on) return;
  std::lock_guard<std::mutex> lk(g_prof.mu);
  if (!g_prof.on || g_prof.n >= kProfMax) { if (g_prof.on) g_prof.open_idx[stage] = -1; return; }
  const int i = g_prof.n++;
  if (i >= g_prof.created) {
    cudaEventCreate(&g_prof.ev[i][0]);
    cudaEventCreate(&g_prof.ev[i][1]);
    g_prof.created = i + 1;
  }
  g_prof.stage[i] = stage;
  g_prof.open_idx[stage] = i;
  cudaEventRecord(g_prof.ev[i][0], st);
}

void prof_end(int stage, cudaStream_t st) {
  if (!g_prof.on) return;
  std::lock_guard<std::mutex> lk(g_prof.mu);
  const int i = g_prof.open_idx[stage];
  if (i >= 0) cudaEventRecord(g_prof.ev[i][1], st);
}

WorkLayout make_work_layout(const qagnn_shape& s) {
  WorkLayout W;
  const size_t N = (size_t)s.N, D = (size_t)s.D, Ep = (size_t)(s.N + s.E), H = (size_t)s.H;
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += align_up(n * 4) / 4; return r; };
  const size_t DP = (size_t)head_dim_padded((int)(D / H));
  W.qkm = take(N * 3 * (D > H * DP ? D : H * DP));
  W.aggr = take(N * D);
  W.hmid = take(N * D);
  W.xa = take(N * D);
  W.xb = take(N * D);
  W.extra = take(N * D);
  W.sinb = take(N * (D / 2));
  const size_t half = N * D / 2 + 8;  // one bf16 plane [N, D], in floats
  W.hp_hi = take(half); W.hp_lo = take(half);
  W.ep_hi = take(half); W.ep_lo = take(half);
  W.xp_hi[0] = take(half); W.xp_lo[0] = take(half);
  W.xp_hi[1] = take(half); W.xp_lo[1] = take(half);
  W.ap_hi = take(half); W.ap_lo = take(half);
  W.mp_hi = take(half); W.mp_lo = take(half);
  const size_t sbh = N * (size_t)round_up8((int)(D / 2)) / 2 + 8;  // one bf16 plane [N, KSh], in floats
  W.sb_hi = take(sbh); W.sb_lo = take(sbh);
  const size_t xsh = N * (size_t)round_up8((int)(D + D / 2)) / 2 + 8;  // one bf16 plane [N, KS], in floats
  for (int i = 0; i < 3; ++i) { W.xs_hi[i] = take(xsh); W.xs_lo[i] = take(xsh); }
  const size_t Eps = (Ep + 3) / 4 * 4;  // per-head stride of the tiled path
  W.score = take(Eps * H);
  W.alpha = take(Eps * H);
  W.alpha2 = take(2 * Eps * H);
  W.total = o;
  return W;
}

namespace {

__global__ void node_feature_prologue_kernel(int64_t N, int D, int T, const int64_t* __restrict__ node_type,
                                             const float* __restrict__ node_score, const float* __restrict__ type_tab,
                                             const float* __restrict__ basis, float* __restrict__ extra,
                                             float* __restrict__ sinb) {
  // extra[v, :D/2] = GELU(emb_node_type(onehot(type)))  == row `type` of the folded table (:65-66)
  // sinb[v, j]     = sin(1.1^j * score[v])                                                (:70-72)
  const int Dh = D / 2;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N * Dh; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / Dh;
    const int j = (int)(i % Dh);
    int64_t t = node_type[v];
    t = t < 0 ? 0 : (t >= T ? T - 1 : t);
    extra[v * D + j] = type_tab[t * Dh + j];
    sinb[i] = sinf(basis[j] * node_score[v]);  // precise sinf: arguments reach ~1e4 * |score|
  }
}

// sin basis of the relevance score as split-bf16 planes [N, ld]: the A operand of emb_score on the tensor-core path (:70-73)
__global__ void sin_basis_planes_kernel(int64_t N, int Dh, int ld, const float* __restrict__ node_score,
                                        const float* __restrict__ basis, __nv_bfloat16* __restrict__ hi,
                                        __nv_bfloat16* __restrict__ lo) {
  const int half = Dh / 2;  // Dh even: two columns per thread
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N * half; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / half;
    const int j = (int)(i % half) * 2;
    const float sc = node_score[v];
    const float a = sinf(basis[j] * sc), b = sinf(basis[j + 1] * sc);  // precise sinf: arguments reach ~1e4 * |score|
    __nv_bfloat162 h2, l2;
    h2.x = __float2bfloat16_rn(a); h2.y = __float2bfloat16_rn(b);
    l2.x = __float2bfloat16_rn(a - __bfloat162float(h2.x)); l2.y = __float2bfloat16_rn(b - __bfloat162float(h2.y));
    *reinterpret_cast<__nv_bfloat162*>(hi + v * ld + j) = h2;
    if (lo != nullptr) *reinterpret_cast<__nv_bfloat162*>(lo + v * ld + j) = l2;  // null: hi plane alone (single pass)
  }
}

// copies `w4` 8-byte words per row (a column block of bf16 planes with row stride `ld8` words) from one hi/lo plane pair into
// two others: score_emb is layer-invariant and has to sit next to x in every [x | score_emb] operand buffer
__global__ void copy_plane_columns_kernel(int64_t N, int w4, int ld8, const uint2* __restrict__ sh, const uint2* __restrict__ sl,
                                          uint2* __restrict__ d1h, uint2* __restrict__ d1l, uint2* __restrict__ d2h,
                                          uint2* __restrict__ d2l) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N * w4; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / w4;
    const int c = (int)(i - r * w4);
    const uint2 h = sh[r * ld8 + c];
    d1h[r * ld8 + c] = h;
    d2h[r * ld8 + c] = h;
    if (sl != nullptr) {  // null: hi planes alone (single pass)
      const uint2 l = sl[r * ld8 + c];
      d1l[r * ld8 + c] = l;
      d2l[r * ld8 + c] = l;
    }
  }
}

// Fused node_feature_extra for D/2 <= 128 (modeling_qagnn.py:62-73,86): one CTA = 64 nodes; emb_score's [D/2, D/2] weight
// and the CTA's sin-basis tile live in shared memory, so the whole prologue (type-table lookup, sin basis, Linear, GELU)
// is one launch that writes `extra` as fp32 and/or as the split-bf16 planes the projection GEMM consumes.
constexpr int kNfNodes = 64;
__global__ void __launch_bounds__(256) node_feature_fused_kernel(int64_t N, int D, int T, const int64_t* __restrict__ node_type,
                                                                  const float* __restrict__ node_score,
                                                                  const float* __restrict__ type_tab, const float* __restrict__ basis,
                                                                  const float* __restrict__ ws, const float* __restrict__ bs,
                                                                  float* __restrict__ extra, __nv_bfloat16* __restrict__ ex_hi,
                                                                  __nv_bfloat16* __restrict__ ex_lo) {
  extern __shared__ __align__(16) float sm_nf[];
  const int Dh = D / 2;                   // Dh % 4 == 0 (checked by the launcher)
  float* Wt = sm_nf;                      // [Dh][Dh]        Wt[k*Dh + j] = ws[j][k]
  float* Bt = Wt + (size_t)Dh * Dh;       // [Dh][kNfNodes]  Bt[k*64 + v] = sin(basis[k] * score[v])
  const int64_t v0 = (int64_t)blockIdx.x * kNfNodes;
  for (int i = threadIdx.x; i < Dh * Dh; i += 256) Wt[(i % Dh) * Dh + i / Dh] = ws[i];
  for (int i = threadIdx.x; i < kNfNodes * Dh; i += 256) {
    const int k = i / kNfNodes, vi = i % kNfNodes;
    const int64_t v = v0 + vi;
    Bt[i] = v < N ? sinf(basis[k] * node_score[v]) : 0.f;  // precise sinf: arguments reach ~1e4 * |score|
  }
  __syncthreads();
  // 4 consecutive columns of one node: one 16-byte fp32 store and/or two 8-byte bf16 stores (hi / lo planes);
  // (v*D + col) is a multiple of 4 because D % 8 == 0 and col % 4 == 0
  auto put4 = [&](int64_t v, int col, const float (&x)[4]) {
    if (extra != nullptr) *reinterpret_cast<float4*>(extra + v * D + col) = make_float4(x[0], x[1], x[2], x[3]);
    if (ex_hi != nullptr) {
      __nv_bfloat16 h[4], l[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        h[c] = __float2bfloat16_rn(x[c]);
        l[c] = __float2bfloat16_rn(x[c] - __bfloat162float(h[c]));
      }
      *reinterpret_cast<uint2*>(ex_hi + v * D + col) = *reinterpret_cast<const uint2*>(h);
      if (ex_lo != nullptr) *reinterpret_cast<uint2*>(ex_lo + v * D + col) = *reinterpret_cast<const uint2*>(l);
    }
  };
  // register tile: 4 nodes x 4 outputs per thread -> two LDS.128 per 16 FMAs
  const int jg = Dh / 4, ntile = (kNfNodes / 4) * jg;
  for (int tl = threadIdx.x; tl < ntile; tl += 256) {
    const int vi0 = (tl / jg) * 4, j0 = (tl % jg) * 4;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
    for (int k = 0; k < Dh; ++k) {
      const float4 b = *reinterpret_cast<const float4*>(Bt + k * kNfNodes + vi0);
      const float4 w = *reinterpret_cast<const float4*>(Wt + k * Dh + j0);
      const float bb[4] = {b.x, b.y, b.z, b.w}, ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = fmaf(bb[a], ww[c], acc[a][c]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int64_t v = v0 + vi0 + a;
      if (v >= N) continue;
      int64_t t = node_type[v];
      t = t < 0 ? 0 : (t >= T ? T - 1 : t);
      float sc[4], ty[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        sc[c] = gelu_tanh(acc[a][c] + bs[j0 + c]);
        ty[c] = type_tab[t * Dh + j0 + c];
      }
      put4(v, Dh + j0, sc);
      put4(v, j0, ty);
    }
  }
}

// alpha_out rows of the edge ids [rowptr_src[N] - N, E) are 0: the unused columns of an edge capacity
// (qagnn_graph_prep_packed).  No row is written when the batch fills E, as every batch the general prep takes does.
__global__ void zero_alpha_holes_kernel(int64_t N, int64_t E, int H, const int32_t* __restrict__ rowptr_src,
                                        float* __restrict__ alpha_out) {
  const int64_t e0 = min(max((int64_t)rowptr_src[N] - N, (int64_t)0), E);
  for (int64_t i = e0 * H + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E * H; i += (int64_t)gridDim.x * blockDim.x)
    alpha_out[i] = 0.f;
}

int32_t zero_alpha_holes(const qagnn_shape& s, const void* prep, const qagnn_prep_layout& pl, float* alpha_out,
                         cudaStream_t st) {
  if (alpha_out == nullptr || s.E == 0) return QAGNN_OK;
  int64_t g = (s.E * s.H + 255) / 256;
  if (g > kNumSMs * 4) g = kNumSMs * 4;
  zero_alpha_holes_kernel<<<(unsigned)g, 256, 0, st>>>(s.N, s.E, s.H, (const int32_t*)((const char*)prep + pl.rowptr_src),
                                                        alpha_out);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

int32_t check_shape_fwd(const qagnn_shape* s) {
  if (!s) return QAGNN_ERR_INVALID_ARGUMENT;
  if (s->N <= 0 || s->E < 0 || s->D <= 0 || s->H <= 0 || s->T <= 0 || s->R <= 0 || s->k < 0)
    return QAGNN_ERR_INVALID_ARGUMENT;
  if (s->D % s->H != 0 || s->D % 2 != 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (s->N + s->E >= (int64_t)1 << 31) return QAGNN_ERR_INVALID_ARGUMENT;
  return QAGNN_OK;
}

// ---- path decision ------------------------------------------------------------------------------------
// Every forward entry point runs the kernels of one ForwardPlan, made once per call by plan_forward.  The switches are read at
// every call: tests and A/B runs cover every path in one process.
struct ForwardPlan {
  int passes;      // 3: split-bf16 GEMMs on fp32 data; 1: single-pass bf16 GEMMs (the bf16 entry points)
  bool tc;         // wgmma GEMMs: the driver exposes TMA descriptors and the row strides meet TMA's 16-byte rule (D % 8 == 0);
                   // else the exact-fp32 FFMA GEMM.  QAGNN_GEMM=ffma forces the latter.
  bool tiled;      // shared-memory-tiled message passing: the batch is made of equal small sub-graphs (shape.n_per_graph > 0,
                   // or a ragged batch) and the tiles fit.  QAGNN_MP_PATH=csr|basic forces the general kernels.
  bool slice;      // without tiles: the column-sliced kernels (edge tables in shared memory) when the head width allows, else
                   // the basic CSR kernels.  QAGNN_MP_PATH=basic forces the latter.
  bool zero_pads;  // tiled on the FFMA GEMM: its head-major projection never writes the pad columns, so the call zeroes them once
  bool fast;       // qagnn_mp_forward's fast-form projection (tiled, tc, k > 0, D/2 % 4 == 0, D/2 >= 8): emb_score on the tensor
                   // cores (a wgmma GEMM of width D/2, which must be at least 8) and the type-embedding half of
                   // node_feature_extra folded into per-node-type bias rows.
                   // QAGNN_MP_FASTPROJ=0 keeps the general [x | extra] projection.
  bool mlp_fused;  // node MLP in one launch with the hidden layer in registers (tc, D <= 208), else mlp.0 and mlp.3 as two
                   // GEMMs with the hidden planes in the workspace.  QAGNN_MLP_FUSED=0 forces the two launches.
};

ForwardPlan plan_forward(const qagnn_shape& s, const Ragged& rg, int passes) {
  const char* path = getenv("QAGNN_MP_PATH");
  const bool basic = path && strcmp(path, "basic") == 0;
  const bool general = basic || (path && strcmp(path, "csr") == 0);
  const char* fastproj = getenv("QAGNN_MP_FASTPROJ");
  const char* fused = getenv("QAGNN_MLP_FUSED");
  ForwardPlan p;
  p.passes = passes;
  p.tc = gemm_tc_available() && s.D % 8 == 0;
  p.tiled = !general && headtile_supported(s, rg);
  p.slice = !p.tiled && !basic && slice_supported(s);
  p.zero_pads = p.tiled && !p.tc;
  p.fast = p.tc && p.tiled && s.k > 0 && (s.D / 2) % 4 == 0 && s.D / 2 >= 8 && !(fastproj && atoi(fastproj) == 0);
  p.mlp_fused = p.tc && !(fused && atoi(fused) == 0) && mlp_tc_shape_ok(s.D);
  return p;
}

// One forward call: its shape and layouts, its plan, and what every stage reads.
struct Fwd {
  qagnn_shape s;
  FoldLayout L;
  WorkLayout W;
  qagnn_prep_layout pl;
  ForwardPlan plan;
  bool in_bf16;  // bf16 inputs (a one-pass call only)
  Ragged rg;
  const void* prep;
  const float* folded;
  float* ws;
  cudaStream_t st;
  const float* layer_block(int l) const { return folded + L.layer0 + (size_t)l * L.layer_stride; }
};

// The checks and setup of every forward entry.  `args_ok`: the entry's own pointer and index checks.  (dtype, in_dtype) is
// (F32, F32) for the fp32 forward (3 passes) or (BF16, F32 | BF16) for bf16 out (1 pass); any other pair is invalid.  Every
// invalid argument is reported ahead of a short workspace.
int32_t setup_forward(const qagnn_shape* shape, int32_t dtype, int32_t in_dtype, bool args_ok, const void* prep,
                      const void* folded, void* workspace, size_t workspace_bytes, void* stream, const Ragged& rg, Fwd& f) {
  QAGNN_RETURN_IF(check_shape_fwd(shape));
  const bool bf16 = dtype == QAGNN_DTYPE_BF16 && (in_dtype == QAGNN_DTYPE_F32 || in_dtype == QAGNN_DTYPE_BF16);
  const bool f32 = dtype == QAGNN_DTYPE_F32 && in_dtype == QAGNN_DTYPE_F32;
  if (!(bf16 || f32) || !args_ok) return QAGNN_ERR_INVALID_ARGUMENT;
  f.s = *shape;
  f.L = make_fold_layout(f.s);
  f.W = make_work_layout(f.s);
  if (workspace_bytes < f.W.total * sizeof(float)) return QAGNN_ERR_WORKSPACE;
  QAGNN_RETURN_IF(qagnn_graph_prep_layout(f.s.N, f.s.E, &f.pl));
  f.plan = plan_forward(f.s, rg, bf16 ? 1 : 3);
  f.in_bf16 = in_dtype == QAGNN_DTYPE_BF16;
  f.rg = rg;
  f.prep = prep;
  f.folded = (const float*)folded;
  f.ws = (float*)workspace;
  f.st = (cudaStream_t)stream;
  return QAGNN_OK;
}

// logits -> per-source softmax -> out-degree rescale -> per-target sum   (:442, :469-484), on the plan's kernels, from the
// projection in the workspace.  aggr_hi / aggr_lo: the tiled kernel also writes the bf16 planes of aggr (tensor-core layer).
int32_t message_passing(const Fwd& f, const float* lb, float* aggr, float* alpha_out, void* aggr_hi, void* aggr_lo) {
  ProfScope ps(QAGNN_PROF_MESSAGE_PASSING, f.st);
  QAGNN_RETURN_IF(zero_alpha_holes(f.s, f.prep, f.pl, alpha_out, f.st));
  const int32_t* prep = (const int32_t*)f.prep;
  const float* qkm = f.ws + f.W.qkm;
  float* score = f.ws + f.W.score;
  if (f.plan.tiled)
    return launch_message_passing_headtile(f.s, prep, f.pl, qkm, lb + f.L.keh, lb + f.L.meh, score, f.ws + f.W.alpha2, aggr,
                                           alpha_out, aggr_hi, aggr_lo, f.st, f.rg);
  if (f.plan.slice)
    return launch_message_passing_slice(f.s, prep, f.pl, qkm, lb + f.L.ke, lb + f.L.me, score, aggr, alpha_out, f.st);
  return launch_message_passing_typed(f.s, prep, f.pl, QAGNN_DTYPE_F32, qkm, lb + f.L.ke, lb + f.L.me, score, f.ws + f.W.alpha,
                                      aggr, alpha_out, f.st);
}

// one GATConvE layer on the exact-fp32 FFMA GEMM; `final_act` = ACT_NONE for the bare layer, ACT_GELU when called from mp_helper
int32_t layer_forward(const Fwd& f, int layer, const float* x, const float* extra, float* out, float* alpha_out,
                      float* aggr_out, Act final_act) {
  const qagnn_shape& s = f.s;
  const FoldLayout& L = f.L;
  const WorkLayout& W = f.W;
  const int D = s.D;
  const float* lb = f.layer_block(layer);
  float* ws = f.ws;
  float* aggr = aggr_out ? aggr_out : ws + W.aggr;
  {  // Q | Kx | Mx = [x ‖ extra] @ Wp^T + bp                     (:440, :464-466 node part, :469)
    ProfScope ps(QAGNN_PROF_PROJECTION, f.st);
    HeadMajorOut hm{f.plan.tiled ? 1 : 0, D, D / s.H, head_dim_padded(D / s.H), s.H};
    QAGNN_RETURN_IF(sgemm_tn(x, D, D, extra, D, D, lb + L.wp, 2 * D, lb + L.bp, ws + W.qkm, 3 * D, s.N, 3 * D, ACT_NONE, f.st, hm));
  }
  QAGNN_RETURN_IF(message_passing(f, lb, aggr, alpha_out, nullptr, nullptr));
  {  // node MLP: Linear -> BatchNorm(eval, folded) -> ReLU -> Linear          (:443, :408)
    ProfScope ps(QAGNN_PROF_NODE_MLP, f.st);
    QAGNN_RETURN_IF(sgemm_tn(aggr, D, D, nullptr, 0, 0, lb + L.w1, D, lb + L.b1, ws + W.hmid, D, s.N, D, ACT_RELU, f.st));
    QAGNN_RETURN_IF(sgemm_tn(ws + W.hmid, D, D, nullptr, 0, 0, lb + L.w2, D, lb + L.b2, out, D, s.N, D, final_act, f.st));
  }
  return QAGNN_OK;
}

struct Planes {  // an operand as bf16 hi / lo planes, row stride ld elements
  void* hi;
  void* lo;
  int ld;
};

// one GATConvE layer on the wgmma GEMMs.  x / extra are [N, D] operand planes; the layer output goes to any of out_f32 (fp32
// [N, D]) and the planes out_hi / out_lo (row stride out_ldp).  row_class selects the fast-form projection (ForwardPlan::fast):
// x rows are [x | score_emb] (K = D + D/2, ONE segment), extra is unused, and the type-embedding half of node_feature_extra
// enters as the bias row of each node's type.  One pass: every GEMM runs on the hi planes alone (lo planes neither read nor
// written, out_lo ignored); the message passing is the same either way.
int32_t layer_forward_tc(const Fwd& f, int layer, Planes x, Planes extra, const int64_t* row_class, float* out_f32, void* out_hi,
                         void* out_lo, int out_ldp, float* alpha_out, float* aggr_out, Act final_act) {
  const qagnn_shape& s = f.s;
  const FoldLayout& L = f.L;
  const WorkLayout& W = f.W;
  const int D = s.D, passes = f.plan.passes;
  cudaStream_t st = f.st;
  float* ws = f.ws;
  float* const ap_lo = passes == 1 ? nullptr : ws + W.ap_lo;
  const float* lb = f.layer_block(layer);
  float* qkm = ws + W.qkm;
  const bool fused_split = f.plan.tiled && (D / s.H) % 2 == 0;  // the tiled kernel emits the bf16 planes of aggr itself
  float* aggr = aggr_out ? aggr_out : (fused_split ? nullptr : ws + W.aggr);
  {  // Q | Kx | Mx = [x ‖ extra] @ Wp^T + bp                     (:440, :464-466 node part, :469)
    ProfScope ps(QAGNN_PROF_PROJECTION, st);
    TcOperand A1{x.hi, x.lo, x.ld, D}, A2{extra.hi, extra.lo, extra.ld, D};
    TcOutput o{};
    if (row_class != nullptr) {  // fast form: T distinct type-embedding rows -> T bias rows
      const int DP = head_dim_padded(D / s.H);
      TcOperand Ax{x.hi, x.lo, x.ld, D + D / 2}, none{nullptr, nullptr, 0, 0};
      TcOperand Wp{lb + L.wps_hi, lb + L.wps_lo, x.ld, D + D / 2};
      o.hm_buf = qkm;
      o.hm = HeadMajorOut{1, D, D / s.H, DP, s.H};
      o.row_class = row_class; o.class_stride = 3 * s.H * DP; o.n_class = s.T;
      // the resident-weight kernel where its slice fits (split-bf16 only), else the general GEMM
      int32_t rc = passes == 3 ? proj_resident(Ax, Wp, lb + L.tbias, s.N, 3 * s.H * DP, o, st) : QAGNN_ERR_UNSUPPORTED;
      if (rc == QAGNN_ERR_UNSUPPORTED) rc = gemm_tc(Ax, none, Wp, lb + L.tbias, s.N, 3 * s.H * DP, ACT_NONE, o, st, passes);
      QAGNN_RETURN_IF(rc);
    } else if (f.plan.tiled) {  // per-head padded weight rows -> the GEMM writes [3][H][N][DP] (pads = exact zeros) itself
      const int DP = head_dim_padded(D / s.H);
      TcOperand Wp{lb + L.wph_hi, lb + L.wph_lo, 2 * D, 2 * D};
      o.hm_buf = qkm;
      o.hm = HeadMajorOut{1, D, D / s.H, DP, s.H};
      QAGNN_RETURN_IF(gemm_tc(A1, A2, Wp, lb + L.bph, s.N, 3 * s.H * DP, ACT_NONE, o, st, passes));
    } else {
      TcOperand Wp{lb + L.wp_hi, lb + L.wp_lo, 2 * D, 2 * D};
      o.f32 = qkm;
      o.ldc = 3 * D;
      QAGNN_RETURN_IF(gemm_tc(A1, A2, Wp, lb + L.bp, s.N, 3 * D, ACT_NONE, o, st, passes));
    }
  }
  QAGNN_RETURN_IF(message_passing(f, lb, aggr, alpha_out, fused_split ? ws + W.ap_hi : nullptr, ap_lo));
  {  // node MLP: Linear -> BatchNorm(eval, folded) -> ReLU -> Linear          (:443, :408)
    ProfScope ps(QAGNN_PROF_NODE_MLP, st);
    if (!fused_split) QAGNN_RETURN_IF(split_bf16(aggr, D, s.N, D, ws + W.ap_hi, ap_lo, D, st));
    TcOperand A{ws + W.ap_hi, ws + W.ap_lo, D, D}, none{nullptr, nullptr, 0, 0};
    TcOperand W1{lb + L.w1_hi, lb + L.w1_lo, D, D}, W2{lb + L.w2_hi, lb + L.w2_lo, D, D};
    if (f.plan.mlp_fused) {  // one launch, the hidden layer never leaves registers
      TcOutput o{};
      o.f32 = out_f32; o.ldc = D; o.hi = out_hi; o.lo = out_lo; o.ldp = out_ldp;
      return mlp_tc(A, W1, lb + L.b1, W2, lb + L.b2, s.N, final_act, o, st, passes);
    }
    TcOutput o1{};
    o1.hi = ws + W.mp_hi; o1.lo = ws + W.mp_lo; o1.ldp = D;
    QAGNN_RETURN_IF(gemm_tc(A, none, W1, lb + L.b1, s.N, D, ACT_RELU, o1, st, passes));
    TcOperand Hm{ws + W.mp_hi, ws + W.mp_lo, D, D};
    TcOutput o2{};
    o2.f32 = out_f32; o2.ldc = D; o2.hi = out_hi; o2.lo = out_lo; o2.ldp = out_ldp;
    QAGNN_RETURN_IF(gemm_tc(Hm, none, W2, lb + L.b2, s.N, D, final_act, o2, st, passes));
  }
  return QAGNN_OK;
}

// node_feature_extra (:62-73,86) as fp32 `extra` and/or as the split-bf16 planes ex_hi / ex_lo (ex_lo null: hi plane alone)
int32_t extra_forward(const Fwd& f, const int64_t* node_type, const float* node_score, float* extra, void* ex_hi, void* ex_lo) {
  ProfScope ps(QAGNN_PROF_PRO_EPILOGUE, f.st);
  const qagnn_shape& s = f.s;
  const FoldLayout& L = f.L;
  const float* folded = f.folded;
  cudaStream_t st = f.st;
  const int D = s.D, Dh = D / 2;
  if (Dh <= 128 && D % 8 == 0) {
    const size_t smem = ((size_t)Dh * Dh + (size_t)kNfNodes * Dh) * sizeof(float);
    static size_t attr[kMaxDevices] = {0};
    const int dev = current_device();
    if (smem > 48 * 1024 && smem > attr[dev]) {
      QAGNN_CHECK_CUDA(cudaFuncSetAttribute(node_feature_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr[dev] = smem;
    }
    node_feature_fused_kernel<<<(unsigned)((s.N + kNfNodes - 1) / kNfNodes), 256, smem, st>>>(
        s.N, D, s.T, node_type, node_score, folded + L.type_tab, folded + L.basis, folded + L.ws, folded + L.bs, extra,
        (__nv_bfloat16*)ex_hi, (__nv_bfloat16*)ex_lo);
    QAGNN_CHECK_LAUNCH();
    return QAGNN_OK;
  }
  const int64_t n = s.N * Dh;
  int64_t g = (n + 255) / 256;
  if (g > kNumSMs * 32) g = kNumSMs * 32;
  node_feature_prologue_kernel<<<(unsigned)g, 256, 0, st>>>(s.N, D, s.T, node_type, node_score, folded + L.type_tab,
                                                            folded + L.basis, extra, f.ws + f.W.sinb);
  QAGNN_CHECK_LAUNCH();
  // extra[:, D/2:] = GELU(emb_score(sinb))                                  (:73)
  QAGNN_RETURN_IF(sgemm_tn(f.ws + f.W.sinb, Dh, Dh, nullptr, 0, 0, folded + L.ws, Dh, folded + L.bs, extra + Dh, D, s.N, Dh,
                           ACT_GELU, st));
  if (ex_hi != nullptr) QAGNN_RETURN_IF(split_bf16(extra, D, s.N, D, ex_hi, ex_lo, D, st));
  return QAGNN_OK;
}

// The fast form's score_emb = GELU(emb_score(sin basis)) (:70-73) as columns [D, D + D/2) of the three [N, KS] plane pairs:
// the sin-basis planes, the emb_score GEMM into pair 0, and a copy into the two activation pairs (layer-invariant: :86)
int32_t score_emb_planes(const Fwd& f, const float* node_score, void* const* hi, void* const* lo, int KS) {
  const qagnn_shape& s = f.s;
  const int D = s.D, Dh = D / 2, KSh = round_up8(Dh);
  const bool single = f.plan.passes == 1;
  float* ws = f.ws;
  const float* fo = f.folded;
  int64_t g = (s.N * (Dh / 2) + 255) / 256;
  if (g > kNumSMs * 32) g = kNumSMs * 32;
  sin_basis_planes_kernel<<<(unsigned)g, 256, 0, f.st>>>(s.N, Dh, KSh, node_score, fo + f.L.basis,
                                                         (__nv_bfloat16*)(ws + f.W.sb_hi),
                                                         single ? nullptr : (__nv_bfloat16*)(ws + f.W.sb_lo));
  QAGNN_CHECK_LAUNCH();
  const size_t off = (size_t)D * 2;  // bytes to column D of a plane
  auto at = [&](void* plane) { return (uint2*)((char*)plane + off); };
  TcOperand A{ws + f.W.sb_hi, ws + f.W.sb_lo, KSh, Dh}, none{nullptr, nullptr, 0, 0}, Wsc{fo + f.L.ws_hi, fo + f.L.ws_lo, KSh, Dh};
  TcOutput o{};
  o.hi = at(hi[0]); o.lo = at(lo[0]); o.ldp = KS;
  QAGNN_RETURN_IF(gemm_tc(A, none, Wsc, fo + f.L.bs, s.N, Dh, ACT_GELU, o, f.st, f.plan.passes));
  const int w4 = Dh * 2 / 8, ld8 = KS * 2 / 8;  // Dh % 4 == 0 and KS % 8 == 0 (ForwardPlan::fast)
  int64_t gc = (s.N * w4 + 255) / 256;
  if (gc > kNumSMs * 16) gc = kNumSMs * 16;
  copy_plane_columns_kernel<<<(unsigned)gc, 256, 0, f.st>>>(s.N, w4, ld8, at(hi[0]), single ? nullptr : at(lo[0]), at(hi[1]),
                                                            at(lo[1]), at(hi[2]), at(lo[2]));
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

// An [N, D] input as the A-operand planes of the call's GEMMs, row stride ldp: the split-bf16 hi / lo planes of an fp32 input
// (3 passes), or the hi plane alone (1 pass) - a bf16 input copied (bf16_rn is the identity on it), an fp32 one rounded to
// nearest even by split_bf16 without its lo plane: autocast's cast, in the same pass that writes the plane
int32_t input_planes(const Fwd& f, const void* src, void* hi, void* lo, int ldp) {
  const int64_t N = f.s.N;
  const int D = f.s.D;
  if (f.in_bf16) {
    QAGNN_CHECK_CUDA(cudaMemcpy2DAsync(hi, (size_t)ldp * 2, src, (size_t)D * 2, (size_t)D * 2, (size_t)N,
                                       cudaMemcpyDeviceToDevice, f.st));
    return QAGNN_OK;
  }
  return split_bf16((const float*)src, D, N, D, hi, f.plan.passes == 1 ? nullptr : lo, ldp, f.st);
}

__global__ void bf16_to_f32_kernel(int64_t n, const __nv_bfloat16* __restrict__ in, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __bfloat162float(in[i]);
}
__global__ void f32_to_bf16_kernel(int64_t n, const float* __restrict__ in, __nv_bfloat16* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16_rn(in[i]);
}
// exact widening / round-to-nearest-even narrowing of n elements (the bf16 entry points on shapes without the wgmma GEMM)
int32_t convert(int64_t n, const void* in, void* out, bool widen, cudaStream_t st) {
  if (n <= 0) return QAGNN_OK;
  int64_t g = (n + 255) / 256;
  if (g > kNumSMs * 32) g = kNumSMs * 32;
  if (widen) bf16_to_f32_kernel<<<(unsigned)g, 256, 0, st>>>(n, (const __nv_bfloat16*)in, (float*)out);
  else f32_to_bf16_kernel<<<(unsigned)g, 256, 0, st>>>(n, (const float*)in, (__nv_bfloat16*)out);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

// A forward on the FFMA GEMM: `run(in32, out32)` is the fp32 path on n_in (<= 2) [N, D] inputs.  An fp32 call runs it on the
// caller's buffers.  A bf16 call runs it on the rounded inputs (widened exactly) and rounds its output once; the split-bf16
// plane buffers, which the FFMA path never touches, stage the fp32 inputs and the output ([hp_hi, ap_hi) spans 4 N*D floats).
template <class Run>
int32_t ffma_forward(const Fwd& f, int n_in, const void* const* in, void* out, Run run) {
  const float* in32[2] = {(const float*)in[0], n_in > 1 ? (const float*)in[1] : nullptr};
  if (f.plan.passes == 3) return run(in32, (float*)out);
  const int64_t ND = f.s.N * (int64_t)f.s.D;
  float* out32 = f.ws + f.W.hp_hi + n_in * ND;
  for (int i = 0; i < n_in; ++i) {
    float* x32 = f.ws + f.W.hp_hi + i * ND;
    if (f.in_bf16) {
      QAGNN_RETURN_IF(convert(ND, in[i], x32, true, f.st));
    } else {  // bf16_rn of the fp32 input, back in fp32
      QAGNN_RETURN_IF(convert(ND, in[i], out32, false, f.st));
      QAGNN_RETURN_IF(convert(ND, out32, x32, true, f.st));
    }
    in32[i] = x32;
  }
  QAGNN_RETURN_IF(run(in32, out32));
  return convert(ND, out32, out, false, f.st);
}

// QAGNN_Message_Passing.forward on the FFMA GEMM, fp32 in and out
int32_t mp_forward_ffma(const Fwd& f, const float* H_in, const int64_t* node_type, const float* node_score, float* out,
                        float* x_layers_out) {
  const qagnn_shape& s = f.s;
  float* extra = f.ws + f.W.extra;
  QAGNN_RETURN_IF(extra_forward(f, node_type, node_score, extra, nullptr, nullptr));
  if (f.plan.zero_pads) QAGNN_RETURN_IF(zero_head_pads(s, f.ws + f.W.qkm, f.st));
  const size_t ND = (size_t)s.N * s.D;
  const float* x = H_in;
  for (int l = 0; l < s.k; ++l) {  // mp_helper, :45-50 (dropout is the identity in eval)
    float* xo = x_layers_out ? x_layers_out + (size_t)l * ND : f.ws + ((l & 1) ? f.W.xb : f.W.xa);
    QAGNN_RETURN_IF(layer_forward(f, l, x, extra, xo, nullptr, nullptr, ACT_GELU));
    x = xo;
  }
  // output = GELU(Vh(H) + Vx(X))                                             (:92)
  ProfScope ps(QAGNN_PROF_PRO_EPILOGUE, f.st);
  return sgemm_tn(H_in, s.D, s.D, x, s.D, s.D, f.folded + f.L.vcat, 2 * s.D, f.folded + f.L.vbias, out, s.D, s.N, s.D, ACT_GELU,
                  f.st);
}

// QAGNN_Message_Passing.forward on the wgmma GEMMs.  The prologue chooses a set of three [N, ld] plane pairs - 0: H_in, 1 and 2:
// the layer activations, ping-pong - and fills it:
// * fast form: ld = KS; columns [D, D + D/2) of every pair hold score_emb, the type embedding enters as per-type bias rows;
// * general form: ld = D; node_feature_extra goes to planes of its own, the projection's second A segment.
// One layer loop and one Vh|Vx GEMM follow for both.
int32_t mp_forward_tc(const Fwd& f, const void* H_in, const int64_t* node_type, const float* node_score, void* out,
                      float* x_layers_out) {
  const qagnn_shape& s = f.s;
  const WorkLayout& W = f.W;
  float* ws = f.ws;
  const int D = s.D;
  const bool fast = f.plan.fast;
  const int ld = fast ? round_up8(D + D / 2) : D;
  void* hi[3];
  void* lo[3];
  for (int i = 0; i < 3; ++i) {
    hi[i] = ws + (fast ? W.xs_hi[i] : i == 0 ? W.hp_hi : W.xp_hi[i - 1]);
    lo[i] = ws + (fast ? W.xs_lo[i] : i == 0 ? W.hp_lo : W.xp_lo[i - 1]);
  }
  Planes extra{nullptr, nullptr, 0};
  if (!fast) {  // `extra` is only ever consumed as planes, so the prologue writes those directly (and fp32 only where D/2 > 128)
    QAGNN_RETURN_IF(extra_forward(f, node_type, node_score, D / 2 <= 128 ? nullptr : ws + W.extra, ws + W.ep_hi,
                                  f.plan.passes == 1 ? nullptr : ws + W.ep_lo));
    extra = Planes{ws + W.ep_hi, ws + W.ep_lo, D};
  }
  {
    ProfScope ps(QAGNN_PROF_PRO_EPILOGUE, f.st);
    if (fast) QAGNN_RETURN_IF(score_emb_planes(f, node_score, hi, lo, ld));
    QAGNN_RETURN_IF(input_planes(f, H_in, hi[0], lo[0], ld));
  }
  const size_t ND = (size_t)s.N * D;
  int cur = 0;  // the pair holding the layer input
  for (int l = 0; l < s.k; ++l) {  // mp_helper, :45-50 (dropout is the identity in eval)
    const int nxt = 1 + (l & 1);
    float* xo32 = x_layers_out ? x_layers_out + (size_t)l * ND : nullptr;
    QAGNN_RETURN_IF(layer_forward_tc(f, l, Planes{hi[cur], lo[cur], ld}, extra, fast ? node_type : nullptr, xo32, hi[nxt],
                                     lo[nxt], ld, nullptr, nullptr, ACT_GELU));
    cur = nxt;
  }
  // output = GELU(Vh(H) + Vx(X)), X = H when k = 0                           (:92)
  ProfScope ps(QAGNN_PROF_PRO_EPILOGUE, f.st);
  TcOperand A1{hi[0], lo[0], ld, D}, A2{hi[cur], lo[cur], ld, D}, Wv{f.folded + f.L.vcat_hi, f.folded + f.L.vcat_lo, 2 * D, 2 * D};
  TcOutput o{};
  if (f.plan.passes == 1) { o.hi = out; o.ldp = D; }
  else { o.f32 = (float*)out; o.ldc = D; }
  return gemm_tc(A1, A2, Wv, f.folded + f.L.vbias, s.N, D, ACT_GELU, o, f.st, f.plan.passes);
}

}  // namespace
}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_abi_version(void) { return QAGNN_ABI_VERSION; }

extern "C" const char* qagnn_status_string(int32_t status) {
  switch (status) {
    case QAGNN_OK: return "ok";
    case QAGNN_ERR_INVALID_ARGUMENT: return "invalid argument";
    case QAGNN_ERR_CUDA: return "CUDA error";
    case QAGNN_ERR_INDEX_RANGE: return "index out of range in edge_index / edge_type / node_type";
    case QAGNN_ERR_WORKSPACE: return "workspace too small";
    case QAGNN_ERR_UNSUPPORTED: return "unsupported shape";
    default: return "unknown status";
  }
}

extern "C" const char* qagnn_last_cuda_error(void) { return g_cuda_err; }

extern "C" int64_t qagnn_launch_count(void) { return (int64_t)g_launches.load(std::memory_order_relaxed); }

extern "C" int32_t qagnn_profile_enable(int32_t on) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  g_prof.on = on != 0;
  g_prof.n = 0;
  for (int i = 0; i < QAGNN_PROF_STAGES; ++i) g_prof.open_idx[i] = -1;
  return QAGNN_OK;
}

extern "C" int32_t qagnn_profile_read(double* ms_out, int64_t* count_out) {
  if (!ms_out || !count_out) return QAGNN_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(g_prof.mu);
  for (int i = 0; i < QAGNN_PROF_STAGES; ++i) { ms_out[i] = 0.0; count_out[i] = 0; }
  for (int i = 0; i < g_prof.n; ++i) {
    QAGNN_CHECK_CUDA(cudaEventSynchronize(g_prof.ev[i][1]));
    float ms = 0.f;
    QAGNN_CHECK_CUDA(cudaEventElapsedTime(&ms, g_prof.ev[i][0], g_prof.ev[i][1]));
    ms_out[g_prof.stage[i]] += ms;
    count_out[g_prof.stage[i]] += 1;
  }
  return QAGNN_OK;
}

extern "C" size_t qagnn_forward_workspace_bytes(const qagnn_shape* shape) {
  if (check_shape_fwd(shape) != QAGNN_OK) return 0;
  return align_up(make_work_layout(*shape).total * sizeof(float));
}

// GATConvE.forward, one layer (:411-484): fp32, or a bf16 output (dtype) from fp32 or bf16 x / extra (in_dtype)
static int32_t gatconve_forward(const qagnn_shape* shape, int32_t dtype, int32_t in_dtype, int32_t layer, const void* x,
                                const void* extra, const void* prep, const void* folded, void* out, float* alpha_out,
                                float* aggr_out, void* workspace, size_t workspace_bytes, void* stream, const Ragged& rg) {
  const bool args_ok = x && extra && prep && folded && out && workspace && shape && layer >= 0 && layer < shape->k;
  Fwd f;
  QAGNN_RETURN_IF(setup_forward(shape, dtype, in_dtype, args_ok, prep, folded, workspace, workspace_bytes, stream, rg, f));
  if (f.plan.tc) {
    const bool single = f.plan.passes == 1;
    const int D = f.s.D;
    float* ws = f.ws;
    const Planes xp{ws + f.W.xp_hi[0], single ? nullptr : ws + f.W.xp_lo[0], D};
    const Planes ep{ws + f.W.ep_hi, single ? nullptr : ws + f.W.ep_lo, D};
    QAGNN_RETURN_IF(input_planes(f, x, xp.hi, xp.lo, D));
    QAGNN_RETURN_IF(input_planes(f, extra, ep.hi, ep.lo, D));
    return layer_forward_tc(f, layer, xp, ep, nullptr, single ? nullptr : (float*)out, single ? out : nullptr, nullptr, D,
                            alpha_out, aggr_out, ACT_NONE);
  }
  const void* in[2] = {x, extra};
  return ffma_forward(f, 2, in, out, [&](const float* const* in32, float* out32) {
    if (f.plan.zero_pads) QAGNN_RETURN_IF(zero_head_pads(f.s, f.ws + f.W.qkm, f.st));
    return layer_forward(f, layer, in32[0], in32[1], out32, alpha_out, aggr_out, ACT_NONE);
  });
}

extern "C" int32_t qagnn_gatconve_forward_typed(const qagnn_shape* shape, int32_t dtype, int32_t in_dtype, int32_t layer,
                                                const void* x, const void* extra, const void* prep, const void* folded,
                                                void* out, float* alpha_out, float* aggr_out, void* workspace,
                                                size_t workspace_bytes, void* stream) {
  return gatconve_forward(shape, dtype, in_dtype, layer, x, extra, prep, folded, out, alpha_out, aggr_out, workspace,
                          workspace_bytes, stream, Ragged{});
}

extern "C" int32_t qagnn_gatconve_forward(const qagnn_shape* shape, int32_t layer, const float* x, const float* extra,
                                          const void* prep, const void* folded, float* out, float* alpha_out,
                                          float* aggr_out, void* workspace, size_t workspace_bytes, void* stream) {
  return qagnn_gatconve_forward_typed(shape, QAGNN_DTYPE_F32, QAGNN_DTYPE_F32, layer, x, extra, prep, folded, out, alpha_out,
                                      aggr_out, workspace, workspace_bytes, stream);
}

// a ragged batch: n_graphs sub-graphs of at most shape->n_per_graph rows at node_ptr, the rest of the N rows a tail
static int32_t check_ragged(const qagnn_shape* shape, int32_t n_graphs, const int64_t* node_ptr, Ragged& rg) {
  if (!shape || !node_ptr || n_graphs <= 0 || n_graphs > shape->N || shape->n_per_graph <= 0) return QAGNN_ERR_INVALID_ARGUMENT;
  rg.node_ptr = node_ptr;
  rg.B = n_graphs;
  return QAGNN_OK;
}

extern "C" int32_t qagnn_gatconve_forward_ragged(const qagnn_shape* shape, int32_t dtype, int32_t in_dtype, int32_t n_graphs,
                                                 const int64_t* node_ptr, int32_t layer, const void* x, const void* extra,
                                                 const void* prep, const void* folded, void* out, float* alpha_out,
                                                 float* aggr_out, void* workspace, size_t workspace_bytes, void* stream) {
  Ragged rg;
  QAGNN_RETURN_IF(check_ragged(shape, n_graphs, node_ptr, rg));
  return gatconve_forward(shape, dtype, in_dtype, layer, x, extra, prep, folded, out, alpha_out, aggr_out, workspace,
                          workspace_bytes, stream, rg);
}

extern "C" int32_t qagnn_mp_path(const qagnn_shape* shape) {
  QAGNN_RETURN_IF(check_shape_fwd(shape));
  const ForwardPlan p = plan_forward(*shape, Ragged{}, 3);
  if (p.tiled) return QAGNN_MP_PATH_TILED;
  return p.slice ? QAGNN_MP_PATH_SLICE : QAGNN_MP_PATH_BASIC;
}

extern "C" int32_t qagnn_node_feature_extra(const qagnn_shape* shape, const int64_t* node_type, const float* node_score,
                                            const void* folded, float* extra_out, void* workspace,
                                            size_t workspace_bytes, void* stream) {
  const bool args_ok = node_type && node_score && folded && extra_out && workspace;
  Fwd f;
  QAGNN_RETURN_IF(setup_forward(shape, QAGNN_DTYPE_F32, QAGNN_DTYPE_F32, args_ok, nullptr, folded, workspace, workspace_bytes,
                                stream, Ragged{}, f));
  return extra_forward(f, node_type, node_score, extra_out, nullptr, nullptr);
}

// QAGNN_Message_Passing.forward (:53-95): fp32, or a bf16 output (dtype) from an fp32 or bf16 H (in_dtype)
static int32_t mp_forward(const qagnn_shape* shape, int32_t dtype, int32_t in_dtype, const void* H_in, const int64_t* node_type,
                          const float* node_score, const void* prep, const void* folded, void* out, float* x_layers_out,
                          void* workspace, size_t workspace_bytes, void* stream, const Ragged& rg) {
  const bool args_ok = H_in && node_type && node_score && prep && folded && out && workspace;
  Fwd f;
  QAGNN_RETURN_IF(setup_forward(shape, dtype, in_dtype, args_ok, prep, folded, workspace, workspace_bytes, stream, rg, f));
  if (f.plan.tc) return mp_forward_tc(f, H_in, node_type, node_score, out, x_layers_out);
  const void* in[1] = {H_in};
  return ffma_forward(f, 1, in, out, [&](const float* const* in32, float* out32) {
    return mp_forward_ffma(f, in32[0], node_type, node_score, out32, x_layers_out);
  });
}

extern "C" int32_t qagnn_mp_forward_typed(const qagnn_shape* shape, int32_t dtype, int32_t in_dtype, const void* H_in,
                                          const int64_t* node_type, const float* node_score, const void* prep,
                                          const void* folded, void* out, float* x_layers_out, void* workspace,
                                          size_t workspace_bytes, void* stream) {
  return mp_forward(shape, dtype, in_dtype, H_in, node_type, node_score, prep, folded, out, x_layers_out, workspace,
                    workspace_bytes, stream, Ragged{});
}

extern "C" int32_t qagnn_mp_forward(const qagnn_shape* shape, const float* H_in, const int64_t* node_type,
                                    const float* node_score, const void* prep, const void* folded, float* out,
                                    float* x_layers_out, void* workspace, size_t workspace_bytes, void* stream) {
  return qagnn_mp_forward_typed(shape, QAGNN_DTYPE_F32, QAGNN_DTYPE_F32, H_in, node_type, node_score, prep, folded, out,
                                x_layers_out, workspace, workspace_bytes, stream);
}

extern "C" int32_t qagnn_mp_forward_ragged(const qagnn_shape* shape, int32_t dtype, int32_t in_dtype, int32_t n_graphs,
                                           const int64_t* node_ptr, const void* H_in, const int64_t* node_type,
                                           const float* node_score, const void* prep, const void* folded, void* out,
                                           float* x_layers_out, void* workspace, size_t workspace_bytes, void* stream) {
  Ragged rg;
  QAGNN_RETURN_IF(check_ragged(shape, n_graphs, node_ptr, rg));
  return mp_forward(shape, dtype, in_dtype, H_in, node_type, node_score, prep, folded, out, x_layers_out, workspace,
                    workspace_bytes, stream, rg);
}

extern "C" size_t qagnn_mp_core_scratch_bytes(const qagnn_shape* shape, int32_t dtype) {
  if (check_shape_fwd(shape) != QAGNN_OK || dtype < QAGNN_DTYPE_F32 || dtype > QAGNN_DTYPE_BF16) return 0;
  return mp_core_scratch_bytes(*shape, dtype);
}

extern "C" int32_t qagnn_mp_core_forward_typed(const qagnn_shape* shape, int32_t dtype, const void* prep, const void* qkm,
                                               const void* ke, const void* me, void* aggr, float* alpha_scaled, float* alpha_out,
                                               float* scratch, void* stream) {
  QAGNN_RETURN_IF(check_shape_fwd(shape));
  if (dtype < QAGNN_DTYPE_F32 || dtype > QAGNN_DTYPE_BF16) return QAGNN_ERR_INVALID_ARGUMENT;
  if (!prep || !qkm || !ke || !me || !aggr || !alpha_scaled || !scratch) return QAGNN_ERR_INVALID_ARGUMENT;
  qagnn_prep_layout pl;
  QAGNN_RETURN_IF(qagnn_graph_prep_layout(shape->N, shape->E, &pl));
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(QAGNN_PROF_MESSAGE_PASSING, st);
  QAGNN_RETURN_IF(zero_alpha_holes(*shape, prep, pl, alpha_out, st));
  return launch_message_passing_typed(*shape, (const int32_t*)prep, pl, dtype, qkm, ke, me, scratch, alpha_scaled, aggr,
                                      alpha_out, st);
}

extern "C" int32_t qagnn_mp_core_forward(const qagnn_shape* shape, const void* prep, const float* qkm, const float* ke,
                                         const float* me, float* aggr, float* alpha_scaled, float* alpha_out, float* scratch,
                                         void* stream) {
  return qagnn_mp_core_forward_typed(shape, QAGNN_DTYPE_F32, prep, qkm, ke, me, aggr, alpha_scaled, alpha_out, scratch, stream);
}

extern "C" int32_t qagnn_mp_core_backward_typed(const qagnn_shape* shape, int32_t dtype, const void* prep,
                                                const int32_t* combo_order, const void* qkm, const void* ke, const void* me,
                                                const float* alpha_scaled, const void* d_aggr, void* d_qkm, void* d_ke,
                                                void* d_me, float* scratch, void* stream) {
  QAGNN_RETURN_IF(check_shape_fwd(shape));
  if (dtype < QAGNN_DTYPE_F32 || dtype > QAGNN_DTYPE_BF16) return QAGNN_ERR_INVALID_ARGUMENT;
  if (!prep || !combo_order || !qkm || !ke || !me || !alpha_scaled || !d_aggr || !d_qkm || !d_ke || !d_me || !scratch)
    return QAGNN_ERR_INVALID_ARGUMENT;
  qagnn_prep_layout pl;
  QAGNN_RETURN_IF(qagnn_graph_prep_layout(shape->N, shape->E, &pl));
  return launch_message_passing_backward_typed(*shape, (const int32_t*)prep, pl, dtype, combo_order, qkm, ke, me, alpha_scaled,
                                               d_aggr, scratch, d_qkm, d_ke, d_me, (cudaStream_t)stream);
}

extern "C" int32_t qagnn_mp_core_backward(const qagnn_shape* shape, const void* prep, const int32_t* combo_order,
                                          const float* qkm, const float* ke, const float* me, const float* alpha_scaled,
                                          const float* d_aggr, float* d_qkm, float* d_ke, float* d_me, float* scratch,
                                          void* stream) {
  return qagnn_mp_core_backward_typed(shape, QAGNN_DTYPE_F32, prep, combo_order, qkm, ke, me, alpha_scaled, d_aggr, d_qkm, d_ke,
                                      d_me, scratch, stream);
}

extern "C" size_t qagnn_mp_core_backward_det_scratch_bytes(const qagnn_shape* shape, int32_t dtype) {
  if (check_shape_fwd(shape) != QAGNN_OK || dtype < QAGNN_DTYPE_F32 || dtype > QAGNN_DTYPE_BF16) return 0;
  return mp_core_det_scratch_bytes(*shape, dtype);
}

extern "C" int32_t qagnn_mp_core_backward_det(const qagnn_shape* shape, int32_t dtype, const void* prep,
                                              const int32_t* combo_order, const int64_t* combo_count, const void* qkm,
                                              const void* ke, const void* me, const float* alpha_scaled, const void* d_aggr,
                                              void* d_qkm, void* d_ke, void* d_me, float* scratch, size_t scratch_bytes,
                                              void* stream) {
  QAGNN_RETURN_IF(check_shape_fwd(shape));
  if (dtype < QAGNN_DTYPE_F32 || dtype > QAGNN_DTYPE_BF16) return QAGNN_ERR_INVALID_ARGUMENT;
  if (!prep || !combo_order || !combo_count || !qkm || !ke || !me || !alpha_scaled || !d_aggr || !d_qkm || !d_ke || !d_me ||
      !scratch)
    return QAGNN_ERR_INVALID_ARGUMENT;
  if (scratch_bytes < mp_core_det_scratch_bytes(*shape, dtype)) return QAGNN_ERR_WORKSPACE;
  qagnn_prep_layout pl;
  QAGNN_RETURN_IF(qagnn_graph_prep_layout(shape->N, shape->E, &pl));
  return launch_message_passing_backward_det(*shape, (const int32_t*)prep, pl, dtype, combo_order, combo_count, qkm, ke, me,
                                             alpha_scaled, d_aggr, scratch, d_qkm, d_ke, d_me, (cudaStream_t)stream);
}

extern "C" size_t qagnn_linear_workspace_bytes(int64_t M, int32_t N, int32_t K1, int32_t K2) {
  if (M <= 0 || N <= 0 || K1 <= 0 || K2 < 0) return 0;
  const size_t K = (size_t)K1 + K2;
  return align_up(2 * 2 * ((size_t)M * K + (size_t)N * K) + 8 * 1024);
}

extern "C" int32_t qagnn_linear_bf16(const void* A1, int32_t lda1, int32_t K1, const void* A2, int32_t lda2, int32_t K2,
                                     const void* Wt, int32_t ldw, const float* bias, float* C, int32_t ldc, void* C_bf16,
                                     int32_t ldp, int64_t M, int32_t N, int32_t act, void* stream) {
  if (!A1 || !Wt || (!C && !C_bf16) || M <= 0 || N <= 0 || K1 <= 0 || K2 < 0 || (K2 > 0 && !A2)) return QAGNN_ERR_INVALID_ARGUMENT;
  if (act < 0 || act > 2) return QAGNN_ERR_INVALID_ARGUMENT;
  if (!gemm_tc_available() || !gemm_tc_shape_ok(K1, K2, lda1, lda2, ldw, N)) return QAGNN_ERR_UNSUPPORTED;
  TcOperand o1{A1, nullptr, lda1, K1}, o2{K2 ? A2 : nullptr, nullptr, lda2, K2}, ow{Wt, nullptr, ldw, K1 + K2};
  TcOutput out{};
  out.f32 = C;
  out.ldc = ldc;
  out.hi = C_bf16;
  out.ldp = ldp;
  return gemm_tc(o1, o2, ow, bias, M, N, (Act)act, out, (cudaStream_t)stream, 1);
}

extern "C" int32_t qagnn_linear_bf16x3(const float* A1, int32_t lda1, int32_t K1, const float* A2, int32_t lda2, int32_t K2,
                                       const float* Wt, int32_t ldw, const float* bias, float* C, int32_t ldc, int64_t M,
                                       int32_t N, int32_t act, void* workspace, size_t workspace_bytes, void* stream) {
  if (!A1 || !Wt || !C || !workspace || M <= 0 || N <= 0 || K1 <= 0 || K2 < 0 || (K2 > 0 && !A2)) return QAGNN_ERR_INVALID_ARGUMENT;
  if (act < 0 || act > 2) return QAGNN_ERR_INVALID_ARGUMENT;
  if (workspace_bytes < qagnn_linear_workspace_bytes(M, N, K1, K2)) return QAGNN_ERR_WORKSPACE;
  if (!gemm_tc_available() || !gemm_tc_shape_ok(K1, K2, K1, K2, K1 + K2, N)) return QAGNN_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  char* w = (char*)workspace;
  auto take = [&](size_t elems) { char* r = w; w += align_up(elems * 2); return (void*)r; };
  const int K = K1 + K2;
  void *a1h = take((size_t)M * K1), *a1l = take((size_t)M * K1);
  void *a2h = K2 ? take((size_t)M * K2) : nullptr, *a2l = K2 ? take((size_t)M * K2) : nullptr;
  void *wh = take((size_t)N * K), *wl = take((size_t)N * K);
  QAGNN_RETURN_IF(split_bf16(A1, lda1, M, K1, a1h, a1l, K1, st));
  if (K2) QAGNN_RETURN_IF(split_bf16(A2, lda2, M, K2, a2h, a2l, K2, st));
  QAGNN_RETURN_IF(split_bf16(Wt, ldw, N, K, wh, wl, K, st));
  TcOperand o1{a1h, a1l, K1, K1}, o2{a2h, a2l, K2, K2}, ow{wh, wl, K, K};
  TcOutput out{};
  out.f32 = C;
  out.ldc = ldc;
  return gemm_tc(o1, o2, ow, bias, M, N, (Act)act, out, st);
}
