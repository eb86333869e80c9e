// The step after the hot path (SURVEY.md §8f #2): QAGNN's masked multi-head attention pooling over the node
// representations (utils/layers.py:324-371 MultiheadAttPoolLayer + :276-299 MatrixVectorScaledDotProductAttention,
// called at modeling/modeling_qagnn.py:180), eval mode.
//
//   qs = w_qs(sent) [B, nh*dk];  ks = w_ks(X) [B, n, nh, dk];  vs = w_vs(X) [B, n, nh, dv]
//   attn[h,b,:] = softmax_i( mask ? -inf : qs[b,h]·ks[b,i,h] / sqrt(dk) );  pooled[b, h*dv:(h+1)*dv] = Σ_i attn·vs[b,i,h]
//
// The reference materialises ks and vs with two [B*n, D] x [D, D] GEMMs.  Both projections are linear, so they fold
// into the query / out of the sum:   qs_h·(W_k,h x_i + b_k,h) = (W_k,hᵀ qs_h)·x_i + qs_h·b_k,h   and
// Σ_i a_i (W_v,h x_i + b_v,h) = W_v,h (Σ_i a_i x_i) + b_v,h   (Σ_i a_i = 1).  One CTA per graph then reads the
// graph's [n, D] node tile ONCE: logits for all heads, masked softmax, attention-weighted node sum; the two tiny
// per-graph matrix-vector products run in the same CTA.  No N-sized GEMM, no ks/vs round trip through HBM.
#include <cuda_bf16.h>

#include "common.cuh"

namespace qagnn {
namespace {

// node features X as fp32 or bf16 (the bf16 eval forward's output): bf16 widens exactly
__device__ __forceinline__ float xval(float v) { return v; }
__device__ __forceinline__ float xval(__nv_bfloat16 v) { return __bfloat162float(v); }

constexpr int kPoolThreads = 256;  // latency-bound kernel: <= 64 registers so that 4 CTAs (graphs) share an SM

// dynamic smem: qk[nh][D] | logit[nh][n] | xs[nh][D] | cst[nh, padded to 8] | part[warps][nh][D]
// RAGGED (decoder tail mode only): X and node_type are a ragged batch of N_rows packed rows, graph b's rows start at
// node_ptr[b]; only its own rows are read, and the positions past them have exact zero weights, as in the padded layout.
template <typename XT, bool RAGGED = false>
__global__ void __launch_bounds__(kPoolThreads, 4) attention_pool_kernel(int n, int D, int nh, const XT* __restrict__ X,
                                                                        const float* __restrict__ qs, const unsigned char* __restrict__ mask,
                                                                        const float* __restrict__ wk, const float* __restrict__ bk,
                                                                        const float* __restrict__ wv, const float* __restrict__ bv,
                                                                        float* __restrict__ pooled, float* __restrict__ attn_out, int B,
                                                                        const int64_t* __restrict__ node_type = nullptr,
                                                                        const int64_t* __restrict__ adj_lengths = nullptr,
                                                                        const float* __restrict__ sent = nullptr, int S = 0,
                                                                        int pooled_ld = 0, const int64_t* __restrict__ node_ptr = nullptr,
                                                                        int64_t N_rows = 0) {
  // mask == nullptr: "decoder tail" mode (modeling_qagnn.py:172-187) — the pool mask is derived here from adj_lengths and
  // node_type, and the row of cat(graph_vecs, sent_vecs, Z) is written in place: pooled -> columns [0, D) of a
  // [B, pooled_ld = 2D+S] buffer, sent_vecs -> [D, D+S), Z = X[b, 0, :] -> [D+S, 2D+S)
  extern __shared__ float sm[];
  float* qk = sm;                  // [nh][D]   W_k,hᵀ qs_h
  float* logit = qk + nh * D;      // [nh][n]
  float* xs = logit + nh * n;      // [nh][D]   Σ_i attn_i x_i
  float* cst = xs + nh * D;        // [nh]      qs_h·b_k,h
  const int b = blockIdx.x, tid = threadIdx.x, dk = D / nh;
  const float inv_temp = 1.0f / sqrtf((float)dk);
  int64_t row0 = (int64_t)b * n;
  int nr = n;  // rows of X that belong to graph b
  if (RAGGED) {
    row0 = min(max(node_ptr[b], (int64_t)0), N_rows);
    nr = (int)min(min((int64_t)n, N_rows - row0), max(node_ptr[b + 1] - row0, (int64_t)0));
  }
  const XT* Xb = X + (size_t)row0 * D;
  const bool tail = mask == nullptr;
  if (!tail) pooled_ld = D;
  int len = n;
  bool all_masked = false;
  if (tail) {
    len = (int)min((int64_t)n, max((int64_t)0, adj_lengths[b]));
    if (RAGGED) nr = min(nr, len);
    // mask = (i >= len) | (type == 3); a fully masked row keeps node 0 (:174-176)
    int any_open = 0;
    for (int i = tid; i < (RAGGED ? nr : len); i += kPoolThreads) any_open |= node_type[RAGGED ? row0 + i : (int64_t)b * n + i] != 3;
    all_masked = __syncthreads_or(any_open) == 0;
  }
  // fold the key projection into the query: qk[h][j] = Σ_{r in head h} qs[b, r] * wk[r, j]
  for (int idx = tid; idx < nh * D; idx += kPoolThreads) {
    const int h = idx / D, j = idx % D;
    float acc = 0.f;
#pragma unroll 10
    for (int r = 0; r < dk; ++r) acc = fmaf(qs[(size_t)b * D + h * dk + r], wk[(size_t)(h * dk + r) * D + j], acc);
    qk[idx] = acc;
  }
  for (int h = tid >> 5; h < nh; h += kPoolThreads / 32) {  // one warp per head: qs_h . b_k,h
    float acc = 0.f;
    for (int r = tid & 31; r < dk; r += 32) acc = fmaf(qs[(size_t)b * D + h * dk + r], bk[h * dk + r], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((tid & 31) == 0) cst[h] = acc;
  }
  __syncthreads();
  // logits: warps split the nodes, lanes the columns; 4 nodes per step so that up to 16 independent 128-byte row-segment
  // loads are in flight per warp (the tile comes from HBM/L2 exactly here)
  const int warp = tid >> 5, lane = tid & 31, nwarps = kPoolThreads / 32;
  for (int i0 = warp * 4; i0 < n; i0 += nwarps * 4) {
    for (int h0 = 0; h0 < nh; h0 += 4) {  // up to 4 heads per pass (register budget)
      float accl[4][4];  // [node][head]
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int hh = 0; hh < 4; ++hh) accl[r][hh] = 0.f;
      for (int j0 = 0; j0 < D; j0 += 32 * 4) {
        float x[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int j = j0 + 32 * c + lane;
            x[r][c] = (i0 + r < (RAGGED ? nr : n) && j < D) ? xval(Xb[(size_t)(i0 + r) * D + j]) : 0.f;
          }
#pragma unroll
        for (int hh = 0; hh < 4; ++hh) {
          if (h0 + hh < nh) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const int j = j0 + 32 * c + lane;
              const float qv = j < D ? qk[(h0 + hh) * D + j] : 0.f;
#pragma unroll
              for (int r = 0; r < 4; ++r) accl[r][hh] = fmaf(qv, x[r][c], accl[r][hh]);
            }
          }
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = i0 + r;
        if (i < n) {
          const bool masked = tail ? ((i >= (RAGGED ? nr : len) || node_type[RAGGED ? row0 + i : (int64_t)b * n + i] == 3) &&
                                      !(all_masked && i == 0))
                                   : mask[(size_t)b * n + i] != 0;
#pragma unroll
          for (int hh = 0; hh < 4; ++hh) {
            if (h0 + hh < nh) {
              float acc = accl[r][hh];
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
              if (lane == 0) logit[(h0 + hh) * n + i] = masked ? -INFINITY : (acc + cst[h0 + hh]) * inv_temp;
            }
          }
        }
      }
    }
  }
  __syncthreads();
  // masked softmax per head (one warp per head)
  for (int h = warp; h < nh; h += nwarps) {
    float m = -INFINITY;
    for (int i = lane; i < n; i += 32) m = fmaxf(m, logit[h * n + i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int i = lane; i < n; i += 32) {
      const float e = expf(logit[h * n + i] - m);
      logit[h * n + i] = e;
      s += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    for (int i = lane; i < n; i += 32) {
      const float a = logit[h * n + i] / s;
      logit[h * n + i] = a;
      attn_out[((size_t)h * B + b) * n + i] = a;  // head-major [nh*B, n] like the reference
    }
  }
  __syncthreads();
  // attention-weighted node sum: xs[h][j] = Σ_i attn[h][i] * X[i][j].  Warps split the nodes, lanes the columns (coalesced
  // 128-byte row segments, every load independent of the accumulators: the kernel is latency bound, so what matters is
  // how many loads are in flight); per-warp partial sums meet in shared memory.
  float* part = cst + ((nh + 7) / 8) * 8;  // [nwarps][nh][D]
  for (int j0 = 0; j0 < D; j0 += 32 * 4) {
    float acc[4][4];  // [column chunk][head] — up to 4 heads per pass
    for (int h0 = 0; h0 < nh; h0 += 4) {
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int hh = 0; hh < 4; ++hh) acc[c][hh] = 0.f;
#pragma unroll 4
      for (int i = warp; i < (RAGGED ? nr : n); i += nwarps) {  // ragged: the positions past nr have weight 0
        float x[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = j0 + 32 * c + lane;
          x[c] = j < D ? xval(Xb[(size_t)i * D + j]) : 0.f;
        }
#pragma unroll
        for (int hh = 0; hh < 4; ++hh) {
          if (h0 + hh < nh) {
            const float a = logit[(h0 + hh) * n + i];
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[c][hh] = fmaf(a, x[c], acc[c][hh]);
          }
        }
      }
#pragma unroll
      for (int hh = 0; hh < 4; ++hh)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = j0 + 32 * c + lane;
          if (h0 + hh < nh && j < D) part[((size_t)warp * nh + h0 + hh) * D + j] = acc[c][hh];
        }
    }
  }
  __syncthreads();
  for (int idx = tid; idx < nh * D; idx += kPoolThreads) {
    float acc = 0.f;
    for (int w = 0; w < nwarps; ++w) acc += part[(size_t)w * nh * D + idx];
    xs[idx] = acc;
  }
  __syncthreads();
  // value projection of the pooled vector: pooled[b, h*dv + r] = wv[h*dv + r, :]·xs[h] + bv   (one warp per output row:
  // coalesced reads of the weight row, shuffle reduction)
  for (int r0 = warp * 4; r0 < D; r0 += nwarps * 4) {  // 4 rows per step: their weight loads are all independent
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = lane; j < D; j += 32) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int idx = min(r0 + r, D - 1);
        acc[r] = fmaf(wv[(size_t)idx * D + j], xs[(idx / dk) * D + j], acc[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float a = acc[r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0 && r0 + r < D) pooled[(size_t)b * pooled_ld + r0 + r] = a + bv[r0 + r];
    }
  }
  if (tail) {
    float* row = pooled + (size_t)b * pooled_ld;
    for (int j = tid; j < S; j += kPoolThreads) row[D + j] = sent[(size_t)b * S + j];
    for (int j = tid; j < D; j += kPoolThreads) row[D + S + j] = (!RAGGED || nr > 0) ? xval(Xb[j]) : 0.f;
  }
}

// Largest dynamic shared memory attention_pool_kernel takes; larger shapes are refused (QAGNN_ERR_UNSUPPORTED) and the
// caller pools with its einsum path.
constexpr size_t kPoolSmemCap = 200 * 1024;

inline size_t pool_smem_bytes(int n, int D, int nh) {
  return ((size_t)2 * nh * D + (size_t)nh * n + nh + 16 + (size_t)(kPoolThreads / 32) * nh * D) * sizeof(float);
}

// Both entry points launch the same kernel, and cudaFuncSetAttribute overwrites the limit rather than raising it, so the
// limit is set once per device and X type, to the cap, for both of them.
template <typename XT, bool RAGGED = false>
int32_t prepare_pool_launch(size_t smem) {
  static bool attr_set[kMaxDevices] = {false};
  const int dev = current_device();
  if (smem > 48 * 1024 && !attr_set[dev]) {
    QAGNN_CHECK_CUDA(cudaFuncSetAttribute(attention_pool_kernel<XT, RAGGED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)kPoolSmemCap));
    attr_set[dev] = true;
  }
  return QAGNN_OK;
}

template <typename XT>
int32_t decoder_tail(int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S, const XT* X, const float* qs,
                     const int64_t* node_type, const int64_t* adj_lengths, const float* sent_vecs, const float* wk,
                     const float* bk, const float* wv, const float* bv, float* concat, float* attn, cudaStream_t st) {
  if (B <= 0 || n <= 0 || D <= 0 || n_head <= 0 || D % n_head != 0 || S < 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (n_head > 8) return QAGNN_ERR_UNSUPPORTED;
  if (!X || !qs || !node_type || !adj_lengths || !sent_vecs || !wk || !bk || !wv || !bv || !concat || !attn)
    return QAGNN_ERR_INVALID_ARGUMENT;
  const size_t smem = pool_smem_bytes(n, D, n_head);
  if (smem > kPoolSmemCap) return QAGNN_ERR_UNSUPPORTED;
  QAGNN_RETURN_IF(prepare_pool_launch<XT>(smem));
  attention_pool_kernel<XT><<<B, kPoolThreads, smem, st>>>(n, D, n_head, X, qs, nullptr, wk, bk, wv, bv, concat, attn, B,
                                                           node_type, adj_lengths, sent_vecs, S, 2 * D + S);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

// decoder_tail on a ragged X [N_rows, D] (graph b's rows start at node_ptr[b])
template <typename XT>
int32_t decoder_tail_ragged(int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S, int64_t N_rows, const XT* X,
                            const int64_t* node_ptr, const float* qs, const int64_t* node_type, const int64_t* adj_lengths,
                            const float* sent_vecs, const float* wk, const float* bk, const float* wv, const float* bv,
                            float* concat, float* attn, cudaStream_t st) {
  if (B <= 0 || n <= 0 || D <= 0 || n_head <= 0 || D % n_head != 0 || S < 0 || N_rows <= 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (n_head > 8) return QAGNN_ERR_UNSUPPORTED;
  if (!X || !node_ptr || !qs || !node_type || !adj_lengths || !sent_vecs || !wk || !bk || !wv || !bv || !concat || !attn)
    return QAGNN_ERR_INVALID_ARGUMENT;
  const size_t smem = pool_smem_bytes(n, D, n_head);
  if (smem > kPoolSmemCap) return QAGNN_ERR_UNSUPPORTED;
  QAGNN_RETURN_IF((prepare_pool_launch<XT, true>(smem)));
  attention_pool_kernel<XT, true><<<B, kPoolThreads, smem, st>>>(n, D, n_head, X, qs, nullptr, wk, bk, wv, bv, concat, attn, B,
                                                                 node_type, adj_lengths, sent_vecs, S, 2 * D + S, node_ptr, N_rows);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

template <typename XT>
int32_t attention_pool(int32_t B, int32_t n, int32_t D, int32_t n_head, const XT* X, const float* qs, const uint8_t* mask,
                       const float* wk, const float* bk, const float* wv, const float* bv, float* pooled, float* attn,
                       cudaStream_t st) {
  if (B <= 0 || n <= 0 || D <= 0 || n_head <= 0 || D % n_head != 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (n_head > 8) return QAGNN_ERR_UNSUPPORTED;
  if (!X || !qs || !mask || !wk || !bk || !wv || !bv || !pooled || !attn) return QAGNN_ERR_INVALID_ARGUMENT;
  const size_t smem = pool_smem_bytes(n, D, n_head);
  if (smem > kPoolSmemCap) return QAGNN_ERR_UNSUPPORTED;
  QAGNN_RETURN_IF(prepare_pool_launch<XT>(smem));
  attention_pool_kernel<XT><<<B, kPoolThreads, smem, st>>>(n, D, n_head, X, qs, mask, wk, bk, wv, bv, pooled, attn, B);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

}  // namespace
}  // namespace qagnn

using namespace qagnn;

namespace qagnn {
namespace {

// The step before the hot path (SURVEY.md §8f #2): QAGNN.forward's input assembly (modeling/modeling_qagnn.py:153-167), eval mode.
//   H[b,0,:]   = ctx[b,:]                      (= GELU(svec2nvec(sent_vecs)), computed by the caller: a [B, sent_dim] GEMM)
//   H[b,i,:]   = table[concept_ids[b,i] - 1]    i >= 1; `table` = the concept embedding AFTER cpt_transform + GELU, folded
//                                               once per weight set (the table is frozen in eval), so this is a pure gather
//   s          = -(score - score[:,0]) * (i < adj_len);  scores_out = s / (sum_i |s| / adj_len + 1e-5)
// One CTA per graph: the rows are copied as float4, the score norm is one block reduction.
__global__ void __launch_bounds__(256) decoder_head_kernel(int n, int D, const int64_t* __restrict__ concept_ids, int64_t n_concept,
                                                            const float* __restrict__ table, const float* __restrict__ ctx,
                                                            const float* __restrict__ node_scores,
                                                            const int64_t* __restrict__ adj_lengths, float* __restrict__ H_out,
                                                            float* __restrict__ scores_out) {
  __shared__ float red[32];
  __shared__ float s_total;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int64_t* cid = concept_ids + (size_t)b * n;
  const int D4 = D / 4;
  float* Hb = H_out + (size_t)b * n * D;
  for (int i = tid; i < n * D4; i += 256) {
    const int row = i / D4, c = i - row * D4;
    const float* srcp;
    if (row == 0) {
      srcp = ctx + (size_t)b * D;
    } else {
      int64_t id = cid[row] - 1;
      id = id < 0 ? 0 : (id >= n_concept ? n_concept - 1 : id);
      srcp = table + (size_t)id * D;
    }
    reinterpret_cast<float4*>(Hb + (size_t)row * D)[c] = __ldg(reinterpret_cast<const float4*>(srcp) + c);
  }
  const float* sc = node_scores + (size_t)b * n;
  const float s0 = -sc[0];
  const int64_t len = adj_lengths[b];
  float part = 0.f;
  for (int i = tid; i < n; i += 256) part += (i < len) ? fabsf(-sc[i] - s0) : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    s_total = t;
  }
  __syncthreads();
  const float denom = s_total / (float)len + 1e-05f;
  for (int i = tid; i < n; i += 256) scores_out[(size_t)b * n + i] = ((i < len) ? (-sc[i] - s0) : 0.f) / denom;
}

// decoder_head_kernel for a ragged batch: graph b's first min(adj_lengths[b], n) positions become the packed rows from
// node_ptr[b] on of H_out [N_rows, D], scores_out [N_rows] and type_out [N_rows] (the loader's node types), with the same
// values the padded kernel writes there.  The tail rows [node_ptr[B], N_rows) get zeros, type 2 and score 0; CTA b clears rows
// node_ptr[B] + b, + B, ...
__global__ void __launch_bounds__(256) decoder_head_ragged_kernel(int n, int D, int64_t N_rows, const int64_t* __restrict__ concept_ids,
                                                                   int64_t n_concept, const float* __restrict__ table,
                                                                   const float* __restrict__ ctx, const float* __restrict__ node_scores,
                                                                   const int64_t* __restrict__ adj_lengths,
                                                                   const int64_t* __restrict__ node_type,
                                                                   const int64_t* __restrict__ node_ptr, float* __restrict__ H_out,
                                                                   float* __restrict__ scores_out, int64_t* __restrict__ type_out) {
  __shared__ float red[32];
  __shared__ float s_total;
  const int b = blockIdx.x, B = gridDim.x, tid = threadIdx.x;
  const int64_t* cid = concept_ids + (size_t)b * n;
  const int D4 = D / 4;
  const int64_t len = adj_lengths[b];
  const int64_t row0 = min(max(node_ptr[b], (int64_t)0), N_rows);
  const int rows = (int)min(min((int64_t)n, max(len, (int64_t)0)), N_rows - row0);
  float* Hb = H_out + (size_t)row0 * D;
  for (int i = tid; i < rows * D4; i += 256) {
    const int row = i / D4, c = i - row * D4;
    const float* srcp;
    if (row == 0) {
      srcp = ctx + (size_t)b * D;
    } else {
      int64_t id = cid[row] - 1;
      id = id < 0 ? 0 : (id >= n_concept ? n_concept - 1 : id);
      srcp = table + (size_t)id * D;
    }
    reinterpret_cast<float4*>(Hb + (size_t)row * D)[c] = __ldg(reinterpret_cast<const float4*>(srcp) + c);
  }
  const float* sc = node_scores + (size_t)b * n;
  const float s0 = -sc[0];
  float part = 0.f;
  for (int i = tid; i < n; i += 256) part += (i < len) ? fabsf(-sc[i] - s0) : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    s_total = t;
  }
  __syncthreads();
  const float denom = s_total / (float)len + 1e-05f;
  for (int i = tid; i < rows; i += 256) {
    scores_out[row0 + i] = (-sc[i] - s0) / denom;
    type_out[row0 + i] = node_type[(size_t)b * n + i];
  }
  const int64_t t0 = min(max(node_ptr[B], (int64_t)0), N_rows);
  for (int64_t r = t0 + b; r < N_rows; r += B) {
    float4* hr = reinterpret_cast<float4*>(H_out + (size_t)r * D);
    for (int c = tid; c < D4; c += 256) hr[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tid == 0) { scores_out[r] = 0.f; type_out[r] = 2; }
  }
}

// Gradient of the ragged decoder tail (attention_pool_kernel<XT, true>), with a = attn (saved by the forward), x_i the
// graph's rows, qk_h = W_k,hᵀ qs_h and xs_h = Σ_i a_hi x_i, given dpooled = d(concat)[:, :D] and dZ = d(concat)[:, D+S:]:
//   dxs_h = W_v,hᵀ dpooled_h;   g_hi = a_hi (dxs_h·x_i - Σ_i' a_hi' dxs_h·x_i') / sqrt(dk)   (the logit gradient, scaled)
//   dX_i  = Σ_h (a_hi dxs_h + g_hi qk_h) + [i = 0] dZ;   dqk_h = Σ_i g_hi x_i;   dcst_h = Σ_i g_hi
//   dqs_h = W_k,h dqk_h + b_k,h dcst_h;   dW_k,h += qs_h ⊗ dqk_h;   dW_v,h += dpooled_h ⊗ xs_h   (summed over graphs)
// Three launches, every sum in a fixed order and no atomics, so two runs give the same bits: pool_backward_head_kernel (one
// CTA per (graph, head)) writes the per-(graph, head) vectors to scratch, pool_backward_rows_kernel (one CTA per graph) sums
// the heads into dX, and pool_backward_weights_kernel (one CTA per weight row) sums the graphs into dW_k, db_k, dW_v, db_v.
// Scratch (fp32): qk | dxs | xs | dqk [B][nh][D] | g [nh*B][n] (the attn layout) | dcst [B][nh].
struct PoolBwdScratch {
  float *qk, *dxs, *xs, *dqk, *g, *dcst;
  __host__ __device__ PoolBwdScratch(float* s, int B, int n, int D, int nh) {
    const size_t v = (size_t)B * nh * D;
    qk = s; dxs = qk + v; xs = dxs + v; dqk = xs + v; g = dqk + v; dcst = g + (size_t)nh * B * n;
  }
  static size_t floats(int B, int n, int D, int nh) { return 4 * (size_t)B * nh * D + (size_t)nh * B * n + (size_t)B * nh; }
};

constexpr int kPoolBwdThreads = 256;

// rows of graph b the forward pooled over: [row0, row0 + nr), the same clamps as attention_pool_kernel<XT, true>
__device__ __forceinline__ void ragged_graph_rows(int b, int n, const int64_t* node_ptr, const int64_t* adj_lengths,
                                                  int64_t N_rows, int64_t& row0, int& nr) {
  row0 = min(max(node_ptr[b], (int64_t)0), N_rows);
  nr = (int)min(min((int64_t)n, N_rows - row0), max(node_ptr[b + 1] - row0, (int64_t)0));
  nr = (int)min((int64_t)nr, max((int64_t)0, adj_lengths[b]));
}

// Sum of one value per lane over a warp, in a fixed order.
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// dynamic smem: qk[D] | dxs[D] | dqk[D] | red[kPoolBwdThreads / 32].  The per-node vectors stay in global memory: a is the
// forward's attn row, and g is built in place in its scratch row (da_i first, then the logit gradient), so the shared memory
// does not grow with n and the kernel takes every node count the forward takes.
template <typename XT>
__global__ void __launch_bounds__(kPoolBwdThreads) pool_backward_head_kernel(int n, int D, int nh, int S, int64_t N_rows,
                                                                            const XT* __restrict__ X, const int64_t* __restrict__ node_ptr,
                                                                            const int64_t* __restrict__ adj_lengths,
                                                                            const float* __restrict__ qs, const float* __restrict__ wk,
                                                                            const float* __restrict__ bk, const float* __restrict__ wv,
                                                                            const float* __restrict__ attn, const float* __restrict__ dconcat,
                                                                            float* __restrict__ dqs, float* __restrict__ scratch) {
  extern __shared__ float sm[];
  const int b = blockIdx.x, h = blockIdx.y, B = gridDim.x, tid = threadIdx.x, dk = D / nh;
  const int warp = tid >> 5, lane = tid & 31, nwarps = kPoolBwdThreads / 32;
  float* qk = sm;
  float* dxs = qk + D;
  float* dqk = dxs + D;
  float* red = dqk + D;
  PoolBwdScratch sc(scratch, B, n, D, nh);
  const float* a = attn + ((size_t)h * B + b) * n;
  float* g = sc.g + ((size_t)h * B + b) * n;
  int64_t row0;
  int nr;
  ragged_graph_rows(b, n, node_ptr, adj_lengths, N_rows, row0, nr);
  const XT* Xb = X + (size_t)row0 * D;
  const float inv_temp = 1.0f / sqrtf((float)dk);
  const float* qsh = qs + (size_t)b * D + h * dk;
  const float* dph = dconcat + (size_t)b * (2 * D + S) + h * dk;  // dpooled_h
  const size_t vo = ((size_t)b * nh + h) * D;
  for (int j = tid; j < D; j += kPoolBwdThreads) {
    float q = 0.f, d = 0.f;
    for (int r = 0; r < dk; ++r) {
      q = fmaf(qsh[r], wk[(size_t)(h * dk + r) * D + j], q);
      d = fmaf(dph[r], wv[(size_t)(h * dk + r) * D + j], d);
    }
    qk[j] = q;
    dxs[j] = d;
    sc.qk[vo + j] = q;
    sc.dxs[vo + j] = d;
  }
  __syncthreads();
  // da_i = dxs·x_i (one warp per node) into g
  for (int i = warp; i < nr; i += nwarps) {
    float acc = 0.f;
    for (int j = lane; j < D; j += 32) acc = fmaf(dxs[j], xval(Xb[(size_t)i * D + j]), acc);
    acc = warp_sum(acc);
    if (lane == 0) g[i] = acc;
  }
  // xs_h = Σ_i a_i x_i (one thread per column, nodes in order)
  __syncthreads();
  for (int j = tid; j < D; j += kPoolBwdThreads) {
    float acc = 0.f;
    for (int i = 0; i < nr; ++i) acc = fmaf(a[i], xval(Xb[(size_t)i * D + j]), acc);
    sc.xs[vo + j] = acc;
  }
  if (warp == 0) {
    float s = 0.f;
    for (int i = lane; i < nr; i += 32) s = fmaf(a[i], g[i], s);
    s = warp_sum(s);
    if (lane == 0) red[0] = s;
  }
  __syncthreads();
  const float sdot = red[0];
  for (int i = tid; i < n; i += kPoolBwdThreads) {
    g[i] = i < nr ? a[i] * (g[i] - sdot) * inv_temp : 0.f;
  }
  __syncthreads();
  for (int j = tid; j < D; j += kPoolBwdThreads) {
    float acc = 0.f;
    for (int i = 0; i < nr; ++i) acc = fmaf(g[i], xval(Xb[(size_t)i * D + j]), acc);
    dqk[j] = acc;
    sc.dqk[vo + j] = acc;
  }
  if (warp == 0) {
    float s = 0.f;
    for (int i = lane; i < nr; i += 32) s += g[i];
    s = warp_sum(s);
    if (lane == 0) red[1] = s;
  }
  __syncthreads();
  const float dcst = red[1];
  if (tid == 0) sc.dcst[(size_t)b * nh + h] = dcst;
  // dqs_h[r] = W_k[h*dk + r, :]·dqk + b_k[h*dk + r] dcst (one warp per row)
  for (int r = warp; r < dk; r += nwarps) {
    const float* w = wk + (size_t)(h * dk + r) * D;
    float acc = 0.f;
    for (int j = lane; j < D; j += 32) acc = fmaf(w[j], dqk[j], acc);
    acc = warp_sum(acc);
    if (lane == 0) dqs[(size_t)b * D + h * dk + r] = fmaf(bk[h * dk + r], dcst, acc);
  }
}

// dX rows of graph b: Σ_h (a_hi dxs_h + g_hi qk_h), plus dZ on row 0.  Other rows are left as the caller zeroed them.
__global__ void __launch_bounds__(kPoolBwdThreads) pool_backward_rows_kernel(int n, int D, int nh, int S, int64_t N_rows,
                                                                            const int64_t* __restrict__ node_ptr,
                                                                            const int64_t* __restrict__ adj_lengths,
                                                                            const float* __restrict__ attn,
                                                                            const float* __restrict__ dconcat,
                                                                            const float* __restrict__ scratch, float* __restrict__ dX) {
  const int b = blockIdx.x, B = gridDim.x;
  PoolBwdScratch sc(const_cast<float*>(scratch), B, n, D, nh);
  int64_t row0;
  int nr;
  ragged_graph_rows(b, n, node_ptr, adj_lengths, N_rows, row0, nr);
  const float* dZ = dconcat + (size_t)b * (2 * D + S) + D + S;
  for (int idx = threadIdx.x; idx < nr * D; idx += kPoolBwdThreads) {
    const int i = idx / D, j = idx - i * D;
    float acc = i == 0 ? dZ[j] : 0.f;
    for (int h = 0; h < nh; ++h) {
      const size_t vo = ((size_t)b * nh + h) * D + j, ao = ((size_t)h * B + b) * n + i;
      acc = fmaf(attn[ao], sc.dxs[vo], acc);
      acc = fmaf(sc.g[ao], sc.qk[vo], acc);
    }
    dX[(size_t)(row0 + i) * D + j] = acc;
  }
}

// Row r of dW_k / dW_v (head h = r / dk) and db_k[r] / db_v[r]: sums over the graphs in order.
__global__ void __launch_bounds__(kPoolBwdThreads) pool_backward_weights_kernel(int B, int n, int D, int nh, int S,
                                                                               const float* __restrict__ qs,
                                                                               const float* __restrict__ dconcat,
                                                                               const float* __restrict__ scratch,
                                                                               float* __restrict__ dwk, float* __restrict__ dbk,
                                                                               float* __restrict__ dwv, float* __restrict__ dbv) {
  const int r = blockIdx.x, h = r / (D / nh);
  PoolBwdScratch sc(const_cast<float*>(scratch), B, n, D, nh);
  const size_t ld = 2 * (size_t)D + S;
  for (int j = threadIdx.x; j < D; j += kPoolBwdThreads) {
    float ak = 0.f, av = 0.f;
    for (int b = 0; b < B; ++b) {
      const size_t vo = ((size_t)b * nh + h) * D + j;
      ak = fmaf(qs[(size_t)b * D + r], sc.dqk[vo], ak);
      av = fmaf(dconcat[b * ld + r], sc.xs[vo], av);
    }
    dwk[(size_t)r * D + j] = ak;
    dwv[(size_t)r * D + j] = av;
  }
  if (threadIdx.x == 0) {
    float ak = 0.f, av = 0.f;
    for (int b = 0; b < B; ++b) {
      ak = fmaf(qs[(size_t)b * D + r], sc.dcst[(size_t)b * nh + h], ak);
      av += dconcat[b * ld + r];
    }
    dbk[r] = ak;
    dbv[r] = av;
  }
}

// (3D + 8) floats: always less than pool_smem_bytes(n, D, nh) (10 nh D + nh n + nh + 16 floats), so the backward takes
// every shape the forward takes.  Above 48 KB (D > 4093) it opts in, once per device and X type, to the forward's cap.
inline size_t pool_backward_smem_bytes(int D) { return ((size_t)3 * D + kPoolBwdThreads / 32) * sizeof(float); }

template <typename XT>
int32_t prepare_pool_backward_launch(size_t smem) {
  static bool attr_set[kMaxDevices] = {false};
  const int dev = current_device();
  if (smem > 48 * 1024 && !attr_set[dev]) {
    QAGNN_CHECK_CUDA(cudaFuncSetAttribute(pool_backward_head_kernel<XT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)kPoolSmemCap));
    attr_set[dev] = true;
  }
  return QAGNN_OK;
}

template <typename XT>
int32_t pool_backward_ragged(int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S, int64_t N_rows, const XT* X,
                             const int64_t* node_ptr, const int64_t* adj_lengths, const float* qs, const float* wk,
                             const float* bk, const float* wv, const float* attn, const float* dconcat, float* dX, float* dqs,
                             float* dwk, float* dbk, float* dwv, float* dbv, float* scratch, size_t scratch_bytes,
                             cudaStream_t st) {
  if (B <= 0 || n <= 0 || D <= 0 || n_head <= 0 || D % n_head != 0 || S < 0 || N_rows <= 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (n_head > 8) return QAGNN_ERR_UNSUPPORTED;
  if (!X || !node_ptr || !adj_lengths || !qs || !wk || !bk || !wv || !attn || !dconcat || !dX || !dqs || !dwk || !dbk || !dwv ||
      !dbv || !scratch)
    return QAGNN_ERR_INVALID_ARGUMENT;
  if (scratch_bytes < PoolBwdScratch::floats(B, n, D, n_head) * sizeof(float)) return QAGNN_ERR_WORKSPACE;
  if (pool_smem_bytes(n, D, n_head) > kPoolSmemCap) return QAGNN_ERR_UNSUPPORTED;  // the forward refuses these too
  const size_t smem = pool_backward_smem_bytes(D);
  QAGNN_RETURN_IF(prepare_pool_backward_launch<XT>(smem));
  QAGNN_CHECK_CUDA(cudaMemsetAsync(dX, 0, (size_t)N_rows * D * sizeof(float), st));
  pool_backward_head_kernel<XT><<<dim3(B, n_head), kPoolBwdThreads, smem, st>>>(n, D, n_head, S, N_rows, X, node_ptr, adj_lengths,
                                                                                qs, wk, bk, wv, attn, dconcat, dqs, scratch);
  QAGNN_CHECK_LAUNCH();
  pool_backward_rows_kernel<<<B, kPoolBwdThreads, 0, st>>>(n, D, n_head, S, N_rows, node_ptr, adj_lengths, attn, dconcat,
                                                           scratch, dX);
  QAGNN_CHECK_LAUNCH();
  pool_backward_weights_kernel<<<D, kPoolBwdThreads, 0, st>>>(B, n, D, n_head, S, qs, dconcat, scratch, dwk, dbk, dwv, dbv);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

}  // namespace
}  // namespace qagnn

extern "C" size_t qagnn_attention_pool_backward_ragged_scratch_bytes(int32_t B, int32_t n, int32_t D, int32_t n_head) {
  if (B <= 0 || n <= 0 || D <= 0 || n_head <= 0 || D % n_head != 0) return 0;
  return qagnn::PoolBwdScratch::floats(B, n, D, n_head) * sizeof(float);
}

extern "C" int32_t qagnn_attention_pool_backward_ragged(int32_t x_dtype, int32_t B, int32_t n, int32_t D, int32_t n_head,
                                                        int32_t S, int64_t N_rows, const void* X, const int64_t* node_ptr,
                                                        const int64_t* adj_lengths, const float* qs, const float* wk,
                                                        const float* bk, const float* wv, const float* attn,
                                                        const float* d_concat, float* dX, float* d_qs, float* d_wk, float* d_bk,
                                                        float* d_wv, float* d_bv, float* scratch, size_t scratch_bytes,
                                                        void* stream) {
  if (x_dtype == QAGNN_DTYPE_F32)
    return pool_backward_ragged(B, n, D, n_head, S, N_rows, (const float*)X, node_ptr, adj_lengths, qs, wk, bk, wv, attn, d_concat,
                                dX, d_qs, d_wk, d_bk, d_wv, d_bv, scratch, scratch_bytes, (cudaStream_t)stream);
  if (x_dtype != QAGNN_DTYPE_BF16) return QAGNN_ERR_INVALID_ARGUMENT;
  return pool_backward_ragged(B, n, D, n_head, S, N_rows, (const __nv_bfloat16*)X, node_ptr, adj_lengths, qs, wk, bk, wv, attn,
                              d_concat, dX, d_qs, d_wk, d_bk, d_wv, d_bv, scratch, scratch_bytes, (cudaStream_t)stream);
}

extern "C" int32_t qagnn_decoder_head_ragged(int32_t B, int32_t n, int32_t D, int64_t N_rows, const int64_t* concept_ids,
                                             int64_t n_concept, const float* table, const float* ctx, const float* node_scores,
                                             const int64_t* adj_lengths, const int64_t* node_type, const int64_t* node_ptr,
                                             float* H_out, float* scores_out, int64_t* type_out, void* stream) {
  if (B <= 0 || n <= 0 || D <= 0 || D % 4 != 0 || n_concept <= 0 || N_rows <= 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (!concept_ids || !table || !ctx || !node_scores || !adj_lengths || !node_type || !node_ptr || !H_out || !scores_out || !type_out)
    return QAGNN_ERR_INVALID_ARGUMENT;
  qagnn::decoder_head_ragged_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n, D, N_rows, concept_ids, n_concept, table, ctx,
                                                                          node_scores, adj_lengths, node_type, node_ptr, H_out,
                                                                          scores_out, type_out);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

extern "C" int32_t qagnn_decoder_tail_ragged(int32_t x_dtype, int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S,
                                             int64_t N_rows, const void* X, const int64_t* node_ptr, const float* qs,
                                             const int64_t* node_type, const int64_t* adj_lengths, const float* sent_vecs,
                                             const float* wk, const float* bk, const float* wv, const float* bv, float* concat,
                                             float* attn, void* stream) {
  if (x_dtype == QAGNN_DTYPE_F32)
    return decoder_tail_ragged(B, n, D, n_head, S, N_rows, (const float*)X, node_ptr, qs, node_type, adj_lengths, sent_vecs, wk,
                               bk, wv, bv, concat, attn, (cudaStream_t)stream);
  if (x_dtype != QAGNN_DTYPE_BF16) return QAGNN_ERR_INVALID_ARGUMENT;
  return decoder_tail_ragged(B, n, D, n_head, S, N_rows, (const __nv_bfloat16*)X, node_ptr, qs, node_type, adj_lengths, sent_vecs,
                             wk, bk, wv, bv, concat, attn, (cudaStream_t)stream);
}

extern "C" int32_t qagnn_decoder_head(int32_t B, int32_t n, int32_t D, const int64_t* concept_ids, int64_t n_concept,
                                      const float* table, const float* ctx, const float* node_scores,
                                      const int64_t* adj_lengths, float* H_out, float* scores_out, void* stream) {
  if (B <= 0 || n <= 0 || D <= 0 || D % 4 != 0 || n_concept <= 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (!concept_ids || !table || !ctx || !node_scores || !adj_lengths || !H_out || !scores_out) return QAGNN_ERR_INVALID_ARGUMENT;
  qagnn::decoder_head_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n, D, concept_ids, n_concept, table, ctx, node_scores,
                                                                   adj_lengths, H_out, scores_out);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

extern "C" int32_t qagnn_decoder_tail(int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S, const float* X, const float* qs,
                                      const int64_t* node_type, const int64_t* adj_lengths, const float* sent_vecs,
                                      const float* wk, const float* bk, const float* wv, const float* bv, float* concat,
                                      float* attn, void* stream) {
  return decoder_tail(B, n, D, n_head, S, X, qs, node_type, adj_lengths, sent_vecs, wk, bk, wv, bv, concat, attn,
                      (cudaStream_t)stream);
}

extern "C" int32_t qagnn_attention_pool(int32_t B, int32_t n, int32_t D, int32_t n_head, const float* X, const float* qs,
                                        const uint8_t* mask, const float* wk, const float* bk, const float* wv, const float* bv,
                                        float* pooled, float* attn, void* stream) {
  return attention_pool(B, n, D, n_head, X, qs, mask, wk, bk, wv, bv, pooled, attn, (cudaStream_t)stream);
}

extern "C" int32_t qagnn_decoder_tail_typed(int32_t x_dtype, int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S,
                                            const void* X, const float* qs, const int64_t* node_type, const int64_t* adj_lengths,
                                            const float* sent_vecs, const float* wk, const float* bk, const float* wv,
                                            const float* bv, float* concat, float* attn, void* stream) {
  if (x_dtype == QAGNN_DTYPE_F32)
    return decoder_tail(B, n, D, n_head, S, (const float*)X, qs, node_type, adj_lengths, sent_vecs, wk, bk, wv, bv, concat,
                        attn, (cudaStream_t)stream);
  if (x_dtype != QAGNN_DTYPE_BF16) return QAGNN_ERR_INVALID_ARGUMENT;
  return decoder_tail(B, n, D, n_head, S, (const __nv_bfloat16*)X, qs, node_type, adj_lengths, sent_vecs, wk, bk, wv, bv, concat,
                      attn, (cudaStream_t)stream);
}

extern "C" int32_t qagnn_attention_pool_typed(int32_t x_dtype, int32_t B, int32_t n, int32_t D, int32_t n_head, const void* X,
                                              const float* qs, const uint8_t* mask, const float* wk, const float* bk,
                                              const float* wv, const float* bv, float* pooled, float* attn, void* stream) {
  if (x_dtype == QAGNN_DTYPE_F32)
    return attention_pool(B, n, D, n_head, (const float*)X, qs, mask, wk, bk, wv, bv, pooled, attn, (cudaStream_t)stream);
  if (x_dtype != QAGNN_DTYPE_BF16) return QAGNN_ERR_INVALID_ARGUMENT;
  return attention_pool(B, n, D, n_head, (const __nv_bfloat16*)X, qs, mask, wk, bk, wv, bv, pooled, attn, (cudaStream_t)stream);
}
