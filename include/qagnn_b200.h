/*
 * qagnn_b200 — C ABI of the H100-native (sm_90a) QA-GNN message-passing path.
 *
 * The reference (michiyasunaga/qagnn) has no FFI layer: its operator API for this path is the
 * Python nn.Module surface in modeling/modeling_qagnn.py.  This header is the boundary a
 * maintainer binds (ctypes stub in INTEGRATION.md) to replace, one-for-one:
 *
 *   qagnn_graph_prep          <- the index work of GATConvE.forward     modeling_qagnn.py:419-438
 *                                + the out-degree count of message()     modeling_qagnn.py:476-479
 *   qagnn_fold_weights        <- edge_encoder on one-hots :30,:433; BatchNorm(eval) :30,:408;
 *                                linear_key/linear_msg/linear_query weight views :401-403,:464-466
 *   qagnn_gatconve_forward    <- GATConvE.forward / GATConvE.message      modeling_qagnn.py:411-484
 *                                (+ torch_geometric propagate/softmax, torch_scatter scatter)
 *   qagnn_node_feature_extra  <- QAGNN_Message_Passing.forward prologue   modeling_qagnn.py:62-73,86
 *   qagnn_mp_forward          <- QAGNN_Message_Passing.forward            modeling_qagnn.py:53-95
 *                                (mp_helper :45-50, Vh/Vx epilogue :92)
 *   qagnn_mp_core_forward /   <- the autograd graph of GATConvE.message + propagate in TRAINING mode
 *   qagnn_mp_core_backward       (modeling_qagnn.py:442,455-484 under qagnn.py:249-278 loss.backward()):
 *                                message passing on node-level projections with the attention kept for backward,
 *                                and its gradient w.r.t. the projections and the two edge tables
 *                                (_typed: the same on fp16 / bf16 operands, for training under torch.autocast)
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in _host; the caller owns every
 *     buffer (inputs, outputs, workspaces); the library never allocates, frees or retains them;
 *   - sizes of the opaque workspaces come from the *_bytes() queries; buffers must be 256-byte
 *     aligned (torch allocations are);
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); calls are re-entrant per
 *     stream and asynchronous, except qagnn_graph_prep with validate != 0, which synchronises the
 *     stream once to report out-of-range indices;
 *   - return value: 0 = ok, negative = error (qagnn_status_string).  No C++ exceptions cross
 *     the boundary;
 *   - dtypes: features fp32 row-major, indices int64 exactly as the reference's loader
 *     (utils/data_utils.py:79-197) produces them.  qagnn_gatconve_forward / qagnn_mp_forward are the eval-mode forward
 *     (dropout = identity, BatchNorm running statistics folded), the reference's evaluate_accuracy path (qagnn.py:30-38);
 *     training mode composes qagnn_mp_core_forward / _backward with the caller's dense layers (qagnn_b200/training.py).
 */
#ifndef QAGNN_B200_H_
#define QAGNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QAGNN_ABI_VERSION 3 /* 3: + training core, packed graph prep, decoder head / tail (round 2); ragged eval entry points; batch assembly */

enum {
  QAGNN_OK = 0,
  QAGNN_ERR_INVALID_ARGUMENT = -1, /* null pointer, non-positive size, D % H != 0, ... */
  QAGNN_ERR_CUDA = -2,             /* a launch or runtime call failed; see qagnn_last_cuda_error */
  QAGNN_ERR_INDEX_RANGE = -3,      /* edge_index / edge_type / node_type outside its range */
  QAGNN_ERR_WORKSPACE = -4,        /* caller-provided workspace is too small */
  QAGNN_ERR_UNSUPPORTED = -5       /* shape outside what the kernels are instantiated for */
};

/* Problem shape.  N nodes in the batched graph, E real directed edges (self loops excluded; the
 * library appends the N self loops itself, modeling_qagnn.py:436-438), D = emb_dim, H = head_count
 * (modeling_qagnn.py:387), T = n_ntype, R = n_etype, k = number of GATConvE layers,
 * n_per_graph = nodes per sub-graph when the batch is made of equal-sized sub-graphs laid out
 * back to back as LM_QAGNN.batch_graph does (modeling_qagnn.py:244-251), else 0 (unknown). */
typedef struct qagnn_shape {
  int64_t N;
  int64_t E;
  int32_t D;
  int32_t H;
  int32_t T;
  int32_t R;
  int32_t k;
  int32_t n_per_graph;
} qagnn_shape;

/* Raw parameters, in the reference's own layout (row-major [out, in], fp32), i.e. pointers into
 * the tensors of the module's state_dict. */
typedef struct qagnn_edge_encoder_params { /* modeling_qagnn.py:30 */
  const float *lin0_w, *lin0_b;            /* [D, R+1+2T], [D]  edge_encoder.0 */
  const float *bn_w, *bn_b, *bn_mean, *bn_var; /* [D] each     edge_encoder.1 */
  const float *lin3_w, *lin3_b;            /* [D, D], [D]      edge_encoder.3 */
} qagnn_edge_encoder_params;

typedef struct qagnn_layer_params { /* GATConvE, modeling_qagnn.py:401-408 */
  const float *key_w, *key_b;       /* [D, 3D], [D] linear_key   */
  const float *msg_w, *msg_b;       /* [D, 3D], [D] linear_msg   */
  const float *query_w, *query_b;   /* [D, 2D], [D] linear_query */
  const float *mlp0_w, *mlp0_b;     /* [D, D], [D]  mlp.0 */
  const float *bn_w, *bn_b, *bn_mean, *bn_var; /* [D] each mlp.1 */
  const float *mlp3_w, *mlp3_b;     /* [D, D], [D]  mlp.3 */
} qagnn_layer_params;

typedef struct qagnn_mp_params { /* QAGNN_Message_Passing, modeling_qagnn.py:19-38 */
  const float *emb_node_type_w, *emb_node_type_b; /* [D/2, T], [D/2]   */
  const float *emb_score_w, *emb_score_b;         /* [D/2, D/2], [D/2] */
  const float *vh_w, *vh_b, *vx_w, *vx_b;         /* [D, D], [D] each  */
  const float *score_basis;                       /* [D/2] = float32 pow(1.1, j), modeling_qagnn.py:70-71 */
} qagnn_mp_params;

int32_t qagnn_abi_version(void);
const char *qagnn_status_string(int32_t status);
/* cudaError_t of the most recent QAGNN_ERR_CUDA on this thread, as text. */
const char *qagnn_last_cuda_error(void);

/* ---- graph prep (once per forward, shared by all k layers) ------------------------------- */

/* Byte offsets of the arrays inside the opaque prep workspace (for inspection / tests).
 * E' = E + N.  All arrays are int32. */
typedef struct qagnn_prep_layout {
  size_t total_bytes;
  size_t src;          /* [E'] source of edge e (self loops at e >= E)                */
  size_t tgt;          /* [E'] target of edge e                                       */
  size_t combo;        /* [E'] (etype*T + type[src])*T + type[tgt]; self loop of v: R*T*T + type[v] */
  size_t rowptr_src;   /* [N+1] CSR by source; out-degree = rowptr_src[v+1]-rowptr_src[v] */
  size_t rowptr_tgt;   /* [N+1] CSR by target                                         */
  size_t perm_src;     /* [E'] edge ids stably sorted by source                        */
  size_t perm_tgt;     /* [E'] edge ids stably sorted by target                        */
  size_t csr_src_tgt;  /* [E'] tgt[perm_src[p]]                                       */
  size_t csr_src_combo;/* [E'] combo[perm_src[p]]                                     */
  size_t csr_tgt_src;  /* [E'] src[perm_tgt[p]]                                       */
  size_t csr_tgt_combo;/* [E'] combo[perm_tgt[p]]                                     */
  size_t csr_tgt_apos; /* [E'] position of edge perm_tgt[p] in the by-source order      */
  size_t pk_src;       /* [E'] (tgt - graph_base) << 16 | combo, by-source order (n_per_graph > 0 only) */
  size_t pk_tgt;       /* [E'] (src - graph_base) << 16 | combo, by-target order (n_per_graph > 0 only) */
  size_t csr_src_tpos; /* [E'] position of edge perm_src[p] in the by-target order       */
  size_t order_src;    /* [N]  per sub-graph: local node ids sorted by out-degree, descending (n_per_graph > 0) */
  size_t order_tgt;    /* [N]  same by in-degree: the tiled kernel gives each warp 4 nodes of similar degree   */
  size_t ninfo_src;    /* [N] x 2 words, per sub-graph in order_src order: {local id | min(out-degree, 65535) << 16, rowptr_src[v]} */
  size_t ninfo_tgt;    /* [N] x 2 words, same in order_tgt order with the in-degree and rowptr_tgt[v] (n_per_graph > 0)   */
  size_t status;       /* [4]  device-side error word + counters                        */
  size_t scratch;      /* internal                                                     */
} qagnn_prep_layout;

int32_t qagnn_graph_prep_layout(int64_t N, int64_t E, qagnn_prep_layout *out_host);
size_t qagnn_graph_prep_bytes(int64_t N, int64_t E);

/* edge_index int64 [2,E] (row 0 = source, row 1 = target), edge_type int64 [E] in [0,R),
 * node_type int64 [N] in [0,T).  validate != 0: synchronise `stream` and return
 * QAGNN_ERR_INDEX_RANGE if any index is out of range (the kernels clamp, never fault).
 * shape->n_per_graph > 0 additionally asserts that no edge crosses a sub-graph boundary
 * (src / n_per_graph == tgt / n_per_graph), which LM_QAGNN.batch_graph guarantees; a violation is
 * reported as QAGNN_ERR_INDEX_RANGE as well.  It enables the shared-memory-tiled kernels. */
int32_t qagnn_graph_prep(const int64_t *edge_index, const int64_t *edge_type, const int64_t *node_type,
                         const qagnn_shape *shape, void *prep, size_t prep_bytes, int32_t validate,
                         void *stream);

/* The same prep for a PACKED batch: the edges of sub-graph g occupy [graph_ptr[g], graph_ptr[g+1]) of edge_index / edge_type (what
 * LM_QAGNN.batch_graph, modeling_qagnn.py:244-251, and qagnn_b200.data.pack_adj produce; graph_ptr int64 [N/n_per_graph + 1] on the
 * DEVICE) and max_edges_per_graph bounds their length (host value).  One CTA builds everything for one sub-graph in shared memory:
 * one launch instead of twelve, bit-identical arrays.  QAGNN_ERR_UNSUPPORTED when a sub-graph does not fit one CTA's shared
 * memory (use qagnn_graph_prep); an edge outside its sub-graph's node range sets the same status bit as qagnn_graph_prep.
 *
 * Edge capacity: shape->E may exceed the batch's edge count.  The real count is graph_ptr[N/n_per_graph], read on the device, so
 * one set of buffer shapes (and one captured CUDA graph) serves batches with different edge counts.  With E' = graph_ptr[B] + N:
 *   - columns [graph_ptr[B], E) of edge_index / edge_type are never read;
 *   - src / tgt / combo hold -1 at those ids; self loops keep the ids E + v, behind every real edge;
 *   - rowptr_src[N] = rowptr_tgt[N] = E', and every CSR-ordered array is defined at positions below E' only;
 *   - graph_ptr[B] > E sets a status bit (QAGNN_ERR_INDEX_RANGE with validate) and nothing past E is read.
 * The forward / training calls take the same shape and touch no entry of the unused ids; alpha_out rows of those ids are 0.
 * When graph_ptr[B] == E every array is what it was without the capacity rule. */
int32_t qagnn_graph_prep_packed(const int64_t *edge_index, const int64_t *edge_type, const int64_t *node_type,
                                const int64_t *graph_ptr, int32_t max_edges_per_graph, const qagnn_shape *shape, void *prep,
                                size_t prep_bytes, int32_t validate, void *stream);

/* The packed prep for a RAGGED batch (eval): sub-graph g < n_graphs owns the rows [node_ptr[g], node_ptr[g+1]) of an N-row batch
 * (shape->N = the node capacity; node_ptr int64 [n_graphs + 1] on the DEVICE, node_ptr[0] = 0) instead of [g*n, (g+1)*n), and its
 * edges the columns [graph_ptr[g], graph_ptr[g+1]) as above.  shape->n_per_graph = n bounds the rows of one sub-graph (it sizes
 * the CTA's shared memory; N need not be a multiple of it).  The tail rows [node_ptr[n_graphs], N) belong to no sub-graph and get
 * their self loops only; the tiled kernel walks them in segments of n rows.  An edge with an endpoint outside its sub-graph's
 * rows sets bit 8; a node_ptr that is not monotone, has a sub-graph of more than n rows, does not start at 0, ends past N, or
 * gives a sub-graph with edges no rows sets bit 32 (that sub-graph is then left untouched).  With validate either is
 * QAGNN_ERR_INDEX_RANGE.  Edge capacity, the status word and QAGNN_ERR_UNSUPPORTED are as for qagnn_graph_prep_packed. */
int32_t qagnn_graph_prep_ragged(const int64_t *edge_index, const int64_t *edge_type, const int64_t *node_type,
                                const int64_t *graph_ptr, const int64_t *node_ptr, int32_t n_graphs, int32_t max_edges_per_graph,
                                const qagnn_shape *shape, void *prep, size_t prep_bytes, int32_t validate, void *stream);

/* ---- weight folding (once per set of weights) --------------------------------------------- */

size_t qagnn_fold_bytes(const qagnn_shape *shape);
/* `layers_host` is a HOST array of shape->k structs holding DEVICE pointers; `mp_host` may be NULL
 * when only qagnn_gatconve_forward will be used. */
int32_t qagnn_fold_weights(const qagnn_shape *shape, const qagnn_edge_encoder_params *edge_encoder_host,
                           const qagnn_layer_params *layers_host, const qagnn_mp_params *mp_host,
                           void *folded, size_t folded_bytes, void *stream);

/* ---- forward ----------------------------------------------------------------------------------- */

size_t qagnn_forward_workspace_bytes(const qagnn_shape *shape);

/* One GATConvE layer `layer` (0-based index into the folded blob):
 *   out[N,D] = mlp(propagate(...))   (NO GELU: that is applied by mp_helper, modeling_qagnn.py:48)
 * alpha_out (optional, may be NULL): [E+N, H] softmax weights BEFORE the out-degree rescale, in
 * edge_index' order (real edges, then self loops) — what return_attention_weights=True returns.
 * aggr_out (optional): [N,D] propagate() output before the node MLP. */
int32_t qagnn_gatconve_forward(const qagnn_shape *shape, int32_t layer, const float *x, const float *extra,
                               const void *prep, const void *folded, float *out, float *alpha_out,
                               float *aggr_out, void *workspace, size_t workspace_bytes, void *stream);

/* Which message-passing kernels qagnn_gatconve_forward / qagnn_mp_forward run for `shape` on the current device, under the
 * current QAGNN_MP_PATH: the shared-memory-tiled per-graph kernel, the column-sliced kernels, or the basic CSR kernels
 * (head counts 1, 2, 4, 8, 16 and D % 4 == 0, D <= 1024; other shapes are refused there with QAGNN_ERR_UNSUPPORTED).
 * Read-only; a negative status for an invalid shape. */
enum { QAGNN_MP_PATH_TILED = 0, QAGNN_MP_PATH_SLICE = 1, QAGNN_MP_PATH_BASIC = 2 };
int32_t qagnn_mp_path(const qagnn_shape *shape);

/* node_feature_extra[N,D] = [GELU(emb_node_type(onehot(type))) ‖ GELU(emb_score(sin(basis*score)))] */
int32_t qagnn_node_feature_extra(const qagnn_shape *shape, const int64_t *node_type, const float *node_score,
                                 const void *folded, float *extra_out, void *workspace, size_t workspace_bytes,
                                 void *stream);

/* Whole QAGNN_Message_Passing.forward (eval): H_in [N,D], node_type int64 [N], node_score [N],
 * out [N,D] = GELU(Vh(H_in) + Vx(X_k)).  x_layers_out (optional): [k,N,D] activations after each
 * layer's GELU. */
int32_t qagnn_mp_forward(const qagnn_shape *shape, const float *H_in, const int64_t *node_type,
                         const float *node_score, const void *prep, const void *folded, float *out,
                         float *x_layers_out, void *workspace, size_t workspace_bytes, void *stream);

/* The eval forward under bf16 autocast.  `dtype` (QAGNN_DTYPE_*, below) is the storage type of out and selects the GEMMs;
 * `in_dtype` that of x / extra / H_in (QAGNN_DTYPE_F32 or QAGNN_DTYPE_BF16; an fp32 input is rounded to nearest even as it is
 * written into the GEMM operand, as autocast's cast would round it).  QAGNN_DTYPE_F32 (with fp32 inputs) runs
 * qagnn_gatconve_forward / qagnn_mp_forward.  QAGNN_DTYPE_BF16: every GEMM of the tensor-core path
 * (emb_score, the projection with its per-type bias rows, mlp.0 / mlp.3 or the fused MLP, Vh|Vx) takes the bf16 operands
 * that path feeds it - the inputs as given, the folded weights rounded to nearest even - and accumulates in fp32 in the same
 * k order; bias and activation are fp32 in the epilogue.  The folds, the Q|Kx|Mx tiles, logits, softmax and aggr sums stay
 * fp32 (the message passing is the fp32 one).  out is the fp32 epilogue value rounded to nearest even; x_layers_out,
 * alpha_out and aggr_out stay fp32.  Shapes without the wgmma GEMM (D % 8 != 0, QAGNN_GEMM=ffma) run the fp32 path on the
 * widened inputs and round its output.  QAGNN_DTYPE_F16: QAGNN_ERR_INVALID_ARGUMENT. */
int32_t qagnn_gatconve_forward_typed(const qagnn_shape *shape, int32_t dtype, int32_t in_dtype, int32_t layer, const void *x,
                                     const void *extra, const void *prep, const void *folded, void *out, float *alpha_out,
                                     float *aggr_out, void *workspace, size_t workspace_bytes, void *stream);
int32_t qagnn_mp_forward_typed(const qagnn_shape *shape, int32_t dtype, int32_t in_dtype, const void *H_in,
                               const int64_t *node_type, const float *node_score, const void *prep, const void *folded,
                               void *out, float *x_layers_out, void *workspace, size_t workspace_bytes, void *stream);

/* qagnn_gatconve_forward_typed / qagnn_mp_forward_typed on a ragged batch built by qagnn_graph_prep_ragged with the same
 * n_graphs and node_ptr: every node array has shape->N rows (the node capacity), tail rows included, and the tiled message
 * passing takes each sub-graph's rows from node_ptr (the column-sliced and CSR kernels take any layout).  Every row of the
 * output of a sub-graph is what the padded layout computes for that row, within the summation-order bounds of the GEMMs'
 * row tiling; tail rows are computed like isolated nodes. */
int32_t qagnn_gatconve_forward_ragged(const qagnn_shape *shape, int32_t dtype, int32_t in_dtype, int32_t n_graphs,
                                      const int64_t *node_ptr, int32_t layer, const void *x, const void *extra, const void *prep,
                                      const void *folded, void *out, float *alpha_out, float *aggr_out, void *workspace,
                                      size_t workspace_bytes, void *stream);
int32_t qagnn_mp_forward_ragged(const qagnn_shape *shape, int32_t dtype, int32_t in_dtype, int32_t n_graphs,
                                const int64_t *node_ptr, const void *H_in, const int64_t *node_type, const float *node_score,
                                const void *prep, const void *folded, void *out, float *x_layers_out, void *workspace,
                                size_t workspace_bytes, void *stream);

/* ---- training (SURVEY.md §8f #3) --------------------------------------------------------------- */

/* Message passing of one layer on caller-computed node-level projections, keeping what backward needs.
 *   qkm [N, 3D] row-major = [Q/sqrt(d) | Kx | Mx]  (Q = linear_query([x|extra])/sqrt(d), Kx / Mx = the [x|extra] part of
 *   linear_key / linear_msg), ke / me [C, D] = edge-table part of linear_key / linear_msg (+ bias) per combo,
 *   C = R*T*T + T (see qagnn_prep_layout.combo).
 * Outputs: aggr [N, D] (propagate() output), alpha_scaled [E+N, H] = softmax * out-degree in BY-SOURCE order (saved for
 * backward), alpha_out (optional) [E+N, H] un-scaled softmax in edge_index' order.  `scratch` = [E+N, H] floats. */
int32_t qagnn_mp_core_forward(const qagnn_shape *shape, const void *prep, const float *qkm, const float *ke, const float *me,
                              float *aggr, float *alpha_scaled, float *alpha_out, float *scratch, void *stream);

/* Gradient of qagnn_mp_core_forward: given d_aggr [N, D] writes d_qkm [N, 3D], d_ke / d_me [C, D] (zeroed here first).
 * combo_order int32 [E']: the by-source edge positions below E' = rowptr_src[N] stably sorted by
 * qagnn_prep_layout.csr_src_combo (the caller builds it once per batch; E' < E + N under an edge capacity).  `scratch` = [E+N, H] floats.  Only dKe / dMe use atomics (a few thousand vector adds). */
int32_t qagnn_mp_core_backward(const qagnn_shape *shape, const void *prep, const int32_t *combo_order, const float *qkm,
                               const float *ke, const float *me, const float *alpha_scaled, const float *d_aggr,
                               float *d_qkm, float *d_ke, float *d_me, float *scratch, void *stream);

/* The same two calls with the node and table operands stored as `dtype`: qkm, ke, me, aggr, d_aggr, d_qkm, d_ke and d_me are
 * arrays of that type (the training loop's autocast dtype, so no cast to fp32 runs around the core); alpha_scaled, alpha_out and
 * scratch stay fp32.  Loads widen exactly and all arithmetic is fp32, as in the fp32 calls: aggr and d_qkm are the fp32 results
 * rounded once to nearest even, and d_ke / d_me are accumulated in fp32 (atomics, in `scratch`) and rounded once at the end.
 * QAGNN_DTYPE_F32 runs the fp32 calls above.  `scratch` holds at least qagnn_mp_core_scratch_bytes(shape, dtype) bytes; 16-bit
 * rows are read and written 4 elements (8 bytes) at a time.  QAGNN_ERR_INVALID_ARGUMENT for an unknown dtype. */
enum { QAGNN_DTYPE_F32 = 0, QAGNN_DTYPE_F16 = 1, QAGNN_DTYPE_BF16 = 2 };
size_t qagnn_mp_core_scratch_bytes(const qagnn_shape *shape, int32_t dtype);
int32_t qagnn_mp_core_forward_typed(const qagnn_shape *shape, int32_t dtype, const void *prep, const void *qkm, const void *ke,
                                    const void *me, void *aggr, float *alpha_scaled, float *alpha_out, float *scratch,
                                    void *stream);
int32_t qagnn_mp_core_backward_typed(const qagnn_shape *shape, int32_t dtype, const void *prep, const int32_t *combo_order,
                                     const void *qkm, const void *ke, const void *me, const float *alpha_scaled,
                                     const void *d_aggr, void *d_qkm, void *d_ke, void *d_me, float *scratch, void *stream);

/* qagnn_mp_core_backward_typed with d_ke / d_me summed without atomics, so that every output is the same, bit for bit, on every
 * run and for every grid size: what training under torch.use_deterministic_algorithms(True) calls.  d_qkm is the same as
 * qagnn_mp_core_backward_typed's, bit for bit.  combo_count int64 [C] and combo_order int32 [E+N] are qagnn_combo_sort's
 * outputs for this prep.  Summation order of row c of d_ke / d_me (fp32 sums; a 16-bit call rounds each row once at the end):
 * the positions [o, o + n) of combo c in combo_order (o = combo_count[0] + ... + combo_count[c-1], n = combo_count[c]) are
 * cut into runs of 64 positions [64r, 64r + 64); each run's part is summed in combo order; a combo inside one run is that
 * sum, and one spanning runs r0 < r1 is (P_0 + P_1) + ... + P_7 with P_k = the parts of runs r0 + k, r0 + k + 8, ... added
 * in ascending order.  A combo without positions gets exact zeros.  E' = rowptr_src[N] is read on the device, so a prep at
 * an edge capacity works without a host synchronisation, and the call can be captured into a CUDA graph.  `scratch` holds
 * qagnn_mp_core_backward_det_scratch_bytes(shape, dtype) bytes (0 for an invalid shape or dtype), else
 * QAGNN_ERR_WORKSPACE. */
size_t qagnn_mp_core_backward_det_scratch_bytes(const qagnn_shape *shape, int32_t dtype);
int32_t qagnn_mp_core_backward_det(const qagnn_shape *shape, int32_t dtype, const void *prep, const int32_t *combo_order,
                                   const int64_t *combo_count, const void *qkm, const void *ke, const void *me,
                                   const float *alpha_scaled, const void *d_aggr, void *d_qkm, void *d_ke, void *d_me,
                                   float *scratch, size_t scratch_bytes, void *stream);

/* What the training path needs per batch besides the prep, without a host synchronisation: a stable counting sort of the
 * by-source positions [0, E') by qagnn_prep_layout.csr_src_combo, with E' = rowptr_src[N] read on the device (shape->N and
 * shape->E are those the prep was built with; E may be an edge capacity, see qagnn_graph_prep_packed).
 *   combo_count_out int64 [C]    number of positions per combo (self loops included), C = R*T*T + T;
 *   combo_order_out int32 [E+N]  the combo_order of qagnn_mp_core_backward in its first E' entries; the rest is not written.
 * Positions with equal combo keep ascending order, so both arrays are unique and the same on every run.  `scratch` is
 * qagnn_combo_sort_bytes(shape) bytes; that query returns 0 for an invalid shape or C > 6144 (QAGNN_ERR_UNSUPPORTED). */
size_t qagnn_combo_sort_bytes(const qagnn_shape *shape);
int32_t qagnn_combo_sort(const qagnn_shape *shape, const void *prep, int64_t *combo_count_out, int32_t *combo_order_out,
                         void *scratch, size_t scratch_bytes, void *stream);

/* A stand-alone dense layer on the same tensor-core path the forward uses (diagnostics / tests):
 *   C[M,N] (ldc) = act( [A1 | A2] @ W^T + bias ),  fp32 row-major operands, W [N, K1+K2] (ldw), act 0/1/2 = none/ReLU/GELU(tanh).
 * Splits the operands into bf16 hi/lo planes in `workspace` and runs the wgmma 3-pass GEMM; returns
 * QAGNN_ERR_UNSUPPORTED when the tensor-core path cannot take the shape (K or ld not multiples of 8). */
size_t qagnn_linear_workspace_bytes(int64_t M, int32_t N, int32_t K1, int32_t K2);
int32_t qagnn_linear_bf16x3(const float *A1, int32_t lda1, int32_t K1, const float *A2, int32_t lda2, int32_t K2,
                            const float *W, int32_t ldw, const float *bias, float *C, int32_t ldc, int64_t M, int32_t N,
                            int32_t act, void *workspace, size_t workspace_bytes, void *stream);
/* The single-pass GEMM of the bf16 forward on its own: bf16 A1 / A2 / W (row strides lda1 / lda2 / ldw, multiples of 8,
 * 16-byte aligned bases), fp32 bias, one wgmma per k16 step with fp32 accumulation.  Writes C (fp32, ldc) and/or C_bf16
 * (the fp32 value rounded to nearest even, ldp); either may be NULL but not both. */
int32_t qagnn_linear_bf16(const void *A1, int32_t lda1, int32_t K1, const void *A2, int32_t lda2, int32_t K2, const void *W,
                          int32_t ldw, const float *bias, float *C, int32_t ldc, void *C_bf16, int32_t ldp, int64_t M, int32_t N,
                          int32_t act, void *stream);

/* The step after the path (SURVEY.md §8f #2): QAGNN's masked multi-head attention pooling of the node representations,
 * MultiheadAttPoolLayer.forward (utils/layers.py:344-371, called at modeling_qagnn.py:180), eval mode, fused into one
 * kernel that reads X [B, n, D] once.  qs [B, D] = w_qs(sent_vecs) (computed by the caller), mask uint8 [B, n]
 * (1 = masked out), wk/wv [D, D] and bk/bv [D] = w_ks / w_vs weights; outputs pooled [B, D], attn [n_head*B, n]. */
int32_t qagnn_attention_pool(int32_t B, int32_t n, int32_t D, int32_t n_head, const float *X, const float *qs,
                             const uint8_t *mask, const float *wk, const float *bk, const float *wv, const float *bv,
                             float *pooled, float *attn, void *stream);

/* The same pooling with the rest of QAGNN.forward's tail (modeling_qagnn.py:172-187) in the kernel: the pool mask is derived
 * from adj_lengths [B] and node_type [B,n] ((i >= len) | (type == 3), node 0 kept if everything is masked) and the row of
 * cat(graph_vecs, sent_vecs, Z) is written in place into concat [B, 2D+S] (Z = X[b,0,:], sent_vecs [B,S]).  The caller
 * all-gathers `concat` (multi-GPU) and applies the answer MLP. */
int32_t qagnn_decoder_tail(int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S, const float *X, const float *qs,
                           const int64_t *node_type, const int64_t *adj_lengths, const float *sent_vecs, const float *wk,
                           const float *bk, const float *wv, const float *bv, float *concat, float *attn, void *stream);

/* qagnn_attention_pool / qagnn_decoder_tail with X stored as `x_dtype` (QAGNN_DTYPE_F32 or QAGNN_DTYPE_BF16: the bf16 eval
 * forward's output, widened exactly); every other operand and output as above. */
int32_t qagnn_attention_pool_typed(int32_t x_dtype, int32_t B, int32_t n, int32_t D, int32_t n_head, const void *X,
                                   const float *qs, const uint8_t *mask, const float *wk, const float *bk, const float *wv,
                                   const float *bv, float *pooled, float *attn, void *stream);
int32_t qagnn_decoder_tail_typed(int32_t x_dtype, int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S, const void *X,
                                 const float *qs, const int64_t *node_type, const int64_t *adj_lengths, const float *sent_vecs,
                                 const float *wk, const float *bk, const float *wv, const float *bv, float *concat, float *attn,
                                 void *stream);

/* The step before the path (SURVEY.md §8f #2): QAGNN.forward's input assembly (modeling_qagnn.py:153-167), eval mode, one kernel:
 *   H_out[b,0,:] = ctx[b,:] (= GELU(svec2nvec(sent_vecs)), caller-computed [B,D]);  H_out[b,i,:] = table[concept_ids[b,i]-1], i >= 1,
 *   with `table` [n_concept, D] the concept embedding after cpt_transform + GELU (folded once by the caller; the table is
 *   frozen in eval);  scores_out [B,n] = the reference's relevance-score normalisation of node_scores [B,n] by adj_lengths. */
int32_t qagnn_decoder_head(int32_t B, int32_t n, int32_t D, const int64_t *concept_ids, int64_t n_concept, const float *table,
                           const float *ctx, const float *node_scores, const int64_t *adj_lengths, float *H_out,
                           float *scores_out, void *stream);

/* The decoder head and tail on a ragged batch of B graphs over N_rows packed rows, graph b's rows from node_ptr[b] (device int64
 * [B + 1], the exclusive cumsum of adj_lengths).  The head reads the padded [B, n] concept_ids / node_scores / node_type as above
 * and writes positions i < adj_lengths[b] as rows node_ptr[b] + i of H_out [N_rows, D], scores_out [N_rows] and type_out int64
 * [N_rows], with the values qagnn_decoder_head writes at [b, i]; the tail rows [node_ptr[B], N_rows) get zeros, score 0 and
 * type 2.  The tail pools graph b over its own rows of X [N_rows, D] (x_dtype as in qagnn_decoder_tail_typed), with node_type
 * the packed [N_rows] type_out of the head, and writes attn [n_head*B, n] in the padded layout, exact zeros at positions
 * >= adj_lengths[b]. */
int32_t qagnn_decoder_head_ragged(int32_t B, int32_t n, int32_t D, int64_t N_rows, const int64_t *concept_ids, int64_t n_concept,
                                  const float *table, const float *ctx, const float *node_scores, const int64_t *adj_lengths,
                                  const int64_t *node_type, const int64_t *node_ptr, float *H_out, float *scores_out,
                                  int64_t *type_out, void *stream);
int32_t qagnn_decoder_tail_ragged(int32_t x_dtype, int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S, int64_t N_rows,
                                  const void *X, const int64_t *node_ptr, const float *qs, const int64_t *node_type,
                                  const int64_t *adj_lengths, const float *sent_vecs, const float *wk, const float *bk,
                                  const float *wv, const float *bv, float *concat, float *attn, void *stream);

/* Gradient of qagnn_decoder_tail_ragged, for autograd through the ragged decoder tail.  Given d_concat [B, 2D+S] (fp32) and the
 * forward's X, qs, attn and weights (node_ptr, adj_lengths as in the forward) it writes d_qs [B, D] (the gradient reaching
 * w_qs(sent_vecs)), dX [N_rows, D] fp32 (zero on the tail rows and on every row the forward did not pool over; row 0 of each
 * graph also receives d(Z)), and d_wk / d_wv [D, D], d_bk / d_bv [D], summed over the B graphs.  The d(sent_vecs) columns of
 * d_concat are the caller's to pass on.  Every sum runs in a fixed order without atomics: two calls give the same bits.
 * `scratch` holds qagnn_attention_pool_backward_ragged_scratch_bytes(B, n, D, n_head) bytes (0 for an invalid shape). */
size_t qagnn_attention_pool_backward_ragged_scratch_bytes(int32_t B, int32_t n, int32_t D, int32_t n_head);
int32_t qagnn_attention_pool_backward_ragged(int32_t x_dtype, int32_t B, int32_t n, int32_t D, int32_t n_head, int32_t S,
                                             int64_t N_rows, const void *X, const int64_t *node_ptr, const int64_t *adj_lengths,
                                             const float *qs, const float *wk, const float *bk, const float *wv, const float *attn,
                                             const float *d_concat, float *dX, float *d_qs, float *d_wk, float *d_bk, float *d_wv,
                                             float *d_bv, float *scratch, size_t scratch_bytes, void *stream);

/* Batch assembly from a split held on the device (qagnn_b200.data.DeviceSplit): the packed adjacency of the B = bs * num_choice
 * sub-graphs of the questions question_ids (device int64 [bs]), equal to FlatAdjCache.pack of the same ids bit for bit.  The split
 * is the FlatAdjCache layout of G sub-graphs: local ids src / tgt int32 [E_split], etype int16 [E_split], graph_ptr int64 [G + 1]
 * and, for a ragged batch, adj_lengths int64 [G]; graph g is choice g % num_choice of question g / num_choice.  Outputs:
 *   edges int64 [3, K]: row 0 src + base, row 1 tgt + base, row 2 etype; columns [graph_ptr_out[B], K) are zero;
 *   graph_ptr_out int64 [B + 1]: the first edge of every graph;
 *   node_ptr_out int64 [B + 1] (N_cap >= 0 only): the exclusive cumsum of the graphs' adj_lengths;
 * with base = b * n_nodes for a padded batch (N_cap = -1) and node_ptr_out[b] for a ragged one.  No host synchronisation and no
 * atomics.  The caller checks the ids and capacities first; the kernels clamp ids to [0, G / num_choice), graph_ptr_out to K and
 * node_ptr_out to N_cap, so a bad id or count never writes past K, N_cap or B + 1 entries.  Two launches (one when K = 0). */
int32_t qagnn_assemble_batch(const int32_t *src, const int32_t *tgt, const int16_t *etype, const int64_t *graph_ptr,
                             const int64_t *adj_lengths, int64_t G, int32_t num_choice, int32_t n_nodes,
                             const int64_t *question_ids, int32_t bs, int64_t K, int64_t N_cap, int64_t *edges,
                             int64_t *graph_ptr_out, int64_t *node_ptr_out, void *stream);

/* One step of the reference's RAdam (utils/optimization_utils.py) over n_tensors fp32 tensors of the current device, in one
 * launch per 512 tensors or 16 distinct groups (qagnn_b200.optim.RAdam).  Tensor i: contiguous params[i], grads[i], exp_avgs[i],
 * exp_avg_sqs[i] of numels[i] elements, its int64 device step counter steps[i], and its group group_index[i] < n_groups.  The
 * per-group host arrays lr, weight_decay, beta1, beta2, eps and degenerated_to_sgd hold the Python values; each scalar the
 * update uses is rounded to fp32 as torch rounds it.  step_tables[g] is a device fp64 [table_len, 2] table of (1.0 when
 * rho_t >= 5 else 0.0, step size) for t = row, built with the reference's formula for the group's betas; the device step after
 * the increment indexes it, so table_len must exceed every step counter.  found_inf (optional, device fp32): nonzero leaves
 * every tensor and step as it is.  grad_scale (optional, device fp32): the gradients are first multiplied by
 * (float)(1.0 / (double)*grad_scale), as GradScaler.unscale_ does, and written back.  counter: a device int32 that is zero
 * between calls (the kernel resets it).  Every element is the eager torch op sequence's result bit for bit; no host
 * synchronisation. */
int32_t qagnn_radam_step(int32_t n_tensors, void *const *params, void *const *grads, void *const *exp_avgs,
                         void *const *exp_avg_sqs, void *const *steps, const int64_t *numels, const int32_t *group_index,
                         int32_t n_groups, const double *lr, const double *weight_decay, const double *beta1,
                         const double *beta2, const double *eps, const int32_t *degenerated_to_sgd,
                         void *const *step_tables, int64_t table_len, const float *found_inf, const float *grad_scale,
                         int32_t *counter, void *stream);

/* Launch counters since load (kernels this library enqueued); for bench.py's gpu_launches. */
int64_t qagnn_launch_count(void);

/* Optional device-side stage timing (diagnostics for bench.py's roofline; single-threaded use).
 * While enabled, every forward brackets its stages with cudaEvents on the launching stream.
 * qagnn_profile_read synchronises those events and returns, per stage, the summed milliseconds and
 * the number of timed intervals since the last enable.  Stages: */
enum {
  QAGNN_PROF_GRAPH_PREP = 0,   /* qagnn_graph_prep                                   */
  QAGNN_PROF_PROJECTION = 1,   /* [x|extra] @ Wp^T  (Q|Kx|Mx)                         */
  QAGNN_PROF_MESSAGE_PASSING = 2, /* logits + per-source softmax + rescale + per-target sum */
  QAGNN_PROF_NODE_MLP = 3,     /* mlp.0 + BN + ReLU + mlp.3 (+GELU)                    */
  QAGNN_PROF_PRO_EPILOGUE = 4, /* node_feature_extra and Vh/Vx                         */
  QAGNN_PROF_STAGES = 5
};
int32_t qagnn_profile_enable(int32_t on);
int32_t qagnn_profile_read(double *ms_out /* [QAGNN_PROF_STAGES] */, int64_t *count_out /* [QAGNN_PROF_STAGES] */);

#ifdef __cplusplus
}
#endif
#endif /* QAGNN_B200_H_ */
