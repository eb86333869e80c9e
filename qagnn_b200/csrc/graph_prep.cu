// Graph prep: the layer-invariant index work of GATConvE (modeling/modeling_qagnn.py:419-438,
// 476-479), done once per forward and reused by all k layers.
//
//   edge_index' = [edge_index | self loops]                                   (:436-438)
//   combo[e]    = (etype*T + type[src])*T + type[tgt] for real edges, R*T*T + type[v] for the self loop of
//                 v — an index of the distinct values the reference's [E', R+1+2T] one-hot edge feature can
//                 take (:419-432); C = R*T*T + T rows in the folded edge tables
//   out-degree by source (self loop included)                                  (:476-479)
//   stable CSR orders by source (softmax groups, :472) and by target (aggregation, :442)
//
// Everything is deterministic: the atomics only count, segment order is restored by an in-segment
// sort on the edge id, so the downstream floating-point sums are run-to-run reproducible.
#include "common.cuh"

namespace qagnn {

namespace {

struct PrepScratch {
  size_t cnt_src, cnt_tgt;  // [N] each (also reused as fill cursors after the scan)
  size_t bsum;              // [2 * nb]
  size_t tmp_src, tmp_tgt;  // [E'] unsorted CSR fill
  size_t inv_src;           // [E'] edge id -> position in the by-source order
  size_t inv_tgt;           // [E'] edge id -> position in the by-target order
  size_t big_list;          // [2N] work list of (node, direction) segments with more than 32 edges
  size_t total;             // int32 words
};

constexpr int kScanChunk = 1024;

inline int64_t scan_blocks(int64_t N) { return (N + kScanChunk - 1) / kScanChunk; }

PrepScratch make_scratch(int64_t N, int64_t E) {
  const size_t Ep = (size_t)(N + E);
  PrepScratch s;
  size_t o = 0;
  auto take = [&](size_t n) { size_t r = o; o += align_up(n * 4) / 4; return r; };
  s.cnt_src = take(N);
  s.cnt_tgt = take(N);
  s.bsum = take(2 * (size_t)scan_blocks(N) + 2);
  s.tmp_src = take(Ep);
  s.tmp_tgt = take(Ep);
  s.inv_src = take(Ep);
  s.inv_tgt = take(Ep);
  s.big_list = take(2 * (size_t)N);
  s.total = o;
  return s;
}

__global__ void prep_edges_kernel(const int64_t* __restrict__ edge_index, const int64_t* __restrict__ edge_type,
                                  const int64_t* __restrict__ node_type, int64_t N, int64_t E, int T, int R, int npg,
                                  int32_t* __restrict__ src_o, int32_t* __restrict__ tgt_o,
                                  int32_t* __restrict__ combo_o, int32_t* __restrict__ cnt_src,
                                  int32_t* __restrict__ cnt_tgt, int32_t* __restrict__ status) {
  const int64_t Ep = E + N;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < Ep; e += (int64_t)gridDim.x * blockDim.x) {
    int64_t s, t, r;
    int bad = 0;
    if (e < E) {
      s = edge_index[e];
      t = edge_index[E + e];
      r = edge_type[e];
      if (s < 0 || s >= N || t < 0 || t >= N) { bad |= 1; s = min(max(s, (int64_t)0), N - 1); t = min(max(t, (int64_t)0), N - 1); }
      if (r < 0 || r >= R) { bad |= 2; r = min(max(r, (int64_t)0), (int64_t)R - 1); }
      if (npg > 0 && s / npg != t / npg) bad |= 8;  // edge crosses a sub-graph boundary
    } else {
      s = t = e - E;  // self loop, own type index R (:420-421)
      r = R;
    }
    int64_t ts = node_type[s], tt = node_type[t];
    if (ts < 0 || ts >= T) { bad |= 4; ts = min(max(ts, (int64_t)0), (int64_t)T - 1); }
    if (tt < 0 || tt >= T) { bad |= 4; tt = min(max(tt, (int64_t)0), (int64_t)T - 1); }
    if (bad) atomicOr(status, bad);
    src_o[e] = (int32_t)s;
    tgt_o[e] = (int32_t)t;
    combo_o[e] = (e < E) ? (int32_t)((r * T + ts) * T + tt) : (int32_t)((int64_t)R * T * T + ts);
    atomicAdd(cnt_src + s, 1);
    atomicAdd(cnt_tgt + t, 1);
  }
}

// ---- 3-phase exclusive scan of two length-N count arrays (blockIdx.y selects the array) ----
__global__ void __launch_bounds__(kScanChunk) scan_block_sums_kernel(const int32_t* __restrict__ cnt_a,
                                                                       const int32_t* __restrict__ cnt_b, int64_t N,
                                                                       int32_t* __restrict__ bsum, int nb) {
  const int32_t* cnt = blockIdx.y ? cnt_b : cnt_a;
  const int64_t i = (int64_t)blockIdx.x * kScanChunk + threadIdx.x;
  int v = i < N ? cnt[i] : 0;
  int total;
  block_exclusive_scan_1024(v, &total);
  if (threadIdx.x == 0) bsum[blockIdx.y * nb + blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanChunk) scan_sums_kernel(int32_t* __restrict__ bsum, int nb) {
  int32_t* b = bsum + blockIdx.y * nb;
  int carry = 0;
  for (int base = 0; base < nb; base += kScanChunk) {
    const int i = base + threadIdx.x;
    int v = i < nb ? b[i] : 0;
    int total;
    int ex = block_exclusive_scan_1024(v, &total);
    if (i < nb) b[i] = carry + ex;
    carry += total;
  }
}

__global__ void __launch_bounds__(kScanChunk) scan_apply_kernel(int32_t* __restrict__ cnt_a, int32_t* __restrict__ cnt_b,
                                                                  int64_t N, const int32_t* __restrict__ bsum, int nb,
                                                                  int32_t* __restrict__ rowptr_a,
                                                                  int32_t* __restrict__ rowptr_b) {
  int32_t* cnt = blockIdx.y ? cnt_b : cnt_a;
  int32_t* rowptr = blockIdx.y ? rowptr_b : rowptr_a;
  const int64_t i = (int64_t)blockIdx.x * kScanChunk + threadIdx.x;
  int v = i < N ? cnt[i] : 0;
  int total;
  int ex = block_exclusive_scan_1024(v, &total) + bsum[blockIdx.y * nb + blockIdx.x];
  if (i < N) {
    rowptr[i] = ex;
    cnt[i] = 0;  // becomes the fill cursor
    if (i == N - 1) rowptr[N] = ex + v;
  }
}

__global__ void prep_fill_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ tgt, int64_t Ep,
                                 const int32_t* __restrict__ rowptr_src, const int32_t* __restrict__ rowptr_tgt,
                                 int32_t* __restrict__ cur_src, int32_t* __restrict__ cur_tgt,
                                 int32_t* __restrict__ tmp_src, int32_t* __restrict__ tmp_tgt) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < Ep; e += (int64_t)gridDim.x * blockDim.x) {
    const int s = src[e], t = tgt[e];
    tmp_src[rowptr_src[s] + atomicAdd(cur_src + s, 1)] = (int32_t)e;
    tmp_tgt[rowptr_tgt[t] + atomicAdd(cur_tgt + t, 1)] = (int32_t)e;
  }
}

// One warp per (node, order): restore ascending edge-id order inside the segment (== stable sort).  Segments with more
// than 32 edges (hub nodes) go to a work list that prep_sort_big_segments_kernel sorts one CTA per segment.
__global__ void prep_sort_segments_kernel(int64_t N, const int32_t* __restrict__ rowptr_src,
                                          const int32_t* __restrict__ rowptr_tgt, const int32_t* __restrict__ tmp_src,
                                          const int32_t* __restrict__ tmp_tgt, int32_t* __restrict__ perm_src,
                                          int32_t* __restrict__ perm_tgt, int32_t* __restrict__ big_list,
                                          int32_t* __restrict__ big_count) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = warp; w < 2 * N; w += nwarps) {
    const bool by_tgt = w >= N;
    const int64_t v = by_tgt ? w - N : w;
    const int32_t* rowptr = by_tgt ? rowptr_tgt : rowptr_src;
    const int32_t* tmp = by_tgt ? tmp_tgt : tmp_src;
    int32_t* perm = by_tgt ? perm_tgt : perm_src;
    const int beg = rowptr[v], deg = rowptr[v + 1] - beg;
    if (deg <= 32) {
      const int id = lane < deg ? tmp[beg + lane] : 0x7fffffff;
      int rank = 0;
      for (int j = 0; j < deg; ++j) rank += (__shfl_sync(0xffffffffu, id, j) < id);
      if (lane < deg) perm[beg + rank] = id;
    } else if (lane == 0) {
      big_list[atomicAdd(big_count, 1)] = (int32_t)w;  // w < 2N < 2^31; the list order does not matter (the result is a sort)
    }
  }
}

// Hub segments: one CTA per segment.  Up to kBigSort edge ids are sorted in shared memory by a bitonic network
// (O(deg log^2 deg / 512) steps); longer segments fall back to rank counting against shared-memory tiles (O(deg^2 / 512)).
constexpr int kBigSort = 8192, kBigThreads = 512;
__global__ void __launch_bounds__(kBigThreads) prep_sort_big_segments_kernel(int64_t N, const int32_t* __restrict__ rowptr_src,
                                                                             const int32_t* __restrict__ rowptr_tgt,
                                                                             const int32_t* __restrict__ tmp_src,
                                                                             const int32_t* __restrict__ tmp_tgt,
                                                                             int32_t* __restrict__ perm_src, int32_t* __restrict__ perm_tgt,
                                                                             const int32_t* __restrict__ big_list,
                                                                             const int32_t* __restrict__ big_count) {
  __shared__ int32_t buf[kBigSort];
  const int count = *big_count;
  for (int item = blockIdx.x; item < count; item += gridDim.x) {
    const int64_t w = big_list[item];
    const bool by_tgt = w >= N;
    const int64_t v = by_tgt ? w - N : w;
    const int32_t* rowptr = by_tgt ? rowptr_tgt : rowptr_src;
    const int32_t* tmp = (by_tgt ? tmp_tgt : tmp_src);
    int32_t* perm = by_tgt ? perm_tgt : perm_src;
    const int beg = rowptr[v], deg = rowptr[v + 1] - beg;
    if (deg <= kBigSort) {
      int n2 = 64;
      while (n2 < deg) n2 <<= 1;
      for (int i = threadIdx.x; i < n2; i += kBigThreads) buf[i] = i < deg ? tmp[beg + i] : 0x7fffffff;
      __syncthreads();
      for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
          for (int i = threadIdx.x; i < n2; i += kBigThreads) {
            const int ixj = i ^ j;
            if (ixj > i) {
              const int32_t a = buf[i], b = buf[ixj];
              const bool up = (i & k) == 0;
              if ((a > b) == up) { buf[i] = b; buf[ixj] = a; }
            }
          }
          __syncthreads();
        }
      }
      for (int i = threadIdx.x; i < deg; i += kBigThreads) perm[beg + i] = buf[i];
      __syncthreads();
    } else {
      for (int i0 = 0; i0 < deg; i0 += kBigThreads) {  // every thread ranks one id per round against all tiles
        const int i = i0 + threadIdx.x;
        const int32_t id = i < deg ? tmp[beg + i] : 0x7fffffff;
        int rank = 0;
        for (int t0 = 0; t0 < deg; t0 += kBigSort) {
          const int tn = min(kBigSort, deg - t0);
          __syncthreads();
          for (int j = threadIdx.x; j < tn; j += kBigThreads) buf[j] = tmp[beg + t0 + j];
          __syncthreads();
          for (int j = 0; j < tn; ++j) rank += (buf[j] < id);
        }
        if (i < deg) perm[beg + rank] = id;
      }
      __syncthreads();
    }
  }
}

__global__ void prep_payload_src_kernel(int64_t Ep, const int32_t* __restrict__ perm_src,
                                        const int32_t* __restrict__ tgt, const int32_t* __restrict__ combo,
                                        int32_t* __restrict__ csr_src_tgt, int32_t* __restrict__ csr_src_combo,
                                        int32_t* __restrict__ inv_src, const int32_t* __restrict__ src, int npg,
                                        int32_t* __restrict__ pk_src) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < Ep; p += (int64_t)gridDim.x * blockDim.x) {
    const int e = perm_src[p];
    const int t = tgt[e], c = combo[e];
    csr_src_tgt[p] = t;
    csr_src_combo[p] = c;
    inv_src[e] = (int32_t)p;
    if (npg > 0) {  // local target id | combo, for the shared-memory-tiled kernels
      int tl = t - (src[e] / npg) * npg;
      tl = min(max(tl, 0), npg - 1);
      pk_src[p] = (int32_t)(((uint32_t)tl << 16) | ((uint32_t)c & 0xffffu));
    }
  }
}

__global__ void prep_payload_tgt_kernel(int64_t Ep, const int32_t* __restrict__ perm_tgt,
                                        const int32_t* __restrict__ src, const int32_t* __restrict__ combo,
                                        const int32_t* __restrict__ inv_src, int32_t* __restrict__ csr_tgt_src,
                                        int32_t* __restrict__ csr_tgt_combo, int32_t* __restrict__ csr_tgt_apos,
                                        const int32_t* __restrict__ tgt, int npg, int32_t* __restrict__ pk_tgt,
                                        int32_t* __restrict__ inv_tgt) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < Ep; p += (int64_t)gridDim.x * blockDim.x) {
    const int e = perm_tgt[p];
    const int s = src[e], c = combo[e];
    inv_tgt[e] = (int32_t)p;
    csr_tgt_src[p] = s;
    csr_tgt_combo[p] = c;
    csr_tgt_apos[p] = inv_src[e];
    if (npg > 0) {
      int sl = s - (tgt[e] / npg) * npg;
      sl = min(max(sl, 0), npg - 1);
      pk_tgt[p] = (int32_t)(((uint32_t)sl << 16) | ((uint32_t)c & 0xffffu));
    }
  }
}

__global__ void prep_tpos_kernel(int64_t Ep, const int32_t* __restrict__ perm_src, const int32_t* __restrict__ inv_tgt,
                                 int32_t* __restrict__ csr_src_tpos) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < Ep; p += (int64_t)gridDim.x * blockDim.x)
    csr_src_tpos[p] = inv_tgt[perm_src[p]];
}

// Per sub-graph (one CTA each, blockIdx.y = direction): local node ids ordered by degree, descending, so that the
// 4 nodes a warp of the tiled kernel walks together have (nearly) the same number of edges.  Ties are broken by a
// shared-memory atomic counter: the order only schedules work, it never changes a summation order.
__global__ void __launch_bounds__(256) prep_degree_order_kernel(int npg, const int32_t* __restrict__ rowptr_src,
                                                                const int32_t* __restrict__ rowptr_tgt,
                                                                int32_t* __restrict__ order_src, int32_t* __restrict__ order_tgt,
                                                                uint2* __restrict__ ninfo_src, uint2* __restrict__ ninfo_tgt) {
  __shared__ int hist[256], base[256];
  const int32_t* rowptr = blockIdx.y ? rowptr_tgt : rowptr_src;
  int32_t* order = (blockIdx.y ? order_tgt : order_src) + (size_t)blockIdx.x * npg;
  uint2* ninfo = (blockIdx.y ? ninfo_tgt : ninfo_src) + (size_t)blockIdx.x * npg;
  const int64_t v0 = (int64_t)blockIdx.x * npg;
  hist[threadIdx.x] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < npg; i += 256) atomicAdd(&hist[min(rowptr[v0 + i + 1] - rowptr[v0 + i], 255)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int b = 255; b >= 0; --b) { base[b] = run; run += hist[b]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < npg; i += 256) {
    const int beg = rowptr[v0 + i], deg = rowptr[v0 + i + 1] - beg;
    const int b = min(deg, 255);
    const int slot = atomicAdd(&base[b], 1);
    order[slot] = i;
    // what a warp of the tiled kernel needs to start on this node, in one 8-byte load: local id | degree, CSR begin
    ninfo[slot] = make_uint2((uint32_t)i | ((uint32_t)min(deg, 0xffff) << 16), (uint32_t)beg);
  }
}

// ---- packed batches: one CTA builds the whole prep of ONE sub-graph in shared memory ------------------------------------
// When the caller knows where each sub-graph's edges start (graph_ptr: the batch generator / pack_adj / batch_graph lay
// the edges out graph by graph), everything above — count, scan, fill, in-segment sort, payloads, degree order — is local
// to a sub-graph: ~1200 edges and 200 nodes at cfg2.  One launch instead of twelve; the result is bit-identical to the
// general pipeline (tests/test_gpu_parity.py) because every array is a function of the stable edge-id order only.
// Local edge index i: real edges i < e_g (edge id gp[g] + i), then the self loop of local node i - e_g (edge id E + g*n + ...).
// E may be an edge capacity larger than the batch (see qagnn_graph_prep_packed in include/qagnn_b200.h): every CSR-ordered
// array then ends at E' = graph_ptr[G] + N, and the positions a sub-graph writes do not depend on E at all.
struct PackedPrepArgs {
  const int64_t *edge_index, *edge_type, *node_type, *graph_ptr;
  const int64_t* node_ptr;  // ragged batches: first row of every sub-graph, [B + 1]
  int64_t N, E;
  int T, R, npg, cap, B;    // B: sub-graphs of a ragged batch (the grid adds the tail segments)
  int32_t *src, *tgt, *combo, *rowptr_src, *rowptr_tgt, *perm_src, *perm_tgt, *csr_src_tgt, *csr_src_combo, *csr_tgt_src,
      *csr_tgt_combo, *csr_tgt_apos, *pk_src, *pk_tgt, *csr_src_tpos, *order_src, *order_tgt, *status;
  uint2 *ninfo_src, *ninfo_tgt;
};

constexpr int kPackedThreads = 256;
constexpr int kNodePtrBit = 32;  // status bit: node_ptr not monotone, a sub-graph over n rows, or node_ptr[B] past N

// RAGGED: sub-graph g owns rows [node_ptr[g], node_ptr[g+1]) (at most npg of them) instead of [g*npg, (g+1)*npg); CTAs
// g >= B build the tail segments (rows past node_ptr[B]: self loops only, see ragged_segment in common.cuh).
template <bool RAGGED>
__global__ void __launch_bounds__(kPackedThreads) prep_packed_graph_kernel(const PackedPrepArgs a) {
  extern __shared__ int32_t sm_pp[];
  const int n = a.npg, cap = a.cap, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = kPackedThreads / 32;
  int32_t* ntype = sm_pp;             // [n]
  int32_t* cnt_s = ntype + n;         // [n + 1]  counts, then exclusive local row pointers
  int32_t* cnt_t = cnt_s + n + 1;     // [n + 1]
  int32_t* cur_s = cnt_t + n + 1;     // [n]      fill cursors, later histogram scratch
  int32_t* cur_t = cur_s + n;         // [n]
  int32_t* lsrc = cur_t + n;          // [cap]    local source of local edge i
  int32_t* ltgt = lsrc + cap;         // [cap]
  int32_t* lcombo = ltgt + cap;       // [cap]
  int32_t* tmp_s = lcombo + cap;      // [cap]    unsorted CSR fill (local edge indices)
  int32_t* tmp_t = tmp_s + cap;       // [cap]
  int32_t* perm_s = tmp_t + cap;      // [cap]    sorted
  int32_t* perm_t = perm_s + cap;     // [cap]
  int32_t* inv_s = perm_t + cap;      // [cap]    local edge -> position
  int32_t* inv_t = inv_s + cap;       // [cap]
  __shared__ int hist[256], hbase[256];

  const int64_t g = blockIdx.x, G = gridDim.x;
  const int64_t Bg = RAGGED ? a.B : G;  // sub-graphs with edges
  // a.E is the edge CAPACITY of edge_index / edge_type; the batch's edges are the first graph_ptr[B] columns (clamped: a
  // graph_ptr past the capacity sets bit 16 in the CTA of the last sub-graph below).  The ids of the unused columns keep
  // src / tgt / combo = -1; the self loops stay at ids E + v, behind every real edge.
  const int64_t e_real = min(max(a.graph_ptr[Bg], (int64_t)0), a.E);
  if (g == (RAGGED ? 0 : G - 1) && tid == 0) {
    a.rowptr_src[a.N] = (int32_t)(e_real + a.N); a.rowptr_tgt[a.N] = (int32_t)(e_real + a.N);
  }
  for (int64_t e = e_real + g * kPackedThreads + tid; e < a.E; e += G * kPackedThreads) {
    a.src[e] = -1; a.tgt[e] = -1; a.combo[e] = -1;
  }
  int64_t v0 = g * n, e0, e1;
  int ng = n;  // rows of this sub-graph
  if (RAGGED) {
    ragged_segment(a.node_ptr, a.B, n, a.N, g, v0, ng);
    if (g < Bg) {
      e0 = a.graph_ptr[g]; e1 = a.graph_ptr[g + 1];
      const int64_t r0 = a.node_ptr[g], r1 = a.node_ptr[g + 1];
      const bool bad_ptr = (g == 0 && r0 != 0) || r1 < r0 || r1 - r0 > n || (g == Bg - 1 && r1 > a.N) || (ng == 0 && e1 > e0);
      if (bad_ptr) {  // nothing of this sub-graph is touched
        if (tid == 0) atomicOr(a.status, kNodePtrBit);
        return;
      }
    } else {
      if (ng == 0) return;  // past the tail
      e0 = e1 = e_real;
    }
  } else {
    e0 = a.graph_ptr[g]; e1 = a.graph_ptr[g + 1];
  }
  const int eg = (int)(e1 - e0), ep = eg + ng;  // real edges, edges incl. self loops (ep <= cap, checked on the host)
  const int64_t base = e0 + v0;  // entries of the CSR orders that belong to earlier sub-graphs
  if (e0 < 0 || e1 < e0 || e1 > a.E || ep > cap) {  // graph_ptr disagrees with E / max_edges_per_graph: nothing is touched
    if (tid == 0) atomicOr(a.status, 16);
    return;
  }
  int bad = 0;
  for (int i = tid; i < ng; i += kPackedThreads) {
    int64_t t = a.node_type[v0 + i];
    if (t < 0 || t >= a.T) { bad |= 4; t = min(max(t, (int64_t)0), (int64_t)a.T - 1); }
    ntype[i] = (int32_t)t;
    cnt_s[i] = 0; cnt_t[i] = 0; cur_s[i] = 0; cur_t[i] = 0;
  }
  if (tid == 0) { cnt_s[ng] = 0; cnt_t[ng] = 0; }
  __syncthreads();
  // edges -> local ids, combo, counts; global src / tgt / combo in edge-id order
  for (int i = tid; i < ep; i += kPackedThreads) {
    int sl, tl, r;
    int64_t gid;
    if (i < eg) {
      gid = e0 + i;
      int64_t s = a.edge_index[gid], t = a.edge_index[a.E + gid], rr = a.edge_type[gid];
      if (s < 0 || s >= a.N || t < 0 || t >= a.N) { bad |= 1; s = min(max(s, (int64_t)0), a.N - 1); t = min(max(t, (int64_t)0), a.N - 1); }
      if (rr < 0 || rr >= a.R) { bad |= 2; rr = min(max(rr, (int64_t)0), (int64_t)a.R - 1); }
      if (RAGGED ? (s < v0 || s >= v0 + ng || t < v0 || t >= v0 + ng) : (s / n != g || t / n != g))
        bad |= 8;  // not an edge of this sub-graph
      sl = (int)min(max(s - v0, (int64_t)0), (int64_t)ng - 1);
      tl = (int)min(max(t - v0, (int64_t)0), (int64_t)ng - 1);
      r = (int)rr;
      a.src[gid] = (int32_t)s; a.tgt[gid] = (int32_t)t;
    } else {
      sl = tl = i - eg;
      r = a.R;
      gid = a.E + v0 + sl;
      a.src[gid] = (int32_t)(v0 + sl); a.tgt[gid] = (int32_t)(v0 + sl);
    }
    const int c = i < eg ? (r * a.T + ntype[sl]) * a.T + ntype[tl] : a.R * a.T * a.T + ntype[sl];
    a.combo[gid] = c;
    lsrc[i] = sl; ltgt[i] = tl; lcombo[i] = c;
    atomicAdd(&cnt_s[sl], 1);
    atomicAdd(&cnt_t[tl], 1);
  }
  if (bad) atomicOr(a.status, bad);
  __syncthreads();
  // exclusive scan of both count arrays (warp 0: by source, warp 1: by target), n <= 65535
  if (warp < 2) {
    int32_t* cnt = warp == 0 ? cnt_s : cnt_t;
    const int chunk = (ng + 31) / 32, b0 = lane * chunk, b1 = min(ng, b0 + chunk);
    int sum = 0;
    for (int i = b0; i < b1; ++i) sum += cnt[i];
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    int run = incl - sum;
    for (int i = b0; i < b1; ++i) { const int c = cnt[i]; cnt[i] = run; run += c; }
    if (lane == 31) cnt[ng] = incl;
  }
  __syncthreads();
  for (int i = tid; i < ng; i += kPackedThreads) {
    a.rowptr_src[v0 + i] = (int32_t)(base + cnt_s[i]);
    a.rowptr_tgt[v0 + i] = (int32_t)(base + cnt_t[i]);
  }
  // unordered fill, then ascending edge order inside every segment (== stable sort by node)
  for (int i = tid; i < ep; i += kPackedThreads) {
    tmp_s[cnt_s[lsrc[i]] + atomicAdd(&cur_s[lsrc[i]], 1)] = i;
    tmp_t[cnt_t[ltgt[i]] + atomicAdd(&cur_t[ltgt[i]], 1)] = i;
  }
  __syncthreads();
  for (int w = warp; w < 2 * ng; w += nwarps) {  // one warp per (node, direction); lanes over the segment's positions
    const bool by_t = w >= ng;
    const int v = by_t ? w - ng : w;
    const int32_t* cnt = by_t ? cnt_t : cnt_s;
    const int32_t* tmp = by_t ? tmp_t : tmp_s;
    int32_t* perm = by_t ? perm_t : perm_s;
    int32_t* inv = by_t ? inv_t : inv_s;
    const int b = cnt[v], deg = cnt[v + 1] - b;
    for (int q = lane; q < deg; q += 32) {
      const int id = tmp[b + q];
      int rank = 0;
      for (int j = 0; j < deg; ++j) rank += (tmp[b + j] < id);
      perm[b + rank] = id;
      inv[id] = b + rank;
    }
  }
  __syncthreads();
  // payloads in both orders
  for (int p = tid; p < ep; p += kPackedThreads) {
    {
      const int i = perm_s[p];
      const int64_t gid = i < eg ? e0 + i : a.E + v0 + (i - eg);
      const int tl = ltgt[i], c = lcombo[i];
      a.perm_src[base + p] = (int32_t)gid;
      a.csr_src_tgt[base + p] = (int32_t)(v0 + tl);
      a.csr_src_combo[base + p] = c;
      a.pk_src[base + p] = (int32_t)(((uint32_t)tl << 16) | ((uint32_t)c & 0xffffu));
      a.csr_src_tpos[base + p] = (int32_t)(base + inv_t[i]);
    }
    {
      const int i = perm_t[p];
      const int64_t gid = i < eg ? e0 + i : a.E + v0 + (i - eg);
      const int sl = lsrc[i], c = lcombo[i];
      a.perm_tgt[base + p] = (int32_t)gid;
      a.csr_tgt_src[base + p] = (int32_t)(v0 + sl);
      a.csr_tgt_combo[base + p] = c;
      a.csr_tgt_apos[base + p] = (int32_t)(base + inv_s[i]);
      a.pk_tgt[base + p] = (int32_t)(((uint32_t)sl << 16) | ((uint32_t)c & 0xffffu));
    }
  }
  // degree-sorted schedule of the tiled kernel, both directions (see prep_degree_order_kernel)
  for (int dir = 0; dir < 2; ++dir) {
    const int32_t* cnt = dir ? cnt_t : cnt_s;
    int32_t* order = (dir ? a.order_tgt : a.order_src) + v0;
    uint2* ninfo = (dir ? a.ninfo_tgt : a.ninfo_src) + v0;
    __syncthreads();
    hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < ng; i += kPackedThreads) atomicAdd(&hist[min(cnt[i + 1] - cnt[i], 255)], 1);
    __syncthreads();
    if (tid == 0) {
      int run = 0;
      for (int b = 255; b >= 0; --b) { hbase[b] = run; run += hist[b]; }
    }
    __syncthreads();
    for (int i = tid; i < ng; i += kPackedThreads) {
      const int deg = cnt[i + 1] - cnt[i];
      const int slot = atomicAdd(&hbase[min(deg, 255)], 1);
      order[slot] = i;
      ninfo[slot] = make_uint2((uint32_t)i | ((uint32_t)min(deg, 0xffff) << 16), (uint32_t)(base + cnt[i]));
    }
  }
}

inline int grid_for(int64_t n, int block, int cap = kNumSMs * 16) {
  int64_t g = (n + block - 1) / block;
  if (g < 1) g = 1;
  return (int)(g < cap ? g : cap);
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_graph_prep_layout(int64_t N, int64_t E, qagnn_prep_layout* out) {
  if (!out || N <= 0 || E < 0 || N + E >= (int64_t)1 << 31) return QAGNN_ERR_INVALID_ARGUMENT;
  const size_t Ep = (size_t)(N + E);
  size_t o = 0;
  auto take = [&](size_t n_words) { size_t r = o; o += align_up(n_words * 4); return r; };
  out->src = take(Ep);
  out->tgt = take(Ep);
  out->combo = take(Ep);
  out->rowptr_src = take(N + 1);
  out->rowptr_tgt = take(N + 1);
  out->perm_src = take(Ep);
  out->perm_tgt = take(Ep);
  out->csr_src_tgt = take(Ep);
  out->csr_src_combo = take(Ep);
  out->csr_tgt_src = take(Ep);
  out->csr_tgt_combo = take(Ep);
  out->csr_tgt_apos = take(Ep);
  out->pk_src = take(Ep);
  out->pk_tgt = take(Ep);
  out->csr_src_tpos = take(Ep);
  out->order_src = take(N);
  out->order_tgt = take(N);
  out->ninfo_src = take(2 * (size_t)N);
  out->ninfo_tgt = take(2 * (size_t)N);
  out->status = take(4);
  out->scratch = o;
  o += make_scratch(N, E).total * 4;
  out->total_bytes = align_up(o);
  return QAGNN_OK;
}

extern "C" size_t qagnn_graph_prep_bytes(int64_t N, int64_t E) {
  qagnn_prep_layout l;
  if (qagnn_graph_prep_layout(N, E, &l) != QAGNN_OK) return 0;
  return l.total_bytes;
}

extern "C" int32_t qagnn_graph_prep(const int64_t* edge_index, const int64_t* edge_type, const int64_t* node_type,
                                    const qagnn_shape* shape, void* prep, size_t prep_bytes, int32_t validate,
                                    void* stream) {
  if (!shape || !node_type || !prep) return QAGNN_ERR_INVALID_ARGUMENT;
  const int64_t N = shape->N, E = shape->E;
  if (E > 0 && (!edge_index || !edge_type)) return QAGNN_ERR_INVALID_ARGUMENT;
  if (shape->T <= 0 || shape->R <= 0) return QAGNN_ERR_INVALID_ARGUMENT;
  qagnn_prep_layout pl;
  QAGNN_RETURN_IF(qagnn_graph_prep_layout(N, E, &pl));
  if (prep_bytes < pl.total_bytes) return QAGNN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  char* base = (char*)prep;
  auto I = [&](size_t off) { return (int32_t*)(base + off); };
  const PrepScratch sc = make_scratch(N, E);
  int32_t* scr = I(pl.scratch);
  const int64_t Ep = N + E;
  const int nb = (int)scan_blocks(N);
  // packed 16|16 local ids need n_per_graph and the combo count to fit in 16 bits
  const int64_t Ccombo = (int64_t)shape->R * shape->T * shape->T + shape->T;
  const int npg = (shape->n_per_graph > 0 && shape->n_per_graph <= 65535 && Ccombo <= 65536 &&
                   N % shape->n_per_graph == 0) ? shape->n_per_graph : 0;

  ProfScope ps(QAGNN_PROF_GRAPH_PREP, st);
  // zero the status word and the count arrays (status .. cnt_tgt are contiguous up to bsum)
  QAGNN_CHECK_CUDA(cudaMemsetAsync(I(pl.status), 0, 16, st));
  QAGNN_CHECK_CUDA(cudaMemsetAsync(scr + sc.cnt_src, 0, (sc.bsum - sc.cnt_src) * 4, st));

  prep_edges_kernel<<<grid_for(Ep, 256), 256, 0, st>>>(edge_index, edge_type, node_type, N, E, shape->T, shape->R,
                                                       shape->n_per_graph > 0 ? shape->n_per_graph : 0, I(pl.src), I(pl.tgt), I(pl.combo), scr + sc.cnt_src,
                                                       scr + sc.cnt_tgt, I(pl.status));
  QAGNN_CHECK_LAUNCH();
  scan_block_sums_kernel<<<dim3(nb, 2), kScanChunk, 0, st>>>(scr + sc.cnt_src, scr + sc.cnt_tgt, N, scr + sc.bsum, nb);
  QAGNN_CHECK_LAUNCH();
  scan_sums_kernel<<<dim3(1, 2), kScanChunk, 0, st>>>(scr + sc.bsum, nb);
  QAGNN_CHECK_LAUNCH();
  scan_apply_kernel<<<dim3(nb, 2), kScanChunk, 0, st>>>(scr + sc.cnt_src, scr + sc.cnt_tgt, N, scr + sc.bsum, nb,
                                                         I(pl.rowptr_src), I(pl.rowptr_tgt));
  QAGNN_CHECK_LAUNCH();
  prep_fill_kernel<<<grid_for(Ep, 256), 256, 0, st>>>(I(pl.src), I(pl.tgt), Ep, I(pl.rowptr_src), I(pl.rowptr_tgt),
                                                      scr + sc.cnt_src, scr + sc.cnt_tgt, scr + sc.tmp_src,
                                                      scr + sc.tmp_tgt);
  QAGNN_CHECK_LAUNCH();
  prep_sort_segments_kernel<<<grid_for(2 * N * 32, 256, kNumSMs * 32), 256, 0, st>>>(
      N, I(pl.rowptr_src), I(pl.rowptr_tgt), scr + sc.tmp_src, scr + sc.tmp_tgt, I(pl.perm_src), I(pl.perm_tgt),
      scr + sc.big_list, I(pl.status) + 1);
  QAGNN_CHECK_LAUNCH();
  // hub nodes (more than 32 edges in a segment): one CTA per listed segment; exits at once when the list is empty
  prep_sort_big_segments_kernel<<<kNumSMs, kBigThreads, 0, st>>>(N, I(pl.rowptr_src), I(pl.rowptr_tgt), scr + sc.tmp_src,
                                                             scr + sc.tmp_tgt, I(pl.perm_src), I(pl.perm_tgt),
                                                             scr + sc.big_list, I(pl.status) + 1);
  QAGNN_CHECK_LAUNCH();
  prep_payload_src_kernel<<<grid_for(Ep, 256), 256, 0, st>>>(Ep, I(pl.perm_src), I(pl.tgt), I(pl.combo),
                                                             I(pl.csr_src_tgt), I(pl.csr_src_combo),
                                                             scr + sc.inv_src, I(pl.src), npg, I(pl.pk_src));
  QAGNN_CHECK_LAUNCH();
  prep_payload_tgt_kernel<<<grid_for(Ep, 256), 256, 0, st>>>(Ep, I(pl.perm_tgt), I(pl.src), I(pl.combo),
                                                             scr + sc.inv_src, I(pl.csr_tgt_src),
                                                             I(pl.csr_tgt_combo), I(pl.csr_tgt_apos), I(pl.tgt), npg,
                                                             I(pl.pk_tgt), scr + sc.inv_tgt);
  QAGNN_CHECK_LAUNCH();
  prep_tpos_kernel<<<grid_for(Ep, 256), 256, 0, st>>>(Ep, I(pl.perm_src), scr + sc.inv_tgt, I(pl.csr_src_tpos));
  QAGNN_CHECK_LAUNCH();
  if (npg > 0) {
    prep_degree_order_kernel<<<dim3((unsigned)(N / npg), 2), 256, 0, st>>>(npg, I(pl.rowptr_src), I(pl.rowptr_tgt),
                                                                          I(pl.order_src), I(pl.order_tgt),
                                                                          (uint2*)I(pl.ninfo_src), (uint2*)I(pl.ninfo_tgt));
    QAGNN_CHECK_LAUNCH();
  }
  if (validate) {
    int32_t h = 0;
    QAGNN_CHECK_CUDA(cudaMemcpyAsync(&h, I(pl.status), 4, cudaMemcpyDeviceToHost, st));
    QAGNN_CHECK_CUDA(cudaStreamSynchronize(st));
    if (h != 0) return QAGNN_ERR_INDEX_RANGE;
  }
  return QAGNN_OK;
}

namespace qagnn {
namespace {

// qagnn_graph_prep_packed (node_ptr == nullptr) and qagnn_graph_prep_ragged
int32_t graph_prep_packed(const int64_t* edge_index, const int64_t* edge_type, const int64_t* node_type, const int64_t* graph_ptr,
                          const int64_t* node_ptr, int32_t n_graphs, int32_t max_edges_per_graph, const qagnn_shape* shape,
                          void* prep, size_t prep_bytes, int32_t validate, void* stream) {
  const bool ragged = node_ptr != nullptr;
  if (!shape || !node_type || !prep || !graph_ptr) return QAGNN_ERR_INVALID_ARGUMENT;
  const int64_t N = shape->N, E = shape->E;
  if (E > 0 && (!edge_index || !edge_type)) return QAGNN_ERR_INVALID_ARGUMENT;
  if (shape->T <= 0 || shape->R <= 0 || max_edges_per_graph < 0) return QAGNN_ERR_INVALID_ARGUMENT;
  if (ragged && (n_graphs <= 0 || n_graphs > N)) return QAGNN_ERR_INVALID_ARGUMENT;
  const int npg = shape->n_per_graph;
  const int64_t Ccombo = (int64_t)shape->R * shape->T * shape->T + shape->T;
  if (npg <= 0 || npg > 65535 || (!ragged && N % npg != 0) || Ccombo > 65536) return QAGNN_ERR_UNSUPPORTED;
  qagnn_prep_layout pl;
  QAGNN_RETURN_IF(qagnn_graph_prep_layout(N, E, &pl));
  if (prep_bytes < pl.total_bytes) return QAGNN_ERR_WORKSPACE;
  const int cap = max_edges_per_graph + npg;
  const size_t smem = ((size_t)5 * npg + 2 + (size_t)9 * cap) * sizeof(int32_t);
  static int smem_c[kMaxDevices] = {0};
  static size_t attr[2][kMaxDevices] = {{0}};
  const int dev = current_device();
  if (smem_c[dev] == 0) cudaDeviceGetAttribute(&smem_c[dev], cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (smem + 4096 > (size_t)smem_c[dev]) return QAGNN_ERR_UNSUPPORTED;  // sub-graphs too large for one CTA: use qagnn_graph_prep
  if (smem + 4096 > 48 * 1024 && smem > attr[ragged][dev]) {  // the kernel also has 2 KB of static shared memory
    QAGNN_CHECK_CUDA(cudaFuncSetAttribute(ragged ? prep_packed_graph_kernel<true> : prep_packed_graph_kernel<false>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr[ragged][dev] = smem;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* base = (char*)prep;
  auto I = [&](size_t off) { return (int32_t*)(base + off); };
  ProfScope ps(QAGNN_PROF_GRAPH_PREP, st);
  QAGNN_CHECK_CUDA(cudaMemsetAsync(I(pl.status), 0, 16, st));
  PackedPrepArgs a;
  a.edge_index = edge_index; a.edge_type = edge_type; a.node_type = node_type; a.graph_ptr = graph_ptr; a.node_ptr = node_ptr;
  a.N = N; a.E = E; a.T = shape->T; a.R = shape->R; a.npg = npg; a.cap = cap; a.B = ragged ? n_graphs : 0;
  a.src = I(pl.src); a.tgt = I(pl.tgt); a.combo = I(pl.combo); a.rowptr_src = I(pl.rowptr_src); a.rowptr_tgt = I(pl.rowptr_tgt);
  a.perm_src = I(pl.perm_src); a.perm_tgt = I(pl.perm_tgt); a.csr_src_tgt = I(pl.csr_src_tgt); a.csr_src_combo = I(pl.csr_src_combo);
  a.csr_tgt_src = I(pl.csr_tgt_src); a.csr_tgt_combo = I(pl.csr_tgt_combo); a.csr_tgt_apos = I(pl.csr_tgt_apos);
  a.pk_src = I(pl.pk_src); a.pk_tgt = I(pl.pk_tgt); a.csr_src_tpos = I(pl.csr_src_tpos); a.order_src = I(pl.order_src);
  a.order_tgt = I(pl.order_tgt); a.status = I(pl.status); a.ninfo_src = (uint2*)I(pl.ninfo_src); a.ninfo_tgt = (uint2*)I(pl.ninfo_tgt);
  if (ragged) {
    prep_packed_graph_kernel<true><<<(unsigned)ragged_max_segments(N, n_graphs, npg), kPackedThreads, smem, st>>>(a);
  } else {
    prep_packed_graph_kernel<false><<<(unsigned)(N / npg), kPackedThreads, smem, st>>>(a);
  }
  QAGNN_CHECK_LAUNCH();
  if (validate) {
    int32_t h = 0;
    QAGNN_CHECK_CUDA(cudaMemcpyAsync(&h, I(pl.status), 4, cudaMemcpyDeviceToHost, st));
    QAGNN_CHECK_CUDA(cudaStreamSynchronize(st));
    if (h != 0) return QAGNN_ERR_INDEX_RANGE;
  }
  return QAGNN_OK;
}

}  // namespace
}  // namespace qagnn

extern "C" int32_t qagnn_graph_prep_packed(const int64_t* edge_index, const int64_t* edge_type, const int64_t* node_type,
                                           const int64_t* graph_ptr, int32_t max_edges_per_graph, const qagnn_shape* shape,
                                           void* prep, size_t prep_bytes, int32_t validate, void* stream) {
  return graph_prep_packed(edge_index, edge_type, node_type, graph_ptr, nullptr, 0, max_edges_per_graph, shape, prep, prep_bytes,
                           validate, stream);
}

extern "C" int32_t qagnn_graph_prep_ragged(const int64_t* edge_index, const int64_t* edge_type, const int64_t* node_type,
                                           const int64_t* graph_ptr, const int64_t* node_ptr, int32_t n_graphs,
                                           int32_t max_edges_per_graph, const qagnn_shape* shape, void* prep, size_t prep_bytes,
                                           int32_t validate, void* stream) {
  if (!node_ptr) return QAGNN_ERR_INVALID_ARGUMENT;
  return graph_prep_packed(edge_index, edge_type, node_type, graph_ptr, node_ptr, n_graphs, max_edges_per_graph, shape, prep,
                           prep_bytes, validate, stream);
}
