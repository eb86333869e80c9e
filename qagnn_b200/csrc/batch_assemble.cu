// Batch assembly from a split held on the device (qagnn_assemble_batch): the packed adjacency of B = bs * num_choice sub-graphs,
// cut out of the split's flat arrays by question id, equal to FlatAdjCache.pack on the host (qagnn_b200/data.py).
//
// Two launches, so the whole assembly can sit inside a captured CUDA graph:
//   1. assemble_scan_kernel  one CTA of 1024 threads walks the B graphs in chunks of 1024: each thread reads its graph's edge
//                            count (and length), a block scan gives graph_ptr (and node_ptr), and a carry joins the chunks
//   2. assemble_copy_kernel  one thread per output column p < K: a binary search over graph_ptr finds the graph b that owns p,
//                            the edge is read from the split and written with b's node base added; columns past graph_ptr[B]
//                            are written as zero
// Every output element has exactly one writer and every sum is a scan in a fixed order, so there are no atomics and the
// result does not depend on scheduling.  Question ids and counts are clamped on the device: graph_ptr stays in [0, K],
// node_ptr in [0, N_cap], no write goes past K columns or B + 1 entries, and no read leaves the split.
#include "common.cuh"

namespace qagnn {

namespace {

constexpr int kScanThreads = 1024;
constexpr int kCopyThreads = 256;

// Exclusive scan of one int64 per thread over a 1024-thread block; *total = the block's sum.  Every thread must call it.
__device__ __forceinline__ int64_t block_exclusive_scan_i64(int64_t v, int64_t* total) {
  __shared__ int64_t warp_sums[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int64_t w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    warp_sums[lane] = w;
  }
  __syncthreads();
  const int64_t base = wid ? warp_sums[wid - 1] : 0;
  *total = warp_sums[31];
  __syncthreads();
  return base + x - v;
}

// Split graph of batch graph b: choice b % nc of question qids[b / nc], the id clamped to [0, Q)
__device__ __forceinline__ int64_t split_graph(const int64_t* __restrict__ qids, int64_t b, int nc, int64_t Q) {
  const int64_t q = min(max(qids[b / nc], (int64_t)0), Q - 1);
  return q * nc + b % nc;
}

__global__ void __launch_bounds__(kScanThreads) assemble_scan_kernel(const int64_t* __restrict__ split_ptr,
                                                                     const int64_t* __restrict__ split_lens, int64_t Q, int nc,
                                                                     int n_nodes, const int64_t* __restrict__ qids, int64_t B,
                                                                     int64_t K, int64_t N_cap, int64_t* __restrict__ graph_ptr,
                                                                     int64_t* __restrict__ node_ptr) {
  int64_t e_carry = 0, n_carry = 0;
  for (int64_t b0 = 0; b0 < B; b0 += kScanThreads) {
    const int64_t b = b0 + threadIdx.x;
    int64_t cnt = 0, len = 0;
    if (b < B) {
      const int64_t g = split_graph(qids, b, nc, Q);
      cnt = max(split_ptr[g + 1] - split_ptr[g], (int64_t)0);
      if (node_ptr) len = min(max(split_lens[g], (int64_t)0), (int64_t)n_nodes);
    }
    int64_t e_total, n_total;
    const int64_t e_off = e_carry + block_exclusive_scan_i64(cnt, &e_total);
    if (b < B) graph_ptr[b] = min(e_off, K);
    e_carry += e_total;
    if (node_ptr) {  // uniform across the block: every thread takes part in the scan
      const int64_t n_off = n_carry + block_exclusive_scan_i64(len, &n_total);
      if (b < B) node_ptr[b] = min(n_off, N_cap);
      n_carry += n_total;
    }
  }
  if (threadIdx.x == 0) {
    graph_ptr[B] = min(e_carry, K);
    if (node_ptr) node_ptr[B] = min(n_carry, N_cap);
  }
}

__global__ void __launch_bounds__(kCopyThreads) assemble_copy_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ tgt,
                                                                     const int16_t* __restrict__ etype,
                                                                     const int64_t* __restrict__ split_ptr, int64_t Q, int nc,
                                                                     int n_nodes, const int64_t* __restrict__ qids, int64_t B,
                                                                     int64_t K, const int64_t* __restrict__ graph_ptr,
                                                                     const int64_t* __restrict__ node_ptr,
                                                                     int64_t* __restrict__ edges) {
  const int64_t total = graph_ptr[B];
  const int64_t E_split = split_ptr[Q * nc];
  for (int64_t p = (int64_t)blockIdx.x * kCopyThreads + threadIdx.x; p < K; p += (int64_t)gridDim.x * kCopyThreads) {
    int64_t s = 0, t = 0, r = 0;
    if (p < total) {
      int64_t lo = 0, hi = B;  // largest b with graph_ptr[b] <= p; graph_ptr[b + 1] > p then holds
      while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (graph_ptr[mid] <= p) lo = mid; else hi = mid;
      }
      const int64_t e = min(max(split_ptr[split_graph(qids, lo, nc, Q)] + (p - graph_ptr[lo]), (int64_t)0), E_split - 1);
      const int64_t base = node_ptr ? node_ptr[lo] : lo * n_nodes;
      s = (int64_t)src[e] + base;
      t = (int64_t)tgt[e] + base;
      r = etype[e];
    }
    edges[p] = s;
    edges[K + p] = t;
    edges[2 * K + p] = r;
  }
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_assemble_batch(const int32_t* src, const int32_t* tgt, const int16_t* etype, const int64_t* graph_ptr,
                                        const int64_t* adj_lengths, int64_t G, int32_t num_choice, int32_t n_nodes,
                                        const int64_t* question_ids, int32_t bs, int64_t K, int64_t N_cap, int64_t* edges,
                                        int64_t* graph_ptr_out, int64_t* node_ptr_out, void* stream) {
  if (!graph_ptr || !question_ids || !graph_ptr_out || num_choice <= 0 || n_nodes <= 0 || bs <= 0 || K < 0 || G < num_choice ||
      G % num_choice != 0 || N_cap < -1)
    return QAGNN_ERR_INVALID_ARGUMENT;
  if (K > 0 && (!src || !tgt || !etype || !edges)) return QAGNN_ERR_INVALID_ARGUMENT;
  const bool ragged = N_cap >= 0;
  if (ragged && (!adj_lengths || !node_ptr_out)) return QAGNN_ERR_INVALID_ARGUMENT;
  const int64_t Q = G / num_choice, B = (int64_t)bs * num_choice;
  int64_t* np_out = ragged ? node_ptr_out : nullptr;
  cudaStream_t st = (cudaStream_t)stream;
  assemble_scan_kernel<<<1, kScanThreads, 0, st>>>(graph_ptr, adj_lengths, Q, num_choice, n_nodes, question_ids, B, K, N_cap,
                                                   graph_ptr_out, np_out);
  QAGNN_CHECK_LAUNCH();
  if (K > 0) {
    const int64_t blocks = min((K + kCopyThreads - 1) / kCopyThreads, (int64_t)kNumSMs * 16);
    assemble_copy_kernel<<<(unsigned)blocks, kCopyThreads, 0, st>>>(src, tgt, etype, graph_ptr, Q, num_choice, n_nodes,
                                                                    question_ids, B, K, graph_ptr_out, np_out, edges);
    QAGNN_CHECK_LAUNCH();
  }
  return QAGNN_OK;
}
