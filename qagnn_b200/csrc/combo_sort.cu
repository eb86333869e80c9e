// Combo sort of a graph prep: the by-source edge positions [0, E') stably sorted by csr_src_combo, and the histogram of the
// combos.  The training backward sums the edge-table gradients in that order (qagnn_mp_core_backward), and the training
// forward weights the edge encoder's BatchNorm moments with the histogram (qagnn_b200/training.py).
//
// A stable counting sort in three launches, with E' = rowptr_src[N] read on the device so that one captured launch sequence
// serves every batch at an edge capacity:
//   1. combo_hist_kernel     one CTA per tile of kTile positions: the tile's histogram, hist[tile][c]
//   2. combo_scan_kernel     one CTA: the bin totals (= combo_count), then hist[tile][c] becomes the first output slot of
//                            bin c in tile `tile` (exclusive scan in (bin, tile) order)
//   3. combo_scatter_kernel  one CTA per tile, one warp per kTile / 8 consecutive positions: each warp takes its own slots
//                            out of the tile's, then walks its positions 32 at a time in order; equal combos inside a step are
//                            ranked by lane (__match_any_sync), so every position lands at its stable rank
// Counts are integer sums, so the shared-memory atomics cannot change any output: the result is unique and bit-identical
// to a stable argsort by combo.
#include "common.cuh"

namespace qagnn {

namespace {

constexpr int kSortThreads = 256, kSortWarps = kSortThreads / 32;
constexpr int kWarpSpan = 512;                    // positions per warp in the scatter
constexpr int kTile = kSortWarps * kWarpSpan;     // positions per tile
constexpr int kMaxCombos = 6144;                  // 8 per-warp cursor rows of C ints fit the 227 KB of opt-in shared memory

inline int64_t combo_tiles(int64_t Ep_cap) { return Ep_cap > 0 ? (Ep_cap + kTile - 1) / kTile : 1; }

__device__ __forceinline__ int64_t real_positions(const int32_t* rowptr_end, int64_t Ep_cap) {
  const int64_t e = *rowptr_end;
  return e < 0 ? 0 : (e > Ep_cap ? Ep_cap : e);
}

__global__ void __launch_bounds__(kSortThreads) combo_hist_kernel(const int32_t* __restrict__ rowptr_end, int64_t Ep_cap, int C,
                                                                  const int32_t* __restrict__ key, int32_t* __restrict__ hist) {
  extern __shared__ int32_t sm_h[];
  const int64_t Ep = real_positions(rowptr_end, Ep_cap);
  for (int c = threadIdx.x; c < C; c += kSortThreads) sm_h[c] = 0;
  __syncthreads();
  const int64_t p0 = (int64_t)blockIdx.x * kTile, p1 = min(p0 + kTile, Ep);
  for (int64_t p = p0 + threadIdx.x; p < p1; p += kSortThreads) atomicAdd(&sm_h[min(max(key[p], 0), C - 1)], 1);
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kSortThreads) hist[(size_t)blockIdx.x * C + c] = sm_h[c];
}

__global__ void __launch_bounds__(1024) combo_scan_kernel(int ntiles, int C, int32_t* __restrict__ hist,
                                                          int64_t* __restrict__ count_out) {
  int carry = 0;
  for (int c0 = 0; c0 < C; c0 += 1024) {
    const int c = c0 + threadIdx.x;
    int total = 0;
    if (c < C)
      for (int t = 0; t < ntiles; ++t) total += hist[(size_t)t * C + c];
    int block_total;
    const int base = carry + block_exclusive_scan_1024(total, &block_total);
    carry += block_total;
    if (c < C) {
      count_out[c] = total;
      int off = base;
      for (int t = 0; t < ntiles; ++t) {
        const int v = hist[(size_t)t * C + c];
        hist[(size_t)t * C + c] = off;
        off += v;
      }
    }
  }
}

__global__ void __launch_bounds__(kSortThreads) combo_scatter_kernel(const int32_t* __restrict__ rowptr_end, int64_t Ep_cap, int C,
                                                                     const int32_t* __restrict__ key,
                                                                     const int32_t* __restrict__ tile_slot,
                                                                     int32_t* __restrict__ order) {
  extern __shared__ int32_t sm_cur[];  // [kSortWarps][C]: per-warp counts, then per-warp next output slot
  const int64_t Ep = real_positions(rowptr_end, Ep_cap);
  const int64_t p0 = (int64_t)blockIdx.x * kTile;
  if (p0 >= Ep) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int32_t* cur = sm_cur + warp * C;
  for (int i = threadIdx.x; i < kSortWarps * C; i += kSortThreads) sm_cur[i] = 0;
  __syncthreads();
  const int64_t w0 = p0 + (int64_t)warp * kWarpSpan, w1 = min(w0 + kWarpSpan, Ep);
  for (int64_t p = w0 + lane; p < w1; p += 32) atomicAdd(&cur[min(max(key[p], 0), C - 1)], 1);
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kSortThreads) {  // warps in position order inside the tile's slots of bin c
    int run = tile_slot[(size_t)blockIdx.x * C + c];
    for (int w = 0; w < kSortWarps; ++w) {
      const int n = sm_cur[w * C + c];
      sm_cur[w * C + c] = run;
      run += n;
    }
  }
  __syncthreads();
  for (int64_t b = w0; b < w1; b += 32) {
    const int64_t p = b + lane;
    const bool valid = p < w1;
    const int k = valid ? min(max(key[p], 0), C - 1) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, k);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (valid) order[cur[k] + rank] = (int32_t)p;
    __syncwarp();
    if (valid && lane == __ffs(peers) - 1) cur[k] += __popc(peers);
    __syncwarp();
  }
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" size_t qagnn_combo_sort_bytes(const qagnn_shape* shape) {
  if (!shape || shape->N <= 0 || shape->E < 0 || shape->T <= 0 || shape->R <= 0) return 0;
  const int64_t C = (int64_t)shape->R * shape->T * shape->T + shape->T;
  if (C > kMaxCombos) return 0;
  return align_up((size_t)combo_tiles(shape->N + shape->E) * (size_t)C * sizeof(int32_t));
}

extern "C" int32_t qagnn_combo_sort(const qagnn_shape* shape, const void* prep, int64_t* combo_count_out,
                                    int32_t* combo_order_out, void* scratch, size_t scratch_bytes, void* stream) {
  if (!shape || !prep || !combo_count_out || !combo_order_out || !scratch) return QAGNN_ERR_INVALID_ARGUMENT;
  const size_t need = qagnn_combo_sort_bytes(shape);
  if (need == 0) {
    const bool valid = shape->N > 0 && shape->E >= 0 && shape->T > 0 && shape->R > 0;
    return valid ? QAGNN_ERR_UNSUPPORTED : QAGNN_ERR_INVALID_ARGUMENT;
  }
  if (scratch_bytes < need) return QAGNN_ERR_WORKSPACE;
  qagnn_prep_layout pl;
  QAGNN_RETURN_IF(qagnn_graph_prep_layout(shape->N, shape->E, &pl));
  const int C = shape->R * shape->T * shape->T + shape->T;
  const int64_t Ep_cap = shape->N + shape->E;
  const int64_t ntiles = combo_tiles(Ep_cap);
  const char* base = (const char*)prep;
  const int32_t* rowptr_end = (const int32_t*)(base + pl.rowptr_src) + shape->N;
  const int32_t* key = (const int32_t*)(base + pl.csr_src_combo);
  int32_t* hist = (int32_t*)scratch;
  const size_t smem_hist = (size_t)C * sizeof(int32_t), smem_scatter = (size_t)kSortWarps * C * sizeof(int32_t);
  static size_t attr[kMaxDevices] = {0};
  const int dev = current_device();
  if (smem_scatter > 48 * 1024 && smem_scatter > attr[dev]) {
    QAGNN_CHECK_CUDA(cudaFuncSetAttribute(combo_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_scatter));
    attr[dev] = smem_scatter;
  }
  cudaStream_t st = (cudaStream_t)stream;
  combo_hist_kernel<<<(unsigned)ntiles, kSortThreads, smem_hist, st>>>(rowptr_end, Ep_cap, C, key, hist);
  QAGNN_CHECK_LAUNCH();
  combo_scan_kernel<<<1, 1024, 0, st>>>((int)ntiles, C, hist, combo_count_out);
  QAGNN_CHECK_LAUNCH();
  combo_scatter_kernel<<<(unsigned)ntiles, kSortThreads, smem_scatter, st>>>(rowptr_end, Ep_cap, C, key, hist, combo_order_out);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}
