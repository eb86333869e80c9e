// The two launches that frame a whole optimiser batch replayed as one CUDA graph (qagnn_b200.pipeline.SplitTrainBatchGraph),
// so a replay needs no host input: qagnn_schedule_batch reads the batch's question ids from a device epoch order at a device
// batch counter, and qagnn_batch_log adds the batch's weighted losses into a device fp64 total and advances the counter.
// Both are launch-bound: one block, no host read.  Also the graph helpers the batch graph is built with.
#include "common.cuh"

namespace qagnn {

namespace {

constexpr int kScheduleThreads = 256;

// ids[i] = order[counter * batch_size + i] for the batch's n_full = (batch_size / mbs) * mbs first questions: micro-batch j
// takes ids[j * mbs, (j + 1) * mbs), which is row j % branches of chunk j / branches of a [chunks, branches, mbs] block.  A
// counter past the epoch's last full batch (or negative) and an id outside [0, Q) set their status bit and read question 0
// instead, so nothing downstream indexes out of range.
__global__ void __launch_bounds__(kScheduleThreads)
    schedule_batch_kernel(const int64_t* __restrict__ order, int64_t n_order, const int64_t* __restrict__ counter,
                          int64_t batch_size, int64_t n_full, int64_t n_questions, int64_t* __restrict__ ids,
                          int32_t* __restrict__ status) {
  const int64_t c = *counter;
  const bool in_epoch = c >= 0 && c < n_order / batch_size;
  if (!in_epoch && threadIdx.x == 0) atomicOr(status, QAGNN_SCHEDULE_PAST_EPOCH);
  bool bad = false;
  for (int64_t i = threadIdx.x; i < n_full; i += kScheduleThreads) {
    int64_t q = in_epoch ? order[c * batch_size + i] : 0;
    if (q < 0 || q >= n_questions) {
      bad = true;
      q = 0;
    }
    ids[i] = q;
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(status, QAGNN_SCHEDULE_BAD_ID);
}

// total += (double)((loss_j * (float)mbs) * (1.f / (float)bs)) for j = 0 ... n_micro - 1 in order, then ++counter.  The weight
// is torch's `loss * mbs / bs` on a CUDA fp32 loss (a multiply by the host scalar, then a multiply by its fp32 reciprocal, as
// torch divides by a CPU scalar), and the double adds are Python's `total_loss += loss.item()`.
__global__ void batch_log_kernel(const float* __restrict__ losses, int32_t n_micro, float mbs, float inv_bs,
                                 double* __restrict__ total, int64_t* __restrict__ counter) {
  if (threadIdx.x != 0) return;
  double acc = *total;
  for (int32_t j = 0; j < n_micro; ++j) acc += (double)__fmul_rn(__fmul_rn(losses[j], mbs), inv_bs);
  *total = acc;
  *counter += 1;
}

int64_t graph_nodes(cudaGraph_t g, bool recursive, int depth = 0) {
  size_t n = 0;
  if (depth > 8 || cudaGraphGetNodes(g, nullptr, &n) != cudaSuccess) return -1;
  if (!recursive || n == 0) return (int64_t)n;
  cudaGraphNode_t* nodes = new cudaGraphNode_t[n];
  int64_t total = 0;
  if (cudaGraphGetNodes(g, nodes, &n) != cudaSuccess) total = -1;
  for (size_t i = 0; i < n && total >= 0; ++i) {
    cudaGraphNodeType t;
    cudaGraph_t child;
    if (cudaGraphNodeGetType(nodes[i], &t) != cudaSuccess) total = -1;
    else if (t != cudaGraphNodeTypeGraph) total += 1;
    else if (cudaGraphChildGraphNodeGetGraph(nodes[i], &child) != cudaSuccess) total = -1;
    else {
      const int64_t k = graph_nodes(child, true, depth + 1);
      total = k < 0 ? -1 : total + k;
    }
  }
  delete[] nodes;
  return total;
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_schedule_batch(const int64_t* order, int64_t n_order, const int64_t* counter, int64_t batch_size,
                                        int32_t micro_batch_size, int64_t n_questions, int64_t* ids, int32_t* status,
                                        void* stream) {
  if (!order || !counter || !ids || !status || n_order < 0 || batch_size < 1 || micro_batch_size < 1 ||
      micro_batch_size > batch_size || n_questions < 1)
    return QAGNN_ERR_INVALID_ARGUMENT;
  const int64_t n_full = batch_size / micro_batch_size * micro_batch_size;
  schedule_batch_kernel<<<1, kScheduleThreads, 0, (cudaStream_t)stream>>>(order, n_order, counter, batch_size, n_full,
                                                                          n_questions, ids, status);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

extern "C" int32_t qagnn_batch_log(const float* losses, int32_t n_micro, int32_t micro_batch_size, int64_t batch_size,
                                   double* total, int64_t* counter, void* stream) {
  if (!losses || !total || !counter || n_micro < 1 || micro_batch_size < 1 || batch_size < 1)
    return QAGNN_ERR_INVALID_ARGUMENT;
  const float inv_bs = 1.f / (float)batch_size;
  batch_log_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(losses, n_micro, (float)micro_batch_size, inv_bs, total, counter);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

extern "C" int32_t qagnn_graph_add_child(void* stream, void* child_graph) {
  if (!child_graph) return QAGNN_ERR_INVALID_ARGUMENT;
  cudaStream_t st = (cudaStream_t)stream;
  cudaStreamCaptureStatus cs;
  cudaGraph_t g;
  const cudaGraphNode_t* deps = nullptr;
  size_t n_deps = 0;
  QAGNN_CHECK_CUDA(cudaStreamGetCaptureInfo(st, &cs, nullptr, &g, &deps, &n_deps));
  if (cs != cudaStreamCaptureStatusActive) return QAGNN_ERR_INVALID_ARGUMENT;
  cudaGraphNode_t node;
  QAGNN_CHECK_CUDA(cudaGraphAddChildGraphNode(&node, g, deps, n_deps, (cudaGraph_t)child_graph));
  QAGNN_CHECK_CUDA(cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies));
  return QAGNN_OK;
}

extern "C" int64_t qagnn_graph_node_count(void* graph, int32_t recursive) {
  return graph ? graph_nodes((cudaGraph_t)graph, recursive != 0) : -1;
}
