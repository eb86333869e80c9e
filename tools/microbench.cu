// Micro-benchmarks that size the message-passing design on the actual GPU:
//   hbm_read / l2_read (streaming float4), table_gather (random 800-B rows from a 1 MB table = the
//   Ke/Me access pattern), smem_read (LDS.128 from a resident tile).
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/bin/microbench tools/microbench.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__global__ void stream_read(const float4* __restrict__ p, size_t n4, int passes, float* out) {
  float acc = 0.f;
  for (int r = 0; r < passes; ++r)
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
      float4 v = p[i];
      acc += v.x + v.y + v.z + v.w;
    }
  if (acc == 123.456f) out[0] = acc;
}

// each warp reads `rows_per_warp` random rows of `row_f4` float4 (lanes stride across the row)
__global__ void table_gather(const float4* __restrict__ tab, int n_rows, int row_f4, int rows_per_warp, float* out) {
  const int lane = threadIdx.x & 31;
  unsigned w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  unsigned s = w * 2654435761u + 12345u;
  float acc = 0.f;
  for (int r = 0; r < rows_per_warp; ++r) {
    s = s * 1664525u + 1013904223u;
    const int row = (s >> 8) % n_rows;
    for (int c = lane; c < row_f4; c += 32) {
      float4 v = tab[(size_t)row * row_f4 + c];
      acc += v.x + v.y + v.z + v.w;
    }
  }
  if (acc == 123.456f) out[0] = acc;
}

__global__ void smem_read(int iters, float* out) {
  extern __shared__ float4 sm[];
  const int n4 = 160 * 1024 / 16;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) sm[i] = make_float4(i, 1, 2, 3);
  __syncthreads();
  float acc = 0.f;
  unsigned idx = threadIdx.x;
  for (int r = 0; r < iters; ++r) {
#pragma unroll 8
    for (int k = 0; k < 8; ++k) {
      float4 v = sm[(idx + k * 1024) % n4];
      acc += v.x + v.y + v.z + v.w;
    }
    idx = (idx + 8 * 1024 + 32) % n4;
  }
  if (acc == 123.456f) out[0] = acc;
}

// The message-passing kernel's access pattern: every quarter-warp (8 lanes) reads one 208-byte row (13 float4 chunks:
// chunks 0-7, then chunks 8-12 with lanes 5-7 re-reading an in-row chunk) of a random row of a table resident in shared
// memory; the four quarter-warps of a warp read four different rows.  Counts quarter-warp wavefronts per clock.
__global__ void smem_row_gather(int iters, int rows, float* out) {
  extern __shared__ float4 sm[];
  const int NCH = 13;
  for (int i = threadIdx.x; i < rows * NCH; i += blockDim.x) sm[i] = make_float4(i, 1, 2, 3);
  __syncthreads();
  const int lane = threadIdx.x & 31, l8 = lane & 7;
  const int c0 = l8, c1 = (l8 + 8 < NCH) ? l8 + 8 : l8 % NCH;
  unsigned state = (threadIdx.x >> 3) * 2654435761u + blockIdx.x * 40503u + 12345u;  // one stream per quarter-warp
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = 0; r < iters; ++r) {
#pragma unroll 4
    for (int k = 0; k < 4; ++k) {
      state = state * 1664525u + 1013904223u;
      const int row = (int)((state >> 8) % (unsigned)rows);
      const float4 a = sm[row * NCH + c0], b = sm[row * NCH + c1];
      acc.x += a.x + b.x; acc.y += a.y + b.y; acc.z += a.z + b.z; acc.w += a.w + b.w;
    }
  }
  if (acc.x + acc.y + acc.z + acc.w == 123.456f) out[0] = acc.x;
}

template <class F>
float time_ms(F f, int reps = 5) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  f();
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int i = 0; i < reps; ++i) {
    cudaEventRecord(a); f(); cudaEventRecord(b); CK(cudaEventSynchronize(b));
    float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms;
  }
  return best;
}

int main() {
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  printf("device %s, %d SMs, L2 %.1f MB, smem/SM %zu KB, clock %d MHz\n", prop.name, prop.multiProcessorCount,
         prop.l2CacheSize / 1e6, prop.sharedMemPerMultiprocessor / 1024, prop.clockRate / 1000);
  float* out; CK(cudaMalloc(&out, 4));
  const int sms = prop.multiProcessorCount;
  {  // HBM
    size_t bytes = (size_t)4 << 30; float4* p; CK(cudaMalloc(&p, bytes)); CK(cudaMemset(p, 0, bytes));
    float ms = time_ms([&] { stream_read<<<sms * 16, 512>>>(p, bytes / 16, 1, out); });
    printf("hbm_read      %8.1f GB/s (4 GiB, %.3f ms)\n", bytes / ms / 1e6, ms);
    cudaFree(p);
  }
  for (size_t mb : {8, 32, 64, 96}) {  // L2 resident
    size_t bytes = mb << 20; float4* p; CK(cudaMalloc(&p, bytes)); CK(cudaMemset(p, 0, bytes));
    int passes = 20;
    float ms = time_ms([&] { stream_read<<<sms * 16, 512>>>(p, bytes / 16, passes, out); });
    printf("l2_read %3zuMB  %8.1f GB/s\n", mb, bytes * (double)passes / ms / 1e6);
    cudaFree(p);
  }
  {  // table gather: 624 rows x 200 floats (x2 tables ~ 1 MB) -> rows of 50 float4
    for (int rows : {624, 1248, 8192}) {
      const int row_f4 = 50; size_t bytes = (size_t)rows * row_f4 * 16; float4* p; CK(cudaMalloc(&p, bytes)); CK(cudaMemset(p, 0, bytes));
      const int rpw = 256; const int blocks = sms * 8, threads = 256;
      float ms = time_ms([&] { table_gather<<<blocks, threads>>>(p, rows, row_f4, rpw, out); });
      double total = (double)blocks * (threads / 32) * rpw * row_f4 * 16;
      printf("table_gather %5d rows x 800 B : %8.1f GB/s  (%.1f M rows/s)\n", rows, total / ms / 1e6, total / 800 / ms / 1e3);
      cudaFree(p);
    }
    for (int rows : {624}) {  // per-head rows of 200 B (50 floats): 12.5 float4 -> use 13
      const int row_f4 = 13; size_t bytes = (size_t)rows * row_f4 * 16; float4* p; CK(cudaMalloc(&p, bytes)); CK(cudaMemset(p, 0, bytes));
      const int rpw = 1024; const int blocks = sms * 8, threads = 256;
      float ms = time_ms([&] { table_gather<<<blocks, threads>>>(p, rows, row_f4, rpw, out); });
      double total = (double)blocks * (threads / 32) * rpw * row_f4 * 16;
      printf("table_gather %5d rows x 208 B : %8.1f GB/s  (%.1f M rows/s)\n", rows, total / ms / 1e6, total / 208 / ms / 1e3);
      cudaFree(p);
    }
  }
  {  // shared memory
    CK(cudaFuncSetAttribute(smem_read, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    const int iters = 2000;
    float ms = time_ms([&] { smem_read<<<sms, 1024, 160 * 1024>>>(iters, out); });
    double total = (double)sms * 1024 * iters * 8 * 16;
    printf("smem_read     %8.1f GB/s aggregate (%.1f B/clk/SM at %d MHz nominal)\n", total / ms / 1e6,
           total / ms / 1e6 * 1e9 / sms / (prop.clockRate * 1e3), prop.clockRate / 1000);
  }
  for (int threads : {800, 1024}) {  // random 208-byte rows per quarter-warp (the message-passing kernel's pattern)
    const int rows = 612 + 200;  // table + one node tile
    const size_t smem = (size_t)rows * 13 * 16;
    CK(cudaFuncSetAttribute(smem_row_gather, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int iters = 4000;
    float ms = time_ms([&] { smem_row_gather<<<sms, threads, smem>>>(iters, rows, out); });
    const double wavefronts = (double)sms * (threads / 8) * iters * 4 * 2;  // 2 quarter-warp LDS.128 per row
    const double clk = ms * 1e-3 * prop.clockRate * 1e3;
    printf("smem_row_gather %4d threads: %.3f quarter-warp wavefronts/clk/SM (%.1f G rows/s aggregate, %.1f B/clk/SM useful)\n", threads,
           wavefronts / sms / clk, (double)sms * (threads / 8) * iters * 4 / ms / 1e6, wavefronts / 2 * 208 / sms / clk);
  }
  return 0;
}
