// Backward of the message passing of one GATConvE layer (the gradient of modeling/modeling_qagnn.py:442,455-484
// with torch_geometric's propagate / softmax and torch_scatter's scatter, on the node-level factorisation):
//
//   forward   s[e,h]  = Q[src] . (Kx[tgt] + Ke[c])        a = softmax over edges sharing SRC        a' = a * outdeg(src)
//             aggr[v] = sum_{e: tgt = v} a'[e,h] (Mx[src] + Me[c])
//   backward  da'[e,h] = dAggr[tgt,h,:] . (Mx[src,h,:] + Me[c,h,:])            da = outdeg(src) * da'
//             ds[e,h]  = a[e,h] (da[e,h] - sum_{e' in out(src)} a[e',h] da[e',h])                  (softmax)
//             dQ[u]  = sum_{e: src = u} ds (Kx[tgt] + Ke[c])      dMx[u] = sum_{e: src = u} a' dAggr[tgt]
//             dKx[v] = sum_{e: tgt = v} ds Q[src]
//             dKe[c] = sum_{e: combo = c} ds Q[src]                dMe[c] = sum_{e: combo = c} a' dAggr[tgt]
//
// Three kernels over the CSR orders of graph prep (general path: any graph):
//   mp_bwd_source_kernel   one warp per SOURCE node: da', softmax backward, ds (kept by-source), dQ, dMx     no atomics
//   mp_bwd_target_kernel   one warp per TARGET node: dKx                                                    no atomics
//   mp_bwd_table_kernel    one warp per run of 64 edges in COMBO order: register partial sums, one vector
//                          atomic add per (run, combo change) into dKe / dMe — the only atomics, a few thousand adds
//
// The deterministic backward (qagnn_mp_core_backward_det) replaces the atomic flush of the table kernel with plain stores:
//   mp_bwd_table_kernel<.., true>   the same walk; a combo whose whole range lies in the run is stored into dKe / dMe, a
//                                   segment that crosses the run's start or end goes to the run's first or last slot
//   mp_bwd_table_combine_kernel     per (combo spanning several runs, 32 columns): the slots of its runs in a fixed order;
//                                   zero rows for combos without edges
// Every sum then has an order fixed by the combo order of the positions alone.
#include <type_traits>

#include "storage.cuh"

namespace qagnn {

namespace {

struct HeadMap4 {
  int first, last;
  int hid[4];
};
__device__ __forceinline__ HeadMap4 head_map4(int c, int d) {
  HeadMap4 m;
#pragma unroll
  for (int t = 0; t < 4; ++t) m.hid[t] = (4 * c + t) / d;
  m.first = m.hid[0];
  m.last = m.hid[3];
  return m;
}

// per-head partial sums of the 4 products of one float4 chunk
template <int H>
__device__ __forceinline__ void add_parts(float (&part)[H], const HeadMap4& hm, float p0, float p1, float p2, float p3) {
  if (hm.first == hm.last) {
    const float s4 = (p0 + p1) + (p2 + p3);
#pragma unroll
    for (int h = 0; h < H; ++h) part[h] += (hm.first == h) ? s4 : 0.f;
  } else {
#pragma unroll
    for (int h = 0; h < H; ++h) {
      part[h] += (hm.hid[0] == h) ? p0 : 0.f;
      part[h] += (hm.hid[1] == h) ? p1 : 0.f;
      part[h] += (hm.hid[2] == h) ? p2 : 0.f;
      part[h] += (hm.hid[3] == h) ? p3 : 0.f;
    }
  }
}
template <int H>
__device__ __forceinline__ float pick(const float (&w)[H], int h) {
  float r = 0.f;
#pragma unroll
  for (int i = 0; i < H; ++i) r = (h == i) ? w[i] : r;
  return r;
}

// S: storage type of the node and table operands (float, __half, __nv_bfloat16): loads widen exactly, the arithmetic is
// fp32 for every S, and d_qkm is rounded once when stored.  ds and alpha_s stay fp32.
template <int H, int CH, typename S>
__global__ void __launch_bounds__(256) mp_bwd_source_kernel(int64_t N, int D, const int32_t* __restrict__ rowptr_src,
                                                            const int32_t* __restrict__ csr_src_tgt,
                                                            const int32_t* __restrict__ csr_src_combo,
                                                            const S* __restrict__ qkm, const S* __restrict__ ke,
                                                            const S* __restrict__ me, const float* __restrict__ alpha_s,
                                                            const S* __restrict__ d_aggr, float* __restrict__ ds,
                                                            S* __restrict__ d_qkm) {
  const int lane = threadIdx.x & 31;
  const int64_t u = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (u >= N) return;
  const int d = D / H, ld = 3 * D;
  HeadMap4 hm[CH];
  bool valid[CH];
  typename Packed4<S>::type mxp[CH];  // Mx[u], widened at each use
  float4 dq[CH], dmx[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    valid[i] = 4 * c < D;
    hm[i] = head_map4(c, d);
    mxp[i] = valid[i] ? load_packed4(qkm + u * ld + 2 * D + 4 * c) : zero_packed4<S>();
    dq[i] = dmx[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int beg = rowptr_src[u], end = rowptr_src[u + 1];
  const float degf = (float)(end - beg), rdeg = 1.f / degf;
  float dot[H];
#pragma unroll
  for (int h = 0; h < H; ++h) dot[h] = 0.f;
  // pass A: da = outdeg * dAggr[tgt] . (Mx[u] + Me[c]) per head, sum_e a da, and dMx[u] += a' dAggr[tgt]
  for (int p = beg; p < end; ++p) {
    const int t = csr_src_tgt[p], cb = csr_src_combo[p];
    float as[H];  // a' of this edge
#pragma unroll
    for (int h = 0; h < H; ++h) as[h] = alpha_s[(int64_t)p * H + h];
    float part[H];
#pragma unroll
    for (int h = 0; h < H; ++h) part[h] = 0.f;
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      if (!valid[i]) continue;
      const int c = lane + 32 * i;
      const float4 g = load4(d_aggr + (int64_t)t * D + 4 * c);
      const float4 mt = load4(me + (int64_t)cb * D + 4 * c);
      const float4 mx = widen4(mxp[i], qkm);
      add_parts<H>(part, hm[i], g.x * (mx.x + mt.x), g.y * (mx.y + mt.y), g.z * (mx.z + mt.z), g.w * (mx.w + mt.w));
      dmx[i].x += pick<H>(as, hm[i].hid[0]) * g.x;
      dmx[i].y += pick<H>(as, hm[i].hid[1]) * g.y;
      dmx[i].z += pick<H>(as, hm[i].hid[2]) * g.z;
      dmx[i].w += pick<H>(as, hm[i].hid[3]) * g.w;
    }
    float mine = 0.f;
#pragma unroll
    for (int h = 0; h < H; ++h) {
      float s = part[h];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float da = s * degf;
      dot[h] += (as[h] * rdeg) * da;
      if (lane == h) mine = da;
    }
    if (lane < H) ds[(int64_t)p * H + lane] = mine;  // da for now
  }
  __syncwarp();
  // pass B: ds = a (da - dot), dQ[u] += ds (Kx[tgt] + Ke[c])
  for (int p = beg; p < end; ++p) {
    const int t = csr_src_tgt[p], cb = csr_src_combo[p];
    float dsv[H];
#pragma unroll
    for (int h = 0; h < H; ++h) dsv[h] = (alpha_s[(int64_t)p * H + h] * rdeg) * (ds[(int64_t)p * H + h] - dot[h]);
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      if (!valid[i]) continue;
      const int c = lane + 32 * i;
      const float4 kx = load4(qkm + (int64_t)t * ld + D + 4 * c);
      const float4 kt = load4(ke + (int64_t)cb * D + 4 * c);
      dq[i].x += pick<H>(dsv, hm[i].hid[0]) * (kx.x + kt.x);
      dq[i].y += pick<H>(dsv, hm[i].hid[1]) * (kx.y + kt.y);
      dq[i].z += pick<H>(dsv, hm[i].hid[2]) * (kx.z + kt.z);
      dq[i].w += pick<H>(dsv, hm[i].hid[3]) * (kx.w + kt.w);
    }
    __syncwarp();  // every lane has read da[p] before it is overwritten
    if (lane < H) {
      float mine = 0.f;
#pragma unroll
      for (int h = 0; h < H; ++h) mine = (lane == h) ? dsv[h] : mine;
      ds[(int64_t)p * H + lane] = mine;
    }
  }
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    if (!valid[i]) continue;
    const int c = lane + 32 * i;
    store4(d_qkm + u * ld + 4 * c, dq[i]);
    store4(d_qkm + u * ld + 2 * D + 4 * c, dmx[i]);
  }
}

template <int H, int CH, typename S>
__global__ void __launch_bounds__(256) mp_bwd_target_kernel(int64_t N, int D, const int32_t* __restrict__ rowptr_tgt,
                                                            const int32_t* __restrict__ csr_tgt_src,
                                                            const int32_t* __restrict__ csr_tgt_apos,
                                                            const S* __restrict__ qkm, const float* __restrict__ ds,
                                                            S* __restrict__ d_qkm) {
  const int lane = threadIdx.x & 31;
  const int64_t v = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (v >= N) return;
  const int d = D / H, ld = 3 * D;
  HeadMap4 hm[CH];
  bool valid[CH];
  float4 acc[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    valid[i] = 4 * c < D;
    hm[i] = head_map4(c, d);
    acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int beg = rowptr_tgt[v], end = rowptr_tgt[v + 1];
  for (int p = beg; p < end; ++p) {
    const int s = csr_tgt_src[p];
    const float* dp = ds + (int64_t)csr_tgt_apos[p] * H;
    float dsv[H];
#pragma unroll
    for (int h = 0; h < H; ++h) dsv[h] = dp[h];
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      if (!valid[i]) continue;
      const int c = lane + 32 * i;
      const float4 q = load4(qkm + (int64_t)s * ld + 4 * c);
      acc[i].x += pick<H>(dsv, hm[i].hid[0]) * q.x;
      acc[i].y += pick<H>(dsv, hm[i].hid[1]) * q.y;
      acc[i].z += pick<H>(dsv, hm[i].hid[2]) * q.z;
      acc[i].w += pick<H>(dsv, hm[i].hid[3]) * q.w;
    }
  }
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    if (!valid[i]) continue;
    store4(d_qkm + v * ld + D + 4 * (lane + 32 * i), acc[i]);
  }
}

constexpr int kTableRun = 64;  // edges per warp in combo order

__device__ __forceinline__ void atomic_add4(float* p, const float4& v) {
  atomicAdd(p, v.x); atomicAdd(p + 1, v.y); atomicAdd(p + 2, v.z); atomicAdd(p + 3, v.w);
}

// d_ke / d_me are fp32 for every S (the accumulators of a 16-bit call, rounded afterwards by round_rows_kernel).
// kDet: no atomics.  A segment (the positions of one combo inside the run) that holds the combo's whole range is stored into
// d_ke / d_me; one that continues past the run's start goes to slot 0 of the run, else (it continues past the run's end) to
// slot 1, except that a segment starting exactly at the run's start also uses slot 0.  Slot k of run w is the 2D floats
// slots[(2w + k) * 2D ...]: dKe's D columns, then dMe's.
template <int H, int CH, typename S, bool kDet>
__global__ void __launch_bounds__(256) mp_bwd_table_kernel(int64_t N, int D, const int32_t* __restrict__ rowptr_src,
                                                           const int32_t* __restrict__ combo_order,
                                                           const int32_t* __restrict__ csr_src_tgt,
                                                           const int32_t* __restrict__ csr_src_combo,
                                                           const int32_t* __restrict__ perm_src,
                                                           const int32_t* __restrict__ src, const S* __restrict__ qkm,
                                                           const float* __restrict__ alpha_s, const float* __restrict__ ds,
                                                           const S* __restrict__ d_aggr, float* __restrict__ d_ke,
                                                           float* __restrict__ d_me, float* __restrict__ slots) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t i0 = w * kTableRun;
  // the real E' of the batch: the grid covers E + N, which may be an edge capacity (qagnn_graph_prep_packed)
  const int64_t Ep = rowptr_src[N];
  if (i0 >= Ep) return;
  const int64_t i1 = min(i0 + (int64_t)kTableRun, Ep);
  const int d = D / H, ld = 3 * D;
  HeadMap4 hm[CH];
  bool valid[CH];
  float4 ak[CH], am[CH];
#pragma unroll
  for (int i = 0; i < CH; ++i) {
    const int c = lane + 32 * i;
    valid[i] = 4 * c < D;
    hm[i] = head_map4(c, d);
    ak[i] = am[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  // the segment [a, b) of combo cb
  auto flush = [&](int cb, int64_t a, int64_t b) {
    float *ok = d_ke + (int64_t)cb * D, *om = d_me + (int64_t)cb * D;
    if constexpr (kDet) {
      const bool open_lo = a == i0 && i0 > 0 && csr_src_combo[combo_order[i0 - 1]] == cb;
      const bool open_hi = b == i1 && i1 < Ep && csr_src_combo[combo_order[i1]] == cb;
      if (open_lo || open_hi) {
        ok = slots + (2 * w + (a == i0 ? 0 : 1)) * (int64_t)(2 * D);
        om = ok + D;
      }
    }
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      if (!valid[i]) continue;
      const int c = lane + 32 * i;
      if constexpr (kDet) {
        store4(ok + 4 * c, ak[i]);
        store4(om + 4 * c, am[i]);
      } else {
        atomic_add4(ok + 4 * c, ak[i]);
        atomic_add4(om + 4 * c, am[i]);
      }
      ak[i] = am[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  int cur = -1;
  int64_t seg = i0;
  for (int64_t i = i0; i < i1; ++i) {
    const int p = combo_order[i];  // by-source position of the i-th edge in combo order
    const int cb = csr_src_combo[p];
    if (cb != cur) {
      if (cur >= 0) flush(cur, seg, i);
      cur = cb;
      seg = i;
    }
    const int t = csr_src_tgt[p], s = src[perm_src[p]];
    float dsv[H], as[H];
#pragma unroll
    for (int h = 0; h < H; ++h) {
      dsv[h] = ds[(int64_t)p * H + h];
      as[h] = alpha_s[(int64_t)p * H + h];
    }
#pragma unroll
    for (int k = 0; k < CH; ++k) {
      if (!valid[k]) continue;
      const int c = lane + 32 * k;
      const float4 q = load4(qkm + (int64_t)s * ld + 4 * c);
      const float4 g = load4(d_aggr + (int64_t)t * D + 4 * c);
      ak[k].x += pick<H>(dsv, hm[k].hid[0]) * q.x; am[k].x += pick<H>(as, hm[k].hid[0]) * g.x;
      ak[k].y += pick<H>(dsv, hm[k].hid[1]) * q.y; am[k].y += pick<H>(as, hm[k].hid[1]) * g.y;
      ak[k].z += pick<H>(dsv, hm[k].hid[2]) * q.z; am[k].z += pick<H>(as, hm[k].hid[2]) * g.z;
      ak[k].w += pick<H>(dsv, hm[k].hid[3]) * q.w; am[k].w += pick<H>(as, hm[k].hid[3]) * g.w;
    }
  }
  if (cur >= 0) flush(cur, seg, i1);
}

// off[c] = sum of combo_count[0, c) (int32: positions are int32), one block of 1024 threads, each scanning a contiguous group
__global__ void __launch_bounds__(1024) combo_offsets_kernel(int C, const int64_t* __restrict__ combo_count,
                                                             int32_t* __restrict__ off) {
  const int per = (C + 1023) / 1024, c0 = threadIdx.x * per, c1 = min(c0 + per, C);
  int local = 0;
  for (int c = c0; c < c1; ++c) local += (int)combo_count[c];
  int total;
  int run = block_exclusive_scan_1024(local, &total);
  for (int c = c0; c < c1; ++c) {
    off[c] = run;
    run += (int)combo_count[c];
  }
}

constexpr int kCombineWarps = 8;

// Rows of the combos the deterministic table kernel did not store.  Block (x, c): columns [32x, 32x + 32) of the 2D columns
// [dKe | dMe] of combo c.  A combo with range [o, o + n), n > 0, spans runs r0 = o / 64 ... r1 = (o + n - 1) / 64; when
// r1 > r0 its row is the sum of one slot per run: slot 1 of r0 when o is not r0's start, slot 0 otherwise.  Warp k adds the
// slots of runs r0 + k, r0 + k + 8, ... in ascending order, then warp 0 adds the 8 partial sums in warp order: the order
// depends on n and o alone.  A combo without edges gets a zero row.
__global__ void __launch_bounds__(32 * kCombineWarps) mp_bwd_table_combine_kernel(int D, const int64_t* __restrict__ combo_count,
                                                                                  const int32_t* __restrict__ off,
                                                                                  const float* __restrict__ slots,
                                                                                  float* __restrict__ d_ke,
                                                                                  float* __restrict__ d_me) {
  __shared__ float part[kCombineWarps][32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int c = blockIdx.y, j = blockIdx.x * 32 + lane;
  const int64_t n = combo_count[c];
  float* out = j < D ? d_ke + (int64_t)c * D + j : d_me + (int64_t)c * D + (j - D);
  if (n == 0) {
    if (wid == 0 && j < 2 * D) *out = 0.f;
    return;
  }
  const int64_t o = off[c], r0 = o / kTableRun, r1 = (o + n - 1) / kTableRun;
  if (r1 == r0) return;  // stored by the table kernel
  float acc = 0.f;
  if (j < 2 * D) {
    const int64_t ld = 2 * (int64_t)D;
#pragma unroll 4
    for (int64_t r = r0 + wid; r <= r1; r += kCombineWarps)
      acc += slots[(2 * r + (r == r0 && o != r0 * kTableRun ? 1 : 0)) * ld + j];
  }
  part[wid][lane] = acc;
  __syncthreads();
  if (wid == 0 && j < 2 * D) {
    float s = part[0][lane];
#pragma unroll
    for (int k = 1; k < kCombineWarps; ++k) s += part[k][lane];
    *out = s;
  }
}

// out[i] = acc[i] rounded to nearest even, 4 elements per thread (n % 4 == 0)
template <typename S>
__global__ void __launch_bounds__(256) round_rows_kernel(int64_t n4, const float* __restrict__ acc, S* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
    store4(out + 4 * i, load4(acc + 4 * i));
}

// The deterministic path's inputs (combo_count == nullptr: the atomic path).  off [C] int32, slots [2 * runs * 2D] floats.
struct DetTable {
  const int64_t* combo_count;
  int32_t* off;
  float* slots;
};

// d_ke / d_me: fp32 outputs (S = float), or fp32 accumulators that are rounded into the S outputs ke_out / me_out
template <int H, int CH, typename S>
int32_t launch_bwd_hc(const qagnn_shape& s, const int32_t* base, const qagnn_prep_layout& pl, const int32_t* combo_order,
                      const S* qkm, const S* ke, const S* me, const float* alpha_s, const S* d_aggr,
                      float* ds, S* d_qkm, float* d_ke, float* d_me, S* ke_out, S* me_out, const DetTable& det,
                      cudaStream_t st) {
  auto I = [&](size_t off) { return (const int32_t*)((const char*)base + off); };
  const int block = 256;
  const unsigned grid = (unsigned)((s.N * 32 + block - 1) / block);
  const int64_t Ep = s.N + s.E;
  const int C = s.R * s.T * s.T + s.T;
  if (det.combo_count) {
    combo_offsets_kernel<<<1, 1024, 0, st>>>(C, det.combo_count, det.off);
    QAGNN_CHECK_LAUNCH();
  } else {
    QAGNN_CHECK_CUDA(cudaMemsetAsync(d_ke, 0, (size_t)C * s.D * sizeof(float), st));
    QAGNN_CHECK_CUDA(cudaMemsetAsync(d_me, 0, (size_t)C * s.D * sizeof(float), st));
  }
  mp_bwd_source_kernel<H, CH, S><<<grid, block, 0, st>>>(s.N, s.D, I(pl.rowptr_src), I(pl.csr_src_tgt), I(pl.csr_src_combo), qkm,
                                                      ke, me, alpha_s, d_aggr, ds, d_qkm);
  QAGNN_CHECK_LAUNCH();
  mp_bwd_target_kernel<H, CH, S><<<grid, block, 0, st>>>(s.N, s.D, I(pl.rowptr_tgt), I(pl.csr_tgt_src), I(pl.csr_tgt_apos), qkm, ds,
                                                      d_qkm);
  QAGNN_CHECK_LAUNCH();
  const int64_t runs = (Ep + kTableRun - 1) / kTableRun;
  const unsigned tgrid = (unsigned)((runs * 32 + block - 1) / block);
  if (det.combo_count) {
    mp_bwd_table_kernel<H, CH, S, true><<<tgrid, block, 0, st>>>(
        s.N, s.D, I(pl.rowptr_src), combo_order, I(pl.csr_src_tgt), I(pl.csr_src_combo), I(pl.perm_src), I(pl.src), qkm, alpha_s, ds,
        d_aggr, d_ke, d_me, det.slots);
    QAGNN_CHECK_LAUNCH();
    mp_bwd_table_combine_kernel<<<dim3((unsigned)((2 * s.D + 31) / 32), (unsigned)C), 32 * kCombineWarps, 0, st>>>(
        s.D, det.combo_count, det.off, det.slots, d_ke, d_me);
    QAGNN_CHECK_LAUNCH();
  } else {
    mp_bwd_table_kernel<H, CH, S, false><<<tgrid, block, 0, st>>>(
        s.N, s.D, I(pl.rowptr_src), combo_order, I(pl.csr_src_tgt), I(pl.csr_src_combo), I(pl.perm_src), I(pl.src), qkm, alpha_s, ds,
        d_aggr, d_ke, d_me, nullptr);
    QAGNN_CHECK_LAUNCH();
  }
  if constexpr (!std::is_same<S, float>::value) {
    const int64_t n4 = (int64_t)C * s.D / 4;
    const int64_t blocks = (n4 + block - 1) / block;
    const unsigned g = (unsigned)(blocks < 8 * kNumSMs ? blocks : 8 * kNumSMs);
    round_rows_kernel<S><<<g, block, 0, st>>>(n4, d_ke, ke_out);
    QAGNN_CHECK_LAUNCH();
    round_rows_kernel<S><<<g, block, 0, st>>>(n4, d_me, me_out);
    QAGNN_CHECK_LAUNCH();
  }
  return QAGNN_OK;
}

template <int H, typename S>
int32_t launch_bwd_h(const qagnn_shape& s, const int32_t* base, const qagnn_prep_layout& pl, const int32_t* combo_order,
                     const S* qkm, const S* ke, const S* me, const float* alpha_s, const S* d_aggr, float* ds,
                     S* d_qkm, float* d_ke, float* d_me, S* ke_out, S* me_out, const DetTable& det, cudaStream_t st) {
  const int ch = (s.D + 127) / 128;
#define QAGNN_BWD_ARGS s, base, pl, combo_order, qkm, ke, me, alpha_s, d_aggr, ds, d_qkm, d_ke, d_me, ke_out, me_out, det, st
  if (ch <= 1) return launch_bwd_hc<H, 1, S>(QAGNN_BWD_ARGS);
  if (ch <= 2) return launch_bwd_hc<H, 2, S>(QAGNN_BWD_ARGS);
  if (ch <= 4) return launch_bwd_hc<H, 4, S>(QAGNN_BWD_ARGS);
  if (ch <= 8) return launch_bwd_hc<H, 8, S>(QAGNN_BWD_ARGS);
#undef QAGNN_BWD_ARGS
  return QAGNN_ERR_UNSUPPORTED;
}

template <typename S>
int32_t launch_bwd(const qagnn_shape& s, const int32_t* prep_base, const qagnn_prep_layout& pl, const int32_t* combo_order,
                   const S* qkm, const S* ke, const S* me, const float* alpha_s, const S* d_aggr, float* ds, S* d_qkm,
                   float* d_ke, float* d_me, S* ke_out, S* me_out, const DetTable& det, cudaStream_t st) {
  if (s.D % 4 != 0 || s.D > 1024) return QAGNN_ERR_UNSUPPORTED;
#define QAGNN_BWD_ARGS s, prep_base, pl, combo_order, qkm, ke, me, alpha_s, d_aggr, ds, d_qkm, d_ke, d_me, ke_out, me_out, det, st
  switch (s.H) {
    case 1: return launch_bwd_h<1>(QAGNN_BWD_ARGS);
    case 2: return launch_bwd_h<2>(QAGNN_BWD_ARGS);
    case 4: return launch_bwd_h<4>(QAGNN_BWD_ARGS);
    case 8: return launch_bwd_h<8>(QAGNN_BWD_ARGS);
    case 16: return launch_bwd_h<16>(QAGNN_BWD_ARGS);
    default: return QAGNN_ERR_UNSUPPORTED;
  }
#undef QAGNN_BWD_ARGS
}

// a 16-bit call accumulates d_ke / d_me in fp32 after the [E+N, H] floats of ds in the scratch, then rounds them once
template <typename S>
int32_t launch_bwd_16(const qagnn_shape& s, const int32_t* prep_base, const qagnn_prep_layout& pl, const int32_t* combo_order,
                      const void* qkm, const void* ke, const void* me, const float* alpha_s, const void* d_aggr, float* scratch,
                      void* d_qkm, void* d_ke, void* d_me, const DetTable& det, cudaStream_t st) {
  const size_t C = (size_t)s.R * s.T * s.T + s.T;
  float* acc = scratch + mp_core_ds_floats(s);
  return launch_bwd(s, prep_base, pl, combo_order, (const S*)qkm, (const S*)ke, (const S*)me, alpha_s, (const S*)d_aggr, scratch,
                    (S*)d_qkm, acc, acc + C * s.D, (S*)d_ke, (S*)d_me, det, st);
}

int32_t launch_bwd_typed(const qagnn_shape& s, const int32_t* prep_base, const qagnn_prep_layout& pl, int32_t dtype,
                         const int32_t* combo_order, const void* qkm, const void* ke, const void* me, const float* alpha_s,
                         const void* d_aggr, float* scratch, void* d_qkm, void* d_ke, void* d_me, const DetTable& det,
                         cudaStream_t st) {
  switch (dtype) {
    case QAGNN_DTYPE_F32:
      return launch_bwd<float>(s, prep_base, pl, combo_order, (const float*)qkm, (const float*)ke, (const float*)me, alpha_s,
                               (const float*)d_aggr, scratch, (float*)d_qkm, (float*)d_ke, (float*)d_me, nullptr, nullptr, det, st);
    case QAGNN_DTYPE_F16:
      return launch_bwd_16<__half>(s, prep_base, pl, combo_order, qkm, ke, me, alpha_s, d_aggr, scratch, d_qkm, d_ke, d_me, det,
                                   st);
    case QAGNN_DTYPE_BF16:
      return launch_bwd_16<__nv_bfloat16>(s, prep_base, pl, combo_order, qkm, ke, me, alpha_s, d_aggr, scratch, d_qkm, d_ke,
                                          d_me, det, st);
    default: return QAGNN_ERR_INVALID_ARGUMENT;
  }
}

// floats of the deterministic path's int32 combo offsets, after ds and the 16-bit accumulators
size_t det_off_floats(const qagnn_shape& s) { return align_up((size_t)s.R * s.T * s.T + s.T, kAlign / sizeof(float)); }

}  // namespace

size_t mp_core_ds_floats(const qagnn_shape& s) { return align_up((size_t)(s.N + s.E) * s.H, kAlign / sizeof(float)); }

size_t mp_core_scratch_bytes(const qagnn_shape& s, int32_t dtype) {
  const size_t C = (size_t)s.R * s.T * s.T + s.T;
  return sizeof(float) * (mp_core_ds_floats(s) + (dtype == QAGNN_DTYPE_F32 ? 0 : 2 * C * s.D));
}

int32_t launch_message_passing_backward_typed(const qagnn_shape& s, const int32_t* prep_base, const qagnn_prep_layout& pl,
                                              int32_t dtype, const int32_t* combo_order, const void* qkm, const void* ke,
                                              const void* me, const float* alpha_s, const void* d_aggr, float* scratch,
                                              void* d_qkm, void* d_ke, void* d_me, cudaStream_t st) {
  return launch_bwd_typed(s, prep_base, pl, dtype, combo_order, qkm, ke, me, alpha_s, d_aggr, scratch, d_qkm, d_ke, d_me,
                          DetTable{}, st);
}

size_t mp_core_det_scratch_bytes(const qagnn_shape& s, int32_t dtype) {
  const size_t runs = ((size_t)(s.N + s.E) + kTableRun - 1) / kTableRun;
  return mp_core_scratch_bytes(s, dtype) + sizeof(float) * (det_off_floats(s) + 2 * runs * 2 * (size_t)s.D);
}

int32_t launch_message_passing_backward_det(const qagnn_shape& s, const int32_t* prep_base, const qagnn_prep_layout& pl,
                                            int32_t dtype, const int32_t* combo_order, const int64_t* combo_count,
                                            const void* qkm, const void* ke, const void* me, const float* alpha_s,
                                            const void* d_aggr, float* scratch, void* d_qkm, void* d_ke, void* d_me,
                                            cudaStream_t st) {
  float* off = scratch + mp_core_scratch_bytes(s, dtype) / sizeof(float);
  const DetTable det{combo_count, (int32_t*)off, off + det_off_floats(s)};
  return launch_bwd_typed(s, prep_base, pl, dtype, combo_order, qkm, ke, me, alpha_s, d_aggr, scratch, d_qkm, d_ke, d_me, det,
                          st);
}

}  // namespace qagnn
