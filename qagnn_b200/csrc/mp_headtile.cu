// Shared-memory-tiled message passing for batches of small sub-graphs (the QA-GNN case: <= 200
// nodes per (question, choice) graph).  One launch per GATConvE layer does
//     logits -> per-SOURCE softmax -> out-degree rescale -> per-TARGET weighted sum
// (modeling/modeling_qagnn.py:442,455-484) with every gathered row served from shared memory.
//
// Why this shape (profiles/r1_microbench.txt, profiles/r1_mp_stall_breakdown.md): each edge needs four row
// gathers (Kx[tgt], Ke[combo], Mx[src], Me[combo]); served from L2 they cap at ~11 G rows/s, so the
// per-head slice of the edge tables (C x d floats, 127 KB at C=612, d=50) has to live in shared
// memory next to the node tile of the current graph.  Hence:
//   * grid = H x floor(#SM / H) persistent CTAs; CTA (h, slot) owns head h of graphs slot, slot+S, ...
//   * phase 1: Ke_h resident, Kx_h tiles streamed through a 2-deep TMA (cp.async.bulk) ring ->
//     logits, softmax per source node; the rescaled weight a'[e] is stored next to the (source row, table row)
//     offsets of its edge at the edge's BY-TARGET position (8 bytes per edge and head, L2-resident);
//   * phase 2: Me_h swapped in, Mx_h tiles streamed the same way -> aggr[:, h*d:(h+1)*d];
//   * ONE loader thread drives the TMA ring (tiles and the two tables); nothing else is staged: the consumers
//     fetch their per-node / per-edge words from L2 one and two work items ahead of use (registers), so the
//     loops never wait on a dependent global load and the 227 KB hold table + 2 tiles for any edge count;
//   * work item = 4 nodes of similar degree ("quad", degree-sorted by graph prep, one packed 8-byte record per
//     node); the consumer warps of a CTA pull quads from a shared-memory counter, heaviest first, across the two
//     graphs whose tiles are resident — no warp waits for a slower one at a graph boundary (round 1 lost 13 % of
//     its time there and 16 % in the od->rowptr->degree set-up chain, profiles/r1_mp_stall_breakdown.md);
//   * consumers: 8 lanes per node (quarter-warp), each lane owning float4 chunks l, l+8 of the padded
//     head row: a quarter-warp LDS.128 covers 128 contiguous bytes = one conflict-free wavefront;
//     fp32 math on float2 pairs; the 8 lane-partials of 8 edges are reduced by a 7-shuffle
//     transposing tree (lane j ends up with the logit of edge j); the softmax runs lane-parallel.
// a' is written and read back by ordinary (generic-proxy) accesses of the same CTA, ordered by a CTA fence and
// the phase-switch mbarrier: no async-proxy fence per graph (5 % in round 1).
// Node rows come from the head-major padded projection layout [3][H][N][DP] written by the
// projection GEMM, so a tile is one contiguous n*DP*4-byte bulk copy.
// No atomics touch the data path and every summation runs in edge-id order: bit-reproducible.
#include <cuda_bf16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace qagnn {

namespace {

struct HeadTileParams {
  int64_t N, Eps;  // Eps = per-head stride of score / alpha2 (E' rounded up to 4)
  int n, G, H, D, d, DP, C, S, W, nquads;
  uint32_t nq_magic;  // floor(2^32 / nquads) + 1: item / nquads == __umulhi(item, nq_magic) for every item a CTA can see
  const int32_t *rowptr_src, *rowptr_tgt, *pk_src, *tpos, *perm_src;
  const uint2 *ninfo_src, *ninfo_tgt;
  const float *qkmh, *keh, *meh;
  float* score;   // [H][Eps] logits past the 8th edge of hub nodes (by-source order)
  uint2* alpha2;  // [H][Eps] {tile byte offset of the source row << 16 | table float4 offset, a'} in by-target order
  float *aggr, *alpha_out;
  void *aggr_hi, *aggr_lo;  // optional split-bf16 planes of aggr [N, D] (A operand of the node-MLP GEMM)
  const int64_t* node_ptr;  // ragged batches: first row of every sub-graph [B + 1]; G is then the most segments
  int B;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_g2s_chunked(char* dst, const char* src, uint32_t bytes, uint64_t* bar) {
  mbar_expect_tx(bar, bytes);
  const uint32_t kChunk = 32768;
  for (uint32_t o = 0; o < bytes; o += kChunk) bulk_g2s(dst + o, src + o, min(kChunk, bytes - o), bar);
}

// 16-byte shared-memory load from a 32-bit shared address (pre-scaled row offsets are added to it)
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float2 lo2(const float4& v) { return make_float2(v.x, v.y); }
__device__ __forceinline__ float2 hi2(const float4& v) { return make_float2(v.z, v.w); }
// element-wise fp32x2 add / fused multiply-add, each lane rounded once (the same bits as a packed FP32x2 unit gives)
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// shared-memory carve-up (bytes from the start of dynamic smem)
struct SmemMap {
  uint32_t tab, tile0, tile_bytes, bars, ctr, total;
};
__host__ __device__ inline SmemMap make_smem_map(int C, int DP, int n) {
  SmemMap m;
  m.tab = 0;
  m.tile0 = (uint32_t)C * DP * 4;
  m.tile_bytes = (uint32_t)n * DP * 4;
  m.bars = m.tile0 + 2 * m.tile_bytes;  // full[2], empty[2], tabbar, ph1done
  m.ctr = m.bars + 6 * 8;               // work-item counters of the two phases
  m.total = m.ctr + 16;
  return m;
}

// Consumer warps per CTA: 24 at <= 80 registers, or 31 (a full 1024-thread CTA) at <= 64.
constexpr int kWarpsWide = 31, kWarpsNarrow = 24;

// CPL: float4 chunks per lane (1: DP <= 32, 2: DP <= 64); WMAX: consumer-warp capacity.  RAGGED: graph g is segment g of a
// ragged batch (ragged_segment in common.cuh: rows [node_ptr[g], node_ptr[g+1]) for g < B, then the tail rows in segments of n)
// and its tile holds only its own rows; quads past a graph's row count are idle work items.
template <int CPL, int WMAX, bool RAGGED = false>
__global__ void __launch_bounds__((WMAX + 1) * 32, 1) mp_headtile_kernel(const HeadTileParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int NCH = p.DP / 4;
  const SmemMap sm = make_smem_map(p.C, p.DP, p.n);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + sm.bars);
  uint64_t* full = bars;         // [2]  tile landed (one expect_tx arrival)
  uint64_t* empty = bars + 2;    // [2]  one arrival per finished work item of the graph in that buffer
  uint64_t* tabbar = bars + 4;   // [1]  edge table landed
  uint64_t* ph1done = bars + 5;  // [1]  every consumer warp has left phase 1
  int* ctr = reinterpret_cast<int*>(smem_raw + sm.ctr);

  const int h = blockIdx.x % p.H;
  const int slot = blockIdx.x / p.H;
  const int G = RAGGED ? (int)ragged_segments(p.node_ptr, p.B, p.n, p.N) : p.G;
  const int Gc = slot < G ? (G - slot + p.S - 1) / p.S : 0;  // graphs slot, slot+S, ...
  if (Gc == 0) return;
  const int nq = p.nquads, total = Gc * nq;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    mbar_init(&empty[0], nq);
    mbar_init(&empty[1], nq);
    mbar_init(tabbar, 1);
    mbar_init(ph1done, p.W);
    ctr[0] = 0;
    ctr[1] = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const size_t head_rows = (size_t)p.N * p.DP;  // floats per [N, DP] slab
  const float* Qh = p.qkmh + (size_t)(0 * p.H + h) * head_rows;
  const float* Kh = p.qkmh + (size_t)(1 * p.H + h) * head_rows;
  const float* Mh = p.qkmh + (size_t)(2 * p.H + h) * head_rows;
  const size_t hE = (size_t)h * p.Eps;

  if (warp == p.W) {
    // ===== loader: ONE thread drives the TMA ring (edge tables + node tiles, cp.async.bulk) =====
    if (lane != 0) return;
    bulk_g2s_chunked((char*)(smem_raw + sm.tab), (const char*)(p.keh + (size_t)h * p.C * p.DP), sm.tile0, tabbar);
    for (int t = 0; t < 2 * Gc; ++t) {
      const int b = t & 1;
      const bool ph2 = t >= Gc;
      if (t == Gc) {
        // phase switch: every consumer warp has arrived, so Ke_h and both tile buffers are free
        mbar_wait(ph1done, 0);
        bulk_g2s_chunked((char*)(smem_raw + sm.tab), (const char*)(p.meh + (size_t)h * p.C * p.DP), sm.tile0, tabbar);
      }
      if (t >= 2) mbar_wait(&empty[b], ((t >> 1) - 1) & 1);
      const int g = slot + (ph2 ? t - Gc : t) * p.S;
      if (RAGGED) {
        int64_t v0;
        int ng;
        ragged_segment(p.node_ptr, p.B, p.n, p.N, g, v0, ng);
        bulk_g2s_chunked((char*)(smem_raw + sm.tile0 + b * sm.tile_bytes), (const char*)((ph2 ? Mh : Kh) + (size_t)v0 * p.DP),
                         (uint32_t)ng * p.DP * 4, &full[b]);
      } else {
        bulk_g2s_chunked((char*)(smem_raw + sm.tile0 + b * sm.tile_bytes),
                         (const char*)((ph2 ? Mh : Kh) + (size_t)g * p.n * p.DP), sm.tile_bytes, &full[b]);
      }
    }
    return;
  }
  if (warp > p.W) return;

  // ========================= consumer warps: 4 nodes per warp, 8 lanes per node =========================
  const int l8 = lane & 7, qbase = lane & 24, qi = lane >> 3;
  int chunk[CPL];
  bool cvalid[CPL];
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    cvalid[k] = (l8 + 8 * k) < NCH;
    // idle lanes (chunk slot past the row) re-read an in-row chunk against q = 0, so the product is 0 * finite.
    // It must stay INSIDE the row: the bytes after a row's last chunk belong to the next row / the next smem region
    // and 0 * NaN would poison the shuffled sum (found with compute-sanitizer, whose smem fill is not finite).
    chunk[k] = cvalid[k] ? l8 + 8 * k : l8 % NCH;
  }
  uint32_t tabu[CPL];  // shared address of the table + this lane's chunk: a row is one add away
#pragma unroll
  for (int k = 0; k < CPL; ++k) tabu[k] = smem_u32(smem_raw + sm.tab) + 16u * (uint32_t)chunk[k];
  const bool b4 = (l8 & 4) != 0, b2 = (l8 & 2) != 0, b1 = (l8 & 1) != 0;
  const uint32_t nch = (uint32_t)NCH, magic = p.nq_magic;
  const uint32_t ctr_u32 = smem_u32(ctr);

  // Offsets word of an edge: low 16 bits = tile-row offset in 16-byte units (< 2^15), high 16 bits = table-row offset in
  // 2-byte units.  A row address is then base + ((w & 0xffff) << 4) resp. base + (w >> 15)  (bit 15 is always 0).
  auto offsets_word = [&](uint32_t tile_row, uint32_t table_row) { return (tile_row * nch) | ((table_row * nch * 8u) << 16); };
  auto tile_addr = [&](uint32_t base, uint32_t w) { return base + ((w & 0xffffu) << 4); };
  auto table_addr = [&](uint32_t base, uint32_t w) { return base + (w >> 15); };

  // next work item of this phase: one shared-memory atomic per warp.  (A static stride — warp w takes items w, w+W, ... —
  // needs no atomic but measured 122 vs 115 us/layer at cfg2: the warps drift apart inside a tile, profiles/r2_mp_tuning.md)
  auto grab = [&](uint32_t counter) {
    int v = 0;
    if (lane == 0) asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(v) : "r"(counter) : "memory");
    return __shfl_sync(0xffffffffu, v, 0);
  };
  auto item_graph = [&](int it) { return (int)__umulhi((uint32_t)it, magic); };  // it / nq
  // first row and row count of this CTA's t-th graph (ragged batches only)
  auto segment = [&](int t, int& ng) {
    int64_t v0;
    ragged_segment(p.node_ptr, p.B, p.n, p.N, slot + (int64_t)t * p.S, v0, ng);
    return v0;
  };
  // packed node record of work item `it` for this lane's node: {local id | degree << 16, CSR begin}; degree 0 = idle
  auto load_ninfo = [&](const uint2* ninfo, int it) {
    uint2 r = make_uint2(0u, 0u);
    if (it < total) {
      const int t = item_graph(it);
      const int si = (it - t * nq) * 4 + qi;
      if (RAGGED) {
        int ng;
        const int64_t v0 = segment(t, ng);
        if (si < ng) r = __ldg(ninfo + v0 + si);
      } else {
        if (si < p.n) r = __ldg(ninfo + (uint32_t)((slot + t * p.S) * p.n + si));
      }
    }
    return r;
  };

  // ---------------------------------- phase 1: attention weights ----------------------------------
  {
    // software pipeline over work items: it2 = record requested, it1 = Q rows + first 8 edge words requested
    int it1 = grab(ctr_u32);
    uint2 ni1 = load_ninfo(p.ninfo_src, it1);
    int it2 = grab(ctr_u32);
    uint2 ni2 = load_ninfo(p.ninfo_src, it2);
    float4 q1[CPL];
    int pk1 = 0, tp1 = 0;
    auto issue = [&](int it, const uint2& ni, float4 (&q)[CPL], int& pk, int& tp) {
      const int deg = (int)(ni.x >> 16);
      pk = 0; tp = 0;
#pragma unroll
      for (int k = 0; k < CPL; ++k) q[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (deg > 0) {  // deg > 0 implies it < total and a valid node
        uint32_t v;
        if (RAGGED) {
          int ng;
          v = (uint32_t)segment(item_graph(it), ng) + (ni.x & 0xffffu);
        } else {
          v = (uint32_t)((slot + item_graph(it) * p.S) * p.n) + (ni.x & 0xffffu);
        }
        const float4* qrow = reinterpret_cast<const float4*>(Qh) + (size_t)v * nch;
#pragma unroll
        for (int k = 0; k < CPL; ++k)
          if (cvalid[k]) q[k] = __ldg(qrow + chunk[k]);
        if (l8 < deg) {
          pk = __ldg(p.pk_src + ni.y + l8);
          tp = __ldg(p.tpos + ni.y + l8);
        }
      }
    };
    issue(it1, ni1, q1, pk1, tp1);
    mbar_wait(tabbar, 0);
    int cur_t = -1;
    while (it1 < total) {
      const int it0 = it1;
      const uint2 ni0 = ni1;
      float4 qc[CPL];
#pragma unroll
      for (int k = 0; k < CPL; ++k) qc[k] = q1[k];
      int pk0 = pk1, tp0 = tp1;
      it1 = it2; ni1 = ni2;
      issue(it1, ni1, q1, pk1, tp1);
      it2 = grab(ctr_u32);
      ni2 = load_ninfo(p.ninfo_src, it2);

      const int t = item_graph(it0);
      const int b = t & 1;
      if (t != cur_t) {
        mbar_wait(&full[b], (t >> 1) & 1);
        cur_t = t;
      }
      const uint32_t vl = ni0.x & 0xffffu;
      const int beg = (int)ni0.y;
      int deg = (int)(ni0.x >> 16);
      if (deg == 0xffff) {  // saturated record: read the true out-degree
        int ng;
        const int64_t v = (RAGGED ? segment(t, ng) : (int64_t)(slot + t * p.S) * p.n) + vl;
        deg = p.rowptr_src[v + 1] - p.rowptr_src[v];
      }
      const int maxdeg = __reduce_max_sync(0xffffffffu, deg);
      uint32_t ktc[CPL];  // shared address of tile base + this lane's chunk: a row is one add away
#pragma unroll
      for (int k = 0; k < CPL; ++k) ktc[k] = smem_u32(smem_raw + sm.tile0 + b * sm.tile_bytes) + 16u * (uint32_t)chunk[k];
      const size_t sbase = hE + (size_t)beg;
      float skeep = -INFINITY;  // lane j keeps the logit of edge j (j < 8)
      uint32_t pko_first = 0;   // offsets word of edge l8 (first block), kept for the a' record below
      for (int i0 = 0; i0 < maxdeg; i0 += 8) {
        if (i0 > 0) pk0 = (i0 + l8 < deg) ? __ldg(p.pk_src + beg + i0 + l8) : 0;  // hub nodes only
        uint32_t pko = 0;
        if (i0 + l8 < deg) pko = offsets_word((uint32_t)pk0 >> 16, (uint32_t)pk0 & 0xffffu);
        if (i0 == 0) pko_first = pko;
        const int lim = min(8, maxdeg - i0);
        // the quarter-warp's 8 offsets words, broadcast up front so that no row load waits on a shuffle
        uint32_t w[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) w[j] = __shfl_sync(0xffffffffu, pko, qbase + j);
#pragma unroll
        for (int j = 4; j < 8; ++j) w[j] = 0u;
        if (lim > 4) {  // warp-uniform
#pragma unroll
          for (int j = 4; j < 8; ++j) w[j] = __shfl_sync(0xffffffffu, pko, qbase + j);
        }
        float v[8];  // this lane's partial dot products of the block's 8 edges
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
        // (quarter-warps past their node's degree read row 0 against a discarded result; predicating these loads
        //  off saves shared-memory wavefronts but cost 143 -> 177 us in issue slots in round 1: measured, reverted)
        auto edge1 = [&](uint32_t w0) {
          float2 a0 = make_float2(0.f, 0.f);
#pragma unroll
          for (int k = 0; k < CPL; ++k) {
            const float4 x0 = lds128(tile_addr(ktc[k], w0)), y0 = lds128(table_addr(tabu[k], w0));
            a0 = ffma2(fadd2(lo2(x0), lo2(y0)), lo2(qc[k]), a0);
            a0 = ffma2(fadd2(hi2(x0), hi2(y0)), hi2(qc[k]), a0);
          }
          return a0.x + a0.y;
        };
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          if (j + 1 < lim) {  // warp-uniform
            const uint32_t w0 = w[j], w1 = w[j + 1];
            float2 a0 = make_float2(0.f, 0.f), a1 = make_float2(0.f, 0.f);
#pragma unroll
            for (int k = 0; k < CPL; ++k) {
              const float4 x0 = lds128(tile_addr(ktc[k], w0)), y0 = lds128(table_addr(tabu[k], w0));
              const float4 x1 = lds128(tile_addr(ktc[k], w1)), y1 = lds128(table_addr(tabu[k], w1));
              a0 = ffma2(fadd2(lo2(x0), lo2(y0)), lo2(qc[k]), a0);
              a0 = ffma2(fadd2(hi2(x0), hi2(y0)), hi2(qc[k]), a0);
              a1 = ffma2(fadd2(lo2(x1), lo2(y1)), lo2(qc[k]), a1);
              a1 = ffma2(fadd2(hi2(x1), hi2(y1)), hi2(qc[k]), a1);
            }
            v[j] = a0.x + a0.y;
            v[j + 1] = a1.x + a1.y;
          } else if (j < lim) {  // odd tail: one edge
            v[j] = edge1(w[j]);
          }
        }
        // transposing reduction over the 8 lanes of the node: after the three stages lane j holds
        // ((v_j[l] + v_j[l^4]) + (v_j[l^2] + v_j[l^6])) + (...[l^1]...), l = j — the butterfly's tree at lane j
        float r4[4], r2[2];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float keep = b4 ? v[i + 4] : v[i], send = b4 ? v[i] : v[i + 4];
          r4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float keep = b2 ? r4[i + 2] : r4[i], send = b2 ? r4[i] : r4[i + 2];
          r2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
        }
        const float keep = b1 ? r2[1] : r2[0], send = b1 ? r2[0] : r2[1];
        const float sj = keep + __shfl_xor_sync(0xffffffffu, send, 1);
        if (i0 == 0) skeep = sj;
        else if (i0 + l8 < deg) p.score[sbase + i0 + l8] = sj;  // hub nodes: logits past the 8th edge
      }
      // softmax over this node's out-edges, lane-parallel (lane j <-> edge j, j + 8, ...)
      const bool hub = maxdeg > 8;  // warp-uniform; logits beyond the 8th edge live in the L2 scratch
      if (hub) __syncwarp();
      float m = (l8 < deg) ? skeep : -INFINITY;
      if (hub)
        for (int j = 8 + l8; j < deg; j += 8) m = fmaxf(m, __ldcg(p.score + sbase + j));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      const float ex0 = (l8 < deg) ? __expf(skeep - m) : 0.f;
      float ssum = ex0;
      if (hub)
        for (int j = 8 + l8; j < deg; j += 8) ssum += __expf(__ldcg(p.score + sbase + j) - m);
      ssum += __shfl_xor_sync(0xffffffffu, ssum, 4);
      ssum += __shfl_xor_sync(0xffffffffu, ssum, 2);
      ssum += __shfl_xor_sync(0xffffffffu, ssum, 1);
      // a = ex / (sum + 1e-16) (torch_geometric.utils.softmax), then * out-degree of the source (:476-481)
      const float rden = __fdividef(1.f, ssum + 1e-16f);
      const float degf = (float)deg;
      const uint32_t src_off = vl * nch;  // row of this SOURCE node in the Mx tile (phase 2), 16-byte units
      if (l8 < deg) {
        const float a = ex0 * rden;
        p.alpha2[hE + (size_t)tp0] = make_uint2(src_off | (pko_first & 0xffff0000u), __float_as_uint(a * degf));
        if (p.alpha_out != nullptr) p.alpha_out[(size_t)p.perm_src[beg + l8] * p.H + h] = a;
      }
      if (hub) {
        for (int j = 8 + l8; j < deg; j += 8) {
          const float a = __expf(__ldcg(p.score + sbase + j) - m) * rden;
          const uint32_t combo = (uint32_t)__ldg(p.pk_src + beg + j) & 0xffffu;
          p.alpha2[hE + (size_t)__ldg(p.tpos + beg + j)] = make_uint2(offsets_word(vl, combo), __float_as_uint(a * degf));
          if (p.alpha_out != nullptr) p.alpha_out[(size_t)p.perm_src[beg + j] * p.H + h] = a;
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[b]);
    }
    // phase switch: this warp's a' records must be visible to the whole CTA before anyone reads them back
    __threadfence_block();
    __syncwarp();
    if (lane == 0) mbar_arrive(ph1done);
    mbar_wait(ph1done, 0);
  }

  // ---------------------------------- phase 2: weighted sum by target ----------------------------------
  {
    int it1 = grab(ctr_u32 + 4);
    uint2 ni1 = load_ninfo(p.ninfo_tgt, it1);
    int it2 = grab(ctr_u32 + 4);
    uint2 ni2 = load_ninfo(p.ninfo_tgt, it2);
    uint2 e1 = make_uint2(0u, 0u);  // {offsets word, a'} of this lane's edge among the node's first 8 in-edges
    auto issue = [&](const uint2& ni, uint2& e) {
      const int deg = (int)(ni.x >> 16);
      e = make_uint2(0u, 0u);
      if (l8 < deg) e = __ldcg(p.alpha2 + hE + ni.y + l8);
    };
    issue(ni1, e1);
    mbar_wait(tabbar, 1);
    int cur_t = -1;
    while (it1 < total) {
      const int it0 = it1;
      const uint2 ni0 = ni1;
      uint2 e0 = e1;
      it1 = it2; ni1 = ni2;
      issue(ni1, e1);
      it2 = grab(ctr_u32 + 4);
      ni2 = load_ninfo(p.ninfo_tgt, it2);

      const int tg = item_graph(it0);  // graph index within this CTA's list
      const int t = Gc + tg;           // ring position
      const int b = t & 1;
      if (t != cur_t) {
        mbar_wait(&full[b], (t >> 1) & 1);
        cur_t = t;
      }
      const int quad = it0 - tg * nq;
      int ng = p.n;
      const int64_t gbase = RAGGED ? segment(tg, ng) : (int64_t)(slot + tg * p.S) * p.n;
      const bool nvalid = quad * 4 + qi < ng;
      const uint32_t vl = ni0.x & 0xffffu;
      const int beg = (int)ni0.y;
      const int64_t v = gbase + vl;
      int deg = (int)(ni0.x >> 16);
      if (deg == 0xffff) deg = p.rowptr_tgt[v + 1] - p.rowptr_tgt[v];  // saturated record: read the true in-degree
      const int maxdeg = __reduce_max_sync(0xffffffffu, deg);
      uint32_t mtc[CPL];
#pragma unroll
      for (int k = 0; k < CPL; ++k) mtc[k] = smem_u32(smem_raw + sm.tile0 + b * sm.tile_bytes) + 16u * (uint32_t)chunk[k];
      float2 acc[CPL][2];
#pragma unroll
      for (int k = 0; k < CPL; ++k) acc[k][0] = acc[k][1] = make_float2(0.f, 0.f);
      for (int i0 = 0; i0 < maxdeg; i0 += 8) {
        if (i0 > 0) {  // hub nodes only
          e0 = make_uint2(0u, 0u);
          if (i0 + l8 < deg) e0 = __ldcg(p.alpha2 + hE + beg + i0 + l8);
        }
        const uint32_t pko = e0.x;
        const float wv = __uint_as_float(e0.y);  // 0 beyond this node's degree
        const int lim = min(8, maxdeg - i0);
        // (broadcasting all 8 {offsets word, a'} pairs up front, as phase 1 does with its offsets words, costs 16 registers
        //  here and measured 123 vs 112 us/layer: reverted, profiles/r2_mp_tuning.md)
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          if (j + 1 < lim) {  // warp-uniform
            const uint32_t w0 = __shfl_sync(0xffffffffu, pko, qbase + j);
            const uint32_t w1 = __shfl_sync(0xffffffffu, pko, qbase + j + 1);
            const float a0 = __shfl_sync(0xffffffffu, wv, qbase + j);
            const float a1 = __shfl_sync(0xffffffffu, wv, qbase + j + 1);
            const float2 aa0 = make_float2(a0, a0), aa1 = make_float2(a1, a1);
#pragma unroll
            for (int k = 0; k < CPL; ++k) {
              const float4 x0 = lds128(tile_addr(mtc[k], w0)), y0 = lds128(table_addr(tabu[k], w0));
              const float4 x1 = lds128(tile_addr(mtc[k], w1)), y1 = lds128(table_addr(tabu[k], w1));
              acc[k][0] = ffma2(fadd2(lo2(x0), lo2(y0)), aa0, acc[k][0]);
              acc[k][1] = ffma2(fadd2(hi2(x0), hi2(y0)), aa0, acc[k][1]);
              acc[k][0] = ffma2(fadd2(lo2(x1), lo2(y1)), aa1, acc[k][0]);
              acc[k][1] = ffma2(fadd2(hi2(x1), hi2(y1)), aa1, acc[k][1]);
            }
          } else if (j < lim) {  // odd tail: one edge
            const uint32_t w0 = __shfl_sync(0xffffffffu, pko, qbase + j);
            const float a0 = __shfl_sync(0xffffffffu, wv, qbase + j);
            const float2 aa0 = make_float2(a0, a0);
#pragma unroll
            for (int k = 0; k < CPL; ++k) {
              const float4 x0 = lds128(tile_addr(mtc[k], w0)), y0 = lds128(table_addr(tabu[k], w0));
              acc[k][0] = ffma2(fadd2(lo2(x0), lo2(y0)), aa0, acc[k][0]);
              acc[k][1] = ffma2(fadd2(hi2(x0), hi2(y0)), aa0, acc[k][1]);
            }
          }
        }
      }
      if (nvalid) {
        const size_t obase = (size_t)v * p.D + (size_t)h * p.d;
#pragma unroll
        for (int k = 0; k < CPL; ++k) {
          const int c0 = 4 * (l8 + 8 * k);
          if (!cvalid[k] || c0 >= p.d) continue;
          const float v0 = acc[k][0].x, v1 = acc[k][0].y, v2 = acc[k][1].x, v3 = acc[k][1].y;
          if (p.aggr != nullptr) {
            float* out = p.aggr + obase;
            if ((p.d & 3) == 0 && (p.D & 3) == 0) {
              *reinterpret_cast<float4*>(out + c0) = make_float4(v0, v1, v2, v3);
            } else if ((p.d & 1) == 0) {
              *reinterpret_cast<float2*>(out + c0) = make_float2(v0, v1);
              if (c0 + 2 < p.d) *reinterpret_cast<float2*>(out + c0 + 2) = make_float2(v2, v3);
            } else {
              out[c0] = v0;
              if (c0 + 1 < p.d) out[c0 + 1] = v1;
              if (c0 + 2 < p.d) out[c0 + 2] = v2;
              if (c0 + 3 < p.d) out[c0 + 3] = v3;
            }
          }
          if (p.aggr_hi != nullptr) {  // d even (D % 8 == 0 on this path): bf16x2 pairs stay 4-byte aligned
            __nv_bfloat16* oh = (__nv_bfloat16*)p.aggr_hi + obase + c0;
            __nv_bfloat16* ol = (__nv_bfloat16*)p.aggr_lo + obase + c0;
            __nv_bfloat162 h01, l01, h23, l23;
            h01.x = __float2bfloat16_rn(v0); h01.y = __float2bfloat16_rn(v1);
            l01.x = __float2bfloat16_rn(v0 - __bfloat162float(h01.x)); l01.y = __float2bfloat16_rn(v1 - __bfloat162float(h01.y));
            *reinterpret_cast<__nv_bfloat162*>(oh) = h01;
            if (p.aggr_lo != nullptr) *reinterpret_cast<__nv_bfloat162*>(ol) = l01;  // null: the hi plane alone (single pass)
            if (c0 + 2 < p.d) {
              h23.x = __float2bfloat16_rn(v2); h23.y = __float2bfloat16_rn(v3);
              l23.x = __float2bfloat16_rn(v2 - __bfloat162float(h23.x)); l23.y = __float2bfloat16_rn(v3 - __bfloat162float(h23.y));
              *reinterpret_cast<__nv_bfloat162*>(oh + 2) = h23;
              if (p.aggr_lo != nullptr) *reinterpret_cast<__nv_bfloat162*>(ol + 2) = l23;
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[b]);
    }
  }
}

__global__ void zero_head_pads_kernel(int64_t rows, int d, int DP, float* __restrict__ buf) {
  const int pad = DP - d;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows * pad; i += (int64_t)gridDim.x * blockDim.x)
    buf[(i / pad) * DP + d + (i % pad)] = 0.f;
}

struct HeadTilePlan {
  bool ok;
  int DP, C, S, W, cpl, nquads;
  uint32_t nq_magic;
  size_t smem;
};

// A/B switch, read at every launch: QAGNN_MP_WARPS=<n> forces the number of consumer warps per CTA (1..31).
int forced_warps() {
  const char* e = getenv("QAGNN_MP_WARPS");
  const int w = e ? atoi(e) : 0;
  return (w >= 1 && w <= kWarpsWide) ? w : 0;
}

// rg.node_ptr != nullptr: a ragged batch of rg.B graphs of at most n_per_graph rows over the N rows
HeadTilePlan make_plan(const qagnn_shape& s, const Ragged& rg) {
  HeadTilePlan pl{};
  pl.ok = false;
  const bool ragged = rg.node_ptr != nullptr;
  if (s.n_per_graph <= 0 || s.n_per_graph > 65535 || (!ragged && s.N % s.n_per_graph != 0)) return pl;
  if (ragged && (rg.B <= 0 || rg.B > s.N)) return pl;
  const int d = s.D / s.H;
  pl.DP = head_dim_padded(d);
  pl.C = s.R * s.T * s.T + s.T;
  if (pl.DP > 64) return pl;
  // the projection writes the head-major [3][H][N][DP] input of this kernel; its tensor-core GEMM must take the shape too
  if (hm_n_step(HeadMajorOut{1, s.D, d, pl.DP, s.H}) == 0) return pl;
  // the 16|16-bit offsets words: tile rows in 16-byte units below 2^15, table rows in 2-byte units below 2^16
  const long nch = pl.DP / 4;
  if ((long)(s.n_per_graph - 1) * nch > 32767 || (long)(pl.C - 1) * nch * 8 > 65535) return pl;
  if (s.E + s.N >= ((int64_t)1 << 31)) return pl;
  pl.cpl = pl.DP <= 32 ? 1 : 2;
  static int sms_c[kMaxDevices] = {0}, smem_c[kMaxDevices] = {0};
  const int dev = current_device();
  if (sms_c[dev] == 0) {
    cudaDeviceGetAttribute(&smem_c[dev], cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaDeviceGetAttribute(&sms_c[dev], cudaDevAttrMultiProcessorCount, dev);
  }
  const int sms = sms_c[dev], max_smem = smem_c[dev];
  if (sms <= 0 || s.H > sms) return pl;
  pl.smem = make_smem_map(pl.C, pl.DP, s.n_per_graph).total;
  if ((long)pl.smem > (long)max_smem) return pl;
  pl.S = sms / s.H;
  pl.nquads = (s.n_per_graph + 3) / 4;
  // item / nquads by multiply-high: exact while item * nquads < 2^32 (items run to graphs-per-CTA * nquads + 2 per warp)
  pl.nq_magic = (uint32_t)((((uint64_t)1) << 32) / (uint64_t)pl.nquads) + 1u;
  const long long G = ragged ? ragged_max_segments(s.N, rg.B, s.n_per_graph) : s.N / s.n_per_graph, Gc = (G + pl.S - 1) / pl.S;
  if ((Gc * pl.nquads + 4 * kWarpsWide) * (long long)pl.nquads >= ((long long)1 << 32)) return pl;
  // two graphs' quads can be in flight at once; more warps than that would only spin
  // (24 warps at 72 registers beat 31 at 64 with spills: 112 vs 115 us/layer at cfg2, profiles/r2_mp_tuning.md)
  int W = 2 * pl.nquads;
  if (W > kWarpsNarrow) W = kWarpsNarrow;
  const int fw = forced_warps();
  if (fw) W = fw;
  pl.W = W;
  pl.ok = true;
  return pl;
}

template <int CPL, int WMAX, bool RAGGED = false>
int32_t launch_t(const HeadTileParams& p, const HeadTilePlan& plan, unsigned grid, unsigned block, cudaStream_t st) {
  static size_t attr_smem[kMaxDevices] = {0};  // the attribute is per device
  const int dev = current_device();
  if (plan.smem > attr_smem[dev]) {
    QAGNN_CHECK_CUDA(cudaFuncSetAttribute(mp_headtile_kernel<CPL, WMAX, RAGGED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)plan.smem));
    attr_smem[dev] = plan.smem;
  }
  mp_headtile_kernel<CPL, WMAX, RAGGED><<<grid, block, plan.smem, st>>>(p);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

}  // namespace

bool headtile_supported(const qagnn_shape& s, const Ragged& rg) { return make_plan(s, rg).ok; }

int32_t zero_head_pads(const qagnn_shape& s, float* qkmh, cudaStream_t st) {
  const int d = s.D / s.H, DP = head_dim_padded(d);
  if (DP == d) return QAGNN_OK;
  const int64_t rows = (int64_t)3 * s.H * s.N;
  int64_t g = (rows * (DP - d) + 255) / 256;
  if (g > kNumSMs * 16) g = kNumSMs * 16;
  zero_head_pads_kernel<<<(unsigned)g, 256, 0, st>>>(rows, d, DP, qkmh);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

int32_t launch_message_passing_headtile(const qagnn_shape& s, const int32_t* prep_base, const qagnn_prep_layout& L,
                                        const float* qkmh, const float* keh, const float* meh, float* score,
                                        float* alpha2, float* aggr, float* alpha_out, void* aggr_hi, void* aggr_lo,
                                        cudaStream_t st, const Ragged& rg) {
  const HeadTilePlan plan = make_plan(s, rg);
  if (!plan.ok) return QAGNN_ERR_UNSUPPORTED;
  auto I = [&](size_t off) { return (const int32_t*)((const char*)prep_base + off); };
  HeadTileParams p;
  p.N = s.N; p.Eps = (s.N + s.E + 3) / 4 * 4;
  p.n = s.n_per_graph; p.G = (int)(s.N / s.n_per_graph);
  p.node_ptr = rg.node_ptr; p.B = rg.B; p.H = s.H; p.D = s.D; p.d = s.D / s.H; p.DP = plan.DP;
  p.C = plan.C; p.S = plan.S; p.W = plan.W; p.nquads = plan.nquads; p.nq_magic = plan.nq_magic;
  p.rowptr_src = I(L.rowptr_src); p.rowptr_tgt = I(L.rowptr_tgt); p.pk_src = I(L.pk_src); p.tpos = I(L.csr_src_tpos); p.perm_src = I(L.perm_src);
  p.ninfo_src = (const uint2*)I(L.ninfo_src); p.ninfo_tgt = (const uint2*)I(L.ninfo_tgt);
  p.qkmh = qkmh; p.keh = keh; p.meh = meh; p.score = score; p.alpha2 = (uint2*)alpha2; p.aggr = aggr; p.alpha_out = alpha_out;
  p.aggr_hi = (s.D % 2 == 0 && (s.D / s.H) % 2 == 0) ? aggr_hi : nullptr; p.aggr_lo = aggr_lo;
  if (aggr_hi != nullptr && p.aggr_hi == nullptr) return QAGNN_ERR_UNSUPPORTED;
  const unsigned grid = (unsigned)(plan.S * s.H), block = (unsigned)(plan.W + 1) * 32;
  const bool wide = plan.W > kWarpsNarrow;  // more than 24 consumer warps: the 64-register build
  if (rg.node_ptr != nullptr) {
    if (plan.cpl == 1)
      return wide ? launch_t<1, kWarpsWide, true>(p, plan, grid, block, st) : launch_t<1, kWarpsNarrow, true>(p, plan, grid, block, st);
    return wide ? launch_t<2, kWarpsWide, true>(p, plan, grid, block, st) : launch_t<2, kWarpsNarrow, true>(p, plan, grid, block, st);
  }
  if (plan.cpl == 1) return wide ? launch_t<1, kWarpsWide>(p, plan, grid, block, st) : launch_t<1, kWarpsNarrow>(p, plan, grid, block, st);
  return wide ? launch_t<2, kWarpsWide>(p, plan, grid, block, st) : launch_t<2, kWarpsNarrow>(p, plan, grid, block, st);
}

}  // namespace qagnn
