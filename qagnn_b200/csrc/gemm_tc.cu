// Tensor-core GEMM for the dense node-level linears of the hot path (the W_q/W_k/W_m projection, the
// node MLP, Vh/Vx — modeling/modeling_qagnn.py:464-466 node part, :443/:408, :92):
//
//     C[M,N] = act( [A1 | A2] @ W^T + bias )          fp32 in, fp32 accumulate, fp32-faithful out
//
// Hopper-native: wgmma.mma_async (bf16 operands from shared memory, fp32 accumulators in registers), operands staged
// by TMA (cp.async.bulk.tensor, 128-byte swizzle) through an mbarrier ring.  Warpgroup 0 is the producer (one thread
// issues the TMA loads); warpgroups 1 and 2 each own 64 rows of the 128-row tile, issue its wgmma chain and run the
// epilogue from their accumulator registers.  By default two CTAs of a cluster work on neighbouring row tiles of the
// same n tile, and each loads HALF of the W tile with a TMA multicast into both CTAs' shared memory, which halves the
// weight bytes each CTA pulls through L2.
//
// Precision: the reference runs these linears in fp32 and parity is 1e-4, which single-pass bf16
// (2^-9) or tf32 (2^-11) cannot hold.  Operands are therefore stored as SPLIT-BF16 planes
//     a = a_hi + a_lo,  a_hi = bf16(a), a_lo = bf16(a - a_hi)        (16 mantissa bits)
// and each k-step issues three MMAs (hi*hi + hi*lo + lo*hi) into the same fp32 accumulator: the
// dropped terms are O(2^-17) relative, ~50x below the parity bar, at 3 tensor passes instead of
// the ~30x slower FFMA path (sgemm.cu, kept as the exact-fp32 fallback).
//
// Single pass (passes = 1: gemm_bf16_kernel / mlp_bf16_kernel, the eval forward under bf16 autocast): the same kernels on
// the hi planes alone - a ring stage is [A hi | W hi], one wgmma per k16 step, and the epilogue writes fp32 and/or the hi
// plane.  The caller has asked for bf16 matmul operands, and hi = bf16_rn(v) is exactly that rounding.
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace qagnn {

namespace {

constexpr int BM = 128;      // rows per CTA tile: two consumer warpgroups x wgmma M = 64
constexpr int BK = 64;       // k-block width in bf16: one 128-byte swizzle span per row
constexpr int kThreads = 384;  // warpgroup 0: TMA producer; warpgroups 1-2: wgmma + epilogue
constexpr size_t kSmemCap = 227 * 1024;  // opt-in shared memory per block on H100
constexpr int kCtrlBytes = 1024;         // mbarriers after the operand ring

// Epilogue staging (after the mbarriers): each consumer warpgroup writes a column chunk of its 64 rows here and one of its
// threads stores it with TMA, so the warpgroup is back at the next tile's MMAs while the copy drains.  13 KB = 64 rows x 52
// fp32 columns, one head of the QA-GNN projection at D = 200.  Two buffers per warpgroup where the ring keeps its stage count
// with them (bn = 208: 2 stages of 86 KB leave 58 KB), else one (bn = 64 / 128 keep 4 / 3 stages, bn = 256 its 2).
constexpr uint32_t kStBytes = 13312;
__host__ __device__ constexpr int st_bufs(int bn) { return bn == 208 ? 2 : 1; }
// bf16 planes per operand: hi and lo for the split-bf16 passes (3), hi alone for the single pass (1)
__host__ __device__ constexpr int planes_of(int passes) { return passes == 1 ? 1 : 2; }
__host__ __device__ constexpr size_t ring_stage_bytes(int bn, int passes = 3) {
  return planes_of(passes) * ((size_t)BM * BK * 2 + (size_t)bn * BK * 2);
}
// bn = 208: 2 stages of 86 KB (split) or 4 of 43 KB (single pass) beside the two staging buffers per warpgroup
__host__ __device__ constexpr int ring_stages(int bn, int passes = 3) {
  return (kSmemCap - kCtrlBytes - 2 * st_bufs(bn) * kStBytes) / ring_stage_bytes(bn, passes) > 6
             ? 6
             : (int)((kSmemCap - kCtrlBytes - 2 * st_bufs(bn) * kStBytes) / ring_stage_bytes(bn, passes));
}

struct TcParams {
  CUtensorMap a_hi[2], a_lo[2], w_hi, w_lo;
  int nseg, kseg[2];
  int n_step, N, stages;
  long long M;
  const float* bias;
  const int64_t* row_class;  // optional: bias row = clamp(row_class[r], 0, n_class-1) * class_stride
  int class_stride, n_class;
  float* c_f32;
  int ldc;
  float* c_hm;
  HeadMajorOut hm;
  __nv_bfloat16 *c_hi, *c_lo;
  int ldp;
  // TMA-store epilogue when st_w > 0: st_chunks chunks of st_w tile columns; boxes of st_w columns x 64 rows over the fp32
  // output ([3H][M][DP] head-major or [1][M][N] row-major) and the bf16 planes ([1][M][N]), clipped to M and N
  CUtensorMap st_f32, st_hi, st_lo;
  int st_w, st_chunks;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
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
// Stage release: arrive on the `empty` barrier at the same shared-memory offset in CTA `cta` of the cluster (CTAS = 1: this
// CTA's own).  Default (.release.cta) semantics on purpose: the only accesses a release orders are the wgmma reads of the
// stage, which are complete once wgmma.wait_group has returned, and the refill it unblocks is a TMA write in the async proxy.
// The .release.cluster form compiles to MEMBAR.ALL.GPU in front of the arrive, which waits for every global store the thread
// has in flight (the previous tile's epilogue) - on the critical path of every k block.
template <int CTAS>
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  if (CTAS == 1) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
  } else {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
  }
}
// one arrival per warp on `empty` in every CTA of the pair: lane c arrives on CTA c, so both arrivals issue at once
template <int CTAS>
__device__ __forceinline__ void release_stage(uint64_t* empty, int lane) {
  __syncwarp();
  if (lane < CTAS) mbar_arrive_cluster<CTAS>(empty, (uint32_t)lane);
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
// the same box lands at the same offset in every CTA of `mask`, each completing its own barrier at `bar`'s offset
__device__ __forceinline__ void tma_load_2d_multicast(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar,
                                                      uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%2, %3}], "
      "[%4], %5;" ::"r"(smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "h"(mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// epilogue staging: the warpgroup's generic-proxy writes are made visible to the TMA engine (async proxy) by each writer's
// proxy fence and a warpgroup barrier; a buffer is rewritten only once the store that read it has finished reading
__device__ __forceinline__ void wg_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void st_shared_f2(uint32_t a, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void st_shared_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {  // at most N committed stores still reading shared memory
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// K-major operand tile, 128-byte swizzle: rows of 128 B, 8-row groups 1024 B apart (wgmma matrix descriptor:
// start >> 4 | LBO (unused for swizzled K-major) = 1 | SBO = 1024 >> 4 | layout type 1 = SWIZZLE_128B)
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void fence_acc(float (&d)[N]) {  // keeps the compiler from moving accumulator accesses
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] . B[16 x N], both operands K-major in shared memory; scale_d = 0 overwrites D
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <>
__device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_bf16<104>(float (&d)[52], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %54, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n104k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51}, %52, %53, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_bf16<208>(float (&d)[104], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %106, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n208k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103}, %104, %105, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_bf16<256>(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d));
}

// the three split-bf16 passes (hi*hi, hi*lo, lo*hi) of the first STEPS k16-steps of one k block, or hi*hi alone when
// P = 1; A / W plane tiles at sa / sw.  STEPS is a compile-time count: a run-time one makes ptxas fence every wgmma of the
// chain.
template <int BN, int STEPS, int P = 3>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint32_t sa, uint32_t sw, uint32_t a_bytes, uint32_t w_bytes) {
#pragma unroll
  for (int k = 0; k < STEPS; ++k) {
    const uint64_t da_hi = wgmma_desc(sa + k * 32), dw_hi = wgmma_desc(sw + k * 32);
    wgmma_bf16<BN>(acc, da_hi, dw_hi, 1u);
    if constexpr (P == 3) {
      const uint64_t da_lo = wgmma_desc(sa + a_bytes + k * 32), dw_lo = wgmma_desc(sw + w_bytes + k * 32);
      wgmma_bf16<BN>(acc, da_hi, dw_lo, 1u);
      wgmma_bf16<BN>(acc, da_lo, dw_hi, 1u);
    }
  }
}

// D[64 x N] += A[64 x 16] . B[16 x N], A from registers (the m64nNk16 A fragment: four bf16x2 words), B K-major in shared
// memory: the second GEMM of the fused MLP (mlp_tc_kernel)
template <int N>
__device__ __forceinline__ void wgmma_bf16_rs(float (&d)[N / 2], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t db);
template <>
__device__ __forceinline__ void wgmma_bf16_rs<72>(float (&d)[36], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %41, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n72k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35}, {%36,%37,%38,%39}, %40, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(db), "r"(1u));
}

// tanh-approximation GELU (utils/layers.py:10-14) with tanh(u) = 1 - 2/(exp(2u)+1) on the fast exp/divide units:
// ~1e-6 absolute, far inside the parity bar, and ~6 instructions instead of tanhf's ~30
__device__ __forceinline__ float gelu_tanh_fast(float x) {
  const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
  const float t = 1.f - __fdividef(2.f, __expf(2.f * u) + 1.f);
  return 0.5f * x * (1.f + t);
}

template <int ACT>
__device__ __forceinline__ float act_fn(float v) {
  if (ACT == ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == ACT_GELU) return gelu_tanh_fast(v);
  return v;
}

// hi = bf16(v), lo = bf16(v - hi) of a column pair, packed low column first (the order of a bf16x2 fragment word)
__device__ __forceinline__ void split_pair(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h2, l2;
  h2.x = __float2bfloat16_rn(v0);
  h2.y = __float2bfloat16_rn(v1);
  l2.x = __float2bfloat16_rn(v0 - __bfloat162float(h2.x));
  l2.y = __float2bfloat16_rn(v1 - __bfloat162float(h2.y));
  hi = *reinterpret_cast<uint32_t*>(&h2);
  lo = *reinterpret_cast<uint32_t*>(&l2);
}
// hi = bf16(v) of a column pair alone (single pass: no lo plane)
__device__ __forceinline__ uint32_t hi_pair(float v0, float v1) {
  __nv_bfloat162 h2;
  h2.x = __float2bfloat16_rn(v0);
  h2.y = __float2bfloat16_rn(v1);
  return *reinterpret_cast<uint32_t*>(&h2);
}

// Persistent CTAs (CTAS = 1) or CTA pairs (CTAS = 2, one cluster) walk the (row block, n tile) grid with n fastest.
// Ring stage = [A hi | A lo | W hi | W lo] (P = 3) or [A hi | W hi] (P = 1), each a 1024-byte aligned K-major tile of 64
// bf16 per row.  Both kernels are the one body in gemm_tc_body.cuh with their pass count.
template <int ACT, int BN, int CTAS>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ TcParams p) {
  constexpr int P = 3;
#include "gemm_tc_body.cuh"
}
template <int ACT, int BN, int CTAS>
__global__ void __launch_bounds__(kThreads, 1) gemm_bf16_kernel(const __grid_constant__ TcParams p) {
  constexpr int P = 1;
#include "gemm_tc_body.cuh"
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused node MLP:  out = act2( W2 . ReLU(W1 . aggr + b1) + b2 ),  D <= 208, every operand a split-bf16 plane pair.
//
// The first GEMM is gemm_tc_kernel's mainloop at BN = 208 (aggr and W1 k blocks through the same ring).  Its accumulator
// fragment is turned into the hidden layer in place: + b1, ReLU, hi = bf16(v), lo = bf16(v - hi) - the rounding of
// gemm_tc_kernel's plane epilogue.  The f32 accumulator fragment of m64nNk16 has the layout of the register A fragment of
// the next m64nNk16, so fragment groups 2t and 2t+1 (columns 16t .. 16t+15) are the four A words of k16 step t.  The second
// GEMM takes A from those registers and streams W2 through the ring in N chunks of 72 rows (all of K in one ring stage), so
// only one 36-register accumulator is live beside the 104 hidden words.  Each output element sees the same k16 steps, in
// the same order and with the same three passes, as the two-launch path (mlp.0 writing the hidden planes, mlp.3 reading them).
constexpr int kMlpMaxD = 208;                      // hidden width held in registers: 13 k16 steps
constexpr int kMlpChunk = 72;                      // W2 rows (output columns) per chunk
// Two warpgroups and no producer warpgroup: 256 threads may hold 255 registers each.  With a third warpgroup (or even one
// extra warp: registers are split per SM sub-partition) every thread is held to 168 - ptxas allocates against that bound
// whatever setmaxnreg hands out at run time - and the 104 hidden words, a chunk accumulator and the epilogue spill there.
// One consumer thread issues the TMA fills instead, `stages` fills ahead of the consumers.
constexpr int kMlpThreads = 256;
constexpr uint32_t kW2Sub = kMlpChunk * BK * 2;    // one W2 plane k block of a chunk: 9216 B (a multiple of 1024)
// epilogue staging per warpgroup: one chunk of its 64 rows, fp32 or both bf16 planes (staged one after the other when
// both are asked for: two buffers would leave room for one ring stage only)
constexpr uint32_t kMlpStBytes = 64 * kMlpChunk * 4;
constexpr int mlp_ring_stages(int passes = 3) {
  return (int)((kSmemCap - kCtrlBytes - 2 * kMlpStBytes) / ring_stage_bytes(kMlpMaxD, passes)) > 6
             ? 6
             : (int)((kSmemCap - kCtrlBytes - 2 * kMlpStBytes) / ring_stage_bytes(kMlpMaxD, passes));
}
static_assert(mlp_ring_stages() >= 2, "the fused MLP's epilogue staging leaves room for two ring stages");

struct MlpParams {
  CUtensorMap a_hi, a_lo, w1_hi, w1_lo, w2_hi, w2_lo;
  int D, stages;
  long long M;
  const float *b1, *b2;
  float* c_f32;
  int ldc;
  __nv_bfloat16 *c_hi, *c_lo;
  int ldp;
  // TMA-store epilogue when set: boxes of one 72-column chunk x 64 rows over the fp32 output and the bf16 planes
  CUtensorMap st_f32, st_hi, st_lo;
  int tma_store;
};

// the three split-bf16 passes of the first STEPS k16 steps of the hidden layer against one W2 chunk (hi planes at sw, lo
// planes lo_off further; k block kb of a plane at kb * kW2Sub), or hh * W2 hi alone when P = 1 (hl is then unused)
template <int STEPS, int P = 3, int HL>
__device__ __forceinline__ void mma_chunk(float (&acc)[kMlpChunk / 2], const uint32_t (&hh)[kMlpMaxD / 4],
                                          const uint32_t (&hl)[HL], uint32_t sw, uint32_t lo_off) {
#pragma unroll
  for (int t = 0; t < STEPS; ++t) {
    const uint32_t off = (uint32_t)(t >> 2) * kW2Sub + (uint32_t)(t & 3) * 32;
    const uint64_t dw_hi = wgmma_desc(sw + off);
    wgmma_bf16_rs<kMlpChunk>(acc, hh[4 * t], hh[4 * t + 1], hh[4 * t + 2], hh[4 * t + 3], dw_hi);
    if constexpr (P == 3) {
      const uint64_t dw_lo = wgmma_desc(sw + lo_off + off);
      wgmma_bf16_rs<kMlpChunk>(acc, hh[4 * t], hh[4 * t + 1], hh[4 * t + 2], hh[4 * t + 3], dw_lo);
      wgmma_bf16_rs<kMlpChunk>(acc, hl[4 * t], hl[4 * t + 1], hl[4 * t + 2], hl[4 * t + 3], dw_hi);
    }
  }
}

// Ring fills per 128-row tile: the k blocks of GEMM1 ([aggr hi | aggr lo | W1 hi | W1 lo], as gemm_tc_kernel at BN = 208),
// then one fill per W2 chunk ([W2 hi kb 0..nkb-1 | W2 lo kb 0..nkb-1], 72 rows each).  Thread 0 issues them.  With CTA
// pairs each CTA loads half of W1's rows and every other W2 k block, multicast into both.  P = 1 (mlp_bf16_kernel): the
// hi planes alone, and the hidden layer is one bf16 fragment (52 words at D = 208 instead of 104).
template <int ACT, int CTAS, int P>
__device__ __forceinline__ void mlp_body(const MlpParams& p) {
  extern __shared__ __align__(1024) unsigned char smem[];
  constexpr int BN = kMlpMaxD;
  constexpr int NP = planes_of(P);
  constexpr uint32_t a_bytes = BM * BK * 2;
  constexpr uint32_t w_bytes = BN * BK * 2;
  constexpr uint32_t stage_bytes = NP * a_bytes + NP * w_bytes;
  static_assert(NP * 4 * kW2Sub <= stage_bytes, "a W2 chunk fills one ring stage");
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const uint32_t rank = CTAS == 2 ? cluster_ctarank() : 0u;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * stage_bytes);
  uint64_t* empty = full + p.stages;
  unsigned char* staging = smem + (size_t)p.stages * stage_bytes + kCtrlBytes;  // [2 warpgroups][kMlpStBytes]

  const int D = p.D;
  const int nkb = (D + BK - 1) / BK;          // k blocks of both GEMMs (K = D)
  const int tail_steps = (D - 1) % BK / 16 + 1;
  const int ksteps = (D + 15) / 16;           // k16 steps of GEMM2 = hidden fragment groups in use
  const int nch = (D + kMlpChunk - 1) / kMlpChunk;
  const uint32_t chunk_bytes = (uint32_t)NP * (uint32_t)nkb * kW2Sub;
  const long long total_tiles = (p.M + BM * CTAS - 1) / (BM * CTAS);
  const long long cl_id = blockIdx.x / CTAS, n_cl = gridDim.x / CTAS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8 * CTAS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CTAS == 2) cluster_sync_all();

  // ---- ring fills: this cluster's tiles, each nkb GEMM1 k blocks then nch W2 chunks; fill f goes to stage f % stages
  const int fills_per_tile = nkb + nch;
  const long long n_fills = (cl_id < total_tiles ? (total_tiles - 1 - cl_id) / n_cl + 1 : 0) * fills_per_tile;
  auto issue = [&](long long f) {
    const long long tile = cl_id + f / fills_per_tile * n_cl;
    const int sub = (int)(f % fills_per_tile);
    unsigned char* st = smem + (size_t)(f % p.stages) * stage_bytes;
    uint64_t* bar = &full[f % p.stages];
    if (sub < nkb) {  // GEMM1 k block: [aggr hi | aggr lo | W1 hi | W1 lo]
      const int kb = sub, m0 = (int)(tile * BM * CTAS + rank * BM);
      mbar_expect_tx(bar, stage_bytes);
      tma_load_2d(st, &p.a_hi, kb * BK, m0, bar);
      if constexpr (P == 3) tma_load_2d(st + a_bytes, &p.a_lo, kb * BK, m0, bar);
      if (CTAS == 1) {
        tma_load_2d(st + NP * a_bytes, &p.w1_hi, kb * BK, 0, bar);
        if constexpr (P == 3) tma_load_2d(st + 2 * a_bytes + w_bytes, &p.w1_lo, kb * BK, 0, bar);
      } else {
        const uint32_t half = w_bytes / 2;
        tma_load_2d_multicast(st + NP * a_bytes + rank * half, &p.w1_hi, kb * BK, (int)rank * (BN / 2), bar, 3);
        if constexpr (P == 3)
          tma_load_2d_multicast(st + 2 * a_bytes + w_bytes + rank * half, &p.w1_lo, kb * BK, (int)rank * (BN / 2), bar, 3);
      }
    } else {  // W2 chunk: [W2 hi kb 0 .. nkb-1 | W2 lo kb 0 .. nkb-1]
      const int ch = sub - nkb;
      mbar_expect_tx(bar, chunk_bytes);
      for (int kb = (int)rank; kb < nkb; kb += CTAS) {
        unsigned char* hi = st + (size_t)kb * kW2Sub;
        unsigned char* lo = st + (size_t)(nkb + kb) * kW2Sub;
        if (CTAS == 1) {
          tma_load_2d(hi, &p.w2_hi, kb * BK, ch * kMlpChunk, bar);
          if constexpr (P == 3) tma_load_2d(lo, &p.w2_lo, kb * BK, ch * kMlpChunk, bar);
        } else {
          tma_load_2d_multicast(hi, &p.w2_hi, kb * BK, ch * kMlpChunk, bar, 3);
          if constexpr (P == 3) tma_load_2d_multicast(lo, &p.w2_lo, kb * BK, ch * kMlpChunk, bar, 3);
        }
      }
    }
  };
  const bool producer = threadIdx.x == 0;
  if (producer)
    for (long long f = 0; f < p.stages && f < n_fills; ++f) issue(f);
  {  // both warpgroups consume: warpgroup wc owns rows wc*64 .. wc*64+63 of the tile
    const int wc = wg;
    const int warp = tid >> 5, lane = tid & 31;
    const int q2 = 2 * (lane & 3);  // fragment column pair 8j + q2
    long long it = 0;
    // fill `it` (stage s) is consumed: release it to both CTAs; once every consumer warp of both has, the producer thread
    // refills the stage with fill it + stages
    auto release = [&](int s) {
      release_stage<CTAS>(&empty[s], lane);
      if (producer && it + p.stages < n_fills) {
        mbar_wait(&empty[s], (uint32_t)(it / p.stages) & 1u);
        issue(it + p.stages);
      }
      __syncwarp();
    };
    for (long long tile = cl_id; tile < total_tiles; tile += n_cl) {
      // ---- GEMM1: acc1 = aggr . W1^T over all 208 (zero-padded) hidden columns
      float acc1[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc1[i] = 0.f;
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = (int)(it % p.stages);
        mbar_wait(&full[s], (uint32_t)(it / p.stages) & 1u);
        const uint32_t sbase = smem_u32(smem + (size_t)s * stage_bytes);
        const uint32_t sa = sbase + (uint32_t)wc * 64 * 128, sw = sbase + NP * a_bytes;
        const int steps = kb == nkb - 1 ? tail_steps : BK / 16;
        fence_acc<BN / 2>(acc1);
        wgmma_fence();
        switch (steps) {
          case 1: mma_kblock<BN, 1, P>(acc1, sa, sw, a_bytes, w_bytes); wgmma_commit(); break;
          case 2: mma_kblock<BN, 2, P>(acc1, sa, sw, a_bytes, w_bytes); wgmma_commit(); break;
          case 3: mma_kblock<BN, 3, P>(acc1, sa, sw, a_bytes, w_bytes); wgmma_commit(); break;
          default: mma_kblock<BN, 4, P>(acc1, sa, sw, a_bytes, w_bytes); wgmma_commit(); break;
        }
        wgmma_wait_all();
        fence_acc<BN / 2>(acc1);
        release(s);
      }
      // ---- hidden layer in registers: fragment group j (columns 8j + q2, +1; rows g and g + 8) -> words 2j, 2j + 1
      uint32_t hh[BN / 4], hl[P == 3 ? BN / 4 : 1];
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + q2;
        const bool in = c < D;  // columns D .. 207 are exact zeros (D even: c + 1 < D too)
        const float bb0 = in ? __ldg(p.b1 + c) : 0.f, bb1 = in ? __ldg(p.b1 + c + 1) : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v0 = acc1[4 * j + 2 * h] + bb0, v1 = acc1[4 * j + 2 * h + 1] + bb1;
          v0 = in ? act_fn<ACT_RELU>(v0) : 0.f;
          v1 = in ? act_fn<ACT_RELU>(v1) : 0.f;
          if constexpr (P == 3) split_pair(v0, v1, hh[2 * j + h], hl[2 * j + h]);
          else hh[2 * j + h] = hi_pair(v0, v1);
        }
      }
      // ---- GEMM2 in N chunks, each followed by its epilogue
      const long long row_g = tile * BM * CTAS + rank * BM + wc * 64 + warp * 16 + (lane >> 2);
      for (int ch = 0; ch < nch; ++ch, ++it) {
        const int s = (int)(it % p.stages);
        float acc2[kMlpChunk / 2];
#pragma unroll
        for (int i = 0; i < kMlpChunk / 2; ++i) acc2[i] = 0.f;
        mbar_wait(&full[s], (uint32_t)(it / p.stages) & 1u);
        const uint32_t sw = smem_u32(smem + (size_t)s * stage_bytes), lo_off = (uint32_t)nkb * kW2Sub;
        fence_acc<kMlpChunk / 2>(acc2);
        wgmma_fence();
        switch (ksteps) {  // compile-time chains: the hidden words are registers, indexed by the step
          case 1: mma_chunk<1, P>(acc2, hh, hl, sw, lo_off); break;
          case 2: mma_chunk<2, P>(acc2, hh, hl, sw, lo_off); break;
          case 3: mma_chunk<3, P>(acc2, hh, hl, sw, lo_off); break;
          case 4: mma_chunk<4, P>(acc2, hh, hl, sw, lo_off); break;
          case 5: mma_chunk<5, P>(acc2, hh, hl, sw, lo_off); break;
          case 6: mma_chunk<6, P>(acc2, hh, hl, sw, lo_off); break;
          case 7: mma_chunk<7, P>(acc2, hh, hl, sw, lo_off); break;
          case 8: mma_chunk<8, P>(acc2, hh, hl, sw, lo_off); break;
          case 9: mma_chunk<9, P>(acc2, hh, hl, sw, lo_off); break;
          case 10: mma_chunk<10, P>(acc2, hh, hl, sw, lo_off); break;
          case 11: mma_chunk<11, P>(acc2, hh, hl, sw, lo_off); break;
          case 12: mma_chunk<12, P>(acc2, hh, hl, sw, lo_off); break;
          default: mma_chunk<13, P>(acc2, hh, hl, sw, lo_off); break;
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_acc<kMlpChunk / 2>(acc2);
        release(s);
        if (p.tma_store) {
          // through this warpgroup's staging buffer: the fp32 box, then the two plane boxes, each stored with TMA by thread
          // 0 of the warpgroup (clipped to M rows and D columns); the buffer is rewritten once the last store has read it
          const uint32_t buf = smem_u32(staging) + (uint32_t)wc * kMlpStBytes;
          const int rl = warp * 16 + (lane >> 2);
          const int r0 = (int)(row_g - rl);
          for (int part = 0; part < 2; ++part) {
            if (part == 0 ? p.c_f32 == nullptr : p.c_hi == nullptr) continue;
            if (tid == 0) bulk_wait_read<0>();
            wg_bar(1 + wc);
#pragma unroll
            for (int j = 0; j < kMlpChunk / 8; ++j) {
              const int cc = 8 * j + q2, gc = ch * kMlpChunk + cc;
              const float bb0 = gc < D ? __ldg(p.b2 + gc) : 0.f, bb1 = gc < D ? __ldg(p.b2 + gc + 1) : 0.f;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float v0 = act_fn<ACT>(acc2[4 * j + 2 * h] + bb0);
                const float v1 = act_fn<ACT>(acc2[4 * j + 2 * h + 1] + bb1);
                const uint32_t e = (uint32_t)((rl + 8 * h) * kMlpChunk + cc);
                if (part == 0) {
                  st_shared_f2(buf + 4 * e, v0, v1);
                } else if constexpr (P == 3) {
                  uint32_t hi, lo;
                  split_pair(v0, v1, hi, lo);
                  st_shared_u32(buf + 2 * e, hi);
                  st_shared_u32(buf + kMlpStBytes / 2 + 2 * e, lo);
                } else {
                  st_shared_u32(buf + 2 * e, hi_pair(v0, v1));
                }
              }
            }
            fence_proxy_async();
            wg_bar(1 + wc);
            if (tid == 0) {
              const unsigned char* b = staging + (size_t)wc * kMlpStBytes;
              if (part == 0) {
                tma_store_3d(&p.st_f32, b, ch * kMlpChunk, r0, 0);
              } else {
                tma_store_3d(&p.st_hi, b, ch * kMlpChunk, r0, 0);
                if constexpr (P == 3) tma_store_3d(&p.st_lo, b + kMlpStBytes / 2, ch * kMlpChunk, r0, 0);
              }
              bulk_commit();
            }
          }
          continue;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long r = row_g + 8 * h;
          if (r >= p.M) continue;
#pragma unroll
          for (int j = 0; j < kMlpChunk / 8; ++j) {
            const int gc = ch * kMlpChunk + 8 * j + q2;
            if (gc >= D) continue;
            const float v0 = act_fn<ACT>(acc2[4 * j + 2 * h] + __ldg(p.b2 + gc));
            const float v1 = act_fn<ACT>(acc2[4 * j + 2 * h + 1] + __ldg(p.b2 + gc + 1));
            if (p.c_f32 != nullptr) *reinterpret_cast<float2*>(p.c_f32 + (size_t)r * p.ldc + gc) = make_float2(v0, v1);
            if (p.c_hi != nullptr) {
              if constexpr (P == 3) {
                uint32_t hi, lo;
                split_pair(v0, v1, hi, lo);
                *reinterpret_cast<uint32_t*>(p.c_hi + (size_t)r * p.ldp + gc) = hi;
                *reinterpret_cast<uint32_t*>(p.c_lo + (size_t)r * p.ldp + gc) = lo;
              } else {
                *reinterpret_cast<uint32_t*>(p.c_hi + (size_t)r * p.ldp + gc) = hi_pair(v0, v1);
              }
            }
          }
        }
      }
    }
    if (tid == 0) bulk_wait_all();  // no store still reads the staging buffers when the CTA exits
  }
  __syncthreads();
  if (CTAS == 2) cluster_sync_all();
}

template <int ACT, int CTAS>
__global__ void __launch_bounds__(kMlpThreads, 1) mlp_tc_kernel(const __grid_constant__ MlpParams p) {
  mlp_body<ACT, CTAS, 3>(p);
}
template <int ACT, int CTAS>
__global__ void __launch_bounds__(kMlpThreads, 1) mlp_bf16_kernel(const __grid_constant__ MlpParams p) {
  mlp_body<ACT, CTAS, 1>(p);
}

// ---------------------------------------------------------------------------------------------------------------------
// The fast-form Q|Kx|Mx projection with a resident weight slice:
//
//     qkm[3][H][M][DP] = [x | score_emb] @ W^T + tbias[clamp(type)]        split-bf16, K = D + D/2 <= 320
//
// gemm_tc_kernel reloads its whole W tile (208 columns x K x 2 planes, 266 KB at D = 200) for every 128-row tile, through
// the same ring as A, and its two consumer warpgroups sit in their epilogue together while the tensor pipe idles.  Here each
// persistent CTA owns one n slice of whole heads (kResBN = 104 columns: two heads of DP 52 at D = 200, six slices over
// Q|Kx|Mx) and loads both of its W planes, every k block, into shared memory once; wgmma reads B from that copy for the
// whole walk.  The ring carries A alone, one 64-row unit of one warpgroup per stage ([A hi | A lo], 16 KB).  The two
// consumer warpgroups own alternate units and take turns on the tensor pipe (named barriers 3 and 4), so one warpgroup's
// epilogue runs under the other's mainloop.  With CTA pairs the two CTAs of a cluster hold neighbouring slices of the same
// rows, and each loads one A plane multicast into both.  The clusters of one slice group walk the units in the same order as
// the other groups, so A comes from HBM about once and from L2 thereafter.
//
// Every output element sees the same k16 steps in the same order with the same three passes (hi*hi, hi*lo, lo*hi) and the
// same exact K tail as in gemm_tc_kernel, and the same bias addition, so the two kernels' outputs are equal bit for bit.
constexpr int kResBN = 104;                                 // wgmma N: one slice of whole heads
constexpr int kResMaxKb = 5;                                // k blocks the resident slice holds: K <= 320
constexpr int kResStages = 4;
constexpr uint32_t kResAPlane = 64 * BK * 2;                // one A plane of one 64-row unit: 8 KB
constexpr uint32_t kResStage = 2 * kResAPlane;              // ring stage [A hi | A lo]
constexpr uint32_t kResWPlane = kResBN * BK * 2;            // one W plane k block of the slice: 13 KB
constexpr uint32_t kResWBytes = kResMaxKb * 2 * kResWPlane;  // resident slice: [kb][hi | lo], 130 KB
// [resident W | ring | mbarriers | one staging buffer (64 rows x one head of fp32) per consumer warpgroup]
constexpr size_t kResSmem = kResWBytes + kResStages * kResStage + kCtrlBytes + 2 * kStBytes;
static_assert(kResSmem <= kSmemCap, "the resident slice, the A ring and the staging buffers fit the opt-in shared memory");
static_assert(kResWPlane % 1024 == 0 && kResStage % 1024 == 0, "swizzled tiles start on 1024-byte boundaries");

struct ResParams {
  CUtensorMap a_hi, a_lo, w_hi, w_lo, st_f32;
  int nkb, tail_steps;
  int n_step, DP;  // slice columns (whole heads) and padded head width
  int groups;      // slice groups: slices / CTAS
  long long M;
  const float* bias;         // [n_class][N]
  const int64_t* row_class;  // bias row of row r = clamp(row_class[r], 0, n_class - 1)
  int class_stride, n_class;
};

__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

template <int CTAS>
__global__ void __launch_bounds__(kThreads, 1) proj_resident_kernel(const __grid_constant__ ResParams p) {
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* const wres = smem;
  unsigned char* const ring = smem + kResWBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + kResStages * kResStage);  // [stages]  TMA -> MMA
  uint64_t* empty = full + kResStages;                                           // [stages]  MMA -> TMA
  uint64_t* w_full = empty + kResStages;                                         // the resident slice has landed
  unsigned char* const staging = ring + kResStages * kResStage + kCtrlBytes;     // [2 warpgroups][kStBytes]
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const uint32_t rank = CTAS == 2 ? cluster_ctarank() : 0u;
  // cluster cl holds slice group cl % groups and walks the 64-row units first, first + walkers, ...
  const int cl = blockIdx.x / CTAS, n_cl = gridDim.x / CTAS;
  const int slice = (cl % p.groups) * CTAS + (int)rank;
  const long long first = cl / p.groups, walkers = n_cl / p.groups;
  const long long units = (p.M + 63) / 64;
  const long long n_mine = first < units ? (units - 1 - first) / walkers + 1 : 0;
  const int n0 = slice * p.n_step;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kResStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4 * CTAS);  // one arrival per warp of the consuming warpgroup in every CTA the stage lands in
    }
    mbar_init(w_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CTAS == 2) cluster_sync_all();  // the peer's barriers are initialised before any multicast or remote arrive

  if (wg == 0) {
    // ===================================== TMA producer =====================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (tid == 0) {
      mbar_expect_tx(w_full, (uint32_t)p.nkb * 2 * kResWPlane);
      for (int kb = 0; kb < p.nkb; ++kb) {
        tma_load_2d(wres + (size_t)(2 * kb) * kResWPlane, &p.w_hi, kb * BK, n0, w_full);
        tma_load_2d(wres + (size_t)(2 * kb + 1) * kResWPlane, &p.w_lo, kb * BK, n0, w_full);
      }
      long long it = 0;  // fill i * nkb + kb: unit i, k block kb
      for (long long i = 0; i < n_mine; ++i) {
        const int m0 = (int)((first + i * walkers) * 64);
        for (int kb = 0; kb < p.nkb; ++kb, ++it) {
          const int s = (int)(it % kResStages);
          // the stage is free once the consuming warpgroup of BOTH CTAs has read it (each CTA's plane lands in both)
          if (it >= kResStages) mbar_wait(&empty[s], (uint32_t)((it / kResStages) - 1) & 1u);
          unsigned char* st = ring + (size_t)s * kResStage;
          mbar_expect_tx(&full[s], kResStage);
          if (CTAS == 1) {
            tma_load_2d(st, &p.a_hi, kb * BK, m0, &full[s]);
            tma_load_2d(st + kResAPlane, &p.a_lo, kb * BK, m0, &full[s]);
          } else {
            tma_load_2d_multicast(st + rank * kResAPlane, rank == 0 ? &p.a_hi : &p.a_lo, kb * BK, m0, &full[s], 3);
          }
        }
      }
    }
  } else {
    // ===================================== consumers (warpgroups 1, 2) =====================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wc = wg - 1;  // units wc, wc + 2, ... of this CTA's walk
    const int warp = tid >> 5, lane = tid & 31;
    const int q2 = 2 * (lane & 3);
    const int rl = warp * 16 + (lane >> 2);  // fragment rows rl, rl + 8 of the unit's 64
    const int DP = p.DP;
    const uint32_t buf = smem_u32(staging) + (uint32_t)wc * kStBytes;
    const uint32_t sw0 = smem_u32(wres);
    mbar_wait(w_full, 0u);
    float acc[kResBN / 2];
    for (long long i = wc; i < n_mine; i += 2) {
      // the other warpgroup's mainloop of unit i - 1 has been issued: this one's turn on the tensor pipe
      if (i > 0) named_bar_sync(3 + wc, 256);
#pragma unroll
      for (int j = 0; j < kResBN / 2; ++j) acc[j] = 0.f;
      // k blocks 0 .. nkb-2 take four k16 steps and the last one the K tail, peeled so that the group left in flight never
      // crosses into a run-time branch (ptxas would serialise every wgmma).  A k block's stage is free once its group is done.
      auto wait_full = [&](int kb) {
        const long long f = i * p.nkb + kb;
        mbar_wait(&full[f % kResStages], (uint32_t)(f / kResStages) & 1u);
        fence_acc<kResBN / 2>(acc);
        wgmma_fence();
        return smem_u32(ring + (size_t)(f % kResStages) * kResStage);
      };
      auto release_prev = [&](int kb) {  // after k block kb's group is committed: release k block kb - 1
        if (kb == 0) return;
        wgmma_wait<1>();
        fence_acc<kResBN / 2>(acc);
        release_stage<CTAS>(&empty[(i * p.nkb + kb - 1) % kResStages], lane);
      };
      const int kt = p.nkb - 1;
      for (int kb = 0; kb < kt; ++kb) {
        const uint32_t sa = wait_full(kb);
        mma_kblock<kResBN, 4>(acc, sa, sw0 + (uint32_t)(2 * kb) * kResWPlane, kResAPlane, kResWPlane);
        wgmma_commit();
        release_prev(kb);
      }
      {
        const uint32_t sa = wait_full(kt), sw = sw0 + (uint32_t)(2 * kt) * kResWPlane;
        switch (p.tail_steps) {
          case 1: mma_kblock<kResBN, 1>(acc, sa, sw, kResAPlane, kResWPlane); break;
          case 2: mma_kblock<kResBN, 2>(acc, sa, sw, kResAPlane, kResWPlane); break;
          case 3: mma_kblock<kResBN, 3>(acc, sa, sw, kResAPlane, kResWPlane); break;
          default: mma_kblock<kResBN, 4>(acc, sa, sw, kResAPlane, kResWPlane); break;
        }
        wgmma_commit();
        release_prev(kt);
      }
      if (i + 1 < n_mine) named_bar_arrive(3 + (1 - wc), 256);  // hand the tensor pipe to unit i + 1
      wgmma_wait<0>();
      fence_acc<kResBN / 2>(acc);
      release_stage<CTAS>(&empty[(i * p.nkb + kt) % kResStages], lane);

      // ---- epilogue: + type-bias row, one head at a time through the staging buffer, stored with TMA (clipped at M)
      const long long row_g = (first + i * walkers) * 64 + rl;
      const int r0 = (int)(row_g - rl);
      int boff[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        long long c = row_g + 8 * h < p.M ? p.row_class[row_g + 8 * h] : 0;
        c = c < 0 ? 0 : (c >= p.n_class ? p.n_class - 1 : c);
        boff[h] = (int)c * p.class_stride;
      }
      for (int h0 = 0; h0 < p.n_step; h0 += DP) {
        if (tid == 0) bulk_wait_read<0>();  // the previous store has read the buffer
        wg_bar(1 + wc);
#pragma unroll
        for (int j = 0; j < kResBN / 8; ++j) {
          const int c = 8 * j + q2;  // DP is even: a column pair never straddles two heads
          if (c < h0 || c >= h0 + DP) continue;
          const int gc = n0 + c;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float v0 = acc[4 * j + 2 * h] + __ldg(p.bias + boff[h] + gc);
            const float v1 = acc[4 * j + 2 * h + 1] + __ldg(p.bias + boff[h] + gc + 1);
            st_shared_f2(buf + 4u * (uint32_t)((rl + 8 * h) * DP + c - h0), v0, v1);
          }
        }
        fence_proxy_async();
        wg_bar(1 + wc);
        if (tid == 0) {
          tma_store_3d(&p.st_f32, staging + (size_t)wc * kStBytes, 0, r0, (n0 + h0) / DP);
          bulk_commit();
        }
      }
    }
    if (tid == 0) bulk_wait_all();  // no store still reads the staging buffers when the CTA exits
  }
  __syncthreads();
  if (CTAS == 2) cluster_sync_all();  // the peer's multicasts and remote arrivals target this CTA: nobody leaves early
}

__global__ void split_bf16_kernel(const float* __restrict__ a, int lda, long long M, int K, __nv_bfloat16* __restrict__ hi,
                                  __nv_bfloat16* __restrict__ lo, int ldp) {
  const long long total = M * (long long)(K / 2);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / (K / 2);
    const int c = (int)(i % (K / 2)) * 2;
    const float2 v = *reinterpret_cast<const float2*>(a + r * lda + c);
    const __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y);
    __nv_bfloat162 hh, ll;
    hh.x = h0; hh.y = h1;
    ll.x = __float2bfloat16_rn(v.x - __bfloat162float(h0));
    ll.y = __float2bfloat16_rn(v.y - __bfloat162float(h1));
    *reinterpret_cast<__nv_bfloat162*>(hi + r * ldp + c) = hh;
    if (lo != nullptr) *reinterpret_cast<__nv_bfloat162*>(lo + r * ldp + c) = ll;
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return (EncodeTiledFn)f;
  }();
  return fn;
}

// [rows, K] bf16 row-major (ld elements) -> 2-D tensor map with a {64, box_rows} box, 128-byte swizzle; out-of-range
// rows and columns of a box are zero-filled
bool make_map(CUtensorMap* m, const void* base, long long rows, int K, int ld, int box_rows) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Epilogue store map: [planes][rows][inner] elements (rows `ld` elements apart, planes `rows` rows apart), a box of
// box_w x 64 x 1, no swizzle.  A store writes only the part of its box inside the extents.
bool make_store_map(CUtensorMap* m, CUtensorMapDataType type, int esize, void* base, int inner, long long rows, int planes,
                    int ld, int box_w) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) return false;
  cuuint64_t dims[3] = {(cuuint64_t)inner, (cuuint64_t)rows, (cuuint64_t)planes};
  cuuint64_t strides[2] = {(cuuint64_t)ld * esize, (cuuint64_t)rows * ld * esize};
  cuuint32_t box[3] = {(cuuint32_t)box_w, 64, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(m, type, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
             CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Largest chunk width 8 <= w <= max_w that divides span and is a multiple of align > 0 (0: none).
int chunk_width(int span, int align, int max_w) {
  for (int w = span < max_w ? span : max_w; w >= 8; --w)
    if (span % w == 0 && w % align == 0) return w;
  return 0;
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// Launches one persistent instantiation; attr_set / max_clusters are that instantiation's per-device caches.
template <typename Params>
int32_t launch_persistent(void (*kernel)(Params), int ctas, cudaLaunchConfig_t cfg, const Params& p, bool* attr_set,
                          int* max_clusters) {
  const int dev = current_device();
  if (!attr_set[dev]) {  // the attribute is per device
    QAGNN_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemCap));
    attr_set[dev] = true;
  }
  if (ctas > 1) {
    // a CTA pair must sit in one GPC, so fewer than #SM / 2 pairs may fit at once; the tiles are walked persistently, and
    // pairs beyond what is resident would only start as a second wave.  Launch at most the resident count.
    if (max_clusters[dev] == 0) {
      cudaLaunchConfig_t q = cfg;
      int n = 0;
      QAGNN_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&n, kernel, &q));
      max_clusters[dev] = n > 0 ? n : 1;
      if (getenv("QAGNN_DEBUG")) fprintf(stderr, "gemm_tc: %d CTA pairs resident at %zu B of shared memory\n", n, cfg.dynamicSmemBytes);
    }
    if (cfg.gridDim.x > (unsigned)(max_clusters[dev] * ctas)) cfg.gridDim.x = (unsigned)(max_clusters[dev] * ctas);
  }
  QAGNN_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
  return QAGNN_OK;
}

template <int ACT, int BN, int CTAS, int P>
int32_t launch(cudaLaunchConfig_t cfg, const TcParams& p) {
  static bool attr_set[kMaxDevices] = {false};
  static int max_clusters[kMaxDevices] = {0};
  return launch_persistent(P == 3 ? gemm_tc_kernel<ACT, BN, CTAS> : gemm_bf16_kernel<ACT, BN, CTAS>, CTAS, cfg, p, attr_set,
                           max_clusters);
}

template <int ACT, int CTAS, int P>
int32_t launch_mlp(cudaLaunchConfig_t cfg, const MlpParams& p) {
  static bool attr_set[kMaxDevices] = {false};
  static int max_clusters[kMaxDevices] = {0};
  return launch_persistent(P == 3 ? mlp_tc_kernel<ACT, CTAS> : mlp_bf16_kernel<ACT, CTAS>, CTAS, cfg, p, attr_set, max_clusters);
}

template <int BN, int CTAS, int P>
int32_t launch_act(Act act, const cudaLaunchConfig_t& cfg, const TcParams& p) {
  if (act == ACT_NONE) return launch<ACT_NONE, BN, CTAS, P>(cfg, p);
  if (act == ACT_RELU) return launch<ACT_RELU, BN, CTAS, P>(cfg, p);
  return launch<ACT_GELU, BN, CTAS, P>(cfg, p);
}

template <int BN>
int32_t launch_bn(int ctas, int passes, Act act, const cudaLaunchConfig_t& cfg, const TcParams& p) {
  if (passes == 1) return ctas == 2 ? launch_act<BN, 2, 1>(act, cfg, p) : launch_act<BN, 1, 1>(act, cfg, p);
  return ctas == 2 ? launch_act<BN, 2, 3>(act, cfg, p) : launch_act<BN, 1, 3>(act, cfg, p);
}

template <int CTAS, int P>
int32_t launch_mlp_act(Act act2, const cudaLaunchConfig_t& cfg, const MlpParams& p) {
  if (act2 == ACT_NONE) return launch_mlp<ACT_NONE, CTAS, P>(cfg, p);
  if (act2 == ACT_RELU) return launch_mlp<ACT_RELU, CTAS, P>(cfg, p);
  return launch_mlp<ACT_GELU, CTAS, P>(cfg, p);
}

// default: CTA pairs (cluster of 2, W tile multicast, half loaded by each); QAGNN_TC_2CTA=0 -> single CTAs.
// Read at every call so that a test can cover both in one process.
int tc_ctas() {
  const char* e = getenv("QAGNN_TC_2CTA");
  return (e && atoi(e) == 0) ? 1 : 2;
}

// default: the epilogue stores through shared memory with TMA; QAGNN_TC_STORE=direct -> stores straight from the registers
// (the same values, bit for bit).  Read at every call, so that one process can compare and time both.
bool tc_store_tma() {
  const char* e = getenv("QAGNN_TC_STORE");
  return !(e && strcmp(e, "direct") == 0);
}

int32_t sm_count(int* sms) {
  static int sms_c[kMaxDevices] = {0};
  const int dev = current_device();
  if (sms_c[dev] == 0) QAGNN_CHECK_CUDA(cudaDeviceGetAttribute(&sms_c[dev], cudaDevAttrMultiProcessorCount, dev));
  *sms = sms_c[dev];
  return QAGNN_OK;
}

}  // namespace

bool gemm_tc_available() {  // QAGNN_GEMM=ffma forces the exact-fp32 FFMA path (read at every call: tests cover both)
  const char* e = getenv("QAGNN_GEMM");
  const bool forced_off = e && strcmp(e, "ffma") == 0;
  return !forced_off && encode_fn() != nullptr;
}

bool gemm_tc_shape_ok(int K1, int K2, int lda1, int lda2, int ldw, int N) {
  // TMA needs 16-byte row strides (ld % 8); K itself may be anything (the tensor map clips and zero-fills), but the second
  // segment's weight columns start at K1, which the k-block arithmetic wants even
  return K1 > 0 && K1 % 2 == 0 && K2 >= 0 && lda1 % 8 == 0 && (K2 == 0 || lda2 % 8 == 0) && ldw % 8 == 0 && N >= 8;
}

int hm_n_step(const HeadMajorOut& hm) {
  // the epilogue stores column pairs, so a tile must start on an even column: DP even keeps every tile start even
  if (hm.DP <= 0 || hm.DP % 2 != 0 || hm.H <= 0) return 0;
  for (int hpt = hm.H; hpt >= 1; --hpt)
    if (hm.H % hpt == 0 && hpt * hm.DP <= 256) return hpt * hm.DP;
  return 0;
}

// lo may be null: the hi plane alone (the single-pass GEMM's operand)
int32_t split_bf16(const float* a, int lda, long long M, int K, void* hi, void* lo, int ldp, cudaStream_t st) {
  if (M <= 0 || K <= 0) return QAGNN_OK;
  if (K % 2 != 0 || lda % 2 != 0) return QAGNN_ERR_UNSUPPORTED;
  long long g = (M * (K / 2) + 255) / 256;
  if (g > kNumSMs * 32) g = kNumSMs * 32;
  split_bf16_kernel<<<(unsigned)g, 256, 0, st>>>(a, lda, M, K, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ldp);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

int32_t gemm_tc(const TcOperand& A1, const TcOperand& A2, const TcOperand& W, const float* bias, long long M, int N, Act act,
                const TcOutput& out, cudaStream_t st, int passes) {
  if (M <= 0 || N <= 0) return QAGNN_OK;
  if (!gemm_tc_available()) return QAGNN_ERR_UNSUPPORTED;
  if (passes != 1 && passes != 3) return QAGNN_ERR_INVALID_ARGUMENT;
  const bool single = passes == 1;
  const int K1 = A1.K, K2 = A2.hi ? A2.K : 0;
  if (!gemm_tc_shape_ok(K1, K2, A1.ld, A2.ld, W.ld, N)) return QAGNN_ERR_UNSUPPORTED;
  TcParams p;
  memset(&p, 0, sizeof(p));
  int n_tiles = (N + 255) / 256;  // wgmma N <= 256
  p.n_step = (N + n_tiles - 1) / n_tiles;
  p.n_step = (p.n_step + 15) / 16 * 16;  // even columns per thread pair; half tiles of whole 8-row swizzle groups
  if (out.hm_buf != nullptr) {  // n tiles of whole heads: hpt heads (hpt | H) of DP padded columns each
    p.n_step = hm_n_step(out.hm);
    if (p.n_step == 0 || N % p.n_step != 0) return QAGNN_ERR_UNSUPPORTED;
    n_tiles = N / p.n_step;
  }
  // wgmma tile width: the smallest compiled one that covers n_step (208 = the H*DP and D of the QA-GNN shapes)
  const int bn = p.n_step <= 64 ? 64 : p.n_step <= 128 ? 128 : p.n_step <= 208 ? 208 : 256;
  p.N = N;
  p.M = M;
  p.nseg = K2 > 0 ? 2 : 1;
  p.kseg[0] = K1;
  p.kseg[1] = K2;
  const int CTAS = tc_ctas();
  const int stages = ring_stages(bn, passes);
  p.stages = stages;
  const size_t smem_bytes = stages * ring_stage_bytes(bn, passes) + kCtrlBytes + 2 * st_bufs(bn) * kStBytes;
  bool ok = make_map(&p.a_hi[0], A1.hi, M, K1, A1.ld, BM) && (single || make_map(&p.a_lo[0], A1.lo, M, K1, A1.ld, BM));
  if (K2 > 0)
    ok = ok && make_map(&p.a_hi[1], A2.hi, M, K2, A2.ld, BM) && (single || make_map(&p.a_lo[1], A2.lo, M, K2, A2.ld, BM));
  ok = ok && make_map(&p.w_hi, W.hi, N, K1 + K2, W.ld, bn / CTAS) &&
       (single || make_map(&p.w_lo, W.lo, N, K1 + K2, W.ld, bn / CTAS));
  if (!ok) return QAGNN_ERR_CUDA;
  if ((out.f32 && (out.ldc % 4 != 0)) || (out.hi && (out.ldp % 8 != 0))) return QAGNN_ERR_UNSUPPORTED;
  p.bias = bias;
  p.row_class = bias != nullptr ? out.row_class : nullptr;
  p.class_stride = out.class_stride;
  p.n_class = out.n_class > 0 ? out.n_class : 1;
  p.c_f32 = out.f32;
  p.ldc = out.ldc;
  p.c_hm = out.hm_buf;
  p.hm = out.hm;
  p.c_hi = (__nv_bfloat16*)out.hi;
  p.c_lo = single ? nullptr : (__nv_bfloat16*)out.lo;
  p.ldp = out.ldp;
  if (tc_store_tma()) {
    // chunks of whole tile columns that never cross a head (head-major) or the tile's n_step: a box must not reach the
    // neighbouring tile's columns.  Box rows of 16-byte multiples: fp32 chunks of 4 columns, bf16 chunks of 8; with one
    // staging buffer a chunk must not share a fragment column group with the next, so multiples of 8.
    const bool f32_out = out.hm_buf != nullptr || out.f32 != nullptr, pl_out = out.hi != nullptr;
    const int col_bytes = 64 * ((f32_out ? 4 : 0) + (pl_out ? 2 * planes_of(passes) : 0));
    const int span = out.hm_buf != nullptr ? out.hm.DP : p.n_step;
    const bool addressable = (!out.hm_buf || aligned16(out.hm_buf)) && (!out.f32 || aligned16(out.f32)) &&
                             (!pl_out || (aligned16(out.hi) && (single || aligned16(out.lo))));
    const int w = addressable && (f32_out || pl_out) ? chunk_width(span, pl_out || st_bufs(bn) == 1 ? 8 : 4, (int)kStBytes / col_bytes) : 0;
    if (w > 0) {
      bool sok = true;
      if (out.hm_buf != nullptr)
        sok = make_store_map(&p.st_f32, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, out.hm_buf, out.hm.DP, M, N / out.hm.DP,
                             out.hm.DP, w);
      else if (out.f32 != nullptr)
        sok = make_store_map(&p.st_f32, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, out.f32, N, M, 1, out.ldc, w);
      if (pl_out)
        sok = sok && make_store_map(&p.st_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, out.hi, N, M, 1, out.ldp, w) &&
              (single || make_store_map(&p.st_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, out.lo, N, M, 1, out.ldp, w));
      if (!sok) return QAGNN_ERR_CUDA;
      p.st_w = w;
      p.st_chunks = p.n_step / w;
    }
  }
  int sms = 0;
  QAGNN_RETURN_IF(sm_count(&sms));
  const long long total_tiles = (long long)n_tiles * ((M + (long long)BM * CTAS - 1) / ((long long)BM * CTAS));
  const long long units = total_tiles < sms / CTAS ? total_tiles : sms / CTAS;  // CTAs (or CTA pairs) to launch
  const unsigned grid = (unsigned)(units * CTAS);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute lattr[1];
  lattr[0].id = cudaLaunchAttributeClusterDimension;
  lattr[0].val.clusterDim.x = CTAS;
  lattr[0].val.clusterDim.y = 1;
  lattr[0].val.clusterDim.z = 1;
  cfg.attrs = lattr;
  cfg.numAttrs = CTAS == 2 ? 1 : 0;
  if (getenv("QAGNN_DEBUG")) fprintf(stderr, "gemm_tc: M=%lld N=%d K1=%d K2=%d act=%d CTAS=%d passes=%d stages=%d smem=%zu grid=%u bn=%d n_step=%d n_tiles=%d st_w=%d\n", M, N, K1, K2, (int)act, CTAS, passes, stages, smem_bytes, grid, bn, p.n_step, n_tiles, p.st_w);
  int32_t rc;
  if (bn == 64) rc = launch_bn<64>(CTAS, passes, act, cfg, p);
  else if (bn == 128) rc = launch_bn<128>(CTAS, passes, act, cfg, p);
  else if (bn == 208) rc = launch_bn<208>(CTAS, passes, act, cfg, p);
  else rc = launch_bn<256>(CTAS, passes, act, cfg, p);
  QAGNN_RETURN_IF(rc);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

// default: the fast-form projection runs proj_resident_kernel where it fits; QAGNN_PROJ_RESIDENT=0 -> gemm_tc_kernel.
// Read at every call, so that tests and A/B runs cover both paths in one process.
static bool proj_resident_enabled() {
  const char* e = getenv("QAGNN_PROJ_RESIDENT");
  return !(e && atoi(e) == 0);
}

// slice width: hpt * DP for the largest divisor hpt of H with hpt * DP <= 104; 0 when one head's fp32 columns of a 64-row
// unit overflow a staging buffer or its TMA-store rows are not 16-byte multiples
static int proj_resident_n_step(const HeadMajorOut& hm) {
  if (hm.H <= 0 || hm.DP <= 0 || hm.DP % 4 != 0 || 64u * hm.DP * 4 > kStBytes) return 0;
  for (int hpt = hm.H; hpt >= 1; --hpt)
    if (hm.H % hpt == 0 && hpt * hm.DP <= kResBN) return hpt * hm.DP;
  return 0;
}

static bool proj_resident_ok(const TcOperand& A, const TcOperand& W, const float* bias, int N, const TcOutput& out, int passes) {
  if (!proj_resident_enabled() || !gemm_tc_available() || passes != 3) return false;
  if (out.hm_buf == nullptr || !aligned16(out.hm_buf) || bias == nullptr || out.row_class == nullptr) return false;
  const int n_step = proj_resident_n_step(out.hm);
  return n_step > 0 && N % n_step == 0 && (A.K + BK - 1) / BK <= kResMaxKb && W.K == A.K &&
         gemm_tc_shape_ok(A.K, 0, A.ld, 0, W.ld, N);
}

int32_t proj_resident(const TcOperand& A, const TcOperand& W, const float* bias, long long M, int N, const TcOutput& out,
                      cudaStream_t st) {
  if (M <= 0) return QAGNN_OK;
  if (!proj_resident_ok(A, W, bias, N, out, 3)) return QAGNN_ERR_UNSUPPORTED;
  const int CTAS = tc_ctas();
  ResParams p;
  memset(&p, 0, sizeof(p));
  p.n_step = proj_resident_n_step(out.hm);
  p.DP = out.hm.DP;
  const int slices = N / p.n_step;
  // CTA pairs hold two slices of the same rows; an odd slice count runs on single CTAs
  const int ctas = slices % 2 == 0 ? CTAS : 1;
  p.groups = slices / ctas;
  p.nkb = (A.K + BK - 1) / BK;
  p.tail_steps = (A.K - 1) % BK / 16 + 1;
  p.M = M;
  p.bias = bias;
  p.row_class = out.row_class;
  p.class_stride = out.class_stride;
  p.n_class = out.n_class > 0 ? out.n_class : 1;
  bool ok = make_map(&p.a_hi, A.hi, M, A.K, A.ld, 64) && make_map(&p.a_lo, A.lo, M, A.K, A.ld, 64) &&
            make_map(&p.w_hi, W.hi, N, W.K, W.ld, kResBN) && make_map(&p.w_lo, W.lo, N, W.K, W.ld, kResBN) &&
            make_store_map(&p.st_f32, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, out.hm_buf, p.DP, M, N / p.DP, p.DP, p.DP);
  if (!ok) return QAGNN_ERR_CUDA;

  void (*kernel)(ResParams) = ctas == 2 ? proj_resident_kernel<2> : proj_resident_kernel<1>;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = kResSmem;
  cfg.stream = st;
  cudaLaunchAttribute lattr[1];
  lattr[0].id = cudaLaunchAttributeClusterDimension;
  lattr[0].val.clusterDim.x = ctas;
  lattr[0].val.clusterDim.y = 1;
  lattr[0].val.clusterDim.z = 1;
  cfg.attrs = lattr;
  cfg.numAttrs = ctas == 2 ? 1 : 0;
  // resident CTAs (pairs), per device and CTA setting: every slice group gets the same number of walkers, so the groups
  // read each unit of A at about the same time
  static bool attr_set[2][kMaxDevices] = {{false}};
  static int resident[2][kMaxDevices] = {{0}};
  const int dev = current_device(), ci = ctas - 1;
  if (!attr_set[ci][dev]) {
    QAGNN_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kResSmem));
    attr_set[ci][dev] = true;
  }
  if (resident[ci][dev] == 0) {
    int n = 0;
    if (ctas == 2) {
      cudaLaunchConfig_t q = cfg;
      q.gridDim = dim3(2);
      QAGNN_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&n, kernel, &q));
    } else {
      QAGNN_RETURN_IF(sm_count(&n));
    }
    resident[ci][dev] = n > 0 ? n : 1;
  }
  const long long units = (M + 63) / 64;
  long long walkers = resident[ci][dev] / p.groups;
  if (walkers > units) walkers = units;
  if (walkers < 1) return QAGNN_ERR_UNSUPPORTED;  // fewer resident CTAs than slices (not on an H100)
  cfg.gridDim = dim3((unsigned)(walkers * p.groups * ctas));
  if (getenv("QAGNN_DEBUG")) fprintf(stderr, "proj_resident: M=%lld N=%d K=%d CTAS=%d slices=%d n_step=%d grid=%u smem=%zu\n", M, N, A.K, ctas, slices, p.n_step, cfg.gridDim.x, kResSmem);
  QAGNN_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

bool mlp_tc_shape_ok(int D) { return D >= 8 && D % 8 == 0 && D <= kMlpMaxD; }

int32_t mlp_tc(const TcOperand& A, const TcOperand& W1, const float* b1, const TcOperand& W2, const float* b2, long long M,
               Act act2, const TcOutput& out, cudaStream_t st, int passes) {
  if (M <= 0) return QAGNN_OK;
  if (!gemm_tc_available()) return QAGNN_ERR_UNSUPPORTED;
  if (passes != 1 && passes != 3) return QAGNN_ERR_INVALID_ARGUMENT;
  const bool single = passes == 1;
  const int D = A.K;
  if (!mlp_tc_shape_ok(D) || W1.K != D || W2.K != D || b1 == nullptr || b2 == nullptr) return QAGNN_ERR_UNSUPPORTED;
  if (A.ld % 8 != 0 || W1.ld % 8 != 0 || W2.ld % 8 != 0) return QAGNN_ERR_UNSUPPORTED;
  if (out.hm_buf != nullptr || out.row_class != nullptr) return QAGNN_ERR_UNSUPPORTED;
  if ((out.f32 && (out.ldc % 4 != 0)) || (out.hi && (out.ldp % 8 != 0))) return QAGNN_ERR_UNSUPPORTED;
  const int CTAS = tc_ctas();
  MlpParams p;
  memset(&p, 0, sizeof(p));
  const int stages = mlp_ring_stages(passes);
  const size_t smem_bytes = stages * ring_stage_bytes(kMlpMaxD, passes) + kCtrlBytes + 2 * kMlpStBytes;
  bool ok = make_map(&p.a_hi, A.hi, M, D, A.ld, BM) && (single || make_map(&p.a_lo, A.lo, M, D, A.ld, BM));
  ok = ok && make_map(&p.w1_hi, W1.hi, D, D, W1.ld, kMlpMaxD / CTAS) &&
       (single || make_map(&p.w1_lo, W1.lo, D, D, W1.ld, kMlpMaxD / CTAS));
  ok = ok && make_map(&p.w2_hi, W2.hi, D, D, W2.ld, kMlpChunk) && (single || make_map(&p.w2_lo, W2.lo, D, D, W2.ld, kMlpChunk));
  if (!ok) return QAGNN_ERR_CUDA;
  p.D = D;
  p.stages = stages;
  p.M = M;
  p.b1 = b1;
  p.b2 = b2;
  p.c_f32 = out.f32;
  p.ldc = out.ldc;
  p.c_hi = (__nv_bfloat16*)out.hi;
  p.c_lo = single ? nullptr : (__nv_bfloat16*)out.lo;
  p.ldp = out.ldp;
  // rows are 16-byte multiples (ldc % 4, ldp % 8 above); the bases must be 16-byte aligned too
  if (tc_store_tma() && (out.f32 || out.hi) && (!out.f32 || aligned16(out.f32)) &&
      (!out.hi || (aligned16(out.hi) && (single || aligned16(out.lo))))) {
    bool sok = true;
    if (out.f32) sok = make_store_map(&p.st_f32, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, out.f32, D, M, 1, out.ldc, kMlpChunk);
    if (out.hi)
      sok = sok && make_store_map(&p.st_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, out.hi, D, M, 1, out.ldp, kMlpChunk) &&
            (single || make_store_map(&p.st_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, out.lo, D, M, 1, out.ldp, kMlpChunk));
    if (!sok) return QAGNN_ERR_CUDA;
    p.tma_store = 1;
  }
  int sms = 0;
  QAGNN_RETURN_IF(sm_count(&sms));
  const long long total_tiles = (M + (long long)BM * CTAS - 1) / ((long long)BM * CTAS);
  const long long units = total_tiles < sms / CTAS ? total_tiles : sms / CTAS;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(units * CTAS));
  cfg.blockDim = dim3(kMlpThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute lattr[1];
  lattr[0].id = cudaLaunchAttributeClusterDimension;
  lattr[0].val.clusterDim.x = CTAS;
  lattr[0].val.clusterDim.y = 1;
  lattr[0].val.clusterDim.z = 1;
  cfg.attrs = lattr;
  cfg.numAttrs = CTAS == 2 ? 1 : 0;
  if (getenv("QAGNN_DEBUG")) fprintf(stderr, "mlp_tc: M=%lld D=%d act2=%d CTAS=%d passes=%d stages=%d smem=%zu grid=%u\n", M, D, (int)act2, CTAS, passes, stages, smem_bytes, cfg.gridDim.x);
  int32_t rc;
  if (single) rc = CTAS == 2 ? launch_mlp_act<2, 1>(act2, cfg, p) : launch_mlp_act<1, 1>(act2, cfg, p);
  else rc = CTAS == 2 ? launch_mlp_act<2, 3>(act2, cfg, p) : launch_mlp_act<1, 3>(act2, cfg, p);
  QAGNN_RETURN_IF(rc);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

}  // namespace qagnn
