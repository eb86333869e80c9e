// The body of gemm_tc_kernel (P = 3: split-bf16, three passes) and gemm_bf16_kernel (P = 1: the hi planes alone), included
// textually in both kernels (gemm_tc.cu) with ACT, BN, CTAS and P in scope and `p` the kernel's __grid_constant__ TcParams.
// A fragment rather than a device function on purpose: read through a `const TcParams&` in an inlined function, the
// parameter's loads compile differently (uniform constant loads become per-thread ones, selects become branches) and the
// split-bf16 instantiations lost their instruction-for-instruction identity with the kernel before the single pass existed;
// included here they keep it (the same count of every SASS opcode).  No include guard: it is included once per kernel.
  extern __shared__ __align__(1024) unsigned char smem[];
  constexpr int NP = planes_of(P);
  constexpr uint32_t a_bytes = BM * BK * 2;  // one A plane tile: 16 KB
  constexpr uint32_t w_bytes = BN * BK * 2;  // one W plane k block
  constexpr uint32_t stage_bytes = NP * a_bytes + NP * w_bytes;
  constexpr int kBufs = st_bufs(BN);
  static_assert(ring_stages(BN, P) >= 2, "the epilogue staging leaves room for two ring stages");
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const uint32_t rank = CTAS == 2 ? cluster_ctarank() : 0u;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * stage_bytes);  // [stages]  TMA -> MMA
  uint64_t* empty = full + p.stages;                                                      // [stages]  MMA -> TMA
  unsigned char* staging = smem + (size_t)p.stages * stage_bytes + kCtrlBytes;           // [2 warpgroups][kBufs]

  // k-blocks across the (up to two) A segments
  int nkb_seg[2];
  nkb_seg[0] = (p.kseg[0] + BK - 1) / BK;
  nkb_seg[1] = p.nseg > 1 ? (p.kseg[1] + BK - 1) / BK : 0;
  const int nkb = nkb_seg[0] + nkb_seg[1];
  // k16 steps of the last k block of each segment: only those that reach its K (the rest would multiply TMA's zero fill)
  const int tail_steps0 = (p.kseg[0] - 1) % BK / 16 + 1;
  const int tail_steps1 = nkb_seg[1] > 0 ? (p.kseg[1] - 1) % BK / 16 + 1 : BK / 16;
  const int n_tiles = (p.N + p.n_step - 1) / p.n_step;
  const long long total_tiles = (p.M + BM * CTAS - 1) / (BM * CTAS) * n_tiles;
  const long long cl_id = blockIdx.x / CTAS, n_cl = gridDim.x / CTAS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8 * CTAS);  // one arrival per consumer warp of every CTA whose W half lands here
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CTAS == 2) cluster_sync_all();  // the peer's barriers are initialised before any multicast or remote arrive

  if (wg == 0) {
    // ===================================== TMA producer =====================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (tid == 0) {
      long long it = 0;  // k-block counter across tiles
      for (long long tile = cl_id; tile < total_tiles; tile += n_cl) {
        const int n0 = (int)(tile % n_tiles) * p.n_step;
        const int m0 = (int)((tile / n_tiles) * BM * CTAS + rank * BM);
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = (int)(it % p.stages);
          // the stage is free once the consumers of BOTH CTAs have read it (the W half of this CTA lands in both)
          if (it >= p.stages) mbar_wait(&empty[s], (uint32_t)((it / p.stages) - 1) & 1u);
          const int seg = kb < nkb_seg[0] ? 0 : 1;
          const int k_in_seg = (seg == 0 ? kb : kb - nkb_seg[0]) * BK;
          const int k_glob = (seg == 0 ? 0 : p.kseg[0]) + k_in_seg;
          unsigned char* st = smem + (size_t)s * stage_bytes;
          mbar_expect_tx(&full[s], stage_bytes);
          tma_load_2d(st, &p.a_hi[seg], k_in_seg, m0, &full[s]);
          if constexpr (P == 3) tma_load_2d(st + a_bytes, &p.a_lo[seg], k_in_seg, m0, &full[s]);
          if (CTAS == 1) {
            tma_load_2d(st + NP * a_bytes, &p.w_hi, k_glob, n0, &full[s]);
            if constexpr (P == 3) tma_load_2d(st + 2 * a_bytes + w_bytes, &p.w_lo, k_glob, n0, &full[s]);
          } else {
            const uint32_t half = w_bytes / 2;
            tma_load_2d_multicast(st + NP * a_bytes + rank * half, &p.w_hi, k_glob, n0 + (int)rank * (BN / 2), &full[s], 3);
            if constexpr (P == 3)
              tma_load_2d_multicast(st + 2 * a_bytes + w_bytes + rank * half, &p.w_lo, k_glob, n0 + (int)rank * (BN / 2), &full[s], 3);
          }
        }
      }
    }
  } else {
    // ===================================== consumers (warpgroups 1, 2) =====================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wc = wg - 1;  // rows wc*64 .. wc*64+63 of the tile
    const int warp = tid >> 5, lane = tid & 31;
    // head-major epilogue: column c = 8j + 2(lane & 3) of a tile is element jj of head hh (c = hh * DP + jj).  The divisions
    // happen once here; the column loop carries (hh, jj) along.
    const bool hm_mode = p.c_hm != nullptr;
    const int DP = hm_mode ? p.hm.DP : 8;
    const int hh0 = 2 * (lane & 3) / DP, jj0 = 2 * (lane & 3) - hh0 * DP;
    const int q8 = 8 / DP, r8 = 8 - q8 * DP;
    float acc[BN / 2];
    long long it = 0;
    int st_it = 0;  // staged chunks so far: buffer st_it % kBufs
    for (long long tile = cl_id; tile < total_tiles; tile += n_cl) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = (int)(it % p.stages);
        mbar_wait(&full[s], (uint32_t)(it / p.stages) & 1u);
        const uint32_t sbase = smem_u32(smem + (size_t)s * stage_bytes);
        const uint32_t sa = sbase + (uint32_t)wc * 64 * 128, sw = sbase + NP * a_bytes;
        const int steps = kb == nkb_seg[0] - 1 ? tail_steps0 : kb == nkb - 1 ? tail_steps1 : BK / 16;
        fence_acc<BN / 2>(acc);
        wgmma_fence();
        // one compile-time chain per step count, each committing its own group
        switch (steps) {
          case 1: mma_kblock<BN, 1, P>(acc, sa, sw, a_bytes, w_bytes); wgmma_commit(); break;
          case 2: mma_kblock<BN, 2, P>(acc, sa, sw, a_bytes, w_bytes); wgmma_commit(); break;
          case 3: mma_kblock<BN, 3, P>(acc, sa, sw, a_bytes, w_bytes); wgmma_commit(); break;
          default: mma_kblock<BN, 4, P>(acc, sa, sw, a_bytes, w_bytes); wgmma_commit(); break;
        }
        wgmma_wait_all();
        fence_acc<BN / 2>(acc);
        release_stage<CTAS>(&empty[s], lane);
      }
      // ---- epilogue: thread holds rows g, g + 8 and column pairs 8j + 2q of the accumulator fragment
      const int n_tile = (int)(tile % n_tiles);
      const int n0 = n_tile * p.n_step;
      const long long row_g = (tile / n_tiles) * BM * CTAS + rank * BM + wc * 64 + warp * 16 + (lane >> 2);
      // head-major output: the tile's first column starts plane n0 / DP (= which * H + head) of [3][H][N][DP]
      const int hm_plane0 = hm_mode ? n0 / DP : 0;
      if (p.st_w > 0) {
        // through shared memory in chunks of W tile columns (W >= 8 divides n_step and, head-major, DP): the fragment is
        // walked in column order, as below, so each accumulator dies once written.  A chunk opens (its buffer free) in the
        // group that holds its first column and closes in the one that holds its last: thread 0 of the warpgroup then
        // stores its [64][W] fp32 / bf16 hi / bf16 lo boxes with TMA.  A group straddles two chunks only with two buffers.
        const int W = p.st_w;
        const int rl = warp * 16 + (lane >> 2);  // fragment rows rl, rl + 8 of the warpgroup's 64
        const int r0 = (int)(row_g - rl);
        int boff[2] = {0, 0};  // per-row bias table offsets
        if (p.bias != nullptr && p.row_class != nullptr) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            long long c = row_g + 8 * h < p.M ? p.row_class[row_g + 8 * h] : 0;
            c = c < 0 ? 0 : (c >= p.n_class ? p.n_class - 1 : c);
            boff[h] = (int)c * p.class_stride;
          }
        }
        const bool f32_out = hm_mode || p.c_f32 != nullptr, pl_out = p.c_hi != nullptr;
        const uint32_t f32_bytes = f32_out ? 64u * W * 4 : 0u, pl_bytes = 64u * W * 2;
        const uint32_t st0 = smem_u32(staging) + (uint32_t)wc * kBufs * kStBytes;
        int open_end = 0;  // columns [0, open_end) are in chunks opened so far
        int close_end = W;  // the oldest open chunk is [close_end - W, close_end)
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (8 * j >= p.n_step) break;
          if (open_end < 8 * j + 8) {  // a chunk starts here: wait until the store that read its buffer last is done
            if (tid == 0) {
              if (kBufs == 2 && open_end == close_end) bulk_wait_read<0>();  // the chunk before is still open
              else bulk_wait_read<kBufs - 1>();
            }
            wg_bar(1 + wc);
            open_end += W;
          }
          const int c = 8 * j + 2 * (lane & 3), gc = n0 + c;
          const bool second = c >= close_end;
          const uint32_t buf = st0 + (uint32_t)((st_it + (second ? 1 : 0)) % kBufs) * kStBytes;
          const int cc = c - (second ? close_end : close_end - W);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if (p.bias != nullptr) {  // columns from N on are clipped by the store
              if (gc < p.N) v0 += __ldg(p.bias + boff[h] + gc);
              if (gc + 1 < p.N) v1 += __ldg(p.bias + boff[h] + gc + 1);
            }
            v0 = act_fn<ACT>(v0);
            v1 = act_fn<ACT>(v1);
            const uint32_t e = (uint32_t)((rl + 8 * h) * W + cc);
            if (f32_out) st_shared_f2(buf + 4 * e, v0, v1);
            if (pl_out) {
              if constexpr (P == 3) {
                uint32_t hi, lo;
                split_pair(v0, v1, hi, lo);
                st_shared_u32(buf + f32_bytes + 2 * e, hi);
                st_shared_u32(buf + f32_bytes + pl_bytes + 2 * e, lo);
              } else {
                st_shared_u32(buf + f32_bytes + 2 * e, hi_pair(v0, v1));
              }
            }
          }
          if (close_end <= 8 * j + 8) {  // the oldest open chunk is complete
            fence_proxy_async();
            wg_bar(1 + wc);
            if (tid == 0) {
              const int cb = close_end - W;
              const unsigned char* b = staging + (size_t)(wc * kBufs + st_it % kBufs) * kStBytes;
              if (f32_out) {
                if (hm_mode) tma_store_3d(&p.st_f32, b, cb % DP, r0, hm_plane0 + cb / DP);
                else tma_store_3d(&p.st_f32, b, n0 + cb, r0, 0);
              }
              if (pl_out) {
                tma_store_3d(&p.st_hi, b + f32_bytes, n0 + cb, r0, 0);
                if constexpr (P == 3) tma_store_3d(&p.st_lo, b + f32_bytes + pl_bytes, n0 + cb, r0, 0);
              }
              bulk_commit();
            }
            close_end += W;
            ++st_it;
          }
        }
        continue;
      }
      // straight from the fragment to global memory (QAGNN_TC_STORE=direct, or outputs TMA cannot address)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = row_g + 8 * h;
        if (r >= p.M) continue;
        const float* bias_row = p.bias;  // per-row bias table (node-type classes)
        if (p.bias != nullptr && p.row_class != nullptr) {
          long long c = p.row_class[r];
          c = c < 0 ? 0 : (c >= p.n_class ? p.n_class - 1 : c);
          bias_row = p.bias + (size_t)c * p.class_stride;
        }
        int hh = hh0, jj = jj0;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (hm_mode && j > 0) {  // c += 8 = q8 heads + r8 columns, r8 < DP
            jj += r8;
            hh += q8;
            if (jj >= DP) { jj -= DP; ++hh; }
          }
          const int c = 8 * j + 2 * (lane & 3);  // tile column (even); n_step is even, so c + 1 < n_step too
          const int gc = n0 + c;
          if (c >= p.n_step || gc >= p.N) continue;
          const bool two = gc + 1 < p.N;
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (p.bias != nullptr) {  // bias is indexed by GEMM column (padded like the weight rows)
            v0 += __ldg(bias_row + gc);
            if (two) v1 += __ldg(bias_row + gc + 1);
          }
          v0 = act_fn<ACT>(v0);
          v1 = act_fn<ACT>(v1);
          if (hm_mode) {  // tile = whole heads of one `which`: column c is element jj of plane hm_plane0 + hh
            float* o = p.c_hm + ((size_t)(hm_plane0 + hh) * p.M + r) * DP + jj;
            *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
          } else if (p.c_f32 != nullptr) {
            float* o = p.c_f32 + (size_t)r * p.ldc + gc;
            if (two) *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
            else o[0] = v0;
          }
          if (p.c_hi != nullptr) {
            if constexpr (P == 3) {
              __nv_bfloat162 h2, l2;
              h2.x = __float2bfloat16_rn(v0);
              h2.y = __float2bfloat16_rn(v1);
              l2.x = __float2bfloat16_rn(v0 - __bfloat162float(h2.x));
              l2.y = __float2bfloat16_rn(v1 - __bfloat162float(h2.y));
              __nv_bfloat16* oh = p.c_hi + (size_t)r * p.ldp + gc;
              __nv_bfloat16* ol = p.c_lo + (size_t)r * p.ldp + gc;
              if (two) {
                *reinterpret_cast<__nv_bfloat162*>(oh) = h2;
                *reinterpret_cast<__nv_bfloat162*>(ol) = l2;
              } else {
                oh[0] = h2.x;
                ol[0] = l2.x;
              }
            } else {
              __nv_bfloat162 h2;
              h2.x = __float2bfloat16_rn(v0);
              h2.y = __float2bfloat16_rn(v1);
              __nv_bfloat16* oh = p.c_hi + (size_t)r * p.ldp + gc;
              if (two) *reinterpret_cast<__nv_bfloat162*>(oh) = h2;
              else oh[0] = h2.x;
            }
          }
        }
      }
    }
    if (tid == 0) bulk_wait_all();  // no store still reads the staging buffers when the CTA exits
  }
  __syncthreads();
  if (CTAS == 2) cluster_sync_all();  // the peer's multicasts and remote arrivals target this CTA: nobody leaves early
