// Keyed dropout (qagnn_keyed_dropout_forward_typed / _backward_typed; qagnn_b200.training.keyed_dropout): a mask that is a
// pure function of what is dropped, not of how many launches ran before it.  x and y are contiguous [A, G, L]; element
// (a, g, l) belongs to question qids[g / nc], choice g % nc, and has the in-graph index e = a L + l.  Its uniform is word
// e & 3 of Philox4x32-10 with
//   key     = (seed lo 32, seed hi 32)
//   counter = (e >> 2, site + 256 choice, question id lo 32, draw lo 32)
// and it is kept when u >= T = min(floor(p 2^32), 2^32 - 1) (none is kept at p = 1).  A kept value is x * scale rounded once
// to the storage type, scale = (float)(1 / (1 - p)); a dropped one is 0.  The forward also writes the keep bits over the
// flat index (bit i of word i / 32), so the backward needs only them: dx = kept ? dy * scale : 0.
//
// A thread owns 4 consecutive flat elements.  When they are one row's and one Philox block's (always when L % 4 == 0), it
// draws once and moves them with one 4-wide load and store; otherwise (row ends, blocks split by L % 4 != 0) it walks them
// one by one and draws once per block it meets.  A warp's 128 elements give 4 mask words, built from 4 ballots.
#include <algorithm>
#include <cmath>

#include "storage.cuh"

namespace qagnn {

namespace {

constexpr int kThreads = 256;
constexpr int64_t kMaxElements = (int64_t)1 << 31;  // 32-bit row arithmetic in the kernels

// Philox4x32-10 (Salmon et al., SC'11), the generator of Random123 and cuRAND's curand_Philox4x32_10
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k.x += 0x9E3779B9u;
      k.y += 0xBB67AE85u;
    }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

__device__ __forceinline__ uint32_t word(const uint4& r, uint32_t j) {
  return j == 0 ? r.x : j == 1 ? r.y : j == 2 ? r.z : r.w;
}

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename S> __device__ __forceinline__ S from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// bit k of the low byte to bit 4k
__device__ __forceinline__ uint32_t spread4(uint32_t x) {
  x &= 0xffu;
  x = (x | (x << 12)) & 0x000F000Fu;
  x = (x | (x << 6)) & 0x03030303u;
  return (x | (x << 3)) & 0x11111111u;
}

struct FwdArgs {
  const void* x;
  void* y;
  uint32_t* mask;
  const int64_t* draw;
  const int64_t* qids;
  int64_t n;        // A G L
  uint32_t L, G, nc, site;
  uint32_t thresh;  // keep when u >= thresh
  int32_t drop_all; // p = 1
  int32_t vec;      // x and y 4-element aligned
  float scale;
  uint2 key;
};

template <typename S>
__global__ void __launch_bounds__(kThreads) keyed_dropout_forward_kernel(const __grid_constant__ FwdArgs a) {
  const S* x = static_cast<const S*>(a.x);
  S* y = static_cast<S*>(a.y);
  const uint32_t draw = (uint32_t)(uint64_t)*a.draw;
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * kThreads * 4;
  const int64_t words = (a.n + 31) >> 5;
  // the loop runs on the warp's first element, so every lane takes the same trips and the ballots see the whole warp
  for (int64_t base = ((int64_t)blockIdx.x * kThreads + (threadIdx.x & ~31)) * 4; base < a.n; base += stride) {
    const int64_t i0 = base + 4 * lane;
    uint32_t keep = 0;
    if (i0 < a.n) {
      uint32_t row = (uint32_t)i0 / a.L, l = (uint32_t)i0 - row * a.L;
      uint32_t ai = row / a.G, g = row - ai * a.G;
      const uint32_t e0 = ai * a.L + l;
      if (a.vec && i0 + 3 < a.n && l + 3 < a.L && (e0 & 3) == 0) {
        const uint32_t q = g / a.nc;
        const uint4 r = philox4x32_10(make_uint4(e0 >> 2, a.site + 256u * (g - q * a.nc), (uint32_t)a.qids[q], draw), a.key);
        keep = a.drop_all ? 0u
                          : (uint32_t)(r.x >= a.thresh) | (uint32_t)(r.y >= a.thresh) << 1 |
                                (uint32_t)(r.z >= a.thresh) << 2 | (uint32_t)(r.w >= a.thresh) << 3;
        const float4 v = load4(x + i0);
        const float s = a.scale;
        store4(y + i0, make_float4(keep & 1 ? v.x * s : 0.f, keep & 2 ? v.y * s : 0.f, keep & 4 ? v.z * s : 0.f,
                                   keep & 8 ? v.w * s : 0.f));
      } else {
        uint4 r = make_uint4(0, 0, 0, 0);
        uint32_t have_row = ~0u, have_blk = ~0u;
        for (int j = 0; j < 4 && i0 + j < a.n; ++j) {
          const uint32_t e = ai * a.L + l;
          if (row != have_row || (e >> 2) != have_blk) {
            const uint32_t q = g / a.nc;
            r = philox4x32_10(make_uint4(e >> 2, a.site + 256u * (g - q * a.nc), (uint32_t)a.qids[q], draw), a.key);
            have_row = row;
            have_blk = e >> 2;
          }
          const bool k = !a.drop_all && word(r, e & 3) >= a.thresh;
          keep |= (uint32_t)k << j;
          y[i0 + j] = k ? from_f<S>(to_f(x[i0 + j]) * a.scale) : from_f<S>(0.f);
          if (++l == a.L) {
            l = 0;
            ++row;
            if (++g == a.G) {
              g = 0;
              ++ai;
            }
          }
        }
      }
    }
    const uint32_t b0 = __ballot_sync(~0u, keep & 1), b1 = __ballot_sync(~0u, keep & 2);
    const uint32_t b2 = __ballot_sync(~0u, keep & 4), b3 = __ballot_sync(~0u, keep & 8);
    // word w of the warp's 4 holds lanes 8w ... 8w + 7, 4 bits each: byte w of every ballot, interleaved
    const int64_t w = (base >> 5) + lane;
    if (lane < 4 && w < words) {
      const int sh = 8 * lane;
      a.mask[w] = spread4(b0 >> sh) | spread4(b1 >> sh) << 1 | spread4(b2 >> sh) << 2 | spread4(b3 >> sh) << 3;
    }
  }
}

struct BwdArgs {
  const uint32_t* mask;
  const void* dy;
  void* dx;
  int64_t n;
  int32_t vec;
  float scale;
};

template <typename S>
__global__ void __launch_bounds__(kThreads) keyed_dropout_backward_kernel(const __grid_constant__ BwdArgs a) {
  const S* dy = static_cast<const S*>(a.dy);
  S* dx = static_cast<S*>(a.dx);
  const float s = a.scale;
  for (int64_t i0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * 4; i0 < a.n; i0 += (int64_t)gridDim.x * kThreads * 4) {
    const uint32_t keep = a.mask[i0 >> 5] >> (i0 & 31);
    if (a.vec && i0 + 3 < a.n) {
      const float4 v = load4(dy + i0);
      store4(dx + i0, make_float4(keep & 1 ? v.x * s : 0.f, keep & 2 ? v.y * s : 0.f, keep & 4 ? v.z * s : 0.f,
                                  keep & 8 ? v.w * s : 0.f));
    } else {
      for (int j = 0; j < 4 && i0 + j < a.n; ++j)
        dx[i0 + j] = (keep >> j) & 1 ? from_f<S>(to_f(dy[i0 + j]) * s) : from_f<S>(0.f);
    }
  }
}

bool bad_p(double p) { return !(p >= 0.0 && p <= 1.0); }  // NaN too

float scale_of(double p) { return p < 1.0 ? (float)(1.0 / (1.0 - p)) : 0.f; }

int32_t elem_bytes(int32_t dtype) {
  return dtype == QAGNN_DTYPE_F32 ? 4 : (dtype == QAGNN_DTYPE_F16 || dtype == QAGNN_DTYPE_BF16) ? 2 : 0;
}

bool aligned4(const void* p, int32_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (uintptr_t)(4 * bytes - 1)) == 0; }

int grid_for(int64_t n) { return (int)std::min<int64_t>((n + 4 * kThreads - 1) / (4 * kThreads), (int64_t)kNumSMs * 16); }

template <typename S>
int32_t launch_fwd(const FwdArgs& a, cudaStream_t st) {
  keyed_dropout_forward_kernel<S><<<grid_for(a.n), kThreads, 0, st>>>(a);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

template <typename S>
int32_t launch_bwd(const BwdArgs& a, cudaStream_t st) {
  keyed_dropout_backward_kernel<S><<<grid_for(a.n), kThreads, 0, st>>>(a);
  QAGNN_CHECK_LAUNCH();
  return QAGNN_OK;
}

}  // namespace

}  // namespace qagnn

using namespace qagnn;

extern "C" int32_t qagnn_keyed_dropout_forward_typed(int32_t dtype, int64_t A, int64_t G, int64_t L, double p, int64_t seed,
                                                     const int64_t* draw, const int64_t* qids, int32_t nc, int32_t site,
                                                     const void* x, void* y, uint32_t* mask, void* stream) {
  const int32_t eb = elem_bytes(dtype);
  if (!eb || A < 0 || G < 0 || L < 0 || bad_p(p) || nc < 1 || nc > (1 << 23) || site < 0 || site > 255 || G % nc)
    return QAGNN_ERR_INVALID_ARGUMENT;
  if (A == 0 || G == 0 || L == 0) return QAGNN_OK;
  if (A > kMaxElements / G || A * G > kMaxElements / L) return QAGNN_ERR_UNSUPPORTED;
  if (!draw || !qids || !x || !y || !mask) return QAGNN_ERR_INVALID_ARGUMENT;
  FwdArgs a;
  a.x = x;
  a.y = y;
  a.mask = mask;
  a.draw = draw;
  a.qids = qids;
  a.n = A * G * L;
  a.L = (uint32_t)L;
  a.G = (uint32_t)G;
  a.nc = (uint32_t)nc;
  a.site = (uint32_t)site;
  a.thresh = (uint32_t)std::min(std::floor(p * 4294967296.0), 4294967295.0);
  a.drop_all = p >= 1.0;
  a.vec = aligned4(x, eb) && aligned4(y, eb);
  a.scale = scale_of(p);
  a.key = make_uint2((uint32_t)(uint64_t)seed, (uint32_t)((uint64_t)seed >> 32));
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case QAGNN_DTYPE_F32: return launch_fwd<float>(a, st);
    case QAGNN_DTYPE_F16: return launch_fwd<__half>(a, st);
    default: return launch_fwd<__nv_bfloat16>(a, st);
  }
}

extern "C" int32_t qagnn_keyed_dropout_backward_typed(int32_t dtype, int64_t n, double p, const uint32_t* mask, const void* dy,
                                                      void* dx, void* stream) {
  const int32_t eb = elem_bytes(dtype);
  if (!eb || n < 0 || bad_p(p)) return QAGNN_ERR_INVALID_ARGUMENT;
  if (n == 0) return QAGNN_OK;
  if (n > kMaxElements) return QAGNN_ERR_UNSUPPORTED;
  if (!mask || !dy || !dx) return QAGNN_ERR_INVALID_ARGUMENT;
  BwdArgs a;
  a.mask = mask;
  a.dy = dy;
  a.dx = dx;
  a.n = n;
  a.vec = aligned4(dy, eb) && aligned4(dx, eb);
  a.scale = scale_of(p);
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case QAGNN_DTYPE_F32: return launch_bwd<float>(a, st);
    case QAGNN_DTYPE_F16: return launch_bwd<__half>(a, st);
    default: return launch_bwd<__nv_bfloat16>(a, st);
  }
}
