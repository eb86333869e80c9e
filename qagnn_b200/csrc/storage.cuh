// Storage types of the training core's node and table operands (qagnn_mp_core_*_typed): fp32, fp16 or bf16 rows.
// Kernels templated on the storage type load 4 consecutive elements as one float4 (16-bit values widen exactly) and do
// all arithmetic in fp32; stores round to nearest even.  The fp32 overloads are plain float4 accesses.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace qagnn {

__device__ __forceinline__ float4 load4(const float* p) { return *reinterpret_cast<const float4*>(p); }
// 16-bit values are unpacked from the two 32-bit words of one 8-byte load with integer ops (no address of a register taken)
__device__ __forceinline__ float h2f(uint32_t bits) { return __half2float(__ushort_as_half((unsigned short)bits)); }

// The same 4 elements kept packed (float4 for fp32, the raw 8 bytes for 16-bit types) and widened where they are used: a
// kernel that holds rows in registers across a loop then needs half the registers for them
template <typename S> struct Packed4 { using type = uint2; };
template <> struct Packed4<float> { using type = float4; };
template <typename S> __device__ __forceinline__ typename Packed4<S>::type load_packed4(const S* p) {
  return *reinterpret_cast<const typename Packed4<S>::type*>(p);
}
template <typename S> __device__ __forceinline__ typename Packed4<S>::type zero_packed4() { return {}; }
template <> __device__ __forceinline__ float4 zero_packed4<float>() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float4 widen4(const float4& v, const float*) { return v; }
__device__ __forceinline__ float4 widen4(const uint2& u, const __half*) {
  return make_float4(h2f(u.x), h2f(u.x >> 16), h2f(u.y), h2f(u.y >> 16));
}
__device__ __forceinline__ float4 widen4(const uint2& u, const __nv_bfloat16*) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xffff0000u));  // bf16 is the top half of an fp32
}
__device__ __forceinline__ float4 load4(const __half* p) { return widen4(load_packed4(p), p); }
__device__ __forceinline__ float4 load4(const __nv_bfloat16* p) { return widen4(load_packed4(p), p); }

__device__ __forceinline__ void store4(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ uint32_t pack_h(float lo, float hi) {
  return (uint32_t)__half_as_ushort(__float2half_rn(lo)) | ((uint32_t)__half_as_ushort(__float2half_rn(hi)) << 16);
}
__device__ __forceinline__ uint32_t pack_bf(float lo, float hi) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(lo)) | ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(hi)) << 16);
}
__device__ __forceinline__ void store4(__half* p, const float4& v) {
  *reinterpret_cast<uint2*>(p) = make_uint2(pack_h(v.x, v.y), pack_h(v.z, v.w));
}
__device__ __forceinline__ void store4(__nv_bfloat16* p, const float4& v) {
  *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf(v.x, v.y), pack_bf(v.z, v.w));
}

}  // namespace qagnn
