// Storage-type loads and stores of the training kernels: float, or 16-bit __half / __nv_bfloat16 under autocast.  A
// 16-bit load converts to float right after it (exact); a 16-bit store rounds the fp32 result once (round to nearest
// even).  Everything in between is fp32.  Four 16-bit channels are one 64-bit load / store.  Loads go through the
// read-only path (__ldg).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace ob {

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld4(const __half* p) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 ld4(const __nv_bfloat16* p) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float2 ld2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ float2 ld2(const __half* p) { return __half22float2(__ldg(reinterpret_cast<const __half2*>(p))); }
__device__ __forceinline__ float2 ld2(const __nv_bfloat16* p) {
  return __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162*>(p)));
}
__device__ __forceinline__ float ld1(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld1(const __half* p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float ld1(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }

__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(__half* p, float4 v) {
  const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  *reinterpret_cast<uint2*>(p) = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
}
__device__ __forceinline__ void st4(__nv_bfloat16* p, float4 v) {
  const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
  *reinterpret_cast<uint2*>(p) = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
}
__device__ __forceinline__ void st2(float* p, float2 v) { *reinterpret_cast<float2*>(p) = v; }
__device__ __forceinline__ void st2(__half* p, float2 v) {
  *reinterpret_cast<__half2*>(p) = __floats2half2_rn(v.x, v.y);
}
__device__ __forceinline__ void st2(__nv_bfloat16* p, float2 v) {
  *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(v.x, v.y);
}
__device__ __forceinline__ void st1(float* p, float v) { *p = v; }
__device__ __forceinline__ void st1(__half* p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void st1(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// The same with a double in registers, for results summed in double: each store rounds the double once to the storage
// type.  The stores keep their own name: as st1 overloads, a double argument could resolve to a float overload and be
// rounded twice on its way to 16 bits.
__device__ __forceinline__ double ld1d(const float* p) { return (double)__ldg(p); }
__device__ __forceinline__ double ld1d(const double* p) { return __ldg(p); }
__device__ __forceinline__ double ld1d(const __half* p) { return (double)__half2float(__ldg(p)); }
__device__ __forceinline__ double ld1d(const __nv_bfloat16* p) { return (double)__bfloat162float(__ldg(p)); }
__device__ __forceinline__ void st1d(float* p, double v) { *p = __double2float_rn(v); }
__device__ __forceinline__ void st1d(double* p, double v) { *p = v; }
__device__ __forceinline__ void st1d(__half* p, double v) { *p = __double2half(v); }
__device__ __forceinline__ void st1d(__nv_bfloat16* p, double v) { *p = __double2bfloat16(v); }

}  // namespace ob
