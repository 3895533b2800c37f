// The attention-mask decision of Mask2Former's decoder for one key, shared by the inference bit-mask kernel
// (attn_simt.cu) and the training bool-mask kernel (mask_head.cu):
//
//   blocked = sigmoid(F.interpolate(logits, (Hl, Wl), "bilinear", align_corners=False)) < 0.5
//
// in torch's CUDA arithmetic for storage type T: the bilinear value is computed in fp32 (upsample_bilinear2d_out_frame:
// source index scale * (dst + 0.5) - 0.5 clamped at 0, truncated, lambdas and the two-level weighted sum) and rounded to
// T, then sigmoid = 1 / (1 + exp(-x)) in fp32, rounded to T, and compared with 0.5.
//
// Every rounding step of the resize is written with an explicit intrinsic, so no FMA contraction by the compiler can
// move a result (the sigmoid's contraction is pinned by its own expression, see mr_sigmoid).  The steps are the ones
// nvcc makes of torch's source expressions
//   src = scale * (dst + 0.5) - 0.5  ->  fma(dst + 0.5, scale, -0.5)
//   val = h0 * (w0 * a + w1 * b) + h1 * (w0 * c + w1 * d)
//       ->  fma(h0, fma(w1, b, w0 * a), h1 * fma(w0, c, w1 * d))
// (read from the SASS of attn_mask_bits_kernel, which evaluated that source expression before this header existed; its
// float instructions are the same with the explicit form).  For T = float both roundings to T are the identity.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace ob {

__device__ __forceinline__ float mr_round(float v, float*) { return v; }
__device__ __forceinline__ float mr_round(float v, __half*) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float mr_round(float v, __nv_bfloat16*) {
  return __bfloat162float(__float2bfloat16_rn(v));
}
__device__ __forceinline__ float mr_load(const float* p) { return *p; }
__device__ __forceinline__ float mr_load(const __half* p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float mr_load(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }

// torch's sigmoid of a value held in T, rounded to T (UnarySpecialOpsKernel.cu: one / (one + exp(-x)) in opmath fp32)
template <typename T>
__device__ __forceinline__ float mr_sigmoid(float x) {
  // Left in torch's source form on purpose: nvcc folds "1 +" into expf's last scaling step (one FFMA, one rounding),
  // as it does when compiling torch's identical expression; "/" is IEEE division under nvcc's default -prec-div=true.
  return mr_round(1.f / (1.f + expf(-x)), static_cast<T*>(nullptr));
}

// key (oy, ox) of the (Hl, Wl) level resized from src [Hm, Wm]; sy = Hm / Hl, sx = Wm / Wl in fp32
template <typename T>
__device__ __forceinline__ bool mr_blocked(const T* __restrict__ src, int Hm, int Wm, int oy, int ox, float sy,
                                           float sx) {
  const float fy = fmaxf(__fmaf_rn(__fadd_rn((float)oy, 0.5f), sy, -0.5f), 0.f);
  const float fx = fmaxf(__fmaf_rn(__fadd_rn((float)ox, 0.5f), sx, -0.5f), 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < Hm - 1 ? 1 : 0), x1 = x0 + (x0 < Wm - 1 ? 1 : 0);
  const float ly = __fsub_rn(fy, (float)y0), lx = __fsub_rn(fx, (float)x0);
  const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  const float a = mr_load(src + y0 * Wm + x0), b = mr_load(src + y0 * Wm + x1);
  const float c = mr_load(src + y1 * Wm + x0), d = mr_load(src + y1 * Wm + x1);
  const float top = __fmaf_rn(lx, b, __fmul_rn(hx, a)), bot = __fmaf_rn(hx, c, __fmul_rn(lx, d));
  const float v = __fmaf_rn(hy, top, __fmul_rn(ly, bot));
  return mr_sigmoid<T>(mr_round(v, static_cast<T*>(nullptr))) < 0.5f;
}

}  // namespace ob
