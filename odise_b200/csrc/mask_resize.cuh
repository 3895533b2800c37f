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

// one axis of torch's bilinear source coordinate for output index o, s = in / out in fp32 (area_pixel_compute_source_index
// and the frame kernels): i0 = trunc(max(s * (o + 0.5) - 0.5, 0)), i1 = i0 + 1 unless i0 is the last of n sources,
// l = the weight of i1, h = 1 - l the weight of i0.  The forward value (mr_bilinear) and the FPN backward's adjoint
// weights and membership (fpn_upsample.cu) both come from here, so they agree bit for bit.
struct MrAxis {
  int i0, i1;
  float h, l;
};

__device__ __forceinline__ MrAxis mr_axis(int o, float s, int n) {
  const float f = fmaxf(__fmaf_rn(__fadd_rn((float)o, 0.5f), s, -0.5f), 0.f);
  MrAxis a;
  a.i0 = (int)f;
  a.i1 = a.i0 + (a.i0 < n - 1 ? 1 : 0);
  a.l = __fsub_rn(f, (float)a.i0);
  a.h = __fsub_rn(1.f, a.l);
  return a;
}

// torch's fp32 bilinear value at (ay, ax) of a source [Hm, Wm] whose element (y, x) is src[(y * Wm + x) * es].
// top_ha selects the contraction of the top row: false fma(l, b, h * a), as in the NHWC frame kernel
// (upsample_bilinear2d_nhwc_out_frame) and the bits of attn_mask_bits_kernel; true fma(h, a, l * b), as in
// upsample_bilinear2d_out_frame where torch runs it for a batch-1 level view (measured on torch 2.11's sm_90 build).
template <typename T, bool top_ha = false>
__device__ __forceinline__ float mr_bilinear(const T* __restrict__ src, int Wm, const MrAxis& ay, const MrAxis& ax,
                                             int es) {
  const float a = mr_load(src + (ay.i0 * Wm + ax.i0) * es), b = mr_load(src + (ay.i0 * Wm + ax.i1) * es);
  const float c = mr_load(src + (ay.i1 * Wm + ax.i0) * es), d = mr_load(src + (ay.i1 * Wm + ax.i1) * es);
  const float top = top_ha ? __fmaf_rn(ax.h, a, __fmul_rn(ax.l, b)) : __fmaf_rn(ax.l, b, __fmul_rn(ax.h, a));
  const float bot = __fmaf_rn(ax.h, c, __fmul_rn(ax.l, d));
  return __fmaf_rn(ay.h, top, __fmul_rn(ay.l, bot));
}

// key (oy, ox) of the (Hl, Wl) level resized from src [Hm, Wm]; sy = Hm / Hl, sx = Wm / Wl in fp32
template <typename T>
__device__ __forceinline__ bool mr_blocked(const T* __restrict__ src, int Hm, int Wm, int oy, int ox, float sy,
                                           float sx) {
  const float v = mr_bilinear(src, Wm, mr_axis(oy, sy, Hm), mr_axis(ox, sx, Wm), 1);
  return mr_sigmoid<T>(mr_round(v, static_cast<T*>(nullptr))) < 0.5f;
}

}  // namespace ob
