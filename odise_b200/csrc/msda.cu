// Multi-scale deformable attention sampling for sm_90a (SURVEY.md §8a rows b4/b5).
//
// Semantics follow ms_deformable_im2col_gpu_kernel / ms_deform_attn_im2col_bilinear of the reference
// (third_party/Mask2Former/mask2former/modeling/pixel_decoder/ops/src/cuda/ms_deform_im2col_cuda.cuh:38-89,
// :242-304): pixel coords h = loc_y*H - 0.5, w = loc_x*W - 0.5, a sample contributes only when
// -1 < h < H and -1 < w < W, out-of-range corners read as zero.  The design does not: the reference runs one
// thread per output scalar (every thread re-reads loc/weight and issues 48 scalar gathers); here LPH = D/4 lanes
// own one (query, head) pair, each lane gathers 16-byte channel vectors, so a D=32 head is 8 lanes x float4 and a
// warp keeps 4 pairs x 48 independent 128-bit gathers in flight.  HBM/L2-bound: value (22 MB/image) stays
// L2-resident, loc/attn/out stream once.
#include <type_traits>

#include "ptx.cuh"
#include "odise_b200.h"
#include "launch_count.h"
#include "storage.cuh"

namespace ob {

// (H_l, W_l) / level_start stay on the device like in the reference (ms_deform_im2col_cuda.cuh:277-281): a
// handful of L1-broadcast int64 loads per thread, no host sync, CUDA-graph capturable.
struct MsdaLevels {
  const int64_t* shapes;
  const int64_t* start;
};

__device__ __forceinline__ void fma4(float4& acc, float w, const float4& v) {
  acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
}

// one sample: adds attn * bilinear(value_level, h_im, w_im) for 4 channels
__device__ __forceinline__ void sample4(float4& acc, const float* __restrict__ vbase, int H, int W, int pix_stride,
                                        float h_im, float w_im, float aw) {
  if (!(h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W)) return;
  const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
  const float lh = h_im - h_low, lw = w_im - w_low;
  const float hh = 1.f - lh, hw = 1.f - lw;
  const int h_high = h_low + 1, w_high = w_low + 1;
  float4 v1 = make_float4(0, 0, 0, 0), v2 = v1, v3 = v1, v4 = v1;
  if (h_low >= 0 && w_low >= 0) v1 = ld4(vbase + (long long)(h_low * W + w_low) * pix_stride);
  if (h_low >= 0 && w_high <= W - 1) v2 = ld4(vbase + (long long)(h_low * W + w_high) * pix_stride);
  if (h_high <= H - 1 && w_low >= 0) v3 = ld4(vbase + (long long)(h_high * W + w_low) * pix_stride);
  if (h_high <= H - 1 && w_high <= W - 1) v4 = ld4(vbase + (long long)(h_high * W + w_high) * pix_stride);
  // same association as the reference: (w1*v1 + w2*v2 + w3*v3 + w4*v4) * weight
  const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
  float4 s;
  s.x = w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
  s.y = w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
  s.z = w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
  s.w = w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
  acc.x += s.x * aw; acc.y += s.y * aw; acc.z += s.z * aw; acc.w += s.w * aw;
}

// FUSED = 0: loc/attn given (reference ABI).  FUSED = 1: raw offsets / logits + reference points.
template <int FUSED>
__global__ void __launch_bounds__(256)
msda_vec4_kernel(const float* __restrict__ value, const MsdaLevels lv, const float* __restrict__ loc_or_off,
                 const float* __restrict__ attn_or_logit, const float* __restrict__ ref, float* __restrict__ out,
                 __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, int N, int S, int M, int D,
                 int L, int Lq, int P, int lph) {
  const long long pairs = (long long)N * Lq * M;
  const long long gid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long pair = gid / lph;
  if (pair >= pairs) return;
  const int c = (int)(gid - pair * lph) * 4;
  const int m = (int)(pair % M);
  const long long nq = pair / M;
  const int n = (int)(nq / Lq);
  const int pix_stride = M * D;
  const float* vb = value + (long long)n * S * pix_stride + m * D + c;
  const float* lp = loc_or_off + pair * L * P * 2;
  const float* ap = attn_or_logit + pair * L * P;

  float mx = 0.f, inv = 1.f;
  if (FUSED) {
    mx = -INFINITY;
    for (int i = 0; i < L * P; ++i) mx = fmaxf(mx, __ldg(ap + i));
    float sum = 0.f;
    for (int i = 0; i < L * P; ++i) sum += expf(__ldg(ap + i) - mx);
    inv = 1.f / sum;
  }
  float4 acc = make_float4(0, 0, 0, 0);
  for (int l = 0; l < L; ++l) {
    const int H = (int)__ldg(lv.shapes + 2 * l), W = (int)__ldg(lv.shapes + 2 * l + 1);
    const float* vl = vb + (long long)__ldg(lv.start + l) * pix_stride;
    float rx = 0.f, ry = 0.f;
    if (FUSED) {
      const float2 r = __ldg(reinterpret_cast<const float2*>(ref + (nq * L + l) * 2));
      rx = r.x; ry = r.y;
    }
#pragma unroll 4
    for (int p = 0; p < P; ++p) {
      const float2 xy = __ldg(reinterpret_cast<const float2*>(lp + (l * P + p) * 2));
      float aw = __ldg(ap + l * P + p);
      float lx = xy.x, ly = xy.y;
      if (FUSED) {
        // ms_deform_attn.py:104-107: loc = ref + off / (W_l, H_l); softmax over L*P (ms_deform_attn.py:100)
        lx = rx + xy.x / (float)W;
        ly = ry + xy.y / (float)H;
        aw = expf(aw - mx) * inv;
      }
      sample4(acc, vl, H, W, pix_stride, ly * H - 0.5f, lx * W - 0.5f, aw);
    }
  }
  const long long o = pair * D + c;
  if (out) *reinterpret_cast<float4*>(out + o) = acc;
  if (out_hi) {
    const float e[4] = {acc.x, acc.y, acc.z, acc.w};
    store_planes<4>(out_hi + o, out_lo ? out_lo + o : nullptr, e);
  }
}

// generic scalar path (any D, e.g. the D=2 problem of the reference's ops/test.py:24-31); T = float or double
template <typename T>
__global__ void msda_scalar_kernel(const T* __restrict__ value, const MsdaLevels lv,
                                   const T* __restrict__ loc, const T* __restrict__ attn,
                                   T* __restrict__ out, int N, int S, int M, int D, int L, int Lq, int P) {
  const long long total = (long long)N * Lq * M * D;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % D);
    const long long pair = idx / D;
    const int m = (int)(pair % M);
    const int n = (int)(pair / M / Lq);
    const int pix_stride = M * D;
    const T* vb = value + (long long)n * S * pix_stride + m * D + c;
    T col = 0;
    for (int l = 0; l < L; ++l) {
      const int H = (int)__ldg(lv.shapes + 2 * l), W = (int)__ldg(lv.shapes + 2 * l + 1);
      const T* vl = vb + (long long)__ldg(lv.start + l) * pix_stride;
      for (int p = 0; p < P; ++p) {
        const T lx = loc[(pair * L * P + l * P + p) * 2], ly = loc[(pair * L * P + l * P + p) * 2 + 1];
        const T aw = attn[pair * L * P + l * P + p];
        const T h_im = ly * H - (T)0.5, w_im = lx * W - (T)0.5;
        if (h_im > (T)-1 && w_im > (T)-1 && h_im < (T)H && w_im < (T)W) {
          const int h_low = (int)floor(h_im), w_low = (int)floor(w_im);
          const T lh = h_im - h_low, lw = w_im - w_low, hh = (T)1 - lh, hw = (T)1 - lw;
          T v1 = 0, v2 = 0, v3 = 0, v4 = 0;
          if (h_low >= 0 && w_low >= 0) v1 = vl[(long long)(h_low * W + w_low) * pix_stride];
          if (h_low >= 0 && w_low + 1 <= W - 1) v2 = vl[(long long)(h_low * W + w_low + 1) * pix_stride];
          if (h_low + 1 <= H - 1 && w_low >= 0) v3 = vl[(long long)((h_low + 1) * W + w_low) * pix_stride];
          if (h_low + 1 <= H - 1 && w_low + 1 <= W - 1) v4 = vl[(long long)((h_low + 1) * W + w_low + 1) * pix_stride];
          col += (hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4) * aw;
        }
      }
    }
    out[idx] = col;
  }
}


// ---------------------------------------------------------------------------------------------------------------
// D = 32 fast path (the ODISE / Mask2Former head: 8 heads x 32 channels).  A block owns PAIRS = 32 (query, head)
// pairs.  Phase 1 ("setup"): one thread per (pair, sample) slot computes — ONCE — what the round-1 kernel (and the
// reference's one-thread-per-scalar kernel) recomputed in every channel lane: the L*P softmax (sub-warp xor shuffles),
// loc = ref + off / (W, H), the bilinear corner weights already multiplied by the attention weight, and the four
// corner offsets as 32-bit element offsets from the (image, head) base (level start folded in, invalid corners ->
// weight 0 / offset 0).  They go to shared memory.  Phase 2 ("gather"): 8 lanes per pair, one float4 of channels
// each; per sample two broadcast LDS.128 + four independent LDG.128 + 16 FMAs.  Instructions per warp drop ~5x
// (ncu r1: 396 M warp instructions, issue-bound); what remains is the L1/L2 data path: 4 corners x 128 B per
// (query, head, sample) = 48 x 128 B lines per pair.
constexpr int MSDA_PAIRS = 32;

// The bilinear footprint of one sample, shared by the D = 32 forward and backward kernels: the four corners
// (top-left, top-right, bottom-left, bottom-right) as 32-bit element offsets from the (image, head) base with the level
// start folded in, their bilinear weights, the fractional position (lh, lw) and a bit per corner that lies inside the
// level.  Corners outside the level (and every corner of a sample outside it) get offset 0, weight 0 and no bit.
struct MsdaCorners {
  int4 off;
  float4 w;
  float lh, lw;
  int valid;
};

__device__ __forceinline__ MsdaCorners msda_corners(float lx, float ly, int H, int W, int start, int pix) {
  MsdaCorners c;
  c.off = make_int4(0, 0, 0, 0);
  c.w = make_float4(0.f, 0.f, 0.f, 0.f);
  c.lh = 0.f; c.lw = 0.f; c.valid = 0;
  const float h_im = ly * H - 0.5f, w_im = lx * W - 0.5f;
  if (h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W) {
    const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
    const float lh = h_im - h_low, lw = w_im - w_low, hh = 1.f - lh, hw = 1.f - lw;
    const bool t = h_low >= 0, b = h_low + 1 <= H - 1, lf = w_low >= 0, rt = w_low + 1 <= W - 1;
    const int base = (start + h_low * W + w_low) * pix;
    c.lh = lh; c.lw = lw;
    if (t && lf) { c.off.x = base; c.w.x = hh * hw; c.valid |= 1; }
    if (t && rt) { c.off.y = base + pix; c.w.y = hh * lw; c.valid |= 2; }
    if (b && lf) { c.off.z = base + W * pix; c.w.z = lh * hw; c.valid |= 4; }
    if (b && rt) { c.off.w = base + (W + 1) * pix; c.w.w = lh * lw; c.valid |= 8; }
  }
  return c;
}

// Phase 1 of a (pair, sample) slot, shared by the D = 32 forward and backward kernels: the sample's level (H, W, start),
// its location and its attention weight; a slot that is not live yields zeros.  FUSED = 1 computes
// loc = ref + off / (W, H) and the softmax over the pair's L*P logits from the raw inputs, so the fused backward
// differentiates exactly the bits its forward sampled with.  The softmax reduces over an aligned sub-warp of SL lanes
// (slot = pair * SL + sample): every lane of the warp must make the call.  T is the storage type of the offsets and
// logits (float, or 16-bit with FUSED = 1); they are converted to float as they are loaded, ref is always float.
// RW is the width of a reference point: 2 = (x, y), 4 = a box (cx, cy, w, h) with loc = ref.xy + off / P * ref.wh * 0.5
// (ms_deform_attn.py:110-112), computed with the roundings of the composed path's torch ops on the device: `off / P` by
// a CUDA tensor is a product with the fp32 reciprocal of P, then the product with w, * 0.5 (exact) and the sum.
struct MsdaSlot {
  float lx, ly, aw;
  int H, W, start;
};

template <int FUSED, typename T, int RW = 2>
__device__ __forceinline__ MsdaSlot msda_slot(const MsdaLevels& lv, const T* __restrict__ loc_or_off,
                                              const T* __restrict__ attn_or_logit, const float* __restrict__ ref,
                                              long long pair, int s, bool live, int M, int L, int P, int SL) {
  const int LP = L * P;
  MsdaSlot r;
  r.aw = 0.f; r.lx = 0.f; r.ly = 0.f;
  r.H = 1; r.W = 1; r.start = 0;
  if (live) {
    const int l = s / P;
    r.H = (int)__ldg(lv.shapes + 2 * l);
    r.W = (int)__ldg(lv.shapes + 2 * l + 1);
    r.start = (int)__ldg(lv.start + l);
    const float2 xy = ld2(loc_or_off + (pair * LP + s) * 2);
    r.aw = ld1(attn_or_logit + pair * LP + s);
    r.lx = xy.x; r.ly = xy.y;
    if constexpr (FUSED && RW == 4) {
      const float4 rp = __ldg(reinterpret_cast<const float4*>(ref + (pair / M * L + l) * 4));
      const float inv_p = 1.f / (float)P;
      r.lx = rp.x + xy.x * inv_p * rp.z * 0.5f;
      r.ly = rp.y + xy.y * inv_p * rp.w * 0.5f;
    } else if (FUSED) {
      const long long nq = pair / M;
      const float2 rp = __ldg(reinterpret_cast<const float2*>(ref + (nq * L + l) * 2));
      r.lx = rp.x + xy.x / (float)r.W;        // ms_deform_attn.py:104-107
      r.ly = rp.y + xy.y / (float)r.H;
    }
  }
  if (FUSED) {                                 // softmax over the L*P logits of the pair (ms_deform_attn.py:100)
    float mx = live ? r.aw : -INFINITY;
    for (int o = SL >> 1; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float e = live ? expf(r.aw - mx) : 0.f;
    float sum = e;
    for (int o = SL >> 1; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    r.aw = e / sum;
  }
  return r;
}

// T: storage type of value, loc_or_off, attn_or_logit and out.  float for both FUSED; __half / __nv_bfloat16 with
// FUSED = 1 (odise_msda_fused_f16 / _bf16: a lane's 4 channels are one 64-bit load per corner, out_hi / out_lo unused).
// RW: reference-point width of msda_slot (4: the odise_msda_fused_box_* entry points); only phase 1 differs.
template <int FUSED, typename T, int RW = 2>
__global__ void __launch_bounds__(256)
msda_d32_kernel(const T* __restrict__ value, const MsdaLevels lv, const T* __restrict__ loc_or_off,
                const T* __restrict__ attn_or_logit, const float* __restrict__ ref, T* __restrict__ out,
                __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, int N, int S, int M, int L,
                int Lq, int P, int SL /* pow2 >= L*P, <= 32 */) {
  extern __shared__ __align__(16) uint8_t msda_smem[];
  const int LP = L * P;
  int4* s_off = reinterpret_cast<int4*>(msda_smem);                       // [PAIRS][LP]
  float4* s_w = reinterpret_cast<float4*>(msda_smem + (size_t)MSDA_PAIRS * LP * sizeof(int4));
  const long long pairs = (long long)N * Lq * M;
  const long long pair0 = (long long)blockIdx.x * MSDA_PAIRS;
  const int pix = M * 32;

  // ---- phase 1: (pair, sample) slots; SL divides 32, so a pair's samples sit in one aligned sub-warp
  for (int slot = threadIdx.x; slot < MSDA_PAIRS * SL; slot += 256) {
    const int pl = slot / SL, s = slot - pl * SL;
    const long long pair = pair0 + pl;
    const bool live = (s < LP) && (pair < pairs);
    const MsdaSlot sl = msda_slot<FUSED, T, RW>(lv, loc_or_off, attn_or_logit, ref, pair, s, live, M, L, P, SL);
    if (live) {
      const float aw = sl.aw;
      const MsdaCorners cn = msda_corners(sl.lx, sl.ly, sl.H, sl.W, sl.start, pix);
      s_off[pl * LP + s] = cn.off;
      s_w[pl * LP + s] = make_float4(cn.w.x * aw, cn.w.y * aw, cn.w.z * aw, cn.w.w * aw);
    }
  }
  __syncthreads();

  // ---- phase 2: 8 lanes per pair, float4 of channels per lane
  const int pl = threadIdx.x >> 3;
  const long long pair = pair0 + pl;
  if (pair >= pairs) return;
  const int c = (threadIdx.x & 7) * 4;
  const int m = (int)(pair % M);
  const int n = (int)(pair / M / Lq);
  const T* vb = value + (long long)n * S * pix + m * 32 + c;
  const int4* po = s_off + pl * LP;
  const float4* pw = s_w + pl * LP;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
  for (int s = 0; s < LP; ++s) {
    const int4 o4 = po[s];
    const float4 w4 = pw[s];
    const float4 v1 = ld4(vb + o4.x), v2 = ld4(vb + o4.y), v3 = ld4(vb + o4.z), v4 = ld4(vb + o4.w);
    fma4(acc, w4.x, v1); fma4(acc, w4.y, v2); fma4(acc, w4.z, v3); fma4(acc, w4.w, v4);
  }
  const long long o = pair * 32 + c;
  if (out) st4(out + o, acc);
  if (out_hi) {
    const float e[4] = {acc.x, acc.y, acc.z, acc.w};
    store_planes<4>(out_hi + o, out_lo ? out_lo + o : nullptr, e);
  }
}

// 32-bit element offsets must cover one image's value block; L*P samples must fit a warp
static bool d32_ok(int S, int M, int D, int L, int P) {
  return D == 32 && L * P <= 32 && (long long)S * M * D < (1LL << 31);
}

template <int FUSED, typename T, int RW = 2>
static void launch_d32(const T* value, const MsdaLevels& lv, const T* a, const T* b, const float* ref,
                       T* out, __nv_bfloat16* hi, __nv_bfloat16* lo, int N, int S, int M, int L, int Lq, int P,
                       cudaStream_t stream) {
  const int LP = L * P;
  int SL = 1;
  while (SL < LP) SL <<= 1;
  const long long pairs = (long long)N * Lq * M;
  const int blocks = (int)((pairs + MSDA_PAIRS - 1) / MSDA_PAIRS);
  const size_t smem = (size_t)MSDA_PAIRS * LP * (sizeof(int4) + sizeof(float4));
  msda_d32_kernel<FUSED, T, RW><<<blocks, 256, smem, stream>>>(value, lv, a, b, ref, out, hi, lo, N, S, M, L, Lq, P,
                                                               SL);
}

static bool vec_ok(int D) { return D % 4 == 0 && D <= 128 && (32 % (D / 4) == 0); }

// ---------------------------------------------------------------------------------------------------------------
// Backward: ms_deformable_col2im_gpu_kernel / ms_deform_attn_col2im_bilinear of the reference (.cuh:92-164, launcher
// ms_deform_attn_cuda.cu:88-158).  For every sample inside its level (-1 < h < H, -1 < w < W) and every corner inside
// the level:
//   grad_value[corner] += w_corner * attn * g,      grad_attn = sum_c g_c * bilinear_c,
//   grad_loc.x = W * attn * sum_c g_c * d bilinear_c / dw,   grad_loc.y = H * attn * sum_c g_c * d bilinear_c / dh.
// Corners outside the level contribute nothing to any of the three (the reference's per-corner `if`: their value is
// never read); samples outside the level get grad_loc = grad_attn = 0.

__device__ __forceinline__ float4 scale4(const float4& v, float s) {
  return make_float4(v.x * s, v.y * s, v.z * s, v.w * s);
}
// The backward kernels' sums of products are written with explicit fmaf / fma: the default (atomic) and the fixed-point
// instantiations share this arithmetic and must give the same bits, while an implicit contraction may associate a sum
// differently in each instantiation.  The association is the one nvcc picked for the default instantiations, whose SASS
// is unchanged by writing it out.
__device__ __forceinline__ float dot4(const float4& a, const float4& b) {
  return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)));
}
// bilinear value w1 v1 + w2 v2 + w3 v3 + w4 v4 and its derivatives d/dh = hw (v3 - v1) + lw (v4 - v2),
// d/dw = hh (v2 - v1) + lh (v4 - v3), for float and double
__device__ __forceinline__ float msda_fma(float a, float b, float c) { return fmaf(a, b, c); }
__device__ __forceinline__ double msda_fma(double a, double b, double c) { return fma(a, b, c); }
template <typename T>
__device__ __forceinline__ T msda_bil(T w1, T w2, T w3, T w4, T v1, T v2, T v3, T v4) {
  return msda_fma(w4, v4, msda_fma(w3, v3, msda_fma(w1, v1, w2 * v2)));
}

// Accumulation policies of grad_value in the backward kernels; only the corner reductions differ between them.
// MsdaAtomicAcc: floating-point atomics into grad_value (the default: fast, bits depend on the order of the reductions).
struct MsdaAtomicAcc {
  static constexpr bool fixed = false;
};

// MsdaFixedAcc: int64 fixed point (the deterministic entry points).  Integer addition is associative, so the sums do not
// depend on the order of the reductions.  Per (image n, head m), with G = max |grad_out[n, :, m, :]|, A = max
// |attn[n, :, m, :, :]| (A = 1 on the fused paths, whose softmax weights are <= 1), e = clog2(G) + clog2(A) (so
// 2^e >= G * A, without forming the product) and K = Lq * P (an element takes at most one contribution per
// (query, point) of its level): s = 61 - ceil(log2 K) - e.  Every contribution g * (w * aw) is computed in the storage arithmetic as
// the atomic path does, scaled by 2^s exactly (|.| <= 2^(61 - ceil(log2 K)) plus product rounding) and rounded to the
// nearest integer, so every sum stays below 2^62.  A contribution that is not finite, or does not fit, marks the
// (n, m) slice non-finite; the finalize pass writes NaN there.
struct MsdaFixedAcc {
  static constexpr bool fixed = true;
  unsigned long long* sum;          // [N, S, M, D] two's-complement int64 sums, zero-filled
  unsigned long long* gmax;         // [N * M] bits of max |grad_out| as a double (>= +inf bits: non-finite slice)
  const unsigned long long* amax;   // [N * M] bits of max |attn| as a double (0 on the fused paths: A taken as 1)
  int log2k;                        // ceil(log2(Lq * P))
};

// least e with 2^e >= x for a finite x > 0; 0 for x = 0 (so A = 0 and A = 1 give the same shift)
__device__ __forceinline__ int msda_clog2(double x) {
  int e;
  const double f = frexp(x, &e);                      // x = f * 2^e, f in [0.5, 1)
  return f == 0.5 ? e - 1 : (x == 0.0 ? 0 : e);
}

__device__ __forceinline__ int msda_fixed_shift(const MsdaFixedAcc& a, long long nm) {
  const double G = __longlong_as_double((long long)a.gmax[nm]), A = __longlong_as_double((long long)a.amax[nm]);
  return 61 - a.log2k - (msda_clog2(G) + msda_clog2(A));
}

// one contribution in fixed point: float c * 2^s in double (exact: sc = 2^s, |s| < 400 for float inputs), double
// c through ldexp (any s); `bad` collects contributions that are not finite or exceed 2^62
__device__ __forceinline__ unsigned long long msda_fixed(float c, double sc, int, bool& bad) {
  const double d = (double)c * sc;
  bad |= !(fabs(d) < 0x1p62);
  return (unsigned long long)__double2ll_rn(d);
}
__device__ __forceinline__ unsigned long long msda_fixed(double c, double, int s, bool& bad) {
  const double d = ldexp(c, s);
  bad |= !(fabs(d) < 0x1p62);
  return (unsigned long long)__double2ll_rn(d);
}

// channels p[0], p[8], p[16], p[24] of a D = 32 head: with lane j of a pair at p = corner + j, each of the four
// reductions covers 64 contiguous bytes (8 channels) across the pair's 8 lanes, two 32-byte sectors
__device__ __forceinline__ void msda_fixed_add4(unsigned long long* p, const float4& c, double sc, bool& bad) {
  atomicAdd(p + 0, msda_fixed(c.x, sc, 0, bad));
  atomicAdd(p + 8, msda_fixed(c.y, sc, 0, bad));
  atomicAdd(p + 16, msda_fixed(c.z, sc, 0, bad));
  atomicAdd(p + 24, msda_fixed(c.w, sc, 0, bad));
}

constexpr unsigned long long MSDA_NAN_BITS = 0x7ff8000000000000ull;   // a quiet NaN: above the bits of +inf
constexpr unsigned long long MSDA_INF_BITS = 0x7ff0000000000000ull;

// D = 32: the forward's block of MSDA_PAIRS pairs.  Phase 1 stores per (pair, sample) the corners of msda_corners with
// their bits and the attention weight; phase 2 runs 8 lanes per pair with one float4 of channels each (grad_out loaded
// once per pair).  Per sample a lane does four LDG.128 of value, three partial dot products (bilinear value, d/dh,
// d/dw) and up to four 128-bit vector reductions into grad_value (atomicAdd(float4*) -> REDG.E.ADD.F32x4, a quarter of
// the reference's scalar atomics).  The partials are summed over the 8 lanes with xor shuffles and one lane stores
// grad_attn and grad_loc: no atomics there, so both are bit-deterministic; only grad_value depends on the order of the
// reductions, as in the reference.
//
// FUSED = 1 is the backward of odise_msda_fused_f32: loc / attn are the raw offsets / logits (+ ref, SL as in the
// forward).  Phase 1 recomputes location and softmax with the forward's msda_slot on the forward's slot layout.  Phase 2
// writes grad_off = grad_loc / (W, H) = (attn * sw, attn * sh) (the W and H of grad_loc cancel) and keeps the
// per-sample grad_attn partial sv in the slot's lh field, which is dead once every lane of the pair has read it; after
// the loop grad_logit[s] = attn_s * (sv_s - sum_t attn_t * sv_t), the softmax backward, with the sum taken in sample
// order in every lane.  grad_off and grad_logit are written without atomics and are bit-deterministic.
//
// T: storage type of value, loc, attn, grad_out, grad_loc and grad_attn (float; __half / __nv_bfloat16 with FUSED = 1).
// grad_value is float for every T: at the 1024^2 shape an element of the coarsest level takes hundreds of contributions,
// which a 16-bit running sum would lose, so the caller rounds the fp32 sum once.
//
// Acc = MsdaFixedAcc (the deterministic entry points): grad_value is unused; each valid corner takes four 64-bit
// integer reductions into acc.sum instead of one 128-bit float reduction.  For them lane j of a pair holds a second,
// interleaved copy of grad_out (channels j, j + 8, j + 16, j + 24), so that each reduction instruction of the pair's 8
// lanes covers 64 contiguous bytes; the contributions are the same products, summed by other lanes.
//
// RW = 4 (FUSED = 1, the odise_msda_fused_box_backward_* entry points): box reference points, phase 1 as in the forward.
// d loc / d off = (w, h) * 0.5 / P does not cancel the W and H of grad_loc, so the storing lane writes
// grad_off = (W * aw * sw * w, H * aw * sh * h) * 0.5 / P, reading (w, h) of its (query, level) from global memory (an L1
// broadcast; the 48 B shared record per slot is full at L*P = 32).  Nothing is divided by w or h: a degenerate box
// (w = 0 or h = 0) gives grad_off = 0 along that axis.
template <int FUSED, typename T, typename Acc = MsdaAtomicAcc, int RW = 2>
__global__ void __launch_bounds__(256)
msda_d32_backward_kernel(const T* __restrict__ value, const MsdaLevels lv, const T* __restrict__ loc,
                         const T* __restrict__ attn, const T* __restrict__ grad_out,
                         float* __restrict__ grad_value, T* __restrict__ grad_loc, T* __restrict__ grad_attn,
                         int N, int S, int M, int L, int Lq, int P, const float* __restrict__ ref, int SL,
                         const Acc acc) {
  extern __shared__ __align__(16) uint8_t msda_smem[];
  const int LP = L * P;
  int4* s_off = reinterpret_cast<int4*>(msda_smem);                                   // [PAIRS][LP]
  float4* s_w = reinterpret_cast<float4*>(msda_smem + (size_t)MSDA_PAIRS * LP * sizeof(int4));
  float4* s_f = s_w + MSDA_PAIRS * LP;                                                // (lh, lw, attn, corner bits)
  const long long pairs = (long long)N * Lq * M;
  const long long pair0 = (long long)blockIdx.x * MSDA_PAIRS;
  const int pix = M * 32;

  // ---- phase 1: (pair, sample) slots; pairs past the end get zero corners so that their lanes do no memory work
  if (FUSED) {
    for (int slot = threadIdx.x; slot < MSDA_PAIRS * SL; slot += 256) {
      const int pl = slot / SL, s = slot - pl * SL;
      const long long pair = pair0 + pl;
      const bool live = (s < LP) && (pair < pairs);
      const MsdaSlot sl = msda_slot<1, T, RW>(lv, loc, attn, ref, pair, s, live, M, L, P, SL);
      if (s < LP) {
        int4 o4 = make_int4(0, 0, 0, 0);
        float4 w4 = make_float4(0.f, 0.f, 0.f, 0.f), f4 = w4;
        if (live) {
          const MsdaCorners cn = msda_corners(sl.lx, sl.ly, sl.H, sl.W, sl.start, pix);
          o4 = cn.off;
          w4 = cn.w;
          f4 = make_float4(cn.lh, cn.lw, sl.aw, __int_as_float(cn.valid));
        }
        s_off[pl * LP + s] = o4;
        s_w[pl * LP + s] = w4;
        s_f[pl * LP + s] = f4;
      }
    }
  } else {
    for (int slot = threadIdx.x; slot < MSDA_PAIRS * LP; slot += 256) {
      const int pl = slot / LP, s = slot - pl * LP;
      const long long pair = pair0 + pl;
      int4 o4 = make_int4(0, 0, 0, 0);
      float4 w4 = make_float4(0.f, 0.f, 0.f, 0.f), f4 = w4;
      if (pair < pairs) {
        const int l = s / P;
        const int H = (int)__ldg(lv.shapes + 2 * l), W = (int)__ldg(lv.shapes + 2 * l + 1);
        const int start = (int)__ldg(lv.start + l);
        const float2 xy = ld2(loc + (pair * LP + s) * 2);
        const MsdaCorners cn = msda_corners(xy.x, xy.y, H, W, start, pix);
        o4 = cn.off;
        w4 = cn.w;
        f4 = make_float4(cn.lh, cn.lw, ld1(attn + pair * LP + s), __int_as_float(cn.valid));
      }
      s_off[slot] = o4;
      s_w[slot] = w4;
      s_f[slot] = f4;
    }
  }
  __syncthreads();

  // ---- phase 2: 8 lanes per pair, float4 of channels per lane; every lane runs every sample (the shuffles need them)
  const int pl = threadIdx.x >> 3;
  const long long pair = pair0 + pl;
  const bool live = pair < pairs;
  const int c = (threadIdx.x & 7) * 4;
  const int m = (int)(pair % M);
  const int n = (int)(pair / M / Lq);
  const long long vbase = (long long)n * S * pix + m * 32 + c;
  const T* vb = value + vbase;
  float* gvb = grad_value + vbase;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 g = live ? ld4(grad_out + pair * 32 + c) : zero;
  const int4* po = s_off + pl * LP;
  const float4* pw = s_w + pl * LP;
  float4* pf = s_f + pl * LP;
  float dot = 0.f;                                    // FUSED: sum_t attn_t * sv_t
  double sc = 0.0;                                    // fixed point: 2^s of the pair's (n, m)
  bool bad = false;
  float4 gt = zero;                                   // fixed point: channels j, j + 8, j + 16, j + 24 of lane j
  if constexpr (Acc::fixed) {
    if (live) {
      sc = ldexp(1.0, msda_fixed_shift(acc, (long long)n * M + m));
      const T* gp = grad_out + pair * 32 + (threadIdx.x & 7);
      gt = make_float4(ld1(gp), ld1(gp + 8), ld1(gp + 16), ld1(gp + 24));
    }
  }
  for (int l = 0, s = 0; l < L; ++l) {
    const float Hf = (float)__ldg(lv.shapes + 2 * l), Wf = (float)__ldg(lv.shapes + 2 * l + 1);
#pragma unroll 2
    for (int p = 0; p < P; ++p, ++s) {
      const int4 o4 = po[s];
      const float4 w4 = pw[s], f4 = pf[s];
      const int valid = __float_as_int(f4.w);
      const float4 v1 = (valid & 1) ? ld4(vb + o4.x) : zero, v2 = (valid & 2) ? ld4(vb + o4.y) : zero,
                   v3 = (valid & 4) ? ld4(vb + o4.z) : zero, v4 = (valid & 8) ? ld4(vb + o4.w) : zero;
      const float lh = f4.x, lw = f4.y, hh = 1.f - lh, hw = 1.f - lw, aw = f4.z;
      float4 bil, dh, dw;
      bil.x = msda_bil(w4.x, w4.y, w4.z, w4.w, v1.x, v2.x, v3.x, v4.x);
      bil.y = msda_bil(w4.x, w4.y, w4.z, w4.w, v1.y, v2.y, v3.y, v4.y);
      bil.z = msda_bil(w4.x, w4.y, w4.z, w4.w, v1.z, v2.z, v3.z, v4.z);
      bil.w = msda_bil(w4.x, w4.y, w4.z, w4.w, v1.w, v2.w, v3.w, v4.w);
      dh.x = hw * (v3.x - v1.x) + lw * (v4.x - v2.x);
      dh.y = hw * (v3.y - v1.y) + lw * (v4.y - v2.y);
      dh.z = hw * (v3.z - v1.z) + lw * (v4.z - v2.z);
      dh.w = hw * (v3.w - v1.w) + lw * (v4.w - v2.w);
      dw.x = hh * (v2.x - v1.x) + lh * (v4.x - v3.x);
      dw.y = hh * (v2.y - v1.y) + lh * (v4.y - v3.y);
      dw.z = hh * (v2.z - v1.z) + lh * (v4.z - v3.z);
      dw.w = hh * (v2.w - v1.w) + lh * (v4.w - v3.w);
      float sv = dot4(g, bil), sh = dot4(g, dh), sw = dot4(g, dw);
      if constexpr (Acc::fixed) {
        // the same per-channel products g_c * (w * aw) as the atomic path, channels interleaved across the lanes
        unsigned long long* sb = acc.sum + (vbase - c) + (threadIdx.x & 7);
        if (valid & 1) msda_fixed_add4(sb + o4.x, scale4(gt, w4.x * aw), sc, bad);
        if (valid & 2) msda_fixed_add4(sb + o4.y, scale4(gt, w4.y * aw), sc, bad);
        if (valid & 4) msda_fixed_add4(sb + o4.z, scale4(gt, w4.z * aw), sc, bad);
        if (valid & 8) msda_fixed_add4(sb + o4.w, scale4(gt, w4.w * aw), sc, bad);
      } else {
        if (valid & 1) atomicAdd(reinterpret_cast<float4*>(gvb + o4.x), scale4(g, w4.x * aw));
        if (valid & 2) atomicAdd(reinterpret_cast<float4*>(gvb + o4.y), scale4(g, w4.y * aw));
        if (valid & 4) atomicAdd(reinterpret_cast<float4*>(gvb + o4.z), scale4(g, w4.z * aw));
        if (valid & 8) atomicAdd(reinterpret_cast<float4*>(gvb + o4.w), scale4(g, w4.w * aw));
      }
      for (int o = 4; o; o >>= 1) {
        sv += __shfl_xor_sync(0xffffffffu, sv, o);
        sh += __shfl_xor_sync(0xffffffffu, sh, o);
        sw += __shfl_xor_sync(0xffffffffu, sw, o);
      }
      if (FUSED) {
        __syncwarp();                                 // all lanes of the pair have read pf[s]: its lh is dead
        if (live && c == 0) {
          if constexpr (RW == 4) {
            const float2 wh = __ldg(reinterpret_cast<const float2*>(ref + (pair / M * L + l) * 4 + 2));
            st2(grad_loc + 2 * (pair * LP + s),
                make_float2(Wf * aw * sw * wh.x * 0.5f / (float)P, Hf * aw * sh * wh.y * 0.5f / (float)P));
          } else {
            st2(grad_loc + 2 * (pair * LP + s), make_float2(aw * sw, aw * sh));
          }
          pf[s].x = sv;
        }
        dot = fmaf(aw, sv, dot);
      } else if (live && c == 0) {
        const long long i = pair * LP + s;
        st1(grad_attn + i, sv);
        st2(grad_loc + 2 * i, make_float2(Wf * aw * sw, Hf * aw * sh));
      }
    }
  }
  if (FUSED) {                                        // softmax backward: the 8 lanes of a pair split its samples
    __syncwarp();
    if (live) {
      for (int s = threadIdx.x & 7; s < LP; s += 8) {
        const float4 f4 = pf[s];
        st1(grad_attn + pair * LP + s, f4.z * (f4.x - dot));
      }
    }
  }
  if constexpr (Acc::fixed) {
    if (bad) atomicMax(acc.gmax + (long long)n * M + m, MSDA_NAN_BITS);   // e.g. NaN softmax weights from NaN logits
  }
}

// Generic path (any D, float or double, 64-bit offsets): one warp per (query, head) pair, lanes stride over the
// channels, the three partials are summed with warp shuffles and lane 0 stores grad_attn / grad_loc.  grad_value takes
// plain scalar atomics (native for double on sm_90); with Acc = MsdaFixedAcc one 64-bit integer reduction per channel
// into acc.sum.
template <typename T, typename Acc = MsdaAtomicAcc>
__global__ void __launch_bounds__(256)
msda_backward_warp_kernel(const T* __restrict__ value, const MsdaLevels lv, const T* __restrict__ loc,
                          const T* __restrict__ attn, const T* __restrict__ grad_out, T* __restrict__ grad_value,
                          T* __restrict__ grad_loc, T* __restrict__ grad_attn, int N, int S, int M, int D, int L,
                          int Lq, int P, const Acc acc) {
  const long long pair = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (pair >= (long long)N * Lq * M) return;        // whole warps leave together
  const int lane = threadIdx.x & 31;
  const int m = (int)(pair % M);
  const long long n = pair / M / Lq;
  const long long pix = (long long)M * D;
  const long long vbase = n * S * pix + (long long)m * D;
  const T* vb = value + vbase;
  T* gvb = grad_value + vbase;
  const T* go = grad_out + pair * D;
  int sh_fx = 0;                                     // fixed point: s and 2^s of the pair's (n, m)
  double sc = 0.0;
  bool bad = false;
  if constexpr (Acc::fixed) {
    sh_fx = msda_fixed_shift(acc, n * M + m);
    sc = ldexp(1.0, sh_fx);
  }
  for (int l = 0; l < L; ++l) {
    const int H = (int)__ldg(lv.shapes + 2 * l), W = (int)__ldg(lv.shapes + 2 * l + 1);
    const long long start = __ldg(lv.start + l);
    for (int p = 0; p < P; ++p) {
      const long long i = (pair * L + l) * P + p;
      const T lx = loc[2 * i], ly = loc[2 * i + 1], aw = attn[i];
      const T h_im = ly * H - (T)0.5, w_im = lx * W - (T)0.5;
      T sv = 0, sh = 0, sw = 0;
      if (h_im > (T)-1 && w_im > (T)-1 && h_im < (T)H && w_im < (T)W) {
        const int h_low = (int)floor(h_im), w_low = (int)floor(w_im);
        const T lh = h_im - h_low, lw = w_im - w_low, hh = (T)1 - lh, hw = (T)1 - lw;
        const T w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
        const bool t = h_low >= 0, b = h_low + 1 <= H - 1, lf = w_low >= 0, rt = w_low + 1 <= W - 1;
        const long long o1 = (start + (long long)h_low * W + w_low) * pix, o2 = o1 + pix, o3 = o1 + W * pix,
                        o4 = o3 + pix;
        for (int c = lane; c < D; c += 32) {
          const T gc = go[c], ga = gc * aw;
          T v1 = 0, v2 = 0, v3 = 0, v4 = 0;
          if constexpr (Acc::fixed) {
            unsigned long long* sb = acc.sum + vbase + c;
            if (t && lf) { v1 = vb[o1 + c]; atomicAdd(sb + o1, msda_fixed(w1 * ga, sc, sh_fx, bad)); }
            if (t && rt) { v2 = vb[o2 + c]; atomicAdd(sb + o2, msda_fixed(w2 * ga, sc, sh_fx, bad)); }
            if (b && lf) { v3 = vb[o3 + c]; atomicAdd(sb + o3, msda_fixed(w3 * ga, sc, sh_fx, bad)); }
            if (b && rt) { v4 = vb[o4 + c]; atomicAdd(sb + o4, msda_fixed(w4 * ga, sc, sh_fx, bad)); }
          } else {
            if (t && lf) { v1 = vb[o1 + c]; atomicAdd(gvb + o1 + c, w1 * ga); }
            if (t && rt) { v2 = vb[o2 + c]; atomicAdd(gvb + o2 + c, w2 * ga); }
            if (b && lf) { v3 = vb[o3 + c]; atomicAdd(gvb + o3 + c, w3 * ga); }
            if (b && rt) { v4 = vb[o4 + c]; atomicAdd(gvb + o4 + c, w4 * ga); }
          }
          sv += gc * msda_bil(w1, w2, w3, w4, v1, v2, v3, v4);
          sh += gc * (hw * (v3 - v1) + lw * (v4 - v2));
          sw += gc * (hh * (v2 - v1) + lh * (v4 - v3));
        }
      }
      for (int o = 16; o; o >>= 1) {
        sv += __shfl_xor_sync(0xffffffffu, sv, o);
        sh += __shfl_xor_sync(0xffffffffu, sh, o);
        sw += __shfl_xor_sync(0xffffffffu, sw, o);
      }
      if (lane == 0) {
        grad_attn[i] = sv;
        grad_loc[2 * i] = (T)W * aw * sw;
        grad_loc[2 * i + 1] = (T)H * aw * sh;
      }
    }
  }
  if constexpr (Acc::fixed) {
    if (bad) atomicMax(acc.gmax + n * M + m, MSDA_NAN_BITS);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Deterministic backward: the passes around the fixed-point instantiations (MsdaFixedAcc above).

// Pre-pass: out[n * M + m] = max (as double bits) of |x[n, q, m, j]| over q < Lq, j < inner, for x [N, Lq, M, inner]
// (grad_out: inner = D; attn: inner = L * P).  A max is exact and the bit patterns of non-negative doubles order like
// their values, so atomicMax on the bits is deterministic; NaN (sign cleared) and +inf land at or above the bits of
// +inf, which marks the slice non-finite.  Block b covers slice b / chunks; its warps take every (chunks * 8)-th query
// row, the lanes stride over the row's `inner` elements.
template <typename T>
__global__ void __launch_bounds__(256)
msda_absmax_kernel(const T* __restrict__ x, unsigned long long* __restrict__ out, int M, int Lq, int inner,
                   int chunks) {
  const long long nm = blockIdx.x / chunks;
  const long long n = nm / M, m = nm % M;
  const int lane = threadIdx.x & 31;
  unsigned long long mx = 0;
  for (int q = (int)(blockIdx.x % chunks) * 8 + (threadIdx.x >> 5); q < Lq; q += chunks * 8) {
    const T* row = x + ((n * Lq + q) * M + m) * inner;
    for (int c = lane; c < inner; c += 32)
      mx = max(mx, (unsigned long long)__double_as_longlong(fabs(ld1d(row + c))));
  }
  for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0 && mx) atomicMax(out + nm, mx);
}

// Finalize: grad_value[n, i, m, c] = sum * 2^-s of its (n, m) slice in Tout; NaN in a non-finite slice.  The sum goes to
// double exactly while |sum| <= 2^53 and is then rounded once to Tout; a larger sum is rounded to double first (two
// roundings, still a function of the sum alone).
// One warp per pixel row (n, i) of M * D elements.
template <typename Tout>
__global__ void __launch_bounds__(256)
msda_fixed_finalize_kernel(const MsdaFixedAcc acc, Tout* __restrict__ grad_value, int N, int S, int M, int D) {
  const int lane = threadIdx.x & 31, MD = M * D;
  const long long rows = (long long)N * S, warps = (long long)gridDim.x * 8;
  for (long long r = blockIdx.x * 8LL + (threadIdx.x >> 5); r < rows; r += warps) {
    const long long n = r / S;
    for (int j = lane; j < MD; j += 32) {
      const long long nm = n * M + j / D, i = r * MD + j;
      double v;
      if (acc.gmax[nm] >= MSDA_INF_BITS || acc.amax[nm] >= MSDA_INF_BITS) v = __longlong_as_double(MSDA_NAN_BITS);
      else v = ldexp((double)(long long)acc.sum[i], -msda_fixed_shift(acc, nm));
      st1d(grad_value + i, v);
    }
  }
}

}  // namespace ob

using namespace ob;

// float: the D = 32 kernel where d32_ok, else the vec4 kernel where vec_ok(D), else the scalar kernel.  double: the
// scalar kernel for every D.
template <typename T>
static int msda_forward(const T* value, const int64_t* spatial_shapes, const int64_t* level_start, const T* loc,
                        const T* attn, T* out, int N, int S, int M, int D, int L, int Lq, int P, void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  if (!value || !spatial_shapes || !level_start || !loc || !attn || !out) return ODISE_ERR_ARG;
  if (N <= 0 || S <= 0 || M <= 0 || D <= 0 || L <= 0 || L > 8 || Lq <= 0 || P <= 0) return ODISE_ERR_ARG;
  MsdaLevels lv{spatial_shapes, level_start};
  bool launched = false;
  if constexpr (std::is_same<T, float>::value) {
    if (d32_ok(S, M, D, L, P)) {
      launch_d32<0>(value, lv, loc, attn, nullptr, out, nullptr, nullptr, N, S, M, L, Lq, P, stream);
      launched = true;
    } else if (vec_ok(D)) {
      const int lph = D / 4;
      const long long threads = (long long)N * Lq * M * lph;
      const int blocks = (int)((threads + 255) / 256);
      msda_vec4_kernel<0><<<blocks, 256, 0, stream>>>(value, lv, loc, attn, nullptr, out, nullptr, nullptr, N, S, M, D,
                                                      L, Lq, P, lph);
      launched = true;
    }
  }
  if (!launched) {
    const long long total = (long long)N * Lq * M * D;
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    msda_scalar_kernel<T><<<blocks, 256, 0, stream>>>(value, lv, loc, attn, out, N, S, M, D, L, Lq, P);
  }
  count_launch(1);
  return (int)cudaGetLastError();
}

#define MSDA_FORWARD(sfx, T)                                                                                           \
  extern "C" int odise_msda_forward_##sfx(const T* value, const int64_t* spatial_shapes, const int64_t* level_start,   \
                                          const T* loc, const T* attn, T* out, int N, int S, int M, int D, int L,      \
                                          int Lq, int P, void* stream) {                                               \
    return msda_forward<T>(value, spatial_shapes, level_start, loc, attn, out, N, S, M, D, L, Lq, P, stream);          \
  }
MSDA_FORWARD(f32, float)
MSDA_FORWARD(f64, double)

// Workspace of the deterministic backward entry points (odise_msda_det_workspace_bytes): the int64 sums [N, S, M, D],
// then per (n, m) the max-|grad_out| and max-|attn| bits of MsdaFixedAcc.
static long long det_ws_bytes(int N, int S, int M, int D) {
  return (long long)sizeof(unsigned long long) * ((long long)N * S * M * D + 2LL * N * M);
}

extern "C" long long odise_msda_det_workspace_bytes(int N, int S, int M, int D) {
  if (N <= 0 || S <= 0 || M <= 0 || D <= 0) return 0;
  return det_ws_bytes(N, S, M, D);
}

static MsdaFixedAcc det_acc(void* ws, int N, int S, int M, int D, int Lq, int P) {
  MsdaFixedAcc a;
  a.sum = static_cast<unsigned long long*>(ws);
  a.gmax = a.sum + (long long)N * S * M * D;
  a.amax = a.gmax + (long long)N * M;
  const long long K = (long long)Lq * P;
  a.log2k = 0;
  while ((1LL << a.log2k) < K) ++a.log2k;
  return a;
}

template <typename T>
static void launch_absmax(const T* x, unsigned long long* out, int N, int M, int Lq, int inner, cudaStream_t stream) {
  const long long slices = (long long)N * M;
  const long long most = (Lq + 7) / 8;                 // one query row per warp at least
  long long chunks = (4LL * num_sms() * 8 + slices - 1) / slices;
  if (chunks > most) chunks = most;
  msda_absmax_kernel<T><<<(unsigned)(slices * chunks), 256, 0, stream>>>(x, out, M, Lq, inner, (int)chunks);
}

// Zero the workspace and run the exponent pre-pass (attn == nullptr: the fused paths, A = 1).
template <typename T>
static int det_begin(const MsdaFixedAcc& a, void* ws, const T* grad_out, const T* attn, int N, int S, int M, int D,
                     int L, int Lq, int P, cudaStream_t stream) {
  cudaError_t e = cudaMemsetAsync(ws, 0, (size_t)det_ws_bytes(N, S, M, D), stream);
  if (e != cudaSuccess) return (int)e;
  launch_absmax<T>(grad_out, a.gmax, N, M, Lq, D, stream);
  if (attn) launch_absmax<T>(attn, const_cast<unsigned long long*>(a.amax), N, M, Lq, L * P, stream);
  return 0;
}

template <typename Tout>
static void det_finish(const MsdaFixedAcc& a, Tout* grad_value, int N, int S, int M, int D, cudaStream_t stream) {
  long long blocks = ((long long)N * S + 7) / 8;
  if (blocks > num_sms() * 16LL) blocks = num_sms() * 16LL;
  msda_fixed_finalize_kernel<Tout><<<(unsigned)blocks, 256, 0, stream>>>(a, grad_value, N, S, M, D);
}

// det = true: the deterministic twin (fixed-point grad_value through `ws`), otherwise the atomic default.
template <typename T>
static int msda_backward(const T* value, const int64_t* spatial_shapes, const int64_t* level_start, const T* loc,
                         const T* attn, const T* grad_out, T* grad_value, T* grad_loc, T* grad_attn, int N, int S, int M,
                         int D, int L, int Lq, int P, bool det, void* ws, void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  if (!value || !spatial_shapes || !level_start || !loc || !attn || !grad_out || !grad_value || !grad_loc || !grad_attn)
    return ODISE_ERR_ARG;
  if (det && !ws) return ODISE_ERR_WORKSPACE;
  if (N <= 0 || S <= 0 || M <= 0 || D <= 0 || L <= 0 || L > 8 || Lq <= 0 || P <= 0) return ODISE_ERR_ARG;
  const long long pairs = (long long)N * Lq * M;
  if ((pairs + 7) / 8 > 0x7fffffffLL) return ODISE_ERR_ARG;   // grid of the generic path
  MsdaLevels lv{spatial_shapes, level_start};
  MsdaFixedAcc fx{};
  if (det) {
    fx = det_acc(ws, N, S, M, D, Lq, P);
    const int rc = det_begin<T>(fx, ws, grad_out, attn, N, S, M, D, L, Lq, P, stream);
    if (rc) return rc;
  } else {
    // the reference returns at::zeros_like(value) plus the scattered contributions
    cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(T) * (size_t)N * S * M * D, stream);
    if (e != cudaSuccess) return (int)e;
  }
  auto run = [&](auto acc) {
    using Acc = decltype(acc);
    bool d32 = false;
    if constexpr (std::is_same<T, float>::value) {
      if (d32_ok(S, M, D, L, P)) {
        // 48 B of shared memory per (pair, sample): at most 32 x 32 x 48 = 48 KB, the default dynamic limit
        const size_t smem = (size_t)MSDA_PAIRS * L * P * (sizeof(int4) + 2 * sizeof(float4));
        const int blocks = (int)((pairs + MSDA_PAIRS - 1) / MSDA_PAIRS);
        msda_d32_backward_kernel<0, float, Acc><<<blocks, 256, smem, stream>>>(
            value, lv, loc, attn, grad_out, grad_value, grad_loc, grad_attn, N, S, M, L, Lq, P, nullptr, 1, acc);
        d32 = true;
      }
    }
    if (!d32) {
      const long long blocks = (pairs + 7) / 8;       // one warp per (query, head) pair
      msda_backward_warp_kernel<T, Acc><<<(unsigned)blocks, 256, 0, stream>>>(
          value, lv, loc, attn, grad_out, grad_value, grad_loc, grad_attn, N, S, M, D, L, Lq, P, acc);
    }
  };
  if (det) {
    run(fx);
    det_finish<T>(fx, grad_value, N, S, M, D, stream);
    count_launch(4);
  } else {
    run(MsdaAtomicAcc{});
    count_launch(1);
  }
  return (int)cudaGetLastError();
}

#define MSDA_BACKWARD(sfx, T)                                                                                          \
  extern "C" int odise_msda_backward_##sfx(const T* value, const int64_t* spatial_shapes, const int64_t* level_start,  \
                                           const T* loc, const T* attn, const T* grad_out, T* grad_value,              \
                                           T* grad_loc, T* grad_attn, int N, int S, int M, int D, int L, int Lq,       \
                                           int P, void* stream) {                                                      \
    return msda_backward<T>(value, spatial_shapes, level_start, loc, attn, grad_out, grad_value, grad_loc, grad_attn,  \
                            N, S, M, D, L, Lq, P, false, nullptr, stream);                                             \
  }                                                                                                                    \
  extern "C" int odise_msda_backward_det_##sfx(const T* value, const int64_t* spatial_shapes,                          \
                                               const int64_t* level_start, const T* loc, const T* attn,                \
                                               const T* grad_out, T* grad_value, T* grad_loc, T* grad_attn, int N,     \
                                               int S, int M, int D, int L, int Lq, int P, void* workspace,             \
                                               void* stream) {                                                         \
    return msda_backward<T>(value, spatial_shapes, level_start, loc, attn, grad_out, grad_value, grad_loc, grad_attn,  \
                            N, S, M, D, L, Lq, P, true, workspace, stream);                                            \
  }
MSDA_BACKWARD(f32, float)
MSDA_BACKWARD(f64, double)

extern "C" int odise_msda_fused_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                    const float* ref, const float* offs, const float* logits, float* out,
                                    void* out_hi, void* out_lo, int N, int S, int M, int D, int L, int Lq, int P,
                                    void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  if (!value || !spatial_shapes || !level_start || !ref || !offs || !logits || (!out && !out_hi)) return ODISE_ERR_ARG;
  if (N <= 0 || S <= 0 || M <= 0 || L <= 0 || L > 8 || Lq <= 0 || P <= 0 || !vec_ok(D)) return ODISE_ERR_ARG;
  MsdaLevels lv{spatial_shapes, level_start};
  if (d32_ok(S, M, D, L, P)) {
    launch_d32<1>(value, lv, offs, logits, ref, out, reinterpret_cast<__nv_bfloat16*>(out_hi),
                  lo_arg(reinterpret_cast<__nv_bfloat16*>(out_lo)), N, S, M, L, Lq, P, stream);
  } else {
    const int lph = D / 4;
    const long long threads = (long long)N * Lq * M * lph;
    const int blocks = (int)((threads + 255) / 256);
    msda_vec4_kernel<1><<<blocks, 256, 0, stream>>>(value, lv, offs, logits, ref, out,
                                                    reinterpret_cast<__nv_bfloat16*>(out_hi),
                                                    lo_arg(reinterpret_cast<__nv_bfloat16*>(out_lo)), N, S, M, D, L, Lq, P, lph);
  }
  count_launch(1);
  return (int)cudaGetLastError();
}

// a box reference point [N, Lq, L, 4] is one 16-byte load
static bool ref_ok(const float* ref, int RW) { return RW == 2 || reinterpret_cast<uintptr_t>(ref) % 16 == 0; }

// The fused forward on the D = 32 kernel alone, without planes: 16-bit storage T with RW = 2 (odise_msda_fused_f16 /
// _bf16), and box reference points [N, Lq, L, 4] (cx, cy, w, h) with RW = 4 in every storage type
// (odise_msda_fused_box_f32 / _f16 / _bf16; include/odise_b200.h states the formulas).
template <typename T, int RW>
static int msda_fused_d32(const void* value_v, const int64_t* spatial_shapes, const int64_t* level_start,
                          const float* ref, const void* offs_v, const void* logits_v, void* out_v, int N, int S, int M,
                          int D, int L, int Lq, int P, void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  if (!value_v || !spatial_shapes || !level_start || !ref || !offs_v || !logits_v || !out_v) return ODISE_ERR_ARG;
  if (N <= 0 || S <= 0 || M <= 0 || D <= 0 || L <= 0 || L > 8 || Lq <= 0 || P <= 0) return ODISE_ERR_ARG;
  if (!ref_ok(ref, RW)) return ODISE_ERR_ARG;
  if (!d32_ok(S, M, D, L, P)) return ODISE_ERR_UNSUPPORTED;
  if (((long long)N * Lq * M + MSDA_PAIRS - 1) / MSDA_PAIRS > 0x7fffffffLL) return ODISE_ERR_ARG;
  MsdaLevels lv{spatial_shapes, level_start};
  launch_d32<1, T, RW>(static_cast<const T*>(value_v), lv, static_cast<const T*>(offs_v),
                       static_cast<const T*>(logits_v), ref, static_cast<T*>(out_v), nullptr, nullptr, N, S, M, L, Lq,
                       P, stream);
  count_launch(1);
  return (int)cudaGetLastError();
}

// Arg: what the entry point's storage pointers point to (float, or void for 16-bit storage).
#define MSDA_FUSED_D32(kind, sfx, Arg, T, RW)                                                                          \
  extern "C" int odise_msda_##kind##_##sfx(const Arg* value, const int64_t* spatial_shapes,                            \
                                           const int64_t* level_start, const float* ref, const Arg* offs,              \
                                           const Arg* logits, Arg* out, int N, int S, int M, int D, int L, int Lq,     \
                                           int P, void* stream) {                                                      \
    return msda_fused_d32<T, RW>(value, spatial_shapes, level_start, ref, offs, logits, out, N, S, M, D, L, Lq, P,     \
                                 stream);                                                                              \
  }
MSDA_FUSED_D32(fused, f16, void, __half, 2)
MSDA_FUSED_D32(fused, bf16, void, __nv_bfloat16, 2)
MSDA_FUSED_D32(fused_box, f32, float, float, 4)
MSDA_FUSED_D32(fused_box, f16, void, __half, 4)
MSDA_FUSED_D32(fused_box, bf16, void, __nv_bfloat16, 4)

// The fused backward for storage type T.  Default (det = false): grad_value is an fp32 buffer for every T, accumulated
// with fp32 atomics.  det = true: grad_value is in T, written by the fixed-point finalize pass through `ws`.  RW = 4:
// box reference points.
template <typename T, int RW>
static int msda_fused_backward(const void* value_v, const int64_t* spatial_shapes, const int64_t* level_start,
                               const float* ref, const void* offs_v, const void* logits_v, const void* grad_out_v,
                               void* grad_value, void* grad_offs_v, void* grad_logits_v, int N, int S, int M, int D,
                               int L, int Lq, int P, bool det, void* ws, void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const T *value = static_cast<const T*>(value_v), *offs = static_cast<const T*>(offs_v);
  const T *logits = static_cast<const T*>(logits_v), *grad_out = static_cast<const T*>(grad_out_v);
  T *grad_offs = static_cast<T*>(grad_offs_v), *grad_logits = static_cast<T*>(grad_logits_v);
  if (!value || !spatial_shapes || !level_start || !ref || !offs || !logits || !grad_out || !grad_value || !grad_offs ||
      !grad_logits)
    return ODISE_ERR_ARG;
  if (det && !ws) return ODISE_ERR_WORKSPACE;
  if (N <= 0 || S <= 0 || M <= 0 || D <= 0 || L <= 0 || L > 8 || Lq <= 0 || P <= 0) return ODISE_ERR_ARG;
  if (!ref_ok(ref, RW)) return ODISE_ERR_ARG;
  if (!d32_ok(S, M, D, L, P)) return ODISE_ERR_UNSUPPORTED;
  const long long pairs = (long long)N * Lq * M;
  const long long blocks = (pairs + MSDA_PAIRS - 1) / MSDA_PAIRS;
  if (blocks > 0x7fffffffLL) return ODISE_ERR_ARG;
  MsdaLevels lv{spatial_shapes, level_start};
  MsdaFixedAcc fx{};
  if (det) {
    fx = det_acc(ws, N, S, M, D, Lq, P);
    const int rc = det_begin<T>(fx, ws, grad_out, nullptr, N, S, M, D, L, Lq, P, stream);
    if (rc) return rc;
  } else {
    cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * (size_t)N * S * M * D, stream);
    if (e != cudaSuccess) return (int)e;
  }
  const int LP = L * P;
  int SL = 1;
  while (SL < LP) SL <<= 1;
  // 48 B of shared memory per (pair, sample), as in the non-fused backward: at most 48 KB at L*P = 32
  const size_t smem = (size_t)MSDA_PAIRS * LP * (sizeof(int4) + 2 * sizeof(float4));
  if (det) {
    msda_d32_backward_kernel<1, T, MsdaFixedAcc, RW><<<(unsigned)blocks, 256, smem, stream>>>(
        value, lv, offs, logits, grad_out, nullptr, grad_offs, grad_logits, N, S, M, L, Lq, P, ref, SL, fx);
    det_finish<T>(fx, static_cast<T*>(grad_value), N, S, M, D, stream);
    count_launch(3);
  } else {
    msda_d32_backward_kernel<1, T, MsdaAtomicAcc, RW><<<(unsigned)blocks, 256, smem, stream>>>(
        value, lv, offs, logits, grad_out, static_cast<float*>(grad_value), grad_offs, grad_logits, N, S, M, L, Lq, P,
        ref, SL, MsdaAtomicAcc{});
    count_launch(1);
  }
  return (int)cudaGetLastError();
}

// The default entry point takes grad_value in fp32; its deterministic twin adds the workspace and takes grad_value in
// the storage type.
#define MSDA_FUSED_BACKWARD(kind, sfx, Arg, T, RW)                                                                     \
  extern "C" int odise_msda_##kind##_backward_##sfx(                                                                   \
      const Arg* value, const int64_t* spatial_shapes, const int64_t* level_start, const float* ref, const Arg* offs,  \
      const Arg* logits, const Arg* grad_out, float* grad_value, Arg* grad_offs, Arg* grad_logits, int N, int S,       \
      int M, int D, int L, int Lq, int P, void* stream) {                                                              \
    return msda_fused_backward<T, RW>(value, spatial_shapes, level_start, ref, offs, logits, grad_out, grad_value,     \
                                      grad_offs, grad_logits, N, S, M, D, L, Lq, P, false, nullptr, stream);           \
  }                                                                                                                    \
  extern "C" int odise_msda_##kind##_backward_det_##sfx(                                                               \
      const Arg* value, const int64_t* spatial_shapes, const int64_t* level_start, const float* ref, const Arg* offs,  \
      const Arg* logits, const Arg* grad_out, Arg* grad_value, Arg* grad_offs, Arg* grad_logits, int N, int S,         \
      int M, int D, int L, int Lq, int P, void* workspace, void* stream) {                                             \
    return msda_fused_backward<T, RW>(value, spatial_shapes, level_start, ref, offs, logits, grad_out, grad_value,     \
                                      grad_offs, grad_logits, N, S, M, D, L, Lq, P, true, workspace, stream);          \
  }
MSDA_FUSED_BACKWARD(fused, f32, float, float, 2)
MSDA_FUSED_BACKWARD(fused, f16, void, __half, 2)
MSDA_FUSED_BACKWARD(fused, bf16, void, __nv_bfloat16, 2)
MSDA_FUSED_BACKWARD(fused_box, f32, float, float, 4)
MSDA_FUSED_BACKWARD(fused_box, f16, void, __half, 4)
MSDA_FUSED_BACKWARD(fused_box, bf16, void, __nv_bfloat16, 4)
