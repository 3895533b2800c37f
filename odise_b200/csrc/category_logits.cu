// Category scoring of ODISE training (CategoryODISE.cal_pred_logits, odise.py:181-207, with
// ensemble_logits_with_labels(..., "max"), helper.py:79-109) on sm_90a, forward and deterministic backward:
//
//   m^_r = x_r / max(|x_r|, 1e-12)        (F.normalize; likewise t^_j for the prompt bank and n^ for the null row)
//   s_rj = scale <m^_r, t^_j>             out[r, k] = max_{j in class k} s_rj,   out[r, K] = scale <m^_r, n^>
//
// The null row is handled as prompt Kp, the single prompt of a class K, so every column of out is a group max and the
// null gradient is a prompt gradient.  Storage type T of mask_embed and out (float, __half or __nv_bfloat16) and Tb of
// the bank (T, or float for a constant float32 bank under autocast); all arithmetic fp32.  In 16 bits every value the
// reference rounds is rounded here in the same place: m^ and t^ to T (autocast casts the fp32 normalised operands to
// the matmul's dtype), the dot product (fp32 accumulation) to T, and scale to T before the multiply (torch casts the
// fp32 0-dim factor to the 16-bit common dtype), whose fp32 product is rounded to T once.
//
// Forward, one launch: a CTA owns CL_RT mask rows; one warp per row normalises it into shared memory.  The CTA walks
// the classes in windows of whole classes covering at most CL_NT prompts (groups have at most 255 prompts, so every
// window holds at least one class); a thread per prompt normalises its bank row and takes its dot products with the
// CTA's rows (fp32 FMA in ascending channel order), and then a thread per (row, class) takes the group max, scanning the
// stored scores in ascending prompt order: the lowest index wins among equal values, and the first NaN wins over every
// number, as torch's max(dim).  The winner's offset in its group is stored as a byte.  CTA 0 also stores the bank's
// clamped norms.  Every CTA normalises the same bank rows with the same instructions, so they agree bit for bit.
//
// Backward, three launches, no atomics:
//   rows   a CTA per mask row: acc = sum_k g[r, k] t^_win(r, k) (ascending k), grad m^ = scale acc, then the normalize
//          backward; the row's scale partial <m^, acc> (= sum_k g s / scale) and m^ itself go to the workspace.
//   bank   a warp per (prompt j, row split): sum over the split's rows, ascending, of g[r, k(j)] m^_r where j won;
//          partials [split][Kp+1][C] in the workspace.
//   final  a warp per prompt: the partials summed in split order, times scale, then the normalize backward; one more
//          CTA sums the scale partials in row order.
// The splits depend on the shape only, so every gradient is bit-reproducible.
#include <stdint.h>

#include "launch_count.h"
#include "odise_b200.h"
#include "storage.cuh"

namespace ob {
namespace {

constexpr int CL_NT = 256;          // threads per CTA
constexpr int CL_W = CL_NT / 32;
constexpr int CL_RT = 8;            // mask rows per forward CTA: one warp each
constexpr int CL_MAX_C = 768;
constexpr int CL_CPL = CL_MAX_C / 32;    // channels per lane (bank kernels)
constexpr int CL_CPT = CL_MAX_C / CL_NT; // channels per thread (row kernel)
constexpr int CL_MAX_KP = 2048;
constexpr int CL_MAX_SPLITS = 16;
constexpr float CL_EPS = 1e-12f;

// v rounded to T and widened back (exact); float is the identity
__device__ __forceinline__ float rt(float v, float*) { return v; }
__device__ __forceinline__ float rt(float v, __half*) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float rt(float v, __nv_bfloat16*) { return __bfloat162float(__float2bfloat16_rn(v)); }
template <typename T>
__device__ __forceinline__ float rt(float v) { return rt(v, (T*)nullptr); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// the clamped norm max(|x|, 1e-12) of a row of C values read by one thread, ascending
template <typename Tb>
__device__ __forceinline__ float row_norm(const Tb* x, int C) {
  float ss = 0.f;
  for (int c = 0; c < C; ++c) {
    const float v = ld1(x + c);
    ss = __fmaf_rn(v, v, ss);
  }
  return fmaxf(__fsqrt_rn(ss), CL_EPS);
}

// the bank row of prompt j (the null row is prompt Kp)
template <typename Tb>
__device__ __forceinline__ const Tb* bank_row(const Tb* te, const Tb* ne, int j, int Kp, int C) {
  return j < Kp ? te + (long long)j * C : ne;
}

template <typename T, typename Tb>
__global__ void __launch_bounds__(CL_NT)
cl_forward_kernel(const T* __restrict__ me, const Tb* __restrict__ te, const Tb* __restrict__ ne,
                  const float* __restrict__ scale_p, const int32_t* __restrict__ group_start, T* __restrict__ out,
                  uint8_t* __restrict__ win, float* __restrict__ norms, int R, int C, int K, int Kp) {
  __shared__ __align__(16) float mh[CL_RT * CL_MAX_C];
  __shared__ float sc[CL_RT][CL_NT];
  __shared__ int gs[CL_MAX_KP + 2];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int r0 = blockIdx.x * CL_RT, nr = min(CL_RT, R - r0);
  for (int k = tid; k < K; k += CL_NT) gs[k] = __ldg(group_start + k);
  if (tid == 0) {
    gs[K] = Kp;
    gs[K + 1] = Kp + 1;
  }
  const float st = rt<T>(__ldg(scale_p));
  {
    float* m = mh + wid * C;
    if (wid < nr) {
      const T* x = me + (long long)(r0 + wid) * C;
      float ss = 0.f;
      for (int c = lane; c < C; c += 32) {
        const float v = ld1(x + c);
        ss = __fmaf_rn(v, v, ss);
      }
      const float d = fmaxf(__fsqrt_rn(warp_sum(ss)), CL_EPS);
      for (int c = lane; c < C; c += 32) m[c] = rt<T>(__fdiv_rn(ld1(x + c), d));
      if (lane == 0) norms[r0 + wid] = d;
    } else {
      for (int c = lane; c < C; c += 32) m[c] = 0.f;
    }
  }
  __syncthreads();
  for (int k0 = 0; k0 <= K;) {
    const int p0 = gs[k0];
    int lo = k0 + 1, hi = K + 1;    // k1: the last class boundary within CL_NT prompts of p0
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (gs[mid] - p0 <= CL_NT)
        lo = mid;
      else
        hi = mid - 1;
    }
    const int k1 = lo, np = gs[k1] - p0;
    if (tid < np) {
      const int j = p0 + tid;
      const Tb* t = bank_row(te, ne, j, Kp, C);
      const float d = row_norm(t, C);
      if (blockIdx.x == 0) norms[R + j] = d;
      float acc[CL_RT];
#pragma unroll
      for (int r = 0; r < CL_RT; ++r) acc[r] = 0.f;
      for (int c = 0; c < C; c += 4) {
        const float t0 = rt<T>(__fdiv_rn(ld1(t + c), d)), t1 = rt<T>(__fdiv_rn(ld1(t + c + 1), d));
        const float t2 = rt<T>(__fdiv_rn(ld1(t + c + 2), d)), t3 = rt<T>(__fdiv_rn(ld1(t + c + 3), d));
#pragma unroll
        for (int r = 0; r < CL_RT; ++r) {
          const float4 m = *reinterpret_cast<const float4*>(mh + r * C + c);
          acc[r] = __fmaf_rn(m.w, t3, __fmaf_rn(m.z, t2, __fmaf_rn(m.y, t1, __fmaf_rn(m.x, t0, acc[r]))));
        }
      }
#pragma unroll
      for (int r = 0; r < CL_RT; ++r) sc[r][tid] = rt<T>(__fmul_rn(rt<T>(acc[r]), st));
    }
    __syncthreads();
    const int nk = k1 - k0;
    for (int e = tid; e < nr * nk; e += CL_NT) {
      const int r = e / nk, k = k0 + e - r * nk;
      const int a = gs[k] - p0, b = gs[k + 1] - p0;
      float best = sc[r][a];
      int bi = a;
      for (int i = a + 1; i < b; ++i) {
        const float v = sc[r][i];
        if (v > best || (v != v && best == best)) {
          best = v;
          bi = i;
        }
      }
      const long long o = (long long)(r0 + r) * (K + 1) + k;
      st1(out + o, best);
      win[o] = (uint8_t)(bi - a);
    }
    __syncthreads();
    k0 = k1;
  }
}

// grad of x from grad y of y = x / d, d = max(|x|, eps): (gy - x^ <gy, x^>) / d, or gy / d where the norm was clamped
__device__ __forceinline__ float normalize_grad(float gy, float xh, float dot, float d) {
  return d > CL_EPS ? __fdiv_rn(__fsub_rn(gy, __fmul_rn(xh, dot)), d) : __fdiv_rn(gy, d);
}

template <typename T, typename Tb>
__global__ void __launch_bounds__(CL_NT)
cl_backward_rows_kernel(const T* __restrict__ me, const Tb* __restrict__ te, const Tb* __restrict__ ne,
                        const float* __restrict__ scale_p, const int32_t* __restrict__ group_start,
                        const uint8_t* __restrict__ win, const float* __restrict__ norms, const T* __restrict__ gout,
                        T* __restrict__ gme, float* __restrict__ ws_m, float* __restrict__ ws_scale, int R, int C, int K,
                        int Kp) {
  __shared__ int sj[CL_MAX_KP + 1];
  __shared__ float sg[CL_MAX_KP + 1];
  __shared__ float red[2][CL_W];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int k = tid; k <= K; k += CL_NT) {
    const long long o = (long long)r * (K + 1) + k;
    sj[k] = (k < K ? __ldg(group_start + k) : Kp) + win[o];
    sg[k] = ld1(gout + o);
  }
  __syncthreads();
  float acc[CL_CPT];
#pragma unroll
  for (int q = 0; q < CL_CPT; ++q) acc[q] = 0.f;
#pragma unroll 4
  for (int k = 0; k <= K; ++k) {
    const int j = sj[k];
    const float g = sg[k], d = __ldg(norms + R + j);
    const Tb* t = bank_row(te, ne, j, Kp, C);
#pragma unroll
    for (int q = 0; q < CL_CPT; ++q) {
      const int c = tid + q * CL_NT;
      if (c < C) acc[q] = __fmaf_rn(g, rt<T>(__fdiv_rn(ld1(t + c), d)), acc[q]);
    }
  }
  const float d = __ldg(norms + r), se = rt<T>(__ldg(scale_p));
  const T* x = me + (long long)r * C;
  float xh[CL_CPT], a = 0.f, b = 0.f;
#pragma unroll
  for (int q = 0; q < CL_CPT; ++q) {
    const int c = tid + q * CL_NT;
    xh[q] = 0.f;
    if (c < C) {
      xh[q] = __fdiv_rn(ld1(x + c), d);
      const float m = rt<T>(xh[q]);
      ws_m[(long long)r * C + c] = m;
      a = __fmaf_rn(m, acc[q], a);
      b = __fmaf_rn(xh[q], __fmul_rn(se, acc[q]), b);
    }
  }
  a = warp_sum(a);
  b = warp_sum(b);
  if (lane == 0) {
    red[0][wid] = a;
    red[1][wid] = b;
  }
  __syncthreads();
  a = 0.f;
  b = 0.f;
#pragma unroll
  for (int w = 0; w < CL_W; ++w) {
    a += red[0][w];
    b += red[1][w];
  }
  if (tid == 0) ws_scale[r] = a;
#pragma unroll
  for (int q = 0; q < CL_CPT; ++q) {
    const int c = tid + q * CL_NT;
    if (c < C) st1(gme + (long long)r * C + c, normalize_grad(__fmul_rn(se, acc[q]), xh[q], b, d));
  }
}

template <typename T>
__global__ void __launch_bounds__(CL_NT)
cl_backward_bank_kernel(const float* __restrict__ ws_m, const int32_t* __restrict__ group_start,
                        const uint8_t* __restrict__ win, const T* __restrict__ gout, float* __restrict__ ws_bank, int R,
                        int C, int K, int Kp, int rows_per_split) {
  const int lane = threadIdx.x & 31, j = blockIdx.x * CL_W + (threadIdx.x >> 5), s = blockIdx.y;
  if (j > Kp) return;
  int k = K, g0 = Kp;    // the class of j and its first prompt (the null row is class K)
  if (j < Kp) {
    int lo = 0, hi = K - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(group_start + mid) <= j)
        lo = mid;
      else
        hi = mid - 1;
    }
    k = lo;
    g0 = __ldg(group_start + k);
  }
  const int off = j - g0;
  float acc[CL_CPL];
#pragma unroll
  for (int q = 0; q < CL_CPL; ++q) acc[q] = 0.f;
  const int rb = s * rows_per_split, re = min(R, rb + rows_per_split);
  for (int c0 = rb; c0 < re; c0 += 32) {
    const int rl = c0 + lane;
    bool hit = false;
    float g = 0.f;
    if (rl < re) {
      const long long o = (long long)rl * (K + 1) + k;
      hit = win[o] == off;
      g = ld1(gout + o);
    }
    for (unsigned hits = __ballot_sync(0xffffffffu, hit); hits; hits &= hits - 1) {
      const int l = __ffs(hits) - 1, rr = c0 + l;
      const float gl = __shfl_sync(0xffffffffu, g, l);
      const float* m = ws_m + (long long)rr * C;
#pragma unroll
      for (int q = 0; q < CL_CPL; ++q) {
        const int c = lane + 32 * q;
        if (c < C) acc[q] = __fmaf_rn(gl, __ldg(m + c), acc[q]);
      }
    }
  }
  float* w = ws_bank + ((long long)s * (Kp + 1) + j) * C;
#pragma unroll
  for (int q = 0; q < CL_CPL; ++q) {
    const int c = lane + 32 * q;
    if (c < C) w[c] = acc[q];
  }
}

template <typename T, typename Tb>
__global__ void __launch_bounds__(CL_NT)
cl_backward_final_kernel(const Tb* __restrict__ te, const Tb* __restrict__ ne, const float* __restrict__ scale_p,
                         const float* __restrict__ norms, const float* __restrict__ ws_bank,
                         const float* __restrict__ ws_scale, Tb* __restrict__ gte, Tb* __restrict__ gne,
                         float* __restrict__ gscale, int R, int C, int Kp, int nsplit) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (blockIdx.x == gridDim.x - 1) {    // the scale gradient: the rows' partials in row order
    if (wid) return;
    float s = 0.f;
    for (int r = lane; r < R; r += 32) s += ws_scale[r];
    s = warp_sum(s);
    if (lane == 0) *gscale = s;
    return;
  }
  const int j = blockIdx.x * CL_W + wid;
  if (j > Kp) return;
  const float se = rt<T>(__ldg(scale_p)), d = __ldg(norms + R + j);
  const Tb* t = bank_row(te, ne, j, Kp, C);
  const float* p = ws_bank + (long long)j * C;
  const long long ps = (long long)(Kp + 1) * C;
  // grad t^ = scale * (the partials in split order); two passes, the first for <grad t^, t / d>
  float b = 0.f;
  for (int c = lane; c < C; c += 32) {
    float v = 0.f;
    for (int s = 0; s < nsplit; ++s) v += p[s * ps + c];
    b = __fmaf_rn(__fmul_rn(se, v), __fdiv_rn(ld1(t + c), d), b);
  }
  b = warp_sum(b);
  Tb* gt = j < Kp ? gte + (long long)j * C : gne;
  for (int c = lane; c < C; c += 32) {
    float v = 0.f;
    for (int s = 0; s < nsplit; ++s) v += p[s * ps + c];
    st1(gt + c, normalize_grad(__fmul_rn(se, v), __fdiv_rn(ld1(t + c), d), b, d));
  }
}

int cl_check(int R, int C, int K, int Kp) {
  if (R <= 0 || C <= 0 || K <= 0 || Kp < K) return ODISE_ERR_ARG;
  if (C % 32 || C > CL_MAX_C || Kp > CL_MAX_KP || (long long)R * (K + 1) >= (1LL << 31) ||
      (long long)R * C >= (1LL << 31))
    return ODISE_ERR_UNSUPPORTED;
  return 0;
}

int cl_splits(int R) { return min((R + 31) / 32, CL_MAX_SPLITS); }

template <typename T, typename Tb>
int cl_forward(const void* me, const void* te, const void* ne, const float* scale, const int32_t* gs, void* out,
               uint8_t* win, float* norms, int R, int C, int K, int Kp, void* stream) {
  if (!me || !te || !ne || !scale || !gs || !out || !win || !norms) return ODISE_ERR_ARG;
  if (const int rc = cl_check(R, C, K, Kp)) return rc;
  cl_forward_kernel<T, Tb><<<(R + CL_RT - 1) / CL_RT, CL_NT, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      (const T*)me, (const Tb*)te, (const Tb*)ne, scale, gs, (T*)out, win, norms, R, C, K, Kp);
  count_launch(1);
  return (int)cudaGetLastError();
}

template <typename T, typename Tb>
int cl_backward(const void* me, const void* te, const void* ne, const float* scale, const int32_t* gs,
                const uint8_t* win, const float* norms, const void* gout, void* gme, void* gte, void* gne,
                float* gscale, int R, int C, int K, int Kp, void* workspace, void* stream) {
  if (!me || !te || !ne || !scale || !gs || !win || !norms || !gout || !gme || !gte || !gne || !gscale)
    return ODISE_ERR_ARG;
  if (const int rc = cl_check(R, C, K, Kp)) return rc;
  if (!workspace) return ODISE_ERR_WORKSPACE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int ns = cl_splits(R), rps = (R + ns - 1) / ns;
  float* ws_bank = (float*)workspace;
  float* ws_m = ws_bank + (long long)ns * (Kp + 1) * C;
  float* ws_scale = ws_m + (long long)R * C;
  cl_backward_rows_kernel<T, Tb><<<R, CL_NT, 0, st>>>((const T*)me, (const Tb*)te, (const Tb*)ne, scale, gs, win,
                                                      norms, (const T*)gout, (T*)gme, ws_m, ws_scale, R, C, K, Kp);
  const int bank_ctas = (Kp + 1 + CL_W - 1) / CL_W;
  cl_backward_bank_kernel<T><<<dim3(bank_ctas, ns), CL_NT, 0, st>>>(ws_m, gs, win, (const T*)gout, ws_bank, R, C, K,
                                                                   Kp, rps);
  cl_backward_final_kernel<T, Tb><<<bank_ctas + 1, CL_NT, 0, st>>>((const Tb*)te, (const Tb*)ne, scale, norms,
                                                                   ws_bank, ws_scale, (Tb*)gte, (Tb*)gne, gscale, R,
                                                                   C, Kp, ns);
  count_launch(3);
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace ob

extern "C" long long odise_category_logits_workspace_bytes(int R, int C, int K, int Kp) {
  if (ob::cl_check(R, C, K, Kp)) return 0;
  return ((long long)ob::cl_splits(R) * (Kp + 1) * C + (long long)R * C + R) * (long long)sizeof(float);
}

#define CL_ENTRY(sfx, T)                                                                                               \
  extern "C" int odise_category_logits_forward_##sfx(                                                                  \
      const void* mask_embed, const void* text_embed, const void* null_embed, const float* logit_scale,                \
      const int32_t* group_start, void* logits, uint8_t* winners, float* norms, int R, int C, int K, int Kp,           \
      int bank_f32, void* stream) {                                                                                    \
    auto fn = bank_f32 ? ob::cl_forward<T, float> : ob::cl_forward<T, T>;                                              \
    return fn(mask_embed, text_embed, null_embed, logit_scale, group_start, logits, winners, norms, R, C, K, Kp,       \
              stream);                                                                                                 \
  }                                                                                                                    \
  extern "C" int odise_category_logits_backward_##sfx(                                                                 \
      const void* mask_embed, const void* text_embed, const void* null_embed, const float* logit_scale,                \
      const int32_t* group_start, const uint8_t* winners, const float* norms, const void* grad_logits,                 \
      void* grad_mask_embed, void* grad_text_embed, void* grad_null_embed, float* grad_logit_scale, int R, int C,      \
      int K, int Kp, int bank_f32, void* workspace, void* stream) {                                                    \
    auto fn = bank_f32 ? ob::cl_backward<T, float> : ob::cl_backward<T, T>;                                            \
    return fn(mask_embed, text_embed, null_embed, logit_scale, group_start, winners, norms, grad_logits,               \
              grad_mask_embed, grad_text_embed, grad_null_embed, grad_logit_scale, R, C, K, Kp, workspace, stream);    \
  }
CL_ENTRY(f32, float)
CL_ENTRY(f16, __half)
CL_ENTRY(bf16, __nv_bfloat16)
