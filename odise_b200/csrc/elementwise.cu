// HBM-bound elementwise / normalisation passes of the ODISE hot path (sm_90a).  Activations are NHWC /
// token-major fp32; every pass that feeds a GEMM also writes the (hi, lo) bf16 operand planes, so the
// fp32 -> bf16x2 split is never a pass of its own.  Reference ops replaced (all individual ATen kernels in
// the reference, SURVEY.md §2.4 "Fused ops: none"): nn.GroupNorm + SiLU (ldm ResBlock / Normalize),
// nn.LayerNorm (+ residual, + with_pos_embed: mask2former_transformer_decoder.py:40-50,98-110,163-167),
// ldm GEGLU, ldm Upsample (nearest x2), F.interpolate (feature_extractor.py:165, msdeformattn.py:349),
// torch.cat skip concat (ldm.py:485), crop paste (feature_extractor.py:243-248), F.normalize + per-class max
// (odise.py:181-207, helper.py:96-100), MaskPooling threshold / normalise (odise.py:945-959).
#include <cstdlib>
#include "ptx.cuh"
#include "odise_b200.h"
#include "launch_count.h"
#include <atomic>

namespace ob {

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static inline int grid_for(long long work, int threads, int max_blocks = 0) {
  if (max_blocks <= 0) max_blocks = num_sms() * 16;
  long long b = (work + threads - 1) / threads;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

__device__ __forceinline__ float act_apply(float v, int act) {
  if (act == ODISE_ACT_RELU) return fmaxf(v, 0.f);
  // SiLU with the MUFU-based intrinsics (~2 ulp): the libm expf + IEEE division made gn_apply ALU-bound
  // (25 instr / element, ncu r1f); 1e-6 relative is far inside the 1e-3 parity budget
  if (act == ODISE_ACT_SILU) return __fdividef(v, 1.f + __expf(-v));
  if (act == ODISE_ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  return v;
}

__device__ __forceinline__ void store_split4(__nv_bfloat16* hi, __nv_bfloat16* lo, float4 v) {
  const float e[4] = {v.x, v.y, v.z, v.w};
  store_planes<4>(hi, lo, e);     // bf16 pair, or fp16 + e5m2 corrections when lo carries the F16Q8 tag (ptx.cuh)
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------- split / add
// generic rows x cols with 4-wide vectors (cols % 4 == 0 required by all callers; checked on the host)
__global__ void add_split_kernel(const float* __restrict__ a, long long lda, const float* __restrict__ b,
                                 long long ldb, long long b_rows, float* __restrict__ y, long long ldy,
                                 __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ldo,
                                 long long rows, int cols4) {
  const long long total = rows * cols4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols4;
    const int c = (int)(i - r * cols4) * 4;
    float4 v = *reinterpret_cast<const float4*>(a + r * lda + c);
    if (b) {
      const long long rb = b_rows > 0 ? r % b_rows : r;
      const float4 w = *reinterpret_cast<const float4*>(b + rb * ldb + c);
      v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
    }
    if (y) *reinterpret_cast<float4*>(y + r * ldy + c) = v;
    if (hi) store_split4(hi + r * ldo + c, lo ? lo + r * ldo + c : nullptr, v);
  }
}

__global__ void copy2d_kernel(const float* __restrict__ src, long long lds, float* __restrict__ dst, long long ldd,
                              long long rows, int cols4, float scale, int accumulate) {
  const long long total = rows * cols4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols4;
    const int c = (int)(i - r * cols4) * 4;
    float4 v = *reinterpret_cast<const float4*>(src + r * lds + c);
    v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
    float4* d = reinterpret_cast<float4*>(dst + r * ldd + c);
    if (accumulate) { const float4 o = *d; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
    *d = v;
  }
}

// ---------------------------------------------------------------------------------------------- GroupNorm
// one block per (image, group): two-pass mean / variance in fp32 with double block reduction (matches
// torch.nn.GroupNorm's fp32 statistics to ~1e-7 relative).
__global__ void __launch_bounds__(256)
gn_stats_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ mean, float* __restrict__ rstd,
                int HW, int C, int G, float eps, long long x_bs) {
  const int b = blockIdx.x / G, g = blockIdx.x % G;
  const int cpg = C / G;
  const float* xb = x + (long long)b * x_bs + g * cpg;
  const long long n = (long long)HW * cpg;
  __shared__ double red[8];
  __shared__ double s_mean;
  double acc = 0.0;
  {
    float part = 0.f;
    int cnt = 0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
      const long long pix = i / cpg;
      const int c = (int)(i - pix * cpg);
      part += xb[pix * ldx + c];
      if (++cnt == 64) { acc += part; part = 0.f; cnt = 0; }
    }
    acc += part;
  }
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
    s_mean = t / (double)n;
  }
  __syncthreads();
  const float mu = (float)s_mean;
  acc = 0.0;
  {
    float part = 0.f;
    int cnt = 0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
      const long long pix = i / cpg;
      const int c = (int)(i - pix * cpg);
      const float d = xb[pix * ldx + c] - mu;
      part = fmaf(d, d, part);
      if (++cnt == 64) { acc += part; part = 0.f; cnt = 0; }
    }
    acc += part;
  }
  acc = warp_sum_d(acc);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
    const double var = t / (double)n;
    mean[blockIdx.x] = mu;
    rstd[blockIdx.x] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

// grid (pixel chunks, B); thread = fixed channel quad (+ pixel lane): the per-channel constants
// (mean, rstd, gamma, beta of the quad) are loaded once, the inner loop is load / 2 FMA-class ops / act / store.
// Up to 1024 threads (C = 4096): the bound keeps the register count launchable.
__global__ void __launch_bounds__(1024) gn_apply_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ mean,
                                const float* __restrict__ rstd, const float* __restrict__ gamma,
                                const float* __restrict__ beta, int act, float* __restrict__ y, long long ldy,
                                __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long ldo,
                                int HW, int C, int G, long long x_bs, long long y_bs, long long o_bs,
                                const float* __restrict__ res, long long ldres, int accumulate, int pix_per_block) {
  const int b = blockIdx.y;
  const int C4 = C >> 2, cpg = C / G;
  const int PL = blockDim.x / C4;
  const int q = threadIdx.x % C4, pl = threadIdx.x / C4;
  if (pl >= PL) return;
  const int c = q * 4;
  float mu[4], rs[4], ga[4], be[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int g = (c + t) / cpg;
    mu[t] = __ldg(mean + b * G + g);
    rs[t] = __ldg(rstd + b * G + g);
    ga[t] = __ldg(gamma + c + t);
    be[t] = __ldg(beta + c + t);
  }
  const float* xb = x + (long long)b * x_bs + c;
  const int p0 = blockIdx.x * pix_per_block, p1 = min(HW, p0 + pix_per_block);
  auto finish = [&](float4 v, float4 r4, float4 prev, int pix) {
    const float in[4] = {v.x, v.y, v.z, v.w};
    float o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) o[t] = fmaf((in[t] - mu[t]) * rs[t], ga[t], be[t]);   // torch order
    if (res) { o[0] += r4.x; o[1] += r4.y; o[2] += r4.z; o[3] += r4.w; }   // BottleneckBlock: relu(gn(conv3) + shortcut)
    if (act != ODISE_ACT_NONE) {
#pragma unroll
      for (int t = 0; t < 4; ++t) o[t] = act_apply(o[t], act);
    }
    float4 ov = make_float4(o[0], o[1], o[2], o[3]);
    if (y) {
      if (accumulate) { ov.x += prev.x; ov.y += prev.y; ov.z += prev.z; ov.w += prev.w; }
      *reinterpret_cast<float4*>(y + (long long)b * y_bs + (long long)pix * ldy + c) = ov;
    }
    if (hi) {
      const long long o_ = (long long)b * o_bs + (long long)pix * ldo + c;
      store_split4(hi + o_, lo ? lo + o_ : nullptr, ov);
    }
  };
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool acc = y && accumulate;
  int pix = p0 + pl;
  for (; pix + 3 * PL < p1; pix += 4 * PL) {   // all loads of 4 pixels in flight before the first use
    float4 v[4], r4[4], pv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int px = pix + u * PL;
      v[u] = *reinterpret_cast<const float4*>(xb + (long long)px * ldx);
      r4[u] = res ? *reinterpret_cast<const float4*>(res + ((long long)b * HW + px) * ldres + c) : z4;
      pv[u] = acc ? *reinterpret_cast<const float4*>(y + (long long)b * y_bs + (long long)px * ldy + c) : z4;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) finish(v[u], r4[u], pv[u], pix + u * PL);
  }
  for (; pix < p1; pix += PL) {
    const float4 v = *reinterpret_cast<const float4*>(xb + (long long)pix * ldx);
    const float4 r4 = res ? *reinterpret_cast<const float4*>(res + ((long long)b * HW + pix) * ldres + c) : z4;
    const float4 pv = acc ? *reinterpret_cast<const float4*>(y + (long long)b * y_bs + (long long)pix * ldy + c) : z4;
    finish(v, r4, pv, pix);
  }
}

// Lean variant for the common case (no residual / accumulate, C % 8 == 0): thread = fixed channel OCTET, 32-byte loads,
// 16-byte plane stores, two pixels in flight, <= 64 registers so that 4 x 256 threads stay resident per SM; the grid is
// exactly one resident wave (grid-stride over pixel chunks).
__device__ __forceinline__ void store_split8(__nv_bfloat16* hi, __nv_bfloat16* lo, const float* v) {
  store_planes<8>(hi, lo, v);
}

__global__ void __launch_bounds__(256, 4)
gn_apply8_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ mean,
                 const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                 int act, float* __restrict__ y, long long ldy, __nv_bfloat16* __restrict__ hi,
                 __nv_bfloat16* __restrict__ lo, long long ldo, int HW, int C, int G, long long x_bs, long long y_bs,
                 long long o_bs, int pix_per_block) {
  const int b = blockIdx.y;
  const int C8 = C >> 3, cpg = C / G;
  const int PL = blockDim.x / C8;
  const int q = threadIdx.x % C8, pl = threadIdx.x / C8;
  if (pl >= PL) return;
  const int c = q * 8;
  // an octet touches at most two groups (launcher guarantees cpg % 4 == 0 or cpg >= 8): the first nb channels use g0
  const int g0 = c / cpg, g1 = min(g0 + 1, G - 1);
  const int nb = min(8, (g0 + 1) * cpg - c);
  const float mu0 = __ldg(mean + b * G + g0), rs0 = __ldg(rstd + b * G + g0);
  const float mu1 = __ldg(mean + b * G + g1), rs1 = __ldg(rstd + b * G + g1);
  float ga[8], be[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) { ga[t] = __ldg(gamma + c + t); be[t] = __ldg(beta + c + t); }
  const float* xb = x + (long long)b * x_bs + c;
  const int p0 = blockIdx.x * pix_per_block, p1 = min(HW, p0 + pix_per_block);
  auto finish = [&](const float4& v0, const float4& v1, int pix) {
    float o[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
    for (int t = 0; t < 8; ++t)
      o[t] = fmaf((o[t] - (t < nb ? mu0 : mu1)) * (t < nb ? rs0 : rs1), ga[t], be[t]);   // torch order
    if (act != ODISE_ACT_NONE) {
#pragma unroll
      for (int t = 0; t < 8; ++t) o[t] = act_apply(o[t], act);
    }
    if (y) {
      float4* yp = reinterpret_cast<float4*>(y + (long long)b * y_bs + (long long)pix * ldy + c);
      yp[0] = make_float4(o[0], o[1], o[2], o[3]);
      yp[1] = make_float4(o[4], o[5], o[6], o[7]);
    }
    if (hi) {
      const long long o_ = (long long)b * o_bs + (long long)pix * ldo + c;
      store_split8(hi + o_, lo ? lo + o_ : nullptr, o);
    }
  };
  int pix = p0 + pl;
  for (; pix + PL < p1; pix += 2 * PL) {
    const float4* s0 = reinterpret_cast<const float4*>(xb + (long long)pix * ldx);
    const float4* s1 = reinterpret_cast<const float4*>(xb + (long long)(pix + PL) * ldx);
    const float4 v00 = s0[0], v01 = s0[1], v10 = s1[0], v11 = s1[1];
    finish(v00, v01, pix);
    finish(v10, v11, pix + PL);
  }
  if (pix < p1) {
    const float4* s0 = reinterpret_cast<const float4*>(xb + (long long)pix * ldx);
    const float4 v00 = s0[0], v01 = s0[1];
    finish(v00, v01, pix);
  }
}

static int launch_gn_apply(const float* x, long long ldx, const float* mean, const float* rstd, const float* gamma,
                           const float* beta, int act, float* y, long long ldy, __nv_bfloat16* hi,
                           __nv_bfloat16* lo, long long ldo, int B, int HW, int C, int G, long long x_bs,
                           long long y_bs, long long o_bs, const float* res, long long ldres, int accumulate,
                           cudaStream_t stream) {
  const int cpg_ = C / G;
  static const bool force_quad = getenv("ODISE_GN_QUAD") != nullptr;   // A/B switch for tools/gn_probe.py
  if (!force_quad && !res && !accumulate && C % 8 == 0 && C / 8 <= 256 && (cpg_ % 4 == 0 || cpg_ >= 8) && ldx % 4 == 0 && x_bs % 4 == 0 && (!y || (ldy % 4 == 0 && y_bs % 4 == 0)) &&
      (!hi || (ldo % 8 == 0 && o_bs % 8 == 0))) {
    const int C8 = C / 8;
    const int PL = 256 / C8;
    const int threads = C8 * PL;
    int chunks = (4 * num_sms() + B - 1) / B;          // one resident wave: 4 blocks per SM
    if (chunks > (HW + 2 * PL - 1) / (2 * PL)) chunks = (HW + 2 * PL - 1) / (2 * PL);
    if (chunks < 1) chunks = 1;
    const int ppb = (HW + chunks - 1) / chunks;
    chunks = (HW + ppb - 1) / ppb;
    gn_apply8_kernel<<<dim3(chunks, B), threads, 0, stream>>>(x, ldx, mean, rstd, gamma, beta, act, y, ldy, hi, lo, ldo, HW,
                                                             C, G, x_bs, y_bs, o_bs, ppb);
    return (int)cudaGetLastError();
  }
  const int C4 = C / 4;
  if (C4 > 1024) return ODISE_ERR_UNSUPPORTED;
  int PL = 256 / C4;
  if (PL < 1) PL = 1;
  const int threads = C4 * PL;
  int chunks = (6 * num_sms() + B - 1) / B;            // ~6 blocks per SM
  if (chunks > (HW + PL - 1) / PL) chunks = (HW + PL - 1) / PL;
  if (chunks < 1) chunks = 1;
  const int ppb = (HW + chunks - 1) / chunks;
  chunks = (HW + ppb - 1) / ppb;
  dim3 grid(chunks, B);
  gn_apply_kernel<<<grid, threads, 0, stream>>>(x, ldx, mean, rstd, gamma, beta, act, y, ldy, hi, lo, ldo, HW, C, G,
                                                x_bs, y_bs, o_bs, res, ldres, accumulate, ppb);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------- GroupNorm stats v2
// One coalesced pass: block = (image, pixel chunk); thread = (pixel lane, channel quad).  Shifted sums
// (pivot = first element of the group) keep E[x^2] - E[x]^2 free of cancellation; per-block partials go to a
// workspace and are combined in fixed order (deterministic), in double.
__global__ void gn_partial_kernel(const float* __restrict__ x, long long ldx, long long x_bs, float* __restrict__ ws,
                                  int HW, int C, int G, int nchunk, int pix_per_chunk) {
  extern __shared__ float sm[];   // [PL][C] sums, [PL][C] sumsq
  const int b = blockIdx.x / nchunk, chunk = blockIdx.x % nchunk;
  const int C4 = C >> 2, cpg = C / G;
  const int PL = blockDim.x / C4;
  const int q = threadIdx.x % C4, pl = threadIdx.x / C4;
  const float* xb = x + (long long)b * x_bs;
  float s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
  if (pl < PL) {
    float pv[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) pv[t] = __ldg(xb + ((q * 4 + t) / cpg) * cpg);
    const int p0 = chunk * pix_per_chunk, p1 = min(HW, p0 + pix_per_chunk);
    int p = p0 + pl;
    for (; p + 3 * PL < p1; p += 4 * PL) {   // 4 independent 16-byte loads in flight per thread
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(xb + (long long)(p + u * PL) * ldx + q * 4);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float d0 = v[u].x - pv[0], d1 = v[u].y - pv[1], d2 = v[u].z - pv[2], d3 = v[u].w - pv[3];
        s[0] += d0; s[1] += d1; s[2] += d2; s[3] += d3;
        ss[0] = fmaf(d0, d0, ss[0]); ss[1] = fmaf(d1, d1, ss[1]); ss[2] = fmaf(d2, d2, ss[2]); ss[3] = fmaf(d3, d3, ss[3]);
      }
    }
    for (; p < p1; p += PL) {
      const float4 v = *reinterpret_cast<const float4*>(xb + (long long)p * ldx + q * 4);
      const float d0 = v.x - pv[0], d1 = v.y - pv[1], d2 = v.z - pv[2], d3 = v.w - pv[3];
      s[0] += d0; s[1] += d1; s[2] += d2; s[3] += d3;
      ss[0] = fmaf(d0, d0, ss[0]); ss[1] = fmaf(d1, d1, ss[1]); ss[2] = fmaf(d2, d2, ss[2]); ss[3] = fmaf(d3, d3, ss[3]);
    }
    float* a = sm + (long long)pl * C + q * 4;
    float* bq = sm + (long long)PL * C + (long long)pl * C + q * 4;
#pragma unroll
    for (int t = 0; t < 4; ++t) { a[t] = s[t]; bq[t] = ss[t]; }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    double ds = 0, dss = 0;
    for (int l = 0; l < PL; ++l)
      for (int c = g * cpg; c < (g + 1) * cpg; ++c) { ds += sm[l * C + c]; dss += sm[(PL + l) * C + c]; }
    float* o = ws + (((long long)b * nchunk + chunk) * G + g) * 2;
    o[0] = (float)ds; o[1] = (float)dss;
  }
}

// one warp per (image, group): lanes stride over the chunk partials, fixed-order shuffle reduction (deterministic)
__global__ void gn_finalize_kernel(const float* __restrict__ x, long long x_bs, const float* __restrict__ ws,
                                   float* __restrict__ mean, float* __restrict__ rstd, int B, int HW, int C, int G,
                                   int nchunk, float eps) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= B * G) return;
  const int lane = threadIdx.x & 31;
  const int b = i / G, g = i % G, cpg = C / G;
  double s = 0, ss = 0;
  for (int k = lane; k < nchunk; k += 32) {
    const float* o = ws + (((long long)b * nchunk + k) * G + g) * 2;
    s += o[0]; ss += o[1];
  }
  s = warp_sum_d(s);
  ss = warp_sum_d(ss);
  if (lane == 0) {
    const double n = (double)HW * cpg;
    const double pivot = x[(long long)b * x_bs + g * cpg];
    const double m = s / n;
    double var = ss / n - m * m;
    if (var < 0) var = 0;
    mean[i] = (float)(pivot + m);
    rstd[i] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

// merge of the (shift, S1, S2) records a GEMM epilogue wrote per (32-row segment, channel): one block per (image, group),
// ONE pass over the records: every record is a (n = 32, mean, M2) triple; a thread folds its strided share in fixed order with
// Chan et al.'s pairwise update, the 32 lanes merge by a fixed xor butterfly, the 8 warps in index order — all in double,
// bit-reproducible.  (Round 1/2a read the records twice: mean first, then M2 about it.)
struct ChanAcc { double n, mu, m2; };
__device__ __forceinline__ void chan_merge(ChanAcc& a, const ChanAcc& b) {
  if (b.n == 0.0) return;
  if (a.n == 0.0) { a = b; return; }
  const double n = a.n + b.n, d = b.mu - a.mu;
  a.mu += d * (b.n / n);
  a.m2 += b.m2 + d * d * (a.n * b.n / n);
  a.n = n;
}
__global__ void __launch_bounds__(256)
gn_finalize_seg_kernel(const float* __restrict__ part, long long seg_stride, long long plane, float* __restrict__ mean,
                       float* __restrict__ rstd, int HW, int C, int G, float eps) {
  __shared__ ChanAcc red[8];
  const int b = blockIdx.x / G, g = blockIdx.x % G, cpg = C / G;
  const int nseg = HW >> 5;
  const int total = nseg * cpg;
  const float* base = part + (long long)b * nseg * seg_stride + g * cpg;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  ChanAcc acc{0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < total; i += 256) {
    const int sg = i / cpg, c = i - sg * cpg;
    const float* r = base + (long long)sg * seg_stride + c;
    const double s1 = r[plane], s2 = r[2 * plane];
    ChanAcc rec{32.0, (double)r[0] + s1 * (1.0 / 32.0), s2 - s1 * s1 * (1.0 / 32.0)};
    chan_merge(acc, rec);
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    ChanAcc other;
    other.n = __shfl_xor_sync(0xffffffffu, acc.n, o);
    other.mu = __shfl_xor_sync(0xffffffffu, acc.mu, o);
    other.m2 = __shfl_xor_sync(0xffffffffu, acc.m2, o);
    // both partners must end with the same value: merge in (lower lane, higher lane) order on both sides
    ChanAcc lo_ = (lane & o) ? other : acc, hi_ = (lane & o) ? acc : other;
    chan_merge(lo_, hi_);
    acc = lo_;
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    ChanAcc t = red[0];
    for (int w = 1; w < 8; ++w) chan_merge(t, red[w]);
    double var = t.m2 / t.n;
    if (var < 0) var = 0;
    mean[blockIdx.x] = (float)t.mu;
    rstd[blockIdx.x] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

// ---------------------------------------------------------------------------------------------- LayerNorm
// one warp per row, row cached in registers (cols <= 4096)
template <int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ res, long long ldres,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ y,
                 long long ldy, const float* __restrict__ post_add, long long ldpa, __nv_bfloat16* __restrict__ hi,
                 __nv_bfloat16* __restrict__ lo, long long ldo, long long rows, int cols) {
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nv = cols / 4;
  float4 v[MAXV];
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int idx = lane + k * 32;
    if (idx < nv) {
      v[k] = *reinterpret_cast<const float4*>(x + row * ldx + idx * 4);
      if (res) {
        const float4 r = *reinterpret_cast<const float4*>(res + row * ldres + idx * 4);
        v[k].x += r.x; v[k].y += r.y; v[k].z += r.z; v[k].w += r.w;
      }
      sum += (v[k].x + v[k].y) + (v[k].z + v[k].w);
    }
  }
  const float mu = warp_sum(sum) / (float)cols;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int idx = lane + k * 32;
    if (idx < nv) {
      const float a = v[k].x - mu, b = v[k].y - mu, c = v[k].z - mu, d = v[k].w - mu;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rs = rsqrtf(warp_sum(sq) / (float)cols + eps);
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int idx = lane + k * 32;
    if (idx < nv) {
      const int c = idx * 4;
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
      const float4 bt = __ldg(reinterpret_cast<const float4*>(beta + c));
      float4 o;
      o.x = fmaf((v[k].x - mu) * rs, g.x, bt.x);
      o.y = fmaf((v[k].y - mu) * rs, g.y, bt.y);
      o.z = fmaf((v[k].z - mu) * rs, g.z, bt.z);
      o.w = fmaf((v[k].w - mu) * rs, g.w, bt.w);
      if (y) *reinterpret_cast<float4*>(y + row * ldy + c) = o;
      if (hi) {
        if (post_add) {
          const float4 pa = *reinterpret_cast<const float4*>(post_add + row * ldpa + c);
          o.x += pa.x; o.y += pa.y; o.z += pa.z; o.w += pa.w;
        }
        store_split4(hi + row * ldo + c, lo ? lo + row * ldo + c : nullptr, o);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- GEGLU
__global__ void geglu_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ hi,
                             __nv_bfloat16* __restrict__ lo, long long ldo, long long rows, int cols) {
  const int c4n = cols / 4;
  const long long total = rows * c4n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c4n;
    const int c = (int)(i - r * c4n) * 4;
    const float4 a = *reinterpret_cast<const float4*>(x + r * ldx + c);
    const float4 g = *reinterpret_cast<const float4*>(x + r * ldx + cols + c);
    float4 o;
    o.x = a.x * act_apply(g.x, ODISE_ACT_GELU);
    o.y = a.y * act_apply(g.y, ODISE_ACT_GELU);
    o.z = a.z * act_apply(g.z, ODISE_ACT_GELU);
    o.w = a.w * act_apply(g.w, ODISE_ACT_GELU);
    store_split4(hi + r * ldo + c, lo ? lo + r * ldo + c : nullptr, o);
  }
}

// ---------------------------------------------------------------------------------------------- resampling
__global__ void upsample2x_split_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ hi,
                                        __nv_bfloat16* __restrict__ lo, long long ldo, int B, int H, int W, int C) {
  const int c4n = C / 4;
  const long long total = (long long)B * 4 * H * W * c4n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4n) * 4;
    long long p = i / c4n;
    const int ox = (int)(p % (2 * W)); p /= 2 * W;
    const int oy = (int)(p % (2 * H));
    const int b = (int)(p / (2 * H));
    const long long src = ((long long)b * H + (oy >> 1)) * W + (ox >> 1);
    const long long dst = ((long long)b * 2 * H + oy) * 2 * W + ox;
    const float4 v = *reinterpret_cast<const float4*>(x + src * ldx + c);
    store_split4(hi + dst * ldo + c, lo ? lo + dst * ldo + c : nullptr, v);
  }
}

__global__ void im2col3x3_split_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ hi,
                                       __nv_bfloat16* __restrict__ lo, int Kpad, int B, int H, int W, int C,
                                       int stride, int pad_lo, int Ho, int Wo) {
  const long long total = (long long)B * Ho * Wo * Kpad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kpad);
    long long p = i / Kpad;
    const int ox = (int)(p % Wo); p /= Wo;
    const int oy = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float v = 0.f;
    if (k < 9 * C) {
      const int tap = k / C, c = k - tap * C;
      const int iy = oy * stride + tap / 3 - pad_lo, ix = ox * stride + tap % 3 - pad_lo;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[(((long long)b * H + iy) * W + ix) * ldx + c];
    }
    store_planes<1>(hi + i, lo ? lo + i : nullptr, &v);
  }
}

// F.interpolate(mode="bilinear", align_corners=False) / mode="nearest" on NHWC
__global__ void resize_nhwc_kernel(const float* __restrict__ src, long long lds, float* __restrict__ dst,
                                   long long ldd, int B, int Hs, int Ws, int Hd, int Wd, int C, int bilinear,
                                   int accumulate, long long src_bs, long long dst_bs) {
  const int c4n = C / 4;
  const long long total = (long long)B * Hd * Wd * c4n;
  const float sy = (float)Hs / (float)Hd, sx = (float)Ws / (float)Wd;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c4n) * 4;
    long long p = i / c4n;
    const int ox = (int)(p % Wd); p /= Wd;
    const int oy = (int)(p % Hd);
    const int b = (int)(p / Hd);
    const float* sb = src + (long long)b * src_bs + c;
    float4 v;
    if (bilinear) {
      // ATen area_pixel_compute_source_index(align_corners=False): max(0, (dst + 0.5) * scale - 0.5)
      float fy = fmaxf((oy + 0.5f) * sy - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sx - 0.5f, 0.f);
      const int y0 = (int)fy, x0 = (int)fx;
      const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
      const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
      const float4 a = *reinterpret_cast<const float4*>(sb + ((long long)y0 * Ws + x0) * lds);
      const float4 bq = *reinterpret_cast<const float4*>(sb + ((long long)y0 * Ws + x1) * lds);
      const float4 cq = *reinterpret_cast<const float4*>(sb + ((long long)y1 * Ws + x0) * lds);
      const float4 d = *reinterpret_cast<const float4*>(sb + ((long long)y1 * Ws + x1) * lds);
      v.x = hy * (hx * a.x + lx * bq.x) + ly * (hx * cq.x + lx * d.x);
      v.y = hy * (hx * a.y + lx * bq.y) + ly * (hx * cq.y + lx * d.y);
      v.z = hy * (hx * a.z + lx * bq.z) + ly * (hx * cq.z + lx * d.z);
      v.w = hy * (hx * a.w + lx * bq.w) + ly * (hx * cq.w + lx * d.w);
    } else {
      const int y0 = min((int)floorf(oy * sy), Hs - 1), x0 = min((int)floorf(ox * sx), Ws - 1);
      v = *reinterpret_cast<const float4*>(sb + ((long long)y0 * Ws + x0) * lds);
    }
    float4* dp = reinterpret_cast<float4*>(dst + (long long)b * dst_bs + ((long long)oy * Wd + ox) * ldd + c);
    if (accumulate) { const float4 o = *dp; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
    *dp = v;
  }
}

// tiled transposes: NCHW [B, C, HW] <-> NHWC [B, HW, C(ld)]
__global__ void transpose_kernel(const float* __restrict__ src, long long src_bs, long long lds,
                                 float* __restrict__ dst, long long dst_bs, long long ldd, int R, int Cc) {
  // src [R rows, Cc cols] (ld lds) -> dst [Cc rows, R cols] (ld ldd), per batch blockIdx.z
  __shared__ float tile[32][33];
  const float* s = src + blockIdx.z * src_bs;
  float* d = dst + blockIdx.z * dst_bs;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < R && c < Cc) tile[j][threadIdx.x] = s[(long long)r * lds + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < R && c < Cc) d[(long long)c * ldd + r] = tile[threadIdx.x][j];
  }
}

// ---------------------------------------------------------------------------------------------- CLIP-match tail
__global__ void l2norm_split_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ hi,
                                    __nv_bfloat16* __restrict__ lo, long long ldo, long long rows, int cols) {
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float sq = 0.f;
  for (int c = lane; c < cols; c += 32) { const float v = x[row * ldx + c]; sq = fmaf(v, v, sq); }
  // F.normalize: x / max(||x||_2, 1e-12)
  const float nrm = fmaxf(sqrtf(warp_sum(sq)), 1e-12f);
  for (int c = lane; c < cols; c += 32) {
    const float v = x[row * ldx + c] / nrm;
    store_planes<1>(hi + row * ldo + c, lo ? lo + row * ldo + c : nullptr, &v);
  }
}

__global__ void class_max_kernel(const float* __restrict__ sims, long long ld, const int32_t* __restrict__ gs,
                                 const float* __restrict__ null_sim, float* __restrict__ out, long long rows,
                                 int K) {
  const long long total = rows * (K + 1);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / (K + 1);
    const int k = (int)(i - r * (K + 1));
    float v;
    if (k == K) {
      v = null_sim[r];
    } else {
      v = -INFINITY;
      for (int j = gs[k]; j < gs[k + 1]; ++j) v = fmaxf(v, sims[r * ld + j]);
    }
    out[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------- mask pooling
// binary mask (sigmoid(x) > 0.5) as bf16 0/1 + per-row count.  grid = (chunks, rows); counts must be zeroed first.
// sigmoid(x) > 0.5 <=> x > 0 except in the fp32 rounding band |x| < ~1.2e-7 where torch's sigmoid rounds to exactly
// 0.5: only there the sigmoid itself is evaluated (MaskPooling, odise.py:945-951).
__global__ void mask_binarize_kernel(const float* __restrict__ logits, __nv_bfloat16* __restrict__ bin,
                                     long long ld_bin, float* __restrict__ counts, int HW) {
  const long long row = blockIdx.y;
  const float* src = logits + row * HW;
  __nv_bfloat16* dst = bin + row * ld_bin;
  float cnt = 0.f;
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4; c < HW; c += gridDim.x * blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(src + c);
    const float in[4] = {v.x, v.y, v.z, v.w};
    __align__(8) __nv_bfloat16 o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      bool on = in[t] > 0.f;
      if (fabsf(in[t]) < 1e-6f) on = (1.f / (1.f + expf(-in[t]))) > 0.5f;
      o[t] = __float2bfloat16_rn(on ? 1.f : 0.f);
      cnt += on ? 1.f : 0.f;
    }
    *reinterpret_cast<uint2*>(dst + c) = *reinterpret_cast<const uint2*>(o);
  }
  cnt = warp_sum(cnt);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
    atomicAdd(counts + row, t);   // integer-valued partial counts < 2^24: exact and order independent
  }
}

__global__ void pool_normalize_kernel(const float* __restrict__ sums, const float* __restrict__ counts,
                                      float* __restrict__ pooled, long long rows, int C) {
  const long long total = rows * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    // einsum(x, mask / (count + 1e-8)): the 0/1 mask makes this sum / (count + 1e-8) up to fp32 rounding order
    pooled[i] = sums[i] / (counts[r] + 1e-8f);
  }
}

// y = act(x) -> (hi, lo)   (SiLU(emb) in front of the ResBlock emb_layers linear)
__global__ void act_split_kernel(const float* __restrict__ x, long long ldx, int act, __nv_bfloat16* __restrict__ hi,
                                 __nv_bfloat16* __restrict__ lo, long long ldo, long long rows, int cols4) {
  const long long total = rows * cols4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols4;
    const int c = (int)(i - r * cols4) * 4;
    float4 v = *reinterpret_cast<const float4*>(x + r * ldx + c);
    v.x = act_apply(v.x, act); v.y = act_apply(v.y, act); v.z = act_apply(v.z, act); v.w = act_apply(v.w, act);
    store_split4(hi + r * ldo + c, lo ? lo + r * ldo + c : nullptr, v);
  }
}

// out[b, t, c] = a0[t, c] + ta[t, c] * p[b, c]   (implicit captioner: cond = uncond + tanh(alpha) * (proj + pos))
__global__ void bcast_fma_kernel(const float* __restrict__ a0, const float* __restrict__ ta,
                                 const float* __restrict__ p, float* __restrict__ out, int B, int T, int C) {
  const long long total = (long long)B * T * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long bt = i / C;
    const int t = (int)(bt % T), b = (int)(bt / T);
    out[i] = fmaf(ta[(long long)t * C + c], p[(long long)b * C + c], a0[(long long)t * C + c]);
  }
}

// y[r, :] *= s[r]
__global__ void rowscale_kernel(float* __restrict__ y, long long ldy, const float* __restrict__ s, long long rows,
                                int cols4) {
  const long long total = rows * cols4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols4;
    const int c = (int)(i - r * cols4) * 4;
    float4* q = reinterpret_cast<float4*>(y + r * ldy + c);
    float4 v = *q;
    const float f = s[r];
    v.x *= f; v.y *= f; v.z *= f; v.w *= f;
    *q = v;
  }
}

// uint8 NCHW image -> normalised NHWC fp32 crop: ((x / 255) - 0.5) / 0.5, i.e. CategoryODISE's (x - 0) / 255
// (odise.py:237) followed by LdmExtractor's (img - 0.5) / 0.5 (ldm.py:556); crop b reads image img_of[b] at (y0[b], x0[b])
__global__ void image_crops_kernel(const uint8_t* __restrict__ img, float* __restrict__ out,
                                   const int32_t* __restrict__ boxes, int n_crops, int H, int W, int ch, int cw) {
  const long long total = (long long)n_crops * ch * cw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % cw);
    long long t = i / cw;
    const int y = (int)(t % ch);
    const int b = (int)(t / ch);
    const int im = boxes[3 * b], y0 = boxes[3 * b + 1], x0 = boxes[3 * b + 2];
    const uint8_t* src = img + ((long long)im * 3 * H + (y0 + y)) * W + x0 + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = (float)src[(long long)c * H * W] / 255.f;
      out[i * 3 + c] = (v - 0.5f) / 0.5f;
    }
  }
}

// float NCHW image in [0, 1] -> normalised NHWC fp32 crops ((x - 0.5) / 0.5): the Backbone plugin entry
// (FeatureExtractorBackbone.forward receives the already /255-normalised tensor, feature_extractor.py:252)
__global__ void image_crops_f32_kernel(const float* __restrict__ img, float* __restrict__ out,
                                       const int32_t* __restrict__ boxes, int n_crops, int H, int W, int ch, int cw) {
  const long long total = (long long)n_crops * ch * cw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % cw);
    long long t = i / cw;
    const int y = (int)(t % ch);
    const int b = (int)(t / ch);
    const int im = boxes[3 * b], y0 = boxes[3 * b + 1], x0 = boxes[3 * b + 2];
    const float* src = img + ((long long)im * 3 * H + (y0 + y)) * W + x0 + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[i * 3 + c] = (src[(long long)c * H * W] - 0.5f) / 0.5f;
  }
}

// ---------------------------------------------------------------------------------------------- CLIP front
// clip_preprocess (odise/modeling/meta_arch/clip.py:94 = open_clip Resize(bicubic) + CenterCrop + Normalize) of a crop
// of the image batch: bicubic (A = -0.75, align_corners=False, no antialias: torchvision 0.14 on tensors), indices
// clamped to the CROP (the reference resizes the already-cropped tensor).  Output NHWC fp32 [n_crops, S, S, 3].
__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }

// PLANAR = true writes NCHW [n_crops, 3, S, S] (the crop re-enters the pipeline as an image batch: T.Resize of
// FeatureExtractorBackbone.single_forward, feature_extractor.py:73-76,144) instead of NHWC.
template <typename T, bool PLANAR = false>
__global__ void clip_preprocess_kernel(const T* __restrict__ img, float* __restrict__ out,
                                       const int32_t* __restrict__ boxes, int n_crops, int H, int W, int ch, int cw,
                                       int S, float in_scale, float m0, float m1, float m2, float s0, float s1,
                                       float s2) {
  const long long total = (long long)n_crops * S * S;
  const float A = -0.75f;
  // square crops only (ODISE crops are short x short): resize ch x cw -> S x S, the centre crop is then the identity
  const float sy = (float)ch / (float)S, sx = (float)cw / (float)S;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % S);
    long long t = i / S;
    const int oy = (int)(t % S);
    const int b = (int)(t / S);
    const int im = boxes[3 * b], y0 = boxes[3 * b + 1], x0 = boxes[3 * b + 2];
    const float fy = (oy + 0.5f) * sy - 0.5f, fx = (ox + 0.5f) * sx - 0.5f;
    const int iy = (int)floorf(fy), ix = (int)floorf(fx);
    const float ty = fy - iy, tx = fx - ix;
    const float wy[4] = {cubic2(ty + 1.f, A), cubic1(ty, A), cubic1(1.f - ty, A), cubic2(2.f - ty, A)};
    const float wx[4] = {cubic2(tx + 1.f, A), cubic1(tx, A), cubic1(1.f - tx, A), cubic2(2.f - tx, A)};
    const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const T* src = img + ((long long)im * 3 + c) * H * W;
      float acc = 0.f;
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int yy = y0 + min(max(iy - 1 + a, 0), ch - 1);
        float row = 0.f;
#pragma unroll
        for (int d = 0; d < 4; ++d) {
          const int xx = x0 + min(max(ix - 1 + d, 0), cw - 1);
          row += wx[d] * ((float)src[(long long)yy * W + xx] * in_scale);
        }
        acc += wy[a] * row;
      }
      if (PLANAR) out[((long long)b * 3 + c) * S * S + (long long)oy * S + ox] = acc;
      else out[i * 3 + c] = (acc - mean[c]) / stdv[c];
    }
  }
}

// out[i, :] = src[idx[i], :] (+ add[i % add_period, :]): token-embedding lookup + positional embedding, EOT-row gather
__global__ void gather_rows_kernel(const float* __restrict__ src, long long lds, const int32_t* __restrict__ idx,
                                   const float* __restrict__ add, long long ld_add, int add_period,
                                   float* __restrict__ out, long long ldo, long long rows, int cols) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i - r * cols);
    float v = src[(long long)idx[r] * lds + c];
    if (add) v += add[(r % add_period) * ld_add + c];
    out[r * ldo + c] = v;
  }
}

// non-overlapping P x P patches of an NHWC image [B, S, S, 3] -> (hi, lo) rows [B*G*G, Kpad], k = c*P*P + ky*P + kx
// (the layout of visual.conv1.weight.reshape(width, 3*P*P); clip.py:179)
__global__ void patchify_split_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi,
                                      __nv_bfloat16* __restrict__ lo, int B, int S, int P, int Kpad) {
  const int G = S / P;
  const long long total = (long long)B * G * G * Kpad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kpad);
    long long r = i / Kpad;
    const int gx = (int)(r % G); r /= G;
    const int gy = (int)(r % G);
    const int b = (int)(r / G);
    float v = 0.f;
    if (k < 3 * P * P) {
      const int c = k / (P * P), rem = k - c * P * P, ky = rem / P, kx = rem - ky * P;
      v = x[(((long long)b * S + gy * P + ky) * S + gx * P + kx) * 3 + c];
    }
    store_planes<1>(hi + i, lo ? lo + i : nullptr, &v);
  }
}

// ---------------------------------------------------------------------------------------------- softmax
// one warp per row
__global__ void softmax_split_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ hi,
                                     __nv_bfloat16* __restrict__ lo, long long ldo, long long rows, int cols,
                                     int cols_pad, float scale) {
  const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * ldx;
  float mx = -INFINITY;
  for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, xr[c] * scale);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < cols; c += 32) sum += expf(xr[c] * scale - mx);
  sum = warp_sum(sum);
  for (int c = lane; c < cols_pad; c += 32) {
    const float v = c < cols ? expf(xr[c] * scale - mx) / sum : 0.f;
    store_planes<1>(hi + row * ldo + c, lo ? lo + row * ldo + c : nullptr, &v);
  }
}

// Long rows (the KL-VAE mid-block attention: 4096 x 4096 scores per crop): the row is read from HBM ONCE into shared memory
// (one warp per row, 4 rows per block so that three blocks share an SM and their load / exp / store phases interleave — with
// one 8-row block per SM the phases ran in lock step at 2.3 TB/s, r2r), exponentials evaluated once (MUFU), planes written 4
// columns at a time — the three-pass kernel above read the 1 GB score matrix three times and stored 2 bytes at a time.
constexpr int kSmRows = 4;
__global__ void __launch_bounds__(32 * kSmRows)
softmax_split_smem_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ hi,
                          __nv_bfloat16* __restrict__ lo, long long ldo, long long rows, int cols, int cols_pad,
                          float scale) {
  extern __shared__ __align__(16) float srow[];                 // [kSmRows warps][cols_pad]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = blockIdx.x * (long long)kSmRows + warp;
  if (row >= rows) return;
  float* rb = srow + (size_t)warp * cols_pad;
  const float* xr = x + row * ldx;
  float mx = -INFINITY;
#pragma unroll 8                                                   // 8 x 16 B per lane in flight (one block per SM: 128 KB of rows)
  for (int c = lane * 4; c < cols; c += 128) {                  // cols % 4 == 0, ldx % 4 == 0 (checked by the launcher)
    float4 v = __ldcs(reinterpret_cast<const float4*>(xr + c));  // streamed: the scores are read exactly once
    v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
    *reinterpret_cast<float4*>(rb + c) = v;
    mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane * 4; c < cols; c += 128) {
    float4 v = *reinterpret_cast<const float4*>(rb + c);
    v.x = __expf(v.x - mx); v.y = __expf(v.y - mx); v.z = __expf(v.z - mx); v.w = __expf(v.w - mx);
    *reinterpret_cast<float4*>(rb + c) = v;
    sum += (v.x + v.y) + (v.z + v.w);
  }
  sum = warp_sum(sum);
  for (int c = lane * 4; c < cols_pad; c += 128) {
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    if (c < cols) {
      const float4 v = *reinterpret_cast<const float4*>(rb + c);
      o[0] = v.x / sum; o[1] = v.y / sum; o[2] = v.z / sum; o[3] = v.w / sum;
    }
    store_planes<4>(hi + row * ldo + c, lo ? lo + row * ldo + c : nullptr, o);
  }
}

}  // namespace ob

using namespace ob;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
// second operand plane as the kernels receive it: tagged when odise_set_operand_format(ODISE_PLANES_F16Q8) is in effect
#define BFL(p) ob::lo_arg(reinterpret_cast<__nv_bfloat16*>(p))
// F16Q8 planes: rows on 128-byte boundaries (the kernels read an element's position in its 64-wide k-block off its address)
#define Q8_CHECK(lo, ld)                                                                                     \
  if ((lo) && ob::operand_format() == ODISE_PLANES_F16Q8 && (((ld) % 64) || (reinterpret_cast<uintptr_t>(lo) & 127))) \
    return ODISE_ERR_ALIGN

namespace ob {
static int g_operand_format = ODISE_PLANES_BF16;
int operand_format() { return g_operand_format; }
}  // namespace ob
extern "C" int odise_set_operand_format(int fmt) {
  if (fmt != ODISE_PLANES_BF16 && fmt != ODISE_PLANES_F16Q8) return ODISE_ERR_ARG;
  ob::g_operand_format = fmt;
  return ODISE_OK;
}
extern "C" int odise_get_operand_format(void) { return ob::g_operand_format; }

extern "C" int odise_version(void) { return 100; }
extern "C" long long odise_launch_count(void) { return g_launches.load(); }
// Shared-memory carve-out policy of the current device: 1 = every kernel runs with the maximum shared-memory carve-out
// (what the TMA-staged GEMM / attention kernels need), so the SMs are not re-partitioned between an elementwise kernel
// and the GEMM that follows it; 0 = driver default (per-kernel choice).
extern "C" int odise_set_carveout_policy(int prefer_shared) {
  return (int)cudaDeviceSetCacheConfig(prefer_shared ? cudaFuncCachePreferShared : cudaFuncCachePreferNone);
}

__global__ void split_f16_kernel(const float* __restrict__ x, long long ldx, uint16_t* __restrict__ hi,
                                 uint16_t* __restrict__ lo, long long ldo, long long rows, int cols) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i - r * cols);
    uint16_t h, l;
    split_f16(x[r * ldx + c], h, l);
    hi[r * ldo + c] = h;
    if (lo) lo[r * ldo + c] = l;
  }
}

extern "C" int odise_split_f16_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, long long rows,
                                   int cols, void* stream) {
  if (!x || !hi || rows <= 0 || cols <= 0) return ODISE_ERR_ARG;
  split_f16_kernel<<<grid_for(rows * cols, 256), 256, 0, STREAM(stream)>>>(x, ldx, reinterpret_cast<uint16_t*>(hi),
                                                                        reinterpret_cast<uint16_t*>(lo), ldo, rows, cols);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_split_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, long long rows,
                               int cols, void* stream) {
  return odise_add_split_f32(x, ldx, nullptr, 0, 0, nullptr, 0, hi, lo, ldo, rows, cols, stream);
}

extern "C" int odise_add_split_f32(const float* a, long long lda, const float* b, long long ldb, long long b_rows,
                                   float* y, long long ldy, void* hi, void* lo, long long ldo, long long rows,
                                   int cols, void* stream) {
  if (!a || rows <= 0 || cols <= 0 || (!y && !hi)) return ODISE_ERR_ARG;
  if (cols % 4 || lda % 4 || (b && ldb % 4) || (y && ldy % 4) || (hi && ldo % 4)) return ODISE_ERR_ALIGN;
  Q8_CHECK(lo, ldo);
  add_split_kernel<<<grid_for(rows * (cols / 4), 256), 256, 0, STREAM(stream)>>>(a, lda, b, ldb, b_rows, y, ldy,
                                                                               BF(hi), BFL(lo), ldo, rows, cols / 4);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_copy2d_f32(const float* src, long long lds, float* dst, long long ldd, long long rows, int cols,
                                float scale, int accumulate, void* stream) {
  if (!src || !dst || rows <= 0 || cols <= 0) return ODISE_ERR_ARG;
  if (cols % 4 || lds % 4 || ldd % 4) return ODISE_ERR_ALIGN;
  copy2d_kernel<<<grid_for(rows * (cols / 4), 256), 256, 0, STREAM(stream)>>>(src, lds, dst, ldd, rows, cols / 4,
                                                                            scale, accumulate);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_groupnorm_stats_f32(const float* x, long long ldx, float* mean, float* rstd, int B, int HW,
                                         int C, int G, float eps, void* stream) {
  return odise_groupnorm_stats_bs_f32(x, ldx, 0, mean, rstd, B, HW, C, G, eps, stream);
}

extern "C" int odise_groupnorm_stats_bs_f32(const float* x, long long ldx, long long x_bs, float* mean, float* rstd,
                                            int B, int HW, int C, int G, float eps, void* stream) {
  if (!x || !mean || !rstd || B <= 0 || HW <= 0 || C <= 0 || G <= 0 || C % G) return ODISE_ERR_ARG;
  gn_stats_kernel<<<B * G, 256, 0, STREAM(stream)>>>(x, ldx, mean, rstd, HW, C, G, eps,
                                                     x_bs ? x_bs : (long long)HW * ldx);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_groupnorm_apply_f32(const float* x, long long ldx, const float* mean, const float* rstd,
                                         const float* gamma, const float* beta, int act, float* y, long long ldy,
                                         void* hi, void* lo, long long ldo, int B, int HW, int C, int G,
                                         void* stream) {
  return odise_groupnorm_apply_bs_f32(x, ldx, 0, mean, rstd, gamma, beta, act, y, ldy, 0, hi, lo, ldo, 0, B, HW, C, G,
                                      stream);
}

extern "C" int odise_groupnorm_apply_bs_f32(const float* x, long long ldx, long long x_bs, const float* mean,
                                            const float* rstd, const float* gamma, const float* beta, int act,
                                            float* y, long long ldy, long long y_bs, void* hi, void* lo,
                                            long long ldo, long long o_bs, int B, int HW, int C, int G, void* stream) {
  if (!x || !mean || !rstd || !gamma || !beta || (!y && !hi) || C % G) return ODISE_ERR_ARG;
  if (C % 4 || ldx % 4 || x_bs % 4 || (y && (ldy % 4 || y_bs % 4)) || (hi && (ldo % 4 || o_bs % 4)))
    return ODISE_ERR_ALIGN;
  Q8_CHECK(lo, ldo);
  int rc = launch_gn_apply(x, ldx, mean, rstd, gamma, beta, act, y, ldy, BF(hi), BFL(lo), ldo, B, HW, C, G,
                           x_bs ? x_bs : (long long)HW * ldx, y_bs ? y_bs : (long long)HW * ldy,
                           o_bs ? o_bs : (long long)HW * ldo, nullptr, 0, 0, STREAM(stream));
  if (rc) return rc;
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_layernorm_f32(const float* x, long long ldx, const float* res, long long ldres,
                                   const float* gamma, const float* beta, float eps, float* y, long long ldy,
                                   const float* post_add, long long ldpa, void* hi, void* lo, long long ldo,
                                   long long rows, int cols, void* stream) {
  if (!x || !gamma || !beta || (!y && !hi) || rows <= 0 || cols <= 0 || cols > 4096) return ODISE_ERR_ARG;
  if (cols % 4 || ldx % 4 || (res && ldres % 4) || (y && ldy % 4) || (hi && ldo % 4) || (post_add && ldpa % 4))
    return ODISE_ERR_ALIGN;
  const int wpb = 8;
  const int blocks = (int)((rows + wpb - 1) / wpb);
  const int nv = cols / 4;
  Q8_CHECK(lo, ldo);
#define LN_LAUNCH(MV)                                                                                              \
  layernorm_kernel<MV><<<blocks, wpb * 32, 0, STREAM(stream)>>>(x, ldx, res, ldres, gamma, beta, eps, y, ldy,       \
                                                               post_add, ldpa, BF(hi), BFL(lo), ldo, rows, cols)
  if (nv <= 64) LN_LAUNCH(2);
  else if (nv <= 128) LN_LAUNCH(4);
  else if (nv <= 320) LN_LAUNCH(10);
  else LN_LAUNCH(32);
#undef LN_LAUNCH
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_geglu_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, long long rows,
                               int cols, void* stream) {
  if (!x || !hi || rows <= 0 || cols <= 0) return ODISE_ERR_ARG;
  if (cols % 4 || ldx % 4 || ldo % 4) return ODISE_ERR_ALIGN;
  Q8_CHECK(lo, ldo);
  geglu_kernel<<<grid_for(rows * (cols / 4), 256), 256, 0, STREAM(stream)>>>(x, ldx, BF(hi), BFL(lo), ldo, rows, cols);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_upsample2x_split_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, int B,
                                          int H, int W, int C, void* stream) {
  if (!x || !hi || B <= 0 || H <= 0 || W <= 0 || C <= 0) return ODISE_ERR_ARG;
  if (C % 4 || ldx % 4 || ldo % 4) return ODISE_ERR_ALIGN;
  Q8_CHECK(lo, ldo);
  upsample2x_split_kernel<<<grid_for((long long)B * 4 * H * W * (C / 4), 256), 256, 0, STREAM(stream)>>>(
      x, ldx, BF(hi), BFL(lo), ldo, B, H, W, C);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_im2col3x3_split_f32(const float* x, long long ldx, void* hi, void* lo, int Kpad, int B, int H,
                                         int W, int C, int stride, int pad_lo, int pad_hi, void* stream) {
  if (!x || !hi || B <= 0 || H <= 0 || W <= 0 || C <= 0 || stride <= 0 || Kpad < 9 * C || Kpad % 8)
    return ODISE_ERR_ARG;
  const int Ho = (H + pad_lo + pad_hi - 3) / stride + 1, Wo = (W + pad_lo + pad_hi - 3) / stride + 1;
  Q8_CHECK(lo, Kpad);
  im2col3x3_split_kernel<<<grid_for((long long)B * Ho * Wo * Kpad, 256), 256, 0, STREAM(stream)>>>(
      x, ldx, BF(hi), BFL(lo), Kpad, B, H, W, C, stride, pad_lo, Ho, Wo);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_resize_nhwc_f32(const float* src, long long lds, float* dst, long long ldd, int B, int Hs,
                                     int Ws, int Hd, int Wd, int C, int bilinear, int accumulate, void* stream) {
  return odise_resize_nhwc_bs_f32(src, lds, 0, dst, ldd, 0, B, Hs, Ws, Hd, Wd, C, bilinear, accumulate, stream);
}

extern "C" int odise_resize_nhwc_bs_f32(const float* src, long long lds, long long src_bs, float* dst, long long ldd,
                                        long long dst_bs, int B, int Hs, int Ws, int Hd, int Wd, int C, int bilinear,
                                        int accumulate, void* stream) {
  if (!src || !dst || B <= 0 || Hs <= 0 || Ws <= 0 || Hd <= 0 || Wd <= 0 || C <= 0) return ODISE_ERR_ARG;
  if (C % 4 || lds % 4 || ldd % 4 || src_bs % 4 || dst_bs % 4) return ODISE_ERR_ALIGN;
  resize_nhwc_kernel<<<grid_for((long long)B * Hd * Wd * (C / 4), 256), 256, 0, STREAM(stream)>>>(
      src, lds, dst, ldd, B, Hs, Ws, Hd, Wd, C, bilinear, accumulate,
      src_bs ? src_bs : (long long)Hs * Ws * lds, dst_bs ? dst_bs : (long long)Hd * Wd * ldd);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_nchw_to_nhwc_f32(const float* src, float* dst, long long ldd, int B, int C, int HW,
                                      void* stream) {
  if (!src || !dst || B <= 0 || C <= 0 || HW <= 0) return ODISE_ERR_ARG;
  dim3 grid((HW + 31) / 32, (C + 31) / 32, B), block(32, 8);
  transpose_kernel<<<grid, block, 0, STREAM(stream)>>>(src, (long long)C * HW, HW, dst, (long long)HW * ldd, ldd, C,
                                                       HW);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_nhwc_to_nchw_f32(const float* src, long long lds, float* dst, int B, int C, int HW,
                                      void* stream) {
  if (!src || !dst || B <= 0 || C <= 0 || HW <= 0) return ODISE_ERR_ARG;
  dim3 grid((C + 31) / 32, (HW + 31) / 32, B), block(32, 8);
  transpose_kernel<<<grid, block, 0, STREAM(stream)>>>(src, (long long)HW * lds, lds, dst, (long long)C * HW, HW, HW,
                                                       C);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_l2_normalize_split_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo,
                                            long long rows, int cols, void* stream) {
  if (!x || !hi || rows <= 0 || cols <= 0) return ODISE_ERR_ARG;
  Q8_CHECK(lo, ldo);
  l2norm_split_kernel<<<(int)((rows + 7) / 8), 256, 0, STREAM(stream)>>>(x, ldx, BF(hi), BFL(lo), ldo, rows, cols);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_class_max_f32(const float* sims, long long ld_sims, const int32_t* group_start,
                                   const float* null_sim, float* out, long long rows, int n_classes, void* stream) {
  if (!sims || !group_start || !null_sim || !out || rows <= 0 || n_classes <= 0) return ODISE_ERR_ARG;
  class_max_kernel<<<grid_for(rows * (n_classes + 1), 256), 256, 0, STREAM(stream)>>>(sims, ld_sims, group_start,
                                                                                    null_sim, out, rows, n_classes);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_mask_binarize_f32(const float* logits, void* bin_bf16, long long ld_bin, float* counts, int B,
                                       int Q, int HW, void* stream) {
  if (!logits || !bin_bf16 || !counts || B <= 0 || Q <= 0 || HW <= 0) return ODISE_ERR_ARG;
  if (HW % 4 || ld_bin % 4) return ODISE_ERR_ALIGN;
  const long long rows = (long long)B * Q;
  cudaError_t e = cudaMemsetAsync(counts, 0, sizeof(float) * rows, STREAM(stream));
  if (e != cudaSuccess) return (int)e;
  int chunks = (HW / 4 + 255) / 256;
  if (chunks > 16) chunks = 16;
  dim3 grid(chunks, (unsigned)rows);
  mask_binarize_kernel<<<grid, 256, 0, STREAM(stream)>>>(logits, BF(bin_bf16), ld_bin, counts, HW);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_pool_normalize_f32(const float* sums, const float* counts, float* pooled, int B, int Q, int C,
                                        void* stream) {
  if (!sums || !counts || !pooled || B <= 0 || Q <= 0 || C <= 0) return ODISE_ERR_ARG;
  const long long rows = (long long)B * Q;
  pool_normalize_kernel<<<grid_for(rows * C, 256), 256, 0, STREAM(stream)>>>(sums, counts, pooled, rows, C);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_softmax_split_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo,
                                       long long rows, int cols, int cols_pad, float scale, void* stream) {
  if (!x || !hi || rows <= 0 || cols <= 0 || cols_pad < cols) return ODISE_ERR_ARG;
  Q8_CHECK(lo, ldo);
  // rows that fit shared memory eight at a time and allow 16-byte accesses: one HBM read of the scores
  const size_t smem = (size_t)kSmRows * cols_pad * sizeof(float);
  if (cols >= 512 && cols % 4 == 0 && cols_pad % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0 && smem <= 200 * 1024 &&
      (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(hi) & 7) == 0 &&
      (!lo || (reinterpret_cast<uintptr_t>(lo) & 7) == 0)) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaError_t e = cudaFuncSetAttribute(softmax_split_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return (int)e;
      attr = smem;
    }
    softmax_split_smem_kernel<<<(int)((rows + kSmRows - 1) / kSmRows), 32 * kSmRows, smem, STREAM(stream)>>>(
        x, ldx, BF(hi), BFL(lo), ldo, rows, cols, cols_pad, scale);
  } else {
    softmax_split_kernel<<<(int)((rows + 7) / 8), 256, 0, STREAM(stream)>>>(x, ldx, BF(hi), BFL(lo), ldo, rows, cols,
                                                                           cols_pad, scale);
  }
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_act_split_f32(const float* x, long long ldx, int act, void* hi, void* lo, long long ldo,
                                   long long rows, int cols, void* stream) {
  if (!x || !hi || rows <= 0 || cols <= 0) return ODISE_ERR_ARG;
  if (cols % 4 || ldx % 4 || ldo % 4) return ODISE_ERR_ALIGN;
  Q8_CHECK(lo, ldo);
  act_split_kernel<<<grid_for(rows * (cols / 4), 256), 256, 0, STREAM(stream)>>>(x, ldx, act, BF(hi), BFL(lo), ldo,
                                                                               rows, cols / 4);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_groupnorm_apply_res_f32(const float* x, long long ldx, const float* mean, const float* rstd,
                                             const float* gamma, const float* beta, const float* res,
                                             long long ldres, int act, float* y, long long ldy, int accumulate,
                                             void* hi, void* lo, long long ldo, int B, int HW, int C, int G,
                                             void* stream) {
  if (!x || !mean || !rstd || !gamma || !beta || (!y && !hi) || C % G) return ODISE_ERR_ARG;
  if (C % 4 || ldx % 4 || (y && ldy % 4) || (hi && ldo % 4) || (res && ldres % 4)) return ODISE_ERR_ALIGN;
  Q8_CHECK(lo, ldo);
  int rc = launch_gn_apply(x, ldx, mean, rstd, gamma, beta, act, y, ldy, BF(hi), BFL(lo), ldo, B, HW, C, G,
                           (long long)HW * ldx, (long long)HW * ldy, (long long)HW * ldo, res, ldres, accumulate,
                           STREAM(stream));
  if (rc) return rc;
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_bcast_fma_f32(const float* a0, const float* ta, const float* p, float* out, int B, int T, int C,
                                   void* stream) {
  if (!a0 || !ta || !p || !out || B <= 0 || T <= 0 || C <= 0) return ODISE_ERR_ARG;
  bcast_fma_kernel<<<grid_for((long long)B * T * C, 256), 256, 0, STREAM(stream)>>>(a0, ta, p, out, B, T, C);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_rowscale_f32(float* y, long long ldy, const float* s, long long rows, int cols, void* stream) {
  if (!y || !s || rows <= 0 || cols <= 0) return ODISE_ERR_ARG;
  if (cols % 4 || ldy % 4) return ODISE_ERR_ALIGN;
  rowscale_kernel<<<grid_for(rows * (cols / 4), 256), 256, 0, STREAM(stream)>>>(y, ldy, s, rows, cols / 4);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_image_crops_u8_f32(const uint8_t* img, float* out, const int32_t* boxes, int n_crops, int H,
                                        int W, int ch, int cw, void* stream) {
  if (!img || !out || !boxes || n_crops <= 0 || H <= 0 || W <= 0 || ch <= 0 || cw <= 0) return ODISE_ERR_ARG;
  image_crops_kernel<<<grid_for((long long)n_crops * ch * cw, 256), 256, 0, STREAM(stream)>>>(img, out, boxes, n_crops,
                                                                                            H, W, ch, cw);
  count_launch(1);
  return (int)cudaGetLastError();
}

// workspace-based, coalesced statistics (see gn_partial_kernel).  ws: >= odise_groupnorm_ws_floats(B, HW, C, G) floats.
extern "C" long long odise_groupnorm_ws_floats(int B, int HW, int C, int G) {
  (void)C;
  int nchunk = (4 * num_sms() + B - 1) / B;
  if (nchunk > HW) nchunk = HW;
  if (nchunk < 1) nchunk = 1;
  return (long long)B * nchunk * G * 2;
}

extern "C" int odise_groupnorm_stats_ws_f32(const float* x, long long ldx, long long x_bs, float* ws, float* mean,
                                            float* rstd, int B, int HW, int C, int G, float eps, void* stream) {
  if (!x || !ws || !mean || !rstd || B <= 0 || HW <= 0 || C <= 0 || G <= 0 || C % G) return ODISE_ERR_ARG;
  if (C % 4 || ldx % 4 || x_bs % 4 || C / 4 > 1024) return ODISE_ERR_ALIGN;
  int nchunk = (4 * num_sms() + B - 1) / B;
  if (nchunk > HW) nchunk = HW;
  if (nchunk < 1) nchunk = 1;
  const int ppc = (HW + nchunk - 1) / nchunk;
  nchunk = (HW + ppc - 1) / ppc;
  const int C4 = C / 4;
  int PL = 256 / C4;
  if (PL < 1) PL = 1;
  if (PL > ppc) PL = ppc;
  const int threads = C4 * PL;
  const size_t smem = (size_t)2 * PL * C * sizeof(float);
  if (smem > 48 * 1024) return ODISE_ERR_UNSUPPORTED;
  const long long xbs = x_bs ? x_bs : (long long)HW * ldx;
  // NOTE: nchunk here must match odise_groupnorm_ws_floats' upper bound (it is <= that value)
  gn_partial_kernel<<<B * nchunk, threads, smem, STREAM(stream)>>>(x, ldx, xbs, ws, HW, C, G, nchunk, ppc);
  gn_finalize_kernel<<<(B * G + 7) / 8, 256, 0, STREAM(stream)>>>(x, xbs, ws, mean, rstd, B, HW, C, G, nchunk, eps);
  count_launch(2);
  return (int)cudaGetLastError();
}

extern "C" int odise_groupnorm_finalize_seg_f32(const float* partial, long long seg_stride, long long plane_stride,
                                                float* mean, float* rstd, int B, int HW, int C, int G, float eps,
                                                void* stream) {
  if (!partial || !mean || !rstd || B <= 0 || HW <= 0 || C <= 0 || G <= 0 || C % G || HW % 32) return ODISE_ERR_ARG;
  gn_finalize_seg_kernel<<<B * G, 256, 0, STREAM(stream)>>>(partial, seg_stride, plane_stride, mean, rstd, HW, C, G, eps);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_image_crops_f32(const float* img, float* out, const int32_t* boxes, int n_crops, int H, int W,
                                     int ch, int cw, void* stream) {
  if (!img || !out || !boxes || n_crops <= 0 || H <= 0 || W <= 0 || ch <= 0 || cw <= 0) return ODISE_ERR_ARG;
  image_crops_f32_kernel<<<grid_for((long long)n_crops * ch * cw, 256), 256, 0, STREAM(stream)>>>(img, out, boxes,
                                                                                                n_crops, H, W, ch, cw);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_clip_preprocess(const void* img, int img_is_u8, float* out, const int32_t* boxes, int n_crops,
                                     int H, int W, int ch, int cw, int S, void* stream) {
  if (!img || !out || !boxes || n_crops <= 0 || H <= 0 || W <= 0 || ch <= 0 || cw <= 0 || S <= 0) return ODISE_ERR_ARG;
  if (ch != cw) return ODISE_ERR_UNSUPPORTED;
  const int blocks = grid_for((long long)n_crops * S * S, 256);
  const float m0 = 0.48145466f, m1 = 0.4578275f, m2 = 0.40821073f, s0 = 0.26862954f, s1 = 0.26130258f, s2 = 0.27577711f;
  if (img_is_u8)
    clip_preprocess_kernel<uint8_t><<<blocks, 256, 0, STREAM(stream)>>>(reinterpret_cast<const uint8_t*>(img), out, boxes,
                                                                        n_crops, H, W, ch, cw, S, 1.f / 255.f, m0, m1, m2,
                                                                        s0, s1, s2);
  else
    clip_preprocess_kernel<float><<<blocks, 256, 0, STREAM(stream)>>>(reinterpret_cast<const float*>(img), out, boxes,
                                                                      n_crops, H, W, ch, cw, S, 1.f, m0, m1, m2, s0, s1, s2);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_crop_resize_bicubic(const void* img, int img_is_u8, float* out, const int32_t* boxes, int n_crops,
                                         int H, int W, int ch, int cw, int S, void* stream) {
  if (!img || !out || !boxes || n_crops <= 0 || H <= 0 || W <= 0 || ch <= 0 || cw <= 0 || S <= 0) return ODISE_ERR_ARG;
  if (ch != cw) return ODISE_ERR_UNSUPPORTED;
  const int blocks = grid_for((long long)n_crops * S * S, 256);
  if (img_is_u8)
    clip_preprocess_kernel<uint8_t, true><<<blocks, 256, 0, STREAM(stream)>>>(
        reinterpret_cast<const uint8_t*>(img), out, boxes, n_crops, H, W, ch, cw, S, 1.f / 255.f, 0, 0, 0, 1, 1, 1);
  else
    clip_preprocess_kernel<float, true><<<blocks, 256, 0, STREAM(stream)>>>(
        reinterpret_cast<const float*>(img), out, boxes, n_crops, H, W, ch, cw, S, 1.f, 0, 0, 0, 1, 1, 1);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_patchify_split_f32(const float* x, void* hi, void* lo, int B, int S, int P, int Kpad, void* stream) {
  if (!x || !hi || B <= 0 || S <= 0 || P <= 0 || S % P || Kpad < 3 * P * P || Kpad % 8) return ODISE_ERR_ARG;
  const int G = S / P;
  Q8_CHECK(lo, Kpad);
  patchify_split_kernel<<<grid_for((long long)B * G * G * Kpad, 256), 256, 0, STREAM(stream)>>>(x, BF(hi), BFL(lo), B, S,
                                                                                            P, Kpad);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_gather_rows_f32(const float* src, long long lds, const int32_t* idx, const float* add, long long ld_add,
                                     int add_period, float* out, long long ldo, long long rows, int cols, void* stream) {
  if (!src || !idx || !out || rows <= 0 || cols <= 0 || (add && add_period <= 0)) return ODISE_ERR_ARG;
  gather_rows_kernel<<<grid_for(rows * cols, 256), 256, 0, STREAM(stream)>>>(src, lds, idx, add, ld_add, add_period, out, ldo,
                                                                          rows, cols);
  count_launch(1);
  return (int)cudaGetLastError();
}
