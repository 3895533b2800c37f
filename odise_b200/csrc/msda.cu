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
#include "ptx.cuh"
#include "odise_b200.h"
#include "launch_count.h"

namespace ob {

// (H_l, W_l) / level_start stay on the device like in the reference (ms_deform_im2col_cuda.cuh:277-281): a
// handful of L1-broadcast int64 loads per thread, no host sync, CUDA-graph capturable.
struct MsdaLevels {
  const int64_t* shapes;
  const int64_t* start;
};

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
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

// generic scalar path (any D, e.g. the D=2 problem of the reference's ops/test.py:24-31)
__global__ void msda_scalar_kernel(const float* __restrict__ value, const MsdaLevels lv,
                                   const float* __restrict__ loc, const float* __restrict__ attn,
                                   float* __restrict__ out, int N, int S, int M, int D, int L, int Lq, int P) {
  const long long total = (long long)N * Lq * M * D;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % D);
    const long long pair = idx / D;
    const int m = (int)(pair % M);
    const int n = (int)(pair / M / Lq);
    const int pix_stride = M * D;
    const float* vb = value + (long long)n * S * pix_stride + m * D + c;
    float col = 0.f;
    for (int l = 0; l < L; ++l) {
      const int H = (int)__ldg(lv.shapes + 2 * l), W = (int)__ldg(lv.shapes + 2 * l + 1);
      const float* vl = vb + (long long)__ldg(lv.start + l) * pix_stride;
      for (int p = 0; p < P; ++p) {
        const float lx = loc[(pair * L * P + l * P + p) * 2], ly = loc[(pair * L * P + l * P + p) * 2 + 1];
        const float aw = attn[pair * L * P + l * P + p];
        const float h_im = ly * H - 0.5f, w_im = lx * W - 0.5f;
        if (h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W) {
          const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
          const float lh = h_im - h_low, lw = w_im - w_low, hh = 1.f - lh, hw = 1.f - lw;
          float v1 = 0, v2 = 0, v3 = 0, v4 = 0;
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

template <int FUSED>
__global__ void __launch_bounds__(256)
msda_d32_kernel(const float* __restrict__ value, const MsdaLevels lv, const float* __restrict__ loc_or_off,
                const float* __restrict__ attn_or_logit, const float* __restrict__ ref, float* __restrict__ out,
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
    float aw = 0.f, lx = 0.f, ly = 0.f;
    int H = 1, W = 1, start = 0;
    if (live) {
      const int l = s / P;
      H = (int)__ldg(lv.shapes + 2 * l);
      W = (int)__ldg(lv.shapes + 2 * l + 1);
      start = (int)__ldg(lv.start + l);
      const float2 xy = __ldg(reinterpret_cast<const float2*>(loc_or_off + (pair * LP + s) * 2));
      aw = __ldg(attn_or_logit + pair * LP + s);
      lx = xy.x; ly = xy.y;
      if (FUSED) {
        const long long nq = pair / M;
        const float2 r = __ldg(reinterpret_cast<const float2*>(ref + (nq * L + l) * 2));
        lx = r.x + xy.x / (float)W;          // ms_deform_attn.py:104-107
        ly = r.y + xy.y / (float)H;
      }
    }
    if (FUSED) {                               // softmax over the L*P logits of the pair (ms_deform_attn.py:100)
      float mx = live ? aw : -INFINITY;
      for (int o = SL >> 1; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float e = live ? expf(aw - mx) : 0.f;
      float sum = e;
      for (int o = SL >> 1; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      aw = e / sum;
    }
    if (live) {
      const float h_im = ly * H - 0.5f, w_im = lx * W - 0.5f;
      int4 o4 = make_int4(0, 0, 0, 0);
      float4 w4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W) {
        const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
        const float lh = h_im - h_low, lw = w_im - w_low, hh = 1.f - lh, hw = 1.f - lw;
        const bool t = h_low >= 0, b = h_low + 1 <= H - 1, lf = w_low >= 0, rt = w_low + 1 <= W - 1;
        const int base = (start + h_low * W + w_low) * pix;
        if (t && lf) { o4.x = base; w4.x = hh * hw * aw; }
        if (t && rt) { o4.y = base + pix; w4.y = hh * lw * aw; }
        if (b && lf) { o4.z = base + W * pix; w4.z = lh * hw * aw; }
        if (b && rt) { o4.w = base + (W + 1) * pix; w4.w = lh * lw * aw; }
      }
      s_off[pl * LP + s] = o4;
      s_w[pl * LP + s] = w4;
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
  const float* vb = value + (long long)n * S * pix + m * 32 + c;
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
  if (out) *reinterpret_cast<float4*>(out + o) = acc;
  if (out_hi) {
    const float e[4] = {acc.x, acc.y, acc.z, acc.w};
    store_planes<4>(out_hi + o, out_lo ? out_lo + o : nullptr, e);
  }
}

// 32-bit element offsets must cover one image's value block; L*P samples must fit a warp
static bool d32_ok(int S, int M, int D, int L, int P) {
  return D == 32 && L * P <= 32 && (long long)S * M * D < (1LL << 31);
}

template <int FUSED>
static void launch_d32(const float* value, const MsdaLevels& lv, const float* a, const float* b, const float* ref,
                       float* out, __nv_bfloat16* hi, __nv_bfloat16* lo, int N, int S, int M, int L, int Lq, int P,
                       cudaStream_t stream) {
  const int LP = L * P;
  int SL = 1;
  while (SL < LP) SL <<= 1;
  const long long pairs = (long long)N * Lq * M;
  const int blocks = (int)((pairs + MSDA_PAIRS - 1) / MSDA_PAIRS);
  const size_t smem = (size_t)MSDA_PAIRS * LP * (sizeof(int4) + sizeof(float4));
  msda_d32_kernel<FUSED><<<blocks, 256, smem, stream>>>(value, lv, a, b, ref, out, hi, lo, N, S, M, L, Lq, P, SL);
}

static bool vec_ok(int D) { return D % 4 == 0 && D <= 128 && (32 % (D / 4) == 0); }

}  // namespace ob

using namespace ob;

extern "C" int odise_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                      const float* loc, const float* attn, float* out, int N, int S, int M, int D,
                                      int L, int Lq, int P, void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  if (!value || !spatial_shapes || !level_start || !loc || !attn || !out) return ODISE_ERR_ARG;
  if (N <= 0 || S <= 0 || M <= 0 || D <= 0 || L <= 0 || L > 8 || Lq <= 0 || P <= 0) return ODISE_ERR_ARG;
  MsdaLevels lv{spatial_shapes, level_start};
  if (d32_ok(S, M, D, L, P)) {
    launch_d32<0>(value, lv, loc, attn, nullptr, out, nullptr, nullptr, N, S, M, L, Lq, P, stream);
  } else if (vec_ok(D)) {
    const int lph = D / 4;
    const long long threads = (long long)N * Lq * M * lph;
    const int blocks = (int)((threads + 255) / 256);
    msda_vec4_kernel<0><<<blocks, 256, 0, stream>>>(value, lv, loc, attn, nullptr, out, nullptr, nullptr, N, S, M, D,
                                                    L, Lq, P, lph);
  } else {
    const long long total = (long long)N * Lq * M * D;
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    msda_scalar_kernel<<<blocks, 256, 0, stream>>>(value, lv, loc, attn, out, N, S, M, D, L, Lq, P);
  }
  count_launch(1);
  return (int)cudaGetLastError();
}

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
