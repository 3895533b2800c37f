// MaskCLIP front-end and the open-vocabulary class merge of ODISE inference (SURVEY.md §8a row b13, §8f-2), sm_90a.
//
// Reference: MaskCLIP.get_mask_embed / encode_image_with_mask (odise/modeling/meta_arch/clip.py:284-339) resizes the
// [0,1] image and the Q mask logits bilinearly to the CLIP resolution, max-pools sigmoid(mask) per 14x14 patch and
// materialises a bool attention mask [B*heads, Q+577, Q+577]; PoolingCLIPHead.forward (odise.py:1506-1536) and the
// tail of CategoryODISE.forward (odise.py:300-323) then merge the two class distributions.  Here:
//   * maskclip_preprocess: bilinear resize of the whole image + CLIP normalisation in one pass (NHWC out);
//   * maskclip_bits: per (image, query) one bit per key of the ViT sequence (class token always on, patch p on iff
//     max over its window of the upsampled mask has sigmoid >= 0.5), in the bit layout odise_attention_tc consumes —
//     the bool mask, the sigmoid map and the pooled map are never materialised;
//   * open_vocab_merge: softmaxes, geometric ensemble (alpha for training classes, beta for novel ones), void merge
//     and the final log in one warp-per-query pass.  Computed in log space, so it stays finite where the reference's
//     pow/log formulation underflows to log(0) * 0 = NaN.
#include "ptx.cuh"
#include "odise_b200.h"
#include "launch_count.h"

namespace ob {

__device__ __forceinline__ float mc_wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float mc_wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ATen upsample_bilinear2d, align_corners=False
__device__ __forceinline__ void bil_coeff(int o, float scale, int n, int& i0, int& i1, float& l1) {
  const float f = fmaxf((o + 0.5f) * scale - 0.5f, 0.f);
  i0 = min((int)f, n - 1);
  i1 = i0 + (i0 < n - 1 ? 1 : 0);
  l1 = f - i0;
}

template <typename T>
__global__ void maskclip_preprocess_kernel(const T* __restrict__ img, float* __restrict__ out, int N, int H, int W, int S,
                                           float denom) {
  const long long total = (long long)N * S * S;
  const float sy = (float)H / (float)S, sx = (float)W / (float)S;
  const float mean[3] = {0.48145466f, 0.4578275f, 0.40821073f}, stdv[3] = {0.26862954f, 0.26130258f, 0.27577711f};
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % S);
    const long long t = i / S;
    const int oy = (int)(t % S), n = (int)(t / S);
    int y0, y1, x0, x1;
    float ly, lx;
    bil_coeff(oy, sy, H, y0, y1, ly);
    bil_coeff(ox, sx, W, x0, x1, lx);
    const float hy = 1.f - ly, hx = 1.f - lx;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const T* src = img + ((long long)n * 3 + c) * H * W;
      const float a = (float)src[(long long)y0 * W + x0] / denom, b = (float)src[(long long)y0 * W + x1] / denom;
      const float d = (float)src[(long long)y1 * W + x0] / denom, e = (float)src[(long long)y1 * W + x1] / denom;
      const float v = hy * (hx * a + lx * b) + ly * (hx * d + lx * e);
      out[i * 3 + c] = (v - mean[c]) / stdv[c];
    }
  }
}

// grid (Q, B), block 32 * n_words: warp w owns word w of the row of mask token q
__global__ void maskclip_bits_kernel(const float* __restrict__ logits, uint32_t* __restrict__ bits,
                                     int32_t* __restrict__ row_any, int Q, int hm, int wm, int S, int P, int Tq, int row0,
                                     int n_words) {
  const int q = blockIdx.x, b = blockIdx.y, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = S / P, Tk = G * G + 1;
  const int key = w * 32 + lane;
  bool on = false;
  if (key == 0) {
    on = true;                                     // the class token is never masked (clip.py:308-314)
  } else if (key < Tk) {
    const int py = (key - 1) / G, px = (key - 1) % G;
    const float* src = logits + ((long long)b * Q + q) * hm * wm;
    const float sy = (float)hm / (float)S, sx = (float)wm / (float)S;
    float mx = -INFINITY;
    for (int dy = 0; dy < P; ++dy) {
      int y0, y1;
      float ly;
      bil_coeff(py * P + dy, sy, hm, y0, y1, ly);
      const float hy = 1.f - ly;
      for (int dx = 0; dx < P; ++dx) {
        int x0, x1;
        float lx;
        bil_coeff(px * P + dx, sx, wm, x0, x1, lx);
        const float hx = 1.f - lx;
        const float v = hy * (hx * src[y0 * wm + x0] + lx * src[y0 * wm + x1]) +
                        ly * (hx * src[y1 * wm + x0] + lx * src[y1 * wm + x1]);
        mx = fmaxf(mx, v);
      }
    }
    // sigmoid is monotone: max-pool of sigmoid == sigmoid of the max; blocked iff that value < 0.5 (clip.py:297-304)
    on = !(1.f / (1.f + expf(-mx)) < 0.5f);
  }
  const uint32_t word = __ballot_sync(0xffffffffu, on);
  const long long row = (long long)b * Tq + row0 + q;
  if (lane == 0 && w < n_words) bits[row * n_words + w] = word;
  if (threadIdx.x == 0) row_any[row] = 1;
}

// warp per (image, query) row.  cat [rows, K+1] (category-head logits incl. void), clip [rows, K] (MaskCLIP logits)
__global__ void open_vocab_merge_kernel(const float* __restrict__ cat, const float* __restrict__ clip, long long ld_clip,
                                        const uint8_t* __restrict__ overlap, float alpha, float beta,
                                        float* __restrict__ out, float* __restrict__ open_logits, int rows, int K) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* c = cat + (long long)r * (K + 1);
  const float* m = clip + (long long)r * ld_clip;
  float cmx = -INFINITY, mmx = -INFINITY;
  for (int k = lane; k < K; k += 32) { cmx = fmaxf(cmx, c[k]); mmx = fmaxf(mmx, m[k]); }
  cmx = mc_wmax(cmx); mmx = mc_wmax(mmx);
  float cs = 0.f, ms = 0.f;
  for (int k = lane; k < K; k += 32) { cs += expf(c[k] - cmx); ms += expf(m[k] - mmx); }
  cs = mc_wsum(cs); ms = mc_wsum(ms);
  const float clse = cmx + logf(cs), mlse = mmx + logf(ms);
  // void probability over the K+1 category logits
  const float vmx = fmaxf(cmx, c[K]);
  const float p_void = expf(c[K] - vmx) / (cs * expf(cmx - vmx) + expf(c[K] - vmx));
  // ensemble logits e_k = (1-a_k) log p_k + a_k log m_k  (odise.py:1513-1524), then softmax over K
  float emx = -INFINITY;
  for (int k = lane; k < K; k += 32) {
    const float a = overlap[k] ? alpha : beta;
    const float e = (1.f - a) * (c[k] - clse) + a * (m[k] - mlse);
    if (open_logits) open_logits[(long long)r * K + k] = e;
    emx = fmaxf(emx, e);
  }
  emx = mc_wmax(emx);
  float es = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float a = overlap[k] ? alpha : beta;
    es += expf((1.f - a) * (c[k] - clse) + a * (m[k] - mlse) - emx);
  }
  es = mc_wsum(es);
  float* o = out + (long long)r * (K + 1);
  const float fg = 1.f - p_void;
  for (int k = lane; k < K; k += 32) {
    const float a = overlap[k] ? alpha : beta;
    const float pk = expf((1.f - a) * (c[k] - clse) + a * (m[k] - mlse) - emx) / es;
    o[k] = logf(pk * fg + 1e-8f);
  }
  if (lane == 0) o[K] = logf(p_void + 1e-8f);
}

}  // namespace ob

using namespace ob;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int odise_maskclip_preprocess(const void* img, int img_is_u8, float* out, int N, int H, int W, int S,
                                         void* stream) {
  if (!img || !out || N <= 0 || H <= 0 || W <= 0 || S <= 0) return ODISE_ERR_ARG;
  const long long total = (long long)N * S * S;
  const int blocks = (int)((total + 255) / 256);
  if (img_is_u8)
    maskclip_preprocess_kernel<uint8_t><<<blocks, 256, 0, STREAM(stream)>>>(reinterpret_cast<const uint8_t*>(img), out, N, H,
                                                                            W, S, 255.f);
  else
    maskclip_preprocess_kernel<float><<<blocks, 256, 0, STREAM(stream)>>>(reinterpret_cast<const float*>(img), out, N, H, W,
                                                                          S, 1.f);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_maskclip_bits_f32(const float* mask_logits, uint32_t* bits, int32_t* row_any, int B, int Q, int hm,
                                       int wm, int S, int P, int Tq, int row0, void* stream) {
  if (!mask_logits || !bits || !row_any || B <= 0 || Q <= 0 || hm <= 0 || wm <= 0 || S <= 0 || P <= 0 || S % P)
    return ODISE_ERR_ARG;
  const int G = S / P, Tk = G * G + 1, n_words = (Tk + 31) / 32;
  if (row0 < 0 || row0 + Q > Tq || n_words * 32 > 1024) return ODISE_ERR_ARG;
  cudaError_t e = cudaMemsetAsync(row_any, 0, sizeof(int32_t) * (size_t)B * Tq, STREAM(stream));
  if (e != cudaSuccess) return (int)e;
  maskclip_bits_kernel<<<dim3(Q, B), 32 * n_words, 0, STREAM(stream)>>>(mask_logits, bits, row_any, Q, hm, wm, S, P, Tq,
                                                                        row0, n_words);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_open_vocab_merge_f32(const float* cat_logits, const float* clip_logits, long long ld_clip,
                                          const uint8_t* overlap, float alpha, float beta, float* out,
                                          float* open_logits, int rows, int K, void* stream) {
  if (!cat_logits || !clip_logits || !overlap || !out || rows <= 0 || K <= 0 || ld_clip < K) return ODISE_ERR_ARG;
  open_vocab_merge_kernel<<<(rows + 7) / 8, 256, 0, STREAM(stream)>>>(cat_logits, clip_logits, ld_clip, overlap, alpha,
                                                                      beta, out, open_logits, rows, K);
  count_launch(1);
  return (int)cudaGetLastError();
}
