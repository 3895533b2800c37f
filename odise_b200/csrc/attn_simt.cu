// Warp-shuffle attention kernels of the Mask2Former transformer decoder (SURVEY.md §8a rows b7-b9), sm_90a.
//
// Reference: nn.MultiheadAttention(256, 8) inside CrossAttentionLayer / SelfAttentionLayer
// (mask2former_transformer_decoder.py:22,80,98-110,40-50) fed a materialised bool attn_mask [B*8, Q, HW] that
// ODISE builds per layer from the previous head's mask logits (odise.py:760-774) plus the
// "row fully masked => unmask" fix-up (odise.py:683).  Here:
//   * attn_mask_bits: one pass over the mask logits -> bilinear resize to the level size (align_corners=False),
//     sigmoid < 0.5 test, 1 bit per (b, q, key) shared by all 8 heads (the reference repeats the mask per head),
//     and a per-row "any key allowed" flag that implements the fix-up without touching the bits.
//   * mha_d32: flash-style (online softmax) attention for head_dim 32: a warp owns a query, lanes own keys for the
//     score pass and channels for the P.V pass (shuffle broadcast of p), K/V tiles staged in shared memory.
#include "ptx.cuh"
#include "odise_b200.h"
#include "launch_count.h"

namespace ob {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block per (b, q) row; bits[b][q][w] bit i = key (w*32+i) may be attended
__global__ void __launch_bounds__(256)
attn_mask_bits_kernel(const float* __restrict__ logits, uint32_t* __restrict__ bits, int32_t* __restrict__ row_any,
                      int Hm, int Wm, int Hl, int Wl) {
  const long long row = blockIdx.x;
  const float* src = logits + row * (long long)Hm * Wm;
  const int HW = Hl * Wl;
  const int words = (HW + 31) / 32;
  uint32_t* dst = bits + row * words;
  const float sy = (float)Hm / (float)Hl, sx = (float)Wm / (float)Wl;
  int any = 0;
  for (int base = (threadIdx.x >> 5) * 32; base < words * 32; base += (blockDim.x >> 5) * 32) {
    const int key = base + (threadIdx.x & 31);
    bool allowed = false;
    if (key < HW) {
      const int oy = key / Wl, ox = key - oy * Wl;
      // F.interpolate(bilinear, align_corners=False) source index (ATen area_pixel_compute_source_index)
      const float fy = fmaxf((oy + 0.5f) * sy - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sx - 0.5f, 0.f);
      const int y0 = (int)fy, x0 = (int)fx;
      const int y1 = y0 + (y0 < Hm - 1 ? 1 : 0), x1 = x0 + (x0 < Wm - 1 ? 1 : 0);
      const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
      const float v = hy * (hx * src[y0 * Wm + x0] + lx * src[y0 * Wm + x1]) +
                      ly * (hx * src[y1 * Wm + x0] + lx * src[y1 * Wm + x1]);
      const float s = 1.f / (1.f + expf(-v));
      allowed = !(s < 0.5f);  // attn_mask = sigmoid(.) < 0.5 means "blocked"
    }
    const uint32_t w = __ballot_sync(0xffffffffu, allowed);
    if ((threadIdx.x & 31) == 0) dst[base >> 5] = w;
    any |= (w != 0);
  }
  any = __syncthreads_or(any);
  if (threadIdx.x == 0) row_any[row] = any;
}

// grid (q_tiles * key_splits, heads, B); 8 warps x QPW queries (register blocked: every K / V element read from
// shared memory feeds QPW FMAs; P is broadcast through shared memory as one float4 per key), head_dim 32.
// key_splits > 1: each block handles a slice of the keys and writes (m, l, o) partials merged by mha_merge_kernel.
template <int QPW>
__global__ void __launch_bounds__(256)
mha_d32_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ k,
               const float* __restrict__ v, long long ldkv, const uint32_t* __restrict__ bits,
               const int32_t* __restrict__ row_any, float* __restrict__ out, __nv_bfloat16* __restrict__ out_hi,
               __nv_bfloat16* __restrict__ out_lo, long long ldo, int Tq, int Tk, int heads, float scale,
               int key_splits, float* __restrict__ part) {
  static_assert(QPW == 4, "P broadcast uses float4");
  constexpr int KT = 128;                // keys per shared-memory tile
  __shared__ float Ks[KT][33];
  __shared__ float Vs[KT][32];
  __shared__ float4 Ps[8][32];
  const int b = blockIdx.z, h = blockIdx.y;
  const int qt = blockIdx.x / key_splits, ksp = blockIdx.x - qt * key_splits;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int words = (Tk + 31) / 32;
  // key range of this split, multiple of KT
  const int tiles = (Tk + KT - 1) / KT;
  const int tps = (tiles + key_splits - 1) / key_splits;
  const int kbeg = ksp * tps * KT, kend = min(Tk, (ksp + 1) * tps * KT);

  float qreg[QPW][32];
  float m[QPW], l[QPW], o[QPW];
  int qi[QPW];
  bool use_mask[QPW];
#pragma unroll
  for (int t = 0; t < QPW; ++t) {
    qi[t] = (qt * 8 + warp) * QPW + t;
    m[t] = -INFINITY; l[t] = 0.f; o[t] = 0.f;
    use_mask[t] = false;
    if (qi[t] < Tq) {
      const float* qp = q + ((long long)b * Tq + qi[t]) * ldq + h * 32;
#pragma unroll
      for (int d = 0; d < 32; ++d) qreg[t][d] = __ldg(qp + d) * scale;
      if (bits) use_mask[t] = row_any[(long long)b * Tq + qi[t]] != 0;
    } else {
#pragma unroll
      for (int d = 0; d < 32; ++d) qreg[t][d] = 0.f;
    }
  }
  const bool warp_active = qi[0] < Tq;   // queries of a warp are consecutive

  for (int k0 = kbeg; k0 < kend; k0 += KT) {
    __syncthreads();
    for (int i = threadIdx.x; i < KT * 8; i += 256) {
      const int r = i >> 3, c4 = (i & 7) * 4;
      float4 kv = make_float4(0, 0, 0, 0), vv = kv;
      if (k0 + r < Tk) {
        kv = *reinterpret_cast<const float4*>(k + ((long long)b * Tk + k0 + r) * ldkv + h * 32 + c4);
        vv = *reinterpret_cast<const float4*>(v + ((long long)b * Tk + k0 + r) * ldkv + h * 32 + c4);
      }
      Ks[r][c4] = kv.x; Ks[r][c4 + 1] = kv.y; Ks[r][c4 + 2] = kv.z; Ks[r][c4 + 3] = kv.w;
      *reinterpret_cast<float4*>(&Vs[r][c4]) = vv;
    }
    __syncthreads();
    if (!warp_active) continue;
#pragma unroll 1
    for (int sb = 0; sb < KT; sb += 32) {
      if (k0 + sb >= Tk) break;
      const int key = k0 + sb + lane;
      float s[QPW];
#pragma unroll
      for (int t = 0; t < QPW; ++t) s[t] = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        const float kd = Ks[sb + lane][d];
#pragma unroll
        for (int t = 0; t < QPW; ++t) s[t] = fmaf(qreg[t][d], kd, s[t]);
      }
      float pv[QPW], alpha[QPW];
#pragma unroll
      for (int t = 0; t < QPW; ++t) {
        bool ok = key < Tk && qi[t] < Tq;
        if (use_mask[t]) {
          const uint32_t w = __ldg(bits + ((long long)b * Tq + qi[t]) * words + ((k0 + sb) >> 5));
          ok = ok && ((w >> lane) & 1u);
        }
        const float sv = ok ? s[t] : -INFINITY;
        const float mnew = fmaxf(m[t], wmax(sv));
        if (mnew == -INFINITY) { pv[t] = 0.f; alpha[t] = 1.f; continue; }   // nothing attendable yet (warp-uniform)
        alpha[t] = __expf(m[t] - mnew);
        pv[t] = ok ? expf(sv - mnew) : 0.f;
        l[t] = l[t] * alpha[t] + wsum(pv[t]);
        m[t] = mnew;
      }
      Ps[warp][lane] = make_float4(pv[0], pv[1], pv[2], pv[3]);
      __syncwarp();
      float acc[QPW];
#pragma unroll
      for (int t = 0; t < QPW; ++t) acc[t] = o[t] * alpha[t];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float4 pj = Ps[warp][j];
        const float vj = Vs[sb + j][lane];
        acc[0] = fmaf(pj.x, vj, acc[0]); acc[1] = fmaf(pj.y, vj, acc[1]);
        acc[2] = fmaf(pj.z, vj, acc[2]); acc[3] = fmaf(pj.w, vj, acc[3]);
      }
#pragma unroll
      for (int t = 0; t < QPW; ++t) o[t] = acc[t];
      __syncwarp();
    }
  }
#pragma unroll
  for (int t = 0; t < QPW; ++t) {
    if (qi[t] >= Tq) continue;
    if (key_splits > 1) {
      // partial: [b][h][q][split][34] = (m, l, o[32])
      float* pp = part + ((((long long)b * heads + h) * Tq + qi[t]) * key_splits + ksp) * 34;
      if (lane == 0) { pp[0] = m[t]; pp[1] = l[t]; }
      pp[2 + lane] = o[t];
      continue;
    }
    const float r = o[t] / l[t];
    const long long idx = ((long long)b * Tq + qi[t]) * ldo + h * 32 + lane;
    if (out) out[idx] = r;
    if (out_hi) {
      store_planes<1>(out_hi + idx, out_lo ? out_lo + idx : nullptr, &r);
    }
  }
}

// one warp per (b, h, q): merge the key-split partials
__global__ void mha_merge_kernel(const float* __restrict__ part, float* __restrict__ out,
                                 __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo,
                                 long long ldo, int B, int Tq, int heads, int key_splits) {
  const long long w = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long total = (long long)B * heads * Tq;
  if (w >= total) return;
  const int lane = threadIdx.x & 31;
  const int qd = (int)(w % Tq);
  const int h = (int)((w / Tq) % heads);
  const int b = (int)(w / ((long long)Tq * heads));
  const float* pp = part + w * key_splits * 34;
  float M = -INFINITY;
  for (int s = 0; s < key_splits; ++s) M = fmaxf(M, pp[s * 34]);
  float L = 0.f, O = 0.f;
  for (int s = 0; s < key_splits; ++s) {
    const float ms = pp[s * 34];
    if (ms == -INFINITY) continue;
    const float f = expf(ms - M);
    L += pp[s * 34 + 1] * f;
    O += pp[s * 34 + 2 + lane] * f;
  }
  const float r = O / L;
  const long long idx = ((long long)b * Tq + qd) * ldo + h * 32 + lane;
  if (out) out[idx] = r;
  if (out_hi) {
    store_planes<1>(out_hi + idx, out_lo ? out_lo + idx : nullptr, &r);
  }
}

}  // namespace ob

using namespace ob;

extern "C" int odise_attn_mask_bits_f32(const float* mask_logits, uint32_t* bits, int32_t* row_any, int B, int Q,
                                        int Hm, int Wm, int Hl, int Wl, void* stream) {
  if (!mask_logits || !bits || !row_any || B <= 0 || Q <= 0 || Hm <= 0 || Wm <= 0 || Hl <= 0 || Wl <= 0)
    return ODISE_ERR_ARG;
  attn_mask_bits_kernel<<<B * Q, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(mask_logits, bits, row_any, Hm,
                                                                                  Wm, Hl, Wl);
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" long long odise_mha_d32_ws_floats(int B, int Tq, int Tk, int heads) {
  const int ks = Tk >= 8192 ? 4 : (Tk >= 2048 ? 2 : 1);
  return ks > 1 ? (long long)B * heads * Tq * ks * 34 : 0;
}

extern "C" int odise_mha_d32_f32(const float* q, long long ldq, const float* k, const float* v, long long ldkv,
                                 const uint32_t* bits, const int32_t* row_any, float* out, void* out_hi,
                                 void* out_lo, long long ldo, int B, int Tq, int Tk, int heads, float scale,
                                 void* stream) {
  return odise_mha_d32_ws_f32(q, ldq, k, v, ldkv, bits, row_any, out, out_hi, out_lo, ldo, B, Tq, Tk, heads, scale,
                              nullptr, stream);
}

// ws: odise_mha_d32_ws_floats() floats (may be NULL: then the keys are not split across blocks)
extern "C" int odise_mha_d32_ws_f32(const float* q, long long ldq, const float* k, const float* v, long long ldkv,
                                    const uint32_t* bits, const int32_t* row_any, float* out, void* out_hi,
                                    void* out_lo, long long ldo, int B, int Tq, int Tk, int heads, float scale,
                                    float* ws, void* stream) {
  if (!q || !k || !v || (!out && !out_hi) || B <= 0 || Tq <= 0 || Tk <= 0 || heads <= 0) return ODISE_ERR_ARG;
  if (ldq < heads * 32 || ldkv < heads * 32 || ldo < heads * 32 || ldkv % 4) return ODISE_ERR_ALIGN;
  if (bits && !row_any) return ODISE_ERR_ARG;
  constexpr int QPW = 4;
  int ks = Tk >= 8192 ? 4 : (Tk >= 2048 ? 2 : 1);
  if (!ws) ks = 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int qtiles = (Tq + 8 * QPW - 1) / (8 * QPW);
  dim3 grid(qtiles * ks, heads, B);
  mha_d32_kernel<QPW><<<grid, 256, 0, st>>>(q, ldq, k, v, ldkv, bits, row_any, out,
                                            reinterpret_cast<__nv_bfloat16*>(out_hi),
                                            lo_arg(reinterpret_cast<__nv_bfloat16*>(out_lo)), ldo, Tq, Tk, heads, scale, ks, ws);
  int n = 1;
  if (ks > 1) {
    const long long warps = (long long)B * heads * Tq;
    mha_merge_kernel<<<(int)((warps + 7) / 8), 256, 0, st>>>(ws, out, reinterpret_cast<__nv_bfloat16*>(out_hi),
                                                             lo_arg(reinterpret_cast<__nv_bfloat16*>(out_lo)), ldo, B, Tq, heads,
                                                             ks);
    n = 2;
  }
  count_launch(n);
  return (int)cudaGetLastError();
}
