// Masked cross-attention for training on sm_90a: the attention core of Mask2Former's CrossAttentionLayer
// (mask2former_transformer_decoder.py:75-135, nn.MultiheadAttention with a bool attn_mask), forward and backward.
//
//   out[q, b, h, :] = softmax_j( (s * q[q, b, h, :]) . k[j, b, h, :], blocked -> -inf ) v[j, b, h, :],  s = 1/sqrt(32)
//
// Head dim 32, sequence-first layouts as the in-projections write them (q [Q, B, H*32], k / v [S, B, H*32], out like q),
// bool mask [B*H, Q, S] or [Q, S] read as bytes (non-zero = blocked).  Storage float, __half or __nv_bfloat16; every
// load is converted to fp32, all arithmetic is fp32 in registers and each output is rounded once.  No [B*H, Q, S]
// tensor is written: the forward saves only lse [B*H, Q] (fp32), the backward recomputes the probabilities from it.
//
// Forward (flash-decoding): a CTA owns 32 queries of one (image, head) and one chunk of the keys.  The chunk count
// depends on the shape only (xa_chunks), so the result bits depend on the inputs only.  The CTA streams 64-key tiles of
// K and V through shared memory; thread (r, g) = (t / 8, t % 8) scores keys 8g..8g+7 of query r against its q row held
// in registers, runs the online softmax of its row (8-lane shuffles) and accumulates channels 4g..4g+3 of P V.  A
// combine pass merges the chunks in chunk order and writes out and lse.
//
// Backward: delta = rowsum(dO o O) first.  dK and dV come from a CTA that owns 64 keys and walks every query tile in
// order, recomputing P = exp(s - lse) and dS = P (dP - delta); no atomics.  dQ is summed per (query tile, key chunk)
// into an fp32 workspace and reduced in chunk order.  So dq, dk and dv are bit-reproducible without any switch.
//
// A row whose keys are all blocked follows torch's math path: its output and its dq row are NaN, and so are dk and dv of
// its whole (image, head) (P of that row is NaN for every key).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "launch_count.h"
#include "odise_b200.h"
#include "storage.cuh"

namespace ob {
namespace {

constexpr int XA_D = 32;              // head dim
constexpr int XA_BQ = 32;             // queries per CTA tile
constexpr int XA_BK = 64;             // keys per shared-memory tile
constexpr int XA_NT = 256;            // threads per CTA
constexpr int XA_PS = XA_BK + 4;      // row stride of the P / dS tiles (float4-aligned)
constexpr int XA_TARGET_CTAS = 528;   // 4 CTAs per SM on 132 SMs: the forward / dQ chunking aims at this many

__device__ __forceinline__ float4 xa_lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void xa_sts4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// 64 rows x 32 channels of k or v (rows k0.. of one (image, head); src points at row 0, rows `rs` elements apart) into
// shared memory, zeros past S.  SWZ: channel chunk ch (4 floats) of row j is stored at chunk ch ^ (j / 8), so that the
// score loop's 8 lanes of a row group (keys 8g + i, g = 0..7) read 8 different bank groups.
template <typename T, bool SWZ>
__device__ __forceinline__ void xa_load_tile(float* dst, const T* src, long long rs, int k0, int S) {
  for (int e = threadIdx.x; e < XA_BK * 8; e += XA_NT) {
    const int j = e >> 3, ch = e & 7;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k0 + j < S) x = ld4(src + (long long)(k0 + j) * rs + ch * 4);
    xa_sts4(dst + j * XA_D + (SWZ ? (ch ^ (j >> 3)) : ch) * 4, x);
  }
}

// bit i set when key kb + i is blocked by the mask or lies past S (mrow: the mask row, or null for no mask)
__device__ __forceinline__ unsigned xa_blocked8(const uint8_t* mrow, int kb, int S, bool vec) {
  unsigned bits = 0;
  if (kb + 8 <= S) {
    if (mrow) {
      if (vec) {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(mrow + kb));
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          bits |= ((u.x >> (8 * i)) & 0xffu) ? (1u << i) : 0u;
          bits |= ((u.y >> (8 * i)) & 0xffu) ? (1u << (i + 4)) : 0u;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) bits |= __ldg(mrow + kb + i) ? (1u << i) : 0u;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int kk = kb + i;
      bits |= (kk >= S || (mrow && __ldg(mrow + kk))) ? (1u << i) : 0u;
    }
  }
  return bits;
}

// 32-channel dot product of a register row with a swizzled shared-memory row read by lane group g (fixed order)
__device__ __forceinline__ float xa_dot_swz(const float* reg, const float* row, int g) {
  float d = 0.f;
#pragma unroll
  for (int ch = 0; ch < 8; ++ch) {
    const float4 x = xa_lds4(row + ((ch ^ g) * 4));
    d = fmaf(reg[4 * ch + 0], x.x, d);
    d = fmaf(reg[4 * ch + 1], x.y, d);
    d = fmaf(reg[4 * ch + 2], x.z, d);
    d = fmaf(reg[4 * ch + 3], x.w, d);
  }
  return d;
}

// the 8 lanes of a row group (lane bits 0-2) agree bit for bit: xor butterflies add / compare the same pairs
__device__ __forceinline__ float xa_max8(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 4));
}
__device__ __forceinline__ float xa_sum8(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  x += __shfl_xor_sync(0xffffffffu, x, 2);
  return x + __shfl_xor_sync(0xffffffffu, x, 4);
}

// a row of 32 channels (q scaled by `scale`, or dO) into registers; zeros for rows past Q
template <typename T>
__device__ __forceinline__ void xa_row_regs(float* reg, const T* p, bool ok, float scale) {
#pragma unroll
  for (int ch = 0; ch < 8; ++ch) {
    float4 x = ok ? ld4(p + ch * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    reg[4 * ch + 0] = x.x * scale;
    reg[4 * ch + 1] = x.y * scale;
    reg[4 * ch + 2] = x.z * scale;
    reg[4 * ch + 3] = x.w * scale;
  }
}

struct XaShape {
  int B, H, Q, S;
  __host__ __device__ long long E() const { return (long long)H * XA_D; }
};

// forward partials: per (chunk, b*H + h, q) the running max m, the sum l and the unnormalised accumulator (fp32)
template <typename T>
__global__ void __launch_bounds__(XA_NT) xattn_fwd_kernel(const T* __restrict__ q, const T* __restrict__ k,
                                                          const T* __restrict__ v, const uint8_t* __restrict__ mask,
                                                          long long mstride, bool mvec, float* __restrict__ ws_acc,
                                                          float* __restrict__ ws_ml, XaShape sh, int tiles_per_chunk,
                                                          float scale) {
  __shared__ __align__(16) float Ks[XA_BK * XA_D];
  __shared__ __align__(16) float Vs[XA_BK * XA_D];
  __shared__ __align__(16) float Ps[XA_BQ * XA_PS];
  const int t = threadIdx.x, r = t >> 3, g = t & 7;
  const int chunk = blockIdx.y, bh = blockIdx.z, b = bh / sh.H, h = bh % sh.H;
  const int qi = blockIdx.x * XA_BQ + r;
  const bool qok = qi < sh.Q;
  const long long E = sh.E(), rs = (long long)sh.B * E, head = (long long)b * E + h * XA_D;
  float qr[XA_D];
  xa_row_regs(qr, q + (long long)qi * rs + head, qok, scale);
  const uint8_t* mrow = (mask && qok) ? mask + (long long)bh * mstride + (long long)qi * sh.S : nullptr;
  const int ntiles = (sh.S + XA_BK - 1) / XA_BK;
  const int kt0 = chunk * tiles_per_chunk, kt1 = min(kt0 + tiles_per_chunk, ntiles);
  float m = -INFINITY, l = 0.f;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int kt = kt0; kt < kt1; ++kt) {
    const int k0 = kt * XA_BK;
    __syncthreads();
    xa_load_tile<T, true>(Ks, k + head, rs, k0, sh.S);
    xa_load_tile<T, false>(Vs, v + head, rs, k0, sh.S);
    const unsigned blk = xa_blocked8(mrow, k0 + g * 8, sh.S, mvec);
    __syncthreads();
    float s[8], mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = xa_dot_swz(qr, Ks + (g * 8 + i) * XA_D, g);
      s[i] = ((blk >> i) & 1u) ? -INFINITY : d;
      mx = fmaxf(mx, s[i]);
    }
    const float mn = fmaxf(m, xa_max8(mx));
    float alpha = 1.f, ps = 0.f;
    if (mn != -INFINITY) {
      alpha = expf(m - mn);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i] = expf(s[i] - mn);
        ps += s[i];
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] = 0.f;
    }
    l = l * alpha + xa_sum8(ps);
    m = mn;
    acc.x *= alpha; acc.y *= alpha; acc.z *= alpha; acc.w *= alpha;
    xa_sts4(Ps + r * XA_PS + g * 8, make_float4(s[0], s[1], s[2], s[3]));
    xa_sts4(Ps + r * XA_PS + g * 8 + 4, make_float4(s[4], s[5], s[6], s[7]));
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < XA_BK; j += 4) {
      const float4 p = xa_lds4(Ps + r * XA_PS + j);
      const float pj[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float4 x = xa_lds4(Vs + (j + jj) * XA_D + g * 4);
        acc.x = fmaf(pj[jj], x.x, acc.x);
        acc.y = fmaf(pj[jj], x.y, acc.y);
        acc.z = fmaf(pj[jj], x.z, acc.z);
        acc.w = fmaf(pj[jj], x.w, acc.w);
      }
    }
  }
  if (qok) {
    const long long row = ((long long)chunk * sh.B * sh.H + bh) * sh.Q + qi;
    xa_sts4(ws_acc + row * XA_D + g * 4, acc);
    if (g == 0) {
      ws_ml[2 * row] = m;
      ws_ml[2 * row + 1] = l;
    }
  }
}

// merge the chunks in chunk order: one warp per (b*H + h, q) row, lane = channel
template <typename T>
__global__ void xattn_combine_kernel(const float* __restrict__ ws_acc, const float* __restrict__ ws_ml, T* __restrict__ out,
                                     float* __restrict__ lse, XaShape sh, int nchunk) {
  const long long BHQ = (long long)sh.B * sh.H * sh.Q;
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= BHQ) return;
  const int bh = (int)(row / sh.Q), qi = (int)(row % sh.Q), b = bh / sh.H, h = bh % sh.H;
  float M = -INFINITY;
  for (int c = 0; c < nchunk; ++c) M = fmaxf(M, ws_ml[2 * (c * BHQ + row)]);
  float o, ls;
  if (M == -INFINITY) {       // every key of the row is blocked: torch's softmax gives NaN
    o = __int_as_float(0x7fffffff);
    ls = -INFINITY;
  } else {
    float L = 0.f, a = 0.f;
    for (int c = 0; c < nchunk; ++c) {
      const long long cr = c * BHQ + row;
      const float w = expf(ws_ml[2 * cr] - M);
      L += ws_ml[2 * cr + 1] * w;
      a += ws_acc[cr * XA_D + lane] * w;
    }
    o = a / L;
    ls = M + logf(L);
  }
  const long long E = sh.E();
  st1(out + (long long)qi * sh.B * E + (long long)b * E + h * XA_D + lane, o);
  if (lane == 0) lse[row] = ls;
}

// delta[b*H + h, q] = sum_c dO * O (fp32, fixed butterfly order): one warp per row
template <typename T>
__global__ void xattn_delta_kernel(const T* __restrict__ out, const T* __restrict__ dout, float* __restrict__ delta,
                                   XaShape sh) {
  const long long BHQ = (long long)sh.B * sh.H * sh.Q;
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= BHQ) return;
  const int bh = (int)(row / sh.Q), qi = (int)(row % sh.Q), b = bh / sh.H, h = bh % sh.H;
  const long long E = sh.E(), off = (long long)qi * sh.B * E + (long long)b * E + h * XA_D + lane;
  float x = ld1(dout + off) * ld1(out + off);
#pragma unroll
  for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  if (lane == 0) delta[row] = x;
}

// P and dS of query row `qok` against 8 keys; `lr` = lse of the row, `dr` = delta
__device__ __forceinline__ void xa_p_ds(float* p, float* ds, const float* qr, const float* dor, const float* Ks,
                                        const float* Vs, int g, unsigned blk, bool qok, float lr, float dr) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = g * 8 + i;
    const float s = xa_dot_swz(qr, Ks + c * XA_D, g);
    const float dp = xa_dot_swz(dor, Vs + c * XA_D, g);
    float pp;
    if (!qok) pp = 0.f;
    else if (lr == -INFINITY) pp = __int_as_float(0x7fffffff);   // fully blocked row: NaN, as torch
    else pp = ((blk >> i) & 1u) ? 0.f : expf(s - lr);
    p[i] = pp;
    ds[i] = pp * (dp - dr);
  }
}

// dK, dV of 64 keys of one (image, head), summed over every query in order
template <typename T>
__global__ void __launch_bounds__(XA_NT, 2) xattn_bwd_dkdv_kernel(
    const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, const uint8_t* __restrict__ mask,
    long long mstride, bool mvec, const float* __restrict__ lse, const float* __restrict__ delta,
    const T* __restrict__ dout, T* __restrict__ dk, T* __restrict__ dv, XaShape sh, float scale) {
  __shared__ __align__(16) float Ks[XA_BK * XA_D];
  __shared__ __align__(16) float Vs[XA_BK * XA_D];
  __shared__ __align__(16) float Qs[XA_BQ * XA_D];
  __shared__ __align__(16) float Ds[XA_BQ * XA_D];
  __shared__ __align__(16) float Ps[XA_BQ * XA_PS];
  __shared__ __align__(16) float Ss[XA_BQ * XA_PS];
  __shared__ float lse_s[XA_BQ], del_s[XA_BQ];
  const int t = threadIdx.x, r = t >> 3, g = t & 7, kc = t >> 2, dg = (t & 3) * 8;
  const int k0 = blockIdx.x * XA_BK, bh = blockIdx.y, b = bh / sh.H, h = bh % sh.H;
  const long long E = sh.E(), rs = (long long)sh.B * E, head = (long long)b * E + h * XA_D;
  xa_load_tile<T, true>(Ks, k + head, rs, k0, sh.S);
  xa_load_tile<T, true>(Vs, v + head, rs, k0, sh.S);
  float dka[8], dva[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) dka[i] = dva[i] = 0.f;
  for (int q0 = 0; q0 < sh.Q; q0 += XA_BQ) {
    __syncthreads();
    {   // 32 rows x 8 chunks of q (scaled) and dO: one chunk of each per thread
      const int j = t >> 3, ch = t & 7;
      const bool ok = q0 + j < sh.Q;
      const long long off = (long long)(q0 + j) * rs + head + ch * 4;
      float4 a = ok ? ld4(q + off) : make_float4(0.f, 0.f, 0.f, 0.f);
      a.x *= scale; a.y *= scale; a.z *= scale; a.w *= scale;
      xa_sts4(Qs + j * XA_D + ch * 4, a);
      xa_sts4(Ds + j * XA_D + ch * 4, ok ? ld4(dout + off) : make_float4(0.f, 0.f, 0.f, 0.f));
      if (t < XA_BQ) {
        const bool okr = q0 + t < sh.Q;
        lse_s[t] = okr ? lse[(long long)bh * sh.Q + q0 + t] : 0.f;
        del_s[t] = okr ? delta[(long long)bh * sh.Q + q0 + t] : 0.f;
      }
    }
    __syncthreads();
    const int qi = q0 + r;
    const bool qok = qi < sh.Q;
    float qr[XA_D], dor[XA_D];
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) {
      const float4 a = xa_lds4(Qs + r * XA_D + ch * 4), d = xa_lds4(Ds + r * XA_D + ch * 4);
      qr[4 * ch] = a.x; qr[4 * ch + 1] = a.y; qr[4 * ch + 2] = a.z; qr[4 * ch + 3] = a.w;
      dor[4 * ch] = d.x; dor[4 * ch + 1] = d.y; dor[4 * ch + 2] = d.z; dor[4 * ch + 3] = d.w;
    }
    const uint8_t* mrow = (mask && qok) ? mask + (long long)bh * mstride + (long long)qi * sh.S : nullptr;
    const unsigned blk = xa_blocked8(mrow, k0 + g * 8, sh.S, mvec);
    float p[8], ds[8];
    xa_p_ds(p, ds, qr, dor, Ks, Vs, g, blk, qok, lse_s[r], del_s[r]);
    xa_sts4(Ps + r * XA_PS + g * 8, make_float4(p[0], p[1], p[2], p[3]));
    xa_sts4(Ps + r * XA_PS + g * 8 + 4, make_float4(p[4], p[5], p[6], p[7]));
    xa_sts4(Ss + r * XA_PS + g * 8, make_float4(ds[0], ds[1], ds[2], ds[3]));
    xa_sts4(Ss + r * XA_PS + g * 8 + 4, make_float4(ds[4], ds[5], ds[6], ds[7]));
    __syncthreads();
    // dV[kc] += P[:, kc]^T dO, dK[kc] += dS[:, kc]^T (s q), channels dg..dg+7, rows in order
#pragma unroll 4
    for (int rr = 0; rr < XA_BQ; ++rr) {
      const float pv = Ps[rr * XA_PS + kc], sv = Ss[rr * XA_PS + kc];
      const float4 o0 = xa_lds4(Ds + rr * XA_D + dg), o1 = xa_lds4(Ds + rr * XA_D + dg + 4);
      const float4 a0 = xa_lds4(Qs + rr * XA_D + dg), a1 = xa_lds4(Qs + rr * XA_D + dg + 4);
      dva[0] = fmaf(pv, o0.x, dva[0]); dva[1] = fmaf(pv, o0.y, dva[1]);
      dva[2] = fmaf(pv, o0.z, dva[2]); dva[3] = fmaf(pv, o0.w, dva[3]);
      dva[4] = fmaf(pv, o1.x, dva[4]); dva[5] = fmaf(pv, o1.y, dva[5]);
      dva[6] = fmaf(pv, o1.z, dva[6]); dva[7] = fmaf(pv, o1.w, dva[7]);
      dka[0] = fmaf(sv, a0.x, dka[0]); dka[1] = fmaf(sv, a0.y, dka[1]);
      dka[2] = fmaf(sv, a0.z, dka[2]); dka[3] = fmaf(sv, a0.w, dka[3]);
      dka[4] = fmaf(sv, a1.x, dka[4]); dka[5] = fmaf(sv, a1.y, dka[5]);
      dka[6] = fmaf(sv, a1.z, dka[6]); dka[7] = fmaf(sv, a1.w, dka[7]);
    }
  }
  if (k0 + kc < sh.S) {
    const long long off = (long long)(k0 + kc) * rs + head + dg;
    st4(dk + off, make_float4(dka[0], dka[1], dka[2], dka[3]));
    st4(dk + off + 4, make_float4(dka[4], dka[5], dka[6], dka[7]));
    st4(dv + off, make_float4(dva[0], dva[1], dva[2], dva[3]));
    st4(dv + off + 4, make_float4(dva[4], dva[5], dva[6], dva[7]));
  }
}

// dQ partials of 32 queries over one key chunk: sum_j dS_ij k_j (without the scale), fp32
template <typename T>
__global__ void __launch_bounds__(XA_NT, 2) xattn_bwd_dq_kernel(
    const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, const uint8_t* __restrict__ mask,
    long long mstride, bool mvec, const float* __restrict__ lse, const float* __restrict__ delta,
    const T* __restrict__ dout, float* __restrict__ ws_dq, XaShape sh, int tiles_per_chunk, float scale) {
  __shared__ __align__(16) float Ks[XA_BK * XA_D];
  __shared__ __align__(16) float Vs[XA_BK * XA_D];
  __shared__ __align__(16) float Ss[XA_BQ * XA_PS];
  const int t = threadIdx.x, r = t >> 3, g = t & 7;
  const int chunk = blockIdx.y, bh = blockIdx.z, b = bh / sh.H, h = bh % sh.H;
  const int qi = blockIdx.x * XA_BQ + r;
  const bool qok = qi < sh.Q;
  const long long E = sh.E(), rs = (long long)sh.B * E, head = (long long)b * E + h * XA_D;
  float qr[XA_D], dor[XA_D];
  xa_row_regs(qr, q + (long long)qi * rs + head, qok, scale);
  xa_row_regs(dor, dout + (long long)qi * rs + head, qok, 1.f);
  const float lr = qok ? lse[(long long)bh * sh.Q + qi] : 0.f, dr = qok ? delta[(long long)bh * sh.Q + qi] : 0.f;
  const uint8_t* mrow = (mask && qok) ? mask + (long long)bh * mstride + (long long)qi * sh.S : nullptr;
  const int ntiles = (sh.S + XA_BK - 1) / XA_BK;
  const int kt0 = chunk * tiles_per_chunk, kt1 = min(kt0 + tiles_per_chunk, ntiles);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int kt = kt0; kt < kt1; ++kt) {
    const int k0 = kt * XA_BK;
    __syncthreads();
    xa_load_tile<T, true>(Ks, k + head, rs, k0, sh.S);
    xa_load_tile<T, true>(Vs, v + head, rs, k0, sh.S);
    const unsigned blk = xa_blocked8(mrow, k0 + g * 8, sh.S, mvec);
    __syncthreads();
    float p[8], ds[8];
    xa_p_ds(p, ds, qr, dor, Ks, Vs, g, blk, qok, lr, dr);
    xa_sts4(Ss + r * XA_PS + g * 8, make_float4(ds[0], ds[1], ds[2], ds[3]));
    xa_sts4(Ss + r * XA_PS + g * 8 + 4, make_float4(ds[4], ds[5], ds[6], ds[7]));
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < XA_BK; j += 4) {
      const float4 d4 = xa_lds4(Ss + r * XA_PS + j);
      const float dj[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int c = j + jj;
        const float4 x = xa_lds4(Ks + c * XA_D + ((g ^ (c >> 3)) * 4));
        acc.x = fmaf(dj[jj], x.x, acc.x);
        acc.y = fmaf(dj[jj], x.y, acc.y);
        acc.z = fmaf(dj[jj], x.z, acc.z);
        acc.w = fmaf(dj[jj], x.w, acc.w);
      }
    }
  }
  if (qok) {
    const long long row = ((long long)chunk * sh.B * sh.H + bh) * sh.Q + qi;
    xa_sts4(ws_dq + row * XA_D + g * 4, acc);
  }
}

// dq = scale * (sum of the chunk partials in chunk order), rounded once: one thread per element
template <typename T>
__global__ void xattn_dq_reduce_kernel(const float* __restrict__ ws_dq, T* __restrict__ dq, XaShape sh, int nchunk,
                                       float scale) {
  const long long BHQ = (long long)sh.B * sh.H * sh.Q;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= BHQ * XA_D) return;
  const long long row = e / XA_D;
  const int c0 = (int)(e % XA_D), bh = (int)(row / sh.Q), qi = (int)(row % sh.Q), b = bh / sh.H, h = bh % sh.H;
  float a = 0.f;
  for (int c = 0; c < nchunk; ++c) a += ws_dq[(c * BHQ + row) * XA_D + c0];
  const long long E = sh.E();
  st1(dq + (long long)qi * sh.B * E + (long long)b * E + h * XA_D + c0, a * scale);
}

// key chunks of the forward and of the dQ pass: a function of the shape only
int xa_chunks(int BH, int Q, int S, int* tiles_per_chunk) {
  const long long ctas = (long long)BH * ((Q + XA_BQ - 1) / XA_BQ);
  const int ntiles = (S + XA_BK - 1) / XA_BK;
  long long n = (XA_TARGET_CTAS + ctas - 1) / ctas;
  if (n > ntiles) n = ntiles;
  if (n < 1) n = 1;
  const int per = (int)((ntiles + n - 1) / n);
  *tiles_per_chunk = per;
  return (ntiles + per - 1) / per;
}

bool xa_shape_ok(int B, int H, int Q, int S) {
  if (B <= 0 || H <= 0 || Q <= 0 || S <= 0) return false;
  if ((long long)B * H > 65535) return false;                       // grid.y / grid.z
  if ((S + XA_BK - 1) / XA_BK > 65535) return false;
  const long long E = (long long)H * XA_D;
  return (long long)Q * B * E < (1LL << 40) && (long long)S * B * E < (1LL << 40);
}

// workspace layout (floats): acc / dq partials [nchunk, B*H, Q, 32], (m, l) [nchunk, B*H, Q, 2], delta [B*H, Q]
struct XaWs {
  float* acc;
  float* ml;
  float* delta;
};
long long xa_ws_floats(int B, int H, int Q, int S, XaWs* w, void* base) {
  int per;
  const long long n = xa_chunks(B * H, Q, S, &per), bhq = (long long)B * H * Q;
  const long long acc = n * bhq * XA_D, ml = (n * bhq * 2 + 3) / 4 * 4, delta = (bhq + 3) / 4 * 4;
  if (w) {
    float* f = static_cast<float*>(base);
    w->acc = f;
    w->ml = f + acc;
    w->delta = f + acc + ml;
  }
  return acc + ml + delta;
}

bool aligned(const void* p, int a) { return ((uintptr_t)p % a) == 0; }

template <typename T>
int xattn_forward(const void* q_v, const void* k_v, const void* v_v, const uint8_t* mask, long long mstride, void* out_v,
                  float* lse, int B, int H, int D, int Q, int S, void* ws, void* stream_v) {
  if (!q_v || !k_v || !v_v || !out_v || !lse) return ODISE_ERR_ARG;
  if (!ws) return ODISE_ERR_WORKSPACE;
  if (D != XA_D) return ODISE_ERR_UNSUPPORTED;
  if (!xa_shape_ok(B, H, Q, S) || (mask && mstride < 0)) return ODISE_ERR_ARG;
  const int va = 4 * (int)sizeof(T);
  if (!aligned(q_v, va) || !aligned(k_v, va) || !aligned(v_v, va) || !aligned(out_v, va) || !aligned(ws, 16))
    return ODISE_ERR_ALIGN;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  XaShape sh{B, H, Q, S};
  XaWs w;
  xa_ws_floats(B, H, Q, S, &w, ws);
  int per;
  const int nchunk = xa_chunks(B * H, Q, S, &per);
  const bool mvec = mask && aligned(mask, 8) && S % 8 == 0 && mstride % 8 == 0;
  const float scale = 1.f / sqrtf((float)XA_D);
  dim3 grid((Q + XA_BQ - 1) / XA_BQ, nchunk, B * H);
  xattn_fwd_kernel<T><<<grid, XA_NT, 0, stream>>>(static_cast<const T*>(q_v), static_cast<const T*>(k_v),
                                                  static_cast<const T*>(v_v), mask, mstride, mvec, w.acc, w.ml, sh, per,
                                                  scale);
  const long long rows = (long long)B * H * Q;
  xattn_combine_kernel<T><<<(unsigned)((rows * 32 + 255) / 256), 256, 0, stream>>>(w.acc, w.ml, static_cast<T*>(out_v),
                                                                                  lse, sh, nchunk);
  count_launch(2);
  return (int)cudaGetLastError();
}

template <typename T>
int xattn_backward(const void* q_v, const void* k_v, const void* v_v, const uint8_t* mask, long long mstride,
                   const void* out_v, const float* lse, const void* dout_v, void* dq_v, void* dk_v, void* dv_v, int B,
                   int H, int D, int Q, int S, void* ws, void* stream_v) {
  if (!q_v || !k_v || !v_v || !out_v || !lse || !dout_v || !dq_v || !dk_v || !dv_v) return ODISE_ERR_ARG;
  if (!ws) return ODISE_ERR_WORKSPACE;
  if (D != XA_D) return ODISE_ERR_UNSUPPORTED;
  if (!xa_shape_ok(B, H, Q, S) || (mask && mstride < 0)) return ODISE_ERR_ARG;
  const int va = 4 * (int)sizeof(T);
  if (!aligned(q_v, va) || !aligned(k_v, va) || !aligned(v_v, va) || !aligned(dout_v, va) || !aligned(dk_v, va) ||
      !aligned(dv_v, va) || !aligned(ws, 16))
    return ODISE_ERR_ALIGN;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  XaShape sh{B, H, Q, S};
  XaWs w;
  xa_ws_floats(B, H, Q, S, &w, ws);
  int per;
  const int nchunk = xa_chunks(B * H, Q, S, &per);
  const bool mvec = mask && aligned(mask, 8) && S % 8 == 0 && mstride % 8 == 0;
  const float scale = 1.f / sqrtf((float)XA_D);
  const T *q = static_cast<const T*>(q_v), *k = static_cast<const T*>(k_v), *v = static_cast<const T*>(v_v);
  const T* dout = static_cast<const T*>(dout_v);
  const long long rows = (long long)B * H * Q;
  xattn_delta_kernel<T><<<(unsigned)((rows * 32 + 255) / 256), 256, 0, stream>>>(static_cast<const T*>(out_v), dout,
                                                                                w.delta, sh);
  dim3 gkv((S + XA_BK - 1) / XA_BK, B * H);
  xattn_bwd_dkdv_kernel<T><<<gkv, XA_NT, 0, stream>>>(q, k, v, mask, mstride, mvec, lse, w.delta, dout,
                                                      static_cast<T*>(dk_v), static_cast<T*>(dv_v), sh, scale);
  dim3 gq((Q + XA_BQ - 1) / XA_BQ, nchunk, B * H);
  xattn_bwd_dq_kernel<T><<<gq, XA_NT, 0, stream>>>(q, k, v, mask, mstride, mvec, lse, w.delta, dout, w.acc, sh, per,
                                                   scale);
  xattn_dq_reduce_kernel<T><<<(unsigned)((rows * XA_D + 255) / 256), 256, 0, stream>>>(w.acc, static_cast<T*>(dq_v), sh,
                                                                                      nchunk, scale);
  count_launch(4);
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace ob

extern "C" long long odise_masked_xattn_workspace_bytes(int B, int H, int Q, int S) {
  if (!ob::xa_shape_ok(B, H, Q, S)) return 0;
  return 4 * ob::xa_ws_floats(B, H, Q, S, nullptr, nullptr);
}

#define XA_FWD(sfx, T)                                                                                                 \
  extern "C" int odise_masked_xattn_forward_##sfx(const void* q, const void* k, const void* v, const uint8_t* mask,    \
                                                  long long mask_bh_stride, void* out, float* lse, int B, int H, int D, \
                                                  int Q, int S, void* workspace, void* stream) {                       \
    return ob::xattn_forward<T>(q, k, v, mask, mask_bh_stride, out, lse, B, H, D, Q, S, workspace, stream);           \
  }
#define XA_BWD(sfx, T)                                                                                                 \
  extern "C" int odise_masked_xattn_backward_##sfx(                                                                    \
      const void* q, const void* k, const void* v, const uint8_t* mask, long long mask_bh_stride, const void* out,     \
      const float* lse, const void* grad_out, void* grad_q, void* grad_k, void* grad_v, int B, int H, int D, int Q,    \
      int S, void* workspace, void* stream) {                                                                          \
    return ob::xattn_backward<T>(q, k, v, mask, mask_bh_stride, out, lse, grad_out, grad_q, grad_k, grad_v, B, H, D,  \
                                 Q, S, workspace, stream);                                                             \
  }
XA_FWD(f32, float)
XA_FWD(f16, __half)
XA_FWD(bf16, __nv_bfloat16)
XA_BWD(f32, float)
XA_BWD(f16, __half)
XA_BWD(bf16, __nv_bfloat16)
