// Attention of the SD-v1 UNet for training on sm_90a: the core of ldm's CrossAttention (oracle/ldm.py:94-117), forward
// and backward, self- and cross-attention.
//
//   out[b, i, h, :] = softmax_j( s * q[b, i, h, :] . k[b, j, h, :] ) v[b, j, h, :],  s = D^-1/2
//
// Head dims D = 40, 80 and 160 (SD-v1's 320 / 640 / 1280 channels over 8 heads), any Tq >= 1 and Tk >= 1, on the
// batch-first layouts to_q / to_k / to_v write (q and out [B, Tq, H*D], k and v [B, Tk, H*D], heads interleaved in the
// last dimension): no permute copies.  The forward saves only lse [B*H, Tq] (fp32); the backward recomputes the
// probabilities from it, so no [B*H, Tq, Tk] tensor is ever written.
//
// Tensor cores: mma.sync (m16n8k16 for 16-bit storage, m16n8k8 TF32 for float).  Every product is a 64 x 64 x D or
// 64 x D x 64 tile whose M = 16 row slices belong to one warp; wgmma's 64-row warpgroup tiles and asynchronous
// accumulators buy nothing at K = 40 and would need a second code path for the three-term float split.
//   - float16 / bfloat16: one MMA per product, fp32 accumulators.  P and dS are rounded to the storage type before they
//     enter a product, as the composed einsum / softmax / einsum path rounds them under autocast.
//   - float32: 3xTF32.  Each operand x is split into big = tf32(x) and small = tf32(x - big) and a product is
//     a_small b_big + a_big b_small + a_big b_big, leaving about 2^-22 of it (the dropped small x small term).  Each
//     k step's three MMAs start from zero and their sum is added to the fp32 accumulator with a rounding add.
// Operand tiles live in shared memory as fp32 (a 16-bit value converts exactly); fragments are packed from there.
//
// Forward: a CTA of 4 warps owns 64 queries of one (image, head) and walks every 64-key tile with an online softmax.
// Backward: delta = rowsum(dO o O) first.  dK and dV come from CTAs that own 64 keys and walk the query tiles of one
// chunk in order; when the keys alone give too few CTAs (cross-attention, Tk = 77) the queries are split into chunks
// whose count depends on the shape only, each chunk writes fp32 partials and a reduce adds them in chunk order.  dQ comes
// from CTAs that own 64 queries and walk every key tile in order.  No atomics: every gradient is bit-reproducible.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

#include "launch_count.h"
#include "odise_b200.h"
#include "storage.cuh"

namespace ob {
namespace {

constexpr int UA_BQ = 64;              // queries per tile (4 warps x 16 rows)
constexpr int UA_BK = 64;              // keys per tile
constexpr int UA_PS = UA_BK + 4;       // row stride of the P / dS tiles
// dK / dV CTAs the query chunking aims at: 4 waves of 2 CTAs per SM on 132 SMs, so that the last partial wave costs
// little (cross-attention at B = 8: 128 key-tile CTAs x 8 chunks at Tq = 4096 and 1024)
constexpr int UA_TARGET_CTAS = 1056;

// D padded to the 16-wide k step of the 16-bit MMA (columns past D are zeros), the smem row stride, and how many warp
// column groups split the D columns of the dK / dV accumulators (2 from D = 80: one warp's 16 x D dK and dV would take
// the float kernel to the register ceiling, and the 121-203 KB of shared memory hold one CTA per SM anyway, which then
// runs 8 warps instead of 4)
template <int D>
struct UaDim {
  static constexpr int DP = (D + 15) / 16 * 16;
  static constexpr int LD = DP + 4;
  static constexpr int NS = D >= 80 ? 2 : 1;
};

struct UaShape {
  int B, H, Tq, Tk;
};

// ------------------------------------------------------------------------------------------------- MMA of one warp
template <typename T>
struct UaOp;
template <>
struct UaOp<__half> {
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
  static __device__ __forceinline__ float round(float x) { return __half2float(__float2half_rn(x)); }
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
};
template <>
struct UaOp<__nv_bfloat16> {
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
  static __device__ __forceinline__ float round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
};
template <>
struct UaOp<float> {
  static __device__ __forceinline__ float round(float x) { return x; }
};

__device__ __forceinline__ uint32_t ua_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
// x = big + small, both TF32 (small carries the 13 bits big drops)
__device__ __forceinline__ void ua_split(float x, uint32_t& big, uint32_t& small) {
  big = ua_tf32(x);
  small = ua_tf32(x - __uint_as_float(big));
}
__device__ __forceinline__ void ua_mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[j] += A[0..16, 0..K) B[0..K, 8j..8j+8) for one warp, from fp32 shared memory: A(r, k) = A[r * ar + k * ak],
// B(k, n) = B[k * bk + n * bn].  acc[j][0..1]: row g, columns 8j + 2t + {0, 1}; acc[j][2..3]: row g + 8
// (g = lane / 4, t = lane % 4).  K steps in order, so a result depends on the operands only.
template <typename T, int NT, int K>
__device__ __forceinline__ void ua_mma(float (&acc)[NT][4], const float* A, int ar, int ak, const float* B, int bk,
                                       int bn) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  if constexpr (std::is_same<T, float>::value) {
    // not unrolled: the split operands of two k steps at once took the float dK / dV and dQ kernels to 232-255 registers
#pragma unroll 1
    for (int k0 = 0; k0 < K; k0 += 8) {
      uint32_t ab[4], as[4];
      ua_split(A[g * ar + (k0 + t) * ak], ab[0], as[0]);
      ua_split(A[(g + 8) * ar + (k0 + t) * ak], ab[1], as[1]);
      ua_split(A[g * ar + (k0 + t + 4) * ak], ab[2], as[2]);
      ua_split(A[(g + 8) * ar + (k0 + t + 4) * ak], ab[3], as[3]);
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        uint32_t b0, b0s, b1, b1s;
        ua_split(B[(k0 + t) * bk + (8 * j + g) * bn], b0, b0s);
        ua_split(B[(k0 + t + 4) * bk + (8 * j + g) * bn], b1, b1s);
        // the tensor cores' fp32 accumulation truncates: a chain of MMAs over thousands of keys drifts (3.5e-6 of
        // the output at Tk = 4096), so each k step's three products start from zero and are added with FADD (RN)
        float d[4] = {0.f, 0.f, 0.f, 0.f};
        ua_mma_tf32(d, as, b0, b1);
        ua_mma_tf32(d, ab, b0s, b1s);
        ua_mma_tf32(d, ab, b0, b1);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[j][e] += d[e];
      }
    }
  } else {
#pragma unroll 2
    for (int k0 = 0; k0 < K; k0 += 16) {
      const int c0 = k0 + 2 * t;
      uint32_t a[4];
      a[0] = UaOp<T>::pack(A[g * ar + c0 * ak], A[g * ar + (c0 + 1) * ak]);
      a[1] = UaOp<T>::pack(A[(g + 8) * ar + c0 * ak], A[(g + 8) * ar + (c0 + 1) * ak]);
      a[2] = UaOp<T>::pack(A[g * ar + (c0 + 8) * ak], A[g * ar + (c0 + 9) * ak]);
      a[3] = UaOp<T>::pack(A[(g + 8) * ar + (c0 + 8) * ak], A[(g + 8) * ar + (c0 + 9) * ak]);
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const float* b = B + (8 * j + g) * bn;
        UaOp<T>::mma(acc[j], a, UaOp<T>::pack(b[c0 * bk], b[(c0 + 1) * bk]),
                     UaOp<T>::pack(b[(c0 + 8) * bk], b[(c0 + 9) * bk]));
      }
    }
  }
}

template <int NT>
__device__ __forceinline__ void ua_zero(float (&acc)[NT][4]) {
#pragma unroll
  for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
}

// rows r0 .. r0 + 63 of one head (src points at row 0, rows `rs` elements apart) into a [64][LD] fp32 tile: zeros for
// rows past R and for the padding columns D .. LD
template <typename T, int D>
__device__ __forceinline__ void ua_load_tile(float* dst, const T* src, long long rs, int r0, int R) {
  constexpr int C4 = UaDim<D>::DP / 4, LD = UaDim<D>::LD;
  for (int e = threadIdx.x; e < 64 * C4; e += blockDim.x) {
    const int j = e / C4, ch = e % C4;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r0 + j < R && ch * 4 < D) x = ld4(src + (long long)(r0 + j) * rs + ch * 4);
    *reinterpret_cast<float4*>(dst + j * LD + ch * 4) = x;
  }
}

// the 4 lanes of a quad (lane bits 0-1, one accumulator row) agree bit for bit
__device__ __forceinline__ float ua_max4(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
__device__ __forceinline__ float ua_sum4(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// ------------------------------------------------------------------------------------------------------- forward
template <int D>
constexpr size_t ua_fwd_smem() {
  return 4 * ((size_t)(UA_BQ + 2 * UA_BK) * UaDim<D>::LD + (size_t)UA_BQ * UA_PS);
}

template <typename T, int D>
__global__ void __launch_bounds__(128) ua_fwd_kernel(const T* __restrict__ q, const T* __restrict__ k,
                                                     const T* __restrict__ v, T* __restrict__ out,
                                                     float* __restrict__ lse, UaShape sh, float scale) {
  constexpr int DP = UaDim<D>::DP, LD = UaDim<D>::LD, NO = D / 8, NS = UA_BK / 8;
  extern __shared__ __align__(16) float ua_smem[];
  float* Qs = ua_smem;
  float* Ks = Qs + UA_BQ * LD;
  float* Vs = Ks + UA_BK * LD;
  float* Ps = Vs + UA_BK * LD;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y, b = bh / sh.H, h = bh % sh.H, q0 = blockIdx.x * UA_BQ;
  const long long E = (long long)sh.H * D;
  const T* kb = k + (long long)b * sh.Tk * E + h * D;
  const T* vb = v + (long long)b * sh.Tk * E + h * D;
  ua_load_tile<T, D>(Qs, q + (long long)b * sh.Tq * E + h * D, E, q0, sh.Tq);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[NO][4];
  ua_zero(o);
  float* Pw = Ps + 16 * w * UA_PS;
  for (int k0 = 0; k0 < sh.Tk; k0 += UA_BK) {
    __syncthreads();
    ua_load_tile<T, D>(Ks, kb, E, k0, sh.Tk);
    ua_load_tile<T, D>(Vs, vb, E, k0, sh.Tk);
    __syncthreads();
    float s[NS][4];
    ua_zero(s);
    ua_mma<T, NS, DP>(s, Qs + 16 * w * LD, LD, 1, Ks, 1, LD);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < NS; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float x = k0 + 8 * j + 2 * t + (e & 1) < sh.Tk ? s[j][e] * scale : -INFINITY;
        s[j][e] = x;
        mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
    float alpha[2], ps[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float mn = fmaxf(m[r], ua_max4(mx[r]));     // finite: every key tile holds a key
      alpha[r] = expf(m[r] - mn);
      m[r] = mn;
    }
#pragma unroll
    for (int j = 0; j < NS; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = expf(s[j][e] - m[e >> 1]);
        ps[e >> 1] += p;
        Pw[(g + 8 * (e >> 1)) * UA_PS + 8 * j + 2 * t + (e & 1)] = UaOp<T>::round(p);
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) l[r] = l[r] * alpha[r] + ua_sum4(ps[r]);
#pragma unroll
    for (int j = 0; j < NO; ++j) {
      o[j][0] *= alpha[0]; o[j][1] *= alpha[0];
      o[j][2] *= alpha[1]; o[j][3] *= alpha[1];
    }
    __syncwarp();
    ua_mma<T, NO, UA_BK>(o, Pw, UA_PS, 1, Vs, LD, 1);
    __syncwarp();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = q0 + 16 * w + g + 8 * r;
    if (qi >= sh.Tq) continue;
    T* orow = out + ((long long)b * sh.Tq + qi) * E + h * D;
#pragma unroll
    for (int j = 0; j < NO; ++j) st2(orow + 8 * j + 2 * t, make_float2(o[j][2 * r] / l[r], o[j][2 * r + 1] / l[r]));
    if (t == 0) lse[(long long)bh * sh.Tq + qi] = m[r] + logf(l[r]);
  }
}

// ------------------------------------------------------------------------------------------------------ backward
// delta[b*H + h, i] = sum_c dO * O (fp32, channels in order): one thread per (b, i, h) row
template <typename T, int D>
__global__ void ua_delta_kernel(const T* __restrict__ out, const T* __restrict__ dout, float* __restrict__ delta,
                                UaShape sh) {
  const long long rows = (long long)sh.B * sh.Tq * sh.H;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows) return;
  const int h = (int)(e % sh.H);
  const long long bi = e / sh.H;
  const int b = (int)(bi / sh.Tq), qi = (int)(bi % sh.Tq);
  const long long off = bi * sh.H * D + h * D;
  float x = 0.f;
#pragma unroll 4
  for (int c = 0; c < D; c += 4) {
    const float4 a = ld4(dout + off + c), o = ld4(out + off + c);
    x = fmaf(a.x, o.x, x);
    x = fmaf(a.y, o.y, x);
    x = fmaf(a.z, o.z, x);
    x = fmaf(a.w, o.w, x);
  }
  delta[((long long)b * sh.H + h) * sh.Tq + qi] = x;
}

template <int D>
constexpr size_t ua_dkdv_smem() {
  return 4 * ((size_t)(2 * UA_BK + 2 * UA_BQ) * UaDim<D>::LD + (size_t)2 * UA_BQ * UA_PS + 2 * UA_BQ);
}

// dK, dV of 64 keys of one (image, head) over the query tiles of chunk blockIdx.z, in order.  ws == null: the results
// go to dk / dv; otherwise fp32 partials [chunk][B*H][Tk][D] (dK) and the same for dV after nchunk * B*H*Tk*D floats
template <typename T, int D>
__global__ void __launch_bounds__(128 * UaDim<D>::NS) ua_bwd_dkdv_kernel(
    const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, const T* __restrict__ dout,
    const float* __restrict__ lse, const float* __restrict__ delta, T* __restrict__ dk, T* __restrict__ dv,
    float* __restrict__ ws, UaShape sh, float scale, int tiles_per_chunk) {
  constexpr int DP = UaDim<D>::DP, LD = UaDim<D>::LD, NSPL = UaDim<D>::NS;
  constexpr int KW = UA_BK / NSPL, DW = D / NSPL;      // keys of a warp's P / dS slice, channels of its dK / dV slice
  extern __shared__ __align__(16) float ua_smem[];
  float* Ks = ua_smem;
  float* Vs = Ks + UA_BK * LD;
  float* Qs = Vs + UA_BK * LD;
  float* Ds = Qs + UA_BQ * LD;
  float* Ps = Ds + UA_BQ * LD;
  float* Ss = Ps + UA_BQ * UA_PS;
  float* ls = Ss + UA_BQ * UA_PS;
  float* dls = ls + UA_BQ;
  const int w = threadIdx.x >> 5, wr = w & 3, wc = w >> 2, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int k0 = blockIdx.x * UA_BK, bh = blockIdx.y, b = bh / sh.H, h = bh % sh.H, chunk = blockIdx.z;
  const long long E = (long long)sh.H * D;
  const T* qb = q + (long long)b * sh.Tq * E + h * D;
  const T* ob = dout + (long long)b * sh.Tq * E + h * D;
  ua_load_tile<T, D>(Ks, k + (long long)b * sh.Tk * E + h * D, E, k0, sh.Tk);
  ua_load_tile<T, D>(Vs, v + (long long)b * sh.Tk * E + h * D, E, k0, sh.Tk);
  float dka[DW / 8][4], dva[DW / 8][4];
  ua_zero(dka);
  ua_zero(dva);
  const int qtiles = (sh.Tq + UA_BQ - 1) / UA_BQ;
  const int qt1 = min((chunk + 1) * tiles_per_chunk, qtiles);
  for (int qt = chunk * tiles_per_chunk; qt < qt1; ++qt) {
    const int q0 = qt * UA_BQ;
    __syncthreads();
    ua_load_tile<T, D>(Qs, qb, E, q0, sh.Tq);
    ua_load_tile<T, D>(Ds, ob, E, q0, sh.Tq);
    if (threadIdx.x < UA_BQ) {
      const bool ok = q0 + threadIdx.x < sh.Tq;
      ls[threadIdx.x] = ok ? lse[(long long)bh * sh.Tq + q0 + threadIdx.x] : 0.f;
      dls[threadIdx.x] = ok ? delta[(long long)bh * sh.Tq + q0 + threadIdx.x] : 0.f;
    }
    __syncthreads();
    // P and dS of queries 16 wr .. and keys wc KW .. of the tile
    float s[KW / 8][4];
    ua_zero(s);
    ua_mma<T, KW / 8, DP>(s, Qs + 16 * wr * LD, LD, 1, Ks + wc * KW * LD, 1, LD);
#pragma unroll
    for (int j = 0; j < KW / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = 16 * wr + g + 8 * (e >> 1), col = wc * KW + 8 * j + 2 * t + (e & 1);
        const bool ok = q0 + row < sh.Tq && k0 + col < sh.Tk;
        const float p = ok ? expf(s[j][e] * scale - ls[row]) : 0.f;
        s[j][e] = p;
        Ps[row * UA_PS + col] = UaOp<T>::round(p);
      }
    float dp[KW / 8][4];
    ua_zero(dp);
    ua_mma<T, KW / 8, DP>(dp, Ds + 16 * wr * LD, LD, 1, Vs + wc * KW * LD, 1, LD);
#pragma unroll
    for (int j = 0; j < KW / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = 16 * wr + g + 8 * (e >> 1), col = wc * KW + 8 * j + 2 * t + (e & 1);
        Ss[row * UA_PS + col] = UaOp<T>::round(s[j][e] * (dp[j][e] - dls[row]) * scale);
      }
    __syncthreads();
    // dV[keys 16 wr .., channels wc DW ..] += P^T dO, dK += (s dS)^T Q, queries in order
    ua_mma<T, DW / 8, UA_BQ>(dva, Ps + 16 * wr, 1, UA_PS, Ds + wc * DW, LD, 1);
    ua_mma<T, DW / 8, UA_BQ>(dka, Ss + 16 * wr, 1, UA_PS, Qs + wc * DW, LD, 1);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = k0 + 16 * wr + g + 8 * r;
    if (key >= sh.Tk) continue;
#pragma unroll
    for (int j = 0; j < DW / 8; ++j) {
      const int c = wc * DW + 8 * j + 2 * t;
      const float2 xk = make_float2(dka[j][2 * r], dka[j][2 * r + 1]), xv = make_float2(dva[j][2 * r], dva[j][2 * r + 1]);
      if (ws) {
        const long long part = (long long)gridDim.z * sh.B * sh.H * sh.Tk * D;
        const long long o = (((long long)chunk * sh.B * sh.H + bh) * sh.Tk + key) * D + c;
        *reinterpret_cast<float2*>(ws + o) = xk;
        *reinterpret_cast<float2*>(ws + part + o) = xv;
      } else {
        const long long o = ((long long)b * sh.Tk + key) * E + h * D + c;
        st2(dk + o, xk);
        st2(dv + o, xv);
      }
    }
  }
}

// dK, dV = the chunk partials added in chunk order, rounded once: one thread per element of dk (and of dv)
template <typename T, int D>
__global__ void ua_dkdv_reduce_kernel(const float* __restrict__ ws, T* __restrict__ dk, T* __restrict__ dv, UaShape sh,
                                      int nchunk) {
  const long long E = (long long)sh.H * D, n = (long long)sh.B * sh.Tk * E;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int c = (int)(e % D), h = (int)(e / D % sh.H);
  const long long bj = e / E;
  const int b = (int)(bj / sh.Tk), key = (int)(bj % sh.Tk);
  const long long step = (long long)sh.B * sh.H * sh.Tk * D, part = nchunk * step;
  const long long o = (((long long)b * sh.H + h) * sh.Tk + key) * D + c;
  float xk = 0.f, xv = 0.f;
  for (int ch = 0; ch < nchunk; ++ch) {
    xk += ws[ch * step + o];
    xv += ws[part + ch * step + o];
  }
  st1(dk + e, xk);
  st1(dv + e, xv);
}

template <int D>
constexpr size_t ua_dq_smem() {
  return 4 * ((size_t)(2 * UA_BQ + 2 * UA_BK) * UaDim<D>::LD + (size_t)UA_BQ * UA_PS);
}

// dQ of 64 queries of one (image, head): s sum_j dS_ij k_j over every key tile in order.  (At D = 40, 2 CTAs per SM:
// the hint lets ptxas go past 128 registers, where the float instance spilled.)
template <typename T, int D>
__global__ void __launch_bounds__(128, D == 40 ? 2 : 1) ua_bwd_dq_kernel(const T* __restrict__ q, const T* __restrict__ k,
                                                        const T* __restrict__ v, const T* __restrict__ dout,
                                                        const float* __restrict__ lse, const float* __restrict__ delta,
                                                        T* __restrict__ dq, UaShape sh, float scale) {
  constexpr int DP = UaDim<D>::DP, LD = UaDim<D>::LD, NO = D / 8, NS = UA_BK / 8;
  extern __shared__ __align__(16) float ua_smem[];
  float* Qs = ua_smem;
  float* Ds = Qs + UA_BQ * LD;
  float* Ks = Ds + UA_BQ * LD;
  float* Vs = Ks + UA_BK * LD;
  float* Ss = Vs + UA_BK * LD;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y, b = bh / sh.H, h = bh % sh.H, q0 = blockIdx.x * UA_BQ;
  const long long E = (long long)sh.H * D;
  const T* kb = k + (long long)b * sh.Tk * E + h * D;
  const T* vb = v + (long long)b * sh.Tk * E + h * D;
  ua_load_tile<T, D>(Qs, q + (long long)b * sh.Tq * E + h * D, E, q0, sh.Tq);
  ua_load_tile<T, D>(Ds, dout + (long long)b * sh.Tq * E + h * D, E, q0, sh.Tq);
  float lr[2], dr[2];
  bool rok[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = q0 + 16 * w + g + 8 * r;
    rok[r] = qi < sh.Tq;
    lr[r] = rok[r] ? lse[(long long)bh * sh.Tq + qi] : 0.f;
    dr[r] = rok[r] ? delta[(long long)bh * sh.Tq + qi] : 0.f;
  }
  float dqa[NO][4];
  ua_zero(dqa);
  float* Sw = Ss + 16 * w * UA_PS;
  for (int k0 = 0; k0 < sh.Tk; k0 += UA_BK) {
    __syncthreads();
    ua_load_tile<T, D>(Ks, kb, E, k0, sh.Tk);
    ua_load_tile<T, D>(Vs, vb, E, k0, sh.Tk);
    __syncthreads();
    float s[NS][4], dp[NS][4];
    ua_zero(s);
    ua_zero(dp);
    ua_mma<T, NS, DP>(s, Qs + 16 * w * LD, LD, 1, Ks, 1, LD);
    ua_mma<T, NS, DP>(dp, Ds + 16 * w * LD, LD, 1, Vs, 1, LD);
#pragma unroll
    for (int j = 0; j < NS; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e >> 1;
        const bool ok = rok[r] && k0 + 8 * j + 2 * t + (e & 1) < sh.Tk;
        const float p = ok ? expf(s[j][e] * scale - lr[r]) : 0.f;
        Sw[(g + 8 * r) * UA_PS + 8 * j + 2 * t + (e & 1)] = UaOp<T>::round(p * (dp[j][e] - dr[r]) * scale);
      }
    __syncwarp();
    ua_mma<T, NO, UA_BK>(dqa, Sw, UA_PS, 1, Ks, LD, 1);
    __syncwarp();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!rok[r]) continue;
    T* row = dq + ((long long)b * sh.Tq + q0 + 16 * w + g + 8 * r) * E + h * D;
#pragma unroll
    for (int j = 0; j < NO; ++j) st2(row + 8 * j + 2 * t, make_float2(dqa[j][2 * r], dqa[j][2 * r + 1]));
  }
}

// ------------------------------------------------------------------------------------------------------- host side
bool ua_shape_ok(int B, int H, int Tq, int Tk) {
  if (B <= 0 || H <= 0 || Tq <= 0 || Tk <= 0) return false;
  if ((long long)B * H > 65535) return false;                        // grid.y
  return (long long)B * Tq * H * 160 < (1LL << 40) && (long long)B * Tk * H * 160 < (1LL << 40);
}
bool ua_dim_ok(int D) { return D == 40 || D == 80 || D == 160; }

// query chunks of the dK / dV pass: a function of the shape only
int ua_chunks(int B, int H, int Tq, int Tk, int* tiles_per_chunk) {
  const long long ctas = (long long)B * H * ((Tk + UA_BK - 1) / UA_BK);
  const int qtiles = (Tq + UA_BQ - 1) / UA_BQ;
  long long n = (UA_TARGET_CTAS + ctas - 1) / ctas;
  if (n > qtiles) n = qtiles;
  if (n < 1) n = 1;
  const int per = (int)((qtiles + n - 1) / n);
  *tiles_per_chunk = per;
  return (qtiles + per - 1) / per;
}

// workspace (floats): delta [B*H, Tq] (rounded up to 4), then with more than one chunk the dK and dV partials
// [2][nchunk][B*H][Tk][D]
long long ua_ws_floats(int B, int H, int D, int Tq, int Tk) {
  int per;
  const int n = ua_chunks(B, H, Tq, Tk, &per);
  const long long delta = ((long long)B * H * Tq + 3) / 4 * 4;
  return delta + (n > 1 ? 2LL * n * B * H * Tk * D : 0);
}

bool aligned(const void* p, int a) { return ((uintptr_t)p % a) == 0; }

template <typename K>
int ua_smem_optin(K kern, size_t smem) {
  // > 48 KB of dynamic shared memory needs an opt-in on the current device (a host-side setting, no stream work)
  return (int)cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

template <typename T, int D>
int ua_forward(const T* q, const T* k, const T* v, T* out, float* lse, UaShape sh, cudaStream_t stream) {
  const size_t smem = ua_fwd_smem<D>();
  if (int e = ua_smem_optin(ua_fwd_kernel<T, D>, smem)) return e;
  const float scale = (float)(1.0 / sqrt((double)D));
  dim3 grid((sh.Tq + UA_BQ - 1) / UA_BQ, sh.B * sh.H);
  ua_fwd_kernel<T, D><<<grid, 128, smem, stream>>>(q, k, v, out, lse, sh, scale);
  count_launch(1);
  return (int)cudaGetLastError();
}

template <typename T, int D>
int ua_backward(const T* q, const T* k, const T* v, const T* out, const float* lse, const T* dout, T* dq, T* dk, T* dv,
                float* ws, UaShape sh, cudaStream_t stream) {
  const size_t s_kv = ua_dkdv_smem<D>(), s_q = ua_dq_smem<D>();
  if (int e = ua_smem_optin(ua_bwd_dkdv_kernel<T, D>, s_kv)) return e;
  if (int e = ua_smem_optin(ua_bwd_dq_kernel<T, D>, s_q)) return e;
  const float scale = (float)(1.0 / sqrt((double)D));
  int per;
  const int nchunk = ua_chunks(sh.B, sh.H, sh.Tq, sh.Tk, &per);
  float* delta = ws;
  float* part = nchunk > 1 ? ws + ((long long)sh.B * sh.H * sh.Tq + 3) / 4 * 4 : nullptr;
  const long long rows = (long long)sh.B * sh.Tq * sh.H;
  ua_delta_kernel<T, D><<<(unsigned)((rows + 255) / 256), 256, 0, stream>>>(out, dout, delta, sh);
  dim3 gkv((sh.Tk + UA_BK - 1) / UA_BK, sh.B * sh.H, nchunk);
  ua_bwd_dkdv_kernel<T, D><<<gkv, 128 * UaDim<D>::NS, s_kv, stream>>>(q, k, v, dout, lse, delta, dk, dv, part, sh,
                                                                      scale, per);
  int launches = 3;
  if (part) {
    const long long n = (long long)sh.B * sh.Tk * sh.H * D;
    ua_dkdv_reduce_kernel<T, D><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(part, dk, dv, sh, nchunk);
    ++launches;
  }
  dim3 gq((sh.Tq + UA_BQ - 1) / UA_BQ, sh.B * sh.H);
  ua_bwd_dq_kernel<T, D><<<gq, 128, s_q, stream>>>(q, k, v, dout, lse, delta, dq, sh, scale);
  count_launch(launches);
  return (int)cudaGetLastError();
}

template <typename T>
int unet_attn_forward(const void* q, const void* k, const void* v, void* out, float* lse, int B, int H, int D, int Tq,
                      int Tk, void* stream_v) {
  if (!q || !k || !v || !out || !lse) return ODISE_ERR_ARG;
  if (!ua_dim_ok(D)) return ODISE_ERR_UNSUPPORTED;
  if (!ua_shape_ok(B, H, Tq, Tk)) return ODISE_ERR_ARG;
  const int va = 4 * (int)sizeof(T);
  if (!aligned(q, va) || !aligned(k, va) || !aligned(v, va) || !aligned(out, va) || !aligned(lse, 4))
    return ODISE_ERR_ALIGN;
  const UaShape sh{B, H, Tq, Tk};
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const T *qt = static_cast<const T*>(q), *kt = static_cast<const T*>(k), *vt = static_cast<const T*>(v);
  T* ot = static_cast<T*>(out);
  if (D == 40) return ua_forward<T, 40>(qt, kt, vt, ot, lse, sh, s);
  if (D == 80) return ua_forward<T, 80>(qt, kt, vt, ot, lse, sh, s);
  return ua_forward<T, 160>(qt, kt, vt, ot, lse, sh, s);
}

template <typename T>
int unet_attn_backward(const void* q, const void* k, const void* v, const void* out, const float* lse,
                       const void* dout, void* dq, void* dk, void* dv, int B, int H, int D, int Tq, int Tk, void* ws,
                       void* stream_v) {
  if (!q || !k || !v || !out || !lse || !dout || !dq || !dk || !dv) return ODISE_ERR_ARG;
  if (!ws) return ODISE_ERR_WORKSPACE;
  if (!ua_dim_ok(D)) return ODISE_ERR_UNSUPPORTED;
  if (!ua_shape_ok(B, H, Tq, Tk)) return ODISE_ERR_ARG;
  const int va = 4 * (int)sizeof(T);
  if (!aligned(q, va) || !aligned(k, va) || !aligned(v, va) || !aligned(out, va) || !aligned(dout, va) ||
      !aligned(dq, va) || !aligned(dk, va) || !aligned(dv, va) || !aligned(lse, 4) || !aligned(ws, 16))
    return ODISE_ERR_ALIGN;
  const UaShape sh{B, H, Tq, Tk};
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_v);
  const T *qt = static_cast<const T*>(q), *kt = static_cast<const T*>(k), *vt = static_cast<const T*>(v);
  const T *ot = static_cast<const T*>(out), *dot = static_cast<const T*>(dout);
  T *dqt = static_cast<T*>(dq), *dkt = static_cast<T*>(dk), *dvt = static_cast<T*>(dv);
  float* w = static_cast<float*>(ws);
  if (D == 40) return ua_backward<T, 40>(qt, kt, vt, ot, lse, dot, dqt, dkt, dvt, w, sh, s);
  if (D == 80) return ua_backward<T, 80>(qt, kt, vt, ot, lse, dot, dqt, dkt, dvt, w, sh, s);
  return ua_backward<T, 160>(qt, kt, vt, ot, lse, dot, dqt, dkt, dvt, w, sh, s);
}

}  // namespace
}  // namespace ob

extern "C" long long odise_unet_attn_workspace_bytes(int B, int H, int D, int Tq, int Tk) {
  if (!ob::ua_dim_ok(D) || !ob::ua_shape_ok(B, H, Tq, Tk)) return 0;
  return 4 * ob::ua_ws_floats(B, H, D, Tq, Tk);
}

#define UA_FWD(sfx, T)                                                                                                 \
  extern "C" int odise_unet_attn_forward_##sfx(const void* q, const void* k, const void* v, void* out, float* lse,    \
                                               int B, int H, int D, int Tq, int Tk, void* stream) {                   \
    return ob::unet_attn_forward<T>(q, k, v, out, lse, B, H, D, Tq, Tk, stream);                                      \
  }
#define UA_BWD(sfx, T)                                                                                                 \
  extern "C" int odise_unet_attn_backward_##sfx(const void* q, const void* k, const void* v, const void* out,         \
                                                const float* lse, const void* grad_out, void* grad_q, void* grad_k,   \
                                                void* grad_v, int B, int H, int D, int Tq, int Tk, void* workspace,   \
                                                void* stream) {                                                        \
    return ob::unet_attn_backward<T>(q, k, v, out, lse, grad_out, grad_q, grad_k, grad_v, B, H, D, Tq, Tk, workspace, \
                                     stream);                                                                          \
  }
UA_FWD(f32, float)
UA_FWD(f16, __half)
UA_FWD(bf16, __nv_bfloat16)
UA_BWD(f32, float)
UA_BWD(f16, __half)
UA_BWD(bf16, __nv_bfloat16)
