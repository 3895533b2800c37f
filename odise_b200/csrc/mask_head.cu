// Decoder prediction heads of Mask2Former-style training on sm_90a: the mask logits, ODISE's hard mask pooling and the
// per-head attention mask (odise.py:729-776 and :923-1015), forward and backward.
//
//   outputs_mask[b, q, p] = sum_c E[b, q, c] X[b, c, p]                        E = mask_embed [B, Q, C], X = [B, C, H*W]
//   m[b, q, p]            = sigmoid(outputs_mask as stored) > threshold         (the hard pooling mask)
//   w[b, q]               = 1 / (sum_p m + 1e-8)                                (rounded to T for 16-bit storage)
//   pooled[b, q, c]       = w[b, q] * sum_p m[b, q, p] X[b, c, p]
//
// Storage float, __half or __nv_bfloat16.  Float: every load is converted to fp32 and products are summed with FFMA.
// 16-bit: the same products run on mma.sync tensor cores with fp32 accumulation (the *_tc_kernel below).  Each output is
// rounded once.  C = 256, Q <= 256.
//
// Forward: a CTA owns 64 queries of one image and a fixed run of 64-pixel tiles (the split count depends on the shape
// only).  Per tile it stages all 256 channels of X in shared memory, computes the 64 x 64 logit tile, rounds and stores
// it, thresholds the stored values into a shared 0 / 1 tile and adds m X^T to its [64, 256] pooled partial in registers,
// while X is still on chip.  A finalize pass sums the split partials in split order and applies w.
//
// Backward: grad E = G X^T is split over pixels into fp32 partials reduced in split order; grad X = [E ; Gp o w]^T [G ; M]
// is one GEMM with K = 2Q, M recomputed from the saved outputs_mask.  No atomics: every gradient is bit-reproducible.
//
// Attention mask: one CTA per (b, q) row resizes the logits to the level (mask_resize.cuh), writes the bool row of
// every head, and writes an all-False row where every key is blocked (odise.py:683).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

#include "launch_count.h"
#include "mask_resize.cuh"
#include "odise_b200.h"
#include "storage.cuh"

namespace ob {
namespace {

constexpr int MH_C = 256;      // mask_dim
constexpr int MH_QMAX = 256;
constexpr int MH_T = 64;       // tile edge (queries / pixels / channels)
constexpr int MH_NT = 256;     // threads per CTA
constexpr int MH_XS = MH_T + 1;           // row stride of the forward's X tile (conflict-free column reads)
constexpr int MH_KC = 32;                 // k per staged chunk of the backward GEMMs
constexpr int MH_GS = MH_T + 4;           // row stride of the backward's staged tiles (float4 rows)
constexpr int MH_TARGET_CTAS = 264;       // 2 per SM on 132 SMs: the split-K counts aim at this many CTAs
constexpr size_t MH_FWD_SMEM = sizeof(float) * (MH_C * MH_T + MH_C * MH_XS + MH_T * MH_T);

template <typename T>
__device__ __forceinline__ float mh_rnd(float v) { return mr_round(v, static_cast<T*>(nullptr)); }

// hard-pool decision on a stored logit (MaskPooling: sigmoid in T, then > threshold against the fp32 scalar)
template <typename T>
__device__ __forceinline__ float mh_hard(float stored, float thr) { return mr_sigmoid<T>(stored) > thr ? 1.f : 0.f; }

__host__ __device__ inline int mh_ptiles(long long HW) { return (int)((HW + MH_T - 1) / MH_T); }

// forward split count: about one wave of one-CTA-per-SM blocks
__host__ __device__ inline int mh_fwd_splits(int B, int Q, long long HW) {
  const int qt = (Q + MH_T - 1) / MH_T;
  const int want = (132 + B * qt - 1) / (B * qt);
  const int pt = mh_ptiles(HW);
  return want < 1 ? 1 : (want > pt ? pt : want);
}

// grad E split count (pixel chunks of MH_KC)
__host__ __device__ inline int mh_bwd_splits(int B, int Q, long long HW) {
  const int tiles = B * ((Q + MH_T - 1) / MH_T) * (MH_C / MH_T);
  const int want = (MH_TARGET_CTAS + tiles - 1) / tiles;
  const int kc = (int)((HW + MH_KC - 1) / MH_KC);
  return want < 1 ? 1 : (want > kc ? kc : want);
}

template <typename T>
__global__ void __launch_bounds__(MH_NT, 1)
mh_fwd_kernel(const T* __restrict__ E, const T* __restrict__ X, T* __restrict__ om, float* __restrict__ ws_pool,
              float* __restrict__ ws_cnt, int B, int Q, long long HW, int splits, float thr) {
  extern __shared__ float smem[];
  float* Es = smem;                         // [C][64]   E^T of this query tile
  float* Xs = Es + MH_C * MH_T;             // [C][65]   X of the current pixel tile
  float* Ms = Xs + MH_C * MH_XS;            // [64][64]  hard mask of the current tile
  const int b = blockIdx.z, q0 = blockIdx.x * MH_T, s = blockIdx.y;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, warp = tid >> 5, lane = tid & 31;
  const T* Eb = E + (long long)b * Q * MH_C;
  const T* Xb = X + (long long)b * MH_C * HW;
  for (int i = tid; i < MH_T * MH_C; i += MH_NT) {
    const int q = i / MH_C, c = i % MH_C;
    Es[c * MH_T + q] = q0 + q < Q ? mr_load(Eb + (long long)(q0 + q) * MH_C + c) : 0.f;
  }
  const int pt = mh_ptiles(HW), per = (pt + splits - 1) / splits;
  const int t0 = s * per, t1 = min(pt, t0 + per);
  float pacc[8][8], cnt[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    cnt[r] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) pacc[r][j] = 0.f;
  }
  for (int t = t0; t < t1; ++t) {
    const long long p0 = (long long)t * MH_T;
    __syncthreads();   // the previous tile's Xs / Ms are consumed (and Es is written, on the first pass)
    for (int i = tid; i < MH_C * MH_T; i += MH_NT) {
      const int c = i / MH_T, p = i % MH_T;
      Xs[c * MH_XS + p] = p0 + p < HW ? mr_load(Xb + (long long)c * HW + p0 + p) : 0.f;
    }
    __syncthreads();
    // logits: thread (ty, tx) owns queries 4ty..4ty+3 and pixels tx + 16i
    float acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[j][i] = 0.f;
#pragma unroll 4
    for (int c = 0; c < MH_C; ++c) {
      const float4 e = *reinterpret_cast<const float4*>(Es + c * MH_T + 4 * ty);
      const float* xr = Xs + c * MH_XS + tx;
      const float ev[4] = {e.x, e.y, e.z, e.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float xv = xr[16 * i];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j][i] = fmaf(ev[j], xv, acc[j][i]);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int q = 4 * ty + j;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int p = tx + 16 * i;
        float m = 0.f;
        if (q0 + q < Q && p0 + p < HW) {
          const float v = mh_rnd<T>(acc[j][i]);
          st1(om + ((long long)b * Q + q0 + q) * HW + p0 + p, v);
          m = mh_hard<T>(v, thr);
        }
        Ms[q * MH_T + p] = m;
      }
    }
    __syncthreads();
    // pooling: warp owns queries 8warp..8warp+7, lane owns channels lane + 32j
#pragma unroll 2
    for (int p = 0; p < MH_T; ++p) {
      float xv[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) xv[j] = Xs[(lane + 32 * j) * MH_XS + p];
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float m = Ms[(8 * warp + r) * MH_T + p];
        cnt[r] += m;
#pragma unroll
        for (int j = 0; j < 8; ++j) pacc[r][j] = fmaf(m, xv[j], pacc[r][j]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int q = q0 + 8 * warp + r;
    if (q >= Q) continue;
    const long long row = ((long long)s * B + b) * Q + q;
#pragma unroll
    for (int j = 0; j < 8; ++j) ws_pool[row * MH_C + lane + 32 * j] = pacc[r][j];
    if (lane == 0) ws_cnt[row] = cnt[r];
  }
}

// one thread per (b, q, c): split partials summed in split order, then w = T(1 / (count + 1e-8)) (0 for an empty mask)
// and one rounding
template <typename T>
__global__ void mh_pool_finalize_kernel(const float* __restrict__ ws_pool, const float* __restrict__ ws_cnt,
                                        T* __restrict__ pooled, float* __restrict__ weights, int B, int Q,
                                        int splits) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long n = (long long)B * Q * MH_C;
  if (i >= n) return;
  const long long row = i / MH_C;
  float sum = 0.f, cnt = 0.f;
  for (int s = 0; s < splits; ++s) {
    sum += ws_pool[(long long)s * n + i];
    cnt += ws_cnt[(long long)s * B * Q + row];
  }
  // an empty mask pools nothing (the reference's operand m / denorm is 0 there); w = 0 also keeps fp16's
  // T(1 / 1e-8) = inf out of the products
  const float w = cnt > 0.f ? mh_rnd<T>(1.f / (cnt + 1e-8f)) : 0.f;
  st1(pooled + i, sum * w);
  if (i % MH_C == 0) weights[row] = w;
}

// ---------------------------------------------------------------------------------------------- backward GEMMs
// C[64 m][64 n] += sum_k A(k, m) B(k, n) over k in [k0, k1), staged MH_KC k at a time.  Loaders: float operator()(k, i)
// (zero outside the problem) and KCONTIG = true when k is the operand's contiguous index (global reads run along k).
template <class L>
__device__ __forceinline__ void mh_stage(const L& ld, int k0, int k1, float* S) {
  for (int i = threadIdx.x; i < MH_KC * MH_T; i += MH_NT) {
    int kk, ii;
    if (L::KCONTIG) { kk = i % MH_KC; ii = i / MH_KC; } else { kk = i / MH_T; ii = i % MH_T; }
    S[kk * MH_GS + ii] = k0 + kk < k1 ? ld(k0 + kk, ii) : 0.f;
  }
}

template <class LA, class LB>
__device__ __forceinline__ void mh_gemm_tile(const LA& la, const LB& lb, int k0, int k1, float (&acc)[4][4]) {
  __shared__ __align__(16) float As[MH_KC * MH_GS];
  __shared__ __align__(16) float Bs[MH_KC * MH_GS];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int kb = k0; kb < k1; kb += MH_KC) {
    __syncthreads();
    mh_stage(la, kb, k1, As);
    mh_stage(lb, kb, k1, Bs);
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < MH_KC; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(As + k * MH_GS + 4 * ty);
      const float4 bb = *reinterpret_cast<const float4*>(Bs + k * MH_GS + 4 * tx);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[j][i] = fmaf(av[j], bv[i], acc[j][i]);
    }
  }
}

// [R, HW] row-major map (G or X of one image), k = pixel: A / B of grad E
template <typename T>
struct MhRowsK {
  static constexpr bool KCONTIG = true;
  const T* base; int r0, R; long long HW;
  __device__ float operator()(int k, int i) const {
    return r0 + i < R && k < HW ? mr_load(base + (long long)(r0 + i) * HW + k) : 0.f;
  }
};

// A of grad X: k < Q -> E[k][c], else Gp[k - Q][c] * w[k - Q]
template <typename T>
struct MhEGp {
  static constexpr bool KCONTIG = false;
  const T *E, *Gp; const float* w; int Q, c0;
  __device__ float operator()(int k, int i) const {
    const int c = c0 + i;
    return k < Q ? mr_load(E + (long long)k * MH_C + c) : mr_load(Gp + (long long)(k - Q) * MH_C + c) * w[k - Q];
  }
};

// B of grad X: k < Q -> G[k][p], else the hard mask of the saved logit om[k - Q][p]
template <typename T>
struct MhGM {
  static constexpr bool KCONTIG = false;
  const T *G, *om; int Q; long long HW, p0; float thr;
  __device__ float operator()(int k, int i) const {
    const long long p = p0 + i;
    if (p >= HW) return 0.f;
    return k < Q ? mr_load(G + (long long)k * HW + p) : mh_hard<T>(mr_load(om + (long long)(k - Q) * HW + p), thr);
  }
};

// grid (C / 64, q tiles, B * splits): fp32 partials of grad E over one pixel range
template <typename T>
__global__ void __launch_bounds__(MH_NT)
mh_grad_embed_kernel(const T* __restrict__ G, const T* __restrict__ X, float* __restrict__ ws, int B, int Q,
                     long long HW, int splits) {
  const int c0 = blockIdx.x * MH_T, q0 = blockIdx.y * MH_T;
  const int b = blockIdx.z % B, s = blockIdx.z / B;
  const int kc = (int)((HW + MH_KC - 1) / MH_KC), per = (kc + splits - 1) / splits;
  const long long k0 = (long long)s * per * MH_KC, k1 = min(HW, k0 + (long long)per * MH_KC);
  float acc[4][4] = {};
  // k is a pixel index; the tile loop runs in int (HW < 2^31 is checked on the host)
  MhRowsK<T> la{G + (long long)b * Q * HW, q0, Q, HW};
  MhRowsK<T> lb{X + (long long)b * MH_C * HW, c0, MH_C, HW};
  if (k0 < k1) mh_gemm_tile(la, lb, (int)k0, (int)k1, acc);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int q = q0 + 4 * ty + j;
    if (q >= Q) continue;
    float* dst = ws + (((long long)s * B + b) * Q + q) * MH_C + c0 + 4 * tx;
    *reinterpret_cast<float4*>(dst) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
  }
}

template <typename T>
__global__ void mh_grad_embed_reduce_kernel(const float* __restrict__ ws, T* __restrict__ gE, long long n, int splits) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float sum = 0.f;
  for (int s = 0; s < splits; ++s) sum += ws[(long long)s * n + i];
  st1(gE + i, sum);
}

// grid (pixel tiles, C / 64, B)
template <typename T>
__global__ void __launch_bounds__(MH_NT)
mh_grad_features_kernel(const T* __restrict__ E, const T* __restrict__ Gp, const float* __restrict__ w,
                        const T* __restrict__ G, const T* __restrict__ om, T* __restrict__ gX, int Q, long long HW,
                        float thr) {
  const long long p0 = (long long)blockIdx.x * MH_T;
  const int c0 = blockIdx.y * MH_T, b = blockIdx.z;
  float acc[4][4] = {};
  MhEGp<T> la{E + (long long)b * Q * MH_C, Gp + (long long)b * Q * MH_C, w + (long long)b * Q, Q, c0};
  MhGM<T> lb{G + (long long)b * Q * HW, om + (long long)b * Q * HW, Q, HW, p0, thr};
  mh_gemm_tile(la, lb, 0, 2 * Q, acc);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = c0 + 4 * ty + j;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long p = p0 + 4 * tx + i;
      if (p < HW) st1(gX + ((long long)b * MH_C + c) * HW + p, acc[j][i]);
    }
  }
}

// ---------------------------------------------------------------------------------------------- 16-bit: tensor cores
// The float16 / bfloat16 paths run the same three products on mma.sync.m16n8k16 (fp32 accumulation, one rounding per
// output).  Operands are staged in shared memory as 16-bit values with k contiguous in every row ("row.col"): a warp's
// A fragment is 4 and its B fragment 2 32-bit loads per k16 step.  Rows are padded by 8 elements, so that the 8 rows a
// fragment load touches start 4 banks apart (conflict-free).
template <typename T> struct MhMma;
template <> struct MhMma<__half> {
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  static __device__ __forceinline__ __half from(float v) { return __float2half_rn(v); }
};
template <> struct MhMma<__nv_bfloat16> {
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  static __device__ __forceinline__ __nv_bfloat16 from(float v) { return __float2bfloat16_rn(v); }
};

// one k16 step of a warp's m16 x (8 NT) tile: acc[j] += A[m0.., k0..k0+15] B[n0 + 8j.., k0..]^T, A [m][lda] and
// B [n][ldb] 16-bit with k contiguous.  acc[j][0..1]: row m0 + g, columns n0 + 8j + 2t + {0, 1}; acc[j][2..3]: row
// m0 + g + 8 (g = lane / 4, t = lane % 4).
template <typename T, int NT>
__device__ __forceinline__ void mh_mma_k16(const T* As, int lda, const T* Bs, int ldb, int m0, int n0, int k0,
                                           float (&acc)[NT][4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const T* a = As + (m0 + g) * lda + k0 + 2 * t;
  uint32_t af[4];
  af[0] = *reinterpret_cast<const uint32_t*>(a);
  af[1] = *reinterpret_cast<const uint32_t*>(a + 8 * lda);
  af[2] = *reinterpret_cast<const uint32_t*>(a + 8);
  af[3] = *reinterpret_cast<const uint32_t*>(a + 8 * lda + 8);
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const T* b = Bs + (n0 + 8 * j + g) * ldb + k0 + 2 * t;
    MhMma<T>::mma(acc[j], af, *reinterpret_cast<const uint32_t*>(b), *reinterpret_cast<const uint32_t*>(b + 8));
  }
}

constexpr int MH_TC_LC = MH_C + 8;        // row length of the [*][C] tiles
constexpr int MH_TC_LT = MH_T + 8;        // row length of the [*][64] tiles
constexpr int MH_TC_LK = MH_KC + 8;       // row length of the backward's [64][32] k chunks
constexpr size_t MH_TC_FWD_SMEM = 2 * ((size_t)2 * MH_T * MH_TC_LC + (size_t)MH_C * MH_TC_LT + (size_t)MH_T * MH_TC_LT);

// forward, 16-bit: as mh_fwd_kernel, with the logit tile (K = C) and the pooling product (K = 64 pixels) on mma.sync.
// Shared: E [64 q][C], X as [64 p][C] (logit B operand) and as [C][64 p] (pooling B operand), m [64 q][64 p].
template <typename T>
__global__ void __launch_bounds__(MH_NT, 1)
mh_fwd_tc_kernel(const T* __restrict__ E, const T* __restrict__ X, T* __restrict__ om, float* __restrict__ ws_pool,
                 float* __restrict__ ws_cnt, int B, int Q, long long HW, int splits, float thr) {
  extern __shared__ __align__(16) unsigned char mh_tc_smem[];
  T* Es = reinterpret_cast<T*>(mh_tc_smem);          // [64][LC]
  T* Xpc = Es + MH_T * MH_TC_LC;                      // [64][LC]
  T* Xcp = Xpc + MH_T * MH_TC_LC;                     // [C][LT]
  T* Ms = Xcp + MH_C * MH_TC_LT;                      // [64][LT]
  const int b = blockIdx.z, q0 = blockIdx.x * MH_T, s = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;
  const T zero = MhMma<T>::from(0.f), one = MhMma<T>::from(1.f);
  const T* Eb = E + (long long)b * Q * MH_C;
  const T* Xb = X + (long long)b * MH_C * HW;
  for (int i = tid; i < MH_T * MH_C; i += MH_NT) {
    const int q = i / MH_C, c = i % MH_C;
    Es[q * MH_TC_LC + c] = q0 + q < Q ? Eb[(long long)(q0 + q) * MH_C + c] : zero;
  }
  const int pt = mh_ptiles(HW), per = (pt + splits - 1) / splits;
  const int t0 = s * per, t1 = min(pt, t0 + per);
  float pacc[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) pacc[j][0] = pacc[j][1] = pacc[j][2] = pacc[j][3] = 0.f;
  float cnt = 0.f;                                    // thread tid < 64: the count of query q0 + tid
  for (int tt = t0; tt < t1; ++tt) {
    const long long p0 = (long long)tt * MH_T;
    __syncthreads();
    for (int i = tid; i < MH_C * MH_T; i += MH_NT) {
      const int c = i / MH_T, p = i % MH_T;
      const T v = p0 + p < HW ? Xb[(long long)c * HW + p0 + p] : zero;
      Xcp[c * MH_TC_LT + p] = v;
      Xpc[p * MH_TC_LC + c] = v;
    }
    __syncthreads();
    // logits: warp (wm, wn) owns queries 16 wm.. and pixels 32 wn..
    float acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll 4
    for (int k0 = 0; k0 < MH_C; k0 += 16) mh_mma_k16<T, 4>(Es, MH_TC_LC, Xpc, MH_TC_LC, 16 * wm, 32 * wn, k0, acc);
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int q = 16 * wm + g + 8 * (e >> 1), p = 32 * wn + 8 * j + 2 * t4 + (e & 1);
        bool m = false;
        if (q0 + q < Q && p0 + p < HW) {
          const float v = mh_rnd<T>(acc[j][e]);
          st1(om + ((long long)b * Q + q0 + q) * HW + p0 + p, v);
          m = mh_hard<T>(v, thr) != 0.f;
        }
        Ms[q * MH_TC_LT + p] = m ? one : zero;
      }
    __syncthreads();
    if (tid < MH_T)
      for (int p = 0; p < MH_T; ++p) cnt += static_cast<float>(Ms[tid * MH_TC_LT + p]);   // 0 or 1, exact
    // pooling: warp (wm, wn) owns queries 16 wm.. and channels 128 wn..; K = the tile's 64 pixels
#pragma unroll
    for (int k0 = 0; k0 < MH_T; k0 += 16) mh_mma_k16<T, 16>(Ms, MH_TC_LT, Xcp, MH_TC_LT, 16 * wm, 128 * wn, k0, pacc);
  }
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int q = q0 + 16 * wm + g + 8 * (e >> 1), c = 128 * wn + 8 * j + 2 * t4 + (e & 1);
      if (q < Q) ws_pool[(((long long)s * B + b) * Q + q) * MH_C + c] = pacc[j][e];
    }
  if (tid < MH_T && q0 + tid < Q) ws_cnt[((long long)s * B + b) * Q + q0 + tid] = cnt;
}

// grad E, 16-bit: grid (C / 64, q tiles, B * splits); A = G [q][p], B = X [c][p], both pixel-contiguous in memory
template <typename T>
__global__ void __launch_bounds__(MH_NT)
mh_grad_embed_tc_kernel(const T* __restrict__ G, const T* __restrict__ X, float* __restrict__ ws, int B, int Q,
                        long long HW, int splits) {
  __shared__ __align__(16) T As[MH_T * MH_TC_LK];
  __shared__ __align__(16) T Bs[MH_T * MH_TC_LK];
  const int c0 = blockIdx.x * MH_T, q0 = blockIdx.y * MH_T;
  const int b = blockIdx.z % B, s = blockIdx.z / B;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;
  const T zero = MhMma<T>::from(0.f);
  const int kc = (int)((HW + MH_KC - 1) / MH_KC), per = (kc + splits - 1) / splits;
  const long long k0 = (long long)s * per * MH_KC, k1 = min(HW, k0 + (long long)per * MH_KC);
  const T* Gb = G + (long long)b * Q * HW;
  const T* Xb = X + (long long)b * MH_C * HW;
  float acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  for (long long kb = k0; kb < k1; kb += MH_KC) {
    __syncthreads();
    for (int i = tid; i < MH_T * MH_KC; i += MH_NT) {
      const int r = i / MH_KC, kk = i % MH_KC;
      const long long p = kb + kk;
      As[r * MH_TC_LK + kk] = q0 + r < Q && p < k1 ? Gb[(long long)(q0 + r) * HW + p] : zero;
      Bs[r * MH_TC_LK + kk] = p < k1 ? Xb[(long long)(c0 + r) * HW + p] : zero;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < MH_KC; k += 16) mh_mma_k16<T, 4>(As, MH_TC_LK, Bs, MH_TC_LK, 16 * wm, 32 * wn, k, acc);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int q = q0 + 16 * wm + g + 8 * (e >> 1), c = c0 + 32 * wn + 8 * j + 2 * t4 + (e & 1);
      if (q < Q) ws[(((long long)s * B + b) * Q + q) * MH_C + c] = acc[j][e];
    }
}

// grad X, 16-bit: grid (pixel tiles, C / 64, B); grad X = [E ; Gp]^T [G ; w o m] with K = 2Q.  The pooling operand
// w o m is the reference's bmm operand T(m / denorm) exactly (m is 0 or 1, w is already rounded to T).  Both operands
// are k-major in memory and are transposed into k-contiguous rows while staged.
template <typename T>
__global__ void __launch_bounds__(MH_NT)
mh_grad_features_tc_kernel(const T* __restrict__ E, const T* __restrict__ Gp, const float* __restrict__ w,
                           const T* __restrict__ G, const T* __restrict__ om, T* __restrict__ gX, int Q, long long HW,
                           float thr) {
  __shared__ __align__(16) T As[MH_T * MH_TC_LK];   // [c][k]
  __shared__ __align__(16) T Bs[MH_T * MH_TC_LK];   // [p][k]
  const long long p0 = (long long)blockIdx.x * MH_T;
  const int c0 = blockIdx.y * MH_T, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;
  const T zero = MhMma<T>::from(0.f);
  const T* Eb = E + (long long)b * Q * MH_C;
  const T* Gpb = Gp + (long long)b * Q * MH_C;
  const T* Gb = G + (long long)b * Q * HW;
  const T* Ob = om + (long long)b * Q * HW;
  const float* wb = w + (long long)b * Q;
  float acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  for (int kb = 0; kb < 2 * Q; kb += MH_KC) {
    __syncthreads();
    for (int i = tid; i < MH_T * MH_KC; i += MH_NT) {
      const int kk = i / MH_T, r = i % MH_T, k = kb + kk;
      T a = zero, bv = zero;
      const long long p = p0 + r;
      if (k < Q) {
        a = Eb[(long long)k * MH_C + c0 + r];
        if (p < HW) bv = Gb[(long long)k * HW + p];
      } else if (k < 2 * Q) {
        a = Gpb[(long long)(k - Q) * MH_C + c0 + r];
        if (p < HW && mh_hard<T>(mr_load(Ob + (long long)(k - Q) * HW + p), thr) != 0.f) bv = MhMma<T>::from(wb[k - Q]);
      }
      As[r * MH_TC_LK + kk] = a;
      Bs[r * MH_TC_LK + kk] = bv;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < MH_KC; k += 16) mh_mma_k16<T, 4>(As, MH_TC_LK, Bs, MH_TC_LK, 16 * wm, 32 * wn, k, acc);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c0 + 16 * wm + g + 8 * (e >> 1);
      const long long p = p0 + 32 * wn + 8 * j + 2 * t4 + (e & 1);
      if (p < HW) st1(gX + ((long long)b * MH_C + c) * HW + p, acc[j][e]);
    }
}

// ---------------------------------------------------------------------------------------------- attention mask
// one CTA per (b, q): the row of head 0 is written first (each thread re-reads only the keys it wrote), then copied to
// the other heads, all False when no key is allowed
template <typename T>
__global__ void __launch_bounds__(256)
mh_attn_mask_kernel(const T* __restrict__ om, uint8_t* __restrict__ out, int Q, int Hm, int Wm, int Hl, int Wl,
                    int heads) {
  const long long row = blockIdx.x;   // b * Q + q
  const int b = (int)(row / Q), q = (int)(row % Q);
  const T* src = om + row * (long long)Hm * Wm;
  const int HW = Hl * Wl;
  const float sy = (float)Hm / (float)Hl, sx = (float)Wm / (float)Wl;
  uint8_t* r0 = out + ((long long)b * heads * Q + q) * HW;
  int any = 0;
  for (int key = threadIdx.x; key < HW; key += blockDim.x) {
    const int oy = key / Wl, ox = key - oy * Wl;
    const bool blk = mr_blocked(src, Hm, Wm, oy, ox, sy, sx);
    r0[key] = blk;
    any |= !blk;
  }
  any = __syncthreads_or(any);
  for (int key = threadIdx.x; key < HW; key += blockDim.x) {
    const uint8_t v = any ? r0[key] : 0;
    if (!any) r0[key] = 0;
    for (int h = 1; h < heads; ++h) r0[(long long)h * Q * HW + key] = v;
  }
}

// ---------------------------------------------------------------------------------------------- host side
bool mh_shape_ok(int B, int Q, int C, int H, int W) {
  return B > 0 && B <= 65535 && Q > 0 && Q <= MH_QMAX && C == MH_C && H > 0 && W > 0 &&
         (long long)H * W < (1LL << 24);   // the per-row mask count is an exact fp32 sum
}

bool mh_aligned(const void* p, int a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

void mh_ws_split(int B, int Q, long long HW, float** pool, float** cnt, float** gE, void* ws) {
  const int sf = mh_fwd_splits(B, Q, HW);
  float* base = static_cast<float*>(ws);
  *pool = base;
  *cnt = base + (long long)sf * B * Q * MH_C;
  *gE = base;
}

long long mh_ws_bytes(int B, int Q, long long HW) {
  const long long fwd = (long long)mh_fwd_splits(B, Q, HW) * B * Q * (MH_C + 1);
  const long long bwd = (long long)mh_bwd_splits(B, Q, HW) * B * Q * MH_C;
  return 4 * (fwd > bwd ? fwd : bwd);
}

template <typename T>
int mh_forward(const void* E, const void* X, void* om, void* pooled, float* weights, int B, int Q, int C, int H, int W,
               float thr, void* ws, void* stream_v) {
  if (!E || !X || !om || !pooled || !weights) return ODISE_ERR_ARG;
  if (!ws) return ODISE_ERR_WORKSPACE;
  if (C != MH_C || Q > MH_QMAX) return ODISE_ERR_UNSUPPORTED;
  if (!mh_shape_ok(B, Q, C, H, W)) return ODISE_ERR_ARG;
  if (!mh_aligned(ws, 16)) return ODISE_ERR_ALIGN;
  // float: the FFMA kernels; 16-bit: the tensor-core kernels
  void (*kern)(const T*, const T*, T*, float*, float*, int, int, long long, int, float);
  size_t smem;
  if constexpr (std::is_same<T, float>::value) {
    kern = mh_fwd_kernel<T>;
    smem = MH_FWD_SMEM;
  } else {
    kern = mh_fwd_tc_kernel<T>;
    smem = MH_TC_FWD_SMEM;
  }
  // > 48 KB of dynamic shared memory needs an opt-in on the current device (a host-side setting, no stream work)
  const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const long long HW = (long long)H * W;
  const int splits = mh_fwd_splits(B, Q, HW);
  float *pool, *cnt, *gE;
  mh_ws_split(B, Q, HW, &pool, &cnt, &gE, ws);
  dim3 grid((Q + MH_T - 1) / MH_T, splits, B);
  kern<<<grid, MH_NT, smem, stream>>>(static_cast<const T*>(E), static_cast<const T*>(X), static_cast<T*>(om), pool,
                                      cnt, B, Q, HW, splits, thr);
  const long long n = (long long)B * Q * MH_C;
  mh_pool_finalize_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(pool, cnt, static_cast<T*>(pooled),
                                                                             weights, B, Q, splits);
  count_launch(2);
  return (int)cudaGetLastError();
}

template <typename T>
int mh_backward(const void* E, const void* X, const void* om, const float* weights, const void* G, const void* Gp,
                void* gE, void* gX, int B, int Q, int C, int H, int W, float thr, void* ws, void* stream_v) {
  if (!E || !X || !om || !weights || !G || !Gp || !gE || !gX) return ODISE_ERR_ARG;
  if (!ws) return ODISE_ERR_WORKSPACE;
  if (C != MH_C || Q > MH_QMAX) return ODISE_ERR_UNSUPPORTED;
  if (!mh_shape_ok(B, Q, C, H, W)) return ODISE_ERR_ARG;
  if (!mh_aligned(ws, 16)) return ODISE_ERR_ALIGN;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const long long HW = (long long)H * W;
  const int splits = mh_bwd_splits(B, Q, HW);
  float *pool, *cnt, *wsE;
  mh_ws_split(B, Q, HW, &pool, &cnt, &wsE, ws);
  dim3 ge(MH_C / MH_T, (Q + MH_T - 1) / MH_T, B * splits);
  if constexpr (std::is_same<T, float>::value)
    mh_grad_embed_kernel<T><<<ge, MH_NT, 0, stream>>>(static_cast<const T*>(G), static_cast<const T*>(X), wsE, B, Q,
                                                      HW, splits);
  else
    mh_grad_embed_tc_kernel<T><<<ge, MH_NT, 0, stream>>>(static_cast<const T*>(G), static_cast<const T*>(X), wsE, B, Q,
                                                         HW, splits);
  const long long n = (long long)B * Q * MH_C;
  mh_grad_embed_reduce_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(wsE, static_cast<T*>(gE), n, splits);
  dim3 gx(mh_ptiles(HW), MH_C / MH_T, B);
  if constexpr (std::is_same<T, float>::value)
    mh_grad_features_kernel<T><<<gx, MH_NT, 0, stream>>>(static_cast<const T*>(E), static_cast<const T*>(Gp), weights,
                                                         static_cast<const T*>(G), static_cast<const T*>(om),
                                                         static_cast<T*>(gX), Q, HW, thr);
  else
    mh_grad_features_tc_kernel<T><<<gx, MH_NT, 0, stream>>>(static_cast<const T*>(E), static_cast<const T*>(Gp),
                                                            weights, static_cast<const T*>(G),
                                                            static_cast<const T*>(om), static_cast<T*>(gX), Q, HW, thr);
  count_launch(3);
  return (int)cudaGetLastError();
}

template <typename T>
int mh_attn_mask(const void* om, uint8_t* out, int B, int Q, int H, int W, int h, int w, int heads, void* stream_v) {
  if (!om || !out) return ODISE_ERR_ARG;
  if (B <= 0 || Q <= 0 || H <= 0 || W <= 0 || h <= 0 || w <= 0 || heads <= 0) return ODISE_ERR_ARG;
  if ((long long)B * Q >= (1LL << 31) || (long long)h * w >= (1LL << 31) || (long long)H * W >= (1LL << 31))
    return ODISE_ERR_ARG;
  mh_attn_mask_kernel<T><<<(unsigned)(B * Q), 256, 0, reinterpret_cast<cudaStream_t>(stream_v)>>>(
      static_cast<const T*>(om), out, Q, H, W, h, w, heads);
  count_launch(1);
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace ob

extern "C" long long odise_mask_head_workspace_bytes(int B, int Q, int C, int H, int W) {
  if (!ob::mh_shape_ok(B, Q, C, H, W)) return 0;
  return ob::mh_ws_bytes(B, Q, (long long)H * W);
}

#define MH_ENTRY(sfx, T)                                                                                               \
  extern "C" int odise_mask_head_forward_##sfx(const void* mask_embed, const void* mask_features, void* outputs_mask, \
                                               void* pooled, float* weights, int B, int Q, int C, int H, int W,       \
                                               float threshold, void* workspace, void* stream) {                      \
    return ob::mh_forward<T>(mask_embed, mask_features, outputs_mask, pooled, weights, B, Q, C, H, W, threshold,      \
                             workspace, stream);                                                                       \
  }                                                                                                                    \
  extern "C" int odise_mask_head_attn_mask_##sfx(const void* outputs_mask, uint8_t* attn_mask, int B, int Q, int H,   \
                                                 int W, int h, int w, int heads, void* stream) {                      \
    return ob::mh_attn_mask<T>(outputs_mask, attn_mask, B, Q, H, W, h, w, heads, stream);                             \
  }                                                                                                                    \
  extern "C" int odise_mask_head_backward_##sfx(                                                                       \
      const void* mask_embed, const void* mask_features, const void* outputs_mask, const float* weights,              \
      const void* grad_mask, const void* grad_pooled, void* grad_embed, void* grad_features, int B, int Q, int C,     \
      int H, int W, float threshold, void* workspace, void* stream) {                                                  \
    return ob::mh_backward<T>(mask_embed, mask_features, outputs_mask, weights, grad_mask, grad_pooled, grad_embed,   \
                              grad_features, B, Q, C, H, W, threshold, workspace, stream);                            \
  }
MH_ENTRY(f32, float)
MH_ENTRY(f16, __half)
MH_ENTRY(bf16, __nv_bfloat16)
