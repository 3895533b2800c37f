// Grounding loss of ODISE(caption) training (MaskGroundingCriterion.get_loss, odise.py:815-907) for all S prediction
// sets of a step in one set of launches, forward and deterministic backward, on sm_90a:
//
//   m^ = x / max(|x|, 1e-12) per row (F.normalize), likewise w^
//   z_iqjk = scale_s <m^_s,i,q, w^_j,k>      mask image i against word image j
//   Score(i, j) = 1/K sum_k sum_q softmax_q(z_i.jk) z_iqjk
//   A[i, b] = Score(i, o+b)   (every gathered mask image against the local words: sim_global_img_txt)
//   D[b, j] = Score(o+b, j)   (the local masks against every gathered word image: sim_img_global_txt)
//   l1 = sum_b v_b CE(A[:, b], o+b) / B,   l2 = sum_b v_b CE(D[b, :], o+b) / sum_b v_b, or, where that is not finite,
//   the unweighted mean of CE(D[b, :], o+b);   loss_s = loss_weight (l1 + l2) / 2
//
// G gathered images, B local ones at offset o (G = B, o = 0 on one rank).  A "pair" is (mask image i, word image j)
// with j local (the A pairs, i-major) or i local and j not (the rest of the D pairs); a pair with both local serves A
// and D.  Storage type T of the masks and their gradients (float, __half or __nv_bfloat16), Tw of the words (T, or float
// for float32 words under autocast); all arithmetic fp32.  In 16 bits the kernels round where torch's autocast rounds:
// m^ and w^ to T (the matmul casts its fp32 operands), the dot product (fp32 accumulation) to T, and scale to T before
// the multiply, whose product is rounded once; softmax, the sums and the cross entropies are fp32, as autocast runs them.
//
// Forward, three launches: normalise (a warp per row: m^, w^ and the clamped norms into the state), pairs (a CTA per
// (pair, set): the Q x K products, the K column softmaxes and Score), final (a CTA per set: both cross entropies, the
// fallback chosen on the device, the loss and the unit gradients dL/dA, dL/dD into the state).
// Backward, three launches, no atomics: pairs (a CTA per (pair, set) recomputes its tile and stores dScore/dp [Q, K]
// and its scale partial in the workspace), partials (a CTA per chunk of 8 word images of a mask image, or of 4
// (set, mask image) pairs of a word image: the chunk's sum into the workspace), grads (a CTA per (set, mask image) and
// per word image adds its partials in chunk order and runs the normalize backward; S more CTAs sum each set's scale
// partials in pair order).  The chunks depend on the shape only, so every gradient is bit-reproducible.
#include <stdint.h>

#include "launch_count.h"
#include "odise_b200.h"
#include "storage.cuh"

namespace ob {
namespace {

constexpr int GR_NT = 256;              // threads per CTA
constexpr int GR_W = GR_NT / 32;
constexpr int GR_MAX_Q = 256;
constexpr int GR_MAX_K = 32;
constexpr int GR_MAX_C = 768;
constexpr int GR_CPL = GR_MAX_C / 32;   // channels per lane
constexpr float GR_EPS = 1e-12f;

__device__ __forceinline__ float rt(float v, float*) { return v; }
__device__ __forceinline__ float rt(float v, __half*) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float rt(float v, __nv_bfloat16*) { return __bfloat162float(__float2bfloat16_rn(v)); }
// v rounded to T and widened back (exact); float is the identity
template <typename T>
__device__ __forceinline__ float rt(float v) { return rt(v, (T*)nullptr); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// grad of x from grad y of y = x / d, d = max(|x|, eps): (gy - x^ <gy, x^>) / d, or gy / d where the norm was clamped
__device__ __forceinline__ float normalize_grad(float gy, float xh, float dot, float d) {
  return d > GR_EPS ? __fdiv_rn(__fsub_rn(gy, __fmul_rn(xh, dot)), d) : __fdiv_rn(gy, d);
}

struct Dims {
  int S, G, B, o, Q, K, C, P;
};

// the state buffer of the forward, read by the backward (float offsets)
struct State {
  float *mh, *wh, *norms, *A, *D, *cA, *cD;
  __host__ __device__ State(float* s, const Dims& d) {
    mh = s;
    wh = mh + (long long)d.S * d.G * d.Q * d.C;
    norms = wh + (long long)d.G * d.K * d.C;
    A = norms + (long long)d.S * d.G * d.Q + (long long)d.G * d.K;
    D = A + (long long)d.S * d.G * d.B;
    cA = D + (long long)d.S * d.B * d.G;
    cD = cA + (long long)d.S * d.G * d.B;
  }
};

__device__ __forceinline__ void pair_ij(const Dims& d, int p, int& i, int& j) {
  if (p < d.G * d.B) {
    i = p / d.B;
    j = d.o + p % d.B;
  } else {
    const int r = p - d.G * d.B, n = d.G - d.B, jj = r % n;
    i = d.o + r / n;
    j = jj < d.o ? jj : jj + d.B;
  }
}

__device__ __forceinline__ int pair_of(const Dims& d, int i, int j) {
  if (j >= d.o && j < d.o + d.B) return i * d.B + (j - d.o);
  return d.G * d.B + (i - d.o) * (d.G - d.B) + (j < d.o ? j : j - d.B);
}

// normalise every gathered mask row and word row: a warp per row; m^, w^ (rounded to T) and the clamped norms
template <typename T, typename Tw>
__global__ void __launch_bounds__(GR_NT)
gr_normalize_kernel(const T* __restrict__ me, const Tw* __restrict__ we, float* __restrict__ state, Dims d) {
  State st(state, d);
  const long long rm = (long long)d.S * d.G * d.Q, rows = rm + (long long)d.G * d.K;
  const long long r = (long long)blockIdx.x * GR_W + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  float v[GR_CPL];
  float ss = 0.f;
  const int ncc = d.C / 32;
  if (r < rm) {
    const T* x = me + r * d.C;
#pragma unroll
    for (int cc = 0; cc < GR_CPL; ++cc)
      if (cc < ncc) {
        v[cc] = ld1(x + lane + 32 * cc);
        ss = __fmaf_rn(v[cc], v[cc], ss);
      }
  } else {
    const Tw* x = we + (r - rm) * d.C;
#pragma unroll
    for (int cc = 0; cc < GR_CPL; ++cc)
      if (cc < ncc) {
        v[cc] = ld1(x + lane + 32 * cc);
        ss = __fmaf_rn(v[cc], v[cc], ss);
      }
  }
  const float n = fmaxf(__fsqrt_rn(warp_sum(ss)), GR_EPS);
  float* y = (r < rm ? st.mh : st.wh - rm * d.C) + r * d.C;
#pragma unroll
  for (int cc = 0; cc < GR_CPL; ++cc)
    if (cc < ncc) y[lane + 32 * cc] = rt<T>(__fdiv_rn(v[cc], n));
  if (lane == 0) st.norms[r] = n;
}

// the rounded products p[q * K + k] = T(<m^_q, w^_k>) of one pair into shared memory: a warp per mask row, lanes over
// channels, each dot product summed by a fixed butterfly
template <typename T>
__device__ __forceinline__ void pair_products(const float* __restrict__ m, const float* __restrict__ w, float* p,
                                              const Dims& d) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, ncc = d.C / 32;
  for (int q = wid; q < d.Q; q += GR_W) {
    float mv[GR_CPL];
#pragma unroll
    for (int cc = 0; cc < GR_CPL; ++cc) mv[cc] = cc < ncc ? m[(long long)q * d.C + lane + 32 * cc] : 0.f;
    for (int k = 0; k < d.K; ++k) {
      const float* wk = w + (long long)k * d.C + lane;
      float a = 0.f;
#pragma unroll
      for (int cc = 0; cc < GR_CPL; ++cc)
        if (cc < ncc) a = __fmaf_rn(mv[cc], __ldg(wk + 32 * cc), a);
      a = warp_sum(a);
      if (lane == 0) p[q * d.K + k] = rt<T>(a);
    }
  }
}

// z of a stored product
template <typename T>
__device__ __forceinline__ float zval(float p, float sc) { return rt<T>(__fmul_rn(p, sc)); }

// per column k, in a warp: the max of z over q, sum e = sum exp(z - max) and s_k = sum e z / sum e
template <typename T>
__device__ __forceinline__ void column_softmax(const float* p, float sc, int k, const Dims& d, float& mx, float& se,
                                               float& sk) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int q = lane; q < d.Q; q += 32) m = fmaxf(m, zval<T>(p[q * d.K + k], sc));
  m = warp_max(m);
  float e = 0.f, ez = 0.f;
  for (int q = lane; q < d.Q; q += 32) {
    const float z = zval<T>(p[q * d.K + k], sc), x = expf(z - m);
    e += x;
    ez = __fmaf_rn(x, z, ez);
  }
  e = warp_sum(e);
  ez = warp_sum(ez);
  mx = m;
  se = e;
  sk = __fdiv_rn(ez, e);
}

template <typename T>
__global__ void __launch_bounds__(GR_NT)
gr_pairs_forward_kernel(const float* __restrict__ scale, float* __restrict__ state, Dims d) {
  __shared__ float p[GR_MAX_Q * GR_MAX_K];
  __shared__ float sk[GR_MAX_K];
  State st(state, d);
  const int s = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int i, j;
  pair_ij(d, blockIdx.x, i, j);
  const float sc = rt<T>(__ldg(scale + s));
  pair_products<T>(st.mh + ((long long)s * d.G + i) * d.Q * d.C, st.wh + (long long)j * d.K * d.C, p, d);
  __syncthreads();
  for (int k = wid; k < d.K; k += GR_W) {
    float mx, se, s_k;
    column_softmax<T>(p, sc, k, d, mx, se, s_k);
    if (lane == 0) sk[k] = s_k;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < d.K; ++k) t += sk[k];
    const float score = __fdiv_rn(t, (float)d.K);
    if (j >= d.o && j < d.o + d.B) st.A[((long long)s * d.G + i) * d.B + (j - d.o)] = score;
    if (i >= d.o && i < d.o + d.B) st.D[((long long)s * d.B + (i - d.o)) * d.G + j] = score;
  }
}

// log-sum-exp of n values x[t * stride] in a warp
__device__ __forceinline__ float warp_lse(const float* x, int n, int stride) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int t = lane; t < n; t += 32) m = fmaxf(m, x[(long long)t * stride]);
  m = warp_max(m);
  float e = 0.f;
  for (int t = lane; t < n; t += 32) e += expf(x[(long long)t * stride] - m);
  return m + logf(warp_sum(e));
}

// a CTA per set: both cross entropies per local image, the losses and the unit gradients dL/dA, dL/dD
__global__ void __launch_bounds__(GR_NT)
gr_final_kernel(const uint8_t* __restrict__ valid, float* __restrict__ losses, float* __restrict__ state,
                float loss_weight, Dims d) {
  __shared__ float ce1[GR_NT], ce2[GR_NT], vb[GR_NT];
  __shared__ float coef[2];
  State st(state, d);
  const int s = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* A = st.A + (long long)s * d.G * d.B;
  const float* D = st.D + (long long)s * d.B * d.G;
  float l1 = 0.f, l2w = 0.f, l2u = 0.f, vs = 0.f;
  bool fallback = false;
  // B may exceed the CTA's slots: the batch is walked in chunks of GR_NT images
  for (int b0 = 0; b0 < d.B; b0 += GR_NT) {
    const int nb = min(GR_NT, d.B - b0);
    for (int bb = wid; bb < nb; bb += GR_W) {
      const int b = b0 + bb, t = d.o + b;
      const float a = warp_lse(A + b, d.G, d.B), c = warp_lse(D + (long long)b * d.G, d.G, 1);
      bool v = false;
      for (int k = lane; k < d.K; k += 32) v |= valid[(long long)t * d.K + k] != 0;
      v = __any_sync(0xffffffffu, v);
      if (lane == 0) {
        ce1[bb] = __fsub_rn(a, A[(long long)t * d.B + b]);
        ce2[bb] = __fsub_rn(c, D[(long long)b * d.G + t]);
        vb[bb] = v ? 1.f : 0.f;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int bb = 0; bb < nb; ++bb) {
        l1 = __fmaf_rn(vb[bb], ce1[bb], l1);
        l2w = __fmaf_rn(vb[bb], ce2[bb], l2w);
        l2u += ce2[bb];
        vs += vb[bb];
      }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float a = __fdiv_rn(l1, (float)d.B), w = __fdiv_rn(l2w, vs);
    fallback = !isfinite(w);    // the reference's `if not torch.isfinite(...)`, taken on the device
    const float c = fallback ? __fdiv_rn(l2u, (float)d.B) : w;
    losses[s] = __fmul_rn(__fmul_rn(0.5f, __fadd_rn(a, c)), loss_weight);
    coef[0] = __fmul_rn(0.5f, loss_weight);
    coef[1] = fallback ? -1.f : vs;
  }
  __syncthreads();
  // dL/dA[j, b] = lw/2 v_b/B (softmax_j A[:, b] - [j = o+b]),  dL/dD[b, j] = lw/2 c_b (softmax_j D[b, :] - [j = o+b])
  const float h = coef[0], den = coef[1];
  for (int b = wid; b < d.B; b += GR_W) {
    const int t = d.o + b;
    const float a = warp_lse(A + b, d.G, d.B), c = warp_lse(D + (long long)b * d.G, d.G, 1);
    bool v = false;
    for (int k = lane; k < d.K; k += 32) v |= valid[(long long)t * d.K + k] != 0;
    v = __any_sync(0xffffffffu, v);
    const float w1 = v ? __fdiv_rn(h, (float)d.B) : 0.f;
    const float w2 = den < 0.f ? __fdiv_rn(h, (float)d.B) : (v ? __fdiv_rn(h, den) : 0.f);
    for (int j = lane; j < d.G; j += 32) {
      const float pa = expf(A[(long long)j * d.B + b] - a), pd = expf(D[(long long)b * d.G + j] - c);
      st.cA[((long long)s * d.G + j) * d.B + b] = __fmul_rn(w1, pa - (j == t ? 1.f : 0.f));
      st.cD[((long long)s * d.B + b) * d.G + j] = __fmul_rn(w2, pd - (j == t ? 1.f : 0.f));
    }
  }
}

// backward per (pair, set): dScore/dp [Q, K] = scale/K P (1 + z - s_k) and the scale partial sum dScore/dz p
template <typename T>
__global__ void __launch_bounds__(GR_NT)
gr_pairs_backward_kernel(const float* __restrict__ scale, const float* __restrict__ state, float* __restrict__ tws,
                         float* __restrict__ sws, Dims d) {
  __shared__ float p[GR_MAX_Q * GR_MAX_K];
  __shared__ float part[GR_MAX_K];
  State st(const_cast<float*>(state), d);
  const int s = blockIdx.y, pr = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int i, j;
  pair_ij(d, pr, i, j);
  const float sc = rt<T>(__ldg(scale + s)), ik = __fdiv_rn(1.f, (float)d.K);
  pair_products<T>(st.mh + ((long long)s * d.G + i) * d.Q * d.C, st.wh + (long long)j * d.K * d.C, p, d);
  __syncthreads();
  float* tw = tws + ((long long)s * d.P + pr) * d.Q * d.K;
  for (int k = wid; k < d.K; k += GR_W) {
    float mx, se, s_k;
    column_softmax<T>(p, sc, k, d, mx, se, s_k);
    float acc = 0.f;
    for (int q = lane; q < d.Q; q += 32) {
      const float pq = p[q * d.K + k], z = zval<T>(pq, sc);
      const float u = __fmul_rn(__fmul_rn(__fdiv_rn(expf(z - mx), se), __fadd_rn(1.f, __fsub_rn(z, s_k))), ik);
      tw[q * d.K + k] = __fmul_rn(u, sc);
      acc = __fmaf_rn(u, pq, acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) part[k] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < d.K; ++k) t += part[k];
    sws[(long long)s * d.P + pr] = t;
  }
}

// The backward's partner sums are split into chunks of a fixed number of partners, each chunk's sum a partial in the
// workspace, and the partials added in chunk order by the final kernel: the work spreads over many CTAs and the order
// of every sum depends on the shape only.
constexpr int GR_PM = 8;    // partners per chunk, mask side (word images)
constexpr int GR_PW = 4;    // partners per chunk, word side ((set, mask image) pairs)

struct Chunks {
  int am, dm, dw, aw;        // chunks: mask A (over local words), mask D (over all words), word D, word A
  long long pmA, pmD, pwD, pwA, end;    // float offsets of the partials in the workspace
  __host__ __device__ Chunks(const Dims& d) {
    am = (d.B + GR_PM - 1) / GR_PM;
    dm = (d.G + GR_PM - 1) / GR_PM;
    dw = (d.S * d.B + GR_PW - 1) / GR_PW;
    aw = (d.S * d.G + GR_PW - 1) / GR_PW;
    pmA = (long long)d.S * d.P * d.Q * d.K + (long long)d.S * d.P;
    pmD = pmA + (long long)d.S * d.G * am * d.Q * d.C;
    pwD = pmD + (long long)d.S * d.B * dm * d.Q * d.C;
    pwA = pwD + (long long)d.G * dw * d.K * d.C;
    end = pwA + (long long)d.B * aw * d.K * d.C;
  }
};

// the partial of one chunk of a mask image's partners: a warp per query row, lanes over channels,
// acc[c] = sum over the chunk's word images j (ascending) of g cA|cD sum_k dScore/dp[q, k] w^[j, k, c]
__device__ __forceinline__ void mask_partial(const Dims& d, const State& st, const float* __restrict__ gl,
                                             const float* __restrict__ tws, int s, int i, bool through_a, int ch,
                                             float* __restrict__ out) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, ncc = d.C / 32;
  const float g = __ldg(gl + s);
  const int n = through_a ? d.B : d.G, j0 = ch * GR_PM, j1 = min(n, j0 + GR_PM);
  for (int q = wid; q < d.Q; q += GR_W) {
    float acc[GR_CPL];
#pragma unroll
    for (int cc = 0; cc < GR_CPL; ++cc) acc[cc] = 0.f;
    for (int x = j0; x < j1; ++x) {
      const int j = through_a ? d.o + x : x;
      const float c = __fmul_rn(g, through_a ? st.cA[((long long)s * d.G + i) * d.B + x]
                                             : st.cD[((long long)s * d.B + (i - d.o)) * d.G + x]);
      const float* t = tws + ((long long)s * d.P + pair_of(d, i, j)) * d.Q * d.K + q * d.K;
      for (int k = 0; k < d.K; ++k) {
        const float u = __fmul_rn(c, t[k]);
        const float* w = st.wh + ((long long)j * d.K + k) * d.C + lane;
#pragma unroll
        for (int cc = 0; cc < GR_CPL; ++cc)
          if (cc < ncc) acc[cc] = __fmaf_rn(u, __ldg(w + 32 * cc), acc[cc]);
      }
    }
    float* y = out + (long long)q * d.C + lane;
#pragma unroll
    for (int cc = 0; cc < GR_CPL; ++cc)
      if (cc < ncc) y[32 * cc] = acc[cc];
  }
}

// the partial of one chunk of a word image's partners: a warp per word, lanes over channels,
// acc[c] = sum over the chunk's (set, mask image) pairs (ascending) of g cD|cA sum_q dScore/dp[q, k] m^[s, i, q, c]
__device__ __forceinline__ void word_partial(const Dims& d, const State& st, const float* __restrict__ gl,
                                             const float* __restrict__ tws, int j, bool through_a, int ch,
                                             float* __restrict__ out) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, ncc = d.C / 32;
  const int per = through_a ? d.G : d.B, n = d.S * per, p0 = ch * GR_PW, p1 = min(n, p0 + GR_PW);
  for (int k = wid; k < d.K; k += GR_W) {
    float acc[GR_CPL];
#pragma unroll
    for (int cc = 0; cc < GR_CPL; ++cc) acc[cc] = 0.f;
    for (int x = p0; x < p1; ++x) {
      const int s = x / per, r = x - s * per, i = through_a ? r : d.o + r;
      const float c = __fmul_rn(__ldg(gl + s), through_a ? st.cA[((long long)s * d.G + i) * d.B + (j - d.o)]
                                                         : st.cD[((long long)s * d.B + r) * d.G + j]);
      const float* t = tws + ((long long)s * d.P + pair_of(d, i, j)) * d.Q * d.K + k;
      const float* m = st.mh + ((long long)s * d.G + i) * d.Q * d.C + lane;
      for (int q = 0; q < d.Q; ++q) {
        const float u = __fmul_rn(c, t[q * d.K]);
#pragma unroll
        for (int cc = 0; cc < GR_CPL; ++cc)
          if (cc < ncc) acc[cc] = __fmaf_rn(u, __ldg(m + (long long)q * d.C + 32 * cc), acc[cc]);
      }
    }
    float* y = out + (long long)k * d.C + lane;
#pragma unroll
    for (int cc = 0; cc < GR_CPL; ++cc)
      if (cc < ncc) y[32 * cc] = acc[cc];
  }
}

// backward, second launch: a CTA per chunk of partners, in four ranges: mask images through A (every gathered mask
// image, chunks of local words), local mask images through D (chunks of all words), word images through D (chunks of
// the sets' local masks), local word images through A (chunks of the sets' gathered masks)
__global__ void __launch_bounds__(GR_NT)
gr_partials_kernel(const float* __restrict__ state, const float* __restrict__ gl, float* __restrict__ ws, Dims d) {
  State st(const_cast<float*>(state), d);
  const Chunks ck(d);
  const float* tws = ws;
  long long x = blockIdx.x;
  const long long nmA = (long long)d.S * d.G * ck.am, nmD = (long long)d.S * d.B * ck.dm;
  const long long nwD = (long long)d.G * ck.dw;
  if (x < nmA) {    // (s, i, chunk)
    const int ch = (int)(x % ck.am), si = (int)(x / ck.am);
    mask_partial(d, st, gl, tws, si / d.G, si % d.G, true, ch, ws + ck.pmA + x * d.Q * d.C);
    return;
  }
  x -= nmA;
  if (x < nmD) {    // (s, b, chunk)
    const int ch = (int)(x % ck.dm), sb = (int)(x / ck.dm);
    mask_partial(d, st, gl, tws, sb / d.B, d.o + sb % d.B, false, ch, ws + ck.pmD + x * d.Q * d.C);
    return;
  }
  x -= nmD;
  if (x < nwD) {    // (j, chunk)
    word_partial(d, st, gl, tws, (int)(x / ck.dw), false, (int)(x % ck.dw), ws + ck.pwD + x * d.K * d.C);
    return;
  }
  x -= nwD;         // (b, chunk)
  word_partial(d, st, gl, tws, d.o + (int)(x / ck.aw), true, (int)(x % ck.aw), ws + ck.pwA + x * d.K * d.C);
}

// a row's partials summed in chunk order (p: the first chunk's row, stride between chunks)
__device__ __forceinline__ void sum_chunks(const float* __restrict__ p, int n, long long stride, int ncc, int lane,
                                           float* acc) {
#pragma unroll
  for (int cc = 0; cc < GR_CPL; ++cc) acc[cc] = 0.f;
  for (int c = 0; c < n; ++c)
#pragma unroll
    for (int cc = 0; cc < GR_CPL; ++cc)
      if (cc < ncc) acc[cc] += p[c * stride + lane + 32 * cc];
}

// the normalize backward of one row of x (norm n) for the gradients ga, gb of its normalised row, stored to ya, yb
template <typename T, typename To>
__device__ __forceinline__ void row_tail(const T* __restrict__ x, float n, const float* ga, To* ya, const float* gb,
                                         To* yb, int ncc, int lane) {
  float xh[GR_CPL], da = 0.f, db = 0.f;
#pragma unroll
  for (int cc = 0; cc < GR_CPL; ++cc)
    if (cc < ncc) {
      xh[cc] = __fdiv_rn(ld1(x + lane + 32 * cc), n);
      da = __fmaf_rn(ga[cc], xh[cc], da);
      if (yb) db = __fmaf_rn(gb[cc], xh[cc], db);
    }
  da = warp_sum(da);
  db = warp_sum(db);
#pragma unroll
  for (int cc = 0; cc < GR_CPL; ++cc)
    if (cc < ncc) {
      st1(ya + lane + 32 * cc, normalize_grad(ga[cc], xh[cc], da, n));
      if (yb) st1(yb + lane + 32 * cc, normalize_grad(gb[cc], xh[cc], db, n));
    }
}

// backward, third launch: CTAs 0 .. S*G-1 a (set, mask image): its partials summed in chunk order, then the normalize
// backward, into the gathered-mask gradient (through A) and for a local image the local-mask gradient (through D);
// the next G CTAs a word image: likewise into the gathered-word gradient (through D) and for a local image the
// local-word gradient (through A); the last S CTAs each set's scale gradient, its pairs' partials in pair order
template <typename T, typename Tw>
__global__ void __launch_bounds__(GR_NT)
gr_grads_kernel(const T* __restrict__ me, const Tw* __restrict__ we, const float* __restrict__ state,
                const float* __restrict__ gl, const float* __restrict__ ws, T* __restrict__ gm_local,
                T* __restrict__ gm_global, Tw* __restrict__ gw_local, Tw* __restrict__ gw_global,
                float* __restrict__ gscale, Dims d) {
  State st(const_cast<float*>(state), d);
  const Chunks ck(d);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, ncc = d.C / 32;
  int x = blockIdx.x;
  if (x < d.S * d.G) {
    const int s = x / d.G, i = x % d.G;
    const bool local = i >= d.o && i < d.o + d.B;
    const long long row0 = ((long long)s * d.G + i) * d.Q, qc = (long long)d.Q * d.C;
    for (int q = wid; q < d.Q; q += GR_W) {
      float aa[GR_CPL], ad[GR_CPL];
      sum_chunks(ws + ck.pmA + (long long)x * ck.am * qc + (long long)q * d.C, ck.am, qc, ncc, lane, aa);
      if (local)
        sum_chunks(ws + ck.pmD + ((long long)s * d.B + (i - d.o)) * ck.dm * qc + (long long)q * d.C, ck.dm, qc, ncc,
                   lane, ad);
      T* yd = local ? gm_local + (((long long)s * d.B + (i - d.o)) * d.Q + q) * d.C : nullptr;
      row_tail(me + (row0 + q) * d.C, st.norms[row0 + q], aa, gm_global + (row0 + q) * d.C, ad, yd, ncc, lane);
    }
    return;
  }
  x -= d.S * d.G;
  if (x < d.G) {
    const int j = x;
    const bool local = j >= d.o && j < d.o + d.B;
    const long long kc = (long long)d.K * d.C;
    for (int k = wid; k < d.K; k += GR_W) {
      float ad[GR_CPL], aa[GR_CPL];
      sum_chunks(ws + ck.pwD + (long long)j * ck.dw * kc + (long long)k * d.C, ck.dw, kc, ncc, lane, ad);
      if (local)
        sum_chunks(ws + ck.pwA + (long long)(j - d.o) * ck.aw * kc + (long long)k * d.C, ck.aw, kc, ncc, lane, aa);
      const long long row = (long long)j * d.K + k;
      Tw* ya = local ? gw_local + ((long long)(j - d.o) * d.K + k) * d.C : nullptr;
      row_tail(we + row * d.C, st.norms[(long long)d.S * d.G * d.Q + row], ad, gw_global + row * d.C, aa, ya, ncc,
               lane);
    }
    return;
  }
  __shared__ float red[GR_W];
  const int s = x - d.G;
  const float* sws = ws + (long long)d.S * d.P * d.Q * d.K;
  float a = 0.f;
  for (int pr = threadIdx.x; pr < d.P; pr += GR_NT) {
    int i, j;
    pair_ij(d, pr, i, j);
    float c = 0.f;
    if (j >= d.o && j < d.o + d.B) c = st.cA[((long long)s * d.G + i) * d.B + (j - d.o)];
    if (i >= d.o && i < d.o + d.B) c = __fadd_rn(c, st.cD[((long long)s * d.B + (i - d.o)) * d.G + j]);
    a = __fmaf_rn(c, sws[(long long)s * d.P + pr], a);
  }
  a = warp_sum(a);
  if (lane == 0) red[wid] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < GR_W; ++w) t += red[w];
    gscale[s] = __fmul_rn(__ldg(gl + s), t);
  }
}

int gr_check(const Dims& d) {
  if (d.S <= 0 || d.B <= 0 || d.G < d.B || d.o < 0 || d.o > d.G - d.B || d.Q <= 0 || d.K <= 0 || d.C <= 0)
    return ODISE_ERR_ARG;
  if (d.Q > GR_MAX_Q || d.K > GR_MAX_K || d.C % 32 || d.C > GR_MAX_C ||
      (long long)d.S * d.G * d.Q * d.C >= (1LL << 31) || (long long)d.S * d.P * d.Q * d.K >= (1LL << 31) ||
      (long long)d.G * d.K * d.C >= (1LL << 31))
    return ODISE_ERR_UNSUPPORTED;
  return 0;
}

Dims gr_dims(int S, int G, int B, int o, int Q, int K, int C) {
  return Dims{S, G, B, o, Q, K, C, G * B + B * (G - B)};
}

template <typename T, typename Tw>
int gr_forward(const void* me, const void* we, const uint8_t* valid, const float* scale, float* losses, float* state,
               const Dims& d, float loss_weight, void* stream) {
  if (!me || !we || !valid || !scale || !losses || !state) return ODISE_ERR_ARG;
  if (const int rc = gr_check(d)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long rows = (long long)d.S * d.G * d.Q + (long long)d.G * d.K;
  gr_normalize_kernel<T, Tw><<<(unsigned)((rows + GR_W - 1) / GR_W), GR_NT, 0, st>>>((const T*)me, (const Tw*)we,
                                                                                     state, d);
  gr_pairs_forward_kernel<T><<<dim3(d.P, d.S), GR_NT, 0, st>>>(scale, state, d);
  gr_final_kernel<<<d.S, GR_NT, 0, st>>>(valid, losses, state, loss_weight, d);
  count_launch(3);
  return (int)cudaGetLastError();
}

template <typename T, typename Tw>
int gr_backward(const void* me, const void* we, const float* scale, const float* state, const float* grad_losses,
                void* gm_local, void* gm_global, void* gw_local, void* gw_global, float* gscale, const Dims& d,
                void* workspace, void* stream) {
  if (!me || !we || !scale || !state || !grad_losses || !gm_local || !gm_global || !gw_local || !gw_global || !gscale)
    return ODISE_ERR_ARG;
  if (const int rc = gr_check(d)) return rc;
  if (!workspace) return ODISE_ERR_WORKSPACE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* ws = (float*)workspace;
  const Chunks ck(d);
  const long long parts = (long long)d.S * d.G * ck.am + (long long)d.S * d.B * ck.dm + (long long)d.G * ck.dw +
                          (long long)d.B * ck.aw;
  gr_pairs_backward_kernel<T><<<dim3(d.P, d.S), GR_NT, 0, st>>>(scale, state, ws, ws + (long long)d.S * d.P * d.Q * d.K,
                                                               d);
  gr_partials_kernel<<<(unsigned)parts, GR_NT, 0, st>>>(state, grad_losses, ws, d);
  gr_grads_kernel<T, Tw><<<d.S * d.G + d.G + d.S, GR_NT, 0, st>>>((const T*)me, (const Tw*)we, state, grad_losses, ws,
                                                                   (T*)gm_local, (T*)gm_global, (Tw*)gw_local,
                                                                   (Tw*)gw_global, gscale, d);
  count_launch(3);
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace ob

extern "C" long long odise_grounding_workspace_bytes(int S, int G, int B, int offset, int Q, int K, int C) {
  const ob::Dims d = ob::gr_dims(S, G, B, offset, Q, K, C);
  if (ob::gr_check(d)) return 0;
  return ob::Chunks(d).end * (long long)sizeof(float);
}

#define GR_ENTRY(sfx, T)                                                                                               \
  extern "C" int odise_grounding_forward_##sfx(const void* mask_embed, const void* word_embed,                         \
                                               const uint8_t* word_valid, const float* logit_scale, float* losses,     \
                                               float* state, int S, int G, int B, int offset, int Q, int K, int C,     \
                                               float loss_weight, int words_f32, void* stream) {                       \
    auto fn = words_f32 ? ob::gr_forward<T, float> : ob::gr_forward<T, T>;                                             \
    return fn(mask_embed, word_embed, word_valid, logit_scale, losses, state, ob::gr_dims(S, G, B, offset, Q, K, C),   \
              loss_weight, stream);                                                                                    \
  }                                                                                                                    \
  extern "C" int odise_grounding_backward_##sfx(                                                                       \
      const void* mask_embed, const void* word_embed, const float* logit_scale, const float* state,                    \
      const float* grad_losses, void* grad_mask_local, void* grad_mask_global, void* grad_word_local,                  \
      void* grad_word_global, float* grad_logit_scale, int S, int G, int B, int offset, int Q, int K, int C,           \
      int words_f32, void* workspace, void* stream) {                                                                  \
    auto fn = words_f32 ? ob::gr_backward<T, float> : ob::gr_backward<T, T>;                                           \
    return fn(mask_embed, word_embed, logit_scale, state, grad_losses, grad_mask_local, grad_mask_global,              \
              grad_word_local, grad_word_global, grad_logit_scale, ob::gr_dims(S, G, B, offset, Q, K, C), workspace,   \
              stream);                                                                                                 \
  }
GR_ENTRY(f32, float)
GR_ENTRY(f16, __half)
GR_ENTRY(bf16, __nv_bfloat16)
