// Mask2Former's SetCriterion on sm_90a: the Hungarian matching costs and the point-sampled mask losses
// (third_party/Mask2Former/mask2former/modeling/matcher.py:15-156, criterion.py:21-197), forward and backward.
//
// Every sample follows detectron2's point_sample (F.grid_sample, bilinear, zeros padding, align_corners=False) at a
// point p in [0, 1)^2 with the fp32 roundings of torch's CUDA grid_sampler_2d_kernel:
//   g = 2p - 1,  ix = fma(W, g + 1, -1) * 0.5,  weights (x1 - ix)(y1 - iy), (ix - x0)(y1 - iy), (x1 - ix)(iy - y0),
//   (ix - x0)(iy - y0),  value = fma chains over the in-bounds corners in the order nw, ne, sw, se, starting from 0.
// So a sampled logit is bit-equal to grid_sample's on the float32 upcast of the map.  Target masks are read as bytes
// (a torch bool or uint8 tensor, 0 / 1) and converted exactly; predictions are float, __half or __nv_bfloat16.
//
// Cost (mc_cost_kernel, one launch per prediction set): a CTA owns 16 queries x 16 targets of one image and walks the
// image's P points in chunks of 128, sampling both sides into shared memory.  Per (q, t) it sums sigma(x) t and x t,
// per q sigma(x) and softplus(x), per t the label, chunk by chunk, and writes
//   C = w_mask (sum softplus(x) - sum x t) / P - w_class prob[q, label_t] + w_dice (1 - (2 sum sigma t + 1) /
//       (sum sigma + sum t + 1)),
// the reference's sigmoid cross entropy (softplus(-x) t + softplus(x) (1 - t) = softplus(x) - x t) and dice cost.
//
// Loss forward (mc_loss_fwd_kernel, one CTA per matched pair): the S = int(P * oversample) candidate logits go to shared
// memory; a 4-pass radix select on the bits of |x| finds the k = int(importance * P) smallest (most uncertain), exact
// ties taken by lowest candidate index; the k selected candidates (in index order) and the P - k random points are
// sampled against the target and the pair's sums (BCE, sigma t, sigma, t) are reduced in a fixed order.  The P loss
// points (selected candidates, then random points) and the sums are the saved state.  mc_loss_final_kernel reduces over pairs in a fixed order.
//
// Backward (mc_loss_bwd_kernel, one CTA per (image, query)): writes every element of grad pred_masks.  The per-point
// gradients of a matched query are summed into the map with the bilinear corner weights in int64 fixed point in shared
// memory (scale 2^(62 - e), P * max|g| < 2^e, computed in the CTA): integer sums do not depend on the order of the
// atomics, so the gradient is bit-reproducible without any switch.
//
// Assignment (mc_assign_kernel, one warp per (set, image) problem): scipy.optimize.linear_sum_assignment's shortest
// augmenting path (scipy/optimize/rectangular_lsap), step for step and in the same fp64 arithmetic, so the matched pairs
// are scipy's for every input, ties included.  A [Q, T] block with T < Q is solved transposed (rows = targets), as
// scipy does.  The sequential column scan's choice (the smallest reduced cost; among equal ones the last unassigned
// column in `remaining` order, else the first) is the warp-wide minimum of the key (cost, rank) with rank = MAX - 1 - it
// for an unassigned column and MAX + it for an assigned one.  Every update is an add or a subtract in scipy's operand
// order: nothing can be contracted into an FMA.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdint.h>

#include "launch_count.h"
#include "odise_b200.h"
#include "storage.cuh"

namespace ob {

// A target mask byte (bool or uint8, 0 / 1) as 0.f / 1.f, one more overload of storage.cuh's ld1.  It is declared in ob
// itself: declared inside the anonymous namespace, it would hide the header's overloads from the kernels below.
__device__ __forceinline__ float ld1(const uint8_t* p) { return __ldg(p) ? 1.f : 0.f; }

namespace {

constexpr int MC_TQ = 16;            // queries per cost CTA
constexpr int MC_TT = 16;            // targets per cost CTA
constexpr int MC_CH = 128;           // points per cost chunk
constexpr int MC_NT = 512;           // threads of the loss kernels
constexpr int MC_SMEM_MAX = 227 * 1024;

// bilinear corners of point (px, py) on an H x W map, as grid_sampler_2d_kernel computes them
struct McCorners {
  int x0, y0;
  float w[4];   // nw, ne, sw, se
};

__device__ __forceinline__ McCorners mc_corners(float px, float py, int H, int W) {
  const float gx = __fadd_rn(__fmul_rn(2.f, px), -1.f), gy = __fadd_rn(__fmul_rn(2.f, py), -1.f);
  const float ix = __fmul_rn(__fmaf_rn((float)W, __fadd_rn(gx, 1.f), -1.f), 0.5f);
  const float iy = __fmul_rn(__fmaf_rn((float)H, __fadd_rn(gy, 1.f), -1.f), 0.5f);
  McCorners c;
  c.x0 = (int)floorf(ix);
  c.y0 = (int)floorf(iy);
  const float e = __fsub_rn((float)(c.x0 + 1), ix), wx = __fsub_rn(ix, (float)c.x0);
  const float s = __fsub_rn((float)(c.y0 + 1), iy), n = __fsub_rn(iy, (float)c.y0);
  c.w[0] = __fmul_rn(e, s);
  c.w[1] = __fmul_rn(wx, s);
  c.w[2] = __fmul_rn(e, n);
  c.w[3] = __fmul_rn(wx, n);
  return c;
}

__device__ __forceinline__ bool mc_in(int y, int x, int H, int W) { return y >= 0 && y < H && x >= 0 && x < W; }

template <typename T>
__device__ __forceinline__ float mc_sample(const T* map, int H, int W, float px, float py) {
  const McCorners c = mc_corners(px, py, H, W);
  float acc = 0.f;
  if (mc_in(c.y0, c.x0, H, W)) acc = __fmaf_rn(c.w[0], ld1(map + (long long)c.y0 * W + c.x0), acc);
  if (mc_in(c.y0, c.x0 + 1, H, W)) acc = __fmaf_rn(c.w[1], ld1(map + (long long)c.y0 * W + c.x0 + 1), acc);
  if (mc_in(c.y0 + 1, c.x0, H, W)) acc = __fmaf_rn(c.w[2], ld1(map + (long long)(c.y0 + 1) * W + c.x0), acc);
  if (mc_in(c.y0 + 1, c.x0 + 1, H, W)) acc = __fmaf_rn(c.w[3], ld1(map + (long long)(c.y0 + 1) * W + c.x0 + 1), acc);
  return acc;
}

__device__ __forceinline__ float mc_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float mc_softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

// ---------------------------------------------------------------------------------------------------------------------
// matching cost

struct McCounts {
  int n[ODISE_MASK_MAX_IMAGES];     // targets of image b
  int off[ODISE_MASK_MAX_IMAGES];   // first target of image b in the [sum T, Hg, Wg] byte masks
};

template <typename T>
__global__ void __launch_bounds__(MC_TQ * MC_TT) mc_cost_kernel(const T* __restrict__ pred, const float* __restrict__ prob,
                                                               const long long* __restrict__ labels,
                                                               const uint8_t* __restrict__ tgt,
                                                               const float* __restrict__ pts, McCounts cnt,
                                                               float* __restrict__ cost, int Q, int H, int W, int K1,
                                                               int Hg, int Wg, int Tmax, int P, float wc, float wm,
                                                               float wd) {
  const int b = blockIdx.z, q0 = blockIdx.x * MC_TQ, t0 = blockIdx.y * MC_TT;
  const int T_b = cnt.n[b];
  if (t0 >= T_b) return;
  __shared__ float sx[MC_TQ][MC_CH + 1], ss[MC_TQ][MC_CH + 1], sp[MC_TQ][MC_CH + 1], st[MC_TT][MC_CH + 1];
  const int tid = threadIdx.x, qi = tid / MC_TT, ti = tid % MC_TT;
  const long long HW = (long long)H * W, HWg = (long long)Hg * Wg;
  const float* pb = pts + (long long)b * P * 2;
  float a_st = 0.f, a_xt = 0.f, a_s = 0.f, a_sp = 0.f, a_t = 0.f;
  for (int p0 = 0; p0 < P; p0 += MC_CH) {
    for (int e = tid; e < MC_TQ * MC_CH; e += MC_TQ * MC_TT) {
      const int r = e / MC_CH, c = e % MC_CH, p = p0 + c;
      float x = 0.f, s = 0.f, f = 0.f, t = 0.f;
      if (p < P) {
        const float px = __ldg(pb + 2 * p), py = __ldg(pb + 2 * p + 1);
        if (q0 + r < Q) {
          x = mc_sample(pred + ((long long)b * Q + q0 + r) * HW, H, W, px, py);
          s = mc_sigmoid(x);
          f = mc_softplus(x);
        }
        if (t0 + r < T_b) t = mc_sample(tgt + (long long)(cnt.off[b] + t0 + r) * HWg, Hg, Wg, px, py);
      }
      sx[r][c] = x;
      ss[r][c] = s;
      sp[r][c] = f;
      st[r][c] = t;
    }
    __syncthreads();
    float c_st = 0.f, c_xt = 0.f, c_s = 0.f, c_sp = 0.f, c_t = 0.f;
#pragma unroll 4
    for (int c = 0; c < MC_CH; ++c) {
      const float t = st[ti][c];
      c_st = fmaf(ss[qi][c], t, c_st);
      c_xt = fmaf(sx[qi][c], t, c_xt);
      c_s += ss[qi][c];
      c_sp += sp[qi][c];
      c_t += t;
    }
    a_st += c_st;
    a_xt += c_xt;
    a_s += c_s;
    a_sp += c_sp;
    a_t += c_t;
    __syncthreads();
  }
  const int q = q0 + qi, t = t0 + ti;
  if (q < Q && t < T_b) {
    const float ce = (a_sp - a_xt) / (float)P;
    const float dice = 1.f - (2.f * a_st + 1.f) / (a_s + a_t + 1.f);
    const long long lab = __ldg(labels + cnt.off[b] + t);   // a label outside [0, K1) gives a NaN cost
    const float pr = (lab >= 0 && lab < K1) ? __ldg(prob + ((long long)b * Q + q) * K1 + lab) : NAN;
    cost[((long long)b * Q + q) * Tmax + t] = wm * ce - wc * pr + wd * dice;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// point selection and mask losses

// exclusive block scan of v over MC_NT threads; *total gets the sum (all threads).  scratch: 32 ints.
__device__ __forceinline__ int mc_block_scan(int v, int* scratch, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) scratch[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int w = lane < MC_NT / 32 ? scratch[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < MC_NT / 32) scratch[lane] = w;   // inclusive warp totals
  }
  __syncthreads();
  const int before = (wid ? scratch[wid - 1] : 0) + x - v;
  *total = scratch[MC_NT / 32 - 1];
  __syncthreads();
  return before;
}

// fixed-order block sum of 4 floats over MC_NT threads; the result is valid in thread 0
__device__ __forceinline__ float4 mc_block_sum4(float4 v, float4* scratch) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
    v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    v.z += __shfl_xor_sync(0xffffffffu, v.z, o);
    v.w += __shfl_xor_sync(0xffffffffu, v.w, o);
  }
  if (lane == 0) scratch[wid] = v;
  __syncthreads();
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if (threadIdx.x == 0) {
    for (int i = 0; i < MC_NT / 32; ++i) {
      r.x += scratch[i].x;
      r.y += scratch[i].y;
      r.z += scratch[i].z;
      r.w += scratch[i].w;
    }
  }
  return r;
}

// the uncertainty order key: the bits of |x| (smaller = more uncertain)
__device__ __forceinline__ unsigned mc_key(float x) { return __float_as_uint(x) & 0x7fffffffu; }

// BCE-with-logits, sigma t, sigma and t of one point, added to a
__device__ __forceinline__ void mc_point_terms(float x, float t, float4& a) {
  const float s = mc_sigmoid(x);
  a.x += (1.f - t) * x + mc_softplus(-x);
  a.y = fmaf(s, t, a.y);
  a.z += s;
  a.w += t;
}

template <typename T>
__global__ void __launch_bounds__(MC_NT) mc_loss_fwd_kernel(const T* __restrict__ pred, const uint8_t* __restrict__ tgt,
                                                           const long long* __restrict__ pairs,
                                                           const float* __restrict__ cand, const float* __restrict__ rnd,
                                                           float* __restrict__ coords, float* __restrict__ sums, int Q, int H,
                                                           int W, int Hg, int Wg, int P, int S, int k) {
  extern __shared__ float sx[];            // S candidate logits
  __shared__ unsigned hist[256];
  __shared__ int scan_scratch[32];
  __shared__ float4 red[MC_NT / 32];
  __shared__ int s_digit, s_rem;
  const int n = blockIdx.x, tid = threadIdx.x;
  const long long b = __ldg(pairs + 3 * n), q = __ldg(pairs + 3 * n + 1), tg = __ldg(pairs + 3 * n + 2);
  const T* map = pred + (b * Q + q) * H * W;
  const uint8_t* tm = tgt + tg * Hg * Wg;
  const float* cn = cand + (long long)n * S * 2;
  for (int i = tid; i < S; i += MC_NT) sx[i] = mc_sample(map, H, W, __ldg(cn + 2 * i), __ldg(cn + 2 * i + 1));
  __syncthreads();

  // radix select: the key of the k-th smallest |x| (thr) and how many candidates with exactly that key to take (need)
  unsigned thr = 0, msk = 0;
  int need = k;
  if (k > 0) {
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = tid; i < 256; i += MC_NT) hist[i] = 0;
      __syncthreads();
      for (int i = tid; i < S; i += MC_NT) {
        const unsigned key = mc_key(sx[i]);
        if ((key & msk) == thr) atomicAdd(&hist[(key >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        int c = 0, d = 0;
        for (; d < 255; ++d) {
          if (c + (int)hist[d] >= need) break;
          c += hist[d];
        }
        s_digit = d;
        s_rem = need - c;
      }
      __syncthreads();
      thr |= (unsigned)s_digit << shift;
      msk |= 255u << shift;
      need = s_rem;
      __syncthreads();
    }
  }

  // the selected candidates in index order: position = #(key < thr before i) + min(#(key == thr before i), need)
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int lt_base = 0, eq_base = 0;
  if (k > 0) {
    for (int c0 = 0; c0 < S; c0 += MC_NT) {
      const int i = c0 + tid;
      const unsigned key = i < S ? mc_key(sx[i]) : 0xffffffffu;
      const int lt = (i < S && key < thr) ? 1 : 0, eq = (i < S && key == thr) ? 1 : 0;
      int tot;
      const int pre = mc_block_scan(lt | (eq << 16), scan_scratch, &tot);
      const int lt_pre = lt_base + (pre & 0xffff), eq_pre = eq_base + (pre >> 16);
      if (lt || (eq && eq_pre < need)) {
        const float px = __ldg(cn + 2 * i), py = __ldg(cn + 2 * i + 1);
        float* dst = coords + ((long long)n * P + lt_pre + min(eq_pre, need)) * 2;
        dst[0] = px;
        dst[1] = py;
        const float t = mc_sample(tm, Hg, Wg, px, py);
        mc_point_terms(sx[i], t, acc);
      }
      lt_base += tot & 0xffff;
      eq_base += tot >> 16;
    }
  }
  const int R = P - k;
  const float* rn = rnd + (long long)n * R * 2;
  for (int j = tid; j < R; j += MC_NT) {
    const float px = __ldg(rn + 2 * j), py = __ldg(rn + 2 * j + 1);
    float* dst = coords + ((long long)n * P + k + j) * 2;
    dst[0] = px;
    dst[1] = py;
    mc_point_terms(mc_sample(map, H, W, px, py), mc_sample(tm, Hg, Wg, px, py), acc);
  }
  const float4 r = mc_block_sum4(acc, red);
  if (tid == 0) reinterpret_cast<float4*>(sums)[n] = r;
}

// loss_mask = sum_n (BCE_n / P) / num_masks, loss_dice = sum_n dice_n / num_masks; one warp, fixed order
__global__ void mc_loss_final_kernel(const float* __restrict__ sums, int N, int P, float num_masks,
                                     float* __restrict__ losses) {
  const int lane = threadIdx.x;
  float m = 0.f, d = 0.f;
  for (int n = lane; n < N; n += 32) {
    const float4 s = reinterpret_cast<const float4*>(sums)[n];
    m += s.x / (float)P;
    d += 1.f - (2.f * s.y + 1.f) / (s.z + s.w + 1.f);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    m += __shfl_xor_sync(0xffffffffu, m, o);
    d += __shfl_xor_sync(0xffffffffu, d, o);
  }
  if (lane == 0) {
    losses[0] = m / num_masks;
    losses[1] = d / num_masks;
  }
}

template <typename T>
__global__ void __launch_bounds__(MC_NT) mc_loss_bwd_kernel(const T* __restrict__ pred, const uint8_t* __restrict__ tgt,
                                                           const long long* __restrict__ pairs,
                                                           const long long* __restrict__ pair_of,
                                                           const float* __restrict__ coords,
                                                           const float* __restrict__ sums,
                                                           const float* __restrict__ grad_losses, T* __restrict__ grad,
                                                           int H, int W, int Hg, int Wg, int P, float num_masks,
                                                           int tile_rows) {
  extern __shared__ __align__(16) unsigned char mc_smem[];
  float* gp = reinterpret_cast<float*>(mc_smem);                                    // P per-point gradients
  long long* acc = reinterpret_cast<long long*>(mc_smem + ((P * 4 + 15) / 16) * 16);  // tile_rows x W cells
  __shared__ float red[MC_NT / 32];
  const long long bq = blockIdx.x, HW = (long long)H * W;
  T* out = grad + bq * HW;
  const long long n = __ldg(pair_of + bq);
  const int tid = threadIdx.x;
  if (n < 0) {
    for (long long i = tid; i < HW; i += MC_NT) st1d(out + i, 0.0);
    return;
  }
  const T* map = pred + bq * HW;
  const uint8_t* tm = tgt + __ldg(pairs + 3 * n + 2) * Hg * Wg;
  const float* pc = coords + n * P * 2;
  const float go_m = __ldg(grad_losses), go_d = __ldg(grad_losses + 1);
  const float4 sm = reinterpret_cast<const float4*>(sums)[n];
  const float D = sm.z + sm.w + 1.f, num = 2.f * sm.y + 1.f;
  const float cm = go_m / ((float)P * num_masks), cd = go_d / (num_masks * D * D);
  float gmax = 0.f;
  for (int j = tid; j < P; j += MC_NT) {
    const float2 p = reinterpret_cast<const float2*>(pc)[j];
    const float x = mc_sample(map, H, W, p.x, p.y), t = mc_sample(tm, Hg, Wg, p.x, p.y);
    const float s = mc_sigmoid(x);
    // d dice / d sigma = -(2 t D - (2 sum sigma t + 1)) / D^2
    const float g = cm * (s - t) + cd * (num - 2.f * t * D) * s * (1.f - s);
    gp[j] = g;
    gmax = fmaxf(gmax, fabsf(g));   // NaN is dropped here and caught below
    if (!(fabsf(g) <= 3.0e38f)) gmax = INFINITY;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) gmax = fmaxf(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
  if ((tid & 31) == 0) red[tid >> 5] = gmax;
  __syncthreads();
  gmax = 0.f;
  for (int i = 0; i < MC_NT / 32; ++i) gmax = fmaxf(gmax, red[i]);
  if (gmax == 0.f || !(gmax <= 3.0e38f)) {
    const double fill = gmax == 0.f ? 0.0 : (double)NAN;
    for (long long i = tid; i < HW; i += MC_NT) st1d(out + i, fill);
    return;
  }
  // every cell sums at most P contributions of |w g| <= gmax: below 2^e, so below 2^62 after scaling by 2^(62 - e)
  int e;
  frexp((double)P * gmax, &e);
  const double scale = ldexp(1.0, 62 - e), unscale = ldexp(1.0, e - 62);
  for (int r0 = 0; r0 < H; r0 += tile_rows) {
    const int rows = min(tile_rows, H - r0), cells = rows * W;
    for (int i = tid; i < cells; i += MC_NT) acc[i] = 0;
    __syncthreads();
    for (int j = tid; j < P; j += MC_NT) {
      const float2 p = reinterpret_cast<const float2*>(pc)[j];
      const McCorners c = mc_corners(p.x, p.y, H, W);
      const float g = gp[j];
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const int y = c.y0 + (m >> 1), x = c.x0 + (m & 1);
        if (y >= r0 && y < r0 + rows && x >= 0 && x < W) {
          const long long v = __double2ll_rn((double)__fmul_rn(c.w[m], g) * scale);
          atomicAdd(reinterpret_cast<unsigned long long*>(acc + (y - r0) * W + x), (unsigned long long)v);
        }
      }
    }
    __syncthreads();
    for (int i = tid; i < cells; i += MC_NT) st1d(out + (long long)r0 * W + i, (double)acc[i] * unscale);
    __syncthreads();
  }
}

// out[n, p] = point_sample(maps[n], points[n, p])
template <typename T>
__global__ void mc_point_sample_kernel(const T* __restrict__ maps, const float* __restrict__ pts, float* __restrict__ out,
                                       long long total, int P, int H, int W) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  out[e] = mc_sample(maps + (e / P) * H * W, H, W, __ldg(pts + 2 * e), __ldg(pts + 2 * e + 1));
}

// ---------------------------------------------------------------------------------------------------------------------
// assignment

constexpr int MA_MAX = ODISE_MASK_MAX_ASSIGN;
constexpr int MA_STAGE_SMEM = 64 * 1024;   // the cost block is staged in shared memory when the CTA stays below this

// shared bytes of the solver's state for max(Q, T) <= M (M a multiple of 8, so every array stays 16-byte aligned):
// u, v, spc fp64, path, row4col, col4row, remaining int16, SR, SC bytes
__host__ __device__ __forceinline__ int ma_state_bytes(int M) { return M * (3 * 8 + 4 * 2 + 2); }

__global__ void __launch_bounds__(32) mc_assign_kernel(const float* __restrict__ cost, McCounts cnt,
                                                       long long* __restrict__ tables, int* __restrict__ status, int B,
                                                       int Q, int Tmax, int M, int N, int staged) {
  extern __shared__ __align__(16) unsigned char ma_smem[];
  double* u = reinterpret_cast<double*>(ma_smem);
  double* v = u + M;
  double* spc = v + M;
  short* path = reinterpret_cast<short*>(spc + M);
  short* row4col = path + M;
  short* col4row = row4col + M;
  short* rem = col4row + M;
  unsigned char* SR = reinterpret_cast<unsigned char*>(rem + M);
  unsigned char* SC = SR + M;
  float* stage = reinterpret_cast<float*>(ma_smem + ma_state_bytes(M));
  const int l = blockIdx.x / B, b = blockIdx.x % B, lane = threadIdx.x;
  const int T = cnt.n[b];
  const bool tr = T < Q;
  const int nr = tr ? T : Q, nc = tr ? Q : T;
  const float* blk = cost + ((long long)l * B + b) * Q * Tmax;

  // scipy's "invalid numeric entries" test (NaN or -inf anywhere), while the block is staged as [nr, nc]
  bool bad = false;
  for (int e = lane; e < Q * T; e += 32) {
    const int q = e / T, t = e % T;
    const float x = __ldg(blk + (long long)q * Tmax + t);
    bad |= x != x || x == -INFINITY;
    if (staged) stage[tr ? t * nc + q : q * nc + t] = x;
  }
  // c(i, j) = c[i * si + j * sj]
  const float* c = staged ? stage : blk;
  const long long si = staged ? nc : (tr ? 1 : Tmax), sj = staged ? 1 : (tr ? Tmax : 1);
  int st = __any_sync(0xffffffffu, bad) ? 1 : 0;
  for (int j = lane; j < nc; j += 32) {
    v[j] = 0.0;
    row4col[j] = -1;
  }
  for (int i = lane; i < nr; i += 32) {
    u[i] = 0.0;
    col4row[i] = -1;
  }
  __syncwarp();

  for (int cur = 0; cur < nr && st == 0; ++cur) {
    for (int j = lane; j < nc; j += 32) {
      spc[j] = INFINITY;
      SC[j] = 0;
      rem[j] = (short)(nc - 1 - j);
    }
    for (int i = lane; i < nr; i += 32) SR[i] = 0;
    __syncwarp();
    int i = cur, nrem = nc, sink = -1;
    double minVal = 0.0;
    while (sink < 0) {
      if (lane == 0) SR[i] = 1;
      const double ui = u[i];
      const float* ci = c + i * si;
      double bv = INFINITY;
      int bk = 2 * MA_MAX;
      for (int it = lane; it < nrem; it += 32) {
        const int j = rem[it];
        const double r = minVal + (double)ci[j * sj] - ui - v[j];
        double s = spc[j];
        if (r < s) {
          path[j] = (short)i;
          spc[j] = r;
          s = r;
        }
        const int k = row4col[j] < 0 ? MA_MAX - 1 - it : MA_MAX + it;
        if (s < bv || (s == bv && k < bk)) {
          bv = s;
          bk = k;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (ov < bv || (ov == bv && ok < bk)) {
          bv = ov;
          bk = ok;
        }
      }
      if (bv == INFINITY) {   // scipy's "cost matrix is infeasible"
        st = 2;
        break;
      }
      minVal = bv;
      const int idx = bk < MA_MAX ? MA_MAX - 1 - bk : bk - MA_MAX;
      const int j = rem[idx], owner = row4col[j];
      __syncwarp();
      if (lane == 0) {
        SC[j] = 1;
        rem[idx] = rem[nrem - 1];
      }
      --nrem;
      if (owner < 0) sink = j;
      else i = owner;
      __syncwarp();
    }
    if (st) break;
    if (lane == 0) u[cur] += minVal;
    for (int r = lane; r < nr; r += 32)
      if (SR[r] && r != cur) u[r] += minVal - spc[col4row[r]];
    for (int j = lane; j < nc; j += 32)
      if (SC[j]) v[j] -= minVal - spc[j];
    __syncwarp();
    if (lane == 0) {
      for (int j = sink;;) {
        const int r = path[j];
        row4col[j] = (short)r;
        const int nj = col4row[r];
        col4row[r] = (short)j;
        j = nj;
        if (r == cur) break;
      }
    }
    __syncwarp();
  }

  // the set's tables: pairs [N, 3], pair_of [B*Q], tg_of [B*Q]; pairs by image, then by query ascending.  A problem
  // that failed gets query r <-> target r for r < min(Q, T), in range for the loss kernels.
  long long* pairs = tables + (long long)l * (3ll * N + 2ll * B * Q);
  long long* pair_of = pairs + 3ll * N + (long long)b * Q;
  long long* tg_of = pair_of + (long long)B * Q;
  int n0 = 0;
  for (int k = 0; k < b; ++k) n0 += min(Q, cnt.n[k]);
  const long long toff = cnt.off[b];
  for (int q0 = 0; q0 < Q; q0 += 32) {
    const int q = q0 + lane;
    int t = -1;
    if (q < Q) t = st ? (q < min(Q, T) ? q : -1) : tr ? row4col[q] : col4row[q];
    const unsigned hit = __ballot_sync(0xffffffffu, t >= 0);
    const long long n = n0 + __popc(hit & ((1u << lane) - 1u));
    if (q < Q) {
      pair_of[q] = t >= 0 ? n : -1;
      tg_of[q] = t >= 0 ? toff + t : -1;
      if (t >= 0) {
        pairs[3 * n] = b;
        pairs[3 * n + 1] = q;
        pairs[3 * n + 2] = toff + t;
      }
    }
    n0 += __popc(hit);
  }
  if (lane == 0) status[(long long)l * B + b] = st;
}

// ---------------------------------------------------------------------------------------------------------------------
// host side

int mc_check_maps(int B, int Q, int H, int W, int Hg, int Wg) {
  if (B <= 0 || Q <= 0 || H <= 0 || W <= 0 || Hg <= 0 || Wg <= 0) return ODISE_ERR_ARG;
  if ((long long)H * W >= (1ll << 31) || (long long)Hg * Wg >= (1ll << 31)) return ODISE_ERR_UNSUPPORTED;
  // the fixed-point corner math takes map sizes exactly in fp32
  if (H > (1 << 24) || W > (1 << 24) || Hg > (1 << 24) || Wg > (1 << 24)) return ODISE_ERR_UNSUPPORTED;
  return ODISE_OK;
}

template <typename T>
int mc_cost(const void* pred, const float* prob, const long long* labels, const uint8_t* tgt, const float* points,
            const int* tgt_counts, float* cost, int B, int Q, int H, int W, int K1, int Hg, int Wg, int Tmax, int P,
            float wc, float wm, float wd, void* stream) {
  if (!pred || !prob || !points || !tgt_counts || !cost || K1 <= 0 || Tmax < 0 || P <= 0) return ODISE_ERR_ARG;
  if (int rc = mc_check_maps(B, Q, H, W, Hg, Wg)) return rc;
  if (B > ODISE_MASK_MAX_IMAGES) return ODISE_ERR_UNSUPPORTED;
  McCounts cnt;
  int off = 0;
  for (int b = 0; b < B; ++b) {
    if (tgt_counts[b] < 0 || tgt_counts[b] > Tmax) return ODISE_ERR_ARG;
    cnt.n[b] = tgt_counts[b];
    cnt.off[b] = off;
    off += tgt_counts[b];
  }
  if (Tmax == 0 || off == 0) return ODISE_OK;
  if (!labels || !tgt) return ODISE_ERR_ARG;
  const dim3 grid((Q + MC_TQ - 1) / MC_TQ, (Tmax + MC_TT - 1) / MC_TT, B);
  if (grid.x > 65535 || grid.y > 65535) return ODISE_ERR_UNSUPPORTED;
  mc_cost_kernel<T><<<grid, MC_TQ * MC_TT, 0, (cudaStream_t)stream>>>(
      static_cast<const T*>(pred), prob, labels, tgt, points, cnt, cost, Q, H, W, K1, Hg, Wg, Tmax, P, wc, wm, wd);
  count_launch(1);
  return (int)cudaGetLastError();
}

int mc_check_loss(int B, int Q, int H, int W, int Hg, int Wg, int N, int P, int S, int k, float num_masks) {
  if (int rc = mc_check_maps(B, Q, H, W, Hg, Wg)) return rc;
  if (N < 0 || P <= 0 || k < 0 || k > P || k > S || S < 0 || !(num_masks > 0.f)) return ODISE_ERR_ARG;
  if (S > ODISE_MASK_MAX_CANDIDATES || P > ODISE_MASK_MAX_POINTS) return ODISE_ERR_UNSUPPORTED;
  return ODISE_OK;
}

int mc_fwd_smem(int S) { return S * 4; }

template <typename T>
int mc_loss_forward(const void* pred, const uint8_t* tgt, const long long* pairs, const float* cand, const float* rnd,
                    void* ws, float* losses, int B, int Q, int H, int W, int Hg, int Wg, int N, int P, int S, int k,
                    float num_masks, void* stream) {
  if (!losses) return ODISE_ERR_ARG;
  if (int rc = mc_check_loss(B, Q, H, W, Hg, Wg, N, P, S, k, num_masks)) return rc;
  if (N > 0 && (!pred || !tgt || !pairs || (S > 0 && !cand) || (P > k && !rnd))) return ODISE_ERR_ARG;
  if (N > 0 && !ws) return ODISE_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(ws) % 16) return ODISE_ERR_ALIGN;
  cudaStream_t st = (cudaStream_t)stream;
  float* sums = static_cast<float*>(ws);
  float* coords = reinterpret_cast<float*>(static_cast<char*>(ws) + (long long)N * 16);
  if (N > 0) {
    const int smem = mc_fwd_smem(S);
    cudaError_t e = cudaFuncSetAttribute(mc_loss_fwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         mc_fwd_smem(ODISE_MASK_MAX_CANDIDATES));
    if (e != cudaSuccess) return (int)e;
    mc_loss_fwd_kernel<T><<<N, MC_NT, smem, st>>>(static_cast<const T*>(pred), tgt, pairs, cand, rnd, coords, sums, Q, H,
                                                  W, Hg, Wg, P, S, k);
    count_launch(1);
  }
  mc_loss_final_kernel<<<1, 32, 0, st>>>(sums, N, P, num_masks, losses);
  count_launch(1);
  return (int)cudaGetLastError();
}

template <typename T>
int mc_loss_backward(const void* pred, const uint8_t* tgt, const long long* pairs, const long long* pair_of,
                     const void* ws, const float* grad_losses, void* grad_pred, int B, int Q, int H, int W, int Hg,
                     int Wg, int N, int P, float num_masks, void* stream) {
  if (!pred || !pair_of || !grad_losses || !grad_pred) return ODISE_ERR_ARG;
  if (int rc = mc_check_loss(B, Q, H, W, Hg, Wg, N, P, 0, 0, num_masks)) return rc;
  if (N > 0 && (!tgt || !pairs)) return ODISE_ERR_ARG;
  if (N > 0 && !ws) return ODISE_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(ws) % 16) return ODISE_ERR_ALIGN;
  const int gp_bytes = ((P * 4 + 15) / 16) * 16;
  const int cells = (MC_SMEM_MAX - 1024 - gp_bytes) / 8;
  int tile_rows = cells / W;
  if (tile_rows < 1) return ODISE_ERR_UNSUPPORTED;
  if (tile_rows > H) tile_rows = H;
  const int smem = gp_bytes + tile_rows * W * 8;
  cudaError_t e = cudaFuncSetAttribute(mc_loss_bwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       MC_SMEM_MAX - 1024);
  if (e != cudaSuccess) return (int)e;
  const float* sums = static_cast<const float*>(ws);
  const float* coords = reinterpret_cast<const float*>(static_cast<const char*>(ws) + (long long)N * 16);
  mc_loss_bwd_kernel<T><<<B * Q, MC_NT, smem, (cudaStream_t)stream>>>(
      static_cast<const T*>(pred), tgt, pairs, pair_of, coords, sums, grad_losses, static_cast<T*>(grad_pred), H, W,
      Hg, Wg, P, num_masks, tile_rows);
  count_launch(1);
  return (int)cudaGetLastError();
}

template <typename T>
int mc_point_sample(const void* maps, const float* points, float* out, int N, int H, int W, int P, void* stream) {
  if (!maps || !points || !out || N <= 0 || P <= 0) return ODISE_ERR_ARG;
  if (int rc = mc_check_maps(1, 1, H, W, 1, 1)) return rc;
  const long long total = (long long)N * P;
  if ((total + 255) / 256 > 0x7fffffffll) return ODISE_ERR_UNSUPPORTED;
  mc_point_sample_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      static_cast<const T*>(maps), points, out, total, P, H, W);
  count_launch(1);
  return (int)cudaGetLastError();
}

int mc_assign(const float* cost, const int* tgt_counts, long long* tables, int* status, int L, int B, int Q, int Tmax,
              void* stream) {
  if (!tgt_counts || !tables || !status || L <= 0 || B <= 0 || Q <= 0 || Tmax < 0 || (!cost && Tmax > 0))
    return ODISE_ERR_ARG;
  if (B > ODISE_MASK_MAX_IMAGES || Q > MA_MAX || Tmax > MA_MAX) return ODISE_ERR_UNSUPPORTED;
  if ((long long)L * B > 0x7fffffffll) return ODISE_ERR_UNSUPPORTED;
  McCounts cnt;
  int off = 0, N = 0;
  for (int b = 0; b < B; ++b) {
    if (tgt_counts[b] < 0 || tgt_counts[b] > Tmax) return ODISE_ERR_ARG;
    cnt.n[b] = tgt_counts[b];
    cnt.off[b] = off;
    off += tgt_counts[b];
    N += min(Q, tgt_counts[b]);
  }
  const int M = (max(Q, Tmax) + 7) / 8 * 8;
  int smem = ma_state_bytes(M);
  const int staged = smem + Q * Tmax * 4 <= MA_STAGE_SMEM;
  if (staged) smem += Q * Tmax * 4;
  cudaError_t e = cudaFuncSetAttribute(mc_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  mc_assign_kernel<<<L * B, 32, smem, (cudaStream_t)stream>>>(cost, cnt, tables, status, B, Q, Tmax, M, N, staged);
  count_launch(1);
  return (int)cudaGetLastError();
}

}  // namespace
}  // namespace ob

extern "C" {

long long odise_mask_loss_workspace_bytes(int N, int P) {
  if (N <= 0 || P <= 0) return 0;
  return (long long)N * 16 + (long long)N * P * 8;
}

#define OB_MC_ENTRIES(SFX, T)                                                                                          \
  int odise_mask_cost_##SFX(const void* pred, const float* prob, const long long* labels, const uint8_t* tgt,          \
                            const float* points, const int* tgt_counts, float* cost, int B, int Q, int H, int W,       \
                            int K1, int Hg, int Wg, int Tmax, int P, float w_class, float w_mask, float w_dice,        \
                            void* stream) {                                                                            \
    return ob::mc_cost<T>(pred, prob, labels, tgt, points, tgt_counts, cost, B, Q, H, W, K1, Hg, Wg, Tmax, P,          \
                          w_class, w_mask, w_dice, stream);                                                            \
  }                                                                                                                    \
  int odise_mask_point_sample_##SFX(const void* maps, const float* points, float* out, int N, int H, int W, int P,     \
                                    void* stream) {                                                                    \
    return ob::mc_point_sample<T>(maps, points, out, N, H, W, P, stream);                                              \
  }                                                                                                                    \
  int odise_mask_loss_forward_##SFX(const void* pred, const uint8_t* tgt, const long long* pairs, const float* cand,   \
                                    const float* rnd, void* ws, float* losses, int B, int Q, int H, int W, int Hg,     \
                                    int Wg, int N, int P, int S, int k, float num_masks, void* stream) {               \
    return ob::mc_loss_forward<T>(pred, tgt, pairs, cand, rnd, ws, losses, B, Q, H, W, Hg, Wg, N, P, S, k, num_masks,  \
                                  stream);                                                                             \
  }                                                                                                                    \
  int odise_mask_loss_backward_##SFX(const void* pred, const uint8_t* tgt, const long long* pairs,                     \
                                     const long long* pair_of, const void* ws, const float* grad_losses,               \
                                     void* grad_pred, int B, int Q, int H, int W, int Hg, int Wg, int N, int P,        \
                                     float num_masks, void* stream) {                                                  \
    return ob::mc_loss_backward<T>(pred, tgt, pairs, pair_of, ws, grad_losses, grad_pred, B, Q, H, W, Hg, Wg, N, P,    \
                                   num_masks, stream);                                                                 \
  }

OB_MC_ENTRIES(f32, float)
OB_MC_ENTRIES(f16, __half)
OB_MC_ENTRIES(bf16, __nv_bfloat16)

int odise_mask_point_sample_u8(const void* maps, const float* points, float* out, int N, int H, int W, int P,
                               void* stream) {
  return ob::mc_point_sample<uint8_t>(maps, points, out, N, H, W, P, stream);
}

int odise_mask_assign_f32(const float* cost, const int* tgt_counts, long long* tables, int* status, int L, int B, int Q,
                          int Tmax, void* stream) {
  return ob::mc_assign(cost, tgt_counts, tables, status, L, B, Q, Tmax, stream);
}

}  // extern "C"
