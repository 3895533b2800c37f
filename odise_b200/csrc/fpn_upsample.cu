// The FPN step of Mask2Former's pixel decoder (msdeformattn.py:349) on sm_90a, float32, forward and deterministic
// backward:
//
//   y[n, c, Y, X] = cur[n, c, Y, X] + bilinear(z)[n, c, Y, X]        (F.interpolate, align_corners=False)
//   grad_z        = bilinear^T(grad_y)                                (grad_cur is grad_y itself)
//
// z is the encoder level as it comes out of the token split: [N, h*w, C] rows, channel-contiguous, batch stride
// z_bs >= h*w*C (a slice of the encoder's memory [N, S, C], read in place).  cur, y and grad_y are NCHW-contiguous
// [N, C, H, W]; grad_z is written token-major with its own batch stride.  C is a multiple of 32.
//
// Forward: a CTA owns 32 output columns of one row and 32 channels.  Lanes run over channels to read the four
// corners (128-byte rows of z), the values go through a shared [32 c][33] tile, and lanes run over columns to read
// cur and write y.  The value is mr_bilinear of mask_resize.cuh, torch's fp32 bilinear with its FMA contraction; the
// add is one fp32 rounding, as torch's add.  torch resizes the reference's strided level view with its NHWC frame
// kernel when N >= 2 and with its NCHW frame kernel when N = 1, and the two contract the top row differently, so the
// kernel takes the matching contraction from N (mr_bilinear's top_ha).
//
// Backward: a gather, no atomics.  A CTA owns 32 source columns of one source row i and 32 channels.  The outputs that
// read source index i along an axis are the contiguous range of o with i0(o) <= i <= i1(o) (i0 and i1 are monotonic in
// o), found by binary search over mr_axis, the forward's own index arithmetic; the weight of o is h where i0 = i plus
// l where i1 = i.  So membership and weights are the forward's.  Per output row Y of the range (ascending) the CTA
// stages grad_y[n, c, Y, X] over the columns its sources read, in chunks of FU_SPAN, and each thread sums
// inner = sum_X wx(X, j) g (ascending X) and then acc = fma(wy(Y, i), inner, acc).  The order depends on the
// geometry only, so the gradient is bit-reproducible and an image's bits do not depend on the batch.
#include <stdint.h>

#include "launch_count.h"
#include "mask_resize.cuh"
#include "odise_b200.h"

namespace ob {
namespace {

constexpr int FU_T = 32;       // output columns (forward) / source columns (backward) per CTA, and channels per CTA
constexpr int FU_NT = 256;     // threads per CTA: 8 warps
constexpr int FU_W = FU_NT / 32;
constexpr int FU_SPAN = 128;   // output columns staged per chunk in the backward

template <bool top_ha>
__global__ void __launch_bounds__(FU_NT)
fu_forward_kernel(const float* __restrict__ z, long long z_bs, const float* __restrict__ cur, float* __restrict__ y,
                  int C, int h, int w, int H, int W, float sy, float sx) {
  __shared__ float t[FU_T][FU_T + 1];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int cb = C / FU_T;
  const int n = blockIdx.z / cb, c0 = (blockIdx.z - n * cb) * FU_T;
  const int X0 = blockIdx.x * FU_T, Y = blockIdx.y;
  const MrAxis ay = mr_axis(Y, sy, h);
  const float* zn = z + n * z_bs + c0 + lane;
  for (int k = wid; k < FU_T; k += FU_W) {
    const int X = X0 + k;
    if (X < W) t[lane][k] = mr_bilinear<float, top_ha>(zn, w, ay, mr_axis(X, sx, w), C);
  }
  __syncthreads();
  const int X = X0 + lane;
  if (X >= W) return;
  for (int k = wid; k < FU_T; k += FU_W) {
    const long long o = (((long long)n * C + c0 + k) * H + Y) * W + X;
    y[o] = __fadd_rn(__ldg(cur + o), t[k][lane]);
  }
}

// first o in [0, n_out) with i1(o) >= i (hi = false) or with i0(o) > i (hi = true); n_out if none
__device__ int fu_first(int n_out, float s, int n_src, int i, bool hi) {
  int lo = 0, up = n_out;
  while (lo < up) {
    const int mid = (lo + up) >> 1;
    const MrAxis a = mr_axis(mid, s, n_src);
    if (hi ? a.i0 > i : a.i1 >= i)
      up = mid;
    else
      lo = mid + 1;
  }
  return lo;
}

__device__ __forceinline__ float fu_weight(const MrAxis& a, int i) {
  return (a.i0 == i ? a.h : 0.f) + (a.i1 == i ? a.l : 0.f);
}

__global__ void __launch_bounds__(FU_NT)
fu_backward_kernel(const float* __restrict__ gy, float* __restrict__ gz, long long gz_bs, int C, int h, int w, int H,
                   int W, float sy, float sx) {
  __shared__ float gs[FU_T][FU_SPAN + 1];
  __shared__ MrAxis xa[FU_SPAN];
  __shared__ int xr[FU_T][2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int cb = C / FU_T;
  const int n = blockIdx.z / cb, c0 = (blockIdx.z - n * cb) * FU_T;
  const int j0 = blockIdx.x * FU_T, i = blockIdx.y;
  const int nj = min(FU_T, w - j0);
  if (wid == 0) {
    const int j = j0 + min(lane, nj - 1);
    xr[lane][0] = fu_first(W, sx, w, j, false);
    xr[lane][1] = fu_first(W, sx, w, j, true);
  }
  const int y_lo = fu_first(H, sy, h, i, false), y_hi = fu_first(H, sy, h, i, true);
  __syncthreads();
  const int x_lo = xr[0][0], x_hi = xr[nj - 1][1];
  constexpr int JQ = FU_T / FU_W;    // source columns per thread: j = j0 + wid + FU_W * q
  float acc[JQ];
#pragma unroll
  for (int q = 0; q < JQ; ++q) acc[q] = 0.f;
  const float* gn = gy + ((long long)n * C + c0) * H * W;
  for (int Y = y_lo; Y < y_hi; ++Y) {
    const float wy = fu_weight(mr_axis(Y, sy, h), i);
    float inner[JQ];
#pragma unroll
    for (int q = 0; q < JQ; ++q) inner[q] = 0.f;
    for (int xs = x_lo; xs < x_hi; xs += FU_SPAN) {
      const int len = min(FU_SPAN, x_hi - xs);
      __syncthreads();    // the previous chunk's reads are done
      for (int k = wid; k < FU_T; k += FU_W)
        for (int x = lane; x < len; x += 32) gs[k][x] = __ldg(gn + ((long long)k * H + Y) * W + xs + x);
      for (int x = threadIdx.x; x < len; x += FU_NT) xa[x] = mr_axis(xs + x, sx, w);
      __syncthreads();
#pragma unroll
      for (int q = 0; q < JQ; ++q) {
        const int jl = wid + FU_W * q;
        if (jl >= nj) continue;
        const int a = max(xr[jl][0], xs) - xs, b = min(xr[jl][1], xs + len) - xs;
        float s = inner[q];
        for (int x = a; x < b; ++x) s = __fmaf_rn(fu_weight(xa[x], j0 + jl), gs[lane][x], s);
        inner[q] = s;
      }
    }
#pragma unroll
    for (int q = 0; q < JQ; ++q) acc[q] = __fmaf_rn(wy, inner[q], acc[q]);
  }
#pragma unroll
  for (int q = 0; q < JQ; ++q) {
    const int jl = wid + FU_W * q;
    if (jl < nj) gz[n * gz_bs + ((long long)i * w + j0 + jl) * C + c0 + lane] = acc[q];
  }
}

// shapes both directions take: C a positive multiple of 32 (ODISE_ERR_UNSUPPORTED otherwise), grid limits, int
// token offsets within one image
int fu_check(int N, int C, int h, int w, int H, int W, long long bs) {
  if (N <= 0 || C <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0) return ODISE_ERR_ARG;
  if (C % FU_T) return ODISE_ERR_UNSUPPORTED;
  if ((long long)N * (C / FU_T) > 65535 || H > 65535 || h > 65535) return ODISE_ERR_UNSUPPORTED;
  if ((long long)h * w * C >= (1LL << 31)) return ODISE_ERR_UNSUPPORTED;
  if (bs < (long long)h * w * C) return ODISE_ERR_ARG;
  return 0;
}

}  // namespace
}  // namespace ob

extern "C" int odise_fpn_upsample_add_f32(const float* z, long long z_batch_stride, const float* cur, float* y, int N,
                                          int C, int h, int w, int H, int W, void* stream) {
  if (!z || !cur || !y) return ODISE_ERR_ARG;
  if (const int rc = ob::fu_check(N, C, h, w, H, W, z_batch_stride)) return rc;
  dim3 grid((W + ob::FU_T - 1) / ob::FU_T, H, N * (C / ob::FU_T));
  auto kern = N == 1 ? ob::fu_forward_kernel<true> : ob::fu_forward_kernel<false>;
  kern<<<grid, ob::FU_NT, 0, reinterpret_cast<cudaStream_t>(stream)>>>(z, z_batch_stride, cur, y, C, h, w, H, W,
                                                                      (float)h / (float)H, (float)w / (float)W);
  ob::count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_fpn_upsample_add_backward_f32(const float* grad_y, float* grad_z, long long grad_z_batch_stride,
                                                   int N, int C, int h, int w, int H, int W, void* stream) {
  if (!grad_y || !grad_z) return ODISE_ERR_ARG;
  if (const int rc = ob::fu_check(N, C, h, w, H, W, grad_z_batch_stride)) return rc;
  dim3 grid((w + ob::FU_T - 1) / ob::FU_T, h, N * (C / ob::FU_T));
  ob::fu_backward_kernel<<<grid, ob::FU_NT, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      grad_y, grad_z, grad_z_batch_stride, C, h, w, H, W, (float)h / (float)H, (float)w / (float)W);
  ob::count_launch(1);
  return (int)cudaGetLastError();
}
