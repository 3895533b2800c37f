// TEST / BENCH INFRASTRUCTURE — not part of the product (only tests/ and tools/ use oracle/).
//
// C-ABI host shim around the REFERENCE's own MSDeformAttn backward kernels, compiled from the reference sources where
// they lie (third_party/Mask2Former/mask2former/modeling/pixel_decoder/ops/src/cuda/ms_deform_im2col_cuda.cuh:92-164
// col2im bilinear, launcher ms_deformable_col2im_cuda :962-1332).  As for the forward shim (ref_msda_host.cu), the
// reference's host file does not compile against torch 2.11, so this file restates the host loop of
// ms_deform_attn_cuda_backward (ms_deform_attn_cuda.cu:126-153: zero-filled gradients, im2col_step chunks) and calls
// the UNMODIFIED launcher.  Built by oracle/backward.mk into oracle/_ref/libref_msda_backward.so; the GPU baseline of
// tools/msda_backward_bench.py and the source of tests/golden/ref_msda_kernel_backward.pt.
#include "cuda/ms_deform_im2col_cuda.cuh"

extern "C" int ref_ms_deform_attn_backward_f32(const float* value, const int64_t* spatial_shapes,
                                               const int64_t* level_start, const float* loc, const float* attn,
                                               const float* grad_out, float* grad_value, float* grad_loc,
                                               float* grad_attn, int N, int S, int M, int D, int L, int Lq, int P,
                                               int im2col_step, void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const int step = N < im2col_step ? N : im2col_step;
  if (step <= 0 || N % step) return 1;                            // reference: AT_ASSERTM(batch % im2col_step_ == 0)
  const long long per_value = (long long)S * M * D, per_loc = (long long)Lq * M * L * P * 2,
                  per_attn = (long long)Lq * M * L * P, per_out = (long long)Lq * M * D;
  // reference: at::zeros_like for all three (some of its kernels accumulate grad_loc / grad_attn with atomics)
  cudaMemsetAsync(grad_value, 0, sizeof(float) * N * per_value, stream);
  cudaMemsetAsync(grad_loc, 0, sizeof(float) * N * per_loc, stream);
  cudaMemsetAsync(grad_attn, 0, sizeof(float) * N * per_attn, stream);
  for (int n = 0; n < N / step; ++n)
    ms_deformable_col2im_cuda<float>(stream, grad_out + n * step * per_out, value + n * step * per_value,
                                     spatial_shapes, level_start, loc + n * step * per_loc,
                                     attn + n * step * per_attn, step, S, M, D, L, Lq, P,
                                     grad_value + n * step * per_value, grad_loc + n * step * per_loc,
                                     grad_attn + n * step * per_attn);
  return (int)cudaGetLastError();
}
