/* odise_b200 C ABI — the drop-in boundary for the ODISE per-image inference hot path on H100 (sm_90a).
 *
 * Plain pointers and sizes only; the caller owns every buffer; every entry point is asynchronous on the CUDA
 * stream it is given (cudaStream_t passed as void*) and returns 0 or an error code (ODISE_ERR_* or a cudaError_t).
 *
 * The ONLY native surface of the reference is the pybind11 module "MultiScaleDeformableAttention"
 * (third_party/Mask2Former/mask2former/modeling/pixel_decoder/ops/src/vision.cpp:18-21); odise_msda_forward_f32
 * replaces ms_deform_attn_forward (.../src/ms_deform_attn.h:26-44 -> cuda/ms_deform_attn_cuda.cu:25-85).
 * The remaining entry points are the kernel families of SURVEY.md §2.4 that the reference executes as individual
 * ATen ops (cuDNN conv / GroupNorm / nn.MultiheadAttention / einsum); each one names the reference call site it
 * replaces.  INTEGRATION.md shows the ctypes binding a reference maintainer would add.
 *
 * Operand convention for tensor-core GEMMs: fp32 values travel as a (hi, lo) pair of bf16 planes with
 * hi = bf16(x), lo = bf16(x - hi); "nmma = 3" issues hi*hi + hi*lo + lo*hi (fp32-grade, the parity mode),
 * "nmma = 1" uses the hi planes only (plain bf16).
 * "nmma = 2" (ODISE_PLANES_F16Q8, round 2): hi = fp16(x); the second plane keeps the byte geometry of a 16-bit plane
 * (2 bytes per element, same leading dimension, which must be a multiple of 64 elements with 128-byte aligned rows) but
 * holds, per block of 64 consecutive k, 64 bytes e5m2(x * 2^-6) followed by 64 bytes e5m2((x - hi) * 2^6).  The GEMM
 * issues hi*hi on kind::f16 and the two first-order cross terms on kind::f8f6f4 at twice the 16-bit rate: 8 MMA slots
 * per 64-wide k-block instead of 12, ~2^-14 per product (UNet taps 1.1e-4 vs the fp32 oracle, bar 1e-3).
 */
#ifndef ODISE_B200_H_
#define ODISE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ODISE_OK 0
#define ODISE_ERR_ARG 10001       /* null / inconsistent argument */
#define ODISE_ERR_ALIGN 10002     /* leading dimension / pointer alignment not supported */
#define ODISE_ERR_DRIVER 10003    /* cuTensorMapEncodeTiled entry point not available */
#define ODISE_ERR_TENSORMAP 10004 /* tensor-map encoding rejected */
#define ODISE_ERR_WORKSPACE 10005 /* workspace missing / too small */
#define ODISE_ERR_UNSUPPORTED 10006

#define ODISE_ACT_NONE 0
#define ODISE_ACT_RELU 1
#define ODISE_ACT_SILU 2
#define ODISE_ACT_GELU 3
#define ODISE_ACT_QUICKGELU 4 /* x * sigmoid(1.702 x): open_clip QuickGELU (CLIP ViT MLP) */

/* operand-plane formats (see the convention above) */
#define ODISE_PLANES_BF16 0   /* (hi, lo) bf16 pair */
#define ODISE_PLANES_F16 1    /* (hi, lo) fp16 pair: V^T of odise_attention_tc */
#define ODISE_PLANES_F16Q8 2  /* fp16 hi + e5m2 correction bytes */
/* Format of the (hi, lo) planes written by every producer entry point launched AFTER this call (odise_split_f32, the
 * groupnorm / layernorm / GEGLU / add / act / upsample / im2col / patchify / softmax / l2-normalise passes, the plane outputs
 * of odise_attention_tc, odise_mha_d32*, odise_msda_fused_f32 and the post-processing kernels): ODISE_PLANES_BF16 (default)
 * or ODISE_PLANES_F16Q8.  A host-side launch parameter (process-global, not thread-safe), captured into CUDA graphs like
 * any other kernel argument.  odise_gemm_bf16 takes its formats from the descriptor instead. */
int odise_set_operand_format(int fmt);
int odise_get_operand_format(void);

int odise_version(void);
/* number of kernels launched through this library since load (bench.py "gpu_launches") */
long long odise_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * Multi-scale deformable attention forward (fp32).  Replaces MSDA.ms_deform_attn_forward
 * (ops/src/cuda/ms_deform_attn_cuda.cu:25-85, kernel ops/src/cuda/ms_deform_im2col_cuda.cuh:242-304).
 *   value          [N, S, M, D]      contiguous
 *   spatial_shapes [L, 2] int64 (H_l, W_l), level_start [L] int64            (device pointers)
 *   loc            [N, Lq, M, L, P, 2] (x, y) in [0,1];  attn [N, Lq, M, L, P]
 *   out            [N, Lq, M*D]   (fully overwritten; the reference allocates at::zeros)
 * D must be a multiple of 4 and <= 128 (ODISE: D = 32). */
int odise_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                           const float* loc, const float* attn, float* out, int N, int S, int M, int D, int L,
                           int Lq, int P, void* stream);

/* Fused front of MSDeformAttn.forward (ops/modules/ms_deform_attn.py:98-113): takes the raw outputs of the
 * sampling_offsets / attention_weights linears, applies the softmax over L*P and loc = ref + off / (W_l, H_l)
 * in registers, then samples.  offs [N, Lq, M, L, P, 2], logits [N, Lq, M, L*P], ref [N, Lq, L, 2]. */
int odise_msda_fused_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                         const float* ref, const float* offs, const float* logits, float* out,
                         void* out_hi, void* out_lo, int N, int S, int M, int D, int L, int Lq, int P, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * wgmma GEMM / implicit-GEMM 3x3 convolution:  out[z][m][n] = epi(alpha * sum_k A[z][m][k] * B[z][n][k]).
 * Replaces F.conv2d / F.linear / torch.einsum call sites of the path (ldm ResBlock & attention linears via
 * odise/modeling/meta_arch/ldm.py:469-491; M2F linears; odise.py:746 mask einsum; odise.py:955-959 pooling;
 * odise.py:192-205 CLIP match).
 *   epi(v) = act(v + bias[n] + bias_m[m] + rowbias[(z*M+m)/rows_per_group][n]) + residual[z][m][n]
 * conv3x3 = 1: A is an NHWC activation [B, H, W, C] (pixel stride lda elements), M = B*H*W, K = 9*C with
 *   k = (kh*3 + kw)*C + c, padding 1, stride 1; C % 64 == 0 and tiles must cover whole rows (W | 128 or 128 | W).
 * All bf16 leading dimensions are multiples of 8 elements, fp32 ones multiples of 4; base pointers 16-byte aligned. */
typedef struct odise_gemm_desc {
  int M, N, K, batch;
  int nmma;     /* 1 = bf16, 3 = bf16x3 (bf16 pairs), 2 = fp16 + e5m2 corrections (both operands ODISE_PLANES_F16Q8) */
  int conv3x3;  /* 0 plain, 1 implicit 3x3 conv */
  int conv_C, conv_H, conv_W;
  const void* a_hi; const void* a_lo; long long lda; long long a_batch_stride; /* 0 = shared across batch */
  const void* b_hi; const void* b_lo; long long ldb; long long b_batch_stride;
  float alpha;
  const float* bias;                 /* [N] or NULL */
  const float* rowbias; int rows_per_group; long long rowbias_ld; /* [groups, N] or NULL */
  int act;
  const float* residual; long long ld_residual; long long residual_batch_stride;
  float* out_f32; long long ld_out; long long out_batch_stride;
  void* out_hi; void* out_lo; long long ld_out_bf16; long long out_bf16_batch_stride;
  int split_k; void* workspace; long long workspace_bytes;
  int force_bn;                      /* 0 = heuristic; 64/128/160/256 */
  const float* bias_m;               /* [M] per-row bias or NULL (transposed-output projections) */
  int conv_mode;                     /* conv3x3: 0 = stride 1 pad 1; 1 = stride 2 pad (1,1) (ldm Downsample);
                                        2 = stride 2 pad (0,1) (ldm VAE Downsample). conv_H/W are INPUT dims,
                                        M = B * (H/stride) * (W/stride) */
  int geglu;                         /* 1: N = 2*Nh, weight rows quad-interleaved (a0-3, g0-3, a4-7, g4-7, ...):
                                        out planes [M, Nh] = a * gelu(gate)  (ldm GEGLU fused into FF1) */
  float* gn_partial;                 /* optional: GroupNorm statistics of the OUTPUT computed in the epilogue (the
                                        producer side of the fused conv + GN + SiLU of ldm ResBlock): per (32-row segment,
                                        column) a record (shift, S1, S2) at gn_partial[seg * gn_seg_stride +
                                        {0,1,2} * gn_plane_stride + n], seg = (z*M + m) / 32.  Needs M % 32 == 0, split_k <= 1.
                                        Merged per (image, group) by odise_groupnorm_finalize_seg_f32. */
  long long gn_seg_stride; long long gn_plane_stride;
  int out_planes_fp16;               /* format of out_hi / out_lo: ODISE_PLANES_BF16 (0), ODISE_PLANES_F16 (1: hi = fp16(v),
                                        lo = fp16(v - hi), the V^T operand of odise_attention_tc) or ODISE_PLANES_F16Q8 (2:
                                        ld_out_bf16 % 64 == 0, rows 128-byte aligned) */
} odise_gemm_desc;
int odise_gemm_bf16(const odise_gemm_desc* desc, void* stream);
/* Host-only: the cost-model tile choice of odise_gemm_bf16 for a problem — output-tile width *bn (64 | 128 | 160 | 256) and
 * *pair (always 0: the sm_90a kernel does not pair CTAs; F16Q8 (nmma 2) uses BN <= 128).  It is what the
 * GEMM uses under CUDA-graph capture / with ODISE_GEMM_AUTOTUNE=0 and the first candidate of the one-time per-shape autotune. */
int odise_gemm_tile_policy(int M, int N, int K, int batch, int conv3x3, int nmma, int* bn, int* pair);
/* optional per-launch timing of odise_gemm_bf16 (CUDA events on the launch stream; not for use under graph capture):
 * begin() starts recording, end() synchronises and returns launch count, summed device ms and algorithmic FLOPs. */
int odise_profile_begin(void);
int odise_profile_end(long long* launches, double* total_ms, double* total_flops);

/* ------------------------------------------------------------------------------------------------------------
 * Elementwise / normalisation passes (HBM-bound).  Every one of them also produces the (hi, lo) bf16 operand
 * planes the next GEMM consumes, so the fp32 -> bf16x2 split never costs an extra pass.  NHWC / token-major. */

/* fp32 -> (hi, lo); rows x cols with leading dims (elements). out_lo may be NULL. */
int odise_split_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, long long rows, int cols,
                    void* stream);
/* the same split into an fp16 pair (V^T of odise_attention_tc when it does not come out of a GEMM epilogue) */
int odise_split_f16_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, long long rows, int cols,
                        void* stream);
/* GroupNorm statistics over NHWC x[B, HW, C] (pixel stride ldx): mean/rstd [B, G].
 * (torch.nn.GroupNorm in ldm ResBlock / SpatialTransformer / d2 BottleneckBlock / M2F input_proj) */
int odise_groupnorm_stats_f32(const float* x, long long ldx, float* mean, float* rstd, int B, int HW, int C, int G,
                              float eps, void* stream);
int odise_groupnorm_stats_bs_f32(const float* x, long long ldx, long long x_bs, float* mean, float* rstd, int B,
                                 int HW, int C, int G, float eps, void* stream);
/* Coalesced single-pass statistics with a caller-provided workspace of odise_groupnorm_ws_floats() floats
 * (deterministic fixed-order combine; shifted sums) — the variant the engines use. */
long long odise_groupnorm_ws_floats(int B, int HW, int C, int G);
int odise_groupnorm_stats_ws_f32(const float* x, long long ldx, long long x_bs, float* ws, float* mean, float* rstd,
                                 int B, int HW, int C, int G, float eps, void* stream);
/* mean / rstd [B, G] from the per-(32-row segment, channel) records an odise_gemm_bf16 epilogue left in `partial`
 * (desc.gn_partial; rows of image b are segments [b*HW/32, (b+1)*HW/32), HW % 32 == 0; channel c at column c of each of
 * the three planes): Chan's parallel-variance merge in double, fixed order -> deterministic.  Replaces the statistics pass
 * over the activation (odise_groupnorm_stats_ws_f32) when the activation was produced by our own GEMM. */
int odise_groupnorm_finalize_seg_f32(const float* partial, long long seg_stride, long long plane_stride, float* mean,
                                     float* rstd, int B, int HW, int C, int G, float eps, void* stream);
/* y = act(gn(x) * gamma + beta): writes fp32 (optional) and (hi, lo) planes (optional). act: NONE/SILU/RELU.
 * The *_bs variants take explicit per-image strides (elements; 0 = dense) so a level can be read from / written
 * into the level-concatenated [B, S, C] token matrix of the pixel decoder (msdeformattn.py:61-78). */
int odise_groupnorm_apply_f32(const float* x, long long ldx, const float* mean, const float* rstd,
                              const float* gamma, const float* beta, int act, float* y, long long ldy, void* hi,
                              void* lo, long long ldo, int B, int HW, int C, int G, void* stream);
int odise_groupnorm_apply_bs_f32(const float* x, long long ldx, long long x_bs, const float* mean, const float* rstd,
                                 const float* gamma, const float* beta, int act, float* y, long long ldy,
                                 long long y_bs, void* hi, void* lo, long long ldo, long long o_bs, int B, int HW,
                                 int C, int G, void* stream);
/* y (+)= act(gn(x) * gamma + beta + res): the tail of detectron2's BottleneckBlock (relu(gn(conv3) + shortcut)),
 * optionally accumulated into y — the per-stride sum of FeatureExtractorBackbone.forward_features
 * (feature_extractor.py:157-179). */
int odise_groupnorm_apply_res_f32(const float* x, long long ldx, const float* mean, const float* rstd,
                                  const float* gamma, const float* beta, const float* res, long long ldres, int act,
                                  float* y, long long ldy, int accumulate, void* hi, void* lo, long long ldo, int B,
                                  int HW, int C, int G, void* stream);
/* out[b, t, c] = a0[t, c] + ta[t, c] * p[b, c]: LdmImplicitCaptionerExtractor.forward (ldm.py:705-714) with the
 * weight-only terms folded: cond = (uncond + tanh(alpha) * pos) + tanh(alpha) * clip_project(prefix). */
int odise_bcast_fma_f32(const float* a0, const float* ta, const float* p, float* out, int B, int T, int C,
                        void* stream);
/* y[r, :] *= s[r]  (slide_forward's division by the crop-overlap count, feature_extractor.py:246-248) */
int odise_rowscale_f32(float* y, long long ldy, const float* s, long long rows, int cols, void* stream);
/* LayerNorm over the last dim (cols <= 4096): optional fp32 output, optional residual add BEFORE the norm
 * (post-norm transformer: y = LN(x + res)), optional `post_add` AFTER the norm written only to the bf16 planes
 * (query_pos / pos added to the GEMM operand, M2F with_pos_embed). */
int odise_layernorm_f32(const float* x, long long ldx, const float* res, long long ldres, const float* gamma,
                        const float* beta, float eps, float* y, long long ldy, const float* post_add,
                        long long ldpa, void* hi, void* lo, long long ldo, long long rows, int cols, void* stream);
/* GEGLU: y[m, j] = x[m, j] * gelu(x[m, j + cols]) for x [rows, 2*cols] -> (hi, lo) [rows, cols]
 * (ldm attention.GEGLU, SURVEY.md App. A) */
int odise_geglu_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, long long rows, int cols,
                    void* stream);
/* y = a + b (optional b, optional fp32 y) -> (hi, lo); b_rows > 0 broadcasts b over rows modulo b_rows */
int odise_add_split_f32(const float* a, long long lda, const float* b, long long ldb, long long b_rows, float* y,
                        long long ldy, void* hi, void* lo, long long ldo, long long rows, int cols, void* stream);
/* y = act(x) -> (hi, lo)  (SiLU(emb) in front of ResBlock.emb_layers) */
int odise_act_split_f32(const float* x, long long ldx, int act, void* hi, void* lo, long long ldo, long long rows,
                        int cols, void* stream);
/* nearest 2x upsample of NHWC x[B,H,W,C] -> (hi, lo) [B,2H,2W,C] (ldm Upsample before its conv3x3) */
int odise_upsample2x_split_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, int B, int H,
                               int W, int C, void* stream);
/* materialised im2col for the few convs the implicit path does not cover (C % 64 != 0, stride 2):
 * x NHWC [B,H,W,C] -> (hi, lo) [B*Ho*Wo, Kpad] with k = (kh*3+kw)*C + c, zero padded to Kpad.
 * pad_lo/pad_hi: zero padding before / after along both H and W (ldm Downsample: 1/1; VAE Downsample: 0/1). */
int odise_im2col3x3_split_f32(const float* x, long long ldx, void* hi, void* lo, int Kpad, int B, int H, int W,
                              int C, int stride, int pad_lo, int pad_hi, void* stream);
/* strided 2-D fp32 copy (skip-concat into a channel slice, crop paste) with optional scale and accumulate */
int odise_copy2d_f32(const float* src, long long lds, float* dst, long long ldd, long long rows, int cols,
                     float scale, int accumulate, void* stream);
/* bilinear (align_corners=False) / nearest resize of NHWC fp32, optional accumulate into dst (FPN top-down add,
 * msdeformattn.py:349; F.interpolate nearest in feature_extractor.py:165) */
int odise_resize_nhwc_f32(const float* src, long long lds, float* dst, long long ldd, int B, int Hs, int Ws, int Hd,
                          int Wd, int C, int bilinear, int accumulate, void* stream);
int odise_resize_nhwc_bs_f32(const float* src, long long lds, long long src_bs, float* dst, long long ldd,
                             long long dst_bs, int B, int Hs, int Ws, int Hd, int Wd, int C, int bilinear,
                             int accumulate, void* stream);
/* uint8 NCHW images [N, 3, H, W] -> normalised NHWC fp32 crops [n_crops, ch, cw, 3] = ((x / 255) - 0.5) / 0.5
 * (odise.py:237 + ldm.py:556); boxes [n_crops, 3] int32 = (image index, y0, x0) (device). */
int odise_image_crops_u8_f32(const uint8_t* img, float* out, const int32_t* boxes, int n_crops, int H, int W, int ch,
                             int cw, void* stream);
/* same for a float NCHW image already in [0, 1] (the Backbone plugin input, feature_extractor.py:252) */
int odise_image_crops_f32(const float* img, float* out, const int32_t* boxes, int n_crops, int H, int W, int ch, int cw,
                          void* stream);
/* CLIP image preprocessing of crops (clip.py:94: bicubic Resize(S) without antialias + CenterCrop(S) + Normalize with
 * the CLIP mean / std): img uint8 (0..255) or float32 in [0, 1], NCHW [N, 3, H, W]; boxes as above; square crops;
 * out NHWC fp32 [n_crops, S, S, 3]. */
int odise_clip_preprocess(const void* img, int img_is_u8, float* out, const int32_t* boxes, int n_crops, int H, int W,
                          int ch, int cw, int S, void* stream);
/* T.Resize(backbone_in_size, BICUBIC) of FeatureExtractorBackbone.single_forward (feature_extractor.py:73-76, :144): a
 * square crop smaller than 512 x 512 is resized to S x S before the feature extractor sees it.  Same sampling as
 * odise_clip_preprocess (bicubic A = -0.75, align_corners=False, no antialias, indices clamped to the crop), no
 * normalisation, no clamping of the overshoot (float tensors are not clamped by torchvision); out is a float image
 * batch NCHW [n_crops, 3, S, S] in (about) [0, 1] that re-enters odise_image_crops_f32 / odise_clip_preprocess. */
int odise_crop_resize_bicubic(const void* img, int img_is_u8, float* out, const int32_t* boxes, int n_crops, int H, int W,
                              int ch, int cw, int S, void* stream);
/* P x P non-overlapping patches of NHWC [B, S, S, 3] -> (hi, lo) rows [B*(S/P)^2, Kpad] with k = c*P*P + ky*P + kx
 * (visual.conv1 as a GEMM, clip.py:179) */
int odise_patchify_split_f32(const float* x, void* hi, void* lo, int B, int S, int P, int Kpad, void* stream);
/* NHWC <-> NCHW transposes at the plugin boundary */
int odise_nchw_to_nhwc_f32(const float* src, float* dst, long long ldd, int B, int C, int HW, void* stream);
int odise_nhwc_to_nchw_f32(const float* src, long long lds, float* dst, int B, int C, int HW, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Fused flash attention on wgmma (UNet SpatialTransformer self- and cross-attention; ldm CrossAttention,
 * SURVEY.md App. A): out[b, t, h*d + j] = softmax_k(scale * q.k) v.
 * Operands are HEAD-PADDED (hi, lo) planes: head h occupies columns [h*HS, h*HS + d) with HS = 64 (d <= 64),
 * 128 (d <= 80) or 192 (d == 160: the 16x16 / 8x8 UNet levels), pad columns zero:  q [B*Tq, heads*HS] (ldq), k [B*tk_stride, heads*HS] (ldk), and V TRANSPOSED
 * vt [vt_rows >= heads*HS, ldvt >= B*tk_stride] with vt[h*HS + j][b*tk_stride + t] = v[b, t, h, j] (the projection
 * GEMM writes it directly by swapping its operands).  tk_stride >= Tk is the per-image row count of the key /
 * value planes (multiple of 8: TMA box starts must be 16-byte aligned); keys t >= Tk are masked out.  d % 8 == 0 and
 * d <= 80, or d == 160 (other head sizes: odise_gemm_bf16 + odise_softmax_split_f32, e.g. the VAE mid block's d = 512).
 * nmma = 3: q, k are bf16 (hi, lo) planes, vt is an **fp16** (hi, lo) pair (odise_gemm_desc.out_planes_fp16 /
 * odise_split_f16_f32): S = Q K^T runs hi*hi + hi*lo + lo*hi, the probabilities are rounded once to fp16 and
 * O = P16 V_hi + P16 V_lo (wgmma needs A and B of one 16-bit type).  nmma = 1: bf16 hi planes only.
 * out fp32 and/or (hi, lo) bf16 planes, UNPADDED [B*Tq, heads*d] with row stride ldo.
 * mask_bits / row_any (optional, from odise_attn_mask_bits_f32): the Mask2Former decoder's masked cross-attention
 * (d = 32) on the same tensor-core kernel — key k of row (b, t) is dropped when its bit is 0 and row_any != 0. */
int odise_attention_tc(const void* q_hi, const void* q_lo, long long ldq, const void* k_hi, const void* k_lo,
                       long long ldk, const void* vt_hi, const void* vt_lo, long long ldvt, long long vt_rows,
                       float* out, void* out_hi, void* out_lo, long long ldo, int B, int heads, int d, int Tq,
                       int Tk, int tk_stride, float scale, int nmma, const uint32_t* mask_bits,
                       const int32_t* row_any, void* stream);
/* row softmax of scale * x over the first `cols` columns -> (hi, lo) planes [rows, ldo], columns [cols, cols_pad)
 * written as zeros (the unfused attention path for head dims > 80 and the VAE mid-block attention). */
int odise_softmax_split_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, long long rows,
                            int cols, int cols_pad, float scale, void* stream);

/* Masked cross-attention of the Mask2Former decoder (odise.py:683-692 + 760-774,
 * mask2former_transformer_decoder.py:98-110).  The boolean attn_mask [B*8, Q, HW] of the reference is replaced by
 * 1 bit per (b, q, key), shared by the 8 heads: bit = !(sigmoid(bilinear(mask_logits -> (Hl, Wl))) < 0.5), and
 * row_any[b, q] = "some key allowed"; rows with row_any == 0 attend everywhere (the odise.py:683 fix-up).
 *   mask_logits [B, Q, Hm, Wm] fp32; bits [B, Q, ceil(Hl*Wl/32)] uint32; row_any [B, Q] int32. */
int odise_attn_mask_bits_f32(const float* mask_logits, uint32_t* bits, int32_t* row_any, int B, int Q, int Hm,
                             int Wm, int Hl, int Wl, void* stream);
/* Multi-head attention for head_dim 32 (nn.MultiheadAttention(256, 8) core of the decoder's cross- and
 * self-attention layers): q [B, Tq, heads*32] (row stride ldq), k, v [B, Tk, heads*32] (row stride ldkv; lets
 * several layers' projections live side by side in one GEMM output) already projected, fp32;
 * out = softmax(scale * q k^T  (+ -inf where bit == 0 and row_any != 0)) v, written as fp32 and/or (hi, lo).
 * bits / row_any may be NULL (unmasked self-attention). */
int odise_mha_d32_f32(const float* q, long long ldq, const float* k, const float* v, long long ldkv,
                      const uint32_t* bits, const int32_t* row_any, float* out, void* out_hi, void* out_lo,
                      long long ldo, int B, int Tq, int Tk, int heads, float scale, void* stream);
/* same with a workspace of odise_mha_d32_ws_floats() floats: long key ranges (>= 2048 keys) are split over 2-4
 * blocks per query tile (flash-decoding style) and merged by a second kernel */
long long odise_mha_d32_ws_floats(int B, int Tq, int Tk, int heads);
int odise_mha_d32_ws_f32(const float* q, long long ldq, const float* k, const float* v, long long ldkv,
                         const uint32_t* bits, const int32_t* row_any, float* out, void* out_hi, void* out_lo,
                         long long ldo, int B, int Tq, int Tk, int heads, float scale, float* ws, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Mask head helpers (odise.py:937-963 MaskPooling, odise.py:746 einsum) */
/* mask_logits [B, Q, HW] fp32 -> binary (logit > 0) as bf16 plane [B, Q, HWpad] + counts [B, Q] */
int odise_mask_binarize_f32(const float* logits, void* bin_bf16, long long ld_bin, float* counts, int B, int Q,
                            int HW, void* stream);
/* pooled[b,q,c] = sums[b,q,c] / (counts[b,q] + 1e-8) */
int odise_pool_normalize_f32(const float* sums, const float* counts, float* pooled, int B, int Q, int C,
                             void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * CLIP match tail (odise.py:181-207 cal_pred_logits + helper.py:79-109 ensemble max):
 *   sims [BQ, Kp] = logit_scale * <normalize(mask_embed), normalize(text_embed)>  (GEMM above on normalised rows)
 *   out [BQ, Kc+1]: per-class max over its synonym columns (group_start [Kc+1] int32 prefix) + null column. */
int odise_l2_normalize_split_f32(const float* x, long long ldx, void* hi, void* lo, long long ldo, long long rows,
                                 int cols, void* stream);
int odise_class_max_f32(const float* sims, long long ld_sims, const int32_t* group_start, const float* null_sim,
                        float* out, long long rows, int n_classes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Post-processing on the device (odise.py:326-370; maskformer_model.py:280-342) — no host syncs.
 * upsample: bilinear (align_corners=False) of mask logits [B, Q, hs, ws] to (H, W), sigmoid, written pixel-major as
 *   (hi, lo) planes [B*H*W, Qpad] (operand of the semantic GEMM) and optionally the upsampled logits up_f32 [B,Q,H,W]. */
/* geom (optional, all three post-processing calls): sem_seg_postprocess (detectron2 modeling/postprocessing.py, called
 * at odise.py:343-347 with sem_seg_postprocess_before_inference=True).  NULL: output (H, W) == padded input size.
 * Otherwise the logits are resampled [hs, ws] -> (pad_h, pad_w) -> crop (img_h, img_w) -> (H, W), both bilinear. */
typedef struct { int pad_h, pad_w, img_h, img_w; } odise_postprocess_geom;
int odise_upsample_sigmoid_split_f32(const float* logits, void* hi, void* lo, float* up_f32, int B, int Q, int Qpad,
                                     int hs, int ws, int H, int W, const odise_postprocess_geom* geom, void* stream);
/* softmax over the K+1 class logits of every query: probs [B*Q, K1] (optional), probs_t [B, K, Qpad] (optional,
 * transposed without the void class, pad columns untouched: pre-zero it), max prob, argmax (first among ties),
 * keep = (label != K) && (score > threshold)   (maskformer_model.py:287-290) */
int odise_query_scores_f32(const float* cls, float* probs, float* probs_t, float* scores, int32_t* labels,
                           int32_t* keep, int B, int Q, int Qpad, int K1, float threshold, void* stream);
/* MaskFormer.panoptic_inference on the device: pan int32 [B, H, W] (0 = void), seg_info int32 [B, Q, 3] =
 * (id, isthing, category) for the first n_segments[b] rows.  ws: odise_panoptic_ws_bytes() bytes. */
long long odise_panoptic_ws_bytes(int B, int Q, int H, int W);
int odise_panoptic_inference_f32(const float* logits, const float* scores, const int32_t* labels, const int32_t* keep,
                                 const uint8_t* is_thing, int32_t* pan, int32_t* seg_info, int32_t* n_segments,
                                 void* ws, int B, int Q, int K, int hs, int ws_, int H, int W, double overlap_thr,
                                 const odise_postprocess_geom* geom, void* stream);

/* MaskFormer.instance_inference (maskformer_model.py:344-380) on the device: top-k over the flattened [Q*K] class
 * probabilities (probs [B*Q, K+1] from odise_query_scores_f32; void column dropped), sorted by probability
 * (descending; ties -> lower flat index), times the mask score sum(sigmoid*m)/(sum(m)+1e-6), m = upsampled logit > 0.
 * scores / classes / query_index / valid: [B, topk]; valid = is_thing[class] (the panoptic_on filter; all 1 when
 * is_thing == NULL); masks u8 [B, Q, H, W] optional (instance i's mask = masks[b, query_index[b, i]]).  topk <= 1024. */
long long odise_instance_ws_bytes(int B, int Q, int H, int W);
int odise_instance_inference_f32(const float* probs, const float* logits, const uint8_t* is_thing, float* scores,
                                 int32_t* classes, int32_t* query_index, int32_t* valid, uint8_t* masks, void* ws, int B,
                                 int Q, int K, int topk, int hs, int ws_, int H, int W,
                                 const odise_postprocess_geom* geom, void* stream);

/* The three inference heads of CategoryODISE.forward (odise.py:326-370) from ONE resampling pass over the mask logits: the
 * stand-alone entry points above each re-evaluate bilinear + sigmoid of every (pixel, query).  Output groups are optional
 * (NULL = skip): semantic operand planes sem_hi / sem_lo [B*H*W, Qpad] (then run the semantic GEMM as before) | panoptic
 * (arguments as odise_panoptic_inference_f32; pan_ws of odise_panoptic_ws_bytes) | instance (arguments as
 * odise_instance_inference_f32; inst_ws of odise_postprocess_fused_ws_bytes; panoptic_filter = apply is_thing to `valid`). */
long long odise_postprocess_fused_ws_bytes(int B, int Q, int H, int W);
int odise_postprocess_fused_f32(const float* logits, void* sem_hi, void* sem_lo, int Qpad, const float* scores,
                                const int32_t* labels, const int32_t* keep, const uint8_t* is_thing, int32_t* pan,
                                int32_t* seg_info, int32_t* n_segments, void* pan_ws, double overlap_thr, const float* probs,
                                float* inst_scores, int32_t* inst_classes, int32_t* inst_query, int32_t* inst_valid,
                                uint8_t* inst_masks, void* inst_ws, int topk, int panoptic_filter, int B, int Q, int K,
                                int hs, int ws_, int H, int W, const odise_postprocess_geom* geom, void* stream);

/* MaskCLIP front-end (odise/modeling/meta_arch/clip.py:284-339) and the open-vocabulary merge (odise.py:1506-1536,
 * :300-323).
 * preprocess: whole image [N,3,H,W] (u8 0..255 or f32 in [0,1]) -> bilinear (align_corners=False) S x S, CLIP
 *   mean/std, NHWC fp32 [N*S*S, 3].
 * bits: mask logits [B,Q,hm,wm] -> attention bits of the Q mask tokens in odise_attention_tc's layout: a token
 *   sequence of Tq rows per image whose rows row0..row0+Q-1 are the mask tokens; bits [B, Tq, ceil(((S/P)^2+1)/32)]
 *   (key 0 = class token, always on; key 1+p = patch p, on iff the max over its PxP window of the mask upsampled to
 *   S x S has sigmoid >= 0.5); row_any [B, Tq] = 1 on mask-token rows, 0 elsewhere (those rows ignore the bits).
 * merge: cat_logits [rows, K+1] (category head, void last), clip_logits [rows, K] (row stride ld_clip), overlap u8 [K]
 *   (class also named in the training vocabulary) -> out [rows, K+1] = log(cat[softmax(e) * (1 - p_void), p_void] +
 *   1e-8), e_k = (1-a_k) log softmax(cat[:K])_k + a_k log softmax(clip)_k, a_k = alpha if overlap[k] else beta;
 *   open_logits [rows, K] = e (optional). */
int odise_maskclip_preprocess(const void* img, int img_is_u8, float* out, int N, int H, int W, int S, void* stream);
int odise_maskclip_bits_f32(const float* mask_logits, uint32_t* bits, int32_t* row_any, int B, int Q, int hm, int wm,
                            int S, int P, int Tq, int row0, void* stream);
int odise_open_vocab_merge_f32(const float* cat_logits, const float* clip_logits, long long ld_clip,
                               const uint8_t* overlap, float alpha, float beta, float* out, float* open_logits, int rows,
                               int K, void* stream);

/* out[i, :] = src[idx[i], :] (+ add[i % add_period, :]) — token-embedding lookup + positional embedding of the CLIP text
 * towers (clip.py:139-140), and the EOT-row gather (clip.py:150). */
int odise_gather_rows_f32(const float* src, long long lds, const int32_t* idx, const float* add, long long ld_add,
                          int add_period, float* out, long long ldo, long long rows, int cols, void* stream);

/* Shared-memory carve-out policy of the current device (cudaDeviceSetCacheConfig): 1 = prefer the maximum shared-memory
 * carve-out for every kernel so the SMs are not re-partitioned between elementwise kernels and the TMA-staged GEMMs;
 * 0 = driver default. */
int odise_set_carveout_policy(int prefer_shared);

#ifdef __cplusplus
}
#endif
#endif /* ODISE_B200_H_ */
