// Fused flash attention on wgmma for the SD-v1 UNet SpatialTransformer (SURVEY.md §8a row a7.2): self-attention
// (4096 / 1024 tokens, head dim 40 / 80) and cross-attention over the 77-token context.  Reference: ldm
// CrossAttention = softmax(q k^T * d^-0.5) v via einsum or xformers (un-vendored; call sites ldm.py:481-489).
//
// One CTA = 128 queries of one (image, head): two consumer warpgroups own 64 query rows each, a producer warpgroup's
// first thread issues the TMA loads.  Per 64-key block j, in each consumer warpgroup:
//     S_j = Q K_j^T            (wgmma, both operands in shared memory, fp32 accumulators in registers)
//     online softmax in registers (a row lives in the 4 lanes of a quad), P_j -> fp16 (bf16x3) / bf16 register fragments
//     O += P_j V_j             (wgmma with A = P_j from registers, accumulated in registers across the key blocks)
// Operands are head-padded planes: head h occupies columns [h*HS, h*HS + DP) of q / k and rows of v^T with
// HS = 64 (d=40, DP=48) or 128 (d=80, DP=80); pad columns are zeros (produced by zero weight rows in the
// projection GEMM).  bf16x3: S = Q K^T uses hi*hi + hi*lo + lo*hi (the logits are exponentiated); O = P V uses
// P16 * V_hi + P16 * V_lo with V^T given as fp16 (hi, lo) planes (odise_gemm_desc.out_planes_fp16; wgmma multiplies
// operands of one 16-bit type) and P in [0, 1] rounded once to fp16 (2^-12 relative, random sign, averaged over the keys;
// bar 1e-3 on the UNet taps).
#include "ptx.cuh"
#include "wgmma.cuh"
#include "odise_b200.h"
#include "launch_count.h"
#include <cuda_fp16.h>
#include <cudaTypedefs.h>
#include <mutex>

namespace ob {

struct AttnParams {
  int B, heads, d, Tq, Tk, TkS;  // TkS: rows per image in the k / v^T planes (>= Tk, multiple of 8)
  float scale_log2;  // softmax scale * log2(e)
  float* out;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  long long ldo;
  const uint32_t* bits;     // optional [B, Tq, ceil(Tk/32)]: bit = key may be attended (Mask2Former masked attention)
  const int32_t* row_any;   // [B, Tq]: 0 -> the row ignores the mask (odise.py:683 fix-up)
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// DP = width of the P V product one CTA computes (= register accumulator width); QK = contraction width of
// Q K^T (head dim padded to 16).  QK > DP: the head's V columns are split over QK / DP CTAs that each recompute S
// (head dim 160 of the 16x16 / 8x8 UNet levels: QK = 160, DP = 80, two CTAs per (tile, head)), which keeps Q, one K
// stage and two V stages of a 160-wide head within shared memory.
template <int DP, int NMMA, int QK = DP>
struct AttnCfg {
  static constexpr int NC = (QK + 63) / 64;          // 64-column chunks per head
  static constexpr int HS = NC * 64;                 // head stride in q / k planes
  static constexpr int NP = (NMMA == 3) ? 2 : 1;
  static constexpr int BK = 64;                      // keys per block
  static constexpr int STAGES = (NC >= 3) ? 1 : 2;           // K stages (three chunks: shared memory allows one)
  static constexpr int VSTAGES = 2;
  static constexpr int Q_BYTES = NC * NP * 128 * 128;       // [chunk][plane][128 rows x 128 B]
  static constexpr int K_BYTES = NC * NP * BK * 128;        // per stage
  static constexpr int V_TILE = DP * 128;                   // one plane: DP rows x 64 tokens
  static constexpr int V_BYTES = NP * V_TILE;               // per stage
  static constexpr int SMEM_BYTES = Q_BYTES + STAGES * K_BYTES + VSTAGES * V_BYTES + 1024 + 256;
  static constexpr int THREADS = 384;
};

__device__ __forceinline__ uint32_t pack2(float a, float b, bool f16) {
  if (f16) {
    const __half2 h2 = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h2);
  }
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h2);
}

template <int DP, int NMMA, int QK = DP>
__global__ void __launch_bounds__(384, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
               const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl,
               const __grid_constant__ CUtensorMap tmVh, const __grid_constant__ CUtensorMap tmVl,
               const AttnParams p) {
  using Cfg = AttnCfg<DP, NMMA, QK>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::Q_BYTES;
  uint8_t* sV = sK + Cfg::STAGES * Cfg::K_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + Cfg::VSTAGES * Cfg::V_BYTES);
  uint64_t* q_full = bars;            // 1
  uint64_t* k_full = bars + 1;        // [2]
  uint64_t* k_empty = bars + 3;       // [2]
  uint64_t* v_full = bars + 5;        // [2]
  uint64_t* v_empty = bars + 7;       // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int VPARTS = QK > DP ? QK / DP : 1;        // CTAs sharing one head (each owns DP columns of V / of the output)
  const int q0 = blockIdx.x * 128, h = blockIdx.y / VPARTS, vpart = blockIdx.y % VPARTS, b = blockIdx.z;
  const int nblk = (p.Tk + Cfg::BK - 1) / Cfg::BK;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQh); tma_prefetch_desc(&tmKh); tma_prefetch_desc(&tmVh);
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 8);   // lane 0 of every consumer warp releases a stage
      mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      // ---------------------------------------------------------------- TMA producer
      mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
      for (int c = 0; c < Cfg::NC; ++c) {
        tma_load_3d(sQ + (c * Cfg::NP) * 16384, &tmQh, q_full, h * Cfg::HS + c * 64, b * p.Tq + q0, 0);
        if (NMMA == 3) tma_load_3d(sQ + (c * Cfg::NP + 1) * 16384, &tmQl, q_full, h * Cfg::HS + c * 64, b * p.Tq + q0, 0);
      }
      for (int j = 0; j < nblk; ++j) {
        const int st = j % Cfg::STAGES;
        mbar_wait(&k_empty[st], ((j / Cfg::STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&k_full[st], Cfg::K_BYTES);
        uint8_t* kd = sK + st * Cfg::K_BYTES;
        for (int c = 0; c < Cfg::NC; ++c) {
          tma_load_3d(kd + (c * Cfg::NP) * 8192, &tmKh, &k_full[st], h * Cfg::HS + c * 64, b * p.TkS + j * 64, 0);
          if (NMMA == 3)
            tma_load_3d(kd + (c * Cfg::NP + 1) * 8192, &tmKl, &k_full[st], h * Cfg::HS + c * 64, b * p.TkS + j * 64, 0);
        }
        const int sv = j % Cfg::VSTAGES;
        mbar_wait(&v_empty[sv], ((j / Cfg::VSTAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&v_full[sv], Cfg::V_BYTES);
        uint8_t* vd = sV + sv * Cfg::V_BYTES;
        tma_load_3d(vd, &tmVh, &v_full[sv], b * p.TkS + j * 64, h * Cfg::HS + vpart * DP, 0);
        if (NMMA == 3)
          tma_load_3d(vd + Cfg::V_TILE, &tmVl, &v_full[sv], b * p.TkS + j * 64, h * Cfg::HS + vpart * DP, 0);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups (64 query rows each)
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, wi = warp & 3;
  const int g = lane >> 2, t = lane & 3;
  // this thread's two rows of the accumulator fragments: g and g + 8 of the warp's 16
  const int rows[2] = {wg * 64 + wi * 16 + g, wg * 64 + wi * 16 + g + 8};
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const int n_words = (p.Tk + 31) / 32;
  const uint32_t* mask_words[2] = {nullptr, nullptr};
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q = q0 + rows[hh];
    if (p.bits && q < p.Tq && p.row_any[(long long)b * p.Tq + q] != 0)
      mask_words[hh] = p.bits + ((long long)b * p.Tq + q) * n_words;
  }
  float o[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
  constexpr int KS = QK / 16;
  const float c = p.scale_log2;
  const uint32_t kq = smem_u32(sQ) + wg * (64 * 128);

  mbar_wait(q_full, 0);
  for (int j = 0; j < nblk; ++j) {
    const int sk = j % Cfg::STAGES;
    mbar_wait(&k_full[sk], (j / Cfg::STAGES) & 1);
    float s[32];
    const uint32_t kk = smem_u32(sK + sk * Cfg::K_BYTES);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const int cc = ks >> 2, off = (ks & 3) * 32;
      const uint64_t qh = wgmma_desc_sw128(kq + (cc * Cfg::NP) * 16384 + off);
      const uint64_t kh = wgmma_desc_sw128(kk + (cc * Cfg::NP) * 8192 + off);
      wgmma_bf16(s, qh, kh, ks > 0 ? 1 : 0);
      if (NMMA == 3) {
        wgmma_bf16(s, qh, wgmma_desc_sw128(kk + (cc * Cfg::NP + 1) * 8192 + off), 1);
        wgmma_bf16(s, wgmma_desc_sw128(kq + (cc * Cfg::NP + 1) * 16384 + off), kh, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    if (lane == 0) mbar_arrive(&k_empty[sk]);

    // s[4 jj + 2 hh + e]: row rows[hh], key 8 jj + 2 t + e of the block
    const int valid = p.Tk - j * 64;  // keys of this block that exist
    if (valid < 64) {                 // only the last block can be ragged
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (8 * (i >> 2) + 2 * t + (i & 1) >= valid) s[i] = -INFINITY;
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      if (mask_words[hh]) {           // per-row predicted-mask bits (masked cross-attention)
        const uint32_t w0 = __ldg(mask_words[hh] + 2 * j);
        const uint32_t w1 = (2 * j + 1 < n_words) ? __ldg(mask_words[hh] + 2 * j + 1) : 0u;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = 8 * jj + 2 * t + e;
            const uint32_t w = key < 32 ? w0 : w1;
            if (!((w >> (key & 31)) & 1u)) s[4 * jj + 2 * hh + e] = -INFINITY;
          }
      }
    }
    float alpha[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float bm = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) bm = fmaxf(bm, fmaxf(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]));
      bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 1));
      bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 2));
      const float mn = fmaxf(m[hh], bm);
      alpha[hh] = (m[hh] == -INFINITY) ? 0.f : fast_exp2((m[hh] - mn) * c);
      m[hh] = mn;
      // guards: a row may have seen no attendable key yet (m = -inf) -> p = 0
      const float mc = (mn == -INFINITY) ? 0.f : -mn * c;
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * jj + 2 * hh + e];
          v = fast_exp2(fmaf(v, c, mc));
          sum += v;
        }
      l[hh] = l[hh] * alpha[hh] + sum;    // this lane's share of the row sum (the quad is summed at the end)
    }
#pragma unroll
    for (int jj = 0; jj < DP / 8; ++jj) {
      o[4 * jj] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
      o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
    }
    // P_j as the A fragments of four k16 slices: the accumulator layout of S is the m64k16 A-fragment layout
    uint32_t pa[4][4];
#pragma unroll
    for (int kk2 = 0; kk2 < 4; ++kk2)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[kk2][r] = pack2(s[8 * kk2 + 2 * r], s[8 * kk2 + 2 * r + 1], NMMA == 3);

    const int sv = j % Cfg::VSTAGES;
    mbar_wait(&v_full[sv], (j / Cfg::VSTAGES) & 1);
    const uint32_t vv = smem_u32(sV + sv * Cfg::V_BYTES);
    reg_fence(o);
    wgmma_fence();
#pragma unroll
    for (int kk2 = 0; kk2 < 4; ++kk2) {
      if (NMMA == 3) {
        wgmma_rs_f16(o, pa[kk2], wgmma_desc_sw128(vv + kk2 * 32), 1);
        wgmma_rs_f16(o, pa[kk2], wgmma_desc_sw128(vv + Cfg::V_TILE + kk2 * 32), 1);
      } else {
        wgmma_rs_bf16(o, pa[kk2], wgmma_desc_sw128(vv + kk2 * 32), 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if (lane == 0) mbar_arrive(&v_empty[sv]);
  }

  const int dpart = p.d / VPARTS;              // columns of the head this CTA owns
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float lt = l[hh];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const int q = q0 + rows[hh];
    if (q >= p.Tq) continue;
    const float inv = 1.f / lt;
    const long long ob = ((long long)b * p.Tq + q) * p.ldo + (long long)h * p.d + vpart * dpart;
#pragma unroll
    for (int jj = 0; jj < DP / 8; ++jj) {
      const int col = 8 * jj + 2 * t;
      if (col >= dpart) continue;
      float ov[2] = {o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv};
      if (p.out) *reinterpret_cast<float2*>(p.out + ob + col) = make_float2(ov[0], ov[1]);
      if (p.out_hi) store_planes<2>(p.out_hi + ob + col, p.out_lo ? p.out_lo + ob + col : nullptr, ov);   // bf16 pair or F16Q8
    }
  }
}

static PFN_cuTensorMapEncodeTiled_v12000 attn_get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
  });
  return fn;
}

static int attn_map(CUtensorMap* tm, const void* base, long long cols, long long rows, long long ld, int box_c,
                    int box_r) {
  auto enc = attn_get_encode();
  if (!enc) return ODISE_ERR_DRIVER;
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, 1};
  cuuint64_t str[2] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * rows * 2};
  cuuint32_t box[3] = {(cuuint32_t)box_c, (cuuint32_t)box_r, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, str, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? ODISE_OK : ODISE_ERR_TENSORMAP;
}

template <int DP, int NMMA, int QK = DP>
static int attn_launch(const CUtensorMap* m, const AttnParams& p, cudaStream_t stream) {
  using Cfg = AttnCfg<DP, NMMA, QK>;
  static_assert(Cfg::SMEM_BYTES <= 232448, "attention tile does not fit shared memory");
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_kernel<DP, NMMA, QK>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  dim3 grid((p.Tq + 127) / 128, p.heads * (QK > DP ? QK / DP : 1), p.B);
  attn_tc_kernel<DP, NMMA, QK><<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(m[0], m[1], m[2], m[3], m[4], m[5], p);
  return (int)cudaGetLastError();
}

}  // namespace ob

using namespace ob;

// q [B*Tq, heads*HS], k [B*TkS, heads*HS] head-padded planes (HS = 64 for d <= 48, 128 for d <= 80);
// vt [heads*HS, ldvt >= B*TkS] (V transposed: row = head-padded channel, col = b*TkS + t); keys t >= Tk are masked.
extern "C" int odise_attention_tc(const void* q_hi, const void* q_lo, long long ldq, const void* k_hi,
                                  const void* k_lo, long long ldk, const void* vt_hi, const void* vt_lo,
                                  long long ldvt, long long vt_rows, float* out, void* out_hi, void* out_lo,
                                  long long ldo, int B, int heads, int d, int Tq, int Tk, int tk_stride, float scale,
                                  int nmma, const uint32_t* mask_bits, const int32_t* row_any, void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  if (!q_hi || !k_hi || !vt_hi || (!out && !out_hi)) return ODISE_ERR_ARG;
  if (nmma != 1 && nmma != 3) return ODISE_ERR_ARG;
  if (nmma == 3 && (!q_lo || !k_lo || !vt_lo)) return ODISE_ERR_ARG;
  if (B <= 0 || heads <= 0 || Tq <= 0 || Tk <= 0 || tk_stride < Tk) return ODISE_ERR_ARG;
  // TMA needs 16-byte aligned box starts: tokens are the inner dimension of v^T
  if (tk_stride % 8) return ODISE_ERR_ALIGN;
  const int TkS = tk_stride;
  if (mask_bits && !row_any) return ODISE_ERR_ARG;
  int DP;
  if (d <= 32) DP = 32; else if (d <= 48) DP = 48; else if (d <= 64) DP = 64; else if (d <= 80) DP = 80;
  else if (d == 160) DP = 160;      // SD-v1 16x16 / 8x8 levels: Q K^T over 160, P V split into two 80-column halves
  else return ODISE_ERR_UNSUPPORTED;
  if (d % 8) return ODISE_ERR_UNSUPPORTED;
  const int HS = DP <= 64 ? 64 : (DP <= 80 ? 128 : 192);
  if (ldq % 8 || ldk % 8 || ldvt % 8 || ldq < (long long)heads * HS || ldk < (long long)heads * HS ||
      vt_rows < (long long)heads * HS || ldvt < (long long)B * TkS)
    return ODISE_ERR_ALIGN;
  if ((out && ldo % 4) || (out_hi && ldo % 8) || (d % 8)) return ODISE_ERR_ALIGN;
  CUtensorMap m[6];
  int rc;
  if ((rc = attn_map(&m[0], q_hi, (long long)heads * HS, (long long)B * Tq, ldq, 64, 128))) return rc;
  if ((rc = attn_map(&m[1], nmma == 3 ? q_lo : q_hi, (long long)heads * HS, (long long)B * Tq, ldq, 64, 128))) return rc;
  if ((rc = attn_map(&m[2], k_hi, (long long)heads * HS, (long long)B * TkS, ldk, 64, 64))) return rc;
  if ((rc = attn_map(&m[3], nmma == 3 ? k_lo : k_hi, (long long)heads * HS, (long long)B * TkS, ldk, 64, 64))) return rc;
  const int vbox = DP == 160 ? 80 : DP;
  if ((rc = attn_map(&m[4], vt_hi, (long long)B * TkS, vt_rows, ldvt, 64, vbox))) return rc;
  if ((rc = attn_map(&m[5], nmma == 3 ? vt_lo : vt_hi, (long long)B * TkS, vt_rows, ldvt, 64, vbox))) return rc;
  AttnParams p{};
  p.B = B; p.heads = heads; p.d = d; p.Tq = Tq; p.Tk = Tk; p.TkS = TkS;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = out; p.out_hi = reinterpret_cast<__nv_bfloat16*>(out_hi); p.out_lo = lo_arg(reinterpret_cast<__nv_bfloat16*>(out_lo));
  if (lo_is_q8(p.out_lo) && (ldo % 64 || (reinterpret_cast<uintptr_t>(out_lo) & 127))) return ODISE_ERR_ALIGN;
  p.ldo = ldo;
  p.bits = mask_bits; p.row_any = row_any;
  if (DP == 32) rc = nmma == 3 ? attn_launch<32, 3>(m, p, stream) : attn_launch<32, 1>(m, p, stream);
  else if (DP == 64) rc = nmma == 3 ? attn_launch<64, 3>(m, p, stream) : attn_launch<64, 1>(m, p, stream);
  else if (DP == 48) rc = nmma == 3 ? attn_launch<48, 3>(m, p, stream) : attn_launch<48, 1>(m, p, stream);
  else if (DP == 160) rc = nmma == 3 ? attn_launch<80, 3, 160>(m, p, stream) : attn_launch<80, 1, 160>(m, p, stream);
  else rc = nmma == 3 ? attn_launch<80, 3>(m, p, stream) : attn_launch<80, 1>(m, p, stream);
  if (rc) return rc;
  count_launch(1);
  return ODISE_OK;
}
