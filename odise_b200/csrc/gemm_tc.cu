// wgmma / TMA GEMM for sm_90a: the tensor-core workhorse behind every dense contraction on the ODISE
// inference hot path (SURVEY.md §8a rows a7.1 ResBlock convs, a7.2 transformer linears, a3 projections,
// b2-b4 pixel-decoder linears, b8-b10 decoder linears / mask einsum / pooling, b12 CLIP match).
//
//   D[z][m][n] = epi( alpha * sum_k A[z][m][k] * B[z][n][k] )        (both operands K-major, bf16)
//
// * A is either a row-major matrix (3-D tensor map {K, M, batch}) or, in conv mode, an NHWC activation read
//   through a 4-D tensor map {C, W, H, B}: the 3x3 / pad-1 / stride-1 convolution is an implicit GEMM whose
//   K loop walks (kh, kw, c-chunk) and lets TMA's out-of-bounds zero fill implement the padding.
//   (reference op: F.conv2d inside ldm ResBlock, call sites odise/modeling/meta_arch/ldm.py:481-489)
// * precision: NMMA=1 plain bf16, NMMA=3 "bf16x3": operands carry a (hi, lo) bf16 pair per fp32 value and the
//   kernel issues hi*hi + hi*lo + lo*hi into the same fp32 accumulator (~16 mantissa bits, the mode that
//   meets the 1e-3 fp32 parity bar of BASELINE.json; see DESIGN.md).  NMMA=2 "f16q8" (ptx.cuh, ODISE_PLANES_F16Q8):
//   hi = fp16 plane, second plane = e5m2 bytes [x * 2^-6 | (x - hi) * 2^6] per 64-wide k-block; per k-block 4 fp16
//   MMAs (hi*hi) + 4 e5m2 MMAs (the two cross terms, K = 32 each, twice the MAC rate) into the same accumulator:
//   8 instruction slots instead of 12, same shared-memory bytes, ~14 mantissa bits.  The e5m2 MMAs accumulate into a
//   register array of their own, added to the fp16 one at the end of the tile: an 8-bit wgmma adds into its accumulator
//   at reduced precision, which would truncate the hi*hi sum.  Two accumulators fit the register file up to BN = 128, so
//   F16Q8 runs 64- and 128-wide tiles.
// * persistent, warp-specialised: one TMA producer warp fills a ring of shared-memory stages; two consumer warpgroups
//   run wgmma on 64 rows each of a 128 x BN tile and then its epilogue (bias / per-image row bias / residual /
//   activation / GEGLU / GroupNorm records -> fp32 and/or (hi, lo) plane stores).
#include "ptx.cuh"
#include "wgmma.cuh"
#include "odise_b200.h"
#include "launch_count.h"
#include <cudaTypedefs.h>
#include <mutex>
#include <map>
#include <cstring>
#include <vector>
#include <cstdlib>
#include <cstdio>

namespace ob {

struct GemmParams {
  int M, N, K, batch;
  int a_batched, b_batched;
  int conv, C, H, W, bw, bh, bb;   // H, W: OUTPUT spatial dims of the conv
  int nseg;                        // > 1: the 128 pixels of a tile are fetched as nseg row segments of bw pixels
  int cstride, cpad;               // conv stride (1 | 2) and low-side zero padding (0 | 1)
  int tiles_m, tiles_n, splits, kblocks;
  float alpha;
  const float* bias;
  const float* bias_m;  // per-row (m) bias, for swapped-operand (transposed-output) projections
  const float* rowbias;
  int rows_per_group;
  long long rowbias_ld;
  const float* res;
  long long ldres, res_bs;
  float* D;
  long long ldd, d_bs;
  __nv_bfloat16* Dh;
  __nv_bfloat16* Dl;
  long long ldh, h_bs;
  int act;
  int geglu;   // N = 2*Nh with quad-interleaved (a, gate) columns: out[:, j] = a_j * gelu(g_j) -> planes [M, Nh]
  int vec_ok;  // all epilogue pointers / leading dims allow 16-byte vector access
  int h16;     // (hi, lo) output planes as fp16 instead of bf16 (V^T operand of the attention kernel)
               // (F16Q8 output planes: Dl carries the q8 tag of ptx.cuh, store_planes() does the rest)
  float* partial;  // [splits][batch][M][N] when splits > 1
  // GroupNorm statistics of the OUTPUT, fused into the epilogue (the consumer's torch.nn.GroupNorm, ldm ResBlock
  // in_layers[0] / out_layers[0], call sites ldm.py:481-489): per (32-row segment, column) a record (shift, S1, S2) with
  // shift = the segment's first row, S1 = sum(x - shift), S2 = sum((x - shift)^2) over the 32 rows.  Layout
  // gnp[seg * gnp_seg + {0,1,2} * gnp_plane + column]; odise_groupnorm_finalize_seg_f32 merges them per (image, group)
  // in fixed order (Chan's formula, double) -> no atomics, bit-reproducible, no second pass over the activation.
  float* gnp;
  long long gnp_seg, gnp_plane;
};

// 4 columns x the 4 rows a lane owns -> per-column (shift, S1, S2) of the warp's 32 rows; lanes 0..3 (rsub == 0) hold
// the result.  `first`: this call carries the rows it = 0 (row 0 of the segment sits in lanes 0..3).
struct GnAcc {
  float sh[4], s1[4], s2[4];
};
__device__ __forceinline__ void gn_acc_rows(GnAcc& a, const float (&e)[4], bool first, int lane) {
  if (first) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      a.sh[j] = __shfl_sync(0xffffffffu, e[j], lane & 3);
      a.s1[j] = 0.f; a.s2[j] = 0.f;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float d = e[j] - a.sh[j];
    a.s1[j] += d;
    a.s2[j] = fmaf(d, d, a.s2[j]);
  }
}
__device__ __forceinline__ void gn_acc_store(GnAcc& a, const GemmParams& p, long long seg, int col, int valid, int lane) {
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {        // fixed-order butterfly over the 8 row-lanes sharing a column quad
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      a.s1[j] += __shfl_xor_sync(0xffffffffu, a.s1[j], o);
      a.s2[j] += __shfl_xor_sync(0xffffffffu, a.s2[j], o);
    }
  }
  if ((lane >> 2) == 0 && valid > 0) {
    float* q = p.gnp + seg * p.gnp_seg + col;
    if (valid == 4 && ((p.gnp_plane | p.gnp_seg) & 3) == 0 && ((reinterpret_cast<uintptr_t>(q) & 15) == 0)) {
      *reinterpret_cast<float4*>(q) = make_float4(a.sh[0], a.sh[1], a.sh[2], a.sh[3]);
      *reinterpret_cast<float4*>(q + p.gnp_plane) = make_float4(a.s1[0], a.s1[1], a.s1[2], a.s1[3]);
      *reinterpret_cast<float4*>(q + 2 * p.gnp_plane) = make_float4(a.s2[0], a.s2[1], a.s2[2], a.s2[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < valid) { q[j] = a.sh[j]; q[p.gnp_plane + j] = a.s1[j]; q[2 * p.gnp_plane + j] = a.s2[j]; }
    }
  }
}

// exact-erf GELU with erf from Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, i.e. fp32 rounding level): one ex2, one
// rcp and six FMAs instead of libdevice's two-branch erff; used by the fused GEGLU epilogue (ldm GEGLU = F.gelu).
__device__ __forceinline__ float gelu_erf_fast(float v) {
  const float x = fabsf(v) * 0.70710678118654752f;
  const float t = __frcp_rn(fmaf(0.3275911f, x, 1.f));
  float pl = fmaf(1.061405429f, t, -1.453152027f);
  pl = fmaf(pl, t, 1.421413741f);
  pl = fmaf(pl, t, -0.284496736f);
  pl = fmaf(pl, t, 0.254829592f);
  const float er = 1.f - pl * t * exp2f(-1.4426950408889634f * x * x);   // erf(|v| / sqrt 2)
  return 0.5f * v * (1.f + copysignf(er, v));
}

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == ODISE_ACT_RELU) return fmaxf(v, 0.f);
  if (act == ODISE_ACT_SILU) return v / (1.f + __expf(-v));
  if (act == ODISE_ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  if (act == ODISE_ACT_QUICKGELU) return v / (1.f + __expf(-1.702f * v));   // open_clip QuickGELU
  return v;
}

// epilogue for 4 consecutive columns [n, n+4) of row m (n % 4 == 0); `valid` = how many of them exist (N tail)
__device__ __forceinline__ void epilogue_quad(const GemmParams& p, int z, int m, int n, int valid, float4 a4,
                                              float* final_vals = nullptr) {
  float acc[4] = {a4.x, a4.y, a4.z, a4.w};
  const bool vec = (valid == 4) && p.vec_ok;
  if (p.alpha != 1.f) {
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] *= p.alpha;
  }
  if (p.bias) {
    if (vec) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + n));
      acc[0] += b.x; acc[1] += b.y; acc[2] += b.z; acc[3] += b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (j < valid) acc[j] += __ldg(p.bias + n + j);
    }
  }
  if (p.bias_m) {
    const float bm = __ldg(p.bias_m + m);
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] += bm;
  }
  if (p.rowbias) {
    const float* rb = p.rowbias + (long long)(((long long)z * p.M + m) / p.rows_per_group) * p.rowbias_ld + n;
    if (vec) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(rb));
      acc[0] += b.x; acc[1] += b.y; acc[2] += b.z; acc[3] += b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (j < valid) acc[j] += __ldg(rb + j);
    }
  }
  if (p.act != ODISE_ACT_NONE) {
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = apply_act(acc[j], p.act);
  }
  if (p.res) {
    const float* r = p.res + (long long)z * p.res_bs + (long long)m * p.ldres + n;
    if (vec) {
      const float4 b = *reinterpret_cast<const float4*>(r);
      acc[0] += b.x; acc[1] += b.y; acc[2] += b.z; acc[3] += b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (j < valid) acc[j] += r[j];
    }
  }
  if (final_vals) {
#pragma unroll
    for (int j = 0; j < 4; ++j) final_vals[j] = acc[j];
  }
  if (p.D) {
    float* d = p.D + (long long)z * p.d_bs + (long long)m * p.ldd + n;
    if (vec) {
      *reinterpret_cast<float4*>(d) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (j < valid) d[j] = acc[j];
    }
  }
  if (p.Dh) {
    __nv_bfloat16* dh = p.Dh + (long long)z * p.h_bs + (long long)m * p.ldh + n;
    __nv_bfloat16* dl = p.Dl ? p.Dl + (long long)z * p.h_bs + (long long)m * p.ldh + n : nullptr;
    if (p.h16) {
      __align__(8) __nv_bfloat16 h[4];
      __align__(8) __nv_bfloat16 l[4];
#pragma unroll
      for (int t = 0; t < 4; ++t)
        split_f16(acc[t], *reinterpret_cast<uint16_t*>(&h[t]), *reinterpret_cast<uint16_t*>(&l[t]));
      if (vec) {
        *reinterpret_cast<uint2*>(dh) = *reinterpret_cast<const uint2*>(h);
        if (dl) *reinterpret_cast<uint2*>(dl) = *reinterpret_cast<const uint2*>(l);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) if (j < valid) { dh[j] = h[j]; if (dl) dl[j] = l[j]; }
      }
    } else if (vec) {
      store_planes<4>(dh, dl, acc);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (j < valid) store_planes<1>(dh + j, dl ? dl + j : nullptr, acc + j);
    }
  }
}

// Two consumer warpgroups (rows [0, 64) and [64, 128) of the tile, fp32 accumulators in registers) and a producer
// warpgroup whose first thread issues the TMA loads (the rest of it only hands its registers to the consumers).  The epilogue scatters the accumulator fragments, 32 columns at a time, into per-warp [32 rows x 16 fp32] staging
// blocks (XOR swizzled) so that every warp then owns 32 whole rows x 16 columns: coalesced global accesses (8 rows x 64
// contiguous bytes per warp-level access) and the 32-row GroupNorm segments.
template <int BN, int NMMA>
struct GemmCfg {
  static constexpr int BM = 128, BK = 64;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int PLANES = (NMMA == 1) ? 1 : 2;
  static constexpr int STAGE_BYTES = PLANES * (A_BYTES + B_BYTES);
  static constexpr int THREADS = 384;
  static constexpr int EPI_BYTES = 8 * 32 * 16 * 4;
  // 227 KB per block on H100, minus the epilogue staging, barriers and the slack for aligning the base to 1024 B
  static constexpr int STAGES_RAW = (232448 - EPI_BYTES - 256 - 1024) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 256 + 1024;
  static_assert(STAGES >= 2, "GEMM tile does not fit shared memory");
};

// EPI selects the compiled epilogue of the interior fast path (the runtime flags it excludes are guaranteed off by the
// host dispatch): 0 = lean (alpha, bias, activation -> fp32 and/or planes), 1 = + row bias / bias_m / residual,
// 2 = fused GEGLU.
template <int BN, int NMMA, int EPI>
__global__ void __launch_bounds__(GemmCfg<BN, NMMA>::THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
               const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl, const GemmParams p) {
  using Cfg = GemmCfg<BN, NMMA>;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* epi_smem = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES + Cfg::EPI_BYTES);
  uint64_t* full = bars;                       // [STAGES]
  uint64_t* empty = bars + Cfg::STAGES;        // [STAGES]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmAh);
    tma_prefetch_desc(&tmBh);
    if (NMMA != 1) {
      tma_prefetch_desc(&tmAl);
      tma_prefetch_desc(&tmBl);
    }
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // lane 0 of every consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int tiles_per_z = p.tiles_m * p.tiles_n * p.splits;
  const int total_tiles = tiles_per_z * p.batch;
  const int kb_per_split = (p.kblocks + p.splits - 1) / p.splits;

  if (warp >= 8) {
    setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      // ------------------------------------------------------------ TMA producer
      int stage = 0;
      uint32_t phase = 0;
      const int cpk = p.conv ? (p.C / 64) : 1;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int z = tile / tiles_per_z;
        int r = tile - z * tiles_per_z;
        const int sp = r / (p.tiles_m * p.tiles_n);
        r -= sp * (p.tiles_m * p.tiles_n);
        const int mt = r / p.tiles_n, nt = r % p.tiles_n;
        const int m0 = mt * 128, n0 = nt * BN;
        const int kb0 = sp * kb_per_split;
        const int kb1 = min(p.kblocks, kb0 + kb_per_split);
        int b0 = 0, h0 = 0, w0 = 0;
        if (p.conv) {
          const int hw = p.H * p.W;
          b0 = m0 / hw;
          const int rem = m0 - b0 * hw;
          h0 = rem / p.W;
          w0 = rem - h0 * p.W;
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* st = smem + stage * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
          if (p.conv) {
            const int tap = kb / cpk, cc = kb - tap * cpk;
            const int kh = tap / 3, kw = tap - kh * 3;
            if (p.nseg == 1) {
              const int cx = w0 * p.cstride + kw - p.cpad, cy = h0 * p.cstride + kh - p.cpad;
              tma_load_4d(st, &tmAh, &full[stage], cc * 64, cx, cy, b0);
              if (NMMA != 1) tma_load_4d(st + Cfg::A_BYTES, &tmAl, &full[stage], cc * 64, cx, cy, b0);
            } else {
              // widths that are neither a divisor nor a multiple of 128: raster-consecutive segments of
              // bw = gcd(W, 128) pixels never straddle an image row; each lands on its 8-row-aligned slice of the tile
              const int hw = p.H * p.W;
              for (int sg = 0; sg < p.nseg; ++sg) {
                const int m = m0 + sg * p.bw;
                const int bi = m / hw, rem = m - bi * hw;
                const int hi_ = rem / p.W, wi = rem - hi_ * p.W;
                const int cx = wi * p.cstride + kw - p.cpad, cy = hi_ * p.cstride + kh - p.cpad;
                uint8_t* sa = st + sg * p.bw * 128;
                tma_load_4d(sa, &tmAh, &full[stage], cc * 64, cx, cy, bi);
                if (NMMA != 1) tma_load_4d(sa + Cfg::A_BYTES, &tmAl, &full[stage], cc * 64, cx, cy, bi);
              }
            }
          } else {
            const int za = p.a_batched ? z : 0;
            tma_load_3d(st, &tmAh, &full[stage], kb * 64, m0, za);
            if (NMMA != 1) tma_load_3d(st + Cfg::A_BYTES, &tmAl, &full[stage], kb * 64, m0, za);
          }
          const int zb = p.b_batched ? z : 0;
          uint8_t* sb = st + Cfg::PLANES * Cfg::A_BYTES;
          tma_load_3d(sb, &tmBh, &full[stage], kb * 64, n0, zb);
          if (NMMA != 1) tma_load_3d(sb + Cfg::B_BYTES, &tmBl, &full[stage], kb * 64, n0, zb);
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ---------------------------------------------------------------- consumer warpgroups: MMAs, then the epilogue
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, wi = warp & 3;
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];
  float acc2[BN / 2];                          // F16Q8: the e5m2 cross terms
  float* stg_wg = epi_smem + wg * (4 * 512);   // the warpgroup's four [32 x 16] staging blocks
  float* stg = stg_wg + wi * 512;              // the block this warp reads back: rows (wi & 1) * 32, columns (wi >> 1) * 16
  const int cq = lane & 3, rsub = lane >> 2;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int z = tile / tiles_per_z;
    int r = tile - z * tiles_per_z;
    const int sp = r / (p.tiles_m * p.tiles_n);
    r -= sp * (p.tiles_m * p.tiles_n);
    const int mt = r / p.tiles_n, nt = r % p.tiles_n;
    const int n0 = nt * BN;
    const int kb0 = sp * kb_per_split;
    const int kb1 = min(p.kblocks, kb0 + kb_per_split);

    // ---- main loop: one k-block of MMAs in flight while the next stage is waited for
    if (kb0 >= kb1) {   // a split with no k-blocks contributes zeros
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      if constexpr (NMMA == 2) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc2[i] = 0.f;
      }
    }
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES) + wg * (64 * 128);
      const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::PLANES * Cfg::A_BYTES);
      reg_fence(acc);
      if constexpr (NMMA == 2) reg_fence(acc2);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t a_hi = wgmma_desc_sw128(sa + k * 32);
        const uint64_t b_hi = wgmma_desc_sw128(sb + k * 32);
        const int accum = (kb > kb0 || k > 0) ? 1 : 0;
        if constexpr (NMMA == 2) wgmma_f16(acc, a_hi, b_hi, accum);
        else wgmma_bf16(acc, a_hi, b_hi, accum);
        if constexpr (NMMA == 3) {
          wgmma_bf16(acc, a_hi, wgmma_desc_sw128(sb + Cfg::B_BYTES + k * 32), 1);
          wgmma_bf16(acc, wgmma_desc_sw128(sa + Cfg::A_BYTES + k * 32), b_hi, 1);
        }
      }
      if constexpr (NMMA == 2) {
        // cross terms on the 8-bit MMAs: the second plane of a stage is [q_hi: 64 B | q_lo: 64 B] per row, i.e. 32-byte
        // chunks 0,1 = q_hi(k 0..31 | 32..63), chunks 2,3 = q_lo;  A.q_hi * B.q_lo + A.q_lo * B.q_hi
        const uint32_t a2 = sa + Cfg::A_BYTES, b2 = sb + Cfg::B_BYTES;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          wgmma_e5m2(acc2, wgmma_desc_sw128(a2 + k * 32), wgmma_desc_sw128(b2 + 64 + k * 32), (kb > kb0 || k > 0) ? 1 : 0);
          wgmma_e5m2(acc2, wgmma_desc_sw128(a2 + 64 + k * 32), wgmma_desc_sw128(b2 + k * 32), 1);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                        // the previous k-block's MMAs are done: its stage may be refilled
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    if constexpr (NMMA == 2) {
      reg_fence(acc2);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] += acc2[i];
    }

    // ---- epilogue
    const int m_base = mt * 128 + wg * 64 + (wi & 1) * 32;
    const bool interior = p.vec_ok && p.splits == 1 && (mt * 128 + 128 <= p.M) && (n0 + BN <= p.N);
    constexpr bool EXTRA = EPI == 1, GEGLU = EPI == 2;
    const bool has_bias = p.bias != nullptr, has_res = EXTRA && p.res != nullptr;
    const bool to_f32 = p.D != nullptr, to_hi = p.Dh != nullptr, to_lo = p.Dl != nullptr;
    const int act = p.act;
    const float alpha = p.alpha;
    const bool has_gn = !GEGLU && p.gnp != nullptr;
    const long long gn_seg = ((long long)z * p.M + m_base) >> 5;
#pragma unroll 1
    for (int ch = 0; ch < BN / 32; ++ch) {
      named_bar_sync(1 + wg, 128);          // the previous chunk's staging has been read
      // fragment of n8 block j: rows wi * 16 + rsub (+ 8), columns 8 j + 2 cq (+ 1)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        if ((j >> 2) != ch) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rw = wi * 16 + rsub + 8 * h, cc = 8 * (j & 3) + 2 * cq;
          const int rr = rw & 31, c16 = cc & 15;
          float* dst = stg_wg + ((rw >> 5) | ((cc >> 4) << 1)) * 512 + rr * 16 + (((c16 >> 2) ^ ((rr >> 1) & 3)) << 2) + (c16 & 3);
          *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
      named_bar_sync(1 + wg, 128);
      const int c0 = ch * 32 + (wi >> 1) * 16;
      if (interior) {
        // fast path: whole tile in range, vector accesses; per-row offsets hoisted out of the column loop
        GnAcc gacc;
        float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (has_bias) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n0 + c0 + cq * 4));
        float4 q[4];
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int rr = it * 8 + rsub;
          q[it] = *reinterpret_cast<const float4*>(stg + rr * 16 + ((cq ^ ((rr >> 1) & 3)) << 2));
        }
        const int nn = n0 + c0 + cq * 4;
        float4 r4[4];
        if (has_res) {
#pragma unroll
          for (int it = 0; it < 4; ++it)
            r4[it] = *reinterpret_cast<const float4*>(p.res + (long long)z * p.res_bs + (long long)(m_base + it * 8 + rsub) * p.ldres + nn);
        }
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const long long m = m_base + it * 8 + rsub;
          float e[4] = {q[it].x, q[it].y, q[it].z, q[it].w};
          const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
          const float bm = (EXTRA && p.bias_m) ? __ldg(p.bias_m + m) : 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) e[j] = fmaf(e[j], alpha, EXTRA ? bb[j] + bm : bb[j]);
          if (EXTRA && p.rowbias) {
            const float4 rb = __ldg(reinterpret_cast<const float4*>(
                p.rowbias + (((long long)z * p.M + m) / p.rows_per_group) * p.rowbias_ld + nn));
            e[0] += rb.x; e[1] += rb.y; e[2] += rb.z; e[3] += rb.w;
          }
          if (GEGLU) {
            // ldm GEGLU fused: lanes with even cq hold 4 `a` values, their xor-1 partner the 4 gates of the same
            // channels (weight rows were quad-interleaved at load time); output planes have N/2 columns
            // both partners work: the even lane finishes channels 0,1 of the quad, the odd lane channels 2,3
            const bool odd = cq & 1;
            const float r0 = __shfl_xor_sync(0xffffffffu, odd ? e[0] : e[2], 1);
            const float r1 = __shfl_xor_sync(0xffffffffu, odd ? e[1] : e[3], 1);
            const float a0 = odd ? r0 : e[0], a1 = odd ? r1 : e[1];
            const float g0 = odd ? e[2] : r0, g1 = odd ? e[3] : r1;
            const float gv[2] = {a0 * gelu_erf_fast(g0), a1 * gelu_erf_fast(g1)};
            const long long og = (long long)z * p.h_bs + m * p.ldh + ((n0 + c0) >> 1) + (cq >> 1) * 4 + (odd ? 2 : 0);
            store_planes<2>(p.Dh + og, to_lo ? p.Dl + og : nullptr, gv);
            continue;
          }
          if (act != ODISE_ACT_NONE) {
#pragma unroll
            for (int j = 0; j < 4; ++j) e[j] = apply_act(e[j], act);
          }
          if (has_res) { e[0] += r4[it].x; e[1] += r4[it].y; e[2] += r4[it].z; e[3] += r4[it].w; }
          if (has_gn) gn_acc_rows(gacc, e, it == 0, lane);
          if (to_f32) *reinterpret_cast<float4*>(p.D + (long long)z * p.d_bs + m * p.ldd + nn) = make_float4(e[0], e[1], e[2], e[3]);
          const long long oh = (long long)z * p.h_bs + m * p.ldh + nn;
          if (to_hi && p.h16) {
            // fp16 (hi, lo) planes: the V^T operand of the attention kernel's P V product
            const __half2 h01 = __floats2half2_rn(e[0], e[1]), h23 = __floats2half2_rn(e[2], e[3]);
            uint2 hv;
            hv.x = *reinterpret_cast<const uint32_t*>(&h01);
            hv.y = *reinterpret_cast<const uint32_t*>(&h23);
            *reinterpret_cast<uint2*>(p.Dh + oh) = hv;
            if (to_lo) {
              const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
              const __half2 l01 = __floats2half2_rn(e[0] - f01.x, e[1] - f01.y);
              const __half2 l23 = __floats2half2_rn(e[2] - f23.x, e[3] - f23.y);
              uint2 lv;
              lv.x = *reinterpret_cast<const uint32_t*>(&l01);
              lv.y = *reinterpret_cast<const uint32_t*>(&l23);
              *reinterpret_cast<uint2*>(p.Dl + oh) = lv;
            }
          } else if (to_hi) {
            // bf16 pair (packed conversions, same values as split_bf16) or, when Dl carries the tag, fp16 + e5m2 bytes
            store_planes<4>(p.Dh + oh, to_lo ? p.Dl + oh : nullptr, e);
          }
        }
        if (has_gn) gn_acc_store(gacc, p, gn_seg, n0 + c0 + cq * 4, 4, lane);
      } else if (n0 + c0 < p.N) {   // warp-uniform
        // fused GroupNorm statistics on edge tiles: whole 32-row segments only (M % 32 == 0 is checked on the host)
        const bool gn_here = p.gnp != nullptr && !p.geglu && p.splits == 1 && m_base < p.M;
        GnAcc gacc;
#pragma unroll 1
        for (int it = 0; it < 4; ++it) {
          const int rr = it * 8 + rsub;
          const float4 q4 = *reinterpret_cast<const float4*>(stg + rr * 16 + ((cq ^ ((rr >> 1) & 3)) << 2));
          const int m = m_base + rr, n = n0 + c0 + cq * 4;
          if (p.geglu) {   // warp-uniform; N % 16 == 0 so a chunk is either fully valid or skipped above
            float e[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) e[j] = fmaf(e[j], p.alpha, p.bias ? __ldg(p.bias + n + j) : 0.f);
            float gt[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) gt[j] = __shfl_xor_sync(0xffffffffu, e[j], 1);
            if ((cq & 1) == 0 && m < p.M) {
              float gv[4];
#pragma unroll
              for (int t = 0; t < 4; ++t) gv[t] = e[t] * gelu_erf_fast(gt[t]);
              const long long og = (long long)z * p.h_bs + (long long)m * p.ldh + ((n0 + c0) >> 1) + (cq >> 1) * 4;
              store_planes<4>(p.Dh + og, p.Dl ? p.Dl + og : nullptr, gv);
            }
            continue;
          }
          float fin[4] = {0.f, 0.f, 0.f, 0.f};
          if (m < p.M && n < p.N) {
            const int valid = min(4, p.N - n);
            if (p.splits > 1) {
              float* dst = p.partial + ((long long)(sp * p.batch + z) * p.M + m) * p.N + n;
              const float e[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
              for (int j = 0; j < 4; ++j) if (j < valid) dst[j] = e[j];
            } else {
              epilogue_quad(p, z, m, n, valid, q4, fin);
            }
          }
          if (gn_here) gn_acc_rows(gacc, fin, it == 0, lane);      // warp-uniform: all lanes shuffle
        }
        if (gn_here) {
          const int n = n0 + c0 + cq * 4;
          gn_acc_store(gacc, p, ((long long)z * p.M + m_base) >> 5, n, n < p.N ? min(4, p.N - n) : 0, lane);
        }
      }
    }
  }
}

// split-K second pass: sum the partials and run the normal epilogue (4 columns per thread)
__global__ void gemm_splitk_reduce_kernel(const GemmParams p) {
  const int quads = (p.N + 3) / 4;
  const long long total = (long long)p.batch * p.M * quads;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int qd = (int)(i % quads);
    const long long zm = i / quads;
    const int m = (int)(zm % p.M);
    const int z = (int)(zm / p.M);
    const int n = qd * 4;
    const int valid = min(4, p.N - n);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int sp = 0; sp < p.splits; ++sp) {
      const float* src = p.partial + ((long long)(sp * p.batch + z) * p.M + m) * p.N + n;
#pragma unroll
      for (int j = 0; j < 4; ++j) if (j < valid) acc[j] += src[j];
    }
    epilogue_quad(p, z, m, n, valid, make_float4(acc[0], acc[1], acc[2], acc[3]));
  }
}

// ------------------------------------------------------------------------------------------------ host side
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
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

static int encode_map(CUtensorMap* tm, const void* base, int rank, const cuuint64_t* dims,
                      const cuuint64_t* strides_bytes, const cuuint32_t* box, int spatial_stride = 1) {
  auto enc = get_encode();
  if (!enc) return ODISE_ERR_DRIVER;
  // strided implicit conv: W and H (dims 1, 2) are traversed with element stride 2
  cuuint32_t estr[5] = {1, (cuuint32_t)spatial_stride, (cuuint32_t)spatial_stride, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides_bytes, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? ODISE_OK : ODISE_ERR_TENSORMAP;
}

// ---- optional per-launch timing (bench.py roofline): CUDA events on the launch stream around every GEMM launch
struct ProfRec { cudaEvent_t a, b; double flops; int M, N, K, batch, conv, bn, nmma, splits; };
static std::vector<ProfRec> g_prof;
static bool g_prof_on = false;

int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

template <int BN, int NMMA, int EPI>
static int launch_cfg(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl,
                      const GemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN, NMMA>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<BN, NMMA, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int total = p.tiles_m * p.tiles_n * p.splits * p.batch;
  const int grid = total < num_sms() ? total : num_sms();
  gemm_tc_kernel<BN, NMMA, EPI><<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(ah, al, bh, bl, p);
  return (int)cudaGetLastError();
}

// Tile choice: output-tile width BN.  eff = shared-memory operand bytes per MAC of a warpgroup's 64 x BN wgmma tile
// ((64 + BN) / (64 BN)), relative to BN = 128: wider tiles re-read A less often.  The per-shape autotune in
// odise_gemm_bf16 replaces this estimate wherever it may launch trial runs.
static int pick_tile(int M, int N, int K, int batch, int forced, bool conv, int nmma) {
  const int cands[4] = {256, 160, 128, 64};
  const double eff[4] = {0.833, 0.933, 1.0, 1.333};
  const double epi_k = 480.0;    // epilogue of a tile in units of MMA k
  const long long tm = (M + 127) / 128;
  double best = 1e30;
  int c = 128;
  for (int i = 0; i < 4; ++i) {
    const int bn = cands[i];
    if (forced && bn != forced) continue;
    if (nmma == 2 && bn > 128) continue;
    const long long tn = (N + bn - 1) / bn;
    const long long units = tm * tn * batch;
    const long long waves = (units + num_sms() - 1) / num_sms();
    double cost;
    if (conv) {          // implicit convs (K >= 576): main-loop bound at every width -> balance waves
      cost = (double)waves * bn * eff[i] + 0.02 * bn;            // mild bias toward smaller tiles on ties
    } else {             // plain GEMMs: per-tile time = max(main loop, epilogue) + fixed fill / drain
      const double mma = (double)bn * K * eff[i], epi = (double)bn * epi_k;
      cost = (double)waves * ((mma > epi ? mma : epi) + 20000.0);
    }
    if (cost < best) { best = cost; c = bn; }
  }
  return c;
}

}  // namespace ob

using namespace ob;

extern "C" int odise_gemm_bf16(const odise_gemm_desc* d, void* stream_v) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  if (!d || !d->a_hi || !d->b_hi) return ODISE_ERR_ARG;
  if (d->nmma != 1 && d->nmma != 2 && d->nmma != 3) return ODISE_ERR_ARG;
  if (d->nmma != 1 && (!d->a_lo || !d->b_lo)) return ODISE_ERR_ARG;
  if (d->M <= 0 || d->N <= 0 || d->K <= 0 || d->batch <= 0) return ODISE_ERR_ARG;
  if (!d->out_f32 && !d->out_hi) return ODISE_ERR_ARG;

  GemmParams p{};
  p.M = d->M; p.N = d->N; p.K = d->K; p.batch = d->batch;
  p.a_batched = d->a_batch_stride != 0; p.b_batched = d->b_batch_stride != 0;
  p.conv = d->conv3x3; p.C = d->conv_C; p.H = d->conv_H; p.W = d->conv_W;
  p.alpha = d->alpha;
  p.bias = d->bias; p.bias_m = d->bias_m; p.rowbias = d->rowbias; p.rows_per_group = d->rows_per_group > 0 ? d->rows_per_group : 1;
  p.rowbias_ld = d->rowbias_ld;
  p.res = d->residual; p.ldres = d->ld_residual; p.res_bs = d->residual_batch_stride;
  p.D = d->out_f32; p.ldd = d->ld_out; p.d_bs = d->out_batch_stride;
  p.Dh = reinterpret_cast<__nv_bfloat16*>(d->out_hi); p.Dl = reinterpret_cast<__nv_bfloat16*>(d->out_lo);
  p.ldh = d->ld_out_bf16; p.h_bs = d->out_bf16_batch_stride;
  p.act = d->act;
  p.geglu = d->geglu;
  p.h16 = d->out_planes_fp16 == ODISE_PLANES_F16 ? 1 : 0;
  if (p.h16 && (d->geglu || !d->out_hi)) return ODISE_ERR_UNSUPPORTED;
  const bool oq8 = d->out_planes_fp16 == ODISE_PLANES_F16Q8 && d->out_hi;
  if (d->out_planes_fp16 < 0 || d->out_planes_fp16 > 2) return ODISE_ERR_ARG;
  if (oq8) {   // F16Q8 output planes: both planes, rows on 128-byte boundaries (store_planes reads k % 64 off the address)
    if (!d->out_lo || d->ld_out_bf16 % 64 || d->out_bf16_batch_stride % 64 || (reinterpret_cast<uintptr_t>(d->out_lo) & 127))
      return ODISE_ERR_ALIGN;
    p.Dl = tag_q8(p.Dl);
  }
  if (d->gn_partial) {
    // whole 32-row segments, final values produced by this kernel (no split-K second pass, no GEGLU re-pairing)
    if (d->M % 32 || d->split_k > 1 || d->geglu || d->gn_seg_stride <= 0 || d->gn_plane_stride <= 0)
      return ODISE_ERR_UNSUPPORTED;
    p.gnp = d->gn_partial; p.gnp_seg = d->gn_seg_stride; p.gnp_plane = d->gn_plane_stride;
  }

  // vector epilogue paths need 16-byte alignment; otherwise the kernel takes the scalar path
  {
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    bool ok = true;
    if (d->out_f32) ok = ok && d->ld_out % 4 == 0 && d->out_batch_stride % 4 == 0 && al16(d->out_f32);
    if (d->residual) ok = ok && d->ld_residual % 4 == 0 && d->residual_batch_stride % 4 == 0 && al16(d->residual);
    if (d->out_hi) ok = ok && d->ld_out_bf16 % 8 == 0 && d->out_bf16_batch_stride % 8 == 0 && al16(d->out_hi) &&
                        (!d->out_lo || al16(d->out_lo));
    if (d->rowbias) ok = ok && d->rowbias_ld % 4 == 0 && al16(d->rowbias);
    if (d->bias) ok = ok && al16(d->bias);
    p.vec_ok = ok ? 1 : 0;
  }

  CUtensorMap ah, al, bh, bl;
  int rc;
  if (p.conv) {
    if (p.C % 64 || d->K != 9 * p.C || d->batch != 1) return ODISE_ERR_ARG;
    // conv_mode 0: stride 1, pad 1 | 1: stride 2, pad (1,1) (ldm Downsample) | 2: stride 2, pad (0,1) (VAE Downsample)
    if (d->conv_mode < 0 || d->conv_mode > 2) return ODISE_ERR_ARG;
    p.cstride = d->conv_mode == 0 ? 1 : 2;
    p.cpad = d->conv_mode == 2 ? 0 : 1;
    const int Hin = d->conv_H, Win = d->conv_W;
    if (Hin % p.cstride || Win % p.cstride) return ODISE_ERR_ARG;
    p.H = Hin / p.cstride; p.W = Win / p.cstride;      // output dims: tiles walk output pixels
    const int hw = p.H * p.W;
    if (d->M % hw) return ODISE_ERR_ARG;
    const int B = d->M / hw;
    p.nseg = 1;
    bool boxed = false;
    if (p.W % 128 == 0) {
      p.bw = 128; p.bh = 1; p.bb = 1;
      boxed = true;
    } else if (128 % p.W == 0) {
      p.bw = p.W;
      p.bh = 128 / p.W < p.H ? 128 / p.W : p.H;
      if (p.H % p.bh == 0 && 128 % (p.bw * p.bh) == 0) {
        p.bb = 128 / (p.bw * p.bh);
        boxed = true;
      }
    }
    if (!boxed) {                       // general widths (e.g. 160 = 640 / 4): segmented fetch
      int g = p.W, r = 128;
      while (r) { const int t = g % r; g = r; r = t; }
      if (g % 8) return ODISE_ERR_UNSUPPORTED;
      p.bw = g; p.bh = 1; p.bb = 1; p.nseg = 128 / g;
    }
    const long long pix = d->lda;  // elements between consecutive pixels (>= C: channel slices of wider buffers)
    if (pix < p.C || pix % 8) return ODISE_ERR_ALIGN;
    cuuint64_t dims[4] = {(cuuint64_t)p.C, (cuuint64_t)Win, (cuuint64_t)Hin, (cuuint64_t)B};
    cuuint64_t str[3] = {(cuuint64_t)pix * 2, (cuuint64_t)pix * Win * 2, (cuuint64_t)pix * Hin * Win * 2};
    // with element stride s the box spans bw*s input columns and yields bw of them
    cuuint32_t box[4] = {64, (cuuint32_t)(p.bw * p.cstride), (cuuint32_t)(p.bh * p.cstride), (cuuint32_t)p.bb};
    rc = encode_map(&ah, d->a_hi, 4, dims, str, box, p.cstride);
    if (rc) return rc;
    rc = encode_map(&al, d->nmma != 1 ? d->a_lo : d->a_hi, 4, dims, str, box, p.cstride);
    if (rc) return rc;
  } else {
    if (d->lda % 8 || d->a_batch_stride % 8) return ODISE_ERR_ALIGN;
    const long long bs = d->a_batch_stride ? d->a_batch_stride : (long long)d->M * d->lda;
    cuuint64_t dims[3] = {(cuuint64_t)d->K, (cuuint64_t)d->M, (cuuint64_t)(d->a_batch_stride ? d->batch : 1)};
    cuuint64_t str[2] = {(cuuint64_t)d->lda * 2, (cuuint64_t)bs * 2};
    cuuint32_t box[3] = {64, 128, 1};
    rc = encode_map(&ah, d->a_hi, 3, dims, str, box);
    if (rc) return rc;
    if (d->nmma == 2) {   // the q bytes of the last (partial) k-block occupy its whole 128-byte slot
      dims[0] = (cuuint64_t)((d->K + 63) / 64 * 64);
      if ((long long)dims[0] > d->lda) return ODISE_ERR_ALIGN;
    }
    rc = encode_map(&al, d->nmma != 1 ? d->a_lo : d->a_hi, 3, dims, str, box);
    if (rc) return rc;
  }
  p.tiles_m = (d->M + 127) / 128;
  if (d->ldb % 8 || d->b_batch_stride % 8) return ODISE_ERR_ALIGN;
  if (d->nmma == 2 && (long long)((d->K + 63) / 64 * 64) > d->ldb) return ODISE_ERR_ALIGN;
  if (d->geglu) {
    // fused GEGLU: (a, gate) quads must share a 16-column chunk; 8-byte plane stores need the aligned path
    if (!d->out_hi || d->out_f32 || d->residual || d->rowbias || d->bias_m || d->split_k > 1 || d->N % 16 ||
        !p.vec_ok || d->act != ODISE_ACT_NONE)
      return ODISE_ERR_UNSUPPORTED;
  }
  p.kblocks = (d->K + 63) / 64;
  p.splits = d->split_k > 1 ? d->split_k : 1;
  if (p.splits > p.kblocks) p.splits = p.kblocks;
  if (p.splits > 1) {
    if (!d->workspace ||
        d->workspace_bytes < (long long)p.splits * d->batch * d->M * d->N * (long long)sizeof(float))
      return ODISE_ERR_WORKSPACE;
    p.partial = reinterpret_cast<float*>(d->workspace);
  }
  const int epi = d->geglu ? 2 : ((d->residual || d->rowbias || d->bias_m) ? 1 : 0);

  // one launch with a given output-tile width: B tensor map (box = bn rows) + dispatch
  auto launch_with = [&](int bn) -> int {
    p.tiles_n = (d->N + bn - 1) / bn;
    const long long bs = d->b_batch_stride ? d->b_batch_stride : (long long)d->N * d->ldb;
    cuuint64_t dims[3] = {(cuuint64_t)d->K, (cuuint64_t)d->N, (cuuint64_t)(d->b_batch_stride ? d->batch : 1)};
    cuuint64_t str[2] = {(cuuint64_t)d->ldb * 2, (cuuint64_t)bs * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)bn, 1};
    int r = encode_map(&bh, d->b_hi, 3, dims, str, box);
    if (r) return r;
    if (d->nmma == 2) dims[0] = (cuuint64_t)((d->K + 63) / 64 * 64);   // whole 64-blocks of q bytes
    r = encode_map(&bl, d->nmma != 1 ? d->b_lo : d->b_hi, 3, dims, str, box);
    if (r) return r;
#define ODISE_LAUNCH(BN_, NM_)                                                   \
  r = epi == 2   ? launch_cfg<BN_, NM_, 2>(ah, al, bh, bl, p, stream)            \
      : epi == 1 ? launch_cfg<BN_, NM_, 1>(ah, al, bh, bl, p, stream)            \
                 : launch_cfg<BN_, NM_, 0>(ah, al, bh, bl, p, stream)
    if (d->nmma == 3) {
      switch (bn) {
        case 64: ODISE_LAUNCH(64, 3); break;
        case 128: ODISE_LAUNCH(128, 3); break;
        case 160: ODISE_LAUNCH(160, 3); break;
        default: ODISE_LAUNCH(256, 3); break;
      }
    } else if (d->nmma == 2) {
      if (bn == 64) ODISE_LAUNCH(64, 2);
      else ODISE_LAUNCH(128, 2);
    } else {
      switch (bn) {
        case 64: ODISE_LAUNCH(64, 1); break;
        case 128: ODISE_LAUNCH(128, 1); break;
        case 160: ODISE_LAUNCH(160, 1); break;
        default: ODISE_LAUNCH(256, 1); break;
      }
    }
#undef ODISE_LAUNCH
    if (r) return r;
    if (p.splits > 1) {
      const long long total = (long long)p.batch * p.M * ((p.N + 3) / 4);
      int blocks = (int)((total + 127) / 128);
      if (blocks > num_sms() * 8) blocks = num_sms() * 8;
      gemm_splitk_reduce_kernel<<<blocks, 128, 0, stream>>>(p);
      r = (int)cudaGetLastError();
    }
    return r;
  };

  // ---- tile width: a per-shape autotune (every candidate is the same arithmetic in the same k order -> bit-identical
  // results, so the choice is free) with the cost model pick_tile() as the fallback under stream capture.
  // ODISE_GEMM_AUTOTUNE=0: cost model only.
  int BN;
  {
    static const bool tune = !(getenv("ODISE_GEMM_AUTOTUNE") && atoi(getenv("ODISE_GEMM_AUTOTUNE")) == 0);
    const int fbn = (d->force_bn == 64 || d->force_bn == 128 || d->force_bn == 160 || d->force_bn == 256) ? d->force_bn : 0;
    BN = pick_tile(d->M, d->N, d->K, d->batch, fbn, d->conv3x3 != 0, d->nmma);
    struct Key {
      int v[13];
      bool operator<(const Key& o) const { return memcmp(v, o.v, sizeof(v)) < 0; }
    };
    static std::map<Key, int> cache;
    static std::mutex mu;
    const Key key{{d->M, d->N, d->K, d->batch, d->conv3x3 ? 1 + d->conv_mode : 0, d->conv_W, d->nmma, epi, p.splits,
                  (d->out_f32 ? 1 : 0) | (d->out_hi ? 2 : 0) | (d->out_planes_fp16 << 2), p.gnp ? 1 : 0, d->act, p.vec_ok}};
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(stream, &cap);
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
      BN = it->second;
    } else if (tune && !fbn && !g_prof_on && cap == cudaStreamCaptureStatusNone &&
               !(d->residual && (const void*)d->residual == (const void*)d->out_f32)) {
      // candidates from wide to narrow (64 only for narrow outputs)
      const int cands[4] = {256, 160, 128, 64};
      cudaEvent_t e0, e1;
      cudaEventCreate(&e0);
      cudaEventCreate(&e1);
      float best = 1e30f;
      int bc = BN;
      for (int i = 0; i < 4; ++i) {
        const int c = cands[i];
        // 64-wide tiles: narrow outputs, or problems too small to fill the SMs with wider ones (decoder linears)
        if (c == 64 && d->N > 96 && (long long)p.tiles_m * ((d->N + 127) / 128) * d->batch >= 2 * num_sms()) continue;
        if (c > 128 && (d->N <= 64 || d->nmma == 2)) continue;
        if (launch_with(c)) { (void)cudaGetLastError(); continue; }     // warm (attributes, L2)
        cudaEventRecord(e0, stream);
        int r2 = launch_with(c);
        if (!r2) r2 = launch_with(c);
        cudaEventRecord(e1, stream);
        if (r2 || cudaEventSynchronize(e1) != cudaSuccess) { (void)cudaGetLastError(); continue; }
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) { best = ms; bc = c; }
      }
      cudaEventDestroy(e0);
      cudaEventDestroy(e1);
      cache[key] = bc;
      BN = bc;
      if (getenv("ODISE_VERBOSE"))
        fprintf(stderr, "odise_b200: gemm %d x %d x %d (batch %d, conv %d, nmma %d, epi %d): BN %d, %.1f us\n", d->M, d->N,
                d->K, d->batch, d->conv3x3, d->nmma, epi, BN, best * 500.f);
    }
  }

  ProfRec rec{};
  if (g_prof_on) {
    cudaEventCreate(&rec.a);
    cudaEventCreate(&rec.b);
    rec.flops = 2.0 * d->M * d->N * (double)d->K * d->batch;
    rec.M = d->M; rec.N = d->N; rec.K = d->K; rec.batch = d->batch; rec.conv = d->conv3x3; rec.bn = BN;
    rec.nmma = d->nmma; rec.splits = p.splits;
    cudaEventRecord(rec.a, stream);
  }
  rc = launch_with(BN);
  if (rc) return rc;
  count_launch(p.splits > 1 ? 2 : 1);
  if (g_prof_on) {
    cudaEventRecord(rec.b, stream);
    g_prof.push_back(rec);
  }
  return rc;
}

// The cost-model choice of odise_gemm_bf16 for a problem (what it uses under stream capture / with ODISE_GEMM_AUTOTUNE=0, and
// the starting point of the per-shape autotune): the output-tile width.  *pair reports CTA pairs, which the sm_90a kernel
// does not use (always 0).  Host only.
extern "C" int odise_gemm_tile_policy(int M, int N, int K, int batch, int conv3x3, int nmma, int* bn, int* pair) {
  if (M <= 0 || N <= 0 || K <= 0 || batch <= 0 || !bn || !pair || nmma < 1 || nmma > 3) return ODISE_ERR_ARG;
  *bn = pick_tile(M, N, K, batch, 0, conv3x3 != 0, nmma);
  *pair = 0;
  return ODISE_OK;
}

extern "C" int odise_profile_begin(void) {
  for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_prof.clear();
  g_prof_on = true;
  return ODISE_OK;
}

// stops recording; returns launches, summed device ms and summed algorithmic FLOPs (2*M*N*K*batch) of the GEMMs;
// if the environment variable ODISE_PROFILE_CSV names a file, one line per launch is appended to it
extern "C" int odise_profile_end(long long* launches, double* total_ms, double* total_flops) {
  g_prof_on = false;
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return (int)e;
  double ms = 0, fl = 0;
  FILE* fcsv = nullptr;
  if (const char* path = getenv("ODISE_PROFILE_CSV")) fcsv = fopen(path, "a");
  if (fcsv) fprintf(fcsv, "M,N,K,batch,conv,bn,nmma,splits,ms,tflops\n");
  for (auto& r : g_prof) {
    float t = 0;
    cudaEventElapsedTime(&t, r.a, r.b);
    ms += t;
    fl += r.flops;
    if (fcsv)
      fprintf(fcsv, "%d,%d,%d,%d,%d,%d,%d,%d,%.4f,%.1f\n", r.M, r.N, r.K, r.batch, r.conv, r.bn, r.nmma, r.splits, t,
              r.flops / (t * 1e9));
  }
  if (fcsv) fclose(fcsv);
  if (launches) *launches = (long long)g_prof.size();
  if (total_ms) *total_ms = ms;
  if (total_flops) *total_flops = fl;
  for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_prof.clear();
  return ODISE_OK;
}
