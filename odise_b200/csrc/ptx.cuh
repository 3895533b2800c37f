// Hopper (sm_90a) PTX wrappers shared by every kernel TU: mbarrier, TMA, wgmma.
// Nothing here is ported from the reference (which has no sm_90 code at all, SURVEY.md §2.4);
// bit layouts follow the PTX ISA (wgmma matrix descriptors, tensor-map swizzle modes).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#include <stdio.h>

namespace ob {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug must abort the kernel (trap -> launch error), never hang the box.  No printf here: a
// function call inside a kernel that runs wgmma makes ptxas serialise the MMAs.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();   // ~2 s at 2 GHz
  }
}
// warpgroup-wide register budget (all four warps of the warpgroup execute it): the TMA producer gives registers back,
// the MMA warpgroups take them
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}

// ---------------------------------------------------------------- TMA (cp.async.bulk.tensor)
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA, accumulators in registers)
// named barrier over `threads` threads (a multiple of 32); ids 1.. (0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// orders this thread's register / shared-memory writes before the wgmma that follow (accumulators, register A fragments)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N committed groups of this warpgroup still in flight (their accumulators / operands are then free)
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major operand tile in the canonical SWIZZLE_128B layout: rows of 128 B (64 16-bit or 128 8-bit elements), 8-row /
// 1024 B swizzle atoms stacked along M/N (SBO = 1024 B); LBO is unused for swizzled K-major (CUTLASS writes 1).  A step of
// 16 (16-bit) or 32 (8-bit) elements along K inside the atom adds 32 bytes to the start address.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);   // [0,14)  start address >> 4
  d |= static_cast<uint64_t>(1) << 16;                       // [16,30) LBO >> 4
  d |= static_cast<uint64_t>(1024 >> 4) << 32;               // [32,46) SBO >> 4
  d |= static_cast<uint64_t>(1) << 62;                       // [62,64) SWIZZLE_128B
  return d;
}

// fp32 -> (hi, lo) bf16 pair with hi + lo ~= x to ~16 mantissa bits (the "bf16x3" operand split)
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// the same split into an fp16 pair (11 + 11 mantissa bits; operands of the attention P V product)
__device__ __forceinline__ void split_f16(float x, uint16_t& hi, uint16_t& lo) {
  const __half h = __float2half_rn(x);
  const __half l = __float2half_rn(x - __half2float(h));
  hi = __half_as_ushort(h);
  lo = __half_as_ushort(l);
}

// ------------------------------------------------------------------------------------------------ operand planes
// Three formats of the (hi, lo) operand planes of an fp32 matrix [rows, K] (ODISE_PLANES_* in odise_b200.h):
//   BF16  hi = bf16(x), lo = bf16(x - hi)                         -> bf16x3: hi*hi + hi*lo + lo*hi, 3 bf16 MMAs
//   F16   the same with fp16 words (V^T of the attention kernel)
//   F16Q8 hi = fp16(x);  the second plane has the SAME byte geometry (2 bytes per element, same row stride) but holds,
//         per block of 64 consecutive k, 64 bytes q_hi[k] = e5m2(x * 2^-S) followed by 64 bytes
//         q_lo[k] = e5m2((x - hi) * 2^S), S = kQ8Shift.  A GEMM in this format issues, per 64-wide k-block,
//         4 x fp16 k16 MMAs (A_hi * B_hi) + 4 x e5m2 k32 MMAs (A.q_hi * B.q_lo and A.q_lo * B.q_hi, the two first-order
//         correction terms; the power-of-two scales cancel; the 8-bit MMAs run at twice the rate) into one fp32
//         accumulator.  Error per product ~2^-14 (e5m2 keeps 3 significant bits of a term that is itself 2^-12 of
//         the product) vs 2^-16 for bf16x3; UNet taps 1.1e-4 vs 2e-5 against the fp32 oracle (tools/precision_budget.py),
//         bar 1e-3.  Out-of-range values degrade gracefully: a saturated / flushed q byte only perturbs a 2^-12 term.
// Rows of F16Q8 planes start on 128-byte boundaries (ld % 64 == 0, checked by the host), so the position of an element
// inside its k-block can be read off its address; device code receives the second plane's pointer with bit 0 set as the
// format tag (set by the launchers from odise_set_operand_format(), never part of the C ABI).
constexpr int kQ8Shift = 6;
constexpr float kQ8Down = 1.f / 64.f, kQ8Up = 64.f;   // 2^-S, 2^S

__host__ __device__ __forceinline__ bool lo_is_q8(const void* lo) { return (reinterpret_cast<uintptr_t>(lo) & 1u) != 0; }
template <typename T>
__host__ __device__ __forceinline__ T* tag_q8(T* lo) {
  return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(lo) | 1u);
}
// two floats -> two e5m2 bytes (first value in the low byte), round-to-nearest, saturating to +-57344
__device__ __forceinline__ uint32_t e5m2x2(float a, float b) {
  return (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E5M2);
}
__device__ __forceinline__ float clamp_f16(float x) { return fminf(fmaxf(x, -65504.f), 65504.f); }

// N (1, 2, 4 or 8) consecutive columns starting at a column that is a multiple of N: `hi` / `lo` point AT the first element
// (2-byte element units in both planes).  lo == nullptr: hi plane only (bf16).  Tagged lo: F16Q8.
template <int N>
__device__ __forceinline__ void store_planes(__nv_bfloat16* hi, __nv_bfloat16* lo, const float* v) {
  static_assert(N == 1 || N == 2 || N == 4 || N == 8, "vector width");
  if (lo_is_q8(lo)) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(lo) & ~static_cast<uintptr_t>(1);
    uint8_t* q = reinterpret_cast<uint8_t*>(a - ((a >> 1) & 63u));   // block base + (column % 64)
    if constexpr (N == 1) {
      const __half h = __float2half_rn(clamp_f16(v[0]));
      *reinterpret_cast<__half*>(hi) = h;
      const uint32_t w = e5m2x2(v[0] * kQ8Down, (v[0] - __half2float(h)) * kQ8Up);
      q[0] = (uint8_t)(w & 0xffu);
      q[64] = (uint8_t)(w >> 8);
    } else {
      uint32_t hw[N / 2], qh[N / 2], ql[N / 2];
#pragma unroll
      for (int j = 0; j < N / 2; ++j) {
        const __half2 h2 = __floats2half2_rn(clamp_f16(v[2 * j]), clamp_f16(v[2 * j + 1]));
        hw[j] = *reinterpret_cast<const uint32_t*>(&h2);
        const float2 f = __half22float2(h2);
        qh[j] = e5m2x2(v[2 * j] * kQ8Down, v[2 * j + 1] * kQ8Down);
        ql[j] = e5m2x2((v[2 * j] - f.x) * kQ8Up, (v[2 * j + 1] - f.y) * kQ8Up);
      }
      if constexpr (N == 2) {
        *reinterpret_cast<uint32_t*>(hi) = hw[0];
        *reinterpret_cast<uint16_t*>(q) = (uint16_t)qh[0];
        *reinterpret_cast<uint16_t*>(q + 64) = (uint16_t)ql[0];
      } else if constexpr (N == 4) {
        *reinterpret_cast<uint2*>(hi) = make_uint2(hw[0], hw[1]);
        *reinterpret_cast<uint32_t*>(q) = qh[0] | (qh[1] << 16);
        *reinterpret_cast<uint32_t*>(q + 64) = ql[0] | (ql[1] << 16);
      } else {
        *reinterpret_cast<uint4*>(hi) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        *reinterpret_cast<uint2*>(q) = make_uint2(qh[0] | (qh[1] << 16), qh[2] | (qh[3] << 16));
        *reinterpret_cast<uint2*>(q + 64) = make_uint2(ql[0] | (ql[1] << 16), ql[2] | (ql[3] << 16));
      }
    }
    return;
  }
  if constexpr (N == 1) {
    __nv_bfloat16 h, l;
    split_bf16(v[0], h, l);
    *hi = h;
    if (lo) *lo = l;
  } else {
    uint32_t hw[N / 2], lw[N / 2];
#pragma unroll
    for (int j = 0; j < N / 2; ++j) {   // packed conversions: same values as split_bf16
      const __nv_bfloat162 h2 = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
      hw[j] = *reinterpret_cast<const uint32_t*>(&h2);
      const float2 f = __bfloat1622float2(h2);
      const __nv_bfloat162 l2 = __floats2bfloat162_rn(v[2 * j] - f.x, v[2 * j + 1] - f.y);
      lw[j] = *reinterpret_cast<const uint32_t*>(&l2);
    }
    if constexpr (N == 2) {
      *reinterpret_cast<uint32_t*>(hi) = hw[0];
      if (lo) *reinterpret_cast<uint32_t*>(lo) = lw[0];
    } else if constexpr (N == 4) {
      *reinterpret_cast<uint2*>(hi) = make_uint2(hw[0], hw[1]);
      if (lo) *reinterpret_cast<uint2*>(lo) = make_uint2(lw[0], lw[1]);
    } else {
      *reinterpret_cast<uint4*>(hi) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
      if (lo) *reinterpret_cast<uint4*>(lo) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
  }
}

// multiprocessors of the current device (grid sizing of persistent and "one resident wave" launches)
int num_sms();

// launch-time operand format of the planes written by the producer kernels (odise_set_operand_format)
int operand_format();
template <typename T>
static inline T* lo_arg(T* lo) {
  return (lo && operand_format() == 2) ? tag_q8(lo) : lo;
}

}  // namespace ob
