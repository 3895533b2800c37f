// GPU post-processing of ODISE / Mask2Former inference (SURVEY.md §8a rows b13 / b14, §8f-3), sm_90a.
//
// Reference: CategoryODISE.forward tail (odise/modeling/meta_arch/odise.py:326-370: F.interpolate of the mask logits to
// the padded image size, then per image semantic / panoptic / instance inference) and
// MaskFormer.semantic_inference / panoptic_inference (third_party/Mask2Former/mask2former/maskformer_model.py:280-342),
// which loops over queries in Python with ~4 `.item()` host syncs per query.  Here nothing leaves the device:
//   * upsample_sigmoid: bilinear x4 (align_corners=False) + sigmoid of the [Q, h, w] logits, written PIXEL-MAJOR as
//     (hi, lo) bf16 planes [H*W, Qpad] — the K-major operand of the semantic GEMM sem[c, p] = sum_q P[q, c] * sig[p, q]
//     (odise_gemm_bf16 with swapped operands writes the reference's [K, H, W] layout directly);
//   * panoptic: per-pixel argmax over kept queries of score_q * sigmoid(mask_q) with the upsample recomputed on the
//     fly, area counters by integer atomics, a single-warp sequential pass that reproduces the reference's segment
//     bookkeeping (overlap test, stuff merging), and a final relabel pass.
#include "ptx.cuh"
#include "odise_b200.h"
#include "launch_count.h"

namespace ob {

__device__ __forceinline__ float bilerp(const float* __restrict__ src, int Hs, int Ws, int oy, int ox, float sy,
                                        float sx) {
  // ATen area_pixel_compute_source_index(align_corners=False) + upsample_bilinear2d
  const float fy = fmaxf((oy + 0.5f) * sy - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sx - 0.5f, 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
  const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
  return hy * (hx * src[y0 * Ws + x0] + lx * src[y0 * Ws + x1]) + ly * (hx * src[y1 * Ws + x0] + lx * src[y1 * Ws + x1]);
}

// Output-pixel sampler of the mask logits.  One stage: [hs, ws] -> (H, W) bilinear (odise.py:326-331, output == padded
// input size).  Two stages (sem_seg_postprocess, detectron2 modeling/postprocessing.py, called at odise.py:343-347):
// [hs, ws] -> (pad_h, pad_w), crop to the un-padded (img_h, img_w), bilinear again to the requested (H, W); the
// 4 stage-2 neighbours are evaluated on the fly, the [Q, pad_h, pad_w] field is never written.
struct Sampler {
  int hs, ws, two, img_h, img_w;
  float sy1, sx1, sy2, sx2;
};
static Sampler make_sampler(int hs, int ws, int H, int W, const odise_postprocess_geom* g) {
  Sampler s{};
  s.hs = hs; s.ws = ws;
  if (g) {
    s.two = 1; s.img_h = g->img_h; s.img_w = g->img_w;
    s.sy1 = (float)hs / (float)g->pad_h; s.sx1 = (float)ws / (float)g->pad_w;
    s.sy2 = (float)g->img_h / (float)H; s.sx2 = (float)g->img_w / (float)W;
  } else {
    s.sy1 = (float)hs / (float)H; s.sx1 = (float)ws / (float)W;
  }
  return s;
}
__device__ __forceinline__ float sample(const float* __restrict__ src, const Sampler& s, int oy, int ox) {
  if (!s.two) return bilerp(src, s.hs, s.ws, oy, ox, s.sy1, s.sx1);
  const float fy = fmaxf((oy + 0.5f) * s.sy2 - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * s.sx2 - 0.5f, 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < s.img_h - 1 ? 1 : 0), x1 = x0 + (x0 < s.img_w - 1 ? 1 : 0);
  const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
  const float v00 = bilerp(src, s.hs, s.ws, y0, x0, s.sy1, s.sx1), v01 = bilerp(src, s.hs, s.ws, y0, x1, s.sy1, s.sx1);
  const float v10 = bilerp(src, s.hs, s.ws, y1, x0, s.sy1, s.sx1), v11 = bilerp(src, s.hs, s.ws, y1, x1, s.sy1, s.sx1);
  return hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
}

// grid (W/32, H, B); block (32 x-pixels, 8): each y-thread strides over queries; smem transpose -> q-fastest writes
__global__ void __launch_bounds__(256)
upsample_sigmoid_split_kernel(const float* __restrict__ logits, __nv_bfloat16* __restrict__ hi,
                              __nv_bfloat16* __restrict__ lo, float* __restrict__ up_f32, int Q, int Qpad, int H, int W,
                              Sampler sp) {
  __shared__ float tile[32][33];   // [q within chunk][x]
  const int b = blockIdx.z, oy = blockIdx.y, ox0 = blockIdx.x * 32;
  const int hs = sp.hs, ws = sp.ws;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int q0 = 0; q0 < Qpad; q0 += 32) {
    for (int qq = ty; qq < 32; qq += 8) {
      const int q = q0 + qq, ox = ox0 + tx;
      float v = 0.f;
      if (q < Q && ox < W) {
        const float lg = sample(logits + ((long long)b * Q + q) * hs * ws, sp, oy, ox);
        if (up_f32) up_f32[(((long long)b * Q + q) * H + oy) * W + ox] = lg;
        v = 1.f / (1.f + expf(-lg));
      }
      tile[qq][tx] = v;
    }
    __syncthreads();
    for (int xx = ty; xx < 32; xx += 8) {
      const int ox = ox0 + xx, q = q0 + tx;
      if (ox < W && q < Qpad) {
        __nv_bfloat16 h, l;
        split_bf16(tile[tx][xx], h, l);
        const long long o = (((long long)b * H + oy) * W + ox) * Qpad + q;
        hi[o] = h;
        if (lo) lo[o] = l;
      }
    }
    __syncthreads();
  }
}

// per-query class statistics: softmax over K+1, P[q, c] (c < K) as planes [Kpad rows?] handled on host via GEMM inputs;
// here: scores[q] = max prob, labels[q] = argmax, keep[q]
__global__ void query_scores_kernel(const float* __restrict__ cls, float* __restrict__ probs, float* __restrict__ scores,
                                    int32_t* __restrict__ labels, int32_t* __restrict__ keep, int BQ, int K1,
                                    float thr, float* __restrict__ probs_t, int Q, int Qpad) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= BQ) return;
  const int lane = threadIdx.x & 31;
  const float* c = cls + (long long)i * K1;
  float mx = -INFINITY;
  for (int k = lane; k < K1; k += 32) mx = fmaxf(mx, c[k]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int k = lane; k < K1; k += 32) sum += expf(c[k] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  float best = -1.f;
  int bi = 0x7fffffff;
  for (int k = lane; k < K1; k += 32) {
    const float pr = expf(c[k] - mx) / sum;
    if (probs) probs[(long long)i * K1 + k] = pr;
    // transposed, per image [K, Qpad] (void class dropped): the A operand of the semantic GEMM
    if (probs_t && k < K1 - 1) probs_t[((long long)(i / Q) * (K1 - 1) + k) * Qpad + (i % Q)] = pr;
    if (pr > best) { best = pr; bi = k; }          // first maximal index within the lane's stride
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {               // torch.max returns the first index among ties
    const float ob_ = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob_ > best || (ob_ == best && oi < bi)) { best = ob_; bi = oi; }
  }
  if (lane == 0) {
    scores[i] = best;
    labels[i] = bi;
    keep[i] = (bi != K1 - 1) && (best > thr);
  }
}

// per pixel: argmax over kept queries of score * sigmoid(upsampled logit); counters per query
//   area[q]  = #pixels whose argmax is q          (mask_area)
//   orig[q]  = #pixels with sigmoid(q) >= 0.5     (original_area)
//   inter[q] = #pixels with argmax == q and sigmoid(q) >= 0.5
__global__ void __launch_bounds__(256)
panoptic_argmax_kernel(const float* __restrict__ logits, const float* __restrict__ scores,
                       const int32_t* __restrict__ keep, int16_t* __restrict__ ids, uint8_t* __restrict__ fg,
                       int32_t* __restrict__ area, int32_t* __restrict__ orig, int32_t* __restrict__ inter, int Q,
                       int H, int W, Sampler sp) {
  extern __shared__ int32_t cnt[];   // [3][Q]
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < 3 * Q; i += blockDim.x) cnt[i] = 0;
  __syncthreads();
  const int hs = sp.hs, ws = sp.ws;
  const long long npix = (long long)H * W;
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(p / W), ox = (int)(p - (long long)oy * W);
    float best = -INFINITY;
    int bq = -1;
    bool bfg = false;
    for (int q = 0; q < Q; ++q) {
      if (!keep[b * Q + q]) continue;      // warp-uniform
      const float lg = sample(logits + ((long long)b * Q + q) * hs * ws, sp, oy, ox);
      const float s = 1.f / (1.f + expf(-lg));
      const bool f = s >= 0.5f;
      if (f) atomicAdd(&cnt[Q + q], 1);
      const float pm = scores[b * Q + q] * s;
      if (pm > best) { best = pm; bq = q; bfg = f; }   // argmax(0): first maximal kept query
    }
    ids[(long long)b * npix + p] = (int16_t)bq;
    fg[(long long)b * npix + p] = bfg ? 1 : 0;
    if (bq >= 0) {
      atomicAdd(&cnt[bq], 1);
      if (bfg) atomicAdd(&cnt[2 * Q + bq], 1);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Q; i += blockDim.x) {
    if (cnt[i]) atomicAdd(&area[b * Q + i], cnt[i]);
    if (cnt[Q + i]) atomicAdd(&orig[b * Q + i], cnt[Q + i]);
    if (cnt[2 * Q + i]) atomicAdd(&inter[b * Q + i], cnt[2 * Q + i]);
  }
}

// one thread per image: the reference's sequential segment bookkeeping (maskformer_model.py:313-340)
__global__ void panoptic_assign_kernel(const int32_t* __restrict__ keep, const int32_t* __restrict__ labels,
                                       const int32_t* __restrict__ area, const int32_t* __restrict__ orig,
                                       const int32_t* __restrict__ inter, const uint8_t* __restrict__ is_thing,
                                       int32_t* __restrict__ seg_of_query, int32_t* __restrict__ seg_info,
                                       int32_t* __restrict__ n_segments, int Q, int K, double overlap_thr) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  extern __shared__ int32_t stuff_seg[];   // [K] segment id of an already created stuff class (0 = none)
  for (int c = 0; c < K; ++c) stuff_seg[c] = 0;
  int cur = 0;
  for (int q = 0; q < Q; ++q) {
    seg_of_query[b * Q + q] = 0;
    if (!keep[b * Q + q]) continue;
    const int a = area[b * Q + q], o = orig[b * Q + q], in = inter[b * Q + q];
    if (!(a > 0 && o > 0 && in > 0)) continue;
    if ((double)a / (double)o < overlap_thr) continue;     // python: int / int -> double, compared with the double threshold
    const int c = labels[b * Q + q];
    const bool thing = is_thing[c] != 0;
    if (!thing) {
      if (stuff_seg[c]) { seg_of_query[b * Q + q] = stuff_seg[c]; continue; }
      stuff_seg[c] = cur + 1;
    }
    ++cur;
    seg_of_query[b * Q + q] = cur;
    seg_info[(b * Q + (cur - 1)) * 3 + 0] = cur;
    seg_info[(b * Q + (cur - 1)) * 3 + 1] = thing ? 1 : 0;
    seg_info[(b * Q + (cur - 1)) * 3 + 2] = c;
  }
  n_segments[b] = cur;
}

__global__ void panoptic_relabel_kernel(const int16_t* __restrict__ ids, const uint8_t* __restrict__ fg,
                                        const int32_t* __restrict__ seg_of_query, int32_t* __restrict__ pan, int Q,
                                        long long npix, int B) {
  const long long total = npix * B;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / npix);
    const int q = ids[i];
    pan[i] = (q >= 0 && fg[i]) ? seg_of_query[b * Q + q] : 0;
  }
}


// ---- MaskFormer.instance_inference (maskformer_model.py:344-380) ------------------------------------------------
// top-k over the flattened [Q*K] class probabilities (void column dropped) by an 8-pass MSB radix select on the
// unique 64-bit key (prob bits << 32 | ~flat index), then a bitonic sort of the <= 1024 winners: deterministic,
// descending score, ties broken towards the lower flat index.  grid B, block 1024.
__global__ void __launch_bounds__(1024)
instance_topk_kernel(const float* __restrict__ probs, const uint8_t* __restrict__ is_thing, float* __restrict__ scores,
                     int32_t* __restrict__ classes, int32_t* __restrict__ query_index, int32_t* __restrict__ valid, int Q,
                     int K, int topk) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long sel[1024];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_remaining, s_count;
  const int b = blockIdx.x, tid = threadIdx.x, n = Q * K, K1 = K + 1;
  const float* pb = probs + (long long)b * Q * K1;
  auto key_of = [&](int i) -> unsigned long long {
    const float v = pb[(i / K) * K1 + (i % K)];
    return ((unsigned long long)__float_as_uint(v) << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
  };
  const int k = topk < n ? topk : n;
  if (tid == 0) { s_prefix = 0ull; s_remaining = k; s_count = 0; }
  __syncthreads();
  for (int pass = 7; pass >= 0; --pass) {
    if (tid < 256) hist[tid] = 0u;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    const unsigned long long hi_mask = pass == 7 ? 0ull : (~0ull << ((pass + 1) * 8));
    for (int i = tid; i < n; i += 1024) {
      const unsigned long long key = key_of(i);
      if ((key & hi_mask) == prefix) atomicAdd(&hist[(unsigned)(key >> (pass * 8)) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      int rem = s_remaining, bin = 255;
      for (; bin > 0; --bin) {
        if ((int)hist[bin] >= rem) break;
        rem -= (int)hist[bin];
      }
      s_remaining = rem;
      s_prefix = prefix | ((unsigned long long)bin << (pass * 8));
    }
    __syncthreads();
  }
  const unsigned long long kth = s_prefix;      // the k-th largest key (keys are unique)
  sel[tid] = 0ull;
  __syncthreads();
  for (int i = tid; i < n; i += 1024) {
    const unsigned long long key = key_of(i);
    if (key >= kth) sel[atomicAdd(&s_count, 1)] = key;
  }
  __syncthreads();
  for (int sz = 2; sz <= 1024; sz <<= 1)         // bitonic sort, descending
    for (int st = sz >> 1; st > 0; st >>= 1) {
      const int j = tid ^ st;
      if (j > tid) {
        const unsigned long long a = sel[tid], c = sel[j];
        const bool desc = (tid & sz) == 0;
        if (desc ? (a < c) : (a > c)) { sel[tid] = c; sel[j] = a; }
      }
      __syncthreads();
    }
  if (tid < topk) {
    const long long o = (long long)b * topk + tid;
    if (tid < k) {
      const unsigned long long key = sel[tid];
      const int i = (int)(0xffffffffu - (unsigned)(key & 0xffffffffu));
      const int c = i % K;
      scores[o] = __uint_as_float((unsigned)(key >> 32));
      classes[o] = c;
      query_index[o] = i / K;
      valid[o] = is_thing ? (int)is_thing[c] : 1;
    } else {
      scores[o] = 0.f; classes[o] = -1; query_index[o] = 0; valid[o] = 0;
    }
  }
}

// per (query, row chunk): sum of sigmoid(up) over up > 0 and the count; optional binary mask u8 [B, Q, H, W].
// grid (chunks, Q, B), block 256; deterministic two-stage reduction (partials [B, Q, chunks, 2]).
__global__ void __launch_bounds__(256)
instance_mask_partial_kernel(const float* __restrict__ logits, uint8_t* __restrict__ masks, float* __restrict__ partial,
                             int Q, int H, int W, int rows_per_chunk, Sampler sp) {
  __shared__ float red[2][8];
  const int chunk = blockIdx.x, q = blockIdx.y, b = blockIdx.z, nchunks = gridDim.x;
  const float* src = logits + ((long long)b * Q + q) * sp.hs * sp.ws;
  const int y0 = chunk * rows_per_chunk, y1 = min(H, y0 + rows_per_chunk);
  float num = 0.f, den = 0.f;
  for (int i = y0 * W + threadIdx.x; i < y1 * W; i += 256) {
    const int oy = i / W, ox = i - oy * W;
    const float lg = sample(src, sp, oy, ox);
    const bool on = lg > 0.f;
    if (on) { num += 1.f / (1.f + expf(-lg)); den += 1.f; }
    if (masks) masks[((long long)b * Q + q) * H * W + i] = on ? 1 : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    num += __shfl_xor_sync(0xffffffffu, num, o);
    den += __shfl_xor_sync(0xffffffffu, den, o);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = num; red[1][threadIdx.x >> 5] = den; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, c = 0.f;
    for (int w = 0; w < 8; ++w) { a += red[0][w]; c += red[1][w]; }
    float* o = partial + (((long long)b * Q + q) * nchunks + chunk) * 2;
    o[0] = a; o[1] = c;
  }
}

// scores[b, i] *= sum(sig * mask) / (sum(mask) + 1e-6) of query_index[b, i]
__global__ void instance_finalize_kernel(const float* __restrict__ partial, const int32_t* __restrict__ query_index,
                                         float* __restrict__ scores, int n, int topk, int Q, int nchunks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = i / topk;
  const float* p = partial + ((long long)b * Q + query_index[i]) * nchunks * 2;
  float a = 0.f, c = 0.f;
  for (int w = 0; w < nchunks; ++w) { a += p[2 * w]; c += p[2 * w + 1]; }
  scores[i] *= a / (c + 1e-6f);
}


// ---------------------------------------------------------------------------------------------------------------
// ONE resampling pass for the three inference heads (round 2).  The stand-alone kernels above each re-evaluate the
// bilinear upsample + sigmoid of every (pixel, query) — ~4e8 evaluations per 4 x 1024^2 batch, three times.  Here a warp
// owns 32 consecutive pixels of one output row, each lane walks all Q queries of its pixel ONCE and feeds
//   * semantic:  sigmoid -> (hi, lo) bf16 of 8 consecutive queries packed in registers -> one 16-byte store per plane
//                into the pixel-major operand [pixel][Qpad] (the stand-alone kernel transposes through shared memory
//                and issues 2-byte stores);
//   * panoptic:  the per-pixel running argmax of score * sigmoid over kept queries lives in the lane's registers; the
//                "sigmoid >= 0.5" pixel count of a query is one ballot + popc per (row segment, query);
//   * instance:  sum(sigmoid * [logit > 0]) and the count per query: fixed-order butterfly per (row segment, query),
//                accumulated in a per-warp shared array over the rows the block walks (deterministic), then combined
//                over the 8 warps in fixed order -> partial [B, Q, chunks, 2] for instance_finalize_kernel; the binary
//                masks leave as 32-byte row segments.
// grid (ceil(W / 32), chunks, B), block 256 = 8 warps; the block walks rows [chunk * rpc, (chunk + 1) * rpc), 8 at a time.
struct FusedPost {
  const float* logits;       // [B, Q, hs, ws]
  __nv_bfloat16* hi;         // semantic planes [B*H*W, Qpad] or null
  __nv_bfloat16* lo;
  const float* scores;       // panoptic: [B*Q] or null
  const int32_t* keep;
  int16_t* ids;              // [B*H*W]
  uint8_t* fg;
  int32_t *area, *orig, *inter;   // [B*Q] (zeroed by the caller)
  float* partial;            // instance: [B, Q, chunks, 2] or null
  uint8_t* masks;            // [B, Q, H, W] or null
  int Q, Qpad, H, W, rows_per_chunk;
};

__global__ void __launch_bounds__(256)
post_fused_kernel(const FusedPost a, const Sampler sp) {
  extern __shared__ __align__(16) uint8_t fsm[];
  const int Q = a.Q, Qpad = a.Qpad;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* inst = reinterpret_cast<float*>(fsm);                    // [8 warps][Q][2]
  int32_t* cnt = reinterpret_cast<int32_t*>(inst + 8 * Q * 2);    // [3][Q]
  const int b = blockIdx.z, chunk = blockIdx.y, ox = blockIdx.x * 32 + lane;
  const bool sem = a.hi != nullptr, pan = a.scores != nullptr, ins = a.partial != nullptr;
  for (int i = threadIdx.x; i < 8 * Q * 2; i += 256) inst[i] = 0.f;
  for (int i = threadIdx.x; i < 3 * Q; i += 256) cnt[i] = 0;
  __syncthreads();
  const int hs = sp.hs, ws = sp.ws;
  const long long npix = (long long)a.H * a.W;
  const int y_begin = chunk * a.rows_per_chunk, y_end = min(a.H, y_begin + a.rows_per_chunk);
  const bool xin = ox < a.W;
  for (int y0r = y_begin; y0r < y_end; y0r += 8) {
    const int oy = y0r + warp;
    if (oy >= y_end) continue;                                    // warp-uniform
    // pixel-dependent half of the bilinear sample (ATen area_pixel_compute_source_index, align_corners=False)
    const float fy = fmaxf((oy + 0.5f) * sp.sy1 - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sp.sx1 - 0.5f, 0.f);
    const int sy0 = (int)fy, sx0 = min((int)fx, ws - 1);
    const int sy1 = sy0 + (sy0 < hs - 1 ? 1 : 0), sx1 = sx0 + (sx0 < ws - 1 ? 1 : 0);
    const float ly = fy - sy0, lx = fx - (int)fx, hy = 1.f - ly, hx = 1.f - lx;
    const int o00 = sy0 * ws + sx0, o01 = sy0 * ws + sx1, o10 = sy1 * ws + sx0, o11 = sy1 * ws + sx1;
    float best = -INFINITY;
    int bq = -1;
    bool bfg = false;
    const float* srcb = a.logits + (long long)b * Q * hs * ws;
    const long long pixel = (long long)b * npix + (long long)oy * a.W + ox;
    for (int q0 = 0; q0 < Qpad; q0 += 8) {
      // 8 queries per step: their (hi, lo) bf16 sigmoids leave as one 16-byte store per plane, pixel-major [pixel][Qpad]
      uint32_t hw[4] = {0u, 0u, 0u, 0u}, lw[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int q = q0 + j;
        if (q >= Q) break;                                        // warp-uniform (pad queries stay zero)
        const float* src = srcb + (long long)q * hs * ws;
        float lg;
        if (!sp.two)
          lg = hy * (hx * __ldg(src + o00) + lx * __ldg(src + o01)) + ly * (hx * __ldg(src + o10) + lx * __ldg(src + o11));
        else
          lg = sample(src, sp, oy, xin ? ox : 0);
        // sigmoid on the MUFU intrinsics (~2 ulp; the semantic map is checked to 1e-4, the 0.5 thresholds only move for
        // |logit| < 1e-7): the IEEE expf + division were ~20 of the ~140 instructions per (pixel, query), ncu r2m
        const float s = __fdividef(1.f, 1.f + __expf(-lg));
        if (sem) {
          __nv_bfloat16 h, l;
          split_bf16(s, h, l);
          const uint32_t hb = __bfloat16_as_ushort(h), lb = __bfloat16_as_ushort(l);
          hw[j >> 1] |= hb << ((j & 1) * 16);
          lw[j >> 1] |= lb << ((j & 1) * 16);
        }
        if (pan && a.keep[b * Q + q]) {                          // warp-uniform
          const bool f = s >= 0.5f;
          const unsigned m = __ballot_sync(0xffffffffu, f && xin);
          if (lane == 0 && m) atomicAdd(&cnt[Q + q], __popc(m));
          const float pm = a.scores[b * Q + q] * s;
          if (pm > best) { best = pm; bq = q; bfg = f; }         // argmax(0): first maximal kept query
        }
        if (ins) {
          const bool on = lg > 0.f && xin;
          float num = on ? s : 0.f;
          const unsigned m = __ballot_sync(0xffffffffu, on);
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) num += __shfl_xor_sync(0xffffffffu, num, o);
          if (lane == 0) { inst[(warp * Q + q) * 2] += num; inst[(warp * Q + q) * 2 + 1] += (float)__popc(m); }
          if (a.masks && xin) a.masks[((long long)b * Q + q) * npix + (long long)oy * a.W + ox] = on ? 1 : 0;
        }
      }
      if (sem && xin) {
        *reinterpret_cast<uint4*>(a.hi + pixel * Qpad + q0) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        if (a.lo) *reinterpret_cast<uint4*>(a.lo + pixel * Qpad + q0) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      }
    }
    if (pan && xin) {
      a.ids[pixel] = (int16_t)bq;
      a.fg[pixel] = bfg ? 1 : 0;
      if (bq >= 0) {
        atomicAdd(&cnt[bq], 1);
        if (bfg) atomicAdd(&cnt[2 * Q + bq], 1);
      }
    }
  }
  __syncthreads();
  if (pan) {
    for (int i = threadIdx.x; i < Q; i += 256) {
      if (cnt[i]) atomicAdd(&a.area[b * Q + i], cnt[i]);
      if (cnt[Q + i]) atomicAdd(&a.orig[b * Q + i], cnt[Q + i]);
      if (cnt[2 * Q + i]) atomicAdd(&a.inter[b * Q + i], cnt[2 * Q + i]);
    }
  }
  if (ins) {
    // partial[b, q, chunk * gridDim.x + blockIdx.x, :] = sum over the 8 warps in fixed order
    const int nparts = gridDim.y * gridDim.x, part = chunk * gridDim.x + blockIdx.x;
    for (int q = threadIdx.x; q < Q; q += 256) {
      float n0 = 0.f, d0 = 0.f;
      for (int w = 0; w < 8; ++w) { n0 += inst[(w * Q + q) * 2]; d0 += inst[(w * Q + q) * 2 + 1]; }
      float* o = a.partial + (((long long)b * Q + q) * nparts + part) * 2;
      o[0] = n0; o[1] = d0;
    }
  }
}

}  // namespace ob

using namespace ob;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

static int geom_bad(const odise_postprocess_geom* g) {
  return g && (g->pad_h <= 0 || g->pad_w <= 0 || g->img_h <= 0 || g->img_w <= 0 || g->img_h > g->pad_h || g->img_w > g->pad_w);
}

extern "C" int odise_upsample_sigmoid_split_f32(const float* logits, void* hi, void* lo, float* up_f32, int B, int Q,
                                                int Qpad, int hs, int ws, int H, int W,
                                                const odise_postprocess_geom* geom, void* stream) {
  if (!logits || !hi || B <= 0 || Q <= 0 || Qpad < Q || hs <= 0 || ws <= 0 || H <= 0 || W <= 0 || geom_bad(geom))
    return ODISE_ERR_ARG;
  dim3 grid((W + 31) / 32, H, B), block(32, 8);
  upsample_sigmoid_split_kernel<<<grid, block, 0, STREAM(stream)>>>(logits, reinterpret_cast<__nv_bfloat16*>(hi),
                                                                    reinterpret_cast<__nv_bfloat16*>(lo), up_f32, Q, Qpad,
                                                                    H, W, make_sampler(hs, ws, H, W, geom));
  count_launch(1);
  return (int)cudaGetLastError();
}

extern "C" int odise_query_scores_f32(const float* cls, float* probs, float* probs_t, float* scores, int32_t* labels,
                                      int32_t* keep, int B, int Q, int Qpad, int K1, float threshold, void* stream) {
  if (!cls || !scores || !labels || !keep || B <= 0 || Q <= 0 || Qpad < Q || K1 <= 1) return ODISE_ERR_ARG;
  const int BQ = B * Q;
  query_scores_kernel<<<(BQ + 7) / 8, 256, 0, STREAM(stream)>>>(cls, probs, scores, labels, keep, BQ, K1, threshold,
                                                                probs_t, Q, Qpad);
  count_launch(1);
  return (int)cudaGetLastError();
}

// logits [B, Q, hs, ws]; scores/labels/keep [B*Q]; is_thing [K] uint8; outputs: pan int32 [B, H, W],
// seg_info int32 [B, Q, 3] (id, isthing, category), n_segments int32 [B].
// workspace: ids int16 [B*H*W] | fg uint8 [B*H*W] | area, orig, inter, seg_of_query int32 [B*Q] each  (see *_ws_bytes)
extern "C" long long odise_panoptic_ws_bytes(int B, int Q, int H, int W) {
  const long long npix = (long long)B * H * W;
  return ((npix * 2 + 255) / 256 * 256) + ((npix + 255) / 256 * 256) + 4LL * B * Q * 4 + 256;
}

extern "C" int odise_panoptic_inference_f32(const float* logits, const float* scores, const int32_t* labels,
                                            const int32_t* keep, const uint8_t* is_thing, int32_t* pan,
                                            int32_t* seg_info, int32_t* n_segments, void* ws, int B, int Q, int K,
                                            int hs, int ws_, int H, int W, double overlap_thr,
                                            const odise_postprocess_geom* geom, void* stream) {
  if (!logits || !scores || !labels || !keep || !is_thing || !pan || !seg_info || !n_segments || !ws || geom_bad(geom))
    return ODISE_ERR_ARG;
  if (B <= 0 || Q <= 0 || Q > 32767 || K <= 0 || K * 4 > 48 * 1024) return ODISE_ERR_ARG;
  cudaStream_t st = STREAM(stream);
  const long long npix = (long long)B * H * W;
  uint8_t* base = reinterpret_cast<uint8_t*>(ws);
  int16_t* ids = reinterpret_cast<int16_t*>(base);
  uint8_t* fg = base + (npix * 2 + 255) / 256 * 256;
  int32_t* counters = reinterpret_cast<int32_t*>(fg + (npix + 255) / 256 * 256);
  int32_t *area = counters, *orig = counters + B * Q, *inter = counters + 2 * B * Q, *seg_of = counters + 3 * B * Q;
  cudaError_t e = cudaMemsetAsync(counters, 0, sizeof(int32_t) * 3 * B * Q, st);
  if (e != cudaSuccess) return (int)e;
  int blocks = (int)(((long long)H * W + 255) / 256);
  if (blocks > num_sms() * 4) blocks = num_sms() * 4;
  panoptic_argmax_kernel<<<dim3(blocks, B), 256, 3 * Q * sizeof(int32_t), st>>>(logits, scores, keep, ids, fg, area, orig,
                                                                            inter, Q, H, W, make_sampler(hs, ws_, H, W, geom));
  panoptic_assign_kernel<<<B, 32, K * sizeof(int32_t), st>>>(keep, labels, area, orig, inter, is_thing, seg_of, seg_info,
                                                          n_segments, Q, K, overlap_thr);
  int rb = (int)((npix + 255) / 256);
  if (rb > num_sms() * 8) rb = num_sms() * 8;
  panoptic_relabel_kernel<<<rb, 256, 0, st>>>(ids, fg, seg_of, pan, Q, (long long)H * W, B);
  count_launch(3);
  return (int)cudaGetLastError();
}

// instance_inference on the device.  probs [B*Q, K+1] (softmax incl. void; odise_query_scores_f32), logits [B, Q, hs, ws].
// Outputs per image, sorted by class probability (descending): scores [B, topk] = class prob * mask score,
// classes / query_index [B, topk], valid [B, topk] (= is_thing[class] when is_thing != NULL: the panoptic_on filter),
// masks u8 [B, Q, H, W] (optional; the mask of instance i is masks[b, query_index[b, i]]).
static inline int instance_chunks(int H) { return H >= 64 ? 16 : 1; }
extern "C" long long odise_instance_ws_bytes(int B, int Q, int H, int W) {
  (void)W;
  return (long long)B * Q * instance_chunks(H) * 2 * sizeof(float) + 256;
}

extern "C" int odise_instance_inference_f32(const float* probs, const float* logits, const uint8_t* is_thing,
                                            float* scores, int32_t* classes, int32_t* query_index, int32_t* valid,
                                            uint8_t* masks, void* ws, int B, int Q, int K, int topk, int hs, int ws_,
                                            int H, int W, const odise_postprocess_geom* geom, void* stream) {
  if (!probs || !logits || !scores || !classes || !query_index || !valid || !ws || geom_bad(geom)) return ODISE_ERR_ARG;
  if (B <= 0 || Q <= 0 || K <= 0 || topk <= 0 || topk > 1024 || hs <= 0 || ws_ <= 0 || H <= 0 || W <= 0) return ODISE_ERR_ARG;
  if ((long long)Q * K >= 0x7fffffffLL) return ODISE_ERR_ARG;
  cudaStream_t st = STREAM(stream);
  const int nchunks = instance_chunks(H), rows = (H + nchunks - 1) / nchunks;
  float* partial = reinterpret_cast<float*>(ws);
  instance_topk_kernel<<<B, 1024, 0, st>>>(probs, is_thing, scores, classes, query_index, valid, Q, K, topk);
  instance_mask_partial_kernel<<<dim3(nchunks, Q, B), 256, 0, st>>>(logits, masks, partial, Q, H, W, rows,
                                                                          make_sampler(hs, ws_, H, W, geom));
  const int n = B * topk;
  instance_finalize_kernel<<<(n + 255) / 256, 256, 0, st>>>(partial, query_index, scores, n, topk, Q, nchunks);
  count_launch(3);
  return (int)cudaGetLastError();
}

// All three inference heads from ONE resampling pass (post_fused_kernel) + the small bookkeeping kernels.  Any of the
// three groups of outputs may be absent (NULL): sem_hi | (pan, seg_info, n_segments, pan_ws) | (inst_scores, ...).
static inline int fused_chunks(int H) { return H >= 128 ? 16 : 1; }
extern "C" long long odise_postprocess_fused_ws_bytes(int B, int Q, int H, int W) {
  const long long parts = (long long)fused_chunks(H) * ((W + 31) / 32);
  return (long long)B * Q * parts * 2 * sizeof(float) + 256;
}

extern "C" int odise_postprocess_fused_f32(const float* logits, void* sem_hi, void* sem_lo, int Qpad,
                                           const float* scores, const int32_t* labels, const int32_t* keep,
                                           const uint8_t* is_thing, int32_t* pan, int32_t* seg_info, int32_t* n_segments,
                                           void* pan_ws, double overlap_thr, const float* probs, float* inst_scores,
                                           int32_t* inst_classes, int32_t* inst_query, int32_t* inst_valid,
                                           uint8_t* inst_masks, void* inst_ws, int topk, int panoptic_filter, int B, int Q,
                                           int K, int hs, int ws_, int H, int W, const odise_postprocess_geom* geom,
                                           void* stream) {
  if (!logits || B <= 0 || Q <= 0 || K <= 0 || hs <= 0 || ws_ <= 0 || H <= 0 || W <= 0 || geom_bad(geom)) return ODISE_ERR_ARG;
  const bool sem = sem_hi != nullptr, panop = pan != nullptr, inst = inst_scores != nullptr;
  if (!sem && !panop && !inst) return ODISE_ERR_ARG;
  if (sem && (Qpad < Q || Qpad % 8)) return ODISE_ERR_ARG;
  if (panop && (!scores || !labels || !keep || !is_thing || !seg_info || !n_segments || !pan_ws || Q > 32767 ||
                K * 4 > 48 * 1024))
    return ODISE_ERR_ARG;
  if (inst && (!probs || !inst_classes || !inst_query || !inst_valid || !inst_ws || topk <= 0 || topk > 1024 ||
               (long long)Q * K >= 0x7fffffffLL))
    return ODISE_ERR_ARG;
  cudaStream_t st = STREAM(stream);
  const long long npix = (long long)B * H * W;
  FusedPost a{};
  a.logits = logits; a.Q = Q; a.Qpad = sem ? Qpad : (Q + 7) / 8 * 8; a.H = H; a.W = W;
  const int chunks = fused_chunks(H);
  a.rows_per_chunk = ((H + chunks - 1) / chunks + 7) / 8 * 8;
  a.hi = reinterpret_cast<__nv_bfloat16*>(sem_hi); a.lo = reinterpret_cast<__nv_bfloat16*>(sem_lo);
  int32_t* seg_of = nullptr;
  if (panop) {
    uint8_t* base = reinterpret_cast<uint8_t*>(pan_ws);
    a.ids = reinterpret_cast<int16_t*>(base);
    a.fg = base + (npix * 2 + 255) / 256 * 256;
    int32_t* counters = reinterpret_cast<int32_t*>(a.fg + (npix + 255) / 256 * 256);
    a.area = counters; a.orig = counters + B * Q; a.inter = counters + 2 * B * Q; seg_of = counters + 3 * B * Q;
    a.scores = scores; a.keep = keep;
    cudaError_t e = cudaMemsetAsync(counters, 0, sizeof(int32_t) * 3 * B * Q, st);
    if (e != cudaSuccess) return (int)e;
  }
  int launches = 1;
  if (inst) {
    a.partial = reinterpret_cast<float*>(inst_ws); a.masks = inst_masks;
    instance_topk_kernel<<<B, 1024, 0, st>>>(probs, panoptic_filter ? is_thing : nullptr, inst_scores, inst_classes,
                                             inst_query, inst_valid, Q, K, topk);
    ++launches;
  }
  dim3 grid((W + 31) / 32, (H + a.rows_per_chunk - 1) / a.rows_per_chunk, B);
  const size_t smem = (size_t)8 * Q * 2 * sizeof(float) + (size_t)3 * Q * sizeof(int32_t);
  if (smem > 48 * 1024) return ODISE_ERR_UNSUPPORTED;
  post_fused_kernel<<<grid, 256, smem, st>>>(a, make_sampler(hs, ws_, H, W, geom));
  if (panop) {
    panoptic_assign_kernel<<<B, 32, K * sizeof(int32_t), st>>>(keep, labels, a.area, a.orig, a.inter, is_thing, seg_of,
                                                            seg_info, n_segments, Q, K, overlap_thr);
    int rb = (int)((npix + 255) / 256);
    if (rb > num_sms() * 8) rb = num_sms() * 8;
    panoptic_relabel_kernel<<<rb, 256, 0, st>>>(a.ids, a.fg, seg_of, pan, Q, (long long)H * W, B);
    launches += 2;
  }
  if (inst) {
    const int n = B * topk;
    instance_finalize_kernel<<<(n + 255) / 256, 256, 0, st>>>(a.partial, inst_query, inst_scores, n, topk, Q,
                                                              (int)(grid.x * grid.y));
    ++launches;
  }
  count_launch(launches);
  return (int)cudaGetLastError();
}
