"""Thin typed wrappers over the C ABI used by the engines (unet.py, head.py).  Activations are token-major /
NHWC fp32 matrices [rows, C]; GEMM operands are lib.Planes.  No torch math on the hot path: torch only allocates.
Every launch goes through lib._launch, which passes tensors as their addresses and the current stream last."""
import torch

from . import lib
from .lib import Planes

ACT_NONE, ACT_RELU, ACT_SILU, ACT_GELU, ACT_QUICKGELU = 0, 1, 2, 3, 4


def empty(rows, cols, device):
    return torch.empty(rows, cols, dtype=torch.float32, device=device)


def _gn_stats(x, ldx, x_bs, B, HW, C, G, eps, stats):
    """-> (mean, rstd) [B*G] of x's groups: from the producer epilogues' records when they exist, else from the
    stand-alone pass over x"""
    mean = torch.empty(B * G, dtype=torch.float32, device=x.device)
    rstd = torch.empty(B * G, dtype=torch.float32, device=x.device)
    if stats is not None and not stats.missing and stats.C == C and stats.rows == B * HW and HW % 32 == 0 and x_bs == 0:
        lib._launch("odise_groupnorm_finalize_seg_f32", stats.ptr, 3 * stats.Ctot, stats.Ctot, mean, rstd, B, HW, C, G,
                    eps)
    else:
        ws = torch.empty(int(lib.load().odise_groupnorm_ws_floats(B, HW, C, G)), dtype=torch.float32, device=x.device)
        lib._launch("odise_groupnorm_stats_ws_f32", x, ldx, x_bs, ws, mean, rstd, B, HW, C, G, eps)
    return mean, rstd


def group_norm(x, B, HW, gamma, beta, eps, act=ACT_NONE, G=32, want_f32=False, want_planes=True, lo=True, ldx=None,
               x_bs=0, y=None, ldy=None, y_bs=0, planes=None, o_bs=0, stats=None):
    """x [B*HW, C] (row stride ldx, per-image stride x_bs) -> (y fp32 | None, planes | None).
    y / planes may be given (with explicit strides) to write into a slice of a larger buffer.
    stats: lib.GnStats filled by the GEMM epilogues that produced x (no statistics pass over x then)."""
    C = gamma.numel()
    ldx = ldx or x.stride(0)
    dev = x.device
    mean, rstd = _gn_stats(x, ldx, x_bs, B, HW, C, G, eps, stats)
    if y is None and want_f32:
        y = empty(B * HW, C, dev)
    if y is not None and ldy is None:
        ldy = y.stride(0)
    p = planes if planes is not None else (Planes.empty(B * HW, C, dev, lo=lo) if want_planes else None)
    lib._launch("odise_groupnorm_apply_bs_f32", x, ldx, x_bs, mean, rstd, gamma, beta, act, y, ldy or C, y_bs,
                *lib.pargs(p), o_bs, B, HW, C, G)
    return y, p


def layer_norm(x, gamma, beta, eps=1e-5, res=None, want_f32=False, want_planes=True, post_add=None, lo=True):
    rows, cols = x.shape
    dev = x.device
    y = empty(rows, cols, dev) if want_f32 else None
    p = Planes.empty(rows, cols, dev, lo=lo) if want_planes else None
    lib._launch("odise_layernorm_f32", x, x.stride(0), res, res.stride(0) if res is not None else 0, gamma, beta, eps,
                y, cols, post_add, post_add.stride(0) if post_add is not None else 0, *lib.pargs(p), rows, cols)
    return y, p


def geglu(x, lo=True):
    rows, c2 = x.shape
    p = Planes.empty(rows, c2 // 2, x.device, lo=lo)
    lib._launch("odise_geglu_f32", x, x.stride(0), *lib.pargs(p), rows, c2 // 2)
    return p


def add_split(a, b=None, b_rows=0, want_f32=False, want_planes=True, lo=True):
    rows, cols = a.shape
    y = empty(rows, cols, a.device) if want_f32 else None
    p = Planes.empty(rows, cols, a.device, lo=lo) if want_planes else None
    lib._launch("odise_add_split_f32", a, a.stride(0), b, b.stride(0) if b is not None else 0, b_rows, y, cols,
                *lib.pargs(p), rows, cols)
    return y, p


def act_split(x, act, lo=True):
    rows, cols = x.shape
    p = Planes.empty(rows, cols, x.device, lo=lo)
    lib._launch("odise_act_split_f32", x, x.stride(0), act, *lib.pargs(p), rows, cols)
    return p


def upsample2x_split(x, B, H, W, lo=True):
    C = x.shape[1]
    p = Planes.empty(B * 4 * H * W, C, x.device, lo=lo)
    lib._launch("odise_upsample2x_split_f32", x, x.stride(0), *lib.pargs(p), B, H, W, C)
    return p


def im2col3x3_split(x, B, H, W, stride=1, pad_lo=1, pad_hi=1, lo=True):
    C = x.shape[1]
    Ho = (H + pad_lo + pad_hi - 3) // stride + 1
    Wo = (W + pad_lo + pad_hi - 3) // stride + 1
    Kpad = (9 * C + 63) // 64 * 64 if lo == lib.Q8 else (9 * C + 7) // 8 * 8
    p = Planes.empty(B * Ho * Wo, Kpad, x.device, lo=lo, ld=Kpad)
    lib._launch("odise_im2col3x3_split_f32", x, x.stride(0), *lib.pargs(p)[:2], Kpad, B, H, W, C, stride, pad_lo,
                pad_hi)
    return p, Ho, Wo


def copy2d(src, dst, scale=1.0, accumulate=False):
    rows, cols = src.shape
    lib._launch("odise_copy2d_f32", src, src.stride(0), dst, dst.stride(0), rows, cols, scale, 1 if accumulate else 0)


def resize_nhwc(src, B, Hs, Ws, Hd, Wd, bilinear, dst=None, accumulate=False, src_bs=0, dst_bs=0):
    C = src.shape[1]
    if dst is None:
        dst = empty(B * Hd * Wd, C, src.device)
    lib._launch("odise_resize_nhwc_bs_f32", src, src.stride(0), src_bs, dst, dst.stride(0), dst_bs, B, Hs, Ws, Hd, Wd,
                C, 1 if bilinear else 0, 1 if accumulate else 0)
    return dst


def nchw_to_nhwc(x):
    B, C, H, W = x.shape
    x = x.contiguous()
    y = empty(B * H * W, C, x.device)
    lib._launch("odise_nchw_to_nhwc_f32", x, y, C, B, C, H * W)
    return y


def nhwc_to_nchw(x, B, H, W):
    C = x.shape[1]
    y = torch.empty(B, C, H, W, dtype=torch.float32, device=x.device)
    lib._launch("odise_nhwc_to_nchw_f32", x, x.stride(0), y, B, C, H * W)
    return y


def attention_tc(q, k, vt, B, heads, d, Tq, Tk, scale, nmma, want_f32=False, want_planes=True, tk_stride=None,
                 mask_bits=None, row_any=None, lo=None):
    """q, k head-padded Planes (bf16 pair / plain bf16); vt Planes [heads*HS, >= B*Tk]. Returns (fp32 | None, Planes | None)
    [B*Tq, heads*d].  nmma = 2 (an engine in the F16Q8 mode) runs the bf16x3 attention; `lo` = format of the output planes
    (default: bf16 pair in the bf16x3 mode; lib.Q8 when the consumer GEMM runs F16Q8)."""
    dev = q.hi.device
    C = heads * d
    if nmma == 2:
        nmma = 3
    if q.fmt != "bf16" or k.fmt != "bf16":
        raise lib.OdiseError("attention_tc: q / k must be bf16 planes (the S = Q K^T product runs bf16x3)")
    if vt.f16 != (nmma == 3):
        raise lib.OdiseError("attention_tc: vt must be fp16 planes in the bf16x3 mode (Planes.empty(..., f16=True) / "
                             "lib.split(..., f16=True)) and bf16 planes in the plain bf16 mode")
    out = empty(B * Tq, C, dev) if want_f32 else None
    p = Planes.empty(B * Tq, C, dev, lo=((nmma == 3) if lo is None else lo)) if want_planes else None
    phi, plo, pld = lib.pargs(p)
    lib._launch("odise_attention_tc", q.hi, q.lo, q.ld, k.hi, k.lo, k.ld, vt.hi, vt.lo, vt.ld, vt.rows, out, phi, plo,
                pld if p else C, B, heads, d, Tq, Tk, tk_stride or Tk, scale, nmma, mask_bits, row_any)
    return out, p


def softmax_split(x, rows, cols, cols_pad, scale, lo=True):
    p = Planes.empty(rows, cols_pad, x.device, lo=lo, ld=cols_pad)
    lib._launch("odise_softmax_split_f32", x, x.stride(0), *lib.pargs(p), rows, cols, cols_pad, scale)
    return p


def head_pad_rows(w, heads, d, HS):
    """[heads*d, K] projection weight -> [heads*HS, K] with zero rows in the pad (host-side, one time)."""
    K = w.shape[1]
    out = torch.zeros(heads, HS, K, dtype=w.dtype, device=w.device)
    out[:, :d] = w.view(heads, d, K)
    return out.view(heads * HS, K)


def head_stride(d):
    if d <= 64:    # incl. the decoder's d = 32 and CLIP's d = 64
        return 64
    if d <= 80:
        return 128
    if d == 160:  # SD-v1 16x16 / 8x8 levels: Q K^T over three 64-column chunks, P V in two 80-column halves
        return 192
    return None   # unfused path


def msda_fused(value, spatial_shapes, level_start, ref, offs, logits, N, S, M, D, L, Lq, P, want_f32=False, lo=True):
    dev = value.device
    out = empty(N * Lq, M * D, dev) if want_f32 else None
    p = Planes.empty(N * Lq, M * D, dev, lo=lo)
    lib._launch("odise_msda_fused_f32", value, spatial_shapes, level_start, ref, offs, logits, out, *lib.pargs(p)[:2],
                N, S, M, D, L, Lq, P)
    return out, p


def attn_mask_bits(mask_logits, B, Q, Hm, Wm, Hl, Wl):
    dev = mask_logits.device
    bits = torch.empty(B * Q * ((Hl * Wl + 31) // 32), dtype=torch.int32, device=dev)
    row_any = torch.empty(B * Q, dtype=torch.int32, device=dev)
    lib._launch("odise_attn_mask_bits_f32", mask_logits, bits, row_any, B, Q, Hm, Wm, Hl, Wl)
    return bits, row_any


def mha_d32(q, ldq, k, v, ldkv, B, Tq, Tk, heads, scale, bits=None, row_any=None, lo=True):
    """q/k/v fp32 device tensors (any views whose data_ptr is the first element); returns Planes [B*Tq, heads*32]."""
    p = Planes.empty(B * Tq, heads * 32, q.device, lo=lo)
    nws = int(lib.load().odise_mha_d32_ws_floats(B, Tq, Tk, heads))
    ws = torch.empty(nws, dtype=torch.float32, device=q.device) if nws else None
    lib._launch("odise_mha_d32_ws_f32", q, ldq, k, v, ldkv, bits, row_any, None, *lib.pargs(p), B, Tq, Tk, heads, scale,
                ws)
    return p


def mask_binarize(logits, B, Q, HW):
    dev = logits.device
    binp = torch.empty(B * Q * HW, dtype=torch.bfloat16, device=dev)
    counts = torch.empty(B * Q, dtype=torch.float32, device=dev)
    lib._launch("odise_mask_binarize_f32", logits, binp, HW, counts, B, Q, HW)
    return binp, counts


def pool_normalize(sums, counts, B, Q, C):
    out = empty(B * Q, C, sums.device)
    lib._launch("odise_pool_normalize_f32", sums, counts, out, B, Q, C)
    return out


def l2_normalize_split(x, lo=True):
    rows, cols = x.shape
    p = Planes.empty(rows, cols, x.device, lo=lo)
    lib._launch("odise_l2_normalize_split_f32", x, x.stride(0), *lib.pargs(p), rows, cols)
    return p


def class_max(sims, group_start, null_sim, rows, n_classes):
    out = empty(rows, n_classes + 1, sims.device)
    lib._launch("odise_class_max_f32", sims, sims.stride(0), group_start, null_sim, out, rows, n_classes)
    return out


def group_norm_res(x, B, HW, gamma, beta, eps, res, act, y, accumulate, G=32, stats=None):
    """y (+)= act(gn(x) + res); x, res, y dense [B*HW, C] fp32."""
    C = gamma.numel()
    mean, rstd = _gn_stats(x, x.stride(0), 0, B, HW, C, G, eps, stats)
    lib._launch("odise_groupnorm_apply_res_f32", x, x.stride(0), mean, rstd, gamma, beta, res,
                res.stride(0) if res is not None else 0, act, y, y.stride(0), 1 if accumulate else 0, None, None, 0,
                B, HW, C, G)
    return y


def bcast_fma(a0, ta, p, B, T, C):
    out = torch.empty(B * T, C, dtype=torch.float32, device=p.device)
    lib._launch("odise_bcast_fma_f32", a0, ta, p, out, B, T, C)
    return out


def rowscale(y, s):
    rows, cols = y.shape
    lib._launch("odise_rowscale_f32", y, y.stride(0), s, rows, cols)
    return y


def _is_u8_image(img, what):
    """1 for a uint8 image (0..255), 0 for a float32 one (in [0, 1]); OdiseError for any other dtype"""
    if img.dtype not in (torch.uint8, torch.float32):
        raise lib.OdiseError(f"{what}: uint8 or float32 image expected")
    return int(img.dtype == torch.uint8)


def image_crops(img, boxes_dev, n_crops, H, W, ch, cw):
    """uint8 [N,3,H,W] (0..255) or float32 [N,3,H,W] in [0,1] -> normalised NHWC crops [n_crops*ch*cw, 3]."""
    fn = "odise_image_crops_u8_f32" if _is_u8_image(img, "image_crops") else "odise_image_crops_f32"
    out = torch.empty(n_crops * ch * cw, 3, dtype=torch.float32, device=img.device)
    lib._launch(fn, img, out, boxes_dev, n_crops, H, W, ch, cw)
    return out


def clip_preprocess(img, boxes_dev, n_crops, H, W, ch, cw, S=336):
    u8 = _is_u8_image(img, "clip_preprocess")
    out = torch.empty(n_crops * S * S, 3, dtype=torch.float32, device=img.device)
    lib._launch("odise_clip_preprocess", img, u8, out, boxes_dev, n_crops, H, W, ch, cw, S)
    return out


def crop_resize_bicubic(img, boxes_dev, n_crops, H, W, ch, cw, S=512):
    """T.Resize((S, S), BICUBIC) of every crop -> float image batch NCHW [n_crops, 3, S, S] (feature_extractor.py:73-76)."""
    u8 = _is_u8_image(img, "crop_resize_bicubic")
    out = torch.empty(n_crops, 3, S, S, dtype=torch.float32, device=img.device)
    lib._launch("odise_crop_resize_bicubic", img, u8, out, boxes_dev, n_crops, H, W, ch, cw, S)
    return out


def patchify_split(x, B, S, P, lo=True):
    Kpad = (3 * P * P + 63) // 64 * 64 if lo == lib.Q8 else (3 * P * P + 7) // 8 * 8
    G = S // P
    p = Planes.empty(B * G * G, Kpad, x.device, lo=lo, ld=Kpad)
    lib._launch("odise_patchify_split_f32", x, *lib.pargs(p)[:2], B, S, P, Kpad)
    return p


def maskclip_preprocess(img, N, H, W, S=336):
    """whole image [N,3,H,W] (u8 0..255 / f32 in [0,1]) -> bilinear S x S + CLIP normalisation, NHWC [N*S*S, 3]."""
    u8 = _is_u8_image(img, "maskclip_preprocess")
    out = torch.empty(N * S * S, 3, dtype=torch.float32, device=img.device)
    lib._launch("odise_maskclip_preprocess", img, u8, out, N, H, W, S)
    return out


def maskclip_bits(mask_logits, B, Q, hm, wm, S, P, Tq, row0):
    """-> (bits uint32 [B, Tq, words], row_any int32 [B, Tq]) for odise_attention_tc (clip.py:291-321)."""
    G = S // P
    words = (G * G + 1 + 31) // 32
    bits = torch.zeros(B, Tq, words, dtype=torch.int32, device=mask_logits.device)
    row_any = torch.empty(B, Tq, dtype=torch.int32, device=mask_logits.device)
    lib._launch("odise_maskclip_bits_f32", mask_logits, bits, row_any, B, Q, hm, wm, S, P, Tq, row0)
    return bits, row_any


def open_vocab_merge(cat_logits, clip_logits, ld_clip, overlap_u8, alpha, beta, rows, K, want_open=False):
    out = torch.empty(rows, K + 1, dtype=torch.float32, device=cat_logits.device)
    op = torch.empty(rows, K, dtype=torch.float32, device=cat_logits.device) if want_open else None
    lib._launch("odise_open_vocab_merge_f32", cat_logits, clip_logits, ld_clip, overlap_u8, alpha, beta, out, op, rows,
                K)
    return out, op


def gather_rows(src, idx, add=None, add_period=1):
    """out[i] = src[idx[i]] (+ add[i % add_period]); src fp32 [n, cols], idx int32 [rows]."""
    rows, cols = idx.numel(), src.shape[1]
    out = empty(rows, cols, src.device)
    lib._launch("odise_gather_rows_f32", src, src.stride(0), idx, add, add.stride(0) if add is not None else 0,
                add_period, out, cols, rows, cols)
    return out
