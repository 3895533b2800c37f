"""Attention chains at the engines' own layouts: fp32 activations and weights through the projection GEMMs, written into
the layouts each engine uses, then the attention, against fp64 softmax(x Wq (x Wk)^T s) x Wv on the same data.

Bars, from the parts' bars: the projections carry 2e-5 of their scale (test_gpu_gemm.py); with q, k ~ N(0, 1) the
logits stay below ~6 in magnitude, so the projected logits are off by at most 2 * 2e-5 * 6 ~ 2.4e-4, which moves P by
as much in relative terms.  Fused attention: TOL3 = 6e-4 (test_gpu_attention.py) + 2.4e-4 + 2e-5 (v) < 1e-3.
VAE (GEMM, softmax_split, GEMM): 2.4e-4 + 2e-5 (softmax_split) + 2e-5 (P V GEMM) + 2e-5 (v) < 3.5e-4."""
import pytest
import torch

pytestmark = pytest.mark.gpu

CHAIN_TOL = 1e-3
VAE_TOL = 3.5e-4


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def _ref(xq, xkv, Wq, Wk, Wv, heads, d, bq=None, bk=None, bv=None, allowed=None, xv=None):
    """fp64 multi-head attention; xq [B, Tq, C], xkv [B, Tk, Ckv] (values from xv when given), W* [heads*d, C*];
    allowed [B, Tq, Tk] or None"""
    def proj(x, W, b):
        y = x.double() @ W.double().T
        return (y if b is None else y + b.double()).view(x.shape[0], x.shape[1], heads, d)
    q, k, v = proj(xq, Wq, bq), proj(xkv, Wk, bk), proj(xkv if xv is None else xv, Wv, bv)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * d ** -0.5
    if allowed is not None:
        s = s.masked_fill(~allowed[:, None], float("-inf"))
    return torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v).reshape(xq.shape[0] * xq.shape[1], heads * d)


def _w(g, rows, cols):
    return torch.randn(rows, cols, generator=g) * cols ** -0.5


def test_unet_self_attention_padded_keys(cuda, record):
    """UNetEngine._st at T = 6 x 6 = 36 tokens (a 48 x 48 latent's 1280-channel level, d = 160): the keys / values come
    from a copy of the tokens with TkS = 40 rows per image, zero rows after the 36 (unet.py:251-257), projected by the
    row slices of the head-padded qk weight and the swapped-operand V^T GEMM (unet.py:199-213)."""
    from odise_b200 import lib, ops
    B, T, heads, d, C = 2, 36, 8, 160, 1280
    TkS, HS = 40, ops.head_stride(d)
    Cp = heads * HS
    g = torch.Generator().manual_seed(36)
    x = torch.randn(B, T, C, generator=g)
    Wq, Wk, Wv = _w(g, C, C), _w(g, C, C), _w(g, C, C)
    wqk = lib.split(torch.cat([ops.head_pad_rows(Wq, heads, d, HS), ops.head_pad_rows(Wk, heads, d, HS)]).to(cuda))
    wv = lib.split(ops.head_pad_rows(Wv, heads, d, HS).to(cuda))
    xd = x.to(cuda)
    n1 = lib.split(xd.view(B * T, C))
    kvp = torch.zeros(B, TkS * C, device=cuda)
    ops.copy2d(xd.view(B, T * C), kvp[:, :T * C])
    kv = lib.split(kvp.view(B * TkS, C))
    qP = lib.Planes.empty(B * T, Cp, cuda)
    lib.gemm(n1, wqk.row_slice(0, Cp), out_planes=qP)
    kP = lib.Planes.empty(B * TkS, Cp, cuda)
    lib.gemm(kv, wqk.row_slice(Cp, Cp), out_planes=kP)
    vt = lib.Planes.empty(Cp, B * TkS, cuda, f16=True)
    lib.gemm(wv, kv, out_planes=vt)
    out, _ = ops.attention_tc(qP, kP, vt, B, heads, d, T, T, d ** -0.5, 3, want_f32=True, want_planes=False,
                              tk_stride=TkS)
    torch.cuda.synchronize()
    e = _rel(out.cpu(), _ref(x, x, Wq, Wk, Wv, heads, d))
    record(f"chain unet self-attention T=36 TkS=40 d=160: rel err {e:.3e}")
    assert e < CHAIN_TOL


def test_unet_cross_attention_context(cuda, record):
    """UNetEngine._attention for attn2 (unet.py:205-213): q from the image tokens, k and V^T from the 77-token context
    held in 80 rows per image with zero rows after the 77 (unet.py:186-187), d = 40."""
    from odise_b200 import lib, ops
    B, T, heads, d, Cc = 2, 256, 8, 40, 768
    C, HS, ctx, TkS = heads * d, ops.head_stride(d), 77, 80
    Cp = heads * HS
    g = torch.Generator().manual_seed(77)
    x = torch.randn(B, T, C, generator=g)
    c = torch.randn(B, ctx, Cc, generator=g)
    Wq, Wk, Wv = _w(g, C, C), _w(g, C, Cc), _w(g, C, Cc)
    cp = torch.zeros(B, TkS, Cc)
    cp[:, :ctx] = c
    ctxP = lib.split(cp.view(B * TkS, Cc).to(cuda))
    qP = lib.Planes.empty(B * T, Cp, cuda)
    lib.gemm(lib.split(x.view(B * T, C).to(cuda)), lib.split(ops.head_pad_rows(Wq, heads, d, HS).to(cuda)), out_planes=qP)
    kP = lib.Planes.empty(B * TkS, Cp, cuda)
    lib.gemm(ctxP, lib.split(ops.head_pad_rows(Wk, heads, d, HS).to(cuda)), out_planes=kP)
    vt = lib.Planes.empty(Cp, B * TkS, cuda, f16=True)
    lib.gemm(lib.split(ops.head_pad_rows(Wv, heads, d, HS).to(cuda)), ctxP, out_planes=vt)
    out, _ = ops.attention_tc(qP, kP, vt, B, heads, d, T, ctx, d ** -0.5, 3, want_f32=True, want_planes=False,
                              tk_stride=TkS)
    torch.cuda.synchronize()
    e = _rel(out.cpu(), _ref(x, c, Wq, Wk, Wv, heads, d))
    record(f"chain unet cross-attention 77/80 d=40: rel err {e:.3e}")
    assert e < CHAIN_TOL


def test_decoder_level_slot(cuda, record):
    """HeadEngine.transformer_decoder at one level (head.py:329-368): hw = 18 x 14 = 252 keys per image at a stride of
    hw8 = 256; K and V^T of all 3 layers reading the level computed at once from the level's rows of the [B*S, 256]
    memory (batched GEMMs, V^T with bias_m and outp_bs = hw8), pad keys zeroed; layer slot 1 attends through col_slice /
    row_slice views with per-row mask bits."""
    import test_gpu_attention as A
    from odise_b200 import lib, ops
    B, Q, heads, d, C, S, start, hw, hw8, nk, slot = 2, 100, 8, 32, 256, 400, 100, 252, 256, 3, 1
    CP = heads * 64
    g = torch.Generator().manual_seed(252)
    kin, vin = torch.randn(B, S, C, generator=g), torch.randn(B, S, C, generator=g)
    qin = torch.randn(B, Q, C, generator=g)
    Wq, Wk, Wv = _w(g, C, C), _w(g, nk * C, C), _w(g, nk * C, C)
    bq, bk = torch.randn(C, generator=g) * 0.3, torch.randn(nk * C, generator=g) * 0.3
    bv = torch.randn(nk * C, generator=g)

    def pad_heads(w):                                     # [n*256, .] -> [n*CP, .], 8 heads of 32 in 64-wide slots
        out = torch.zeros(w.shape[0] // C, heads, 64, *w.shape[1:])
        out[:, :, :d] = w.view(w.shape[0] // C, heads, d, *w.shape[1:])
        return out.view(-1, *w.shape[1:])

    kin_p = lib.split(kin.view(B * S, C).to(cuda))
    vin_p = lib.split(vin.view(B * S, C).to(cuda))
    k = lib.Planes.empty(B * hw8, nk * CP, cuda)
    lib.gemm(kin_p.row_slice(start, hw), lib.split(pad_heads(Wk).to(cuda)), M=hw, N=nk * CP, K=C, batch=B,
             a_bs=S * kin_p.ld, bias=pad_heads(bk).to(cuda), out_planes=k, outp_bs=hw8 * k.ld)
    vt = lib.Planes.empty(nk * CP, B * hw8, cuda, f16=True)
    lib.gemm(lib.split(pad_heads(Wv).to(cuda)), vin_p.row_slice(start, hw), M=nk * CP, N=hw, K=C, batch=B,
             b_bs=S * vin_p.ld, bias_m=pad_heads(bv).to(cuda), out_planes=vt, outp_bs=hw8)
    for plane in (k.hi, k.lo):
        plane.view(B, hw8, k.ld)[:, hw:].zero_()
    for plane in (vt.hi, vt.lo):
        plane.view(nk * CP, B, hw8)[:, :, hw:].zero_()
    qc = lib.Planes.empty(B * Q, CP, cuda)
    lib.gemm(lib.split(qin.view(B * Q, C).to(cuda)), lib.split(pad_heads(Wq).to(cuda)), bias=pad_heads(bq).to(cuda),
             out_planes=qc)
    allowed, row_any = A._random_mask(B, Q, hw, g)
    out, _ = ops.attention_tc(qc, k.col_slice(slot * CP, CP), vt.row_slice(slot * CP, CP), B, heads, d, Q, hw,
                              d ** -0.5, 3, want_f32=True, want_planes=False, tk_stride=hw8,
                              mask_bits=A.pack_bits(allowed).to(cuda), row_any=row_any.to(cuda))
    torch.cuda.synchronize()
    sl = slice(slot * C, (slot + 1) * C)
    lvl = slice(start, start + hw)
    ref = _ref(qin, kin[:, lvl], Wq, Wk[sl], Wv[sl], heads, d, bq, bk[sl], bv[sl], A.effective_mask(allowed, row_any),
               xv=vin[:, lvl])
    e = _rel(out.cpu(), ref)
    record(f"chain decoder level hw=252 hw8=256 slot 1/3 d=32: rel err {e:.3e}")
    assert e < CHAIN_TOL


def test_vae_mid_block_attention(cuda, record):
    """VaeEngine._attn (vae.py:118-132) at T = 64 x 64 = 4096, one head of d = 512: qk projection into one [M, 1024]
    planes buffer, V^T by the swapped-operand GEMM with bias_m into bf16 planes, S by a batched GEMM over column slices,
    softmax_split on 4096-wide rows (the shared-memory kernel), and P V into planes with outp_bs."""
    from odise_b200 import lib, ops
    B, T, C = 2, 4096, 512
    M = B * T
    g = torch.Generator().manual_seed(4096)
    x = torch.randn(B, T, C, generator=g)
    Wq, Wk, Wv = _w(g, C, C), _w(g, C, C), _w(g, C, C)
    bqk, bv = torch.randn(2 * C, generator=g) * 0.1, torch.randn(C, generator=g)
    xn = lib.split(x.view(M, C).to(cuda))
    qk = lib.Planes.empty(M, 2 * C, cuda)
    lib.gemm(xn, lib.split(torch.cat([Wq, Wk]).to(cuda)), bias=bqk.to(cuda), out_planes=qk)
    vt = lib.Planes.empty(C, M, cuda)
    lib.gemm(lib.split(Wv.to(cuda)), xn, bias_m=bv.to(cuda), out_planes=vt)
    S = torch.empty(B, T, T, device=cuda)
    lib.gemm(qk.col_slice(0, C), qk.col_slice(C, C), M=T, N=T, K=C, batch=B, a_bs=T * qk.ld, b_bs=T * qk.ld, out=S,
             ld_out=T, out_bs=T * T)
    P = ops.softmax_split(S.view(M, T), M, T, T, float(C) ** -0.5)
    del S
    o = lib.Planes.empty(M, C, cuda)
    lib.gemm(P, vt, M=T, N=C, K=T, batch=B, a_bs=T * P.ld, b_bs=T, out_planes=o, outp_bs=T * o.ld)
    torch.cuda.synchronize()
    got = o.float()
    del P
    e = _rel(got.cpu(), _ref(x, x, Wq, Wk, Wv, 1, C, bqk[:C], bqk[C:], bv))
    record(f"chain vae mid-block T=4096 d=512: rel err {e:.3e}")
    assert e < VAE_TOL
