"""GPU parity of the fused wgmma flash attention (odise_attention_tc) vs fp64 softmax attention.
Shapes are the SD-v1 UNet ones: self-attention d=40 / d=80 / d=160, cross-attention over 77 context tokens.
Tolerance in the bf16x3 mode: the probabilities enter the P V product rounded ONCE to fp16 (2^-12 relative per element,
random sign -> ~1.5e-4 of the output scale on random data); the budget behind that choice is tools/precision_budget.py
(5e-5 on the UNet taps, bar 1e-3).  S = Q K^T stays bf16x3 (2^-16)."""
# Expected size (round 2 note): each probability carries an independent relative rounding error of rms 2^-11 / sqrt(3) =
# 2.8e-4; with n_eff = n / e effective keys for N(0, 1) scores the output error is 2.8e-4 |v| / sqrt(n_eff) rms, while the
# outputs themselves are ~|v| / sqrt(n_eff): the max-error / max-output ratio this file measures is therefore ~2.8e-4
# whatever n is, and one realisation lands anywhere in 1.5e-4 .. 4e-4.  The bound is 2x that expectation.
TOL3 = 6e-4
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("cfg", [(2, 8, 40, 256, 256), (1, 8, 40, 1024, 1024), (2, 8, 80, 256, 256), (3, 8, 40, 128, 77),
                                 (2, 8, 80, 64, 77), (1, 4, 80, 64, 64), (2, 2, 40, 200, 130), (1, 8, 40, 4096, 4096),
                                 (2, 8, 160, 256, 256), (3, 8, 160, 64, 64), (2, 8, 160, 256, 77), (1, 3, 160, 144, 144)])
def test_attention_tc(cuda, nmma, cfg):
    from odise_b200 import lib, ops
    B, heads, d, Tq, Tk = cfg
    g = torch.Generator().manual_seed(Tq * 3 + Tk + d)
    q = torch.randn(B, Tq, heads, d, generator=g).to(cuda)
    k = torch.randn(B, Tk, heads, d, generator=g).to(cuda)
    v = torch.randn(B, Tk, heads, d, generator=g).to(cuda)
    HS = ops.head_stride(d)
    TkS = (Tk + 7) // 8 * 8            # rows per image in the key / value planes (TMA alignment)
    qp = torch.zeros(B * Tq, heads, HS, device=cuda)
    qp[:, :, :d] = q.view(B * Tq, heads, d)
    kp = torch.zeros(B, TkS, heads, HS, device=cuda)
    kp[:, :Tk, :, :d] = k
    kp[:, Tk:] = 7.0                   # pad keys must be masked, not merely zero
    vt = torch.zeros(heads, HS, B, TkS, device=cuda)
    vt[:, :d, :, :Tk] = v.permute(2, 3, 0, 1)
    vt[:, :, :, Tk:] = 5.0
    qP, kP = lib.split(qp.view(B * Tq, heads * HS)), lib.split(kp.view(B * TkS, heads * HS))
    vP = lib.split(vt.view(heads * HS, B * TkS), f16=nmma == 3)
    scale = d ** -0.5
    out, outp = ops.attention_tc(qP, kP, vP, B, heads, d, Tq, Tk, scale, nmma, want_f32=True, want_planes=True,
                                 tk_stride=TkS)
    torch.cuda.synchronize()
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), k.double()) * scale
    ref = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v.double()).reshape(B * Tq, heads * d)
    tol = TOL3 if nmma == 3 else 3e-2
    assert _rel(out, ref) < tol
    assert _rel(outp.float(), ref) < tol + 1e-2 * (nmma == 1)


def test_softmax_split(cuda):
    from odise_b200 import ops
    x = torch.randn(300, 77, device=cuda) * 3
    p = ops.softmax_split(x, 300, 77, 80, 0.5)
    ref = (x.double() * 0.5).softmax(-1)
    got = p.float()
    assert _rel(got[:, :77], ref) < 2e-5 and got[:, 77:].abs().max() == 0


@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("cfg", [(2, 100, 32 * 32, 64, 64), (1, 100, 64 * 64, 256, 256), (2, 37, 8 * 8, 32, 32)])
def test_masked_attention_tc_d32(cuda, nmma, cfg):
    """Mask2Former masked cross-attention (odise.py:683-692, 760-774) on the wgmma kernel: head dim 32, mask bits from
    odise_attn_mask_bits_f32, fully-masked rows attend everywhere."""
    import torch.nn.functional as F
    from odise_b200 import lib, ops
    B, Tq, Tk, Hm, Wm = cfg
    heads, d, HS = 8, 32, 64
    Hl = Wl = int(Tk ** 0.5)
    g = torch.Generator().manual_seed(Tk + Tq)
    q = torch.randn(B, Tq, heads, d, generator=g).to(cuda)
    k = torch.randn(B, Tk, heads, d, generator=g).to(cuda)
    v = torch.randn(B, Tk, heads, d, generator=g).to(cuda)
    ml = (torch.randn(B, Tq, Hm, Wm, generator=g) * 3 - 2.0).to(cuda)
    ml[0, 3] = -5.0                      # fully masked row -> must attend everywhere
    ml[0, 5, : Hm // 2] = -9.0           # first key blocks fully masked for this row (exercises the -inf guards)
    bits, row_any = ops.attn_mask_bits(ml, B, Tq, Hm, Wm, Hl, Wl)
    qp = torch.zeros(B * Tq, heads, HS, device=cuda)
    qp[:, :, :d] = q.view(B * Tq, heads, d)
    kp = torch.zeros(B * Tk, heads, HS, device=cuda)
    kp[:, :, :d] = k.view(B * Tk, heads, d)
    vt = torch.zeros(heads, HS, B * Tk, device=cuda)
    vt[:, :d] = v.view(B * Tk, heads, d).permute(1, 2, 0)
    scale = d ** -0.5
    out, _ = ops.attention_tc(lib.split(qp.view(B * Tq, -1)), lib.split(kp.view(B * Tk, -1)), lib.split(vt.view(heads * HS, -1), f16=nmma == 3),
                              B, heads, d, Tq, Tk, scale, nmma, want_f32=True, want_planes=False, tk_stride=Tk,
                              mask_bits=bits, row_any=row_any)
    torch.cuda.synchronize()
    am = F.interpolate(ml, size=(Hl, Wl), mode="bilinear", align_corners=False).sigmoid().flatten(2) < 0.5
    am[torch.where(am.sum(-1) == am.shape[-1])] = False
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), k.double()) * scale
    s = s.masked_fill(am[:, None], float("-inf"))
    ref = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v.double()).reshape(B * Tq, heads * d)
    assert _rel(out, ref) < (TOL3 if nmma == 3 else 3e-2)
