"""GPU parity of the elementwise / normalisation / small-attention kernels against plain PyTorch on the same inputs."""
import pytest
import torch
import torch.nn.functional as F

from odise_b200 import lib

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("shape", [(2, 64 * 64, 320, 32), (3, 16 * 16, 1920, 32), (1, 8 * 8, 2560, 32), (2, 100, 256, 32)])
@pytest.mark.parametrize("act", [0, 2, 1])
def test_groupnorm(cuda, shape, act):
    B, HW, C, G = shape
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(B, HW, C, generator=g) * 2 + 0.7).to(cuda)
    gamma, beta = torch.randn(C, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)
    mean, rstd = torch.empty(B * G, device=cuda), torch.empty(B * G, device=cuda)
    y = torch.empty_like(x)
    yp = lib.Planes.empty(B * HW, C, cuda)
    lib._launch("odise_groupnorm_stats_f32", x, C, mean, rstd, B, HW, C, G, 1e-5)
    lib._launch("odise_groupnorm_apply_f32", x, C, mean, rstd, gamma, beta, act, y, C, yp.hi, yp.lo, yp.ld, B, HW, C, G)
    ref = F.group_norm(x.double().transpose(1, 2), G, gamma.double(), beta.double(), 1e-5).transpose(1, 2)
    ref = [lambda t: t, F.relu, F.silu][act](ref)
    assert _rel(y, ref) < 2e-6
    assert _rel(yp.float().view_as(y), ref) < 2e-5


@pytest.mark.parametrize("cols", [256, 320, 640, 1280, 2048])
def test_layernorm(cuda, cols):
    rows = 333
    g = torch.Generator().manual_seed(cols)
    x, res = torch.randn(rows, cols, generator=g).to(cuda), torch.randn(rows, cols, generator=g).to(cuda)
    pa = torch.randn(rows, cols, generator=g).to(cuda)
    gamma, beta = torch.randn(cols, generator=g).to(cuda), torch.randn(cols, generator=g).to(cuda)
    y = torch.empty_like(x)
    yp = lib.Planes.empty(rows, cols, cuda)
    lib._launch("odise_layernorm_f32", x, cols, res, cols, gamma, beta, 1e-5, y, cols, pa, cols, yp.hi, yp.lo, yp.ld,
                rows, cols)
    ref = F.layer_norm((x + res).double(), (cols,), gamma.double(), beta.double(), 1e-5)
    assert _rel(y, ref) < 2e-6
    assert _rel(yp.float(), ref + pa.double()) < 2e-5


def test_geglu_add_upsample_copy(cuda):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(77, 2 * 640, generator=g).to(cuda)
    p = lib.Planes.empty(77, 640, cuda)
    lib._launch("odise_geglu_f32", x, 1280, p.hi, p.lo, p.ld, 77, 640)
    ref = x[:, :640].double() * F.gelu(x[:, 640:].double())
    assert _rel(p.float(), ref) < 2e-5
    a, b = torch.randn(200, 256, generator=g).to(cuda), torch.randn(100, 256, generator=g).to(cuda)
    y = torch.empty_like(a)
    p = lib.Planes.empty(200, 256, cuda)
    lib._launch("odise_add_split_f32", a, 256, b, 256, 100, y, 256, p.hi, p.lo, p.ld, 200, 256)
    assert torch.equal(y, a + b.repeat(2, 1))
    assert _rel(p.float(), y) < 2e-5
    u = torch.randn(2, 5, 7, 64, generator=g).to(cuda)
    p = lib.Planes.empty(2 * 10 * 14, 64, cuda)
    lib._launch("odise_upsample2x_split_f32", u, 64, p.hi, p.lo, p.ld, 2, 5, 7, 64)
    ref = F.interpolate(u.permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1).reshape(-1, 64)
    assert _rel(p.float(), ref) < 2e-5
    dst = torch.ones(50, 128, device=cuda)
    src = torch.randn(50, 64, generator=g).to(cuda)
    lib._launch("odise_copy2d_f32", src, 64, dst[:, 32:], 128, 50, 64, 0.5, 1)
    assert torch.allclose(dst[:, 32:96], 1 + 0.5 * src) and dst[:, :32].eq(1).all() and dst[:, 96:].eq(1).all()


@pytest.mark.parametrize("cfg", [(2, 8, 8, 16, 16, 64, 1), (1, 16, 16, 64, 64, 32, 1), (2, 64, 64, 16, 16, 8, 0),
                                 (1, 16, 16, 64, 64, 8, 0), (1, 32, 32, 32, 32, 16, 0), (1, 256, 256, 128, 128, 4, 1),
                                 # the pixel decoder's FPN add (head.py::pixel_decoder): s3 rows of the [B, S, 256] encoder
                                 # memory (after the s5 and s4 rows) bilinearly added into s2, portrait 576 x 448 input
                                 (2, 72, 56, 144, 112, 256, 1, 18 * 14 + 36 * 28),
                                 (2, 12, 20, 24, 40, 64, 1, 37), (1, 9, 7, 18, 14, 32, 1, 5), (2, 7, 9, 16, 20, 8, 1, 3)])
def test_resize(cuda, cfg):
    """cfgs with an 8th field (rows before the level in each image's source block) run ops.resize_nhwc with a per-image
    source stride and accumulate=True into a non-zero destination; reference F.interpolate + add in fp64, 1e-6."""
    B, Hs, Ws, Hd, Wd, C, bil = cfg[:7]
    g = torch.Generator().manual_seed(Hs + Hd)
    x = torch.randn(B, Hs, Ws, C, generator=g).to(cuda)
    xn = x.permute(0, 3, 1, 2)
    ref = F.interpolate(xn.double(), size=(Hd, Wd), mode="bilinear", align_corners=False) if bil else \
        F.interpolate(xn, size=(Hd, Wd))
    ref = ref.permute(0, 2, 3, 1)
    if len(cfg) == 7:
        y = torch.zeros(B, Hd, Wd, C, device=cuda)
        lib._launch("odise_resize_nhwc_f32", x, C, y, C, B, Hs, Ws, Hd, Wd, C, bil, 0)
    else:
        from odise_b200 import ops
        r0 = cfg[7]
        S = r0 + Hs * Ws + 11                          # rows per image of the source block: other levels around this one
        src = torch.full((B, S, C), 1e4, device=cuda)  # finite junk outside the level: read only through a wrong stride
        src[:, r0:r0 + Hs * Ws] = x.reshape(B, Hs * Ws, C)
        y0 = torch.randn(B, Hd, Wd, C, generator=g).to(cuda)
        y = y0.clone()
        ops.resize_nhwc(src.view(B * S, C)[r0:], B, Hs, Ws, Hd, Wd, True, dst=y.view(B * Hd * Wd, C), accumulate=True,
                        src_bs=S * C)
        ref = ref + y0.double()
    assert _rel(y, ref) < 1e-6


@pytest.mark.parametrize("cfg", [(2, 9, 9, 4, 1, 1, 1), (1, 16, 16, 320, 2, 1, 1), (1, 16, 16, 128, 2, 0, 1), (2, 8, 8, 3, 1, 1, 1)])
def test_im2col(cuda, cfg):
    B, H, W, C, stride, plo, phi = cfg
    g = torch.Generator().manual_seed(C)
    x = torch.randn(B, C, H, W, generator=g).to(cuda)
    w = torch.randn(24, C, 3, 3, generator=g).to(cuda)
    xp = F.pad(x, (plo, phi, plo, phi))
    ref = F.conv2d(xp.double(), w.double(), stride=stride)
    Ho, Wo = ref.shape[-2:]
    Kpad = (9 * C + 7) // 8 * 8
    xh = x.permute(0, 2, 3, 1).contiguous()
    cols = lib.Planes.empty(B * Ho * Wo, Kpad, cuda, ld=Kpad)
    lib._launch("odise_im2col3x3_split_f32", xh, C, cols.hi, cols.lo, Kpad, B, H, W, C, stride, plo, phi)
    wm = torch.zeros(24, Kpad, device=cuda)
    wm[:, :9 * C] = w.permute(0, 2, 3, 1).reshape(24, 9 * C)
    out = torch.empty(B * Ho * Wo, 24, device=cuda)
    lib.gemm(cols, lib.split(wm), out=out)
    assert _rel(out, ref.permute(0, 2, 3, 1).reshape(-1, 24)) < 2e-5


def test_transposes(cuda):
    x = torch.randn(2, 37, 50, device=cuda)       # NCHW [B, C, HW]
    y = torch.empty(2, 50, 40, device=cuda)
    lib._launch("odise_nchw_to_nhwc_f32", x, y, 40, 2, 37, 50)
    assert torch.equal(y[:, :, :37], x.transpose(1, 2))
    z = torch.empty(2, 37, 50, device=cuda)
    lib._launch("odise_nhwc_to_nchw_f32", y, 40, z, 2, 37, 50)
    assert torch.equal(z, x)


def test_clip_tail(cuda):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(100, 256, generator=g).to(cuda)
    p = lib.Planes.empty(100, 256, cuda)
    lib._launch("odise_l2_normalize_split_f32", x, 256, p.hi, p.lo, p.ld, 100, 256)
    assert _rel(p.float(), F.normalize(x.double(), dim=-1)) < 2e-5
    sizes = torch.randint(1, 5, (20,), generator=g)
    gs = torch.cat([torch.zeros(1, dtype=torch.long), sizes.cumsum(0)]).int().to(cuda)
    Kp = int(sizes.sum())
    sims = torch.randn(100, Kp, generator=g).to(cuda)
    null = torch.randn(100, generator=g).to(cuda)
    out = torch.empty(100, 21, device=cuda)
    lib._launch("odise_class_max_f32", sims, Kp, gs, null, out, 100, 20)
    ref = torch.stack([sims[:, gs[i]:gs[i + 1]].max(-1).values for i in range(20)] + [null], -1)
    assert torch.equal(out, ref)


def test_mask_pool_helpers(cuda):
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(2, 10, 64 * 64, generator=g).to(cuda)
    binm = torch.empty(2, 10, 64 * 64, dtype=torch.bfloat16, device=cuda)
    cnt = torch.empty(2, 10, device=cuda)
    lib._launch("odise_mask_binarize_f32", logits, binm, 64 * 64, cnt, 2, 10, 64 * 64)
    ref = (logits.sigmoid() > 0.5).float()
    assert torch.equal(binm.float(), ref) and torch.equal(cnt, ref.sum(-1))
    sums = torch.randn(2, 10, 256, generator=g).to(cuda)
    pooled = torch.empty_like(sums)
    lib._launch("odise_pool_normalize_f32", sums, cnt, pooled, 2, 10, 256)
    assert torch.allclose(pooled, sums / (cnt[..., None] + 1e-8), rtol=1e-6)


def check_mask_bits(bits, rowany, ml, Hl, Wl):
    """odise_attn_mask_bits_f32 output vs the reference recipe (F.interpolate bilinear, sigmoid < 0.5 = blocked), bit for
    bit.  A bit may differ only where the interpolated logit lies within 1e-6 of 0 (where the sigmoid < 0.5 decision of
    two fp32 evaluations can tie differently), and fewer than 1e-4 of the bits may fall in that band.  Pad bits of the last
    word must be 0; row_any = some key is allowed."""
    B, Tq = ml.shape[:2]
    Tk = Hl * Wl
    li = F.interpolate(ml, size=(Hl, Wl), mode="bilinear", align_corners=False).flatten(2)
    want = ~(li.sigmoid() < 0.5)
    words = bits.view(B, Tq, -1)
    assert words.shape[-1] == (Tk + 31) // 32
    got = ((words[..., None] >> torch.arange(32, device=bits.device, dtype=torch.int32)) & 1).flatten(2).bool()
    assert not got[..., Tk:].any()                                          # ragged last word: pad bits clear
    got = got[..., :Tk]
    band = li.abs() <= 1e-6
    assert band.float().mean().item() < 1e-4, band.float().mean().item()
    assert torch.equal(got | band, want | band)                             # bit for bit outside the tie band
    assert torch.equal(rowany.view(B, Tq) != 0, got.any(-1))


@pytest.mark.parametrize("cfg", [(2, 100, 32 * 32, 256, 256), (1, 100, 128 * 128, 256, 256), (2, 100, 100, 0, 0), (1, 37, 65, 0, 0),
                                 # the decoder's masks at H/4 x W/4 resized to its H/32 and H/16 levels, portrait 576 x 448
                                 # (252 and 1008 keys: ragged last bit words), landscape 256 x 384, and an odd 7 x 9 level
                                 (2, 100, 18 * 14, 144, 112, 18, 14), (2, 100, 36 * 28, 144, 112, 36, 28),
                                 (2, 100, 8 * 12, 64, 96, 8, 12), (1, 37, 7 * 9, 28, 36, 7, 9)])
def test_mha_d32(cuda, cfg):
    """odise_attn_mask_bits_f32 + odise_mha_d32_f32 vs the reference recipe: bilinear resize, sigmoid<0.5 bool mask,
    fully-masked rows unmasked (odise.py:683,760-774), then softmax attention with -inf bias.  (Hl, Wl) is the level the
    mask is resized to (square sqrt(Tk) when not given)."""
    B, Tq, Tk, Hm, Wm = cfg[:5]
    heads, d = 8, 32
    g = torch.Generator().manual_seed(Tk)
    q = torch.randn(B, Tq, heads * d, generator=g).to(cuda)
    k = torch.randn(B, Tk, heads * d, generator=g).to(cuda)
    v = torch.randn(B, Tk, heads * d, generator=g).to(cuda)
    out = torch.empty_like(q)
    scale = d ** -0.5
    bias = None
    bits = rowany = None
    if Hm:
        Hl, Wl = cfg[5:] if len(cfg) > 5 else (int(Tk ** 0.5),) * 2
        assert Hl * Wl == Tk
        ml = (torch.randn(B, Tq, Hm, Wm, generator=g) * 3 - 2.5).to(cuda)
        ml[0, 3] = -5.0          # a fully masked row -> must attend everywhere
        bits = torch.empty(B, Tq, (Tk + 31) // 32, dtype=torch.int32, device=cuda)
        rowany = torch.empty(B, Tq, dtype=torch.int32, device=cuda)
        lib._launch("odise_attn_mask_bits_f32", ml, bits, rowany, B, Tq, Hm, Wm, Hl, Wl)
        check_mask_bits(bits, rowany, ml, Hl, Wl)
        am = F.interpolate(ml, size=(Hl, Wl), mode="bilinear", align_corners=False).sigmoid().flatten(2) < 0.5
        am[torch.where(am.sum(-1) == am.shape[-1])] = False
        assert rowany[0, 3].item() == 0
        bias = torch.zeros(B, 1, Tq, Tk, device=cuda, dtype=torch.float64).masked_fill(am[:, None], float("-inf"))
    lib._launch("odise_mha_d32_f32", q, heads * d, k, v, heads * d, bits, rowany, out, None, None, heads * d, B, Tq, Tk,
                heads, scale)
    qh = q.double().view(B, Tq, heads, d).transpose(1, 2)
    kh = k.double().view(B, Tk, heads, d).transpose(1, 2)
    vh = v.double().view(B, Tk, heads, d).transpose(1, 2)
    s = qh @ kh.transpose(-1, -2) * scale
    if bias is not None:
        s = s + bias
    ref = (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, Tq, heads * d)
    assert _rel(out, ref) < 1e-5
    # the engine path: key-split (flash-decoding) variant with workspace, planes out
    from odise_b200 import ops
    p = ops.mha_d32(q, heads * d, k, v, heads * d, B, Tq, Tk, heads, scale, bits, rowany)
    assert _rel(p.float().view(B, Tq, heads * d), ref) < 2e-5


@pytest.mark.parametrize("shape", [(16, 64 * 64, 320), (4, 16 * 16, 1920), (2, 8 * 8, 2560), (3, 100, 256), (1, 512 * 64, 128), (2, 7, 512)])
def test_groupnorm_workspace_stats(cuda, shape):
    """ops.group_norm -> odise_groupnorm_stats_ws_f32 (coalesced single pass, shifted sums) incl. a large-mean input
    and a strided (column-slice) input."""
    from odise_b200 import ops
    B, HW, C = shape
    g = torch.Generator().manual_seed(C + HW)
    wide = (torch.randn(B * HW, C + 64, generator=g) * 1.7 + 25.0).to(cuda)       # mean >> std: cancellation test
    x = wide[:, 32:32 + C]
    gamma, beta = torch.randn(C, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)
    y, p = ops.group_norm(x, B, HW, gamma, beta, 1e-6, act=2, want_f32=True)
    ref = F.silu(F.group_norm(x.double().view(B, HW, C).transpose(1, 2), 32, gamma.double(), beta.double(), 1e-6)).transpose(1, 2)
    assert _rel(y.view(B, HW, C), ref) < 5e-6
    assert _rel(p.float().view(B, HW, C), ref) < 2e-5
