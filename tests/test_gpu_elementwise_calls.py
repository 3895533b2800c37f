"""Elementwise passes at the shapes the engines call them with, against float64 on the same fp32 inputs: the backbone's
residual GroupNorm tail and both GroupNorm apply kernels, every activation code of every kernel that takes one, the implicit
captioner's broadcast FMA, the crop-overlap row scaling, the CLIP token gathers and the bicubic crop resize."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ACTS = [0, 1, 2, 3, 4]           # ODISE_ACT_NONE, RELU, SILU, GELU, QUICKGELU
U = 2.0 ** -23                   # fp32 ulp of 1: one ulp of v is at most U * |v|
TINY = 1e-35                     # above |act(z)| wherever a kernel underflows to 0 or a subnormal (|z| <= 100: < 100 * 2^-126)


def _gn64(x, B, HW, G, gamma, beta, eps):
    C = gamma.numel()
    xt = x.double().reshape(B, HW, C).transpose(1, 2)
    return F.group_norm(xt, G, gamma.double(), beta.double(), eps).transpose(1, 2).reshape(B * HW, C)


def _act64(z, act):
    z = z.double()
    if act == 0:
        return z
    if act == 1:
        return z.clamp_min(0)
    if act == 2:
        return z * torch.sigmoid(z)
    if act == 3:
        return 0.5 * z * (1 + torch.erf(z / math.sqrt(2)))
    return z * torch.sigmoid(1.702 * z)


def _act_bound(z, act):
    """Per-element bound on |act(z) as the kernels compute it - act(z) in float64|, z an fp32 value."""
    a = z.double().abs()
    r = _act64(z, act).abs()
    if act in (0, 1):
        return torch.zeros_like(r)                     # identity and fmaxf are exact
    if act in (2, 4):
        # r = z / (1 + E), E = __expf(-k z), k = 1 (SiLU) | 1.702f (QuickGELU).  __expf(x) is within 2 + 1.173 |x| ulps
        # (CUDA C++ Programming Guide, intrinsic functions); rounding -k*z to fp32 (0.5 ulp) and 1.702f - 1.702 (0.11 ulp)
        # move E's argument by 0.61 k|z| U, i.e. E by 0.61 k|z| ulps; r inherits E's relative error times E / (1 + E) <= 1;
        # 1 + E rounds (0.5 ulp), the division rounds (__fdividef: 2 ulps, IEEE: 0.5 ulp).  -> (4.5 + 1.8 k|z|) ulps of r.
        k = 1.0 if act == 2 else 1.702
        return (4.5 + 1.8 * k * a) * U * r + TINY
    # GELU 0.5 z (1 + erff(z * 0.70710678f)): erff is within 2 ulps (<= 2^-23 absolute, |erf| <= 1), the argument's rounding
    # moves erf by <= 2/sqrt(pi) * max(t exp(-t^2)) * 0.6 U < 0.3 U, and 1 + erf rounds by <= 0.5 U: the sum is off by
    # < 1.8 U absolute however small it is (the cancellation torch's fp32 F.gelu shares) -> 0.9 |z| U; the product rounds by
    # 0.5 ulp of r.
    return (a + r) * U + TINY


def _check_act(got, z, act, planes=False):
    """max of |got - act64(z)| / bound over the elements (<= 1 passes); planes: the (hi, lo) bf16 pair, whose sum is
    within 2^-17 of the fp32 value it encodes (the 2e-5 bar of the plane readback)."""
    ref = _act64(z, act)
    bound = _act_bound(z, act)
    if planes:
        bound = 2e-5 * ref.abs() + 2 * bound
    err = (got.double() - ref).abs()
    ok = bound > 0
    assert torch.equal(err[~ok], torch.zeros_like(err[~ok])), (act, err[~ok].max().item())
    return (err[ok] / bound[ok]).max().item() if ok.any() else 0.0


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


# ---------------------------------------------------------------------------------------------- GroupNorm
@pytest.mark.parametrize("stats", ["records", "pass"])
@pytest.mark.parametrize("side", [128, 64, 32, 16])
def test_backbone_tail(cuda, record, side, stats):
    """BackboneEngine.project's tail at a 512 crop's s2..s5 maps: t3 = conv3 (a GEMM leaving its GroupNorm records), then
    y = relu(gn(t3) + shortcut), then y += relu(gn(t3') + shortcut') for the next tap of the same stride.  Statistics from
    the GEMM's records or from the stand-alone pass."""
    from odise_b200 import lib, ops
    B, HW, C = 2, side * side, 512
    g = torch.Generator().manual_seed(side)
    gamma, beta = torch.randn(C, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)

    def conv3():
        a2 = torch.randn(B * HW, 128, generator=g).relu().to(cuda)        # the ReLU'd conv2 GroupNorm
        w = (torch.randn(C, 128, generator=g) * 0.1).to(cuda)
        t, s = ops.empty(B * HW, C, cuda), lib.GnStats(B * HW, C, cuda)
        lib.gemm(lib.split(a2), lib.split(w), out=t, gn=s)
        assert not s.missing
        return t, (s if stats == "records" else None), torch.randn(B * HW, C, generator=g).to(cuda)

    t1, s1, sc1 = conv3()
    t2, s2, sc2 = conv3()
    y = ops.empty(B * HW, C, cuda)
    ops.group_norm_res(t1, B, HW, gamma, beta, 1e-5, sc1, ops.ACT_RELU, y, accumulate=False, stats=s1)
    y0 = y.clone()
    ops.group_norm_res(t2, B, HW, gamma, beta, 1e-5, sc2, ops.ACT_RELU, y, accumulate=True, stats=s2)
    e1 = _rel(y0, (_gn64(t1, B, HW, 32, gamma, beta, 1e-5) + sc1.double()).relu())
    e2 = _rel(y, y0.double() + (_gn64(t2, B, HW, 32, gamma, beta, 1e-5) + sc2.double()).relu())
    record(f"elementwise_calls backbone tail {side}x{side} stats={stats}: {e1:.2e} / accumulated {e2:.2e} of max|ref|")
    assert e1 < 2e-6 and e2 < 2e-6


def _gn_input(B, HW, C, G, g):
    """per-(image, group) offsets and scales, so that a channel normalised with a neighbouring group's statistics is far off"""
    cpg = C // G
    off = (torch.rand(B, 1, G, generator=g) * 40 - 20).repeat_interleave(cpg, -1)
    sc = (torch.rand(B, 1, G, generator=g) * 3.5 + 0.5).repeat_interleave(cpg, -1)
    return torch.randn(B, HW, C, generator=g) * sc + off


@pytest.mark.parametrize("C", [320, 512, 640, 1280])
@pytest.mark.parametrize("act", ACTS)
def test_octet_and_quad_apply_agree(cuda, C, act):
    """The 8-channel apply kernel (ops.group_norm) and the 4-channel one (ops.group_norm_res with accumulate into zeros)
    evaluate the same fmaf((x - mu) * rs, gamma, beta) and activation: identical bits up to the sign of zero."""
    from odise_b200 import ops
    B, HW = 2, 24 * 24
    g = torch.Generator().manual_seed(C + act)
    x = _gn_input(B, HW, C, 32, g).view(B * HW, C).to(cuda)
    gamma = ((torch.rand(C, generator=g) - 0.5) * 120).to(cuda)            # pre-activations over about [-100, 100]
    beta = torch.randn(C, generator=g).to(cuda)
    y8, _ = ops.group_norm(x, B, HW, gamma, beta, 1e-5, act=act, want_f32=True, want_planes=False)
    yq = torch.zeros_like(x)
    ops.group_norm_res(x, B, HW, gamma, beta, 1e-5, None, act, yq, accumulate=True)
    assert torch.equal(y8, yq)


# (B, HW, C, ldo of the planes); G = 32, cpg = C / 32
GN_SLICES = [(2, 300, 128, 136),     # cpg 4: every octet spans two groups
             (2, 250, 288, 296),     # cpg 9: octets straddle group boundaries at every offset
             (2, 256, 320, 328),     # cpg 10
             (2, 200, 384, 392),     # cpg 12
             (2, 150, 640, 648),     # cpg 20
             (2, 64, 1280, 1288),    # cpg 40: octets inside one group
             (2, 100, 96, 104),      # cpg 3: 4-channel kernel
             (2, 100, 192, 200),     # cpg 6: 4-channel kernel
             (2, 64, 2560, 2568),    # C / 8 > 256: 4-channel kernel
             (2, 100, 512, 516)]     # plane rows not on 8-element boundaries: 4-channel kernel


@pytest.mark.parametrize("cfg", GN_SLICES)
def test_group_norm_slices(cuda, record, cfg):
    """ops.group_norm reading a level from a [B, S, ldx] block (x_bs) and writing it into slices of larger fp32 and plane
    buffers (y_bs, o_bs), as the pixel decoder writes its input projections into the level-concatenated token matrix.
    Against float64 GroupNorm + SiLU; everything outside the slices keeps its sentinel."""
    from odise_b200 import lib, ops
    B, HW, C, ldo = cfg
    G = 32
    g = torch.Generator().manual_seed(C + HW)
    x = _gn_input(B, HW, C, G, g)
    gamma, beta = torch.randn(C, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)
    ldx, Sx, rx = C + 12, HW + 37, 29                 # x: rows [rx, rx + HW), columns [4, 4 + C) of each image's block
    xblk = torch.full((B, Sx, ldx), 1e4)
    xblk[:, rx:rx + HW, 4:4 + C] = x
    xblk = xblk.to(cuda)
    ldy, Sy, ry = C + 8, HW + 21, 13                  # y: rows [ry, ry + HW), columns [4, 4 + C)
    yblk = torch.full((B, Sy, ldy), 777.0, device=cuda)
    Sp, rp = HW + 9, 5                                # planes: rows [rp, rp + HW) of each image's Sp rows, ld = ldo
    sent = torch.tensor(-3.0, dtype=torch.bfloat16)
    p = lib.Planes(torch.full((B * Sp * ldo,), -3.0, dtype=torch.bfloat16, device=cuda),
                   torch.full((B * Sp * ldo,), -3.0, dtype=torch.bfloat16, device=cuda), B * Sp, C, ldo)
    ops.group_norm(xblk.view(-1)[rx * ldx + 4:], B, HW, gamma, beta, 1e-5, act=ops.ACT_SILU, ldx=ldx, x_bs=Sx * ldx,
                   y=yblk.view(-1)[ry * ldy + 4:], ldy=ldy, y_bs=Sy * ldy, planes=p.row_slice(rp, B * Sp - rp),
                   o_bs=Sp * ldo)
    ref = F.silu(_gn64(x, B, HW, G, gamma.cpu(), beta.cpu(), 1e-5)).view(B, HW, C)
    y = yblk[:, ry:ry + HW, 4:4 + C].cpu()
    ph = p.hi.view(B, Sp, ldo).cpu()
    pl = p.lo.view(B, Sp, ldo).cpu()
    planes = (ph[:, rp:rp + HW, :C].float() + pl[:, rp:rp + HW, :C].float())
    ey, ep = _rel(y, ref), _rel(planes, ref)
    record(f"elementwise_calls group_norm slices B={B} HW={HW} C={C} ldo={ldo}: fp32 {ey:.2e}, planes {ep:.2e} of max|ref|")
    assert ey < 2e-6 and ep < 2e-5
    ymask = torch.ones(B, Sy, ldy, dtype=torch.bool)
    ymask[:, ry:ry + HW, 4:4 + C] = False
    assert yblk.cpu()[ymask].eq(777.0).all()
    pmask = torch.ones(B, Sp, ldo, dtype=torch.bool)
    pmask[:, rp:rp + HW, :C] = False
    assert ph[pmask].eq(sent).all() and pl[pmask].eq(sent).all()
    assert torch.equal(xblk[:, rx:rx + HW, 4:4 + C].cpu(), x)


# ---------------------------------------------------------------------------------------------- activations
def _sweep(n):
    """n fp32 values over [-100, 100]: a uniform grid plus +-0 and tiny magnitudes"""
    special = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 1e-7, -1e-7, 100.0, -100.0])
    return torch.cat([special, torch.linspace(-100, 100, n - special.numel())])


@pytest.mark.parametrize("act", ACTS)
def test_act_split(cuda, record, act):
    """ops.act_split at the UNet's [2, 1280] time embedding (unet.py: SiLU(emb) ahead of each ResBlock emb linear)."""
    from odise_b200 import ops
    x = _sweep(2 * 1280).view(2, 1280).to(cuda)
    p = ops.act_split(x, act)
    worst = _check_act(p.float(), x, act, planes=True)
    record(f"elementwise_calls act_split act={act}: planes {worst:.3f} of the bound")
    assert worst <= 1.0


@pytest.mark.parametrize("act", ACTS)
def test_act_group_norm(cuda, record, act):
    """The activation of both GroupNorm apply kernels, per element, against float64 act() of the kernel's own fp32
    pre-activation (the same call with ACT_NONE): the 8-channel kernel (fp32 and planes), the 4-channel kernel without and
    with a residual.  Pre-activations cover [-100, 100]; gamma = 0, beta = -0 channels give +0 and -0."""
    from odise_b200 import ops
    B, HW, C, G = 2, 256, 320, 32
    g = torch.Generator().manual_seed(100 + act)
    x = (torch.rand(B * HW, C, generator=g) * 2 - 1).to(cuda)
    mag = 58.0 * 10.0 ** (-4 * torch.rand(C, generator=g))                # |x - mu| * rs <= sqrt(3): |z| up to ~100
    gamma = mag * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0)
    beta = torch.randn(C, generator=g) * 0.5
    gamma[::16], beta[::16] = 0.0, -0.0
    gamma, beta = gamma.to(cuda), beta.to(cuda)
    res = torch.randn(B * HW, C, generator=g).to(cuda)
    z8, _ = ops.group_norm(x, B, HW, gamma, beta, 1e-5, act=0, want_f32=True, want_planes=False)
    assert z8.abs().max().item() > 80 and (z8 == 0).any() and torch.signbit(z8[z8 == 0]).any()
    y8, p8 = ops.group_norm(x, B, HW, gamma, beta, 1e-5, act=act, want_f32=True)
    zq = torch.zeros_like(x)
    ops.group_norm_res(x, B, HW, gamma, beta, 1e-5, None, 0, zq, accumulate=True)
    yq = torch.zeros_like(x)
    ops.group_norm_res(x, B, HW, gamma, beta, 1e-5, None, act, yq, accumulate=True)
    zr = ops.group_norm_res(x, B, HW, gamma, beta, 1e-5, res, 0, torch.empty_like(x), accumulate=False)
    yr = ops.group_norm_res(x, B, HW, gamma, beta, 1e-5, res, act, torch.empty_like(x), accumulate=False)
    worst = {"octet": _check_act(y8, z8, act), "octet planes": _check_act(p8.float(), z8, act, planes=True),
             "quad": _check_act(yq, zq, act), "quad residual": _check_act(yr, zr, act)}
    record(f"elementwise_calls group_norm act={act}: " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()) +
           " of the bound")
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("act", [5, -1])
def test_unknown_act_code_is_refused(cuda, act):
    """An act code outside ODISE_ACT_NONE..ODISE_ACT_QUICKGELU is an argument error, never a silent identity."""
    from odise_b200 import lib, ops
    x = torch.randn(64, 64, device=cuda)
    gamma, beta = torch.ones(64, device=cuda), torch.zeros(64, device=cuda)
    with pytest.raises(lib.OdiseError):
        ops.act_split(x, act)
    with pytest.raises(lib.OdiseError):
        ops.group_norm(x, 2, 32, gamma, beta, 1e-5, act=act, want_f32=True)
    with pytest.raises(lib.OdiseError):
        ops.group_norm_res(x, 2, 32, gamma, beta, 1e-5, x, act, torch.empty_like(x), accumulate=False)
    with pytest.raises(lib.OdiseError):
        lib.gemm(lib.split(x), lib.split(x), act=act, out=torch.empty_like(x))
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- conditioning, scaling, gathers
def _ulp(v):
    a = v.float().abs()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


@pytest.mark.parametrize("B", [1, 2, 4])
@pytest.mark.parametrize("TC", [(77, 768), (1, 1280)])
def test_bcast_fma(cuda, record, B, TC):
    """The implicit captioner's cond = a0 + ta * proj (context [B, 77, 768], time embedding [B, 1, 1280]): one fmaf, so
    within 1 ulp of the float64 value per element (ta * p is exact in float64)."""
    from odise_b200 import ops
    T, C = TC
    g = torch.Generator().manual_seed(B * T + C)
    a0 = torch.randn(T, C, generator=g).to(cuda)
    ta = torch.tanh(torch.randn(T, C, generator=g)).to(cuda)
    p = (torch.randn(B, C, generator=g) * 3).to(cuda)
    out = ops.bcast_fma(a0, ta, p, B, T, C).view(B, T, C)
    ref = ta.double()[None] * p.double()[:, None] + a0.double()[None]
    worst = ((out.double() - ref).abs() / _ulp(ref)).max().item()
    record(f"elementwise_calls bcast_fma B={B} T={T} C={C}: {worst:.2f} ulp")
    assert worst <= 1.0


def test_rowscale_strided(cuda):
    """The crop-overlap averaging (1 / count per row) on a strided [M, 512] view: the s2 map of two 384 x 640 images.
    Bit-equal to torch's fp32 product; the columns around the view are not touched."""
    from odise_b200 import ops
    M = 2 * 96 * 160
    g = torch.Generator().manual_seed(11)
    buf = torch.randn(M, 524, generator=g).to(cuda)
    s = (1.0 / torch.randint(1, 5, (M,), generator=g).float()).to(cuda)
    before = buf.clone()
    view = buf[:, 4:516]
    assert view.stride(0) == 524
    ops.rowscale(view, s)
    assert torch.equal(view, before[:, 4:516] * s[:, None])
    assert torch.equal(buf[:, :4], before[:, :4]) and torch.equal(buf[:, 516:], before[:, 516:])


def test_gather_rows_clip_text(cuda):
    """ClipTextEngine.encode: token embedding + positional add over a [49408, 768] table, then the EOT-row gather.
    Ids include 0 (padding, repeated), the last row and repeats; bit-equal to torch's fp32 index + add."""
    from odise_b200 import ops
    V, W, TS, N = 49408, 768, 77, 3
    g = torch.Generator().manual_seed(12)
    table = torch.randn(V, W, generator=g).to(cuda)
    pos = (torch.randn(TS, W, generator=g) * 0.01).to(cuda)
    ids = torch.randint(1, V - 1, (N, TS), generator=g)
    ids[:, 0] = V - 2                                        # start of text
    ids[0, 5], ids[0, 6], ids[1, 7] = V - 1, V - 1, V - 1    # the last row, repeated
    ids[1, 10:20] = ids[1, 9]                                # a repeated token
    ids[2, 12:] = 0                                          # padding
    ids[2, 11] = V - 1
    idx = ids.view(-1).to(torch.int32).to(cuda)
    h = ops.gather_rows(table, idx, add=pos, add_period=TS)
    assert torch.equal(h, table[idx.long()] + pos.repeat(N, 1))
    eot = (ids.argmax(dim=-1) + torch.arange(N) * TS).to(torch.int32).to(cuda)
    rows = ops.gather_rows(h, eot)
    assert torch.equal(rows, h[eot.long()])


# ---------------------------------------------------------------------------------------------- bicubic crop resize
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32], ids=["u8", "f32"])
@pytest.mark.parametrize("side", [384, 448, 640])
def test_crop_resize_bicubic(cuda, record, dtype, side):
    """T.Resize((512, 512), BICUBIC) of square crops (384 and 448: the engine's upsample; 640: a downscale, no antialias)
    against float64 F.interpolate of the cropped tensor.  Three crops of three images: touching the right and bottom edges,
    inside the image, at the top-left corner.  Every pixel outside a crop is far from the crop's values, so sampling must
    clamp to the crop, not to the image."""
    from odise_b200 import ops
    S = 512
    H, W = side + 24, side + 40
    boxes = [(0, H - side, W - side), (1, 13, 21), (2, 0, 0)]
    g = torch.Generator().manual_seed(side)
    if dtype == torch.uint8:
        img = torch.full((3, 3, H, W), 255, dtype=torch.uint8)
        crops = [torch.randint(0, 101, (3, side, side), generator=g, dtype=torch.uint8) for _ in boxes]
        scale = 1.0 / 255
    else:
        img = torch.full((3, 3, H, W), 1e3)
        crops = [torch.rand(3, side, side, generator=g) for _ in boxes]
        scale = 1.0
    for (i, y0, x0), c in zip(boxes, crops):
        img[i, :, y0:y0 + side, x0:x0 + side] = c
    bx = torch.tensor(boxes, dtype=torch.int32).to(cuda)
    out = ops.crop_resize_bicubic(img.to(cuda), bx, len(boxes), H, W, side, side, S).cpu()
    ref = torch.cat([F.interpolate(c[None].double() * scale, size=(S, S), mode="bicubic", align_corners=False)
                     for c in crops])
    err = (out.double() - ref).abs().max().item()
    record(f"elementwise_calls crop_resize_bicubic {dtype} {side}->{S}: {err:.2e} absolute")
    assert err < 2e-6
