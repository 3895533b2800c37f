"""GPU parity of the wgmma GEMM / implicit conv (odise_gemm_bf16) against fp64 torch on the same inputs.
Tolerances: bf16x3 (nmma=3) is the parity mode -> 2e-5 of the output scale; plain bf16 (nmma=1) -> 2e-2."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


TOL = {1: 2e-2, 3: 2e-5}


@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("bn", [0, 64, 128, 160, 256])
@pytest.mark.parametrize("mnk", [(128, 128, 64), (256, 320, 320), (1000, 77, 200), (4096, 640, 2880), (100, 1342, 256)])
def test_gemm_plain(cuda, nmma, bn, mnk):
    from odise_b200 import lib
    M, N, K = mnk
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, generator=g).to(cuda)
    b = torch.randn(N, K, generator=g).to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    res = torch.randn(M, N, generator=g).to(cuda)
    ap, bp = lib.split(a), lib.split(b)
    out = torch.full((M, N), float("nan"), device=cuda)
    outp = lib.Planes.empty(M, N, cuda)
    lib.gemm(ap, bp, nmma=nmma, bias=bias, residual=res, out=out, out_planes=outp, force_bn=bn)
    torch.cuda.synchronize()
    ref = a.double() @ b.double().t() + bias.double() + res.double()
    assert _rel(out, ref) < TOL[nmma]
    assert _rel(outp.float(), out) < 1e-4   # (hi, lo) planes reproduce the fp32 output to ~2^-16
    if nmma == 3:
        assert _rel(ap.float(), a) < 1e-4


@pytest.mark.parametrize("act", [0, 1, 2, 3, 4])
def test_gemm_epilogue(cuda, act):
    from odise_b200 import lib
    M, N, K, G = 512, 256, 192, 4
    g = torch.Generator().manual_seed(act)
    a, b = torch.randn(M, K, generator=g).to(cuda), torch.randn(N, K, generator=g).to(cuda)
    rb = torch.randn(G, N, generator=g).to(cuda)
    out = torch.empty(M, N, device=cuda)
    lib.gemm(lib.split(a), lib.split(b), alpha=0.5, rowbias=rb, rows_per_group=M // G, act=act, out=out)
    ref = 0.5 * (a.double() @ b.double().t()) + rb.double().repeat_interleave(M // G, 0)
    ref = [lambda x: x, F.relu, F.silu, F.gelu, lambda x: x * torch.sigmoid(1.702 * x)][act](ref)   # 4: QuickGELU
    assert _rel(out, ref) < 2e-5


def test_gemm_batched_and_splitk(cuda):
    from odise_b200 import lib
    Bz, M, N, K = 3, 100, 256, 4096
    g = torch.Generator().manual_seed(5)
    a = torch.randn(Bz, M, K, generator=g).to(cuda)
    b = torch.randn(Bz, N, K, generator=g).to(cuda)
    ap, bp = lib.split(a), lib.split(b)
    ref = torch.bmm(a.double(), b.double().transpose(1, 2))
    out = torch.empty(Bz, M, N, device=cuda)
    lib.gemm(ap, bp, M=M, N=N, K=K, batch=Bz, a_bs=M * ap.ld, b_bs=N * bp.ld, out=out, out_bs=M * N)
    assert _rel(out, ref) < 2e-5
    ws = torch.empty(8 * Bz * M * N, device=cuda)
    out2 = torch.empty(Bz, M, N, device=cuda)
    lib.gemm(ap, bp, M=M, N=N, K=K, batch=Bz, a_bs=M * ap.ld, b_bs=N * bp.ld, out=out2, out_bs=M * N, split_k=8,
             workspace=ws)
    assert _rel(out2, ref) < 2e-5
    # shared B across the batch (weights)
    out3 = torch.empty(Bz, M, N, device=cuda)
    lib.gemm(ap, bp.row_slice(0, N), M=M, N=N, K=K, batch=Bz, a_bs=M * ap.ld, b_bs=0, out=out3, out_bs=M * N)
    ref3 = a.double() @ b[0].double().t()
    assert _rel(out3, ref3) < 2e-5


@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("shape", [(2, 64, 64, 64, 128), (3, 8, 8, 128, 64), (2, 16, 16, 320, 320), (1, 32, 32, 192, 100),
                                   (1, 128, 128, 64, 64), (1, 4, 256, 64, 32),
                                   # widths that neither divide nor are multiples of 128 (segmented fetch), e.g. 640 / 4
                                   (2, 24, 160, 64, 64), (1, 10, 40, 128, 96), (3, 7, 96, 64, 32), (1, 6, 8, 64, 64)])
def test_conv3x3_implicit(cuda, nmma, shape):
    """F.conv2d(x, w, padding=1) on NCHW == implicit GEMM on NHWC with k = (kh*3+kw)*C + c."""
    from odise_b200 import lib
    B, H, W, C, Co = shape
    g = torch.Generator().manual_seed(B + H + C)
    x = torch.randn(B, C, H, W, generator=g).to(cuda)
    w = (torch.randn(Co, C, 3, 3, generator=g) / (3 * C ** 0.5)).to(cuda)
    bias = torch.randn(Co, generator=g).to(cuda)
    ref = F.conv2d(x.double(), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1).reshape(B * H * W, Co)
    xp = lib.split(x.permute(0, 2, 3, 1).contiguous().view(B * H * W, C))
    wp = lib.split(w.permute(0, 2, 3, 1).contiguous().view(Co, 9 * C))
    out = torch.empty(B * H * W, Co, device=cuda)
    lib.gemm(xp, wp, M=B * H * W, N=Co, nmma=nmma, conv=(C, H, W), bias=bias, out=out)
    assert _rel(out, ref) < TOL[nmma]


def test_gemm_channel_slice_output(cuda):
    """epilogue writes into a column slice of a wider buffer (skip-concat without a copy)."""
    from odise_b200 import lib
    M, N, K, LD = 256, 128, 64, 320
    g = torch.Generator().manual_seed(9)
    a, b = torch.randn(M, K, generator=g).to(cuda), torch.randn(N, K, generator=g).to(cuda)
    buf = torch.zeros(M, LD, device=cuda)
    lib.gemm(lib.split(a), lib.split(b), out=buf[:, 64:64 + N], ld_out=LD)
    ref = a.double() @ b.double().t()
    assert _rel(buf[:, 64:64 + N], ref) < 2e-5
    assert buf[:, :64].abs().max() == 0 and buf[:, 64 + N:].abs().max() == 0


@pytest.mark.parametrize("M", [512, 64, 200])
def test_gemm_geglu_fused(cuda, M):
    """FF1 + GEGLU in one launch: quad-interleaved (a, gate) weight rows, out planes = a * gelu(gate)."""
    from odise_b200 import lib
    C = 320
    g = torch.Generator().manual_seed(12)
    x = torch.randn(M, C, generator=g).to(cuda)
    w = (torch.randn(8 * C, C, generator=g) / C ** 0.5).to(cuda)
    b = torch.randn(8 * C, generator=g).to(cuda)
    h4 = 4 * C
    wi = torch.stack([w[:h4].reshape(h4 // 4, 4, C), w[h4:].reshape(h4 // 4, 4, C)], 1).reshape(2 * h4, C).contiguous()
    bi = torch.stack([b[:h4].reshape(h4 // 4, 4), b[h4:].reshape(h4 // 4, 4)], 1).reshape(2 * h4).contiguous()
    out = lib.Planes.empty(M, h4, cuda)
    lib.gemm(lib.split(x), lib.split(wi), bias=bi, out_planes=out, geglu=True)
    y = x.double() @ w.double().t() + b.double()
    ref = y[:, :h4] * F.gelu(y[:, h4:])
    assert _rel(out.float(), ref) < 3e-5


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("shape", [(2, 64, 64, 64, 96), (1, 16, 16, 320, 320), (3, 8, 8, 128, 64), (1, 256, 256, 64, 64), (1, 512, 512, 128, 32),
                                   (2, 12, 160, 64, 64), (1, 20, 48, 128, 64)])
def test_conv3x3_stride2_implicit(cuda, mode, shape):
    """stride-2 3x3 conv as a strided implicit GEMM: mode 1 = pad (1,1) (ldm Downsample), mode 2 = F.pad(0,1,0,1) + no pad (VAE)."""
    from odise_b200 import lib
    B, H, W, C, Co = shape
    g = torch.Generator().manual_seed(B + H + C + mode)
    x = torch.randn(B, C, H, W, generator=g).to(cuda)
    w = (torch.randn(Co, C, 3, 3, generator=g) / (3 * C ** 0.5)).to(cuda)
    bias = torch.randn(Co, generator=g).to(cuda)
    if mode == 1:
        ref = F.conv2d(x.double(), w.double(), bias.double(), stride=2, padding=1)
    else:
        ref = F.conv2d(F.pad(x.double(), (0, 1, 0, 1)), w.double(), bias.double(), stride=2)
    Ho, Wo = ref.shape[-2:]
    assert (Ho, Wo) == (H // 2, W // 2)
    xp = lib.split(x.permute(0, 2, 3, 1).contiguous().view(B * H * W, C))
    wp = lib.split(w.permute(0, 2, 3, 1).contiguous().view(Co, 9 * C))
    out = torch.empty(B * Ho * Wo, Co, device=cuda)
    lib.gemm(xp, wp, M=B * Ho * Wo, N=Co, conv=(C, H, W), conv_mode=mode, bias=bias, out=out)
    assert _rel(out, ref.permute(0, 2, 3, 1).reshape(B * Ho * Wo, Co)) < 2e-5


@pytest.mark.parametrize("cfg", [(16, 8, 8, 1280, 1280, 160, 2), (16, 8, 8, 128, 192, 128, 4), (4, 16, 16, 640, 320, 256, 3)])
def test_conv3x3_split_k_with_fused_epilogue(cuda, cfg):
    """low-resolution UNet levels: implicit conv + split-K (lib.auto_split), epilogue (bias, time-embedding row bias,
    residual) applied by the reduce kernel."""
    from odise_b200 import lib
    B, H, W, C, Co, bn, sk = cfg
    g = torch.Generator().manual_seed(C + sk)
    x = torch.randn(B, C, H, W, generator=g).to(cuda)
    w = (torch.randn(Co, C, 3, 3, generator=g) / (3 * C ** 0.5)).to(cuda)
    bias, emb = torch.randn(Co, generator=g).to(cuda), torch.randn(B, Co, generator=g).to(cuda)
    res = torch.randn(B * H * W, Co, generator=g).to(cuda)
    ref = F.conv2d(x.double(), w.double(), bias.double(), padding=1) + emb.double()[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(B * H * W, Co) + res.double()
    xp = lib.split(x.permute(0, 2, 3, 1).contiguous().view(B * H * W, C))
    wp = lib.split(w.permute(0, 2, 3, 1).contiguous().view(Co, 9 * C))
    out = torch.empty(B * H * W, Co, device=cuda)
    M = B * H * W
    lib.gemm(xp, wp, M=M, N=Co, conv=(C, H, W), bias=bias, rowbias=emb, rows_per_group=H * W, residual=res, out=out,
             split_k=sk, force_bn=bn, workspace=lib.workspace(sk * M * Co * 4, cuda))
    assert _rel(out, ref) < 2e-5
    assert lib.auto_split(1024, 1280, 11520) == (160, 2) and lib.auto_split(65536, 320, 2880) == (0, 1)


def _gn_ref(x, B, HW, G, eps):
    xx = x.double().view(B, HW, G, -1).permute(0, 2, 1, 3).reshape(B, G, -1)
    return xx.mean(-1).reshape(-1), 1.0 / torch.sqrt(xx.var(-1, unbiased=False) + eps).reshape(-1)


@pytest.mark.parametrize("cfg", [
    dict(B=2, HW=1024, N=320, K=320, bn=0, extra=False),       # interior tiles, lean epilogue
    dict(B=2, HW=1024, N=320, K=320, bn=256, extra=True),      # edge tile in N (320 = 256 + 64), residual + row bias
    dict(B=4, HW=64, N=1280, K=640, bn=0, extra=True),         # 8x8 maps: a 128-row tile spans two images
    dict(B=1, HW=4096, N=640, K=128, bn=160, extra=False),
    dict(B=3, HW=96, N=64, K=64, bn=64, extra=False),          # M = 288: ragged last tile, whole 32-row segments
])
def test_gemm_groupnorm_statistics_in_epilogue(cuda, cfg):
    """desc.gn_partial: the producer half of the fused conv + GroupNorm (ldm ResBlock): per-(32-row segment, channel)
    records written by the epilogue, merged by odise_groupnorm_finalize_seg_f32 == torch group statistics of the output."""
    from odise_b200 import lib, ops
    B, HW, N, K = cfg["B"], cfg["HW"], cfg["N"], cfg["K"]
    M, G, eps = B * HW, 32, 1e-5
    g = torch.Generator().manual_seed(N + K + HW)
    a, b = torch.randn(M, K, generator=g).to(cuda), torch.randn(N, K, generator=g).to(cuda)
    bias = (torch.randn(N, generator=g) * 30).to(cuda)         # |mean| >> std inside some groups: the shifted sums must hold
    kw = {}
    if cfg["extra"]:
        kw = dict(residual=torch.randn(M, N, generator=g).to(cuda), rowbias=torch.randn(B, N, generator=g).to(cuda),
                  rows_per_group=HW)
    out = torch.empty(M, N, device=cuda)
    st = lib.GnStats(M, N, cuda)
    lib.gemm(lib.split(a), lib.split(b), bias=bias, out=out, force_bn=cfg["bn"], gn=st, **kw)
    assert not st.missing
    gamma, beta = torch.ones(N, device=cuda), torch.zeros(N, device=cuda)
    y_f, _ = ops.group_norm(out, B, HW, gamma, beta, eps, want_f32=True, want_planes=False, stats=st)
    y_s, _ = ops.group_norm(out, B, HW, gamma, beta, eps, want_f32=True, want_planes=False)
    torch.cuda.synchronize()
    mean, rstd = _gn_ref(out.cpu(), B, HW, G, eps)
    want = ((out.cpu().double().view(B, HW, G, -1) - mean.view(B, 1, G, 1)) * rstd.view(B, 1, G, 1)).view(M, N)
    assert _rel(y_f.cpu(), want) < 2e-5 and _rel(y_s.cpu(), want) < 2e-5
    assert _rel(y_f, y_s) < 1e-5


def test_groupnorm_statistics_of_a_concat_and_fallbacks(cuda):
    """Two producers write disjoint column ranges of one buffer (UNet skip concat, ldm.py:485) and of its records; a
    split-K producer marks the records missing and group_norm falls back to the stand-alone pass."""
    from odise_b200 import lib, ops
    B, HW, C1, C2, K = 2, 256, 640, 320, 256
    M = B * HW
    g = torch.Generator().manual_seed(9)
    a = torch.randn(M, K, generator=g).to(cuda)
    w1, w2 = torch.randn(C1, K, generator=g).to(cuda), torch.randn(C2, K, generator=g).to(cuda)
    buf = torch.empty(M, C1 + C2, device=cuda)
    st = lib.GnStats(M, C1 + C2, cuda)
    lib.gemm(lib.split(a), lib.split(w1), out=buf[:, :C1], gn=st.cols(0, C1))
    lib.gemm(lib.split(a), lib.split(w2), out=buf[:, C1:], gn=st.cols(C1, C2))
    gamma, beta = torch.randn(C1 + C2, generator=g).to(cuda), torch.randn(C1 + C2, generator=g).to(cuda)
    y_f, _ = ops.group_norm(buf, B, HW, gamma, beta, 1e-6, want_f32=True, want_planes=False, stats=st)
    want = torch.nn.functional.group_norm(buf.view(B, HW, -1).permute(0, 2, 1).double(), 32, gamma.double(), beta.double(), 1e-6)
    assert _rel(y_f.view(B, HW, -1).permute(0, 2, 1), want) < 2e-5
    # a column-slice consumer (the next block reads only the right half)
    y_r, _ = ops.group_norm(buf[:, C1:], B, HW, gamma[C1:].contiguous(), beta[C1:].contiguous(), 1e-6, want_f32=True,
                            want_planes=False, stats=st.cols(C1, C2))
    want_r = torch.nn.functional.group_norm(buf[:, C1:].reshape(B, HW, -1).permute(0, 2, 1).double(), 32, gamma[C1:].double(),
                                            beta[C1:].double(), 1e-6)
    assert _rel(y_r.view(B, HW, -1).permute(0, 2, 1), want_r) < 2e-5
    st2 = lib.GnStats(M, C2, cuda)
    out2 = torch.empty(M, C2, device=cuda)
    lib.gemm(lib.split(a), lib.split(w2), out=out2, gn=st2, split_k=2, workspace=lib.workspace(2 * M * C2 * 4, cuda))
    assert st2.missing
    y2, _ = ops.group_norm(out2, B, HW, gamma[:C2].contiguous(), beta[:C2].contiguous(), 1e-6, want_f32=True,
                           want_planes=False, stats=st2)
    want2 = torch.nn.functional.group_norm(out2.view(B, HW, -1).permute(0, 2, 1).double(), 32, gamma[:C2].double(),
                                           beta[:C2].double(), 1e-6)
    assert _rel(y2.view(B, HW, -1).permute(0, 2, 1), want2) < 2e-5
    assert lib.GnStats(100, 64, cuda).missing                     # ragged rows: no records


@pytest.mark.parametrize("kind", ["f32", "planes", "planes_hi_only", "planes_f16"])
@pytest.mark.parametrize("cfg", [
    dict(M=512, N=320, K=320, bn=0, batch=1, extra=False),       # interior tiles only
    dict(M=1000, N=333 // 4 * 4 + 4, K=200, bn=128, batch=1, extra=True),   # ragged M and N: edge tiles take the plain path
    dict(M=4096, N=640, K=128, bn=256, batch=1, extra=True),     # 640 = 2 x 256 + 128: interior + edge tile per row
    dict(M=256, N=256, K=64, bn=64, batch=3, extra=False),       # batched (decoder-style), one k-block
])
def test_gemm_tma_store_epilogue(cuda, kind, cfg):
    """Single-output GEMMs (fp32 OR planes) on interior and edge tiles: values must equal the fp64 product to the GEMM
    tolerance, also when the output is a column slice of a wider buffer."""
    from odise_b200 import lib
    M, N, K, Bz = cfg["M"], cfg["N"], cfg["K"], cfg["batch"]
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(Bz, M, K, generator=g).to(cuda)
    b = torch.randn(Bz, N, K, generator=g).to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    kw = dict(bias=bias, act=2 if cfg["extra"] else 0, force_bn=cfg["bn"])
    ref = torch.einsum("zmk,znk->zmn", a.double(), b.double()) + bias.double()
    if cfg["extra"]:
        ref = torch.nn.functional.silu(ref)
        res = torch.randn(Bz, M, N, generator=g).to(cuda)
        kw.update(residual=res, ld_res=N, res_bs=M * N)
        ref = ref + res.double()
    if Bz > 1:
        kw.update(batch=Bz, a_bs=M * K, b_bs=N * K)
    ap, bp = lib.split(a.view(Bz * M, K)), lib.split(b.view(Bz * N, K))
    pad = 32                                       # outputs live in columns [pad, pad + N) of a wider buffer
    if kind == "f32":
        buf = torch.full((Bz, M, N + 2 * pad), 7.0, device=cuda)
        lib.gemm(ap, bp, M=M, N=N, K=K, out=buf[:, :, pad:], ld_out=N + 2 * pad, out_bs=M * (N + 2 * pad), **kw)
        torch.cuda.synchronize()
        assert _rel(buf[:, :, pad:pad + N], ref) < 2e-5
        assert (buf[:, :, :pad] == 7.0).all() and (buf[:, :, pad + N:] == 7.0).all()        # nothing outside the slice
    else:
        f16 = kind == "planes_f16"
        P = lib.Planes.empty(Bz * M, N + 2 * pad, cuda, lo=kind != "planes_hi_only", f16=f16)
        P.hi.fill_(0)
        if P.lo is not None:
            P.lo.fill_(0)
        out = P.col_slice(pad, N)
        lib.gemm(ap, bp, M=M, N=N, K=K, out_planes=out, outp_bs=M * P.ld, **kw)
        torch.cuda.synchronize()
        got = P.float().view(Bz, M, -1)
        tol = 1e-4 if kind != "planes_hi_only" else 6e-3
        assert _rel(got[:, :, pad:pad + N], ref) < tol
        assert (got[:, :, :pad] == 0).all() and (got[:, :, pad + N:N + 2 * pad] == 0).all()


@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
@pytest.mark.parametrize("case", ["unet", "clip", "clip_hi_only", "decoder", "vae_bf16", "clip_split_k"])
def test_gemm_vt_producer(cuda, record, nmma, bn, case):
    """The attention kernels' V^T operand, written by the swapped-operand GEMM V^T = W X^T + bias_m[:, None] into
    (hi, lo) planes: fp16 pairs for odise_attention_tc (clip.py:56, head.py:338, unet.py:212), bf16 pairs for the VAE's
    P V GEMM (vae.py:126).  unet: M = heads * HS with zero pad rows in W, no bias_m | clip: M = 1024, N = B * 584 |
    decoder: batch = B over image row blocks of the level memory (b_bs), image z written at column z * hw8, N = hw = 252,
    whose 4 pad columns per image must stay untouched | clip_split_k: bias_m applied by the split-K reduce kernel.
    Ragged N and forced tile widths send tiles through both the interior epilogue and epilogue_quad."""
    from odise_b200 import lib, ops
    g = torch.Generator().manual_seed(len(case) * 13 + bn + nmma)
    f16, lo, batch, split_k = True, True, 1, 1
    if case == "unet":
        heads, d, HS, C, N = 8, 40, 64, 320, 2 * 1024
        W = ops.head_pad_rows(torch.randn(heads * d, C, generator=g) * C ** -0.5, heads, d, HS)
        bm = None
    elif case == "decoder":
        B, S, start, hw, hw8, C = 2, 400, 100, 252, 256, 256
        W = torch.randn(3 * 8 * 64, C, generator=g) * C ** -0.5
        bm = torch.randn(W.shape[0], generator=g)
        N, batch = hw, B
    else:
        C, B, TS = 1024, 2, 584
        if case == "vae_bf16":
            C, B, TS = 512, 1, 4096
        W = torch.randn(C, C, generator=g) * C ** -0.5
        bm = torch.randn(C, generator=g)
        N = B * TS
        f16 = case != "vae_bf16"
        lo = case != "clip_hi_only"
        split_k = 4 if case == "clip_split_k" else 1
    M = W.shape[0]
    Wp = lib.split(W.to(cuda))
    kw = dict(nmma=nmma, force_bn=bn, bias_m=None if bm is None else bm.to(cuda))
    if split_k > 1:
        kw.update(split_k=split_k, workspace=torch.empty(split_k * M * N, device=cuda))
    if case == "decoder":
        mem = torch.randn(B, S, C, generator=g)                  # level rows [start, start + hw) of every image
        X = mem[:, start:start + hw]
        xp = lib.split(mem.view(B * S, C).to(cuda)).row_slice(start, hw)
        out = lib.Planes.empty(M, B * hw8, cuda, lo=lo, f16=f16)
        kw.update(N=hw, batch=B, b_bs=S * xp.ld, outp_bs=hw8)
        ref = torch.einsum("mc,btc->mbt", W.double(), X.double())
    else:
        X = torch.randn(N, C, generator=g)
        xp = lib.split(X.to(cuda))
        out = lib.Planes.empty(M, N, cuda, lo=lo, f16=f16)
        ref = W.double() @ X.double().T
    if bm is not None:
        ref = ref + (bm.double().view(-1, 1, 1) if case == "decoder" else bm.double().view(-1, 1))
    for t in (out.hi, out.lo):
        if t is not None:
            t.view(torch.int16).fill_(0x3C01)                   # a sentinel: 1.0009765625 in fp16, 1.0078125 in bf16
    lib.gemm(Wp, xp, out_planes=out, **kw)
    torch.cuda.synchronize()
    got = out.float().cpu()
    if case == "decoder":
        got = got.view(M, B, hw8)
        for t in (out.hi, out.lo):
            if t is not None:
                assert (t.view(torch.int16).view(M, B, hw8)[:, :, hw:] == 0x3C01).all()   # pad keys untouched
        got = got[:, :, :hw]
    tol = TOL[nmma] if lo else max(TOL[nmma], 1e-3 if f16 else 6e-3)   # hi only: one fp16 / bf16 rounding of the output
    e = _rel(got, ref)
    record(f"gemm V^T {case} bn={bn} nmma={nmma}: rel err {e:.3e}")
    assert e < tol
