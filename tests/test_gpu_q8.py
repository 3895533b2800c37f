"""GPU tests of the F16Q8 operand mode (ODISE_PLANES_F16Q8, odise_gemm_desc.nmma = 2): fp16 hi plane + e5m2 correction
bytes, A_hi*B_hi on kind::f16 and the two cross terms on kind::f8f6f4 (csrc/ptx.cuh, csrc/gemm_tc.cu).

Two kinds of checks:
* EXACT scheme: the GEMM result must equal a torch emulation of the same operand rounding (fp16 hi, e5m2 of x*2^-6 and of
  (x - hi)*2^6, three exact products accumulated in fp64) to fp32-accumulation level -> proves the byte layout, the pairing of
  the q_hi / q_lo halves and the scales, independent of how good the scheme is;
* ACCURACY: against fp64 torch on the unrounded inputs, 2e-4 of the output scale (bf16x3: 2e-5; the end-to-end bar is 1e-3
  and the UNet taps land at ~1e-4, tests/test_gpu_unet.py)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

S = 6


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def _e5m2(x):
    return x.clamp(-57344.0, 57344.0).to(torch.float8_e5m2).double()


def _q8_terms(x):
    """(hi, q_hi, q_lo) as the kernels store them, in fp64"""
    x = x.float()
    hi = x.clamp(-65504.0, 65504.0).half().float()
    return hi.double(), _e5m2(x * 2.0 ** -S), _e5m2((x - hi) * 2.0 ** S)


def _emul(a, b):
    ah, aqh, aql = _q8_terms(a)
    bh, bqh, bql = _q8_terms(b)
    return ah @ bh.t() + aqh @ bql.t() + aql @ bqh.t()


def test_q8_split_layout_and_value(cuda):
    from odise_b200 import lib
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(70, 200, generator=g) * torch.logspace(-3, 2, 200)).to(cuda)   # 5 decades of magnitudes
    p = lib.split(x, lo=lib.Q8)
    assert p.fmt == "q8" and p.ld == 256
    hi, qh, ql = _q8_terms(x.cpu())
    got_hi = p.hi.view(torch.float16).view(70, 256)[:, :200].cpu().double()
    assert torch.equal(got_hi, hi)
    qb = p.lo.view(torch.uint8).view(70, 4, 2, 64).cpu()
    got_qh = qb[:, :, 0, :].reshape(70, 256)[:, :200].contiguous().view(torch.float8_e5m2).double()
    got_ql = qb[:, :, 1, :].reshape(70, 256)[:, :200].contiguous().view(torch.float8_e5m2).double()
    assert torch.equal(got_qh, qh) and torch.equal(got_ql, ql)
    assert qb[:, 3, :, 8:].abs().max() == 0                     # pad bytes of the last k-block stay zero
    assert _rel(p.float(), x) < 2e-4


@pytest.mark.parametrize("bn", [0, 64, 128, 160, 256])
@pytest.mark.parametrize("mnk", [(128, 128, 64), (256, 320, 320), (1000, 77, 200), (4096, 640, 2880), (100, 1342, 256)])
def test_q8_gemm_plain(cuda, bn, mnk):
    from odise_b200 import lib
    M, N, K = mnk
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, generator=g)
    b = torch.randn(N, K, generator=g) * 0.05
    bias = torch.randn(N, generator=g).to(cuda)
    res = torch.randn(M, N, generator=g).to(cuda)
    ap, bp = lib.split(a.to(cuda), lo=lib.Q8), lib.split(b.to(cuda), lo=lib.Q8)
    out = torch.full((M, N), float("nan"), device=cuda)
    outp = lib.Planes.empty(M, N, cuda, lo=lib.Q8)
    lib.gemm(ap, bp, bias=bias, residual=res, out=out, out_planes=outp, force_bn=bn)
    torch.cuda.synchronize()
    extra = bias.double().cpu() + res.double().cpu()
    assert _rel(out.cpu(), _emul(a, b) + extra) < 2e-5                      # exact scheme, fp32 accumulation
    assert _rel(out.cpu() - extra, a.double() @ b.double().t()) < 2e-4      # accuracy of the scheme
    assert _rel(outp.float(), out) < 2e-4
    if N % 4 == 0:                                                          # the epilogue writes the same bytes as split()
        ref_p = lib.split(out, lo=lib.Q8)
        assert torch.equal(outp.hi, ref_p.hi) and torch.equal(outp.lo, ref_p.lo)


def test_q8_gemm_batched_splitk_and_mixed_outputs(cuda):
    from odise_b200 import lib
    Bz, M, N, K = 3, 100, 256, 4096
    g = torch.Generator().manual_seed(5)
    a = torch.randn(Bz, M, K, generator=g)
    b = torch.randn(Bz, N, K, generator=g)
    ap, bp = lib.split(a.to(cuda), lo=lib.Q8), lib.split(b.to(cuda), lo=lib.Q8)
    ref = torch.stack([_emul(a[i], b[i]) for i in range(Bz)])
    out = torch.empty(Bz, M, N, device=cuda)
    lib.gemm(ap, bp, M=M, N=N, K=K, batch=Bz, a_bs=M * ap.ld, b_bs=N * bp.ld, out=out, out_bs=M * N)
    assert _rel(out.cpu(), ref) < 2e-5
    ws = torch.empty(8 * Bz * M * N, device=cuda)
    out2 = torch.empty(Bz, M, N, device=cuda)
    lib.gemm(ap, bp, M=M, N=N, K=K, batch=Bz, a_bs=M * ap.ld, b_bs=N * bp.ld, out=out2, out_bs=M * N, split_k=8, workspace=ws)
    assert _rel(out2.cpu(), ref) < 2e-5
    # F16Q8 operands -> bf16-pair and fp16-pair output planes (the q / k / V^T operands of the attention kernel)
    pb = lib.Planes.empty(M, N, cuda, lo=True)
    pf = lib.Planes.empty(M, N, cuda, lo=True, f16=True)
    lib.gemm(ap.row_slice(0, M), bp.row_slice(0, N), out_planes=pb)
    lib.gemm(ap.row_slice(0, M), bp.row_slice(0, N), out_planes=pf)
    assert pb.fmt == "bf16" and pf.fmt == "f16"
    assert _rel(pb.float().cpu(), ref[0]) < 1e-4 and _rel(pf.float().cpu(), ref[0]) < 1e-4
    with pytest.raises(lib.OdiseError):
        lib.gemm(ap.row_slice(0, M), lib.split(b[0].to(cuda)), out_planes=pb)      # formats of the operands must agree


@pytest.mark.parametrize("shape", [(2, 64, 64, 64, 128), (3, 8, 8, 128, 64), (2, 16, 16, 320, 320), (1, 128, 128, 64, 64),
                                   (2, 24, 160, 64, 64), (1, 10, 40, 128, 96)])
def test_q8_conv3x3_implicit(cuda, shape):
    from odise_b200 import lib
    B, H, W, C, Co = shape
    g = torch.Generator().manual_seed(B + H + C)
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(Co, C, 3, 3, generator=g) / (3 * C ** 0.5)
    bias = torch.randn(Co, generator=g)
    ref = F.conv2d(x.double(), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1).reshape(B * H * W, Co)
    xp = lib.split(x.permute(0, 2, 3, 1).contiguous().view(B * H * W, C).to(cuda), lo=lib.Q8)
    wp = lib.split(w.permute(0, 2, 3, 1).contiguous().view(Co, 9 * C).to(cuda), lo=lib.Q8)
    out = torch.empty(B * H * W, Co, device=cuda)
    lib.gemm(xp, wp, M=B * H * W, N=Co, conv=(C, H, W), bias=bias.to(cuda), out=out)
    assert _rel(out.cpu(), ref) < 2e-4
    # exact scheme: the implicit conv equals the GEMM over the materialised im2col matrix in the same format
    cols = F.unfold(x, 3, padding=1).view(B, C, 9, H * W).permute(0, 3, 2, 1).reshape(B * H * W, 9 * C)
    em = _emul(cols, w.permute(0, 2, 3, 1).reshape(Co, 9 * C)) + bias.double()
    assert _rel(out.cpu(), em) < 2e-5


@pytest.mark.parametrize("mode", [1, 2])
def test_q8_conv3x3_stride2(cuda, mode):
    from odise_b200 import lib
    B, H, W, C, Co = 2, 64, 64, 64, 96
    g = torch.Generator().manual_seed(3 + mode)
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(Co, C, 3, 3, generator=g) / (3 * C ** 0.5)
    xin = x if mode == 1 else F.pad(x, (0, 1, 0, 1))
    ref = F.conv2d(xin.double(), w.double(), None, stride=2, padding=1 if mode == 1 else 0)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, Co)
    xp = lib.split(x.permute(0, 2, 3, 1).contiguous().view(B * H * W, C).to(cuda), lo=lib.Q8)
    wp = lib.split(w.permute(0, 2, 3, 1).contiguous().view(Co, 9 * C).to(cuda), lo=lib.Q8)
    out = torch.empty(B * (H // 2) * (W // 2), Co, device=cuda)
    lib.gemm(xp, wp, M=out.shape[0], N=Co, conv=(C, H, W), conv_mode=mode, out=out)
    assert _rel(out.cpu(), ref) < 2e-4


@pytest.mark.parametrize("kind", ["f32", "planes"])
@pytest.mark.parametrize("cfg", [(1024, 512, 320, False), (65536, 640, 320, True), (896, 320, 1280, True)])
def test_q8_tma_store_epilogue(cuda, kind, cfg):
    """single-output GEMMs in the F16Q8 mode, fp32 or F16Q8 output planes (fp16 tile + the two e5m2 byte blocks per 64 columns)"""
    from odise_b200 import lib
    M, N, K, extra = cfg
    g = torch.Generator().manual_seed(M + N)
    a = torch.randn(M, K, generator=g).to(cuda)
    b = (torch.randn(N, K, generator=g) * 0.05).to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    res = torch.randn(M, N, generator=g).to(cuda) if extra else None
    ap, bp = lib.split(a, lo=lib.Q8), lib.split(b, lo=lib.Q8)
    both = torch.empty(M, N, device=cuda)
    bothp = lib.Planes.empty(M, N, cuda, lo=lib.Q8)
    lib.gemm(ap, bp, bias=bias, residual=res, out=both, out_planes=bothp)       # two outputs: transposing epilogue
    if kind == "f32":
        out = torch.empty(M, N, device=cuda)
        lib.gemm(ap, bp, bias=bias, residual=res, out=out)
        assert torch.equal(out, both)
    else:
        outp = lib.Planes.empty(M, N, cuda, lo=lib.Q8)
        lib.gemm(ap, bp, bias=bias, residual=res, out_planes=outp)
        assert torch.equal(outp.hi, bothp.hi) and torch.equal(outp.lo, bothp.lo)


@pytest.mark.parametrize("M", [512, 200])
def test_q8_geglu_fused(cuda, M):
    from odise_b200 import lib
    C = 320
    g = torch.Generator().manual_seed(12)
    x = torch.randn(M, C, generator=g).to(cuda)
    w = (torch.randn(8 * C, C, generator=g) / C ** 0.5).to(cuda)
    b = torch.randn(8 * C, generator=g).to(cuda)
    h4 = 4 * C
    wi = torch.stack([w[:h4].reshape(h4 // 4, 4, C), w[h4:].reshape(h4 // 4, 4, C)], 1).reshape(2 * h4, C).contiguous()
    bi = torch.stack([b[:h4].reshape(h4 // 4, 4), b[h4:].reshape(h4 // 4, 4)], 1).reshape(2 * h4).contiguous()
    out = lib.Planes.empty(M, h4, cuda, lo=lib.Q8)
    lib.gemm(lib.split(x, lo=lib.Q8), lib.split(wi, lo=lib.Q8), bias=bi, out_planes=out, geglu=True)
    y = x.double() @ w.double().t() + b.double()
    ref = y[:, :h4] * F.gelu(y[:, h4:])
    assert _rel(out.float(), ref) < 3e-4


def test_q8_gemm_gn_records_and_chain(cuda):
    """conv (records in the epilogue) -> GroupNorm + SiLU (F16Q8 planes) -> conv: the ResBlock pattern in the new format"""
    from odise_b200 import lib, ops
    B, H, W, C = 2, 32, 32, 64
    g = torch.Generator().manual_seed(21)
    x = torch.randn(B, C, H, W, generator=g)
    w1 = torch.randn(C, C, 3, 3, generator=g) / (3 * C ** 0.5)
    w2 = torch.randn(C, C, 3, 3, generator=g) / (3 * C ** 0.5)
    gam, bet = torch.randn(C, generator=g), torch.randn(C, generator=g)
    h = F.conv2d(x.double(), w1.double(), None, padding=1)
    y = F.silu(F.group_norm(h, 32, gam.double(), bet.double(), 1e-5))
    ref = F.conv2d(y, w2.double(), None, padding=1).permute(0, 2, 3, 1).reshape(B * H * W, C)
    M = B * H * W
    xp = lib.split(x.permute(0, 2, 3, 1).contiguous().view(M, C).to(cuda), lo=lib.Q8)
    cw = lambda w: lib.split(w.permute(0, 2, 3, 1).contiguous().view(C, 9 * C).to(cuda), lo=lib.Q8)
    hbuf = torch.empty(M, C, device=cuda)
    st = lib.GnStats(M, C, cuda)
    lib.gemm(xp, cw(w1), M=M, N=C, conv=(C, H, W), out=hbuf, gn=st)
    assert not st.missing
    _, yp = ops.group_norm(hbuf, B, H * W, gam.to(cuda), bet.to(cuda), 1e-5, ops.ACT_SILU, lo=lib.Q8, stats=st)
    assert yp.fmt == "q8"
    assert _rel(yp.float().cpu(), y.permute(0, 2, 3, 1).reshape(M, C)) < 3e-4
    out = torch.empty(M, C, device=cuda)
    lib.gemm(yp, cw(w2), M=M, N=C, conv=(C, H, W), out=out)
    assert _rel(out.cpu(), ref) < 3e-4


def test_q8_producers_match_the_bf16_pair(cuda):
    """every pass that writes operand planes: the F16Q8 planes decode to the same values as the bf16 pair (both ~2^-14)"""
    from odise_b200 import lib, ops
    g = torch.Generator().manual_seed(33)
    rows, cols = 300, 320
    x = torch.randn(rows, cols, generator=g).to(cuda)
    gam, bet = torch.randn(cols, generator=g).to(cuda), torch.randn(cols, generator=g).to(cuda)

    def both(fn):
        a, b = fn(True), fn(lib.Q8)
        assert a.fmt == "bf16" and b.fmt == "q8"
        assert _rel(b.float(), a.float()) < 2e-4, fn
        # and the bytes are exactly the encoding of the fp32 values the bf16 pair approximates to 2^-16
        assert _rel(b.float(), lib.split(a.float(), lo=lib.Q8).float()) < 2e-4

    both(lambda lo: ops.layer_norm(x, gam, bet, lo=lo)[1])
    both(lambda lo: ops.layer_norm(x, gam, bet, res=x, post_add=x, lo=lo)[1])
    both(lambda lo: ops.add_split(x, x, lo=lo)[1])
    both(lambda lo: ops.act_split(x, ops.ACT_SILU, lo=lo))
    both(lambda lo: ops.geglu(torch.cat([x, x], 1).contiguous(), lo=lo))
    both(lambda lo: ops.l2_normalize_split(x, lo=lo))
    both(lambda lo: ops.softmax_split(x, rows, 300, cols, 0.3, lo=lo))
    # long rows take the single-read shared-memory kernel (the KL-VAE 4096-key attention): against torch, both formats
    xl = (torch.randn(40, 1024, generator=g) * 3).to(cuda)
    want = torch.softmax(xl[:, :1000].double() * 0.3, -1)
    for lo_ in (True, lib.Q8):
        pl = ops.softmax_split(xl, 40, 1000, 1024, 0.3, lo=lo_)
        assert _rel(pl.float()[:, :1000], want) < 2e-4 and pl.float()[:, 1000:].abs().max() == 0
    both(lambda lo: ops.softmax_split(xl, 40, 1000, 1024, 0.3, lo=lo))
    both(lambda lo: ops.group_norm(x[:256].contiguous(), 2, 128, gam, bet, 1e-5, ops.ACT_SILU, lo=lo)[1])
    xs = torch.randn(2 * 8 * 8, 64, generator=g).to(cuda)
    both(lambda lo: ops.upsample2x_split(xs, 2, 8, 8, lo=lo))
    img = torch.randn(2, 3, 28, 28, generator=g).to(cuda)
    a, b = ops.patchify_split(img, 2, 28, 14, lo=True), ops.patchify_split(img, 2, 28, 14, lo=lib.Q8)
    assert (a.ld, b.ld) == (592, 640) and _rel(b.float()[:, :588], a.float()[:, :588]) < 2e-4 and b.float()[:, 588:].abs().max() == 0
    x4 = torch.randn(2 * 6 * 6, 4, generator=g).to(cuda)
    a, b = ops.im2col3x3_split(x4, 2, 6, 6, lo=True)[0], ops.im2col3x3_split(x4, 2, 6, 6, lo=lib.Q8)[0]
    assert b.ld == 64 and _rel(b.float()[:, :36], a.float()[:, :36]) < 2e-4 and b.float()[:, 36:].abs().max() == 0


def test_q8_attention_and_msda_outputs(cuda):
    from odise_b200 import lib, ops
    g = torch.Generator().manual_seed(44)
    B, heads, d, T = 2, 8, 40, 256
    HS = ops.head_stride(d)
    qf = torch.randn(B * T, heads * HS, generator=g).to(cuda)
    kf = torch.randn(B * T, heads * HS, generator=g).to(cuda)
    vf = torch.randn(heads * HS, B * T, generator=g).to(cuda)
    q, k, vt = lib.split(qf), lib.split(kf), lib.split(vf, f16=True)
    _, o3 = ops.attention_tc(q, k, vt, B, heads, d, T, T, d ** -0.5, 3)
    _, o2 = ops.attention_tc(q, k, vt, B, heads, d, T, T, d ** -0.5, 2, lo=lib.Q8)
    assert o3.fmt == "bf16" and o2.fmt == "q8" and o2.ld == 320
    assert _rel(o2.float(), o3.float()) < 2e-4
    # decoder self-attention (SIMT, d = 32)
    Q = 100
    qkv = torch.randn(B * Q, 768, generator=g).to(cuda)
    m3 = ops.mha_d32(qkv, 768, qkv[:, 256:], qkv[:, 512:], 768, B, Q, Q, 8, 32 ** -0.5, lo=True)
    m2 = ops.mha_d32(qkv, 768, qkv[:, 256:], qkv[:, 512:], 768, B, Q, Q, 8, 32 ** -0.5, lo=lib.Q8)
    assert _rel(m2.float(), m3.float()) < 2e-4
    # MSDeformAttn output planes
    N, M, D, L, P = 2, 8, 32, 3, 4
    shapes = torch.tensor([[8, 8], [16, 16], [32, 32]], dtype=torch.int64)
    S = int((shapes[:, 0] * shapes[:, 1]).sum())
    starts = torch.cat([torch.zeros(1, dtype=torch.int64), (shapes[:, 0] * shapes[:, 1]).cumsum(0)[:-1]])
    value = torch.randn(N, S, M, D, generator=g).to(cuda)
    ref = torch.rand(N, S, L, 2, generator=g).to(cuda)
    offs = (torch.randn(N, S, M, L, P, 2, generator=g) * 2).to(cuda)
    logits = torch.randn(N, S, M, L * P, generator=g).to(cuda)
    a = ops.msda_fused(value, shapes.to(cuda), starts.to(cuda), ref, offs, logits, N, S, M, D, L, S, P, lo=True)[1]
    b = ops.msda_fused(value, shapes.to(cuda), starts.to(cuda), ref, offs, logits, N, S, M, D, L, S, P, lo=lib.Q8)[1]
    assert _rel(b.float(), a.float()) < 2e-4
