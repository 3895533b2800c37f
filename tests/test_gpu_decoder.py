"""The fused decoder prediction heads (odise_mask_head_* kernels, odise_b200.decoder) on the GPU: kernel parity against
float64, threshold bits against torch's composition, autocast error against the reference composition's, the fused
decoder against the float64 oracle with forced masks, dispatch, host synchronisation, determinism, CUDA graphs and
torch.compile."""

import pytest
import torch
import torch.nn.functional as F

from odise_b200 import lib
from odise_b200 import decoder as dec
from oracle import m2f

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib.load()
    return torch.device("cuda:0")


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def _torch_attn_mask(om, size, heads):
    """the reference's attention mask on a given outputs_mask, with the decoder's fix-up (odise.py:683, :760-774)"""
    am = F.interpolate(om, size=size, mode="bilinear", align_corners=False)
    am = (am.sigmoid().flatten(2).unsqueeze(1).repeat(1, heads, 1, 1).flatten(0, 1) < 0.5).bool()
    am[torch.where(am.sum(-1) == am.shape[-1])] = False
    return am


@pytest.mark.parametrize("shape", [(2, 100, 37, 53), (1, 100, 64, 96), (2, 7, 5, 3)])
def test_kernel_parity_f32(cuda, shape):
    """outputs_mask and pooled features within 1e-5 x max|ref| of float64, pooling with the kernel's own hard mask, and
    both gradients against float64 autograd of the composed formulas with that mask"""
    B, Q, H, W = shape
    g = torch.Generator().manual_seed(H * W + Q)
    E = torch.randn(B, Q, 256, generator=g).to(cuda)
    X = torch.randn(B, 256, H, W, generator=g).to(cuda)
    om, pooled, w = lib.mask_head_forward(E, X)
    E64, X64 = E.double().requires_grad_(), X.double().requires_grad_()
    om64 = torch.einsum("bqc,bchw->bqhw", E64, X64)
    assert _rel(om, om64) < 1e-5
    m = (om.sigmoid() > 0.5).double()
    cnt = m.sum((-1, -2))
    assert torch.equal(w, torch.where(cnt > 0, 1.0 / (cnt.float() + 1e-8), 0.0))
    pooled64 = torch.einsum("bchw,bqhw->bqc", X64, m / (cnt[..., None, None] + 1e-8))
    assert _rel(pooled, pooled64) < 1e-5
    G = torch.randn(B, Q, H, W, generator=g).to(cuda)
    Gp = torch.randn(B, Q, 256, generator=g).to(cuda)
    ge, gx = lib.mask_head_backward(E, X, om, w, G, Gp)
    torch.autograd.backward([om64, pooled64], [G.double(), Gp.double()])
    assert _rel(ge, E64.grad) < 1e-5
    assert _rel(gx, X64.grad) < 1e-5


def _adversarial(dtype, B, Q, HW, g):
    """logits in dtype: random, 0, +-1e-8, values around which the dtype's sigmoid rounds to 0.5, whole rows blocked
    (all very negative) and a full row"""
    x = torch.randn(B, Q, HW, generator=g) * 2
    ulp = 2.0 ** -11 if dtype == torch.float16 else (2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -24)
    special = torch.tensor([0.0, 1e-8, -1e-8, ulp, -ulp, 2 * ulp, -2 * ulp, 4 * ulp, -4 * ulp, 1e-3, -1e-3, 3e-3,
                            -3e-3, 5e-4, -5e-4])
    for q in range(0, Q, 3):
        x[:, q, : special.numel()] = special[torch.randperm(special.numel(), generator=g)]
    x[:, 1] = -8.0            # empty pooling mask, every key blocked
    x[:, 2] = 8.0             # full pooling mask
    x[:, 4] = torch.linspace(-6 * ulp, 6 * ulp, HW)
    return x.to(dtype)


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_threshold_bits(cuda, dt):
    """hard mask and attention mask (fix-up included) bit-equal to torch's composition on the kernel's own outputs_mask.
    With one-hot features (X[c, p] = [c == p], H*W <= 256) the kernel's outputs_mask is exactly the chosen logits and
    pooled[b, q, c] = w m[b, q, c], so the kernel's hard mask is read off pooled != 0."""
    dtype = DT[dt]
    g = torch.Generator().manual_seed(11)
    B, Q, H, W = 2, 24, 12, 20
    logits = _adversarial(dtype, B, Q, H * W, g).to(cuda)
    E = torch.zeros(B, Q, 256, dtype=dtype, device=cuda)
    E[:, :, : H * W] = logits
    X = torch.zeros(B, 256, H * W, dtype=dtype, device=cuda)
    X[:, torch.arange(H * W), torch.arange(H * W)] = 1
    X = X.view(B, 256, H, W)
    om, pooled, w = lib.mask_head_forward(E, X)
    n_om = int((om.view(B, Q, H * W) != logits).sum())
    want = om.sigmoid() > 0.5
    got = pooled[:, :, : H * W] != 0
    n_hard = int((got != want.flatten(2)).sum())
    print(f"{dt}: outputs_mask values that differ {n_om}, hard-mask bits that differ {n_hard}")
    assert n_om == 0 and n_hard == 0
    assert not want[:, 1].any() and want[:, 2].all() and (pooled[:, 1] == 0).all()
    for size in [(5, 7), (3, 10), (12, 20), (24, 40), (1, 1)]:
        am = lib.mask_head_attn_mask(om, size, 8)
        ref = _torch_attn_mask(om, size, 8)
        n = (am != ref).sum().item()
        print(f"{dt}: attention-mask bits that differ at {size}: {n}")
        assert n == 0, (dt, size, n)
        assert not am.view(B, 8, Q, -1)[:, :, 1].any()       # all-blocked row cleared


@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_autocast_error(cuda, dt):
    """under autocast: outputs_mask and pooled features of the fused kernel against float64 (pooling with the kernel's
    own hard mask), within the error of the reference composition under the same autocast (its own mask)"""
    dtype = DT[dt]
    g = torch.Generator().manual_seed(5)
    B, Q, H, W = 2, 100, 48, 40
    E = torch.randn(B, Q, 256, generator=g).to(cuda) * 0.1
    X = torch.randn(B, 256, H, W, generator=g).to(cuda)
    om, pooled, w = lib.mask_head_forward(E.to(dtype), X.to(dtype))
    om64 = torch.einsum("bqc,bchw->bqhw", E.double(), X.double())

    def pool64(mask):
        m = (mask.sigmoid() > 0.5).double()     # sigmoid in the mask's dtype, as MaskPooling computes it
        return torch.einsum("bchw,bqhw->bqc", X.double(), m / (m.sum((-1, -2), keepdim=True) + 1e-8))

    with torch.autocast("cuda", dtype=dtype):
        om_ref = torch.einsum("bqc,bchw->bqhw", E, X)
        pooled_ref = dec.MaskPooling()(X, om_ref)["mask_pooled_features"]
    e_om, r_om = _rel(om, om64), _rel(om_ref, om64)
    e_p, r_p = _rel(pooled, pool64(om)), _rel(pooled_ref, pool64(om_ref))
    print(f"{dt}: outputs_mask err fused {e_om:.2e} / composed {r_om:.2e}; pooled err fused {e_p:.2e} / "
          f"composed {r_p:.2e}")
    # both paths accumulate in fp32 and round once, so the worst error is set by that rounding; the 10 % covers only a
    # different fp32 summation order moving one value across a rounding boundary
    assert e_om <= 1.1 * r_om and e_p <= 1.1 * r_p


@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_autocast_gradients(cuda, dt):
    """16-bit backward (tensor-core kernels) against float64 autograd of the composed formulas, with the kernel's own
    hard mask, within the error of the same composition run under autocast"""
    dtype = DT[dt]
    g = torch.Generator().manual_seed(6)
    B, Q, H, W = 2, 100, 48, 40
    E = (torch.randn(B, Q, 256, generator=g) * 0.1).to(cuda)
    X = torch.randn(B, 256, H, W, generator=g).to(cuda)
    G = (torch.randn(B, Q, H, W, generator=g) * 1e-3).to(cuda, dtype)
    Gp = (torch.randn(B, Q, 256, generator=g) * 1e-2).to(cuda, dtype)
    Et, Xt = E.to(dtype), X.to(dtype)
    om, pooled, w = lib.mask_head_forward(Et, Xt)
    ge, gx = lib.mask_head_backward(Et, Xt, om, w, G, Gp)
    m = (om.sigmoid() > 0.5).float()          # sigmoid in the dtype, as MaskPooling thresholds a 16-bit tensor

    def composed(e, x, mask):
        om_ = torch.einsum("bqc,bchw->bqhw", e, x)
        pooled_ = torch.einsum("bchw,bqhw->bqc", x, mask / (mask.sum((-1, -2), keepdim=True) + 1e-8))
        torch.autograd.backward([om_, pooled_], [G.to(om_.dtype), Gp.to(pooled_.dtype)])

    E64, X64 = Et.double().requires_grad_(), Xt.double().requires_grad_()
    composed(E64, X64, m.double())
    Ea, Xa = Et.float().requires_grad_(), Xt.float().requires_grad_()
    with torch.autocast("cuda", dtype=dtype):
        composed(Ea, Xa, m)
    e_e, r_e = _rel(ge, E64.grad), _rel(Ea.grad, E64.grad)
    e_x, r_x = _rel(gx, X64.grad), _rel(Xa.grad, X64.grad)
    print(f"{dt}: grad mask_embed err fused {e_e:.2e} / composed {r_e:.2e}; grad mask_features err fused {e_x:.2e} / "
          f"composed {r_x:.2e}")
    assert e_e <= 1.1 * r_e and e_x <= 1.1 * r_x


def _decoder(seed=0, Q=100):
    torch.manual_seed(seed)
    return dec.ODISEMultiScaleMaskedTransformerDecoder(
        in_channels=256, num_classes=16, hidden_dim=256, num_queries=Q, nheads=8, dim_feedforward=2048, dec_layers=9,
        pre_norm=False, mask_dim=256, enforce_input_project=False,
        post_mask_embed=dec.PooledMaskEmbed(hidden_dim=256, mask_dim=256, projection_dim=128))


def _inputs(B, H, W, device, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = [torch.randn(B, 256, H // 2 ** (3 - i), W // 2 ** (3 - i), generator=g).to(device) for i in range(3)]
    mf = torch.randn(B, 256, H, W, generator=g).to(device)
    return x, mf


def _loss(out):
    t = out["pred_masks"].float().mean() + out["mask_embed"].float().pow(2).mean()
    for a in out["aux_outputs"]:
        t = t + a["pred_masks"].float().mean() + a["mask_embed"].float().pow(2).mean()
    return t


def test_decoder_against_oracle(cuda):
    """the fused float32 decoder against oracle.m2f.transformer_decoder in float64 with the fused run's per-head
    outputs_mask forced as every threshold's input: forward and the gradients of mask_features and the parameters.
    Attention-mask bits that differ from the float64 evaluation (logits within a few ulps of the threshold) are counted
    and reported."""
    B, H, W = 2, 48, 40
    m = _decoder().to(cuda)
    x, mf = _inputs(B, H, W, cuda)
    mf.requires_grad_()
    out = m(x, mf)
    _loss(out).backward()
    heads = [a["pred_masks"] for a in out["aux_outputs"]] + [out["pred_masks"]]
    sd = {k: v.detach().double().cpu().requires_grad_() for k, v in m.state_dict().items()}
    mf64 = mf.detach().double().cpu().requires_grad_()
    forced = [h.detach().double().cpu() for h in heads]
    ref, masks = m2f.transformer_decoder(sd, [t.double().cpu() for t in x], mf64, forced_masks=forced)
    assert _rel(out["pred_masks"].cpu(), ref["pred_masks"]) < 1e-4
    assert _rel(out["mask_embed"].cpu(), ref["mask_embed"]) < 1e-4
    for a, r in zip(out["aux_outputs"], ref["aux_outputs"]):
        assert _rel(a["pred_masks"].cpu(), r["pred_masks"]) < 1e-4
        assert _rel(a["mask_embed"].cpu(), r["mask_embed"]) < 1e-4
    _loss(ref).backward()
    assert _rel(mf.grad.cpu(), mf64.grad) < 1e-4
    params = dict(m.named_parameters())
    worst = max(_rel(params[k].grad.cpu(), sd[k].grad) for k in sd if sd[k].grad is not None and
                params[k].grad is not None and sd[k].grad.abs().max() > 0)
    sizes = [t.shape[-2:] for t in x]
    flips = sum(int((lib.mask_head_attn_mask(h.detach(), sizes[i % 3], 8).cpu() !=
                     _torch_attn_mask(f, sizes[i % 3], 8)).sum()) for i, (h, f) in enumerate(zip(heads[:-1], forced)))
    print(f"decoder vs float64 oracle: worst parameter-gradient rel err {worst:.2e}, attention-mask bits that differ "
          f"from the float64 threshold: {flips}")
    assert worst < 3e-3


def _run(m, x, mf, dtype=None):
    mf = mf.detach().clone().requires_grad_()
    m.zero_grad(set_to_none=True)
    if dtype is None:
        out = m(x, mf)
    else:
        with torch.autocast("cuda", dtype=dtype):
            out = m(x, mf)
    _loss(out).backward()
    return out, [mf.grad] + [p.grad for p in m.parameters() if p.grad is not None]


class _OtherPooledEmbed(torch.nn.Module):
    """a post_mask_embed that is not this module's PooledMaskEmbed (the same computation, another class)"""

    def __init__(self):
        super().__init__()
        self.inner = dec.PooledMaskEmbed(hidden_dim=256, mask_dim=256, projection_dim=128)

    def forward(self, *args):
        return self.inner(*args)


def _heads_only(m, mf, dtype):
    """forward_prediction_heads of m on a seeded [Q, B, 256] decoder state, its outputs and gradients"""
    g = torch.Generator().manual_seed(9)
    out = (torch.randn(m.num_queries, mf.shape[0], 256, generator=g)).to(mf.device, dtype).requires_grad_()
    mf = mf.detach().clone().requires_grad_()
    m.zero_grad(set_to_none=True)
    cls, om, am, extra = m.forward_prediction_heads(out, mf, (6, 5))
    (om.float().mean() + extra["mask_embed"].float().pow(2).mean()).backward()
    return [om, am, extra["mask_embed"]], [out.grad, mf.grad] + [p.grad for p in m.parameters() if p.grad is not None]


def test_dispatch(cuda, monkeypatch):
    """fused cases reach the kernels; each composed case (float64, another post_mask_embed, soft pooling, a 16-bit module
    without autocast) never does and gives the bits of the composed ops (use_fused = False) in every output and
    gradient.  A 16-bit module without autocast cannot run the whole decoder (the position encoding is float32, in the
    reference too), so that case runs forward_prediction_heads."""
    B, H, W = 1, 32, 24
    x, mf = _inputs(B, H, W, cuda)
    calls = []
    real = lib.mask_head_forward
    monkeypatch.setattr(lib, "mask_head_forward", lambda *a, **k: calls.append(1) or real(*a, **k))
    m = _decoder(Q=20).to(cuda)
    _run(m, x, mf)
    assert len(calls) == 10
    _run(m, x, mf, torch.bfloat16)
    assert len(calls) == 20

    def same(a, b):
        return len(a) == len(b) and all(torch.equal(u, v) for u, v in zip(a, b))

    f64 = _decoder(Q=20).to(cuda).double()
    other = _decoder(Q=20).to(cuda)
    other.post_mask_embed = _OtherPooledEmbed().to(cuda)
    soft = _decoder(Q=20).to(cuda)
    soft.post_mask_embed.mask_pooling.hard_pooling = False
    for mod, xi, mfi in ((f64, [t.double() for t in x], mf.double()), (other, x, mf), (soft, x, mf)):
        calls.clear()
        o1, g1 = _run(mod, xi, mfi)
        assert not calls
        mod.use_fused = False
        o2, g2 = _run(mod, xi, mfi)
        assert torch.equal(o1["pred_masks"], o2["pred_masks"]) and torch.equal(o1["mask_embed"], o2["mask_embed"])
        assert same(g1, g2)
    m16 = _decoder(Q=20).to(cuda).half()
    calls.clear()
    o1, g1 = _heads_only(m16, mf.half(), torch.float16)
    assert not calls
    m16.use_fused = False
    o2, g2 = _heads_only(m16, mf.half(), torch.float16)
    assert same(o1, o2) and same(g1, g2)


def test_overridden_forward_prediction_heads(cuda):
    """forward() calls forward_prediction_heads, as the reference's does, so a subclass's override is used"""
    seen = []

    class Sub(dec.ODISEMultiScaleMaskedTransformerDecoder):
        def forward_prediction_heads(self, *a, **k):
            seen.append(1)
            return super().forward_prediction_heads(*a, **k)

    torch.manual_seed(0)
    m = Sub(in_channels=256, num_classes=16, hidden_dim=256, num_queries=20, nheads=8, dim_feedforward=64,
            dec_layers=3, pre_norm=False, mask_dim=256, enforce_input_project=False,
            post_mask_embed=dec.PooledMaskEmbed(hidden_dim=256, mask_dim=256, projection_dim=128)).to(cuda)
    x, mf = _inputs(1, 32, 24, cuda)
    m(x, mf)
    assert len(seen) == 4


def test_decoder_and_criterion_sync_once(cuda):
    """the fused decoder + the fused SetCriterion (odise_b200.criterion), forward and backward, synchronise exactly once:
    the criterion's copy of the matching costs to the host"""
    import warnings
    from odise_b200.criterion import HungarianMatcher, SetCriterion
    B, H, W = 2, 48, 40
    m = _decoder().to(cuda)
    x, mf = _inputs(B, H, W, cuda)
    g = torch.Generator().manual_seed(2)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, 4 * H), torch.linspace(0, 1, 4 * W), indexing="ij")
    targets = []
    for T in (3, 5):
        c = torch.rand(T, 2, generator=g)
        masks = ((yy - c[:, 0, None, None]) ** 2 + (xx - c[:, 1, None, None]) ** 2) < 0.1
        targets.append({"labels": torch.randint(0, 16, (T,), generator=g).to(cuda), "masks": masks.to(cuda)})
    crit = SetCriterion(16, HungarianMatcher(2.0, 5.0, 5.0, num_points=1024), 2.0, 5.0, 5.0, 9, 0.1,
                        ["labels", "masks"], 1024, 3.0, 0.75).to(cuda)

    def step():
        m.zero_grad(set_to_none=True)
        losses = crit(m(x, mf), targets)
        sum(losses.values()).backward()

    step()
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [str(x.message) for x in w if "called a synchronizing CUDA operation" in str(x.message)]
    print(f"decoder + criterion syncs: {len(syncs)}")
    assert len(syncs) == 1, syncs


@pytest.mark.parametrize("dt", [None, torch.float16, torch.bfloat16])
def test_no_sync_and_determinism(cuda, dt):
    """the fused decoder's forward + backward makes no host synchronisation, and two runs give the same bits in every
    gradient, in default mode and under torch.use_deterministic_algorithms(True)"""
    B, H, W = 2, 48, 40
    m = _decoder().to(cuda)
    x, mf = _inputs(B, H, W, cuda)
    _run(m, x, mf, dt)                                     # warm-up (module loading, algorithm choice)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        o1, g1 = _run(m, x, mf, dt)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    o2, g2 = _run(m, x, mf, dt)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    torch.use_deterministic_algorithms(True)
    try:
        o3, g3 = _run(m, x, mf, dt)
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(a, b) for a, b in zip(g1, g3))


def test_cuda_graph_replay(cuda):
    """the head's kernels (forward, attention mask, backward) captured in a CUDA graph replay bit-equal to eager"""
    g = torch.Generator().manual_seed(3)
    E = torch.randn(2, 100, 256, generator=g).to(cuda)
    X = torch.randn(2, 256, 40, 36, generator=g).to(cuda)
    G = torch.randn(2, 100, 40, 36, generator=g).to(cuda)
    Gp = torch.randn(2, 100, 256, generator=g).to(cuda)

    def step():
        om, pooled, w = torch.ops.odise_b200.mask_head_forward(E, X, 0.5)
        am = torch.ops.odise_b200.mask_head_attn_mask(om, 10, 9, 8)
        ge, gx = torch.ops.odise_b200.mask_head_backward(E, X, om, w, G, Gp, 0.5)
        return om, pooled, am, ge, gx

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(eager, captured))


def test_compile_fullgraph(cuda):
    """torch.compile(fullgraph=True) traces the head's forward + backward with the custom ops in the graph"""
    g = torch.Generator().manual_seed(4)
    E = torch.randn(2, 20, 256, generator=g).to(cuda).requires_grad_()
    X = torch.randn(2, 256, 24, 20, generator=g).to(cuda).requires_grad_()

    def f(E, X):
        om, pooled, _ = dec.MaskHeadFunction.apply(E, X, X.detach(), 0.5)
        am = torch.ops.odise_b200.mask_head_attn_mask(om.detach(), 6, 5, 8)
        return om.mean() + pooled.pow(2).sum() + am.float().mean()

    torch._dynamo.reset()
    cf = torch.compile(f, fullgraph=True)
    loss = cf(E, X)
    loss.backward()
    ge, gx = E.grad.clone(), X.grad.clone()
    E.grad = X.grad = None
    f(E, X).backward()
    assert torch.equal(ge, E.grad) and torch.equal(gx, X.grad)
