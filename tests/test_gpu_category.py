"""Category scoring on the H100: odise_b200.category's fused kernels against float64 and against the composed path, with
the COCO training bank (133 classes, 254 prompts), Q = 100 and C in {256, 768}."""
import warnings

import pytest
import torch
import torch.nn.functional as F

from category_ref import coco_labels, inputs
from odise_b200 import category, lib

pytestmark = pytest.mark.gpu

LABELS = coco_labels()
SIZES = [len(l) for l in LABELS]
GS = lib.category_group_start(SIZES)
K, KP = len(SIZES), sum(SIZES)
NAMES = ("mask_embed", "text_embed", "null_embed", "logit_scale")


def _outputs(B, C, device, dtype=torch.float32, bank=None, seed=0, labels=LABELS):
    me, te, ne, ls = inputs(B, 100, C, [len(l) for l in labels], dtype=torch.float32, device=device, seed=seed)
    bank = bank or dtype
    o = dict(mask_embed=me.to(dtype), text_embed=te.to(bank), null_embed=ne.to(bank), logit_scale=ls, labels=labels)
    for k in NAMES:
        o[k].requires_grad_()
    return o


def _weights(shape, device, seed=3):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(device)


def _grads(out, o, w):
    return list(torch.autograd.grad((out.float() * w).sum(), [o[k] for k in NAMES]))


def _f64_forced(o, win, w):
    """float64 values and gradients of the scores at the kernel's winners (each output the scaled similarity of its
    saved winner)"""
    x = {k: o[k].detach().double().requires_grad_() for k in NAMES}
    m, t, n = (F.normalize(x[k], dim=-1) for k in ("mask_embed", "text_embed", "null_embed"))
    s = x["logit_scale"] * (m @ t.t())
    idx = torch.tensor(GS[:-1], device=win.device)[None, None] + win[..., :K].long()
    out = torch.cat([s.gather(-1, idx), x["logit_scale"] * (m @ n.t())], -1)
    grads = torch.autograd.grad((out * w.double()).sum(), [x[k] for k in NAMES])
    return out.detach(), grads, s.detach()


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def _relf(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.mark.parametrize("C", [256, 768])
@pytest.mark.parametrize("B", [1, 2, 4])
def test_float32_against_float64(cuda, B, C, record):
    o = _outputs(B, C, cuda, seed=B)
    n0 = lib.launch_count()
    out = category.cal_pred_logits(o)
    assert lib.launch_count() == n0 + 1 and out.dtype == torch.float32 and out.shape == (B, 100, K + 1)
    _, win, _ = torch.ops.odise_b200.category_logits(*[o[k].detach() for k in NAMES[:3]], o["logit_scale"].detach(),
                                                     category.group_start(SIZES, cuda))
    w = _weights(out.shape, cuda)
    got = _grads(out, o, w)
    ref, ref_grads, s64 = _f64_forced(o, win, w)
    errs = [_rel(out, ref)] + [_rel(g, r) for g, r in zip(got, ref_grads)]
    record(f"category fp32 B={B} C={C}: out / grad mask, text, null, scale rel err vs float64 (kernel winners) "
           + " ".join(f"{e:.1e}" for e in errs))
    assert max(errs) < 1e-5, errs
    # each saved winner is the group's max up to float32 rounding
    for k in range(K):
        top = s64[..., GS[k]:GS[k + 1]].max(-1).values
        assert (ref[..., k] >= top - 1e-5 * top.abs().max()).all()


def test_ties_lowest_index(cuda):
    """duplicated prompt rows score equal; the gradient goes to the lowest index, as in the composed path"""
    o = _outputs(4, 256, cuda, seed=11)
    with torch.no_grad():
        for k in range(K):
            if SIZES[k] > 1:
                o["text_embed"][GS[k] + 1] = o["text_embed"][GS[k]]
    w = _weights((4, 100, K + 1), cuda)
    gf = _grads(category.cal_pred_logits(o), o, w)
    gc = _grads(category.cal_pred_logits(o, use_fused=False), o, w)
    dup = torch.tensor([GS[k] + 1 for k in range(K) if SIZES[k] > 1], device=cuda)
    first = dup - 1
    assert (gf[1][dup] == 0).all() and (gc[1][dup] == 0).all()
    assert (gf[1][first].abs().sum(-1) > 0).any()
    assert torch.equal(gf[1].abs().sum(-1) == 0, gc[1].abs().sum(-1) == 0)
    assert _rel(gf[1], gc[1]) < 1e-5


@pytest.mark.parametrize("dtype,bank", [(torch.float16, torch.float16), (torch.bfloat16, torch.bfloat16),
                                        (torch.float16, torch.float32)])
def test_autocast(cuda, dtype, bank, record):
    """output dtype as the composed path's; errors against float64 no worse than the composed path's under the same
    autocast; the null column in torch's rounding of logit_scale"""
    C = 768 if bank == torch.float32 else 256     # a float32 bank is text_proj = Identity's, at C = 768
    o = _outputs(4, C, cuda, dtype=dtype, bank=bank, seed=5)
    w = _weights((4, 100, K + 1), cuda)
    with torch.autocast("cuda", dtype=dtype):
        n0 = lib.launch_count()
        of = category.cal_pred_logits(o)
        assert lib.launch_count() == n0 + 1
        oc = category.cal_pred_logits(o, use_fused=False)
    assert of.dtype == oc.dtype == dtype
    gf, gc = _grads(of, o, w), _grads(oc, o, w)
    for g, k in zip(gf, NAMES):
        assert g.dtype == o[k].dtype
    x = {k: (o[k].detach().double().requires_grad_() if k in NAMES else o[k]) for k in o}
    o64 = category.cal_pred_logits(x)
    g64 = torch.autograd.grad((o64 * w.double()).sum(), [x[k] for k in NAMES])
    ef = [_rel(of, o64)] + [_relf(g, r) for g, r in zip(gf, g64)]
    ec = [_rel(oc, o64)] + [_relf(g, r) for g, r in zip(gc, g64)]
    record(f"category autocast {str(dtype)[6:]} bank {str(bank)[6:]} C={C}: fused / composed err vs float64, out "
           f"(max) {ef[0]:.2e} / {ec[0]:.2e}, grads (norm) mask {ef[1]:.2e} / {ec[1]:.2e}, text {ef[2]:.2e} / "
           f"{ec[2]:.2e}, null {ef[3]:.2e} / {ec[3]:.2e}, scale {ef[4]:.2e} / {ec[4]:.2e}")
    for a, b in zip(ef, ec):
        assert a <= b * 1.1 + 1e-7, (ef, ec)
    # torch rounds the float32 0-dim factor to the 16-bit dtype before the multiply, and so does the kernel
    with torch.autocast("cuda", dtype=dtype), torch.no_grad():
        m = F.normalize(o["mask_embed"], dim=-1)
        p = m @ F.normalize(o["null_embed"], dim=-1).t()
        ls = o["logit_scale"].detach()
        torch_null = ls * p
    assert torch.equal(torch_null, (p.float() * ls.to(dtype).float()).to(dtype))
    assert not torch.equal(torch_null, (p.float() * ls).to(dtype))
    same = (of[..., K].detach() == oc[..., K].detach()).float().mean().item()
    record(f"category autocast {str(dtype)[6:]}: null column bit-equal to the composed path's at {same:.1%} of rows, "
           f"max diff {_rel(of[..., K], oc[..., K]):.1e} of max")
    assert same > 0.9


def _fwd_bwd(o, w):
    return _grads(category.cal_pred_logits(o), o, w)


def test_deterministic(cuda):
    o = _outputs(4, 256, cuda, seed=2)
    w = _weights((4, 100, K + 1), cuda)
    a, b = _fwd_bwd(o, w), _fwd_bwd(o, w)
    torch.use_deterministic_algorithms(True)
    try:
        c = _fwd_bwd(o, w)
    finally:
        torch.use_deterministic_algorithms(False)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_no_sync(cuda):
    o = _outputs(4, 256, cuda, seed=2)
    w = _weights((4, 100, K + 1), cuda)
    _fwd_bwd(o, w)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for dtype in (None, torch.float16):
            with torch.autocast("cuda", dtype=dtype or torch.float16, enabled=dtype is not None):
                out = category.cal_pred_logits(o)
            _grads(out, o, w)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_cuda_graph_replay(cuda):
    o = _outputs(2, 256, cuda, seed=4)
    w = _weights((2, 100, K + 1), cuda)

    def step():
        out = category.cal_pred_logits(o)
        return [out.detach()] + _grads(out, o, w)

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(eager, captured))


def test_compile_fullgraph(cuda):
    o = _outputs(2, 256, cuda, seed=6)
    w = _weights((2, 100, K + 1), cuda)

    def f(me, te, ne, ls):
        return category.cal_pred_logits(dict(mask_embed=me, text_embed=te, null_embed=ne, logit_scale=ls,
                                             labels=LABELS))

    args = [o[k] for k in NAMES]
    eager = torch.autograd.grad((f(*args) * w).sum(), args)
    torch._dynamo.reset()
    cf = torch.compile(f, fullgraph=True, backend="aot_eager")
    comp = torch.autograd.grad((cf(*args) * w).sum(), args)
    assert all(torch.equal(a, b) for a, b in zip(eager, comp))


def test_kernels_per_ten_calls(cuda, record):
    """10 calls, forward and backward: four scoring launches each on the fused path, plus autograd's sums of the shared
    bank's and scale's gradients over the calls; thousands of launches on the composed path"""
    from torch.profiler import ProfilerActivity, profile
    o = _outputs(4, 256, cuda, seed=8)
    sets = [torch.randn(4, 100, 256, device=cuda, requires_grad=True) for _ in range(10)]
    w = _weights((4, 100, K + 1), cuda)
    shared = [o[k] for k in ("text_embed", "null_embed", "logit_scale")]
    counts = {}
    for fused in (True, False):
        def step():
            outs = [category.cal_pred_logits(dict(o, mask_embed=me), use_fused=fused) for me in sets]
            torch.autograd.grad(outs, sets + shared, [w] * 10)
        step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        kern = [n for n in names if "Memcpy" not in n and "Memset" not in n]
        counts[fused] = (len(kern), sum("cl_" in n for n in kern))
    record(f"category 10 calls fwd+bwd, B=4: kernels fused {counts[True][0]} ({counts[True][1]} scoring kernels), "
           f"composed {counts[False][0]}")
    assert counts[True][1] == 40 and counts[True][0] <= 40 + 3 * 9 + 3, counts
    assert counts[False][0] > 1000, counts


def test_stack_syncs_once(cuda, record):
    """fused decoder + scoring of all 10 sets + fused SetCriterion, forward and backward, synchronise exactly once:
    the criterion's copy of the matching costs"""
    from odise_b200 import decoder as dec
    from odise_b200.criterion import HungarianMatcher, SetCriterion
    torch.manual_seed(0)
    d = dec.ODISEMultiScaleMaskedTransformerDecoder(
        in_channels=256, num_classes=16, hidden_dim=256, num_queries=100, nheads=8, dim_feedforward=2048,
        dec_layers=9, pre_norm=False, mask_dim=256, enforce_input_project=False,
        post_mask_embed=dec.PooledMaskEmbed(hidden_dim=256, mask_dim=256, projection_dim=256)).to(cuda).train()
    crit = SetCriterion(K, HungarianMatcher(2.0, 5.0, 5.0, num_points=1024), 2.0, 5.0, 5.0, 9, 0.1,
                        ["labels", "masks"], 1024, 3.0, 0.75).to(cuda)
    B, H, W = 2, 128, 96
    g = torch.Generator().manual_seed(1)
    ms = [torch.randn(B, 256, H // s, W // s, generator=g).to(cuda) for s in (8, 4, 2)]
    mf = torch.randn(B, 256, H, W, generator=g).to(cuda)
    te = torch.randn(KP, 256, generator=g).to(cuda).requires_grad_()
    ne = torch.randn(1, 256, generator=g).to(cuda).requires_grad_()
    targets = [{"labels": torch.randint(0, K, (n,), generator=g).to(cuda),
                "masks": (torch.rand(n, 4 * H, 4 * W, generator=g) > 0.5).to(cuda)} for n in (3, 5)]

    def step():
        torch.manual_seed(2)
        out = d(ms, mf)
        head = {"text_embed": te, "null_embed": ne, "labels": LABELS}
        for s in [out] + out["aux_outputs"]:
            s.update(head)
            s["pred_logits"] = category.cal_pred_logits(s)
        losses = crit(out, targets)
        sum(losses.values()).backward()

    step()
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [str(x.message) for x in caught if "called a synchronizing CUDA operation" in str(x.message)]
    record(f"decoder + 10-set category scoring + criterion syncs: {len(syncs)}")
    assert len(syncs) == 1, syncs
