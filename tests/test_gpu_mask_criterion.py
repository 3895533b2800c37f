"""GPU checks of the SetCriterion / HungarianMatcher drop-in (odise_b200/criterion.py, odise_mask_* kernels): sampling
bit-equal to F.grid_sample, matching costs against float64, point selection against torch.topk, mask losses and their
gradient against float64 at the kernel's points, the whole 10-set criterion fused vs composed (float32 and autocast),
determinism, the synchronisation count and the memory bound.  Inputs are smooth logit fields (upsampled low-resolution
noise) and blob targets at 4x the prediction resolution."""
import warnings

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

K = 133


def _logits(g, B, Q, H, W, scale=6.0):
    low = torch.randn(B, Q, max(H // 16, 2), max(W // 16, 2), generator=g) * scale
    return F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)


def _blobs(g, T, H, W):
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    c = torch.rand(T, 2, generator=g)
    r = 0.08 + 0.3 * torch.rand(T, 1, 1, generator=g)
    return ((yy - c[:, 0, None, None]) ** 2 + (xx - c[:, 1, None, None]) ** 2) < r ** 2


def _problem(cuda, counts, Q=100, pred_hw=(256, 256), tgt_hw=(1024, 1024), sets=10, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(seed)
    B = len(counts)

    def one():
        return {"pred_logits": (torch.randn(B, Q, K + 1, generator=g) * 2).to(cuda),
                "pred_masks": _logits(g, B, Q, *pred_hw).to(cuda, dtype).requires_grad_(True)}
    outputs = one()
    outputs["aux_outputs"] = [one() for _ in range(sets - 1)]
    targets = [{"labels": torch.randint(0, K, (T,), generator=g).to(cuda), "masks": _blobs(g, T, *tgt_hw).to(cuda)}
               for T in counts]
    return outputs, targets


def _criterion(cuda, P=12544):
    from odise_b200.criterion import HungarianMatcher, SetCriterion
    m = HungarianMatcher(cost_class=2.0, cost_mask=5.0, cost_dice=5.0, num_points=P)
    return SetCriterion(K, m, 2.0, 5.0, 5.0, 9, 0.1, ["labels", "masks"], P, 3.0, 0.75).to(cuda)


def _sets(outputs):
    return [{k: v for k, v in outputs.items() if k != "aux_outputs"}] + outputs.get("aux_outputs", [])


def _run(crit, outputs, targets, fused, seed=0):
    crit.use_fused = fused
    torch.manual_seed(seed)
    losses = crit(outputs, targets)
    total = sum(crit.weight_dict[k] * v for k, v in losses.items())
    grads = torch.autograd.grad(total, [s["pred_masks"] for s in _sets(outputs)])
    return {k: v.detach() for k, v in losses.items()}, grads


def _ulp(x, dtype):
    m = {torch.float16: 10, torch.bfloat16: 7}[dtype]
    tiny = {torch.float16: 2.0 ** -14, torch.bfloat16: 2.0 ** -126}[dtype]
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp(min=tiny))) - m)


# 1 ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.bool])
@pytest.mark.parametrize("hw", [(64, 64), (48, 80), (7, 5)])
def test_sampling_bit_equal_to_grid_sample(cuda, dtype, hw):
    from odise_b200 import lib
    g = torch.Generator().manual_seed(1)
    N, P = 3, 4096
    maps = (torch.rand(N, *hw, generator=g) < 0.5) if dtype == torch.bool else (torch.randn(N, *hw, generator=g) * 4)
    maps = maps.to(cuda, dtype)
    pts = torch.rand(N, P, 2, generator=g)
    edge = torch.tensor([0.0, 1.0 - 2 ** -24, 0.5, 0.25, 1.0 / hw[0], 1.0 / hw[1], 0.5 / hw[1]])
    pts[:, :49] = torch.cartesian_prod(edge, edge)
    pts = pts.to(cuda)
    got = lib.mask_point_sample(maps, pts)
    want = F.grid_sample(maps[:, None].float(), 2.0 * pts[:, :, None] - 1.0, align_corners=False)[:, 0, :, 0]
    assert torch.equal(got, want)


# 2 ---------------------------------------------------------------------------------------------------------------------

def _cost64(outputs, targets, points, m):
    """float64 matching costs at the given points: [B] of [Q, T_b]"""
    out = []
    for b, t in enumerate(targets):
        x = F.grid_sample(outputs["pred_masks"][b, :, None].double(), 2.0 * points[b][0][None, :, None].double()
                          .expand(outputs["pred_masks"].shape[1], -1, -1, -1) - 1.0, align_corners=False)[:, 0, :, 0]
        T = len(t["labels"])
        y = F.grid_sample(t["masks"][:, None].double(), 2.0 * points[b][0][None, :, None].double()
                          .expand(T, -1, -1, -1) - 1.0, align_corners=False)[:, 0, :, 0]
        ce = (F.softplus(x) @ torch.ones_like(y).T - x @ y.T) / x.shape[1]
        s = x.sigmoid()
        dice = 1 - (2 * s @ y.T + 1) / (s.sum(1)[:, None] + y.sum(1)[None, :] + 1)
        prob = outputs["pred_logits"][b].double().softmax(-1)[:, t["labels"]]
        out.append(m.cost_mask * ce - m.cost_class * prob + m.cost_dice * dice)
    return out


@pytest.mark.parametrize("counts", [(0, 120, 7), (30,), (5, 17, 60, 1)])
def test_matcher_costs_and_indices(cuda, counts):
    from odise_b200.criterion import HungarianMatcher, _Targets
    outputs, targets = _problem(cuda, counts, sets=1, pred_hw=(64, 96), tgt_hw=(256, 384))
    m = HungarianMatcher(2.0, 5.0, 5.0, num_points=4096)
    tg = _Targets(targets)
    B, Q = len(counts), 100
    torch.manual_seed(3)
    pts = m._draw(B, cuda)
    C = torch.zeros(B, Q, tg.Tmax, device=cuda)
    m._costs(outputs, tg, pts, C)
    for b, want in enumerate(_cost64(outputs, targets, pts, m)):
        got = C[b, :, :counts[b]].double()
        assert ((got - want).abs() <= 1e-5 * want.abs().clamp(min=1)).all(), (got - want).abs().max()
    torch.manual_seed(5)
    fused = m(outputs, targets)
    m.use_fused = False
    torch.manual_seed(5)
    composed = m(outputs, targets)
    for (a, b_), (c, d) in zip(fused, composed):
        assert a.device.type == "cpu" and a.dtype == torch.int64
        assert torch.equal(a, c) and torch.equal(b_, d)


# 3 ---------------------------------------------------------------------------------------------------------------------

def _loss_problem(cuda, dtype, P=12544, N=24, seed=2):
    g = torch.Generator().manual_seed(seed)
    B, Q = 3, 20
    pred = _logits(g, B, Q, 256, 192).to(cuda, dtype)
    tgt = _blobs(g, N, 1024, 768).to(cuda)
    perm = torch.randperm(B * Q, generator=g)[:N]
    pairs = torch.stack([perm // Q, perm % Q, torch.arange(N)], 1).to(cuda)
    pair_of = torch.full((B * Q,), -1, dtype=torch.int64)
    pair_of[perm] = torch.arange(N)
    S, k = int(P * 3.0), int(0.75 * P)
    cand = torch.rand(N, S, 2, generator=g).to(cuda)
    rnd = torch.rand(N, P - k, 2, generator=g).to(cuda)
    return pred, tgt, pairs, pair_of.to(cuda), cand, rnd, P, k


def _loss64(pred, tgt, pairs, coords, num_masks):
    """float64 losses of the pairs at coords [N, P, 2] and the gradient of (loss_mask, loss_dice) . (go_m, go_d)"""
    p = pred.detach().double().requires_grad_(True)
    src = p[pairs[:, 0], pairs[:, 1]][:, None]
    x = F.grid_sample(src, 2.0 * coords[:, :, None].double() - 1.0, align_corners=False)[:, 0, :, 0]
    t = F.grid_sample(tgt[pairs[:, 2]][:, None].double(), 2.0 * coords[:, :, None].double() - 1.0,
                      align_corners=False)[:, 0, :, 0]
    lm = F.binary_cross_entropy_with_logits(x, t, reduction="none").mean(1).sum() / num_masks
    s = x.sigmoid()
    ld = (1 - (2 * (s * t).sum(1) + 1) / (s.sum(1) + t.sum(1) + 1)).sum() / num_masks
    return lm, ld, p


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_mask_losses_selection_and_gradient(cuda, dtype):
    from odise_b200 import lib
    from odise_b200.criterion import MaskLossFunction
    pred, tgt, pairs, pair_of, cand, rnd, P, k = _loss_problem(cuda, dtype)
    N, num_masks = pairs.shape[0], 30.0
    losses, state = lib.mask_loss_forward(pred, tgt, pairs, cand, rnd, num_masks, P, k)
    coords = state[N * 16:N * 16 + N * P * 8].view(torch.float32).view(N, P, 2)
    assert torch.equal(coords[:, k:], rnd)
    # the selected set is torch.topk's on grid_sample values, up to exact ties: the same multiset of |logit|, and every
    # selected point is a candidate (in candidate order)
    src = pred.float()[pairs[:, 0], pairs[:, 1]][:, None]
    x = F.grid_sample(src, 2.0 * cand[:, :, None] - 1.0, align_corners=False)[:, 0, :, 0]
    xs = F.grid_sample(src, 2.0 * coords[:, :k, None] - 1.0, align_corners=False)[:, 0, :, 0]
    top = torch.topk(-x.abs(), k, dim=1)[0]
    assert torch.equal(xs.abs().sort(1).values, (-top).sort(1).values)
    key = cand[..., 0] * 4 + cand[..., 1]
    pos = torch.searchsorted(key.sort(1).values, coords[:, :k, 0] * 4 + coords[:, :k, 1])
    assert torch.equal(key.sort(1).values.gather(1, pos), coords[:, :k, 0] * 4 + coords[:, :k, 1])
    lm, ld, p = _loss64(pred, tgt, pairs, coords, num_masks)
    torch.testing.assert_close(losses[0].double(), lm.detach(), rtol=1e-5, atol=0)
    torch.testing.assert_close(losses[1].double(), ld.detach(), rtol=1e-5, atol=0)
    go = torch.tensor([0.7, -1.3], device=cuda)
    grad = lib.mask_loss_backward(pred, tgt, pairs, pair_of, state, go, num_masks, P)
    assert grad.dtype == dtype and grad.shape == pred.shape
    want = torch.autograd.grad(go[0].double() * lm + go[1].double() * ld, p)[0]
    if dtype == torch.float32:
        assert (grad.double() - want).abs().max() <= 1e-5 * want.abs().max()
    else:
        # one unit of the rounded float64 gradient, plus the fp32 bar where opposite-signed contributions cancel
        r = want.to(dtype).double()
        assert ((grad.double() - r).abs() <= _ulp(r, dtype) + 1e-5 * want.abs().max()).all()
    unmatched = (pair_of < 0).view(pred.shape[:2])
    assert (grad[unmatched] == 0).all()
    # through autograd: the [2] loss tensor's gradient
    pr = pred.detach().requires_grad_(True)
    out = MaskLossFunction.apply(pr, tgt, pairs, pair_of, cand, rnd, num_masks, P, k)
    assert torch.equal(out, losses)
    (out[0] * 0.7 - out[1] * 1.3).backward()
    assert torch.equal(pr.grad, grad)


# 4 ---------------------------------------------------------------------------------------------------------------------

def _record_assign(monkeypatch):
    from odise_b200 import criterion
    seen = []
    real = criterion._assign

    def rec(C, counts):
        r = real(C, counts)
        seen.append(r)
        return r
    monkeypatch.setattr(criterion, "_assign", rec)
    return seen


def test_criterion_fused_vs_composed(cuda, monkeypatch, record):
    seen = _record_assign(monkeypatch)
    outputs, targets = _problem(cuda, (6, 15), Q=100)
    crit = _criterion(cuda)
    lf, gf = _run(crit, outputs, targets, True)
    lc, gc = _run(crit, outputs, targets, False)
    assert len(seen) == 2
    for a_set, b_set in zip(*seen):
        for (a, b), (c, d) in zip(a_set, b_set):
            assert torch.equal(a, c) and torch.equal(b, d)
    assert list(lf) == list(lc) and len(lf) == 30
    for k_ in lf:
        assert lf[k_].dtype == torch.float32 and lf[k_].dim() == 0
        torch.testing.assert_close(lf[k_], lc[k_], rtol=1e-5, atol=0, msg=k_)
    worst = 0.0
    for a, b in zip(gf, gc):
        e = ((a - b).abs().max() / b.abs().max()).item()
        worst = max(worst, e)
        assert e <= 1e-5
    record(f"mask criterion fused vs composed (10 sets, 1024^2 targets, fp32): worst grad err {worst:.2e} x max|ref|")


# 5 ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_criterion_autocast(cuda, dtype):
    outputs, targets = _problem(cuda, (6, 15), Q=100, sets=3, dtype=dtype)
    crit = _criterion(cuda)
    with torch.autocast("cuda", dtype=dtype):
        lf, gf = _run(crit, outputs, targets, True)
        lc, gc = _run(crit, outputs, targets, False)
    for k_ in lf:
        assert lf[k_].dtype == torch.float32
        torch.testing.assert_close(lf[k_], lc[k_], rtol=1e-5, atol=0, msg=k_)
    for a, s in zip(gf, _sets(outputs)):
        assert a.dtype == dtype and a.shape == s["pred_masks"].shape


# 6 ---------------------------------------------------------------------------------------------------------------------

def test_determinism(cuda):
    outputs, targets = _problem(cuda, (6, 15, 30), Q=100, sets=3)
    crit = _criterion(cuda)
    l1, g1 = _run(crit, outputs, targets, True)
    l2, g2 = _run(crit, outputs, targets, True)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        l3, g3 = _run(crit, outputs, targets, True)
        with pytest.raises(RuntimeError):
            _run(crit, outputs, targets, False)
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b, c in zip(g1, g2, g3):
        assert torch.equal(a, b) and torch.equal(a, c)
    for k_ in l1:
        assert torch.equal(l1[k_], l2[k_]) and torch.equal(l1[k_], l3[k_]), k_


# 7 ---------------------------------------------------------------------------------------------------------------------

def test_at_most_two_syncs_per_forward(cuda):
    outputs, targets = _problem(cuda, (6, 15, 30, 60), Q=100)
    crit = _criterion(cuda)
    crit.use_fused = True
    torch.manual_seed(0)
    crit(outputs, targets)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            crit(outputs, targets)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [x for x in w if "synchroniz" in str(x.message)]
    assert len(syncs) <= 2, [str(x.message) for x in syncs]


# 8 ---------------------------------------------------------------------------------------------------------------------

def test_memory_below_one_float_copy_of_targets(cuda):
    counts = (6, 15, 30, 60)
    outputs, targets = _problem(cuda, counts, Q=100)
    crit = _criterion(cuda)
    crit.use_fused = True
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(0)
    losses = crit(outputs, targets)
    total = sum(crit.weight_dict[k] * v for k, v in losses.items())
    grads = torch.autograd.grad(total, [s["pred_masks"] for s in _sets(outputs)])
    torch.cuda.synchronize()
    grad_bytes = sum(g.numel() * g.element_size() for g in grads)
    peak = torch.cuda.max_memory_allocated() - base - grad_bytes   # the gradients are outputs of pred_masks' size
    float_copy = sum(counts) * 1024 * 1024 * 4
    assert peak < float_copy, (peak, float_copy)
