"""Grounding loss on the H100: odise_b200.grounding's fused kernels against float64 and against the composed path, for
all 10 prediction sets at once, Q = 100, C in {256, 768}, K in {1, 8}, on one rank and at emulated ranks (the gathered
tensors passed straight to the functions)."""
import warnings

import pytest
import torch

import grounding_ref
from category_ref import coco_labels
from odise_b200 import category, grounding

pytestmark = pytest.mark.gpu

S, Q = 10, 100


def _leaves(G, C, K, dtype=torch.float32, wdtype=None, seed=0, valid=None):
    """the gathered masks [S, G, Q, C], words [G, K, C] and scales [S] as leaves, and valid bool [G, K]"""
    ranks, sc = grounding_ref.inputs([G], S, Q, K, C, dtype=torch.float64, device="cuda", seed=seed, valid=valid)
    (m, w, v), = ranks
    return (m.to(dtype).requires_grad_(), w.to(wdtype or dtype).requires_grad_(), v,
            sc.to(torch.float64 if dtype == torch.float64 else torch.float32).requires_grad_())


def _run(leaves, B, o, use_fused, autocast=None, concat=False):
    """losses [S] and the gradients of a weighted sum against masks, words and scales; concat: the gathered tensors
    carry no gradient, so only the local rows' uses count"""
    m, w, v, sc = leaves
    G = m.shape[1]
    with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
        if G == B:
            losses = grounding.grounding_losses(m, m, w, w, v, sc, 0, 0.7, use_fused=use_fused)
        elif concat:
            losses = grounding.grounding_losses(m[:, o:o + B], m.detach(), w[o:o + B], w.detach(), v, sc, o, 0.7,
                                                local_in_global=False, use_fused=use_fused)
        else:
            losses = grounding.grounding_losses(m[:, o:o + B], m, w[o:o + B], w, v, sc, o, 0.7, use_fused=use_fused)
    wts = torch.randn(S, generator=torch.Generator().manual_seed(5)).cuda()
    grads = torch.autograd.grad((losses.float() * wts).sum(), [m, w, sc])
    return [losses.detach()] + [g.detach() for g in grads]


def _err(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def _case(G, B, o, C, K, valid=None, dtype=torch.float32, autocast=None, wdtype=None, concat=False):
    ref = _run(_leaves(G, C, K, torch.float64, valid=valid), B, o, False, concat=concat)
    fused = _run(_leaves(G, C, K, dtype, wdtype, valid=valid), B, o, True, autocast, concat)
    comp = _run(_leaves(G, C, K, dtype, wdtype, valid=valid), B, o, False, autocast, concat)
    return [_err(f, r) for f, r in zip(fused, ref)], [_err(c, r) for c, r in zip(comp, ref)]


CASES = [(B, B, 0) for B in (1, 2, 4, 8)] + [(64, 8, o) for o in (0, 24, 56)] + [(13, 3, 5)]
NAMES = ("losses", "masks", "words", "scales")


@pytest.mark.parametrize("K", [1, 8])
@pytest.mark.parametrize("C", [256, 768])
@pytest.mark.parametrize("G,B,o", CASES)
def test_float32_against_float64(cuda, G, B, o, C, K, record):
    fe, ce = _case(G, B, o, C, K)
    record(f"grounding fp32 G={G} B={B} o={o} C={C} K={K}: fused / composed rel err vs float64 "
           + ", ".join(f"{n} {a:.1e} / {b:.1e}" for n, a, b in zip(NAMES, fe, ce)))
    for n, a, b in zip(NAMES, fe, ce):
        assert a <= max(1e-5, 2 * b), (n, a, b)


@pytest.mark.parametrize("C", [256, 768])
@pytest.mark.parametrize("G,B,o", [(64, 8, 24), (13, 3, 5)])
def test_concat_against_float64(cuda, G, B, o, C, record):
    """"concat": the gathered rows carry no gradient; the local masks' gradient is the one through D and the local
    words' the one through A, and every other row's gradient is zero"""
    fe, ce = _case(G, B, o, C, 8, concat=True)
    record(f"grounding fp32 concat G={G} B={B} o={o} C={C}: fused / composed rel err vs float64 "
           + ", ".join(f"{n} {a:.1e} / {b:.1e}" for n, a, b in zip(NAMES, fe, ce)))
    for n, a, b in zip(NAMES, fe, ce):
        assert a <= max(1e-5, 2 * b), (n, a, b)
    _, gm, gw, _ = _run(_leaves(G, C, 8), B, o, True, concat=True)
    assert not gm[:, :o].any() and not gm[:, o + B:].any() and not gw[:o].any() and not gw[o + B:].any()


@pytest.mark.parametrize("G,B,o", [(4, 4, 0), (64, 8, 24)])
def test_fallback(cuda, G, B, o, record):
    """the local images have no valid word: l2's weighted mean is 0/0 and the kernels take the unweighted one"""
    valid = torch.rand(G, 8, generator=torch.Generator().manual_seed(2)) < 0.5
    valid[o:o + B] = False
    fe, ce = _case(G, B, o, 256, 8, valid=valid)
    record(f"grounding fp32 fallback G={G} B={B}: fused / composed rel err "
           + ", ".join(f"{n} {a:.1e} / {b:.1e}" for n, a, b in zip(NAMES, fe, ce)))
    for n, a, b in zip(NAMES, fe, ce):
        assert a <= max(1e-5, 2 * b), (n, a, b)


@pytest.mark.parametrize("wdtype", [None, torch.float32])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("G,B,o", [(4, 4, 0), (64, 8, 24)])
def test_autocast_against_float64(cuda, G, B, o, dtype, wdtype, record):
    fe, ce = _case(G, B, o, 256, 8, dtype=dtype, autocast=dtype, wdtype=wdtype)
    record(f"grounding autocast {str(dtype)[6:]} words {str(wdtype or dtype)[6:]} G={G} B={B}: fused / composed rel "
           "err vs float64 " + ", ".join(f"{n} {a:.1e} / {b:.1e}" for n, a, b in zip(NAMES, fe, ce)))
    for n, a, b in zip(NAMES, fe, ce):
        assert a <= 1.5 * b, (n, a, b)


@pytest.mark.parametrize("deterministic", [False, True])
def test_bit_reproducible(cuda, deterministic):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        for G, B, o in [(8, 8, 0), (64, 8, 24)]:
            a = _run(_leaves(G, 256, 8), B, o, True)
            b = _run(_leaves(G, 256, 8), B, o, True)
            for x, y in zip(a, b):
                assert torch.equal(x, y)
    finally:
        torch.use_deterministic_algorithms(prev)


ONES = None


def _module_step(crit, outputs, targets, forward=None):
    """the module's 10 losses and the gradients of their sum against every set's masks and the words"""
    global ONES
    losses = (forward or (lambda o, t: torch.stack(list(crit(o, t).values()))))(outputs, targets)
    leaves = [outputs["mask_embed"]] + [a["mask_embed"] for a in outputs["aux_outputs"]] + [outputs["word_embed"]]
    if ONES is None:
        ONES = torch.ones(S, device="cuda")
    return [losses.detach()], torch.autograd.grad(losses, leaves, grad_outputs=ONES)


def _module_inputs(B=4, C=256, K=8):
    m, w, v, sc = _leaves(B, C, K)
    m, w = m.detach(), w.detach()
    sets = [{"mask_embed": m[s].clone().requires_grad_(), "word_embed": None, "logit_scale": sc[s].detach().clone()}
            for s in range(S)]
    w = w.clone().requires_grad_()
    for x in sets:
        x["word_embed"] = w
    outputs = dict(sets[0], aux_outputs=sets[1:])
    return outputs, [{"word_valid_mask": v[b]} for b in range(B)]


def test_module_makes_no_host_sync(cuda):
    crit = grounding.MaskGroundingCriterion(collect_mode="diff")
    outputs, targets = _module_inputs()
    _module_step(crit, outputs, targets)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _module_step(crit, outputs, targets)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_kernels_per_step(cuda, record):
    crit = grounding.MaskGroundingCriterion(collect_mode="diff")
    outputs, targets = _module_inputs()
    _module_step(crit, outputs, targets)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _module_step(crit, outputs, targets)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and not e.name.startswith(("Memcpy", "Memset"))]
    record(f"grounding module W=1 B=4, 10 sets fwd+bwd: {len(names)} kernels: {sorted(set(names))}")
    assert len(names) <= 16, names


def test_cuda_graph_and_compile_match_eager(cuda):
    crit = grounding.MaskGroundingCriterion(collect_mode="diff")
    outputs, targets = _module_inputs()
    eager = _module_step(crit, outputs, targets)
    compiled = torch.compile(lambda o, t: torch.stack(list(crit(o, t).values())), fullgraph=True,
                             backend="aot_eager")
    got = _module_step(crit, outputs, targets, compiled)
    for a, b in zip(eager[0] + list(eager[1]), got[0] + list(got[1])):
        assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _module_step(crit, outputs, targets)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = _module_step(crit, outputs, targets)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager[0] + list(eager[1]), captured[0] + list(captured[1])):
        assert torch.equal(a, b)


def test_stack_syncs_once(cuda, record):
    """fused decoder + scoring of all 10 sets + the grounding loss + fused SetCriterion, forward and backward,
    synchronise exactly once: the criterion's copy of the matching costs"""
    from odise_b200 import decoder as dec
    from odise_b200.criterion import HungarianMatcher, SetCriterion
    labels = coco_labels()
    K = len(labels)
    torch.manual_seed(0)
    d = dec.ODISEMultiScaleMaskedTransformerDecoder(
        in_channels=256, num_classes=16, hidden_dim=256, num_queries=100, nheads=8, dim_feedforward=2048,
        dec_layers=9, pre_norm=False, mask_dim=256, enforce_input_project=False,
        post_mask_embed=dec.PooledMaskEmbed(hidden_dim=256, mask_dim=256, projection_dim=256)).to(cuda).train()
    crit = SetCriterion(K, HungarianMatcher(2.0, 5.0, 5.0, num_points=1024), 2.0, 5.0, 5.0, 9, 0.1,
                        ["labels", "masks"], 1024, 3.0, 0.75).to(cuda)
    grounding_crit = grounding.MaskGroundingCriterion(collect_mode="diff")
    B, H, W = 2, 128, 96
    g = torch.Generator().manual_seed(1)
    ms = [torch.randn(B, 256, H // s, W // s, generator=g).to(cuda) for s in (8, 4, 2)]
    mf = torch.randn(B, 256, H, W, generator=g).to(cuda)
    te = torch.randn(sum(len(l) for l in labels), 256, generator=g).to(cuda).requires_grad_()
    ne = torch.randn(1, 256, generator=g).to(cuda).requires_grad_()
    we = torch.randn(B, 8, 256, generator=g).to(cuda).requires_grad_()
    targets = [{"labels": torch.randint(0, K, (n,), generator=g).to(cuda),
                "masks": (torch.rand(n, 4 * H, 4 * W, generator=g) > 0.5).to(cuda),
                "word_valid_mask": (torch.rand(8, generator=g) > 0.3).to(cuda)} for n in (3, 5)]

    def step():
        torch.manual_seed(2)
        out = d(ms, mf)
        head = {"text_embed": te, "null_embed": ne, "labels": labels, "word_embed": we}
        for s in [out] + out["aux_outputs"]:
            s.update(head)
            s["pred_logits"] = category.cal_pred_logits(s)
        losses = crit(out, targets)
        losses.update(grounding_crit(out, targets))
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
    record(f"decoder + 10-set category scoring + grounding loss + criterion syncs: {len(syncs)}")
    assert len(syncs) == 1, syncs
