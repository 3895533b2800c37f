"""Grounding loss without a GPU: the composed path of odise_b200.grounding against the reference's
MaskGroundingCriterion.get_loss (values and float64 gradients, pinned in tests/golden/ref_pinned_grounding.pt) on one
rank and at emulated ranks, the gather over gloo at world 2 and 3 with its collective count, the fake implementations
of the custom ops, the shape checks and the dispatch."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch._subclasses.fake_tensor import FakeTensorMode

from odise_b200 import grounding, lib
from oracle import refshim
import grounding_ref

FIXTURE = "ref_pinned_grounding.pt"
S, Q, K, C = 3, 5, 4, 8


def _leaves(sizes, seed=0, valid=None, S=S):
    ranks, scales = grounding_ref.inputs(sizes, S, Q, K, C, seed=seed, valid=valid)
    ranks = [tuple(t.clone().requires_grad_(t.is_floating_point()) for t in r) for r in ranks]
    scales = [[scales[s].clone().requires_grad_() for s in range(S)] for _ in sizes]
    return ranks, scales


def _grads(losses, ranks, scales):
    """every rank's losses and the gradients of their weighted sum against every leaf"""
    g = torch.Generator().manual_seed(9)
    flat = [l for per_rank in losses for l in per_rank]
    w = [torch.randn((), generator=g, dtype=torch.float64) for _ in flat]
    leaves = [t for m, wd, _ in ranks for t in (m, wd)] + [s for per_rank in scales for s in per_rank]
    grads = torch.autograd.grad(flat, leaves, grad_outputs=w, allow_unused=True)
    return dict(losses=torch.stack([l.detach() for l in flat]),
                grads=[torch.zeros_like(t) if x is None else x for t, x in zip(leaves, grads)])


def _reference(sizes, mode, seed=0, valid=None):
    ranks, scales = _leaves(sizes, seed, valid)
    return _grads(grounding_ref.reference_losses(ranks, scales, mode, loss_weight=0.7), ranks, scales)


def _composed(sizes, mode, seed=0, valid=None):
    ranks, scales = _leaves(sizes, seed, valid)
    mg = torch.cat([m for m, _, _ in ranks], dim=1)
    wg = torch.cat([w for _, w, _ in ranks])
    vg = torch.cat([v for _, _, v in ranks])
    if mode == "concat":
        mg, wg = mg.detach(), wg.detach()
    losses, o = [], 0
    for r, (m, w, v) in enumerate(ranks):
        if len(sizes) == 1:
            mg, wg, vg = m, w, v
        ls = grounding.grounding_losses(m, mg, w, wg, vg, torch.stack(scales[r]), o, 0.7,
                                        local_in_global=mode != "concat", use_fused=False)
        losses.append(list(ls.unbind(0)))
        o += sizes[r]
    return _grads(losses, ranks, scales)


def _no_valid(sizes, rank):
    g = torch.Generator().manual_seed(3)
    v = torch.rand(sum(sizes), K, generator=g) < 0.5
    v[:, 0] = True
    o = sum(sizes[:rank])
    v[o:o + sizes[rank]] = False
    return v


CASES = {
    "w1_b1": ([1], None, None),
    "w1_b4": ([4], None, None),
    "w1_b4_diff": ([4], "diff", None),
    "w1_b4_novalid": ([4], None, _no_valid([4], 0)),
    "w3_diff": ([2, 3, 1], "diff", None),
    "w3_concat": ([2, 3, 1], "concat", None),
    "w3_diff_novalid": ([2, 3, 1], "diff", _no_valid([2, 3, 1], 1)),
    "w3_concat_novalid": ([2, 3, 1], "concat", _no_valid([2, 3, 1], 2)),
}


def _pinned(case):
    sizes, mode, valid = CASES[case]

    def ref():
        import mask_criterion_ref
        mask_criterion_ref.classes()
        return _reference(sizes, mode, valid=valid)
    return refshim.pinned(f"grounding/{case}", ref, fixture=FIXTURE)


@pytest.mark.parametrize("case", sorted(CASES))
def test_composed_path_matches_reference(case):
    """the composed path runs the reference's ops: equal losses and float64 gradients at every rank (bit-equal on one
    rank; at emulated ranks the sums over ranks' gradient contributions may associate differently)"""
    sizes, mode, valid = CASES[case]
    want = _pinned(case)
    got = _composed(sizes, mode, valid=valid)
    exact = len(sizes) == 1
    if exact:
        assert torch.equal(got["losses"], want["losses"])
    else:
        torch.testing.assert_close(got["losses"], want["losses"], rtol=0, atol=1e-13)
    assert torch.isfinite(want["losses"]).all()
    for a, b in zip(got["grads"], want["grads"]):
        if exact:
            assert torch.equal(a, b)
        else:
            torch.testing.assert_close(a, b, rtol=0, atol=1e-12 * max(1.0, b.abs().max().item()))


def test_fallback_case_takes_the_fallback():
    """a rank without a valid word: the weighted CE is 0/0 and the reference falls back to the unweighted mean"""
    want = _pinned("w3_diff_novalid")
    assert torch.isfinite(want["losses"]).all()


def test_module_interface():
    crit = grounding.MaskGroundingCriterion(collect_mode="diff", loss_weight=2.0)
    assert crit.extra_repr() == "collect_mode=diff, \nloss_weight=2.0 \n"
    assert grounding.MaskGroundingCriterion().collect_mode == "concat"
    with pytest.raises(ValueError):
        grounding.MaskGroundingCriterion(collect_mode="sum")
    (m, w, v), = grounding_ref.inputs([2], 4, Q, K, C)[0]
    outputs = {"mask_embed": m[0], "word_embed": w, "logit_scale": torch.tensor(12.0, dtype=torch.float64),
               "aux_outputs": [{"mask_embed": m[s], "word_embed": w, "logit_scale": torch.tensor(12.0, dtype=torch.float64)}
                               for s in range(1, 4)]}
    targets = [{"word_valid_mask": v[b]} for b in range(2)]
    out = crit(outputs, targets)
    assert list(out) == ["loss_mask_word", "loss_mask_word_0", "loss_mask_word_1", "loss_mask_word_2"]
    sc = torch.full((4,), 12.0, dtype=torch.float64)
    want = grounding.grounding_losses(m, m, w, w, v, sc, 0, 2.0, use_fused=False)
    assert torch.equal(torch.stack(list(out.values())), want)


def test_op_schemas():
    ops = torch.ops.odise_b200
    assert str(ops.grounding.default._schema) == (
        "odise_b200::grounding(Tensor mask_embed, Tensor word_embed, Tensor word_valid, Tensor logit_scale, "
        "int batch, int offset, float loss_weight) -> (Tensor, Tensor)")
    assert str(ops.grounding_backward.default._schema) == (
        "odise_b200::grounding_backward(Tensor mask_embed, Tensor word_embed, Tensor logit_scale, Tensor state, "
        "Tensor grad_losses, int batch, int offset) -> (Tensor, Tensor, Tensor, Tensor, Tensor)")


@pytest.mark.parametrize("dtype,wdtype", [(torch.float32, torch.float32), (torch.float16, torch.float16),
                                          (torch.bfloat16, torch.float32)])
def test_fakes(dtype, wdtype, monkeypatch):
    monkeypatch.setattr(lib, "load", lambda: pytest.fail("a fake loaded the library"))
    Sx, G, B, o = 10, 12, 4, 8
    with FakeTensorMode(allow_non_fake_inputs=False) as mode:
        dev = torch.device("cuda")
        m = torch.empty(Sx, G, 100, 256, dtype=dtype, device=dev)
        w = torch.empty(G, 8, 256, dtype=wdtype, device=dev)
        v = torch.empty(G, 8, dtype=torch.bool, device=dev)
        sc = torch.empty(Sx, dtype=torch.float32, device=dev)
        losses, state = torch.ops.odise_b200.grounding(m, w, v, sc, B, o, 1.0)
        assert losses.shape == (Sx,) and losses.dtype == torch.float32
        assert state.shape == (lib.grounding_state_size(Sx, G, B, 100, 8, 256),) and state.dtype == torch.float32
        g = torch.empty(Sx, dtype=torch.float32, device=dev)
        gml, gmg, gwl, gwg, gs = torch.ops.odise_b200.grounding_backward(m, w, sc, state, g, B, o)
        assert (gml.shape, gml.dtype) == ((Sx, B, 100, 256), dtype)
        assert (gmg.shape, gmg.dtype) == ((Sx, G, 100, 256), dtype)
        assert (gwl.shape, gwl.dtype) == ((B, 8, 256), wdtype)
        assert (gwg.shape, gwg.dtype) == ((G, 8, 256), wdtype)
        assert (gs.shape, gs.dtype) == ((Sx,), torch.float32)
        with pytest.raises(lib.OdiseError):
            torch.ops.odise_b200.grounding(m, w, v, sc, B, G - B + 1, 1.0)      # offset past the last image
    del mode


def test_limit_checks():
    def shapes(Q=100, K=8, C=256, G=4, B=4, o=0, dtype=torch.float32, wdtype=torch.float32):
        with FakeTensorMode():
            dev = torch.device("cuda")
            lib._grounding_shapes(torch.empty(2, G, Q, C, dtype=dtype, device=dev),
                                  torch.empty(G, K, C, dtype=wdtype, device=dev),
                                  torch.empty(2, dtype=torch.float32, device=dev), B, o)
    shapes()
    shapes(Q=256, K=32, C=768)
    shapes(dtype=torch.float16, wdtype=torch.float32)
    for bad in (dict(Q=257), dict(K=33), dict(K=0), dict(C=48), dict(C=800), dict(B=5), dict(B=0), dict(o=1),
                dict(dtype=torch.float64, wdtype=torch.float64), dict(wdtype=torch.float16)):
        with pytest.raises(lib.OdiseError):
            shapes(**bad)
    with pytest.raises(lib.OdiseError):
        lib.grounding_forward(torch.zeros(1, 1, 4, 32), torch.zeros(1, 2, 32), torch.ones(1, 2, dtype=torch.bool),
                              torch.ones(1), 1, 0, 1.0)     # CPU tensors: no fallback


def test_dispatch_rules(monkeypatch):
    """CPU, float64 and use_fused=False take the composed path; the fused test needs no GPU"""
    calls = []
    monkeypatch.setattr(grounding.GroundingFunction, "apply", lambda *a: calls.append(a))
    (m, w, v), = grounding_ref.inputs([2], 2, Q, K, C)[0]
    sc = torch.ones(2, dtype=torch.float64)
    grounding.grounding_losses(m, m, w, w, v, sc, 0)
    assert not calls
    assert not grounding._fused_ok(m, m, w, v, sc)
    assert not grounding._fused_ok(m.float(), m.float(), w.float(), v, sc.float())      # CPU


def test_dispatch_sends_oversize_shapes_to_the_composed_path():
    """a global batch past the kernels' 32-bit element counts takes the composed path instead of raising"""
    with FakeTensorMode():
        dev = torch.device("cuda")

        def ok(G, B=8, S=10, Q=100, K=8, C=256):
            return grounding._fused_ok(torch.empty(S, B, Q, C, device=dev), torch.empty(S, G, Q, C, device=dev),
                                       torch.empty(B, K, C, device=dev), torch.empty(G, K, dtype=torch.bool, device=dev),
                                       torch.empty(S, device=dev))
        assert ok(64)
        assert not ok(8400)         # S·G·Q·C >= 2^31
        assert not ok(64, K=33)
    assert lib.grounding_supported(10, 8000, 8, 100, 8, 256)
    assert not lib.grounding_supported(10, 8400, 8, 100, 8, 256)
    assert not lib.grounding_supported(10, 8000, 8, 100, 32, 256)     # S·P·Q·K >= 2^31


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


_GLOO_SIZES = {2: [2, 3], 3: [2, 3, 1]}


def _worker(rank, world, port, mode, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        counts = {"fwd": 0, "bwd": 0}
        phase = ["fwd"]
        for name in ("all_gather", "all_reduce", "all_gather_into_tensor", "reduce_scatter", "broadcast", "reduce",
                     "gather", "scatter", "all_to_all"):
            fn = getattr(dist, name)

            def wrapped(*a, _fn=fn, **k):
                counts[phase[0]] += 1
                return _fn(*a, **k)
            setattr(dist, name, wrapped)
        sizes = _GLOO_SIZES[world]
        Sx = 10
        ranks, scales = _leaves(sizes, seed=5, S=Sx)
        m, w, v = ranks[rank]
        sc = scales[rank]
        outputs = {"mask_embed": m[0], "word_embed": w, "logit_scale": sc[0],
                   "aux_outputs": [{"mask_embed": m[s], "word_embed": w, "logit_scale": sc[s]} for s in range(1, Sx)]}
        targets = [{"word_valid_mask": v[b]} for b in range(v.shape[0])]
        crit = grounding.MaskGroundingCriterion(collect_mode=mode, loss_weight=0.7)
        out = crit(outputs, targets)
        losses = torch.stack(list(out.values()))
        g = torch.Generator().manual_seed(11)
        wts = torch.randn(Sx, generator=g, dtype=torch.float64)
        phase[0] = "bwd"
        grads = torch.autograd.grad((losses * wts).sum(), [m, w] + sc)
        q.put((rank, losses.detach(), [x.detach() for x in grads], counts))
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(240)
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ["diff", "concat"])
def test_gloo_world(world, mode):
    """every rank's losses and local gradients against the emulated oracle; at most 2 collectives forward and 1
    backward per step of 10 sets"""
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, mode, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        r, *rest = q.get(timeout=200)
        res[r] = rest
    for p in procs:
        p.join(30)
        assert p.exitcode == 0
    sizes = _GLOO_SIZES[world]
    Sx = 10
    ranks, scales = _leaves(sizes, seed=5, S=Sx)
    losses = grounding_ref.reference_losses(ranks, scales, mode, loss_weight=0.7)
    g = torch.Generator().manual_seed(11)
    wts = torch.randn(Sx, generator=g, dtype=torch.float64)
    total = sum((torch.stack(l) * wts).sum() for l in losses)
    leaves = [t for m, w, _ in ranks for t in (m, w)] + [s for per in scales for s in per]
    want = torch.autograd.grad(total, leaves)
    for r in range(world):
        got_losses, got_grads, counts = res[r]
        assert counts["fwd"] <= 3 and counts["bwd"] <= 1, counts
        want_r = [want[2 * r], want[2 * r + 1]] + list(want[2 * world + Sx * r: 2 * world + Sx * (r + 1)])
        tol = 1e-12      # all_reduce and autograd may add the ranks' contributions in different orders
        torch.testing.assert_close(got_losses, torch.stack(losses[r]).detach(), rtol=0, atol=tol)
        for a, b in zip(got_grads, want_r):
            torch.testing.assert_close(a, b, rtol=0, atol=tol * max(1.0, b.abs().max().item()))
