"""CPU checks of the SetCriterion / HungarianMatcher drop-in (odise_b200/criterion.py): the surface against the
reference's classes, the composed path pinned against the reference's own forward (live where the reference tree is
present, from tests/golden/ref_pinned_mask_criterion.pt otherwise), lib's argument checks without data, and the C ABI's
exports and argument checks."""
import ctypes
import inspect

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from oracle import refshim

FIXTURE = "ref_pinned_mask_criterion.pt"
Q, K, P, LAYERS = 5, 4, 40, 9
COUNTS = (0, 7, 3)          # an image without targets, one with more targets than queries
PRED_HW, TGT_HW = (12, 10), (24, 20)


def _problem(seed=0):
    g = torch.Generator().manual_seed(seed)
    B = len(COUNTS)

    def one_set():
        return {"pred_logits": torch.randn(B, Q, K + 1, generator=g) * 2,
                "pred_masks": torch.randn(B, Q, *PRED_HW, generator=g) * 3}
    outputs = one_set()
    outputs["aux_outputs"] = [one_set() for _ in range(LAYERS)]
    targets = [{"labels": torch.randint(0, K, (T,), generator=g),
                "masks": torch.rand(T, *TGT_HW, generator=g) < 0.4} for T in COUNTS]
    return outputs, targets


def _kwargs():
    return dict(num_classes=K, class_weight=2.0, mask_weight=5.0, dice_weight=5.0, num_layers=LAYERS, eos_coef=0.1,
                losses=["labels", "masks"], num_points=P, oversample_ratio=3.0, importance_sample_ratio=0.75)


def _run(crit_cls, matcher_cls, seed=0):
    """indices of every set (the matcher alone, seeded per set), the criterion's losses and pred_masks gradients (seeded)"""
    matcher = matcher_cls(cost_class=2.0, cost_mask=5.0, cost_dice=5.0, num_points=P)
    crit = crit_cls(matcher=matcher, **_kwargs())
    outputs, targets = _problem()
    sets = [outputs] + outputs["aux_outputs"]
    indices = []
    for i, s in enumerate(sets):
        torch.manual_seed(100 + i)
        indices.append([(a.clone(), b.clone()) for a, b in matcher({k: v for k, v in s.items() if k != "aux_outputs"},
                                                                   targets)])
    for s in sets:
        s["pred_masks"].requires_grad_(True)
    torch.manual_seed(seed)
    losses = crit(outputs, targets)
    total = sum(crit.weight_dict[k] * v for k, v in losses.items())
    grads = torch.autograd.grad(total, [s["pred_masks"] for s in sets])
    return dict(indices=indices, losses={k: v.detach() for k, v in losses.items()}, grads=[g.clone() for g in grads],
                rng_after=torch.rand(4))


def _surface(crit_cls, matcher_cls):
    def sig(f):
        ps = inspect.signature(f).parameters
        return ([p for p in ps if p != "self"],
                {n: p.default for n, p in ps.items() if p.default is not inspect.Parameter.empty})
    crit = crit_cls(matcher=matcher_cls(2.0, 5.0, 5.0, P), **_kwargs())
    return dict(crit_sig=sig(crit_cls.__init__), matcher_sig=sig(matcher_cls.__init__), weight_dict=crit.weight_dict,
                state_dict={k: v.clone() for k, v in crit.state_dict().items()}, repr=repr(crit),
                matcher_repr=repr(crit.matcher))


@pytest.fixture(scope="module")
def ref():
    def compute():
        import mask_criterion_ref
        crit_cls, matcher_cls = mask_criterion_ref.classes()
        return dict(surface=_surface(crit_cls, matcher_cls), run=_run(crit_cls, matcher_cls))
    return refshim.pinned(None, compute, fixture=FIXTURE)


def _mine():
    from odise_b200.criterion import HungarianMatcher, SetCriterion
    return SetCriterion, HungarianMatcher


def test_surface_matches_reference(ref):
    s = _surface(*_mine())
    r = ref["surface"]
    assert s["crit_sig"] == tuple(r["crit_sig"]) or list(s["crit_sig"]) == list(r["crit_sig"])
    assert s["matcher_sig"][0] == list(r["matcher_sig"][0]) and s["matcher_sig"][1] == dict(r["matcher_sig"][1])
    assert s["weight_dict"] == r["weight_dict"]
    assert list(s["state_dict"]) == list(r["state_dict"]) == ["empty_weight"]
    assert torch.equal(s["state_dict"]["empty_weight"], r["state_dict"]["empty_weight"])
    assert s["repr"] == r["repr"] and s["matcher_repr"] == r["matcher_repr"]
    crit_cls, matcher_cls = _mine()
    with pytest.raises(AssertionError, match="all costs cant be 0"):
        matcher_cls(0, 0, 0)
    # state dicts load both ways
    mine = crit_cls(matcher=matcher_cls(2.0, 5.0, 5.0, P), **_kwargs())
    mine.load_state_dict(r["state_dict"])
    if refshim.available():
        import mask_criterion_ref
        theirs_cls, theirs_matcher = mask_criterion_ref.classes()
        theirs_cls(matcher=theirs_matcher(2.0, 5.0, 5.0, P), **_kwargs()).load_state_dict(mine.state_dict())


def test_composed_path_pinned_to_reference(ref):
    """Same seed -> the reference's indices, losses (every key of a 10-set forward), gradients and RNG state after."""
    got = _run(*_mine())
    want = ref["run"]
    tol = 0 if refshim.available() else 1e-6
    for gi, wi in zip(got["indices"], want["indices"]):
        assert len(gi) == len(wi) == len(COUNTS)
        for (a, b), (c, d) in zip(gi, wi):
            assert a.dtype == b.dtype == torch.int64 and a.device.type == "cpu"
            assert torch.equal(a, c) and torch.equal(b, d)
    assert list(got["losses"]) == list(want["losses"])
    assert len(got["losses"]) == 3 * (LAYERS + 1)
    for k, v in got["losses"].items():
        assert v.dtype == torch.float32 and v.dim() == 0, k
        torch.testing.assert_close(v, want["losses"][k], rtol=0, atol=tol, msg=k)
    # the reference's loss functions are TorchScript, whose autodiff backward rounds differently from eager's
    for g, w in zip(got["grads"], want["grads"]):
        torch.testing.assert_close(g, w, rtol=1e-5, atol=1e-8)
    # the same number of random draws in the same order: the generator ends in the same state
    assert torch.equal(got["rng_after"], want["rng_after"])


def test_matcher_alone_matches_reference_indices_and_shapes():
    crit_cls, matcher_cls = _mine()
    outputs, targets = _problem(seed=3)
    m = matcher_cls(1, 1, 1, num_points=P)
    idx = m(outputs, targets)
    for (i, j), T in zip(idx, COUNTS):
        assert len(i) == len(j) == min(Q, T)
        assert torch.equal(i, i.sort().values)


def test_other_matcher_is_called_per_set():
    crit_cls, matcher_cls = _mine()
    calls = []
    inner = matcher_cls(2.0, 5.0, 5.0, P)

    def matcher(out, targets):
        calls.append(out["pred_masks"].shape)
        return inner(out, targets)
    crit = crit_cls(matcher=matcher, **_kwargs())
    outputs, targets = _problem()
    torch.manual_seed(0)
    a = crit(outputs, targets)
    assert len(calls) == LAYERS + 1
    torch.manual_seed(0)
    b = crit_cls(matcher=inner, **_kwargs())(outputs, targets)
    for k in a:
        assert torch.equal(a[k], b[k]), k


# ---- lib's argument checks (no data, no library) ----

@pytest.fixture
def nolib(monkeypatch):
    from odise_b200 import lib

    def no_library():
        raise AssertionError("an argument check loaded the shared library")
    monkeypatch.setattr(lib, "load", no_library)
    return lib


def test_lib_argument_checks(nolib):
    lib = nolib
    with FakeTensorMode():
        d = "cuda"
        pred = torch.empty(2, 5, 16, 12, device=d)
        tgt = torch.empty(4, 32, 24, dtype=torch.bool, device=d)
        prob = torch.empty(2, 5, 7, device=d)
        labels = torch.empty(4, dtype=torch.int64, device=d)
        pts = torch.empty(2, 50, 2, device=d)
        pairs = torch.empty(4, 3, dtype=torch.int64, device=d)
        cand = torch.empty(4, 150, 2, device=d)
        rnd = torch.empty(4, 13, 2, device=d)
        pair_of = torch.empty(10, dtype=torch.int64, device=d)
        state = torch.empty(4 * (16 + 8 * 50), dtype=torch.uint8, device=d)
        bad = {
            "pred float64": lambda: lib.mask_cost(pred.double(), prob, labels, tgt, pts, [1, 3], 1, 1, 1),
            "float targets": lambda: lib.mask_cost(pred, prob, labels, tgt.float(), pts, [1, 3], 1, 1, 1),
            "pred 3-D": lambda: lib.mask_cost(pred[0], prob, labels, tgt, pts, [1, 3], 1, 1, 1),
            "counts": lambda: lib.mask_cost(pred, prob, labels, tgt, pts, [1, 2], 1, 1, 1),
            "prob shape": lambda: lib.mask_cost(pred, prob[:1], labels, tgt, pts, [1, 3], 1, 1, 1),
            "prob dtype": lambda: lib.mask_cost(pred, prob.half(), labels, tgt, pts, [1, 3], 1, 1, 1),
            "labels dtype": lambda: lib.mask_cost(pred, prob, labels.int(), tgt, pts, [1, 3], 1, 1, 1),
            "points": lambda: lib.mask_cost(pred, prob, labels, tgt, pts[:, :, :1], [1, 3], 1, 1, 1),
            "non-contiguous": lambda: lib.mask_cost(pred.transpose(2, 3), prob, labels, tgt, pts, [1, 3], 1, 1, 1),
            "too many candidates": lambda: lib.mask_loss_forward(
                pred, tgt, pairs, torch.empty(4, lib.MASK_MAX_CANDIDATES + 1, 2, device=d), rnd, 4.0, 50, 37),
            "k > P": lambda: lib.mask_loss_forward(pred, tgt, pairs, cand, rnd, 4.0, 50, 51),
            "rnd rows": lambda: lib.mask_loss_forward(pred, tgt, pairs, cand, rnd[:, :5], 4.0, 50, 37),
            "pairs dtype": lambda: lib.mask_loss_forward(pred, tgt, pairs.int(), cand, rnd, 4.0, 50, 37),
            "pair_of": lambda: lib.mask_loss_backward(pred, tgt, pairs, torch.empty(9, dtype=torch.int64, device=d),
                                                      state, torch.empty(2, device=d), 4.0, 50),
            "grad_losses": lambda: lib.mask_loss_backward(pred, tgt, pairs, pair_of, state, torch.empty(3, device=d),
                                                          4.0, 50),
            "state size": lambda: lib.mask_loss_backward(pred, tgt, pairs, pair_of, state[:100],
                                                         torch.empty(2, device=d), 4.0, 50),
        }
        for what, call in bad.items():
            with pytest.raises(lib.OdiseError):
                call()
                pytest.fail(what)
    with pytest.raises(lib.OdiseError):       # real CPU tensors
        lib.mask_cost(torch.zeros(1, 2, 4, 4), torch.zeros(1, 2, 3), torch.zeros(1, dtype=torch.int64),
                      torch.zeros(1, 4, 4, dtype=torch.bool), torch.zeros(1, 5, 2), [1], 1, 1, 1)


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


NAMES = ["odise_mask_loss_workspace_bytes", "odise_mask_point_sample_u8"] + [
    f"odise_mask_{d}_{s}" for d in ("cost", "loss_forward", "loss_backward", "point_sample") for s in ("f32", "f16", "bf16")]


def test_cabi_exports_prototypes_and_checks(built):
    from odise_b200 import lib
    dll = ctypes.CDLL(built)
    for n in NAMES:
        assert hasattr(dll, n), n
        assert n in lib._PROTOS
    L = lib.load()
    assert L.odise_mask_loss_workspace_bytes(0, 10) == 0
    assert L.odise_mask_loss_workspace_bytes(111, 12544) == 111 * 16 + 111 * 12544 * 8
    p = 256
    cnt = (ctypes.c_int * 2)(1, 3)
    for s in ("f32", "f16", "bf16"):
        cost = getattr(L, "odise_mask_cost_" + s)
        fwd, bwd = getattr(L, "odise_mask_loss_forward_" + s), getattr(L, "odise_mask_loss_backward_" + s)
        assert cost(None, p, p, p, p, cnt, p, 2, 5, 8, 8, 7, 16, 16, 3, 50, 1., 1., 1., None) == 10001      # null pred
        assert cost(p, p, p, p, p, cnt, p, 2, 5, 8, 8, 7, 16, 16, 2, 50, 1., 1., 1., None) == 10001         # T > Tmax
        assert cost(p, p, p, p, p, cnt, p, 300, 5, 8, 8, 7, 16, 16, 3, 50, 1., 1., 1., None) == 10006       # images
        assert cost(p, p, p, p, p, cnt, p, 2, 5, 8, 8, 7, 16, 16, 3, 0, 1., 1., 1., None) == 10001          # P = 0
        big = lib.MASK_MAX_CANDIDATES + 1
        assert fwd(p, p, p, p, p, p, p, 2, 5, 8, 8, 16, 16, 4, 50, big, 37, 4., None) == 10006           # candidates
        assert fwd(p, p, p, p, p, p, p, 2, 5, 8, 8, 16, 16, 4, 50, 150, 51, 4., None) == 10001           # k > P
        assert fwd(p, p, p, p, p, p, p, 2, 5, 8, 8, 16, 16, 4, 50, 150, 37, 0., None) == 10001           # num_masks
        assert fwd(p, p, p, p, p, None, p, 2, 5, 8, 8, 16, 16, 4, 50, 150, 37, 4., None) == 10005        # workspace
        assert fwd(p, p, p, p, p, p + 4, p, 2, 5, 8, 8, 16, 16, 4, 50, 150, 37, 4., None) == 10002       # align
        ps = getattr(L, "odise_mask_point_sample_" + s)
        assert ps(None, p, p, 2, 8, 8, 5, None) == 10001 and ps(p, p, p, 2, 8, 0, 5, None) == 10001
        assert bwd(p, p, p, None, p, p, p, 2, 5, 8, 8, 16, 16, 4, 50, 4., None) == 10001                   # pair_of
        assert bwd(p, p, p, p, None, p, p, 2, 5, 8, 8, 16, 16, 4, 50, 4., None) == 10005                   # state
        assert bwd(p, p, p, p, p, p, p, 2, 5, 8, 8, 16, 16, 4, lib.MASK_MAX_POINTS + 1, 4., None) == 10006
