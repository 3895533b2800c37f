"""Category scoring without a GPU: the composed path of odise_b200.category against the reference's
CategoryODISE.cal_pred_logits + ensemble_logits_with_labels (values and float64 gradients, pinned in
tests/golden/ref_pinned_category.pt), the fake implementations of its custom ops, the shape checks and the dispatch."""
import ctypes

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from odise_b200 import category, lib
from oracle import refshim
from category_ref import coco_labels, inputs

FIXTURE = "ref_pinned_category.pt"


def _labels(case):
    if case == "coco":
        return coco_labels()
    if case == "singletons":
        return [[f"c{i}"] for i in range(7)]
    return [["a"], ["b", "b", "b2"], ["c"], ["d", "d"]]     # duplicated prompts within a group


def _outputs(case, seed=0):
    labels = _labels(case)
    B, Q, C = (2, 4, 16) if case == "coco" else (2, 5, 8)
    me, te, ne, ls = inputs(B, Q, C, [len(l) for l in labels], seed=seed)
    if case == "duplicates":
        te[2] = te[1]           # "b" twice: equal rows, equal scores
        te[5] = te[4]
    for t in (me, te, ne, ls):
        t.requires_grad_()
    return dict(mask_embed=me, text_embed=te, null_embed=ne, labels=labels, logit_scale=ls)


def _value_and_grads(fn, outputs):
    out = fn(outputs)
    g = torch.Generator().manual_seed(9)
    w = torch.randn(out.shape, generator=g, dtype=out.dtype)
    grads = torch.autograd.grad((out * w).sum(), [outputs[k] for k in ("mask_embed", "text_embed", "null_embed",
                                                                       "logit_scale")])
    return dict(out=out.detach(), grads=[x.detach() for x in grads])


@pytest.mark.parametrize("case", ["coco", "singletons", "duplicates"])
def test_composed_path_matches_reference(case):
    """the composed path runs the reference's ops: bit-equal values and float64 gradients"""
    def ref():
        # the point_rend helpers that ODISE's imports reach are set first, as the criterion tests need them before
        # mask2former's matcher first loads, whichever test runs first
        import mask_criterion_ref
        mask_criterion_ref.classes()
        m = refshim.modules()
        return _value_and_grads(lambda o: m.CategoryODISE.cal_pred_logits(None, o), _outputs(case))
    want = refshim.pinned(f"category/{case}", ref, fixture=FIXTURE)
    got = _value_and_grads(category.cal_pred_logits, _outputs(case))
    assert got["out"].shape == want["out"].shape
    assert torch.equal(got["out"], want["out"])
    for a, b in zip(got["grads"], want["grads"]):
        assert torch.equal(a, b)


def test_coco_bank():
    labels = coco_labels()
    sizes = [len(l) for l in labels]
    assert (len(labels), sum(sizes), max(sizes)) == (133, 254, 17)
    gs = lib.category_group_start(sizes)
    assert gs[0] == 0 and gs[-1] == 254 and len(gs) == 134


def test_op_schemas():
    ops = torch.ops.odise_b200
    assert str(ops.category_logits.default._schema) == (
        "odise_b200::category_logits(Tensor mask_embed, Tensor text_embed, Tensor null_embed, Tensor logit_scale, "
        "Tensor group_start) -> (Tensor, Tensor, Tensor)")
    assert str(ops.category_logits_backward.default._schema) == (
        "odise_b200::category_logits_backward(Tensor mask_embed, Tensor text_embed, Tensor null_embed, "
        "Tensor logit_scale, Tensor group_start, Tensor winners, Tensor norms, Tensor grad_logits) -> "
        "(Tensor, Tensor, Tensor, Tensor)")


@pytest.mark.parametrize("dtype,bank", [(torch.float32, torch.float32), (torch.float16, torch.float16),
                                        (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float32)])
def test_fakes(dtype, bank):
    ops = torch.ops.odise_b200
    with FakeTensorMode():
        me = torch.empty(4, 100, 256, device="cuda", dtype=dtype)
        te = torch.empty(254, 256, device="cuda", dtype=bank)
        ne = torch.empty(1, 256, device="cuda", dtype=bank)
        ls = torch.empty((), device="cuda")
        gs = torch.empty(134, device="cuda", dtype=torch.int32)
        out, win, norms = ops.category_logits(me, te, ne, ls, gs)
        assert out.shape == (4, 100, 134) and out.dtype == dtype
        assert win.shape == (4, 100, 134) and win.dtype == torch.uint8
        assert norms.shape == (400 + 255,) and norms.dtype == torch.float32
        gm, gt, gn, gl = ops.category_logits_backward(me, te, ne, ls, gs, win, norms, out)
        assert (gm.shape, gm.dtype, gt.shape, gt.dtype, gn.shape, gn.dtype) == (me.shape, dtype, te.shape, bank,
                                                                                 ne.shape, bank)
        assert gl.shape == () and gl.dtype == torch.float32


def test_shape_checks():
    ops = torch.ops.odise_b200
    with FakeTensorMode():
        me = torch.empty(4, 100, 256, device="cuda")
        te = torch.empty(254, 256, device="cuda")
        ne = torch.empty(1, 256, device="cuda")
        ls = torch.empty((), device="cuda")
        gs = torch.empty(134, device="cuda", dtype=torch.int32)
        bad = [
            (me.half(), te.half(), ne, ls, gs),                                           # mixed dtypes
            (me, te.half(), ne.half(), ls, gs),
            (me, te, ne.half(), ls, gs),
            (me.double(), te.double(), ne.double(), ls, gs),                              # float64
            (torch.empty(4, 100, 100, device="cuda"), torch.empty(254, 100, device="cuda"),
             torch.empty(1, 100, device="cuda"), ls, gs),                                 # C not a multiple of 32
            (torch.empty(4, 100, 1024, device="cuda"), torch.empty(254, 1024, device="cuda"),
             torch.empty(1, 1024, device="cuda"), ls, gs),                                # C > 768
            (me, torch.empty(2049, 256, device="cuda"), ne, ls, gs),                      # too many prompts
            (me, te, ne, ls, torch.empty(300, device="cuda", dtype=torch.int32)),         # K > Kp
            (me, te, ne, ls, gs.long()),
            (me, te, ne, torch.empty(1, device="cuda"), gs),                              # scale not a scalar
            (me.transpose(0, 1), te, ne, ls, gs),                                         # non-contiguous
            (me, te, torch.empty(2, 256, device="cuda"), ls, gs),
        ]
        for args in bad:
            with pytest.raises(lib.OdiseError):
                ops.category_logits(*args)
        out, win, norms = ops.category_logits(me, te, ne, ls, gs)
        with pytest.raises(lib.OdiseError):
            ops.category_logits_backward(me, te, ne, ls, gs, win.int(), norms, out)
        with pytest.raises(lib.OdiseError):
            ops.category_logits_backward(me, te, ne, ls, gs, win, norms, out.half())
    with pytest.raises(lib.OdiseError):       # CPU tensors are refused before any launch
        lib.category_logits_forward(torch.zeros(1, 4, 32), torch.zeros(3, 32), torch.zeros(1, 32), torch.ones(()),
                                    torch.tensor([0, 1, 3], dtype=torch.int32))
    for sizes in ([], [1, 0, 2], [256]):
        with pytest.raises(lib.OdiseError):
            lib.category_group_start(sizes)


def test_cabi_argument_checks():
    L = lib.load()
    for sfx in ("f32", "f16", "bf16"):
        for kind in ("forward", "backward"):
            assert hasattr(L, f"odise_category_logits_{kind}_{sfx}")
    assert L.odise_category_logits_workspace_bytes(400, 256, 133, 254) > 0
    assert L.odise_category_logits_workspace_bytes(400, 1024, 133, 254) == 0
    assert L.odise_category_logits_workspace_bytes(400, 256, 133, 4096) == 0
    ERR_ARG, ERR_WS, ERR_UNSUP = 10001, 10005, 10006
    p = ctypes.c_void_p(16)
    assert L.odise_category_logits_forward_f32(None, p, p, p, p, p, p, p, 400, 256, 133, 254, 0, None) == ERR_ARG
    assert L.odise_category_logits_forward_f16(p, p, p, p, p, p, p, p, 0, 256, 133, 254, 0, None) == ERR_ARG
    assert L.odise_category_logits_forward_bf16(p, p, p, p, p, p, p, p, 400, 100, 133, 254, 1, None) == ERR_UNSUP
    assert L.odise_category_logits_forward_f32(p, p, p, p, p, p, p, p, 400, 256, 300, 254, 0, None) == ERR_ARG
    assert L.odise_category_logits_backward_f32(p, p, p, p, p, p, p, p, p, p, p, p, 400, 256, 133, 254, 0, None,
                                                None) == ERR_WS
    assert L.odise_category_logits_backward_f16(p, p, p, p, p, p, p, None, p, p, p, p, 400, 256, 133, 254, 0, p,
                                                None) == ERR_ARG
    assert L.odise_category_logits_backward_bf16(p, p, p, p, p, p, p, p, p, p, p, p, 400, 256, 133, 3000, 0, p,
                                                 None) == ERR_UNSUP


def test_dispatch_cpu_and_float64(monkeypatch):
    """CPU inputs, in any dtype, take the composed path; the fused op is never called"""
    calls = []
    monkeypatch.setattr(category.CategoryLogitsFunction, "apply", lambda *a: calls.append(a))
    for dtype in (torch.float32, torch.float64):
        o = _outputs("duplicates")
        o.update({k: o[k].detach().to(dtype) for k in ("mask_embed", "text_embed", "null_embed")})
        out = category.cal_pred_logits(o)
        assert out.shape == (2, 5, 5) and out.dtype == dtype
    assert not calls
    assert not category._fused_ok(*[torch.empty(1)] * 4, [1])
