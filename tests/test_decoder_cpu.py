"""odise_b200.decoder on the CPU: the drop-in classes against ODISE's own (reached through oracle.refshim, pinned in
tests/golden/ref_pinned_decoder.pt where the reference tree is absent), the custom-op schemas, fakes and their errors,
and the mask-head C ABI's exports and argument checks."""
import ctypes
import inspect

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from odise_b200 import decoder as dec
from odise_b200 import lib
from oracle import refshim

FIX = "ref_pinned_decoder.pt"
KW = dict(in_channels=256, mask_classification=True, num_classes=5, hidden_dim=256, num_queries=7, nheads=8,
          dim_feedforward=64, dec_layers=3, pre_norm=False, mask_dim=256, enforce_input_project=False)


def _inputs():
    g = torch.Generator().manual_seed(1)
    x = [torch.randn(2, 256, 3 * 2 ** i, 2 * 2 ** i, generator=g, dtype=torch.float64) for i in range(3)]
    return x, torch.randn(2, 256, 24, 16, generator=g, dtype=torch.float64)


def _build(mod, pme_mod):
    torch.manual_seed(0)
    return mod.ODISEMultiScaleMaskedTransformerDecoder(post_mask_embed=pme_mod.PooledMaskEmbed(256, 256, 32), **KW)


def _run(m):
    """float64 forward + backward of a small non-square 3-level problem -> dict of results and gradients"""
    m = m.double()
    x, mf = _inputs()
    mf.requires_grad_()
    o = m(x, mf)
    loss = o["pred_masks"].sum() + o["mask_embed"].pow(2).sum() + o["pred_logits"].sum()
    for a in o["aux_outputs"]:
        loss = loss + a["pred_masks"].mean() + a["mask_pooled_features"].pow(2).sum() + a["pred_logits"].mean()
    loss.backward()
    res = {"pred_masks": o["pred_masks"], "pred_logits": o["pred_logits"], "mask_embed": o["mask_embed"],
           "pooled": o["mask_pooled_features"], "aux_masks": torch.stack([a["pred_masks"] for a in o["aux_outputs"]]),
           "grad_mf": mf.grad}
    for n, p in m.named_parameters():
        res["grad." + n] = p.grad if p.grad is not None else torch.zeros(0)
    return {k: v.detach() for k, v in res.items()}


def _ref_modules():
    """refshim.modules(), after the point_rend helpers that ODISE's imports reach are set to their restatements (the
    criterion tests need those in place before mask2former's matcher first loads, whichever test runs first)"""
    import mask_criterion_ref
    mask_criterion_ref.classes()
    return refshim.modules()


def _ref_surface():
    R = _ref_modules()
    m = _build(R, R)
    sd = m.state_dict()
    return dict(keys=list(sd), shapes=[list(v.shape) for v in sd.values()],
                params=torch.cat([v.reshape(-1) for v in sd.values()]),
                kwargs=sorted(inspect.signature(R.MultiScaleMaskedTransformerDecoder.__init__).parameters) +
                sorted(inspect.signature(R.ODISEMultiScaleMaskedTransformerDecoder.__init__).parameters),
                pme=sorted(inspect.signature(R.PooledMaskEmbed.__init__).parameters),
                pool=sorted(inspect.signature(R.MaskPooling.__init__).parameters))


def _ref_run():
    R = _ref_modules()
    return _run(_build(R, R))


def _sampled(d):
    """stored stand-ins a few hundred KB in all: 256 seeded values of each gradient, 4096 of everything else"""
    return {k: refshim.sample(v, k=256 if k.startswith("grad.") else 4096) if torch.is_tensor(v) and v.numel() > 256
            else v for k, v in d.items()}


def test_surface_matches_reference():
    ref = refshim.pinned("surface", _ref_surface, FIX, store=_sampled)
    m = _build(dec, dec)
    sd = m.state_dict()
    assert list(sd) == ref["keys"]
    assert [list(v.shape) for v in sd.values()] == ref["shapes"]
    got, want = refshim.at_sample(torch.cat([v.reshape(-1) for v in sd.values()]), ref["params"])
    assert torch.equal(got, want)
    kw = sorted(inspect.signature(dec.ODISEMultiScaleMaskedTransformerDecoder.__init__).parameters)
    assert set(kw) == set(ref["kwargs"]) - {"kwargs"}
    assert sorted(inspect.signature(dec.PooledMaskEmbed.__init__).parameters) == ref["pme"]
    assert sorted(inspect.signature(dec.MaskPooling.__init__).parameters) == ref["pool"]


def test_composed_path_matches_reference():
    """CPU (the composed path): forward and every parameter and input gradient equal the reference's, bit for bit where
    the tree is present and within 1e-10 of the pinned float64 values elsewhere"""
    ref = refshim.pinned("run", _ref_run, FIX, store=_sampled)
    got = _run(_build(dec, dec))
    assert set(got) == set(ref)
    for k, r in ref.items():
        g, w = refshim.at_sample(got[k], r)
        if refshim.available():
            assert torch.equal(g, w), k
        elif w.numel():
            assert (g - w).abs().max().item() <= 1e-10 * max(1.0, w.abs().max().item()), k


def test_state_dict_static_query_conversion():
    m = _build(dec, dec)
    sd = {k.replace("query_feat", "static_query"): v.clone() for k, v in m.state_dict().items()}
    m2 = _build(dec, dec)
    with torch.no_grad():
        m2.query_feat.weight.zero_()
    m2.load_state_dict(sd)          # no version metadata: the reference's v1 conversion applies
    assert torch.equal(m2.query_feat.weight, m.query_feat.weight)


def test_op_schemas():
    ops = torch.ops.odise_b200
    assert str(ops.mask_head_forward.default._schema) == \
        "odise_b200::mask_head_forward(Tensor embed, Tensor features, float threshold) -> (Tensor, Tensor, Tensor)"
    assert str(ops.mask_head_backward.default._schema) == (
        "odise_b200::mask_head_backward(Tensor embed, Tensor features, Tensor outputs_mask, Tensor weights, "
        "Tensor grad_mask, Tensor grad_pooled, float threshold) -> (Tensor, Tensor)")
    assert str(ops.mask_head_attn_mask.default._schema) == \
        "odise_b200::mask_head_attn_mask(Tensor outputs_mask, int h, int w, int heads) -> Tensor"


def test_fakes_and_errors():
    ops = torch.ops.odise_b200
    with FakeTensorMode():
        E = torch.empty(2, 100, 256, device="cuda")
        X = torch.empty(2, 256, 37, 53, device="cuda")
        om, pooled, w = ops.mask_head_forward(E, X, 0.5)
        assert om.shape == (2, 100, 37, 53) and pooled.shape == (2, 100, 256) and w.dtype == torch.float32
        am = ops.mask_head_attn_mask(om, 5, 7, 8)
        assert am.shape == (16, 100, 35) and am.dtype == torch.bool
        ge, gx = ops.mask_head_backward(E, X, om, w, om, pooled, 0.5)
        assert ge.shape == E.shape and gx.shape == X.shape
        bad = [(torch.empty(2, 100, 128, device="cuda"), X), (torch.empty(2, 300, 256, device="cuda"), X),
               (E, torch.empty(2, 256, 37, 53, device="cuda", dtype=torch.float16)),
               (E.double(), X.double()), (E, torch.empty(3, 256, 37, 53, device="cuda"))]
        for e, x in bad:
            with pytest.raises(lib.OdiseError):
                ops.mask_head_forward(e, x, 0.5)
        with pytest.raises(lib.OdiseError):
            ops.mask_head_backward(E, X, om, w.half(), om, pooled, 0.5)
        with pytest.raises(lib.OdiseError):
            ops.mask_head_attn_mask(om, 0, 7, 8)
    with pytest.raises(lib.OdiseError):       # CPU tensors are refused before any launch
        lib.mask_head_forward(torch.zeros(1, 4, 256), torch.zeros(1, 256, 3, 3))


def test_cabi_exports_and_argument_checks():
    L = lib.load()
    for sfx in ("f32", "f16", "bf16"):
        for kind in ("forward", "attn_mask", "backward"):
            assert hasattr(L, f"odise_mask_head_{kind}_{sfx}")
    assert L.odise_mask_head_workspace_bytes(2, 100, 256, 256, 256) > 0
    assert L.odise_mask_head_workspace_bytes(2, 300, 256, 64, 64) == 0
    assert L.odise_mask_head_workspace_bytes(2, 100, 128, 64, 64) == 0
    assert L.odise_mask_head_workspace_bytes(2, 100, 256, 4096, 4096) == 0
    ERR_ARG, ERR_WS, ERR_UNSUP = 10001, 10005, 10006
    p = ctypes.c_void_p(16)
    assert L.odise_mask_head_forward_f32(None, p, p, p, p, 2, 100, 256, 8, 8, 0.5, p, None) == ERR_ARG
    assert L.odise_mask_head_forward_f16(p, p, p, p, p, 2, 100, 256, 8, 8, 0.5, None, None) == ERR_WS
    assert L.odise_mask_head_forward_bf16(p, p, p, p, p, 2, 100, 128, 8, 8, 0.5, p, None) == ERR_UNSUP
    assert L.odise_mask_head_forward_f32(p, p, p, p, p, 2, 257, 256, 8, 8, 0.5, p, None) == ERR_UNSUP
    assert L.odise_mask_head_forward_f32(p, p, p, p, p, 0, 100, 256, 8, 8, 0.5, p, None) == ERR_ARG
    assert L.odise_mask_head_backward_f32(p, p, p, p, p, None, p, p, 2, 100, 256, 8, 8, 0.5, p, None) == ERR_ARG
    assert L.odise_mask_head_backward_bf16(p, p, p, p, p, p, p, p, 2, 100, 256, 8, 8, 0.5, None, None) == ERR_WS
    assert L.odise_mask_head_attn_mask_f32(None, p, 2, 100, 8, 8, 4, 4, 8, None) == ERR_ARG
    assert L.odise_mask_head_attn_mask_f16(p, p, 2, 100, 8, 8, 0, 4, 8, None) == ERR_ARG
