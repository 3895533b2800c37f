"""CPU checks of the masked cross-attention drop-in (odise_b200/masked_attn.py): the layer's surface against the
reference's CrossAttentionLayer (live where the reference tree is present, pinned in tests/golden otherwise), the
composed path on CPU, the custom ops' schemas, fake implementations and errors under FakeTensorMode (which makes "cuda"
tensors without a device), and the C ABI's exports and argument checks."""
import ctypes
import importlib
import inspect

import pytest
import torch
from torch import nn
from torch._subclasses.fake_tensor import FakeTensorMode

from oracle import refshim

FIXTURE = "ref_pinned_masked_xattn.pt"


def _ref_class():
    refshim.install()
    return importlib.import_module(
        "mask2former.modeling.transformer_decoder.mask2former_transformer_decoder").CrossAttentionLayer


def _inputs(Q=5, B=2, S=7, C=64, H=2, seed=1):
    g = torch.Generator().manual_seed(seed)
    tgt, mem = torch.randn(Q, B, C, generator=g), torch.randn(S, B, C, generator=g)
    pos, qpos = torch.randn(S, B, C, generator=g), torch.randn(Q, B, C, generator=g)
    mask = torch.rand(B * H, Q, S, generator=g) < 0.4
    mask[:, :, 0] = False
    return tgt, mem, pos, qpos, mask


def _reference_surface():
    cls = _ref_class()
    out = dict(init_kwargs=[p for p in inspect.signature(cls.__init__).parameters if p != "self"],
               defaults={p.name: p.default for p in inspect.signature(cls.__init__).parameters.values()
                         if p.default is not inspect.Parameter.empty})
    for fn in ("forward", "forward_post", "forward_pre"):
        out[fn] = [p for p in inspect.signature(getattr(cls, fn)).parameters if p != "self"]
    torch.manual_seed(0)
    layer = cls(64, 2)
    out["state_dict"] = {k: v.clone() for k, v in layer.state_dict().items()}
    tgt, mem, pos, qpos, mask = _inputs()
    with torch.no_grad():
        out["post"] = layer(tgt, mem, memory_mask=mask, pos=pos, query_pos=qpos)
        layer.normalize_before = True
        out["pre"] = layer(tgt, mem, memory_mask=mask, pos=pos, query_pos=qpos)
    return out


@pytest.fixture(scope="module")
def ref():
    return refshim.pinned(None, _reference_surface, fixture=FIXTURE)


def test_surface_matches_reference(ref):
    from odise_b200.masked_attn import CrossAttentionLayer
    sig = inspect.signature(CrossAttentionLayer.__init__).parameters
    assert [p for p in sig if p != "self"] == ref["init_kwargs"]
    assert {p.name: p.default for p in sig.values() if p.default is not inspect.Parameter.empty} == ref["defaults"]
    for fn in ("forward", "forward_post", "forward_pre"):
        assert [p for p in inspect.signature(getattr(CrossAttentionLayer, fn)).parameters if p != "self"] == ref[fn]
    torch.manual_seed(0)
    mine = CrossAttentionLayer(64, 2)
    sd = mine.state_dict()
    assert list(sd) == list(ref["state_dict"])
    for k, v in sd.items():                    # same initialisation, parameter by parameter, from the same seed
        assert torch.equal(v, ref["state_dict"][k]), k
    assert isinstance(mine.multihead_attn, nn.MultiheadAttention) and isinstance(mine.norm, nn.LayerNorm)
    assert isinstance(mine.dropout, nn.Dropout)
    # state dicts load both ways
    mine.load_state_dict(ref["state_dict"])
    if refshim.available():
        theirs = _ref_class()(64, 2)
        theirs.load_state_dict(mine.state_dict())


def test_cpu_layer_matches_reference(ref):
    from odise_b200.masked_attn import CrossAttentionLayer
    mine = CrossAttentionLayer(64, 2)
    mine.load_state_dict(ref["state_dict"])
    tgt, mem, pos, qpos, mask = _inputs()
    with torch.no_grad():
        post = mine(tgt, mem, memory_mask=mask, pos=pos, query_pos=qpos)
        mine.normalize_before = True
        pre = mine(tgt, mem, memory_mask=mask, pos=pos, query_pos=qpos)
    # the reference's arithmetic on CPU, recorded on another machine where the tree is absent: BLAS bits may differ
    tol = 0 if refshim.available() else 1e-6
    torch.testing.assert_close(post, ref["post"], rtol=0, atol=tol)
    torch.testing.assert_close(pre, ref["pre"], rtol=0, atol=tol)


@pytest.mark.parametrize("normalize_before", [False, True])
def test_cpu_path_is_multihead_attention_and_layernorm(normalize_before):
    """On CPU the layer is nn.MultiheadAttention + dropout + residual + LayerNorm, bit for bit, forward and backward."""
    from odise_b200.masked_attn import CrossAttentionLayer
    torch.manual_seed(3)
    layer = CrossAttentionLayer(64, 2, normalize_before=normalize_before)
    tgt, mem, pos, qpos, mask = _inputs(seed=4)
    tgt.requires_grad_(True)
    out = layer(tgt, mem, memory_mask=mask, pos=pos, query_pos=qpos)
    g1 = torch.autograd.grad(out.sum(), [tgt] + list(layer.parameters()))
    mha, norm = layer.multihead_attn, layer.norm
    x = norm(tgt) if normalize_before else tgt
    a = mha(query=x + qpos, key=mem + pos, value=mem, attn_mask=mask, key_padding_mask=None)[0]
    want = tgt + a if normalize_before else norm(tgt + a)
    g2 = torch.autograd.grad(want.sum(), [tgt] + list(layer.parameters()))
    assert torch.equal(out, want)
    for a_, b_ in zip(g1, g2):
        assert torch.equal(a_, b_)


def test_activation_names():
    from odise_b200.masked_attn import CrossAttentionLayer
    for name in ("relu", "gelu", "glu"):
        CrossAttentionLayer(64, 2, activation=name)
    with pytest.raises(RuntimeError):
        CrossAttentionLayer(64, 2, activation="tanh")


SCHEMAS = {
    "masked_xattn_forward": "odise_b200::masked_xattn_forward(Tensor q, Tensor k, Tensor v, Tensor? mask, int heads) "
                            "-> (Tensor, Tensor)",
    "masked_xattn_backward": "odise_b200::masked_xattn_backward(Tensor q, Tensor k, Tensor v, Tensor? mask, "
                             "Tensor out, Tensor lse, Tensor grad_out, int heads) -> (Tensor, Tensor, Tensor)",
}


@pytest.fixture
def ops(monkeypatch):
    from odise_b200 import lib, masked_attn  # noqa: F401  (importing masked_attn defines the ops)

    def no_library():
        raise AssertionError("a fake implementation loaded the shared library")
    monkeypatch.setattr(lib, "load", no_library)
    return torch.ops.odise_b200


def test_schemas(ops):
    for name, schema in SCHEMAS.items():
        assert str(getattr(ops, name).default._schema) == schema


def _args(Q=7, B=2, S=33, H=3, D=32, dtype=torch.float32, mask="full"):
    E = H * D
    q = torch.empty(Q, B, E, dtype=dtype, device="cuda")
    k, v = torch.empty(S, B, E, dtype=dtype, device="cuda"), torch.empty(S, B, E, dtype=dtype, device="cuda")
    m = {"full": lambda: torch.empty(B * H, Q, S, dtype=torch.bool, device="cuda"),
         "bcast": lambda: torch.empty(Q, S, dtype=torch.bool, device="cuda"), "none": lambda: None}[mask]()
    return q, k, v, m


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mask", ["full", "bcast", "none"])
def test_fake_results(ops, dtype, mask):
    with FakeTensorMode():
        q, k, v, m = _args(dtype=dtype, mask=mask)
        out, lse = ops.masked_xattn_forward(q, k, v, m, 3)
        assert (tuple(out.shape), out.dtype, out.device.type) == ((7, 2, 96), dtype, "cuda")
        assert (tuple(lse.shape), lse.dtype, lse.device.type) == ((6, 7), torch.float32, "cuda")
        gq, gk, gv = ops.masked_xattn_backward(q, k, v, m, out, lse, torch.empty_like(out), 3)
        for g, t in ((gq, q), (gk, k), (gv, v)):
            assert (g.shape, g.dtype, g.device.type) == (t.shape, t.dtype, "cuda")


def test_fake_errors(ops):
    with FakeTensorMode():
        q, k, v, m = _args()
        bad = {
            "head dim 64": lambda: ops.masked_xattn_forward(*_args(H=2, D=64)[:4], 2),
            "heads do not divide": lambda: ops.masked_xattn_forward(q, k, v, None, 5),
            "float64": lambda: ops.masked_xattn_forward(*_args(dtype=torch.float64, mask="none"), 3),
            "mixed dtypes": lambda: ops.masked_xattn_forward(q, k.half(), v, m, 3),
            "float mask": lambda: ops.masked_xattn_forward(q, k, v, m.float(), 3),
            "mask shape": lambda: ops.masked_xattn_forward(q, k, v, m[:, :, :-1], 3),
            "non-contiguous": lambda: ops.masked_xattn_forward(q.transpose(0, 1), k, v, None, 3),
            "k / v disagree": lambda: ops.masked_xattn_forward(q, k, v[:-1], None, 3),
            "batch": lambda: ops.masked_xattn_forward(q[:, :1].contiguous(), k, v, None, 3),
            "cpu": lambda: ops.masked_xattn_forward(*[t.cpu() for t in _args(mask="none")[:3]], None, 3),
            "lse shape": lambda: ops.masked_xattn_backward(q, k, v, m, q, torch.empty(6, 8, device="cuda"), q, 3),
            "lse dtype": lambda: ops.masked_xattn_backward(q, k, v, m, q, torch.empty(6, 7, dtype=torch.float16,
                                                                                       device="cuda"), q, 3),
            "grad_out dtype": lambda: ops.masked_xattn_backward(q, k, v, m, q, torch.empty(6, 7, device="cuda"),
                                                                q.half(), 3),
        }
        for what, call in bad.items():
            with pytest.raises(RuntimeError):
                call()
                pytest.fail(what)


def test_real_op_on_cpu_raises():
    from odise_b200 import masked_attn  # noqa: F401
    q = torch.zeros(2, 1, 32)
    with pytest.raises(RuntimeError):
        torch.ops.odise_b200.masked_xattn_forward(q, q, q, None, 1)


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


NAMES = ["odise_masked_xattn_workspace_bytes"] + [f"odise_masked_xattn_{d}_{s}" for d in ("forward", "backward")
                                                  for s in ("f32", "f16", "bf16")]


def test_cabi_exports_prototypes_and_checks(built):
    from odise_b200 import lib
    dll = ctypes.CDLL(built)
    for n in NAMES:
        assert hasattr(dll, n), n
        assert n in lib._PROTOS
    L = lib.load()
    ws = L.odise_masked_xattn_workspace_bytes(2, 8, 100, 16384)
    assert ws >= 4 * (2 * 8 * 100 * 34) and ws % 16 == 0
    assert L.odise_masked_xattn_workspace_bytes(2, 8, 100, 0) == 0
    assert L.odise_masked_xattn_workspace_bytes(2, 8, 0, 16) == 0
    p = 256   # a non-null, aligned dummy address: every check below returns before anything is launched
    for s in ("f32", "f16", "bf16"):
        fwd, bwd = getattr(L, "odise_masked_xattn_forward_" + s), getattr(L, "odise_masked_xattn_backward_" + s)
        assert fwd(None, p, p, None, 0, p, p, 2, 8, 32, 10, 10, p, None) == 10001                          # null q
        assert fwd(p, p, p, None, 0, p, p, 2, 8, 32, 10, 10, None, None) == 10005                          # workspace
        assert fwd(p, p, p, None, 0, p, p, 2, 8, 64, 10, 10, p, None) == lib.ODISE_ERR_UNSUPPORTED         # D = 64
        assert fwd(p, p, p, None, 0, p, p, 2, 8, 32, 0, 10, p, None) == 10001                              # Q = 0
        assert fwd(p, p, p, None, 0, p, p, 2, 8, 32, 10, -1, p, None) == 10001                             # S < 0
        assert fwd(p, p, p, p, -1, p, p, 2, 8, 32, 10, 10, p, None) == 10001                               # stride
        assert fwd(p + 2, p, p, None, 0, p, p, 2, 8, 32, 10, 10, p, None) == 10002                         # align
        assert bwd(p, p, p, None, 0, p, p, p, p, p, None, 2, 8, 32, 10, 10, p, None) == 10001
        assert bwd(p, p, p, None, 0, p, p, p, p, p, p, 2, 8, 16, 10, 10, p, None) == lib.ODISE_ERR_UNSUPPORTED
        assert bwd(p, p, p, None, 0, p, p, p, p, p, p, 2, 8, 32, 10, 10, None, None) == 10005
