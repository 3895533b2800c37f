"""CPU checks of the UNet attention drop-in (odise_b200/unet_attn.py): the module's surface and composed path against
oracle.ldm.CrossAttention, replace_attention on oracle.ldm.UNetModel, the dispatch rules, the custom ops' schemas,
fake implementations and errors under FakeTensorMode (which makes "cuda" tensors without a device), and the C ABI's
exports and argument checks."""
import ctypes
import inspect

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from odise_b200 import lib, unet_attn
from odise_b200.unet_attn import CrossAttention, replace_attention
from oracle import ldm


def _pair(query_dim=64, context_dim=32, heads=4, dim_head=16, dtype=torch.float32):
    torch.manual_seed(0)
    o = ldm.CrossAttention(query_dim, context_dim, heads, dim_head).to(dtype)
    m = CrossAttention(query_dim, context_dim, heads, dim_head).to(dtype)
    m.load_state_dict(o.state_dict())
    return m, o


def test_surface_and_state_dict_both_ways():
    sig = inspect.signature(CrossAttention.__init__).parameters
    assert list(sig)[1:] == ["query_dim", "context_dim", "heads", "dim_head", "dropout"]
    assert [p for p in inspect.signature(CrossAttention.forward).parameters][1:] == ["x", "context", "mask"]
    m, o = _pair()
    assert list(m.state_dict()) == ["to_q.weight", "to_k.weight", "to_v.weight", "to_out.0.weight", "to_out.0.bias"]
    assert list(m.state_dict()) == list(o.state_dict())
    o2 = ldm.CrossAttention(64, 32, 4, 16)
    o2.load_state_dict(m.state_dict())
    for k, v in o2.state_dict().items():
        assert torch.equal(v, m.state_dict()[k])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("cross", [False, True])
def test_composed_path_is_the_oracle_bit_for_bit(dtype, cross):
    m, o = _pair(dtype=dtype)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 10, 64, generator=g, dtype=dtype)
    ctx = torch.randn(2, 7, 32, generator=g, dtype=dtype) if cross else None
    if not cross:
        m, o = _pair(context_dim=None, dtype=dtype)
    results = []
    for mod in (m, o):
        xs = [x.clone().requires_grad_(True)] + ([ctx.clone().requires_grad_(True)] if cross else [])
        out = mod(*xs)
        w = torch.randn(out.shape, generator=torch.Generator().manual_seed(2), dtype=dtype)
        results.append([out] + list(torch.autograd.grad((out * w).sum(), xs + list(mod.parameters()))))
    for a, b in zip(*results):
        assert torch.equal(a, b)


def _small_unet():
    torch.manual_seed(0)
    return ldm.UNetModel(model_channels=32, context_dim=32).eval()


def test_replace_attention_on_the_oracle_unet():
    unet = _small_unet()
    keys = list(unet.state_dict())
    tensors = {k: v.clone() for k, v in unet.state_dict().items()}
    params = dict(unet.named_parameters())
    g = torch.Generator().manual_seed(3)
    x, ctx, cond = torch.randn(1, 4, 16, 16, generator=g), torch.randn(1, 5, 32, generator=g), torch.randn(1, 128)
    with torch.no_grad():
        before = ldm.unet_features(unet, x, ctx, cond)
    assert replace_attention(unet) == 32
    assert sum(isinstance(m, CrossAttention) for m in unet.modules()) == 32
    assert list(unet.state_dict()) == keys
    for k, v in unet.state_dict().items():
        assert torch.equal(v, tensors[k]), k
    for n, p in unet.named_parameters():
        assert p is params[n], n
    with torch.no_grad():
        after = ldm.unet_features(unet, x, ctx, cond)
    for a, b in zip(before, after):
        assert torch.equal(a, b)
    assert replace_attention(unet) == 0          # already swapped


def test_replace_attention_counts_32_on_sd_v1():
    with torch.device("meta"):
        unet = ldm.UNetModel()
    params = dict(unet.named_parameters())
    assert replace_attention(unet) == 32
    assert all(p is params[n] for n, p in unet.named_parameters())


@pytest.fixture
def fused_calls(monkeypatch):
    """CPU tensors pass for CUDA ones, and UNetAttnFunction records its calls instead of launching"""
    calls = []
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda t: True))

    def record(q, k, v, heads):
        calls.append((q.dtype, tuple(q.shape), tuple(k.shape), heads))
        return torch.zeros_like(q)
    monkeypatch.setattr(unet_attn.UNetAttnFunction, "apply", record)
    return calls


def test_dispatch_rules(fused_calls):
    m = CrossAttention(320, 768, 8, 40)
    x, ctx = torch.randn(1, 64, 320), torch.randn(1, 77, 768)
    s = CrossAttention(320, None, 8, 40)
    m(x, ctx)                                           # cross-attention: fused
    s(x)                                                # self-attention at 64 keys: fused
    assert len(fused_calls) == 2
    m.use_fused = False
    m(x, ctx)
    m.use_fused = True
    m(x, ctx, mask=torch.ones(1, 77, dtype=torch.bool))
    m.double()(x.double(), ctx.double())               # float64 projections
    m.float()
    d64 = CrossAttention(512, 768, 8, 64)
    d64(torch.randn(1, 64, 512), ctx)                  # head dim 64
    assert len(fused_calls) == 2
    drop = CrossAttention(320, 768, 8, 40, dropout=0.1)
    drop.train()(x, ctx)                                # output dropout in effect
    assert len(fused_calls) == 2
    drop.eval()(x, ctx)                                 # dropout off in eval mode
    assert len(fused_calls) == 3
    odd = CrossAttention(320, 768, 8, 40)
    odd.scale = 0.1                                     # not d^-1/2: the kernels would compute another attention
    odd(x, ctx)
    assert len(fused_calls) == 3
    # by shape: composed at 1024 keys in every dtype; fused at 77, up to 256 and at 4096 keys
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        assert unet_attn.fused_faster(dt, 77) and unet_attn.fused_faster(dt, 256) and unet_attn.fused_faster(dt, 4096)
        assert not unet_attn.fused_faster(dt, 1024)
    s(torch.randn(1, 1024, 320))
    assert len(fused_calls) == 3
    s(torch.randn(1, 4096, 320))
    assert len(fused_calls) == 4


SCHEMAS = {
    "unet_attn_forward": "odise_b200::unet_attn_forward(Tensor q, Tensor k, Tensor v, int heads) -> (Tensor, Tensor)",
    "unet_attn_backward": "odise_b200::unet_attn_backward(Tensor q, Tensor k, Tensor v, Tensor out, Tensor lse, "
                          "Tensor grad_out, int heads) -> (Tensor, Tensor, Tensor)",
}


@pytest.fixture
def ops(monkeypatch):
    def no_library():
        raise AssertionError("a fake implementation loaded the shared library")
    monkeypatch.setattr(lib, "load", no_library)
    return torch.ops.odise_b200


def test_schemas(ops):
    for name, schema in SCHEMAS.items():
        assert str(getattr(ops, name).default._schema) == schema


def _args(Tq=7, Tk=77, B=2, H=8, D=40, dtype=torch.float32):
    return (torch.empty(B, Tq, H * D, dtype=dtype, device="cuda"), torch.empty(B, Tk, H * D, dtype=dtype, device="cuda"),
            torch.empty(B, Tk, H * D, dtype=dtype, device="cuda"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D", [40, 80, 160])
def test_fake_results(ops, dtype, D):
    with FakeTensorMode():
        q, k, v = _args(D=D, dtype=dtype)
        out, lse = ops.unet_attn_forward(q, k, v, 8)
        assert (tuple(out.shape), out.dtype, out.device.type) == ((2, 7, 8 * D), dtype, "cuda")
        assert (tuple(lse.shape), lse.dtype, lse.device.type) == ((16, 7), torch.float32, "cuda")
        gq, gk, gv = ops.unet_attn_backward(q, k, v, out, lse, torch.empty_like(out), 8)
        for g, t in ((gq, q), (gk, k), (gv, v)):
            assert (g.shape, g.dtype, g.device.type) == (t.shape, t.dtype, "cuda")


def test_fake_errors(ops):
    with FakeTensorMode():
        q, k, v = _args()
        lse = torch.empty(16, 7, device="cuda")
        bad = {
            "head dim 64": lambda: ops.unet_attn_forward(*_args(H=5, D=64), 5),
            "head dim 32": lambda: ops.unet_attn_forward(*_args(D=32), 8),
            "heads do not divide": lambda: ops.unet_attn_forward(q, k, v, 7),
            "float64": lambda: ops.unet_attn_forward(*_args(dtype=torch.float64), 8),
            "mixed dtypes": lambda: ops.unet_attn_forward(q, k.half(), v, 8),
            "non-contiguous": lambda: ops.unet_attn_forward(q.transpose(0, 1), k, v, 8),
            "strided k": lambda: ops.unet_attn_forward(q, k[:, ::2], v[:, ::2], 8),
            "k / v disagree": lambda: ops.unet_attn_forward(q, k, v[:, :-1], 8),
            "batch": lambda: ops.unet_attn_forward(q[:1], k, v, 8),
            "empty keys": lambda: ops.unet_attn_forward(q, k[:, :0], v[:, :0], 8),
            "2-D q": lambda: ops.unet_attn_forward(q[0], k, v, 8),
            "cpu": lambda: ops.unet_attn_forward(*[t.cpu() for t in _args()], 8),
            "lse shape": lambda: ops.unet_attn_backward(q, k, v, q, torch.empty(16, 8, device="cuda"), q, 8),
            "lse dtype": lambda: ops.unet_attn_backward(q, k, v, q, lse.half(), q, 8),
            "grad_out dtype": lambda: ops.unet_attn_backward(q, k, v, q, lse, q.half(), 8),
            "out shape": lambda: ops.unet_attn_backward(q, k, v, q[:, :-1], lse, q, 8),
        }
        for what, call in bad.items():
            with pytest.raises(lib.OdiseError):
                call()
                pytest.fail(what)


def test_supported():
    assert lib.unet_attn_supported(8, 8, 40, 4096, 4096) and lib.unet_attn_supported(8, 8, 160, 1, 77)
    assert not lib.unet_attn_supported(8, 8, 64, 4096, 4096)
    assert not lib.unet_attn_supported(8, 8, 40, 0, 77) and not lib.unet_attn_supported(8, 8, 40, 77, 0)
    assert not lib.unet_attn_supported(65536, 1, 40, 1, 1)


def test_real_op_on_cpu_raises():
    q = torch.zeros(1, 2, 320)
    with pytest.raises(RuntimeError):
        torch.ops.odise_b200.unet_attn_forward(q, q, q, 8)


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


NAMES = ["odise_unet_attn_workspace_bytes"] + [f"odise_unet_attn_{d}_{s}" for d in ("forward", "backward")
                                               for s in ("f32", "f16", "bf16")]


def test_cabi_exports_prototypes_and_checks(built):
    dll = ctypes.CDLL(built)
    for n in NAMES:
        assert hasattr(dll, n), n
        assert n in lib._PROTOS
    L = lib.load()
    # delta only at self-attention; query-chunk partials of dK / dV where the keys give few blocks (cross-attention)
    assert L.odise_unet_attn_workspace_bytes(8, 8, 40, 4096, 4096) == 4 * 8 * 8 * 4096
    assert L.odise_unet_attn_workspace_bytes(8, 8, 40, 4096, 77) > 4 * 8 * 8 * 4096
    assert L.odise_unet_attn_workspace_bytes(8, 8, 64, 10, 10) == 0
    assert L.odise_unet_attn_workspace_bytes(8, 8, 40, 0, 10) == 0
    p = 256   # a non-null, aligned dummy address: every check below returns before anything is launched
    for s in ("f32", "f16", "bf16"):
        fwd, bwd = getattr(L, "odise_unet_attn_forward_" + s), getattr(L, "odise_unet_attn_backward_" + s)
        assert fwd(None, p, p, p, p, 2, 8, 40, 10, 10, None) == lib.ODISE_ERR_ARG                   # null q
        assert fwd(p, p, p, p, p, 2, 8, 64, 10, 10, None) == lib.ODISE_ERR_UNSUPPORTED               # D = 64
        assert fwd(p, p, p, p, p, 2, 8, 40, 0, 10, None) == lib.ODISE_ERR_ARG                        # Tq = 0
        assert fwd(p, p, p, p, p, 2, 8, 40, 10, -1, None) == lib.ODISE_ERR_ARG                       # Tk < 0
        assert fwd(p + 2, p, p, p, p, 2, 8, 40, 10, 10, None) == lib.ODISE_ERR_ALIGN                 # align
        assert bwd(p, p, p, p, p, p, p, p, None, 2, 8, 40, 10, 10, p, None) == lib.ODISE_ERR_ARG     # null grad_v
        assert bwd(p, p, p, p, p, p, p, p, p, 2, 8, 80, 10, 10, None, None) == lib.ODISE_ERR_WORKSPACE
        assert bwd(p, p, p, p, p, p, p, p, p, 2, 8, 32, 10, 10, p, None) == lib.ODISE_ERR_UNSUPPORTED
        assert bwd(p, p, p, p, p, p, p, p, p, 2, 8, 160, 10, 10, p + 4, None) == lib.ODISE_ERR_ALIGN
