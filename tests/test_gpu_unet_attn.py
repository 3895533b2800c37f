"""The UNet attention drop-in on the GPU (odise_b200/unet_attn.py, odise_b200/csrc/unet_attn.cu).

Parity is measured as err(t) = max|t - t64| / max|t64| against a float64 run of the same module on the composed path
(use_fused = False), for the output and the gradients of x, context and the four weights.  The fused path is held to
the composed path's own error at the same storage type: float32 err <= max(4 x composed, 2e-6); float16 / bfloat16 under
autocast err <= 2 x composed."""
import copy

import pytest
import torch

from odise_b200 import lib, unet_attn
from odise_b200.unet_attn import CrossAttention, UNetAttnFunction, replace_attention
from oracle import ldm

pytestmark = pytest.mark.gpu

NAMES = ["out", "x", "context", "to_q", "to_k", "to_v", "to_out"]

# (d, Tq, Tk): SD-v1's self-attention (Tk = Tq) and cross-attention (Tk = 77) at each head dim, and ragged lengths
SD_CASES = [(40, 4096, 4096), (80, 1024, 1024), (160, 256, 256), (160, 64, 64),
            (40, 4096, 77), (80, 1024, 77), (160, 256, 77), (160, 64, 77)]
RAGGED_CASES = [(40, 4095, 4095), (80, 65, 65), (160, 1, 1), (40, 65, 77), (80, 1, 77), (40, 4095, 77)]


def _problem(d, Tq, Tk, B=2, heads=8, seed=0):
    torch.manual_seed(seed)
    cross = Tk == 77
    m = CrossAttention(heads * d, 768 if cross else None, heads, d).cuda()
    with torch.no_grad():
        m.to_out[0].bias.add_(torch.randn_like(m.to_out[0].bias) * 0.1)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    x = torch.randn(B, Tq, heads * d, generator=g, device="cuda")
    ctx = torch.randn(B, Tk, 768, generator=g, device="cuda") if cross else None
    return m, x, ctx


def _run(m, x, ctx, dtype=None, seed=5):
    """output and gradients (x, context, to_q / to_k / to_v / to_out.0 weights) of one forward + backward"""
    xs = [x.detach().clone().requires_grad_(True)]
    if ctx is not None:
        xs.append(ctx.detach().clone().requires_grad_(True))
    with torch.autocast("cuda", dtype=dtype, enabled=dtype is not None):
        out = m(xs[0], xs[1] if ctx is not None else None)
    g = torch.Generator(device=out.device).manual_seed(seed)
    w = torch.randn(out.shape, generator=g, device=out.device, dtype=torch.float32)
    ws = [m.to_q.weight, m.to_k.weight, m.to_v.weight, m.to_out[0].weight]
    grads = torch.autograd.grad((out.float() * w.to(out.dtype).float()).sum(), xs + ws)
    return [out] + list(grads[:len(xs)]) + ([None] if ctx is None else []) + list(grads[len(xs):])


def _fp64(m, x, ctx):
    ref = copy.deepcopy(m).double()
    ref.use_fused = False
    return _run(ref, x.double(), None if ctx is None else ctx.double())


def _err(a, b):
    """relative error; absolute where the reference is exactly zero (one key: the q and to_q gradients vanish)"""
    scale = b.abs().max().item()
    return (a.double() - b).abs().max().item() / (scale if scale > 0 else 1.0)


def _errors(got, want):
    return {n: _err(a, b) for n, a, b in zip(NAMES, got, want) if b is not None}


def _count_fused(monkeypatch):
    """counts the fused path's launches; the shape dispatch is lifted so that the kernels run at every shape"""
    monkeypatch.setattr(unet_attn, "fused_faster", lambda dtype, Tk: True)
    calls = []
    fwd = lib.unet_attn_forward

    def counted(*a):
        calls.append(1)
        return fwd(*a)
    monkeypatch.setattr(lib, "unet_attn_forward", counted)
    return calls


@pytest.fixture
def all_fused(monkeypatch):
    """the kernels at every supported shape, whatever the shape dispatch would pick"""
    monkeypatch.setattr(unet_attn, "fused_faster", lambda dtype, Tk: True)


def _ids(c):
    return f"d{c[0]}-Tq{c[1]}-Tk{c[2]}"


@pytest.mark.parametrize("case", SD_CASES + RAGGED_CASES, ids=_ids)
def test_float32_parity(cuda, case, record, monkeypatch):
    calls = _count_fused(monkeypatch)
    m, x, ctx = _problem(*case)
    got = _run(m, x, ctx)
    assert calls, "the fused path was not taken"
    m.use_fused = False
    comp = _run(m, x, ctx)
    want = _fp64(m, x, ctx)
    errs, errs_c = _errors(got, want), _errors(comp, want)
    record(f"unet_attn fp32 {_ids(case)}: fused {max(errs.values()):.2e}, composed {max(errs_c.values()):.2e}")
    for n in errs:
        assert errs[n] <= max(4 * errs_c[n], 2e-6), (n, errs[n], errs_c[n])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", SD_CASES + RAGGED_CASES, ids=_ids)
def test_autocast_parity(cuda, case, dtype, record, monkeypatch):
    calls = _count_fused(monkeypatch)
    m, x, ctx = _problem(*case)
    got = _run(m, x, ctx, dtype=dtype)
    assert calls and got[0].dtype == dtype
    m.use_fused = False
    comp = _run(m, x, ctx, dtype=dtype)
    want = _fp64(m, x, ctx)
    errs, errs_c = _errors(got, want), _errors(comp, want)
    record(f"unet_attn {str(dtype)[6:]} {_ids(case)}: fused {max(errs.values()):.2e}, "
           f"composed {max(errs_c.values()):.2e}")
    for n in errs:
        # a gradient that is exactly zero in fp64 (one key: q gets none) is held to an absolute 1e-5 instead
        floor = 1e-5 if not want[NAMES.index(n)].any() else 0.0
        assert errs[n] <= max(2 * errs_c[n], floor), (n, errs[n], errs_c[n])


def _qkv(Tq, Tk, d, B=2, heads=8, dtype=torch.float32, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, Tq, heads * d, generator=g, device="cuda").to(dtype)
    k = torch.randn(B, Tk, heads * d, generator=g, device="cuda").to(dtype)
    v = torch.randn(B, Tk, heads * d, generator=g, device="cuda").to(dtype)
    return q, k, v, torch.randn(B, Tq, heads * d, generator=g, device="cuda").to(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("Tk", [1024, 77])
def test_reproducible_deterministic_and_graph_replay(cuda, dtype, Tk):
    q, k, v, go = _qkv(1024, Tk, 80, dtype=dtype)

    def both():
        out, lse = lib.unet_attn_forward(q, k, v, 8)
        return [out, lse, *lib.unet_attn_backward(q, k, v, out, lse, go, 8)]
    first, second = both(), both()
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    torch.use_deterministic_algorithms(True)
    try:
        third = both()
    finally:
        torch.use_deterministic_algorithms(False)
    for a, b in zip(first, third):
        assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        both()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = both()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(captured, first):
        assert torch.equal(a, b)


def test_no_host_sync(cuda, all_fused):
    m, x, ctx = _problem(40, 4096, 77)
    _run(m, x, ctx)                                  # warm-up: library load, opt-ins
    xs = [x.clone().requires_grad_(True), ctx.clone().requires_grad_(True)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = m(*xs)
        out.backward(torch.ones_like(out))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_saved_tensors_and_peak_memory(cuda, record, all_fused):
    q, k, v, _ = _qkv(64, 77, 40)
    xs = [t.clone().requires_grad_(True) for t in (q, k, v)]
    saved = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: saved.append(t) or t, lambda t: t):
        out = UNetAttnFunction.apply(*xs, 8)
    assert len(saved) == 5
    for t, want in zip(saved[:3], xs):
        assert t.data_ptr() == want.data_ptr() and t.shape == want.shape
    assert saved[3].data_ptr() == out.data_ptr() and saved[3].shape == out.shape
    assert saved[4].shape == (2 * 8, 64) and saved[4].dtype == torch.float32

    m, x, _ = _problem(40, 4096, 4096, B=8)

    def peak(fused):
        m.use_fused = fused
        xx = x.clone().requires_grad_(True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = m(xx)
        out.backward(torch.ones_like(out))
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated() - base
        del out, xx
        m.zero_grad(set_to_none=True)
        return p
    pf, pc = peak(True), peak(False)
    record(f"unet_attn B=8 d=40 T=4096 fp32 fwd+bwd peak: fused {pf / 2 ** 20:.0f} MiB, composed {pc / 2 ** 20:.0f} MiB")
    assert pf * 20 <= pc, (pf, pc)


def test_torch_compile_fullgraph(cuda, all_fused):
    m, x, ctx = _problem(40, 1024, 77)
    eager = _run(m, x, ctx)
    torch._dynamo.reset()
    compiled = torch.compile(m, fullgraph=True)
    got = _run(compiled, x, ctx)
    for n, a, b in zip(NAMES, got, eager):
        assert torch.equal(a, b), n
    explain = torch._dynamo.explain(m)(x, ctx)
    assert explain.graph_break_count == 0


def test_whole_unet_against_fp64(cuda, record, monkeypatch, all_fused):
    """oracle.ldm.UNetModel (random init) at a 64^2 latent, B = 2, through oracle.ldm.unet_features: the four taps and
    the gradients of context and cond_emb of a fixed random linear functional of the taps, composed and patched with
    replace_attention (every attention layer on the kernels), against a float64 run."""
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        torch.manual_seed(0)
        unet = ldm.UNetModel().cuda()
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(2, 4, 64, 64, generator=g, device="cuda")
        ctx = torch.randn(2, 77, 768, generator=g, device="cuda")
        cond = torch.randn(2, 1280, generator=g, device="cuda") * 0.5

        def run(model, dtype=torch.float32):
            c, e = ctx.to(dtype).requires_grad_(True), cond.to(dtype).requires_grad_(True)
            taps = ldm.unet_features(model, x.to(dtype), c, e)
            gw = torch.Generator(device="cuda").manual_seed(2)
            f = sum((t * torch.randn(t.shape, generator=gw, device="cuda").to(dtype)).sum() for t in taps)
            return taps + list(torch.autograd.grad(f, [c, e]))
        ref = copy.deepcopy(unet).double()
        ref.time_embed.register_forward_pre_hook(lambda mod, a: (a[0].double(),))   # timestep_embedding is float32
        with monkeypatch.context() as mp:          # GroupNorm32 computes in float32; a no-op cast for the fp32 runs
            mp.setattr(ldm.GroupNorm32, "forward", torch.nn.GroupNorm.forward)
            want = run(ref, torch.float64)
        comp = run(unet)
        assert replace_attention(unet) == 32
        fused = run(unet)
        names = ["tap0", "tap1", "tap2", "tap3", "context", "cond_emb"]
        ef = {n: _err(a, b) for n, a, b in zip(names, fused, want)}
        ec = {n: _err(a, b) for n, a, b in zip(names, comp, want)}
        record(f"unet_attn whole UNet B=2 64^2 fp32: fused {max(ef.values()):.2e}, composed {max(ec.values()):.2e}")
        for n in names:
            assert ef[n] <= 2 * ec[n], (n, ef[n], ec[n])
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def _oracle_twin(m):
    o = ldm.CrossAttention(m.to_q.in_features, m.to_k.in_features, m.heads, m.to_q.out_features // m.heads)
    o.load_state_dict(m.state_dict())
    return o.to(m.to_q.weight.device)


@pytest.mark.parametrize("what", ["mask", "dropout", "d64", "cpu"])
def test_fallback_is_the_oracle_bit_for_bit(cuda, what, monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(lib, "_launch", refuse)
    dev = "cpu" if what == "cpu" else "cuda"
    d = 64 if what == "d64" else 40
    torch.manual_seed(0)
    m = CrossAttention(8 * d, 768, 8, d, dropout=0.1 if what == "dropout" else 0.0).to(dev).train()
    ref = _oracle_twin(m)
    if what == "dropout":
        ref.to_out = m.to_out
    g = torch.Generator(device=dev).manual_seed(1)
    x, ctx = torch.randn(2, 256, 8 * d, generator=g, device=dev), torch.randn(2, 77, 768, generator=g, device=dev)
    mask = None
    if what == "mask":         # a mask that blocks no key: ldm's masked_fill changes nothing, so the oracle's bits
        mask = torch.ones(2, 77, dtype=torch.bool, device=dev)
    torch.manual_seed(7)
    out = m(x, ctx, mask=mask)
    got = [out] + list(torch.autograd.grad(out.sum(), [m.to_q.weight, m.to_k.weight, m.to_v.weight]))
    torch.manual_seed(7)
    out = ref(x, ctx)
    want = [out] + list(torch.autograd.grad(out.sum(), [ref.to_q.weight, ref.to_k.weight, ref.to_v.weight]))
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_mask_against_sdpa_fp64(cuda, monkeypatch):
    """A key mask (False = blocked) takes the composed path; its output and weight gradients against float64
    F.scaled_dot_product_attention with the same boolean mask on the same projections (an independent computation)."""
    def refuse(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(lib, "_launch", refuse)
    torch.manual_seed(0)
    m = CrossAttention(320, 768, 8, 40).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    x, ctx = torch.randn(2, 256, 320, generator=g, device="cuda"), torch.randn(2, 77, 768, generator=g, device="cuda")
    mask = torch.rand(2, 77, generator=g, device="cuda") < 0.5
    mask[:, 0] = True
    ws = [m.to_q.weight, m.to_k.weight, m.to_v.weight]
    out = m(x, ctx, mask=mask)
    got = [out] + list(torch.autograd.grad(out.sum(), ws))
    w64 = [w.detach().double().requires_grad_(True) for w in ws]
    q, k, v = x.double() @ w64[0].T, ctx.double() @ w64[1].T, ctx.double() @ w64[2].T
    q, k, v = (t.view(2, t.shape[1], 8, 40).transpose(1, 2) for t in (q, k, v))
    a = torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=mask[:, None, None, :])
    ref = torch.nn.functional.linear(a.transpose(1, 2).reshape(2, 256, 320), m.to_out[0].weight.double(),
                                     m.to_out[0].bias.double())
    want = [ref] + list(torch.autograd.grad(ref.sum(), w64))
    for a_, b_ in zip(got, want):
        assert _err(a_, b_) <= 1e-5


def test_lib_rejects_before_launch(cuda, monkeypatch):
    q, k, v, go = _qkv(64, 77, 40)

    def refuse(*a, **kw):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(lib, "_launch", refuse)
    bad = {
        "head dim 64": lambda: lib.unet_attn_forward(q, k, v, 5),
        "heads do not divide": lambda: lib.unet_attn_forward(q, k, v, 7),
        "float64": lambda: lib.unet_attn_forward(q.double(), k.double(), v.double(), 8),
        "mixed dtypes": lambda: lib.unet_attn_forward(q, k.half(), v, 8),
        "non-contiguous": lambda: lib.unet_attn_forward(q.transpose(0, 1), k, v, 8),
        "k / v disagree": lambda: lib.unet_attn_forward(q, k, v[:, :-1], 8),
        "batch": lambda: lib.unet_attn_forward(q[:1], k, v, 8),
        "cpu": lambda: lib.unet_attn_forward(q.cpu(), k.cpu(), v.cpu(), 8),
    }
    for what, call in bad.items():
        with pytest.raises(lib.OdiseError):
            call()
            pytest.fail(what)
