"""The masked cross-attention drop-in on the GPU (odise_b200/masked_attn.py, odise_b200/csrc/masked_xattn.cu).

Parity is measured against a float64 evaluation of the same layer: a copy of it in float64 taking nn.MultiheadAttention
(use_fused = False) on the same weights and inputs, for the output and the gradients of tgt, memory, pos, query_pos and
every parameter.  The bars sit next to each comparison."""
import copy

import pytest
import torch

from odise_b200 import lib
from odise_b200.masked_attn import CrossAttentionLayer, MaskedCrossAttnFunction

pytestmark = pytest.mark.gpu

ODISE_LEVELS = [32 * 32, 64 * 64, 128 * 128]
ROUNDOFF = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}


def _mask(kind, B, H, Q, S, g, device):
    """bool masks (True = blocked) of the kinds the decoder makes"""
    if kind == "none":
        return None
    if kind == "allowed":
        return torch.zeros(B * H, Q, S, dtype=torch.bool, device=device)
    if kind == "sparse":
        m = torch.rand(B * H, Q, S, generator=g, device=device) < 0.8
        m[torch.arange(B * H, device=device)[:, None], torch.arange(Q, device=device)[None, :],
          torch.randint(0, S, (B * H, Q), generator=g, device=device)] = False
        return m
    if kind == "one":
        m = torch.ones(B * H, Q, S, dtype=torch.bool, device=device)
        m[torch.arange(B * H, device=device)[:, None], torch.arange(Q, device=device)[None, :],
          torch.randint(0, S, (B * H, Q), generator=g, device=device)] = False
        return m
    if kind in ("logits", "bcast"):
        # odise.py: sigmoid(mask logits) < 0.5 is blocked, per image, repeated over the heads; then the fix-up of
        # odise.py:683 (a row with every key blocked attends everywhere)
        shape = (Q, S) if kind == "bcast" else (B, Q, S)
        m = torch.randn(*shape, generator=g, device=device).sigmoid() < 0.5
        m[:3] = True           # a few fully blocked rows for the fix-up to clear
        if kind == "logits":
            m = m.unsqueeze(1).repeat(1, H, 1, 1).flatten(0, 1)
        m[torch.where(m.sum(-1) == m.shape[-1])] = False
        return m
    raise ValueError(kind)


def _problem(Q, S, B=2, C=256, H=8, kind="logits", seed=0, normalize_before=False, device="cuda"):
    torch.manual_seed(seed)
    layer = CrossAttentionLayer(C, H, normalize_before=normalize_before).to(device)
    with torch.no_grad():          # non-trivial LayerNorm and biases
        for p in layer.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.1)
    g = torch.Generator(device=device).manual_seed(seed + 1)
    tgt, memory = torch.randn(Q, B, C, generator=g, device=device), torch.randn(S, B, C, generator=g, device=device)
    pos, qpos = torch.randn(S, B, C, generator=g, device=device), torch.randn(Q, B, C, generator=g, device=device)
    return layer, (tgt, memory, pos, qpos), _mask(kind, B, H, Q, S, g, device)


def _run(layer, inputs, mask, dtype=None, seed=5):
    """output and gradients (tgt, memory, pos, query_pos, parameters) of one forward + backward; dtype = autocast dtype"""
    xs = [x.detach().clone().requires_grad_(True) for x in inputs]
    with torch.autocast("cuda", dtype=dtype, enabled=dtype is not None):
        out = layer(xs[0], xs[1], memory_mask=mask, pos=xs[2], query_pos=xs[3])
    g = torch.Generator(device=out.device).manual_seed(seed)
    w = torch.randn(out.shape, generator=g, device=out.device, dtype=torch.float32)
    grads = torch.autograd.grad((out.float() * w.to(out.dtype).float()).sum(), xs + list(layer.parameters()))
    return [out] + list(grads)


def _fp64(layer, inputs, mask):
    ref = copy.deepcopy(layer).double()
    ref.use_fused = False
    return _run(ref, [x.double() for x in inputs], mask)


NAMES = ["out", "tgt", "memory", "pos", "query_pos"]


def _errors(got, want, layer):
    names = NAMES + [n for n, _ in layer.named_parameters()]
    return {n: ((a.double() - b).abs().max().item(), max(1.0, b.abs().max().item())) for n, a, b in zip(names, got, want)}


def _count_fused(monkeypatch):
    calls = []
    fwd = lib.masked_xattn_forward

    def counted(*a):
        calls.append(1)
        return fwd(*a)
    monkeypatch.setattr(lib, "masked_xattn_forward", counted)
    return calls


FP32_CASES = [
    dict(Q=100, S=32 * 32, kind="logits"), dict(Q=100, S=64 * 64, kind="sparse"), dict(Q=100, S=128 * 128, kind="logits"),
    dict(Q=1, S=1000, kind="sparse"), dict(Q=300, S=1024, kind="one"), dict(Q=100, S=1, kind="none"),
    dict(Q=37, S=777, kind="allowed"), dict(Q=100, S=500, kind="bcast"),
    dict(Q=100, S=256, kind="logits", normalize_before=True),
]


@pytest.mark.parametrize("case", FP32_CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_float32_parity(cuda, case, record, monkeypatch):
    calls = _count_fused(monkeypatch)
    layer, inputs, mask = _problem(**case)
    got = _run(layer, inputs, mask)
    assert calls, "the fused path was not taken"
    want = _fp64(layer, inputs, mask)
    errs = _errors(got, want, layer)
    worst = max(e / s for e, s in errs.values())
    record(f"masked_xattn fp32 {case}: max err / max(1, max|ref|) = {worst:.2e}")
    for n, (e, s) in errs.items():
        assert e <= 1e-5 * s, (n, e, s)          # float32 bar: 1e-5 x max(1, max |ref|)


AUTOCAST_CASES = [dict(Q=100, S=s, kind="logits") for s in ODISE_LEVELS] + [dict(Q=300, S=777, kind="sparse")]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", AUTOCAST_CASES, ids=lambda c: f"Q{c['Q']}-S{c['S']}")
def test_autocast_parity(cuda, case, dtype, record, monkeypatch):
    calls = _count_fused(monkeypatch)
    layer, inputs, mask = _problem(**case)
    layer.fused_16bit_max_keys = None       # the kernels at every length (by default 128^2 keys stay composed)
    got = _run(layer, inputs, mask, dtype=dtype)
    assert calls
    layer.use_fused = False
    comp = _run(layer, inputs, mask, dtype=dtype)
    want = _fp64(layer, inputs, mask)
    errs, errs_c = _errors(got, want, layer), _errors(comp, want, layer)
    u = ROUNDOFF[dtype]
    record(f"masked_xattn {dtype} {case}: fused {max(e / s for e, s in errs.values()):.2e}, "
           f"composed {max(e / s for e, s in errs_c.values()):.2e} (x max(1, max|ref|))")
    for n, (e, s) in errs.items():
        # 16-bit bar: a few units of roundoff of the storage type relative to max(1, max |ref|), or no more than twice
        # the error of nn.MultiheadAttention under the same autocast where that is larger (sums over many rows)
        assert e <= max(8 * u * s, 2 * errs_c[n][0]), (n, e, s, errs_c[n][0])


def test_eval_no_grad(cuda):
    layer, inputs, mask = _problem(100, 4096, kind="logits")
    layer.eval()
    with torch.no_grad():
        out = layer(inputs[0], inputs[1], memory_mask=mask, pos=inputs[2], query_pos=inputs[3])
        ref = copy.deepcopy(layer).double()
        ref.use_fused = False
        want = ref(*[x.double() for x in inputs[:2]], memory_mask=mask, pos=inputs[2].double(),
                   query_pos=inputs[3].double())
    assert (out.double() - want).abs().max().item() <= 1e-5 * max(1.0, want.abs().max().item())


def _qkv(Q, S, B=2, H=8, dtype=torch.float32, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(Q, B, H * 32, generator=g, device="cuda").to(dtype)
    k = torch.randn(S, B, H * 32, generator=g, device="cuda").to(dtype)
    v = torch.randn(S, B, H * 32, generator=g, device="cuda").to(dtype)
    return q, k, v, torch.randn(Q, B, H * 32, generator=g, device="cuda").to(dtype), g


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_deterministic_and_graph_replay(cuda, dtype):
    Q, S, B, H = 100, 64 * 64, 2, 8
    q, k, v, go, g = _qkv(Q, S, dtype=dtype)
    mask = _mask("sparse", B, H, Q, S, g, "cuda")
    out, lse = lib.masked_xattn_forward(q, k, v, mask, H)
    first = lib.masked_xattn_backward(q, k, v, mask, out, lse, go, H)
    second = lib.masked_xattn_backward(q, k, v, mask, out, lse, go, H)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    out2, lse2 = lib.masked_xattn_forward(q, k, v, mask, H)
    assert torch.equal(out, out2) and torch.equal(lse, lse2)
    # the whole forward + backward captured in a CUDA graph and replayed gives the eager bits
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lib.masked_xattn_backward(q, k, v, mask, *lib.masked_xattn_forward(q, k, v, mask, H), go, H)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out, g_lse = lib.masked_xattn_forward(q, k, v, mask, H)
        g_grads = lib.masked_xattn_backward(q, k, v, mask, g_out, g_lse, go, H)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_out, out) and torch.equal(g_lse, lse)
    for a, b in zip(g_grads, first):
        assert torch.equal(a, b)


def test_fully_masked_rows_give_torchs_nans(cuda):
    """A row whose keys are all blocked: NaN output row and dq row, NaN dk / dv over its (image, head), as torch's math
    path gives; every other (image, head) stays finite."""
    Q, S, B, H = 40, 300, 2, 4
    q, k, v, go, g = _qkv(Q, S, B=B, H=H)
    mask = _mask("sparse", B, H, Q, S, g, "cuda")
    mask[3, 7] = True          # (b 0, head 3), query 7
    mask[5, 0] = True          # (b 1, head 1), query 0
    xs = [t.clone().requires_grad_(True) for t in (q, k, v)]
    out = MaskedCrossAttnFunction.apply(*xs, mask, H)
    got = [out] + list(torch.autograd.grad(out, xs, go))
    ts = [t.clone().requires_grad_(True) for t in (q, k, v)]

    def heads(t):        # [L, B, H*32] -> [B*H, L, 32]
        return t.view(t.shape[0], B * H, 32).transpose(0, 1)
    sc = torch.baddbmm(torch.zeros_like(mask, dtype=torch.float32).masked_fill(mask, float("-inf")),
                       heads(ts[0]) * 32 ** -0.5, heads(ts[1]).transpose(1, 2))
    ref = torch.bmm(sc.softmax(-1), heads(ts[2])).transpose(0, 1).reshape(Q, B, H * 32)
    want = [ref] + list(torch.autograd.grad(ref, ts, go))
    for a, b in zip(got, want):
        assert torch.equal(a.isnan(), b.isnan())
        assert a.isnan().any()
        fin = ~b.isnan()
        assert (a[fin] - b[fin]).abs().max().item() < 1e-4


def _reference_composition(layer, tgt, memory, mask, kpm, pos, qpos):
    mha = layer.multihead_attn
    x = layer.norm(tgt) if layer.normalize_before else tgt
    a = mha(query=x + qpos, key=memory + pos, value=memory, attn_mask=mask, key_padding_mask=kpm)[0]
    y = tgt + layer.dropout(a)
    return y if layer.normalize_before else layer.norm(y)


@pytest.mark.parametrize("what", ["dropout", "float_mask", "key_padding_mask", "d64"])
def test_fallback_is_the_reference_bit_for_bit(cuda, what, monkeypatch):
    def refuse(*a):
        raise AssertionError("the fused path was taken")
    monkeypatch.setattr(lib, "masked_xattn_forward", refuse)
    Q, S, B = 100, 1024, 2
    H = 4 if what == "d64" else 8
    torch.manual_seed(0)
    layer = CrossAttentionLayer(256, H, dropout=0.1 if what == "dropout" else 0.0).cuda().train()
    g = torch.Generator(device="cuda").manual_seed(1)
    tgt, memory = torch.randn(Q, B, 256, generator=g, device="cuda"), torch.randn(S, B, 256, generator=g, device="cuda")
    pos, qpos = torch.randn(S, B, 256, generator=g, device="cuda"), torch.randn(Q, B, 256, generator=g, device="cuda")
    mask = _mask("logits", B, H, Q, S, g, "cuda")
    kpm = None
    if what == "float_mask":
        mask = torch.zeros(mask.shape, device="cuda").masked_fill(mask, float("-inf"))
    if what == "key_padding_mask":
        kpm = torch.zeros(B, S, dtype=torch.bool, device="cuda")
        kpm[:, -100:] = True
    results = []
    for fn in (lambda: layer(tgt, memory, memory_mask=mask, memory_key_padding_mask=kpm, pos=pos, query_pos=qpos),
               lambda: _reference_composition(layer, tgt, memory, mask, kpm, pos, qpos)):
        torch.manual_seed(7)
        out = fn()
        results.append([out] + list(torch.autograd.grad(out.sum(), list(layer.parameters()))))
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_torch_compile_fullgraph(cuda):
    layer, inputs, mask = _problem(100, 1024, kind="logits")
    eager = _run(layer, inputs, mask)
    torch._dynamo.reset()
    compiled = torch.compile(layer, fullgraph=True)
    got = _run(compiled, inputs, mask)
    for n, a, b in zip(NAMES + [n for n, _ in layer.named_parameters()], got, eager):
        assert (a - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item()), n
    # the kernels run inside the compiled graph: the op appears in the traced graph, not a graph break
    explain = torch._dynamo.explain(layer)(inputs[0], inputs[1], memory_mask=mask, pos=inputs[2], query_pos=inputs[3])
    assert explain.graph_break_count == 0


def test_decoder_stack_fused_against_composed(cuda, record):
    """9 cross-attention layers over the three ODISE levels, each mask rebuilt with the odise.py:683 fix-up, as
    ODISEMultiScaleMaskedTransformerDecoder runs them (self-attention and FFN layers left out)."""
    B, Q, C, H = 2, 100, 256, 8
    torch.manual_seed(0)
    layers = torch.nn.ModuleList([CrossAttentionLayer(C, H) for _ in range(9)]).cuda()
    g = torch.Generator(device="cuda").manual_seed(3)
    srcs = [torch.randn(s, B, C, generator=g, device="cuda") for s in ODISE_LEVELS]
    poss = [torch.randn(s, B, C, generator=g, device="cuda") for s in ODISE_LEVELS]
    masks = [_mask("logits", B, H, Q, ODISE_LEVELS[i % 3], g, "cuda") for i in range(9)]
    tgt0, qpos = torch.randn(Q, B, C, generator=g, device="cuda"), torch.randn(Q, B, C, generator=g, device="cuda")

    def run(fused):
        for layer in layers:
            layer.use_fused = fused
        xs = [t.clone().requires_grad_(True) for t in [tgt0] + srcs]
        out = xs[0]
        for i, layer in enumerate(layers):
            out = layer(out, xs[1 + i % 3], memory_mask=masks[i], pos=poss[i % 3], query_pos=qpos)
        return [out] + list(torch.autograd.grad(out.square().sum(), xs + list(layers.parameters())))
    fused, comp = run(True), run(False)
    worst = 0.0
    for a, b in zip(fused, comp):
        e = (a - b).abs().max().item() / max(1.0, b.abs().max().item())
        worst = max(worst, e)
        assert e <= 1e-4
    record(f"masked_xattn 9-layer stack fp32 fused vs composed: max rel err {worst:.2e}")


def test_dispatch_rules(cuda, monkeypatch):
    calls = _count_fused(monkeypatch)
    layer, inputs, mask = _problem(20, 300, kind="bcast")
    layer(inputs[0], inputs[1], memory_mask=mask, pos=inputs[2], query_pos=inputs[3])
    layer(inputs[0], inputs[1], memory_mask=None, pos=inputs[2], query_pos=inputs[3])
    assert len(calls) == 2
    layer.use_fused = False
    layer(inputs[0], inputs[1], memory_mask=mask, pos=inputs[2], query_pos=inputs[3])
    layer.use_fused = True
    kpm = torch.zeros(inputs[1].shape[1], inputs[1].shape[0], dtype=torch.bool, device="cuda")
    layer(inputs[0], inputs[1], memory_mask=mask, memory_key_padding_mask=kpm, pos=inputs[2],
          query_pos=inputs[3])                                                                      # padding mask
    layer.double()(*[x.double() for x in inputs[:2]], memory_mask=mask, pos=inputs[2].double(),
                   query_pos=inputs[3].double())                                                    # float64
    assert len(calls) == 2
    layer.float()
    big, big_mask = torch.randn(4097, 2, 256, device="cuda"), torch.zeros(20, 4097, dtype=torch.bool,
                                                                        device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        layer(inputs[0], big, memory_mask=big_mask, pos=big, query_pos=inputs[3])      # 16-bit above the key limit
        assert len(calls) == 2
        layer(inputs[0], inputs[1], memory_mask=mask, pos=inputs[2], query_pos=inputs[3])
        assert len(calls) == 3
        layer.fused_16bit_max_keys = None
        layer(inputs[0], big, memory_mask=big_mask, pos=big, query_pos=inputs[3])
        assert len(calls) == 4
    layer(inputs[0], big, memory_mask=big_mask, pos=big, query_pos=inputs[3])          # float32: no limit
    assert len(calls) == 5
    q, k, v, _, _ = _qkv(4, 8, H=2)
    with pytest.raises(RuntimeError):
        lib.masked_xattn_forward(q, k, v, None, 4)                       # head dim 16
    with pytest.raises(RuntimeError):
        lib.masked_xattn_forward(q[:, :1].contiguous(), k, v, None, 2)   # batch of q and k differ
    with pytest.raises(RuntimeError):
        lib.masked_xattn_forward(q, k, v, torch.zeros(4, 8, dtype=torch.bool), 2)   # mask on the CPU
