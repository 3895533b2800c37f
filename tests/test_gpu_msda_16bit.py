"""GPU checks of MSDeformAttn with 16-bit storage (odise_msda_fused_f16 / _bf16 and their backward, and the module under
torch.autocast or cast to float16 / bfloat16): the entry points against the fp64 oracle at the rounded inputs,
bit-equality with the float32 kernels, determinism and CUDA-graph capture, module steps on both dispatch paths against
each other and against the fp64 module oracle, a short mixed-precision training run, and the error classes.

u is the unit roundoff of the storage type: 2^-11 for float16, 2^-8 for bfloat16."""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}

# tests/test_gpu_msda_module.py::FUSED_CASES, restated
FUSED_CASES = [
    dict(seed=4, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64)], Lq=5376, P=4),               # 512^2 release
    dict(seed=5, N=1, M=8, D=32, shapes=[(32, 32), (64, 64), (128, 128)], Lq=21504, P=4),            # 1024^2
    dict(seed=8, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64), (128, 128)], Lq=300, P=4),    # C4: L = 4
    dict(seed=9, N=1, M=8, D=32, shapes=[(9, 7), (5, 3)], Lq=37, P=3),           # L*P = 6: ragged sub-warp, tail block
    dict(seed=10, N=2, M=5, D=32, shapes=[(4, 4)] * 8, Lq=19, P=4),              # L*P = 32: the largest D = 32 block
    dict(seed=11, N=2, M=8, D=32, shapes=[(5, 7), (3, 2)], Lq=23, P=4, far=True),  # far outside: all grads exactly 0
]
NAMES = ("grad_value", "grad_offsets", "grad_logits")


def _id(cfg):
    return f"L{len(cfg['shapes'])}-P{cfg['P']}-Lq{cfg['Lq']}" + ("-far" if cfg.get("far") else "")


def _dt(dtype):
    return {torch.float16: "f16", torch.bfloat16: "bf16"}[dtype]


def _on(dev, tensors):
    return [t.to(dev) for t in tensors]


def _problem(cfg, dtype):
    from oracle.msda_16bit import fused_problem_16bit
    return fused_problem_16bit(**cfg, dtype=dtype)


def _within(got, want, u):
    """element-wise |got - ref| <= u |ref| + 1e-5 max(1, max |ref|): one rounding of an fp32 result that meets the float32
    kernels' bar -> (ok, worst ratio of error to bar)"""
    g, w = got.detach().cpu().double(), want.double()
    bar = u * w.abs() + 1e-5 * max(1.0, w.abs().max().item())
    ratio = ((g - w).abs() / bar).max().item()
    return ratio <= 1.0, ratio


@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("cfg", FUSED_CASES, ids=_id)
def test_fused_16bit_vs_fp64_oracle(cuda, cfg, dtype, record):
    from odise_b200 import lib
    from oracle.msda_16bit import oracle_fused_forward
    from oracle.msda_module import oracle_fused_grads
    prob = _problem(cfg, dtype)
    want_out = oracle_fused_forward(*prob[:6])
    want = oracle_fused_grads(*prob)
    args = _on(cuda, prob)
    out = lib.msda_fused_forward_16bit(*args[:6])
    got = lib.msda_fused_backward_16bit(*args)
    torch.cuda.synchronize()
    assert out.dtype == dtype and out.shape == want_out.shape
    ok, r = _within(out, want_out, U[dtype])
    assert ok, ("out", r)
    ratios = [f"out {r:.2f}"]
    for name, g, w in zip(NAMES, got, want):
        assert g.shape == w.shape and g.dtype == dtype, name
        ok, r = _within(g, w, U[dtype])
        assert ok, (name, r)
        ratios.append(f"{name} {r:.2f}")
        if cfg.get("far"):
            assert g.abs().max().item() == 0, name
    if cfg.get("far"):
        assert out.abs().max().item() == 0
    record(f"msda fused {_dt(dtype)} vs fp64 oracle {_id(cfg)}: max err / bar: " + " ".join(ratios))


def _grad_value_close(got, want, dtype, scale):
    """|got - want| <= one 16-bit ulp of the larger + 1e-6 * scale: two roundings of fp32 sums whose atomics ran in
    different orders.  The 1e-6 is the float32 kernel's own order dependence (tests/test_gpu_msda_module.py's determinism
    bar); it matters where a sum cancels to nearly zero, so that its 16-bit ulp is smaller than the reordering."""
    from oracle.msda_16bit import ulp
    a, b = got.double(), want.double()
    return ((a - b).abs() <= ulp(torch.maximum(a.abs(), b.abs()), dtype) + 1e-6 * scale).all().item()


@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("cfg", [FUSED_CASES[0], FUSED_CASES[3], FUSED_CASES[4]], ids=_id)
def test_bit_equality_with_float32_kernels(cuda, cfg, dtype):
    """The 16-bit kernels load exactly, compute the float32 kernels' fp32 arithmetic in the same order and round once:
    out, grad_offsets and grad_logits equal the float32 entry points' results on the upcast inputs, rounded, bit for bit.
    grad_value (fp32 atomics in both, order-dependent) is within one 16-bit ulp of the float32 result rounded, plus the
    float32 kernel's own order dependence (_grad_value_close)."""
    from odise_b200 import lib
    value, ss, lsi, ref, offs, logits, go = _on(cuda, _problem(cfg, dtype))
    up = [t.float() for t in (value, offs, logits, go)]
    o32 = lib.msda_fused_forward(up[0], ss, lsi, ref, up[1], up[2])
    o16 = lib.msda_fused_forward_16bit(value, ss, lsi, ref, offs, logits)
    assert torch.equal(o16, o32.to(dtype))
    g32 = lib.msda_fused_backward(up[0], ss, lsi, ref, up[1], up[2], up[3])
    g16 = lib.msda_fused_backward_16bit(value, ss, lsi, ref, offs, logits, go)
    assert torch.equal(g16[1], g32[1].to(dtype)) and torch.equal(g16[2], g32[2].to(dtype))
    assert _grad_value_close(g16[0], g32[0].to(dtype), dtype, g32[0].abs().max().item())


@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("cfg", [FUSED_CASES[0], FUSED_CASES[4]], ids=_id)
def test_determinism_and_graph_capture(cuda, cfg, dtype):
    """grad_offsets / grad_logits: bit-identical across eager calls and a CUDA-graph replay into NaN-filled buffers; the
    forward output too.  grad_value goes through fp32 atomics (order-dependent) and one rounding (_grad_value_close)."""
    from odise_b200 import lib
    args = _on(cuda, _problem(cfg, dtype))
    a = lib.msda_fused_backward_16bit(*args)
    b = lib.msda_fused_backward_16bit(*args)
    fa = lib.msda_fused_forward_16bit(*args[:6])
    torch.cuda.synchronize()
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    scale = a[0].abs().max().item()
    assert _grad_value_close(b[0], a[0], dtype, scale)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lib.msda_fused_backward_16bit(*args)             # warm-up on the side stream before capture
        lib.msda_fused_forward_16bit(*args[:6])
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = lib.msda_fused_backward_16bit(*args)
        fc = lib.msda_fused_forward_16bit(*args[:6])
    for t in list(c) + [fc]:
        t.fill_(float("nan"))                            # the replay must overwrite every buffer
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(c[1], a[1]) and torch.equal(c[2], a[2]) and torch.equal(fc, fa)
    assert _grad_value_close(c[0], a[0], dtype, scale)


@pytest.fixture
def dispatch_spy(monkeypatch):
    """records which Function MSDeformAttn.forward applied ("fused" / "composed")"""
    from odise_b200 import msda
    calls = []

    def spy(fn, tag):
        class Spy:
            @staticmethod
            def apply(*a):
                calls.append(tag)
                return fn.apply(*a)
        return Spy
    monkeypatch.setattr(msda, "MSDeformAttnFusedFunction", spy(msda.MSDeformAttnFusedFunction, "fused"))
    monkeypatch.setattr(msda, "MSDeformAttnFunction", spy(msda.MSDeformAttnFunction, "composed"))
    return calls


MODULE_CASES = {
    # D = 32: both paths, with a padding mask and reference points that require grad
    "d32_padding_refgrad": (dict(seed=51, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4,
                                 padding=True), True, ("fused", "composed")),
    # the ODISE pixel decoder's configuration (d_model 256, 8 heads, 3 levels, 4 points)
    "odise": (dict(seed=52, N=1, d_model=256, n_heads=8, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4), False,
              ("fused", "composed")),
    # D = 64 (d_model 256, 4 heads) and 4-column box reference points: the composed path whatever use_fused says
    "d64_padding": (dict(seed=53, N=1, d_model=256, n_heads=4, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4,
                         padding=True), False, ("composed", "composed")),
    "box_refgrad": (dict(seed=54, N=2, d_model=64, n_heads=2, shapes=[(4, 4), (8, 8)], n_points=3, box=True), True,
                    ("composed", "composed")),
}
# Bar against the fp64 module oracle, which runs at the module's 16-bit-rounded parameters and inputs (so input rounding
# is not counted).  What the module still rounds to 16 bits is, on any path from an input to a result, at most four
# tensors in sequence: forward value / logits (the offsets are exactly the 16-bit bias), the sampled output and the
# output projection; backward the incoming gradient of a Linear, the sampled output's gradient, the value / offset /
# logit gradients and the Linear's own result.  Each rounding is at most u relative to that tensor's largest element, and
# each stage after it passes an error on with a gain of at most 2 (a convex combination for the sampling, a Linear whose
# C^-0.5-scaled weights have spectral norm about 2, two rounded factors in a weight gradient).  Four roundings with two
# later gain-2 stages at most: 4 * 4 u = 16 u of max(1, max |ref|).
ORACLE_BAR_U = 16
# The two dispatch paths share every op except the sampling, which both compute in fp32 from the same 16-bit inputs and
# round once: they can differ by a 16-bit ulp where the fp32 results straddle a rounding boundary, in the sampled output,
# its three gradients and the results they feed: 4 u of max(1, max |ref|).
PATHS_BAR_U = 4


def _module_run(dev, cfg, pr, dtype, mode, use_fused, ref_grad):
    """one forward + backward of MSDeformAttn: mode "autocast" = float32 module under torch.autocast("cuda", dtype),
    "cast" = module and inputs cast to dtype -> (output, {name: gradient})"""
    from odise_b200.msda import MSDeformAttn
    m = MSDeformAttn(cfg["d_model"], len(cfg["shapes"]), cfg["n_heads"], cfg["n_points"]).to(dev)
    m.load_state_dict(pr["params"])
    in_dtype = torch.float32
    if mode == "cast":
        m, in_dtype = m.to(dtype), dtype
    m.use_fused = use_fused
    q, x = (pr[k].to(dev, in_dtype).requires_grad_(True) for k in ("query", "input_flatten"))
    ref = pr["reference_points"].to(dev).requires_grad_(ref_grad)
    mask = None if pr["padding_mask"] is None else pr["padding_mask"].to(dev)
    ctx = torch.autocast("cuda", dtype=dtype) if mode == "autocast" else contextlib.nullcontext()
    with ctx:
        out = m(q, ref, x, pr["spatial_shapes"].to(dev), pr["level_start_index"].to(dev), mask)
    assert out.dtype == dtype
    out.backward(pr["grad_output"].to(dev, dtype))
    grads = {k: p.grad for k, p in m.named_parameters()}
    grads.update(query=q.grad, input_flatten=x.grad)
    if ref_grad:
        grads["reference_points"] = ref.grad
    else:
        assert ref.grad is None
    for k, g in grads.items():
        assert g is not None and torch.isfinite(g).all(), k
    return out, grads


@pytest.mark.parametrize("mode", ["autocast", "cast"])
@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
@pytest.mark.parametrize("name", sorted(MODULE_CASES))
def test_module_16bit_both_paths(cuda, name, dtype, mode, dispatch_spy):
    """Forward + backward of MSDeformAttn with 16-bit activations: use_fused = True and False take the paths named in
    MODULE_CASES, return the value's dtype, agree with each other to PATHS_BAR_U u and with the fp64 module oracle to
    ORACLE_BAR_U u (derivations beside the constants)."""
    from oracle.msda_16bit import MARGIN, round_module_problem
    from oracle.msda_module import module_problem, oracle_module_grads, sample_margin
    cfg, ref_grad, paths = MODULE_CASES[name]
    pr = round_module_problem(module_problem(**cfg), cfg["n_points"], dtype)
    assert sample_margin(pr["params"], pr["query"], pr["reference_points"], pr["spatial_shapes"], cfg["n_heads"],
                         cfg["n_points"]) >= MARGIN
    want_out, want = oracle_module_grads(pr["params"], pr["query"], pr["reference_points"], pr["input_flatten"],
                                         pr["spatial_shapes"], pr["level_start_index"], pr["padding_mask"],
                                         pr["grad_output"], cfg["n_heads"], cfg["n_points"], ref_grad=ref_grad)
    want["output"] = want_out
    runs = []
    for use_fused in (True, False):
        dispatch_spy.clear()
        out, grads = _module_run(cuda, cfg, pr, dtype, mode, use_fused, ref_grad)
        assert dispatch_spy == [paths[0] if use_fused else "composed"]
        grads["output"] = out
        assert sorted(grads) == sorted(want)
        runs.append(grads)
    u = U[dtype]
    for k in sorted(want):
        scale = max(1.0, want[k].abs().max().item())
        for tag, got in zip(("use_fused", "composed"), runs):
            err = (got[k].detach().cpu().double() - want[k]).abs().max().item()
            assert err <= ORACLE_BAR_U * u * scale, (k, tag, err / (u * scale))
        err = (runs[0][k].detach().double() - runs[1][k].detach().double()).abs().max().item()
        assert err <= PATHS_BAR_U * u * scale, (k, "paths", err / (u * scale))


def _stack_run(dev, dtype, use_fused, steps, lr):
    """SGD on a 2-layer float32 stack x <- x + MSDeformAttn(x, ref, x) (D = 32) under torch.autocast("cuda", dtype);
    float16 scales the loss with torch.amp.GradScaler -> losses.  Every gradient is checked finite at every step."""
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_16bit import round_module_problem
    from oracle.msda_module import module_problem
    cfg = dict(N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4)
    prs = [round_module_problem(module_problem(seed=60 + i, **cfg), 4, dtype) for i in range(2)]
    layers = []
    for pr in prs:
        m = MSDeformAttn(64, 3, 2, 4).to(dev)
        m.load_state_dict(pr["params"])
        m.use_fused = use_fused
        layers.append(m)
    pr = prs[0]
    ss, lsi, ref = pr["spatial_shapes"].to(dev), pr["level_start_index"].to(dev), pr["reference_points"].to(dev)
    x0 = pr["input_flatten"].to(dev, torch.float32)
    target = torch.randn(x0.shape, generator=torch.Generator().manual_seed(5)).to(dev)
    params = [p for m in layers for p in m.parameters()]
    opt = torch.optim.SGD(params, lr=lr)
    # a fixed, moderate scale: the loss is O(1), so 2^8 neither overflows float16 gradients nor skips a step
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 8) if dtype == torch.float16 else None
    losses = []
    for _ in range(steps):
        with torch.autocast("cuda", dtype=dtype):
            x = x0
            for m in layers:
                x = x + m(x, ref, x, ss, lsi)
            loss = ((x.float() - target) ** 2).mean()
        opt.zero_grad()
        if scaler is not None:
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
        else:
            loss.backward()
        for p in params:
            assert p.grad is not None and torch.isfinite(p.grad).all()
        if scaler is not None:
            scaler.step(opt)
            scaler.update()
            assert scaler.get_scale() == 2.0 ** 8          # no step was skipped
        else:
            opt.step()
        losses.append(loss.item())
    return losses


@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
def test_mixed_precision_training_run_fused_vs_composed(cuda, dtype, dispatch_spy):
    """Four SGD steps of a 2-layer stack under autocast (float16 with a GradScaler, bfloat16 without): the fused and the
    composed path give the same loss trajectory to PATHS_BAR_U u, the loss goes down and every gradient is finite.  The
    loss is a continuous function of the sample positions (bilinear weights vanish at the level's border), so a sample
    that lands on a cell edge after a step changes the gradient, not the loss."""
    fused = _stack_run(cuda, dtype, True, 4, 0.1)
    assert set(dispatch_spy) == {"fused"}
    dispatch_spy.clear()
    composed = _stack_run(cuda, dtype, False, 4, 0.1)
    assert set(dispatch_spy) == {"composed"}
    assert fused[-1] < fused[0]
    for a, b in zip(fused, composed):
        assert abs(a - b) <= PATHS_BAR_U * U[dtype] * max(1.0, abs(b)), (fused, composed)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dt)
def test_16bit_errors(cuda, dtype):
    from odise_b200 import lib
    from oracle.msda_16bit import fused_problem_16bit
    args = _on(cuda, fused_problem_16bit(seed=3, N=2, M=2, D=32, shapes=[(6, 4)], Lq=3, P=2, dtype=dtype))
    value, ss, lsi, ref, offs, logits, go = args
    other = torch.bfloat16 if dtype == torch.float16 else torch.float16
    fwd, bwd = lib.msda_fused_forward_16bit, lib.msda_fused_backward_16bit
    with pytest.raises(RuntimeError):                   # CPU tensors
        bwd(*[t.cpu() for t in args])
    with pytest.raises(RuntimeError):
        fwd(value.cpu(), ss, lsi, ref, offs, logits)
    with pytest.raises(RuntimeError):                   # non-contiguous
        bwd(value, ss, lsi, ref, offs, logits, go.transpose(0, 1).contiguous().transpose(0, 1))
    with pytest.raises(RuntimeError):
        fwd(value, ss, lsi, ref.transpose(0, 1).contiguous().transpose(0, 1), offs, logits)
    with pytest.raises(RuntimeError):                   # float32 value: the float32 functions' case
        fwd(value.float(), ss, lsi, ref, offs.float(), logits.float())
    with pytest.raises(RuntimeError):
        bwd(value.float(), ss, lsi, ref, offs.float(), logits.float(), go.float())
    with pytest.raises(RuntimeError):                   # offsets / logits / grad_output not in the value's dtype
        fwd(value, ss, lsi, ref, offs.to(other), logits)
    with pytest.raises(RuntimeError):
        fwd(value, ss, lsi, ref, offs, logits.float())
    with pytest.raises(RuntimeError):
        bwd(value, ss, lsi, ref, offs, logits, go.float())
    with pytest.raises(RuntimeError):                   # reference points not float32
        fwd(value, ss, lsi, ref.to(dtype), offs, logits)
    with pytest.raises(RuntimeError):                   # shapes that disagree
        bwd(value, ss, lsi, ref, offs, logits[..., :1].contiguous(), go)
    with pytest.raises(RuntimeError):
        fwd(value, ss, lsi, ref[:, :2].contiguous(), offs, logits)
    for bad in (dict(seed=3, N=1, M=2, D=64, shapes=[(6, 4)], Lq=3, P=2),         # D = 64
                dict(seed=3, N=1, M=2, D=32, shapes=[(3, 3)] * 4, Lq=3, P=9)):    # L * P = 36 > 32
        b = _on(cuda, fused_problem_16bit(**bad, dtype=dtype))
        with pytest.raises(RuntimeError):
            fwd(*b[:6])
        with pytest.raises(RuntimeError):
            bwd(*b)
    # the float32 functions keep refusing 16-bit tensors
    with pytest.raises(RuntimeError):
        lib.msda_fused_forward(value, ss, lsi, ref, offs, logits)
    with pytest.raises(RuntimeError):
        lib.msda_fused_backward(value, ss, lsi, ref, offs, logits, go)
