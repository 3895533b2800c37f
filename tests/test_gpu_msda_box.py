"""GPU checks of MSDeformAttn with box reference points (cx, cy, w, h) on the fused kernels (odise_msda_fused_box_*):
float32 forward and backward against the fp64 oracle (tests/msda_box_oracle.py), degenerate and far-outside boxes, the
fused output against the composed op on torch-computed locations, 16-bit storage, deterministic mode, the module's
dispatch and training steps, and torch.compile / torch.export.  Bars are the 2-column tests' for the same quantity:
1e-5 x max(1, max |ref|) in float32 (tests/test_gpu_msda_module.py), u |ref| + 1e-5 max(1, max |ref|) in 16 bits
(tests/test_gpu_msda_16bit.py, u the unit roundoff), ORACLE_BAR_U / PATHS_BAR_U for 16-bit modules (derived there)."""
import contextlib
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# shapes of tests/test_gpu_msda_module.py::FUSED_CASES
CASES = [
    dict(seed=8, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64), (128, 128)], Lq=300, P=4),    # C4: L = 4
    dict(seed=9, N=1, M=8, D=32, shapes=[(9, 7), (5, 3)], Lq=37, P=3),           # L*P = 6: ragged sub-warp, tail block
    dict(seed=10, N=2, M=5, D=32, shapes=[(4, 4)] * 8, Lq=19, P=4),              # L*P = 32: the largest D = 32 block
    dict(seed=11, N=2, M=8, D=32, shapes=[(5, 7), (3, 2)], Lq=23, P=4, far=True),  # far outside: all grads exactly 0
]
DTYPES16 = [torch.float16, torch.bfloat16]
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
DT = {torch.float32: "f32", torch.float16: "f16", torch.bfloat16: "bf16"}
ORACLE_BAR_U, PATHS_BAR_U = 16, 4
NAMES = ("grad_value", "grad_offsets", "grad_logits")


def _id(cfg):
    return f"L{len(cfg['shapes'])}-P{cfg['P']}-Lq{cfg['Lq']}" + ("-far" if cfg.get("far") else "")


def _on(dev, tensors):
    return [t.to(dev) for t in tensors]


def _close(got, want, tol=1e-5):
    scale = max(1.0, want.abs().max().item())
    err = (got.detach().cpu().double() - want.detach().cpu().double()).abs().max().item()
    return err < tol * scale, err, scale


def _within(got, want, u):
    g, w = got.detach().cpu().double(), want.double()
    bar = u * w.abs() + 1e-5 * max(1.0, w.abs().max().item())
    ratio = ((g - w).abs() / bar).max().item()
    return ratio <= 1.0, ratio


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8),
                                                                     b.contiguous().view(torch.uint8))


def _problem(cfg, dtype):
    from msda_box_oracle import fused_problem_box, fused_problem_box_16bit
    if dtype in U:
        return fused_problem_box_16bit(**cfg, dtype=dtype)
    return fused_problem_box(**cfg, dtype=torch.float32)


def _fwd(args):
    from odise_b200 import lib
    fn = lib.msda_fused_forward_16bit if args[0].dtype in U else lib.msda_fused_forward
    return fn(*args[:6])


def _bwd(args, deterministic=False):
    from odise_b200 import lib
    fn = lib.msda_fused_backward_16bit if args[0].dtype in U else lib.msda_fused_backward
    return fn(*args[:7], deterministic=deterministic)


def _check_degenerate_and_far(cfg, ref, out, grads):
    """grad_offsets along a zero box side is exactly 0; far outside, every output is exactly 0"""
    go = grads[1].detach().cpu()
    flat = (ref.cpu()[:, :, None, :, None, 2:] == 0).expand_as(go)
    assert flat.any() and go[flat].abs().max().item() == 0
    if cfg.get("far"):
        assert out.abs().max().item() == 0
        for name, g in zip(NAMES, grads):
            assert g.abs().max().item() == 0, name


# ---- the entry points ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cfg", CASES, ids=_id)
def test_box_f32_vs_fp64_oracle(cuda, cfg, record):
    """the oracle runs at the float32 box locations the kernel samples at (fp32_locations): a box location is rounded in
    the product with w and the sum with the centre, and for a P that is not a power of two in 1/P and the product with
    it, where the 2-column location at power-of-two level sizes is rounded in its sum only.  test_box_fused_vs_composed_op
    checks that arithmetic against the composed path's torch ops"""
    from msda_box_oracle import oracle_fused_forward, oracle_fused_grads
    prob = _problem(cfg, torch.float32)
    want_out = oracle_fused_forward(*prob[:6], fp32_locations=True)
    want = oracle_fused_grads(*prob, fp32_locations=True)
    args = _on(cuda, prob)
    out = _fwd(args)
    got = _bwd(args)
    torch.cuda.synchronize()
    ok, err, scale = _close(out, want_out)
    assert out.dtype == torch.float32 and ok, ("out", err, scale)
    rel = [f"out {err / scale:.2e}"]
    for name, g, w in zip(NAMES, got, want):
        assert g.shape == w.shape and g.dtype == torch.float32
        ok, err, scale = _close(g, w)
        assert ok, (name, err, scale)
        rel.append(f"{name} {err / scale:.2e}")
    _check_degenerate_and_far(cfg, args[3], out, got)
    record(f"msda fused box f32 vs fp64 oracle {_id(cfg)}: max err / max(1, |ref|): " + " ".join(rel))


@pytest.mark.parametrize("cfg", CASES[:3], ids=_id)
def test_box_fused_vs_composed_op(cuda, cfg):
    """the fused box forward against lib.msda_forward on the locations and softmax weights computed by the composed
    path's torch ops (MSDeformAttn.forward), on the device in float32.  P = 3 included: torch computes `offsets / P` on
    the GPU as the product with the float32 reciprocal of P, and so does the kernel"""
    from odise_b200 import lib
    value, ss, lsi, ref, offs, logits, _ = _on(cuda, _problem(cfg, torch.float32))
    N, Lq, M, L, P, _ = offs.shape
    loc = ref[:, :, None, :, None, :2] + offs / P * ref[:, :, None, :, None, 2:] * 0.5
    aw = torch.softmax(logits, -1).view(N, Lq, M, L, P)
    want = lib.msda_forward(value, ss, lsi, loc.contiguous(), aw.contiguous())
    got = lib.msda_fused_forward(value, ss, lsi, ref, offs, logits)
    err = (got - want).abs().max().item()
    assert err <= 1e-6 * max(1.0, want.abs().max().item()), err


@pytest.mark.parametrize("dtype", DTYPES16, ids=DT.get)
@pytest.mark.parametrize("cfg", CASES, ids=_id)
def test_box_16bit_vs_fp64_oracle_and_f32_kernels(cuda, cfg, dtype, record):
    """within the 16-bit bars of the fp64 oracle; out, grad_offsets and grad_logits equal the float32 box kernels'
    results on the upcast inputs, rounded, bit for bit"""
    from msda_box_oracle import oracle_fused_forward, oracle_fused_grads
    prob = _problem(cfg, dtype)
    want_out = oracle_fused_forward(*prob[:6])
    want = oracle_fused_grads(*prob)
    args = _on(cuda, prob)
    out = _fwd(args)
    got = _bwd(args)
    up = [t.float() if t.dtype == dtype else t for t in args]
    o32, g32 = _fwd(up), _bwd(up)
    torch.cuda.synchronize()
    ok, r = _within(out, want_out, U[dtype])
    assert out.dtype == dtype and ok, ("out", r)
    ratios = [f"out {r:.2f}"]
    for name, g, w in zip(NAMES, got, want):
        assert g.shape == w.shape and g.dtype == dtype, name
        ok, r = _within(g, w, U[dtype])
        assert ok, (name, r)
        ratios.append(f"{name} {r:.2f}")
    _check_degenerate_and_far(cfg, args[3], out, got)
    assert torch.equal(out, o32.to(dtype))
    assert torch.equal(got[1], g32[1].to(dtype)) and torch.equal(got[2], g32[2].to(dtype))
    record(f"msda fused box {DT[dtype]} vs fp64 oracle {_id(cfg)}: max err / bar: " + " ".join(ratios))


# ---- deterministic mode --------------------------------------------------------------------------------------------------

DET_DTYPES = [torch.float32, torch.float16, torch.bfloat16]


@pytest.mark.parametrize("dtype", DET_DTYPES, ids=DT.get)
@pytest.mark.parametrize("cfg", CASES, ids=_id)
def test_box_deterministic_vs_oracle_and_default(cuda, cfg, dtype):
    """grad_value within the default path's bars of the fp64 oracle; grad_offsets and grad_logits bit-equal to the
    default path's"""
    from msda_box_oracle import oracle_fused_grads
    prob = _problem(cfg, dtype)
    want = oracle_fused_grads(*prob, fp32_locations=dtype == torch.float32)
    args = _on(cuda, prob)
    det, dflt = _bwd(args, True), _bwd(args, False)
    torch.cuda.synchronize()
    assert det[0].dtype == dtype
    if dtype == torch.float32:
        ok, err, scale = _close(det[0], want[0])
        assert ok, (err, scale)
    else:
        ok, r = _within(det[0], want[0], U[dtype])
        assert ok, r
    assert _bits_equal(det[1], dflt[1]) and _bits_equal(det[2], dflt[2])


@pytest.mark.parametrize("dtype", DET_DTYPES, ids=DT.get)
def test_box_deterministic_order_independence(cuda, dtype):
    """deterministic grad_value bit-identical across repeated calls, a CUDA-graph replay, a permutation of the queries
    and a batch split"""
    args = _on(cuda, _problem(CASES[2], dtype))
    a, b = _bwd(args, True), _bwd(args, True)
    torch.cuda.synchronize()
    assert all(_bits_equal(x, y) for x, y in zip(a, b))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _bwd(args, True)                                 # warm-up on the side stream before capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = _bwd(args, True)
    for t in c:
        t.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert all(_bits_equal(x, y) for x, y in zip(a, c))
    perm = torch.randperm(args[3].shape[1], generator=torch.Generator().manual_seed(7)).to(cuda)
    pargs = [t.index_select(1, perm).contiguous() if i in (3, 4, 5, 6) else t for i, t in enumerate(args)]
    p = _bwd(pargs, True)
    assert _bits_equal(a[0], p[0])
    assert _bits_equal(a[1].index_select(1, perm), p[1]) and _bits_equal(a[2].index_select(1, perm), p[2])
    assert args[0].shape[0] == 2
    for n in range(2):
        one = _bwd([t[n:n + 1].contiguous() if i in (0, 3, 4, 5, 6) else t for i, t in enumerate(args)], True)
        torch.cuda.synchronize()
        assert all(_bits_equal(x[n:n + 1], y) for x, y in zip(a, one)), n


_TRAIN_SCRIPT = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from odise_b200 import lib
from odise_b200.msda import MSDeformAttn
from oracle.msda_module import module_problem

torch.use_deterministic_algorithms(True)
dev = torch.device("cuda:0")
CFG = dict(seed=74, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4, box=True)


def train(amp):
    pr = module_problem(**CFG, dtype=torch.float32)
    m = MSDeformAttn(64, 3, 2, 4).to(dev)
    m.load_state_dict(pr["params"])
    q, ref, x = (pr[k].to(dev) for k in ("query", "reference_points", "input_flatten"))
    ss, lsi = pr["spatial_shapes"].to(dev), pr["level_start_index"].to(dev)
    target = torch.randn(q.shape, generator=torch.Generator().manual_seed(5)).to(dev)
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    for _ in range(4):
        with torch.autocast("cuda", dtype=amp, enabled=amp is not None):
            out = m(q, ref, x, ss, lsi)
            loss = ((out.float() - target) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    return [p.detach().clone() for p in m.parameters()]


seen = []
for name in ("msda_backward", "msda_fused_backward", "msda_fused_backward_16bit"):
    def wrap(fn, name=name):
        def spy(*a, **kw):
            seen.append((name, kw.get("deterministic", False), a[3].shape[-1]))
            return fn(*a, **kw)
        return spy
    setattr(lib, name, wrap(getattr(lib, name)))
res = {}
for name, amp in (("fused_f32", None), ("fused_bf16_autocast", torch.bfloat16)):
    seen.clear()
    a, b = train(amp), train(amp)
    res[name] = dict(identical=all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(a, b)),
                     calls=sorted(set(seen)))
print("RESULT " + json.dumps(res))
"""


def test_box_module_training_is_bit_reproducible(cuda):
    """two 4-step SGD runs of MSDeformAttn with box reference points (no gradient) under
    torch.use_deterministic_algorithms(True) and CUBLAS_WORKSPACE_CONFIG=:4096:8 (set before CUDA starts, hence the
    subprocess) end with bit-identical parameters, in float32 and under bfloat16 autocast, on the fused box kernels"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _TRAIN_SCRIPT, ROOT]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])
    want = {"fused_f32": [["msda_fused_backward", True, 4]],
            "fused_bf16_autocast": [["msda_fused_backward_16bit", True, 4]]}
    assert sorted(res) == sorted(want)
    for name, v in res.items():
        assert v["calls"] == want[name], (name, v)
        assert v["identical"], name


# ---- the module ----------------------------------------------------------------------------------------------------------

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
    "box_small": dict(seed=54, N=2, d_model=64, n_heads=2, shapes=[(4, 4), (8, 8)], n_points=3, box=True),
    "box_padding": dict(seed=55, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4, box=True,
                        padding=True),
    "box_odise": dict(seed=56, N=1, d_model=256, n_heads=8, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4, box=True),
}


def _module(dev, cfg, params):
    from odise_b200.msda import MSDeformAttn
    m = MSDeformAttn(cfg["d_model"], len(cfg["shapes"]), cfg["n_heads"], cfg["n_points"]).to(dev)
    m.load_state_dict(params)
    return m


@pytest.mark.parametrize("name", sorted(MODULE_CASES))
def test_box_module_fp32_vs_fp64_oracle(cuda, name, dispatch_spy):
    """boxes that do not require grad take the fused path; the output and every parameter and input gradient match the
    fp64 module oracle at 1e-5 x max(1, max |ref|)"""
    from oracle.msda_module import module_problem, oracle_module_grads, sample_margin
    cfg = MODULE_CASES[name]
    pr = module_problem(**cfg, dtype=torch.float32)
    assert sample_margin(pr["params"], pr["query"], pr["reference_points"], pr["spatial_shapes"], cfg["n_heads"],
                         cfg["n_points"]) >= 0.02
    want_out, want = oracle_module_grads(pr["params"], pr["query"], pr["reference_points"], pr["input_flatten"],
                                         pr["spatial_shapes"], pr["level_start_index"], pr["padding_mask"],
                                         pr["grad_output"], cfg["n_heads"], cfg["n_points"])
    m = _module(cuda, cfg, pr["params"])
    q, x = (pr[k].to(cuda).requires_grad_(True) for k in ("query", "input_flatten"))
    ref = pr["reference_points"].to(cuda)
    mask = None if pr["padding_mask"] is None else pr["padding_mask"].to(cuda)
    out = m(q, ref, x, pr["spatial_shapes"].to(cuda), pr["level_start_index"].to(cuda), mask)
    out.backward(pr["grad_output"].to(cuda))
    assert dispatch_spy == ["fused"]
    got = {k: p.grad for k, p in m.named_parameters()}
    got.update(query=q.grad, input_flatten=x.grad)
    assert sorted(got) == sorted(want)
    for k in ["output"] + sorted(want):
        ok, err, scale = _close(out if k == "output" else got[k], want_out if k == "output" else want[k])
        assert ok, (k, err, scale)


@pytest.mark.parametrize("mode", ["autocast", "cast"])
@pytest.mark.parametrize("dtype", DTYPES16, ids=DT.get)
@pytest.mark.parametrize("name", ["box_small", "box_padding"])
def test_box_module_16bit(cuda, name, dtype, mode, dispatch_spy):
    """under autocast and in a module cast to 16 bits, boxes take the fused path; both paths match the fp64 module
    oracle to ORACLE_BAR_U u and each other to PATHS_BAR_U u"""
    from oracle.msda_16bit import MARGIN, round_module_problem
    from oracle.msda_module import module_problem, oracle_module_grads, sample_margin
    cfg = MODULE_CASES[name]
    pr = round_module_problem(module_problem(**cfg), cfg["n_points"], dtype)
    assert sample_margin(pr["params"], pr["query"], pr["reference_points"], pr["spatial_shapes"], cfg["n_heads"],
                         cfg["n_points"]) >= MARGIN
    want_out, want = oracle_module_grads(pr["params"], pr["query"], pr["reference_points"], pr["input_flatten"],
                                         pr["spatial_shapes"], pr["level_start_index"], pr["padding_mask"],
                                         pr["grad_output"], cfg["n_heads"], cfg["n_points"])
    want["output"] = want_out
    runs = []
    for use_fused in (True, False):
        dispatch_spy.clear()
        m = _module(cuda, cfg, pr["params"])
        in_dtype = torch.float32
        if mode == "cast":
            m, in_dtype = m.to(dtype), dtype
        m.use_fused = use_fused
        q, x = (pr[k].to(cuda, in_dtype).requires_grad_(True) for k in ("query", "input_flatten"))
        mask = None if pr["padding_mask"] is None else pr["padding_mask"].to(cuda)
        ctx = torch.autocast("cuda", dtype=dtype) if mode == "autocast" else contextlib.nullcontext()
        with ctx:
            out = m(q, pr["reference_points"].to(cuda), x, pr["spatial_shapes"].to(cuda),
                    pr["level_start_index"].to(cuda), mask)
        assert out.dtype == dtype
        out.backward(pr["grad_output"].to(cuda, dtype))
        assert dispatch_spy == ["fused" if use_fused else "composed"]
        grads = {k: p.grad for k, p in m.named_parameters()}
        grads.update(query=q.grad, input_flatten=x.grad, output=out)
        runs.append(grads)
    u = U[dtype]
    for k in sorted(want):
        scale = max(1.0, want[k].abs().max().item())
        for tag, got in zip(("fused", "composed"), runs):
            err = (got[k].detach().cpu().double() - want[k]).abs().max().item()
            assert err <= ORACLE_BAR_U * u * scale, (k, tag, err / (u * scale))
        err = (runs[0][k].detach().double() - runs[1][k].detach().double()).abs().max().item()
        assert err <= PATHS_BAR_U * u * scale, (k, "paths", err / (u * scale))


def test_box_requiring_grad_dispatch(cuda, dispatch_spy):
    """a box that requires grad takes the composed path (and gets its gradient), except under torch.no_grad, where the
    fused path gives the same output to 1e-5; MSDeformAttnFusedFunction raises for it"""
    from odise_b200.msda import MSDeformAttnFusedFunction
    from oracle.msda_module import module_problem
    cfg = MODULE_CASES["box_small"]
    pr = module_problem(**cfg, dtype=torch.float32)
    m = _module(cuda, cfg, pr["params"])
    q, x, ss, lsi = (pr[k].to(cuda) for k in ("query", "input_flatten", "spatial_shapes", "level_start_index"))
    ref = pr["reference_points"].to(cuda).requires_grad_(True)
    out = m(q, ref, x, ss, lsi)
    out.sum().backward()
    assert dispatch_spy == ["composed"] and ref.grad is not None
    dispatch_spy.clear()
    with torch.no_grad():
        fused = m(q, ref, x, ss, lsi)
    assert dispatch_spy == ["fused"]
    ok, err, scale = _close(fused, out)
    assert ok, (err, scale)
    from msda_box_oracle import fused_problem_box
    value, ss2, lsi2, ref2, offs, logits, _ = _on(cuda, fused_problem_box(**CASES[1], dtype=torch.float32))
    with pytest.raises(RuntimeError):
        MSDeformAttnFusedFunction.apply(value, ss2, lsi2, ref2.requires_grad_(True), offs, logits)


def test_box_misaligned_view(cuda, dispatch_spy):
    """a box view whose storage offset is not a multiple of 4 floats: lib refuses it before any launch, the module copies
    it and gives the bits of the aligned tensor on the fused path"""
    from odise_b200 import lib
    from oracle.msda_module import module_problem
    value, ss, lsi, ref, offs, logits, go = _on(cuda, _problem(CASES[1], torch.float32))
    shifted = torch.empty(ref.numel() + 2, device=cuda)[2:].view(ref.shape).copy_(ref)
    with pytest.raises(RuntimeError, match="16 bytes"):
        lib.msda_fused_forward(value, ss, lsi, shifted, offs, logits)
    with pytest.raises(RuntimeError, match="16 bytes"):
        lib.msda_fused_backward(value, ss, lsi, shifted, offs, logits, go)
    cfg = MODULE_CASES["box_small"]
    pr = module_problem(**cfg, dtype=torch.float32)
    m = _module(cuda, cfg, pr["params"])
    q, x, ss, lsi, r = (pr[k].to(cuda) for k in ("query", "input_flatten", "spatial_shapes", "level_start_index",
                                                 "reference_points"))
    rv = torch.empty(r.numel() + 2, device=cuda)[2:].view(r.shape).copy_(r)
    with torch.no_grad():
        want, got = m(q, r, x, ss, lsi), m(q, rv, x, ss, lsi)
    assert dispatch_spy == ["fused", "fused"]
    assert torch.equal(got, want)


def _stack_run(dev, use_fused, amp, steps=4, lr=0.1):
    """SGD on a 2-layer stack x <- x + MSDeformAttn(x, boxes, x) with detached boxes, float32 or under autocast (float16
    with a GradScaler) -> (losses, smallest sample margin, or None under autocast)"""
    from oracle.msda_16bit import round_module_problem
    from oracle.msda_module import module_problem, sample_margin
    cfg = dict(N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4, box=True)
    prs = [module_problem(seed=80 + i, **cfg, dtype=torch.float32) for i in range(2)]
    if amp is not None:
        prs = [round_module_problem(module_problem(seed=80 + i, **cfg), 4, amp) for i in range(2)]
    layers = []
    for pr in prs:
        m = _module(dev, cfg, pr["params"])
        m.use_fused = use_fused
        layers.append(m)
    pr = prs[0]
    ss, lsi, ref = pr["spatial_shapes"].to(dev), pr["level_start_index"].to(dev), pr["reference_points"].to(dev)
    x0 = pr["input_flatten"].to(dev, torch.float32)
    target = torch.randn(x0.shape, generator=torch.Generator().manual_seed(5)).to(dev)
    params = [p for m in layers for p in m.parameters()]
    opt = torch.optim.SGD(params, lr=lr)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 8) if amp == torch.float16 else None
    losses, margin = [], float("inf")
    for _ in range(steps):
        with torch.autocast("cuda", dtype=amp or torch.float16, enabled=amp is not None):
            x = x0
            for m in layers:
                if amp is None:
                    margin = min(margin, sample_margin(m.state_dict(), x.detach(), ref, ss, 2, 4))
                x = x + m(x, ref, x, ss, lsi)
            loss = ((x.float() - target) ** 2).mean()
        opt.zero_grad()
        if scaler is not None:
            scaler.scale(loss).backward()
            scaler.step(opt)
            scaler.update()
            assert scaler.get_scale() == 2.0 ** 8          # no step was skipped
        else:
            loss.backward()
            opt.step()
        losses.append(loss.item())
    return losses, margin


@pytest.mark.parametrize("amp", [None, torch.float16], ids=["f32", "f16_autocast"])
def test_box_training_run_fused_vs_composed(cuda, amp, dispatch_spy):
    """four SGD steps of a 2-layer stack with detached boxes: the same losses on the fused and the composed path (1e-5 in
    float32, every sample 0.02 px from a cell edge at every step; PATHS_BAR_U u under float16 autocast)"""
    fused, m_fused = _stack_run(cuda, True, amp)
    assert set(dispatch_spy) == {"fused"}
    dispatch_spy.clear()
    composed, m_composed = _stack_run(cuda, False, amp)
    assert set(dispatch_spy) == {"composed"}
    assert fused[-1] < fused[0]
    tol = 1e-5 if amp is None else PATHS_BAR_U * U[amp]
    if amp is None:
        assert min(m_fused, m_composed) >= 0.02, (m_fused, m_composed)
    for a, b in zip(fused, composed):
        assert abs(a - b) <= tol * max(1.0, abs(b)), (fused, composed)


# ---- torch.compile / torch.export ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("dtype", DET_DTYPES, ids=DT.get)
def test_box_opcheck(cuda, dtype, det):
    """schema and fake implementation of both fused ops with box arguments; AOT dispatch with dynamic shapes for the
    forward, and for the backward with deterministic=True (float atomics make the default grad_value's bits vary)"""
    import odise_b200.msda  # noqa: F401
    ops = torch.ops.odise_b200
    args = _on(cuda, _problem(CASES[1], dtype))
    every = ("test_schema", "test_faketensor", "test_aot_dispatch_dynamic")
    torch.library.opcheck(ops.msda_fused_forward.default, tuple(args[:6]), test_utils=every)
    torch.library.opcheck(ops.msda_fused_backward.default, (*args, det),
                          test_utils=every if det else ("test_schema", "test_faketensor"))


def _op_names(gms):
    found = set()
    for gm in gms:
        for mod in gm.modules():
            if isinstance(mod, torch.fx.GraphModule):
                found |= {str(n.target).removesuffix(".default") for n in mod.graph.nodes
                          if n.op == "call_function" and str(n.target).startswith("odise_b200.")}
    return found


def test_box_module_compile_fullgraph_same_bits(cuda):
    """torch.compile(MSDeformAttn, fullgraph=True) (aot_eager) with box reference points: the graph holds the fused ops
    and the output and gradients equal eager's bit for bit (deterministic mode, so that grad_value is reproducible)"""
    from oracle.msda_module import module_problem
    torch._dynamo.reset()
    cfg = MODULE_CASES["box_padding"]
    pr = module_problem(**cfg, dtype=torch.float32)
    m = _module(cuda, cfg, pr["params"])
    graphs = []
    backend = torch._dynamo.lookup_backend("aot_eager")

    def rec(gm, example_inputs):
        graphs.append(gm)
        return backend(gm, example_inputs)

    def run(f):
        m.zero_grad()
        q, x = (pr[k].to(cuda).requires_grad_(True) for k in ("query", "input_flatten"))
        out = f(q, pr["reference_points"].to(cuda), x, pr["spatial_shapes"].to(cuda), pr["level_start_index"].to(cuda),
                pr["padding_mask"].to(cuda))
        out.backward(pr["grad_output"].to(cuda))
        return [out.detach(), q.grad, x.grad] + [p.grad.clone() for p in m.parameters()]

    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        eager = run(m)
        compiled = run(torch.compile(m, fullgraph=True, backend=rec))
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
        torch._dynamo.reset()
    assert _op_names(graphs) == {"odise_b200.msda_fused_forward", "odise_b200.msda_fused_backward"}
    for i, (c, e) in enumerate(zip(compiled, eager)):
        assert _bits_equal(c, e), i


def test_box_export_forward(cuda):
    """torch.export.export of an eval-mode MSDeformAttn with box reference points holds the fused forward op, and the
    exported program's output equals eager's"""
    from oracle.msda_module import module_problem
    cfg = MODULE_CASES["box_odise"]
    pr = module_problem(**cfg, dtype=torch.float32)
    m = _module(cuda, cfg, pr["params"]).eval()
    args = tuple(pr[k].to(cuda) for k in ("query", "reference_points", "input_flatten", "spatial_shapes",
                                           "level_start_index"))
    ep = torch.export.export(m, args)
    targets = {str(n.target).removesuffix(".default") for n in ep.graph.nodes if n.op == "call_function"}
    assert "odise_b200.msda_fused_forward" in targets
    with torch.no_grad():
        assert torch.equal(ep.module()(*args), m(*args))
