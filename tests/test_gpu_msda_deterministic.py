"""GPU checks of the deterministic MSDeformAttn backward (odise_msda_*_det_*, lib's deterministic=True and
torch.use_deterministic_algorithms in odise_b200.msda): grad_value against the fp64 oracles within the default paths'
bars with every other gradient bit-equal to the default path's, bit-for-bit independence of the reduction order
(repeated calls, CUDA-graph replay, permuted queries, batch split), the fixed-point scale (exact power-of-two scaling,
NaN in exactly the non-finite slice), gradcheck in fp64 under deterministic mode, and bit-reproducible training of the
module in a subprocess."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the shapes of tests/test_gpu_msda_backward.py / test_gpu_msda_module.py
D32_CASES = [
    dict(seed=4, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64)], Lq=5376, P=4),               # 512^2 release
    dict(seed=5, N=1, M=8, D=32, shapes=[(32, 32), (64, 64), (128, 128)], Lq=21504, P=4),            # 1024^2
    dict(seed=8, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64), (128, 128)], Lq=300, P=4),    # C4: L = 4
    dict(seed=9, N=1, M=8, D=32, shapes=[(9, 7), (5, 3)], Lq=37, P=3),           # L*P = 6: ragged sub-warp, tail block
    dict(seed=10, N=2, M=5, D=32, shapes=[(4, 4)] * 8, Lq=19, P=4),              # L*P = 32: the largest D = 32 block
    dict(seed=11, N=2, M=8, D=32, shapes=[(5, 7), (3, 2)], Lq=23, P=4, far=True),  # far outside: all grads exactly 0
]
WARP_CASES = [dict(seed=20 + D, N=2, M=2, D=D, shapes=[(6, 4), (3, 2)], Lq=37, P=2) for D in (30, 64, 71)]
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
DT = {torch.float32: "f32", torch.float64: "f64", torch.float16: "f16", torch.bfloat16: "bf16"}


def _id(cfg):
    return f"D{cfg['D']}-L{len(cfg['shapes'])}-P{cfg['P']}-Lq{cfg['Lq']}" + ("-far" if cfg.get("far") else "")


def _on(dev, tensors):
    return [t.to(dev) for t in tensors]


def _close(got, want, tol):
    scale = max(1.0, want.abs().max().item())
    err = (got.detach().cpu().double() - want.double()).abs().max().item()
    return err < tol * scale, err, scale


# --------------------------------------------------------------------------------------------------------------------
# the five entry points behind one interface: "op" = msda_backward (inputs value, ss, lsi, loc, attn, grad_out),
# "fused" = msda_fused_backward / _16bit (inputs value, ss, lsi, ref, offsets, logits, grad_out)

PATHS = {     # name -> (kind, dtype, case)
    "op_d32_f32": ("op", torch.float32, D32_CASES[0]),
    "op_warp_f32": ("op", torch.float32, WARP_CASES[1]),
    "op_warp_f64": ("op", torch.float64, WARP_CASES[0]),
    "fused_f32": ("fused", torch.float32, D32_CASES[0]),
    "fused_f16": ("fused", torch.float16, D32_CASES[0]),
    "fused_bf16": ("fused", torch.bfloat16, D32_CASES[0]),
}
QUERY_ARGS = {"op": (3, 4, 5), "fused": (3, 4, 5, 6)}            # arguments with a query dimension (dim 1)
BATCH_ARGS = {"op": (0, 3, 4, 5), "fused": (0, 3, 4, 5, 6)}      # arguments with a batch dimension (dim 0)


def _problem(kind, dtype, cfg):
    """CPU problem of the path"""
    if kind == "op":
        from oracle.msda_grad import grad_problem
        return grad_problem(**cfg, dtype=dtype)
    if dtype in U:
        from oracle.msda_16bit import fused_problem_16bit
        return fused_problem_16bit(**cfg, dtype=dtype)
    from oracle.msda_module import fused_problem
    return fused_problem(**cfg, dtype=dtype)


def _backward(kind, dtype, args, deterministic=True):
    from odise_b200 import lib
    if kind == "op":
        return lib.msda_backward(*args, 64, deterministic=deterministic)
    fn = lib.msda_fused_backward_16bit if dtype in U else lib.msda_fused_backward
    return fn(*args, deterministic=deterministic)


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8),
                                                                     b.contiguous().view(torch.uint8))


# --------------------------------------------------------------------------------------------------------------------
# accuracy against the fp64 oracles; every other gradient bit-equal to the default path's

OP_CASES = ([pytest.param(c, torch.float32, id=_id(c) + "-f32") for c in D32_CASES + WARP_CASES]
            + [pytest.param(c, torch.float64, id=_id(c) + "-f64") for c in WARP_CASES])


@pytest.mark.parametrize("cfg,dtype", OP_CASES)
def test_op_deterministic_vs_fp64_oracle(cuda, cfg, dtype, record):
    """float32 D = 32 (the vectorised kernel) and D = 30 / 64 / 71 (the warp kernel), float64 on the warp kernel: 1e-5
    x max(1, max |ref|) in float32 as the default path, 1e-12 in float64 as tests/test_gpu_msda_backward.py's fp64 bar."""
    from oracle.msda_grad import oracle_grads
    prob = _problem("op", dtype, cfg)
    want = oracle_grads(*prob)
    args = _on(cuda, prob)
    det = _backward("op", dtype, args)
    dflt = _backward("op", dtype, args, deterministic=False)
    torch.cuda.synchronize()
    tol = 1e-5 if dtype == torch.float32 else 1e-12
    ok, err, scale = _close(det[0], want[0], tol)
    assert det[0].dtype == dtype and ok, ("grad_value", err, scale)
    assert _bits_equal(det[1], dflt[1]) and _bits_equal(det[2], dflt[2])
    if cfg.get("far"):
        assert det[0].abs().max().item() == 0
    record(f"msda deterministic backward {DT[dtype]} vs fp64 oracle {_id(cfg)}: grad_value max err / max(1, |ref|) "
           f"{err / scale:.2e}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=DT.get)
@pytest.mark.parametrize("cfg", D32_CASES, ids=_id)
def test_fused_deterministic_vs_fp64_oracle(cuda, cfg, dtype, record):
    """float32: 1e-5 x max(1, max |ref|) as the default fused path; 16 bits: the element-wise bar of
    tests/test_gpu_msda_16bit.py, u |ref| + 1e-5 max(1, max |ref|) (one rounding of a result that meets the float32 bar)."""
    from oracle.msda_module import oracle_fused_grads
    prob = _problem("fused", dtype, cfg)
    want = oracle_fused_grads(*prob)
    args = _on(cuda, prob)
    det = _backward("fused", dtype, args)
    dflt = _backward("fused", dtype, args, deterministic=False)
    torch.cuda.synchronize()
    g, w = det[0].detach().cpu().double(), want[0].double()
    assert det[0].dtype == dtype
    if dtype == torch.float32:
        ok, err, scale = _close(det[0], want[0], 1e-5)
        assert ok, ("grad_value", err, scale)
        ratio = err / (1e-5 * scale)
    else:
        bar = U[dtype] * w.abs() + 1e-5 * max(1.0, w.abs().max().item())
        ratio = ((g - w).abs() / bar).max().item()
        assert ratio <= 1.0, ("grad_value", ratio)
    assert _bits_equal(det[1], dflt[1]) and _bits_equal(det[2], dflt[2])
    if cfg.get("far"):
        assert det[0].abs().max().item() == 0
    record(f"msda deterministic fused backward {DT[dtype]} vs fp64 oracle {_id(cfg)}: grad_value max err / bar "
           f"{ratio:.2e}")


# --------------------------------------------------------------------------------------------------------------------
# order independence, bit for bit

@pytest.mark.parametrize("path", sorted(PATHS))
def test_repeat_and_graph_replay(cuda, path):
    kind, dtype, cfg = PATHS[path]
    args = _on(cuda, _problem(kind, dtype, cfg))
    a = _backward(kind, dtype, args)
    b = _backward(kind, dtype, args)
    torch.cuda.synchronize()
    assert all(_bits_equal(x, y) for x, y in zip(a, b))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _backward(kind, dtype, args)                     # warm-up on the side stream before capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = _backward(kind, dtype, args)
    for t in c:
        t.fill_(float("nan"))                            # the replay must overwrite every buffer
    graph.replay()
    torch.cuda.synchronize()
    assert all(_bits_equal(x, y) for x, y in zip(a, c))


@pytest.mark.parametrize("path", sorted(PATHS))
def test_query_permutation(cuda, path):
    """The queries in a random order (inputs and grad_output permuted together): the same grad_value bits, and the other
    gradients permuted.  Float atomics fail this: the order of the queries is the order of the reductions."""
    kind, dtype, cfg = PATHS[path]
    args = _on(cuda, _problem(kind, dtype, cfg))
    perm = torch.randperm(args[3].shape[1], generator=torch.Generator().manual_seed(7)).to(cuda)
    pargs = [t.index_select(1, perm).contiguous() if i in QUERY_ARGS[kind] else t for i, t in enumerate(args)]
    a = _backward(kind, dtype, args)
    b = _backward(kind, dtype, pargs)
    torch.cuda.synchronize()
    assert _bits_equal(a[0], b[0])
    assert _bits_equal(a[1].index_select(1, perm), b[1]) and _bits_equal(a[2].index_select(1, perm), b[2])


@pytest.mark.parametrize("path", sorted(PATHS))
def test_batch_split(cuda, path):
    """One N = 2 call gives, per image, the bits of an N = 1 call on that image."""
    kind, dtype, cfg = PATHS[path]
    args = _on(cuda, _problem(kind, dtype, cfg))
    assert args[0].shape[0] == 2
    both = _backward(kind, dtype, args)
    for n in range(2):
        one = _backward(kind, dtype, [t[n:n + 1].contiguous() if i in BATCH_ARGS[kind] else t
                                      for i, t in enumerate(args)])
        torch.cuda.synchronize()
        assert all(_bits_equal(x[n:n + 1], y) for x, y in zip(both, one)), n


# --------------------------------------------------------------------------------------------------------------------
# the fixed-point scale

SCALE_K = {torch.float32: 60, torch.float64: 60, torch.bfloat16: 60, torch.float16: 8}
TINY = {torch.float32: 2.0 ** -126, torch.float64: 2.0 ** -1022, torch.bfloat16: 2.0 ** -126, torch.float16: 2.0 ** -14}


@pytest.mark.parametrize("path", sorted(PATHS))
def test_power_of_two_scaling_is_exact(cuda, path):
    """grad_output * 2^k gives exactly grad_value * 2^k (k = +-60; +-8 in float16, whose exponent range is narrow), on
    every output that is a normal number at both scales: the shift s moves by exactly k, the integer sums do not change.
    (An output that rounds to zero, to a subnormal or up to the smallest normal at one scale need not scale exactly.)"""
    kind, dtype, cfg = PATHS[path]
    args = _on(cuda, _problem(kind, dtype, cfg))
    go = args[-1]
    if dtype == torch.float16:       # keep grad_output * 2^-8 normal, so that the scaled input is exact
        go = torch.where(go.abs() < 2.0 ** -5, torch.zeros_like(go), go)
        args[-1] = go
    base = _backward(kind, dtype, args)[0].double()
    k0 = SCALE_K[dtype]
    for k in (k0, -k0):
        sgo = (go.double() * 2.0 ** k).to(dtype)
        assert torch.equal(sgo.double(), go.double() * 2.0 ** k)
        got = _backward(kind, dtype, args[:-1] + [sgo])[0].double()
        want = base * 2.0 ** k
        # strictly above the smallest normal: a result that rounded up to it from the subnormal range was rounded on the
        # coarser subnormal grid at that scale
        normal = (base.abs() > TINY[dtype]) & (want.abs() > TINY[dtype])
        assert normal.float().mean().item() > 0.5
        assert torch.equal(got[normal], want[normal]), k


@pytest.mark.parametrize("path", ["op_d32_f32", "op_warp_f32", "op_warp_f64", "fused_f32", "fused_bf16"])
def test_non_finite_slice(cuda, path):
    """An inf in grad_output[1, q, 1, :] (and, on the op, a NaN in attn[0, q, 0]) gives NaN in exactly those
    grad_value[n, :, m, :] slices; every other slice keeps the bits of the clean run."""
    kind, dtype, cfg = PATHS[path]
    args = _on(cuda, _problem(kind, dtype, cfg))
    clean = _backward(kind, dtype, args)[0]
    M, D = args[0].shape[2], args[0].shape[3]
    go = args[-1].clone()
    go.view(go.shape[0], go.shape[1], M, D)[1, 3, 1, 5] = float("inf")
    bad = args[:-1] + [go]
    hit = {(1, 1)}
    if kind == "op":
        aw = args[4].clone()
        aw[0, 7, 0, 0, 1] = float("nan")
        bad[4] = aw
        hit.add((0, 0))
    got = _backward(kind, dtype, bad)[0]
    torch.cuda.synchronize()
    for n in range(got.shape[0]):
        for m in range(M):
            if (n, m) in hit:
                assert torch.isnan(got[n, :, m]).all(), (n, m)
            else:
                assert _bits_equal(got[n, :, m], clean[n, :, m]), (n, m)


# --------------------------------------------------------------------------------------------------------------------
# autograd and the module

OPS_TEST = dict(seed=3, N=1, M=2, D=2, shapes=[(6, 4), (3, 2)], Lq=2, P=2, small_values=True)   # ops/test.py:24-31


@pytest.fixture
def deterministic_mode():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


@pytest.mark.parametrize("D", [30, 32, 64, 71])
def test_gradcheck_fp64_under_deterministic_mode(cuda, D, deterministic_mode):
    """ops/test.py check_gradient_numerical(D) with torch.use_deterministic_algorithms(True)."""
    from odise_b200.msda import MSDeformAttnFunction
    from oracle.msda_grad import grad_problem
    value, ss, lsi, loc, aw, _ = _on(cuda, grad_problem(**dict(OPS_TEST, D=D, seed=30 + D)))
    for t in (value, loc, aw):
        t.requires_grad_(True)
    assert torch.autograd.gradcheck(MSDeformAttnFunction.apply, (value, ss, lsi, loc, aw, 2))


@pytest.fixture
def backward_spy(monkeypatch):
    """records (deterministic flag, returned gradients) of every lib backward call made by odise_b200.msda"""
    from odise_b200 import lib
    calls = []

    def wrap(fn):
        def spy(*a, deterministic=False, **kw):
            res = fn(*a, deterministic=deterministic, **kw)
            calls.append((deterministic, res))
            return res
        return spy
    for name in ("msda_backward", "msda_fused_backward", "msda_fused_backward_16bit"):
        monkeypatch.setattr(lib, name, wrap(getattr(lib, name)))
    return calls


@pytest.mark.parametrize("mode", ["off", "on", "warn_only"])
def test_functions_follow_the_torch_switch(cuda, mode, backward_spy):
    """MSDeformAttnFunction and MSDeformAttnFusedFunction (float32 and bfloat16) call the lib backward with
    deterministic = torch.are_deterministic_algorithms_enabled() (warn_only included) and hand its gradients to autograd
    unchanged: with the switch off, the gradients are bit-equal to the default lib call's."""
    from odise_b200.msda import MSDeformAttnFunction, MSDeformAttnFusedFunction
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        if mode != "off":
            torch.use_deterministic_algorithms(True, warn_only=mode == "warn_only")
        for kind, dtype in (("op", torch.float32), ("fused", torch.float32), ("fused", torch.bfloat16)):
            args = _on(cuda, _problem(kind, dtype, D32_CASES[3]))
            backward_spy.clear()
            if kind == "op":
                leaves = {i: args[i].clone().requires_grad_(True) for i in (0, 3, 4)}
                out = MSDeformAttnFunction.apply(leaves[0], args[1], args[2], leaves[3], leaves[4], 64)
                order = (0, 3, 4)
            else:
                leaves = {i: args[i].clone().requires_grad_(True) for i in (0, 4, 5)}
                out = MSDeformAttnFusedFunction.apply(leaves[0], args[1], args[2], args[3], leaves[4], leaves[5])
                order = (0, 4, 5)
            out.backward(args[-1].to(out.dtype).view_as(out))
            assert len(backward_spy) == 1
            det, res = backward_spy[0]
            assert det == (mode != "off")
            for i, r in zip(order, res):
                assert _bits_equal(leaves[i].grad, r), (kind, dtype, i)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


_MODULE_SCRIPT = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from odise_b200.msda import MSDeformAttn
from oracle.msda_module import module_problem

torch.use_deterministic_algorithms(True)
dev = torch.device("cuda:0")
RUNS = {  # name -> (module problem, use_fused, autocast dtype)
    "fused_f32": (dict(seed=70, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4), True, None),
    "fused_bf16_autocast": (dict(seed=71, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4),
                            True, torch.bfloat16),
    "composed": (dict(seed=72, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4), False, None),
    "d64": (dict(seed=73, N=2, d_model=256, n_heads=4, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4), True, None),
}


def train(cfg, use_fused, amp):
    pr = module_problem(**cfg, dtype=torch.float32)
    m = MSDeformAttn(cfg["d_model"], len(cfg["shapes"]), cfg["n_heads"], cfg["n_points"]).to(dev)
    m.load_state_dict(pr["params"])
    m.use_fused = use_fused
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


from odise_b200 import lib
seen = []
for name in ("msda_backward", "msda_fused_backward", "msda_fused_backward_16bit"):
    def wrap(fn, name=name):
        def spy(*a, **kw):
            seen.append((name, kw.get("deterministic", False)))
            return fn(*a, **kw)
        return spy
    setattr(lib, name, wrap(getattr(lib, name)))
res = {}
for name, (cfg, use_fused, amp) in RUNS.items():
    seen.clear()
    a = train(cfg, use_fused, amp)
    b = train(cfg, use_fused, amp)
    res[name] = dict(identical=all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(a, b)),
                     calls=sorted(set(seen)))
print("RESULT " + json.dumps(res))
"""


def test_module_training_is_bit_reproducible(cuda):
    """Two 4-step SGD runs of MSDeformAttn with torch.use_deterministic_algorithms(True) and
    CUBLAS_WORKSPACE_CONFIG=:4096:8 (set before CUDA starts, hence the subprocess) end with bit-identical parameters:
    fused float32, fused bfloat16 under autocast, the composed path (use_fused = False) and D = 64 (composed)."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _MODULE_SCRIPT, ROOT]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])
    want_calls = {"fused_f32": [["msda_fused_backward", True]],
                  "fused_bf16_autocast": [["msda_fused_backward_16bit", True]],
                  "composed": [["msda_backward", True]], "d64": [["msda_backward", True]]}
    for name, v in res.items():
        assert v["calls"] == want_calls[name], (name, v)
        assert v["identical"], name
    assert sorted(res) == sorted(want_calls)
