"""GPU checks of the MSDeformAttn drop-ins under torch.compile and torch.export: torch.library.opcheck of the four custom
ops (torch.ops.odise_b200.*); the autograd Functions compiled with fullgraph=True giving eager's bits; the module
compiled with Inductor against the fp64 module oracle on both dispatch paths, in float32 and under autocast; a short
training run under mode="reduce-overhead" (CUDA graphs), bit-reproducible under torch.use_deterministic_algorithms;
the deterministic switch recompiling; dynamic shapes; and torch.export of the forward.

Which path a compiled module took is read from the recorded FX graphs (the fused or the composed op node): the dispatch
spies of the eager tests do not see a traced call."""
import contextlib
import json
import os
import subprocess
import sys

import pytest
import torch
import torch._dynamo.testing

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# L*P = 6 with a ragged sub-warp and a tail block (tests/test_gpu_msda_module.py::FUSED_CASES[3])
SMALL = dict(seed=9, N=1, M=8, D=32, shapes=[(9, 7), (5, 3)], Lq=37, P=3)
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
ORACLE_BAR_U = 16                  # tests/test_gpu_msda_16bit.py::ORACLE_BAR_U, derivation there

# tests/test_gpu_msda_module.py::MODULE_CASES, restated: name -> (module problem, reference points require grad, path)
MODULE_CASES = {
    "fused_d32_padding_refgrad": (dict(seed=51, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)],
                                       n_points=4, padding=True), True, "fused"),
    "fused_odise": (dict(seed=52, N=1, d_model=256, n_heads=8, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4), False,
                    "fused"),
    "composed_d64_padding": (dict(seed=53, N=1, d_model=256, n_heads=4, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4,
                                  padding=True), False, "composed"),
    "composed_box_refgrad": (dict(seed=54, N=2, d_model=64, n_heads=2, shapes=[(4, 4), (8, 8)], n_points=3, box=True),
                             True, "composed"),
}
FORWARD_OP = {"fused": "odise_b200.msda_fused_forward", "composed": "odise_b200.msda_forward"}
BACKWARD_OP = {"fused": "odise_b200.msda_fused_backward", "composed": "odise_b200.msda_backward"}


def _op_name(target):
    """"odise_b200.<op>" of an FX node's target (an OpOverloadPacket in Dynamo's graphs, an OpOverload in export's)"""
    return str(target).removesuffix(".default")


@pytest.fixture(autouse=True)
def fresh_dynamo():
    torch._dynamo.reset()
    yield
    torch._dynamo.reset()


@contextlib.contextmanager
def deterministic(on):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


class Recorder:
    """a torch.compile backend that records every FX graph Dynamo hands it (with the subgraphs of autograd.Function
    bodies) and compiles it with the named backend"""

    def __init__(self, backend):
        self.backend = torch._dynamo.lookup_backend(backend)
        self.graphs = []

    def __call__(self, gm, example_inputs):
        self.graphs.append(gm)
        return self.backend(gm, example_inputs)

    def ops(self):
        """{odise_b200 op name: set of the dtypes of its first result} over all recorded graphs"""
        found = {}
        for gm in self.graphs:
            for mod in gm.modules():
                if not isinstance(mod, torch.fx.GraphModule):
                    continue
                for n in mod.graph.nodes:
                    if n.op == "call_function" and str(n.target).startswith("odise_b200."):
                        ev = n.meta.get("example_value")
                        ev = ev[0] if isinstance(ev, (tuple, list)) else ev
                        found.setdefault(_op_name(n.target), set()).add(getattr(ev, "dtype", None))
        return found


def _on(dev, tensors):
    return [t.to(dev) for t in tensors]


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8),
                                                                     b.contiguous().view(torch.uint8))


def _close(got, want, tol=1e-5):
    scale = max(1.0, want.abs().max().item())
    err = (got.detach().cpu().double() - want.detach().cpu().double()).abs().max().item()
    return err < tol * scale, err, scale


def _problem(kind, dtype, cfg=SMALL):
    """CPU inputs: "op" -> value, ss, lsi, loc, attn, grad_output; "fused" -> value, ss, lsi, ref, offsets, logits,
    grad_output"""
    if kind == "op":
        from oracle.msda_grad import grad_problem
        return grad_problem(**cfg, dtype=dtype)
    if dtype in U:
        from oracle.msda_16bit import fused_problem_16bit
        return fused_problem_16bit(**cfg, dtype=dtype)
    from oracle.msda_module import fused_problem
    return fused_problem(**cfg, dtype=dtype)


# --------------------------------------------------------------------------------------------------------------------
# torch.library.opcheck

OPCHECK = [("op", torch.float32), ("op", torch.float64), ("fused", torch.float32), ("fused", torch.float16),
           ("fused", torch.bfloat16)]


@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("kind,dtype", OPCHECK, ids=[f"{k}-{str(d)[6:]}" for k, d in OPCHECK])
def test_opcheck(cuda, kind, dtype, det):
    """schema, fake implementation and AOT dispatch with dynamic shapes of each op.  test_aot_dispatch_dynamic compares
    the op's results across runs bit for bit, so the backward ops run it with deterministic=True only: with
    deterministic=False grad_value is summed with float atomics and its bits depend on the order of the sums."""
    import odise_b200.msda  # noqa: F401  (defines the ops)
    ops = torch.ops.odise_b200
    args = _on(cuda, _problem(kind, dtype))
    every = ("test_schema", "test_faketensor", "test_aot_dispatch_dynamic")
    bwd_tests = every if det else ("test_schema", "test_faketensor")
    if kind == "op":
        fwd_call, bwd_call = (ops.msda_forward.default, (*args[:5], 64)), (ops.msda_backward.default, (*args, 64, det))
    else:
        fwd_call, bwd_call = (ops.msda_fused_forward.default, tuple(args[:6])), (ops.msda_fused_backward.default,
                                                                                 (*args, det))
    torch.library.opcheck(*fwd_call, test_utils=every)
    torch.library.opcheck(*bwd_call, test_utils=bwd_tests)


# --------------------------------------------------------------------------------------------------------------------
# the Functions compiled whole: the same kernels, the same bits

@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("kind", ["op", "fused"])
def test_functions_fullgraph_same_bits(cuda, kind, det):
    """MSDeformAttnFunction / MSDeformAttnFusedFunction compiled with fullgraph=True (aot_eager): no graph break, the
    ops in the graph, and out, grad_loc / grad_attn, grad_offsets / grad_logits bit-equal to eager; grad_value bit-equal
    with the deterministic switch on, within 1e-6 x max |grad_value| with it off (float atomics).  The fused case also
    differentiates the reference points (ctx.needs_input_grad[3] under tracing)."""
    from odise_b200.msda import MSDeformAttnFunction, MSDeformAttnFusedFunction
    args = _on(cuda, _problem(kind, torch.float32))
    go = args[-1]
    if kind == "op":
        grad_idx = (0, 3, 4)

        def fn(value, ss, lsi, loc, aw):
            return MSDeformAttnFunction.apply(value, ss, lsi, loc, aw, 64)
    else:
        grad_idx = (0, 3, 4, 5)

        def fn(value, ss, lsi, ref, offs, logits):
            return MSDeformAttnFusedFunction.apply(value, ss, lsi, ref, offs, logits)

    def run(f):
        leaves = [t.clone().requires_grad_(i in grad_idx) for i, t in enumerate(args[:-1])]
        out = f(*leaves)
        out.backward(go.view_as(out))
        return [out.detach()] + [leaves[i].grad for i in grad_idx]

    rec = Recorder("aot_eager")
    with deterministic(det):
        eager = run(fn)
        assert torch._dynamo.explain(fn)(*[t.clone().requires_grad_(True) if i in grad_idx else t
                                           for i, t in enumerate(args[:-1])]).graph_break_count == 0
        torch._dynamo.reset()
        compiled = run(torch.compile(fn, fullgraph=True, backend=rec))
    names = ("out", "grad_value") + (("grad_loc", "grad_attn") if kind == "op" else
                                     ("grad_ref", "grad_offsets", "grad_logits"))
    path = "composed" if kind == "op" else "fused"
    assert set(rec.ops()) == {FORWARD_OP[path], BACKWARD_OP[path]}
    for name, c, e in zip(names, compiled, eager):
        if name == "grad_value" and not det:
            assert (c - e).abs().max().item() <= 1e-6 * e.abs().max().item(), name
        elif name == "grad_ref":          # torch ops on grad_offsets, which is bit-equal
            assert torch.allclose(c, e, rtol=1e-6, atol=0), name
        else:
            assert _bits_equal(c, e), name


# --------------------------------------------------------------------------------------------------------------------
# the module under Inductor

def _module_inputs(dev, pr, ref_grad, dtype=torch.float32):
    q, x = (pr[k].to(dev, dtype).requires_grad_(True) for k in ("query", "input_flatten"))
    ref = pr["reference_points"].to(dev).requires_grad_(ref_grad)
    mask = None if pr["padding_mask"] is None else pr["padding_mask"].to(dev)
    return q, ref, x, pr["spatial_shapes"].to(dev), pr["level_start_index"].to(dev), mask


def _grads(m, q, ref, x, ref_grad):
    got = {k: p.grad for k, p in m.named_parameters()}
    got.update(query=q.grad, input_flatten=x.grad)
    if ref_grad:
        got["reference_points"] = ref.grad
    else:
        assert ref.grad is None
    return got


@pytest.mark.parametrize("name", sorted(MODULE_CASES))
def test_module_inductor_vs_fp64_oracle(cuda, name):
    """torch.compile(MSDeformAttn, fullgraph=True) with Inductor, forward and backward, against the fp64 module oracle at
    the eager tests' bar (1e-5 x max(1, max |ref|)); the path is the one the eager module takes."""
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_module import module_problem, oracle_module_grads
    cfg, ref_grad, path = MODULE_CASES[name]
    pr = module_problem(**cfg, dtype=torch.float32)
    want_out, want = oracle_module_grads(pr["params"], pr["query"], pr["reference_points"], pr["input_flatten"],
                                         pr["spatial_shapes"], pr["level_start_index"], pr["padding_mask"],
                                         pr["grad_output"], cfg["n_heads"], cfg["n_points"], ref_grad=ref_grad)
    m = MSDeformAttn(cfg["d_model"], len(cfg["shapes"]), cfg["n_heads"], cfg["n_points"]).to(cuda)
    m.load_state_dict(pr["params"])
    rec = Recorder("inductor")
    cm = torch.compile(m, fullgraph=True, backend=rec)
    q, ref, x, ss, lsi, mask = _module_inputs(cuda, pr, ref_grad)
    out = cm(q, ref, x, ss, lsi, mask)
    out.backward(pr["grad_output"].to(cuda))
    assert set(rec.ops()) == {FORWARD_OP[path], BACKWARD_OP[path]}
    got = _grads(m, q, ref, x, ref_grad)
    assert sorted(got) == sorted(want)
    for k in ["output"] + sorted(want):
        ok, err, scale = _close(out if k == "output" else got[k], want_out if k == "output" else want[k])
        assert ok, (k, err, scale)


AUTOCAST = [(n, d) for n in ("d32_padding_refgrad", "odise") for d in (torch.float16, torch.bfloat16)]
AUTOCAST_CASES = {   # tests/test_gpu_msda_16bit.py::MODULE_CASES, the two with a fused path
    "d32_padding_refgrad": (dict(seed=51, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4,
                                 padding=True), True),
    "odise": (dict(seed=52, N=1, d_model=256, n_heads=8, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4), False),
}


@pytest.mark.parametrize("use_fused", [True, False], ids=["fused", "composed"])
@pytest.mark.parametrize("name,dtype", AUTOCAST, ids=[f"{n}-{str(d)[6:]}" for n, d in AUTOCAST])
def test_module_inductor_autocast(cuda, name, dtype, use_fused):
    """a float32 module compiled with Inductor and run under torch.autocast: against the fp64 module oracle at the
    16-bit-rounded problem to ORACLE_BAR_U u; the fused path runs the 16-bit fused op, the composed one the float32 op"""
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_16bit import round_module_problem
    from oracle.msda_module import module_problem, oracle_module_grads
    cfg, ref_grad = AUTOCAST_CASES[name]
    pr = round_module_problem(module_problem(**cfg), cfg["n_points"], dtype)
    want_out, want = oracle_module_grads(pr["params"], pr["query"], pr["reference_points"], pr["input_flatten"],
                                         pr["spatial_shapes"], pr["level_start_index"], pr["padding_mask"],
                                         pr["grad_output"], cfg["n_heads"], cfg["n_points"], ref_grad=ref_grad)
    want["output"] = want_out
    m = MSDeformAttn(cfg["d_model"], len(cfg["shapes"]), cfg["n_heads"], cfg["n_points"]).to(cuda)
    m.load_state_dict(pr["params"])
    m.use_fused = use_fused
    rec = Recorder("inductor")
    cm = torch.compile(m, fullgraph=True, backend=rec)
    q, ref, x, ss, lsi, mask = _module_inputs(cuda, pr, ref_grad)
    with torch.autocast("cuda", dtype=dtype):
        out = cm(q, ref, x, ss, lsi, mask)
    assert out.dtype == dtype
    out.backward(pr["grad_output"].to(cuda, dtype))
    ops = rec.ops()
    if use_fused:
        assert ops == {FORWARD_OP["fused"]: {dtype}, BACKWARD_OP["fused"]: {dtype}}
    else:
        assert ops == {FORWARD_OP["composed"]: {torch.float32}, BACKWARD_OP["composed"]: {torch.float32}}
    got = _grads(m, q, ref, x, ref_grad)
    got["output"] = out
    assert sorted(got) == sorted(want)
    u = U[dtype]
    for k in sorted(want):
        scale = max(1.0, want[k].abs().max().item())
        err = (got[k].detach().cpu().double() - want[k]).abs().max().item()
        assert err <= ORACLE_BAR_U * u * scale, (k, err / (u * scale))


# --------------------------------------------------------------------------------------------------------------------
# training under CUDA graphs (mode="reduce-overhead")

def train(dev, mode, steps=4, lr=0.1):
    """SGD on a 2-layer stack x <- x + MSDeformAttn(x, ref, x) (D = 32, the encoder's setting), the forward and loss
    eager (mode None) or compiled with torch.compile(mode=mode, fullgraph=True) -> (losses, parameters)"""
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_module import module_problem
    cfg = dict(N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4)
    prs = [module_problem(seed=60 + i, **cfg, dtype=torch.float32) for i in range(2)]
    layers = []
    for pr in prs:
        m = MSDeformAttn(64, 3, 2, 4).to(dev)
        m.load_state_dict(pr["params"])
        layers.append(m)
    pr = prs[0]
    ss, lsi, ref = pr["spatial_shapes"].to(dev), pr["level_start_index"].to(dev), pr["reference_points"].to(dev)
    x0 = pr["input_flatten"].to(dev)
    target = torch.randn(x0.shape, generator=torch.Generator().manual_seed(5)).to(dev)

    def loss_fn(x):
        for m in layers:
            x = x + m(x, ref, x, ss, lsi)
        return ((x - target) ** 2).mean()

    if mode is not None:
        loss_fn = torch.compile(loss_fn, mode=mode, fullgraph=True)
    params = [p for m in layers for p in m.parameters()]
    opt = torch.optim.SGD(params, lr=lr)
    losses = []
    for _ in range(steps):
        torch.compiler.cudagraph_mark_step_begin()
        loss = loss_fn(x0)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    return losses, [p.detach().clone() for p in params]


def test_training_under_cuda_graphs(cuda):
    """Four SGD steps of a 2-layer stack compiled with mode="reduce-overhead": the loss trajectory of eager to the
    fused-vs-composed bar of tests/test_gpu_msda_module.py (1e-5 relative), and the loss goes down."""
    eager, _ = train(cuda, None)
    graphs, _ = train(cuda, "reduce-overhead")
    assert graphs[-1] < graphs[0]
    for a, b in zip(graphs, eager):
        assert abs(a - b) <= 1e-5 * abs(b), (graphs, eager)


_DET_SCRIPT = r"""
import json, os, sys
sys.path[:0] = [sys.argv[1], os.path.join(sys.argv[1], "tests")]
import torch
from test_gpu_msda_compile import train
torch.use_deterministic_algorithms(True)
dev = torch.device("cuda:0")
a = train(dev, "reduce-overhead")
torch._dynamo.reset()
b = train(dev, "reduce-overhead")
same = all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(a[1], b[1]))
print("RESULT " + json.dumps(dict(identical=same, losses=[a[0], b[0]])))
"""


def test_training_under_cuda_graphs_is_bit_reproducible(cuda):
    """Two compiled 4-step runs (mode="reduce-overhead", each compiled afresh) with torch.use_deterministic_algorithms
    (True) and CUBLAS_WORKSPACE_CONFIG=:4096:8 (set before CUDA starts, hence the subprocess) end with bit-identical
    parameters."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _DET_SCRIPT, ROOT]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])
    assert res["identical"], res


# --------------------------------------------------------------------------------------------------------------------
# the deterministic switch, dynamic shapes, export

@pytest.mark.parametrize("kind", ["op", "fused"])
def test_switch_recompiles(cuda, kind):
    """torch.use_deterministic_algorithms is read when the graph is traced and Dynamo guards on it: a function compiled
    and run with the switch off recompiles when it is turned on, and then returns eager's deterministic grad_value, bit
    for bit"""
    from odise_b200.msda import MSDeformAttnFunction, MSDeformAttnFusedFunction
    args = _on(cuda, _problem(kind, torch.float32))
    go = args[-1]
    fn_cls = MSDeformAttnFunction if kind == "op" else MSDeformAttnFusedFunction
    extra = (64,) if kind == "op" else ()

    def fn(*a):
        return fn_cls.apply(*a, *extra)

    def grad_value(f):
        value = args[0].clone().requires_grad_(True)
        out = f(value, *args[1:-1])
        out.backward(go.view_as(out))
        return value.grad

    counter = torch._dynamo.testing.CompileCounterWithBackend("aot_eager")
    cf = torch.compile(fn, fullgraph=True, backend=counter)
    with deterministic(False):
        grad_value(cf)
    assert counter.frame_count == 1
    with deterministic(True):
        got = grad_value(cf)
        want = grad_value(fn)
    assert counter.frame_count == 2
    assert _bits_equal(got, want)


def test_dynamic_shapes(cuda):
    """torch.compile(MSDeformAttn, dynamic=True): two image sizes (different S and Lq) with at most one recompile, each
    matching eager to 1e-5 x max(1, max |eager|)"""
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_module import module_problem
    sizes = ([(8, 8), (16, 16), (32, 32)], [(6, 10), (12, 20), (24, 40)])
    prs = [module_problem(seed=55, N=2, d_model=64, n_heads=2, shapes=s, n_points=4, dtype=torch.float32)
           for s in sizes]
    m = MSDeformAttn(64, 3, 2, 4).to(cuda)
    m.load_state_dict(prs[0]["params"])
    counter = torch._dynamo.testing.CompileCounterWithBackend("inductor")
    cm = torch.compile(m, dynamic=True, fullgraph=True, backend=counter)
    for pr in prs:
        runs = []
        for f in (m, cm):
            m.zero_grad()
            q, ref, x, ss, lsi, _ = _module_inputs(cuda, pr, False)
            out = f(q, ref, x, ss, lsi)
            out.backward(pr["grad_output"].to(cuda))
            runs.append([out.detach(), q.grad, x.grad] + [p.grad.clone() for p in m.parameters()])
        for got, want in zip(runs[1], runs[0]):
            ok, err, scale = _close(got, want)
            assert ok, (err, scale)
    assert counter.frame_count <= 2


def test_export_forward(cuda):
    """torch.export.export of an eval-mode MSDeformAttn forward holds the fused op, and the exported program's output
    equals eager's"""
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_module import module_problem
    cfg, _, _ = MODULE_CASES["fused_odise"]
    pr = module_problem(**cfg, dtype=torch.float32)
    m = MSDeformAttn(cfg["d_model"], len(cfg["shapes"]), cfg["n_heads"], cfg["n_points"]).to(cuda).eval()
    m.load_state_dict(pr["params"])
    args = tuple(pr[k].to(cuda) for k in ("query", "reference_points", "input_flatten", "spatial_shapes",
                                           "level_start_index"))
    ep = torch.export.export(m, args)
    targets = {_op_name(n.target) for n in ep.graph.nodes if n.op == "call_function"}
    assert FORWARD_OP["fused"] in targets
    with torch.no_grad():
        assert torch.equal(ep.module()(*args), m(*args))
