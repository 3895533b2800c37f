"""GPU checks of the fused MSDeformAttn backward (odise_msda_fused_backward_f32) and of the module drop-in
odise_b200.msda.MSDeformAttn: the entry point against the fp64 CPU autograd oracle (oracle/msda_module.py), forward
equality with the inference path's fused op, determinism and CUDA-graph capture, full module training steps on both
sides of the dispatch against the fp64 module oracle, a short training run through both paths, and the error classes.
Bar: 1e-5 x max(1, max |ref|), as in tests/test_gpu_msda_backward.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# the D = 32 cases of tests/test_gpu_msda_backward.py::FP32_CASES
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
    return f"D{cfg['D']}-L{len(cfg['shapes'])}-P{cfg['P']}-Lq{cfg['Lq']}" + ("-far" if cfg.get("far") else "")


def _on(dev, tensors):
    return [t.to(dev) for t in tensors]


def _close(got, want, tol=1e-5):
    scale = max(1.0, want.abs().max().item())
    err = (got.detach().cpu().double() - want.double()).abs().max().item()
    return err < tol * scale, err, scale


@pytest.mark.parametrize("cfg", FUSED_CASES, ids=_id)
def test_fused_backward_vs_fp64_oracle(cuda, cfg, record):
    from odise_b200 import lib
    from oracle.msda_module import fused_problem, oracle_fused_grads
    # the oracle differentiates at the fp32-rounded inputs, so that only the kernel's own rounding is measured
    prob = fused_problem(**cfg, dtype=torch.float32)
    want = oracle_fused_grads(*prob)
    got = lib.msda_fused_backward(*_on(cuda, prob))
    torch.cuda.synchronize()
    rel = []
    for name, g, w in zip(NAMES, got, want):
        assert g.shape == w.shape and g.dtype == torch.float32
        ok, err, scale = _close(g, w)
        assert ok, (name, err, scale)
        if cfg.get("far"):
            assert g.abs().max().item() == 0, name
        rel.append(f"{name} {err / scale:.2e}")
    record(f"msda fused backward fp32 vs fp64 oracle {_id(cfg)}: max err / max(1, |ref|): " + " ".join(rel))


def test_fused_function_reference_point_grad(cuda):
    """MSDeformAttnFusedFunction: the gradient of the reference points (computed in torch from grad_offsets) against the
    oracle, and value / offsets / logits gradients equal to the entry point's."""
    from odise_b200 import lib
    from odise_b200.msda import MSDeformAttnFusedFunction
    from oracle.msda_module import fused_problem, oracle_fused_grads
    prob = fused_problem(**FUSED_CASES[2], dtype=torch.float32)
    want = oracle_fused_grads(*prob, ref_grad=True)
    value, ss, lsi, ref, offs, logits, go = _on(cuda, prob)
    leaves = [t.clone().requires_grad_(True) for t in (value, ref, offs, logits)]
    out = MSDeformAttnFusedFunction.apply(leaves[0], ss, lsi, *leaves[1:])
    out.backward(go)
    ok, err, scale = _close(leaves[1].grad, want[3])
    assert ok, ("grad_reference_points", err, scale)
    direct = lib.msda_fused_backward(value, ss, lsi, ref, offs, logits, go)
    assert torch.equal(leaves[2].grad, direct[1]) and torch.equal(leaves[3].grad, direct[2])
    ok, err, scale = _close(leaves[0].grad, want[0])
    assert ok, ("grad_value", err, scale)


def test_module_forward_equals_inference_fused_op(cuda):
    """The module's fused path runs the inference path's kernel: its output equals ops.msda_fused(..., want_f32=True)
    followed by the same output projection, bit for bit."""
    from odise_b200 import lib, ops
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_module import module_problem
    pr = module_problem(seed=50, N=2, d_model=256, n_heads=8, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4,
                        dtype=torch.float32)
    m = MSDeformAttn(256, 3, 8, 4).to(cuda)
    m.load_state_dict(pr["params"])
    q, ref, x, ss, lsi = _on(cuda, [pr[k] for k in ("query", "reference_points", "input_flatten", "spatial_shapes",
                                                     "level_start_index")])
    with torch.no_grad():
        got = m(q, ref, x, ss, lsi)
        N, S, _ = x.shape
        value = m.value_proj(x).view(N, S, 8, 32)
        offs = m.sampling_offsets(q).view(N, S, 8, 3, 4, 2)
        logits = m.attention_weights(q).view(N, S, 8, 12)
        o32, _ = ops.msda_fused(value, ss, lsi, ref, offs, logits, N, S, 8, 32, 3, S, 4, want_f32=True)
        assert torch.equal(lib.msda_fused_forward(value, ss, lsi, ref, offs, logits).view(N * S, 256), o32)
        want = m.output_proj(o32.view(N, S, 256))
    assert torch.equal(got, want)


@pytest.mark.parametrize("cfg", [FUSED_CASES[0], FUSED_CASES[4]], ids=_id)
def test_fused_determinism_and_graph_capture(cuda, cfg):
    """grad_offsets / grad_logits are written without atomics: bit-identical across eager calls and a CUDA-graph replay
    into NaN-filled buffers.  grad_value is accumulated with atomics (order-dependent)."""
    from odise_b200 import lib
    from oracle.msda_module import fused_problem
    args = _on(cuda, fused_problem(**cfg, dtype=torch.float32))
    a = lib.msda_fused_backward(*args)
    b = lib.msda_fused_backward(*args)
    torch.cuda.synchronize()
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert (a[0] - b[0]).abs().max().item() <= 1e-6 * a[0].abs().max().item()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lib.msda_fused_backward(*args)                   # warm-up on the side stream before capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = lib.msda_fused_backward(*args)
    for t in c:
        t.fill_(float("nan"))                            # the replay must overwrite all three buffers
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(c[1], a[1]) and torch.equal(c[2], a[2])
    assert (c[0] - a[0]).abs().max().item() <= 1e-6 * a[0].abs().max().item()


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
    # D = 32: the fused path, with a padding mask and reference points that require grad
    "fused_d32_padding_refgrad": (dict(seed=51, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)],
                                       n_points=4, padding=True), True, "fused"),
    # the ODISE pixel decoder's configuration (d_model 256, 8 heads, 3 levels, 4 points)
    "fused_odise": (dict(seed=52, N=1, d_model=256, n_heads=8, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4), False,
                    "fused"),
    # D = 64 (d_model 256, 4 heads): the composed path
    "composed_d64_padding": (dict(seed=53, N=1, d_model=256, n_heads=4, shapes=[(4, 4), (8, 8), (16, 16)], n_points=4,
                                  padding=True), False, "composed"),
    # 4-column box reference points: the composed path
    "composed_box_refgrad": (dict(seed=54, N=2, d_model=64, n_heads=2, shapes=[(4, 4), (8, 8)], n_points=3, box=True),
                             True, "composed"),
}


@pytest.mark.parametrize("name", sorted(MODULE_CASES))
def test_module_training_step_vs_fp64_oracle(cuda, name, dispatch_spy):
    """One forward + backward of MSDeformAttn in fp32 on the GPU: output and the gradients of all Linear weights and
    biases, query, input_flatten (and reference_points where it requires grad) against the fp64 module oracle."""
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_module import module_problem, oracle_module_grads, sample_margin
    cfg, ref_grad, path = MODULE_CASES[name]
    pr = module_problem(**cfg, dtype=torch.float32)
    assert sample_margin(pr["params"], pr["query"], pr["reference_points"], pr["spatial_shapes"], cfg["n_heads"],
                         cfg["n_points"]) >= 0.02
    want_out, want = oracle_module_grads(pr["params"], pr["query"], pr["reference_points"], pr["input_flatten"],
                                         pr["spatial_shapes"], pr["level_start_index"], pr["padding_mask"],
                                         pr["grad_output"], cfg["n_heads"], cfg["n_points"], ref_grad=ref_grad)
    m = MSDeformAttn(cfg["d_model"], len(cfg["shapes"]), cfg["n_heads"], cfg["n_points"]).to(cuda)
    m.load_state_dict(pr["params"])
    q, ref, x = (pr[k].to(cuda).requires_grad_(k != "reference_points" or ref_grad)
                 for k in ("query", "reference_points", "input_flatten"))
    mask = None if pr["padding_mask"] is None else pr["padding_mask"].to(cuda)
    out = m(q, ref, x, pr["spatial_shapes"].to(cuda), pr["level_start_index"].to(cuda), mask)
    out.backward(pr["grad_output"].to(cuda))
    assert dispatch_spy == [path]
    got = {k: p.grad for k, p in m.named_parameters()}
    got.update(query=q.grad, input_flatten=x.grad)
    if ref_grad:
        got["reference_points"] = ref.grad
    else:
        assert ref.grad is None
    assert sorted(got) == sorted(want)
    for k in ["output"] + sorted(want):
        ok, err, scale = _close(out if k == "output" else got[k], want_out if k == "output" else want[k])
        assert ok, (k, err, scale)


def _stack_run(dev, use_fused, steps, lr):
    """SGD on a 2-layer stack x <- x + MSDeformAttn(x, ref, x) (D = 32, the encoder's setting) -> (losses, smallest
    sample margin over all layers and steps)."""
    from odise_b200.msda import MSDeformAttn
    from oracle.msda_module import module_problem, sample_margin
    cfg = dict(N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4)
    prs = [module_problem(seed=60 + i, **cfg, dtype=torch.float32) for i in range(2)]
    layers = []
    for pr in prs:
        m = MSDeformAttn(64, 3, 2, 4).to(dev)
        m.load_state_dict(pr["params"])
        m.use_fused = use_fused
        layers.append(m)
    pr = prs[0]
    ss, lsi, ref = pr["spatial_shapes"].to(dev), pr["level_start_index"].to(dev), pr["reference_points"].to(dev)
    x0 = pr["input_flatten"].to(dev)
    target = torch.randn(x0.shape, generator=torch.Generator().manual_seed(5)).to(dev)
    opt = torch.optim.SGD([p for m in layers for p in m.parameters()], lr=lr)
    losses, margin = [], float("inf")
    for _ in range(steps):
        x = x0
        for m in layers:
            margin = min(margin, sample_margin(m.state_dict(), x.detach(), ref, ss, 2, 4))
            x = x + m(x, ref, x, ss, lsi)
        loss = ((x - target) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    return losses, margin


def test_short_training_run_fused_vs_composed(cuda, dispatch_spy):
    """Four SGD steps of a 2-layer stack: the fused and the composed path give the same loss trajectory (every sample
    stays at least 0.02 px from a cell edge at every step, so both paths pick the same cells)."""
    fused, m_fused = _stack_run(cuda, True, 4, 0.1)
    assert set(dispatch_spy) == {"fused"}
    dispatch_spy.clear()
    composed, m_composed = _stack_run(cuda, False, 4, 0.1)
    assert set(dispatch_spy) == {"composed"}
    assert min(m_fused, m_composed) >= 0.02, (m_fused, m_composed)
    assert fused[-1] < fused[0]
    for a, b in zip(fused, composed):
        assert abs(a - b) <= 1e-5 * abs(b), (fused, composed)


def test_fused_errors(cuda):
    from odise_b200 import lib
    from oracle.msda_module import fused_problem
    args = _on(cuda, fused_problem(seed=3, N=2, M=2, D=32, shapes=[(6, 4)], Lq=3, P=2, dtype=torch.float32))
    value, ss, lsi, ref, offs, logits, go = args
    with pytest.raises(RuntimeError):                   # CPU tensors
        lib.msda_fused_backward(*[t.cpu() for t in args])
    with pytest.raises(RuntimeError):
        lib.msda_fused_forward(value.cpu(), ss, lsi, ref, offs, logits)
    with pytest.raises(RuntimeError):                   # non-contiguous
        lib.msda_fused_backward(value, ss, lsi, ref, offs, logits, go.transpose(0, 1).contiguous().transpose(0, 1))
    with pytest.raises(RuntimeError):
        lib.msda_fused_forward(value, ss, lsi, ref.transpose(0, 1).contiguous().transpose(0, 1), offs, logits)
    with pytest.raises(RuntimeError):                   # float16
        lib.msda_fused_backward(value.half(), ss, lsi, ref.half(), offs.half(), logits.half(), go.half())
    with pytest.raises(RuntimeError):                   # float64 (the fused op is float32 only)
        lib.msda_fused_forward(value.double(), ss, lsi, ref.double(), offs.double(), logits.double())
    with pytest.raises(RuntimeError):                   # shapes that disagree
        lib.msda_fused_backward(value, ss, lsi, ref, offs, logits[..., :1].contiguous(), go)
    with pytest.raises(RuntimeError):
        lib.msda_fused_forward(value, ss, lsi, ref[:, :2].contiguous(), offs, logits)
    with pytest.raises(RuntimeError):                   # D = 64: no fused backward
        lib.msda_fused_backward(*_on(cuda, fused_problem(seed=3, N=1, M=2, D=64, shapes=[(6, 4)], Lq=3, P=2,
                                                         dtype=torch.float32)))
    with pytest.raises(RuntimeError):                   # L * P = 36 > 32
        lib.msda_fused_backward(*_on(cuda, fused_problem(seed=3, N=1, M=2, D=32, shapes=[(3, 3)] * 4, Lq=3, P=9,
                                                         dtype=torch.float32)))
