"""GPU checks of the MSDeformAttn backward (odise_msda_backward_f32 / _f64, odise_msda_forward_f64) and of the autograd
drop-in odise_b200.msda: fp32 against the fp64 CPU autograd oracle (oracle/msda_grad.py), the reference's own test
(ops/test.py: gradcheck and the fp64 forward check) in fp64, the stored sample of the reference's CUDA backward,
determinism and CUDA-graph capture, a training step through MSDeformAttn's front, and the error classes."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")

OPS_TEST = dict(seed=3, N=1, M=2, D=2, shapes=[(6, 4), (3, 2)], Lq=2, P=2, small_values=True)   # ops/test.py:24-31

FP32_CASES = [
    OPS_TEST,
    dict(seed=4, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64)], Lq=5376, P=4),               # 512^2 release
    dict(seed=5, N=1, M=8, D=32, shapes=[(32, 32), (64, 64), (128, 128)], Lq=21504, P=4),            # 1024^2
    dict(seed=8, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64), (128, 128)], Lq=300, P=4),    # C4: L = 4
    dict(seed=9, N=1, M=8, D=32, shapes=[(9, 7), (5, 3)], Lq=37, P=3),           # L*P = 6: ragged sub-warp, tail block
    dict(seed=10, N=2, M=5, D=32, shapes=[(4, 4)] * 8, Lq=19, P=4),              # L*P = 32: the largest D = 32 block
    dict(seed=11, N=2, M=8, D=32, shapes=[(5, 7), (3, 2)], Lq=23, P=4, far=True),  # far outside: all grads exactly 0
] + [dict(seed=20 + D, N=1, M=2, D=D, shapes=[(6, 4), (3, 2)], Lq=5, P=2) for D in (30, 64, 71, 1025, 2048, 3096)]

# shapes of tests/test_gpu_msda.py::REFKERNEL_CASES with boundary-safe inputs; the reference kernel's gradients are
# stored (sampled) in tests/golden/ref_msda_kernel_backward.pt by tools/make_golden_msda_ref_backward.py
REFKERNEL_BWD_CASES = (dict(seed=4, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64)], Lq=5376, P=4),
                       dict(seed=8, N=2, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64), (128, 128)], Lq=300, P=4),
                       dict(seed=6, N=3, M=4, D=64, shapes=[(7, 5), (3, 9)], Lq=11, P=3))


def _id(cfg):
    return f"D{cfg['D']}-L{len(cfg['shapes'])}-P{cfg['P']}-Lq{cfg['Lq']}" + ("-far" if cfg.get("far") else "")


def _on(dev, tensors, dtype=None):
    return [t.to(dev) if dtype is None or not t.is_floating_point() else t.to(dev, dtype) for t in tensors]


def _close(got, want, tol):
    scale = max(1.0, want.abs().max().item())
    err = (got.detach().cpu().double() - want.double()).abs().max().item()
    return err < tol * scale, err, scale


@pytest.mark.parametrize("cfg", FP32_CASES, ids=_id)
def test_backward_fp32_vs_fp64_oracle(cuda, cfg, record):
    from odise_b200 import lib
    from oracle.msda_grad import grad_problem, oracle_grads
    # the oracle differentiates at the fp32-rounded inputs, so that only the kernel's own rounding is measured
    prob = grad_problem(**cfg, dtype=torch.float32)
    want = oracle_grads(*prob)
    value, ss, lsi, loc, aw, go = _on(cuda, prob)
    got = lib.msda_backward(value, ss, lsi, loc, aw, go, 64)
    torch.cuda.synchronize()
    rel = []
    for name, g, w in zip(("grad_value", "grad_loc", "grad_attn"), got, want):
        assert g.shape == w.shape and g.dtype == torch.float32
        ok, err, scale = _close(g, w, 1e-5)
        assert ok, (name, err, scale)
        if cfg.get("far"):
            assert g.abs().max().item() == 0, name
        rel.append(f"{name} {err / scale:.2e}")
    record(f"msda backward fp32 vs fp64 oracle {_id(cfg)}: max err / max(1, |ref|): " + " ".join(rel))


@pytest.mark.parametrize("D", [30, 32, 64, 71])
def test_gradcheck_fp64_reference_test(cuda, D):
    """ops/test.py check_gradient_numerical(D): torch.autograd.gradcheck of MSDeformAttnFunction in double."""
    from odise_b200.msda import MSDeformAttnFunction
    from oracle.msda_grad import grad_problem
    value, ss, lsi, loc, aw, _ = _on(cuda, grad_problem(**dict(OPS_TEST, D=D, seed=30 + D)))
    value.requires_grad_(True)
    loc.requires_grad_(True)
    aw.requires_grad_(True)
    assert torch.autograd.gradcheck(MSDeformAttnFunction.apply, (value, ss, lsi, loc, aw, 2))


@pytest.mark.parametrize("D", [1025, 2048, 3096])
def test_backward_fp64_wide_vs_oracle(cuda, D):
    """ops/test.py's widest D: a dense numerical Jacobian runs to tens of GB, so the fp64 backward is held to the fp64
    CPU autograd oracle at 1e-12 relative instead."""
    from odise_b200 import lib
    from oracle.msda_grad import grad_problem, oracle_grads
    prob = grad_problem(**dict(OPS_TEST, D=D, seed=30 + D))
    want = oracle_grads(*prob)
    got = lib.msda_backward(*_on(cuda, prob), 2)
    for name, g, w in zip(("grad_value", "grad_loc", "grad_attn"), got, want):
        assert g.dtype == torch.float64
        ok, err, scale = _close(g, w, 1e-12)
        assert ok, (name, err, scale)


def test_forward_fp64_reference_test(cuda):
    """ops/test.py check_forward_equal_with_pytorch_double: torch.allclose with its default tolerances."""
    from odise_b200.msda import MSDA, MSDeformAttnFunction
    from oracle.msda import msda_forward
    from oracle.msda_grad import grad_problem
    value, ss, lsi, loc, aw, _ = grad_problem(**OPS_TEST)
    want = msda_forward(value, ss, lsi, loc, aw)
    d = _on(cuda, (value, ss, lsi, loc, aw))
    out = MSDeformAttnFunction.apply(*d, 2)
    assert out.dtype == torch.float64 and torch.allclose(out.cpu(), want)
    assert torch.allclose(MSDA.ms_deform_attn_forward(*d, 2).cpu(), want)
    # a D = 32 release problem through the same fp64 entry point
    value, ss, lsi, loc, aw, _ = grad_problem(**FP32_CASES[1])
    assert torch.allclose(MSDA.ms_deform_attn_forward(*_on(cuda, (value, ss, lsi, loc, aw)), 64).cpu(),
                          msda_forward(value, ss, lsi, loc, aw))


def test_backward_vs_reference_kernel(cuda):
    """Same inputs as the REFERENCE's own CUDA backward (ms_deformable_col2im_cuda, run through
    oracle/_ref/libref_msda_backward.so when the golden file was made): fp32, only the summation order differs."""
    from odise_b200 import lib
    from oracle.msda_grad import grad_problem
    cases = torch.load(os.path.join(GOLD, "ref_msda_kernel_backward.pt"))
    assert [c["cfg"] for c in cases] == list(REFKERNEL_BWD_CASES)
    for c in cases:
        got = lib.msda_backward(*_on(cuda, grad_problem(**c["cfg"]), torch.float32), 128)
        torch.cuda.synchronize()
        for name, g in zip(("grad_value", "grad_loc", "grad_attn"), got):
            s = c[name]
            err = (g.flatten()[s["idx"].long().to(cuda)].cpu() - s["values"]).abs().max().item()
            assert err < 1e-5 * max(1.0, s["absmax"]), (c["cfg"], name, err)


@pytest.mark.parametrize("cfg", [FP32_CASES[1], FP32_CASES[-1]], ids=_id)
def test_determinism_and_graph_capture(cuda, cfg):
    """grad_loc / grad_attn are written without atomics: bit-identical across eager calls and a CUDA-graph replay.
    grad_value is accumulated with atomics (order-dependent, as in the reference)."""
    from odise_b200 import lib
    from oracle.msda_grad import grad_problem
    args = _on(cuda, grad_problem(**cfg), torch.float32)
    a = lib.msda_backward(*args, 64)
    b = lib.msda_backward(*args, 64)
    torch.cuda.synchronize()
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert (a[0] - b[0]).abs().max().item() <= 1e-6 * a[0].abs().max().item()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lib.msda_backward(*args, 64)                    # warm-up on the side stream before capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = lib.msda_backward(*args, 64)
    for t in c:
        t.fill_(float("nan"))                           # the replay must overwrite all three buffers
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(c[1], a[1]) and torch.equal(c[2], a[2])
    assert (c[0] - a[0]).abs().max().item() <= 1e-6 * a[0].abs().max().item()


def test_training_step_through_drop_in(cuda):
    """MSDeformAttn.forward's front (softmax over L*P, loc = ref + off / (W, H)) in torch ops on CUDA, fed to
    MSDeformAttnFunction, backpropagated from a scalar loss; the gradients w.r.t. value, the raw sampling offsets and the
    attention logits match the same graph run in fp64 on the CPU with oracle.msda.msda_forward."""
    from odise_b200.msda import MSDeformAttnFunction
    from oracle.msda import msda_forward, msdeformattn_front
    from oracle.msda_grad import grad_problem
    N, M, D, P, shapes, Lq = 2, 8, 32, 4, [(16, 16), (32, 32), (64, 64)], 5376
    L = len(shapes)
    value, ss, lsi, loc0, _, go = grad_problem(seed=40, N=N, M=M, D=D, shapes=shapes, Lq=Lq, P=P)
    g = torch.Generator().manual_seed(41)
    ref_pts = torch.rand(N, Lq, L, 2, generator=g, dtype=torch.float64) * 0.2 + 0.4
    norm = torch.stack([ss[:, 1], ss[:, 0]], -1).double()                        # (W, H)
    # offsets that put every sample at the boundary-safe location of grad_problem: loc0 = ref + off / (W, H)
    offs = ((loc0 - ref_pts[:, :, None, :, None, :]) * norm[None, None, None, :, None, :]).reshape(N, Lq, M * L * P * 2)
    logits = torch.randn(N, Lq, M * L * P, generator=g, dtype=torch.float64)

    def step(dev, dtype, fwd):
        v, o, lg = (t.detach().to(dev, dtype, copy=True).requires_grad_(True) for t in (value, offs, logits))
        loc, aw = msdeformattn_front(None, ref_pts.to(dev, dtype), o, lg, ss.to(dev), M, L, P)
        out = fwd(v, ss.to(dev), lsi.to(dev), loc.contiguous(), aw.contiguous())
        (out * go.to(dev, dtype)).sum().backward()
        return v.grad, o.grad, lg.grad

    want = step("cpu", torch.float64, msda_forward)
    got = step(cuda, torch.float32, lambda *a: MSDeformAttnFunction.apply(*a, 64))
    for name, gt, w in zip(("value", "sampling_offsets", "attention_logits"), got, want):
        ok, err, scale = _close(gt, w, 1e-5)
        assert ok, (name, err, scale)


def test_backward_errors(cuda):
    from odise_b200 import lib
    from oracle.msda_grad import grad_problem
    value, ss, lsi, loc, aw, go = _on(cuda, grad_problem(seed=3, N=2, M=2, D=4, shapes=[(6, 4)], Lq=2, P=2),
                                      torch.float32)
    with pytest.raises(RuntimeError):               # non-contiguous (reference .cu:98-103)
        lib.msda_backward(value.transpose(2, 3), ss, lsi, loc, aw, go, 2)
    with pytest.raises(RuntimeError):
        lib.msda_backward(value, ss, lsi, loc, aw, go.transpose(1, 2), 2)
    with pytest.raises(RuntimeError):               # mixed dtypes
        lib.msda_backward(value.double(), ss, lsi, loc, aw, go, 2)
    with pytest.raises(RuntimeError):
        lib.msda_backward(value, ss, lsi, loc, aw, go.double(), 2)
    with pytest.raises(RuntimeError):               # batch 3 with im2col_step 2: 3 % min(3, 2) != 0 (reference .cu:121)
        lib.msda_backward(*_on(cuda, grad_problem(seed=3, N=3, M=2, D=4, shapes=[(6, 4)], Lq=2, P=2),
                               torch.float32), 2)
    with pytest.raises(RuntimeError):               # float16 is not dispatched (the reference: float and double)
        lib.msda_backward(value.half(), ss, lsi, loc.half(), aw.half(), go.half(), 2)
