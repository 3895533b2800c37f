"""CPU checks of the MSDeformAttn backward: the fp64 autograd oracle (oracle/msda_grad.py) is pinned against the grads
of the reference's own ms_deform_attn_core_pytorch (F.grid_sample backward); the new C entry points validate their
arguments without a GPU; the Python drop-in refuses CPU tensors (there is no CPU fallback)."""
import pytest
import torch

# the reference's ops/test.py problem (ops/test.py:24-31) and the ODISE 512^2 pixel-decoder shape at batch 1
PIN_CASES = {
    "ops_test": dict(seed=3, N=1, M=2, D=2, shapes=[(6, 4), (3, 2)], Lq=2, P=2, small_values=True),
    "release_512": dict(seed=4, N=1, M=8, D=32, shapes=[(16, 16), (32, 32), (64, 64)], Lq=5376, P=4),
}


def _reference_grads(cfg):
    from oracle import refshim
    from oracle.msda_grad import grad_problem
    core = refshim.modules().ms_deform_attn_core_pytorch
    value, ss, _, loc, aw, go = grad_problem(**cfg)
    v, lc, a = (t.clone().requires_grad_(True) for t in (value, loc, aw))
    out = core(v, [(int(h), int(w)) for h, w in ss], lc, a)
    return list(torch.autograd.grad(out, (v, lc, a), go))


@pytest.mark.parametrize("name", sorted(PIN_CASES))
def test_oracle_grads_pinned_to_reference(name):
    """autograd of the explicit-gather oracle == grid_sample backward of the reference's PyTorch restatement (fp64)."""
    from oracle import refshim
    from oracle.msda_grad import grad_problem, oracle_grads
    cfg = PIN_CASES[name]
    ref = refshim.pinned(name, lambda: _reference_grads(cfg), fixture="ref_pinned_msda_grad.pt",
                         store=lambda v: [refshim.sample(t, seed=i) for i, t in enumerate(v)])
    got = oracle_grads(*grad_problem(**cfg))
    for i, (gt, rt) in enumerate(zip(got, ref)):
        a, b = refshim.at_sample(gt, rt)
        scale = max(1.0, b.abs().max().item())
        assert (a - b).abs().max().item() < 1e-10 * scale, (name, i)


def test_far_outside_locations_have_zero_oracle_grads():
    from oracle.msda_grad import grad_problem, oracle_grads
    gv, gl, ga = oracle_grads(*grad_problem(seed=5, N=1, M=2, D=4, shapes=[(5, 7), (3, 2)], Lq=6, P=3, far=True))
    assert gv.abs().max() == 0 and gl.abs().max() == 0 and ga.abs().max() == 0


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


def test_backward_argument_validation_without_gpu(built):
    from odise_b200 import lib
    L = lib.load()
    p = 16       # any non-null address: every call below fails its checks before anything is dereferenced or launched
    for fn in (L.odise_msda_backward_f32, L.odise_msda_backward_f64):
        assert fn(None, None, None, None, None, None, None, None, None, 1, 1, 1, 4, 1, 1, 1, None) == 10001
        assert fn(p, p, p, p, p, p, p, p, None, 1, 1, 1, 4, 1, 1, 1, None) == 10001        # grad_attn missing
        for bad in range(7):                                                                  # N S M D L Lq P
            dims = [1, 1, 1, 4, 1, 1, 1]
            dims[bad] = 0
            assert fn(p, p, p, p, p, p, p, p, p, *dims, None) == 10001
        assert fn(p, p, p, p, p, p, p, p, p, 1, 1, 1, 4, 9, 1, 1, None) == 10001             # L > 8
    assert L.odise_msda_forward_f64(None, None, None, None, None, None, 1, 1, 1, 4, 1, 1, 1, None) == 10001
    assert L.odise_msda_forward_f64(p, p, p, p, p, p, 1, -1, 1, 4, 1, 1, 1, None) == 10001


def test_backward_has_no_cpu_fallback():
    from odise_b200 import lib
    from odise_b200.msda import MSDA, MSDeformAttnFunction
    value, ss, lsi, loc, aw, go = (torch.zeros(1, 4, 1, 4), torch.tensor([[2, 2]]), torch.tensor([0]),
                                   torch.zeros(1, 1, 1, 1, 1, 2), torch.zeros(1, 1, 1, 1, 1), torch.zeros(1, 1, 4))
    with pytest.raises(RuntimeError):
        lib.msda_backward(value, ss, lsi, loc, aw, go, 128)
    with pytest.raises(RuntimeError):
        MSDA.ms_deform_attn_backward(value.double(), ss, lsi, loc.double(), aw.double(), go.double(), 128)
    with pytest.raises(RuntimeError):
        MSDA.ms_deform_attn_forward(value.double(), ss, lsi, loc.double(), aw.double(), 128)
    with pytest.raises(RuntimeError):
        MSDeformAttnFunction.apply(value.requires_grad_(), ss, lsi, loc, aw, 128)
