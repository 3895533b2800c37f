"""Oracle side of the MSDeformAttn backward (CPU, torch fp64).  TEST INFRASTRUCTURE ONLY.

grad_problem() draws seeded inputs for gradient checks; oracle_grads() differentiates oracle.msda.msda_forward (explicit
gathers) with torch autograd.  tests/test_msda_backward_cpu.py pins oracle_grads() against the grads of the reference's
own ms_deform_attn_core_pytorch (F.grid_sample backward, ops/functions/ms_deform_attn_func.py:52-72).

Why the sampling locations are drawn away from cell edges: the derivative of bilinear interpolation jumps where the
pixel coordinate loc * H - 0.5 crosses an integer.  fp32 on the device and fp64 on the CPU can pick different cells for
a coordinate within a few ulps of an integer, which turns a rounding difference into an O(1) difference of grad_loc.
So every coordinate is an integer cell in [-1, H - 1] (the first and last include samples that lie partly outside the
level) plus a fractional part in [0.02, 0.98].
"""
import torch

from .msda import msda_forward


def _coord(g, shape, size, dtype):
    cell = torch.randint(-1, size, shape, generator=g).to(dtype)          # -1 .. size-1
    frac = 0.02 + 0.96 * torch.rand(shape, generator=g, dtype=dtype)
    return (cell + frac + 0.5) / size                                      # loc with loc * size - 0.5 = cell + frac


def grad_problem(seed, N, M, D, shapes, Lq, P, small_values=False, far=False, dtype=torch.float64):
    """-> value, spatial_shapes, level_start_index, sampling_locations, attention_weights, grad_output (CPU, dtype).
    small_values: value = rand * 0.01 as in the reference's ops/test.py (else randn).  far: every location lies far
    outside its level (all gradients are exactly zero)."""
    g = torch.Generator().manual_seed(seed)
    ss = torch.as_tensor(shapes, dtype=torch.long)
    lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
    S = int(ss.prod(1).sum())
    L = len(shapes)
    value = (torch.rand(N, S, M, D, generator=g, dtype=torch.float64) * 0.01 if small_values
             else torch.randn(N, S, M, D, generator=g, dtype=torch.float64))
    loc = torch.empty(N, Lq, M, L, P, 2, dtype=torch.float64)
    for l, (H, W) in enumerate(shapes):
        loc[:, :, :, l, :, 0] = _coord(g, (N, Lq, M, P), W, torch.float64)
        loc[:, :, :, l, :, 1] = _coord(g, (N, Lq, M, P), H, torch.float64)
    if far:
        sign = torch.randint(0, 2, loc.shape, generator=g).to(torch.float64) * 2 - 1
        loc = 0.5 + sign * (3.0 + torch.rand(loc.shape, generator=g, dtype=torch.float64))
    aw = torch.rand(N, Lq, M, L, P, generator=g, dtype=torch.float64) + 1e-5
    aw = aw / aw.sum(-1, keepdim=True).sum(-2, keepdim=True)
    grad_out = torch.randn(N, Lq, M * D, generator=g, dtype=torch.float64)
    return tuple(t.to(dtype) if t.is_floating_point() else t for t in (value, ss, lsi, loc, aw, grad_out))


def oracle_grads(value, spatial_shapes, level_start_index, sampling_locations, attention_weights, grad_output):
    """[grad_value, grad_sampling_loc, grad_attn_weight] of oracle.msda.msda_forward by torch autograd, in fp64."""
    v, loc, aw = (t.detach().double().requires_grad_(True) for t in (value, sampling_locations, attention_weights))
    out = msda_forward(v, spatial_shapes, level_start_index, loc, aw)
    return list(torch.autograd.grad(out, (v, loc, aw), grad_output.double()))
