"""Oracle side of the 16-bit fused MSDeformAttn kernels (odise_msda_fused_f16 / _bf16 and their backward).  TEST
INFRASTRUCTURE ONLY.

fused_problem_16bit() draws oracle/msda_module.py's fused problems with value, offsets, logits and grad_output rounded to
float16 or bfloat16 and the reference points rounded to float32, the types the kernels read.  The fp64 oracle
(oracle_fused_grads) then differentiates at those rounded inputs, so a test measures only the kernels' own rounding.

Rounding moves samples: an offset of tens of pixels in bfloat16 is quantised to 0.25-0.5 px, which can put a sample on a
cell edge, where the bilinear derivative jumps (see oracle/msda_grad.py).  So every rounded offset whose sample lies within
MARGIN px of an edge is stepped by whole 16-bit ulps until it does not, and sample_margin_16bit() measures the result.
"""
import math

import torch

from .msda_module import fused_problem

MARGIN = 0.02
UNIT_ROUNDOFF = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}


def ulp(x, dtype):
    """spacing of the 16-bit grid at each element of x (fp64 tensor of values representable in dtype)"""
    mant, emin = {torch.float16: (10, -14), torch.bfloat16: (7, -126)}[dtype]
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.pow(2.0, e - mant)


def pixel_coords(reference_points, offsets, spatial_shapes):
    """fp64 pixel coordinates loc * size - 0.5 of every sample, loc = ref + off / (W, H) -> [N, Lq, M, L, P, 2]"""
    wh = torch.stack([spatial_shapes[:, 1], spatial_shapes[:, 0]], -1).double()[None, None, None, :, None, :]
    loc = reference_points.double()[:, :, None, :, None, :] + offsets.double() / wh
    return loc * wh - 0.5


def edge_distance(reference_points, offsets, spatial_shapes):
    """distance in px of every sample coordinate from the nearest cell edge; samples outside (-2, size + 1) in either
    axis (they read nothing, and rounding cannot bring them in) count as infinitely far"""
    px = pixel_coords(reference_points, offsets, spatial_shapes)
    size = torch.stack([spatial_shapes[:, 1], spatial_shapes[:, 0]], -1).double()[None, None, None, :, None, :]
    d = (px - torch.round(px)).abs()
    outside = ((px <= -2) | (px >= size + 1)).any(-1, keepdim=True).expand_as(d)
    return torch.where(outside, torch.full_like(d, math.inf), d)


def sample_margin_16bit(reference_points, offsets, spatial_shapes):
    return edge_distance(reference_points, offsets, spatial_shapes).min().item()


def keep_off_edges(reference_points, offsets, spatial_shapes, dtype, max_steps=64):
    """offsets (fp64 values representable in dtype) with every coordinate within MARGIN px of a cell edge stepped by
    whole ulps of dtype, +1, -1, +2, -2, ... until it holds; the result is still representable in dtype."""
    offs = offsets.clone()
    base = offsets.clone()
    for k in range(1, max_steps + 1):
        bad = edge_distance(reference_points, offs, spatial_shapes) < MARGIN
        if not bad.any():
            return offs
        step = (k + 1) // 2 * (1 if k % 2 else -1)
        cand = (base + step * ulp(base, dtype)).to(dtype).double()
        offs = torch.where(bad, cand, offs)
    raise AssertionError("keep_off_edges: no 16-bit offset within reach keeps the margin")


def fused_problem_16bit(seed, N, M, D, shapes, Lq, P, dtype, small_values=False, far=False):
    """fused_problem() rounded to what the 16-bit kernels read -> (value, spatial_shapes, level_start_index,
    reference_points float32, offsets, logits, grad_output) on the CPU, the four 16-bit tensors in dtype.  Every sample
    that can touch its level lies at least MARGIN px from a cell edge, asserted."""
    value, ss, lsi, ref, offs, logits, go = fused_problem(seed, N, M, D, shapes, Lq, P, small_values=small_values,
                                                          far=far)
    ref32 = ref.to(torch.float32)
    offs16 = keep_off_edges(ref32, offs.to(dtype).double(), ss, dtype).to(dtype)
    assert sample_margin_16bit(ref32, offs16, ss) >= MARGIN
    return value.to(dtype), ss, lsi, ref32, offs16, logits.to(dtype), go.to(dtype)


def oracle_fused_forward(value, spatial_shapes, level_start_index, reference_points, offsets, logits):
    """the fused op's output [N, Lq, M*D] in fp64: msdeformattn_front, then oracle.msda.msda_forward"""
    from .msda import msda_forward, msdeformattn_front
    N, Lq, M, L, P, _ = offsets.shape
    loc, aw = msdeformattn_front(None, reference_points.double(), offsets.double().reshape(N, Lq, -1),
                                 logits.double().reshape(N, Lq, -1), spatial_shapes, M, L, P)
    return msda_forward(value.double(), spatial_shapes, level_start_index, loc, aw)


def round_module_problem(pr, n_points, dtype):
    """module_problem() (fp64 or fp32) with its parameters and floating inputs rounded to dtype, and sampling_offsets.bias
    stepped by whole ulps so that every sample keeps MARGIN px from a cell edge after rounding.  With
    sampling_offsets.weight = 0 the module's offsets are exactly the 16-bit bias, in a float32 module under autocast and
    in a module cast to dtype alike.  Returns a new dict; the fp64 oracle runs at these values."""
    from .msda_module import _locations
    params = {k: v.to(dtype) for k, v in pr["params"].items()}
    assert params["sampling_offsets.weight"].abs().max() == 0
    ss = pr["spatial_shapes"]
    ref = pr["reference_points"].to(torch.float32).double()
    N, Lq = pr["query"].shape[:2]
    L = ss.shape[0]
    P = n_points
    M = params["sampling_offsets.bias"].numel() // (L * P * 2)
    size = torch.stack([ss[:, 1], ss[:, 0]], -1).double()[None, None, None, :, None, :]

    def bad_entries(bias):
        px = _locations(ref, bias.expand(N, Lq, -1), ss, M, L, P) * size - 0.5
        return ((px - torch.round(px)).abs() < MARGIN).reshape(-1, M * L * P * 2).any(0)

    base = params["sampling_offsets.bias"].double()[None, None, :]
    bias = base.clone()
    for k in range(1, 65):
        bad = bad_entries(bias)
        if not bad.any():
            break
        step = (k + 1) // 2 * (1 if k % 2 else -1)
        bias = torch.where(bad, (base + step * ulp(base, dtype)).to(dtype).double(), bias)
    else:
        raise AssertionError("round_module_problem: no 16-bit bias within reach keeps the margin")
    params["sampling_offsets.bias"] = bias.reshape(-1).to(dtype)
    out = dict(pr, params=params, reference_points=pr["reference_points"].to(torch.float32))
    for k in ("query", "input_flatten", "grad_output"):
        out[k] = pr[k].to(dtype)
    return out
