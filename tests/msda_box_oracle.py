"""Box reference points (cx, cy, w, h) for the fused MSDeformAttn oracles.  TEST INFRASTRUCTURE ONLY.

The box forms of oracle/msda_module.py's fused_problem / oracle_fused_grads and of oracle/msda_16bit.py's
fused_problem_16bit / oracle_fused_forward, built on those modules and on the same rules: grad_problem()'s sampling
locations (each coordinate an integer cell plus a fraction in [0.02, 0.98], see oracle/msda_grad.py), expressed as the
raw offsets of a box, loc = ref.xy + off / P * ref.wh * 0.5 (ms_deform_attn.py:110-112, oracle.msda_module._locations).
"""
import torch

from oracle.msda import msda_forward
from oracle.msda_16bit import MARGIN, ulp
from oracle.msda_grad import grad_problem
from oracle.msda_module import _locations


def fused_problem_box(seed, N, M, D, shapes, Lq, P, small_values=False, far=False, dtype=torch.float64):
    """-> value, spatial_shapes, level_start_index, reference_points [N, Lq, L, 4], offsets [N, Lq, M, L, P, 2], logits,
    grad_output, as oracle.msda_module.fused_problem but with boxes: centres in [0.3, 0.7], w and h in [0.05, 0.6], and
    about one box in eight with w = 0 and one in eight with h = 0 (never both).  The offsets are solved so that the fp64
    location is grad_problem()'s; along a degenerate axis every sample sits at the centre, which is drawn 0.02-0.98 px
    into a cell (its offset is random and moves nothing).  Every sample keeps MARGIN px from a cell edge at the locations
    computed in float32 from the inputs rounded to `dtype` (asserted for float32; the 16-bit form steps offsets)."""
    value, ss, lsi, loc, _, go = grad_problem(seed, N, M, D, shapes, Lq, P, small_values=small_values, far=far)
    g = torch.Generator().manual_seed(seed + 2000)
    L = len(shapes)
    size = torch.stack([ss[:, 1], ss[:, 0]], -1).double()                      # (W, H) per level
    centre = torch.rand(N, Lq, L, 2, generator=g, dtype=torch.float64) * 0.4 + 0.3
    wh = torch.rand(N, Lq, L, 2, generator=g, dtype=torch.float64) * 0.55 + 0.05
    u = torch.rand(N, Lq, L, generator=g, dtype=torch.float64)
    flat = torch.stack([u < 0.125, (u >= 0.125) & (u < 0.25)], -1)            # w = 0 | h = 0
    wh = torch.where(flat, torch.zeros_like(wh), wh)
    # a degenerate axis samples at its centre: put the centre 0.02-0.98 px into a cell
    cell = torch.floor(centre * size - 0.5)
    frac = 0.02 + 0.96 * torch.rand(N, Lq, L, 2, generator=g, dtype=torch.float64)
    centre = torch.where(flat, (cell + frac + 0.5) / size, centre)
    c, s = centre[:, :, None, :, None, :], wh[:, :, None, :, None, :]
    raw = torch.randn(N, Lq, M, L, P, 2, generator=g, dtype=torch.float64) * P
    offs = torch.where(s > 0, (loc - c) * P / torch.where(s > 0, s * 0.5, torch.ones_like(s)), raw)
    ref = torch.cat([centre, wh], -1)
    logits = torch.randn(N, Lq, M, L * P, generator=g, dtype=torch.float64) * 2
    out = tuple(t.to(dtype) if t.is_floating_point() else t for t in (value, ss, lsi, ref, offs, logits, go))
    if dtype == torch.float32:
        assert box_sample_margin(out[3], out[4], ss) >= MARGIN
    return out


def box_locations_fp32(reference_points, offsets):
    """the float32 box locations [N, Lq, M, L, P, 2] the kernels sample at, with the roundings of the composed path's
    torch ops on the device: `offsets / P` by a CUDA tensor is the product with the float32 reciprocal of P (on the CPU
    torch divides exactly, so the reciprocal is formed here explicitly), then * w, * 0.5 and the sum with the centre"""
    P = offsets.shape[4]
    ref = reference_points.float()[:, :, None, :, None, :]
    inv_p = torch.ones((), dtype=torch.float32) / P                     # 1/P rounded once to float32
    return ref[..., :2] + offsets.float() * inv_p * ref[..., 2:] * 0.5


def box_pixel_coords(reference_points, offsets, spatial_shapes):
    """pixel coordinates loc * size - 0.5 [N, Lq, M, L, P, 2] (fp64) of box_locations_fp32"""
    loc = box_locations_fp32(reference_points, offsets)
    size = torch.stack([spatial_shapes[:, 1], spatial_shapes[:, 0]], -1).double()[None, None, None, :, None, :]
    return loc.double() * size - 0.5


def box_edge_distance(reference_points, offsets, spatial_shapes):
    """distance in px of every sample coordinate from the nearest cell edge; samples outside (-2, size + 1) in either
    axis read nothing and count as infinitely far (as oracle.msda_16bit.edge_distance)"""
    px = box_pixel_coords(reference_points, offsets, spatial_shapes)
    size = torch.stack([spatial_shapes[:, 1], spatial_shapes[:, 0]], -1).double()[None, None, None, :, None, :]
    d = (px - torch.round(px)).abs()
    outside = ((px <= -2) | (px >= size + 1)).any(-1, keepdim=True).expand_as(d)
    return torch.where(outside, torch.full_like(d, float("inf")), d)


def box_sample_margin(reference_points, offsets, spatial_shapes):
    return box_edge_distance(reference_points, offsets, spatial_shapes).min().item()


def keep_box_off_edges(reference_points, offsets, spatial_shapes, dtype, max_steps=64):
    """oracle.msda_16bit.keep_off_edges for boxes: offsets (fp64 values representable in dtype) within MARGIN px of a
    cell edge are stepped by whole ulps of dtype, +1, -1, +2, -2, ... until every sample keeps the margin"""
    offs, base = offsets.clone(), offsets.clone()
    for k in range(1, max_steps + 1):
        bad = box_edge_distance(reference_points, offs, spatial_shapes) < MARGIN
        if not bad.any():
            return offs
        step = (k + 1) // 2 * (1 if k % 2 else -1)
        offs = torch.where(bad, (base + step * ulp(base, dtype)).to(dtype).double(), offs)
    raise AssertionError("keep_box_off_edges: no 16-bit offset within reach keeps the margin")


def fused_problem_box_16bit(seed, N, M, D, shapes, Lq, P, dtype, small_values=False, far=False):
    """fused_problem_box() rounded to what the 16-bit kernels read (as oracle.msda_16bit.fused_problem_16bit): value,
    offsets, logits and grad_output in dtype, boxes in float32.  The margin is asserted on the float32 locations."""
    value, ss, lsi, ref, offs, logits, go = fused_problem_box(seed, N, M, D, shapes, Lq, P, small_values=small_values,
                                                              far=far)
    ref32 = ref.to(torch.float32)
    offs16 = keep_box_off_edges(ref32, offs.to(dtype).double(), ss, dtype).to(dtype)
    assert box_sample_margin(ref32, offs16, ss) >= MARGIN
    return value.to(dtype), ss, lsi, ref32, offs16, logits.to(dtype), go.to(dtype)


def _front(reference_points, offsets, logits, spatial_shapes, fp32_locations=False):
    """fp64 locations and softmax weights.  fp32_locations (boxes): the location values are the float32 ones the kernel
    samples at (box_locations_fp32), with the fp64 derivative w / (2P) of the offsets"""
    N, Lq, M, L, P, _ = offsets.shape
    loc = _locations(reference_points, offsets.reshape(N, Lq, -1), spatial_shapes, M, L, P)
    if fp32_locations:
        loc = box_locations_fp32(reference_points, offsets.detach()).double() + (loc - loc.detach())
    aw = torch.softmax(logits.reshape(N, Lq, M, L * P), -1).view(N, Lq, M, L, P)
    return loc, aw


def oracle_fused_forward(value, spatial_shapes, level_start_index, reference_points, offsets, logits,
                         fp32_locations=False):
    """the fused op's output [N, Lq, M*D] in fp64 for either reference-point width: _locations and the softmax, then
    oracle.msda.msda_forward"""
    loc, aw = _front(reference_points.double(), offsets.double(), logits.double(), spatial_shapes, fp32_locations)
    return msda_forward(value.double(), spatial_shapes, level_start_index, loc, aw)


def oracle_fused_grads(value, spatial_shapes, level_start_index, reference_points, offsets, logits, grad_output,
                       fp32_locations=False):
    """[grad_value, grad_offsets, grad_logits] of the fused op for either reference-point width, by fp64 autograd.
    fp32_locations=True evaluates at the float32 box locations the kernel computes (box_locations_fp32), so that a
    float32 test measures the sampling and its backward rather than the rounding of the location arithmetic, which
    tests/test_gpu_msda_box.py checks against the composed path's torch ops"""
    v, off, lg = (t.detach().double().requires_grad_(True) for t in (value, offsets, logits))
    loc, aw = _front(reference_points.detach().double(), off, lg, spatial_shapes, fp32_locations)
    out = msda_forward(v, spatial_shapes, level_start_index, loc, aw)
    return list(torch.autograd.grad(out, (v, off, lg), grad_output.double()))
