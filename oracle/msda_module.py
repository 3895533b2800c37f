"""Oracle side of the MSDeformAttn module drop-in and of the fused op's backward (CPU, torch fp64).  TEST INFRASTRUCTURE
ONLY.

fused_problem() / oracle_fused_grads(): oracle/msda_grad.py's gradient problems expressed as inputs of the fused op (raw
offsets and logits + reference points) and their fp64 autograd through msdeformattn_front and oracle.msda.msda_forward.
module_problem() / oracle_module_grads(): the whole MSDeformAttn module (ops/modules/ms_deform_attn.py:34-125), pinned
against the reference's own module by tests/test_msda_module_cpu.py.  Why samples are kept off cell edges: see the
docstring of oracle/msda_grad.py.
"""
import torch
import torch.nn.functional as F

from .msda import msda_forward, msdeformattn_front
from .msda_grad import grad_problem


# ---- module level: MSDeformAttn (ops/modules/ms_deform_attn.py:34-125) --------------------------------------------------
# The module's sampling offsets are outputs of a Linear, so locations cannot be placed one by one as in grad_problem().
# module_problem() starts from the reference's own initial state instead: sampling_offsets.weight = 0 (the offsets are the
# bias), reference points from the pixel decoder's grid (msdeformattn.py:141-153, valid ratios 1), and a bias whose
# fractional parts in pixel units keep every sample coordinate off a cell edge on every level.

MODULE_PARAMS = ("sampling_offsets.weight", "sampling_offsets.bias", "attention_weights.weight", "attention_weights.bias",
                 "value_proj.weight", "value_proj.bias", "output_proj.weight", "output_proj.bias")


def grid_reference_points(shapes, N, dtype=torch.float64):
    """Reference points of MSDeformAttnTransformerEncoder.get_reference_points with valid ratios 1: the centre of every
    pixel of every level, in level order, repeated over the levels -> [N, S, L, 2] (x, y)."""
    pts = []
    for H, W in shapes:
        y, x = torch.meshgrid(torch.linspace(0.5, H - 0.5, H, dtype=dtype), torch.linspace(0.5, W - 0.5, W, dtype=dtype),
                              indexing="ij")
        pts.append(torch.stack((x.reshape(-1) / W, y.reshape(-1) / H), -1))
    ref = torch.cat(pts, 0)
    return ref[None, :, None, :].expand(N, -1, len(shapes), -1).contiguous()


def _best_fraction(coords):
    """(c, d): the shift c in [0, 1) that keeps coords + c farthest from an integer, and that distance d."""
    frac = torch.unique(torch.remainder(coords.reshape(-1), 1.0))
    cand = torch.arange(1024, dtype=torch.float64) / 1024
    x = torch.remainder(frac[None, :] + cand[:, None], 1.0)
    dist = torch.minimum(x, 1 - x).min(1).values
    i = int(dist.argmax())
    return float(cand[i]), float(dist[i])


def module_problem(seed, N, d_model, n_heads, shapes, n_points, box=False, padding=False, dtype=torch.float64):
    """Seeded inputs of one MSDeformAttn call in the encoder's setting (queries = the S pixels of all levels) -> dict:
    params (the module's state dict), query [N, S, C], reference_points [N, S, L, 2] (box: [N, S, L, 4] with
    (w, h) = (2P / W_l, 2P / H_l), which puts the samples where the 2-column form does), input_flatten [N, S, C],
    spatial_shapes, level_start_index, padding_mask ([N, S] bool, about 20 % True, or None), grad_output [N, S, C].
    Every sample coordinate lies at least 0.02 px from a cell edge (sample_margin() measures it)."""
    g = torch.Generator().manual_seed(seed)
    M, L, P, C = n_heads, len(shapes), n_points, d_model
    ss = torch.as_tensor(shapes, dtype=torch.long)
    lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
    S = int(ss.prod(1).sum())
    ref = grid_reference_points(shapes, N)
    # bias = the reference's directional grid rounded to whole pixels + a random whole shift + the best fraction per
    # (level, axis) + a jitter that keeps 0.02 px of margin
    theta = torch.arange(M, dtype=torch.float64) * (2.0 * torch.pi / M)
    grid = torch.stack([theta.cos(), theta.sin()], -1)
    grid = (grid / grid.abs().max(-1, keepdim=True)[0]).view(M, 1, 1, 2) * torch.arange(1, P + 1).view(1, 1, P, 1)
    bias = torch.round(grid.expand(M, L, P, 2)) + torch.randint(-1, 2, (M, L, P, 2), generator=g).to(torch.float64)
    for l, (H, W) in enumerate(shapes):
        for a, size in ((0, W), (1, H)):
            c, d = _best_fraction(ref[0, :, l, a] * size - 0.5)
            jit = max(d - 0.02, 0.0) * 0.5
            bias[:, l, :, a] += c + jit * (2 * torch.rand(M, P, generator=g, dtype=torch.float64) - 1)
    rnd = lambda *s, scale=1.0: torch.randn(*s, generator=g, dtype=torch.float64) * scale  # noqa: E731
    params = {
        "sampling_offsets.weight": torch.zeros(M * L * P * 2, C, dtype=torch.float64),
        "sampling_offsets.bias": bias.reshape(-1),
        "attention_weights.weight": rnd(M * L * P, C, scale=C ** -0.5),
        "attention_weights.bias": rnd(M * L * P, scale=0.5),
        "value_proj.weight": rnd(C, C, scale=C ** -0.5), "value_proj.bias": rnd(C, scale=0.1),
        "output_proj.weight": rnd(C, C, scale=C ** -0.5), "output_proj.bias": rnd(C, scale=0.1),
    }
    if box:
        wh = torch.stack([2.0 * P / ss[:, 1].double(), 2.0 * P / ss[:, 0].double()], -1)      # [L, 2]
        ref = torch.cat([ref, wh[None, None].expand(N, S, L, 2)], -1)
    mask = torch.rand(N, S, generator=g) < 0.2 if padding else None
    out = dict(params=params, query=rnd(N, S, C), reference_points=ref, input_flatten=rnd(N, S, C), spatial_shapes=ss,
               level_start_index=lsi, padding_mask=mask, grad_output=rnd(N, S, C))
    cast = lambda t: t.to(dtype) if torch.is_tensor(t) and t.is_floating_point() else t  # noqa: E731
    out["params"] = {k: cast(v) for k, v in params.items()}
    return {k: (cast(v) if k != "params" else v) for k, v in out.items()}


def _locations(reference_points, offsets, spatial_shapes, M, L, P):
    """sampling locations of ms_deform_attn.py:106-113 for both reference-point forms; offsets [N, Lq, M*L*P*2]."""
    N, Lq = offsets.shape[:2]
    off = offsets.view(N, Lq, M, L, P, 2)
    if reference_points.shape[-1] == 2:
        wh = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1).to(off.dtype)
        return reference_points[:, :, None, :, None, :] + off / wh[None, None, None, :, None, :]
    return reference_points[:, :, None, :, None, :2] + off / P * reference_points[:, :, None, :, None, 2:] * 0.5


def sample_margin(params, query, reference_points, spatial_shapes, n_heads, n_points):
    """Smallest distance in pixels, over every sample and both axes, from the sample's pixel coordinate
    (loc * size - 0.5) to a cell edge, in fp64 for the given parameters."""
    M, L, P = n_heads, spatial_shapes.shape[0], n_points
    with torch.no_grad():
        off = F.linear(query.double().cpu(), params["sampling_offsets.weight"].double().cpu(),
                       params["sampling_offsets.bias"].double().cpu())
        loc = _locations(reference_points.double().cpu(), off, spatial_shapes.cpu(), M, L, P)
        size = torch.stack([spatial_shapes[:, 1], spatial_shapes[:, 0]], -1).double().cpu()    # (W, H)
        px = loc * size[None, None, None, :, None, :] - 0.5
        return (px - torch.round(px)).abs().min().item()


def oracle_module_grads(params, query, reference_points, input_flatten, spatial_shapes, level_start_index,
                        padding_mask, grad_output, n_heads, n_points, ref_grad=False):
    """MSDeformAttn.forward in fp64 on the CPU (the four linears, msdeformattn_front or the box form of the locations,
    oracle.msda.msda_forward) and its torch autograd -> (output, grads): grads maps every parameter name, "query",
    "input_flatten" and (ref_grad) "reference_points" to its gradient for grad_output."""
    M, L, P = n_heads, spatial_shapes.shape[0], n_points
    p = {k: v.detach().double().cpu().requires_grad_(True) for k, v in params.items()}
    q, x = (t.detach().double().cpu().requires_grad_(True) for t in (query, input_flatten))
    ref = reference_points.detach().double().cpu().requires_grad_(ref_grad)
    ss, lsi = spatial_shapes.cpu(), level_start_index.cpu()
    N, Lq, C = q.shape
    S = x.shape[1]
    value = F.linear(x, p["value_proj.weight"], p["value_proj.bias"])
    if padding_mask is not None:
        value = value.masked_fill(padding_mask.cpu()[..., None], 0.0)
    value = value.view(N, S, M, C // M)
    off = F.linear(q, p["sampling_offsets.weight"], p["sampling_offsets.bias"])
    logits = F.linear(q, p["attention_weights.weight"], p["attention_weights.bias"])
    if ref.shape[-1] == 2:
        loc, aw = msdeformattn_front(None, ref, off, logits, ss, M, L, P)
    else:
        loc = _locations(ref, off, ss, M, L, P)
        aw = torch.softmax(logits.view(N, Lq, M, L * P), -1).view(N, Lq, M, L, P)
    out = F.linear(msda_forward(value, ss, lsi, loc, aw), p["output_proj.weight"], p["output_proj.bias"])
    names = list(MODULE_PARAMS) + ["query", "input_flatten"] + (["reference_points"] if ref_grad else [])
    leaves = [p[k] for k in MODULE_PARAMS] + [q, x] + ([ref] if ref_grad else [])
    grads = torch.autograd.grad(out, leaves, grad_output.double().cpu())
    return out.detach(), dict(zip(names, grads))


def fused_problem(seed, N, M, D, shapes, Lq, P, small_values=False, far=False, dtype=torch.float64):
    """grad_problem()'s locations expressed as inputs of the fused op -> value, spatial_shapes, level_start_index,
    reference_points [N, Lq, L, 2] (in [0.4, 0.6]), offsets [N, Lq, M, L, P, 2] with ref + off / (W, H) = the location,
    logits [N, Lq, M, L*P], grad_output."""
    value, ss, lsi, loc, _, go = grad_problem(seed, N, M, D, shapes, Lq, P, small_values=small_values, far=far)
    g = torch.Generator().manual_seed(seed + 1000)
    L = len(shapes)
    ref = torch.rand(N, Lq, L, 2, generator=g, dtype=torch.float64) * 0.2 + 0.4
    wh = torch.stack([ss[:, 1], ss[:, 0]], -1).double()
    offs = (loc - ref[:, :, None, :, None, :]) * wh[None, None, None, :, None, :]
    logits = torch.randn(N, Lq, M, L * P, generator=g, dtype=torch.float64) * 2
    return tuple(t.to(dtype) if t.is_floating_point() else t for t in (value, ss, lsi, ref, offs, logits, go))


def oracle_fused_grads(value, spatial_shapes, level_start_index, reference_points, offsets, logits, grad_output,
                       ref_grad=False):
    """[grad_value, grad_offsets, grad_logits] (+ grad_reference_points with ref_grad) of the fused op (softmax and
    locations of msdeformattn_front, then oracle.msda.msda_forward) by torch autograd in fp64."""
    v, off, lg = (t.detach().double().requires_grad_(True) for t in (value, offsets, logits))
    ref = reference_points.detach().double().requires_grad_(ref_grad)
    N, Lq, M, L, P, _ = off.shape
    loc, aw = msdeformattn_front(None, ref, off.reshape(N, Lq, -1), lg.reshape(N, Lq, -1), spatial_shapes, M, L, P)
    out = msda_forward(v, spatial_shapes, level_start_index, loc, aw)
    leaves = (v, off, lg) + ((ref,) if ref_grad else ())
    return list(torch.autograd.grad(out, leaves, grad_output.double()))
