"""Training drop-ins for the reference's MSDeformAttn ops package
(third_party/Mask2Former/mask2former/modeling/pixel_decoder/ops: the native module MultiScaleDeformableAttention,
the autograd Function and the nn.Module).

    from odise_b200.msda import MSDA          # in place of: import MultiScaleDeformableAttention as MSDA
    from odise_b200.msda import MSDeformAttn  # in place of: from .ops.modules import MSDeformAttn

MSDA exposes the native module's two entry points with its arguments and results, for float32 and float64 CUDA tensors;
MSDeformAttnFunction is the autograd Function of ops/functions/ms_deform_attn_func.py:32-49 on top of them.
MSDeformAttnFusedFunction differentiates the fused op (odise_msda_fused_f32 / odise_msda_fused_backward_f32: softmax and
sampling locations computed inside the kernels, for 2-column reference points and for boxes; float16 and bfloat16 storage
under autocast), and MSDeformAttn is the
module of ops/modules/ms_deform_attn.py, which takes the fused op where it applies.  All of them run the library's sm_90a
kernels; there is no CPU path.  Under torch.use_deterministic_algorithms(True) every backward here returns a
bit-reproducible grad_value (fixed-point sums, lib's deterministic=True); the other gradients are deterministic anyway.
They reach the kernels through four torch custom ops (torch.ops.odise_b200.msda_forward, msda_backward,
msda_fused_forward, msda_fused_backward) with fake implementations, so torch.compile (fullgraph=True included) and
torch.export trace them without a graph break."""
import math
import warnings

import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib


_LOW = (torch.float16, torch.bfloat16)


# The kernels as torch custom ops (lib.custom_op).  lib's functions are looked up at call time, so that a test that
# patches them sees every call.
def _msda_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
    fwd = lib.msda_forward_f64 if value.dtype == torch.float64 else lib.msda_forward
    return fwd(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step)


def _msda_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, im2col_step,
                   deterministic):
    return tuple(lib.msda_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                                   im2col_step, deterministic=deterministic))


def _msda_fused_forward(value, spatial_shapes, level_start_index, reference_points, offsets, logits):
    fwd = lib.msda_fused_forward_16bit if value.dtype in _LOW else lib.msda_fused_forward
    return fwd(value, spatial_shapes, level_start_index, reference_points, offsets, logits)


def _msda_fused_backward(value, spatial_shapes, level_start_index, reference_points, offsets, logits, grad_output,
                         deterministic):
    bwd = lib.msda_fused_backward_16bit if value.dtype in _LOW else lib.msda_fused_backward
    return bwd(value, spatial_shapes, level_start_index, reference_points, offsets, logits, grad_output,
               deterministic=deterministic)


lib.custom_op("msda_forward(Tensor value, Tensor spatial_shapes, Tensor level_start_index, Tensor sampling_loc, "
              "Tensor attn_weight, int im2col_step) -> Tensor", _msda_forward)
lib.custom_op("msda_backward(Tensor value, Tensor spatial_shapes, Tensor level_start_index, Tensor sampling_loc, "
              "Tensor attn_weight, Tensor grad_output, int im2col_step, bool deterministic) -> (Tensor, Tensor, Tensor)",
              _msda_backward)
lib.custom_op("msda_fused_forward(Tensor value, Tensor spatial_shapes, Tensor level_start_index, "
              "Tensor reference_points, Tensor offsets, Tensor logits) -> Tensor", _msda_fused_forward)
lib.custom_op("msda_fused_backward(Tensor value, Tensor spatial_shapes, Tensor level_start_index, "
              "Tensor reference_points, Tensor offsets, Tensor logits, Tensor grad_output, bool deterministic) "
              "-> (Tensor, Tensor, Tensor)", _msda_fused_backward)


class MSDA:
    """Stand-in for the pybind module: ms_deform_attn_forward / ms_deform_attn_backward (ops/src/vision.cpp:19-20)."""

    @staticmethod
    def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
        return torch.ops.odise_b200.msda_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                                                 im2col_step)

    @staticmethod
    def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                                im2col_step):
        """Under torch.use_deterministic_algorithms(True) (warn_only too) grad_value is summed in fixed point and is
        bit-reproducible; otherwise float atomics, as in the reference.  Under torch.compile the switch is read when the
        graph is traced (Dynamo guards on it: flipping it recompiles)."""
        return list(torch.ops.odise_b200.msda_backward(value, spatial_shapes, level_start_index, sampling_loc,
                                                       attn_weight, grad_output, im2col_step,
                                                       torch.are_deterministic_algorithms_enabled()))


class MSDeformAttnFunction(Function):
    """MSDeformAttnFunction of ms_deform_attn_func.py:32-49: gradients for value, sampling_locations and
    attention_weights; None for the spatial shapes, the level start index and im2col_step."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights,
                im2col_step):
        ctx.im2col_step = im2col_step
        output = MSDA.ms_deform_attn_forward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                                             attention_weights, ctx.im2col_step)
        ctx.save_for_backward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                              attention_weights)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights = ctx.saved_tensors
        grad_value, grad_sampling_loc, grad_attn_weight = MSDA.ms_deform_attn_backward(
            value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights,
            grad_output.contiguous(), ctx.im2col_step)
        return grad_value, None, None, grad_sampling_loc, grad_attn_weight, None


class MSDeformAttnFusedFunction(Function):
    """Autograd through the fused op: forward odise_msda_fused_f32, backward odise_msda_fused_backward_f32, or their
    16-bit forms (odise_msda_fused_f16 / _bf16 and the backward) when value is float16 or bfloat16.

    Inputs: value [N, S, M, D], spatial_shapes [L, 2], level_start_index [L], reference_points [N, Lq, L, 2] or boxes
    [N, Lq, L, 4] (cx, cy, w, h), offsets [N, Lq, M, L, P, 2] (raw output of the sampling_offsets linear) and logits
    [N, Lq, M, L*P] (raw output of the attention_weights linear); CUDA tensors, value / offsets / logits float32 or all of
    one 16-bit dtype, reference_points float32; D = 32 and L*P <= 32 for the backward (and for the 16-bit and the box
    forward).  Gradients for value, offsets and logits in their dtype.  For 2-column reference_points that require one,
    grad_ref[n, q, l] = sum over (m, p) of grad_offsets * (W_l, H_l), computed in float32.  Boxes get no gradient here:
    it cannot be recovered from grad_offsets without dividing by w and h, so forward raises RuntimeError for a box that
    requires grad (MSDeformAttn sends those to the composed path)."""

    @staticmethod
    def forward(ctx, value, spatial_shapes, level_start_index, reference_points, offsets, logits):
        if ctx.needs_input_grad[3] and lib._msda_box(reference_points):
            raise RuntimeError("MSDeformAttnFusedFunction: box reference points [N, Lq, L, 4] that require grad are not "
                               "supported by the fused op; detach them or use the composed path "
                               "(MSDeformAttn with use_fused = False)")
        output = torch.ops.odise_b200.msda_fused_forward(value, spatial_shapes, level_start_index, reference_points,
                                                         offsets, logits)
        ctx.save_for_backward(value, spatial_shapes, level_start_index, reference_points, offsets, logits)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, spatial_shapes, level_start_index, reference_points, offsets, logits = ctx.saved_tensors
        grad_value, grad_offsets, grad_logits = torch.ops.odise_b200.msda_fused_backward(
            value, spatial_shapes, level_start_index, reference_points, offsets, logits,
            grad_output.to(value.dtype).contiguous(), torch.are_deterministic_algorithms_enabled())
        grad_ref = None
        if ctx.needs_input_grad[3]:
            go = grad_offsets.float()
            wh = torch.stack([spatial_shapes[:, 1], spatial_shapes[:, 0]], -1).to(go)
            grad_ref = (go * wh[None, None, None, :, None, :]).sum((2, 4))
        return grad_value, None, None, grad_ref, grad_offsets, grad_logits


def _is_power_of_2(n):
    if not isinstance(n, int) or n < 0:
        raise ValueError(f"invalid input for _is_power_of_2: {n} (type: {type(n)})")
    return n != 0 and (n & (n - 1)) == 0


class MSDeformAttn(nn.Module):
    """Multi-scale deformable attention, the module of ops/modules/ms_deform_attn.py:34-125: same constructor, parameter
    names and shapes (state dicts load both ways), initialisation and forward signature.

    forward() runs MSDeformAttnFusedFunction (softmax, sampling locations and bilinear sampling in one kernel, and one
    kernel for their backward) for float32 CUDA inputs with 2-column reference points or 4-column boxes,
    D = d_model / n_heads = 32, n_levels * n_points <= 32 and S * d_model < 2^31.  A box that needs a gradient
    (grad mode on and reference_points.requires_grad) is the exception: the fused kernels return the gradient of the raw
    offsets, from which a box's own gradient cannot be recovered without dividing by w and h, so it takes the composed
    path.  Decoders that detach their boxes between layers (box refinement) stay fused, as does torch.no_grad.  Every
    other input (other D, float64, or use_fused = False) takes the reference's composition: softmax and locations in
    torch ops, then MSDeformAttnFunction.  CPU tensors raise: there is no CPU path.

    Under torch.autocast, or in a module cast to float16 / bfloat16, value, offsets and logits come out of the Linears in
    16 bits.  Where the fused conditions hold, the 16-bit fused kernels take them as they are (reference points cast to
    float32, which is exact) and return the value's dtype.  Elsewhere the composition runs in float32 on upcast inputs
    and its output is cast back to the value's dtype before output_proj, as the reference's grid_sample fallback does."""

    def __init__(self, d_model=256, n_levels=4, n_heads=8, n_points=4):
        super().__init__()
        if d_model % n_heads != 0:
            raise ValueError(f"d_model must be divisible by n_heads, but got {d_model} and {n_heads}")
        if not _is_power_of_2(d_model // n_heads):
            warnings.warn("MSDeformAttn: d_model / n_heads is not a power of 2; the CUDA kernels are most efficient "
                          "when it is")
        self.im2col_step = 128
        self.d_model, self.n_levels, self.n_heads, self.n_points = d_model, n_levels, n_heads, n_points
        self.use_fused = True          # False forces the composed path (for comparisons)
        self.sampling_offsets = nn.Linear(d_model, n_heads * n_levels * n_points * 2)
        self.attention_weights = nn.Linear(d_model, n_heads * n_levels * n_points)
        self.value_proj = nn.Linear(d_model, d_model)
        self.output_proj = nn.Linear(d_model, d_model)
        self._reset_parameters()

    def _reset_parameters(self):
        """Zero sampling_offsets.weight; its bias points head h in direction 2*pi*h / n_heads, scaled so that the larger
        of |x|, |y| is 1 and multiplied by point index + 1; zero attention_weights; xavier-uniform projections with zero
        biases."""
        M, L, P = self.n_heads, self.n_levels, self.n_points
        nn.init.constant_(self.sampling_offsets.weight, 0.0)
        theta = torch.arange(M, dtype=torch.float32) * (2.0 * math.pi / M)
        grid = torch.stack([theta.cos(), theta.sin()], -1)
        grid = grid / grid.abs().max(-1, keepdim=True)[0]
        grid = grid.view(M, 1, 1, 2).repeat(1, L, P, 1) * torch.arange(1, P + 1, dtype=torch.float32).view(1, 1, P, 1)
        with torch.no_grad():
            self.sampling_offsets.bias.copy_(grid.reshape(-1))
        nn.init.constant_(self.attention_weights.weight, 0.0)
        nn.init.constant_(self.attention_weights.bias, 0.0)
        nn.init.xavier_uniform_(self.value_proj.weight)
        nn.init.constant_(self.value_proj.bias, 0.0)
        nn.init.xavier_uniform_(self.output_proj.weight)
        nn.init.constant_(self.output_proj.bias, 0.0)

    def forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask=None):
        """query [N, Lq, C]; reference_points [N, Lq, L, 2] in [0, 1] (x, y) or [N, Lq, L, 4] boxes (x, y, w, h);
        input_flatten [N, S, C] with S = sum of H_l * W_l; input_spatial_shapes [L, 2] (H_l, W_l);
        input_level_start_index [L]; input_padding_mask [N, S], True at padding -> [N, Lq, C]."""
        return self._attend(query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                            input_padding_mask, check_shapes=True)

    def _attend(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask, check_shapes):
        """forward(); check_shapes = False skips its host read of input_spatial_shapes (a synchronisation), for callers
        that built the shapes from the same ints as input_flatten (odise_b200.pixel_decoder's encoder layers)"""
        if not (query.is_cuda and input_flatten.is_cuda and reference_points.is_cuda):
            raise lib.OdiseError("MSDeformAttn: expected CUDA tensors (odise_b200 kernels only run on the GPU)")
        N, Lq, _ = query.shape
        _, S, _ = input_flatten.shape
        # reads the shapes on the host, which a traced graph cannot: skipped there
        if check_shapes and not torch.compiler.is_compiling():
            assert (input_spatial_shapes[:, 0] * input_spatial_shapes[:, 1]).sum() == S
        M, L, P = self.n_heads, self.n_levels, self.n_points
        D = self.d_model // M
        if reference_points.shape[-1] not in (2, 4):
            raise ValueError(f"Last dim of reference_points must be 2 or 4, but get {reference_points.shape[-1]} "
                             "instead.")

        value = self.value_proj(input_flatten)
        if input_padding_mask is not None:
            value = value.masked_fill(input_padding_mask[..., None], 0.0)
        value = value.view(N, S, M, D)
        offsets = self.sampling_offsets(query).view(N, Lq, M, L, P, 2)
        logits = self.attention_weights(query).view(N, Lq, M, L * P)
        low = value.dtype in _LOW
        # float32 needs float32 reference points; a 16-bit value takes them in float32 or 16 bits (cast exactly below)
        ref_ok = reference_points.dtype in ((torch.float32,) + _LOW if low else (torch.float32,))
        # a box that needs a gradient stays composed (MSDeformAttnFusedFunction has no box gradient)
        box_grad = reference_points.shape[-1] == 4 and torch.is_grad_enabled() and reference_points.requires_grad
        fused = (self.use_fused and (value.dtype == torch.float32 or low) and offsets.dtype == logits.dtype == value.dtype
                 and ref_ok and not box_grad and D == 32 and L * P <= 32 and S * M * D < 2 ** 31)
        if fused:
            ref = reference_points.to(torch.float32).contiguous()
            if ref.shape[-1] == 4:     # here grad mode is off or the box needs no gradient
                ref = ref.detach()
                # a view that the box kernels' 16-byte loads cannot read is copied.  Dynamo cannot trace
                # storage_offset(), so a traced graph leaves the check to the op's fake implementation (lib's validator)
                if not torch.compiler.is_compiling() and ref.storage_offset() % 4:
                    ref = ref.clone()
            output = MSDeformAttnFusedFunction.apply(value, input_spatial_shapes, input_level_start_index, ref, offsets,
                                                     logits)
        else:
            out_dtype = value.dtype
            if low:                    # sample in float32 (what the reference's grid_sample fallback does under autocast)
                value, offsets, logits = value.float(), offsets.float(), logits.float()
                reference_points = reference_points.float()
            attention_weights = F.softmax(logits, -1).view(N, Lq, M, L, P)
            if reference_points.shape[-1] == 2:
                wh = torch.stack([input_spatial_shapes[..., 1], input_spatial_shapes[..., 0]], -1)
                sampling_locations = reference_points[:, :, None, :, None, :] + offsets / wh[None, None, None, :, None, :]
            else:
                sampling_locations = (reference_points[:, :, None, :, None, :2]
                                      + offsets / P * reference_points[:, :, None, :, None, 2:] * 0.5)
            output = MSDeformAttnFunction.apply(value, input_spatial_shapes, input_level_start_index,
                                                sampling_locations, attention_weights, self.im2col_step)
            if low:
                output = output.to(out_dtype)
        return self.output_proj(output)
