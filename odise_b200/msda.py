"""Training drop-in for the reference's only native module, MultiScaleDeformableAttention
(third_party/Mask2Former/mask2former/modeling/pixel_decoder/ops/src/vision.cpp:18-21).

    from odise_b200.msda import MSDA          # in place of: import MultiScaleDeformableAttention as MSDA

MSDA exposes the module's two entry points with its arguments and results, for float32 and float64 CUDA tensors;
MSDeformAttnFunction is the autograd Function of ops/functions/ms_deform_attn_func.py:32-49 on top of them.  Both run
the library's sm_90a kernels (odise_msda_forward_* / odise_msda_backward_*); there is no CPU path."""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib


class MSDA:
    """Stand-in for the pybind module: ms_deform_attn_forward / ms_deform_attn_backward (ops/src/vision.cpp:19-20)."""

    @staticmethod
    def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
        if value.dtype == torch.float64:
            return lib.msda_forward_f64(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step)
        return lib.msda_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step)

    @staticmethod
    def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                                im2col_step):
        return lib.msda_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                                 im2col_step)


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
