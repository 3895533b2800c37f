"""TEST / BENCH INFRASTRUCTURE (not shipped, not imported by odise_b200/).

ctypes binding of oracle/_ref/libref_msda_backward.so = the REFERENCE's own MSDeformAttn backward CUDA kernels
(ops/src/cuda/ms_deform_im2col_cuda.cuh, launcher ms_deformable_col2im_cuda) compiled unmodified for sm_90a by
oracle/backward.mk behind the C shim oracle/ref_msda_backward_host.cu.  Used as (1) a parity oracle for
odise_msda_backward_f32 (tools/make_golden_msda_ref_backward.py) and (2) the GPU baseline of
tools/msda_backward_bench.py."""
import ctypes
import os

import torch

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libref_msda_backward.so")
_lib = None


def available():
    return os.path.exists(_PATH)


def _load():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(_PATH)
        _lib.ref_ms_deform_attn_backward_f32.argtypes = [ctypes.c_void_p] * 9 + [ctypes.c_int] * 8 + [ctypes.c_void_p]
        _lib.ref_ms_deform_attn_backward_f32.restype = ctypes.c_int
    return _lib


def backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, im2col_step=128,
             out=None):
    """Same arguments and result as MSDA.ms_deform_attn_backward (ops/src/vision.cpp:20): [grad_value, grad_loc,
    grad_attn]; CUDA fp32 contiguous tensors.  out: optional preallocated (grad_value, grad_loc, grad_attn)."""
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_loc.shape
    gv, gl, ga = out if out is not None else (torch.empty_like(value), torch.empty_like(sampling_loc),
                                              torch.empty_like(attn_weight))
    rc = _load().ref_ms_deform_attn_backward_f32(
        value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(), sampling_loc.data_ptr(),
        attn_weight.data_ptr(), grad_output.data_ptr(), gv.data_ptr(), gl.data_ptr(), ga.data_ptr(),
        N, S, M, D, L, Lq, P, im2col_step, torch.cuda.current_stream().cuda_stream)
    if rc:
        raise RuntimeError(f"reference ms_deform_attn_backward failed with code {rc}")
    return [gv, gl, ga]
