"""TEST / BENCH INFRASTRUCTURE (not shipped, not imported by odise_b200/).

ctypes binding of oracle/_ref/libref_msda.so = the REFERENCE's own MSDeformAttn forward CUDA kernel
(ops/src/cuda/ms_deform_im2col_cuda.cuh:242-304, launcher :928-958) compiled unmodified for sm_90a by oracle/Makefile
behind the C shim oracle/ref_msda_host.cu.  Used as (1) a second parity oracle for odise_msda_forward_f32 and (2) the GPU
baseline the engine's kernel has to beat in the C4 microbench (bench.py --config c4)."""
import ctypes
import os

import torch

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libref_msda.so")
_lib = None


def available():
    return os.path.exists(_PATH)


def _load():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(_PATH)
        _lib.ref_ms_deform_attn_forward_f32.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_int] * 8 + [ctypes.c_void_p]
        _lib.ref_ms_deform_attn_forward_f32.restype = ctypes.c_int
    return _lib


def forward(value, spatial_shapes, level_start_index, sampling_locations, attention_weights, im2col_step=128, out=None):
    """Same arguments as MSDA.ms_deform_attn_forward (ops/src/vision.cpp:19); CUDA fp32 contiguous tensors."""
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_locations.shape
    if out is None:
        out = torch.empty(N, Lq, M * D, dtype=torch.float32, device=value.device)
    rc = _load().ref_ms_deform_attn_forward_f32(
        value.data_ptr(), spatial_shapes.data_ptr(), level_start_index.data_ptr(), sampling_locations.data_ptr(),
        attention_weights.data_ptr(), out.data_ptr(), N, S, M, D, L, Lq, P, im2col_step,
        torch.cuda.current_stream().cuda_stream)
    if rc:
        raise RuntimeError(f"reference ms_deform_attn_forward failed with code {rc}")
    return out
