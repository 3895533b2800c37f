"""ctypes binding of libodise_b200.so (include/odise_b200.h).

PyTorch is used for device memory and streams only; every op here launches hand-written sm_90a kernels through
the C ABI.  There is NO fallback: if the library is missing or a call fails, an exception is raised.
"""
import ctypes
import os
from ctypes import c_int, c_float, c_longlong, c_void_p, POINTER

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libodise_b200.so")

ACT_NONE, ACT_RELU, ACT_SILU, ACT_GELU, ACT_QUICKGELU = 0, 1, 2, 3, 4


class OdiseError(RuntimeError):
    pass


class GemmDesc(ctypes.Structure):
    _fields_ = [
        ("M", c_int), ("N", c_int), ("K", c_int), ("batch", c_int),
        ("nmma", c_int), ("conv3x3", c_int),
        ("conv_C", c_int), ("conv_H", c_int), ("conv_W", c_int),
        ("a_hi", c_void_p), ("a_lo", c_void_p), ("lda", c_longlong), ("a_batch_stride", c_longlong),
        ("b_hi", c_void_p), ("b_lo", c_void_p), ("ldb", c_longlong), ("b_batch_stride", c_longlong),
        ("alpha", c_float),
        ("bias", c_void_p),
        ("rowbias", c_void_p), ("rows_per_group", c_int), ("rowbias_ld", c_longlong),
        ("act", c_int),
        ("residual", c_void_p), ("ld_residual", c_longlong), ("residual_batch_stride", c_longlong),
        ("out_f32", c_void_p), ("ld_out", c_longlong), ("out_batch_stride", c_longlong),
        ("out_hi", c_void_p), ("out_lo", c_void_p), ("ld_out_bf16", c_longlong), ("out_bf16_batch_stride", c_longlong),
        ("split_k", c_int), ("workspace", c_void_p), ("workspace_bytes", c_longlong),
        ("force_bn", c_int),
        ("bias_m", c_void_p),
        ("conv_mode", c_int),
        ("geglu", c_int),
        ("gn_partial", c_void_p), ("gn_seg_stride", c_longlong), ("gn_plane_stride", c_longlong),
        ("out_planes_fp16", c_int),
    ]


_lib = None

# name -> argtypes (all return int); kept in one place so tests can check every header symbol is bound
_SIGS = {
    "odise_msda_forward_f32": [c_void_p] * 6 + [c_int] * 7 + [c_void_p],
    "odise_msda_fused_f32": [c_void_p] * 9 + [c_int] * 7 + [c_void_p],
    "odise_gemm_bf16": [POINTER(GemmDesc), c_void_p],
    "odise_gemm_tile_policy": [c_int] * 6 + [c_void_p, c_void_p],
    "odise_profile_begin": [],
    "odise_profile_end": [c_void_p, c_void_p, c_void_p],
    "odise_split_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong, c_int, c_void_p],
    "odise_split_f16_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong, c_int, c_void_p],
    "odise_groupnorm_stats_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float,
                                  c_void_p],
    "odise_groupnorm_apply_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                  c_longlong, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int, c_int, c_void_p],
    "odise_groupnorm_finalize_seg_f32": [c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                         c_float, c_void_p],
    "odise_groupnorm_stats_bs_f32": [c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                     c_float, c_void_p],
    "odise_groupnorm_stats_ws_f32": [c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                     c_int, c_int, c_float, c_void_p],
    "odise_groupnorm_apply_bs_f32": [c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                     c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong,
                                     c_int, c_int, c_int, c_int, c_void_p],
    "odise_resize_nhwc_bs_f32": [c_void_p, c_longlong, c_longlong, c_void_p, c_longlong, c_longlong, c_int, c_int,
                                 c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "odise_groupnorm_apply_res_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_longlong, c_int, c_void_p, c_longlong, c_int, c_void_p, c_void_p, c_longlong,
                                      c_int, c_int, c_int, c_int, c_void_p],
    "odise_bcast_fma_f32": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "odise_rowscale_f32": [c_void_p, c_longlong, c_void_p, c_longlong, c_int, c_void_p],
    "odise_layernorm_f32": [c_void_p, c_longlong, c_void_p, c_longlong, c_void_p, c_void_p, c_float, c_void_p,
                            c_longlong, c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong, c_int,
                            c_void_p],
    "odise_geglu_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong, c_int, c_void_p],
    "odise_add_split_f32": [c_void_p, c_longlong, c_void_p, c_longlong, c_longlong, c_void_p, c_longlong, c_void_p,
                            c_void_p, c_longlong, c_longlong, c_int, c_void_p],
    "odise_upsample2x_split_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int, c_int,
                                   c_void_p],
    "odise_im2col3x3_split_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                  c_int, c_int, c_void_p],
    "odise_copy2d_f32": [c_void_p, c_longlong, c_void_p, c_longlong, c_longlong, c_int, c_float, c_int, c_void_p],
    "odise_resize_nhwc_f32": [c_void_p, c_longlong, c_void_p, c_longlong, c_int, c_int, c_int, c_int, c_int, c_int,
                              c_int, c_int, c_void_p],
    "odise_image_crops_u8_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "odise_image_crops_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "odise_clip_preprocess": [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "odise_crop_resize_bicubic": [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "odise_patchify_split_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "odise_nchw_to_nhwc_f32": [c_void_p, c_void_p, c_longlong, c_int, c_int, c_int, c_void_p],
    "odise_nhwc_to_nchw_f32": [c_void_p, c_longlong, c_void_p, c_int, c_int, c_int, c_void_p],
    "odise_attn_mask_bits_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "odise_mha_d32_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p,
                          c_void_p, c_longlong, c_int, c_int, c_int, c_int, c_float, c_void_p],
    "odise_mha_d32_ws_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_longlong, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p],
    "odise_mask_binarize_f32": [c_void_p, c_void_p, c_longlong, c_void_p, c_int, c_int, c_int, c_void_p],
    "odise_pool_normalize_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "odise_l2_normalize_split_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong, c_int,
                                     c_void_p],
    "odise_class_max_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_void_p],
    "odise_act_split_f32": [c_void_p, c_longlong, c_int, c_void_p, c_void_p, c_longlong, c_longlong, c_int, c_void_p],
    "odise_softmax_split_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong, c_int, c_int,
                                c_float, c_void_p],
    "odise_upsample_sigmoid_split_f32": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                         c_int, c_void_p, c_void_p],
    "odise_query_scores_f32": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                               c_float, c_void_p],
    "odise_panoptic_inference_f32": [c_void_p] * 9 + [c_int] * 7 + [ctypes.c_double, c_void_p, c_void_p],
    "odise_instance_inference_f32": [c_void_p] * 9 + [c_int] * 8 + [c_void_p, c_void_p],
    "odise_postprocess_fused_f32": [c_void_p, c_void_p, c_void_p, c_int] + [c_void_p] * 8 + [ctypes.c_double] + [c_void_p] * 7 +
                                   [c_int] * 9 + [c_void_p, c_void_p],
    "odise_set_carveout_policy": [c_int],
    "odise_set_operand_format": [c_int],
    "odise_get_operand_format": [],
    "odise_gather_rows_f32": [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_int, c_void_p, c_longlong, c_longlong,
                              c_int, c_void_p],
    "odise_maskclip_preprocess": [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "odise_maskclip_bits_f32": [c_void_p] * 3 + [c_int] * 8 + [c_void_p],
    "odise_open_vocab_merge_f32": [c_void_p, c_void_p, c_longlong, c_void_p, c_float, c_float, c_void_p, c_void_p, c_int,
                                   c_int, c_void_p],
    "odise_attention_tc": [c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p,
                           c_longlong, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_int,
                           c_int, c_int, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p],
}


def load():
    """Load the shared library (building is __graft_entry__.build()'s job). Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise OdiseError(
            f"{_LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(odise_b200 has no CPU / eager fallback)")
    lib = ctypes.CDLL(_LIB_PATH)
    lib.odise_version.restype = c_int
    lib.odise_launch_count.restype = c_longlong
    lib.odise_groupnorm_ws_floats.restype = c_longlong
    lib.odise_groupnorm_ws_floats.argtypes = [c_int, c_int, c_int, c_int]
    lib.odise_mha_d32_ws_floats.restype = c_longlong
    lib.odise_panoptic_ws_bytes.restype = c_longlong
    lib.odise_panoptic_ws_bytes.argtypes = [c_int, c_int, c_int, c_int]
    lib.odise_instance_ws_bytes.restype = c_longlong
    lib.odise_instance_ws_bytes.argtypes = [c_int, c_int, c_int, c_int]
    lib.odise_postprocess_fused_ws_bytes.restype = c_longlong
    lib.odise_postprocess_fused_ws_bytes.argtypes = [c_int, c_int, c_int, c_int]
    lib.odise_mha_d32_ws_floats.argtypes = [c_int, c_int, c_int, c_int]
    for name, args in _SIGS.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = c_int
    _lib = lib
    return lib


def launch_count():
    return int(load().odise_launch_count())


def _check(rc, what):
    if rc != 0:
        raise OdiseError(f"{what} failed with code {rc}")


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _req(t, dtype, name):
    if not t.is_cuda:
        raise OdiseError(f"{name}: expected a CUDA tensor (odise_b200 kernels only run on the GPU)")
    if t.dtype != dtype:
        raise OdiseError(f"{name}: expected {dtype}, got {t.dtype}")
    return t


class PostprocessGeom(ctypes.Structure):
    """odise_postprocess_geom (include/odise_b200.h): padded size and un-padded image size of sem_seg_postprocess."""
    _fields_ = [("pad_h", c_int), ("pad_w", c_int), ("img_h", c_int), ("img_w", c_int)]


Q8 = "q8"          # value of the engines' `lo` switch in the F16Q8 operand mode (truthy: a second plane exists)
Q8_SHIFT = 6       # kQ8Shift of csrc/ptx.cuh
PLANES_BF16, PLANES_F16, PLANES_F16Q8 = 0, 1, 2


class Planes:
    """(hi, lo) operand planes of a 2-D fp32 matrix [rows, cols] (row stride ld elements of 2 bytes, both planes).
    fmt: "bf16" = bf16 pair (lo may be None: plain bf16) | "f16" = fp16 pair (V^T of the attention kernel) | "q8" = fp16 hi +
    e5m2 correction bytes [x * 2^-6 | (x - hi) * 2^6] per 64-wide k-block (ODISE_PLANES_F16Q8, include/odise_b200.h)."""

    __slots__ = ("hi", "lo", "rows", "cols", "ld", "fmt")

    def __init__(self, hi, lo, rows, cols, ld, f16=False, fmt=None):
        self.hi, self.lo, self.rows, self.cols, self.ld = hi, lo, rows, cols, ld
        self.fmt = fmt or ("f16" if f16 else "bf16")

    @property
    def f16(self):
        return self.fmt == "f16"

    @property
    def code(self):
        return {"bf16": PLANES_BF16, "f16": PLANES_F16, "q8": PLANES_F16Q8}[self.fmt]

    @staticmethod
    def empty(rows, cols, device, lo=True, ld=None, f16=False):
        """lo: False = hi plane only | True = bf16 pair (fp16 pair with f16=True) | lib.Q8 = the F16Q8 format (rows padded to
        whole 64-element k-blocks, pad bytes zero)."""
        q8 = lo == Q8 and not f16
        ld = ld or ((cols + 7) // 8 * 8)
        if q8:
            ld = (ld + 63) // 64 * 64
        hi = torch.empty(rows * ld, dtype=torch.bfloat16, device=device)
        lo_t = torch.empty(rows * ld, dtype=torch.bfloat16, device=device) if lo else None
        if ld != cols:
            hi.zero_()
            if lo_t is not None:
                lo_t.zero_()
        return Planes(hi, lo_t, rows, cols, ld, fmt="q8" if q8 else ("f16" if f16 else "bf16"))

    def float(self):
        if self.fmt == "q8":        # test helper: hi + the decoded low-order correction
            h = self.hi.view(torch.float16).view(self.rows, self.ld)[:, : self.cols].float()
            qb = self.lo.view(torch.uint8).view(self.rows, self.ld // 64, 2, 64)
            ql = qb[:, :, 1, :].reshape(self.rows, self.ld)[:, : self.cols].contiguous().view(torch.float8_e5m2).float()
            return h + ql * 2.0 ** -Q8_SHIFT
        vw = (lambda t: t.view(torch.float16)) if self.f16 else (lambda t: t)
        h = vw(self.hi).view(self.rows, self.ld)[:, : self.cols].float()
        if self.lo is not None:
            h = h + vw(self.lo).view(self.rows, self.ld)[:, : self.cols].float()
        return h

    def col_slice(self, c0, cols):
        """Planes viewing columns [c0, c0+cols) of every row (same ld); c0 % 8 == 0 (q8: whole 64-wide k-blocks)."""
        assert c0 % (64 if self.fmt == "q8" else 8) == 0
        return Planes(self.hi[c0:], None if self.lo is None else self.lo[c0:], self.rows, cols, self.ld, fmt=self.fmt)

    def row_slice(self, r0, rows):
        return Planes(self.hi[r0 * self.ld:], None if self.lo is None else self.lo[r0 * self.ld:], rows, self.cols,
                      self.ld, fmt=self.fmt)


_FMT_STATE = [PLANES_BF16]


def pargs(p):
    """(hi pointer, lo pointer, ld) of output planes for a producer entry point, and tell the library which format the
    kernels launched next must write (odise_set_operand_format is a launch-time host parameter)."""
    if p is None:
        return None, None, 0
    if p.fmt == "f16":
        raise OdiseError("fp16-pair planes are written by odise_gemm_bf16 / odise_split_f16_f32 only")
    code = p.code
    if _FMT_STATE[0] != code:
        _check(load().odise_set_operand_format(code), "odise_set_operand_format")
        _FMT_STATE[0] = code
    return _ptr(p.hi), _ptr(p.lo), p.ld


class GnStats:
    """Per-(32-row segment, channel) GroupNorm records of an fp32 activation [rows, C], filled by the epilogues of the GEMMs
    that produce the activation (possibly several: the two halves of a skip concat write disjoint column ranges of one
    buffer, see cols()) and merged by ops.group_norm().  `missing` (shared by all views of a buffer) is set by a producer that
    could not fill its columns (split-K, ragged rows): group_norm() then falls back to the stand-alone statistics pass."""

    __slots__ = ("t", "rows", "C", "Ctot", "col", "_flag")

    def __init__(self, rows, C, device, _root=None, _col=0):
        self.rows, self.C, self.col = rows, C, _col
        if _root is None:
            self._flag = [rows % 32 != 0]
            self.Ctot = C
            self.t = None if self._flag[0] else torch.empty(rows // 32, 3, C, dtype=torch.float32, device=device)
        else:
            self._flag, self.Ctot, self.t = _root._flag, _root.Ctot, _root.t

    @property
    def missing(self):
        return self._flag[0]

    @missing.setter
    def missing(self, v):
        self._flag[0] = bool(v)

    def cols(self, c0, C):
        """records of columns [c0, c0 + C) of the same activation buffer"""
        return GnStats(self.rows, C, None, _root=self, _col=self.col + c0)

    @property
    def ptr(self):
        return self.t.data_ptr() + 4 * self.col


def split(x, out=None, lo=True, f16=False):
    """fp32 [rows, cols] (last dim contiguous) -> Planes (bf16 pair; f16=True: fp16 pair; lo=lib.Q8: F16Q8)."""
    _req(x, torch.float32, "x")
    x2 = x.reshape(-1, x.shape[-1])
    rows, cols = x2.shape
    assert x2.stride(1) == 1
    if out is None:
        out = Planes.empty(rows, cols, x.device, lo=lo, f16=f16)
    if out.f16:
        _check(load().odise_split_f16_f32(_ptr(x2), x2.stride(0), _ptr(out.hi), _ptr(out.lo), out.ld, rows, cols, _stream()),
               "odise_split_f16_f32")
    else:
        if out.fmt == "q8" and cols % 4:
            raise OdiseError("split: F16Q8 planes need cols % 4 == 0")
        hi, lo_p, ld = pargs(out)
        _check(load().odise_split_f32(_ptr(x2), x2.stride(0), hi, lo_p, ld, rows, cols, _stream()), "odise_split_f32")
    return out


_WS = {}


def workspace(nbytes, device):
    """Grow-only scratch buffer per device for split-K partials (GEMMs of one stream run in order, so it is shared)."""
    key = str(device)
    if key not in _WS or _WS[key].numel() < nbytes:
        _WS[key] = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
    return _WS[key]


def auto_split(M, N, K, batch=1, sms=132):
    """(force_bn, split_k) for GEMMs that cannot fill the GPU with output tiles alone (e.g. the 8x8 / 16x16 UNet levels:
    M = 1024 -> 80 tiles of 128 x 128 on 132 SMs).  Cost model in units of K * BN per wave (tools/gemm_one.py), plus
    ~6 us for the reduce launch; (0, 1) = leave it to the kernel's own heuristic."""
    tm = (M + 127) // 128
    kblocks = (K + 63) // 64
    unit = 0.68 / (64 * 128)                      # us per (k element x output column) of a 128-row tile, bf16x3
    best = (None, 1e30)
    for bn in (128, 160, 256):
        tiles = tm * ((N + bn - 1) // bn) * batch
        for s in (1, 2, 3, 4):
            if s > 1 and kblocks // s < 16:
                continue
            waves = (tiles * s + sms - 1) // sms
            cost = waves * (K / s) * bn * unit
            if s > 1:                             # reduce launch + the partial sums written and read back through HBM / L2
                cost += 6.0 + 8.0 * s * M * N * batch / 5.0e6
            if cost < best[1]:
                best = ((bn, s), cost)
    bn, s = best[0]
    return (bn, s) if s > 1 else (0, 1)


def conv_ok(H, W):
    """Can odise_gemm_bf16 run a 3x3 conv with OUTPUT size H x W as an implicit GEMM (gemm_tc.cu host checks)?  Widths whose
    gcd with the 128-pixel tile is below 8 (e.g. 12, 6: latents of crops that are not 512^2) take the materialised
    im2col path instead."""
    import math
    if W % 128 == 0:
        return True
    if 128 % W == 0:
        bh = min(128 // W, H)
        if H % bh == 0 and 128 % (W * bh) == 0:
            return True
    return math.gcd(W, 128) % 8 == 0


def gemm(a, b, *, M=None, N=None, K=None, nmma=3, batch=1, a_bs=0, b_bs=0, conv=None, alpha=1.0, bias=None, bias_m=None,
         rowbias=None, rows_per_group=1, act=ACT_NONE, residual=None, ld_res=None, res_bs=0, out=None, ld_out=None,
         out_bs=0, out_planes=None, outp_bs=0, split_k=1, workspace=None, force_bn=0, geglu=False, conv_mode=0, gn=None):
    """out[z] = epi(alpha * A[z] @ B[z]^T).  a, b: Planes (K-major).  conv = (C, H, W) for implicit 3x3."""
    d = GemmDesc()
    d.M = M if M is not None else a.rows
    d.N = N if N is not None else b.rows
    d.K = K if K is not None else (9 * conv[0] if conv else a.cols)
    d.batch = batch
    if conv:
        d.conv3x3, d.conv_C, d.conv_H, d.conv_W = 1, conv[0], conv[1], conv[2]
    if a.f16 or b.f16:
        raise OdiseError("gemm: fp16 planes are attention-kernel operands (V^T), not GEMM inputs")
    if a.fmt != b.fmt:
        raise OdiseError(f"gemm: operand formats differ ({a.fmt} x {b.fmt})")
    if a.fmt == "q8":
        if nmma == 1:
            raise OdiseError("gemm: F16Q8 operands have no plain-bf16 mode")
        nmma = 2               # fp16 hi*hi + e5m2 cross terms; the engines pass their own nmma (2) or the default 3
    elif nmma == 2:
        nmma = 3               # an engine in the F16Q8 mode calling with bf16-pair operands (attention / binary-mask GEMMs)
    d.nmma = nmma
    d.a_hi, d.a_lo, d.lda, d.a_batch_stride = _ptr(a.hi), _ptr(a.lo), a.ld, a_bs
    d.b_hi, d.b_lo, d.ldb, d.b_batch_stride = _ptr(b.hi), _ptr(b.lo), b.ld, b_bs
    d.alpha = alpha
    d.bias = _ptr(bias)
    d.bias_m = _ptr(bias_m)
    if rowbias is not None:
        d.rowbias, d.rows_per_group, d.rowbias_ld = _ptr(rowbias), rows_per_group, rowbias.stride(0)
    d.act = act
    if residual is not None:
        d.residual = _ptr(residual)
        d.ld_residual = ld_res if ld_res is not None else residual.stride(-2)
        d.residual_batch_stride = res_bs
    if out is not None:
        d.out_f32 = _ptr(out)
        d.ld_out = ld_out if ld_out is not None else out.stride(-2)
        d.out_batch_stride = out_bs
    if out_planes is not None:
        d.out_hi, d.out_lo, d.ld_out_bf16 = _ptr(out_planes.hi), _ptr(out_planes.lo), out_planes.ld
        d.out_bf16_batch_stride = outp_bs
        d.out_planes_fp16 = out_planes.code
    d.split_k = split_k
    if split_k > 1:
        need = split_k * batch * d.M * d.N * 4
        if workspace is None or workspace.numel() * workspace.element_size() < need:
            raise OdiseError("gemm: split_k needs a workspace of %d bytes" % need)
        d.workspace, d.workspace_bytes = _ptr(workspace), workspace.numel() * workspace.element_size()
    d.force_bn = force_bn
    if gn is not None:        # GroupNorm records of the output (a GnStats view of the output's columns)
        if split_k > 1 or gn.missing or d.M % 32 or gn.C != d.N or gn.rows != d.M * batch:
            gn.missing = True
        else:
            d.gn_partial = gn.ptr
            d.gn_seg_stride, d.gn_plane_stride = 3 * gn.Ctot, gn.Ctot
    d.geglu = 1 if geglu else 0
    d.conv_mode = conv_mode
    _check(load().odise_gemm_bf16(ctypes.byref(d), _stream()), "odise_gemm_bf16")
    return out if out is not None else out_planes


def gemm_tile_policy(M, N, K, batch=1, conv=False, nmma=2):
    """(BN, pair) the GEMM's cost model picks for a problem (host only; include/odise_b200.h odise_gemm_tile_policy)."""
    bn, pair = c_int(0), c_int(0)
    _check(load().odise_gemm_tile_policy(M, N, K, batch, 1 if conv else 0, nmma, ctypes.byref(bn), ctypes.byref(pair)),
           "odise_gemm_tile_policy")
    return bn.value, bool(pair.value)


def msda_forward(value, spatial_shapes, level_start_index, sampling_locations, attention_weights, im2col_step=128):
    """Drop-in for MSDA.ms_deform_attn_forward (reference ops/src/vision.cpp:19): same arguments, same result
    shape [N, Lq, M*D], same error behaviour class (RuntimeError on non-contiguous / non-CUDA input)."""
    for t, nm in ((value, "value"), (sampling_locations, "sampling_loc"), (attention_weights, "attn_weight")):
        if not t.is_cuda:
            raise OdiseError(f"{nm} must be a CUDA tensor")  # reference: AT_ERROR("Not implemented on the CPU")
        if not t.is_contiguous():
            raise OdiseError(f"{nm} tensor has to be contiguous")  # reference .cu:33-37
        _req(t, torch.float32, nm)
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_locations.shape
    step = min(N, im2col_step)
    if N % step != 0:
        raise OdiseError(f"batch({N}) must divide im2col_step({step})")  # reference .cu:57
    ss = spatial_shapes.to(device=value.device, dtype=torch.int64).contiguous()
    ls = level_start_index.to(device=value.device, dtype=torch.int64).contiguous()
    out = torch.empty(N, Lq, M * D, dtype=torch.float32, device=value.device)
    _check(load().odise_msda_forward_f32(_ptr(value), _ptr(ss), _ptr(ls), _ptr(sampling_locations),
                                         _ptr(attention_weights), _ptr(out), N, S, M, D, L, Lq, P, _stream()),
           "odise_msda_forward_f32")
    return out


class nvtx:
    """NVTX range around a pipeline stage (SURVEY.md §5 tracing): visible in nsys / ncu --nvtx timelines, free otherwise."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        torch.cuda.nvtx.range_pop()
        return False


def profile_begin():
    _check(load().odise_profile_begin(), "odise_profile_begin")


def profile_end():
    """-> (launches, total_ms, total_flops) of the GEMM launches since profile_begin()"""
    n, ms, fl = ctypes.c_longlong(0), ctypes.c_double(0), ctypes.c_double(0)
    _check(load().odise_profile_end(ctypes.byref(n), ctypes.byref(ms), ctypes.byref(fl)), "odise_profile_end")
    return n.value, ms.value, fl.value
