"""ctypes binding of libodise_b200.so (include/odise_b200.h).

PyTorch is used for device memory and streams only; every op here launches hand-written sm_90a kernels through
the C ABI.  There is NO fallback: if the library is missing or a call fails, an exception is raised.
"""
import contextvars
import ctypes
import os
import re
from ctypes import c_double, c_float, c_int, c_longlong, c_void_p, POINTER

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libodise_b200.so")

ACT_NONE, ACT_RELU, ACT_SILU, ACT_GELU, ACT_QUICKGELU = 0, 1, 2, 3, 4


class OdiseError(RuntimeError):
    pass


_HEADER = os.path.normpath(os.path.join(_HERE, os.pardir, "include", "odise_b200.h"))
# the C scalar types the header may use; any other non-pointer type is an error, never a guess
_SCALARS = {"int": c_int, "long long": c_longlong, "int64_t": c_longlong, "float": c_float, "double": c_double}


def _decls(decl, structs):
    """[(name, ctypes type)] of one C declaration: a parameter "const float* x" or a field statement "int M, N, K".
    const is dropped; a pointer to a struct in `structs` is POINTER(that Structure), any other pointer c_void_p."""
    err = f"{_HEADER}: no ctypes type for `{' '.join(decl.split())}`"
    first, *more = [d.strip() for d in decl.split(",")]
    m = re.fullmatch(r"([\w\s]+?)\s*(\*?\s*\w+)", first)
    if m is None:
        raise OdiseError(err)
    base = " ".join(w for w in m.group(1).split() if w != "const")
    out = []
    for d in [m.group(2)] + more:
        dm = re.fullmatch(r"(\*?)\s*(\w+)", d)
        if dm is None or not (dm.group(1) or base in _SCALARS):
            raise OdiseError(err)
        if dm.group(1):
            out.append((dm.group(2), POINTER(structs[base]) if base in structs else c_void_p))
        else:
            out.append((dm.group(2), _SCALARS[base]))
    return out


def _parse_header(text):
    """-> (structs, protos) of the C ABI header's text: each `typedef struct {...} name;` as a ctypes.Structure class
    called `name`, and name -> (restype, argtypes) of each odise_* prototype."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
    structs = {}
    for body, name in re.findall(r"typedef\s+struct\s*\w*\s*\{([^}]*)\}\s*(\w+)\s*;", text):
        fields = [f for stmt in body.split(";") if stmt.strip() for f in _decls(stmt, structs)]
        structs[name] = type(name, (ctypes.Structure,), {"_fields_": fields})
    protos = {}
    for ret, name, args in re.findall(r"([\w\s*]+?)\b(odise_\w+)\s*\(([^()]*)\)\s*;", text):
        argtypes = [] if args.strip() == "void" else [_decls(a, structs)[0][1] for a in args.split(",")]
        protos[name] = (_decls(f"{ret} {name}", structs)[0][1], argtypes)
    return structs, protos


# every signature and struct layout comes from include/odise_b200.h, the one statement of the ABI the .cu files compile
# against: a new entry point is declared there only
if not os.path.exists(_HEADER):
    raise OdiseError(f"{_HEADER} not found: odise_b200/lib.py binds the library from its declarations")
with open(_HEADER) as _f:
    _STRUCTS, _PROTOS = _parse_header(_f.read())
GemmDesc = _STRUCTS["odise_gemm_desc"]
PostprocessGeom = _STRUCTS["odise_postprocess_geom"]     # sem_seg_postprocess's padded size and un-padded image size

_lib = None


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
    for name, (restype, argtypes) in _PROTOS.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
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


# set while a custom op's fake implementation runs (custom_op): _launch then returns before loading the library
_NO_LAUNCH = contextvars.ContextVar("odise_b200_no_launch", default=False)
_Tensor = torch.Tensor


def _launch(name, *args, workspace=None):
    """Run entry point `name` on the current stream; OdiseError if it returns an error code.  Tensor arguments are
    passed as their addresses; ints, floats, None, ctypes arrays and byref() as they are.  workspace, if given, maps the
    loaded library to a byte count: a _scratch buffer of that size on the first argument's device goes last.
    Every entry point that takes a stream is called through here; host-only calls, which take none (the workspace size
    queries, odise_gemm_tile_policy, odise_set_operand_format, the launch counter, profile_*), call load() directly."""
    if _NO_LAUNCH.get():
        return
    dll = load()
    if workspace is not None:
        args += (_scratch(workspace(dll), args[0].device),)
    # None and ints are tested first: isinstance against torch.Tensor (a class with a metaclass) is slow for them
    _check(getattr(dll, name)(*[a if a is None or type(a) is int else a.data_ptr() if isinstance(a, _Tensor) else a
                                for a in args], _stream()), name)


# The training drop-ins' kernels as torch custom ops in namespace odise_b200, the one place where a traced graph
# (torch.compile, torch.export) meets the ctypes calls, which Dynamo cannot trace.  torch.library.Library rather than
# torch.library.custom_op: its eager call goes straight to the dispatcher, without custom_op's Python wrapper (DESIGN.md
# §3, "Under torch.compile").
_OPS = torch.library.Library("odise_b200", "FRAGMENT")


def custom_op(schema, impl):
    """Define torch.ops.odise_b200.<name> by its schema and run it with impl, a call of a wrapper of this module, on
    every device, so that a CPU tensor reaches the wrapper's own check.  The fake implementation is the same impl with
    launching switched off: the wrapper's checks read no data and need no library, so the fake refuses what the real
    call refuses for reasons visible without data, and allocates exactly the results the real call returns.  The ops
    have no autograd formula: each drop-in's autograd.Function is the one autograd definition, and Dynamo traces it with
    the ops inside."""
    name = schema.split("(")[0]
    _OPS.define(schema)
    _OPS.impl(name, impl, "CompositeExplicitAutograd")

    def fake(*args, **kwargs):
        token = _NO_LAUNCH.set(True)
        try:
            return impl(*args, **kwargs)
        finally:
            _NO_LAUNCH.reset(token)
    torch.library.register_fake(f"odise_b200::{name}", fake, lib=_OPS)


# the entry-point suffix of each storage dtype (bool masks are read as bytes); each wrapper states which dtypes it takes
_SFX = {torch.float32: "f32", torch.float64: "f64", torch.float16: "f16", torch.bfloat16: "bf16", torch.uint8: "u8",
        torch.bool: "u8"}
_FLOATS = (torch.float32, torch.float16, torch.bfloat16)     # the storage types of the training kernels


def _tensor(t, name, dtypes, shape=None, contiguous=True):
    """Raise OdiseError unless t is a CUDA tensor of `dtypes` (one dtype or a tuple), contiguous (unless
    contiguous=False: strided operands) and, if given, of `shape`.  Reads no data and needs no library."""
    dtypes = dtypes if isinstance(dtypes, tuple) else (dtypes,)
    if not t.is_cuda:
        raise OdiseError(f"{name} must be a CUDA tensor")
    if t.dtype not in dtypes:
        raise OdiseError(f"{name}: expected {' or '.join(str(d)[6:] for d in dtypes)}, got {t.dtype}")
    if contiguous and not t.is_contiguous():
        raise OdiseError(f"{name} tensor has to be contiguous")
    if shape is not None and t.shape != shape:
        raise OdiseError(f"{name}: expected shape {shape}, got {tuple(t.shape)}")


def _scratch(nbytes, device):
    """One call's device scratch of nbytes from torch's allocator (stream-ordered, and private to a captured CUDA
    graph).  Unlike workspace() it is never shared: mask_loss_forward returns its buffer as the backward's state."""
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device)


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
    _tensor(x, "x", torch.float32, contiguous=False)
    x2 = x.reshape(-1, x.shape[-1])
    rows, cols = x2.shape
    assert x2.stride(1) == 1
    if out is None:
        out = Planes.empty(rows, cols, x.device, lo=lo, f16=f16)
    if out.f16:
        _launch("odise_split_f16_f32", x2, x2.stride(0), out.hi, out.lo, out.ld, rows, cols)
    else:
        if out.fmt == "q8" and cols % 4:
            raise OdiseError("split: F16Q8 planes need cols % 4 == 0")
        _launch("odise_split_f32", x2, x2.stride(0), *pargs(out), rows, cols)
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
    _launch("odise_gemm_bf16", ctypes.byref(d))
    return out if out is not None else out_planes


def gemm_tile_policy(M, N, K, batch=1, conv=False, nmma=2):
    """(BN, pair) the GEMM's cost model picks for a problem (host only; include/odise_b200.h odise_gemm_tile_policy)."""
    bn, pair = c_int(0), c_int(0)
    _check(load().odise_gemm_tile_policy(M, N, K, batch, 1 if conv else 0, nmma, ctypes.byref(bn), ctypes.byref(pair)),
           "odise_gemm_tile_policy")
    return bn.value, bool(pair.value)


def _msda_inputs(tensors, im2col_step, dtypes=(torch.float32, torch.float64)):
    """Checks of ms_deform_attn_cuda_forward / _backward (reference .cu:33-57, :98-121) for the float / double entry
    points: CUDA, contiguous, all of value's dtype, one of `dtypes`, batch divisible by min(batch, im2col_step).
    -> the entry points' dtype suffix"""
    (value, _), *rest = tensors
    _tensor(value, "value", dtypes)
    for t, nm in rest:
        _tensor(t, nm, value.dtype)
    N = value.shape[0]
    step = min(N, im2col_step)
    if step <= 0 or N % step != 0:
        raise OdiseError(f"batch({N}) must divide im2col_step({step})")  # reference .cu:57
    return _SFX[value.dtype]


def _msda_index(device, spatial_shapes, level_start_index):
    """spatial_shapes and level_start_index as the MSDA kernels read them: contiguous int64 on the value's device"""
    return [t.to(device=device, dtype=torch.int64).contiguous() for t in (spatial_shapes, level_start_index)]


def _msda_forward(dtypes, value, spatial_shapes, level_start_index, sampling_locations, attention_weights, im2col_step):
    sfx = _msda_inputs(((value, "value"), (sampling_locations, "sampling_loc"), (attention_weights, "attn_weight")),
                       im2col_step, dtypes)
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_locations.shape
    ss, ls = _msda_index(value.device, spatial_shapes, level_start_index)
    out = torch.empty(N, Lq, M * D, dtype=value.dtype, device=value.device)
    _launch("odise_msda_forward_" + sfx, value, ss, ls, sampling_locations, attention_weights, out, N, S, M, D, L, Lq, P)
    return out


def msda_forward(value, spatial_shapes, level_start_index, sampling_locations, attention_weights, im2col_step=128):
    """Drop-in for MSDA.ms_deform_attn_forward (reference ops/src/vision.cpp:19): same arguments, same result
    shape [N, Lq, M*D], same error behaviour class (RuntimeError on non-contiguous / non-CUDA input).  float32."""
    return _msda_forward(torch.float32, value, spatial_shapes, level_start_index, sampling_locations,
                         attention_weights, im2col_step)


def msda_forward_f64(value, spatial_shapes, level_start_index, sampling_locations, attention_weights, im2col_step=128):
    """msda_forward in float64 (the reference's AT_DISPATCH_FLOATING_TYPES double instantiation)."""
    return _msda_forward(torch.float64, value, spatial_shapes, level_start_index, sampling_locations,
                         attention_weights, im2col_step)


def msda_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, im2col_step=128,
                  *, deterministic=False):
    """Drop-in for MSDA.ms_deform_attn_backward (reference ops/src/vision.cpp:20): same arguments, returns
    [grad_value, grad_sampling_loc, grad_attn_weight] shaped like value / sampling_loc / attn_weight.  float32 or
    float64 (all tensors of one dtype); RuntimeError on CPU, non-contiguous or mixed-dtype input and on a batch that
    min(batch, im2col_step) does not divide.  The whole batch is one launch (im2col_step only checked).
    deterministic=True runs odise_msda_backward_det_f32 / _f64: grad_value summed in int64 fixed point, so its bits depend
    on the inputs only (include/odise_b200.h states the error bound); the other two results are the same bits."""
    sfx = _msda_inputs(((value, "value"), (sampling_loc, "sampling_loc"), (attn_weight, "attn_weight"),
                        (grad_output, "grad_output")), im2col_step)
    # value [N, S, M, D], sampling_loc [N, Lq, M, L, P, 2]
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_loc.shape
    if grad_output.numel() != N * Lq * M * D:
        raise OdiseError(f"grad_output: expected {N * Lq * M * D} elements, got {grad_output.numel()}")
    ss, ls = _msda_index(value.device, spatial_shapes, level_start_index)
    grad_value = torch.empty_like(value)
    grad_loc = torch.empty_like(sampling_loc)
    grad_attn = torch.empty_like(attn_weight)
    _launch(f"odise_msda_backward_{'det_' if deterministic else ''}{sfx}", value, ss, ls, sampling_loc, attn_weight,
            grad_output, grad_value, grad_loc, grad_attn, N, S, M, D, L, Lq, P,
            workspace=(lambda dll: dll.odise_msda_det_workspace_bytes(N, S, M, D)) if deterministic else None)
    return [grad_value, grad_loc, grad_attn]


ODISE_ERR_ARG, ODISE_ERR_ALIGN, ODISE_ERR_WORKSPACE = 10001, 10002, 10005     # the header's ODISE_ERR_*
ODISE_ERR_UNSUPPORTED = 10006


def _msda_box(reference_points):
    """True for box reference points [N, Lq, L, 4] (cx, cy, w, h): the odise_msda_fused_box_* entry points."""
    return reference_points.dim() == 4 and reference_points.shape[-1] == 4


def _msda_fused_call(value, spatial_shapes, level_start_index, reference_points, offsets, logits, grad_output=None,
                     deterministic=False, dtypes=_FLOATS):
    """Checks of a fused MSDA call, the forward or (grad_output given) the backward, without data and without the
    library: CUDA, contiguous, value of one of `dtypes` and offsets, logits and grad_output of its dtype,
    reference_points float32, in the layouts of odise_msda_fused_f32
    (value [N, S, M, D], reference_points [N, Lq, L, 2] or boxes [N, Lq, L, 4] with a storage offset that keeps them
    16-byte aligned, offsets [N, Lq, M, L, P, 2], logits [N, Lq, M, L*P], grad_output [N, Lq, M*D]).  The 16-bit, the
    box and every backward entry point take D = 32, L*P <= 32 and S*M*D < 2^31 only (d32_ok in msda.cu; they return
    ODISE_ERR_UNSUPPORTED on any other): such shapes raise here, before any launch.
    -> (entry point, N, S, M, D, L, Lq, P)"""
    _tensor(value, "value", dtypes)
    if value.dim() != 4 or offsets.dim() != 6:
        raise OdiseError(f"value must be [N, S, M, D] and offsets [N, Lq, M, L, P, 2], got {tuple(value.shape)} and "
                         f"{tuple(offsets.shape)}")
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = offsets.shape
    box = _msda_box(reference_points)
    _tensor(reference_points, "reference_points", torch.float32, (N, Lq, L, 4 if box else 2))
    _tensor(offsets, "offsets", value.dtype, (N, Lq, M, L, P, 2))
    _tensor(logits, "logits", value.dtype, (N, Lq, M, L * P))
    if grad_output is not None:
        _tensor(grad_output, "grad_output", value.dtype, (N, Lq, M * D))
    for t, nm, want in ((spatial_shapes, "spatial_shapes", (L, 2)), (level_start_index, "level_start_index", (L,))):
        if t.shape != want:
            raise OdiseError(f"{nm}: expected shape {want}, got {tuple(t.shape)}")
    if box and reference_points.storage_offset() % 4:
        # a box is one 16-byte load (the entry points return ODISE_ERR_ARG otherwise); checked on the storage offset,
        # which a fake tensor has too, so that a view into an allocation fails here and not at the launch
        raise OdiseError("reference_points: box reference points must start 16 bytes into their storage "
                         f"(storage offset a multiple of 4 floats, got {reference_points.storage_offset()}); pass a "
                         "copy")
    fn = (f"odise_msda_fused_{'box_' if box else ''}{'' if grad_output is None else 'backward_'}"
          f"{'det_' if deterministic else ''}{_SFX[value.dtype]}")
    d32_only = box or grad_output is not None or value.dtype != torch.float32
    if d32_only and not (D == 32 and L * P <= 32 and S * M * D < 2 ** 31):
        raise OdiseError(f"{fn}: D = {D}, L*P = {L * P} not supported (D = 32, L*P <= 32 and S*M*D < 2^31 only)")
    return fn, N, S, M, D, L, Lq, P


def _msda_fused_forward(dtypes, value, spatial_shapes, level_start_index, reference_points, offsets, logits):
    fn, N, S, M, D, L, Lq, P = _msda_fused_call(value, spatial_shapes, level_start_index, reference_points, offsets,
                                                logits, dtypes=dtypes)
    ss, ls = _msda_index(value.device, spatial_shapes, level_start_index)
    out = torch.empty(N, Lq, M * D, dtype=value.dtype, device=value.device)
    planes = (None, None) if fn == "odise_msda_fused_f32" else ()    # its out_hi / out_lo, which only the engines use
    _launch(fn, value, ss, ls, reference_points, offsets, logits, out, *planes, N, S, M, D, L, Lq, P)
    return out


def _msda_fused_backward(dtypes, value, spatial_shapes, level_start_index, reference_points, offsets, logits,
                         grad_output, deterministic):
    fn, N, S, M, D, L, Lq, P = _msda_fused_call(value, spatial_shapes, level_start_index, reference_points, offsets,
                                                logits, grad_output, deterministic, dtypes)
    ss, ls = _msda_index(value.device, spatial_shapes, level_start_index)
    # the default 16-bit entry points accumulate grad_value in a float32 buffer, rounded once below
    grad_value = torch.empty(value.shape, dtype=value.dtype if deterministic else torch.float32, device=value.device)
    grad_offs = torch.empty_like(offsets)
    grad_logits = torch.empty_like(logits)
    _launch(fn, value, ss, ls, reference_points, offsets, logits, grad_output, grad_value, grad_offs, grad_logits,
            N, S, M, D, L, Lq, P,
            workspace=(lambda dll: dll.odise_msda_det_workspace_bytes(N, S, M, D)) if deterministic else None)
    if grad_value.dtype != value.dtype:
        grad_value = grad_value.to(value.dtype)
    return grad_value, grad_offs, grad_logits


def msda_fused_forward(value, spatial_shapes, level_start_index, reference_points, offsets, logits):
    """MSDeformAttn's sampling from the raw linear outputs (odise_msda_fused_f32: softmax over L*P and
    loc = ref + off / (W_l, H_l) inside the kernel) -> out [N, Lq, M*D] float32.  Box reference points [N, Lq, L, 4]
    take odise_msda_fused_box_f32 (loc = ref.xy + off / P * ref.wh * 0.5), D = 32, L*P <= 32 and S*M*D < 2^31 only.
    RuntimeError on CPU, non-contiguous or non-float32 tensors, on shapes that disagree and on a D the kernel does not
    take."""
    return _msda_fused_forward(torch.float32, value, spatial_shapes, level_start_index, reference_points, offsets,
                               logits)


def msda_fused_backward(value, spatial_shapes, level_start_index, reference_points, offsets, logits, grad_output, *,
                        deterministic=False):
    """Backward of msda_fused_forward (odise_msda_fused_backward_f32) -> (grad_value, grad_offsets, grad_logits) shaped
    like value / offsets / logits.  D = 32 and L*P <= 32 only; RuntimeError otherwise and on the input errors of
    msda_fused_forward.  grad_offsets and grad_logits are bit-deterministic; deterministic=True
    (odise_msda_fused_backward_det_f32) makes grad_value so too.  Box reference points take
    odise_msda_fused_box_backward_f32 / _det_f32."""
    return _msda_fused_backward(torch.float32, value, spatial_shapes, level_start_index, reference_points, offsets,
                                logits, grad_output, deterministic)


_16BIT = (torch.float16, torch.bfloat16)


def msda_fused_forward_16bit(value, spatial_shapes, level_start_index, reference_points, offsets, logits):
    """msda_fused_forward with 16-bit storage (odise_msda_fused_f16 / _bf16, chosen by value.dtype): value, offsets and
    logits float16 or bfloat16 (one dtype), reference_points float32 -> out [N, Lq, M*D] in the value's dtype, one rounding
    of the fp32 result.  D = 32 and L*P <= 32 only.  Box reference points [N, Lq, L, 4] take odise_msda_fused_box_f16 /
    _bf16.  RuntimeError on CPU or non-contiguous tensors, on a float32 value, on mixed dtypes, on shapes that disagree
    and on unsupported shapes."""
    return _msda_fused_forward(_16BIT, value, spatial_shapes, level_start_index, reference_points, offsets, logits)


def msda_fused_backward_16bit(value, spatial_shapes, level_start_index, reference_points, offsets, logits, grad_output,
                              *, deterministic=False):
    """Backward of msda_fused_forward_16bit (odise_msda_fused_backward_f16 / _bf16) -> (grad_value, grad_offsets,
    grad_logits), each in the value's dtype.  grad_value is accumulated in a float32 buffer and rounded once here;
    grad_offsets and grad_logits are rounded once in the kernel and are bit-deterministic.  grad_output has the value's
    dtype.  Errors as msda_fused_forward_16bit.  deterministic=True (odise_msda_fused_backward_det_f16 / _bf16) sums
    grad_value in int64 fixed point and the kernels write it in the value's dtype: its bits depend on the inputs only.
    Box reference points take odise_msda_fused_box_backward_* (and _det_*)."""
    return _msda_fused_backward(_16BIT, value, spatial_shapes, level_start_index, reference_points, offsets, logits,
                                grad_output, deterministic)


def _xattn_shapes(q, k, v, mask, heads, out=None, lse=None, grad_out=None):
    """Checks of the masked cross-attention entry points, without data and without the library: q [Q, B, E], k and v
    [S, B, E], E = heads * 32, CUDA,
    contiguous, one dtype of float32 / float16 / bfloat16; mask None or a contiguous CUDA bool [B*heads, Q, S] or
    [Q, S]; for the backward out and grad_out like q and lse [B*heads, Q] float32.  -> (Q, B, E, S, mask_bh_stride)"""
    _tensor(q, "q", _FLOATS)
    if q.dim() != 3 or k.dim() != 3:
        raise OdiseError(f"q and k: expected 3-D tensors, got {tuple(q.shape)} and {tuple(k.shape)}")
    Q, B, E = q.shape
    S = k.shape[0]
    if heads <= 0 or E % heads:
        raise OdiseError(f"embed dim {E} is not divisible by heads = {heads}")
    if E // heads != 32:
        raise OdiseError(f"masked cross-attention: head dim {E // heads} not supported (32 only)")
    for t, nm, want in ((k, "k", (S, B, E)), (v, "v", (S, B, E)), (out, "out", (Q, B, E)),
                        (grad_out, "grad_out", (Q, B, E))):
        if t is not None:
            _tensor(t, nm, q.dtype, want)
    if S <= 0 or Q <= 0 or B <= 0:
        raise OdiseError(f"empty sequence: Q = {Q}, S = {S}, B = {B}")
    if B * heads > 65535 or (S + 63) // 64 > 65535:
        raise OdiseError(f"masked cross-attention: B*heads = {B * heads} or S = {S} too large")
    if lse is not None:
        _tensor(lse, "lse", torch.float32, (B * heads, Q))
    stride = 0
    if mask is not None:
        _tensor(mask, "mask", torch.bool)     # True = blocked
        if mask.shape == (B * heads, Q, S):
            stride = Q * S
        elif mask.shape != (Q, S):
            raise OdiseError(f"mask: expected shape {(B * heads, Q, S)} or {(Q, S)}, got {tuple(mask.shape)}")
    return Q, B, E, S, stride


def masked_xattn_forward(q, k, v, mask, heads):
    """Masked cross-attention core of nn.MultiheadAttention (odise_masked_xattn_forward_f32 / _f16 / _bf16 by q.dtype):
    q [Q, B, heads*32], k and v [S, B, heads*32] (the in-projection outputs, sequence first), mask None or bool
    [B*heads, Q, S] / [Q, S] with True = blocked -> (out [Q, B, heads*32] in q's dtype, lse [B*heads, Q] float32).
    RuntimeError on CPU, non-contiguous or mixed-dtype tensors, shapes that disagree and a head dim other than 32."""
    Q, B, E, S, stride = _xattn_shapes(q, k, v, mask, heads)
    out = torch.empty_like(q)
    lse = torch.empty(B * heads, Q, dtype=torch.float32, device=q.device)
    _launch("odise_masked_xattn_forward_" + _SFX[q.dtype], q, k, v, mask, stride, out, lse, B, heads, 32, Q, S,
            workspace=lambda dll: dll.odise_masked_xattn_workspace_bytes(B, heads, Q, S))
    return out, lse


def masked_xattn_backward(q, k, v, mask, out, lse, grad_out, heads):
    """Backward of masked_xattn_forward (odise_masked_xattn_backward_*) -> (grad_q, grad_k, grad_v) shaped and typed like
    q / k / v.  grad_out has q's dtype.  Every result is bit-reproducible (fixed-order sums, no atomics).  Errors as
    masked_xattn_forward, and for out / lse / grad_out of the wrong shape or dtype."""
    Q, B, E, S, stride = _xattn_shapes(q, k, v, mask, heads, out=out, lse=lse, grad_out=grad_out)
    gq, gk, gv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    _launch("odise_masked_xattn_backward_" + _SFX[q.dtype], q, k, v, mask, stride, out, lse, grad_out, gq, gk, gv, B,
            heads, 32, Q, S, workspace=lambda dll: dll.odise_masked_xattn_workspace_bytes(B, heads, Q, S))
    return gq, gk, gv


UNET_ATTN_HEAD_DIMS = (40, 80, 160)     # SD-v1's 320 / 640 / 1280 channels over 8 heads


def unet_attn_supported(B, heads, dim_head, Tq, Tk):
    """whether the UNet attention kernels take B images of `heads` heads of dim_head channels, Tq queries and Tk keys:
    a head dim of UNET_ATTN_HEAD_DIMS, non-empty sequences and at most 65535 (image, head) pairs"""
    return (dim_head in UNET_ATTN_HEAD_DIMS and min(B, heads, Tq, Tk) >= 1 and B * heads <= 65535
            and max(Tq, Tk) * B * heads * 160 < 2 ** 40)


def _unet_attn_shapes(q, k, v, heads, out=None, lse=None, grad_out=None):
    """Checks of the UNet attention entry points, without data and without the library: q [B, Tq, heads*D], k and v
    [B, Tk, heads*D] as to_q / to_k / to_v write them, contiguous CUDA tensors of one dtype of float32 / float16 /
    bfloat16, unet_attn_supported(B, heads, D, Tq, Tk); for the backward out and grad_out like q and lse [B*heads, Tq]
    float32.  -> (B, Tq, Tk, D)"""
    _tensor(q, "q", _FLOATS)
    if q.dim() != 3 or k.dim() != 3:
        raise OdiseError(f"q and k: expected 3-D tensors, got {tuple(q.shape)} and {tuple(k.shape)}")
    B, Tq, E = q.shape
    Tk = k.shape[1]
    if heads <= 0 or E % heads:
        raise OdiseError(f"inner dim {E} is not divisible by heads = {heads}")
    D = E // heads
    if not unet_attn_supported(B, heads, D, Tq, Tk):
        raise OdiseError(f"UNet attention: B = {B}, heads = {heads}, head dim {D}, Tq = {Tq}, Tk = {Tk} not supported "
                         f"(head dim one of {UNET_ATTN_HEAD_DIMS}, non-empty sequences, B*heads <= 65535)")
    for t, nm, want in ((k, "k", (B, Tk, E)), (v, "v", (B, Tk, E)), (out, "out", (B, Tq, E)),
                        (grad_out, "grad_out", (B, Tq, E))):
        if t is not None:
            _tensor(t, nm, q.dtype, want)
    if lse is not None:
        _tensor(lse, "lse", torch.float32, (B * heads, Tq))
    return B, Tq, Tk, D


def unet_attn_forward(q, k, v, heads):
    """Attention core of ldm's CrossAttention (odise_unet_attn_forward_f32 / _f16 / _bf16 by q.dtype): q [B, Tq,
    heads*D], k and v [B, Tk, heads*D], D = 40, 80 or 160 -> (out [B, Tq, heads*D] in q's dtype, lse [B*heads, Tq]
    float32).  OdiseError on CPU, non-contiguous or mixed-dtype tensors, shapes that disagree and unsupported shapes."""
    B, Tq, Tk, D = _unet_attn_shapes(q, k, v, heads)
    out = torch.empty_like(q)
    lse = torch.empty(B * heads, Tq, dtype=torch.float32, device=q.device)
    _launch("odise_unet_attn_forward_" + _SFX[q.dtype], q, k, v, out, lse, B, heads, D, Tq, Tk)
    return out, lse


def unet_attn_backward(q, k, v, out, lse, grad_out, heads):
    """Backward of unet_attn_forward (odise_unet_attn_backward_*) -> (grad_q, grad_k, grad_v) shaped and typed like
    q / k / v.  grad_out has q's dtype.  Every result is bit-reproducible (fixed-order sums, no atomics).  Errors as
    unet_attn_forward, and for out / lse / grad_out of the wrong shape or dtype."""
    B, Tq, Tk, D = _unet_attn_shapes(q, k, v, heads, out=out, lse=lse, grad_out=grad_out)
    gq, gk, gv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    _launch("odise_unet_attn_backward_" + _SFX[q.dtype], q, k, v, out, lse, grad_out, gq, gk, gv, B, heads, D, Tq, Tk,
            workspace=lambda dll: dll.odise_unet_attn_workspace_bytes(B, heads, D, Tq, Tk))
    return gq, gk, gv


MASK_MAX_IMAGES, MASK_MAX_CANDIDATES, MASK_MAX_POINTS = 256, 53248, 32768    # ODISE_MASK_MAX_* of the header
MASK_MAX_ASSIGN = 1024                                                          # ODISE_MASK_MAX_ASSIGN
_MASK_BYTES = (torch.bool, torch.uint8)


def _mask_maps(pred, tgt):
    """Checks shared by the mask-criterion entry points: pred [B, Q, H, W] float32 / float16 / bfloat16 and the target
    masks tgt [sum T, Hg, Wg] bool or uint8, both CUDA and contiguous.  -> (suffix, B, Q, H, W, Hg, Wg)"""
    _tensor(pred, "pred_masks", _FLOATS)
    _tensor(tgt, "target masks", _MASK_BYTES)
    if pred.dim() != 4 or tgt.dim() != 3:
        raise OdiseError(f"pred_masks must be [B, Q, H, W] and target masks [T, Hg, Wg], got {tuple(pred.shape)} and "
                         f"{tuple(tgt.shape)}")
    B, Q, H, W = pred.shape
    if min(B, Q, H, W) <= 0 or min(tgt.shape[1:]) <= 0:
        raise OdiseError(f"empty maps: pred_masks {tuple(pred.shape)}, target masks {tuple(tgt.shape)}")
    if B > MASK_MAX_IMAGES:
        raise OdiseError(f"mask criterion: at most {MASK_MAX_IMAGES} images, got {B}")
    return _SFX[pred.dtype], B, Q, H, W, tgt.shape[1], tgt.shape[2]


def _u8(t):
    return t.view(torch.uint8) if t.dtype == torch.bool else t


def mask_point_sample(maps, points):
    """detectron2's point_sample on the device, as the mask-criterion kernels sample (odise_mask_point_sample_*):
    maps [N, H, W] float32 / float16 / bfloat16 / bool / uint8, points [N, P, 2] float32 in [0, 1)^2 -> [N, P] float32,
    bit-equal to F.grid_sample(maps[:, None].float(), 2 * points[:, :, None] - 1, align_corners=False)."""
    _tensor(maps, "maps", _FLOATS + _MASK_BYTES)
    if maps.dim() != 3:
        raise OdiseError(f"maps: expected [N, H, W], got {tuple(maps.shape)}")
    N, H, W = maps.shape
    if points.dim() != 3 or points.shape[0] != N or points.shape[2] != 2:
        raise OdiseError(f"points: expected [{N}, P, 2], got {tuple(points.shape)}")
    _tensor(points, "points", torch.float32)
    out = torch.empty(N, points.shape[1], dtype=torch.float32, device=maps.device)
    _launch("odise_mask_point_sample_" + _SFX[maps.dtype], _u8(maps), points, out, N, H, W, points.shape[1])
    return out


def mask_cost(pred, prob, labels, tgt, points, counts, w_class, w_mask, w_dice, out=None):
    """Matching costs of one prediction set (odise_mask_cost_f32 / _f16 / _bf16 by pred.dtype): pred [B, Q, H, W],
    prob [B, Q, K1] float32 (softmax of the class logits), labels [sum T] int64, tgt [sum T, Hg, Wg] bool / uint8 with
    image b's counts[b] targets after those of images 0..b-1 (counts: a Python list), points [B, P, 2] float32 ->
    cost [B, Q, max(counts)] float32 (out: a tensor of that shape and dtype to write into; columns t >= counts[b] are
    left as they are).  OdiseError on CPU, non-contiguous or wrongly typed tensors and on shapes that disagree."""
    sfx, B, Q, H, W, Hg, Wg = _mask_maps(pred, tgt)
    counts = [int(c) for c in counts]
    if len(counts) != B or min(counts, default=0) < 0 or sum(counts) != tgt.shape[0]:
        raise OdiseError(f"target counts {counts} do not match {B} images and {tgt.shape[0]} target masks")
    if prob.dim() != 3 or tuple(prob.shape[:2]) != (B, Q):
        raise OdiseError(f"prob: expected [B, Q, K1] = [{B}, {Q}, K1], got {tuple(prob.shape)}")
    K1 = prob.shape[2]
    if points.dim() != 3 or points.shape[0] != B or points.shape[2] != 2 or points.shape[1] <= 0:
        raise OdiseError(f"points: expected [{B}, P, 2] with P > 0, got {tuple(points.shape)}")
    P = points.shape[1]
    _tensor(prob, "prob", torch.float32)
    _tensor(labels, "labels", torch.int64, (tgt.shape[0],))
    _tensor(points, "points", torch.float32)
    Tmax = max(counts, default=0)
    if out is None:
        out = torch.empty(B, Q, Tmax, dtype=torch.float32, device=pred.device)
    _tensor(out, "out", torch.float32, (B, Q, Tmax))
    cnt = (ctypes.c_int * B)(*counts)
    _launch("odise_mask_cost_" + sfx, pred, prob, labels, _u8(tgt), points, cnt, out, B, Q, H, W, K1, Hg, Wg, Tmax, P,
            float(w_class), float(w_mask), float(w_dice))
    return out


def mask_assign(cost, counts):
    """scipy.optimize.linear_sum_assignment of every [Q, counts[b]] block of cost [L, B, Q, Tmax] float32 on the device
    (odise_mask_assign_f32), scipy's indices for every input, ties included; counts: a Python list ->
    (tables, status).  tables int64 holds, set after set, pairs [N, 3] (image, query, global target) by image then
    query, pair_of [B*Q] and tg_of [B*Q] (-1 if unmatched), N = sum_b min(Q, counts[b]); status [L, B] int32 is
    0 (solved), 1 (a NaN or -inf cost) or 2 (infeasible), where scipy raises.  No synchronisation, CUDA-graph
    capturable.  OdiseError on CPU, non-contiguous or wrongly typed costs, counts that disagree, B > MASK_MAX_IMAGES
    and Q or Tmax > MASK_MAX_ASSIGN."""
    _tensor(cost, "cost", torch.float32)
    if cost.dim() != 4:
        raise OdiseError(f"cost must be [L, B, Q, Tmax], got {tuple(cost.shape)}")
    L, B, Q, Tmax = cost.shape
    counts = [int(c) for c in counts]
    if min(L, B, Q) <= 0 or len(counts) != B or not all(0 <= c <= Tmax for c in counts):
        raise OdiseError(f"target counts {counts} do not match cost {tuple(cost.shape)}")
    if B > MASK_MAX_IMAGES or max(Q, Tmax) > MASK_MAX_ASSIGN:
        raise OdiseError(f"mask assign: at most {MASK_MAX_IMAGES} images and {MASK_MAX_ASSIGN} queries and targets, "
                         f"got cost {tuple(cost.shape)}")
    N = sum(min(Q, c) for c in counts)
    tables = torch.empty(L * (3 * N + 2 * B * Q), dtype=torch.int64, device=cost.device)
    status = torch.empty(L, B, dtype=torch.int32, device=cost.device)
    _launch("odise_mask_assign_f32", cost, (ctypes.c_int * B)(*counts), tables, status, L, B, Q, Tmax)
    return tables, status


def _mask_loss_shapes(pred, tgt, pairs, num_points):
    """Checks shared by the mask-loss entry points: pairs [N, 3] int64 and 0 < num_points <= MASK_MAX_POINTS.
    -> (suffix, B, Q, H, W, Hg, Wg, N)"""
    sfx, B, Q, H, W, Hg, Wg = _mask_maps(pred, tgt)
    if pairs.dim() != 2 or pairs.shape[1] != 3:
        raise OdiseError(f"pairs must be [N, 3], got {tuple(pairs.shape)}")
    _tensor(pairs, "pairs", torch.int64)
    if not 0 < num_points <= MASK_MAX_POINTS:
        raise OdiseError(f"mask loss: num_points = {num_points} not supported (1 .. {MASK_MAX_POINTS})")
    return sfx, B, Q, H, W, Hg, Wg, pairs.shape[0]


def mask_loss_forward(pred, tgt, pairs, cand, rnd, num_masks, num_points, k):
    """Point-sampled mask losses of N matched pairs (odise_mask_loss_forward_* by pred.dtype): pairs [N, 3] int64 =
    (image, query, row of tgt), cand [N, S, 2] the oversampled candidates, of which the k with the smallest |logit| are
    kept, rnd [N, num_points - k, 2] the random points -> (losses [2] float32 = (loss_mask, loss_dice), state): state is
    the workspace the backward reads: sums [N, 4] float32, then the P loss points of each pair [N, P, 2] float32 (the
    selected candidates in candidate order, then the random points)."""
    sfx, B, Q, H, W, Hg, Wg, N = _mask_loss_shapes(pred, tgt, pairs, num_points)
    if cand.dim() != 3:
        raise OdiseError(f"cand must be [N, S, 2], got {tuple(cand.shape)}")
    S = cand.shape[1]
    if not (S <= MASK_MAX_CANDIDATES and 0 <= k <= min(num_points, S)):
        raise OdiseError(f"mask loss: {S} candidates, k = {k} not supported (candidates <= {MASK_MAX_CANDIDATES}, "
                         f"k <= min(num_points, candidates))")
    _tensor(cand, "cand", torch.float32, (N, S, 2))
    _tensor(rnd, "rnd", torch.float32, (N, num_points - k, 2))
    # at least 16 bytes: the buffer is also the state mask_loss_backward takes, never empty
    ws = _scratch(max(load().odise_mask_loss_workspace_bytes(N, num_points), 16), pred.device)
    losses = torch.empty(2, dtype=torch.float32, device=pred.device)
    _launch("odise_mask_loss_forward_" + sfx, pred, _u8(tgt), pairs, cand, rnd, ws, losses, B, Q, H, W, Hg, Wg, N,
            num_points, S, k, float(num_masks))
    return losses, ws


def mask_loss_backward(pred, tgt, pairs, pair_of, state, grad_losses, num_masks, num_points):
    """Backward of mask_loss_forward (odise_mask_loss_backward_*): state as it returned, grad_losses [2] float32 on the
    device -> grad_pred shaped and typed like pred, zero on the queries pair_of [B*Q] int64 maps to -1.
    Bit-reproducible (int64 fixed-point sums)."""
    sfx, B, Q, H, W, Hg, Wg, N = _mask_loss_shapes(pred, tgt, pairs, num_points)
    _tensor(pair_of, "pair_of", torch.int64, (B * Q,))
    _tensor(grad_losses, "grad_losses", torch.float32, (2,))
    if not state.is_cuda or state.dtype != torch.uint8 or state.numel() < N * (16 + 8 * num_points):
        raise OdiseError("state: expected the workspace mask_loss_forward returned")
    grad = torch.empty_like(pred)
    _launch("odise_mask_loss_backward_" + sfx, pred, _u8(tgt), pairs, pair_of, state, grad_losses, grad, B, Q, H, W,
            Hg, Wg, N, num_points, float(num_masks))
    return grad


MASK_HEAD_C, MASK_HEAD_MAX_Q = 256, 256    # the mask width and query count the mask-head kernels take


def _mask_head_shapes(embed, features, outputs_mask=None, weights=None, grad_mask=None, grad_pooled=None):
    """Checks of the mask-head entry points, without data and without the library: embed [B, Q, 256] and features
    [B, 256, H, W] contiguous CUDA tensors of one dtype of float32 / float16 / bfloat16, Q <= 256, H * W < 2^24; for the
    backward outputs_mask and grad_mask
    [B, Q, H, W] and grad_pooled [B, Q, 256] of that dtype and weights [B, Q] float32.  -> (suffix, B, Q, H, W)"""
    _tensor(embed, "mask_embed", _FLOATS)
    if embed.dim() != 3 or features.dim() != 4:
        raise OdiseError(f"mask_embed must be [B, Q, C] and mask_features [B, C, H, W], got {tuple(embed.shape)} and "
                         f"{tuple(features.shape)}")
    B, Q, C = embed.shape
    H, W = features.shape[2:]
    if C != MASK_HEAD_C or not 0 < Q <= MASK_HEAD_MAX_Q:
        raise OdiseError(f"mask head: C = {C}, Q = {Q} not supported (C = {MASK_HEAD_C}, Q <= {MASK_HEAD_MAX_Q})")
    if min(B, H, W) <= 0 or H * W >= 2 ** 24 or B > 65535:
        raise OdiseError(f"mask head: B = {B}, H x W = {H} x {W} not supported (B <= 65535, 0 < H*W < 2^24)")
    for t, nm, want in ((features, "mask_features", (B, C, H, W)), (outputs_mask, "outputs_mask", (B, Q, H, W)),
                        (grad_mask, "grad_mask", (B, Q, H, W)), (grad_pooled, "grad_pooled", (B, Q, C))):
        if t is not None:
            _tensor(t, nm, embed.dtype, want)
    if weights is not None:
        _tensor(weights, "weights", torch.float32, (B, Q))
    return _SFX[embed.dtype], B, Q, H, W


def mask_head_forward(embed, features, threshold=0.5):
    """The prediction head's mask logits and hard mask pooling (odise_mask_head_forward_* by dtype): embed [B, Q, 256],
    features [B, 256, H, W] -> (outputs_mask [B, Q, H, W], pooled [B, Q, 256], both in embed's dtype, weights [B, Q]
    float32 = the per-(b, q) factor 1 / (count + 1e-8) as the pooling applied it).  OdiseError on CPU, non-contiguous or
    mixed-dtype tensors and on shapes the kernels do not take."""
    sfx, B, Q, H, W = _mask_head_shapes(embed, features)
    om = torch.empty(B, Q, H, W, dtype=embed.dtype, device=embed.device)
    pooled = torch.empty_like(embed)
    weights = torch.empty(B, Q, dtype=torch.float32, device=embed.device)
    _launch("odise_mask_head_forward_" + sfx, embed, features, om, pooled, weights, B, Q, MASK_HEAD_C, H, W,
            float(threshold), workspace=lambda dll: dll.odise_mask_head_workspace_bytes(B, Q, MASK_HEAD_C, H, W))
    return om, pooled, weights


def mask_head_attn_mask(outputs_mask, size, heads):
    """The decoder's attention mask (odise_mask_head_attn_mask_*): outputs_mask [B, Q, H, W] -> bool
    [B*heads, Q, h*w], True = blocked = sigmoid(bilinear resize to size = (h, w)) < 0.5 in torch's roundings for the
    dtype, with every all-blocked row written all False (odise.py:683)."""
    _tensor(outputs_mask, "outputs_mask", _FLOATS)
    if outputs_mask.dim() != 4:
        raise OdiseError(f"outputs_mask must be [B, Q, H, W], got {tuple(outputs_mask.shape)}")
    B, Q, H, W = outputs_mask.shape
    h, w = (int(s) for s in size)
    if min(B, Q, H, W, h, w, heads) <= 0 or B * Q >= 2 ** 31 or h * w >= 2 ** 31:
        raise OdiseError(f"attention mask: outputs_mask {tuple(outputs_mask.shape)}, size {(h, w)}, heads {heads} not "
                         "supported")
    out = torch.empty(B * heads, Q, h * w, dtype=torch.bool, device=outputs_mask.device)
    _launch("odise_mask_head_attn_mask_" + _SFX[outputs_mask.dtype], outputs_mask, out, B, Q, H, W, h, w, heads)
    return out


def mask_head_backward(embed, features, outputs_mask, weights, grad_mask, grad_pooled, threshold=0.5):
    """Backward of mask_head_forward (odise_mask_head_backward_*) -> (grad_embed, grad_features) in embed's dtype:
    grad_mask X^T and E^T grad_mask + (grad_pooled o weights)^T m, m the hard mask of outputs_mask.  Bit-reproducible
    (fixed-order sums, no atomics).  Errors as mask_head_forward, and for the saved tensors or gradients of the wrong
    shape or dtype."""
    sfx, B, Q, H, W = _mask_head_shapes(embed, features, outputs_mask, weights, grad_mask, grad_pooled)
    ge, gx = torch.empty_like(embed), torch.empty_like(features)
    _launch("odise_mask_head_backward_" + sfx, embed, features, outputs_mask, weights, grad_mask, grad_pooled, ge, gx,
            B, Q, MASK_HEAD_C, H, W, float(threshold),
            workspace=lambda dll: dll.odise_mask_head_workspace_bytes(B, Q, MASK_HEAD_C, H, W))
    return ge, gx


# the category-scoring kernels' limits: C a multiple of 32 up to 768, up to 2048 prompts, groups of 1..255 prompts
CATEGORY_C_MULTIPLE, CATEGORY_MAX_C, CATEGORY_MAX_PROMPTS, CATEGORY_MAX_GROUP = 32, 768, 2048, 255


def _category_shapes(mask_embed, text_embed, null_embed, logit_scale, group_start, winners=None, norms=None,
                     grad_logits=None):
    """Checks of the category-scoring entry points, without data and without the library: mask_embed [B, Q, C]
    float32 / float16 / bfloat16, text_embed [Kp, C] and null_embed [1, C] of mask_embed's dtype or (16-bit mask_embed only) both float32, logit_scale a float32 scalar,
    group_start int32 [K + 1], all contiguous CUDA tensors; for the backward winners uint8 and grad_logits of
    mask_embed's dtype [B, Q, K + 1], norms float32 [B*Q + Kp + 1].  -> (suffix, bank_f32, B, Q, C, K, Kp)"""
    _tensor(mask_embed, "mask_embed", _FLOATS)
    if mask_embed.dim() != 3 or text_embed.dim() != 2 or group_start.dim() != 1:
        raise OdiseError(f"mask_embed must be [B, Q, C], text_embed [Kp, C] and group_start [K + 1], got "
                         f"{tuple(mask_embed.shape)}, {tuple(text_embed.shape)} and {tuple(group_start.shape)}")
    B, Q, C = mask_embed.shape
    Kp, K = text_embed.shape[0], group_start.shape[0] - 1
    if min(B, Q) <= 0 or C % CATEGORY_C_MULTIPLE or not 0 < C <= CATEGORY_MAX_C or not 1 <= K <= Kp \
            or Kp > CATEGORY_MAX_PROMPTS or B * Q * max(K + 1, C) >= 2 ** 31:
        raise OdiseError(f"category scoring: B = {B}, Q = {Q}, C = {C}, K = {K}, Kp = {Kp} not supported (C a multiple "
                         f"of {CATEGORY_C_MULTIPLE} up to {CATEGORY_MAX_C}, 1 <= K <= Kp <= {CATEGORY_MAX_PROMPTS})")
    _tensor(text_embed, "text_embed", (mask_embed.dtype, torch.float32), (Kp, C))    # float32 = a float32 bank
    _tensor(null_embed, "null_embed", text_embed.dtype, (1, C))
    _tensor(logit_scale, "logit_scale", torch.float32, ())
    _tensor(group_start, "group_start", torch.int32)
    if winners is not None:
        _tensor(winners, "winners", torch.uint8, (B, Q, K + 1))
    if norms is not None:
        _tensor(norms, "norms", torch.float32, (B * Q + Kp + 1,))
    if grad_logits is not None:
        _tensor(grad_logits, "grad_logits", mask_embed.dtype, (B, Q, K + 1))
    return _SFX[mask_embed.dtype], int(text_embed.dtype != mask_embed.dtype), B, Q, C, K, Kp


def category_group_start(sizes):
    """group_start of the category-scoring kernels, as Python ints, for the classes' prompt counts (each 1..255)"""
    if not sizes or min(sizes) < 1 or max(sizes) > CATEGORY_MAX_GROUP:
        raise OdiseError(f"category scoring: groups of 1..{CATEGORY_MAX_GROUP} prompts, got sizes from "
                         f"{min(sizes, default=None)} to {max(sizes, default=None)}")
    out = [0]
    for n in sizes:
        out.append(out[-1] + n)
    return out


def category_logits_forward(mask_embed, text_embed, null_embed, logit_scale, group_start):
    """CategoryODISE.cal_pred_logits with the "max" ensemble (odise_category_logits_forward_* by mask_embed's dtype):
    -> (logits [B, Q, K + 1] in mask_embed's dtype, winners uint8 [B, Q, K + 1] = each max's prompt offset in its
    group, norms float32 [B*Q + Kp + 1] = the clamped row norms of mask_embed, text_embed and null_embed).  group_start
    int32 [K + 1] on the device holds the classes' prompt offsets (category_group_start); it is not read on the host.
    OdiseError on CPU, non-contiguous or mixed-dtype tensors and on shapes the kernels do not take."""
    sfx, bank_f32, B, Q, C, K, Kp = _category_shapes(mask_embed, text_embed, null_embed, logit_scale, group_start)
    dev = mask_embed.device
    out = torch.empty(B, Q, K + 1, dtype=mask_embed.dtype, device=dev)
    win = torch.empty(B, Q, K + 1, dtype=torch.uint8, device=dev)
    norms = torch.empty(B * Q + Kp + 1, dtype=torch.float32, device=dev)
    _launch("odise_category_logits_forward_" + sfx, mask_embed, text_embed, null_embed, logit_scale, group_start, out,
            win, norms, B * Q, C, K, Kp, bank_f32)
    return out, win, norms


def category_logits_backward(mask_embed, text_embed, null_embed, logit_scale, group_start, winners, norms,
                             grad_logits):
    """Backward of category_logits_forward (odise_category_logits_backward_*) -> (grad_mask_embed, grad_text_embed,
    grad_null_embed, grad_logit_scale): each in its input's dtype, the scale's a float32 scalar.  Each gradient goes to
    the prompt the forward chose; fixed-order sums without atomics, so every gradient is bit-reproducible."""
    sfx, bank_f32, B, Q, C, K, Kp = _category_shapes(mask_embed, text_embed, null_embed, logit_scale, group_start,
                                                     winners, norms, grad_logits)
    gm, gt, gn = torch.empty_like(mask_embed), torch.empty_like(text_embed), torch.empty_like(null_embed)
    gs = torch.empty((), dtype=torch.float32, device=mask_embed.device)
    _launch("odise_category_logits_backward_" + sfx, mask_embed, text_embed, null_embed, logit_scale, group_start,
            winners, norms, grad_logits, gm, gt, gn, gs, B * Q, C, K, Kp, bank_f32,
            workspace=lambda dll: dll.odise_category_logits_workspace_bytes(B * Q, C, K, Kp))
    return gm, gt, gn, gs


# the grounding-loss kernels' limits: Q up to 256 queries, 1..32 words, C a multiple of 32 up to 768
GROUNDING_MAX_Q, GROUNDING_MAX_K, GROUNDING_C_MULTIPLE, GROUNDING_MAX_C = 256, 32, 32, 768


def _grounding_shapes(mask_embed, word_embed, logit_scale, batch, offset, word_valid=None, state=None,
                      grad_losses=None):
    """Checks of the grounding-loss entry points, without data and without the library: mask_embed [S, G, Q, C]
    float32 / float16 / bfloat16, word_embed [G, K, C] of mask_embed's dtype or (16-bit mask_embed only) float32,
    logit_scale float32 [S], 1 <= batch <= G, 0 <= offset <= G - batch, all contiguous CUDA tensors; word_valid bool
    [G, K], state float32 [grounding_state_size(...)], grad_losses float32 [S].
    -> (suffix, words_f32, S, G, Q, K, C)"""
    _tensor(mask_embed, "mask_embed", _FLOATS)
    if mask_embed.dim() != 4 or word_embed.dim() != 3:
        raise OdiseError(f"mask_embed must be [S, G, Q, C] and word_embed [G, K, C], got {tuple(mask_embed.shape)} and "
                         f"{tuple(word_embed.shape)}")
    S, G, Q, C = mask_embed.shape
    K = word_embed.shape[1]
    if not 0 <= offset <= G - batch or not grounding_supported(S, G, batch, Q, K, C):
        raise OdiseError(f"grounding loss: S = {S}, G = {G}, B = {batch}, offset = {offset}, Q = {Q}, K = {K}, C = {C} "
                         f"not supported (1 <= B <= G, Q <= {GROUNDING_MAX_Q}, 1 <= K <= {GROUNDING_MAX_K}, C a "
                         f"multiple of {GROUNDING_C_MULTIPLE} up to {GROUNDING_MAX_C})")
    _tensor(word_embed, "word_embed", (mask_embed.dtype, torch.float32), (G, K, C))     # float32 words under autocast
    _tensor(logit_scale, "logit_scale", torch.float32, (S,))
    if word_valid is not None:
        _tensor(word_valid, "word_valid", torch.bool, (G, K))
    if state is not None:
        _tensor(state, "state", torch.float32, (grounding_state_size(S, G, batch, Q, K, C),))
    if grad_losses is not None:
        _tensor(grad_losses, "grad_losses", torch.float32, (S,))
    return _SFX[mask_embed.dtype], int(word_embed.dtype != mask_embed.dtype), S, G, Q, K, C


def grounding_supported(S, G, B, Q, K, C):
    """whether the grounding kernels take S sets of G gathered images (B local), Q queries, K words, C channels: the
    limits above and 32-bit element counts of the gathered masks, the words and the backward's per-pair tiles"""
    P = B * (2 * G - B)     # (mask image, word image) pairs with the mask or the word image local
    return (min(S, Q) > 0 and 1 <= B <= G and Q <= GROUNDING_MAX_Q and 1 <= K <= GROUNDING_MAX_K
            and C % GROUNDING_C_MULTIPLE == 0 and 0 < C <= GROUNDING_MAX_C and S * G * Q * C < 2 ** 31
            and S * P * Q * K < 2 ** 31 and G * K * C < 2 ** 31)


def grounding_state_size(S, G, B, Q, K, C):
    """float32 elements of the grounding forward's state (include/odise_b200.h)"""
    return S * G * Q * C + G * K * C + S * G * Q + G * K + 4 * S * G * B


def grounding_forward(mask_embed, word_embed, word_valid, logit_scale, batch, offset, loss_weight):
    """MaskGroundingCriterion.get_loss for S prediction sets (odise_grounding_forward_* by mask_embed's dtype) on the
    gathered mask_embed [S, G, Q, C], word_embed [G, K, C] and word_valid [G, K], this rank's `batch` images at rows
    offset .. offset + batch - 1 -> (losses float32 [S], state float32, read by grounding_backward).  OdiseError on
    CPU, non-contiguous or mixed-dtype tensors and on shapes the kernels do not take."""
    sfx, wf32, S, G, Q, K, C = _grounding_shapes(mask_embed, word_embed, logit_scale, batch, offset, word_valid)
    dev = mask_embed.device
    losses = torch.empty(S, dtype=torch.float32, device=dev)
    state = torch.empty(grounding_state_size(S, G, batch, Q, K, C), dtype=torch.float32, device=dev)
    _launch("odise_grounding_forward_" + sfx, mask_embed, word_embed, word_valid, logit_scale, losses, state, S, G,
            batch, offset, Q, K, C, float(loss_weight), wf32)
    return losses, state


def grounding_backward(mask_embed, word_embed, logit_scale, state, grad_losses, batch, offset):
    """Backward of grounding_forward (odise_grounding_backward_*) -> (grad_mask_local [S, B, Q, C], grad_mask_global
    [S, G, Q, C], grad_word_local [B, K, C], grad_word_global [G, K, C], grad_logit_scale float32 [S]): the gradients
    through the uses of the local and of the gathered rows, kept apart for the caller to combine; each in its input's
    dtype.  Fixed-order sums without atomics, so every gradient is bit-reproducible."""
    sfx, wf32, S, G, Q, K, C = _grounding_shapes(mask_embed, word_embed, logit_scale, batch, offset, None, state,
                                                 grad_losses)
    gml = mask_embed.new_empty(S, batch, Q, C)
    gmg = torch.empty_like(mask_embed)
    gwl = word_embed.new_empty(batch, K, C)
    gwg = torch.empty_like(word_embed)
    gs = torch.empty_like(logit_scale)
    _launch("odise_grounding_backward_" + sfx, mask_embed, word_embed, logit_scale, state, grad_losses, gml, gmg, gwl,
            gwg, gs, S, G, batch, offset, Q, K, C, wf32,
            workspace=lambda dll: dll.odise_grounding_workspace_bytes(S, G, batch, offset, Q, K, C))
    return gml, gmg, gwl, gwg, gs


FPN_C_MULTIPLE = 32     # the FPN upsample-add kernels take C a multiple of this


def _fpn_nchw(t, name):
    """-> (N, C, H, W) of an NCHW-contiguous CUDA float32 operand of the FPN upsample-add kernels, checked"""
    if t.dim() != 4:
        raise OdiseError(f"{name} must be [N, C, H, W], got {tuple(t.shape)}")
    _tensor(t, name, torch.float32)
    return tuple(t.shape)


def _fpn_limits(N, C, h, w, H, W):
    if min(N, C, h, w, H, W) <= 0:
        raise OdiseError(f"FPN upsample-add: empty shape N={N}, C={C}, {h}x{w} -> {H}x{W}")
    if C % FPN_C_MULTIPLE or N * (C // FPN_C_MULTIPLE) > 65535 or max(H, h) > 65535 or h * w * C >= 2 ** 31:
        raise OdiseError(f"FPN upsample-add: N={N}, C={C}, {h}x{w} -> {H}x{W} not supported (C a multiple of "
                         f"{FPN_C_MULTIPLE}, N * C / {FPN_C_MULTIPLE} <= 65535, H, h <= 65535, h*w*C < 2^31)")


def fpn_upsample_add(z, cur, size):
    """The pixel decoder's FPN step (odise_fpn_upsample_add_f32): cur + F.interpolate(level, cur's H x W, "bilinear",
    align_corners=False) of the level z [N, h*w, C] (token-major, read in place; size = (h, w)) -> y [N, C, H, W],
    bit-equal to torch's CUDA result.  z is float32 CUDA with channel-contiguous rows (strides (>= h*w*C, C, 1); a
    token slice of the encoder's memory qualifies), cur contiguous float32 CUDA.  OdiseError on CPU or non-float32
    tensors, layouts and shapes the kernel does not take."""
    h, w = (int(s) for s in size)
    N, C, H, W = _fpn_nchw(cur, "cur")
    _tensor(z, "z", torch.float32, (N, h * w, C), contiguous=False)
    _fpn_limits(N, C, h, w, H, W)
    bs = z.stride(0) if N > 1 else h * w * C
    if z.stride(2) != 1 or (h * w > 1 and z.stride(1) != C) or bs < h * w * C:
        raise OdiseError(f"z: rows must be channel-contiguous with a batch stride >= h*w*C, got strides {z.stride()}")
    y = torch.empty_like(cur)
    _launch("odise_fpn_upsample_add_f32", z, bs, cur, y, N, C, h, w, H, W)
    return y


def fpn_upsample_add_backward(grad_y, size):
    """Backward of fpn_upsample_add for the level (odise_fpn_upsample_add_backward_f32): grad_y [N, C, H, W]
    contiguous float32 -> grad_z [N, h*w, C] contiguous, the adjoint of the bilinear resize, summed in a fixed order
    without atomics (bit-reproducible).  The gradient of cur is grad_y itself."""
    h, w = (int(s) for s in size)
    N, C, H, W = _fpn_nchw(grad_y, "grad_y")
    _fpn_limits(N, C, h, w, H, W)
    gz = torch.empty(N, h * w, C, dtype=torch.float32, device=grad_y.device)
    _launch("odise_fpn_upsample_add_backward_f32", grad_y, gz, h * w * C, N, C, h, w, H, W)
    return gz


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
