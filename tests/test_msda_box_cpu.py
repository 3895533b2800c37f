"""CPU checks of MSDeformAttn with box reference points (cx, cy, w, h) on the fused path: argument validation of the nine
odise_msda_fused_box_* entry points, the fake implementations of the fused ops for box arguments, and the box oracles of
tests/msda_box_oracle.py (margins, and the fused forward equal to oracle.msda.msda_forward on the locations of
oracle.msda_module._locations, the formula tests/test_msda_module_cpu.py pins to the reference module)."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

FWD = ["odise_msda_fused_box_f32", "odise_msda_fused_box_f16", "odise_msda_fused_box_bf16"]
BWD = ["odise_msda_fused_box_backward_f32", "odise_msda_fused_box_backward_f16", "odise_msda_fused_box_backward_bf16"]
DET = ["odise_msda_fused_box_backward_det_f32", "odise_msda_fused_box_backward_det_f16",
       "odise_msda_fused_box_backward_det_bf16"]
FUSED_DTYPES = [torch.float32, torch.float16, torch.bfloat16]


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


def test_box_prototypes_match_their_twins():
    """each box entry point takes its 2-column twin's arguments (the f32 forward without out_hi / out_lo)"""
    from odise_b200 import lib
    assert lib._PROTOS["odise_msda_fused_box_f32"][1] == lib._PROTOS["odise_msda_fused_f16"][1]
    for name in FWD[1:] + BWD + DET:
        assert lib._PROTOS[name][1] == lib._PROTOS[name.replace("box_", "")][1], name


@pytest.mark.parametrize("name", FWD + BWD + DET)
def test_box_argument_validation_without_gpu(built, name):
    """return codes as the 2-column entry points': ODISE_ERR_ARG for null pointers, bad dimensions (L > 8 included) and
    a reference-point array that is not 16-byte aligned; ODISE_ERR_WORKSPACE for a null workspace; ODISE_ERR_UNSUPPORTED
    unless D = 32, L*P <= 32 and S*M*D < 2^31.  Every call fails its checks before anything is dereferenced or launched."""
    from odise_b200 import lib
    fn = getattr(lib.load(), name)
    nptr = 7 if name in FWD else 10                       # pointer arguments before the dimensions
    tail = [16, None] if name in DET else [None]          # (workspace,) stream
    p = 16
    assert fn(*([None] * nptr), 1, 1, 1, 32, 1, 1, 1, *tail) == 10001
    assert fn(*([p] * (nptr - 1)), None, 1, 1, 1, 32, 1, 1, 1, *tail) == 10001           # last output missing
    for bad in range(7):                                                                  # N S M D L Lq P
        dims = [1, 1, 1, 32, 1, 1, 1]
        dims[bad] = 0
        assert fn(*([p] * nptr), *dims, *tail) == 10001
    assert fn(*([p] * nptr), 1, 1, 1, 32, 9, 1, 1, *tail) == 10001                       # L > 8
    ref8 = [p] * nptr
    ref8[3] = 8                                                                           # ref only 8-byte aligned
    assert fn(*ref8, 1, 1, 1, 32, 1, 1, 1, *tail) == 10001
    assert fn(*([p] * nptr), 1, 1, 1, 64, 1, 1, 1, *tail) == lib.ODISE_ERR_UNSUPPORTED    # D != 32
    assert fn(*([p] * nptr), 1, 1, 1, 16, 1, 1, 1, *tail) == lib.ODISE_ERR_UNSUPPORTED    # D = 16: f32 too
    assert fn(*([p] * nptr), 1, 1, 1, 32, 3, 1, 11, *tail) == lib.ODISE_ERR_UNSUPPORTED   # L * P = 33 > 32
    assert fn(*([p] * nptr), 1, 1 << 26, 1, 32, 1, 1, 1, *tail) == lib.ODISE_ERR_UNSUPPORTED  # S * M * D >= 2^31
    if name in DET:
        assert fn(*([p] * nptr), 1, 1, 1, 32, 1, 1, 1, None, None) == 10005                                  # ODISE_ERR_WORKSPACE


# ---- fake implementations ------------------------------------------------------------------------------------------------

@pytest.fixture
def ops(monkeypatch):
    from odise_b200 import lib, msda  # noqa: F401  (importing msda defines the ops)

    def no_library():
        raise AssertionError("a fake implementation loaded the shared library")
    monkeypatch.setattr(lib, "load", no_library)
    return torch.ops.odise_b200


def _box_args(N=2, S=24, M=2, D=32, L=1, Lq=3, P=2, dtype=torch.float32, device="cuda", rw=4):
    """value, spatial_shapes, level_start_index, reference_points [N, Lq, L, rw] (float32), offsets, logits, grad_output"""
    return [torch.empty(N, S, M, D, dtype=dtype, device=device), torch.empty(L, 2, dtype=torch.int64, device=device),
            torch.empty(L, dtype=torch.int64, device=device), torch.empty(N, Lq, L, rw, device=device),
            torch.empty(N, Lq, M, L, P, 2, dtype=dtype, device=device),
            torch.empty(N, Lq, M, L * P, dtype=dtype, device=device),
            torch.empty(N, Lq, M * D, dtype=dtype, device=device)]


def _shifted(t, by=2):
    """a contiguous view with t's shape and dtype whose storage offset is `by` elements"""
    return torch.empty(t.numel() + by, dtype=t.dtype, device=t.device)[by:].view(t.shape)


def _meta(t):
    return tuple(t.shape), t.dtype, t.device.type, t.is_contiguous()


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("dtype", FUSED_DTYPES, ids=str)
def test_box_fake_results(ops, dtype, deterministic):
    with FakeTensorMode():
        value, ss, lsi, ref, offs, logits, go = _box_args(dtype=dtype)
        out = ops.msda_fused_forward(value, ss, lsi, ref, offs, logits)
        grads = ops.msda_fused_backward(value, ss, lsi, ref, offs, logits, go, deterministic)
    assert _meta(out) == ((2, 3, 64), dtype, "cuda", True)
    assert len(grads) == 3
    for g, like in zip(grads, (value, offs, logits)):
        assert _meta(g) == (tuple(like.shape), dtype, "cuda", True)


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("dtype", FUSED_DTYPES, ids=str)
def test_box_fake_errors(ops, dtype, deterministic):
    """3-column reference points, and the shapes the box kernels do not take, in the float32 forward too (the 2-column
    float32 forward takes D = 64 and L*P = 36); mixed dtypes; a box view that is not 16-byte aligned in its storage"""
    other = torch.float16 if dtype != torch.float16 else torch.bfloat16
    fwd, bwd = ops.msda_fused_forward, ops.msda_fused_backward
    with FakeTensorMode():
        args = _box_args(dtype=dtype)
        value, ss, lsi, ref, offs, logits, go = args
        bad = [_box_args(dtype=dtype, rw=3), _box_args(dtype=dtype, rw=5),
               _box_args(N=1, D=64, dtype=dtype), _box_args(N=1, S=36, L=4, P=9, dtype=dtype),
               _box_args(N=1, S=2 ** 26, M=1, D=32, dtype=dtype),
               [value, ss, lsi, ref, offs.to(other), logits, go], [value, ss, lsi, ref.to(other), offs, logits, go],
               [value, ss, lsi, _shifted(ref), offs, logits, go],
               [value, ss, lsi, ref, offs, logits, go.to(other)]]
        cases = [(fwd, b[:6]) for b in bad[:-1]] + [(bwd, b + [deterministic]) for b in bad]
        for i, (fn, a) in enumerate(cases):
            with pytest.raises(RuntimeError):
                fn(*a)
                pytest.fail(f"case {i} did not raise")
        # the same shapes with 2-column reference points: the float32 forward takes D = 64 and L*P = 36
        if dtype == torch.float32:
            fwd(*_box_args(N=1, D=64, rw=2)[:6])
            fwd(*_box_args(N=1, S=36, L=4, P=9, rw=2)[:6])
        # a view whose storage offset is a multiple of 4 floats stays 16-byte aligned
        fwd(value, ss, lsi, _shifted(ref, 4), offs, logits)


# ---- oracle helpers ------------------------------------------------------------------------------------------------------

ORACLE_CASES = [
    dict(seed=9, N=1, M=8, D=32, shapes=[(9, 7), (5, 3)], Lq=37, P=3),
    dict(seed=10, N=2, M=5, D=32, shapes=[(4, 4)] * 8, Lq=19, P=4),
    dict(seed=11, N=2, M=8, D=32, shapes=[(5, 7), (3, 2)], Lq=23, P=4, far=True),
]


@pytest.mark.parametrize("cfg", ORACLE_CASES, ids=lambda c: f"seed{c['seed']}")
def test_box_problem_margins_and_degenerate_boxes(cfg):
    from oracle.msda_16bit import MARGIN
    from msda_box_oracle import box_sample_margin, fused_problem_box, fused_problem_box_16bit
    value, ss, lsi, ref, offs, logits, go = fused_problem_box(**cfg, dtype=torch.float32)
    assert ref.shape[-1] == 4 and box_sample_margin(ref, offs, ss) >= MARGIN
    wh = ref[..., 2:]
    assert ((wh[..., 0] == 0) & (wh[..., 1] > 0)).any() and ((wh[..., 1] == 0) & (wh[..., 0] > 0)).any()
    assert not ((wh[..., 0] == 0) & (wh[..., 1] == 0)).any()
    live = wh > 0
    assert wh[live].min() >= 0.05 and wh.max() <= 0.6
    c = ref[..., :2][live]                                 # a degenerate axis moves its centre into a cell
    assert c.min() >= 0.3 - 1e-6 and c.max() <= 0.7 + 1e-6
    for dtype in (torch.float16, torch.bfloat16):
        p16 = fused_problem_box_16bit(**cfg, dtype=dtype)
        assert p16[4].dtype == dtype and p16[3].dtype == torch.float32
        assert box_sample_margin(p16[3], p16[4], ss) >= MARGIN


def test_box_fp64_locations_are_grad_problems():
    """the solved offsets put every non-degenerate coordinate at grad_problem()'s location (fp64)"""
    from oracle.msda_grad import grad_problem
    from oracle.msda_module import _locations
    from msda_box_oracle import fused_problem_box
    cfg = ORACLE_CASES[0]
    value, ss, lsi, ref, offs, logits, go = fused_problem_box(**cfg)
    loc = grad_problem(**cfg)[3]
    N, Lq, M, L, P, _ = offs.shape
    got = _locations(ref, offs.reshape(N, Lq, -1), ss, M, L, P)
    live = (ref[:, :, None, :, None, 2:] > 0).expand_as(got)
    assert (got - loc)[live].abs().max() < 1e-12


@pytest.mark.parametrize("cfg", ORACLE_CASES, ids=lambda c: f"seed{c['seed']}")
def test_box_oracle_forward_is_msda_on_module_locations(cfg):
    from oracle.msda import msda_forward
    from oracle.msda_module import _locations
    from msda_box_oracle import fused_problem_box, oracle_fused_forward
    value, ss, lsi, ref, offs, logits, go = fused_problem_box(**cfg)
    N, Lq, M, L, P, _ = offs.shape
    loc = _locations(ref, offs.reshape(N, Lq, -1), ss, M, L, P)
    aw = torch.softmax(logits, -1).view(N, Lq, M, L, P)
    want = msda_forward(value, ss, lsi, loc, aw)
    assert torch.equal(oracle_fused_forward(value, ss, lsi, ref, offs, logits), want)
    if cfg.get("far"):
        assert want.abs().max() == 0
