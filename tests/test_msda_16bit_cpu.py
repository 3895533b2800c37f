"""CPU checks of the 16-bit fused MSDeformAttn support: the problem generator of oracle/msda_16bit.py rounds to the
kernels' input types and keeps every sample off cell edges after rounding; the four 16-bit C entry points validate their
arguments without a GPU; the 16-bit Python entry points refuse CPU tensors."""
import pytest
import torch

DTYPES = [torch.float16, torch.bfloat16]
ERR_ARG = 10001       # ODISE_ERR_ARG of include/odise_b200.h


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_problem_rounding_and_margin(dtype):
    from oracle.msda_16bit import MARGIN, fused_problem_16bit, sample_margin_16bit
    from oracle.msda_module import fused_problem
    cfg = dict(seed=5, N=1, M=8, D=32, shapes=[(32, 32), (64, 64), (128, 128)], Lq=512, P=4)
    value, ss, lsi, ref, offs, logits, go = fused_problem_16bit(**cfg, dtype=dtype)
    assert value.dtype == offs.dtype == logits.dtype == go.dtype == dtype and ref.dtype == torch.float32
    assert sample_margin_16bit(ref, offs, ss) >= MARGIN
    v64, _, _, r64, o64, l64, g64 = fused_problem(**cfg)
    # value / logits / grad_output are plain roundings, the reference points are rounded to float32
    for got, want in ((value, v64), (logits, l64), (go, g64)):
        assert torch.equal(got, want.to(dtype))
    assert torch.equal(ref, r64.float())
    # offsets: rounded, then moved by at most a few ulps where the rounding put a sample near an edge
    rounded = o64.to(dtype)
    moved = offs != rounded
    step = 2.0 ** -(10 if dtype == torch.float16 else 7)
    assert ((offs.double() - rounded.double()).abs() <= 8 * step * rounded.double().abs().clamp_min(1)).all()
    # bfloat16 offsets of tens of pixels move samples by up to a quarter pixel: some must have been stepped off an edge,
    # and the plain rounding would have violated the margin
    if dtype == torch.bfloat16:
        assert moved.any()
        assert sample_margin_16bit(ref, rounded, ss) < MARGIN


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_module_problem_rounding(dtype):
    from oracle.msda_16bit import MARGIN, round_module_problem
    from oracle.msda_module import module_problem, sample_margin
    cfg = dict(seed=51, N=2, d_model=64, n_heads=2, shapes=[(8, 8), (16, 16), (32, 32)], n_points=4, padding=True)
    pr = round_module_problem(module_problem(**cfg), cfg["n_points"], dtype)
    assert all(v.dtype == dtype for v in pr["params"].values())
    assert pr["query"].dtype == pr["input_flatten"].dtype == dtype and pr["reference_points"].dtype == torch.float32
    assert sample_margin(pr["params"], pr["query"], pr["reference_points"], pr["spatial_shapes"], cfg["n_heads"],
                         cfg["n_points"]) >= MARGIN


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


@pytest.mark.parametrize("sfx", ["f16", "bf16"])
def test_entry_point_argument_validation_without_gpu(built, sfx):
    from odise_b200 import lib
    L = lib.load()
    fwd, bwd = getattr(L, "odise_msda_fused_" + sfx), getattr(L, "odise_msda_fused_backward_" + sfx)
    p = 16       # any non-null address: every call below fails its checks before anything is dereferenced or launched
    dims = [1, 1, 1, 32, 1, 1, 1]
    assert fwd(*([None] * 7), *dims, None) == ERR_ARG
    assert bwd(*([None] * 10), *dims, None) == ERR_ARG
    for i in range(7):                                                   # each pointer missing in turn
        args = [p] * 7
        args[i] = None
        assert fwd(*args, *dims, None) == ERR_ARG
    for i in range(10):
        args = [p] * 10
        args[i] = None
        assert bwd(*args, *dims, None) == ERR_ARG
    for bad in range(7):                                                 # N S M D L Lq P
        d = list(dims)
        d[bad] = 0
        assert fwd(*([p] * 7), *d, None) == ERR_ARG
        assert bwd(*([p] * 10), *d, None) == ERR_ARG
    for fn, n in ((fwd, 7), (bwd, 10)):
        assert fn(*([p] * n), 1, 1, 1, 32, 9, 1, 1, None) == ERR_ARG                    # L > 8
        assert fn(*([p] * n), 1, 1, 1, 64, 1, 1, 1, None) == lib.ODISE_ERR_UNSUPPORTED            # D != 32
        assert fn(*([p] * n), 1, 1, 1, 32, 3, 1, 11, None) == lib.ODISE_ERR_UNSUPPORTED           # L * P = 33 > 32
        assert fn(*([p] * n), 1, 1 << 26, 1, 32, 1, 1, 1, None) == lib.ODISE_ERR_UNSUPPORTED      # S * M * D >= 2^31


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_16bit_entry_points_have_no_cpu_path(dtype):
    from odise_b200 import lib
    ss, lsi = torch.tensor([[2, 2], [1, 1]]), torch.tensor([0, 4])
    value, offs, logits = (torch.zeros(1, 5, 2, 32, dtype=dtype), torch.zeros(1, 5, 2, 2, 2, 2, dtype=dtype),
                           torch.zeros(1, 5, 2, 4, dtype=dtype))
    r = torch.zeros(1, 5, 2, 2)
    with pytest.raises(RuntimeError):
        lib.msda_fused_forward_16bit(value, ss, lsi, r, offs, logits)
    with pytest.raises(RuntimeError):
        lib.msda_fused_backward_16bit(value, ss, lsi, r, offs, logits, torch.zeros(1, 5, 64, dtype=dtype))
    with pytest.raises(RuntimeError):                    # float32 belongs to msda_fused_forward
        lib.msda_fused_forward_16bit(value.float(), ss, lsi, r, offs.float(), logits.float())
