"""CPU checks of the MSDeformAttn custom ops (torch.ops.odise_b200.*, defined in odise_b200/msda.py) that torch.compile
and torch.export trace: their schemas, the results of their fake implementations under FakeTensorMode (which makes
"cuda" tensors without a device) for every dtype and both settings of `deterministic`, and the errors the fake
implementations raise on the inputs lib refuses.  The fake implementations never load the shared library; lib.load is
made to fail here to show it.  A CPU tensor given to the real op reaches lib's own check and raises RuntimeError."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

SCHEMAS = {
    "msda_forward": "odise_b200::msda_forward(Tensor value, Tensor spatial_shapes, Tensor level_start_index, "
                    "Tensor sampling_loc, Tensor attn_weight, int im2col_step) -> Tensor",
    "msda_backward": "odise_b200::msda_backward(Tensor value, Tensor spatial_shapes, Tensor level_start_index, "
                     "Tensor sampling_loc, Tensor attn_weight, Tensor grad_output, int im2col_step, bool deterministic) "
                     "-> (Tensor, Tensor, Tensor)",
    "msda_fused_forward": "odise_b200::msda_fused_forward(Tensor value, Tensor spatial_shapes, "
                          "Tensor level_start_index, Tensor reference_points, Tensor offsets, Tensor logits) -> Tensor",
    "msda_fused_backward": "odise_b200::msda_fused_backward(Tensor value, Tensor spatial_shapes, "
                           "Tensor level_start_index, Tensor reference_points, Tensor offsets, Tensor logits, "
                           "Tensor grad_output, bool deterministic) -> (Tensor, Tensor, Tensor)",
}
FUSED_DTYPES = [torch.float32, torch.float16, torch.bfloat16]
OP_DTYPES = [torch.float32, torch.float64]


@pytest.fixture
def ops(monkeypatch):
    from odise_b200 import lib, msda  # noqa: F401  (importing msda defines the ops)

    def no_library():
        raise AssertionError("a fake implementation loaded the shared library")
    monkeypatch.setattr(lib, "load", no_library)
    return torch.ops.odise_b200


def _op_args(N=2, S=30, M=2, D=32, L=2, Lq=5, P=2, dtype=torch.float32, device="cuda"):
    """value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output of msda_forward / _backward"""
    return [torch.empty(N, S, M, D, dtype=dtype, device=device), torch.empty(L, 2, dtype=torch.int64, device=device),
            torch.empty(L, dtype=torch.int64, device=device), torch.empty(N, Lq, M, L, P, 2, dtype=dtype, device=device),
            torch.empty(N, Lq, M, L, P, dtype=dtype, device=device), torch.empty(N, Lq, M * D, dtype=dtype, device=device)]


def _fused_args(N=2, S=24, M=2, D=32, L=1, Lq=3, P=2, dtype=torch.float32, device="cuda"):
    """value, spatial_shapes, level_start_index, reference_points (float32), offsets, logits, grad_output of the fused
    ops: the shapes of fused_problem(seed=3, N=2, M=2, D=32, shapes=[(6, 4)], Lq=3, P=2) by default"""
    return [torch.empty(N, S, M, D, dtype=dtype, device=device), torch.empty(L, 2, dtype=torch.int64, device=device),
            torch.empty(L, dtype=torch.int64, device=device), torch.empty(N, Lq, L, 2, device=device),
            torch.empty(N, Lq, M, L, P, 2, dtype=dtype, device=device),
            torch.empty(N, Lq, M, L * P, dtype=dtype, device=device),
            torch.empty(N, Lq, M * D, dtype=dtype, device=device)]


def _meta(t):
    return tuple(t.shape), t.dtype, t.device.type, t.is_contiguous()


def test_schemas(ops):
    for name, schema in SCHEMAS.items():
        assert str(getattr(ops, name).default._schema) == schema


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("dtype", OP_DTYPES, ids=str)
def test_op_fake_results(ops, dtype, deterministic):
    """msda_forward -> [N, Lq, M*D]; msda_backward -> shaped like value / sampling_loc / attn_weight; all in the value's
    dtype on its device, as lib.msda_forward(_f64) and lib.msda_backward return them"""
    with FakeTensorMode():
        value, ss, lsi, loc, aw, go = _op_args(dtype=dtype)
        out = ops.msda_forward(value, ss, lsi, loc, aw, 64)
        grads = ops.msda_backward(value, ss, lsi, loc, aw, go, 64, deterministic)
    assert _meta(out) == ((2, 5, 64), dtype, "cuda", True)
    assert len(grads) == 3
    for g, like in zip(grads, (value, loc, aw)):
        assert _meta(g) == (tuple(like.shape), dtype, "cuda", True)


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("dtype", FUSED_DTYPES, ids=str)
def test_fused_fake_results(ops, dtype, deterministic):
    """msda_fused_forward -> [N, Lq, M*D] in the value's dtype; msda_fused_backward -> shaped like value / offsets /
    logits in the value's dtype (grad_value too: lib rounds the 16-bit default path's float32 buffer)"""
    with FakeTensorMode():
        value, ss, lsi, ref, offs, logits, go = _fused_args(dtype=dtype)
        out = ops.msda_fused_forward(value, ss, lsi, ref, offs, logits)
        grads = ops.msda_fused_backward(value, ss, lsi, ref, offs, logits, go, deterministic)
    assert _meta(out) == ((2, 3, 64), dtype, "cuda", True)
    assert len(grads) == 3
    for g, like in zip(grads, (value, offs, logits)):
        assert _meta(g) == (tuple(like.shape), dtype, "cuda", True)


def _nc(t):
    """t with the same shape and values, not contiguous"""
    return t.transpose(0, 1).contiguous().transpose(0, 1)


@pytest.mark.parametrize("deterministic", [False, True])
def test_fused_fake_errors_float32(ops, deterministic):
    """the inputs tests/test_gpu_msda_module.py::test_fused_errors gives lib.msda_fused_forward / _backward"""
    fwd, bwd = ops.msda_fused_forward, ops.msda_fused_backward
    with FakeTensorMode():
        args = _fused_args()
        value, ss, lsi, ref, offs, logits, go = args
        bad = [
            (bwd, [t.cpu() for t in args]),                                                  # CPU tensors
            (fwd, [value.cpu(), ss, lsi, ref, offs, logits]),
            (bwd, [value, ss, lsi, ref, offs, logits, _nc(go)]),                             # non-contiguous
            (fwd, [value, ss, lsi, _nc(ref), offs, logits]),
            (bwd, [value.half(), ss, lsi, ref.half(), offs.half(), logits.half(), go.half()]),  # float16
            (fwd, [value.double(), ss, lsi, ref.double(), offs.double(), logits.double()]),     # float64
            (bwd, [value, ss, lsi, ref, offs, logits[..., :1].contiguous(), go]),             # shapes that disagree
            (fwd, [value, ss, lsi, ref[:, :2].contiguous(), offs, logits]),
            (bwd, _fused_args(N=1, D=64)),                                                    # D = 64: no fused backward
            (bwd, _fused_args(N=1, S=36, L=4, P=9)),                                          # L * P = 36 > 32
            (bwd, _fused_args(N=1, S=2 ** 26, M=1, D=32)),                                    # S * M * D = 2^31
        ]
        for i, (fn, a) in enumerate(bad):
            a = a + [deterministic] if fn is bwd else a
            with pytest.raises(RuntimeError):
                fn(*a)
                pytest.fail(f"case {i} did not raise")


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=str)
def test_fused_fake_errors_16bit(ops, dtype, deterministic):
    """the inputs tests/test_gpu_msda_16bit.py::test_16bit_errors gives lib.msda_fused_forward_16bit / _backward_16bit
    (its float32 cases run the float32 path through the op, which test_fused_fake_errors_float32 covers)"""
    other = torch.bfloat16 if dtype == torch.float16 else torch.float16
    fwd, bwd = ops.msda_fused_forward, ops.msda_fused_backward
    with FakeTensorMode():
        args = _fused_args(dtype=dtype)
        value, ss, lsi, ref, offs, logits, go = args
        bad = [
            (bwd, [t.cpu() for t in args]),                                                  # CPU tensors
            (fwd, [value.cpu(), ss, lsi, ref, offs, logits]),
            (bwd, [value, ss, lsi, ref, offs, logits, _nc(go)]),                             # non-contiguous
            (fwd, [value, ss, lsi, _nc(ref), offs, logits]),
            (fwd, [value, ss, lsi, ref, offs.to(other), logits]),                            # mixed dtypes
            (fwd, [value, ss, lsi, ref, offs, logits.float()]),
            (bwd, [value, ss, lsi, ref, offs, logits, go.float()]),
            (fwd, [value, ss, lsi, ref.to(dtype), offs, logits]),                            # reference points 16 bits
            (bwd, [value, ss, lsi, ref, offs, logits[..., :1].contiguous(), go]),             # shapes that disagree
            (fwd, [value, ss, lsi, ref[:, :2].contiguous(), offs, logits]),
        ]
        for shape in (dict(N=1, D=64), dict(N=1, S=36, L=4, P=9), dict(N=1, S=2 ** 26, M=1, D=32)):
            b = _fused_args(**shape, dtype=dtype)                                             # unsupported shapes
            bad += [(fwd, b[:6]), (bwd, b)]
        for i, (fn, a) in enumerate(bad):
            a = a + [deterministic] if fn is bwd else a
            with pytest.raises(RuntimeError):
                fn(*a)
                pytest.fail(f"case {i} did not raise")


@pytest.mark.parametrize("deterministic", [False, True])
def test_op_fake_errors(ops, deterministic):
    """msda_forward / msda_backward refuse what lib.msda_forward(_f64) / lib.msda_backward refuse: CPU, non-contiguous,
    mixed or unsupported dtypes, a grad_output of the wrong size and a batch that min(batch, im2col_step) does not
    divide"""
    fwd, bwd = ops.msda_forward, ops.msda_backward
    with FakeTensorMode():
        args = _op_args()
        value, ss, lsi, loc, aw, go = args
        bad = [
            (bwd, [t.cpu() for t in args]),
            (fwd, [value, ss, lsi, loc.cpu(), aw]),
            (fwd, [value, ss, lsi, _nc(loc), aw]),
            (bwd, [value, ss, lsi, loc, aw, _nc(go)]),
            (fwd, [value.half(), ss, lsi, loc.half(), aw.half()]),
            (fwd, [value.double(), ss, lsi, loc, aw]),
            (bwd, [value, ss, lsi, loc, aw, go.double()]),
            (bwd, [value, ss, lsi, loc, aw, go[:, :1].contiguous()]),
        ]
        for i, (fn, a) in enumerate(bad):
            with pytest.raises(RuntimeError):
                fn(*a, 64, deterministic) if fn is bwd else fn(*a, 64)
                pytest.fail(f"case {i} did not raise")
        a3 = _op_args(N=3)
        with pytest.raises(RuntimeError):                                # min(3, 2) = 2 does not divide 3
            fwd(*a3[:5], 2)
        with pytest.raises(RuntimeError):
            bwd(*a3, 2, deterministic)


def test_real_op_on_cpu_raises_runtime_error():
    """the implementation is registered for every device: CPU tensors reach lib's check (a RuntimeError, not the
    dispatcher's NotImplementedError for a missing kernel), before the library is needed"""
    from odise_b200 import msda  # noqa: F401
    for fn, args in ((torch.ops.odise_b200.msda_fused_forward, _fused_args(device="cpu")[:6]),
                     (torch.ops.odise_b200.msda_fused_backward, _fused_args(device="cpu") + [False]),
                     (torch.ops.odise_b200.msda_forward, _op_args(device="cpu")[:5] + [64]),
                     (torch.ops.odise_b200.msda_backward, _op_args(device="cpu") + [64, True])):
        with pytest.raises(RuntimeError) as e:
            fn(*args)
        assert not isinstance(e.value, NotImplementedError)
        assert "CUDA" in str(e.value)
