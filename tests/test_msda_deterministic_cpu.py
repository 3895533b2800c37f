"""CPU checks of the deterministic MSDeformAttn backward entry points (odise_msda_*_det_*): they are bound from
lib._PROTOS, return ODISE_ERR_ARG / ODISE_ERR_WORKSPACE / ODISE_ERR_UNSUPPORTED without touching a device, and the
workspace size is the int64 accumulator plus two 8-byte maxima per (image, head)."""
import pytest
import torch

ERR_ARG, ERR_WORKSPACE, ERR_UNSUPPORTED = 10001, 10005, 10006      # include/odise_b200.h

# name -> number of pointer arguments before the seven sizes (N, S, M, D, L, Lq, P)
TWINS = {
    "odise_msda_backward_det_f32": 9,
    "odise_msda_backward_det_f64": 9,
    "odise_msda_fused_backward_det_f32": 10,
    "odise_msda_fused_backward_det_f16": 10,
    "odise_msda_fused_backward_det_bf16": 10,
}


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


def test_bindings_follow_header_prototypes(built):
    from odise_b200 import lib
    L = lib.load()
    for name, n in TWINS.items():
        default = name.replace("_det", "")
        assert lib._PROTOS[name][1] == lib._PROTOS[default][1][:-1] + [lib.c_void_p, lib.c_void_p], name
        assert len(lib._PROTOS[name][1]) == n + 7 + 2
        assert getattr(L, name).restype is lib.c_int
    assert "odise_msda_det_workspace_bytes" in lib._PROTOS
    assert L.odise_msda_det_workspace_bytes.restype is lib.c_longlong


def test_workspace_bytes(built):
    from odise_b200 import lib
    L = lib.load()
    assert L.odise_msda_det_workspace_bytes(2, 10, 3, 32) == 8 * (2 * 10 * 3 * 32 + 2 * 2 * 3)
    # the ODISE 1024^2 shape at N = 4: beyond 32 bits, returned in full
    S = 128 * 128 + 64 * 64 + 32 * 32
    assert L.odise_msda_det_workspace_bytes(4, S, 8, 32) == 8 * (4 * S * 8 * 32 + 2 * 4 * 8)
    assert L.odise_msda_det_workspace_bytes(512, S, 8, 32) > 2 ** 32
    assert L.odise_msda_det_workspace_bytes(0, 10, 3, 32) == 0


@pytest.mark.parametrize("name", sorted(TWINS))
def test_argument_validation_without_gpu(built, name):
    from odise_b200 import lib
    fn = getattr(lib.load(), name)
    n = TWINS[name]
    p = 16       # any non-null address: every call below fails its checks before anything is dereferenced or launched
    dims = [1, 1, 1, 32, 1, 1, 1]
    assert fn(*([None] * n), *dims, None, None) == ERR_ARG
    for i in range(n):                                                   # each pointer missing in turn
        args = [p] * n
        args[i] = None
        assert fn(*args, *dims, p, None) == ERR_ARG, i
    assert fn(*([p] * n), *dims, None, None) == ERR_WORKSPACE            # only the workspace missing
    for bad in range(7):                                                 # N S M D L Lq P
        d = list(dims)
        d[bad] = 0
        assert fn(*([p] * n), *d, p, None) == ERR_ARG, bad
    assert fn(*([p] * n), 1, 1, 1, 32, 9, 1, 1, p, None) == ERR_ARG      # L > 8
    if "fused" in name:
        assert fn(*([p] * n), 1, 1, 1, 64, 1, 1, 1, p, None) == ERR_UNSUPPORTED         # D != 32
        assert fn(*([p] * n), 1, 1, 1, 32, 3, 1, 11, p, None) == ERR_UNSUPPORTED        # L * P = 33 > 32


def test_deterministic_python_entry_points_have_no_cpu_path():
    from odise_b200 import lib
    ss, lsi = torch.tensor([[2, 2], [1, 1]]), torch.tensor([0, 4])
    value = torch.zeros(1, 5, 2, 32)
    loc, aw = torch.zeros(1, 5, 2, 2, 2, 2), torch.zeros(1, 5, 2, 2, 2)
    offs, logits, r = torch.zeros(1, 5, 2, 2, 2, 2), torch.zeros(1, 5, 2, 4), torch.zeros(1, 5, 2, 2)
    go = torch.zeros(1, 5, 64)
    with pytest.raises(RuntimeError):
        lib.msda_backward(value, ss, lsi, loc, aw, go, 64, deterministic=True)
    with pytest.raises(RuntimeError):
        lib.msda_fused_backward(value, ss, lsi, r, offs, logits, go, deterministic=True)
    with pytest.raises(RuntimeError):
        lib.msda_fused_backward_16bit(value.bfloat16(), ss, lsi, r, offs.bfloat16(), logits.bfloat16(), go.bfloat16(),
                                      deterministic=True)
