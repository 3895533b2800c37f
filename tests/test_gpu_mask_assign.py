"""GPU checks of the device assignment (odise_mask_assign_f32, lib.mask_assign) and of SetCriterion.match_on_device:
scipy's pair tables bit for bit on 27 260 problems of five cost families (ties, duplicates, constants, sprinkled +inf),
status codes where scipy raises, the criterion's losses, gradients and RNG state against the scipy path, no
synchronisation (alone and in a single-rank NCCL group), the fallbacks to scipy and CUDA-graph capture."""
import warnings

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

from test_gpu_mask_criterion import _criterion, _problem, _sets
from test_mask_assign_cpu import FAMILIES, _family

pytestmark = pytest.mark.gpu


def _want(C, counts):
    """the tables the scipy path builds (SetCriterion._tables of criterion._assign)"""
    from odise_b200.criterion import SetCriterion, _assign
    return SetCriterion._tables(_assign(C, counts), counts, C.shape[2], C.device)


def _got(C, counts):
    from odise_b200 import lib
    from odise_b200.criterion import SetCriterion
    L, B, Q = C.shape[:3]
    buf, status = lib.mask_assign(C, counts)
    assert buf.numel() == L * (3 * sum(min(Q, T) for T in counts) + 2 * B * Q)
    return SetCriterion._split_tables(buf, [sum(min(Q, T) for T in counts)] * L, B, Q), status


def _assert_tables_equal(got, want, what):
    assert len(got) == len(want)
    for l, (a, b) in enumerate(zip(got, want)):
        for k in ("pairs", "pair_of", "tg_of"):
            assert torch.equal(a[k], b[k]), (what, l, k)


def _costs(rng, kind, L, Q, counts, cuda):
    """[L, B, Q, Tmax] of one family; the columns t >= T_b are NaN, which the solver must never read"""
    C = np.full((L, len(counts), Q, max(counts, default=0)), np.nan, np.float32)
    for l in range(L):
        for b, T in enumerate(counts):
            C[l, b, :, :T] = _family(rng, kind, Q, T)
    return torch.from_numpy(C).to(cuda)


def _counts(rng, Q, B):
    """B target counts around Q (0, 1, Q - 1, Q, Q + 1), a few up to MASK_MAX_ASSIGN, the rest random"""
    from odise_b200 import lib
    edge = [0, 1, max(Q - 1, 0), Q, Q + 1, lib.MASK_MAX_ASSIGN]
    out = [edge[b] if b < len(edge) else int(rng.integers(0, 3 * Q + 3)) for b in range(B)]
    rng.shuffle(out)
    return out


# (Q, B, L): the largest problems at small B, so that the cost buffer stays below ~150 MB
SHAPES = [(1, 256, 10), (7, 256, 10), (100, 32, 10), (300, 6, 2)]


@pytest.mark.parametrize("kind", FAMILIES)
def test_bit_identical_to_scipy(cuda, kind):
    rng = np.random.default_rng(FAMILIES.index(kind))
    n = 0
    for Q, B, L in SHAPES:
        counts = _counts(rng, Q, B)
        C = _costs(rng, kind, L, Q, counts, cuda)
        got, status = _got(C, counts)
        assert torch.equal(status, torch.zeros(L, B, dtype=torch.int32, device=cuda)), (kind, Q)
        _assert_tables_equal(got, _want(C, counts), (kind, Q, counts))
        n += L * B
    assert n >= 5400        # x 5 families: over 20 000 problems


def test_invalid_costs_give_status_and_in_range_tables(cuda):
    from odise_b200.criterion import SetCriterion
    rng = np.random.default_rng(7)
    Q, counts = 6, [4, 6, 9]
    C = _costs(rng, "gauss", 2, Q, counts, cuda)
    C[0, 1, 2, 3] = float("nan")
    C[1, 0, 1, 1] = float("-inf")
    C[1, 2, 3, :9] = float("inf")            # query 3 of a T > Q problem has no finite cost: infeasible
    failed = {(0, 1): 1, (1, 0): 1, (1, 2): 2}
    host = C.cpu().numpy()
    indices = []
    for l in range(2):
        per = []
        for b, T in enumerate(counts):
            if (l, b) in failed:
                with pytest.raises(ValueError):
                    linear_sum_assignment(host[l, b, :, :T])
                m = min(Q, T)
                per.append((torch.arange(m), torch.arange(m)))
            else:
                i, j = linear_sum_assignment(host[l, b, :, :T])
                per.append((torch.as_tensor(i, dtype=torch.int64), torch.as_tensor(j, dtype=torch.int64)))
        indices.append(per)
    got, status = _got(C, counts)
    want_status = torch.zeros(2, 3, dtype=torch.int32)
    for (l, b), s in failed.items():
        want_status[l, b] = s
    assert torch.equal(status.cpu(), want_status)
    _assert_tables_equal(got, SetCriterion._tables(indices, counts, Q, cuda), "invalid")
    offs = np.cumsum([0] + counts)
    for tab in got:
        p = tab["pairs"].cpu()
        for b in range(3):
            rows = p[p[:, 0] == b]
            assert ((rows[:, 1] >= 0) & (rows[:, 1] < Q)).all()
            assert ((rows[:, 2] >= offs[b]) & (rows[:, 2] < offs[b + 1])).all()


def _record_assign(monkeypatch):
    from odise_b200 import criterion
    seen = []
    real = criterion._assign

    def rec(C, counts):
        seen.append(C.shape)
        return real(C, counts)
    monkeypatch.setattr(criterion, "_assign", rec)
    return seen


def _step(crit, outputs, targets, dtype, on_device, seed=0):
    """seeded forward + backward -> (losses, pred_masks gradients, CUDA RNG state after)"""
    crit.match_on_device = on_device
    torch.manual_seed(seed)
    with torch.autocast("cuda", dtype=dtype, enabled=dtype is not None):
        losses = crit(outputs, targets)
    total = sum(crit.weight_dict[k] * v for k, v in losses.items())
    grads = torch.autograd.grad(total, [s["pred_masks"] for s in _sets(outputs)])
    return {k: v.detach() for k, v in losses.items()}, grads, torch.cuda.get_rng_state()


@pytest.mark.parametrize("dtype", [None, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("counts", [(6, 15), (0, 120, 7)])
def test_criterion_device_vs_scipy(cuda, monkeypatch, dtype, counts):
    outputs, targets = _problem(cuda, counts, Q=100, pred_hw=(64, 64), tgt_hw=(256, 256))
    crit = _criterion(cuda)
    ls, gs, rs = _step(crit, outputs, targets, dtype, False)
    seen = _record_assign(monkeypatch)
    runs = [_step(crit, outputs, targets, dtype, True), _step(crit, outputs, targets, dtype, True)]
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        runs.append(_step(crit, outputs, targets, dtype, True))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert seen == []
    assert crit.match_status.shape == (10, len(counts)) and not crit.match_status.any()
    for ld, gd, rd in runs:
        assert list(ld) == list(ls) and len(ld) == 30
        for k in ls:
            assert torch.equal(ld[k], ls[k]), k
        for a, b in zip(gd, gs):
            assert torch.equal(a, b)
        assert torch.equal(rd, rs)


def _count_syncs(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return [str(x.message) for x in w if "called a synchronizing" in str(x.message)]


def test_no_syncs(cuda, tmp_path):
    import torch.distributed as dist
    outputs, targets = _problem(cuda, (6, 15, 30, 60), Q=100, pred_hw=(64, 64), tgt_hw=(256, 256))
    crit = _criterion(cuda)
    _step(crit, outputs, targets, None, True)
    torch.cuda.synchronize()
    syncs = _count_syncs(lambda: _step(crit, outputs, targets, None, True))
    assert syncs == [], syncs

    dist.init_process_group("nccl", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0, world_size=1)
    try:
        lh, gh, _ = _step(crit, outputs, targets, None, False)
        ld, gd, _ = _step(crit, outputs, targets, None, True)
        torch.cuda.synchronize()
        syncs = _count_syncs(lambda: _step(crit, outputs, targets, None, True))
        assert syncs == [], syncs
        for k in lh:
            torch.testing.assert_close(ld[k], lh[k], rtol=1e-6, atol=0, msg=k)
        for a, b in zip(gd, gh):
            assert (a - b).abs().max() <= 1e-6 * b.abs().max()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("case", ["use_fused_off", "Q_over_limit"])
def test_fallbacks_take_scipy(cuda, monkeypatch, case):
    """Sets off the fused path, or max(Q, T) > MASK_MAX_ASSIGN: match_on_device runs scipy and computes what the default
    path computes (the composed path's gradients up to the order of grid_sample's backward atomics)."""
    from odise_b200 import lib
    Q = lib.MASK_MAX_ASSIGN + 1 if case == "Q_over_limit" else 100
    outputs, targets = _problem(cuda, (3, 5), Q=Q, pred_hw=(32, 32), tgt_hw=(64, 64), sets=3)
    crit = _criterion(cuda, P=1024)
    crit.use_fused = case != "use_fused_off"
    seen = _record_assign(monkeypatch)
    lw, gw, rw = _step(crit, outputs, targets, None, False)
    ld, gd, rd = _step(crit, outputs, targets, None, True)
    assert len(seen) == 2 and crit.match_status is None
    for k in lw:
        assert torch.equal(ld[k], lw[k]), k
    for a, b in zip(gd, gw):
        if crit.use_fused:
            assert torch.equal(a, b)
        else:
            assert (a - b).abs().max() <= 1e-6 * b.abs().max()
    assert torch.equal(rd, rw)


def test_graph_capture(cuda):
    from odise_b200 import lib
    rng = np.random.default_rng(11)
    L, Q, counts = 3, 100, [0, 37, 100, 160, 99]
    C = _costs(rng, "int012", L, Q, counts, cuda)
    lib.mask_assign(C, counts)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        buf, status = lib.mask_assign(C, counts)
    from odise_b200.criterion import SetCriterion
    N = sum(min(Q, T) for T in counts)
    for kind in ("gauss", "dup", "inf"):
        C.copy_(_costs(rng, kind, L, Q, counts, cuda))
        g.replay()
        assert not status.any()
        _assert_tables_equal(SetCriterion._split_tables(buf, [N] * L, len(counts), Q), _want(C, counts), kind)
