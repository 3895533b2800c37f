"""CPU checks of the device assignment (odise_mask_assign_f32, lib.mask_assign, SetCriterion.match_on_device): scipy's
algorithm restated in the form the kernel computes it, compared with scipy itself on mixed and tie-heavy problems;
lib's argument checks without data and without the library; the C ABI's argument checks without a device."""
import ctypes

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment
from torch._subclasses.fake_tensor import FakeTensorMode

MAX = 1024      # ODISE_MASK_MAX_ASSIGN: the rank offset of the kernel's column key


def lsap_restated(cost):
    """scipy's shortest augmenting path as mc_assign_kernel runs it: fp64, scipy's operand order, and the column choice
    as the warp reduction makes it, the minimum of (reduced cost, rank) with rank = MAX - 1 - it for an unassigned
    column and MAX + it for an assigned one.  -> (rows, cols) as scipy returns them; ValueError where scipy raises."""
    c = np.asarray(cost, dtype=np.float64)
    if c.shape[0] == 0 or c.shape[1] == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    tr = c.shape[1] < c.shape[0]
    if tr:
        c = c.T
    if np.isnan(c).any() or (c == -np.inf).any():
        raise ValueError("matrix contains invalid numeric entries")
    nr, nc = c.shape
    u, v = np.zeros(nr), np.zeros(nc)
    path, row4col, col4row = np.full(nc, -1), np.full(nc, -1), np.full(nr, -1)
    for cur in range(nr):
        spc = np.full(nc, np.inf)
        SR, SC = np.zeros(nr, bool), np.zeros(nc, bool)
        rem = np.arange(nc - 1, -1, -1)
        nrem, minVal, i, sink = nc, 0.0, cur, -1
        while sink < 0:
            SR[i] = True
            js = rem[:nrem]
            r = ((minVal + c[i, js]) - u[i]) - v[js]
            upd = r < spc[js]
            path[js[upd]] = i
            spc[js[upd]] = r[upd]
            s, its = spc[js], np.arange(nrem)
            rank = np.where(row4col[js] < 0, MAX - 1 - its, MAX + its)
            m = s.min()
            if m == np.inf:
                raise ValueError("cost matrix is infeasible")
            tied = np.flatnonzero(s == m)
            idx = tied[np.argmin(rank[tied])]
            minVal, j = m, rem[idx]
            if row4col[j] < 0:
                sink = j
            else:
                i = row4col[j]
            SC[j] = True
            nrem -= 1
            rem[idx] = rem[nrem]
        u[cur] += minVal
        others = np.flatnonzero(SR)
        others = others[others != cur]
        u[others] += minVal - spc[col4row[others]]
        v[SC] -= minVal - spc[SC]
        j = sink
        while True:
            i = path[j]
            row4col[j] = i
            col4row[i], j = j, col4row[i]
            if i == cur:
                break
    if tr:
        order = np.argsort(col4row)
        return col4row[order].astype(np.int64), order.astype(np.int64)
    return np.arange(nr, dtype=np.int64), col4row.astype(np.int64)


def _family(rng, kind, Q, T):
    """one float32 [Q, T] cost of a family: gauss, int012, dup (duplicated rows and columns), const, inf (sprinkled
    +inf, kept feasible by a finite diagonal)"""
    if kind == "gauss":
        c = rng.standard_normal((Q, T))
    elif kind == "int012":
        c = rng.integers(0, 3, (Q, T)).astype(np.float64)
    elif kind == "dup":
        c = rng.integers(0, 4, (Q, T)) * 0.25 + rng.standard_normal((Q, T)) * (rng.random() < 0.5)
        if T > 1:
            c[:, rng.integers(0, T, T // 2)] = c[:, rng.integers(0, T, T // 2)]
        if Q > 1:
            c[rng.integers(0, Q, Q // 2)] = c[rng.integers(0, Q, Q // 2)]
    elif kind == "const":
        c = np.full((Q, T), float(rng.integers(-2, 3)))
    else:
        c = rng.standard_normal((Q, T))
        keep = np.arange(min(Q, T))
        c[rng.random((Q, T)) < 0.3] = np.inf
        c[keep, keep] = rng.standard_normal(len(keep))
    return c.astype(np.float32)


FAMILIES = ("gauss", "int012", "dup", "const", "inf")


def test_restatement_matches_scipy():
    """The kernel's form of the algorithm gives scipy's exact indices on 2000+ problems, ties included (fails first if
    scipy ever changes its algorithm or its tie rule)."""
    rng = np.random.default_rng(0)
    n = 0
    for rep in range(420):
        for kind in FAMILIES:
            Q = int(rng.integers(1, 41))
            T = int(rng.choice([0, 1, max(Q - 1, 0), Q, Q + 1, int(rng.integers(0, 51))]))
            c = _family(rng, kind, Q, T)
            i, j = linear_sum_assignment(c)
            a, b = lsap_restated(c)
            assert np.array_equal(i, a) and np.array_equal(j, b), (rep, kind, Q, T)
            n += 1
    assert n >= 2000


@pytest.mark.parametrize("bad", ["nan", "-inf", "infeasible"])
def test_restatement_raises_where_scipy_raises(bad):
    c = np.random.default_rng(1).standard_normal((6, 4)).astype(np.float32)
    if bad == "infeasible":
        c[:, 2] = np.inf
    else:
        c[3, 1] = np.nan if bad == "nan" else -np.inf
    for fn in (linear_sum_assignment, lsap_restated):
        with pytest.raises(ValueError):
            fn(c)


# ---- lib's argument checks (no data, no library) ----

@pytest.fixture
def nolib(monkeypatch):
    from odise_b200 import lib

    def no_library():
        raise AssertionError("an argument check loaded the shared library")
    monkeypatch.setattr(lib, "load", no_library)
    return lib


def test_lib_argument_checks(nolib):
    lib = nolib
    with FakeTensorMode():
        d = "cuda"
        C = torch.empty(2, 3, 5, 4, device=d)
        bad = {
            "float64": lambda: lib.mask_assign(C.double(), [1, 4, 0]),
            "3-D": lambda: lib.mask_assign(C[0], [1, 4, 0]),
            "counts length": lambda: lib.mask_assign(C, [1, 4]),
            "count > Tmax": lambda: lib.mask_assign(C, [1, 5, 0]),
            "negative count": lambda: lib.mask_assign(C, [1, -1, 0]),
            "non-contiguous": lambda: lib.mask_assign(C.transpose(2, 3), [1, 4, 0]),
            "images": lambda: lib.mask_assign(torch.empty(1, lib.MASK_MAX_IMAGES + 1, 2, 1, device=d),
                                              [1] * (lib.MASK_MAX_IMAGES + 1)),
            "queries": lambda: lib.mask_assign(torch.empty(1, 1, lib.MASK_MAX_ASSIGN + 1, 1, device=d), [1]),
            "targets": lambda: lib.mask_assign(torch.empty(1, 1, 2, lib.MASK_MAX_ASSIGN + 1, device=d), [3]),
        }
        for what, call in bad.items():
            with pytest.raises(lib.OdiseError):
                call()
                pytest.fail(what)
    with pytest.raises(lib.OdiseError):       # a real CPU tensor
        lib.mask_assign(torch.zeros(1, 1, 2, 2), [2])


def test_match_on_device_is_a_plain_attribute():
    """Not a constructor argument, not in repr or the state dict; off by default.  On CPU tensors (no fused set) the
    criterion takes the scipy path with it set, and computes what it computes without it."""
    from test_mask_criterion_cpu import _kwargs, _problem, P
    from odise_b200.criterion import HungarianMatcher, SetCriterion
    crit = SetCriterion(matcher=HungarianMatcher(2.0, 5.0, 5.0, P), **_kwargs())
    assert crit.match_on_device is False and "match_on_device" not in repr(crit)
    assert list(crit.state_dict()) == ["empty_weight"]
    outputs, targets = _problem()
    torch.manual_seed(0)
    want = crit(outputs, targets)
    crit.match_on_device = True
    torch.manual_seed(0)
    got = crit(outputs, targets)
    assert crit.match_status is None
    for k in want:
        assert torch.equal(got[k], want[k]), k


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


def test_cabi_export_and_checks(built):
    from odise_b200 import lib
    dll = ctypes.CDLL(built)
    assert hasattr(dll, "odise_mask_assign_f32") and "odise_mask_assign_f32" in lib._PROTOS
    f = lib.load().odise_mask_assign_f32
    p = 256
    cnt = (ctypes.c_int * 3)(1, 4, 0)
    assert f(None, cnt, p, p, 2, 3, 5, 4, None) == 10001            # null cost
    assert f(p, None, p, p, 2, 3, 5, 4, None) == 10001              # null counts
    assert f(p, cnt, None, p, 2, 3, 5, 4, None) == 10001            # null tables
    assert f(p, cnt, p, None, 2, 3, 5, 4, None) == 10001            # null status
    assert f(p, cnt, p, p, 0, 3, 5, 4, None) == 10001               # L = 0
    assert f(p, cnt, p, p, 2, 3, 0, 4, None) == 10001               # Q = 0
    assert f(p, cnt, p, p, 2, 3, 5, 3, None) == 10001               # T_b > Tmax
    assert f(p, cnt, p, p, 2, 300, 5, 4, None) == 10006             # images
    assert f(p, cnt, p, p, 2, 3, lib.MASK_MAX_ASSIGN + 1, 4, None) == 10006
    assert f(p, cnt, p, p, 2, 3, 5, lib.MASK_MAX_ASSIGN + 1, None) == 10006
