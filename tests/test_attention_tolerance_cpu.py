"""The error bar of tests/test_gpu_attention.py (TOL3, bf16x3 mode) checked against a CPU emulation of the kernel's
arithmetic on every case of that file's tables, with the same data.

Emulated rounding (odise_b200/csrc/attn_tc.cu): q and k split into bf16 (hi, lo) pairs, S = hi.hi + hi.lo + lo.hi in
fp32; P = exp(S - rowmax) rounded once to fp16 for the P V product, the row sum l taken from the unrounded P; V^T as an
fp16 (hi, lo) pair.  Every emulated error must sit below half the bar, so that the bar keeps a 2x margin for what the
emulation leaves out (the online rescale, fp32 accumulation order, ex2.approx) as cases are added."""
import pytest
import torch

import test_gpu_attention as G


def _bf(x):
    return x.to(torch.bfloat16).float()


def _hf(x):
    return x.to(torch.float16).float()


def emulate_rel(q, k, v, scale, allowed=None):
    """max |emulated - fp64| / max |fp64| over the whole output, one (image, head) at a time"""
    B, Tq, H, d = q.shape
    qh, kh, vh = _bf(q), _bf(k), _hf(v)
    ql, kl, vl = _bf(q - qh), _bf(k - kh), _hf(v - vh)
    err = ref_max = 0.0
    for b in range(B):
        blocked = None if allowed is None else ~allowed[b]
        for h in range(H):
            s = (qh[b, :, h] @ kh[b, :, h].T + qh[b, :, h] @ kl[b, :, h].T + ql[b, :, h] @ kh[b, :, h].T) * scale
            s64 = (q[b, :, h].double() @ k[b, :, h].double().T) * scale
            if blocked is not None:
                s = s.masked_fill(blocked, float("-inf"))
                s64 = s64.masked_fill(blocked, float("-inf"))
            p = torch.exp(s - s.max(-1, keepdim=True).values)
            p16 = _hf(p)
            o = (p16 @ vh[b, :, h] + p16 @ vl[b, :, h]) / p.sum(-1, keepdim=True)
            ref = s64.softmax(-1) @ v[b, :, h].double()
            err = max(err, (o.double() - ref).abs().max().item())
            ref_max = max(ref_max, ref.abs().max().item())
    return err / ref_max


def _check(record_line, e):
    print(f"{record_line}: emulated rel err {e:.3e} (bar {G.TOL3:.0e})")
    assert e < G.TOL3 / 2


@pytest.mark.parametrize("cfg", G.TC_CASES)
def test_bar_covers_unmasked_cases(cfg):
    q, k, v = G.tc_case(cfg)
    _check(f"attention_tc {cfg}", emulate_rel(q, k, v, cfg[2] ** -0.5))


@pytest.mark.parametrize("case", G.MASKED_CASES, ids=lambda c: "-".join(map(str, c)))
def test_bar_covers_masked_cases(case):
    q, k, v, allowed, row_any, _, _ = G.masked_case(case)
    _check(f"attention_tc masked {case}", emulate_rel(q, k, v, case[3] ** -0.5, G.effective_mask(allowed, row_any)))


@pytest.mark.parametrize("case", G.STRESS_CASES, ids=lambda c: "-".join(map(str, c)))
def test_bar_covers_stress_cases(case):
    q, k, v = G.stress_case(case)
    _check(f"attention_tc stress {case}", emulate_rel(q, k, v, case[3] ** -0.5))

