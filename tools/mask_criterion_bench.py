"""Benchmark of the SetCriterion drop-in (odise_b200.criterion): the full criterion forward + backward over 10 prediction
sets (final + 9 aux), fused (odise_mask_* kernels) against use_fused = False (the composed torch path), arms alternated:

  fused_f32 / fused_f32_dev / composed_f32      float32 pred_masks
  fused_bf16 / fused_bf16_dev / composed_bf16   bfloat16 pred_masks under torch.autocast("cuda", torch.bfloat16)

The _dev arms set match_on_device (the assignment on the device, no synchronisation); the others match with scipy.

Shapes: ODISE LSJ training, 1024 x 1024 bool target masks, pred_masks [B, 100, 256, 256], pred_logits with 133 classes +
no-object, the ODISE criterion (12544 points, oversample 3.0, importance 0.75); B = 4 with T = (6, 15, 30, 60) and
B = 8 with that list twice.  Per (shape, arm): median ms over --iters iterations (host clock around a step that ends in
a device synchronise; the step synchronises anyway for scipy), and torch.cuda.max_memory_allocated above the inputs for
one forward + backward, gradients included, and the median host ms until forward returns (the host's enqueue time, plus
the wait for the cost copy on the scipy arms).  The assignment alone at B = 4, 8 and 32 (T = (6, 15, 30, 60) repeated,
costs of 10 prediction sets from the matcher): the median ms of lib.mask_assign by CUDA events against the host route
(cost copy, synchronisation, scipy, tables sent back; host clock up to a device synchronise).  The device name and power
limit are read in the same run.  Prints one JSON line.

    python tools/mask_criterion_bench.py [--iters 20] [--warmup 3]
"""
import argparse
import contextlib
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from odise_b200 import lib  # noqa: E402
from odise_b200.criterion import HungarianMatcher, SetCriterion, _assign, _Targets  # noqa: E402
from msda_backward_bench import gpu_info  # noqa: E402

Q, K, SETS, P = 100, 133, 10, 12544
SHAPES = {"B4": (6, 15, 30, 60), "B8": (6, 15, 30, 60) * 2}
ARMS = {"fused_f32": (None, True, False), "fused_f32_dev": (None, True, True), "composed_f32": (None, False, False),
        "fused_bf16": (torch.bfloat16, True, False), "fused_bf16_dev": (torch.bfloat16, True, True),
        "composed_bf16": (torch.bfloat16, False, False)}
ASSIGN_B = (4, 8, 32)


def problem(counts, dtype, seed=0, sets=SETS):
    g = torch.Generator().manual_seed(seed)
    B = len(counts)

    def one():
        low = torch.randn(B, Q, 16, 16, generator=g) * 6
        pm = F.interpolate(low, size=(256, 256), mode="bilinear", align_corners=False)
        return {"pred_logits": (torch.randn(B, Q, K + 1, generator=g) * 2).cuda(),
                "pred_masks": pm.to("cuda", dtype).requires_grad_(True)}
    outputs = one()
    outputs["aux_outputs"] = [one() for _ in range(sets - 1)]
    yy, xx = torch.meshgrid(torch.linspace(0, 1, 1024), torch.linspace(0, 1, 1024), indexing="ij")
    targets = []
    for T in counts:
        c, r = torch.rand(T, 2, generator=g), 0.08 + 0.3 * torch.rand(T, 1, 1, generator=g)
        m = ((yy - c[:, 0, None, None]) ** 2 + (xx - c[:, 1, None, None]) ** 2) < r ** 2
        targets.append({"labels": torch.randint(0, K, (T,), generator=g).cuda(), "masks": m.cuda()})
    return outputs, targets


def leaves(outputs):
    return [outputs["pred_masks"]] + [a["pred_masks"] for a in outputs["aux_outputs"]]


def step(crit, outputs, targets, arm):
    """one forward + backward -> (gradients, host ms until forward returned)"""
    dtype, fused, dev = ARMS[arm]
    crit.use_fused, crit.match_on_device = fused, dev
    t0 = time.perf_counter()
    with (torch.autocast("cuda", dtype=dtype) if dtype is not None else contextlib.nullcontext()):
        losses = crit(outputs, targets)
    fwd = (time.perf_counter() - t0) * 1e3
    total = sum(crit.weight_dict[k] * v for k, v in losses.items())
    return torch.autograd.grad(total, leaves(outputs)), fwd


def assign_times(crit, B, iters, warmup):
    """median ms of the assignment of 10 sets' costs: lib.mask_assign (CUDA events) and the host route"""
    counts = SHAPES["B4"] * (B // 4)
    outputs, targets = problem(counts, torch.float32, sets=1)
    m, tg = crit.matcher, _Targets(targets)
    C = torch.empty(SETS, B, Q, tg.Tmax, device="cuda")
    with torch.no_grad():
        for l in range(SETS):
            m._costs(outputs, tg, m._draw(B, C.device), C[l])
    del outputs
    dev, host = [], []
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for i in range(warmup + iters):
        torch.cuda.synchronize()
        ev[0].record()
        lib.mask_assign(C, counts)
        ev[1].record()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        SetCriterion._tables(_assign(C, counts), counts, Q, C.device)
        torch.cuda.synchronize()
        if i >= warmup:
            dev.append(ev[0].elapsed_time(ev[1]))
            host.append((time.perf_counter() - t0) * 1e3)
    med = lambda v: round(sorted(v)[len(v) // 2], 3)  # noqa: E731
    return {"T": list(counts), "device_ms": med(dev), "host_route_ms": med(host)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mask_criterion_bench needs a CUDA device")
    name, power, clock = gpu_info()
    crit = SetCriterion(K, HungarianMatcher(2.0, 5.0, 5.0, P), 2.0, 5.0, 5.0, SETS - 1, 0.1, ["labels", "masks"], P,
                        3.0, 0.75).cuda()
    res = {"device": name, "power_limit": power, "max_sm_clock": clock, "iters": a.iters, "shapes": {}}
    for shape, counts in SHAPES.items():
        data = {dt: problem(counts, dt) for dt in (torch.float32, torch.bfloat16)}
        times = {arm: [] for arm in ARMS}
        fwd = {arm: [] for arm in ARMS}
        peaks = {}
        for arm in ARMS:
            outputs, targets = data[ARMS[arm][0] or torch.float32]
            for _ in range(a.warmup):
                step(crit, outputs, targets, arm)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            g, _ = step(crit, outputs, targets, arm)
            torch.cuda.synchronize()
            peaks[arm] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
            del g
        for _ in range(a.iters):
            for arm in ARMS:
                outputs, targets = data[ARMS[arm][0] or torch.float32]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                g, f = step(crit, outputs, targets, arm)
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t0) * 1e3)
                fwd[arm].append(f)
                del g
        med = {arm: round(sorted(v)[len(v) // 2], 2) for arm, v in times.items()}
        res["shapes"][shape] = {"T": list(counts), "median_ms": med, "peak_mib_above_inputs": peaks,
                                "forward_host_ms": {arm: round(sorted(v)[len(v) // 2], 2) for arm, v in fwd.items()},
                                "speedup_f32": round(med["composed_f32"] / med["fused_f32"], 2),
                                "speedup_bf16": round(med["composed_bf16"] / med["fused_bf16"], 2),
                                "speedup_dev_f32": round(med["fused_f32"] / med["fused_f32_dev"], 3),
                                "speedup_dev_bf16": round(med["fused_bf16"] / med["fused_bf16_dev"], 3)}
        del data
        torch.cuda.empty_cache()
    res["assign"] = {f"B{B}": assign_times(crit, B, a.iters, a.warmup) for B in ASSIGN_B}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
