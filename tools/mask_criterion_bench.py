"""Benchmark of the SetCriterion drop-in (odise_b200.criterion): the full criterion forward + backward over 10 prediction
sets (final + 9 aux), fused (odise_mask_* kernels) against use_fused = False (the composed torch path), arms alternated:

  fused_f32 / composed_f32      float32 pred_masks
  fused_bf16 / composed_bf16    bfloat16 pred_masks under torch.autocast("cuda", torch.bfloat16)

Shapes: ODISE LSJ training, 1024 x 1024 bool target masks, pred_masks [B, 100, 256, 256], pred_logits with 133 classes +
no-object, the ODISE criterion (12544 points, oversample 3.0, importance 0.75); B = 4 with T = (6, 15, 30, 60) and
B = 8 with that list twice.  Per (shape, arm): median ms over --iters iterations (host clock around a step that ends in
a device synchronise; the step synchronises anyway for scipy), and torch.cuda.max_memory_allocated above the inputs for
one forward + backward, gradients included.  The device name and power limit are read in the same run.  Prints one JSON
line.

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
from odise_b200.criterion import HungarianMatcher, SetCriterion  # noqa: E402
from msda_backward_bench import gpu_info  # noqa: E402

Q, K, SETS, P = 100, 133, 10, 12544
SHAPES = {"B4": (6, 15, 30, 60), "B8": (6, 15, 30, 60) * 2}
ARMS = {"fused_f32": (None, True), "composed_f32": (None, False),
        "fused_bf16": (torch.bfloat16, True), "composed_bf16": (torch.bfloat16, False)}


def problem(counts, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    B = len(counts)

    def one():
        low = torch.randn(B, Q, 16, 16, generator=g) * 6
        pm = F.interpolate(low, size=(256, 256), mode="bilinear", align_corners=False)
        return {"pred_logits": (torch.randn(B, Q, K + 1, generator=g) * 2).cuda(),
                "pred_masks": pm.to("cuda", dtype).requires_grad_(True)}
    outputs = one()
    outputs["aux_outputs"] = [one() for _ in range(SETS - 1)]
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
    dtype, fused = ARMS[arm]
    crit.use_fused = fused
    with (torch.autocast("cuda", dtype=dtype) if dtype is not None else contextlib.nullcontext()):
        losses = crit(outputs, targets)
    total = sum(crit.weight_dict[k] * v for k, v in losses.items())
    return torch.autograd.grad(total, leaves(outputs))


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
        peaks = {}
        for arm in ARMS:
            outputs, targets = data[ARMS[arm][0] or torch.float32]
            for _ in range(a.warmup):
                step(crit, outputs, targets, arm)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            g = step(crit, outputs, targets, arm)
            torch.cuda.synchronize()
            peaks[arm] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
            del g
        for _ in range(a.iters):
            for arm in ARMS:
                outputs, targets = data[ARMS[arm][0] or torch.float32]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                g = step(crit, outputs, targets, arm)
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t0) * 1e3)
                del g
        med = {arm: round(sorted(v)[len(v) // 2], 2) for arm, v in times.items()}
        res["shapes"][shape] = {"T": list(counts), "median_ms": med, "peak_mib_above_inputs": peaks,
                                "speedup_f32": round(med["composed_f32"] / med["fused_f32"], 2),
                                "speedup_bf16": round(med["composed_bf16"] / med["fused_bf16"], 2)}
        del data
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
