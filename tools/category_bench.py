"""Category scoring (CategoryODISE.cal_pred_logits over the 10 prediction sets of a training step): the fused sm_90a
kernels against the reference's composed ops, alternated in one process, in float32, fp16 autocast and bf16 autocast,
at B = 4 and 8 with Q = 100, C = 256 and the COCO training bank (133 classes, 254 prompts).

Per arm it reports
  - the median ms of the 10 calls' forward + backward alone (CUDA events),
  - the median ms of a decoder + scoring + SetCriterion step at 1024^2 crops (mask features 256 x 256),
  - the host enqueue time of the 10 forward calls (a host clock with no synchronisation inside: what the CPU spends
    issuing the work, not GPU time),
  - kernels per 10-call forward + backward, from a separate torch.profiler run,
  - synchronising calls per decoder + scoring + criterion step.
The device name and power limit are read in the same run.  Output: one JSON line per arm, and a markdown table."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from category_ref import coco_labels  # noqa: E402
from odise_b200 import category  # noqa: E402
from odise_b200 import decoder as dec  # noqa: E402
from odise_b200.criterion import HungarianMatcher, SetCriterion  # noqa: E402

LABELS = coco_labels()
K, KP = len(LABELS), sum(len(l) for l in LABELS)
DTYPES = {"fp32": None, "fp16": torch.float16, "bf16": torch.bfloat16}


def scoring_inputs(B, dt, dev, C=256):
    g = torch.Generator().manual_seed(0)
    store = dt or torch.float32
    sets = [torch.randn(B, 100, C, generator=g).to(dev, store).requires_grad_() for _ in range(10)]
    te = torch.randn(KP, C, generator=g).to(dev, store).requires_grad_()
    ne = torch.randn(1, C, generator=g).to(dev, store).requires_grad_()
    ls = torch.tensor(14.3, device=dev, requires_grad=True)
    w = torch.randn(B, 100, K + 1, generator=g).to(dev)
    return sets, te, ne, ls, w


def scoring_step(inp, dt, fused):
    sets, te, ne, ls, w = inp
    for t in sets + [te, ne, ls]:       # as zero_grad(set_to_none=True) leaves them at the start of a step
        t.grad = None
    with torch.autocast("cuda", dtype=dt or torch.float16, enabled=dt is not None):
        outs = [category.cal_pred_logits(dict(mask_embed=m, text_embed=te, null_embed=ne, logit_scale=ls,
                                              labels=LABELS), use_fused=fused) for m in sets]
    torch.autograd.backward(outs, [w.to(o.dtype) for o in outs])


def enqueue_ms(inp, dt, fused, reps):
    sets, te, ne, ls, _ = inp
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad(), torch.autocast("cuda", dtype=dt or torch.float16, enabled=dt is not None):
            for m in sets:
                category.cal_pred_logits(dict(mask_embed=m, text_embed=te, null_embed=ne, logit_scale=ls,
                                              labels=LABELS), use_fused=fused)
        ts.append((time.perf_counter() - t0) * 1e3)
    torch.cuda.synchronize()
    return statistics.median(ts)


def stack(B, dev):
    torch.manual_seed(0)
    d = dec.ODISEMultiScaleMaskedTransformerDecoder(
        in_channels=256, num_classes=K, hidden_dim=256, num_queries=100, nheads=8, dim_feedforward=2048, dec_layers=9,
        pre_norm=False, mask_dim=256, enforce_input_project=False,
        post_mask_embed=dec.PooledMaskEmbed(hidden_dim=256, mask_dim=256, projection_dim=256)).to(dev).train()
    crit = SetCriterion(K, HungarianMatcher(2.0, 5.0, 5.0, num_points=12544), 2.0, 5.0, 5.0, 9, 0.1,
                        ["labels", "masks"], 12544, 3.0, 0.75).to(dev)
    g = torch.Generator().manual_seed(1)
    S = 256      # mask features of a 1024^2 crop at stride 4
    ms = [torch.randn(B, 256, S // s, S // s, generator=g).to(dev) for s in (8, 4, 2)]
    mf = torch.randn(B, 256, S, S, generator=g).to(dev)
    te = torch.randn(KP, 256, generator=g).to(dev).requires_grad_()
    ne = torch.randn(1, 256, generator=g).to(dev).requires_grad_()
    yy, xx = torch.meshgrid(torch.linspace(0, 1, 4 * S), torch.linspace(0, 1, 4 * S), indexing="ij")
    targets = []
    for _ in range(B):
        c = torch.rand(6, 2, generator=g)
        masks = ((yy - c[:, 0, None, None]) ** 2 + (xx - c[:, 1, None, None]) ** 2) < 0.05
        targets.append({"labels": torch.randint(0, K, (6,), generator=g).to(dev), "masks": masks.to(dev)})
    return d, crit, ms, mf, te, ne, targets


def stack_step(st, dt, fused):
    d, crit, ms, mf, te, ne, targets = st
    torch.manual_seed(2)
    d.zero_grad(set_to_none=True)
    te.grad = ne.grad = None
    with torch.autocast("cuda", dtype=dt or torch.float16, enabled=dt is not None):
        out = d(ms, mf)
        head = {"text_embed": te, "null_embed": ne, "labels": LABELS}
        for s in [out] + out["aux_outputs"]:
            s.update(head)
            s["pred_logits"] = category.cal_pred_logits(s, use_fused=fused)
        losses = crit(out, targets)
    sum(losses.values()).backward()


def timed(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "Memcpy" not in e.name and "Memset" not in e.name)


def syncs(fn):
    fn()
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="4,8")
    ap.add_argument("--dtypes", default="fp32,fp16,bf16")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--stack-iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("category_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print(f"device: {smi}")
    rows = []
    for B in (int(b) for b in args.batches.split(",")):
        st = stack(B, dev)
        for name in args.dtypes.split(","):
            dt = DTYPES[name]
            inp = scoring_inputs(B, dt, dev)
            res = {True: {"alone": [], "stack": []}, False: {"alone": [], "stack": []}}
            for fused in (True, False):                       # warm-up
                for _ in range(3):
                    scoring_step(inp, dt, fused)
                stack_step(st, dt, fused)
            torch.cuda.synchronize()
            for _ in range(args.iters):                       # alternated
                for fused in (True, False):
                    res[fused]["alone"] += timed(lambda: scoring_step(inp, dt, fused), 1)
            for _ in range(args.stack_iters):
                for fused in (True, False):
                    res[fused]["stack"] += timed(lambda: stack_step(st, dt, fused), 1)
            for fused in (True, False):
                r = dict(B=B, dtype=name, arm="fused" if fused else "composed", device=smi,
                         scoring_fwd_bwd_ms=statistics.median(res[fused]["alone"]),
                         step_ms=statistics.median(res[fused]["stack"]),
                         host_enqueue_fwd_ms=enqueue_ms(inp, dt, fused, 20),
                         kernels_10_calls=kernels(lambda: scoring_step(inp, dt, fused)),
                         syncs_per_step=syncs(lambda: stack_step(st, dt, fused)))
                rows.append(r)
                print(json.dumps(r), flush=True)
            del inp
        del st
        torch.cuda.empty_cache()
    print(f"\nmeasured on {smi}\n")
    print("| B | dtype | arm | 10-set fwd+bwd ms | step ms | host enqueue, 10 fwd, ms | kernels / 10 calls | syncs / step |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['B']} | {r['dtype']} | {r['arm']} | {r['scoring_fwd_bwd_ms']:.2f} | {r['step_ms']:.1f} | "
              f"{r['host_enqueue_fwd_ms']:.2f} | {r['kernels_10_calls']} | {r['syncs_per_step']} |")
    if args.out:
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
