"""Forward + backward of ODISE's 9-layer transformer decoder (odise_b200.decoder) at the training geometry: 1024^2
crops, mask_features [B, 256, 256, 256], levels 32^2 / 64^2 / 128^2, Q = 100.  Alternates the fused prediction heads
(odise_mask_head_* kernels) with the composed reference ops (use_fused = False) in float32 and under fp16 / bf16 autocast,
and prints per arm the median ms, the peak max_memory_allocated above the inputs and the number of synchronising CUDA
calls of one step, with the device name and power limit read in the same run.

    python tools/mask_head_bench.py [--batches 4 8] [--iters 10] [--rounds 3] [--size 256] [--queries 100] [--out f]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from odise_b200 import decoder as dec  # noqa: E402

ARMS = {"fp32": None, "fp16": torch.float16, "bf16": torch.bfloat16}


def build(Q, device):
    torch.manual_seed(0)
    return dec.ODISEMultiScaleMaskedTransformerDecoder(
        in_channels=256, num_classes=150, hidden_dim=256, num_queries=Q, nheads=8, dim_feedforward=2048, dec_layers=9,
        pre_norm=False, mask_dim=256, enforce_input_project=False,
        post_mask_embed=dec.PooledMaskEmbed(hidden_dim=256, mask_dim=256, projection_dim=768)).to(device)


def inputs(B, size, device):
    g = torch.Generator(device=device).manual_seed(1)
    # the pixel decoder's three levels (1/32, 1/16, 1/8 of the crop) and its 1/4 mask features
    x = [torch.randn(B, 256, size // 2 ** (3 - i), size // 2 ** (3 - i), device=device, generator=g) for i in range(3)]
    mf = torch.randn(B, 256, size, size, device=device, generator=g, requires_grad=True)
    return x, mf


def step(m, x, mf, dtype):
    if dtype is None:
        out = m(x, mf)
    else:
        with torch.autocast("cuda", dtype=dtype):
            out = m(x, mf)
    loss = out["pred_masks"].float().mean() + out["mask_embed"].float().pow(2).mean()
    for a in out["aux_outputs"]:
        loss = loss + a["pred_masks"].float().mean() + a["mask_embed"].float().pow(2).mean()
    loss.backward()


def syncs(m, x, mf, dtype):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step(m, x, mf, dtype)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(x.message) for x in w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 8])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--size", type=int, default=256, help="mask-feature side (crop / 4)")
    ap.add_argument("--queries", type=int, default=100)
    ap.add_argument("--arms", nargs="+", default=list(ARMS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mask_head_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi: {smi}")
    m = build(a.queries, dev)
    results = []
    for B in a.batches:
        x, mf = inputs(B, a.size, dev)
        for arm in a.arms:
            dtype = ARMS[arm]
            times = {True: [], False: []}
            peak, nsync = {}, {}
            for fused in (True, False):           # warm-up, memory and sync count of each path
                m.use_fused = fused
                m.zero_grad(set_to_none=True)
                mf.grad = None
                step(m, x, mf, dtype)
                m.zero_grad(set_to_none=True)
                mf.grad = None
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated(dev)
                torch.cuda.reset_peak_memory_stats(dev)
                step(m, x, mf, dtype)
                torch.cuda.synchronize()
                peak[fused] = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20
                nsync[fused] = syncs(m, x, mf, dtype)
            for _ in range(a.rounds):              # alternate the two paths
                for fused in (True, False):
                    m.use_fused = fused
                    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                    for i in range(a.iters):
                        m.zero_grad(set_to_none=True)
                        mf.grad = None
                        ev[0].record()
                        step(m, x, mf, dtype)
                        ev[1].record()
                        torch.cuda.synchronize()
                        times[fused].append(ev[0].elapsed_time(ev[1]))
            for fused in (True, False):
                r = dict(B=B, arm=arm, path="fused" if fused else "composed",
                         median_ms=round(statistics.median(times[fused]), 2), peak_mib=round(peak[fused]),
                         syncs=nsync[fused])
                results.append(r)
                print(json.dumps(r), flush=True)
        del x, mf
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(device=torch.cuda.get_device_name(dev), nvidia_smi=smi, results=results), f, indent=1)


if __name__ == "__main__":
    main()
