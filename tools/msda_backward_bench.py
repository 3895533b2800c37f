"""Microbenchmark of the MSDeformAttn backward: odise_msda_backward_f32 against the reference's own CUDA backward
(oracle/_ref/libref_msda_backward.so), with the forwards, timed with CUDA events, arms alternated in one run.

Shapes: the ODISE 1024^2 pixel decoder (N = 4, S = Lq = 21504, M = 8, D = 32, L = 3 levels 128^2..32^2, P = 4) and C4
(the op's default L = 4: levels 128^2..16^2, S = Lq = 21760).  Prints one JSON line: device name and power limit
(read-only nvidia-smi query in the same run), per shape and arm the median ms of backward alone and of forward +
backward, the compulsory HBM bytes of the backward and the GB/s they imply, and the number of global reductions the
backward issues into grad_value (ours: one float4 per in-range corner and 4-channel group; the reference: one scalar
per in-range corner and channel; counted with all four corners in range, so an upper bound).  Before timing, the two arms' gradients are compared at the timed size with the bar
of tests/test_gpu_msda_backward.py::test_backward_vs_reference_kernel (1e-5 x max(1, max |ref|)).

    python tools/msda_backward_bench.py [--iters 100] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from odise_b200 import lib  # noqa: E402
from oracle import refmsda, refmsda_backward  # noqa: E402
from oracle.msda_grad import grad_problem  # noqa: E402

SHAPES = {
    "odise_1024": dict(seed=1, N=4, M=8, D=32, shapes=[(128, 128), (64, 64), (32, 32)], P=4),
    "c4": dict(seed=2, N=4, M=8, D=32, shapes=[(128, 128), (64, 64), (32, 32), (16, 16)], P=4),
}


def gpu_info():
    """(name, power limit, max SM clock) of GPU 0, read-only."""
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if r.returncode != 0 or not r.stdout.strip():
        return torch.cuda.get_device_name(0), "unknown", "unknown"
    name, power, clock = (f.strip() for f in r.stdout.strip().splitlines()[0].split(","))
    return name, power, clock


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    name, power, clock = gpu_info()
    res = dict(device=name, power_limit=power, max_sm_clock=clock, iters=a.iters, shapes={})
    for key, cfg in SHAPES.items():
        S = sum(h * w for h, w in cfg["shapes"])
        N, M, D, L, P = cfg["N"], cfg["M"], cfg["D"], len(cfg["shapes"]), cfg["P"]
        prob = grad_problem(Lq=S, **cfg)
        value, ss, lsi, loc, aw, go = (t.to(dev, torch.float32) if t.is_floating_point() else t.to(dev) for t in prob)
        ref_out = (torch.empty_like(value), torch.empty_like(loc), torch.empty_like(aw))
        fwd_out = torch.empty(N, S, M * D, device=dev)

        def ours_bwd():
            return lib.msda_backward(value, ss, lsi, loc, aw, go, 64)

        def ref_bwd():
            return refmsda_backward.backward(value, ss, lsi, loc, aw, go, 64, out=ref_out)

        arms = {
            "ours": (ours_bwd, lambda: lib.msda_forward(value, ss, lsi, loc, aw, 64)),
            "reference": (ref_bwd, lambda: refmsda.forward(value, ss, lsi, loc, aw, 64, out=fwd_out)),
        }
        # parity at the timed size
        g_ours, g_ref = ours_bwd(), [t.clone() for t in ref_bwd()]
        torch.cuda.synchronize()
        parity = {}
        for nm, x, y in zip(("grad_value", "grad_loc", "grad_attn"), g_ours, g_ref):
            scale = max(1.0, y.abs().max().item())
            parity[nm] = (x - y).abs().max().item() / scale
        parity_ok = all(v < 1e-5 for v in parity.values())
        del g_ours, g_ref

        times = {k: {"bwd": [], "fwd_bwd": []} for k in arms}
        for it in range(a.warmup + a.iters):
            for k, (bwd, fwd) in arms.items():
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                fwd()
                e1.record()
                bwd()
                e2.record()
                e2.synchronize()
                if it >= a.warmup:
                    times[k]["bwd"].append(e1.elapsed_time(e2))
                    times[k]["fwd_bwd"].append(e0.elapsed_time(e2))

        # compulsory HBM traffic of one backward: value, grad_out, loc, attn read; the three grads written; zero fill
        f = 4
        rd = N * (S * M * D + S * M * D + S * M * L * P * 2 + S * M * L * P) * f
        wr = N * (S * M * D + S * M * L * P * 2 + S * M * L * P) * f + N * S * M * D * f
        samples = N * S * M * L * P
        out = dict(N=N, Lq=S, S=S, M=M, D=D, L=L, P=P, hbm_bytes_bwd=rd + wr, parity_rel_err=parity,
                   parity_ok=parity_ok, arms={})
        for k in arms:
            bwd = sorted(times[k]["bwd"])[len(times[k]["bwd"]) // 2]
            fb = sorted(times[k]["fwd_bwd"])[len(times[k]["fwd_bwd"]) // 2]
            red = samples * 4 * (D // 4) if k == "ours" else samples * 4 * D
            out["arms"][k] = dict(bwd_ms=round(bwd, 4), fwd_bwd_ms=round(fb, 4),
                                  bwd_hbm_GBps=round((rd + wr) / bwd / 1e6, 1),
                                  reductions=red, reduction_kind="float4" if k == "ours" else "scalar",
                                  reductions_per_us=round(red / bwd / 1e3, 1))
        out["speedup_bwd"] = round(out["arms"]["reference"]["bwd_ms"] / out["arms"]["ours"]["bwd_ms"], 3)
        out["speedup_fwd_bwd"] = round(out["arms"]["reference"]["fwd_bwd_ms"] / out["arms"]["ours"]["fwd_bwd_ms"], 3)
        res["shapes"][key] = out
        del value, loc, aw, go, ref_out, fwd_out
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
