"""Grounding loss, fused against composed, on one GPU: forward + backward of all 10 prediction sets at Q = 100, K = 8,
C = 256, for B in {4, 8}, float32 and fp16 / bf16 autocast.  Per arm: the CUDA-event median of the two paths run
alternately in one process, the host enqueue time of the fused forward, kernels per step (torch.profiler, a separate
run) and host synchronisations per step (torch.cuda.set_sync_debug_mode("warn") counts).  Then the fused kernels at an
emulated W = 8 (G = 64, B = 8, the gathered tensors passed in, no collectives) against the composed ops on the same
tensors.  Prints the card's name and power limit read in the same run, then one line per arm.

    python tools/grounding_bench.py [--reps 30]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from odise_b200 import grounding  # noqa: E402

S, Q, K, C = 10, 100, 8, 256


def _inputs(G, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    m = torch.randn(S, G, Q, C, generator=g).cuda().to(dtype).requires_grad_()
    w = torch.randn(G, K, C, generator=g).cuda().to(dtype).requires_grad_()
    v = (torch.rand(G, K, generator=g) < 0.7).cuda()
    v[:, 0] = True
    sc = (10 + 5 * torch.rand(S, generator=g)).cuda().requires_grad_()
    return m, w, v, sc


def _step(x, B, o, fused, autocast):
    m, w, v, sc = x
    G = m.shape[1]
    with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
        ml, wl = (m, w) if G == B else (m[:, o:o + B], w[o:o + B])
        losses = grounding.grounding_losses(ml, m, wl, w, v, sc, o, 1.0, use_fused=fused)
    torch.autograd.grad(losses.sum(), [m, w, sc])


def _time(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def _kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset")))


def _syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(c.message) for c in caught)


def _arm(label, G, B, o, dtype, autocast, reps):
    x = _inputs(G, dtype)
    fused = lambda: _step(x, B, o, True, autocast)        # noqa: E731
    comp = lambda: _step(x, B, o, False, autocast)        # noqa: E731
    for _ in range(3):
        fused()
        comp()
    tf, tc = [], []
    for _ in range(reps):
        tf.append(_time(fused))
        tc.append(_time(comp))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
        ml, wl = (x[0], x[1]) if G == B else (x[0][:, o:o + B], x[1][o:o + B])
        grounding.grounding_losses(ml, x[0], wl, x[1], x[2], x[3], o, 1.0)
    enqueue = (time.perf_counter() - t0) * 1e3
    torch.cuda.synchronize()
    print(f"{label}: fwd+bwd 10 sets median fused {statistics.median(tf):.3f} ms, composed "
          f"{statistics.median(tc):.3f} ms; fused forward enqueue {enqueue:.3f} ms; kernels fused {_kernels(fused)}, "
          f"composed {_kernels(comp)}; syncs fused {_syncs(fused)}, composed {_syncs(comp)}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/grounding_bench.py measures on a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"GPU: {smi}", flush=True)
    for B in (4, 8):
        for name, dtype, ac in (("fp32", torch.float32, None), ("fp16 autocast", torch.float16, torch.float16),
                                ("bf16 autocast", torch.bfloat16, torch.bfloat16)):
            _arm(f"W=1 B={B} {name}", B, B, 0, dtype, ac, a.reps)
    for name, dtype, ac in (("fp32", torch.float32, None), ("bf16 autocast", torch.bfloat16, torch.bfloat16)):
        _arm(f"emulated W=8 G=64 B=8 offset 24 {name}", 64, 8, 24, dtype, ac, max(5, a.reps // 3))


if __name__ == "__main__":
    main()
