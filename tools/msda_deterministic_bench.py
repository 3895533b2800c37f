"""Microbenchmark of the deterministic MSDeformAttn backward (fixed-point grad_value) against the default one (float
atomics), arms alternated in one run:

  op          lib.msda_backward (odise_msda_backward_f32 vs odise_msda_backward_det_f32): the native op's backward
  fused_f32   lib.msda_fused_backward (odise_msda_fused_backward_f32 vs _det_f32)
  fused_bf16  lib.msda_fused_backward_16bit on bfloat16 storage (odise_msda_fused_backward_bf16 vs _det_bf16)
  layer_f32   a whole float32 MSDeformAttn layer, forward + backward, torch.use_deterministic_algorithms off vs on
  layer_bf16  the same under torch.autocast("cuda", torch.bfloat16)

Shapes as tools/msda_16bit_bench.py: the ODISE 1024^2 pixel decoder (N = 4, S = Lq = 21504, d_model 256, 8 heads, L = 3,
4 points) and C4 (L = 4, S = Lq = 21760).  Per shape, arm and mode: median ms over --iters iterations (CUDA events,
--warmup first), default and deterministic alternated call by call; for the three backward arms the peak memory a
call allocates (torch.cuda.max_memory_allocated above what was allocated before it: the outputs, plus the workspace in
deterministic mode).  Before timing, each backward arm's deterministic grad_value is compared with the default one
(max |diff| / max |default|) and its other gradients checked bit-equal.  CUBLAS_WORKSPACE_CONFIG=:4096:8 is set for the
whole run (deterministic mode needs it for the Linears), so both layer modes run the same cuBLAS configuration.  The
device name and power limit are read in the same run.  Prints one JSON line.

    python tools/msda_deterministic_bench.py [--iters 100] [--warmup 10]
"""
import argparse
import contextlib
import json
import os
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")      # before CUDA starts

import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from odise_b200 import lib, msda  # noqa: E402
from oracle.msda_module import grid_reference_points, module_problem  # noqa: E402
from msda_backward_bench import gpu_info  # noqa: E402

SHAPES = {
    "odise_1024": [(128, 128), (64, 64), (32, 32)],
    "c4": [(128, 128), (64, 64), (32, 32), (16, 16)],
}
N, C, HEADS, POINTS = 4, 256, 8, 4
ARMS = ("op", "fused_f32", "fused_bf16", "layer_f32", "layer_bf16")
MODES = ("default", "deterministic")


@contextlib.contextmanager
def det_mode(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def median(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    name, power, clock = gpu_info()
    res = dict(device=name, power_limit=power, max_sm_clock=clock, iters=a.iters, arms=list(ARMS), shapes={})
    g = torch.Generator(device=dev).manual_seed(0)
    for key, shapes in SHAPES.items():
        L = len(shapes)
        S = sum(h * w for h, w in shapes)
        D = C // HEADS
        params = module_problem(seed=1, N=1, d_model=C, n_heads=HEADS, shapes=shapes, n_points=POINTS,
                                dtype=torch.float32)["params"]
        ss = torch.as_tensor(shapes, dtype=torch.long, device=dev)
        lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
        ref = grid_reference_points(shapes, N, torch.float32).to(dev)
        m = msda.MSDeformAttn(C, L, HEADS, POINTS).to(dev)
        m.load_state_dict(params)
        q = torch.randn(N, S, C, device=dev, generator=g).requires_grad_(True)
        x = torch.randn(N, S, C, device=dev, generator=g).requires_grad_(True)
        go = torch.randn(N, S, C, device=dev, generator=g)
        with torch.no_grad():
            value = m.value_proj(x).view(N, S, HEADS, D)
            offs = m.sampling_offsets(q).view(N, S, HEADS, L, POINTS, 2)
            logits = m.attention_weights(q).view(N, S, HEADS, L * POINTS)
            aw = torch.softmax(logits, -1).view(N, S, HEADS, L, POINTS).contiguous()
            wh = torch.stack([ss[..., 1], ss[..., 0]], -1)
            loc = (ref[:, :, None, :, None, :] + offs / wh[None, None, None, :, None, :]).contiguous()
        bf = [t.bfloat16() for t in (value, offs, logits, go)]
        bwd = {
            "op": lambda det: lib.msda_backward(value, ss, lsi, loc, aw, go, 64, deterministic=det),
            "fused_f32": lambda det: lib.msda_fused_backward(value, ss, lsi, ref, offs, logits, go, deterministic=det),
            "fused_bf16": lambda det: lib.msda_fused_backward_16bit(bf[0], ss, lsi, ref, bf[1], bf[2], bf[3],
                                                                    deterministic=det),
        }

        def layer(amp):
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                out = m(q, ref, x, ss, lsi)
            out.backward(go.to(out.dtype))

        run = {arm: fn for arm, fn in bwd.items()}
        run["layer_f32"] = lambda det: layer(False)
        run["layer_bf16"] = lambda det: layer(True)

        # deterministic against default: grad_value close, the other gradients bit-equal
        parity, mem = {}, {}
        for arm, fn in bwd.items():
            d0, d1 = fn(False), fn(True)
            torch.cuda.synchronize()
            parity[arm] = dict(
                grad_value_rel_diff=((d1[0].double() - d0[0].double()).abs().max() / d0[0].double().abs().max()).item(),
                other_grads_bit_equal=bool(torch.equal(d0[1], d1[1]) and torch.equal(d0[2], d1[2])))
            del d0, d1
            mem[arm] = {}
            for mode in MODES:
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                r = fn(mode == "deterministic")
                torch.cuda.synchronize()
                mem[arm][mode] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
                del r

        times = {arm: {mode: [] for mode in MODES} for arm in ARMS}
        for it in range(a.warmup + a.iters):
            for arm in ARMS:
                for mode in MODES:
                    det = mode == "deterministic"
                    with det_mode(det):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        r = run[arm](det)
                        e1.record()
                        e1.synchronize()
                        del r
                    if it >= a.warmup:
                        times[arm][mode].append(e0.elapsed_time(e1))
            for t in [q, x] + list(m.parameters()):
                t.grad = None
        out = dict(N=N, S=S, Lq=S, L=L, d_model=C, heads=HEADS, points=POINTS,
                   workspace_MiB=round(lib.load().odise_msda_det_workspace_bytes(N, S, HEADS, D) / 2 ** 20, 1),
                   parity=parity, arms={})
        for arm in ARMS:
            t0, t1 = median(times[arm]["default"]), median(times[arm]["deterministic"])
            out["arms"][arm] = dict(default_ms=round(t0, 4), deterministic_ms=round(t1, 4), ratio=round(t1 / t0, 3))
            if arm in mem:
                out["arms"][arm].update(default_peak_MiB=mem[arm]["default"],
                                        deterministic_peak_MiB=mem[arm]["deterministic"])
        res["shapes"][key] = out
        del m, q, x, go, value, offs, logits, aw, loc, bf, bwd, run
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
