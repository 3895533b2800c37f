"""Microbenchmark of MSDeformAttn with 16-bit activations (odise_b200.msda.MSDeformAttn under torch.autocast), forward +
backward, arms alternated in one run:

  f32            the float32 module as before (fused float32 kernels)
  fused_bf16     under torch.autocast("cuda", torch.bfloat16): odise_msda_fused_bf16 and its backward
  fused_f16      under torch.autocast("cuda", torch.float16): odise_msda_fused_f16 and its backward
  composed_bf16  use_fused = False under bfloat16 autocast: value, locations and weights upcast to float32, then
                 MSDeformAttnFunction (what the module does without the 16-bit kernels)
  composed_f16   the same under float16 autocast

Shapes as tools/msda_module_bench.py: the ODISE 1024^2 pixel decoder (N = 4, S = Lq = 21504, d_model 256, 8 heads, L = 3,
4 points) and C4 (L = 4, S = Lq = 21760).  Per shape and arm: median ms over --iters iterations (CUDA events, --warmup
first) of the whole layer (four Linears included; query and input require grad) and of the layer without the four
Linears (value, offsets and logits given in the arm's dtype: the sampling op, its front and their backward), and
torch.cuda.max_memory_allocated above the inputs for the forward + backward of a 6-layer stack.  Before timing, the fused
and composed arms of each dtype are compared at the timed size (output and every gradient, max |diff| / max(1, max |ref|)).
The device name and power limit are read in the same run.  Prints one JSON line.

    python tools/msda_16bit_bench.py [--iters 100] [--warmup 10]
"""
import argparse
import contextlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from odise_b200 import msda  # noqa: E402
from oracle.msda_module import grid_reference_points, module_problem  # noqa: E402
from msda_backward_bench import gpu_info  # noqa: E402

SHAPES = {
    "odise_1024": [(128, 128), (64, 64), (32, 32)],
    "c4": [(128, 128), (64, 64), (32, 32), (16, 16)],
}
N, C, HEADS, POINTS = 4, 256, 8, 4
ARMS = {  # name -> (autocast dtype or None, use_fused)
    "f32": (None, True),
    "fused_bf16": (torch.bfloat16, True),
    "fused_f16": (torch.float16, True),
    "composed_bf16": (torch.bfloat16, False),
    "composed_f16": (torch.float16, False),
}


@contextlib.contextmanager
def arm_context(arm, modules):
    dtype, fused = ARMS[arm]
    for m in modules:
        m.use_fused = fused
    with (torch.autocast("cuda", dtype=dtype) if dtype is not None else contextlib.nullcontext()):
        yield


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
        params = module_problem(seed=1, N=1, d_model=C, n_heads=HEADS, shapes=shapes, n_points=POINTS,
                                dtype=torch.float32)["params"]
        ss = torch.as_tensor(shapes, dtype=torch.long, device=dev)
        lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
        ref = grid_reference_points(shapes, N, torch.float32).to(dev)
        layers = []
        for _ in range(6):
            m = msda.MSDeformAttn(C, L, HEADS, POINTS).to(dev)
            m.load_state_dict(params)
            layers.append(m)
        m = layers[0]
        q = torch.randn(N, S, C, device=dev, generator=g).requires_grad_(True)
        x = torch.randn(N, S, C, device=dev, generator=g).requires_grad_(True)
        go = torch.randn(N, S, C, device=dev, generator=g)
        with torch.no_grad():
            value = m.value_proj(x).view(N, S, HEADS, C // HEADS)
            offs = m.sampling_offsets(q).view(N, S, HEADS, L, POINTS, 2)
            logits = m.attention_weights(q).view(N, S, HEADS, L * POINTS)
        core_in = {}
        for dt in (torch.float32, torch.bfloat16, torch.float16):
            core_in[dt] = [t.to(dt).requires_grad_(True) for t in (value, offs, logits)]
        go_core = torch.randn(N, S, C, device=dev, generator=g)

        def layer():
            out = m(q, ref, x, ss, lsi)
            out.backward(go.to(out.dtype))

        def core(arm):
            dt, fused = ARMS[arm]
            v, o, lg = core_in[dt or torch.float32]
            if fused:
                out = msda.MSDeformAttnFusedFunction.apply(v, ss, lsi, ref, o, lg)
            else:                          # MSDeformAttn.forward's composed branch for a 16-bit value
                vf, of, lf = v.float(), o.float(), lg.float()
                aw = torch.softmax(lf, -1).view(N, S, HEADS, L, POINTS)
                wh = torch.stack([ss[..., 1], ss[..., 0]], -1)
                loc = ref[:, :, None, :, None, :] + of / wh[None, None, None, :, None, :]
                out = msda.MSDeformAttnFunction.apply(vf, ss, lsi, loc, aw, m.im2col_step).to(v.dtype)
            out.backward(go_core.to(out.dtype))

        # parity of the fused and composed arms of each dtype at the timed size
        parity = {}
        for dt, pair in (("bf16", ("fused_bf16", "composed_bf16")), ("f16", ("fused_f16", "composed_f16"))):
            got = {}
            for arm in pair:
                with arm_context(arm, layers):
                    for t in [q, x] + list(m.parameters()):
                        t.grad = None
                    out = m(q, ref, x, ss, lsi)
                    out.backward(go.to(out.dtype))
                    got[arm] = [out.detach()] + [t.grad.clone() for t in [q, x] + list(m.parameters())]
            parity[dt] = max(((u.double() - w.double()).abs().max() / w.double().abs().max().clamp_min(1.0)).item()
                             for u, w in zip(got[pair[0]], got[pair[1]]))
            del got

        times = {arm: {"layer": [], "core": []} for arm in ARMS}
        for it in range(a.warmup + a.iters):
            for arm in ARMS:
                with arm_context(arm, layers):
                    for kind, fn in (("layer", layer), ("core", lambda: core(arm))):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        fn()
                        e1.record()
                        e1.synchronize()
                        if it >= a.warmup:
                            times[arm][kind].append(e0.elapsed_time(e1))
        for t in [q, x] + [t for ts in core_in.values() for t in ts] + [p for l_ in layers for p in l_.parameters()]:
            t.grad = None

        mem = {}
        for arm in ARMS:
            with arm_context(arm, layers):
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                h = x
                for l_ in layers:
                    h = h + l_(h, ref, h, ss, lsi)
                h.backward(go)
                torch.cuda.synchronize()
                mem[arm] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
                del h
                for t in [q, x] + [p for l_ in layers for p in l_.parameters()]:
                    t.grad = None
        out = dict(N=N, S=S, Lq=S, L=L, d_model=C, heads=HEADS, points=POINTS, parity_fused_vs_composed=parity, arms={})
        for arm in ARMS:
            out["arms"][arm] = dict(layer_fwd_bwd_ms=round(median(times[arm]["layer"]), 4),
                                    no_linears_fwd_bwd_ms=round(median(times[arm]["core"]), 4),
                                    stack6_fwd_bwd_peak_MiB=mem[arm])
        res["shapes"][key] = out
        del layers, m, q, x, go, value, offs, logits, core_in, go_core
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
