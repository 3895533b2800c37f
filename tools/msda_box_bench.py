"""Microbenchmark of MSDeformAttn with box reference points (cx, cy, w, h): the cross-attention of a DETR-style decoder
layer, forward + backward, fused (odise_msda_fused_box_*) against composed (use_fused = False), arms alternated:

  fused_f32 / composed_f32      float32 module
  fused_bf16 / composed_bf16    under torch.autocast("cuda", torch.bfloat16)
  fused_f16 / composed_f16      under torch.autocast("cuda", torch.float16)

Shape: an 800 x 1333 input, 4 levels (100, 167), (50, 84), (25, 42), (13, 21) (S = 22223), N = 2, d_model 256, 8 heads,
4 points, Lq = 300 and 900 queries.  The boxes are detached (decoders with box refinement detach them between layers);
memory and queries require grad.  Per (Lq, arm) and run: median ms over --iters iterations (CUDA events, --warmup first)
of the whole layer and of the layer without its four Linears (value, offsets and logits given in the arm's dtype), and
torch.cuda.max_memory_allocated above the inputs for the forward + backward of a 6-layer stack (queries pass from layer to
layer, the memory is shared).  Before timing, the fused and composed arms of each dtype are compared at the timed size
(output and every gradient, max |diff| / max(1, max |ref|)).  The device name and power limit are read in the same run.
Prints one JSON line.

    python tools/msda_box_bench.py [--iters 50] [--warmup 10] [--runs 2]
"""
import argparse
import contextlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from odise_b200 import msda  # noqa: E402
from oracle.msda_module import module_problem  # noqa: E402
from msda_backward_bench import gpu_info  # noqa: E402

SHAPES = [(100, 167), (50, 84), (25, 42), (13, 21)]
N, C, HEADS, POINTS = 2, 256, 8, 4
QUERIES = (300, 900)
ARMS = {  # name -> (autocast dtype or None, use_fused)
    "fused_f32": (None, True),
    "composed_f32": (None, False),
    "fused_bf16": (torch.bfloat16, True),
    "composed_bf16": (torch.bfloat16, False),
    "fused_f16": (torch.float16, True),
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
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    name, power, clock = gpu_info()
    res = dict(device=name, power_limit=power, max_sm_clock=clock, iters=a.iters, runs=a.runs, arms=list(ARMS),
               queries={})
    g = torch.Generator(device=dev).manual_seed(0)
    L = len(SHAPES)
    S = sum(h * w for h, w in SHAPES)
    params = module_problem(seed=1, N=1, d_model=C, n_heads=HEADS, shapes=[(2, 2)] * L, n_points=POINTS,
                            dtype=torch.float32)["params"]
    ss = torch.as_tensor(SHAPES, dtype=torch.long, device=dev)
    lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
    for Lq in QUERIES:
        layers = []
        for _ in range(6):
            m = msda.MSDeformAttn(C, L, HEADS, POINTS).to(dev)
            m.load_state_dict(params)
            layers.append(m)
        m = layers[0]
        centre = torch.rand(N, Lq, 1, 2, device=dev, generator=g) * 0.8 + 0.1
        wh = torch.rand(N, Lq, 1, 2, device=dev, generator=g) * 0.45 + 0.05
        ref = torch.cat([centre, wh], -1).expand(N, Lq, L, 4).contiguous()
        q = torch.randn(N, Lq, C, device=dev, generator=g).requires_grad_(True)
        x = torch.randn(N, S, C, device=dev, generator=g).requires_grad_(True)
        go = torch.randn(N, Lq, C, device=dev, generator=g)
        with torch.no_grad():
            value = m.value_proj(x).view(N, S, HEADS, C // HEADS)
            offs = m.sampling_offsets(q).view(N, Lq, HEADS, L, POINTS, 2)
            logits = m.attention_weights(q).view(N, Lq, HEADS, L * POINTS)
        core_in = {dt: [t.to(dt).requires_grad_(True) for t in (value, offs, logits)]
                   for dt in (torch.float32, torch.bfloat16, torch.float16)}
        leaves = [q, x] + list(m.parameters())

        def layer():
            out = m(q, ref, x, ss, lsi)
            out.backward(go.to(out.dtype))

        def core(arm):
            dt, fused = ARMS[arm]
            v, o, lg = core_in[dt or torch.float32]
            if fused:
                out = msda.MSDeformAttnFusedFunction.apply(v, ss, lsi, ref, o, lg)
            else:                          # MSDeformAttn.forward's composed branch for boxes
                vf, of, lf = v.float(), o.float(), lg.float()
                aw = torch.softmax(lf, -1).view(N, Lq, HEADS, L, POINTS)
                loc = ref[:, :, None, :, None, :2] + of / POINTS * ref[:, :, None, :, None, 2:] * 0.5
                out = msda.MSDeformAttnFunction.apply(vf, ss, lsi, loc, aw, m.im2col_step).to(v.dtype)
            out.backward(go.to(out.dtype))

        parity = {}
        for dt in ("f32", "bf16", "f16"):
            got = {}
            for arm in (f"fused_{dt}", f"composed_{dt}"):
                with arm_context(arm, layers):
                    for t in leaves:
                        t.grad = None
                    out = m(q, ref, x, ss, lsi)
                    out.backward(go.to(out.dtype))
                    got[arm] = [out.detach()] + [t.grad.clone() for t in leaves]
            parity[dt] = max(((u.double() - w.double()).abs().max() / w.double().abs().max().clamp_min(1.0)).item()
                             for u, w in zip(got[f"fused_{dt}"], got[f"composed_{dt}"]))
            del got

        runs = []
        for _ in range(a.runs):
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
            runs.append({arm: dict(layer_fwd_bwd_ms=round(median(times[arm]["layer"]), 4),
                                   no_linears_fwd_bwd_ms=round(median(times[arm]["core"]), 4)) for arm in ARMS})
        for t in leaves + [t for ts in core_in.values() for t in ts] + [p for l_ in layers for p in l_.parameters()]:
            t.grad = None

        mem = {}
        for arm in ARMS:
            with arm_context(arm, layers):
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                h = q
                for l_ in layers:
                    h = h + l_(h, ref, x, ss, lsi)
                h.backward(go.to(h.dtype))
                torch.cuda.synchronize()
                mem[arm] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
                del h
                for t in leaves + [p for l_ in layers for p in l_.parameters()]:
                    t.grad = None
        res["queries"][str(Lq)] = dict(N=N, S=S, Lq=Lq, L=L, d_model=C, heads=HEADS, points=POINTS,
                                       parity_fused_vs_composed=parity, runs=runs, stack6_fwd_bwd_peak_MiB=mem)
        del layers, m, q, x, go, value, offs, logits, core_in, leaves
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
