"""Microbenchmark of the MSDeformAttn module drop-in (odise_b200.msda.MSDeformAttn), forward + backward, three arms
alternated in one run:

  fused      the module as shipped: MSDeformAttnFusedFunction (softmax and locations inside odise_msda_fused_f32 and
             odise_msda_fused_backward_f32)
  composed   the same module with use_fused = False: softmax and locations in torch ops, then MSDeformAttnFunction
             (odise_msda_forward_f32 / odise_msda_backward_f32)
  reference  the composed module on the reference's own CUDA kernels (oracle/_ref/libref_msda*.so), when present

Shapes: the ODISE 1024^2 pixel decoder (N = 4, S = Lq = 21504, d_model 256, 8 heads, L = 3 levels 128^2..32^2, 4 points)
and C4 (L = 4: levels 128^2..16^2, S = Lq = 21760).  Per shape and arm: median ms over --iters iterations (CUDA events,
--warmup first) of the whole layer (four Linears included; query and input require grad) and of the layer without the
four Linears (value, offsets and logits given, front + sampling and their backward), and torch.cuda.max_memory_allocated
above the inputs for the forward + backward of a 6-layer stack.  Before timing, the fused and composed arms' outputs and
gradients are compared at the timed size.  The device name and power limit are read in the same run.  Prints one JSON
line.

    python tools/msda_module_bench.py [--iters 100] [--warmup 10]
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
from oracle import refmsda, refmsda_backward  # noqa: E402
from oracle.msda_module import grid_reference_points, module_problem  # noqa: E402
from msda_backward_bench import gpu_info  # noqa: E402

SHAPES = {
    "odise_1024": [(128, 128), (64, 64), (32, 32)],
    "c4": [(128, 128), (64, 64), (32, 32), (16, 16)],
}
N, C, HEADS, POINTS = 4, 256, 8, 4


class RefFunction(torch.autograd.Function):
    """MSDeformAttnFunction on the reference's own forward and backward kernels"""

    @staticmethod
    def forward(ctx, value, ss, lsi, loc, aw, im2col_step):
        ctx.im2col_step = im2col_step
        ctx.save_for_backward(value, ss, lsi, loc, aw)
        return refmsda.forward(value, ss, lsi, loc, aw, im2col_step)

    @staticmethod
    def backward(ctx, go):
        value, ss, lsi, loc, aw = ctx.saved_tensors
        gv, gl, ga = refmsda_backward.backward(value, ss, lsi, loc, aw, go.contiguous(), ctx.im2col_step)
        return gv, None, None, gl, ga, None


@contextlib.contextmanager
def arm_context(arm, modules):
    """fused / composed: set use_fused; reference: composed path with MSDeformAttnFunction swapped for RefFunction"""
    for m in modules:
        m.use_fused = arm == "fused"
    saved = msda.MSDeformAttnFunction
    if arm == "reference":
        msda.MSDeformAttnFunction = RefFunction
    try:
        yield
    finally:
        msda.MSDeformAttnFunction = saved


def median(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    name, power, clock = gpu_info()
    arms = ["fused", "composed"] + (["reference"] if refmsda.available() and refmsda_backward.available() else [])
    res = dict(device=name, power_limit=power, max_sm_clock=clock, iters=a.iters, arms=arms, shapes={})
    g = torch.Generator(device=dev).manual_seed(0)
    for key, shapes in SHAPES.items():
        L = len(shapes)
        S = sum(h * w for h, w in shapes)
        # parameters with every sample off a cell edge, so that the arms' gradients can be compared
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
        core_in = [t.clone().requires_grad_(True) for t in (value, offs, logits)]
        go_core = torch.randn(N, S, C, device=dev, generator=g)

        def layer():
            out = m(q, ref, x, ss, lsi)
            out.backward(go)

        def core(arm):
            v, o, lg = core_in
            if arm == "fused":
                out = msda.MSDeformAttnFusedFunction.apply(v, ss, lsi, ref, o, lg)
            else:
                aw = torch.softmax(lg, -1).view(N, S, HEADS, L, POINTS)
                wh = torch.stack([ss[..., 1], ss[..., 0]], -1)
                loc = ref[:, :, None, :, None, :] + o / wh[None, None, None, :, None, :]
                out = msda.MSDeformAttnFunction.apply(v, ss, lsi, loc, aw, m.im2col_step)
            out.backward(go_core)

        # parity of the fused and composed arms at the timed size
        got = {}
        for arm in ("fused", "composed"):
            with arm_context(arm, layers):
                for t in [q, x] + list(m.parameters()):
                    t.grad = None
                out = m(q, ref, x, ss, lsi)
                out.backward(go)
                got[arm] = [out.detach()] + [t.grad.clone() for t in [q, x] + list(m.parameters())]
        parity = max(((u - w).abs().max() / w.abs().max().clamp_min(1.0)).item()
                     for u, w in zip(got["fused"], got["composed"]))
        del got

        times = {arm: {"layer": [], "core": []} for arm in arms}
        for it in range(a.warmup + a.iters):
            for arm in arms:
                with arm_context(arm, layers):
                    for kind, fn in (("layer", layer), ("core", lambda: core(arm))):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        fn()
                        e1.record()
                        e1.synchronize()
                        if it >= a.warmup:
                            times[arm][kind].append(e0.elapsed_time(e1))
        for t in [q, x] + core_in + [p for l_ in layers for p in l_.parameters()]:
            t.grad = None

        mem = {}
        for arm in arms:
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
        for arm in arms:
            out["arms"][arm] = dict(layer_fwd_bwd_ms=round(median(times[arm]["layer"]), 4),
                                    no_linears_fwd_bwd_ms=round(median(times[arm]["core"]), 4),
                                    stack6_fwd_bwd_peak_MiB=mem[arm])
        res["shapes"][key] = out
        del layers, m, q, x, go, value, offs, logits, core_in, go_core
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
