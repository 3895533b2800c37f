"""Microbenchmark of the MSDeformAttn drop-in under torch.compile: a 6-layer encoder stack, forward + backward, arms
alternated in one run:

  eager            the stack as written
  inductor         torch.compile(stack) (default mode, Inductor)
  reduce_overhead  torch.compile(stack, mode="reduce-overhead") (Inductor and CUDA graphs)

each in float32 and under torch.autocast("cuda", torch.bfloat16).  The stack is the deformable encoder's layer:
x <- LayerNorm(x + MSDeformAttn(x, ref, x)), x <- LayerNorm(x + FFN(x)) with FFN 256 -> 1024 -> ReLU -> 256.

Shapes: the ODISE 1024^2 pixel decoder (N = 4, S = Lq = 21504, d_model 256, 8 heads, L = 3 levels 128^2..32^2, 4 points)
and C4 (L = 4: levels 128^2..16^2, S = Lq = 21760).  Per shape and arm: median, 25th and 75th percentile ms over --iters
iterations (CUDA events, --warmup first) and the first call's wall time (the compile).  Then the eager cost of the custom
ops: one MSDeformAttn layer forward + backward through the module as shipped (custom ops) against the same layer on a
restated copy of the previous MSDeformAttnFusedFunction, which called lib directly ("direct"), alternated; and the host
time per call of the fused forward op against lib.msda_fused_forward on a tiny problem (launch-bound, so the difference
is the op's dispatch).  The device name and power limit are read in the same run.  Prints one JSON line.

    python tools/msda_compile_bench.py [--iters 100] [--warmup 10]
"""
import argparse
import json
import os
import sys
import time

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from odise_b200 import lib, msda  # noqa: E402
from oracle.msda_module import grid_reference_points, module_problem  # noqa: E402
from msda_backward_bench import gpu_info  # noqa: E402

SHAPES = {
    "odise_1024": [(128, 128), (64, 64), (32, 32)],
    "c4": [(128, 128), (64, 64), (32, 32), (16, 16)],
}
N, C, HEADS, POINTS, FFN, LAYERS = 4, 256, 8, 4, 1024, 6
ARMS = [(mode, amp) for amp in ("f32", "bf16") for mode in ("eager", "inductor", "reduce_overhead")]


class DirectFusedFunction(torch.autograd.Function):
    """MSDeformAttnFusedFunction as it was before the custom ops: lib called directly"""

    @staticmethod
    def forward(ctx, value, spatial_shapes, level_start_index, reference_points, offsets, logits):
        fwd = lib.msda_fused_forward_16bit if value.dtype in msda._LOW else lib.msda_fused_forward
        output = fwd(value, spatial_shapes, level_start_index, reference_points, offsets, logits)
        ctx.save_for_backward(value, spatial_shapes, level_start_index, reference_points, offsets, logits)
        return output

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_output):
        value, spatial_shapes, level_start_index, reference_points, offsets, logits = ctx.saved_tensors
        bwd = lib.msda_fused_backward_16bit if value.dtype in msda._LOW else lib.msda_fused_backward
        grad_value, grad_offsets, grad_logits = bwd(
            value, spatial_shapes, level_start_index, reference_points, offsets, logits,
            grad_output.to(value.dtype).contiguous(), deterministic=torch.are_deterministic_algorithms_enabled())
        grad_ref = None
        if ctx.needs_input_grad[3]:
            go = grad_offsets.float()
            wh = torch.stack([spatial_shapes[:, 1], spatial_shapes[:, 0]], -1).to(go)
            grad_ref = (go * wh[None, None, None, :, None, :]).sum((2, 4))
        return grad_value, None, None, grad_ref, grad_offsets, grad_logits


class EncoderLayer(nn.Module):
    def __init__(self, L):
        super().__init__()
        self.attn = msda.MSDeformAttn(C, L, HEADS, POINTS)
        self.norm1, self.norm2 = nn.LayerNorm(C), nn.LayerNorm(C)
        self.ffn = nn.Sequential(nn.Linear(C, FFN), nn.ReLU(), nn.Linear(FFN, C))

    def forward(self, x, ref, ss, lsi):
        x = self.norm1(x + self.attn(x, ref, x, ss, lsi))
        return self.norm2(x + self.ffn(x))


class Stack(nn.Module):
    def __init__(self, L):
        super().__init__()
        self.layers = nn.ModuleList(EncoderLayer(L) for _ in range(LAYERS))

    def forward(self, x, ref, ss, lsi):
        for layer in self.layers:
            x = layer(x, ref, ss, lsi)
        return x


def pct(xs, q):
    return sorted(xs)[min(len(xs) - 1, int(q * len(xs)))]


def summary(xs):
    return dict(median_ms=round(pct(xs, 0.5), 4), p25_ms=round(pct(xs, 0.25), 4), p75_ms=round(pct(xs, 0.75), 4))


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    name, power, clock = gpu_info()
    res = dict(device=name, power_limit=power, max_sm_clock=clock, torch=torch.__version__, iters=a.iters, shapes={})
    g = torch.Generator(device=dev).manual_seed(0)
    for key, shapes in SHAPES.items():
        L = len(shapes)
        S = sum(h * w for h, w in shapes)
        params = module_problem(seed=1, N=1, d_model=C, n_heads=HEADS, shapes=shapes, n_points=POINTS,
                                dtype=torch.float32)["params"]
        ss = torch.as_tensor(shapes, dtype=torch.long, device=dev)
        lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
        ref = grid_reference_points(shapes, N, torch.float32).to(dev)
        stack = Stack(L).to(dev)
        for layer in stack.layers:
            layer.attn.load_state_dict(params)
        x = torch.randn(N, S, C, device=dev, generator=g).requires_grad_(True)
        go = torch.randn(N, S, C, device=dev, generator=g)

        def step_of(fn, amp):
            def step():
                torch.compiler.cudagraph_mark_step_begin()
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp == "bf16"):
                    out = fn(x, ref, ss, lsi)
                out.backward(go.to(out.dtype))
            return step

        steps, compile_s = {}, {}
        for mode, amp in ARMS:
            fn = stack if mode == "eager" else torch.compile(
                stack, mode="reduce-overhead" if mode == "reduce_overhead" else None, fullgraph=True)
            steps[(mode, amp)] = step_of(fn, amp)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            steps[(mode, amp)]()
            torch.cuda.synchronize()
            compile_s[(mode, amp)] = time.perf_counter() - t0
        times = {arm: [] for arm in ARMS}
        for it in range(a.warmup + a.iters):
            for arm in ARMS:
                for t in [x] + list(stack.parameters()):
                    t.grad = None
                ms = timed(steps[arm])
                if it >= a.warmup:
                    times[arm].append(ms)
        out = dict(N=N, S=S, Lq=S, L=L, d_model=C, heads=HEADS, points=POINTS, layers=LAYERS, ffn=FFN, arms={})
        for mode, amp in ARMS:
            out["arms"][f"{mode}_{amp}"] = dict(**summary(times[(mode, amp)]),
                                                first_call_s=round(compile_s[(mode, amp)], 2))

        # eager cost of the custom ops: one layer forward + backward, custom ops against the direct lib calls
        m = stack.layers[0].attn
        q = torch.randn(N, S, C, device=dev, generator=g).requires_grad_(True)
        layer_ms = {"custom_op": [], "direct": []}
        shipped = msda.MSDeformAttnFusedFunction
        for it in range(a.warmup + a.iters):
            for arm in layer_ms:
                msda.MSDeformAttnFusedFunction = shipped if arm == "custom_op" else DirectFusedFunction
                try:
                    for t in [q] + list(m.parameters()):
                        t.grad = None
                    ms = timed(lambda: m(q, ref, q, ss, lsi).backward(go))
                finally:
                    msda.MSDeformAttnFusedFunction = shipped
                if it >= a.warmup:
                    layer_ms[arm].append(ms)
        out["eager_layer_fwd_bwd"] = {arm: summary(v) for arm, v in layer_ms.items()}
        res["shapes"][key] = out
        del stack, x, go, q, steps
        torch._dynamo.reset()
        torch.cuda.empty_cache()

    # host time per call: the fused forward op against lib on a tiny problem (N = 1, Lq = 1, one 2x2 level)
    tiny = [torch.randn(1, 4, 8, 32, device=dev), torch.tensor([[2, 2]], device=dev), torch.zeros(1, dtype=torch.long,
            device=dev), torch.rand(1, 1, 1, 2, device=dev), torch.randn(1, 1, 8, 1, 4, 2, device=dev),
            torch.randn(1, 1, 8, 4, device=dev)]
    calls = {"custom_op": lambda: torch.ops.odise_b200.msda_fused_forward(*tiny),
             "direct": lambda: lib.msda_fused_forward(*tiny)}
    per_call = {arm: [] for arm in calls}
    for rep in range(11):
        for arm, fn in calls.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(2000):
                fn()
            torch.cuda.synchronize()
            if rep:
                per_call[arm].append((time.perf_counter() - t0) / 2000 * 1e6)
    res["fused_forward_host_us_per_call"] = {arm: dict(median=round(pct(v, 0.5), 2), min=round(min(v), 2),
                                                       max=round(max(v), 2)) for arm, v in per_call.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
