"""Microbenchmark of the masked cross-attention drop-in (odise_b200.masked_attn.CrossAttentionLayer): one layer,
forward + backward, fused (odise_masked_xattn_*) against use_fused = False (nn.MultiheadAttention's math path), arms
alternated (the fused arms lift the layer's 16-bit key limit, so they time the kernels at every level):

  fused_f32 / composed_f32      float32 layer
  fused_bf16 / composed_bf16    under torch.autocast("cuda", torch.bfloat16)
  fused_f16 / composed_f16      under torch.autocast("cuda", torch.float16)

Shapes: the ODISE decoder at a 1024 x 1024 training crop: B = 2, Q = 100 queries, d_model 256, 8 heads, keys of the three
levels 32^2, 64^2 and 128^2, bool masks from mask logits with the odise.py:683 fix-up, [B*8, Q, S].  Per (level, arm)
and run: median ms over --iters iterations (CUDA events, --warmup first).  Then torch.cuda.max_memory_allocated above
the inputs for the forward + backward of the 9-layer cross-attention stack (levels 0, 1, 2, 0, ...), per arm.  The
device name and power limit are read in the same run.  Prints one JSON line.

    python tools/masked_xattn_bench.py [--iters 30] [--warmup 5] [--runs 2]
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
from odise_b200.masked_attn import CrossAttentionLayer  # noqa: E402
from msda_backward_bench import gpu_info  # noqa: E402

B, Q, C, H = 2, 100, 256, 8
LEVELS = [32 * 32, 64 * 64, 128 * 128]
ARMS = {  # name -> (autocast dtype or None, use_fused)
    "fused_f32": (None, True),
    "composed_f32": (None, False),
    "fused_bf16": (torch.bfloat16, True),
    "composed_bf16": (torch.bfloat16, False),
    "fused_f16": (torch.float16, True),
    "composed_f16": (torch.float16, False),
}


@contextlib.contextmanager
def arm_context(arm, layers):
    dtype, fused = ARMS[arm]
    for m in layers:
        m.use_fused = fused
        m.fused_16bit_max_keys = None       # the fused arms run the kernels at every level
    with (torch.autocast("cuda", dtype=dtype) if dtype is not None else contextlib.nullcontext()):
        yield


def median(xs):
    return sorted(xs)[len(xs) // 2]


def make_mask(S, g):
    m = torch.randn(B, Q, S, generator=g, device="cuda").sigmoid() < 0.5
    m = m.unsqueeze(1).repeat(1, H, 1, 1).flatten(0, 1)
    m[torch.where(m.sum(-1) == m.shape[-1])] = False
    return m


def step(layer, tgt, mem, mask, pos, qpos):
    out = layer(tgt, mem, memory_mask=mask, pos=pos, query_pos=qpos)
    out.float().sum().backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "masked_xattn_bench needs a GPU"
    dev = torch.device("cuda")
    torch.manual_seed(0)
    g = torch.Generator(device=dev).manual_seed(1)
    layer = CrossAttentionLayer(C, H).to(dev)
    tgt = torch.randn(Q, B, C, generator=g, device=dev, requires_grad=True)
    qpos = torch.randn(Q, B, C, generator=g, device=dev)
    data = {}
    for S in LEVELS:
        data[S] = (torch.randn(S, B, C, generator=g, device=dev, requires_grad=True),
                   torch.randn(S, B, C, generator=g, device=dev), make_mask(S, g))
    times = {run: {S: {a: [] for a in ARMS} for S in LEVELS} for run in range(args.runs)}
    for run in range(args.runs):
        for S in LEVELS:
            mem, pos, mask = data[S]
            for arm in ARMS:
                with arm_context(arm, [layer]):
                    for _ in range(args.warmup):
                        step(layer, tgt, mem, mask, pos, qpos)
            torch.cuda.synchronize()
            for _ in range(args.iters):
                for arm in ARMS:            # alternate the arms iteration by iteration
                    with arm_context(arm, [layer]):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        step(layer, tgt, mem, mask, pos, qpos)
                        e1.record()
                        e1.synchronize()
                        times[run][S][arm].append(e0.elapsed_time(e1))
    layer_ms = {f"run{run}": {str(S): {a: round(median(v), 4) for a, v in times[run][S].items()} for S in LEVELS}
                for run in range(args.runs)}
    # peak memory of the 9-layer cross-attention stack, forward + backward
    stack = torch.nn.ModuleList([CrossAttentionLayer(C, H) for _ in range(9)]).to(dev)
    masks = [make_mask(LEVELS[i % 3], g) for i in range(9)]
    peak = {}
    for arm in ARMS:
        with arm_context(arm, stack):
            for attempt in range(2):      # the first pass warms the allocator and libraries
                tgt.grad = None
                for m in data.values():
                    m[0].grad = None
                stack.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                out = tgt
                for i, lyr in enumerate(stack):
                    mem, pos, _ = data[LEVELS[i % 3]]
                    out = lyr(out, mem, memory_mask=masks[i], pos=pos, query_pos=qpos)
                out.float().sum().backward()
                torch.cuda.synchronize()
                peak[arm] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
                del out
    print(json.dumps(dict(bench="masked_xattn", gpu=gpu_info(), B=B, Q=Q, d_model=C, heads=H, levels=LEVELS,
                          iters=args.iters, layer_fwd_bwd_ms=layer_ms, stack9_peak_mib=peak)))


if __name__ == "__main__":
    main()
