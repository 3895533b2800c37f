"""UNet attention for training: the fused sm_90a kernels (odise_b200/unet_attn.py) against ldm's composed
einsum / softmax / einsum, at every attention shape of the SD-v1 UNet at B = 8, the per-pass batch of ODISE's recipe
(64 images per step on 8 GPUs, each image cut into 512^2 slide crops: 4 UNet passes of B = 8 on a 64^2 latent).

Per shape (head dim d, Tq, Tk; 8 heads) and arm it reports the forward and forward + backward time of the attention
core alone (q / k / v already projected): the median and the min-max over rounds in which the arms alternate, each round
one CUDA-event window of back-to-back calls lasting about --window-ms; the peak allocation of forward + backward above
the inputs; and the achieved TFLOP/s under the FLOP model below.  Arms: fused and composed in float32 and in float16 /
bfloat16 storage under torch.autocast, as the module runs them (the composed softmax is then float32); torch SDPA (its
default backend choice) is recorded for context only.  A composed arm whose [B*h, Tq, Tk] tensors would not fit in free
memory is reported as "does not fit" without running it.

It also times one forward + backward of the whole UNet (oracle.ldm.UNetModel, random init, float32) through
oracle.ldm.unet_features at a B = 8 crop pass on a 64^2 latent, with context and cond_emb requiring grad, patched by
replace_attention, fused against composed.

FLOP model (multiply-add = 2): forward 4 B h Tq Tk d (q k^T and P v); backward 8 B h Tq Tk d (dV = P^T dO,
dP = dO v^T, dQ = dS k, dK = dS^T q); the fused backward's recomputation of q k^T is not counted.
The device name and power limit are read in the same run.  Output: one JSON line per measurement, and a markdown table."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from odise_b200.unet_attn import CrossAttention, UNetAttnFunction, replace_attention  # noqa: E402
from oracle import ldm  # noqa: E402

B, HEADS = 8, 8
SHAPES = [(40, 4096, 4096), (80, 1024, 1024), (160, 256, 256), (160, 64, 64),
          (40, 4096, 77), (80, 1024, 77), (160, 256, 77), (160, 64, 77)]
DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def composed(q, k, v):
    """oracle/ldm.py's CrossAttention core, op for op"""
    b, n, _ = q.shape
    q, k, v = (t.reshape(b, t.shape[1], HEADS, -1).permute(0, 2, 1, 3) for t in (q, k, v))
    sim = torch.einsum("bhid,bhjd->bhij", q, k) * q.shape[-1] ** -0.5
    out = torch.einsum("bhij,bhjd->bhid", sim.softmax(dim=-1), v)
    return out.permute(0, 2, 1, 3).reshape(b, n, -1)


def sdpa(q, k, v):
    b, n, _ = q.shape
    q, k, v = (t.reshape(b, t.shape[1], HEADS, -1).transpose(1, 2) for t in (q, k, v))
    return F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(b, n, -1)


ARMS = {"fused": lambda q, k, v: UNetAttnFunction.apply(q, k, v, HEADS), "composed": composed, "sdpa": sdpa}


def window_ms(fn, calls):
    """ms per call over one CUDA-event window of `calls` back-to-back calls"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / calls


def composed_bytes(Tq, Tk, dtype):
    """the [B*h, Tq, Tk] tensors the composed forward + backward can hold at once.  float32: the scores, their softmax
    (saved) and the backward's gradient of each, 4 bytes.  Under autocast the scores are 16-bit, softmax runs in float32
    and saves its fp32 output, the second einsum saves a 16-bit copy, and the backward makes 16-bit and fp32 gradients:
    2 + 4 + 2 + 2 + 4 + 4 + 2 bytes"""
    return B * HEADS * Tq * Tk * (16 if dtype == torch.float32 else 20)


def attention_rows(rounds, window):
    """per shape and dtype: every arm timed in `rounds` rounds, the arms alternating inside each round; each round is
    one CUDA-event window of enough calls to last about `window` ms.  The 16-bit arms run under torch.autocast, as the
    module runs them (the composed path's softmax is then float32)."""
    rows = []
    for d, Tq, Tk in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(0)
        for dname, dt in DTYPES.items():
            q = torch.randn(B, Tq, HEADS * d, generator=g, device="cuda").to(dt).requires_grad_(True)
            k = torch.randn(B, Tk, HEADS * d, generator=g, device="cuda").to(dt).requires_grad_(True)
            v = torch.randn(B, Tk, HEADS * d, generator=g, device="cuda").to(dt).requires_grad_(True)
            go = torch.randn(B, Tq, HEADS * d, generator=g, device="cuda").to(dt)
            ac = dict(device_type="cuda", dtype=dt, enabled=dt != torch.float32)
            arms, out = {}, {}
            for arm, fn in ARMS.items():
                row = dict(d=d, Tq=Tq, Tk=Tk, B=B, dtype=dname, arm=arm)
                out[arm] = row
                if arm == "composed" and composed_bytes(Tq, Tk, dt) > 0.9 * torch.cuda.mem_get_info()[0]:
                    row["result"] = "does not fit"
                    continue

                def fwd(fn=fn):
                    with torch.no_grad(), torch.autocast(**ac):
                        fn(q, k, v)

                def fwd_bwd(fn=fn):
                    with torch.autocast(**ac):
                        o = fn(q, k, v)
                    torch.autograd.grad(o, (q, k, v), go.to(o.dtype))
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                fwd_bwd()
                torch.cuda.synchronize()
                row["peak_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
                calls = {}
                for name, f in (("fwd", fwd), ("fwd_bwd", fwd_bwd)):
                    f()
                    calls[name] = max(1, min(200, int(window / max(window_ms(f, 1), 1e-3))))
                arms[arm] = (fwd, fwd_bwd, calls)
                row["fwd_all"], row["fwd_bwd_all"] = [], []
            for _ in range(rounds):
                for arm, (fwd, fwd_bwd, calls) in arms.items():
                    out[arm]["fwd_all"].append(window_ms(fwd, calls["fwd"]))
                    out[arm]["fwd_bwd_all"].append(window_ms(fwd_bwd, calls["fwd_bwd"]))
            f = 4 * B * HEADS * Tq * Tk * d
            for arm, row in out.items():
                if arm in arms:
                    for key in ("fwd", "fwd_bwd"):
                        xs = row.pop(key + "_all")
                        row[key + "_ms"], row[key + "_min"], row[key + "_max"] = statistics.median(xs), min(xs), max(xs)
                    row["fwd_tflops"] = f / row["fwd_ms"] / 1e9
                    row["fwd_bwd_tflops"] = 3 * f / row["fwd_bwd_ms"] / 1e9
                rows.append(row)
                print(json.dumps(row), flush=True)
            del q, k, v, go
    return rows


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        ts.append(window_ms(fn, 1))
    return statistics.median(ts)


def unet_rows(iters, warmup):
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)
    unet = ldm.UNetModel().cuda()
    assert replace_attention(unet) == 32
    attn = [m for m in unet.modules() if isinstance(m, CrossAttention)]
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(B, 4, 64, 64, generator=g, device="cuda")
    ctx = torch.randn(B, 77, 768, generator=g, device="cuda").requires_grad_(True)
    cond = (torch.randn(B, 1280, generator=g, device="cuda") * 0.5).requires_grad_(True)

    def step():
        unet.zero_grad(set_to_none=True)
        taps = ldm.unet_features(unet, x, ctx, cond)
        torch.autograd.backward(taps, [torch.ones_like(t) for t in taps])
    rows = []
    for arm in ("fused", "composed"):
        for m in attn:
            m.use_fused = arm == "fused"
        row = dict(what="unet_features fwd+bwd", B=B, latent=64, dtype="fp32", arm=arm)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        try:
            step()
        except torch.OutOfMemoryError:
            row["result"] = "out of memory"
            rows.append(row)
            print(json.dumps(row), flush=True)
            continue
        torch.cuda.synchronize()
        row["peak_gib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
        row["ms"] = timed(step, iters, warmup)
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--window-ms", type=float, default=20.0)
    ap.add_argument("--skip-unet", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(), nvidia_smi=smi)), flush=True)
    rows = attention_rows(args.rounds, args.window_ms)
    print("\n| d | Tq | Tk | dtype | arm | fwd ms (min-max) | fwd+bwd ms (min-max) | peak MiB | fwd+bwd TFLOP/s |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        if "result" in r:
            print(f"| {r['d']} | {r['Tq']} | {r['Tk']} | {r['dtype']} | {r['arm']} | {r['result']} | | | |")
        else:
            print(f"| {r['d']} | {r['Tq']} | {r['Tk']} | {r['dtype']} | {r['arm']} | {r['fwd_ms']:.3f} "
                  f"({r['fwd_min']:.3f}-{r['fwd_max']:.3f}) | {r['fwd_bwd_ms']:.3f} ({r['fwd_bwd_min']:.3f}-"
                  f"{r['fwd_bwd_max']:.3f}) | {r['peak_mib']:.0f} | {r['fwd_bwd_tflops']:.1f} |")
    if not args.skip_unet:
        for r in unet_rows(5, 1):
            print(f"| UNet B={B} 64^2 fp32 fwd+bwd | {r['arm']} | {r.get('result', '%.1f ms' % r.get('ms', 0))} | "
                  f"peak {r.get('peak_gib', float('nan')):.1f} GiB |")


if __name__ == "__main__":
    main()
