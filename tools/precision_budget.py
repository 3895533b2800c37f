"""Error budget of cheaper tensor-core precision modes for the UNet feature pass (VERDICT r1 item 4a), by EMULATION on the
CPU oracle: every contraction of the SD-v1 UNet (3x3 convs | 1x1 convs + linears | attention QK^T and PV) is run with its
operands rounded the way a given tensor-core scheme would see them, and the four taps are compared with the plain fp32 oracle
(the parity reference; bar 1e-3 on max|a-b| / max|b|, ship rule: >= 3x margin -> <= 3.3e-4).

Schemes (cost in bf16-MMA units per k-step; bf16x3 = what the engine ships):
  bf16x3     hi*hi + hi*lo + lo*hi, bf16 planes                         cost 3
  fp16x3     same with fp16 planes                                      cost 3
  fp16x2     (A_hi + A_lo) * W_hi, fp16 planes: weight / second operand rounded to fp16, first exact     cost 2
  bf16x2     same with bf16 planes                                      cost 2
  tf32       kind::tf32, both operands rounded to 10 mantissa bits (RN; the hardware truncates: tf32t)   cost 2
  bf16       plain bf16                                                 cost 1
Usage: python tools/precision_budget.py [--latent 64]"""
import argparse
import os
import sys
import time

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from odise_b200 import spec  # noqa: E402
from oracle import ldm  # noqa: E402


def q_bf16(x): return x.bfloat16().float()
def q_fp16(x): return x.half().float()


def q_tf32(x, truncate=False):
    i = x.contiguous().view(torch.int32)
    if not truncate:
        i = i + 0x1000
    return (i & ~0x1FFF).view(torch.float32)


def contract(op, a, b, mode):
    """op(a, b) with operands as the scheme `mode` presents them (b = weight / second operand)."""
    if mode == "fp32":
        return op(a, b)
    if mode == "bf16":
        return op(q_bf16(a), q_bf16(b))
    if mode == "tf32":
        return op(q_tf32(a), q_tf32(b))
    if mode == "tf32t":
        return op(q_tf32(a, True), q_tf32(b, True))
    if mode == "fp16x2":
        return op(a, q_fp16(b))
    if mode == "bf16x2":
        return op(a, q_bf16(b))
    if mode in ("bf16x3", "fp16x3"):                    # all terms but lo*lo (lo planes themselves rounded once more)
        q = q_bf16 if mode == "bf16x3" else q_fp16
        ah, bh = q(a), q(b)
        al, bl = q(a - ah), q(b - bh)
        return op(ah, bh) + op(ah, bl) + op(al, bh)
    if mode == "fp16x2c8":
        # fp16 2-term + the dropped cross term A * W_lo recovered by ONE fp8 MMA at twice the rate (kind::f8f6f4):
        # A rounded to 2 mantissa bits (e5m2), W_lo to 3 (e4m3); range / scaling not modelled -> an upper bound on the gain
        bh = q_fp16(b)
        return op(a, bh) + op(q_bits(a, 2), q_bits(b - bh, 3))
    if mode.startswith("f16c8"):
        # fp16 main product + BOTH cross terms on fp8 MMAs (kind::f8f6f4, twice the 16-bit rate) -> cost 2:
        #   A_hi*W_hi [fp16]  +  e5m2(A * 2^-a) * e5m2(W_lo * 2^a)  +  e5m2(A_lo * 2^b) * e5m2(W * 2^-b)
        # with the real e5m2 range / subnormals / saturation (torch.float8_e5m2) and global power-of-two scales (a, b)
        t8 = torch.float8_e4m3fn if mode.endswith("e4") else torch.float8_e5m2
        lim = 448.0 if mode.endswith("e4") else 57344.0
        q8 = lambda x: x.clamp(-lim, lim).to(t8).float()
        sa, sb = float(os.environ.get("PB_SA", 8)), float(os.environ.get("PB_SB", 4))
        ah, bh = q_fp16(a), q_fp16(b)
        al, bl = a - ah, b - bh
        return op(ah, bh) + op(q8(a * 2.0 ** -sa), q8(bl * 2.0 ** sa)) + op(q8(al * 2.0 ** sb), q8(b * 2.0 ** -sb))
    raise ValueError(mode)


def q_bits(x, k):
    """round to k explicit mantissa bits (RN, ties away), exponent range unchanged"""
    i = x.contiguous().view(torch.int32)
    sh = 23 - k
    return ((i + (1 << (sh - 1))) & ~((1 << sh) - 1)).view(torch.float32)


MODES = {"conv3": "fp32", "lin": "fp32", "attn": "fp32"}


def patch(unet):
    for m in unet.modules():
        if isinstance(m, nn.Conv2d):
            cls = "conv3" if m.kernel_size[0] == 3 else "lin"
            def fwd(x, m=m, cls=cls):
                y = contract(lambda a, b: F.conv2d(a, b, None, m.stride, m.padding), x, m.weight, MODES[cls])
                return y if m.bias is None else y + m.bias.view(1, -1, 1, 1)
            m.forward = fwd
        elif isinstance(m, nn.Linear):
            def fwd(x, m=m):
                y = contract(lambda a, b: F.linear(a, b), x, m.weight, MODES["lin"])
                return y if m.bias is None else y + m.bias
            m.forward = fwd
        elif isinstance(m, ldm.CrossAttention):
            def fwd(x, context=None, m=m):
                h = m.heads
                q = m.to_q(x)
                context = x if context is None else context
                k, v = m.to_k(context), m.to_v(context)
                b, n, _ = q.shape
                q, k, v = (t.reshape(b, t.shape[1], h, -1).permute(0, 2, 1, 3) for t in (q, k, v))
                if MODES["attn"] == "p16":
                    # shipped attention scheme: S in bf16x3; P rounded ONCE to fp16 (one plane), V as (hi, lo) bf16 planes:
                    # O = P16 * V_hi + P16 * V_lo.  P is the un-normalised exp(s - rowmax) in [0, 1] (normalised at the end)
                    sim = contract(lambda a, c: torch.einsum("bhid,bhjd->bhij", a, c), q, k, "bf16x3") * m.scale
                    p = torch.exp(sim - sim.amax(-1, keepdim=True))
                    vh = q_bf16(v)
                    v2 = vh + q_bf16(v - vh)
                    out = torch.einsum("bhij,bhjd->bhid", q_fp16(p), v2) / p.sum(-1, keepdim=True)
                else:
                    sim = contract(lambda a, c: torch.einsum("bhid,bhjd->bhij", a, c), q, k, MODES["attn"]) * m.scale
                    out = contract(lambda a, c: torch.einsum("bhij,bhjd->bhid", a, c), sim.softmax(dim=-1), v, MODES["attn"])
                return m.to_out(out.permute(0, 2, 1, 3).reshape(b, n, -1))
            m.forward = fwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent", type=int, default=64)
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    sd = spec.synth_state_dict(spec.unet_params(), 0)
    with torch.device("meta"):
        unet = ldm.UNetModel()
    unet.load_state_dict({k[len(spec.UNET_PREFIX):]: v for k, v in sd.items()}, assign=True)
    unet.eval()
    g = torch.Generator().manual_seed(7)
    L = a.latent
    x, ctx, cond = torch.randn(1, 4, L, L, generator=g), torch.randn(1, 77, 768, generator=g), torch.randn(1, 1280, generator=g) * 0.5
    with torch.no_grad():
        ref = ldm.unet_features(unet, x, ctx, cond)
    patch(unet)

    def run(conv3, lin, attn):
        MODES.update(conv3=conv3, lin=lin, attn=attn)
        t0 = time.time()
        with torch.no_grad():
            out = ldm.unet_features(unet, x, ctx, cond)
        errs = [((o.double() - r.double()).abs().max() / r.double().abs().max()).item() for o, r in zip(out, ref)]
        return errs, time.time() - t0

    cost = {"fp32": None, "bf16x3": 3, "fp16x3": 3, "fp16x2": 2, "bf16x2": 2, "tf32": 2, "tf32t": 2, "bf16": 1, "fp16x2c8": 2.5,
            "p16": 2.5, "f16c8": 2, "f16c8e4": 2}
    # MMA-FLOP share of the three classes in the minimal feature pass (per-GEMM shapes of one step, tools/gemm_shapes.py:
    # convs ~ 62 %, linears / 1x1 ~ 30 %, attention ~ 8 %) -> relative tensor time of a mix vs all-bf16x3
    share = {"conv3": 0.62, "lin": 0.30, "attn": 0.08}
    print(f"# UNet taps (blocks 2, 5, 8, 11) at a {L}x{L} latent, synthetic weights seed 0; rel = max|a-b| / max|b| vs the fp32 oracle")
    print(f"# {'conv3x3':8s} {'linear':8s} {'attn':8s} | {'tap2':>9s} {'tap5':>9s} {'tap8':>9s} {'tap11':>9s} | {'worst':>9s} | tensor time vs bf16x3 | ships (<= 3.3e-4)")
    rows = [("bf16x3",) * 3, ("fp16x3",) * 3, ("fp16x2",) * 3, ("bf16x2",) * 3, ("tf32",) * 3, ("tf32t",) * 3, ("bf16",) * 3,
            ("fp16x2", "bf16x3", "bf16x3"), ("bf16x3", "fp16x2", "bf16x3"), ("bf16x3", "bf16x3", "fp16x2"),
            ("tf32", "bf16x3", "bf16x3"), ("bf16x3", "bf16x3", "bf16"), ("fp16x2", "fp16x2", "bf16x3"),
            ("bf16x3", "bf16x3", "p16"), ("fp16x2c8", "fp16x2c8", "p16")]
    if os.environ.get("PB_ROWS"):
        rows = [tuple(r.split(",")) for r in os.environ["PB_ROWS"].split(";")]
    for conv3, lin, attn in rows:
        errs, dt = run(conv3, lin, attn)
        rel_t = (share["conv3"] * cost[conv3] + share["lin"] * cost[lin] + share["attn"] * cost[attn]) / 3.0
        w = max(errs)
        print(f"  {conv3:8s} {lin:8s} {attn:8s} | " + " ".join(f"{e:9.2e}" for e in errs) + f" | {w:9.2e} | {rel_t:21.2f} | "
              f"{'yes' if w <= 3.3e-4 else 'NO'}", flush=True)


if __name__ == "__main__":
    main()
