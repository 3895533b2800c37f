"""Per-block diagnostic: runs oracle UNet blocks on CPU and the engine on GPU, prints where they diverge."""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from odise_b200 import lib, ops, spec  # noqa: E402
from odise_b200.unet import UNetEngine  # noqa: E402
from oracle import ldm  # noqa: E402


def rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def main():
    hw = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    nmma = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    B = 2
    dev = torch.device("cuda")
    sd = spec.synth_state_dict(spec.unet_params(), 0)
    with torch.device("meta"):
        m = ldm.UNetModel()
    m.load_state_dict({k[len(spec.UNET_PREFIX):]: v for k, v in sd.items()}, assign=True)
    m.eval()
    eng = UNetEngine(sd, dev, nmma=nmma)
    g = torch.Generator().manual_seed(1)
    ctx = torch.randn(B, 77, 768, generator=g)
    cond = torch.randn(B, 1280, generator=g) * 0.5
    t = torch.zeros(B, dtype=torch.long)
    with torch.no_grad():
        emb = m.time_embed(ldm.timestep_embedding(t, 320)) + cond
    # engine-side shared tensors
    embd, _ = ops.add_split(cond.to(dev), eng.emb0, b_rows=1, want_f32=True, want_planes=False)
    print("emb", rel(embd.cpu(), emb))
    e_silu = ops.act_split(embd, 2, lo=eng.lo)
    emb_all = ops.empty(B, eng.emb_total, dev)
    eng._gemm(e_silu, "emb_all", "emb_all.b", out=emb_all)
    cpad = torch.zeros(B, 80, 768, device=dev)
    cpad[:, :77] = ctx.to(dev)
    ctxp = lib.split(cpad.view(B * 80, 768), lo=eng.lo)

    def nhwc(x):
        return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1]).contiguous().to(dev)

    def nchw(y, h, w):
        return y.view(B, h, w, -1).permute(0, 3, 1, 2).cpu()

    # individual layers on random inputs at each resolution
    for name, blocks in (("input_blocks", eng.inp), ("middle_block", [eng.mid]), ("output_blocks", eng.out[:11])):
        for i, layers in enumerate(blocks):
            q = f"{name}.{i}." if name != "middle_block" else "middle_block."
            mod = getattr(m, name)[i] if name != "middle_block" else m.middle_block
            for j, l in enumerate(layers):
                size = hw
                # find a plausible spatial size from channel count
                cin = l[1]
                s = {320: hw, 640: hw // 2, 1280: hw // 4}.get(l[2] if l[0] == "res" else l[1], hw // 8)
                if l[0] == "res":
                    x = torch.randn(B, cin, s, s, generator=g)
                    with torch.no_grad():
                        ref = mod[j](x, emb)
                    dst = ops.empty(B * s * s, l[2], dev)
                    eng._resblock(f"{q}{j}.", nhwc(x), B, s, s, cin, l[2], emb_all, dst)
                    print(f"{q}{j} res {cin}->{l[2]} @{s}: {rel(nchw(dst, s, s), ref):.3e}", flush=True)
                elif l[0] == "st":
                    x = torch.randn(B, cin, s, s, generator=g)
                    with torch.no_grad():
                        ref = mod[j](x, ctx)
                    dst = ops.empty(B * s * s, cin, dev)
                    eng._st(f"{q}{j}.", nhwc(x), B, s, s, cin, ctxp, dst)
                    print(f"{q}{j} st {cin} @{s}: {rel(nchw(dst, s, s), ref):.3e}", flush=True)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
