"""Forward + backward of Mask2Former's pixel decoder (odise_b200.pixel_decoder, 6 encoder layers, GN) at the training
geometry: 1024^2 crops, s2..s5 at 256^2 / 128^2 / 64^2 / 32^2 with 512 channels.  Alternates the fused FPN step
(odise_fpn_upsample_add_* kernels) with the composed F.interpolate + add (use_fused = False) and prints per arm the
median ms, the peak max_memory_allocated above the inputs and the number of synchronising CUDA calls of one step.
Then the FPN op alone (128^2 -> 256^2, C = 256): forward and backward kernel time from CUDA events, and the bytes the
algorithm needs over that time against the 3.35 TB/s data-sheet HBM3 figure.  The device name and power limit are read
in the same run.

    python tools/pixel_decoder_bench.py [--batches 4 8] [--iters 10] [--rounds 3] [--out f]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from odise_b200 import lib  # noqa: E402
from odise_b200 import pixel_decoder as pd  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


class Shape:
    def __init__(self, channels, stride):
        self.channels, self.stride = channels, stride


def build(device):
    torch.manual_seed(0)
    return pd.MSDeformAttnPixelDecoder(
        {f"s{i}": Shape(512, 2 ** i) for i in (2, 3, 4, 5)}, transformer_dropout=0.0, transformer_nheads=8,
        transformer_dim_feedforward=1024, transformer_enc_layers=6, conv_dim=256, mask_dim=256, norm="GN",
        transformer_in_features=["s3", "s4", "s5"], common_stride=4).to(device).train()


def inputs(B, size, device):
    g = torch.Generator(device=device).manual_seed(1)
    return {f"s{i}": torch.randn(B, 512, size // 2 ** i, size // 2 ** i, device=device, generator=g,
                                 requires_grad=True) for i in (2, 3, 4, 5)}


def step(m, feats):
    mf, o0, ms = m.forward_features(feats)
    (mf.mean() + o0.mean() + sum(o.mean() for o in ms)).backward()


def syncs(m, feats):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            step(m, feats)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def timed(m, feats, iters):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        m.zero_grad(set_to_none=True)
        a.record()
        step(m, feats)
        b.record()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def op_alone(N, device, reps=50):
    """forward and backward kernel ms of the FPN op at the ODISE step (128^2 -> 256^2, C = 256), median of reps"""
    C, h, w, H, W = 256, 128, 128, 256, 256
    mem = torch.randn(N, h * w + 80 * 80, C, device=device)
    z = mem[:, 4096:4096 + h * w]
    cur = torch.randn(N, C, H, W, device=device)
    out = {}
    for name, fn in (("forward", lambda: lib.fpn_upsample_add(z, cur, (h, w))),
                     ("backward", lambda: lib.fpn_upsample_add_backward(cur, (h, w))),
                     ("torch_forward", lambda: cur + F.interpolate(z.transpose(1, 2).view(N, C, h, w), size=(H, W),
                                                                    mode="bilinear", align_corners=False))):
        for _ in range(5):
            fn()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        out[name] = statistics.median(ts)
    # bytes the algorithm needs: forward reads z and cur and writes y; backward reads grad_y and writes grad_z
    fwd_bytes = 4 * N * C * (h * w + 2 * H * W)
    bwd_bytes = 4 * N * C * (H * W + h * w)
    return dict(N=N, forward_ms=out["forward"], backward_ms=out["backward"], torch_forward_ms=out["torch_forward"],
                forward_bytes=fwd_bytes, backward_bytes=bwd_bytes,
                forward_TBps=fwd_bytes / out["forward"] / 1e9, backward_TBps=bwd_bytes / out["backward"] / 1e9,
                forward_share_of_hbm=fwd_bytes / out["forward"] / 1e-3 / HBM_BYTES_PER_S,
                backward_share_of_hbm=bwd_bytes / out["backward"] / 1e-3 / HBM_BYTES_PER_S)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 8])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pixel_decoder_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi, size=args.size, rows=[], op=[])
    m = build(dev)
    for B in args.batches:
        feats = inputs(B, args.size, dev)
        times = {"fused": [], "composed": []}
        peak, nsync = {}, {}
        for arm in times:                       # warm-up, peak memory and sync count per arm
            m.use_fused = arm == "fused"
            for _ in range(2):
                m.zero_grad(set_to_none=True)
                step(m, feats)
            m.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            step(m, feats)
            torch.cuda.synchronize()
            peak[arm] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
            m.zero_grad(set_to_none=True)
            nsync[arm] = syncs(m, feats)
        for _ in range(args.rounds):            # alternate the arms
            for arm in times:
                m.use_fused = arm == "fused"
                times[arm] += timed(m, feats, args.iters)
        for arm in times:
            row = dict(B=B, arm=arm, median_ms=statistics.median(times[arm]), n=len(times[arm]),
                       peak_mib_above_inputs=peak[arm], syncs=nsync[arm])
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
        del feats
        m.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()
    for B in args.batches:
        r = op_alone(B, dev)
        res["op"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps(dict(device=res["device"], nvidia_smi=smi)))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
