"""Eager step with per-GEMM CUDA-event timing -> gpurun_out/gemm_shapes.csv (+ grouped summary on stdout)."""
import os
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
out = os.path.join("gpurun_out", "gemm_shapes.csv")
os.makedirs("gpurun_out", exist_ok=True)
if os.path.exists(out):
    os.remove(out)
os.environ["ODISE_PROFILE_CSV"] = out
from odise_b200 import lib, spec  # noqa: E402
from odise_b200.pipeline import ODISEEngine, full_param_list, synthetic_vocabulary  # noqa: E402

full = "--full" in sys.argv
nmma = 1 if "--bf16" in sys.argv else (3 if "--bf16x3" in sys.argv else 2)      # default: the F16Q8 operand mode
dev = torch.device("cuda:0")
eng = ODISEEngine(spec.synth_state_dict(full_param_list(with_vae=full, with_clip=full), 0), dev, synthetic_uncond=True, nmma=nmma, with_vae=full,
                  with_clip=full)
eng.set_synthetic_vocabulary("ade150", 150, 403)
for _ in range(2):
    eng.step(4, 1024, 1024)
torch.cuda.synchronize()
lib.profile_begin()
eng.step(4, 1024, 1024)
n, ms, fl = lib.profile_end()
print(f"{n} gemm launches, {ms:.2f} ms, {fl/ms/1e9:.1f} TFLOP/s algorithmic")
agg = defaultdict(lambda: [0, 0.0, 0.0])
for line in open(out).read().splitlines()[1:]:
    M, N, K, b, conv, bn, nm, sp, t, tf = line.split(",")
    k = (int(M), int(N), int(K), int(b), int(conv), int(bn), int(sp), int(nm))
    agg[k][0] += 1
    agg[k][1] += float(t)
    agg[k][2] += 2.0 * int(M) * int(N) * int(K) * int(b)
print("   ms    n   TF/s  (M, N, K, batch, conv, BN, splits, nmma)")
for k, (c, t, f) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:45]:
    print(f"{t:7.3f} {c:4d} {f/t/1e9:6.0f}  {k}")
