"""Generate tests/golden/msda_*.pt by running the REFERENCE's own PyTorch restatement
ms_deform_attn_core_pytorch (third_party/Mask2Former/.../ops/functions/ms_deform_attn_func.py:52-72), imported
from /root/reference (only available in the build container).  Inputs follow ops/test.py:24-39."""
import os
import sys

import torch

REF = "/root/reference/third_party/Mask2Former/mask2former/modeling/pixel_decoder"
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from ops.functions.ms_deform_attn_func import ms_deform_attn_core_pytorch  # noqa: E402
from oracle.msda import msda_forward  # noqa: E402

OUT = os.path.join(os.path.dirname(__file__), "..", "tests", "golden")


def make(name, seed, N, M, D, shapes, Lq, P, spread=1.0):
    torch.manual_seed(seed)
    ss = torch.as_tensor(shapes, dtype=torch.long)
    lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
    S = int(ss.prod(1).sum())
    L = len(shapes)
    value = torch.rand(N, S, M, D) * 0.01
    loc = torch.rand(N, Lq, M, L, P, 2) * spread - (spread - 1) / 2
    aw = torch.rand(N, Lq, M, L, P) + 1e-5
    aw /= aw.sum(-1, keepdim=True).sum(-2, keepdim=True)
    out64 = ms_deform_attn_core_pytorch(value.double(), ss, loc.double(), aw.double())
    out32 = ms_deform_attn_core_pytorch(value, ss, loc, aw)
    mine = msda_forward(value.double(), ss, lsi, loc.double(), aw.double())
    err = (mine - out64).abs().max().item()
    assert err < 1e-12, (name, err)
    print(f"{name}: oracle-vs-reference fp64 max err {err:.2e}; fp32-vs-fp64 {(out32.double()-out64).abs().max():.2e}")
    torch.save(dict(value=value, spatial_shapes=ss, level_start_index=lsi, sampling_locations=loc,
                    attention_weights=aw, output=out64.float()), os.path.join(OUT, f"msda_{name}.pt"))


if __name__ == "__main__":
    make("reftest", 3, 1, 2, 2, [(6, 4), (3, 2)], 2, 2)                       # exact ops/test.py problem
    make("d32_small", 11, 2, 8, 32, [(4, 4), (8, 8), (12, 12)], 100, 4, spread=1.3)
    make("oob", 12, 1, 4, 8, [(5, 7), (3, 2)], 41, 3, spread=3.0)
