"""Generate tests/golden/ref_msda_kernel.pt: outputs of the REFERENCE's own MSDeformAttn CUDA kernel (oracle/_ref/libref_msda.so,
built by oracle/Makefile where the reference tree is present) on the seeded problems of
tests/test_gpu_msda.py::test_msda_vs_reference_kernel.  Needs a GPU.  The outputs are large, so a fixed, seeded sample of
4096 elements per problem is stored, with the problem's maximum |output| for the tolerance.

    python tools/make_golden_msda_ref.py [OUT_DIR]      (default tests/golden)
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import refmsda  # noqa: E402
from test_gpu_msda import REFKERNEL_CASES, _problem, refkernel_sample  # noqa: E402


def main(out_dir):
    dev = torch.device("cuda:0")
    cases = []
    for cfg in REFKERNEL_CASES:
        value, ss, lsi, loc, aw = (t.to(dev) for t in _problem(**cfg))
        want = refmsda.forward(value, ss, lsi, loc, aw, 128)
        torch.cuda.synchronize()
        idx = refkernel_sample(want.numel(), cfg["seed"])
        cases.append(dict(cfg=cfg, idx=idx, want=want.flatten()[idx.to(dev)].cpu(), absmax=want.abs().max().item()))
    os.makedirs(out_dir, exist_ok=True)
    torch.save(cases, os.path.join(out_dir, "ref_msda_kernel.pt"))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
