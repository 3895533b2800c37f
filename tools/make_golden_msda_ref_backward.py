"""Generate tests/golden/ref_msda_kernel_backward.pt: gradients of the REFERENCE's own MSDeformAttn CUDA backward
(oracle/_ref/libref_msda_backward.so, built by oracle/backward.mk where the reference tree is present) on the seeded,
boundary-safe problems of tests/test_gpu_msda_backward.py::test_backward_vs_reference_kernel.  Needs a GPU.  The
gradients are large, so a fixed, seeded sample of 4096 positions per gradient tensor is stored, with the tensor's
maximum |.| for the tolerance.

    python tools/make_golden_msda_ref_backward.py [OUT_DIR]      (default tests/golden)
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import refmsda_backward, refshim  # noqa: E402
from oracle.msda_grad import grad_problem  # noqa: E402
from test_gpu_msda_backward import REFKERNEL_BWD_CASES  # noqa: E402


def main(out_dir):
    dev = torch.device("cuda:0")
    cases = []
    for cfg in REFKERNEL_BWD_CASES:
        args = [t.to(dev, torch.float32) if t.is_floating_point() else t.to(dev) for t in grad_problem(**cfg)]
        grads = refmsda_backward.backward(*args, 128)
        torch.cuda.synchronize()
        c = dict(cfg=cfg)
        for i, (name, g) in enumerate(zip(("grad_value", "grad_loc", "grad_attn"), grads)):
            s = refshim.sample(g.cpu(), seed=1000 + 10 * cfg["seed"] + i)
            c[name] = dict(idx=s["idx"], values=s["values"], absmax=g.abs().max().item())
        cases.append(c)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "ref_msda_kernel_backward.pt")
    torch.save(cases, path)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
