"""GroupNorm statistics / apply bandwidth at the release shapes (CUDA events, inputs >> L2 or L2 flushed between runs)."""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from odise_b200 import lib, ops  # noqa: E402
from odise_b200.lib import Planes  # noqa: E402

dev = torch.device("cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, n=5):
    fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        s, e = torch.cuda.Event(True), torch.cuda.Event(True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return sorted(ts)[len(ts) // 2]


for (B, HW, C) in [(16, 262144, 128), (16, 65536, 256), (16, 16384, 512), (16, 4096, 320), (16, 4096, 640),
                   (16, 1024, 1280), (16, 4096, 960), (4, 65536, 256)]:
    x = torch.randn(B * HW, C, device=dev)
    ga, be = torch.randn(C, device=dev), torch.randn(C, device=dev)
    mean, rstd = ops._gn_stats(x, C, 0, B, HW, C, 32, 1e-5, None)
    t_stats = timeit(lambda: ops._gn_stats(x, C, 0, B, HW, C, 32, 1e-5, None))
    p = Planes.empty(B * HW, C, dev)
    t_apply = timeit(lambda: lib._launch("odise_groupnorm_apply_f32", x, C, mean, rstd, ga, be, 2, None, 0, p.hi, p.lo,
                                         p.ld, B, HW, C, 32))
    n = B * HW * C
    print(f"B={B} HW={HW} C={C}: stats {t_stats*1000:8.1f} us {4*n/t_stats/1e6:7.0f} GB/s | apply {t_apply*1000:8.1f} us "
          f"{8*n/t_apply/1e6:7.0f} GB/s", flush=True)
    del x, p
