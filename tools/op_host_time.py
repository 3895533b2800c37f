"""Host time per call of the training custom ops on a launch-bound problem (one 2x2 level, one query; the kernels take
a few microseconds, so the time is the op's dispatch and lib's checks, allocations and launch), for one or more source
trees run alternately on one machine.

    python tools/op_host_time.py [--trees DIR [DIR ...]] [--rounds 10] [--calls 2000]

Each round runs one fresh process per tree, with that tree first on sys.path, so that two versions of odise_b200 (for
instance a change and its parent checked out side by side, each with its built library) are measured in turns, the
order reversed every other round.  A
process calls each op --calls times to warm up, then times --calls calls per op between two device synchronisations.
Reported per tree and op: median, min and max microseconds per call over the rounds.  The device name and power limit
are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def one(tree, calls):
    """-> {op: microseconds per call} of this process, with tree's odise_b200"""
    sys.path.insert(0, tree)
    import torch
    from odise_b200 import lib, masked_attn, msda  # noqa: F401  (importing them defines the ops)
    assert os.path.dirname(os.path.abspath(lib.__file__)) == os.path.join(os.path.abspath(tree), "odise_b200")
    dev = torch.device("cuda:0")
    ops = torch.ops.odise_b200
    # MSDA: N = 1, Lq = 1, one 2x2 level, 8 heads of D = 32, 4 points; masked cross-attention: Q = S = B = 1, one head
    fused = (torch.randn(1, 4, 8, 32, device=dev), torch.tensor([[2, 2]], device=dev),
             torch.zeros(1, dtype=torch.long, device=dev), torch.rand(1, 1, 1, 2, device=dev),
             torch.randn(1, 1, 8, 1, 4, 2, device=dev), torch.randn(1, 1, 8, 4, device=dev))
    grad = torch.randn(1, 1, 256, device=dev)
    q = torch.randn(1, 1, 32, device=dev)
    calls_of = {
        "msda_fused_forward": lambda: ops.msda_fused_forward(*fused),
        "lib.msda_fused_forward": lambda: lib.msda_fused_forward(*fused),
        "msda_fused_backward": lambda: ops.msda_fused_backward(*fused, grad, False),
        "msda_fused_backward_det": lambda: ops.msda_fused_backward(*fused, grad, True),
        "masked_xattn_forward": lambda: ops.masked_xattn_forward(q, q, q, None, 1),
    }
    res = {}
    for _ in range(2):          # the first pass warms up; the second one's times are kept
        for name, fn in calls_of.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(calls):
                fn()
            torch.cuda.synchronize()
            res[name] = (time.perf_counter() - t0) / calls * 1e6
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="+", default=[ROOT])
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--one", help=argparse.SUPPRESS)      # the per-process measurement of one tree
    a = ap.parse_args()
    if a.one:
        print(json.dumps(one(a.one, a.calls)))
        return
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    us = {tree: {} for tree in a.trees}
    for r in range(a.rounds):
        for tree in a.trees[::-1] if r % 2 else a.trees:
            cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
                os.path.abspath(__file__), "--one", tree, "--calls", str(a.calls)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode:
                sys.exit(f"{tree}: {r.stderr[-4000:]}")
            for op, t in json.loads(r.stdout.splitlines()[-1]).items():
                us[tree].setdefault(op, []).append(t)
    print(json.dumps(dict(device=smi, rounds=a.rounds, calls=a.calls, us_per_call={
        tree: {op: dict(median=round(statistics.median(v), 2), min=round(min(v), 2), max=round(max(v), 2))
               for op, v in ops.items()} for tree, ops in us.items()})))


if __name__ == "__main__":
    main()
