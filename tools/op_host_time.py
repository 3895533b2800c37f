"""Host time per call of the training custom ops on a launch-bound problem (one 2x2 level, one query; the kernels take
a few microseconds, so the time is the op's dispatch and lib's checks, allocations and launch), and of the eager engine
calls of the inference path, for one or more source trees run alternately on one machine.

    python tools/op_host_time.py [--trees DIR [DIR ...]] [--rounds 10] [--calls 2000] [--forwards 20]

Each round runs one fresh process per tree, with that tree first on sys.path, so that two versions of odise_b200 (for
instance a change and its parent checked out side by side, each with its built library) are measured in turns, the
order reversed every other round.  A
process calls each op --calls times to warm up, then times --calls calls per op between two device synchronisations.
The engine arms, which run eagerly and pay lib._launch's argument loop on every launch, time --forwards calls each, every
call between two device synchronisations: one HeadEngine.forward at B = 1 and 128 x 128 (386 launches of the ops
wrappers, lib.split and lib.gemm) and one PostProcessor call (4 launches; 100 queries, 133 classes, semantic, panoptic
and instance outputs at 128 x 128).
Reported per tree and arm: median, min and max microseconds per call over the rounds.  The device name and power limit
are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def one(tree, calls, forwards):
    """-> {arm: microseconds per call} of this process, with tree's odise_b200"""
    sys.path.insert(0, tree)
    import torch
    from odise_b200 import lib, masked_attn, msda, spec  # noqa: F401  (importing them defines the ops)
    from odise_b200.head import HeadEngine
    from odise_b200.postprocess import PostProcessor
    assert os.path.dirname(os.path.abspath(lib.__file__)) == os.path.join(os.path.abspath(tree), "odise_b200")
    dev = torch.device("cuda:0")
    ops = torch.ops.odise_b200
    # MSDA: N = 1, Lq = 1, one 2x2 level, 8 heads of D = 32, 4 points; masked cross-attention: Q = S = B = 1, one head
    fused = (torch.randn(1, 4, 8, 32, device=dev), torch.tensor([[2, 2]], device=dev),
             torch.zeros(1, dtype=torch.long, device=dev), torch.rand(1, 1, 1, 2, device=dev),
             torch.randn(1, 1, 8, 1, 4, 2, device=dev), torch.randn(1, 1, 8, 4, device=dev))
    grad = torch.randn(1, 1, 256, device=dev)
    q = torch.randn(1, 1, 32, device=dev)
    g = torch.Generator().manual_seed(0)
    head = HeadEngine(spec.synth_state_dict(spec.head_params(), seed=1), dev, nmma=3)
    feats = {f"s{i}": (torch.randn((128 >> i) ** 2, 512, generator=g).to(dev), 128 >> i, 128 >> i) for i in (2, 3, 4, 5)}
    post = PostProcessor(dev, 133, range(0, 133, 2))
    logits, masks = torch.randn(1, 100, 134, generator=g).to(dev), torch.randn(1, 100, 32, 32, generator=g).to(dev)
    # arm -> (call, calls per timing, synchronise after every call)
    arms = {
        "msda_fused_forward": (lambda: ops.msda_fused_forward(*fused), calls, False),
        "lib.msda_fused_forward": (lambda: lib.msda_fused_forward(*fused), calls, False),
        "msda_fused_backward": (lambda: ops.msda_fused_backward(*fused, grad, False), calls, False),
        "msda_fused_backward_det": (lambda: ops.msda_fused_backward(*fused, grad, True), calls, False),
        "masked_xattn_forward": (lambda: ops.masked_xattn_forward(q, q, q, None, 1), calls, False),
        "HeadEngine.forward": (lambda: head.forward(feats, 1), forwards, True),
        "PostProcessor": (lambda: post(logits, masks, 128, 128, instance=True), forwards, True),
    }
    res = {}
    for _ in range(2):          # the first pass warms up; the second one's times are kept
        for name, (fn, n, sync_each) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n):
                fn()
                if sync_each:
                    torch.cuda.synchronize()
            torch.cuda.synchronize()
            res[name] = (time.perf_counter() - t0) / n * 1e6
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="+", default=[ROOT])
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--forwards", type=int, default=20)
    ap.add_argument("--one", help=argparse.SUPPRESS)      # the per-process measurement of one tree
    a = ap.parse_args()
    if a.one:
        print(json.dumps(one(a.one, a.calls, a.forwards)))
        return
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    us = {tree: {} for tree in a.trees}
    for r in range(a.rounds):
        for tree in a.trees[::-1] if r % 2 else a.trees:
            cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
                os.path.abspath(__file__), "--one", tree, "--calls", str(a.calls), "--forwards", str(a.forwards)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode:
                sys.exit(f"{tree}: {r.stderr[-4000:]}")
            for op, t in json.loads(r.stdout.splitlines()[-1]).items():
                us[tree].setdefault(op, []).append(t)
    print(json.dumps(dict(device=smi, rounds=a.rounds, calls=a.calls, forwards=a.forwards, us_per_call={
        tree: {op: dict(median=round(statistics.median(v), 2), min=round(min(v), 2), max=round(max(v), 2))
               for op, v in ops.items()} for tree, ops in us.items()})))


if __name__ == "__main__":
    main()
