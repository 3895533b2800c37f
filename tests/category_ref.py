"""Inputs shared by the category-scoring tests: the COCO training bank's synonym groups and seeded score inputs."""
import os

import torch

from oracle import refshim


def coco_labels():
    """get_openseg_labels("coco_panoptic", prompt_engineered=True): 133 classes, 254 prompts, as pinned in
    tests/golden/ref_pinned.pt (tests/test_vocab_cpu.py checks that value against the reference's function).  Read from
    the fixture even where the reference is present: importing its odise.data package here would install stand-ins
    that later tests in the same process do not expect."""
    pinned = torch.load(os.path.join(refshim.GOLDEN, "ref_pinned.pt"), weights_only=True)
    return pinned["openseg_labels"]["labels"]["coco_panoptic"]


def inputs(B, Q, C, sizes, dtype=torch.float64, device="cpu", seed=0, scale=14.3):
    """(mask_embed [B, Q, C], text_embed [sum(sizes), C], null_embed [1, C], logit_scale) drawn from a seed"""
    g = torch.Generator().manual_seed(seed)
    me = torch.randn(B, Q, C, generator=g, dtype=torch.float64)
    te = torch.randn(sum(sizes), C, generator=g, dtype=torch.float64)
    ne = torch.randn(1, C, generator=g, dtype=torch.float64)
    return (me.to(device, dtype), te.to(device, dtype), ne.to(device, dtype),
            torch.tensor(scale, dtype=torch.float32 if dtype != torch.float64 else dtype, device=device))
