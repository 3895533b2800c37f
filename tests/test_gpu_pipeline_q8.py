"""The assembled pipeline in the F16Q8 operand mode (ODISEEngine(nmma=2): VAE, CLIP image tower, UNet and projections on
fp16 hi x hi + e5m2 cross-term MMAs; head / post-processing bf16x3) against the same composed oracle and the same 1e-3 bars
as tests/test_gpu_pipeline.py — the test bodies are shared, only the engine differs."""
import pytest
import torch

import test_gpu_pipeline as P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def world_q8(cuda):
    from odise_b200 import spec
    from odise_b200.pipeline import ODISEEngine, full_param_list, synthetic_vocabulary
    sd = spec.synth_state_dict(full_param_list(with_vae=True, with_clip=True), seed=0)
    eng = ODISEEngine(sd, cuda, nmma=2, with_vae=True, with_clip=True, synthetic_uncond=True)
    assert eng.backbone.unet.lo == "q8" and eng.head.nmma == 3
    bank, null, sizes = synthetic_vocabulary(20, 31)
    clip_bank = torch.randn(31, 768, generator=torch.Generator().manual_seed(77))
    ov = [(k % 3) == 0 for k in range(20)]
    eng.set_vocabulary("v20", bank, null, sizes, thing_ids=list(range(0, 20, 2)), clip_text_bank=clip_bank, overlapping=ov)
    img = torch.randint(0, 256, (1, 3, 512, 512), generator=torch.Generator().manual_seed(5), dtype=torch.uint8)
    return dict(sd=sd, eng=eng, img=img, bank=bank, null=null, sizes=sizes, clip_bank=clip_bank, ov=ov)


def test_q8_backbone_end_to_end(cuda, world_q8):
    P.test_backbone_end_to_end(cuda, world_q8)


def test_q8_step_graph_and_clip_head(cuda, world_q8):
    """also covers CUDA-graph capture with the operand format switching between producers inside one step"""
    P.test_step_graph_and_clip_head(cuda, world_q8)


def test_q8_c1_end_to_end(cuda, world_q8, record):
    def rec(line):
        record("[F16Q8] " + line)
    P.test_c1_end_to_end_mask_logits_and_class_scores(cuda, world_q8, rec)


def test_q8_c1_end_to_end_portrait_576x448(cuda, world_q8, record):
    def rec(line):
        record("[F16Q8] " + line)
    P.test_c1_end_to_end_portrait_576x448(cuda, world_q8, rec)


def test_q8_full_size_batch4_1024_paste(cuda, world_q8, record):
    def rec(line):
        record("[F16Q8] " + line)
    P.test_full_size_batch4_1024_paste(cuda, world_q8, rec)


def test_q8_short_side_below_512(cuda, world_q8, record):
    """384^2 crops -> 48 x 48 latent: 24 / 12 / 6-pixel maps take the materialised-im2col and odd-width paths in F16Q8"""
    def rec(line):
        record("[F16Q8] " + line)
    P.test_short_side_below_512(cuda, world_q8, rec)
