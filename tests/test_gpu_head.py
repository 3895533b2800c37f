"""GPU parity of the Mask2Former/ODISE head engine (odise_b200/head.py) against the CPU oracle (oracle/m2f.py, itself
pinned against the reference's code) with the same synthetic weights.  The decoder thresholds mask logits twice per
head (attention mask odise.py:772, hard pooling odise.py:951), so heads after the first are compared with the
oracle's mask logits teacher-forced on both sides (SURVEY.md §7 "Discontinuities"); the un-forced run is compared
on the first head exactly and on the final masks by agreement rate.

Every test runs at three input geometries (B = 2, different content per image, so image 1's keys sit at a per-image
stride): 256 x 256 (the `setup` fixture); and, through the *_non_square wrappers, 256 x 384 landscape (s5 8 x 12) and
576 x 448 portrait (s5 18 x 14 = 252 keys, not a multiple of 8: the decoder pads each image's keys to 256, and 2 x 252
rows is not a whole number of 32-row GroupNorm records, so the pixel decoder's s5 input GroupNorm takes the stand-alone
statistics pass)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GEOMETRIES = [(256, 256), (256, 384), (576, 448)]


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


_SETUPS = {}


def _setup(cuda, H, W):
    """engine, device features and the oracle's pixel decoder + decoder outputs at H x W (built once per geometry)"""
    if (H, W) in _SETUPS:
        return _SETUPS[H, W]
    from odise_b200 import spec
    from odise_b200.head import HeadEngine
    from oracle import m2f
    sd = spec.synth_state_dict(spec.head_params(), seed=1)
    B = 2
    g = torch.Generator().manual_seed(5)
    feats = {f"s{i}": torch.randn(B, 512, H // 2 ** i, W // 2 ** i, generator=g) for i in (2, 3, 4, 5)}
    eng = HeadEngine(sd, cuda, nmma=3)
    dfe = {k: (v.permute(0, 2, 3, 1).reshape(-1, 512).contiguous().to(cuda), v.shape[2], v.shape[3]) for k, v in feats.items()}
    with torch.no_grad():
        mf, _, ms = m2f.pixel_decoder(sd, feats, "sem_seg_head.pixel_decoder.")
        ref, ref_masks = m2f.transformer_decoder(sd, ms, mf, "sem_seg_head.predictor.")
    _SETUPS[H, W] = dict(sd=sd, eng=eng, dfe=dfe, B=B, hw=(H, W), mf=mf, ms=ms, ref=ref, ref_masks=ref_masks)
    return _SETUPS[H, W]


@pytest.fixture(scope="module")
def setup(cuda):
    return _setup(cuda, *GEOMETRIES[0])


NON_SQUARE = pytest.mark.parametrize("hw", GEOMETRIES[1:], ids=[f"{h}x{w}" for h, w in GEOMETRIES[1:]])


def test_pixel_decoder(cuda, setup):
    eng, dfe, B, mf, ms = setup["eng"], setup["dfe"], setup["B"], setup["mf"], setup["ms"]
    pd = eng.pixel_decoder(dfe, B, want_mask_features_f32=True)
    torch.cuda.synchronize()
    S = pd["geo"]["S"]
    mem = pd["memory"].view(B, S, 256).cpu()
    for lvl, (h, w) in enumerate(pd["shapes"]):
        st = pd["geo"]["starts"][lvl]
        got = mem[:, st:st + h * w].transpose(1, 2).reshape(B, 256, h, w)
        assert _rel(got, ms[lvl]) < 1e-3, (lvl, _rel(got, ms[lvl]))        # oracle encoder memory, 1e-3
    h2, w2 = pd["mask_hw"]
    got = pd["mf"].view(B, h2, w2, 256).permute(0, 3, 1, 2).cpu()
    assert _rel(got, mf) < 1e-3                                             # oracle mask features, 1e-3
    assert _rel(pd["mf_p"].float().view(B, h2 * w2, 256).cpu(), got.flatten(2).transpose(1, 2)) < 1e-4
    assert _rel(pd["mft_p"].float().view(256, B, h2 * w2).permute(1, 0, 2).cpu(), got.flatten(2)) < 1e-4


@NON_SQUARE
def test_pixel_decoder_non_square(cuda, hw):
    test_pixel_decoder(cuda, _setup(cuda, *hw))


def _check_teacher_forced(heads, refs, B):
    """every head's mask logits, mask embeddings and pooled features vs the oracle's, 1e-3 each; returns the worst"""
    worst = 0.0
    for i, (h, r) in enumerate(zip(heads, refs)):
        e1 = _rel(h["pred_masks"].view_as(r["pred_masks"]).cpu(), r["pred_masks"])
        e2 = _rel(h["mask_embed"].view_as(r["mask_embed"]).cpu(), r["mask_embed"])
        e3 = _rel(h["mask_pooled_features"].view_as(r["mask_pooled_features"]).cpu(), r["mask_pooled_features"])
        worst = max(worst, e1, e2, e3)
        assert max(e1, e2, e3) < 1e-3, (i, e1, e2, e3)
    return worst


def test_decoder_teacher_forced_and_scoring(cuda, setup, record):
    from oracle import m2f
    sd, eng, dfe, B, ref, ref_masks = (setup[k] for k in ("sd", "eng", "dfe", "B", "ref", "ref_masks"))
    pd = eng.pixel_decoder(dfe, B)
    forced = [m.reshape(B, 100, -1).contiguous().to(cuda) for m in ref_masks]
    heads = eng.transformer_decoder(pd, B, forced_masks=forced)
    torch.cuda.synchronize()
    worst = _check_teacher_forced(heads, ref["aux_outputs"] + [ref], B)
    record(f"head {setup['hw'][0]} x {setup['hw'][1]} (B = 2): decoder teacher-forced worst rel err {worst:.2e}")
    assert abs(eng.logit_scale - float(ref["logit_scale"])) < 1e-5
    # scoring (cal_pred_logits + per-class max + null column)
    g = torch.Generator().manual_seed(11)
    sizes = [1, 3, 2, 1, 4] * 4
    te, ne = torch.randn(sum(sizes), 768, generator=g), torch.randn(1, 768, generator=g)
    eng.set_vocabulary("t", te, ne, sizes)
    with torch.no_grad():
        tp, npj = m2f.category_embed(sd, te, ne)
        want = m2f.cal_pred_logits(ref["mask_embed"], tp, npj, ref["logit_scale"], sizes)
    got = eng.score(ref["mask_embed"].reshape(-1, 256).contiguous().to(cuda), "t").view(B, 100, -1).cpu()
    assert _rel(got, want) < 1e-3, _rel(got, want)


@NON_SQUARE
def test_decoder_teacher_forced_and_scoring_non_square(cuda, hw, record):
    test_decoder_teacher_forced_and_scoring(cuda, _setup(cuda, *hw), record)


def test_decoder_unforced_first_head_and_agreement(cuda, setup, record):
    eng, dfe, B, ref_masks = setup["eng"], setup["dfe"], setup["B"], setup["ref_masks"]
    out = eng.forward(dfe, B)
    torch.cuda.synchronize()
    h0 = out["heads"][0]
    assert _rel(h0["pred_masks"].view_as(ref_masks[0]).cpu(), ref_masks[0]) < 1e-3     # no threshold before head 0
    last = out["heads"][-1]["pred_masks"].view_as(ref_masks[-1]).cpu()
    agree = ((last > 0) == (ref_masks[-1] > 0)).float().mean().item()
    record(f"head {setup['hw'][0]} x {setup['hw'][1]} (B = 2): unforced final-mask sign agreement {agree:.5f}, "
           f"rel err {_rel(last, ref_masks[-1]):.2e}")
    assert agree > 0.99


@NON_SQUARE
def test_decoder_unforced_first_head_and_agreement_non_square(cuda, hw, record):
    test_decoder_unforced_first_head_and_agreement(cuda, _setup(cuda, *hw), record)


def test_decoder_from_plugin_tensors_portrait(cuda, record):
    """HeadEngine.pd_from_tensors (the decoder's NCHW inputs at the plugin boundary, odise.py:642-660) + transformer_decoder
    vs m2f.transformer_decoder on the same NCHW maps, teacher-forced, 1e-3 on every head.  Portrait 576 x 448: its s5
    level has 252 keys per image."""
    s = _setup(cuda, 576, 448)
    eng, B, ms, mf, ref, ref_masks = (s[k] for k in ("eng", "B", "ms", "mf", "ref", "ref_masks"))
    pd = eng.pd_from_tensors([t.to(cuda) for t in ms], mf.to(cuda))
    assert pd["shapes"][0] == (18, 14)
    forced = [m.reshape(B, 100, -1).contiguous().to(cuda) for m in ref_masks]
    heads = eng.transformer_decoder(pd, B, forced_masks=forced)
    torch.cuda.synchronize()
    worst = _check_teacher_forced(heads, ref["aux_outputs"] + [ref], B)
    record(f"head from plugin tensors 576 x 448 (B = 2): decoder teacher-forced worst rel err {worst:.2e}")
