"""End-to-end GPU parity of the assembled pipeline (odise_b200/pipeline.py::ODISEEngine) against the oracle pieces
composed the way the reference composes them:
  LdmImplicitCaptionerExtractor.forward (ldm.py:697-718) -> LdmExtractor.forward (ldm.py:543-613)
  -> FeatureExtractorBackbone.forward_features (feature_extractor.py:157-179), then the clip_head branch of
  CategoryODISE.forward (odise.py:292-323).  One 512^2 image = one crop, full-size SD-v1 / ViT-L/14-336 / KL-VAE."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


@pytest.fixture(scope="module")
def world(cuda):
    from odise_b200 import spec
    from odise_b200.pipeline import ODISEEngine, full_param_list, synthetic_vocabulary
    sd = spec.synth_state_dict(full_param_list(with_vae=True, with_clip=True), seed=0)
    eng = ODISEEngine(sd, cuda, nmma=3, with_vae=True, with_clip=True, synthetic_uncond=True)
    bank, null, sizes = synthetic_vocabulary(20, 31)
    clip_bank = torch.randn(31, 768, generator=torch.Generator().manual_seed(77))
    ov = [(k % 3) == 0 for k in range(20)]
    eng.set_vocabulary("v20", bank, null, sizes, thing_ids=list(range(0, 20, 2)), clip_text_bank=clip_bank, overlapping=ov)
    img = torch.randint(0, 256, (1, 3, 512, 512), generator=torch.Generator().manual_seed(5), dtype=torch.uint8)
    return dict(sd=sd, eng=eng, img=img, bank=bank, null=null, sizes=sizes, clip_bank=clip_bank, ov=ov)


@torch.no_grad()
def test_backbone_end_to_end(cuda, world):
    """uint8 image -> s2..s5 through VAE taps, CLIP image embedding, implicit captioner, UNet taps, projections."""
    from odise_b200 import spec
    from oracle import clip as oclip, ldm, m2f
    sd, eng, img = world["sd"], world["eng"], world["img"]
    got = eng.backbone.forward(1, 512, 512, images_u8=img.to(cuda))
    torch.cuda.synchronize()

    def load(cls, prefix):
        with torch.device("meta"):
            m = cls()
        m.load_state_dict({k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}, assign=True)
        return m.eval()
    unet, vae, vis = load(ldm.UNetModel, spec.UNET_PREFIX), load(ldm.AutoencoderKL, spec.VAE_PREFIX), load(oclip.VisionTransformer, spec.CLIP_PREFIX)
    img01 = img.float() / 255.0
    e = "backbone.feature_extractor."
    lin = torch.nn.functional.linear
    emb = oclip.embed_image(vis, img01)                                                        # ldm.py:705
    uncond = torch.randn(1, 77, 768, generator=torch.Generator().manual_seed(17))              # BackboneEngine default
    ctx = uncond + torch.tanh(sd[e + "alpha_cond"]) * (
        lin(emb, sd[e + "clip_project.linear.weight"], sd[e + "clip_project.linear.bias"]).unsqueeze(1)
        + sd[e + "clip_project.positional_embedding"])
    cemb = torch.tanh(sd[e + "alpha_cond_time_embed"]) * (
        lin(emb, sd[e + "time_embed_project.linear.weight"], sd[e + "time_embed_project.linear.bias"]).unsqueeze(1)
        + sd[e + "time_embed_project.positional_embedding"])
    lat, ef = ldm.encoder_features(vae, (img01 - 0.5) / 0.5)
    uf = ldm.unet_features(unet, ldm.q_sample_t0(lat, ldm.shared_noise()), ctx, cemb[:, 0])
    df = ldm.decoder_features(vae, lat)
    want = m2f.forward_features(sd, [*ef, *uf, *df], (512, 512))
    for k, w in want.items():
        t, h, ww = got[k]
        r = _rel(t.view(1, h, ww, 512).permute(0, 3, 1, 2).cpu(), w)
        assert r < 1e-3, (k, r)


@torch.no_grad()
def test_step_graph_and_clip_head(cuda, world):
    """eager step == CUDA-graph replay == infer(); the merged class scores equal the oracle's clip_head branch applied
    to the engine's own category logits / mask logits (the decoder's hard thresholds make a fully independent CPU
    run discontinuous: the decoder itself is covered teacher-forced in test_gpu_head.py)."""
    from odise_b200 import spec
    from oracle import clip as oclip
    sd, eng, img = world["sd"], world["eng"], world["img"]
    dimg = img.to(cuda)
    a = eng.step(1, 512, 512, images_u8=dimg)
    torch.cuda.synchronize()
    assert a["pred_logits"].shape == (1, 100, 21) and a["pred_masks"].shape == (1, 100, 128, 128)
    assert torch.isfinite(a["pred_logits"]).all()
    assert (a["pred_logits"].exp().sum(-1) - 1).abs().max() < 1e-3         # log-probabilities (+ 21e-8)
    ea = {k: a[k].clone() for k in ("pred_logits", "pred_masks", "pred_logits_category")}
    host = eng.infer(img.pin_memory())                                      # graph capture + replay, H2D/D2H inside
    assert torch.equal(host["pred_logits"], ea["pred_logits"].cpu())
    assert torch.equal(host["pred_masks"], ea["pred_masks"].cpu())
    with torch.device("meta"):
        vis = oclip.VisionTransformer()
    vis.load_state_dict({k[len(spec.CLIP_PREFIX):]: v for k, v in sd.items() if k.startswith(spec.CLIP_PREFIX)}, assign=True)
    cat, masks = ea["pred_logits_category"].cpu(), ea["pred_masks"].cpu()
    me = oclip.get_mask_embed(vis.eval(), img.float() / 255.0, masks)
    lg = oclip.maskclip_pred_logits(me, world["clip_bank"], world["sizes"], 100.0)
    want = oclip.merge_with_void(cat, oclip.pooling_clip_ensemble(cat[..., :-1], lg, torch.tensor(world["ov"]).long(), 0.3, 0.7))
    # a patch whose pooled mask value sits within rounding of the 0.5 threshold may flip one attention bit of one
    # query: require every query but (at most) two to match tightly
    err = (ea["pred_logits"].cpu() - want).abs().amax(-1)[0]
    assert (err < 3e-2).sum() >= 98, err
    # post-processing on the merged scores runs end to end
    post = eng.postprocess(a, 512, 512)
    assert post["sem_seg"].shape == (1, 20, 512, 512) and post["panoptic_seg"].shape == (1, 512, 512)


@torch.no_grad()
def test_maskclip_image_tokens_share_the_crop_pass(cuda, world):
    """step() sends MaskCLIP's image tokens through the CLIP tower together with the crops and keeps their keys / values;
    the mask tokens then run alone (nobody attends to them, clip.py:306).  Must equal the stand-alone MaskCLIP pass bit for
    bit (same rows, same k order), for a batch of 2 images x 4 crops."""
    eng = world["eng"]
    img = torch.randint(0, 256, (2, 3, 1024, 1024), generator=torch.Generator().manual_seed(6), dtype=torch.uint8).to(cuda)
    eng.use_vocabulary("v20")
    a = eng.step(2, 1024, 1024, images_u8=img)
    assert eng.clip_head.visual._kv is None                                   # consumed
    alone = eng.clip_head.visual.mask_embed(img, a["pred_masks"].contiguous(), 2, 1024, 1024)
    torch.cuda.synchronize()
    assert torch.equal(a["clip_mask_embed"], alone)


@torch.no_grad()
def test_vocabulary_from_tokens(cuda, world):
    """tokenised prompts -> CLIP text bank on the device -> category + MaskCLIP vocabularies (odise.py:1281-1288)."""
    from odise_b200 import spec
    from oracle import clip as oclip
    eng = world["eng"]
    tsd = spec.synth_state_dict(spec.clip_text_params(), seed=8)
    eng._sd_text, eng.text = tsd, None
    eng._null_embed = torch.randn(1, 768, generator=torch.Generator().manual_seed(3))
    g = torch.Generator().manual_seed(6)
    sizes = [2, 1, 1, 3]
    ids = torch.zeros(sum(sizes), 77, dtype=torch.int64)
    for i in range(ids.shape[0]):
        n = 3 + i
        ids[i, :n] = torch.randint(1000, 40000, (n,), generator=g)
        ids[i, 0], ids[i, n - 1] = 49406, 49407
    bank = eng.set_vocabulary_from_tokens("tok4", ids, sizes, thing_ids=[0, 2], overlapping=[1, 0, 0, 1])
    with torch.device("meta"):
        m = oclip.TextTransformer()
    m.load_state_dict({k[len(spec.CLIP_TEXT_PREFIX):]: v for k, v in tsd.items()}, assign=True)
    m.attn_mask = torch.empty(77, 77).fill_(float("-inf")).triu_(1)
    want, _ = oclip.encode_text(m.eval(), ids)
    assert _rel(bank.cpu(), want) < 1e-3
    out = eng.step(1, 512, 512, images_u8=world["img"].to(cuda))
    assert out["pred_logits"].shape == (1, 100, 5) and torch.isfinite(out["pred_logits"]).all()
    eng.set_vocabulary("v20", world["bank"], world["null"], world["sizes"], thing_ids=list(range(0, 20, 2)),
                       clip_text_bank=world["clip_bank"], overlapping=world["ov"])


@torch.no_grad()
def test_category_odise_plugin_ragged_batch(cuda, world):
    """B200CategoryODISE: two images of different, non-64-divisible sizes in one batch, outputs at the datasets' original
    sizes; checked against the oracle post-processing applied to the engine's own logits.  The batch pads to 512 x 640."""
    _plugin_ragged_batch(cuda, world, ((500, 620), (470, 640)), ((250, 310), (600, 817)), (512, 640))


@torch.no_grad()
def test_category_odise_plugin_ragged_batch_portrait(cuda, world):
    """the same with a portrait batch that pads to 576 x 448: s5 18 x 14 = 252 keys per image in the decoder's first
    cross-attention"""
    _plugin_ragged_batch(cuda, world, ((560, 430), (576, 400)), ((280, 215), (720, 500)), (576, 448))


def _plugin_ragged_batch(cuda, world, sizes, outs, padded):
    from odise_b200.plugin import B200CategoryODISE
    from oracle import postprocess as opp
    eng = world["eng"]
    g = torch.Generator().manual_seed(21)
    ims = [torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8) for h, w in sizes]
    req = [dict(image=im, height=h, width=w) for im, (h, w) in zip(ims, outs)]
    model = B200CategoryODISE(eng).eval()
    res = model(req)
    torch.cuda.synchronize()
    assert len(res) == 2
    for r, hw in zip(res, outs):
        assert r["sem_seg"].shape == (20, *hw) and r["panoptic_seg"][0].shape == hw
    # re-run the network part to get the raw outputs the plugin post-processed (the padded batch)
    ph, pw = padded
    mh, mw = max(h for h, _ in sizes), max(w for _, w in sizes)
    net = torch.zeros(2, 3, ph, pw, dtype=torch.uint8)
    for i, (h, w) in enumerate(sizes):
        net[i, :, :h, :w] = ims[i]
    out = eng.step(2, ph, pw, images_u8=net.to(cuda), clip_images=net[:, :, :mh, :mw].contiguous().to(cuda))
    things = list(range(0, 20, 2))
    for i, (r, rq) in enumerate(zip(res, req)):
        cls, masks = out["pred_logits"][i].cpu(), out["pred_masks"][i:i + 1].cpu()
        up = opp.sem_seg_postprocess(opp.upsample_masks(masks, padded)[0], ims[i].shape[-2:], rq["height"], rq["width"])
        sem = opp.semantic_inference(cls, up)
        assert ((r["sem_seg"].cpu().double() - sem.double()).abs().max() / sem.abs().max()).item() < 1e-3
        pan, info = opp.panoptic_inference(cls, up, 20, things)
        assert r["panoptic_seg"][1] == info
        assert (r["panoptic_seg"][0].cpu() == pan).float().mean().item() > 0.999
        ins = r["instances"]
        assert ins["pred_masks"].shape[1:] == (rq["height"], rq["width"]) and ins["scores"].numel() == ins["pred_classes"].numel()


# ------------------------------------------------------------------------------------------------ round-2 parity closure
def _nchw(t, h, w):
    return t.view(-1, h, w, 512).permute(0, 3, 1, 2).cpu()


UNCOND17 = lambda: torch.randn(1, 77, 768, generator=torch.Generator().manual_seed(17))      # synthetic_uncond=True


@torch.no_grad()
def test_c1_end_to_end_mask_logits_and_class_scores(cuda, world, record):
    """BASELINE.json configs[0] / BASELINE.md §4 as stated: ONE 512 x 512 image, Q = 100, 20-class vocabulary; FINAL mask
    logits and FINAL class scores of the whole pipeline vs the composed oracle within 1e-3 (max |a-b| / max |b|, one global
    norm per tensor).  The three hard thresholds of the path (attention mask sigmoid < 0.5, odise.py:772; MaskPooling mask > 0,
    odise.py:951; MaskCLIP patch mask >= 0.5, clip.py:291-321) are teacher-forced with the ORACLE's mask logits — everything
    continuous is computed independently by both sides from the uint8 image — and the un-forced decisions are compared
    separately as a bit-flip rate."""
    _end_to_end(cuda, world, record, world["img"], "512^2")


@torch.no_grad()
def test_c1_end_to_end_portrait_576x448(cuda, world, record):
    """The C1 comparison (same oracle, same three 1e-3 bars, same flip bound) on a 576 x 448 portrait image: two vertically
    stacked, overlapping 448^2 crops; s5 18 x 14 = 252 keys, not a multiple of 8, in the decoder's first cross-attention;
    MaskCLIP masks of 144 x 112."""
    from odise_b200.backbone import BackboneEngine
    assert BackboneEngine.crop_grid(576, 448) == ([(0, 0), (128, 0)], 448)
    img = torch.randint(0, 256, (1, 3, 576, 448), generator=torch.Generator().manual_seed(82), dtype=torch.uint8)
    _end_to_end(cuda, world, record, img, "576 x 448")


def _end_to_end(cuda, world, record, img, label):
    from oracle import clip as oclip, compose, m2f
    sd, eng = world["sd"], world["eng"]
    H, W = img.shape[-2:]
    mods = compose.load_modules(sd)
    img01 = img.float() / 255.0
    feats = compose.slide_forward(sd, mods, img01, UNCOND17())
    mf, _, ms = m2f.pixel_decoder(sd, feats, "sem_seg_head.pixel_decoder.")
    ref, ref_masks = m2f.transformer_decoder(sd, ms, mf, "sem_seg_head.predictor.")
    te, ne = m2f.category_embed(sd, world["bank"], world["null"])
    cat_ref = m2f.cal_pred_logits(ref["mask_embed"], te, ne, ref["logit_scale"], world["sizes"])
    me = oclip.get_mask_embed(mods["vis"], img01, ref["pred_masks"])
    lg = oclip.maskclip_pred_logits(me, world["clip_bank"], world["sizes"], 100.0)
    want_cls = oclip.merge_with_void(cat_ref, oclip.pooling_clip_ensemble(cat_ref[..., :-1], lg, torch.tensor(world["ov"]).long(), 0.3, 0.7))
    # engine, thresholds forced to the oracle's decisions
    dimg = img.to(cuda)
    eng.use_vocabulary("v20")
    f_e = eng.backbone.forward(1, H, W, images_u8=dimg)
    pd = eng.head.pixel_decoder(f_e, 1)
    forced = [m.reshape(1, 100, -1).contiguous().to(cuda) for m in ref_masks]
    heads = eng.head.transformer_decoder(pd, 1, forced_masks=forced)
    cat = eng.head.score(heads[-1]["mask_embed"], "v20").view(1, 100, -1)
    got = eng.clip_head.forward("v20", dimg, 1, H, W, ref["pred_masks"].to(cuda).contiguous(), cat)
    torch.cuda.synchronize()
    assert ref["pred_masks"].shape[-2:] == (H // 4, W // 4)
    e_mask = _rel(heads[-1]["pred_masks"].view_as(ref["pred_masks"]).cpu(), ref["pred_masks"])
    e_cat = _rel(cat.cpu(), cat_ref)
    e_cls = _rel(got["pred_logits"].cpu(), want_cls)
    # un-forced run: how many discrete decisions differ (reported, bounded loosely: they are discontinuities, not errors)
    out = eng.step(1, H, W, images_u8=dimg)
    flips = [((h["pred_masks"].view_as(r).cpu() > 0) != (r > 0)).float().mean().item()
             for h, r in zip(out["aux"] + [dict(pred_masks=out["pred_masks"])], ref_masks)]
    record(f"C1 end to end ({label}, Q=100, 20 classes): final mask logits rel {e_mask:.2e}, category scores rel {e_cat:.2e}, "
           f"merged class scores rel {e_cls:.2e}; un-forced sign flips per head {['%.1e' % f for f in flips]}")
    # oracle (compose + m2f + MaskCLIP), 1e-3 relative on each of the three outputs
    assert e_mask < 1e-3 and e_cat < 1e-3 and e_cls < 1e-3, (e_mask, e_cat, e_cls)
    assert max(flips) < 1e-2


@torch.no_grad()
def test_full_size_batch4_1024_paste(cuda, world, record):
    """B = 4 x 1024^2 (BASELINE.json configs[1] shape): the real 4-crop paste with real VAE / CLIP / UNet taps.  The
    oracle runs ONE of the four images (4 crops on the host cores); the other three are checked against the engine's own
    single-image result (batch composition must not change an image's features)."""
    from oracle import compose
    sd, eng = world["sd"], world["eng"]
    g = torch.Generator().manual_seed(77)
    imgs = torch.randint(0, 256, (4, 3, 1024, 1024), generator=g, dtype=torch.uint8)
    got = eng.backbone.forward(4, 1024, 1024, images_u8=imgs.to(cuda))
    torch.cuda.synchronize()
    got = {k: _nchw(t, h, w) for k, (t, h, w) in got.items()}
    want = compose.slide_forward(sd, compose.load_modules(sd), imgs[2:3].float() / 255.0, UNCOND17())
    record("B=4 x 1024^2 backbone vs oracle (image 2): " + ", ".join(f"{k} {_rel(got[k][2:3], w_):.2e}" for k, w_ in want.items()))
    for k, w_ in want.items():
        assert got[k].shape == (4, 512, 1024 // 2 ** int(k[1]), 1024 // 2 ** int(k[1]))
        assert _rel(got[k][2:3], w_) < 1e-3, (k, _rel(got[k][2:3], w_))
    one = eng.backbone.forward(1, 1024, 1024, images_u8=imgs[1:2].to(cuda))
    torch.cuda.synchronize()
    for k, (t, h, w) in one.items():           # same arithmetic up to the tile / split-K choices that depend on the batch rows
        assert _rel(got[k][1:2], _nchw(t, h, w)) < 1e-4, k


@torch.no_grad()
def test_1280_nine_overlapping_crops(cuda, world, record):
    """1280 x 1280 (BASELINE.json configs[4]): 3 x 3 crops of 512 with stride 512 clamped to the border -> overlaps of 256
    pixels, paste-add + count + divide (feature_extractor.py:197-250)."""
    from odise_b200.backbone import BackboneEngine
    from oracle import compose
    sd, eng = world["sd"], world["eng"]
    boxes, short = BackboneEngine.crop_grid(1280, 1280)
    assert short == 512 and boxes == [(y, x) for y in (0, 512, 768) for x in (0, 512, 768)]
    img = torch.randint(0, 256, (1, 3, 1280, 1280), generator=torch.Generator().manual_seed(78), dtype=torch.uint8)
    got = eng.backbone.forward(1, 1280, 1280, images_u8=img.to(cuda))
    torch.cuda.synchronize()
    want = compose.slide_forward(sd, compose.load_modules(sd), img.float() / 255.0, UNCOND17())
    record("1280^2, 9 overlapping crops, backbone vs oracle: " + ", ".join(
        f"{k} {_rel(_nchw(*got[k]), w_):.2e}" for k, w_ in want.items()))
    for k, w_ in want.items():
        t, h, w = got[k]
        assert _rel(_nchw(t, h, w), w_) < 1e-3, (k, _rel(_nchw(t, h, w), w_))


@torch.no_grad()
def test_short_side_below_512(cuda, world, record):
    """A 384 x 640 image: two overlapping 384^2 crops, each bicubic-resized to 512^2 before the extractor
    (single_forward's T.Resize, feature_extractor.py:73-76,144) and brought back by the nearest resize of forward_features;
    then the whole engine runs on it (round 1 raised here)."""
    from oracle import compose
    sd, eng = world["sd"], world["eng"]
    img = torch.randint(0, 256, (1, 3, 384, 640), generator=torch.Generator().manual_seed(79), dtype=torch.uint8)
    got = eng.backbone.forward(1, 384, 640, images_u8=img.to(cuda))
    torch.cuda.synchronize()
    want = compose.slide_forward(sd, compose.load_modules(sd), img.float() / 255.0, UNCOND17())
    record("384 x 640 (two 384^2 crops resized to 512^2), backbone vs oracle: " + ", ".join(
        f"{k} {_rel(_nchw(*got[k]), w_):.2e}" for k, w_ in want.items()))
    for k, w_ in want.items():
        t, h, w = got[k]
        assert (h, w) == tuple(w_.shape[-2:]) and _rel(_nchw(t, h, w), w_) < 1e-3, (k, _rel(_nchw(t, h, w), w_))
    eng.use_vocabulary("v20")
    out = eng.step_full(1, 384, 640, images_u8=img.to(cuda))
    assert out["pred_masks"].shape == (1, 100, 96, 160) and out["post"]["panoptic_seg"].shape == (1, 384, 640)
    assert torch.isfinite(out["pred_logits"]).all()


@torch.no_grad()
def test_latent_other_than_64(cuda, world):
    """LdmExtractor at a latent that is not 64 x 64 (ldm.py:583-592: the shared noise is bicubic-resized): a 384^2 crop
    WITHOUT the backbone's resize -> 48 x 48 latent, UNet levels 48 / 24 / 12 / 6 (the last two take the materialised
    im2col path: their widths cannot be tiled by the implicit-GEMM TMA boxes)."""
    from odise_b200 import spec
    from oracle import ldm
    eng = world["eng"]
    sd = world["sd"]
    with torch.device("meta"):
        unet = ldm.UNetModel()
    unet.load_state_dict({k[len(spec.UNET_PREFIX):]: v for k, v in sd.items() if k.startswith(spec.UNET_PREFIX)}, assign=True)
    g = torch.Generator().manual_seed(80)
    lat, ctx, cemb = torch.randn(1, 4, 48, 48, generator=g), torch.randn(1, 77, 768, generator=g), torch.randn(1, 1280, generator=g) * 0.5
    want = ldm.unet_features(unet.eval(), ldm.q_sample_t0(lat, ldm.shared_noise((48, 48))), ctx, cemb)
    bb = eng.backbone
    x = bb.q_sample(lat.permute(0, 2, 3, 1).reshape(-1, 4).contiguous().to(cuda), 1, 48, 48)
    taps = bb.unet.forward(x, 1, 48, 48, ctx.view(77, 768).to(cuda), cemb.to(cuda))
    torch.cuda.synchronize()
    for (t, h, w), r in zip(taps, want):
        assert _rel(t.view(1, h, w, -1).permute(0, 3, 1, 2).cpu(), r) < 1e-3


@torch.no_grad()
def test_ade847_vocabulary_scoring(cuda, world):
    """K = 847 classes / K' = 1342 prompts (BASELINE.json configs[4]): cal_pred_logits + per-class max at full size."""
    from odise_b200.pipeline import synthetic_vocabulary
    from oracle import m2f
    sd, eng = world["sd"], world["eng"]
    bank, null, sizes = synthetic_vocabulary(847, 1342)
    eng.head.set_vocabulary("ade847", bank, null, sizes)
    me = torch.randn(400, 256, generator=torch.Generator().manual_seed(81))
    te, ne = m2f.category_embed(sd, bank, null)
    want = m2f.cal_pred_logits(me.view(4, 100, 256), te, ne, torch.tensor(eng.head.logit_scale), sizes)
    got = eng.head.score(me.to(cuda), "ade847").view(4, 100, -1).cpu()
    assert got.shape == (4, 100, 848) and _rel(got, want) < 1e-3
