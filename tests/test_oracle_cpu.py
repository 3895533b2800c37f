"""CPU tests that PIN the oracle (oracle/) against the reference's own code and check the parameter inventory of
odise_b200/spec.py.  The reference side runs live where the reference tree is present; elsewhere what it computed is read
from tests/golden/ref_pinned*.pt (oracle.refshim.pinned)."""
import os
import types

import torch

from odise_b200 import spec
from oracle import ldm as oldm
from oracle import cases, m2f, refshim


def _same(a, b):
    """Bit equality where the reference runs in this process.  Against stored reference results the CPU kernels of another
    machine may sum in another order: fp32 rounding level, max |a - b| <= 1e-5 max |b| (~1.5e-6 seen between hosts)."""
    if refshim.available():
        return torch.equal(a, b)
    return a.shape == b.shape and bool((a - b).abs().max() <= 1e-5 * b.abs().max())


def _shapes(params, prefix):
    return {n[len(prefix):]: tuple(s) for n, s, _ in params}


def test_unet_and_vae_inventory_matches_oracle_modules():
    with torch.device("meta"):
        unet, vae = oldm.UNetModel(), oldm.AutoencoderKL()
    assert _shapes(spec.unet_params(), spec.UNET_PREFIX) == {k: tuple(v.shape) for k, v in unet.state_dict().items()}
    assert _shapes(spec.vae_params(), spec.VAE_PREFIX) == {k: tuple(v.shape) for k, v in vae.state_dict().items()}
    n = sum(torch.Size(s).numel() for _, s, _ in spec.unet_params())
    assert n == 859_520_964          # the published SD-v1 UNet parameter count
    assert sum(torch.Size(s).numel() for _, s, _ in spec.vae_params()) == 83_653_863


def test_tap_table():
    """reset_dim_stride expectations of the reference (ldm.py:284-346): tap channels / strides."""
    inp, mid, out = spec.unet_blocks()
    assert [out[i][0][1] for i in (2, 5, 8, 11)] == [2560, 1920, 960, 640]
    assert spec.FEATURE_DIMS == (512, 512, 2560, 1920, 960, 640, 512, 512)


def _head_sd(seed=0):
    return spec.synth_state_dict(spec.head_params(), seed)


def test_head_inventory_matches_reference_modules():
    def ref():
        pd, dec = _ref_head(refshim.modules())
        return {**{"sem_seg_head.pixel_decoder." + k: tuple(v.shape) for k, v in pd.state_dict().items()},
                **{"sem_seg_head.predictor." + k: tuple(v.shape) for k, v in dec.state_dict().items()}}
    want = refshim.pinned("head_inventory", ref)
    got = {n: tuple(s) for n, s, _ in spec.pixel_decoder_params() + spec.decoder_params()}
    assert got == want


def _ref_head(m):
    S = m.ShapeSpec
    shape = {f"s{i}": S(channels=512, stride=2 ** i) for i in (2, 3, 4, 5)}
    pd = m.MSDeformAttnPixelDecoder(shape, transformer_dropout=0.0, transformer_nheads=8,
                                    transformer_dim_feedforward=1024, transformer_enc_layers=6, conv_dim=256,
                                    mask_dim=256, norm="GN", transformer_in_features=["s3", "s4", "s5"],
                                    common_stride=4).eval()
    dec = m.ODISEMultiScaleMaskedTransformerDecoder(
        class_embed=m.PseudoClassEmbed(133), post_mask_embed=m.PooledMaskEmbed(256, 256, 256), in_channels=256,
        mask_classification=True, num_classes=133, hidden_dim=256, num_queries=100, nheads=8, dim_feedforward=2048,
        dec_layers=9, pre_norm=False, enforce_input_project=False, mask_dim=256).eval()
    return pd, dec


def _strip(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


@torch.no_grad()
def test_head_oracle_equals_reference():
    """The reference's MSDeformAttnPixelDecoder / ODISE decoder (every head) / cal_pred_logits with the same weights on 2
    images of 128x128 input features.  Both decoders read the oracle's pixel-decoder outputs, so the decoder comparison is
    isolated from the pixel decoder's.  Stored reference results (no reference tree) are seeded samples of each tensor."""
    sd = _head_sd(1)
    g = torch.Generator().manual_seed(5)
    feats = {f"s{i}": torch.randn(2, 512, 128 // 2 ** i, 128 // 2 ** i, generator=g) for i in (2, 3, 4, 5)}
    sizes = [1, 3, 2, 1, 4] * 4
    te = torch.randn(sum(sizes), 256, generator=g)
    ne = torch.randn(1, 256, generator=g)
    me = torch.randn(2, 100, 256, generator=g)
    mf_o, t_o, ms_o = m2f.pixel_decoder(sd, feats, "sem_seg_head.pixel_decoder.")

    def ref():
        m = refshim.modules()
        pd, dec = _ref_head(m)
        pd.load_state_dict(_strip(sd, "sem_seg_head.pixel_decoder."))
        dec.load_state_dict(_strip(sd, "sem_seg_head.predictor."))
        mf_r, _, ms_r = pd.forward_features(feats)
        out_r = dec(ms_o, mf_o)
        # scoring: CategoryODISE.cal_pred_logits on the reference class itself
        logits = m.CategoryODISE.cal_pred_logits(None, dict(mask_embed=me, text_embed=te, null_embed=ne,
                                                            labels=[["x"] * n for n in sizes],
                                                            logit_scale=out_r["logit_scale"]))
        return dict(mask_features=mf_r, multi_scale=list(ms_r), logit_scale=out_r["logit_scale"], pred_logits=logits,
                    aux_pred_masks=[a["pred_masks"] for a in out_r["aux_outputs"]],
                    **{k: out_r[k] for k in ("pred_masks", "mask_embed", "mask_pooled_features")})

    def store(r):
        return {k: ([refshim.sample(t) for t in v] if isinstance(v, list) else
                    v.detach().clone() if v.numel() == 1 else refshim.sample(v)) for k, v in r.items()}
    r = refshim.pinned("head", ref, "ref_pinned_head.pt", store)

    def close(got, want, rtol, atol):
        a, b = refshim.at_sample(got, want)
        return torch.allclose(a, b, rtol=rtol, atol=atol)
    assert close(mf_o, r["mask_features"], 1e-4, 1e-5)
    assert len(ms_o) == len(r["multi_scale"]) == 3
    for a, b in zip(ms_o, r["multi_scale"]):
        assert close(a, b, 1e-4, 1e-5)
    out_o, _ = m2f.transformer_decoder(sd, ms_o, mf_o, "sem_seg_head.predictor.")
    for k in ("pred_masks", "mask_embed", "mask_pooled_features"):
        assert close(out_o[k], r[k], 1e-3, 1e-4), k
    assert torch.equal(out_o["logit_scale"], r["logit_scale"])
    assert len(out_o["aux_outputs"]) == len(r["aux_pred_masks"]) == 9
    for a, b in zip(out_o["aux_outputs"], r["aux_pred_masks"]):
        assert close(a["pred_masks"], b, 1e-3, 1e-4)
    mine = m2f.cal_pred_logits(me, te, ne, r["logit_scale"], sizes)
    assert close(mine, r["pred_logits"], 1e-5, 1e-5)


@torch.no_grad()
def test_position_embedding_and_msdeformattn_equal_reference():
    x = torch.zeros(2, 256, 7, 9)
    ref = refshim.pinned("position_embedding_sine", lambda: refshim.modules().PositionEmbeddingSine(128, normalize=True)(x))
    assert torch.allclose(m2f.position_embedding_sine(2, 7, 9), ref, atol=1e-6)


@torch.no_grad()
def test_reference_ldm_driver_runs_on_oracle_unet():
    """The reference's LdmExtractor.unet_forward / encoder_forward / decoder_forward (ldm.py:424-533) executed
    VERBATIM on the oracle modules == oracle.ldm.unet_features / encoder_features / decoder_features.  The case is
    oracle/cases.py::ldm_case, whose reference outputs tools/make_golden_ref.py stores in tests/golden/ref_ldm_driver.pt."""
    import importlib
    d = cases.ldm_case()
    unet, vae = d["unet"], d["vae"]

    def ref():
        refshim.install()
        rl = importlib.import_module("odise.modeling.meta_arch.ldm")
        rl.timestep_embedding = oldm.timestep_embedding
        rl.DiagonalGaussianDistribution = oldm.DiagonalGaussianDistribution
        fu = types.SimpleNamespace(ldm=types.SimpleNamespace(unet=unet),
                                   unet_blocks=[unet.output_blocks[i] for i in oldm.UNET_TAP_BLOCKS])
        _, ref_feats = rl.LdmExtractor.unet_forward(fu, d["x"], torch.zeros(2, dtype=torch.long), d["ctx"],
                                                    cond_emb=d["cond"].clone())
        enc_blocks = [vae.encoder.down[i].block[j] for i in range(4) for j in range(2)]
        dec_blocks = [vae.decoder.up[i].block[j] for i in reversed(range(4)) for j in range(3)]
        fv = types.SimpleNamespace(
            ldm=types.SimpleNamespace(encoder=vae.encoder, decoder=vae.decoder,
                                      ldm=types.SimpleNamespace(first_stage_model=vae, scale_factor=oldm.SCALE_FACTOR)),
            encoder_blocks=[enc_blocks[i] for i in oldm.ENC_TAP_BLOCKS],
            decoder_blocks=[dec_blocks[i] for i in oldm.DEC_TAP_BLOCKS])
        fv.encoder_forward = lambda im: rl.LdmExtractor.encoder_forward(fv, im)
        fv.decoder_forward = lambda z: rl.LdmExtractor.decoder_forward(fv, z)
        lat_r, ef_r = rl.LdmExtractor.encode_to_latent(fv, d["img"])
        _, df_r = rl.LdmExtractor.decode_to_image(fv, lat_r)
        c = lambda t: t.detach().clone().to(torch.float32)
        return dict(unet_feats=[c(t) for t in ref_feats], latent=c(lat_r), enc_feats=[c(t) for t in ef_r],
                    dec_feats=[c(t) for t in df_r])
    r = refshim.pinned(None, ref, "ref_ldm_driver.pt")
    mine = oldm.unet_features(unet, d["x"], d["ctx"], d["cond"])
    assert len(mine) == len(r["unet_feats"]) == 4
    for a, b in zip(mine, r["unet_feats"]):
        assert _same(a, b)
    lat_o, ef_o = oldm.encoder_features(vae, d["img"])
    assert _same(lat_o, r["latent"]) and len(ef_o) == len(r["enc_feats"])
    assert all(_same(a, b) for a, b in zip(ef_o, r["enc_feats"]))
    df_o = oldm.decoder_features(vae, lat_o)
    assert len(r["dec_feats"]) == 2 and all(_same(a, b) for a, b in zip(df_o, r["dec_feats"]))


def test_q_sample_constants():
    a, b = oldm.SQRT_ALPHA_BAR_0, oldm.SQRT_ONE_MINUS_ALPHA_BAR_0
    assert abs(a - 0.999575) < 1e-6 and abs(b - 0.029155) < 1e-6   # SURVEY.md §8a row a6
    n = oldm.shared_noise()
    assert n.shape == (1, 4, 64, 64)


@torch.no_grad()
def test_postprocess_oracle_equals_reference_methods():
    """oracle/postprocess.py vs the reference's MaskFormer.semantic_inference / panoptic_inference
    (maskformer_model.py:280-342) called on a fake self through the shim."""
    import importlib
    from oracle import postprocess as opp
    g = torch.Generator().manual_seed(4)
    Q, K, H, W = 30, 9, 40, 56
    cls = torch.randn(Q, K + 1, generator=g) * 3
    cls[:, -1] -= 2
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    pred = torch.stack([(6 + 10 * torch.rand(1, generator=g) - ((yy - torch.rand(1, generator=g) * H) ** 2 +
                                                               (xx - torch.rand(1, generator=g) * W) ** 2).sqrt()) * 2
                        for _ in range(Q)])
    things = [0, 2, 4]
    fake = types.SimpleNamespace(sem_seg_head=types.SimpleNamespace(num_classes=K), object_mask_threshold=0.0,
                                 overlap_threshold=0.8, num_queries=Q, test_topk_per_image=10, panoptic_on=True,
                                 metadata=types.SimpleNamespace(thing_dataset_id_to_contiguous_id={i: t for i, t in enumerate(things)}))

    def ref():
        refshim.install()
        MF = importlib.import_module("mask2former.maskformer_model").MaskFormer
        return (MF.semantic_inference(fake, cls, pred),) + tuple(MF.panoptic_inference(fake, cls, pred))
    sr, pr, ir = refshim.pinned("maskformer_inference", ref)
    assert torch.equal(sr, opp.semantic_inference(cls, pred))
    po, io = opp.panoptic_inference(cls, pred, K, things)
    assert torch.equal(pr, po) and ir == io and len(ir) > 0


def test_clip_inventory_matches_oracle_module():
    from oracle import clip as oclip
    with torch.device("meta"):
        v = oclip.VisionTransformer()
    got = {n[len(spec.CLIP_PREFIX):]: tuple(s) for n, s, _ in spec.clip_visual_params()}
    assert got == {k: tuple(t.shape) for k, t in v.state_dict().items()}
    assert 303e6 < sum(torch.Size(s).numel() for s in got.values()) < 305e6      # ViT-L/14-336 image tower


@torch.no_grad()
def test_reference_clip_glue_runs_on_oracle_visual():
    """ClipAdapter._encode_image (clip.py:177-222) executed verbatim on the oracle VisionTransformer == oracle.encode_image."""
    import importlib
    from oracle import clip as oclip
    torch.manual_seed(0)
    v = oclip.VisionTransformer(image_size=56, patch=14, width=64, layers=2, heads=4, out_dim=32).eval()
    for p in v.parameters():
        torch.nn.init.normal_(p, std=0.1)
    img = torch.randn(2, 3, 56, 56)
    fake = types.SimpleNamespace(clip=types.SimpleNamespace(visual=v))

    def ref():
        refshim.install()
        rc = importlib.import_module("odise.modeling.meta_arch.clip")
        import einops
        rc.rearrange = einops.rearrange
        return rc.ClipAdapter._encode_image(fake, img)[0]
    emb_ref = refshim.pinned("clip_encode_image", ref)
    assert torch.allclose(emb_ref, oclip.encode_image(v, img), rtol=1e-5, atol=1e-6)


@torch.no_grad()
def test_reference_maskclip_runs_on_oracle_visual():
    """MaskCLIP.get_mask_embed / pred_logits (clip.py:252-351) executed verbatim on the oracle VisionTransformer."""
    import importlib
    from oracle import clip as oclip
    torch.manual_seed(1)
    v = oclip.VisionTransformer(image_size=56, patch=14, width=128, layers=2, heads=2, out_dim=32).eval()
    for p in v.parameters():
        torch.nn.init.normal_(p, std=0.1)
    img = torch.rand(2, 3, 96, 96)
    masks = torch.randn(2, 5, 24, 24) * 3
    masks[0, 0] = -5.0                                         # a query whose mask touches no patch at all
    fake = types.SimpleNamespace(clip=types.SimpleNamespace(visual=v), image_size=(56, 56),
                                 clip_preprocess=lambda im: oclip.preprocess(im, 56), logit_scale=torch.tensor(37.0))
    text = torch.randn(7, 32)
    labels = [["a", "b"], ["c"], ["d", "e", "f"], ["g"]]

    def reference():
        refshim.install()
        rc = importlib.import_module("odise.modeling.meta_arch.clip")
        fake._mask_clip_forward = lambda *a: rc.MaskCLIP._mask_clip_forward(fake, *a)
        fake.encode_image_with_mask = lambda *a: rc.MaskCLIP.encode_image_with_mask(fake, *a)
        emb = rc.MaskCLIP.get_mask_embed(fake, img, masks)
        return emb, rc.MaskCLIP.pred_logits(fake, emb, text, labels)
    ref, lr = refshim.pinned("maskclip", reference)
    got = oclip.get_mask_embed(v, img, masks)
    assert ref.shape == (2, 5, 32) and torch.allclose(ref, got, rtol=1e-5, atol=1e-6)
    lo = oclip.maskclip_pred_logits(got, text, [len(l) for l in labels], fake.logit_scale)
    assert torch.allclose(lr, lo, rtol=1e-5, atol=1e-5)


@torch.no_grad()
def test_reference_pooling_clip_head_ensemble():
    """PoolingCLIPHead.forward (odise.py:1469-1542) run verbatim with a stubbed MaskCLIP == oracle ensemble."""
    from oracle import clip as oclip
    import importlib
    torch.manual_seed(2)
    test_labels = [["cat", "kitty"], ["unicorn"], ["dog"], ["spaceship", "rocket"]]
    train_labels = [["cat"], ["dog", "puppy"], ["tree"]]
    cat_logits, clip_logits = torch.randn(2, 6, 4) * 4, torch.randn(2, 6, 4) * 4
    fake = types.SimpleNamespace(training=False, test_labels=test_labels, train_labels=train_labels, prompt="photo",
                                 with_bg=False, bg_labels=None, alpha=0.3, beta=0.7, normalize_logits=True,
                                 get_and_cache_test_text_embed=lambda labels: None,
                                 clip=lambda im, m, t, l: {"mask_pred_open_logits": clip_logits})

    def ref():
        refshim.install()
        ro = importlib.import_module("odise.modeling.meta_arch.odise")
        return ro.PoolingCLIPHead.forward(fake, {"pred_open_logits": cat_logits.clone(), "images": torch.zeros(1),
                                                 "pred_masks": None})["pred_open_logits"]
    want = refshim.pinned("pooling_clip_head", ref)
    ov = torch.tensor([1, 0, 1, 0])
    got = oclip.pooling_clip_ensemble(cat_logits, clip_logits, ov, 0.3, 0.7)
    assert torch.allclose(want, got, rtol=1e-6, atol=1e-6)
    full = torch.randn(2, 6, 5)
    merged = oclip.merge_with_void(full, got)
    assert torch.allclose(merged.exp().sum(-1), torch.ones(2, 6) + 5e-8, atol=1e-5)


def test_clip_text_inventory_matches_oracle_module():
    from oracle import clip as oclip
    with torch.device("meta"):
        t = oclip.TextTransformer()
    got = {n[len(spec.CLIP_TEXT_PREFIX):]: tuple(s) for n, s, _ in spec.clip_text_params()}
    assert got == {k: tuple(v.shape) for k, v in t.state_dict().items()}
    # the SD-v1 cond_stage_model (HF names) maps onto the same module minus projection / logit_scale
    hf = spec.synth_state_dict(spec.sd_text_params(width=64, layers=2, vocab=100), 0)
    conv = spec.hf_text_to_openai(hf, dst_prefix="")
    small = oclip.TextTransformer(vocab=100, width=64, layers=2, heads=2, out_dim=64)
    missing = set(small.state_dict()) - set(conv)
    assert missing == {"text_projection", "logit_scale"} and not (set(conv) - set(small.state_dict()))


@torch.no_grad()
def test_reference_encode_text_runs_on_oracle_text_tower():
    """ClipAdapter._encode_text (clip.py:138-152) executed verbatim on the oracle TextTransformer == oracle.encode_text."""
    import importlib
    from oracle import clip as oclip
    torch.manual_seed(3)
    m = oclip.TextTransformer(vocab=50, ctx=9, width=64, layers=2, heads=2, out_dim=32).eval()
    for p in m.parameters():
        torch.nn.init.normal_(p, std=0.1)
    ids = torch.randint(1, 40, (3, 9))
    ids[0, 4], ids[1, 8], ids[2, 2] = 49, 49, 49                          # EOT = highest id
    fake = types.SimpleNamespace(clip=m)

    def ref():
        refshim.install()
        return importlib.import_module("odise.modeling.meta_arch.clip").ClipAdapter._encode_text(fake, ids)
    emb_ref, enc_ref = refshim.pinned("clip_encode_text", ref)
    emb, enc = oclip.encode_text(m, ids)
    assert torch.allclose(emb_ref, emb, rtol=1e-5, atol=1e-6) and torch.allclose(enc_ref, enc, rtol=1e-5, atol=1e-6)


def test_plugin_surface_matches_reference_modules():
    """SURVEY §8b B-1 / B-2: the B200* plugin classes take the constructor keywords the LazyConfigs pass
    (configs/common/models/odise_with_label.py:16-29, mask_generator_with_label.py:29-66) and expect exactly the state-dict
    keys of the reference modules they replace."""
    import inspect
    from odise_b200 import plugin
    bb_kw = {"feature_extractor", "out_features", "use_checkpoint", "slide_training"}
    fe_kw = {"encoder_block_indices", "unet_block_indices", "decoder_block_indices", "steps", "learnable_time_embed",
             "num_timesteps", "clip_model_name"}
    names = ("MSDeformAttnPixelDecoder", "ODISEMultiScaleMaskedTransformerDecoder", "PooledMaskEmbed", "PseudoClassEmbed")

    def ref():
        m = refshim.modules()
        pd, dec = _ref_head(m)
        keys = sorted({"pixel_decoder." + k for k in pd.state_dict()} | {"predictor." + k for k in dec.state_dict()})
        kws = {n: [p for c in getattr(m, n).__mro__ if c.__module__.startswith(("odise", "mask2former"))
                   for p in inspect.signature(c.__init__).parameters if p not in ("self", "kwargs", "args")] for n in names}
        # the config file's keyword sets, parsed from the file itself: only whether each keyword is passed is kept
        cfg = open(os.path.join(refshim.REF, "configs/common/models/odise_with_label.py")).read()
        return dict(keys=keys, kwargs=kws, cfg_passes={k: k + "=" in cfg for k in bb_kw | fe_kw})
    r = refshim.pinned("plugin_surface", ref)
    head = plugin.B200MaskFormerHead(num_classes=133, device="cpu")
    assert set(head.expected_keys()) == set(r["keys"])
    for n in names:
        mine = getattr(plugin, "B200" + n)
        mine_kw = set(inspect.signature(mine.__init__).parameters)
        assert set(r["kwargs"][n]) <= mine_kw, (mine.__name__, set(r["kwargs"][n]) - mine_kw)
    assert all(r["cfg_passes"][k] for k in bb_kw)
    assert bb_kw <= set(inspect.signature(plugin.B200FeatureExtractorBackbone.__init__).parameters)
    assert all(r["cfg_passes"][k] for k in fe_kw)
    assert fe_kw <= set(inspect.signature(plugin.B200LdmImplicitCaptionerExtractor.__init__).parameters)
    fe = plugin.B200LdmImplicitCaptionerExtractor(frozen_state_dict={}, device="cpu")
    bb = plugin.B200FeatureExtractorBackbone(fe, ["s2", "s3", "s4", "s5"], use_checkpoint=True, slide_training=True)
    got = set(bb.expected_keys())
    assert {k for k in got if k.startswith("feature_extractor.")} == {
        "feature_extractor." + k for k in ("clip_project.linear.weight", "clip_project.linear.bias",
                                           "clip_project.positional_embedding", "alpha_cond",
                                           "time_embed_project.linear.weight", "time_embed_project.linear.bias",
                                           "time_embed_project.positional_embedding", "alpha_cond_time_embed")}
    assert len([k for k in got if k.startswith("feature_projections.")]) == 8 * 9 + 4 * 3   # 4 of 8 blocks have a shortcut
