"""The reference's plugin surface, backed by the H100 engines (SURVEY.md §8b B-1 / B-2 / B-3).

`B200FeatureExtractorBackbone` and `B200MaskFormerHead` keep the forward contracts of
odise.modeling.backbone.FeatureExtractorBackbone (feature_extractor.py:29-256) and
mask2former MaskFormerHead + ODISEMultiScaleMaskedTransformerDecoder (mask_former_head.py:115-132,
odise.py:713-727): NCHW tensors in, the same dict keys out — so a LazyConfig can point `model.backbone` /
`model.sem_seg_head` at them.  NCHW <-> NHWC conversion happens once at this boundary (odise_nchw_to_nhwc_f32).
detectron2 is not required: `output_shape()` returns lightweight ShapeSpec objects with .channels / .stride.
"""
from collections import OrderedDict, namedtuple

import torch
import torch.nn as nn

from . import ops, spec
from .backbone import BackboneEngine
from .head import HeadEngine

ShapeSpec = namedtuple("ShapeSpec", ["channels", "height", "width", "stride"])


def _expect(name, got, want):
    if tuple(got) != tuple(want) if isinstance(want, (tuple, list)) else got != want:
        raise NotImplementedError(f"{name}={got!r}: the engine implements the released ODISE configuration "
                                  f"({name}={want!r}, configs/common/models/odise_with_label.py)")


class B200LdmImplicitCaptionerExtractor(nn.Module):
    """Stands where LazyConfig puts `LdmImplicitCaptionerExtractor(...)` (odise_with_label.py:17-25, ldm.py:636-670,
    LdmExtractor kwargs ldm.py:225-236): same keyword arguments, plus the FROZEN weights the reference's constructor
    pulls from disk itself (LatentDiffusion(init_checkpoint=sd-v1-3.ckpt), open_clip ViT-L-14-336): here they are
    handed over as one state dict (`model.diffusion_model.*`, `first_stage_model.*`, `clip.visual.*`, and either
    `cond_stage_model.*` or an explicit `uncond_inputs` [1, 77, 768]) — see odise_b200.checkpoint.
    The learnable parameters (`clip_project.*`, `alpha_cond`, `time_embed_project.*`, `alpha_cond_time_embed`) arrive
    later through the backbone's load_state_dict, exactly as in the reference."""

    def __init__(self, learnable_time_embed=True, num_timesteps=1, clip_model_name="ViT-L-14-336", ldm=None,
                 encoder_block_indices=(5, 7), unet_block_indices=(2, 5, 8, 11), decoder_block_indices=(2, 5),
                 steps=(0,), share_noise=True, enable_resize=False, *, frozen_state_dict=None, uncond_inputs=None,
                 synthetic_uncond=False, device="cuda", nmma=3):
        super().__init__()
        _expect("encoder_block_indices", encoder_block_indices, (5, 7))
        _expect("unet_block_indices", unet_block_indices, (2, 5, 8, 11))
        _expect("decoder_block_indices", decoder_block_indices, (2, 5))
        _expect("steps", steps, (0,))
        _expect("share_noise", share_noise, True)
        _expect("enable_resize", enable_resize, False)
        _expect("learnable_time_embed", learnable_time_embed, True)
        _expect("num_timesteps", num_timesteps, 1)
        _expect("clip_model_name", clip_model_name, "ViT-L-14-336")
        if ldm is not None:
            raise NotImplementedError("ldm=<module>: pass the frozen weights as frozen_state_dict instead")
        self.frozen_state_dict = dict(frozen_state_dict) if frozen_state_dict is not None else None
        self.uncond_inputs, self.synthetic_uncond = uncond_inputs, synthetic_uncond
        self.device_, self.nmma = torch.device(device), nmma
        self.learnable_time_embed = learnable_time_embed

    # the attributes FeatureExtractorBackbone.__init__ reads (feature_extractor.py:53-99; values: ldm.py:330-346)
    feature_dims = tuple(spec.FEATURE_DIMS)
    feature_strides = tuple(spec.FEATURE_STRIDES)
    num_groups = 8                               # ldm.py:361-366: one group per tapped block

    @property
    def grouped_indices(self):
        return [[i] for i in range(8)]           # ldm.py:369-388 with steps = (0,)

    LEARNABLE = ("clip_project.linear.weight", "clip_project.linear.bias", "clip_project.positional_embedding",
                 "alpha_cond", "time_embed_project.linear.weight", "time_embed_project.linear.bias",
                 "time_embed_project.positional_embedding", "alpha_cond_time_embed")


class B200FeatureExtractorBackbone(nn.Module):
    """Drop-in for FeatureExtractorBackbone (feature_extractor.py:28-256) — same constructor keywords as
    configs/common/models/odise_with_label.py:16-29, same state-dict keys (`feature_projections.{i}.0.*`,
    `feature_extractor.{clip_project,alpha_cond,...}`), same forward contract:
    forward(img: [B, 3, H, W] in [0, 1], H, W % 64 == 0) -> {"s2".."s5": [B, 512, H/2^k, W/2^k]}.
    The engine is built when the learnable weights arrive (load_state_dict), from them + the extractor's frozen weights."""

    def __init__(self, feature_extractor, out_features, backbone_in_size=(512, 512), min_stride=4, max_stride=32,
                 projection_dim=512, num_res_blocks=1, use_checkpoint=False, slide_training=False):
        super().__init__()
        if not isinstance(feature_extractor, B200LdmImplicitCaptionerExtractor):
            raise TypeError("feature_extractor must be a B200LdmImplicitCaptionerExtractor")
        if isinstance(backbone_in_size, int):
            raise NotImplementedError("backbone_in_size=int (whole-image resize, no sliding window) is not the released "
                                      "configuration; pass (512, 512)")
        _expect("backbone_in_size", backbone_in_size, (512, 512))
        _expect("min_stride", min_stride, 4)
        _expect("max_stride", max_stride, 32)
        _expect("projection_dim", projection_dim, 512)
        _expect("num_res_blocks", num_res_blocks, 1)
        self.feature_extractor = feature_extractor
        self.use_checkpoint = use_checkpoint        # activation checkpointing: training only, no effect here
        self._slide_training, self._slide_inference = slide_training, True
        self.backbone_in_size = tuple(backbone_in_size)
        self._out_features = [n for n in ("s2", "s3", "s4", "s5") if n in out_features]
        self._out_feature_strides = {f"s{k}": 2 ** k for k in (2, 3, 4, 5)}
        self._out_feature_channels = {f"s{k}": projection_dim for k in (2, 3, 4, 5)}
        self.engine = None
        self._learnable = None

    @classmethod
    def from_state_dict(cls, state_dict, device, out_features=("s2", "s3", "s4", "s5"), nmma=3, uncond_inputs=None,
                        synthetic_uncond=False):
        """One dict with everything (frozen + learnable, keys prefixed `backbone.` as in an ODISE checkpoint)."""
        fe = B200LdmImplicitCaptionerExtractor(frozen_state_dict=state_dict, uncond_inputs=uncond_inputs,
                                               synthetic_uncond=synthetic_uncond, device=device, nmma=nmma)
        bb = cls(fe, list(out_features), slide_training=True)
        bb.load_state_dict({k[len("backbone."):]: v for k, v in state_dict.items() if k.startswith("backbone.")})
        return bb

    @staticmethod
    def expected_keys():
        keys = ["feature_extractor." + k for k in B200LdmImplicitCaptionerExtractor.LEARNABLE]
        for name, _, _ in spec.backbone_params(prefix="backbone."):
            if name.startswith("backbone.feature_projections."):
                keys.append(name[len("backbone."):])
        return keys

    def load_state_dict(self, state_dict, strict=True):
        """Reference keys (what FeatureExtractorBackbone.state_dict() minus ignored_state_dict() holds)."""
        want = self.expected_keys()
        missing = [k for k in want if k not in state_dict]
        unexpected = [k for k in state_dict if k not in set(want)]
        if strict and (missing or unexpected):
            raise RuntimeError(f"B200FeatureExtractorBackbone.load_state_dict: missing {missing[:5]} "
                               f"({len(missing)}), unexpected {unexpected[:5]} ({len(unexpected)})")
        fe = self.feature_extractor
        if fe.frozen_state_dict is None:
            raise RuntimeError("the feature extractor has no frozen weights (frozen_state_dict=...)")
        sd = dict(fe.frozen_state_dict)
        sd.update({"backbone." + k: v for k, v in state_dict.items()})
        vae = clip = None
        if any(k.startswith(spec.VAE_PREFIX) for k in sd):
            from .vae import VAEEngine
            vae = VAEEngine(sd, fe.device_, nmma=fe.nmma)
        if any(k.startswith(spec.CLIP_PREFIX) for k in sd):   # ClipAdapter image tower (clip.py:177-231)
            from .clip import ClipVisualEngine
            clip = ClipVisualEngine(sd, fe.device_, nmma=fe.nmma)
        self.engine = BackboneEngine(sd, fe.device_, nmma=fe.nmma, vae=vae, clip=clip, uncond=fe.uncond_inputs,
                                     synthetic_uncond=fe.synthetic_uncond)
        self._learnable = OrderedDict((k, state_dict[k].detach().cpu()) for k in want if k in state_dict)
        return missing, unexpected

    def state_dict(self, destination=None, prefix="", keep_vars=False):
        d = OrderedDict() if destination is None else destination
        for k, v in (self._learnable or {}).items():
            d[prefix + k] = v
        return d

    @property
    def size_divisibility(self):
        return 64                                # feature_extractor.py:126-128

    def output_shape(self):
        return {n: ShapeSpec(self._out_feature_channels[n], None, None, self._out_feature_strides[n])
                for n in self._out_features}

    def ignored_state_dict(self, destination=None, prefix=""):
        return OrderedDict() if destination is None else destination     # frozen SD / CLIP weights: nothing to save

    @torch.no_grad()
    def forward(self, img):
        if self.engine is None:
            raise RuntimeError("B200FeatureExtractorBackbone: load_state_dict() first (the engine is built from the weights)")
        if not img.is_cuda:
            raise RuntimeError("B200FeatureExtractorBackbone: CUDA tensor required (no CPU path)")
        B, _, H, W = img.shape
        if H % 64 or W % 64:
            raise RuntimeError("input must be padded to a multiple of size_divisibility=64")
        feats = self.engine.forward(B, H, W, images_u8=img.contiguous().float())
        return {k: ops.nhwc_to_nchw(t, B, h, w) for k, (t, h, w) in feats.items() if k in self._out_features}


class _HeadPart(nn.Module):
    """Shared plumbing of the two sub-modules of the head: both are views on ONE HeadEngine (owned by B200MaskFormerHead)."""

    def __init__(self):
        super().__init__()
        self._owner = None

    @property
    def engine(self):
        if self._owner is None or self._owner.engine is None:
            raise RuntimeError("load_state_dict() on the B200MaskFormerHead first (the engine is built from the weights)")
        return self._owner.engine


class B200MSDeformAttnPixelDecoder(_HeadPart):
    """MSDeformAttnPixelDecoder (msdeformattn.py:165-358) with the keyword arguments of
    configs/common/models/mask_generator_with_label.py:32-43; forward_features(features) ->
    (mask_features [B, 256, H/4, W/4], out[0] = encoder output of the coarsest level, multi_scale_features [s5, s4, s3])."""

    def __init__(self, input_shape=None, *, transformer_dropout=0.0, transformer_nheads=8, transformer_dim_feedforward=1024,
                 transformer_enc_layers=6, conv_dim=256, mask_dim=256, norm="GN",
                 transformer_in_features=("s3", "s4", "s5"), common_stride=4):
        super().__init__()
        _expect("transformer_nheads", transformer_nheads, 8)
        _expect("transformer_dim_feedforward", transformer_dim_feedforward, 1024)
        _expect("conv_dim", conv_dim, 256)
        _expect("mask_dim", mask_dim, 256)
        _expect("norm", norm, "GN")
        _expect("transformer_in_features", list(transformer_in_features), ["s3", "s4", "s5"])
        _expect("common_stride", common_stride, 4)
        self.transformer_enc_layers = transformer_enc_layers
        self.transformer_in_features = list(transformer_in_features)
        self.conv_dim, self.mask_dim, self.common_stride = conv_dim, mask_dim, common_stride
        self.maskformer_num_feature_levels = 3

    @torch.no_grad()
    def forward_features(self, features):
        eng = self.engine
        B = features["s2"].shape[0]
        feats = {k: (ops.nchw_to_nhwc(v.float()), v.shape[2], v.shape[3]) for k, v in features.items()}
        pd = eng.pixel_decoder(feats, B, want_mask_features_f32=True)
        h2, w2 = pd["mask_hw"]
        mask_features = ops.nhwc_to_nchw(pd["mf"], B, h2, w2)
        S, starts = pd["geo"]["S"], pd["geo"]["starts"]
        mem = pd["memory"].view(B, S, 256)
        ms = []
        for i, (h, w) in enumerate(pd["shapes"]):
            lvl = ops.empty(B * h * w, 256, mem.device)
            ops.copy2d(mem.view(B, S * 256)[:, starts[i] * 256:(starts[i] + h * w) * 256], lvl.view(B, h * w * 256))
            ms.append(ops.nhwc_to_nchw(lvl, B, h, w))
        mask_features._b200_pd = (pd, tuple(ms))         # lets the predictor skip the NCHW -> token-major round trip
        return mask_features, ms[0], ms


class B200ODISEMultiScaleMaskedTransformerDecoder(_HeadPart):
    """ODISEMultiScaleMaskedTransformerDecoder (odise.py:642-776; ctor mask2former_transformer_decoder.py:236-340 +
    odise.py:966-982) with the keyword arguments of mask_generator_with_label.py:46-65.
    forward(x = multi_scale_features, mask_features, mask=None) -> the reference's dict (pred_logits = PseudoClassEmbed
    output, pred_masks, mask_embed, mask_pooled_features, logit_scale, aux_outputs)."""

    def __init__(self, in_channels=256, mask_classification=True, *, num_classes=133, hidden_dim=256, num_queries=100,
                 nheads=8, dim_feedforward=2048, dec_layers=9, pre_norm=False, mask_dim=256, enforce_input_project=False,
                 class_embed=None, mask_embed=None, post_mask_embed=None):
        super().__init__()
        if mask_embed is not None:
            raise NotImplementedError("mask_embed=<module>: ODISE configs use post_mask_embed=PooledMaskEmbed (odise.py:636-640)")
        _expect("in_channels", in_channels, 256)
        _expect("hidden_dim", hidden_dim, 256)
        _expect("nheads", nheads, 8)
        _expect("dim_feedforward", dim_feedforward, 2048)
        _expect("pre_norm", pre_norm, False)
        _expect("mask_dim", mask_dim, 256)
        _expect("enforce_input_project", enforce_input_project, False)
        _expect("mask_classification", mask_classification, True)
        self.num_queries, self.num_layers, self.num_classes = num_queries, dec_layers, num_classes
        self.num_feature_levels = 3
        self.class_embed, self.post_mask_embed = class_embed, post_mask_embed     # config objects; weights live in the engine

    @torch.no_grad()
    def forward(self, x, mask_features, mask=None, *, inputs_dict=None):
        del mask, inputs_dict                    # odise.py:649-650: the mask is discarded; inputs_dict only feeds caption heads
        eng, own = self.engine, self._owner
        cached = getattr(mask_features, "_b200_pd", None)
        if cached is not None and len(cached[1]) == len(x) and all(a is b for a, b in zip(cached[1], x)):
            pd = cached[0]
        else:
            pd = eng.pd_from_tensors(x, mask_features)
        B = mask_features.shape[0]
        heads = eng.transformer_decoder(pd, B)
        h2, w2 = pd["mask_hw"]
        Q, dev = eng.Q, mask_features.device

        def pack(hd):
            return dict(pred_logits=own._pseudo_logits(B, Q, dev), pred_masks=hd["pred_masks"].view(B, Q, h2, w2),
                        mask_embed=hd["mask_embed"].view(B, Q, -1),
                        mask_pooled_features=hd["mask_pooled_features"].view(B, Q, -1),
                        logit_scale=torch.tensor(eng.logit_scale, device=dev))

        res = pack(heads[-1])
        res["aux_outputs"] = [pack(h) for h in heads[:-1]]
        return res


class B200PseudoClassEmbed(nn.Module):
    """PseudoClassEmbed (odise.py:906-920): config holder (num_classes); the constant logits are produced by the head."""

    def __init__(self, num_classes):
        super().__init__()
        self.num_classes = num_classes


class B200PooledMaskEmbed(nn.Module):
    """PooledMaskEmbed (odise.py:966-1015): config holder; its weights (`post_mask_embed.*`) live in the HeadEngine."""

    def __init__(self, hidden_dim=256, mask_dim=256, projection_dim=256, temperature=0.07):
        super().__init__()
        _expect("hidden_dim", hidden_dim, 256)
        _expect("mask_dim", mask_dim, 256)
        _expect("projection_dim", projection_dim, 256)
        self.hidden_dim, self.mask_dim, self.projection_dim = hidden_dim, mask_dim, projection_dim


class B200MaskFormerHead(nn.Module):
    """Drop-in for MaskFormerHead (mask_former_head.py:48-132) over MSDeformAttnPixelDecoder +
    ODISEMultiScaleMaskedTransformerDecoder(class_embed=PseudoClassEmbed, post_mask_embed=PooledMaskEmbed): the
    constructor keywords of mask_generator_with_label.py:29-66, `.pixel_decoder.forward_features`, `.predictor(...)`,
    `.layers`, `.num_classes`, and load_state_dict with the reference's keys (`pixel_decoder.*`, `predictor.*`)."""

    def __init__(self, input_shape=None, *, num_classes=133, pixel_decoder=None, loss_weight=1.0, ignore_value=-1,
                 transformer_predictor=None, transformer_in_feature="multi_scale_pixel_decoder", device="cuda", nmma=3):
        super().__init__()
        _expect("transformer_in_feature", transformer_in_feature, "multi_scale_pixel_decoder")
        self.pixel_decoder = pixel_decoder if pixel_decoder is not None else B200MSDeformAttnPixelDecoder()
        self.predictor = transformer_predictor if transformer_predictor is not None \
            else B200ODISEMultiScaleMaskedTransformerDecoder(num_classes=num_classes)
        for part in (self.pixel_decoder, self.predictor):
            if not isinstance(part, _HeadPart):
                raise TypeError("pixel_decoder / transformer_predictor must be the B200* plugin classes")
            object.__setattr__(part, "_owner", self)
        self.in_features = ["s2", "s3", "s4", "s5"] if input_shape is None else \
            [k for k, v in sorted(input_shape.items(), key=lambda kv: kv[1].stride)]
        self.ignore_value, self.loss_weight, self.common_stride = ignore_value, loss_weight, 4
        self.transformer_in_feature = transformer_in_feature
        self.num_classes = num_classes          # set by OpenPanopticInference through open_state_dict (odise.py:135)
        ce = getattr(self.predictor, "class_embed", None)
        self._pseudo_classes = ce.num_classes if ce is not None else num_classes   # NOT updated by the wrapper (SURVEY §8b B-2)
        self._dev, self._nmma = torch.device(device), nmma
        self.engine = None
        self._sd = None

    @classmethod
    def from_state_dict(cls, state_dict, device, num_classes=133, num_queries=100, nmma=3):
        """Keys prefixed `sem_seg_head.` as in an ODISE checkpoint."""
        head = cls(num_classes=num_classes, device=device, nmma=nmma,
                   transformer_predictor=B200ODISEMultiScaleMaskedTransformerDecoder(
                       num_classes=num_classes, num_queries=num_queries, class_embed=B200PseudoClassEmbed(num_classes),
                       post_mask_embed=B200PooledMaskEmbed()))
        head.load_state_dict({k[len("sem_seg_head."):]: v for k, v in state_dict.items() if k.startswith("sem_seg_head.")})
        return head

    @staticmethod
    def expected_keys():
        return [n[len("sem_seg_head."):] for n, _, _ in spec.head_params() if n.startswith("sem_seg_head.")]

    def load_state_dict(self, state_dict, strict=True):
        want = self.expected_keys()
        missing = [k for k in want if k not in state_dict]
        unexpected = [k for k in state_dict if k not in set(want)]
        if strict and (missing or unexpected):
            raise RuntimeError(f"B200MaskFormerHead.load_state_dict: missing {missing[:5]} ({len(missing)}), "
                               f"unexpected {unexpected[:5]} ({len(unexpected)})")
        self.engine = HeadEngine(dict(state_dict), self._dev, nmma=self._nmma, pd_prefix="pixel_decoder.",
                                 dec_prefix="predictor.", n_enc=self.pixel_decoder.transformer_enc_layers,
                                 n_dec=self.predictor.num_layers, num_queries=self.predictor.num_queries)
        self._sd = OrderedDict((k, state_dict[k].detach().cpu()) for k in want if k in state_dict)
        return missing, unexpected

    def state_dict(self, destination=None, prefix="", keep_vars=False):
        d = OrderedDict() if destination is None else destination
        for k, v in (self._sd or {}).items():
            d[prefix + k] = v
        return d

    def _pseudo_logits(self, B, Q, dev):
        # PseudoClassEmbed (odise.py:910-920): ones for every class, zero for background
        lg = torch.ones(B, Q, self._pseudo_classes + 1, device=dev)
        lg[..., -1] = 0
        return lg

    def forward(self, features, mask=None):
        return self.layers(features, mask)

    @torch.no_grad()
    def layers(self, features, mask=None):
        # mask_former_head.py:118-120
        mask_features, _, multi_scale_features = self.pixel_decoder.forward_features(features)
        return self.predictor(multi_scale_features, mask_features, mask)


class B200PoolingCLIPHead(nn.Module):
    """Drop-in for PoolingCLIPHead (odise.py:1420-1542), inference only, normalize_logits=True, no bg labels:
    forward(outputs) pops "pred_open_logits" [B, Q, K] and returns {"pred_open_logits": ensemble logits [B, Q, K]}
    from outputs["images"] ([B, 3, H, W] in [0, 1]) and outputs["pred_masks"].  The vocabulary (CLIP text embeddings of
    the prompts, prompt counts per class, overlap with the training vocabulary) is set with set_vocabulary()."""

    def __init__(self, state_dict, device, alpha=0.35, beta=0.65, nmma=3, visual=None):
        super().__init__()
        from .clip import ClipVisualEngine, MaskClipHead
        self.visual = visual if visual is not None else ClipVisualEngine(state_dict, device, nmma=nmma)
        import math
        self.engine = MaskClipHead(self.visual, alpha=alpha, beta=beta,
                                   logit_scale=math.exp(float(state_dict.get("clip.logit_scale", math.log(100.0)))))
        self.alpha, self.beta = alpha, beta

    @property
    def with_bg(self):
        return False

    def set_vocabulary(self, text_embed, group_sizes, overlapping):
        self.engine.set_vocabulary("test", text_embed, group_sizes, overlapping)

    @torch.no_grad()
    def forward(self, outputs, targets=None):
        assert not self.training, "PoolingCLIPHead only supports inference"
        assert targets is None and "test" in self.engine._vocab
        open_logits = outputs.pop("pred_open_logits")
        img, masks = outputs["images"], outputs["pred_masks"]
        if not img.is_cuda:
            raise RuntimeError("B200PoolingCLIPHead: CUDA tensors required (no CPU path)")
        B, Q, K = open_logits.shape
        # the device kernel takes the category logits with a void column; it only enters the merged output, which the
        # plugin surface does not return (the caller merges, odise.py:300-323)
        cat = torch.cat([open_logits.float(), torch.zeros(B, Q, 1, device=img.device)], dim=-1)
        r = self.engine.forward("test", img.contiguous().float(), B, img.shape[2], img.shape[3], masks.float(), cat,
                                want_open=True)
        return {"pred_open_logits": r["pred_open_logits"]}


class B200CategoryODISE(nn.Module):
    """Drop-in for the eval branch of CategoryODISE.forward (odise.py:209-246, :282-370): a list of
    {"image": uint8 [3, h, w] (0..255), "height": H_out, "width": W_out} in, a list of
    {"sem_seg": [K, H_out, W_out], "panoptic_seg": (int32 [H_out, W_out], segments_info), "instances": {...}} out.
    Batching follows detectron2's ImageList.from_tensors: images are top-left aligned in a zero-padded batch whose size
    is the per-batch maximum rounded up to size_divisibility (64) for the network, and un-rounded for MaskCLIP.
    `engine` is an ODISEEngine with a vocabulary set (set_vocabulary / set_vocabulary_from_tokens)."""

    def __init__(self, engine, size_divisibility=64, semantic_on=True, panoptic_on=True, instance_on=True,
                 test_topk_per_image=100, tokenizer=None, train_labels=None, category_prompt=None, clip_prompt="photo",
                 metadata=None):
        super().__init__()
        self.engine = engine
        self.size_divisibility = size_divisibility
        self.semantic_on, self.panoptic_on, self.instance_on = semantic_on, panoptic_on, instance_on
        self.test_topk_per_image = test_topk_per_image
        self.tokenizer, self.train_labels = tokenizer, train_labels
        self.category_prompt, self.clip_prompt = category_prompt, clip_prompt   # odise.py:1225 (None), :1428 ("photo")
        self.metadata = metadata
        self.num_classes = None
        self.test_labels = None

    # ---- vocabulary protocol of OpenPanopticInference (odise/modeling/wrapper/pano_wrapper.py:36-68, odise.py:133-166)
    def open_state_dict(self, destination=None, prefix=""):
        d = OrderedDict() if destination is None else destination
        d[prefix + "sem_seg_head.num_classes"] = self.num_classes
        d[prefix + "metadata"] = self.metadata
        d[prefix + "test_topk_per_image"] = self.test_topk_per_image
        d[prefix + "semantic_on"] = self.semantic_on
        d[prefix + "panoptic_on"] = self.panoptic_on
        d[prefix + "instance_on"] = self.instance_on
        d[prefix + "category_head.test_labels"] = self.test_labels
        d[prefix + "clip_head.test_labels"] = self.test_labels
        return d

    def load_open_state_dict(self, state_dict):
        """Same keys as open_state_dict().  New `test_labels` (list of synonym lists) build — or re-activate from the cache,
        like get_and_cache_test_text_embed — the vocabulary on the device; `metadata.thing_dataset_id_to_contiguous_id`
        names the "thing" classes of the panoptic merge (maskformer_model.py:318)."""
        known = set(self.open_state_dict())
        for k, v in state_dict.items():
            if k not in known:
                raise KeyError(f"{k} is not part of the open state dict")
        g = state_dict.get
        self.num_classes = g("sem_seg_head.num_classes", self.num_classes)
        self.metadata = g("metadata", self.metadata)
        self.test_topk_per_image = g("test_topk_per_image", self.test_topk_per_image)
        self.semantic_on = g("semantic_on", self.semantic_on)
        self.panoptic_on = g("panoptic_on", self.panoptic_on)
        self.instance_on = g("instance_on", self.instance_on)
        cat, clip = g("category_head.test_labels", self.test_labels), g("clip_head.test_labels", self.test_labels)
        if "category_head.test_labels" in state_dict and "clip_head.test_labels" in state_dict and cat != clip:
            raise ValueError("category_head and clip_head must share one test vocabulary")
        labels = cat if "category_head.test_labels" in state_dict else clip
        if labels is not None and labels != self.test_labels:
            self._activate(labels)
        self.test_labels = labels
        for k, v in state_dict.items():                       # the reference asserts every key took (odise.py:166)
            assert self.open_state_dict()[k] == v, f"{k} is not loaded correctly"

    def _activate(self, labels):
        from . import vocab
        key = tuple(tuple(s) for s in labels)
        if self.num_classes is not None and self.num_classes != len(labels):
            raise ValueError(f"num_classes = {self.num_classes} but {len(labels)} test labels")
        if self.engine.has_vocabulary(key):
            self.engine.use_vocabulary(key)
            return
        if self.tokenizer is None:
            raise RuntimeError("a new test vocabulary needs a tokenizer (odise_b200.vocab.SimpleTokenizer)")
        if self.metadata is None or not hasattr(self.metadata, "thing_dataset_id_to_contiguous_id"):
            raise RuntimeError("a new test vocabulary needs `metadata.thing_dataset_id_to_contiguous_id` (the thing classes "
                               "of the panoptic merge, maskformer_model.py:318)")
        things = sorted(self.metadata.thing_dataset_id_to_contiguous_id.values())
        if self.engine.clip_head is not None and self.train_labels is None:
            raise RuntimeError("a new test vocabulary needs `train_labels` (PoolingCLIPHead.train_labels, odise.py:1446-1449: "
                               "the COCO panoptic prompt-engineered labels) to assign the alpha / beta exponents")
        vocab.build_vocabulary(self.engine, self.tokenizer, key, labels, self.train_labels, things, self.category_prompt,
                               self.clip_prompt)

    @torch.no_grad()
    def forward(self, batched_inputs):
        assert not self.training, "B200CategoryODISE is inference only"
        eng, dev = self.engine, self.engine.dev
        imgs = [x["image"] for x in batched_inputs]
        sizes = [(int(im.shape[-2]), int(im.shape[-1])) for im in imgs]
        mh, mw = max(s[0] for s in sizes), max(s[1] for s in sizes)
        d = self.size_divisibility
        ph, pw = (mh + d - 1) // d * d, (mw + d - 1) // d * d
        n = len(imgs)
        net = torch.zeros(n, 3, ph, pw, dtype=torch.uint8, device=dev)
        for i, im in enumerate(imgs):
            if im.dtype != torch.uint8:
                raise RuntimeError('"image" must be uint8 CHW in 0..255 (detectron2 DatasetMapper format)')
            net[i, :, :sizes[i][0], :sizes[i][1]] = im.to(dev, non_blocking=True)
        clip_in = net[:, :, :mh, :mw].contiguous() if (mh, mw) != (ph, pw) else net
        out = eng.step(n, ph, pw, images_u8=net, clip_images=clip_in)
        results = []
        for i, x in enumerate(batched_inputs):
            H, W = int(x.get("height", sizes[i][0])), int(x.get("width", sizes[i][1]))
            post = eng.post(out["pred_logits"][i:i + 1], out["pred_masks"][i:i + 1], H, W, semantic=self.semantic_on,
                            panoptic=self.panoptic_on, instance=self.instance_on, topk=self.test_topk_per_image,
                            panoptic_on=self.panoptic_on, padded_size=(ph, pw), image_size=sizes[i])
            r = {}
            if self.semantic_on:
                r["sem_seg"] = post["sem_seg"][0]
            if self.panoptic_on:
                r["panoptic_seg"] = (post["panoptic_seg"][0], eng.post.segments_info(post["seg_info"], post["n_segments"])[0])
            if self.instance_on:
                ins = post["instances"]
                keep = ins["valid"][0].bool()
                qi = ins["query_index"][0][keep].long()
                r["instances"] = dict(pred_masks=ins["query_masks"][0][qi], scores=ins["scores"][0][keep],
                                      pred_classes=ins["pred_classes"][0][keep].long(), image_size=(H, W))
            results.append(r)
        return results
