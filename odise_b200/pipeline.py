"""Inference meta-arch of the H100 engine: the eval branch of CategoryODISE.forward
(odise/modeling/meta_arch/odise.py:209-246, :282-331) restricted to the north-star hot path:

    images -> [sliding 512^2 crops] -> UNet feature pass -> projections -> pixel decoder -> masked-attention decoder
           -> mask_embed x CLIP-text scoring -> (pred_logits [B, Q, K+1], pred_masks [B, Q, H/4, W/4])

One process per GPU; images shard over ranks with a single NCCL all-gather of the final logits (reference analogue:
d2 evaluator gather, SURVEY.md §2.4).  A step at fixed (batch, H, W) is captured once into a CUDA graph and replayed.
"""
import math
import os

import torch

from . import lib, spec
from .backbone import BackboneEngine
from .head import HeadEngine


def full_param_list(with_vae=False, with_clip=False):
    return (spec.unet_params() + spec.backbone_params() + spec.head_params() + (spec.vae_params() if with_vae else [])
            + (spec.clip_visual_params() if with_clip else []))


class ODISEEngine:
    def __init__(self, sd, device, nmma=3, num_queries=100, with_vae=False, with_clip=False, with_clip_head=None,
                 alpha=0.3, beta=0.7, uncond=None, synthetic_uncond=False):
        """with_clip: CLIP ViT-L/14-336 image tower (implicit captioner input, §8f-2); with_clip_head (default = with_clip):
        MaskCLIP + PoolingCLIPHead ensemble (odise_with_label.py: alpha 0.3, beta 0.7) on the same frozen tower."""
        self.dev = torch.device(device)
        self.nmma = nmma
        vae = None
        if with_vae:                      # SURVEY.md §8f-1: real KL-VAE taps instead of synthetic ones
            from .vae import VAEEngine
            vae = VAEEngine(sd, device, nmma=nmma)
        clip = None
        if with_clip:                     # SURVEY.md §8f-2: real CLIP ViT-L/14-336 image embedding of every crop
            from .clip import ClipVisualEngine
            clip = ClipVisualEngine(sd, device, nmma=nmma)
        self.with_vae, self.with_clip = with_vae, with_clip
        self.clip_head = None
        if with_clip_head if with_clip_head is not None else with_clip:
            from .clip import MaskClipHead
            assert clip is not None, "the MaskCLIP head shares the CLIP image tower: with_clip=True required"
            self.clip_head = MaskClipHead(clip, alpha=alpha, beta=beta,
                                          logit_scale=math.exp(float(sd.get("clip.logit_scale", math.log(100.0)))))
        self.backbone = BackboneEngine(sd, device, nmma=nmma, vae=vae, clip=clip, uncond=uncond,
                                       synthetic_uncond=synthetic_uncond)
        self.text = None                  # ClipTextEngine, built on demand (set_vocabulary_from_tokens)
        self._sd_text = {k: v for k, v in sd.items() if k.startswith(spec.CLIP_TEXT_PREFIX) and not k.startswith(spec.CLIP_PREFIX)}
        self._null_embed = sd.get("category_head.null_embed")
        self.head = HeadEngine(sd, device, nmma=nmma, num_queries=num_queries)
        self.Q = num_queries
        self._graphs = {}
        self.vocab_key = None
        self.launches_per_step = None

    def set_vocabulary(self, key, text_bank, null_bank, group_sizes, thing_ids=None, clip_text_bank=None,
                       overlapping=None):
        """OpenPanopticInference / CategoryEmbed.test_labels analogue (pano_wrapper.py:58-68, odise.py:1281-1307):
        the vocabulary is a [K', 768] CLIP text bank + per-class prompt counts (+ which classes are "things" for
        the panoptic merge, metadata.thing_dataset_id_to_contiguous_id in the reference).  With a MaskCLIP head:
        clip_text_bank = the CLIP text embeddings of the PoolingCLIPHead prompts ("a photo of a {}.": odise.py:1428,1475 —
        NOT the category head's raw class names, odise.py:1225), overlapping[k] = class k shares a name with the training
        vocabulary (odise.py:1483-1493).  thing_ids / overlapping have no defaults: a silently wrong thing/stuff split or
        alpha/beta assignment changes the results (synthetic runs: set_synthetic_vocabulary)."""
        K = len(group_sizes)
        if thing_ids is None:
            raise lib.OdiseError("set_vocabulary: thing_ids is required (metadata.thing_dataset_id_to_contiguous_id "
                                 "values; pass () for a stuff-only vocabulary)")
        if self.clip_head is not None and (overlapping is None or clip_text_bank is None):
            raise lib.OdiseError("set_vocabulary: the MaskCLIP head needs `clip_text_bank` (prompted labels) and "
                                 "`overlapping` (vocab.overlapping_mask(test_labels, train_labels))")
        self.head.set_vocabulary(key, text_bank, null_bank, group_sizes)
        if self.clip_head is not None:
            self.clip_head.set_vocabulary(key, clip_text_bank, group_sizes, list(overlapping))
        from .postprocess import PostProcessor
        if not hasattr(self, "_posts"):
            self._posts = {}
        self._posts[key] = PostProcessor(self.dev, K, thing_ids, nmma=self.nmma)
        self.use_vocabulary(key)

    def set_synthetic_vocabulary(self, key, n_classes, n_prompts, seed=11):
        """Benchmarks / tests only: seeded random text banks (category bank and an independent MaskCLIP bank), every
        other class a "thing", every other class "seen in training"."""
        bank, null, sizes = synthetic_vocabulary(n_classes, n_prompts, seed)
        clip_bank = torch.randn(n_prompts, 768, generator=torch.Generator().manual_seed(seed + 66))
        self.set_vocabulary(key, bank, null, sizes, thing_ids=list(range(0, n_classes, 2)), clip_text_bank=clip_bank,
                            overlapping=[(k % 2) == 0 for k in range(n_classes)])

    def has_vocabulary(self, key):
        return key in getattr(self, "_posts", {})

    def use_vocabulary(self, key):
        """Switch to a vocabulary that was set before (the reference caches text banks per label tuple, odise.py:1281-1288)."""
        if not self.has_vocabulary(key):
            raise lib.OdiseError(f"vocabulary {key!r} has not been set")
        self.vocab_key = key
        self.post = self._posts[key]

    @classmethod
    def from_checkpoints(cls, ldm_path, odise_path, clip_path, device, trusted=False, **kw):
        """The reference's three downloads (sd-v1-3.ckpt, OpenAI CLIP ViT-L-14-336, odise_*.pth) -> a ready engine:
        weights verified against the spec inventory, `uncond_inputs` computed by the SD text encoder (ldm.py:116)."""
        from . import checkpoint
        from .clip import uncond_inputs
        sd, _ = checkpoint.load_reference_checkpoints(ldm_path, odise_path, clip_path, trusted=trusted)
        nmma = kw.get("nmma", 3)
        un = uncond_inputs(sd, device, nmma=nmma).cpu()
        return cls(sd, device, with_vae=True, with_clip=True, uncond=un, **kw)

    @torch.no_grad()
    def set_vocabulary_from_tokens(self, key, token_ids, group_sizes, null_token_ids=None, thing_ids=None, overlapping=None,
                                   clip_token_ids=None):
        """CategoryEmbed.get_and_cache_test_text_embed (odise.py:1281-1288): tokenised prompts [K', 77] (all synonyms of
        all classes, class-major) -> CLIP text bank on the device -> set_vocabulary.  clip_token_ids: the same labels under
        the PoolingCLIPHead prompt (odise.py:1475) — a second bank; None = same tokens (caption model: both 'photo').
        The null embedding is the checkpoint's `category_head.null_embed` parameter, or the text embedding of
        `null_token_ids` ("" at init)."""
        from .clip import ClipTextEngine, build_text_bank
        if self.text is None:
            if not self._sd_text:
                raise lib.OdiseError("no CLIP text tower weights (`clip.token_embedding.weight`, ...) in the state dict")
            self.text = ClipTextEngine(self._sd_text, self.dev, nmma=self.nmma)
        bank = build_text_bank(self.text, token_ids)
        if self._null_embed is not None:
            null = self._null_embed.view(1, -1)
        elif null_token_ids is not None:
            null = self.text.encode(null_token_ids.view(1, -1))[0]
        else:
            raise lib.OdiseError("no category_head.null_embed in the state dict and no null_token_ids given")
        clip_bank = bank if clip_token_ids is None else build_text_bank(self.text, clip_token_ids)
        self.set_vocabulary(key, bank, null, group_sizes, thing_ids=thing_ids, clip_text_bank=clip_bank, overlapping=overlapping)
        return bank

    @torch.no_grad()
    def postprocess(self, out, H, W, semantic=True, panoptic=True, instance=False, padded_size=None, image_size=None):
        """semantic / panoptic / instance inference on the device (odise.py:326-370).  (H, W) = requested output size;
        padded_size / image_size as in sem_seg_postprocess when the output is not the padded input itself."""
        return self.post(out["pred_logits"], out["pred_masks"], H, W, semantic=semantic, panoptic=panoptic,
                         instance=instance, padded_size=padded_size, image_size=image_size)

    # ------------------------------------------------------------------------------------------- device step
    @torch.no_grad()
    def step(self, n_images, H, W, vae_taps=None, images_u8=None, clip_images=None):
        """One pass of the hot path for n_images resident images (eager). Returns device tensors.
        clip_images: what MaskCLIP looks at when it differs from the network input — the reference feeds it the batch
        padded only to its own maximum size, not to size_divisibility (odise.py:240-246)."""
        if images_u8 is None and (self.with_vae or self.with_clip):
            images_u8 = self._image_buffer(n_images, H, W)
        ci = clip_images if clip_images is not None else images_u8
        # MaskCLIP's image-token stream does not depend on the masks: it rides through the CLIP tower together with the crops
        joint = self.clip_head is not None and self.vocab_key is not None and ci is not None and \
            not os.environ.get("ODISE_NO_CLIP_JOINT")                       # A/B switch: stand-alone MaskCLIP pass
        self.backbone.maskclip_images = (ci, n_images, ci.shape[2], ci.shape[3]) if joint else None
        try:
            feats = self.backbone.forward(n_images, H, W, vae_taps, images_u8)
        finally:
            self.backbone.maskclip_images = None
        out = self.head.forward(feats, n_images, vocab_key=self.vocab_key)
        h2, w2 = out["pd"]["mask_hw"]
        last = out["heads"][-1]
        res = dict(pred_masks=last["pred_masks"].view(n_images, self.Q, h2, w2),
                   mask_embed=last["mask_embed"].view(n_images, self.Q, -1),
                   mask_pooled_features=last["mask_pooled_features"].view(n_images, self.Q, -1))
        if "pred_logits" in out:
            res["pred_logits"] = out["pred_logits"]
            if self.clip_head is not None:        # odise.py:292-323: MaskCLIP ensemble replaces the class scores
                with lib.nvtx("maskclip_ensemble"):
                    ch = self.clip_head.forward(self.vocab_key, ci, n_images, ci.shape[2], ci.shape[3], res["pred_masks"],
                                                out["pred_logits"])
                res["pred_logits_category"] = out["pred_logits"]
                res["pred_logits"] = ch["pred_logits"]
                res["clip_mask_embed"] = ch["mask_embed"]
        res["aux"] = out["heads"][:-1]
        return res

    @torch.no_grad()
    def step_full(self, n_images, H, W, images_u8=None, semantic=True, panoptic=True, instance=True, topk=100):
        """step() + the inference heads of CategoryODISE.forward (odise.py:326-370: semantic / panoptic / instance
        inference at the input resolution) — what the metric "panoptic inference" times.  All on the device."""
        res = self.step(n_images, H, W, images_u8=images_u8)
        with lib.nvtx("semantic_panoptic_instance_inference"):
            res["post"] = self.post(res["pred_logits"], res["pred_masks"], H, W, semantic=semantic, panoptic=panoptic,
                                    instance=instance, topk=topk)
        return res

    def _image_buffer(self, n_images, H, W):
        shp = (n_images, 3, H, W)
        if not hasattr(self, "_img_dev") or tuple(self._img_dev.shape) != shp:
            g = torch.Generator().manual_seed(99)
            self._img_dev = torch.randint(0, 256, shp, generator=g, dtype=torch.uint8).to(self.dev)
        return self._img_dev

    def capture(self, n_images, H, W, post=False):
        """Warm up eagerly, then capture the step into a CUDA graph (static shapes, static buffers).
        post=True captures step_full (network + semantic / panoptic / instance inference)."""
        key = (n_images, H, W, self.vocab_key, bool(post))
        if key in self._graphs:
            return self._graphs[key]
        fn = self.step_full if post else self.step
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            for _ in range(2):
                fn(n_images, H, W)
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        before = lib.launch_count()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fn(n_images, H, W)
        self.launches_per_step = lib.launch_count() - before
        self._graphs[key] = (g, out)
        return self._graphs[key]

    # ------------------------------------------------------------------------------------------- user API
    @torch.no_grad()
    def infer(self, images_u8_pinned, use_graph=True, outputs="raw"):
        """End-to-end call on a host batch: uint8 [B, 3, H, W] in pinned memory -> host dict.  H2D and D2H inside.
        outputs="raw": pred_logits [B, Q, K+1] + pred_masks [B, Q, H/4, W/4] (the network outputs);
        outputs="panoptic": the inference results at the input resolution — panoptic_seg int32 [B, H, W], seg_info
        [B, Q, 3] + n_segments [B], semantic label map uint8/int16 is NOT shipped (the [K, H, W] score tensor stays on the
        device like in the reference), instance scores / classes / query index [B, topk], plus pred_logits."""
        B, _, H, W = images_u8_pinned.shape
        self._image_buffer(B, H, W).copy_(images_u8_pinned, non_blocking=True)
        post = outputs == "panoptic"
        if use_graph:
            g, out = self.capture(B, H, W, post=post)
            g.replay()
        else:
            out = (self.step_full if post else self.step)(B, H, W, images_u8=self._img_dev)
        if post:
            src = dict(pred_logits=out["pred_logits"], panoptic_seg=out["post"]["panoptic_seg"],
                       seg_info=out["post"]["seg_info"], n_segments=out["post"]["n_segments"])
            if "instances" in out["post"]:
                ins = out["post"]["instances"]
                src.update(instance_scores=ins["scores"], instance_classes=ins["pred_classes"],
                           instance_query=ins["query_index"], instance_valid=ins["valid"])
        else:
            src = dict(pred_logits=out["pred_logits"], pred_masks=out["pred_masks"])
        hk = (outputs, B, H, W, self.vocab_key)
        if getattr(self, "_host_key", None) != hk:
            self._host = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in src.items()}
            self._host_key = hk
        for k, v in src.items():
            self._host[k].copy_(v, non_blocking=True)
        torch.cuda.current_stream(self.dev).synchronize()
        return dict(self._host)

    def d2h_bytes(self):
        """bytes infer() last copied back per call"""
        return int(sum(v.numel() * v.element_size() for v in getattr(self, "_host", {}).values()))


def gather_logits(local_logits):
    """Image-sharded inference: one all-gather of the final class logits over the ranks (NCCL on NVLink)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local_logits
    out = torch.empty((dist.get_world_size() * local_logits.shape[0],) + tuple(local_logits.shape[1:]),
                      dtype=local_logits.dtype, device=local_logits.device)
    dist.all_gather_into_tensor(out, local_logits.contiguous())
    return out


def synthetic_vocabulary(n_classes, n_prompts, seed=11):
    """Seeded stand-in for the CLIP text bank of a vocabulary with n_classes classes and n_prompts prompt strings
    (ADE-150: 150 / 403, COCO-133: 133 / 254, ADE-847: 847 / 1342; SURVEY.md §8d) -> (bank, null, group sizes)."""
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(n_prompts, 768, generator=g)
    null = torch.randn(1, 768, generator=torch.Generator().manual_seed(13))
    base, extra = divmod(n_prompts, n_classes)
    sizes = [base + (1 if i < extra else 0) for i in range(n_classes)]
    return bank, null, sizes
