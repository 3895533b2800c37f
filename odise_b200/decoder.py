"""Training drop-in for ODISE's Mask2Former transformer decoder and its pooled mask embedding
(ODISEMultiScaleMaskedTransformerDecoder, PooledMaskEmbed and MaskPooling of odise/modeling/meta_arch/odise.py, over
MultiScaleMaskedTransformerDecoder of mask2former_transformer_decoder.py).

    from odise_b200.decoder import ODISEMultiScaleMaskedTransformerDecoder, PooledMaskEmbed   # in place of odise's

The classes keep the reference's constructors and defaults, submodule names, initialisation order (the same seed gives
the same parameters) and state-dict keys, so state dicts load both ways.  The decoder's cross-attention layers are
odise_b200.masked_attn.CrossAttentionLayer; the self-attention, FFN, MLP and position-encoding modules are restated
here in torch.

forward_prediction_heads takes the fused path when mask_features is on CUDA, the mask einsum would run in float32 or in
16 bits under torch.autocast, post_mask_embed is this module's PooledMaskEmbed with hard pooling, mask_dim = 256,
num_queries <= 256 and use_fused is True.  It then runs MaskHeadFunction: one sm_90a kernel pass writes the mask logits
and the hard-pooled features together (MaskPooling once, not twice), and odise_mask_head_attn_mask_* builds the
attention mask with the all-blocked-row fix-up of odise.py:683 inside the kernel, so the decoder's forward and backward
make no host synchronisation.  forward() calls forward_prediction_heads as the reference does, so a subclass's override
is used.  Every other input runs the reference's ops in its order, torch.where included.

Under autocast, MaskPooling's sum is a float32 op: the pooling weight is w = dtype(float32(1 / (count + 1e-8))), applied
in fp32 and rounded once per pooled value, as the reference's bmm operand is rounded.  A 16-bit module without autocast
(.half()) takes the composed path, whose fp16 sum the kernels do not reproduce."""
import logging
import math

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib
from .masked_attn import CrossAttentionLayer, _activation

# The kernels as torch custom ops (lib.custom_op).  lib's functions are looked up at call time, so that a test that
# patches them sees every call.
lib.custom_op("mask_head_forward(Tensor embed, Tensor features, float threshold) -> (Tensor, Tensor, Tensor)",
              lambda *args: lib.mask_head_forward(*args))
lib.custom_op("mask_head_backward(Tensor embed, Tensor features, Tensor outputs_mask, Tensor weights, Tensor grad_mask, "
              "Tensor grad_pooled, float threshold) -> (Tensor, Tensor)", lambda *args: lib.mask_head_backward(*args))
lib.custom_op("mask_head_attn_mask(Tensor outputs_mask, int h, int w, int heads) -> Tensor",
              lambda outputs_mask, h, w, heads: lib.mask_head_attn_mask(outputs_mask, (h, w), heads))


class MaskHeadFunction(Function):
    """(outputs_mask, pooled) = (E X, w * sum_hw m X) of embed E [B, Q, 256] and features X [B, 256, H, W] (CUDA,
    contiguous, one of float32 / float16 / bfloat16), m = sigmoid(outputs_mask) > threshold, w = 1 / (count + 1e-8).
    The pooling is hard (no gradient through m), so the gradients are grad E = G X^T and grad X = E^T G + (Gp w)^T m.
    features is the tensor the gradient is for and features_t its contiguous copy in embed's dtype that the kernels read
    (the same tensor in float32; under autocast one detached copy shared by the decoder's heads).  grad X is computed in
    embed's dtype, rounded once, and returned in features' dtype, so that autograd sums the heads' gradients there.
    Saves E, features_t, outputs_mask and w; the backward recomputes m and is bit-reproducible."""

    @staticmethod
    def forward(ctx, embed, features, features_t, threshold):
        om, pooled, weights = torch.ops.odise_b200.mask_head_forward(embed, features_t, threshold)
        ctx.threshold = threshold
        ctx.features_dtype = features.dtype
        ctx.save_for_backward(embed, features_t, om, weights)
        ctx.mark_non_differentiable(weights)
        return om, pooled, weights

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_mask, grad_pooled, _grad_weights):
        embed, features, om, weights = ctx.saved_tensors
        grad_mask = torch.zeros_like(om) if grad_mask is None else grad_mask.to(om.dtype).contiguous()
        grad_pooled = torch.zeros_like(embed) if grad_pooled is None else grad_pooled.to(embed.dtype).contiguous()
        ge, gx = torch.ops.odise_b200.mask_head_backward(embed, features, om, weights, grad_mask, grad_pooled,
                                                         ctx.threshold)
        return ge, gx.to(ctx.features_dtype), None, None


# ---------------------------------------------------------------------------------------------- the reference's layers
class SelfAttentionLayer(nn.Module):
    """Mask2Former's SelfAttentionLayer: nn.MultiheadAttention over (tgt + query_pos, tgt + query_pos, tgt), dropout,
    residual and LayerNorm, post-norm or (normalize_before) pre-norm."""

    def __init__(self, d_model, nhead, dropout=0.0, activation="relu", normalize_before=False):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.norm = nn.LayerNorm(d_model)
        self.dropout = nn.Dropout(dropout)
        self.activation = _activation(activation)
        self.normalize_before = normalize_before
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)

    @staticmethod
    def with_pos_embed(tensor, pos):
        return tensor if pos is None else tensor + pos

    def forward(self, tgt, tgt_mask=None, tgt_key_padding_mask=None, query_pos=None):
        x = self.norm(tgt) if self.normalize_before else tgt
        q = k = self.with_pos_embed(x, query_pos)
        tgt = tgt + self.dropout(self.self_attn(q, k, value=x, attn_mask=tgt_mask,
                                                key_padding_mask=tgt_key_padding_mask)[0])
        return tgt if self.normalize_before else self.norm(tgt)


class FFNLayer(nn.Module):
    """Mask2Former's FFNLayer: linear2(dropout(act(linear1(x)))), dropout, residual and LayerNorm (post or pre)."""

    def __init__(self, d_model, dim_feedforward=2048, dropout=0.0, activation="relu", normalize_before=False):
        super().__init__()
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm = nn.LayerNorm(d_model)
        self.activation = _activation(activation)
        self.normalize_before = normalize_before
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)

    def forward(self, tgt):
        x = self.norm(tgt) if self.normalize_before else tgt
        tgt = tgt + self.dropout(self.linear2(self.dropout(self.activation(self.linear1(x)))))
        return tgt if self.normalize_before else self.norm(tgt)


class MLP(nn.Module):
    """num_layers Linear layers with ReLU between them (layers.0 .. layers.{num_layers - 1})."""

    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        dims = [input_dim] + [hidden_dim] * (num_layers - 1) + [output_dim]
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip(dims[:-1], dims[1:]))

    def forward(self, x):
        for i, layer in enumerate(self.layers):
            x = F.relu(layer(x)) if i < self.num_layers - 1 else layer(x)
        return x


class PositionEmbeddingSine(nn.Module):
    """DETR's sine position encoding of an [N, C, H, W] map (Mask2Former's position_encoding.py): per pixel the
    cumulative row / column index, normalised to (0, scale], divided by temperature^(2 floor(i/2) / num_pos_feats), then
    interleaved sin / cos, y features first -> [N, 2 num_pos_feats, H, W] float32."""

    def __init__(self, num_pos_feats=64, temperature=10000, normalize=False, scale=None):
        super().__init__()
        self.num_pos_feats = num_pos_feats
        self.temperature = temperature
        self.normalize = normalize
        if scale is not None and normalize is False:
            raise ValueError("normalize should be True if scale is passed")
        self.scale = 2 * math.pi if scale is None else scale

    def forward(self, x, mask=None):
        if mask is None:
            mask = torch.zeros((x.size(0), x.size(2), x.size(3)), device=x.device, dtype=torch.bool)
        not_mask = ~mask
        y = not_mask.cumsum(1, dtype=torch.float32)
        xx = not_mask.cumsum(2, dtype=torch.float32)
        if self.normalize:
            y = y / (y[:, -1:, :] + 1e-6) * self.scale
            xx = xx / (xx[:, :, -1:] + 1e-6) * self.scale
        dim_t = torch.arange(self.num_pos_feats, dtype=torch.float32, device=x.device)
        dim_t = self.temperature ** (2 * (dim_t // 2) / self.num_pos_feats)
        px, py = xx[:, :, :, None] / dim_t, y[:, :, :, None] / dim_t
        px = torch.stack((px[:, :, :, 0::2].sin(), px[:, :, :, 1::2].cos()), dim=4).flatten(3)
        py = torch.stack((py[:, :, :, 0::2].sin(), py[:, :, :, 1::2].cos()), dim=4).flatten(3)
        return torch.cat((py, px), dim=3).permute(0, 3, 1, 2)

    def __repr__(self, _repr_indent=4):
        body = [f"num_pos_feats: {self.num_pos_feats}", f"temperature: {self.temperature}",
                f"normalize: {self.normalize}", f"scale: {self.scale}"]
        return "\n".join(["Positional encoding " + self.__class__.__name__] + [" " * _repr_indent + b for b in body])


# ---------------------------------------------------------------------------------------------- pooling
class MaskPooling(nn.Module):
    """ODISE's MaskPooling: einsum("bchw,bqhw->bqc", x, m / (sum_hw m + 1e-8)) with m = sigmoid(mask.detach()), hard:
    (m > mask_threshold) as mask's dtype.  Called on its own it runs these composed ops."""

    def __init__(self, hard_pooling=True, mask_threshold=0.5):
        super().__init__()
        self.hard_pooling = hard_pooling
        self.mask_threshold = mask_threshold

    def extra_repr(self) -> str:
        return f"hard_pooling={self.hard_pooling}\n" f"mask_threshold={self.mask_threshold}\n"

    def forward(self, x, mask):
        assert x.shape[-2:] == mask.shape[-2:]
        mask = mask.detach().sigmoid()
        if self.hard_pooling:
            mask = (mask > self.mask_threshold).to(mask.dtype)
        denorm = mask.sum(dim=(-1, -2), keepdim=True) + 1e-8
        return {"mask_pooled_features": torch.einsum("bchw,bqhw->bqc", x, mask / denorm)}


class PooledMaskEmbed(nn.Module):
    """ODISE's PooledMaskEmbed: mask-pooled features -> pool_proj (LayerNorm, Linear) + decoder_output -> mask_embed
    (LayerNorm, 3-layer MLP), and logit_scale = min(exp(logit_scale), 100).  Called on its own it pools with the
    composed ops (twice, as the reference does); the decoder's fused path hands it the kernel's pooled features."""

    def __init__(self, hidden_dim, mask_dim, projection_dim, temperature=0.07):
        super().__init__()
        self.pool_proj = nn.Sequential(nn.LayerNorm(hidden_dim), nn.Linear(hidden_dim, hidden_dim))
        self.mask_embed = nn.Sequential(nn.LayerNorm(mask_dim), MLP(mask_dim, hidden_dim, projection_dim, 3))
        self.logit_scale = nn.Parameter(torch.ones([]) * np.log(1 / temperature))
        self.mask_pooling = MaskPooling()

    def forward(self, decoder_output, input_mask_embed, mask_features, pred_logits, pred_masks):
        self.mask_pooling(mask_features, pred_masks)        # the reference pools twice and keeps the second result
        res = self.mask_pooling(mask_features, pred_masks)
        out = self.from_pooled(decoder_output, res["mask_pooled_features"])
        if res.get("outputs_mask") is not None:
            out["outputs_mask"] = res["outputs_mask"]
        return out

    def from_pooled(self, decoder_output, mask_pooled_x):
        mask_pooled_x = self.pool_proj(mask_pooled_x)
        mask_pooled_x += decoder_output
        mask_embed = self.mask_embed(mask_pooled_x)
        logit_scale = torch.clamp(self.logit_scale.exp(), max=100)
        return {"mask_embed": mask_embed, "mask_pooled_features": mask_pooled_x, "logit_scale": logit_scale}


# ---------------------------------------------------------------------------------------------- the decoder
class ODISEMultiScaleMaskedTransformerDecoder(nn.Module):
    """Mask2Former's multi-scale masked transformer decoder with ODISE's class_embed / mask_embed / post_mask_embed
    overrides.  See the module docstring for the fused prediction heads; use_fused = False forces the reference's
    composed ops."""

    _version = 2

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        version = local_metadata.get("version", None)
        if version is None or version < 2:
            scratch = True
            for k in list(state_dict.keys()):
                if "static_query" in k:
                    state_dict[k.replace("static_query", "query_feat")] = state_dict.pop(k)
                    scratch = False
            if not scratch:
                logging.getLogger(__name__).warning(
                    f"Weight format of {self.__class__.__name__} have changed! Please upgrade your models. Applying "
                    "automatic conversion now ...")
        # as in the reference, nothing else: the decoder holds no parameter of its own, its children load theirs

    def __init__(self, in_channels, mask_classification=True, *, num_classes, hidden_dim, num_queries, nheads,
                 dim_feedforward, dec_layers, pre_norm, mask_dim, enforce_input_project, class_embed=None,
                 mask_embed=None, post_mask_embed=None):
        super().__init__()
        assert mask_classification, "Only support mask classification model"
        self.mask_classification = mask_classification
        self.pe_layer = PositionEmbeddingSine(hidden_dim // 2, normalize=True)
        self.num_heads = nheads
        self.num_layers = dec_layers
        self.transformer_self_attention_layers = nn.ModuleList()
        self.transformer_cross_attention_layers = nn.ModuleList()
        self.transformer_ffn_layers = nn.ModuleList()
        for _ in range(self.num_layers):
            self.transformer_self_attention_layers.append(
                SelfAttentionLayer(d_model=hidden_dim, nhead=nheads, dropout=0.0, normalize_before=pre_norm))
            self.transformer_cross_attention_layers.append(
                CrossAttentionLayer(d_model=hidden_dim, nhead=nheads, dropout=0.0, normalize_before=pre_norm))
            self.transformer_ffn_layers.append(
                FFNLayer(d_model=hidden_dim, dim_feedforward=dim_feedforward, dropout=0.0, normalize_before=pre_norm))
        self.decoder_norm = nn.LayerNorm(hidden_dim)
        self.num_queries = num_queries
        self.query_feat = nn.Embedding(num_queries, hidden_dim)
        self.query_embed = nn.Embedding(num_queries, hidden_dim)
        self.num_feature_levels = 3
        self.level_embed = nn.Embedding(self.num_feature_levels, hidden_dim)
        self.input_proj = nn.ModuleList()
        for _ in range(self.num_feature_levels):
            if in_channels != hidden_dim or enforce_input_project:
                conv = nn.Conv2d(in_channels, hidden_dim, kernel_size=1)
                nn.init.kaiming_uniform_(conv.weight, a=1)      # fvcore's c2_xavier_fill
                nn.init.constant_(conv.bias, 0)
                self.input_proj.append(conv)
            else:
                self.input_proj.append(nn.Sequential())
        self.class_embed = nn.Linear(hidden_dim, num_classes + 1)
        self.mask_embed = MLP(hidden_dim, hidden_dim, mask_dim, 3)
        if class_embed is not None:
            self.class_embed = class_embed
        if mask_embed is not None:
            self.mask_embed = mask_embed
        if post_mask_embed is not None:
            assert mask_embed is None
        self.post_mask_embed = post_mask_embed
        self.use_fused = True          # False forces the composed path (for comparisons)
        self._casts = None             # within forward(): mask_features' detached 16-bit copy, shared by the heads
        self._fixed_up = False         # set by forward_prediction_heads: its attn_mask has no all-blocked row

    def forward(self, x, mask_features, mask=None, *, inputs_dict=None):
        assert len(x) == self.num_feature_levels
        del mask
        src, pos, size_list = [], [], []
        for i in range(self.num_feature_levels):
            size_list.append(x[i].shape[-2:])
            pos.append(self.pe_layer(x[i], None).flatten(2).permute(2, 0, 1))
            src.append((self.input_proj[i](x[i]).flatten(2) + self.level_embed.weight[i][None, :, None])
                       .permute(2, 0, 1))
        _, bs, _ = src[0].shape
        query_embed = self.query_embed.weight.unsqueeze(1).repeat(1, bs, 1)
        output = self.query_feat.weight.unsqueeze(1).repeat(1, bs, 1)
        predictions_class, predictions_mask, predictions_extra = [], [], []
        self._casts = {}
        try:
            return self._decode(output, src, pos, size_list, query_embed, mask_features, inputs_dict)
        finally:
            self._casts = None

    def _heads_step(self, output, mask_features, size, inputs_dict):
        """forward_prediction_heads as the reference's forward calls it (so a subclass's override is used), and whether
        the attention mask it returned still needs the all-blocked-row fix-up"""
        self._fixed_up = False
        res = self.forward_prediction_heads(output, mask_features, attn_mask_target_size=size, inputs_dict=inputs_dict)
        return res, self._fixed_up

    def _decode(self, output, src, pos, size_list, query_embed, mask_features, inputs_dict):
        predictions_class, predictions_mask, predictions_extra = [], [], []
        (cls, om, attn_mask, extra), fixed = self._heads_step(output, mask_features, size_list[0], inputs_dict)
        predictions_class.append(cls)
        predictions_mask.append(om)
        predictions_extra.append(extra)
        for i in range(self.num_layers):
            level_index = i % self.num_feature_levels
            if not fixed:
                attn_mask[torch.where(attn_mask.sum(-1) == attn_mask.shape[-1])] = False
            output = self.transformer_cross_attention_layers[i](
                output, src[level_index], memory_mask=attn_mask, memory_key_padding_mask=None, pos=pos[level_index],
                query_pos=query_embed)
            output = self.transformer_self_attention_layers[i](output, tgt_mask=None, tgt_key_padding_mask=None,
                                                               query_pos=query_embed)
            output = self.transformer_ffn_layers[i](output)
            (cls, om, attn_mask, extra), fixed = self._heads_step(
                output, mask_features, size_list[(i + 1) % self.num_feature_levels], inputs_dict)
            predictions_class.append(cls)
            predictions_mask.append(om)
            predictions_extra.append(extra)
        assert len(predictions_class) == self.num_layers + 1
        out = {"pred_logits": predictions_class[-1], "pred_masks": predictions_mask[-1],
               "aux_outputs": self._set_aux_loss(predictions_class, predictions_mask)}
        for k in predictions_extra[-1].keys():
            out[k] = predictions_extra[-1][k]
            for i in range(len(predictions_extra) - 1):
                out["aux_outputs"][i][k] = predictions_extra[i][k]
        return out

    def _fused_dtype(self, mask_embed, mask_features):
        """the dtype the fused path runs in, or None when the head takes the composed path"""
        pme = self.post_mask_embed
        if not (self.use_fused and mask_features.is_cuda and mask_embed.is_cuda and isinstance(pme, PooledMaskEmbed)
                and isinstance(pme.mask_pooling, MaskPooling) and pme.mask_pooling.hard_pooling):
            return None
        if mask_embed.dim() != 3 or mask_features.dim() != 4 or mask_embed.shape[0] != mask_features.shape[0]:
            return None
        if mask_embed.shape[2] != lib.MASK_HEAD_C or mask_features.shape[1] != lib.MASK_HEAD_C:
            return None
        if not 0 < mask_embed.shape[1] <= lib.MASK_HEAD_MAX_Q or mask_features.shape[2] * mask_features.shape[3] >= 2 ** 24:
            return None
        if torch.is_autocast_enabled("cuda"):
            dt = torch.get_autocast_dtype("cuda")
            return dt if dt in (torch.float16, torch.bfloat16) else None
        return torch.float32 if mask_embed.dtype == mask_features.dtype == torch.float32 else None

    def forward_prediction_heads(self, output, mask_features, attn_mask_target_size, *, inputs_dict=None):
        """-> (outputs_class, outputs_mask, attn_mask, extra_results) as the reference returns them, except that on the
        fused path attn_mask already has its all-blocked rows cleared (the decoder's next step does that in the
        reference); self._fixed_up tells forward() so."""
        decoder_output = self.decoder_norm(output).transpose(0, 1)
        outputs_class = self.class_embed(decoder_output)
        extra_results = dict()
        mask_embed_results = self.mask_embed(decoder_output)
        if isinstance(mask_embed_results, dict):
            mask_embed = mask_embed_results.pop("mask_embed")
            extra_results.update(mask_embed_results)
        else:
            mask_embed = mask_embed_results
        dt = self._fused_dtype(mask_embed, mask_features)
        if dt is not None:
            pme = self.post_mask_embed
            # one detached copy of mask_features in dt per forward; each head's gradient is returned in
            # mask_features' own dtype, so autograd sums the heads there, as it sums the reference's per-use casts
            casts = {} if self._casts is None else self._casts
            if dt not in casts:
                casts[dt] = mask_features.detach().to(dt).contiguous()
            outputs_mask, pooled, _ = MaskHeadFunction.apply(mask_embed.to(dt).contiguous(), mask_features, casts[dt],
                                                             float(pme.mask_pooling.mask_threshold))
            extra_results.update(pme.from_pooled(decoder_output, pooled))
            h, w = (int(s) for s in attn_mask_target_size)
            attn_mask = torch.ops.odise_b200.mask_head_attn_mask(outputs_mask.detach(), h, w, self.num_heads)
            self._fixed_up = True
            return outputs_class, outputs_mask, attn_mask, extra_results
        outputs_mask = torch.einsum("bqc,bchw->bqhw", mask_embed, mask_features)
        if self.post_mask_embed is not None:
            post = self.post_mask_embed(decoder_output, mask_embed, mask_features, outputs_class, outputs_mask)
            if "outputs_mask" in post:
                outputs_mask = post.pop("outputs_mask")
            extra_results.update(post)
        attn_mask = F.interpolate(outputs_mask, size=attn_mask_target_size, mode="bilinear", align_corners=False)
        attn_mask = (attn_mask.sigmoid().flatten(2).unsqueeze(1).repeat(1, self.num_heads, 1, 1).flatten(0, 1)
                     < 0.5).bool().detach()
        return outputs_class, outputs_mask, attn_mask, extra_results

    @torch.jit.unused
    def _set_aux_loss(self, outputs_class, outputs_seg_masks):
        return [{"pred_logits": a, "pred_masks": b} for a, b in zip(outputs_class[:-1], outputs_seg_masks[:-1])]
