"""Training drop-in for Mask2Former's pixel decoder (MSDeformAttnPixelDecoder and its
MSDeformAttnTransformerEncoderOnly / MSDeformAttnTransformerEncoder / MSDeformAttnTransformerEncoderLayer of
third_party/Mask2Former/mask2former/modeling/pixel_decoder/msdeformattn.py).

    from odise_b200.pixel_decoder import MSDeformAttnPixelDecoder   # in place of mask2former's

The classes keep the reference's constructor keywords and defaults (input_shape is a dict of objects with .channels and
.stride, as LazyConfig passes detectron2's ShapeSpec), submodule names, initialisation order (the same seed gives the
same parameters) and state-dict keys, so state dicts load both ways.  The attention is odise_b200.msda.MSDeformAttn and
the position encoding odise_b200.decoder.PositionEmbeddingSine.  Conv2d is detectron2's conv-with-norm/activation
(its norm's parameters under "<name>.norm").

The FPN step (msdeformattn.py:349, y = cur + F.interpolate(level, "bilinear")) runs FpnUpsampleAddFunction when both
operands are float32 CUDA tensors, autocast is off there (forward_features turns it off in training, as the reference
does) and use_fused is True: one sm_90a kernel reads the encoder level token-major in place and writes cur + the
resize, bit-equal to torch's, and the backward is a fixed-order gather without atomics, so the whole pixel decoder is
deterministic, in default mode and under torch.use_deterministic_algorithms(True) (where torch's upsample backward
raises).  Every other case (CPU, float64, eval under autocast, use_fused = False) runs the reference's F.interpolate
+ add.

The host bookkeeping uses Python ints from the input shapes: level sizes, split sections and views, and the reference
points (the reference's own linspace / division arithmetic on the device).  spatial_shapes and level_start_index are
device tensors built from those ints without a host-to-device copy and cached per (shapes, device), outside the state
dict; the encoder layers skip MSDeformAttn.forward's host check of them.  So forward and backward make no host
synchronisation and can be captured in a CUDA graph or traced by torch.compile(fullgraph=True)."""
import copy

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib
from .decoder import PositionEmbeddingSine
from .masked_attn import _activation
from .msda import MSDeformAttn

# The kernels as torch custom ops (lib.custom_op).  lib's functions are looked up at call time, so that a test that
# patches them sees every call.
lib.custom_op("fpn_upsample_add(Tensor z, Tensor cur, int h, int w) -> Tensor",
              lambda z, cur, h, w: lib.fpn_upsample_add(z, cur, (h, w)))
lib.custom_op("fpn_upsample_add_backward(Tensor grad_y, int h, int w) -> Tensor",
              lambda grad_y, h, w: lib.fpn_upsample_add_backward(grad_y, (h, w)))


class FpnUpsampleAddFunction(Function):
    """y = cur + F.interpolate(level, cur's size, "bilinear", align_corners=False) for the level z [N, h*w, C]
    (float32 CUDA, channel-contiguous rows, e.g. a token slice of the encoder's memory) and cur [N, C, H, W] (float32
    CUDA, contiguous).  Gradients: grad_z from the deterministic gather kernel, grad_cur = grad_y itself."""

    @staticmethod
    def forward(ctx, z, cur, h, w):
        ctx.hw = (h, w)
        return torch.ops.odise_b200.fpn_upsample_add(z, cur, h, w)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_y):
        h, w = ctx.hw
        return torch.ops.odise_b200.fpn_upsample_add_backward(grad_y.contiguous(), h, w), grad_y, None, None


# ---------------------------------------------------------------------------------------------- detectron2's layers
class Conv2d(nn.Conv2d):
    """detectron2.layers.Conv2d: the convolution, then the optional norm module (a child, so its parameters are
    "<name>.norm.*") and the optional activation function."""

    def __init__(self, *args, **kwargs):
        norm = kwargs.pop("norm", None)
        activation = kwargs.pop("activation", None)
        super().__init__(*args, **kwargs)
        self.norm = norm
        self.activation = activation

    def forward(self, x):
        x = F.conv2d(x, self.weight, self.bias, self.stride, self.padding, self.dilation, self.groups)
        if self.norm is not None:
            x = self.norm(x)
        if self.activation is not None:
            x = self.activation(x)
        return x


def get_norm(norm, out_channels):
    """detectron2.layers.get_norm for the norms a pixel decoder config names: None or "" -> None, "GN" ->
    GroupNorm(32, C), "BN" / "SyncBN" -> BatchNorm2d / SyncBatchNorm, or a callable of the channel count"""
    if norm is None or norm == "":
        return None
    if callable(norm):
        return norm(out_channels)
    makers = {"GN": lambda c: nn.GroupNorm(32, c), "BN": nn.BatchNorm2d, "SyncBN": nn.SyncBatchNorm}
    if norm not in makers:
        raise ValueError(f"unsupported norm {norm!r} (None, '', 'GN', 'BN', 'SyncBN' or a callable)")
    return makers[norm](out_channels)


def c2_xavier_fill(module):
    """fvcore's c2_xavier_fill: kaiming_uniform_(a=1) weight, zero bias"""
    nn.init.kaiming_uniform_(module.weight, a=1)
    if module.bias is not None:
        nn.init.constant_(module.bias, 0)


# ---------------------------------------------------------------------------------------------- the encoder
class MSDeformAttnTransformerEncoderLayer(nn.Module):
    """Deformable DETR's encoder layer: MSDeformAttn self-attention, dropout, residual, LayerNorm, then the FFN
    (linear2(dropout(act(linear1))), dropout, residual, LayerNorm)."""

    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8, n_points=4):
        super().__init__()
        self.self_attn = MSDeformAttn(d_model, n_levels, n_heads, n_points)
        self.dropout1 = nn.Dropout(dropout)
        self.norm1 = nn.LayerNorm(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.activation = _activation(activation)
        self.dropout2 = nn.Dropout(dropout)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.dropout3 = nn.Dropout(dropout)
        self.norm2 = nn.LayerNorm(d_model)

    @staticmethod
    def with_pos_embed(tensor, pos):
        return tensor if pos is None else tensor + pos

    def forward_ffn(self, src):
        src2 = self.linear2(self.dropout2(self.activation(self.linear1(src))))
        return self.norm2(src + self.dropout3(src2))

    def forward(self, src, pos, reference_points, spatial_shapes, level_start_index, padding_mask=None):
        """spatial_shapes must describe src's S tokens: the attention does not read them on the host to check"""
        src2 = self.self_attn._attend(self.with_pos_embed(src, pos), reference_points, src, spatial_shapes,
                                      level_start_index, padding_mask, check_shapes=False)
        src = self.norm1(src + self.dropout1(src2))
        return self.forward_ffn(src)


class MSDeformAttnTransformerEncoder(nn.Module):
    def __init__(self, encoder_layer, num_layers):
        super().__init__()
        self.layers = nn.ModuleList([copy.deepcopy(encoder_layer) for _ in range(num_layers)])
        self.num_layers = num_layers

    @staticmethod
    def get_reference_points(spatial_shapes, valid_ratios, device):
        """the reference's reference points: level centres in (x, y) over [0, 1], scaled by the valid ratios
        [N, L, 2].  spatial_shapes is iterated on the host: pass (h, w) ints to avoid reading a device tensor."""
        reference_points_list = []
        for lvl, (H_, W_) in enumerate(spatial_shapes):
            ref_y, ref_x = torch.meshgrid(torch.linspace(0.5, H_ - 0.5, H_, dtype=torch.float32, device=device),
                                          torch.linspace(0.5, W_ - 0.5, W_, dtype=torch.float32, device=device),
                                          indexing="ij")
            ref_y = ref_y.reshape(-1)[None] / (valid_ratios[:, None, lvl, 1] * H_)
            ref_x = ref_x.reshape(-1)[None] / (valid_ratios[:, None, lvl, 0] * W_)
            reference_points_list.append(torch.stack((ref_x, ref_y), -1))
        reference_points = torch.cat(reference_points_list, 1)
        return reference_points[:, :, None] * valid_ratios[:, None]

    def forward(self, src, spatial_shapes, level_start_index, valid_ratios, pos=None, padding_mask=None, *,
                shapes=None):
        """shapes: the levels' (h, w) as ints; without them spatial_shapes is read on the host, as the reference does"""
        if shapes is None:
            shapes = [tuple(s) for s in spatial_shapes.tolist()]
        output = src
        reference_points = self.get_reference_points(shapes, valid_ratios, device=src.device)
        for layer in self.layers:
            output = layer(output, pos, reference_points, spatial_shapes, level_start_index, padding_mask)
        return output


def level_geometry(shapes, device):
    """(spatial_shapes [L, 2] int64, level_start_index [L] int64) on `device` for the levels' (h, w) ints, written by
    fill kernels rather than copied from the host (a copy from pageable memory synchronises)"""
    starts = [0]
    for h, w in shapes[:-1]:
        starts.append(starts[-1] + h * w)

    def col(vals):
        return torch.stack([torch.full((), v, dtype=torch.long, device=device) for v in vals])

    return col([v for hw in shapes for v in hw]).view(len(shapes), 2), col(starts)


class MSDeformAttnTransformerEncoderOnly(nn.Module):
    def __init__(self, d_model=256, nhead=8, num_encoder_layers=6, dim_feedforward=1024, dropout=0.1,
                 activation="relu", num_feature_levels=4, enc_n_points=4):
        super().__init__()
        self.d_model = d_model
        self.nhead = nhead
        encoder_layer = MSDeformAttnTransformerEncoderLayer(d_model, dim_feedforward, dropout, activation,
                                                            num_feature_levels, nhead, enc_n_points)
        self.encoder = MSDeformAttnTransformerEncoder(encoder_layer, num_encoder_layers)
        self.level_embed = nn.Parameter(torch.Tensor(num_feature_levels, d_model))
        self._geometry = {}            # (shapes, device) -> (spatial_shapes, level_start_index); not module state
        self._reset_parameters()

    def _reset_parameters(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if isinstance(m, MSDeformAttn):
                m._reset_parameters()
        nn.init.normal_(self.level_embed)

    def get_valid_ratio(self, mask):
        _, H, W = mask.shape
        valid_H = torch.sum(~mask[:, :, 0], 1)
        valid_W = torch.sum(~mask[:, 0, :], 1)
        return torch.stack([valid_W.float() / W, valid_H.float() / H], -1)

    def level_geometry(self, shapes, device):
        """level_geometry(shapes, device), cached in eager mode; a traced graph builds it in the graph"""
        if torch.compiler.is_compiling():
            return level_geometry(shapes, device)
        key = (tuple(shapes), device)
        if key not in self._geometry:
            self._geometry[key] = level_geometry(shapes, device)
        return self._geometry[key]

    def forward(self, srcs, pos_embeds):
        """srcs, pos_embeds: per level [N, C, h, w] -> (memory [N, S, C], spatial_shapes [L, 2], level_start_index
        [L]).  The reference's all-False padding masks are dropped: masking nothing changes no value and no gradient,
        and their valid ratios are exactly 1."""
        shapes = [(int(s.shape[2]), int(s.shape[3])) for s in srcs]
        src_flatten = torch.cat([s.flatten(2).transpose(1, 2) for s in srcs], 1)
        lvl_pos_embed_flatten = torch.cat([p.flatten(2).transpose(1, 2) + self.level_embed[lvl].view(1, 1, -1)
                                           for lvl, p in enumerate(pos_embeds)], 1)
        spatial_shapes, level_start_index = self.level_geometry(shapes, src_flatten.device)
        valid_ratios = src_flatten.new_ones(src_flatten.shape[0], len(srcs), 2, dtype=torch.float32)
        memory = self.encoder(src_flatten, spatial_shapes, level_start_index, valid_ratios, lvl_pos_embed_flatten,
                              None, shapes=shapes)
        return memory, spatial_shapes, level_start_index


# ---------------------------------------------------------------------------------------------- the pixel decoder
class MSDeformAttnPixelDecoder(nn.Module):
    """Mask2Former's MSDeformAttnPixelDecoder; see the module docstring for the fused FPN step.  use_fused = False
    forces the reference's F.interpolate + add (for comparisons)."""

    def __init__(self, input_shape, *, transformer_dropout, transformer_nheads, transformer_dim_feedforward,
                 transformer_enc_layers, conv_dim, mask_dim, norm=None, transformer_in_features, common_stride):
        super().__init__()
        transformer_input_shape = {k: v for k, v in input_shape.items() if k in transformer_in_features}
        input_shape = sorted(input_shape.items(), key=lambda x: x[1].stride)
        self.in_features = [k for k, v in input_shape]
        self.feature_strides = [v.stride for k, v in input_shape]
        self.feature_channels = [v.channels for k, v in input_shape]
        transformer_input_shape = sorted(transformer_input_shape.items(), key=lambda x: x[1].stride)
        self.transformer_in_features = [k for k, v in transformer_input_shape]
        transformer_in_channels = [v.channels for k, v in transformer_input_shape]
        self.transformer_feature_strides = [v.stride for k, v in transformer_input_shape]
        self.transformer_num_feature_levels = len(self.transformer_in_features)
        # from low to high resolution (res5 -> res2); one level takes the last channel count, as in the reference
        in_list = transformer_in_channels[::-1] if self.transformer_num_feature_levels > 1 else \
            transformer_in_channels[-1:]
        self.input_proj = nn.ModuleList([nn.Sequential(nn.Conv2d(c, conv_dim, kernel_size=1), nn.GroupNorm(32, conv_dim))
                                         for c in in_list])
        for proj in self.input_proj:
            nn.init.xavier_uniform_(proj[0].weight, gain=1)
            nn.init.constant_(proj[0].bias, 0)
        self.transformer = MSDeformAttnTransformerEncoderOnly(
            d_model=conv_dim, dropout=transformer_dropout, nhead=transformer_nheads,
            dim_feedforward=transformer_dim_feedforward, num_encoder_layers=transformer_enc_layers,
            num_feature_levels=self.transformer_num_feature_levels)
        self.pe_layer = PositionEmbeddingSine(conv_dim // 2, normalize=True)
        self.mask_dim = mask_dim
        self.mask_features = Conv2d(conv_dim, mask_dim, kernel_size=1, stride=1, padding=0)
        c2_xavier_fill(self.mask_features)
        self.maskformer_num_feature_levels = 3  # always use 3 scales
        self.common_stride = common_stride
        stride = min(self.transformer_feature_strides)
        self.num_fpn_levels = int(np.log2(stride) - np.log2(self.common_stride))
        lateral_convs, output_convs = [], []
        use_bias = norm == ""
        for idx, in_channels in enumerate(self.feature_channels[:self.num_fpn_levels]):
            lateral_norm = get_norm(norm, conv_dim)
            output_norm = get_norm(norm, conv_dim)
            lateral_conv = Conv2d(in_channels, conv_dim, kernel_size=1, bias=use_bias, norm=lateral_norm)
            output_conv = Conv2d(conv_dim, conv_dim, kernel_size=3, stride=1, padding=1, bias=use_bias,
                                 norm=output_norm, activation=F.relu)
            c2_xavier_fill(lateral_conv)
            c2_xavier_fill(output_conv)
            self.add_module("adapter_{}".format(idx + 1), lateral_conv)
            self.add_module("layer_{}".format(idx + 1), output_conv)
            lateral_convs.append(lateral_conv)
            output_convs.append(output_conv)
        # top-down order (from low to high resolution)
        self.lateral_convs = lateral_convs[::-1]
        self.output_convs = output_convs[::-1]
        self.use_fused = True          # False forces the composed FPN step (for comparisons)

    def _fused(self, prev, cur):
        """whether the FPN step of prev [N, C, h, w] onto cur takes FpnUpsampleAddFunction"""
        if not (self.use_fused and prev.is_cuda and cur.is_cuda and prev.dtype == cur.dtype == torch.float32):
            return False
        if torch.is_autocast_enabled("cuda") or prev.dim() != 4 or cur.dim() != 4:
            return False
        (N, C, h, w), (H, W) = prev.shape, cur.shape[-2:]
        return (tuple(cur.shape[:2]) == (N, C) and C % lib.FPN_C_MULTIPLE == 0 and N * C // lib.FPN_C_MULTIPLE <= 65535
                and max(H, h) <= 65535 and h * w * C < 2 ** 31)

    def _fpn_add(self, prev, z, cur):
        """cur + F.interpolate(prev, cur's size, "bilinear"); z is prev's token-major [N, h*w, C] form when prev is an
        encoder level, None when it is an FPN output"""
        if self._fused(prev, cur):
            h, w = prev.shape[-2:]
            if z is None:
                z = prev.flatten(2).transpose(1, 2).contiguous()
            return FpnUpsampleAddFunction.apply(z, cur.contiguous(), h, w)
        return cur + F.interpolate(prev, size=cur.shape[-2:], mode="bilinear", align_corners=False)

    def forward_features(self, features):
        """features: name -> [N, C_in, H, W] -> (mask_features, out[0], the first 3 multi-scale maps)"""
        with torch.autocast("cuda", enabled=not self.training and torch.is_autocast_enabled("cuda")):
            srcs, pos = [], []
            for idx, f in enumerate(self.transformer_in_features[::-1]):
                x = features[f].float()  # deformable detr does not support half precision
                srcs.append(self.input_proj[idx](x))
                pos.append(self.pe_layer(x))
            y, spatial_shapes, level_start_index = self.transformer(srcs, pos)
            bs = y.shape[0]
            shapes = [(int(s.shape[2]), int(s.shape[3])) for s in srcs]
            tokens = list(torch.split(y, [h * w for h, w in shapes], dim=1))
            out = [z.transpose(1, 2).view(bs, -1, h, w) for z, (h, w) in zip(tokens, shapes)]
            for idx, f in enumerate(self.in_features[:self.num_fpn_levels][::-1]):
                x = features[f].float()
                cur_fpn = self.lateral_convs[idx](x)
                y = self.output_convs[idx](self._fpn_add(out[-1], tokens[-1], cur_fpn))
                out.append(y)
                tokens.append(None)
            multi_scale_features = out[:self.maskformer_num_feature_levels]
            return self.mask_features(out[-1]), out[0], multi_scale_features
