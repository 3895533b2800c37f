"""H100 engine for the Mask2Former half of ODISE (SURVEY.md §8a rows b1-b12): MSDeformAttn pixel decoder
(M2F/modeling/pixel_decoder/msdeformattn.py:314-358), ODISE masked-attention transformer decoder with its pooled
mask-embedding heads (odise/modeling/meta_arch/odise.py:642-776, :937-1015) and the CLIP-text scoring
(odise.py:181-207, helper.py:79-109).

Token-major fp32 activations + (hi, lo) bf16 GEMM operands; every contraction is odise_gemm_bf16 (wgmma), the
deformable sampling is odise_msda_fused_f32 (softmax + location math + bilinear gathers in one kernel), the masked
cross-attention never materialises the [B*8, Q, HW] boolean mask (1 bit per (b, q, key), shared by the heads), and
K / V of the three decoder layers that share a feature level come out of ONE GEMM per level.
"""
import math

import torch

from . import lib, ops
from .lib import Planes
from .ops import ACT_RELU

M_HEADS, D_HEAD, N_POINTS, N_LEVELS = 8, 32, 4, 3


def pos_sine(H, W, num_pos_feats=128, temperature=10000.0):
    """PositionEmbeddingSine(normalize=True) for an unmasked H x W map -> [H*W, 2*num_pos_feats] (token-major).
    Input independent, so it is folded once per resolution on the host (position_encoding.py:29-52)."""
    scale, eps = 2 * math.pi, 1e-6
    y = torch.arange(1, H + 1, dtype=torch.float32).view(H, 1).expand(H, W)
    x = torch.arange(1, W + 1, dtype=torch.float32).view(1, W).expand(H, W)
    y = y / (y[-1:, :] + eps) * scale
    x = x / (x[:, -1:] + eps) * scale
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    px, py = x[:, :, None] / dim_t, y[:, :, None] / dim_t
    px = torch.stack((px[:, :, 0::2].sin(), px[:, :, 1::2].cos()), dim=3).flatten(2)
    py = torch.stack((py[:, :, 0::2].sin(), py[:, :, 1::2].cos()), dim=3).flatten(2)
    return torch.cat((py, px), dim=2).reshape(H * W, 2 * num_pos_feats)


def ref_points(shapes):
    """get_reference_points with valid_ratios == 1 (msdeformattn.py:141-153): pixel centres / (W, H) -> [S, L, 2]."""
    pts = []
    for H, W in shapes:
        ry = torch.linspace(0.5, H - 0.5, H, dtype=torch.float32)
        rx = torch.linspace(0.5, W - 0.5, W, dtype=torch.float32)
        gy, gx = torch.meshgrid(ry, rx, indexing="ij")
        pts.append(torch.stack((gx.reshape(-1) / W, gy.reshape(-1) / H), -1))
    ref = torch.cat(pts, 0)
    return ref[:, None, :].expand(-1, len(shapes), -1).contiguous()


class HeadEngine:
    def __init__(self, sd, device, nmma=3, pd_prefix="sem_seg_head.pixel_decoder.",
                 dec_prefix="sem_seg_head.predictor.", cat_prefix="category_head.", n_enc=6, n_dec=9, num_queries=100):
        self.dev = torch.device(device)
        # The head stays in the bf16x3 parity mode when the rest of the pipeline runs F16Q8 (nmma = 2): its outputs feed hard
        # thresholds (mask > 0 pooling, attention-mask bits) and it is < 6 % of the tensor time.
        nmma = 3 if nmma == 2 else nmma
        self.nmma, self.lo = nmma, nmma == 3
        self.n_enc, self.n_dec, self.Q = n_enc, n_dec, num_queries
        self.W, self.F = {}, {}
        self._geo = {}
        self._vocab = {}
        self._prep(sd, pd_prefix, dec_prefix, cat_prefix)

    # ------------------------------------------------------------------------------------------- weights
    def _planes(self, w):
        return lib.split(w.to(self.dev, torch.float32).contiguous(), lo=self.lo)

    def _f(self, t):
        return t.to(self.dev, torch.float32).contiguous()

    def _lin(self, name, w, b=None):
        self.W[name] = self._planes(w.reshape(w.shape[0], -1))
        if b is not None:
            self.F[name + ".b"] = self._f(b)

    def _norm(self, name, sd, key):
        self.F[name + ".g"], self.F[name + ".be"] = self._f(sd[key + ".weight"]), self._f(sd[key + ".bias"])

    def _prep(self, sd, pp, dp, cp):
        for i in range(3):
            self._lin(f"pd.in{i}", sd[f"{pp}input_proj.{i}.0.weight"], sd[f"{pp}input_proj.{i}.0.bias"])
            self._norm(f"pd.in{i}.gn", sd, f"{pp}input_proj.{i}.1")
        self.pd_level_embed = sd[pp + "transformer.level_embed"].float()
        for l in range(self.n_enc):
            q = f"{pp}transformer.encoder.layers.{l}."
            n = f"pd.l{l}."
            for a in ("sampling_offsets", "attention_weights", "value_proj", "output_proj"):
                self._lin(n + a, sd[q + f"self_attn.{a}.weight"], sd[q + f"self_attn.{a}.bias"])
            self._lin(n + "linear1", sd[q + "linear1.weight"], sd[q + "linear1.bias"])
            self._lin(n + "linear2", sd[q + "linear2.weight"], sd[q + "linear2.bias"])
            self._norm(n + "norm1", sd, q + "norm1")
            self._norm(n + "norm2", sd, q + "norm2")
        self._lin("pd.adapter", sd[pp + "adapter_1.weight"])
        self._norm("pd.adapter.gn", sd, pp + "adapter_1.norm")
        self.W["pd.layer"] = self._planes(sd[pp + "layer_1.weight"].permute(0, 2, 3, 1).reshape(256, -1))
        self._norm("pd.layer.gn", sd, pp + "layer_1.norm")
        self._lin("pd.mask_features", sd[pp + "mask_features.weight"], sd[pp + "mask_features.bias"])
        # decoder
        C = 256
        self.dec_level_embed = sd[dp + "level_embed.weight"].float()
        # num_feature_levels of the decoder (mask2former_transformer_decoder.py:296: 3 in every ODISE config; the C4
        # microbench of BASELINE.json runs 4 scales) and the query count come from the weights
        self.n_lvl = int(self.dec_level_embed.shape[0])
        self.F["query_embed"] = self._f(sd[dp + "query_embed.weight"])
        self.query_feat = sd[dp + "query_feat.weight"].float()
        if self.query_feat.shape[0] != self.Q:
            raise lib.OdiseError(f"num_queries = {self.Q} but query_feat has {self.query_feat.shape[0]} rows")
        for lvl in range(self.n_lvl):   # K / V projections of the layers that read level lvl, concatenated along N and
            # head-padded 32 -> 64 columns per head (zero rows): the operands of the wgmma attention kernel
            ids = [i for i in range(self.n_dec) if i % self.n_lvl == lvl]
            pad = lambda w: ops.head_pad_rows(w, M_HEADS, D_HEAD, 64)
            padb = lambda b: ops.head_pad_rows(b.view(-1, 1), M_HEADS, D_HEAD, 64).view(-1)
            wk = torch.cat([pad(sd[f"{dp}transformer_cross_attention_layers.{i}.multihead_attn.in_proj_weight"][C:2 * C]) for i in ids])
            bk = torch.cat([padb(sd[f"{dp}transformer_cross_attention_layers.{i}.multihead_attn.in_proj_bias"][C:2 * C]) for i in ids])
            wv = torch.cat([pad(sd[f"{dp}transformer_cross_attention_layers.{i}.multihead_attn.in_proj_weight"][2 * C:]) for i in ids])
            bv = torch.cat([padb(sd[f"{dp}transformer_cross_attention_layers.{i}.multihead_attn.in_proj_bias"][2 * C:]) for i in ids])
            self._lin(f"dec.k{lvl}", wk, bk)
            self._lin(f"dec.v{lvl}", wv, bv)
        for i in range(self.n_dec):
            c, s, f = (f"{dp}transformer_cross_attention_layers.{i}.", f"{dp}transformer_self_attention_layers.{i}.",
                       f"{dp}transformer_ffn_layers.{i}.")
            n = f"dec.l{i}."
            w, b = sd[c + "multihead_attn.in_proj_weight"], sd[c + "multihead_attn.in_proj_bias"]
            self._lin(n + "cq", ops.head_pad_rows(w[:C], M_HEADS, D_HEAD, 64),
                      ops.head_pad_rows(b[:C].view(-1, 1), M_HEADS, D_HEAD, 64).view(-1))
            self._lin(n + "co", sd[c + "multihead_attn.out_proj.weight"], sd[c + "multihead_attn.out_proj.bias"])
            self._norm(n + "cn", sd, c + "norm")
            w, b = sd[s + "self_attn.in_proj_weight"], sd[s + "self_attn.in_proj_bias"]
            self._lin(n + "sqk", w[:2 * C], b[:2 * C])
            self._lin(n + "sv", w[2 * C:], b[2 * C:])
            self._lin(n + "so", sd[s + "self_attn.out_proj.weight"], sd[s + "self_attn.out_proj.bias"])
            self._norm(n + "sn", sd, s + "norm")
            self._lin(n + "f1", sd[f + "linear1.weight"], sd[f + "linear1.bias"])
            self._lin(n + "f2", sd[f + "linear2.weight"], sd[f + "linear2.bias"])
            self._norm(n + "fn", sd, f + "norm")
        self._norm("dec.norm", sd, dp + "decoder_norm")
        for j in range(3):
            self._lin(f"dec.me{j}", sd[f"{dp}mask_embed.layers.{j}.weight"], sd[f"{dp}mask_embed.layers.{j}.bias"])
            self._lin(f"dec.pme{j}", sd[f"{dp}post_mask_embed.mask_embed.1.layers.{j}.weight"],
                      sd[f"{dp}post_mask_embed.mask_embed.1.layers.{j}.bias"])
        self._norm("dec.pool_ln", sd, dp + "post_mask_embed.pool_proj.0")
        self._lin("dec.pool_proj", sd[dp + "post_mask_embed.pool_proj.1.weight"], sd[dp + "post_mask_embed.pool_proj.1.bias"])
        self._norm("dec.pme_ln", sd, dp + "post_mask_embed.mask_embed.0")
        # logit_scale = clamp(exp(s), max=100)  (odise.py:1004)
        self.logit_scale = float(min(math.exp(float(sd[dp + "post_mask_embed.logit_scale"])), 100.0))
        if cp + "text_proj.weight" in sd:
            self._lin("cat.text_proj", sd[cp + "text_proj.weight"], sd[cp + "text_proj.bias"])

    def _gemm(self, a, wname, bias=True, **kw):
        b = self.F.get(wname + ".b") if bias else None
        return lib.gemm(a, self.W[wname], nmma=self.nmma, bias=b, **kw)

    def _ln(self, x, name, **kw):
        return ops.layer_norm(x, self.F[name + ".g"], self.F[name + ".be"], lo=self.lo, **kw)

    # ------------------------------------------------------------------------------------------- geometry consts
    def _geometry(self, B, shapes):
        key = (B, tuple(shapes))
        if key in self._geo:
            return self._geo[key]
        dev = self.dev
        S = sum(h * w for h, w in shapes)
        starts = [0]
        for h, w in shapes[:-1]:
            starts.append(starts[-1] + h * w)
        pos = [pos_sine(h, w) for h, w in shapes]
        g = dict(S=S, starts=starts)
        if len(shapes) <= self.pd_level_embed.shape[0]:       # the pixel decoder's own levels (absent for decoder-only use)
            g["pd_pos"] = torch.cat([p + self.pd_level_embed[i][None] for i, p in enumerate(pos)], 0).to(dev)
        g["dec_kpos"] = torch.cat([p + self.dec_level_embed[i][None] for i, p in enumerate(pos)], 0).to(dev)
        g["dec_lvl"] = torch.cat([self.dec_level_embed[i][None].expand(h * w, -1) for i, (h, w) in enumerate(shapes)], 0).contiguous().to(dev)
        g["ref"] = ref_points(shapes)[None].expand(B, -1, -1, -1).contiguous().to(dev)
        g["ss"] = torch.as_tensor(shapes, dtype=torch.int64).to(dev)
        g["lsi"] = torch.as_tensor(starts, dtype=torch.int64).to(dev)
        g["query0"] = self.query_feat[None].expand(B, -1, -1).reshape(B * self.Q, -1).contiguous().to(dev)
        self._geo[key] = g
        return g

    # ------------------------------------------------------------------------------------------- pixel decoder
    @torch.no_grad()
    def pixel_decoder(self, feats, B, want_mask_features_f32=False):
        """feats: {"s2".."s5": (NHWC fp32 [B*h*w, 512], h, w)}.  Returns a dict with the encoder memory
        (token-major, levels s5|s4|s3), mask features as GEMM operands (and fp32 on request)."""
        dev = self.dev
        names = ["s5", "s4", "s3"]
        shapes = [(feats[n][1], feats[n][2]) for n in names]
        g = self._geometry(B, shapes)
        S, starts = g["S"], g["starts"]
        src = ops.empty(B * S, 256, dev)
        for i, n in enumerate(names):
            x, h, w = feats[n]
            t, ts = ops.empty(B * h * w, 256, dev), lib.GnStats(B * h * w, 256, dev)
            self._gemm(ops.split(x, lo=self.lo), f"pd.in{i}", out=t, gn=ts)
            ops.group_norm(t, B, h * w, self.F[f"pd.in{i}.gn.g"], self.F[f"pd.in{i}.gn.be"], 1e-5, want_planes=False,
                           y=src[starts[i]:], ldy=256, y_bs=S * 256, stats=ts)
        src_p = ops.split(src, lo=self.lo)
        for l in range(self.n_enc):
            n = f"pd.l{l}."
            _, q_p = ops.add_split(src, g["pd_pos"], b_rows=S, lo=self.lo)
            value = ops.empty(B * S, 256, dev)
            self._gemm(src_p, n + "value_proj", out=value)
            offs = ops.empty(B * S, M_HEADS * N_LEVELS * N_POINTS * 2, dev)
            self._gemm(q_p, n + "sampling_offsets", out=offs)
            logits = ops.empty(B * S, M_HEADS * N_LEVELS * N_POINTS, dev)
            self._gemm(q_p, n + "attention_weights", out=logits)
            _, o_p = ops.msda_fused(value, g["ss"], g["lsi"], g["ref"], offs, logits, B, S, M_HEADS, D_HEAD, N_LEVELS, S,
                                    N_POINTS, lo=self.lo)
            t = ops.empty(B * S, 256, dev)
            self._gemm(o_p, n + "output_proj", residual=src, out=t)
            y, y_p = self._ln(t, n + "norm1", want_f32=True)
            f_p = Planes.empty(B * S, 1024, dev, lo=self.lo)
            self._gemm(y_p, n + "linear1", act=ACT_RELU, out_planes=f_p)
            t2 = ops.empty(B * S, 256, dev)
            self._gemm(f_p, n + "linear2", residual=y, out=t2)
            src, src_p = self._ln(t2, n + "norm2", want_f32=True)
        # FPN level on s2 (msdeformattn.py:343-351)
        x2, h2, w2 = feats["s2"]
        h3, w3 = shapes[2]
        lat, lat_s = ops.empty(B * h2 * w2, 256, dev), lib.GnStats(B * h2 * w2, 256, dev)
        self._gemm(ops.split(x2, lo=self.lo), "pd.adapter", bias=False, out=lat, gn=lat_s)
        cur, _ = ops.group_norm(lat, B, h2 * w2, self.F["pd.adapter.gn.g"], self.F["pd.adapter.gn.be"], 1e-5,
                                want_f32=True, want_planes=False, stats=lat_s)
        ops.resize_nhwc(src[starts[2]:], B, h3, w3, h2, w2, True, dst=cur, accumulate=True, src_bs=S * 256)
        conv, conv_s = ops.empty(B * h2 * w2, 256, dev), lib.GnStats(B * h2 * w2, 256, dev)
        self._gemm(ops.split(cur, lo=self.lo), "pd.layer", bias=False, M=B * h2 * w2, N=256, conv=(256, h2, w2), out=conv,
                   gn=conv_s)
        _, y2_p = ops.group_norm(conv, B, h2 * w2, self.F["pd.layer.gn.g"], self.F["pd.layer.gn.be"], 1e-5, ACT_RELU,
                                 lo=self.lo, stats=conv_s)
        HW = h2 * w2
        mf_p = Planes.empty(B * HW, 256, dev, lo=self.lo)                 # [B*HW, C]: B operand of the mask einsum
        mf = ops.empty(B * HW, 256, dev) if want_mask_features_f32 else None
        self._gemm(y2_p, "pd.mask_features", out=mf, out_planes=mf_p)
        mft_p = Planes.empty(256, B * HW, dev, lo=self.lo)                 # [C, B*HW]: B operand of the pooling
        lib.gemm(self.W["pd.mask_features"], y2_p, nmma=self.nmma, bias_m=self.F["pd.mask_features.b"], out_planes=mft_p)
        return dict(memory=src, memory_p=src_p, shapes=shapes, geo=g, mf_p=mf_p, mft_p=mft_p, mf=mf, mask_hw=(h2, w2))

    @torch.no_grad()
    def pd_from_tensors(self, multi_scale, mask_features):
        """The decoder's inputs from the plugin boundary (ODISEMultiScaleMaskedTransformerDecoder.forward(x, mask_features),
        odise.py:642-660): x = 3 NCHW maps [B, 256, h, w] (coarse -> fine), mask_features NCHW [B, 256, H/4, W/4]
        -> the dict transformer_decoder() consumes (token-major memory of the levels, mask features as GEMM operands)."""
        dev = self.dev
        B = mask_features.shape[0]
        shapes = [(int(t.shape[2]), int(t.shape[3])) for t in multi_scale]
        g = self._geometry(B, shapes)
        S, starts = g["S"], g["starts"]
        mem = ops.empty(B * S, 256, dev)
        for i, t in enumerate(multi_scale):
            h, w = shapes[i]
            lvl = ops.nchw_to_nhwc(t.float())
            ops.copy2d(lvl.view(B, h * w * 256), mem.view(B, S * 256)[:, starts[i] * 256:(starts[i] + h * w) * 256])
        h2, w2 = int(mask_features.shape[2]), int(mask_features.shape[3])
        HW = h2 * w2
        mf = ops.nchw_to_nhwc(mask_features.float())                       # [B*HW, 256]
        mf_p = ops.split(mf, lo=self.lo)
        mft = ops.empty(256, B * HW, dev)                                  # [C, B*HW]: image z at column offset z*HW
        src = mask_features.float().contiguous().view(B, 256, HW)
        for z in range(B):
            ops.copy2d(src[z], mft[:, z * HW:(z + 1) * HW])
        mft_p = ops.split(mft, lo=self.lo)
        return dict(memory=mem, memory_p=None, shapes=shapes, geo=g, mf_p=mf_p, mft_p=mft_p, mf=mf, mask_hw=(h2, w2))

    # ------------------------------------------------------------------------------------------- decoder
    def _mlp3(self, x_p, base, rows, out_f32):
        a = Planes.empty(rows, 256, self.dev, lo=self.lo)
        self._gemm(x_p, base + "0", act=ACT_RELU, out_planes=a)
        b = Planes.empty(rows, 256, self.dev, lo=self.lo)
        self._gemm(a, base + "1", act=ACT_RELU, out_planes=b)
        if out_f32:
            o = ops.empty(rows, 256, self.dev)
            self._gemm(b, base + "2", out=o)
            return o
        o = Planes.empty(rows, 256, self.dev, lo=self.lo)
        self._gemm(b, base + "2", out_planes=o)
        return o

    def _pred_head(self, output, pd, B, next_level_hw, forced_masks=None):
        """forward_prediction_heads + PooledMaskEmbed (odise.py:729-776, :984-1015).
        forced_masks: teacher-forced mask logits for the two thresholds (tests; discontinuity control)."""
        Q, dev = self.Q, self.dev
        h2, w2 = pd["mask_hw"]
        HW = h2 * w2
        dec, dec_p = self._ln(output, "dec.norm", want_f32=True)
        me_p = self._mlp3(dec_p, "dec.me", B * Q, out_f32=False)
        masks = torch.empty(B, Q, HW, dtype=torch.float32, device=dev)
        lib.gemm(me_p, pd["mf_p"], M=Q, N=HW, K=256, nmma=self.nmma, batch=B, a_bs=Q * me_p.ld, b_bs=HW * pd["mf_p"].ld,
                 out=masks, ld_out=HW, out_bs=Q * HW)
        thr = masks if forced_masks is None else forced_masks
        binp, counts = ops.mask_binarize(thr, B, Q, HW)
        # pooled sums = binary mask [Q, HW] x mask_features^T [C, HW]^T ; the 0/1 mask is exact in one bf16 plane
        bin_p = Planes(binp, None, B * Q, HW, HW)
        mft = pd["mft_p"]
        split_k = 16 if HW >= 4096 else 1
        ws = torch.empty(split_k * B * Q * 256, dtype=torch.float32, device=dev) if split_k > 1 else None
        sums = torch.empty(B, Q, 256, dtype=torch.float32, device=dev)
        lib.gemm(bin_p, Planes(mft.hi, None, 256, HW, mft.ld), M=Q, N=256, K=HW, nmma=1, batch=B, a_bs=Q * HW, b_bs=HW,
                 out=sums, ld_out=256, out_bs=Q * 256, split_k=split_k, workspace=ws)
        if self.lo:
            sums2 = torch.empty_like(sums)
            lib.gemm(bin_p, Planes(mft.lo, None, 256, HW, mft.ld), M=Q, N=256, K=HW, nmma=1, batch=B, a_bs=Q * HW,
                     b_bs=HW, residual=sums, ld_res=256, res_bs=Q * 256, out=sums2, ld_out=256, out_bs=Q * 256,
                     split_k=split_k, workspace=ws)
            sums = sums2
        pooled = ops.pool_normalize(sums, counts, B, Q, 256)
        _, pp = self._ln(pooled, "dec.pool_ln")
        mpf = ops.empty(B * Q, 256, dev)
        self._gemm(pp, "dec.pool_proj", residual=dec, out=mpf)
        _, ep = self._ln(mpf, "dec.pme_ln")
        mask_embed = self._mlp3(ep, "dec.pme", B * Q, out_f32=True)
        bits = row_any = None
        if next_level_hw is not None:
            bits, row_any = ops.attn_mask_bits(thr, B, Q, h2, w2, next_level_hw[0], next_level_hw[1])
        return dict(pred_masks=masks, mask_embed=mask_embed, mask_pooled_features=mpf), bits, row_any

    @torch.no_grad()
    def transformer_decoder(self, pd, B, forced_masks=None):
        """ODISEMultiScaleMaskedTransformerDecoder.forward (odise.py:642-727) on the pixel-decoder outputs."""
        dev, Q = self.dev, self.Q
        g, shapes = pd["geo"], pd["shapes"]
        S, starts = g["S"], g["starts"]
        mem = pd["memory"]
        _, kin_p = ops.add_split(mem, g["dec_kpos"], b_rows=S, lo=self.lo)
        _, vin_p = ops.add_split(mem, g["dec_lvl"], b_rows=S, lo=self.lo)
        K, V = [], []
        CP = M_HEADS * 64                      # head-padded width of one layer's K / V
        nl = self.n_lvl
        if len(shapes) != nl:
            raise lib.OdiseError(f"the decoder has {nl} feature levels, got {len(shapes)} maps")
        for lvl, (h, w) in enumerate(shapes):
            hw = h * w
            nk = self.W[f"dec.k{lvl}"].rows // CP                         # layers reading this level (i % nl == lvl)
            k = Planes.empty(B * hw, nk * CP, dev, lo=self.lo)           # [B*hw, nk layers x 8 heads x 64]
            lib.gemm(kin_p.row_slice(starts[lvl], hw), self.W[f"dec.k{lvl}"], M=hw, N=nk * CP, K=256, nmma=self.nmma,
                     batch=B, a_bs=S * kin_p.ld, bias=self.F[f"dec.k{lvl}.b"], out_planes=k, outp_bs=hw * k.ld)
            # V^T [nk*CP, B*hw]: swapped operands, image z lands at column offset z*hw
            vt = Planes.empty(nk * CP, B * hw, dev, lo=self.lo, f16=self.lo)
            lib.gemm(self.W[f"dec.v{lvl}"], vin_p.row_slice(starts[lvl], hw), M=nk * CP, N=hw, K=256, nmma=self.nmma,
                     batch=B, b_bs=S * vin_p.ld, bias_m=self.F[f"dec.v{lvl}.b"], out_planes=vt, outp_bs=hw)
            K.append(k)
            V.append(vt)
        fm = (lambda i: None) if forced_masks is None else (lambda i: forced_masks[i])
        output = g["query0"]
        heads = []
        res, bits, row_any = self._pred_head(output, pd, B, shapes[0], fm(0))
        heads.append(res)
        scale = D_HEAD ** -0.5
        qe = self.F["query_embed"]
        for i in range(self.n_dec):
            lvl, slot = i % nl, i // nl
            hw = shapes[lvl][0] * shapes[lvl][1]
            n = f"dec.l{i}."
            # masked cross-attention (mask2former_transformer_decoder.py:98-110, odise.py:683-692)
            _, qin_p = ops.add_split(output, qe, b_rows=Q, lo=self.lo)
            qc = Planes.empty(B * Q, CP, dev, lo=self.lo)
            self._gemm(qin_p, n + "cq", out_planes=qc)
            _, o_p = ops.attention_tc(qc, K[lvl].col_slice(slot * CP, CP), V[lvl].row_slice(slot * CP, CP), B, M_HEADS,
                                      D_HEAD, Q, hw, scale, self.nmma, tk_stride=hw, mask_bits=bits, row_any=row_any)
            t = ops.empty(B * Q, 256, dev)
            self._gemm(o_p, n + "co", residual=output, out=t)
            output, _ = self._ln(t, n + "cn", want_f32=True, want_planes=False)
            # self-attention
            _, qk_p = ops.add_split(output, qe, b_rows=Q, lo=self.lo)
            out_p = ops.split(output, lo=self.lo)
            qkv = ops.empty(B * Q, 768, dev)
            self._gemm(qk_p, n + "sqk", out=qkv[:, :512], ld_out=768)
            self._gemm(out_p, n + "sv", out=qkv[:, 512:], ld_out=768)
            o_p = ops.mha_d32(qkv, 768, qkv[:, 256:], qkv[:, 512:], 768, B, Q, Q, M_HEADS, scale, lo=self.lo)
            t = ops.empty(B * Q, 256, dev)
            self._gemm(o_p, n + "so", residual=output, out=t)
            output, out_p = self._ln(t, n + "sn", want_f32=True)
            # FFN
            f_p = Planes.empty(B * Q, 2048, dev, lo=self.lo)
            self._gemm(out_p, n + "f1", act=ACT_RELU, out_planes=f_p)
            t = ops.empty(B * Q, 256, dev)
            self._gemm(f_p, n + "f2", residual=output, out=t)
            output, _ = self._ln(t, n + "fn", want_f32=True, want_planes=False)
            nxt = shapes[(i + 1) % nl] if i + 1 < self.n_dec else None
            res, bits, row_any = self._pred_head(output, pd, B, nxt, fm(i + 1))
            heads.append(res)
        return heads

    # ------------------------------------------------------------------------------------------- scoring
    def set_vocabulary(self, key, text_bank, null_bank, group_sizes):
        """CategoryEmbed eval branch (odise.py:1298-1307): text_proj of the cached CLIP text bank [K', 768] and of the
        null embedding, L2-normalised once per vocabulary (they are constants of the vocabulary)."""
        dev = self.dev
        tb = self._f(text_bank)
        te = ops.empty(tb.shape[0], 256, dev)
        self._gemm(ops.split(tb, lo=self.lo), "cat.text_proj", out=te)
        ne = ops.empty(1, 256, dev)
        self._gemm(ops.split(self._f(null_bank).view(1, -1), lo=self.lo), "cat.text_proj", out=ne)
        gs = torch.zeros(len(group_sizes) + 1, dtype=torch.int32)
        gs[1:] = torch.as_tensor(group_sizes, dtype=torch.int32).cumsum(0)
        self._vocab[key] = dict(te=te, ne=ne, te_p=ops.l2_normalize_split(te, lo=self.lo),
                                ne_p=ops.l2_normalize_split(ne, lo=self.lo), gs=gs.to(dev), K=len(group_sizes),
                                Kp=tb.shape[0])
        return self._vocab[key]

    @torch.no_grad()
    def score(self, mask_embed, key):
        """cal_pred_logits (odise.py:181-207): logit_scale * cos-sim against the prompt bank, per-class max over
        synonym prompts (helper.py:96-100), null column appended -> [rows, K + 1]."""
        v = self._vocab[key]
        rows = mask_embed.shape[0]
        me_p = ops.l2_normalize_split(mask_embed, lo=self.lo)
        sims = ops.empty(rows, v["Kp"], self.dev)
        lib.gemm(me_p, v["te_p"], nmma=self.nmma, alpha=self.logit_scale, out=sims)
        null = ops.empty(rows, 1, self.dev)
        lib.gemm(me_p, v["ne_p"], nmma=self.nmma, alpha=self.logit_scale, out=null)
        return ops.class_max(sims, v["gs"], null, rows, v["K"])

    @torch.no_grad()
    def forward(self, feats, B, vocab_key=None, want_mask_features_f32=False):
        with lib.nvtx("pixel_decoder"):
            pd = self.pixel_decoder(feats, B, want_mask_features_f32)
        with lib.nvtx("masked_attention_decoder"):
            heads = self.transformer_decoder(pd, B)
        out = dict(heads=heads, pd=pd)
        if vocab_key is not None:
            with lib.nvtx("clip_text_scoring"):
                out["pred_logits"] = self.score(heads[-1]["mask_embed"], vocab_key).view(B, self.Q, -1)
        return out
