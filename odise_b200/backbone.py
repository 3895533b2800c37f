"""H100 engine for ODISE's diffusion backbone glue (SURVEY.md §8a rows a2-a6): the sliding 512x512 crops of
FeatureExtractorBackbone.slide_forward (odise/modeling/backbone/feature_extractor.py:181-250), the implicit
captioner front of LdmImplicitCaptionerExtractor.forward (odise/modeling/meta_arch/ldm.py:697-718), q_sample at
t = 0 (odise/modeling/diffusion/gaussian_diffusion.py:275-292) with the reference's shared noise (ldm.py:271-277),
the UNet feature pass (unet.py) and the eight BottleneckBlock projections summed per stride
(feature_extractor.py:157-179).

All crops of all images of a step run as ONE batch through the UNet (B = images x crops): the reference loops over
crops sequentially (feature_extractor.py:205-227).

The KL-VAE encoder / truncated decoder and the CLIP image tower are §8(f) rows; until their engines land, their
outputs enter through a `TapProvider` (synthetic, seeded) — see DESIGN.md.
"""
import math

import torch

from . import lib, ops, spec
from .ops import ACT_RELU
from .unet import UNetEngine, CTX_T

FEATURE_DIMS = spec.FEATURE_DIMS
FEATURE_STRIDES = spec.FEATURE_STRIDES
TAP_ORDER = ("enc5", "enc7", "unet2", "unet5", "unet8", "unet11", "dec2", "dec5")


def t0_coefficients():
    """sqrt(alpha_bar_0), sqrt(1 - alpha_bar_0) of the "ldm_linear" schedule with 1000 steps, rounded to fp32 like
    _extract_into_tensor(...).float() does (gaussian_diffusion.py:125-135, :288-291)."""
    import numpy as np
    betas = np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=np.float64) ** 2
    ac = np.cumprod(1.0 - betas, axis=0)
    return float(np.float32(np.sqrt(ac)[0])), float(np.float32(np.sqrt(1.0 - ac)[0]))


class SyntheticTaps:
    """Stand-in for the KL-VAE (encoder taps, latent, decoder taps) and the CLIP image embedding: deterministic
    seeded tensors of the reference's shapes (ldm.py:284-346).  NOT part of the measured hot path."""

    def __init__(self, device, seed=21):
        self.dev = torch.device(device)
        self.seed = seed
        self._cache = {}

    def __call__(self, B, crop_hw=(512, 512)):
        key = (B, crop_hw)
        if key not in self._cache:
            g = torch.Generator().manual_seed(self.seed)
            H, W = crop_hw
            mk = lambda h, w, c: torch.randn(B * h * w, c, generator=g).to(self.dev)
            self._cache[key] = dict(
                latent=(mk(H // 8, W // 8, 4), H // 8, W // 8),
                enc5=(mk(H // 4, W // 4, 512), H // 4, W // 4), enc7=(mk(H // 8, W // 8, 512), H // 8, W // 8),
                dec2=(mk(H // 8, W // 8, 512), H // 8, W // 8), dec5=(mk(H // 4, W // 4, 512), H // 4, W // 4),
                clip_embed=torch.randn(B, 768, generator=g).to(self.dev))
        return self._cache[key]


class BackboneEngine:
    def __init__(self, sd, device, nmma=3, prefix="backbone.", unet_prefix=spec.UNET_PREFIX, uncond=None, vae=None, clip=None,
                 synthetic_uncond=False, backbone_in_size=512):
        """sd: state dict with `backbone.feature_projections.*`, `backbone.feature_extractor.*` and the UNet.
        uncond: the frozen text-encoder output for "" ([1, 77, 768]; ldm.py:116) — an input of the path.
        vae: optional VAEEngine (SURVEY.md §8f-1); without it the VAE taps / latent are synthetic.
        clip: optional ClipVisualEngine (§8f-2); without it the CLIP image embedding is a seeded synthetic tensor."""
        self.dev = torch.device(device)
        self.nmma, self.lo = nmma, (lib.Q8 if nmma == 2 else nmma == 3)     # 2 = F16Q8 operand mode (lib.Q8)
        self.vae = vae
        self.clip = clip
        self._boxes = {}
        self._inv_cnt = {}
        self.in_size = backbone_in_size            # FeatureExtractorBackbone(backbone_in_size=(512, 512))
        self.unet = UNetEngine(sd, device, nmma=nmma, prefix=unet_prefix)
        self.W, self.F = {}, {}
        f = lambda t: t.to(self.dev, torch.float32).contiguous()
        pl = lambda w: lib.split(f(w.reshape(w.shape[0], -1)), lo=self.lo)
        for i, cin in enumerate(FEATURE_DIMS):
            q = f"{prefix}feature_projections.{i}.0."
            n = f"p{i}."
            self.W[n + "c1"] = pl(sd[q + "conv1.weight"])
            self.W[n + "c2"] = lib.split(f(sd[q + "conv2.weight"].permute(0, 2, 3, 1).reshape(128, -1)), lo=self.lo)
            self.W[n + "c3"] = pl(sd[q + "conv3.weight"])
            for c in ("conv1", "conv2", "conv3"):
                self.F[n + c + ".g"], self.F[n + c + ".b"] = f(sd[q + c + ".norm.weight"]), f(sd[q + c + ".norm.bias"])
            if cin != 512:
                self.W[n + "sc"] = pl(sd[q + "shortcut.weight"])
                self.F[n + "sc.g"], self.F[n + "sc.b"] = f(sd[q + "shortcut.norm.weight"]), f(sd[q + "shortcut.norm.bias"])
        e = prefix + "feature_extractor."
        self.W["clip_project"] = pl(sd[e + "clip_project.linear.weight"])
        self.F["clip_project.b"] = f(sd[e + "clip_project.linear.bias"])
        self.W["time_project"] = pl(sd[e + "time_embed_project.linear.weight"])
        self.F["time_project.b"] = f(sd[e + "time_embed_project.linear.bias"])
        if uncond is None:
            # ADVICE r1: never condition a real checkpoint on noise.  With the SD text encoder in the state dict the
            # empty-prompt embedding (ldm.py:116) is computed here; a seeded random stand-in is an explicit opt-in.
            if any(k.startswith(spec.SD_TEXT_PREFIX) for k in sd):
                from .clip import uncond_inputs
                uncond = uncond_inputs(sd, device, nmma=nmma).cpu()
            elif synthetic_uncond:
                uncond = torch.randn(1, CTX_T, 768, generator=torch.Generator().manual_seed(17))
            else:
                raise lib.OdiseError("BackboneEngine: no `uncond` given and no cond_stage_model.* weights to compute it "
                                     "from; pass synthetic_uncond=True for a seeded stand-in (benchmarks / tests)")
        # weight-only terms of cond = uncond + tanh(alpha) * (proj + pos)   (ldm.py:707-709)
        ta = torch.tanh(sd[e + "alpha_cond"].float())
        self.F["cond.ta"] = f(ta.view(CTX_T, 768))
        self.F["cond.a0"] = f((uncond.float() + ta * sd[e + "clip_project.positional_embedding"].float()).view(CTX_T, 768))
        tt = torch.tanh(sd[e + "alpha_cond_time_embed"].float()).view(1, 1280)
        self.F["temb.ta"] = f(tt)
        self.F["temb.a0"] = f(tt * sd[e + "time_embed_project.positional_embedding"].float().view(1, 1280))
        c0, c1 = t0_coefficients()
        self.c0 = c0
        self.c1 = c1
        self._noise = torch.randn(1, 4, 64, 64, generator=torch.Generator().manual_seed(42))      # ldm.py:273-276
        self._noise_c1 = {(64, 64): f((c1 * self._noise).permute(0, 2, 3, 1).reshape(64 * 64, 4))}
        self.taps_provider = SyntheticTaps(device)

    # ------------------------------------------------------------------------------------------- pieces
    def conditioning(self, clip_embed, B):
        """-> (context [B*77, 768], cond_emb [B, 1280])"""
        e_p = lib.split(clip_embed, lo=self.lo)
        proj = ops.empty(B, 768, self.dev)
        lib.gemm(e_p, self.W["clip_project"], nmma=self.nmma, bias=self.F["clip_project.b"], out=proj)
        ctx = ops.bcast_fma(self.F["cond.a0"], self.F["cond.ta"], proj, B, CTX_T, 768)
        tp = ops.empty(B, 1280, self.dev)
        lib.gemm(e_p, self.W["time_project"], nmma=self.nmma, bias=self.F["time_project.b"], out=tp)
        cemb = ops.bcast_fma(self.F["temb.a0"], self.F["temb.ta"], tp, B, 1, 1280)
        return ctx, cemb

    def shared_noise(self, h, w):
        """sqrt(1 - abar_0) * shared noise for an h x w latent, NHWC [h*w, 4] on the device.  Latents other than 64 x 64
        get the bicubic resize of the 64 x 64 noise (ldm.py:583-592: F.interpolate(mode="bicubic", align_corners=False));
        a constant of (h, w), computed once on the host and cached."""
        if (h, w) not in self._noise_c1:
            n = torch.nn.functional.interpolate(self._noise, size=(h, w), mode="bicubic", align_corners=False)
            self._noise_c1[(h, w)] = (self.c1 * n).permute(0, 2, 3, 1).reshape(h * w, 4).contiguous().to(self.dev)
        return self._noise_c1[(h, w)]

    def q_sample(self, latent, B, h, w):
        """x_t = sqrt(abar_0) * z + sqrt(1 - abar_0) * eps with the shared noise (gaussian_diffusion.py:275-292)."""
        x = ops.empty(B * h * w, 4, self.dev)
        ops.copy2d(latent, x, scale=self.c0)
        y, _ = ops.add_split(x, self.shared_noise(h, w), b_rows=h * w, want_f32=True, want_planes=False)
        return y

    def project(self, taps, B, crop_hw):
        """forward_features (feature_extractor.py:157-179): -> {"s2".."s5": (NHWC fp32 [B*h*w, 512], h, w)}"""
        H, W = crop_hw
        out = {}
        for idx, name in enumerate(TAP_ORDER):
            x, h, w = taps[name]
            s = FEATURE_STRIDES[idx]
            th, tw = H // s, W // s
            if (h, w) != (th, tw):
                x = ops.resize_nhwc(x, B, h, w, th, tw, bilinear=False)       # F.interpolate default = nearest
            M = B * th * tw
            n = f"p{idx}."
            x_p = lib.split(x, lo=self.lo)
            # every conv leaves the GroupNorm records of its output in its epilogue (lib.GnStats): no statistics passes
            t1, s1 = ops.empty(M, 128, self.dev), lib.GnStats(M, 128, self.dev)
            lib.gemm(x_p, self.W[n + "c1"], nmma=self.nmma, out=t1, gn=s1)
            _, a1 = ops.group_norm(t1, B, th * tw, self.F[n + "conv1.g"], self.F[n + "conv1.b"], 1e-5, ACT_RELU, lo=self.lo,
                                   stats=s1)
            t2, s2 = ops.empty(M, 128, self.dev), lib.GnStats(M, 128, self.dev)
            if lib.conv_ok(th, tw):
                lib.gemm(a1, self.W[n + "c2"], M=M, N=128, nmma=self.nmma, conv=(128, th, tw), out=t2, gn=s2)
            else:     # map widths the implicit-GEMM boxes cannot tile (e.g. 12 = 384 / 32): materialised im2col
                lib.gemm(ops.im2col3x3_split(a1.float(), B, th, tw, lo=self.lo)[0], self.W[n + "c2"], nmma=self.nmma, out=t2,
                         gn=s2)
            _, a2 = ops.group_norm(t2, B, th * tw, self.F[n + "conv2.g"], self.F[n + "conv2.b"], 1e-5, ACT_RELU, lo=self.lo,
                                   stats=s2)
            t3, s3 = ops.empty(M, 512, self.dev), lib.GnStats(M, 512, self.dev)
            lib.gemm(a2, self.W[n + "c3"], nmma=self.nmma, out=t3, gn=s3)
            if FEATURE_DIMS[idx] != 512:
                sc, ss = ops.empty(M, 512, self.dev), lib.GnStats(M, 512, self.dev)
                lib.gemm(x_p, self.W[n + "sc"], nmma=self.nmma, out=sc, gn=ss)
                sc, _ = ops.group_norm(sc, B, th * tw, self.F[n + "sc.g"], self.F[n + "sc.b"], 1e-5, want_f32=True,
                                       want_planes=False, stats=ss)
            else:
                sc = x
            key = f"s{int(math.log2(s))}"
            first = key not in out
            if first:
                out[key] = (ops.empty(M, 512, self.dev), th, tw)
            ops.group_norm_res(t3, B, th * tw, self.F[n + "conv3.g"], self.F[n + "conv3.b"], 1e-5, sc, ACT_RELU,
                               out[key][0], accumulate=not first, stats=s3)
        return out

    @torch.no_grad()
    def extract(self, B, crop_hw=(512, 512), vae_taps=None, crops=None, clip_embed=None, out_hw=None):
        """single_forward for a batch of B crops.  out_hw: the crop size BEFORE T.Resize (input_image_size of
        forward_features, feature_extractor.py:141-155): the projections run at out_hw / stride.  crops: normalised NHWC fp32 [B*h*w, 3] -> the VAE engine produces
        latent + taps; otherwise they are given / synthetic.  clip_embed: [B, 768] from the CLIP image tower
        (ldm.py:705); synthetic when no ClipVisualEngine is attached."""
        t = vae_taps if vae_taps is not None else self.taps_provider(B, crop_hw)
        if clip_embed is not None:
            t = dict(t, clip_embed=clip_embed)
        if crops is not None and self.vae is not None:
            with lib.nvtx("vae_encoder_taps"):
                enc = self.vae.encode(crops, B, crop_hw[0], crop_hw[1])
            lat, lh, lw = enc["latent"]
            with lib.nvtx("vae_decoder_taps"):
                dec = self.vae.decode_taps(lat, B, lh, lw)
            t = dict(latent=enc["latent"], enc5=enc["enc5"], enc7=enc["enc7"], dec2=dec["dec2"], dec5=dec["dec5"],
                     clip_embed=t["clip_embed"])
        with lib.nvtx("implicit_captioner+q_sample"):
            ctx, cemb = self.conditioning(t["clip_embed"], B)
            lat, lh, lw = t["latent"]
            x = self.q_sample(lat, B, lh, lw)
        with lib.nvtx("unet_feature_pass"):
            u = self.unet.forward(x, B, lh, lw, ctx, cemb)
        taps = dict(enc5=t["enc5"], enc7=t["enc7"], dec2=t["dec2"], dec5=t["dec5"],
                    unet2=u[0], unet5=u[1], unet8=u[2], unet11=u[3])
        with lib.nvtx("feature_projections"):
            return self.project(taps, B, out_hw or crop_hw)

    # ------------------------------------------------------------------------------------------- sliding window
    @staticmethod
    def crop_grid(h_img, w_img, crop=512):
        """slide_forward's crop boxes (feature_extractor.py:197-218): (y1, x1) list and the crop side."""
        short = min(crop, min(h_img, w_img))
        hg = max(h_img - short + short - 1, 0) // short + 1
        wg = max(w_img - short + short - 1, 0) // short + 1
        boxes = []
        for hi in range(hg):
            for wi in range(wg):
                y2 = min(hi * short + short, h_img)
                x2 = min(wi * short + short, w_img)
                boxes.append((max(y2 - short, 0), max(x2 - short, 0)))
        return boxes, short

    @torch.no_grad()
    def forward(self, n_images, h_img, w_img, vae_taps=None, images_u8=None):
        """slide_forward over n_images images of h_img x w_img: all crops in one batch, paste + average.
        images_u8: device image batch [n_images, 3, H, W], uint8 (0..255) or float32 in [0, 1] (used when a VAE
        engine is attached).
        Returns {"s2".."s5": (NHWC fp32 [n_images * H/s * W/s, 512], H/s, W/s)}."""
        boxes, short = self.crop_grid(h_img, w_img)
        nc = len(boxes)
        B = n_images * nc                                # crop batch, image-major: b = img * nc + crop
        crops = clip_embed = None
        net = short                                          # side of what the feature extractor sees
        if images_u8 is not None and (self.vae is not None or self.clip is not None):
            key = (n_images, h_img, w_img)
            if key not in self._boxes:
                self._boxes[key] = torch.tensor([[i, y, x] for i in range(n_images) for (y, x) in boxes],
                                                dtype=torch.int32).to(self.dev)
            src, bx, sh, sw = images_u8, self._boxes[key], h_img, w_img
            if short != self.in_size:
                # single_forward's image_preprocess = T.Resize((512, 512), BICUBIC) (feature_extractor.py:73-76, :144):
                # crops of images whose short side is below 512 are upsampled before the extractor, so the latent is
                # always 64 x 64; the features are brought back to crop / stride in project() (F.interpolate nearest)
                net = self.in_size
                src = ops.crop_resize_bicubic(images_u8, bx, B, h_img, w_img, short, short, net)
                ikey = ("id", B)
                if ikey not in self._boxes:
                    self._boxes[ikey] = torch.tensor([[i, 0, 0] for i in range(B)], dtype=torch.int32).to(self.dev)
                bx, sh, sw = self._boxes[ikey], net, net
            if self.vae is not None:
                crops = ops.image_crops(src, bx, B, sh, sw, net, net)
            if self.clip is not None:
                with lib.nvtx("clip_image_tower"):
                    # maskclip_images (set by ODISEEngine.step): the images the MaskCLIP head will encode later in the step;
                    # their image tokens share this pass, their keys / values are cached inside the CLIP engine
                    clip_embed = self.clip.embed(src, bx, B, sh, sw, net, net,
                                                 maskclip_images=getattr(self, "maskclip_images", None))
        elif short != self.in_size and vae_taps is None:
            net = self.in_size
        feats = self.extract(B, (net, net), vae_taps, crops, clip_embed, out_hw=(short, short))
        if nc == 1 and short == h_img == w_img:
            return feats
        out = {}
        for k, (f, fh, fw) in feats.items():
            s = short // fh
            Hd, Wd = h_img // s, w_img // s
            dst = torch.zeros(n_images * Hd * Wd, 512, dtype=torch.float32, device=self.dev)
            ckey = (n_images, h_img, w_img, s)
            if ckey not in self._inv_cnt:                  # cached on the device: no H2D copy inside a graph capture
                cnt = torch.zeros(Hd, Wd)
                for ci, (y1, x1) in enumerate(boxes):
                    cnt[y1 // s:y1 // s + fh, x1 // s:x1 // s + fw] += 1
                self._inv_cnt[ckey] = (1.0 / cnt).reshape(-1).repeat(n_images).to(self.dev) if float(cnt.max()) > 1 else None
            for img in range(n_images):
                for ci, (y1, x1) in enumerate(boxes):
                    b = img * nc + ci
                    src = f[b * fh * fw:(b + 1) * fh * fw].view(fh, fw * 512)
                    d0 = (img * Hd + y1 // s) * Wd + x1 // s
                    dv = dst[d0:d0 + (fh - 1) * Wd + fw].as_strided((fh, fw * 512), (Wd * 512, 1))
                    ops.copy2d(src, dv, accumulate=True)
            if self._inv_cnt[ckey] is not None:
                ops.rowscale(dst, self._inv_cnt[ckey])
            out[k] = (dst, Hd, Wd)
        return out
