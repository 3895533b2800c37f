"""H100 engine for the CLIP ViT-L/14-336 image tower behind ClipAdapter.embed_image (SURVEY.md §8f-2;
odise/modeling/meta_arch/clip.py:177-231, called from LdmImplicitCaptionerExtractor.forward, ldm.py:705).

crop [B, 3, 512, 512] in [0,1] -> bicubic 336 + CLIP normalisation (odise_clip_preprocess) -> 14x14 patch embedding as a
GEMM -> 24 pre-LN transformer blocks (QKV / out / MLP on the wgmma GEMM with fused bias, QuickGELU and residual
epilogues; attention on the wgmma flash kernel, d = 64) -> ln_post + projection of the class token -> [B, 768].
Tokens per image are padded 577 -> 584 rows so every TMA box start stays 16-byte aligned; pad keys are masked.
"""
import torch

from . import lib, ops, spec
from .lib import Planes
from .ops import ACT_QUICKGELU


class _ResBlocks:
    """`layers` open_clip ResidualAttentionBlocks (x += attn(ln_1 x); x += c_proj(QuickGELU(c_fc(ln_2 x)))) as operand
    planes + the loop that runs them on a token matrix [B*TS, width] whose first Tk rows per image are the keys."""

    def __init__(self, sd, prefix, device, nmma, width, layers, heads):
        # nmma: 3 = bf16x3 | 2 = F16Q8 operands for the linears (lib.Q8; the attention core keeps bf16x3 q / k, fp16 V^T) | 1
        self.dev, self.nmma, self.lo = torch.device(device), nmma, (lib.Q8 if nmma == 2 else nmma == 3)
        self.lb = bool(self.lo)
        self.width, self.layers, self.heads = width, layers, heads
        f = lambda t: t.to(self.dev, torch.float32).contiguous()
        pl = lambda w: lib.split(f(w), lo=self.lo)
        self.W, self.F = {}, {}
        for i in range(layers):
            q = f"{prefix}transformer.resblocks.{i}."
            n = f"l{i}."
            w, b = sd[q + "attn.in_proj_weight"], sd[q + "attn.in_proj_bias"]
            self.W[n + "qk"], self.F[n + "qk.b"] = pl(w[:2 * width]), f(b[:2 * width])
            self.W[n + "v"], self.F[n + "v.b"] = pl(w[2 * width:]), f(b[2 * width:])
            self.W[n + "o"], self.F[n + "o.b"] = pl(sd[q + "attn.out_proj.weight"]), f(sd[q + "attn.out_proj.bias"])
            self.W[n + "fc"], self.F[n + "fc.b"] = pl(sd[q + "mlp.c_fc.weight"]), f(sd[q + "mlp.c_fc.bias"])
            self.W[n + "pr"], self.F[n + "pr.b"] = pl(sd[q + "mlp.c_proj.weight"]), f(sd[q + "mlp.c_proj.bias"])
            for ln in ("ln_1", "ln_2"):
                self.F[n + ln + ".g"], self.F[n + ln + ".b"] = f(sd[q + ln + ".weight"]), f(sd[q + ln + ".bias"])

    def _gemm(self, a, name, **kw):
        return lib.gemm(a, self.W[name], nmma=self.nmma, bias=self.F.get(name + ".b"), **kw)

    def run(self, h, B, TS, Tk, bits=None, row_any=None, keep=None):
        """keep = (first_image, n_images): also return, per layer, the K planes and V^T planes of those images' tokens
        (views into the layer's projection outputs) — the keys / values a later run_queries() attends to."""
        dev, Wd = self.dev, self.width
        M = B * TS
        d = Wd // self.heads
        cache = []
        for i in range(self.layers):
            n = f"l{i}."
            _, y = ops.layer_norm(h, self.F[n + "ln_1.g"], self.F[n + "ln_1.b"], lo=self.lo)
            qk = Planes.empty(M, 2 * Wd, dev, lo=self.lb)
            self._gemm(y, n + "qk", out_planes=qk)
            vt = Planes.empty(Wd, M, dev, lo=self.lb, f16=self.lb)
            lib.gemm(self.W[n + "v"], y, nmma=self.nmma, bias_m=self.F[n + "v.b"], out_planes=vt)
            if keep is not None:
                cache.append((qk.col_slice(Wd, Wd).row_slice(keep[0] * TS, keep[1] * TS), vt.col_slice(keep[0] * TS, keep[1] * TS)))
            _, o = ops.attention_tc(qk.col_slice(0, Wd), qk.col_slice(Wd, Wd), vt, B, self.heads, d, TS, Tk, d ** -0.5,
                                    self.nmma, tk_stride=TS, mask_bits=bits, row_any=row_any, lo=self.lo)
            h2 = ops.empty(M, Wd, dev)
            self._gemm(o, n + "o", residual=h, out=h2)
            _, y2 = ops.layer_norm(h2, self.F[n + "ln_2.g"], self.F[n + "ln_2.b"], lo=self.lo)
            u = Planes.empty(M, 4 * Wd, dev, lo=self.lo)
            self._gemm(y2, n + "fc", act=ACT_QUICKGELU, out_planes=u)
            h = ops.empty(M, Wd, dev)
            self._gemm(u, n + "pr", residual=h2, out=h)
        return (h, cache) if keep is not None else h

    def run_queries(self, hq, cache, B, Q, TS, Tk, bits, row_any):
        """Extra query tokens (MaskCLIP's mask tokens, clip.py:291-321) through the blocks: per layer they attend to the
        cached keys / values of their image's first Tk tokens under their own key mask; nobody attends to THEM (the
        reference masks the mask-token columns for every row), so only their q projection is needed and the image tokens'
        stream — computed once by run(..., keep=...) — is untouched.  hq: fp32 [B*Q, width] (after ln_pre)."""
        dev, Wd = self.dev, self.width
        M = B * Q
        d = Wd // self.heads
        # a few hundred rows: four M tiles, so a CTA's k loop is a serial chain of TMA round trips -> split K to spread it
        # (K = 1024: 4 splits of 4 k-blocks; K = 4096: 8 splits), the reduce kernel applies the epilogue
        sk1 = 4 if M <= 1024 and Wd >= 1024 else 1
        sk4 = 8 if M <= 1024 and Wd >= 1024 else 1
        ws = lib.workspace(max(sk1 * M * 4 * Wd, sk4 * M * Wd) * 4, dev) if sk1 > 1 else None
        kw1 = dict(split_k=sk1, workspace=ws) if sk1 > 1 else {}
        kw4 = dict(split_k=sk4, workspace=ws) if sk4 > 1 else {}
        for i in range(self.layers):
            n = f"l{i}."
            kP, vt = cache[i]
            _, y = ops.layer_norm(hq, self.F[n + "ln_1.g"], self.F[n + "ln_1.b"], lo=self.lo)
            qP = Planes.empty(M, Wd, dev, lo=self.lb)
            lib.gemm(y, self.W[n + "qk"].row_slice(0, Wd), nmma=self.nmma, bias=self.F[n + "qk.b"][:Wd], out_planes=qP, **kw1)
            _, o = ops.attention_tc(qP, kP, vt, B, self.heads, d, Q, Tk, d ** -0.5, self.nmma, tk_stride=TS,
                                    mask_bits=bits, row_any=row_any, lo=self.lo)
            h2 = ops.empty(M, Wd, dev)
            self._gemm(o, n + "o", residual=hq, out=h2, **kw1)
            _, y2 = ops.layer_norm(h2, self.F[n + "ln_2.g"], self.F[n + "ln_2.b"], lo=self.lo)
            u = Planes.empty(M, 4 * Wd, dev, lo=self.lo)
            self._gemm(y2, n + "fc", act=ACT_QUICKGELU, out_planes=u, **kw1)
            hq = ops.empty(M, Wd, dev)
            self._gemm(u, n + "pr", residual=h2, out=hq, **kw4)
        return hq


class ClipVisualEngine:
    def __init__(self, sd, device, nmma=3, prefix=spec.CLIP_PREFIX, width=1024, layers=24, heads=16, patch=14, image=336):
        self.dev = torch.device(device)
        self.nmma, self.lo = nmma, (lib.Q8 if nmma == 2 else nmma == 3)
        self.width, self.layers, self.heads, self.patch, self.image = width, layers, heads, patch, image
        self.G = image // patch
        self.T = self.G * self.G + 1             # 577
        self.TS = (self.T + 7) // 8 * 8          # 584 rows per image
        f = lambda t: t.to(self.dev, torch.float32).contiguous()
        g = lambda n: sd[prefix + n]

        def pl(w):
            w = f(w)
            if w.shape[1] % 8:
                w = torch.nn.functional.pad(w, (0, 8 - w.shape[1] % 8))
            return lib.split(w, lo=self.lo)

        self.W, self.F = {}, {}
        self.W["conv1"] = pl(g("conv1.weight").reshape(width, -1))
        pos = g("positional_embedding").float()
        self.F["pos_patches"] = f(pos[1:])                                   # [576, width]
        self.F["cls_row"] = f((g("class_embedding").float() + pos[0]).view(1, width))
        self.F["ln_pre.g"], self.F["ln_pre.b"] = f(g("ln_pre.weight")), f(g("ln_pre.bias"))
        self.blocks = _ResBlocks(sd, prefix, device, nmma, width, layers, heads)
        self.F["ln_post.g"], self.F["ln_post.b"] = f(g("ln_post.weight")), f(g("ln_post.bias"))
        self.W["proj"] = pl(g("proj").t())                                   # x @ proj == x @ (proj^T)^T

    def _tokens(self, parts):
        """parts: [(normalised NHWC image batch [n*S*S, 3], n), ...] -> pre-ln_pre token matrix [B*TS, width] of all the
        images in order: per image row 0 = class token, rows 1..576 = patches (+ positional embedding), zero pad rows."""
        dev, Wd, T, TS = self.dev, self.width, self.T, self.TS
        B = sum(n for _, n in parts)
        tok = torch.zeros(B * TS, Wd, dtype=torch.float32, device=dev)
        b0 = 0
        for x, n in parts:
            patches = ops.patchify_split(x, n, self.image, self.patch, lo=self.lo)
            lib.gemm(patches, self.W["conv1"], M=T - 1, N=Wd, K=patches.cols, nmma=self.nmma, batch=n,
                     a_bs=(T - 1) * patches.ld, residual=self.F["pos_patches"], ld_res=Wd, res_bs=0,
                     out=tok[b0 * TS + 1:], ld_out=Wd, out_bs=TS * Wd)
            b0 += n
        ops.copy2d(self.F["cls_row"].expand(B, Wd), tok.view(B, TS * Wd)[:, :Wd])
        return tok, B

    def _tower(self, tok, B, keep=None):
        """ln_pre + the 24 residual attention blocks on [B*TS, width]; keys = the first 577 rows of every image."""
        h, _ = ops.layer_norm(tok, self.F["ln_pre.g"], self.F["ln_pre.b"], want_f32=True, want_planes=False, lo=self.lo)
        return self.blocks.run(h, B, self.TS, self.T, keep=keep)

    @torch.no_grad()
    def embed(self, img, boxes_dev, n_crops, H, W, ch, cw, maskclip_images=None):
        """ClipAdapter.embed_image (clip.py:225-231) of every crop.
        img: device uint8 / float32 [N, 3, H, W]; boxes [n_crops, 3] int32 -> image_embed fp32 [n_crops, 768].
        maskclip_images = (images [N, 3, Hi, Wi], N, Hi, Wi): the images MaskCLIP will look at later in the step.  Their
        image-token stream does not depend on the masks (see _ResBlocks.run_queries), so it rides through the SAME GEMMs as
        the crops (one batch of n_crops + N images) and its per-layer keys / values are kept for mask_embed()."""
        B, Wd, TS = n_crops, self.width, self.TS
        parts = [(ops.clip_preprocess(img, boxes_dev, B, H, W, ch, cw, self.image), B)]
        keep = None
        if maskclip_images is not None:
            mi, Nm, Hm, Wm = maskclip_images
            parts.append((ops.maskclip_preprocess(mi, Nm, Hm, Wm, self.image), Nm))
            keep = (B, Nm)
        tok, Ball = self._tokens(parts)
        h = self._tower(tok, Ball, keep)
        self._kv = None
        if keep is not None:
            h, cache = h
            self._kv = (mi.data_ptr(), Nm, Hm, Wm, cache)
        cls = h.view(Ball, TS * Wd)[:B, :Wd]                                   # token 0 of every crop (strided rows)
        _, c = ops.layer_norm(cls, self.F["ln_post.g"], self.F["ln_post.b"], lo=self.lo)
        out = ops.empty(B, self.W["proj"].rows, self.dev)
        lib.gemm(c, self.W["proj"], nmma=self.nmma, out=out)
        return out

    @torch.no_grad()
    def mask_embed(self, img, mask_logits, N, H, W):
        """MaskCLIP.get_mask_embed (clip.py:325-339): img [N,3,H,W] (u8 / f32 in [0,1]), mask logits [N,Q,hm,wm]
        -> fp32 [N*Q, 768].  The Q mask tokens are rows 577.. of each image's token block; their attention mask
        is 1 bit per (token, key) built straight from the low-resolution logits (odise_maskclip_bits_f32)."""
        Wd, T, TS = self.width, self.T, self.TS
        Q, hm, wm = mask_logits.shape[1:]
        kv = getattr(self, "_kv", None)
        if kv is not None and kv[:4] == (img.data_ptr(), N, H, W):
            cache = kv[4]                       # image-token keys / values left by embed(..., maskclip_images=...)
        else:                                   # stand-alone call: the image-token stream of these N images first
            tok, _ = self._tokens([(ops.maskclip_preprocess(img, N, H, W, self.image), N)])
            _, cache = self._tower(tok, N, keep=(0, N))
        self._kv = None
        # the mask tokens start as copies of the (ln_pre'd) class token (clip.py:271-274) and attend to the class token + the
        # patches under their mask; 1 bit per (token, key)
        bits, row_any = ops.maskclip_bits(mask_logits.contiguous(), N, Q, hm, wm, self.image, self.patch, Q, 0)
        hq0 = ops.empty(N * Q, Wd, self.dev)
        ops.copy2d(self.F["cls_row"].expand(N * Q, Wd), hq0)
        hq, _ = ops.layer_norm(hq0, self.F["ln_pre.g"], self.F["ln_pre.b"], want_f32=True, want_planes=False, lo=self.lo)
        hq = self.blocks.run_queries(hq, cache, N, Q, TS, T, bits, row_any)
        _, c = ops.layer_norm(hq, self.F["ln_post.g"], self.F["ln_post.b"], lo=self.lo)
        out = ops.empty(N * Q, self.W["proj"].rows, self.dev)
        lib.gemm(c, self.W["proj"], nmma=self.nmma, out=out)
        return out


class MaskClipHead:
    """PoolingCLIPHead + the clip_head branch of CategoryODISE.forward (odise.py:1469-1542, :292-323) on the device:
    MaskCLIP mask embeddings x CLIP text bank -> per-class max over synonym prompts -> geometric ensemble with the
    category head (alpha for classes of the training vocabulary, beta for novel ones) -> void merge -> log-probs."""

    def __init__(self, visual, alpha=0.3, beta=0.7, logit_scale=100.0):
        self.visual, self.dev = visual, visual.dev
        self.nmma, self.lo = visual.nmma, bool(visual.lo)     # the CLIP match itself (one small GEMM) stays bf16x3 in every mode
        self.alpha, self.beta = float(alpha), float(beta)
        self.logit_scale = float(min(logit_scale, 100.0))            # clamp(exp(clip.logit_scale), max=100), clip.py:247
        self._vocab = {}

    def set_vocabulary(self, key, text_bank, group_sizes, overlapping):
        """text_bank: raw CLIP text embeddings of every prompt [K', 768] (get_and_cache_test_text_embed);
        overlapping[k]: class k shares a name with the training vocabulary (odise.py:1483-1493)."""
        tb = text_bank.to(self.dev, torch.float32).contiguous()
        gs = torch.zeros(len(group_sizes) + 1, dtype=torch.int32)
        gs[1:] = torch.as_tensor(group_sizes, dtype=torch.int32).cumsum(0)
        self._vocab[key] = dict(te_p=ops.l2_normalize_split(tb, lo=self.lo), gs=gs.to(self.dev), K=len(group_sizes),
                                Kp=tb.shape[0],
                                ov=torch.as_tensor(overlapping).to(torch.uint8).to(self.dev).contiguous())

    @torch.no_grad()
    def forward(self, key, img, N, H, W, pred_masks, cat_logits, want_open=False):
        """pred_masks [N,Q,hm,wm] logits, cat_logits [N,Q,K+1] -> dict(pred_logits [N,Q,K+1] merged log-probs,
        mask_embed [N*Q,768], mask_pred_open_logits [N*Q,K] (row stride K+1), pred_open_logits (optional))."""
        v = self._vocab[key]
        Q, K = pred_masks.shape[1], v["K"]
        rows = N * Q
        me = self.visual.mask_embed(img, pred_masks, N, H, W)
        me_p = ops.l2_normalize_split(me, lo=self.lo)
        sims = ops.empty(rows, v["Kp"], self.dev)
        lib.gemm(me_p, v["te_p"], nmma=self.nmma, alpha=self.logit_scale, out=sims)
        if not hasattr(self, "_zero") or self._zero.shape[0] < rows:
            self._zero = torch.zeros(rows, 1, dtype=torch.float32, device=self.dev)
        clip_logits = ops.class_max(sims, v["gs"], self._zero, rows, K)         # [rows, K+1], last column unused
        cl = cat_logits.contiguous().view(rows, K + 1)
        merged, op = ops.open_vocab_merge(cl, clip_logits, K + 1, v["ov"], self.alpha, self.beta, rows, K, want_open)
        out = dict(pred_logits=merged.view(N, Q, K + 1), mask_embed=me, mask_pred_open_logits=clip_logits)
        if want_open:
            out["pred_open_logits"] = op.view(N, Q, K)
        return out


class ClipTextEngine:
    """CLIP text tower on the device (f-4 text-bank builder): ClipAdapter._encode_text / open_clip CLIP.encode_text
    (odise/modeling/meta_arch/clip.py:138-152, :29-73) for the vocabulary's prompt bank, and — with the SD-v1
    `cond_stage_model` weights renamed by spec.hf_text_to_openai and project=False — ldm's FrozenCLIPEmbedder, whose
    output for "" is `uncond_inputs` (ldm.py:116).  Token ids come from the caller (the BPE vocabulary file is not part
    of this repo); ctx 77 is padded to 80 rows per prompt, the causal mask is 1 bit per (query, key)."""

    def __init__(self, sd, device, nmma=3, prefix=spec.CLIP_TEXT_PREFIX, width=768, layers=12, heads=12, ctx=77, project=True):
        self.dev = torch.device(device)
        nmma = 3 if nmma == 2 else nmma             # the text tower runs once per vocabulary: always the bf16x3 parity mode
        self.nmma, self.lo = nmma, nmma == 3
        self.width, self.ctx = width, ctx
        self.TS = (ctx + 7) // 8 * 8
        f = lambda t: t.to(self.dev, torch.float32).contiguous()
        self.table = f(sd[prefix + "token_embedding.weight"])
        self.pos = torch.zeros(self.TS, width, dtype=torch.float32, device=self.dev)
        self.pos[:ctx] = f(sd[prefix + "positional_embedding"])
        self.blocks = _ResBlocks(sd, prefix, device, nmma, width, layers, heads)
        self.ln_g, self.ln_b = f(sd[prefix + "ln_final.weight"]), f(sd[prefix + "ln_final.bias"])
        self.proj = lib.split(f(sd[prefix + "text_projection"].t()), lo=self.lo) if project else None
        words = (ctx + 31) // 32
        q = torch.arange(self.TS).view(-1, 1, 1)
        key = (torch.arange(words).view(1, -1, 1) * 32 + torch.arange(32).view(1, 1, -1))
        allowed = ((key <= q) & (key < ctx)).to(torch.int64)                       # causal: query i sees keys <= i
        self._row_bits = (allowed << torch.arange(32).view(1, 1, -1)).sum(-1)      # [TS, words] as uint32 values
        self._row_bits = torch.where(self._row_bits >= 2 ** 31, self._row_bits - 2 ** 32, self._row_bits).to(torch.int32)
        self._row_any = (torch.arange(self.TS) < ctx).to(torch.int32)

    @torch.no_grad()
    def encode(self, token_ids):
        """token_ids int [N, ctx] (host or device) -> (text_embed fp32 [N, out] or None, encodings fp32 [N, ctx, width])."""
        N = token_ids.shape[0]
        assert token_ids.shape[1] == self.ctx
        TS, Wd, dev = self.TS, self.width, self.dev
        ids = torch.zeros(N, TS, dtype=torch.int32)
        ids[:, :self.ctx] = token_ids.cpu().to(torch.int32)
        h = ops.gather_rows(self.table, ids.view(-1).to(dev), add=self.pos, add_period=TS)
        bits = self._row_bits.unsqueeze(0).expand(N, -1, -1).contiguous().to(dev)
        row_any = self._row_any.unsqueeze(0).expand(N, -1).contiguous().to(dev)
        h = self.blocks.run(h, N, TS, self.ctx, bits, row_any)
        x, xp = ops.layer_norm(h, self.ln_g, self.ln_b, want_f32=True, want_planes=self.proj is not None, lo=self.lo)
        enc = x.view(N, TS, Wd)[:, :self.ctx]
        if self.proj is None:
            return None, enc
        eot = (token_ids.cpu().argmax(dim=-1) + torch.arange(N) * TS).to(torch.int32).to(dev)      # clip.py:150
        rows = ops.gather_rows(x, eot)
        out = ops.empty(N, self.proj.rows, dev)
        lib.gemm(ops.split(rows, lo=self.lo), self.proj, nmma=self.nmma, out=out)
        return out, enc


def build_text_bank(text_engine, token_ids, batch=256):
    """build_clip_text_embed (clip.py:29-73): prompts are encoded in chunks of 256 -> raw text embeddings [K', 768]."""
    outs = [text_engine.encode(token_ids[i:i + batch])[0] for i in range(0, token_ids.shape[0], batch)]
    return torch.cat(outs)


EMPTY_PROMPT_IDS = [49406] + [49407] * 76          # "<|startoftext|>" + "<|endoftext|>" padding: the tokens of ""


def uncond_inputs(sd, device, nmma=3):
    """LdmExtractor `uncond_inputs` = ldm.embed_text([""]) (ldm.py:116): the SD-v1 text encoder applied to the empty
    prompt -> [1, 77, 768], from the `cond_stage_model.*` weights of an sd-v1 checkpoint."""
    conv = spec.hf_text_to_openai(sd, dst_prefix="sd_text.")
    eng = ClipTextEngine(conv, device, nmma=nmma, prefix="sd_text.", project=False)
    return eng.encode(torch.tensor([EMPTY_PROMPT_IDS]))[1].contiguous()
