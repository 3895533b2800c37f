"""H100 engine for the KL-VAE stages of ODISE's feature extractor (SURVEY.md §8f row f-1): the encoder pass that
yields the latent + 2 encoder taps (LdmExtractor.encoder_forward / encode_to_latent, ldm.py:424-467) and the decoder
pass TRUNCATED after the last tap (decoder_forward, ldm.py:493-533: taps are the inputs of up-blocks 2 and 5; the
reference runs on to the full 512x512 RGB image and discards it — ~75 % of the decoder FLOPs are dead code).

Same kernels as the UNet ResBlocks: GN(eps 1e-6)+SiLU+split pass -> implicit-GEMM conv3x3 on wgmma.  The single-head
4096-token mid-block attention (d = 512) goes through GEMM + odise_softmax_split_f32 + GEMM.
"""
import torch

from . import lib, ops, spec
from .lib import Planes
from .ops import ACT_NONE, ACT_SILU

SCALE_FACTOR = 0.18215


def _conv_w(w):
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


class VAEEngine:
    def __init__(self, sd, device, nmma=3, prefix=spec.VAE_PREFIX):
        self.dev = torch.device(device)
        # nmma: 3 = bf16x3 | 2 = F16Q8 (lib.Q8: fp16 + e5m2 cross terms) | 1 = plain bf16.  The two mid-block attentions
        # (~2 % of the FLOPs; their batched S / P V GEMMs slice operands at token offsets) stay bf16x3 in the F16Q8 mode.
        self.nmma, self.lo = nmma, (lib.Q8 if nmma == 2 else nmma == 3)
        self.lb = bool(self.lo)
        self.W, self.F = {}, {}
        p = prefix
        g = lambda n: sd[p + n]
        f = lambda t: t.to(self.dev, torch.float32).contiguous()

        def planes(w2d, lo=None):
            w2d = f(w2d)
            if w2d.shape[1] % 8:
                w2d = torch.nn.functional.pad(w2d, (0, 8 - w2d.shape[1] % 8))
            return lib.split(w2d, lo=self.lo if lo is None else lo)

        def conv(name, key, lo=None):
            self.W[name] = planes(_conv_w(g(key + ".weight")), lo)
            self.F[name + ".b"] = f(g(key + ".bias"))

        def lin(name, key, lo=None):
            w = g(key + ".weight")
            self.W[name] = planes(w.reshape(w.shape[0], -1), lo)
            self.F[name + ".b"] = f(g(key + ".bias"))

        def norm(name, key):
            self.F[name + ".g"], self.F[name + ".be"] = f(g(key + ".weight")), f(g(key + ".bias"))

        def res(name, key, cin, cout):
            norm(name + "n1", key + "norm1"); conv(name + "c1", key + "conv1")
            norm(name + "n2", key + "norm2"); conv(name + "c2", key + "conv2")
            if cin != cout:
                lin(name + "sc", key + "nin_shortcut")

        def attn(name, key):
            norm(name + "n", key + "norm")
            w = torch.cat([g(key + "q.weight"), g(key + "k.weight")], 0)
            self.W[name + "qk"] = planes(w.reshape(w.shape[0], -1), self.lb)
            self.F[name + "qk.b"] = f(torch.cat([g(key + "q.bias"), g(key + "k.bias")], 0))
            lin(name + "v", key + "v", self.lb)
            lin(name + "o", key + "proj_out", self.lb)

        ch, mult = 128, (1, 2, 4, 4)
        # 3 -> 128 channels at 512^2: K = 27.  F16Q8 planes come in whole 64-wide k-blocks, the bf16 pair pads to 32 only: this
        # one layer keeps the bf16 pair in every mode (half the im2col bytes over 4.2 M pixels, half the k-blocks)
        conv("e.conv_in", "encoder.conv_in", self.lb)
        in_mult = (1,) + mult
        self.enc_blocks = []
        for i in range(4):
            bi, bo = ch * in_mult[i], ch * mult[i]
            for j in range(2):
                res(f"e.d{i}.b{j}.", f"encoder.down.{i}.block.{j}.", bi, bo)
                self.enc_blocks.append((f"e.d{i}.b{j}.", bi, bo, i))
                bi = bo
            if i != 3:
                conv(f"e.d{i}.down", f"encoder.down.{i}.downsample.conv")
        res("e.m1.", "encoder.mid.block_1.", 512, 512); attn("e.ma.", "encoder.mid.attn_1."); res("e.m2.", "encoder.mid.block_2.", 512, 512)
        norm("e.norm_out", "encoder.norm_out"); conv("e.conv_out", "encoder.conv_out")
        lin("quant", "quant_conv")
        lin("post_quant", "post_quant_conv")
        conv("d.conv_in", "decoder.conv_in")
        res("d.m1.", "decoder.mid.block_1.", 512, 512); attn("d.ma.", "decoder.mid.attn_1."); res("d.m2.", "decoder.mid.block_2.", 512, 512)
        for j in range(3):
            res(f"d.u3.b{j}.", f"decoder.up.3.block.{j}.", 512, 512)
        conv("d.u3.up", "decoder.up.3.upsample.conv")
        for j in range(2):                      # up.2.block.2 onward is dead code for ODISE (tap idx 5 = its input)
            res(f"d.u2.b{j}.", f"decoder.up.2.block.{j}.", 512, 512)

    def _gemm(self, a, name, **kw):
        return lib.gemm(a, self.W[name], nmma=self.nmma, bias=self.F.get(name + ".b"), **kw)

    def _gn(self, x, B, HW, name, act, lo=None, **kw):
        return ops.group_norm(x, B, HW, self.F[name + ".g"], self.F[name + ".be"], 1e-6, act,
                              lo=self.lo if lo is None else lo, **kw)

    def _res(self, n, x, B, H, W, cin, cout, xs=None):
        """ldm ResnetBlock.  xs: GroupNorm records of x left by its producer's epilogue (lib.GnStats) or None;
        returns (out, records of out)."""
        M = B * H * W
        _, a1 = self._gn(x, B, H * W, n + "n1", ACT_SILU, stats=xs)
        h = ops.empty(M, cout, self.dev)
        hs = lib.GnStats(M, cout, self.dev)
        self._gemm(a1, n + "c1", M=M, N=cout, conv=(cin, H, W), out=h, gn=hs)
        _, a2 = self._gn(h, B, H * W, n + "n2", ACT_SILU, stats=hs)
        if cin != cout:
            skip = ops.empty(M, cout, self.dev)
            self._gemm(ops.split(x, lo=self.lo), n + "sc", out=skip)
        else:
            skip = x
        out = ops.empty(M, cout, self.dev)
        os_ = lib.GnStats(M, cout, self.dev)
        self._gemm(a2, n + "c2", M=M, N=cout, conv=(cout, H, W), residual=skip, out=out, gn=os_)
        return out, os_

    def _attn(self, n, x, B, H, W, xs=None):
        """ldm AttnBlock: single head, d = C = 512, softmax(q k^T / sqrt(C)) v, 1x1 projections with bias."""
        T, C = H * W, 512
        M = B * T
        _, xn = self._gn(x, B, T, n + "n", ACT_NONE, stats=xs, lo=self.lb)
        qk = Planes.empty(M, 2 * C, self.dev, lo=self.lb)
        self._gemm(xn, n + "qk", out_planes=qk)
        vt = Planes.empty(C, M, self.dev, lo=self.lb)
        lib.gemm(self.W[n + "v"], xn, nmma=self.nmma, bias_m=self.F[n + "v.b"], out_planes=vt)
        S = torch.empty(B, T, T, dtype=torch.float32, device=self.dev)
        lib.gemm(qk.col_slice(0, C), qk.col_slice(C, C), M=T, N=T, K=C, nmma=self.nmma, batch=B, a_bs=T * qk.ld,
                 b_bs=T * qk.ld, out=S, ld_out=T, out_bs=T * T)
        P = ops.softmax_split(S.view(M, T), M, T, T, float(C) ** -0.5, lo=self.lb)
        o = Planes.empty(M, C, self.dev, lo=self.lb)
        lib.gemm(P, vt, M=T, N=C, K=T, nmma=self.nmma, batch=B, a_bs=T * P.ld, b_bs=T, out_planes=o, outp_bs=T * o.ld)
        out = ops.empty(M, C, self.dev)
        os_ = lib.GnStats(M, C, self.dev)
        self._gemm(o, n + "o", residual=x, out=out, gn=os_)
        return out, os_

    @torch.no_grad()
    def encode(self, img, B, H, W):
        """img: NHWC fp32 [B*H*W, 3], already (x - 0.5) / 0.5.  Returns dict(latent, enc5, enc7) of (tensor, h, w)."""
        cols, _, _ = ops.im2col3x3_split(img, B, H, W, lo=self.lb)
        h = ops.empty(B * H * W, 128, self.dev)
        hs = lib.GnStats(B * H * W, 128, self.dev)
        self._gemm(cols, "e.conv_in", out=h, gn=hs)
        taps = {}
        ch, cw = H, W
        for idx, (n, cin, cout, lvl) in enumerate(self.enc_blocks):
            if idx == 5:
                taps["enc5"] = (h, ch, cw)
            if idx == 7:
                taps["enc7"] = (h, ch, cw)
            h, hs = self._res(n, h, B, ch, cw, cin, cout, hs)
            if idx % 2 == 1 and lvl != 3:
                # ldm Downsample (with_conv): F.pad(x, (0,1,0,1)) then conv3x3 stride 2, no padding
                # strided implicit GEMM: conv_mode 2 = stride 2 with zero padding on the high side only
                d = ops.empty(B * (ch // 2) * (cw // 2), cout, self.dev)
                hs = lib.GnStats(B * (ch // 2) * (cw // 2), cout, self.dev)
                self._gemm(ops.split(h, lo=self.lo), f"e.d{lvl}.down", M=B * (ch // 2) * (cw // 2), N=cout,
                           conv=(cout, ch, cw), conv_mode=2, out=d, gn=hs)
                ch, cw = ch // 2, cw // 2
                h = d
        h, hs = self._res("e.m1.", h, B, ch, cw, 512, 512, hs)
        h, hs = self._attn("e.ma.", h, B, ch, cw, hs)
        h, hs = self._res("e.m2.", h, B, ch, cw, 512, 512, hs)
        _, a = self._gn(h, B, ch * cw, "e.norm_out", ACT_SILU, stats=hs)
        mom_p = Planes.empty(B * ch * cw, 8, self.dev, lo=self.lo)
        self._gemm(a, "e.conv_out", M=B * ch * cw, N=8, conv=(512, ch, cw), out_planes=mom_p)
        # quant_conv (1x1, 8 -> 8); posterior mean = first 4 channels; latent = 0.18215 * mean (ldm.py:461-465)
        mom = ops.empty(B * ch * cw, 8, self.dev)
        self._gemm(mom_p, "quant", out=mom)
        lat = ops.empty(B * ch * cw, 4, self.dev)
        ops.copy2d(mom[:, :4], lat, scale=SCALE_FACTOR)
        taps["latent"] = (lat, ch, cw)
        return taps

    @torch.no_grad()
    def decode_taps(self, latent, B, h, w):
        """latent NHWC [B*h*w, 4] (scaled).  Returns dict(dec2, dec5)."""
        z = ops.empty(B * h * w, 4, self.dev)
        ops.copy2d(latent, z, scale=1.0 / SCALE_FACTOR)          # ldm.py:536: z = 1/scale_factor * z
        z8 = torch.zeros(B * h * w, 8, dtype=torch.float32, device=self.dev)
        ops.copy2d(z, z8[:, :4])
        pq = ops.empty(B * h * w, 4, self.dev)
        self._gemm(ops.split(z8, lo=self.lo), "post_quant", out=pq)
        cols, _, _ = ops.im2col3x3_split(pq, B, h, w, lo=self.lo)
        x = ops.empty(B * h * w, 512, self.dev)
        xs = lib.GnStats(B * h * w, 512, self.dev)
        self._gemm(cols, "d.conv_in", out=x, gn=xs)
        x, xs = self._res("d.m1.", x, B, h, w, 512, 512, xs)
        x, xs = self._attn("d.ma.", x, B, h, w, xs)
        x, xs = self._res("d.m2.", x, B, h, w, 512, 512, xs)
        x, xs = self._res("d.u3.b0.", x, B, h, w, 512, 512, xs)
        x, xs = self._res("d.u3.b1.", x, B, h, w, 512, 512, xs)
        taps = {"dec2": (x, h, w)}
        x, xs = self._res("d.u3.b2.", x, B, h, w, 512, 512, xs)
        up = ops.upsample2x_split(x, B, h, w, lo=self.lo)
        y = ops.empty(B * 4 * h * w, 512, self.dev)
        ys = lib.GnStats(B * 4 * h * w, 512, self.dev)
        self._gemm(up, "d.u3.up", M=B * 4 * h * w, N=512, conv=(512, 2 * h, 2 * w), out=y, gn=ys)
        y, ys = self._res("d.u2.b0.", y, B, 2 * h, 2 * w, 512, 512, ys)
        y, _ = self._res("d.u2.b1.", y, B, 2 * h, 2 * w, 512, 512, ys)
        taps["dec5"] = (y, 2 * h, 2 * w)
        return taps
