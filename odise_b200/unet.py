"""H100 engine for the frozen SD-v1 UNet feature pass of ODISE (SURVEY.md §8a rows a6, a7, a7.1-a7.3).

Computes exactly what LdmExtractor.unet_forward (odise/modeling/meta_arch/ldm.py:469-491) needs from the UNet at
t = 0: the inputs of output_blocks[2, 5, 8, 11].  output_blocks[11] and unet.out are never executed (their results
are discarded by the reference, ldm.py:600).  Layout is NHWC / token-major throughout, so every conv / linear /
attention projection is one call of the wgmma GEMM (odise_gemm_bf16) and the skip concatenations of the up path
(torch.cat, ldm.py:485) cost nothing: down-path blocks write their outputs straight into the right half of the
concat buffer their mirror block will read, up-path blocks into the left half.

All arithmetic runs in libodise_b200.so; torch only owns the memory.
"""
import torch

from . import lib, ops, spec
from .lib import Planes
from .ops import ACT_NONE, ACT_SILU

HEADS = 8
CTX_T = 77
CTX_TS = 80    # context rows per image in the key / value planes (zero padded; TMA alignment)


def _conv_w(w):
    """[Co, Ci, 3, 3] -> [Co, 9*Ci] with k = (kh*3 + kw)*Ci + ci (the implicit-GEMM K order)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


class UNetEngine:
    def __init__(self, sd, device, nmma=3, prefix=spec.UNET_PREFIX):
        self.dev = torch.device(device)
        self.nmma = nmma            # 3 = bf16x3 (bf16 pairs) | 2 = F16Q8 (fp16 + e5m2 cross terms, lib.Q8) | 1 = plain bf16
        self.lo = lib.Q8 if nmma == 2 else (nmma == 3)
        self.lb = bool(self.lo)     # attention operands (q, k: bf16 pair; V^T: fp16 pair) keep their formats in every mode
        self.p = prefix
        self.inp, self.mid, self.out = spec.unet_blocks()
        self.W = {}     # name -> Planes (GEMM weights)
        self.F = {}     # name -> fp32 device tensor (biases, norm params)
        self._prep(sd)

    # ------------------------------------------------------------------------------------------- weights
    def _planes(self, w2d):
        w2d = w2d.to(self.dev, torch.float32).contiguous()
        K = w2d.shape[1]
        if K % 8:
            w2d = torch.nn.functional.pad(w2d, (0, 8 - K % 8))
        return lib.split(w2d, lo=self.lo)

    def _f(self, t):
        return t.to(self.dev, torch.float32).contiguous()

    def _prep(self, sd):
        p = self.p
        g = lambda n: sd[p + n]
        emb_w, emb_b = [], []
        self.emb_off = {}
        off = 0

        def res(q, cin, cout):
            nonlocal off
            self.F[q + "gn1.g"], self.F[q + "gn1.b"] = self._f(g(q + "in_layers.0.weight")), self._f(g(q + "in_layers.0.bias"))
            self.W[q + "conv1"] = self._planes(_conv_w(g(q + "in_layers.2.weight")))
            self.F[q + "conv1.b"] = self._f(g(q + "in_layers.2.bias"))
            emb_w.append(g(q + "emb_layers.1.weight"))
            emb_b.append(g(q + "emb_layers.1.bias"))
            self.emb_off[q] = (off, cout)
            off += cout
            self.F[q + "gn2.g"], self.F[q + "gn2.b"] = self._f(g(q + "out_layers.0.weight")), self._f(g(q + "out_layers.0.bias"))
            self.W[q + "conv2"] = self._planes(_conv_w(g(q + "out_layers.3.weight")))
            self.F[q + "conv2.b"] = self._f(g(q + "out_layers.3.bias"))
            if cin != cout:
                self.W[q + "skip"] = self._planes(g(q + "skip_connection.weight").reshape(cout, cin))
                self.F[q + "skip.b"] = self._f(g(q + "skip_connection.bias"))

        def st(q, ch):
            d = ch // HEADS
            HS = ops.head_stride(d)
            t = q + "transformer_blocks.0."
            self.F[q + "norm.g"], self.F[q + "norm.b"] = self._f(g(q + "norm.weight")), self._f(g(q + "norm.bias"))
            self.W[q + "proj_in"] = self._planes(g(q + "proj_in.weight").reshape(ch, ch))
            self.F[q + "proj_in.b"] = self._f(g(q + "proj_in.bias"))
            for a in ("attn1", "attn2"):
                wq, wk, wv = g(t + a + ".to_q.weight"), g(t + a + ".to_k.weight"), g(t + a + ".to_v.weight")
                if HS is not None:   # fused kernel: head-padded projections (zero rows in the pad)
                    wq, wk, wv = (ops.head_pad_rows(w, HEADS, d, HS) for w in (wq, wk, wv))
                if a == "attn1":
                    self.W[t + a + ".qk"] = self._planes(torch.cat([wq, wk], 0))
                else:
                    self.W[t + a + ".q"] = self._planes(wq)
                    self.W[t + a + ".k"] = self._planes(wk)
                self.W[t + a + ".v"] = self._planes(wv)
                self.W[t + a + ".out"] = self._planes(g(t + a + ".to_out.0.weight"))
                self.F[t + a + ".out.b"] = self._f(g(t + a + ".to_out.0.bias"))
            # GEGLU fused into the FF1 epilogue: interleave (a, gate) rows in quads so both land in one lane pair
            w1, b1 = g(t + "ff.net.0.proj.weight"), g(t + "ff.net.0.proj.bias")
            h4 = 4 * ch
            w1 = torch.stack([w1[:h4].reshape(h4 // 4, 4, ch), w1[h4:].reshape(h4 // 4, 4, ch)], 1).reshape(2 * h4, ch)
            b1 = torch.stack([b1[:h4].reshape(h4 // 4, 4), b1[h4:].reshape(h4 // 4, 4)], 1).reshape(2 * h4)
            self.W[t + "ff1"] = self._planes(w1)
            self.F[t + "ff1.b"] = self._f(b1)
            self.W[t + "ff2"] = self._planes(g(t + "ff.net.2.weight"))
            self.F[t + "ff2.b"] = self._f(g(t + "ff.net.2.bias"))
            for n in ("norm1", "norm2", "norm3"):
                self.F[t + n + ".g"], self.F[t + n + ".b"] = self._f(g(t + n + ".weight")), self._f(g(t + n + ".bias"))
            self.W[q + "proj_out"] = self._planes(g(q + "proj_out.weight").reshape(ch, ch))
            self.F[q + "proj_out.b"] = self._f(g(q + "proj_out.bias"))

        def block(q, layers):
            for j, l in enumerate(layers):
                r = f"{q}{j}."
                if l[0] == "conv_in":
                    self.W[r + "conv"] = self._planes(_conv_w(g(r + "weight")))
                    self.F[r + "conv.b"] = self._f(g(r + "bias"))
                elif l[0] == "res":
                    res(r, l[1], l[2])
                elif l[0] == "st":
                    st(r, l[1])
                elif l[0] == "down":
                    self.W[r + "conv"] = self._planes(_conv_w(g(r + "op.weight")))
                    self.F[r + "conv.b"] = self._f(g(r + "op.bias"))
                elif l[0] == "up":
                    self.W[r + "conv"] = self._planes(_conv_w(g(r + "conv.weight")))
                    self.F[r + "conv.b"] = self._f(g(r + "conv.bias"))

        for i, layers in enumerate(self.inp):
            block(f"input_blocks.{i}.", layers)
        block("middle_block.", self.mid)
        for i, layers in enumerate(self.out[:11]):   # output_blocks[11] is dead code for ODISE
            block(f"output_blocks.{i}.", layers)
        self.W["emb_all"] = self._planes(torch.cat(emb_w, 0))
        self.F["emb_all.b"] = self._f(torch.cat(emb_b, 0))
        self.emb_total = off
        # time embedding at t = 0 is a constant of the weights: timestep_embedding(0, 320) = [1]*160 + [0]*160
        # (cos first; SURVEY.md App. A) -> time_embed MLP, folded once at load time with our own GEMM.
        t_emb = torch.cat([torch.ones(1, 160), torch.zeros(1, 160)], 1).to(self.dev)
        w0, w2 = self._planes(g("time_embed.0.weight")), self._planes(g("time_embed.2.weight"))
        h = Planes.empty(1, 1280, self.dev, lo=self.lo)
        lib.gemm(lib.split(t_emb, lo=self.lo), w0, nmma=self.nmma, bias=self._f(g("time_embed.0.bias")), act=ACT_SILU,
                 out_planes=h)
        self.emb0 = ops.empty(1, 1280, self.dev)
        lib.gemm(h, w2, nmma=self.nmma, bias=self._f(g("time_embed.2.bias")), out=self.emb0)

    # ------------------------------------------------------------------------------------------- primitives
    def _gemm(self, a, wname, bias=None, **kw):
        if "conv" in kw and kw.get("conv_mode", 0) == 0:
            # low-resolution levels cannot fill 132 SMs with output tiles: split K (lib.auto_split)
            Mc, Nc, Kc = kw["M"], kw["N"], 9 * kw["conv"][0]
            bn, sk = lib.auto_split(Mc, Nc, Kc)
            if sk > 1:
                kw.update(split_k=sk, force_bn=bn, workspace=lib.workspace(sk * Mc * Nc * 4, self.dev))
        return lib.gemm(a, self.W[wname], nmma=self.nmma, bias=self.F[bias] if bias else None, **kw)

    def _resblock(self, q, x, B, H, W, cin, cout, emb_all, dst, xs=None, ds=None):
        """x: fp32 view [B*H*W, cin]; dst: fp32 view [B*H*W, cout] (may be a column slice of a concat buffer).
        xs / ds: lib.GnStats views of x / dst — the GroupNorm statistics travel with the activations: every GEMM that
        writes an activation a GroupNorm will read leaves the per-segment records in its epilogue (conv + GN fusion, producer
        side), so in_layers[0] / out_layers[0] never re-read the activation for its statistics."""
        M = B * H * W
        imp = lib.conv_ok(H, W)          # False: map width the implicit-GEMM TMA boxes cannot tile -> materialised im2col
        y1, a1 = ops.group_norm(x, B, H * W, self.F[q + "gn1.g"], self.F[q + "gn1.b"], 1e-5, ACT_SILU, lo=self.lo,
                                want_f32=not imp, want_planes=imp, stats=xs)
        eo, ec = self.emb_off[q]
        h = ops.empty(M, cout, self.dev)
        hs = lib.GnStats(M, cout, self.dev)
        if imp:
            self._gemm(a1, q + "conv1", q + "conv1.b", M=M, N=cout, conv=(cin, H, W), rowbias=emb_all[:, eo:eo + ec],
                       rows_per_group=H * W, out=h, gn=hs)
        else:
            self._gemm(ops.im2col3x3_split(y1, B, H, W, lo=self.lo)[0], q + "conv1", q + "conv1.b",
                       rowbias=emb_all[:, eo:eo + ec], rows_per_group=H * W, out=h, gn=hs)
        y2, a2 = ops.group_norm(h, B, H * W, self.F[q + "gn2.g"], self.F[q + "gn2.b"], 1e-5, ACT_SILU, lo=self.lo,
                                want_f32=not imp, want_planes=imp, stats=hs)
        if cin != cout:
            skip = ops.empty(M, cout, self.dev)
            self._gemm(lib.split(x, lo=self.lo), q + "skip", q + "skip.b", out=skip)
        else:
            skip = x
        if imp:
            self._gemm(a2, q + "conv2", q + "conv2.b", M=M, N=cout, conv=(cout, H, W), residual=skip, out=dst, gn=ds)
        else:
            self._gemm(ops.im2col3x3_split(y2, B, H, W, lo=self.lo)[0], q + "conv2", q + "conv2.b", residual=skip, out=dst,
                       gn=ds)
        return dst

    def _attention(self, t, a, xq, kv_src, B, T, Tk, ch, TkS=None):
        """Returns Planes [B*T, ch] = softmax(q k^T / sqrt(d)) v.  xq: LN'd planes [B*T, ch];
        kv_src: planes [B*TkS, Kdim] (== xq for self-attention; the context carries TkS = 80 rows per image,
        zero rows after the 77 tokens, so every TMA box start is 16-byte aligned)."""
        TkS = TkS or Tk
        d = ch // HEADS
        HS = ops.head_stride(d)
        scale = d ** -0.5
        M = B * T
        if HS is not None:
            Cp = HEADS * HS
            if a == "attn1" and kv_src is xq:
                qk = Planes.empty(M, 2 * Cp, self.dev, lo=self.lb)
                self._gemm(xq, t + a + ".qk", out_planes=qk)
                qP, kP = qk.col_slice(0, Cp), qk.col_slice(Cp, Cp)
            elif a == "attn1":           # keys / values from the row-padded copy of the tokens (T % 8 != 0)
                wqk = self.W[t + a + ".qk"]
                qP = Planes.empty(M, Cp, self.dev, lo=self.lb)
                lib.gemm(xq, wqk.row_slice(0, Cp), nmma=self.nmma, out_planes=qP)
                kP = Planes.empty(B * TkS, Cp, self.dev, lo=self.lb)
                lib.gemm(kv_src, wqk.row_slice(Cp, Cp), nmma=self.nmma, out_planes=kP)
            else:
                qP = Planes.empty(M, Cp, self.dev, lo=self.lb)
                self._gemm(xq, t + a + ".q", out_planes=qP)
                kP = Planes.empty(B * TkS, Cp, self.dev, lo=self.lb)
                self._gemm(kv_src, t + a + ".k", out_planes=kP)
            vt = Planes.empty(Cp, B * TkS, self.dev, lo=self.lb, f16=self.lb)   # fp16 pair in the bf16x3 mode
            # V^T = Wv_pad @ X^T: the same K-major GEMM with the operands swapped
            lib.gemm(self.W[t + a + ".v"], kv_src, nmma=self.nmma, out_planes=vt)
            _, o = ops.attention_tc(qP, kP, vt, B, HEADS, d, T, Tk, scale, self.nmma, tk_stride=TkS, lo=self.lo)
            return o
        if self.nmma == 2:
            raise lib.OdiseError("UNetEngine: the unfused attention path (head dims outside 40 / 80 / 160) has no F16Q8 mode")
        # head dim 160 (16x16 and 8x8 levels, < 2 % of the FLOPs): unfused S / softmax / PV through the GEMM
        src, Tkp = kv_src, TkS
        if a == "attn1":
            qk = Planes.empty(M, 2 * ch, self.dev, lo=self.lo)
            self._gemm(xq, t + a + ".qk", out_planes=qk)
            qP, kP = qk.col_slice(0, ch), qk.col_slice(ch, ch)
        else:
            qP = Planes.empty(M, ch, self.dev, lo=self.lo)
            self._gemm(xq, t + a + ".q", out_planes=qP)
            kP = Planes.empty(B * Tkp, ch, self.dev, lo=self.lo)
            self._gemm(src, t + a + ".k", out_planes=kP)
        vt = Planes.empty(ch, B * Tkp, self.dev, lo=self.lo)
        lib.gemm(self.W[t + a + ".v"], src, nmma=self.nmma, out_planes=vt)
        o = Planes.empty(M, ch, self.dev, lo=self.lo)
        S = torch.empty(B, T, Tkp, dtype=torch.float32, device=self.dev)
        for h in range(HEADS):
            lib.gemm(qP.col_slice(h * d, d), kP.col_slice(h * d, d), M=T, N=Tkp, K=d, nmma=self.nmma, batch=B,
                     a_bs=T * qP.ld, b_bs=Tkp * kP.ld, out=S, ld_out=Tkp, out_bs=T * Tkp)
            P = ops.softmax_split(S.view(B * T, Tkp), B * T, Tk, Tkp, scale, lo=self.lo)
            lib.gemm(P, vt.row_slice(h * d, d), M=T, N=d, K=Tkp, nmma=self.nmma, batch=B, a_bs=T * P.ld, b_bs=Tkp,
                     out_planes=o.col_slice(h * d, d), outp_bs=T * o.ld)
        return o

    def _st(self, q, x, B, H, W, ch, ctx, dst, xs=None, ds=None):
        T = H * W
        M = B * T
        t = q + "transformer_blocks.0."
        _, xn = ops.group_norm(x, B, T, self.F[q + "norm.g"], self.F[q + "norm.b"], 1e-6, ACT_NONE, lo=self.lo, stats=xs)
        h = ops.empty(M, ch, self.dev)
        self._gemm(xn, q + "proj_in", q + "proj_in.b", out=h)
        if T % 8 == 0:
            _, n1 = ops.layer_norm(h, self.F[t + "norm1.g"], self.F[t + "norm1.b"], lo=self.lo)
            o1 = self._attention(t, "attn1", n1, n1, B, T, T, ch)
        else:
            # token counts that are not a multiple of 8 (6 x 6 = 36 at a 48 x 48 latent): the key / value planes carry
            # TkS = ceil8(T) rows per image (zero rows, masked as keys) so the attention kernel's TMA box starts stay aligned
            TkS = (T + 7) // 8 * 8
            y1, n1 = ops.layer_norm(h, self.F[t + "norm1.g"], self.F[t + "norm1.b"], lo=self.lo, want_f32=True)
            kvp = torch.zeros(B, TkS * ch, dtype=torch.float32, device=self.dev)
            ops.copy2d(y1.view(B, T * ch), kvp[:, :T * ch])
            o1 = self._attention(t, "attn1", n1, lib.split(kvp.view(B * TkS, ch), lo=self.lo), B, T, T, ch, TkS=TkS)
        h2 = ops.empty(M, ch, self.dev)
        self._gemm(o1, t + "attn1.out", t + "attn1.out.b", residual=h, out=h2)
        _, n2 = ops.layer_norm(h2, self.F[t + "norm2.g"], self.F[t + "norm2.b"], lo=self.lo)
        o2 = self._attention(t, "attn2", n2, ctx, B, T, CTX_T, ch, TkS=CTX_TS)
        h3 = ops.empty(M, ch, self.dev)
        self._gemm(o2, t + "attn2.out", t + "attn2.out.b", residual=h2, out=h3)
        _, n3 = ops.layer_norm(h3, self.F[t + "norm3.g"], self.F[t + "norm3.b"], lo=self.lo)
        gg = Planes.empty(M, 4 * ch, self.dev, lo=self.lo)
        self._gemm(n3, t + "ff1", t + "ff1.b", out_planes=gg, geglu=True)
        h4p = Planes.empty(M, ch, self.dev, lo=self.lo)
        self._gemm(gg, t + "ff2", t + "ff2.b", residual=h3, out_planes=h4p)
        self._gemm(h4p, q + "proj_out", q + "proj_out.b", residual=x, out=dst, gn=ds)
        return dst

    # ------------------------------------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, x, B, H, W, context, cond_emb=None):
        """x: noisy latent, NHWC fp32 [B*H*W, 4]; context [B*77, 768] fp32; cond_emb [B, 1280] fp32 or None.
        Returns the 4 taps as NHWC fp32 matrices [(tensor [B*h*w, C], h, w), ...] for output blocks 2, 5, 8, 11."""
        dev = self.dev
        if cond_emb is not None:
            emb, _ = ops.add_split(cond_emb, self.emb0, b_rows=1, want_f32=True, want_planes=False)
        else:
            emb = self.emb0.expand(B, 1280).contiguous()
        e_silu = ops.act_split(emb, ACT_SILU, lo=self.lo)
        emb_all = ops.empty(B, self.emb_total, dev)
        self._gemm(e_silu, "emb_all", "emb_all.b", out=emb_all)
        # context with 80 rows per image (3 zero rows): keeps the v^T box starts of the attention kernel aligned
        cpad = torch.zeros(B, CTX_TS, context.shape[1], dtype=torch.float32, device=dev)
        nc = CTX_T * context.shape[1]
        ops.copy2d(context.view(B, nc), cpad.view(B, CTX_TS * context.shape[1])[:, :nc])
        ctx = lib.split(cpad.view(B * CTX_TS, -1), lo=self.lo)

        # spatial size / channels of every down-path output (= skip), to lay out the concat buffers
        sizes = []
        h_, w_ = H, W
        for layers in self.inp:
            if layers[0][0] == "down":
                h_, w_ = h_ // 2, w_ // 2
            cout = layers[0][2] if layers[0][0] in ("conv_in", "res") else layers[0][1]
            sizes.append((h_, w_, cout))
        # cat[i] = input of output block i = [h (left) | skip hs[11 - i] (right)]
        ch_in = [l[0][1] for l in self.out]                      # channels of the concat
        cat, cst = [], []
        for i in range(12):
            hh, ww, cs = sizes[11 - i]
            cat.append((torch.empty(B * hh * ww, ch_in[i], dtype=torch.float32, device=dev), ch_in[i] - cs, hh, ww))
            cst.append(lib.GnStats(B * hh * ww, ch_in[i], dev))   # GroupNorm records of the whole concat [h | skip]

        def skip_view(j):   # where down-path output j lives (+ the matching columns of the statistics records)
            buf, cl, hh, ww = cat[11 - j]
            return buf[:, cl:], cst[11 - j].cols(cl, buf.shape[1] - cl)

        cur, cur_s, ch_, cw_ = None, None, H, W
        for j, layers in enumerate(self.inp):
            q = f"input_blocks.{j}."
            dst, dst_s = skip_view(j)
            kind = layers[0][0]
            if kind == "conv_in":
                cols, _, _ = ops.im2col3x3_split(x, B, H, W, lo=self.lo)
                self._gemm(cols, q + "0.conv", q + "0.conv.b", out=dst, gn=dst_s)
            elif kind == "down":
                # ldm Downsample = conv3x3 stride 2 pad 1: strided implicit GEMM (TMA element strides), no im2col
                cdim = layers[0][1]
                if lib.conv_ok(ch_ // 2, cw_ // 2):
                    self._gemm(lib.split(cur, lo=self.lo), q + "0.conv", q + "0.conv.b", M=B * (ch_ // 2) * (cw_ // 2),
                               N=cdim, conv=(cdim, ch_, cw_), conv_mode=1, out=dst, gn=dst_s)
                else:
                    self._gemm(ops.im2col3x3_split(cur, B, ch_, cw_, stride=2, lo=self.lo)[0], q + "0.conv", q + "0.conv.b",
                               out=dst, gn=dst_s)
                ch_, cw_ = ch_ // 2, cw_ // 2
            else:
                _, cin, cout = layers[0]
                if len(layers) == 1:
                    self._resblock(q + "0.", cur, B, ch_, cw_, cin, cout, emb_all, dst, cur_s, dst_s)
                else:
                    tmp = ops.empty(B * ch_ * cw_, cout, dev)
                    tmp_s = lib.GnStats(B * ch_ * cw_, cout, dev)
                    self._resblock(q + "0.", cur, B, ch_, cw_, cin, cout, emb_all, tmp, cur_s, tmp_s)
                    self._st(q + "1.", tmp, B, ch_, cw_, cout, ctx, dst, tmp_s, dst_s)
            cur, cur_s = dst, dst_s
        # middle block -> left part of cat[0]
        c = self.mid[0][1]
        Mm = B * ch_ * cw_
        t1, t1s = ops.empty(Mm, c, dev), lib.GnStats(Mm, c, dev)
        self._resblock("middle_block.0.", cur, B, ch_, cw_, c, c, emb_all, t1, cur_s, t1s)
        t2, t2s = ops.empty(Mm, c, dev), lib.GnStats(Mm, c, dev)
        self._st("middle_block.1.", t1, B, ch_, cw_, c, ctx, t2, t1s, t2s)
        self._resblock("middle_block.2.", t2, B, ch_, cw_, c, c, emb_all, cat[0][0][:, :cat[0][1]], t2s,
                       cst[0].cols(0, cat[0][1]))

        taps = []
        for i in range(12):
            buf, cl, hh, ww = cat[i]
            if i in (2, 5, 8, 11):
                taps.append((buf, hh, ww))
            if i == 11:
                break
            layers = self.out[i]
            q = f"output_blocks.{i}."
            nbuf, ncl, nh, nw = cat[i + 1]
            dst, dst_s = nbuf[:, :ncl], cst[i + 1].cols(0, ncl)
            _, cin, cout = layers[0]
            last_is_res = len(layers) == 1
            t, ts = (dst, dst_s) if last_is_res else (ops.empty(B * hh * ww, cout, dev), lib.GnStats(B * hh * ww, cout, dev))
            self._resblock(q + "0.", buf, B, hh, ww, cin, cout, emb_all, t, cst[i], ts)
            k = 1
            if k < len(layers) and layers[k][0] == "st":
                t_out, to_s = (dst, dst_s) if k == len(layers) - 1 else (ops.empty(B * hh * ww, cout, dev), None)
                self._st(f"{q}{k}.", t, B, hh, ww, cout, ctx, t_out, ts, to_s)
                t = t_out
                k += 1
            if k < len(layers) and layers[k][0] == "up":
                if lib.conv_ok(2 * hh, 2 * ww):
                    up = ops.upsample2x_split(t, B, hh, ww, lo=self.lo)
                    self._gemm(up, f"{q}{k}.conv", f"{q}{k}.conv.b", M=B * 4 * hh * ww, N=cout,
                               conv=(cout, 2 * hh, 2 * ww), out=dst, gn=dst_s)
                else:
                    up = ops.resize_nhwc(t, B, hh, ww, 2 * hh, 2 * ww, bilinear=False)
                    self._gemm(ops.im2col3x3_split(up, B, 2 * hh, 2 * ww, lo=self.lo)[0], f"{q}{k}.conv", f"{q}{k}.conv.b",
                               out=dst, gn=dst_s)
        return taps
