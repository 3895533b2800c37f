"""GPU parity of the fused wgmma flash attention (odise_attention_tc) vs fp64 softmax attention.
Shapes are those of the four engines that call it: the SD-v1 UNet (self-attention d=40 / d=80 / d=160, cross-attention
over 77 context tokens), the CLIP image and text towers (d=64), MaskCLIP's mask tokens and the Mask2Former decoder (d=32).
Tolerance in the bf16x3 mode: the probabilities enter the P V product rounded ONCE to fp16 (2^-12 relative per element,
random sign -> ~1.5e-4 of the output scale on random data); the budget behind that choice is tools/precision_budget.py
(5e-5 on the UNet taps, bar 1e-3).  S = Q K^T stays bf16x3 (2^-16).  tests/test_attention_tolerance_cpu.py emulates that
arithmetic on the CPU for every case of the tables below and checks that the emulated error stays under half the bar."""
# Expected size (round 2 note): each probability carries an independent relative rounding error of rms 2^-11 / sqrt(3) =
# 2.8e-4; with n_eff = n / e effective keys for N(0, 1) scores the output error is 2.8e-4 |v| / sqrt(n_eff) rms, while the
# outputs themselves are ~|v| / sqrt(n_eff): the max-error / max-output ratio this file measures is therefore ~2.8e-4
# whatever n is, and one realisation lands anywhere in 1.5e-4 .. 4e-4.  The bound is 2x that expectation.
TOL3 = 6e-4
TOL1 = 3e-2
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def _tol(nmma):
    return TOL3 if nmma == 3 else TOL1


def ceil8(n):
    return (n + 7) // 8 * 8


# ------------------------------------------------------------------------------------------------ case tables (CPU data)
# (B, heads, d, Tq, Tk); the key / value planes carry TkS = ceil8(Tk) rows per image
TC_CASES = [
    (2, 8, 40, 256, 256), (1, 8, 40, 1024, 1024), (2, 8, 80, 256, 256), (3, 8, 40, 128, 77), (2, 8, 80, 64, 77),
    (1, 4, 80, 64, 64), (2, 2, 40, 200, 130), (1, 8, 40, 4096, 4096), (2, 8, 160, 256, 256), (3, 8, 160, 64, 64),
    (2, 8, 160, 256, 77), (1, 3, 160, 144, 144),
    (2, 16, 64, 584, 577),     # CLIP ViT-L/14 image tower (clip.py:59): 577 tokens in 584-row image blocks
    (2, 12, 64, 80, 77),       # CLIP text tower: ctx 77 padded to 80 rows (unmasked here; causal in MASKED_CASES)
    (2, 4, 48, 200, 130),      # DP = 48
    (2, 4, 56, 256, 200),      # DP = 64 with 8 unused pad lanes (dpart < DP)
    (2, 4, 72, 192, 160),      # DP = 80: two 64-column chunks, the second one 8 columns wide
    (2, 4, 16, 130, 100),      # DP = 32 with half of it unused
    (3, 4, 64, 1, 77), (2, 2, 160, 1, 64),     # a single query row
    (2, 4, 40, 64, 4), (2, 2, 64, 130, 4),     # Tk = 4 in 8-row blocks: one ragged key block
]

# (kind, B, heads, d, Tq, Tk, TkS).  causal: ClipTextEngine's recipe | maskclip: MaskCLIP's mask tokens, bits from
# ops.maskclip_bits | random: random per-(image, row) bits with the edge rows of _random_mask
MASKED_CASES = [
    ("causal", 2, 12, 64, 80, 77, 80), ("causal", 3, 8, 40, 80, 77, 80), ("causal", 2, 8, 32, 80, 77, 80),
    ("maskclip", 2, 16, 64, 150, 577, 584), ("maskclip", 2, 4, 40, 150, 577, 584),
    ("random", 2, 4, 64, 200, 96, 96), ("random", 2, 4, 40, 200, 96, 104), ("random", 2, 8, 32, 200, 96, 96),
    ("random", 2, 4, 64, 130, 577, 584), ("random", 3, 4, 40, 64, 200, 200),
]

# (kind, B, heads, d, Tq, Tk).  peaked: logits of std ~8 | rising: every row's logits grow by ~5 per 64-key block |
# dominant: one key 30 above the rest, alone in the ragged last block (577 = 9 * 64 + 1)
STRESS_CASES = [(kind, 2, 4, d, 256, 577) for kind in ("peaked", "rising", "dominant") for d in (40, 64, 160)]


def attention_inputs(B, heads, d, Tq, Tk, seed, qscale=1.0):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Tq, heads, d, generator=g) * qscale
    k = torch.randn(B, Tk, heads, d, generator=g)
    v = torch.randn(B, Tk, heads, d, generator=g)
    return q, k, v


def tc_case(cfg):
    """-> q, k, v [B, T, heads, d] fp32 (CPU) of a TC_CASES entry"""
    B, heads, d, Tq, Tk = cfg
    return attention_inputs(B, heads, d, Tq, Tk, Tq * 3 + Tk + d)


def causal_bits(ctx, TS):
    """ClipTextEngine.__init__'s causal mask: [TS, ceil(ctx / 32)] int32 words, row_any [TS] (0 on the pad query rows)"""
    words = (ctx + 31) // 32
    q = torch.arange(TS).view(-1, 1, 1)
    key = (torch.arange(words).view(1, -1, 1) * 32 + torch.arange(32).view(1, 1, -1))
    allowed = ((key <= q) & (key < ctx)).to(torch.int64)                       # causal: query i sees keys <= i
    row_bits = (allowed << torch.arange(32).view(1, 1, -1)).sum(-1)            # [TS, words] as uint32 values
    row_bits = torch.where(row_bits >= 2 ** 31, row_bits - 2 ** 32, row_bits).to(torch.int32)
    return row_bits, (torch.arange(TS) < ctx).to(torch.int32)


def pack_bits(allowed):
    """bool [B, Tq, Tk] -> int32 words [B, Tq, ceil(Tk / 32)], bit t % 32 of word t // 32 = key t may be attended"""
    B, Tq, Tk = allowed.shape
    W = (Tk + 31) // 32
    a = torch.zeros(B, Tq, W * 32, dtype=torch.int64)
    a[..., :Tk] = allowed.long()
    w = (a.view(B, Tq, W, 32) << torch.arange(32)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def unpack_bits(bits, Tk):
    return ((bits.long().unsqueeze(-1) >> torch.arange(32, device=bits.device)) & 1).bool().flatten(-2)[..., :Tk]


def maskclip_logits(B, Q, seed, hm=16, wm=16):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, Q, hm, wm, generator=g) * 3 - 1.0


def maskclip_allowed(logits, S=336, P=14):
    """MaskCLIP's key mask (clip.py:291-321): class token always on, patch on iff sigmoid(max over its window of the
    bilinearly upsampled mask) >= 0.5.  [B, Q, 1 + (S / P)^2] bool"""
    up = F.interpolate(logits, size=(S, S), mode="bilinear", align_corners=False)
    on = F.max_pool2d(up, P).sigmoid().flatten(2) >= 0.5
    return torch.cat([torch.ones_like(on[..., :1]), on], -1)


def _random_mask(B, Tq, Tk, g):
    allowed = torch.rand(B, Tq, Tk, generator=g) < 0.4
    for r in (0, min(130, Tq - 1)):          # the only attendable key sits in the last, ragged key block
        allowed[:, r] = False
        allowed[:, r, Tk - 1] = True
    allowed[:, 1] = False                    # two keys, the last block's first and last
    allowed[:, 1, (Tk - 1) // 64 * 64] = True
    allowed[:, 1, Tk - 1] = True
    allowed[0, 2] = False                    # fully blocked: row_any = 0, the row attends everywhere (odise.py:683)
    row_any = allowed.any(-1).to(torch.int32)
    row_any[-1, 3] = 0                       # a row whose bits exist but must be ignored
    return allowed, row_any


def masked_case(case):
    """-> q, k, v, allowed [B, Tq, Tk] bool, row_any [B, Tq] int32, bits int32 words or None (maskclip: the kernel's
    bits come from ops.maskclip_bits on the logits returned as the last item; `allowed` is the torch recipe)"""
    kind, B, heads, d, Tq, Tk, TkS = case
    seed = 1000 * len(kind) + B * 100 + d * 7 + Tq + Tk
    q, k, v = attention_inputs(B, heads, d, Tq, Tk, seed)
    logits = None
    if kind == "causal":
        rb, ra = causal_bits(Tk, Tq)
        bits, row_any = rb.expand(B, -1, -1).contiguous(), ra.expand(B, -1).contiguous()
        allowed = unpack_bits(bits, Tk)
    elif kind == "maskclip":
        logits = maskclip_logits(B, Tq, seed)
        allowed = maskclip_allowed(logits)
        row_any = torch.ones(B, Tq, dtype=torch.int32)
        bits = None
    else:
        allowed, row_any = _random_mask(B, Tq, Tk, torch.Generator().manual_seed(seed + 1))
        bits = pack_bits(allowed)
    return q, k, v, allowed, row_any, bits, logits


def stress_case(case):
    """-> q, k, v of a STRESS_CASES entry"""
    kind, B, heads, d, Tq, Tk = case
    scale = d ** -0.5
    q, k, v = attention_inputs(B, heads, d, Tq, Tk, 77 + d + len(kind), qscale=8.0 if kind == "peaked" else 1.0)
    if kind == "rising":
        # a shared direction: q . e = 4, k_t . e ramps so that the logits gain ~5 per 64-key block; the ramp is centred
        # on 0 (logits in about [-22, 22]) because S = Q K^T carries an absolute error proportional to |S|
        q[..., 0] += 4.0
        k[..., 0] += (torch.arange(Tk).view(1, Tk, 1) - Tk / 2) * (5.0 / 64) / (4.0 * scale)
    elif kind == "dominant":
        q[..., 0] += 4.0
        k[:, Tk - 1, :, 0] += 30.0 / (4.0 * scale)
    return q, k, v


def effective_mask(allowed, row_any):
    """the kernel's semantics: a row with row_any = 0 ignores its bits"""
    return allowed | (row_any == 0).unsqueeze(-1)


def reference(q, k, v, scale, allowed=None):
    """fp64 softmax attention -> [B*Tq, heads*d]; allowed [B, Tq, Tk] bool (None: every key)"""
    B, Tq, heads, d = q.shape
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), k.double()) * scale
    if allowed is not None:
        s = s.masked_fill(~allowed.to(s.device)[:, None], float("-inf"))
    return torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v.double()).reshape(B * Tq, heads * d)


# ------------------------------------------------------------------------------------------------ GPU operands
def _planes(q, k, v, TkS, nmma, dev):
    """head-padded operand planes under the kernel's contract (attn_tc.cu:10-15): zero head pad columns in q and k;
    large finite junk in the pad keys of k and v^T and in the head pad rows of v^T"""
    from odise_b200 import lib, ops
    B, Tq, heads, d = q.shape
    Tk = k.shape[1]
    HS = ops.head_stride(d)
    qp = torch.zeros(B * Tq, heads, HS)
    qp[:, :, :d] = q.reshape(B * Tq, heads, d)
    kp = torch.zeros(B, TkS, heads, HS)
    kp[:, :Tk, :, :d] = k
    kp[:, Tk:] = 7.0                     # pad keys must be masked, not merely zero
    vt = torch.full((heads, HS, B, TkS), 3.0)
    vt[:, :d, :, :Tk] = v.permute(2, 3, 0, 1)
    vt[:, :, :, Tk:] = 1e3               # finite: exp(-inf) = 0 must zero them, 0 * 1e3 stays 0
    qP = lib.split(qp.view(B * Tq, heads * HS).to(dev))
    kP = lib.split(kp.view(B * TkS, heads * HS).to(dev))
    vP = lib.split(vt.view(heads * HS, B * TkS).to(dev), f16=nmma == 3)
    return qP, kP, vP


def _run(q, k, v, TkS, nmma, dev, bits=None, row_any=None):
    from odise_b200 import ops
    B, Tq, heads, d = q.shape
    qP, kP, vP = _planes(q, k, v, TkS, nmma, dev)
    out, outp = ops.attention_tc(qP, kP, vP, B, heads, d, Tq, k.shape[1], d ** -0.5, nmma, want_f32=True,
                                 want_planes=True, tk_stride=TkS, mask_bits=bits, row_any=row_any)
    torch.cuda.synchronize()
    return out, outp


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("cfg", TC_CASES)
def test_attention_tc(cuda, record, nmma, cfg):
    B, heads, d, Tq, Tk = cfg
    q, k, v = tc_case(cfg)
    out, outp = _run(q, k, v, ceil8(Tk), nmma, cuda)
    ref = reference(q, k, v, d ** -0.5).to(cuda)
    e, ep = _rel(out, ref), _rel(outp.float(), ref)
    record(f"attention_tc {cfg} nmma={nmma}: rel err {e:.3e} (planes {ep:.3e})")
    assert e < _tol(nmma)
    assert ep < _tol(nmma) + 1e-2 * (nmma == 1)


@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("case", MASKED_CASES, ids=lambda c: "-".join(map(str, c)))
def test_attention_tc_masked(cuda, record, nmma, case):
    """1-bit key masks at the engines' own configurations: the text tower's causal mask (3 words per row, an odd count;
    row_any = 0 on the 3 pad query rows), MaskCLIP's 19-word rows from ops.maskclip_bits, Tq > 128 (CTAs with q0 > 0
    read mask rows), Tk = 96 (3 words: the second key block reads word 2 and the guard supplies word 3), rows whose only
    attendable key is in the ragged last block, fully blocked rows and rows with row_any = 0.  Images get different
    masks, so a mask row read from the wrong image shows."""
    from odise_b200 import ops
    kind, B, heads, d, Tq, Tk, TkS = case
    q, k, v, allowed, row_any, bits, logits = masked_case(case)
    if kind == "maskclip":
        bits_d, row_any_d = ops.maskclip_bits(logits.to(cuda), B, Tq, logits.shape[2], logits.shape[3], 336, 14, Tq, 0)
        allowed = unpack_bits(bits_d, Tk).cpu()          # the kernel is checked against the bits it was given
        assert (row_any_d == 1).all()
    else:
        bits_d, row_any_d = bits.to(cuda), row_any.to(cuda)
    assert bits_d.shape[-1] == (Tk + 31) // 32
    out, outp = _run(q, k, v, TkS, nmma, cuda, bits_d, row_any_d)
    ref = reference(q, k, v, d ** -0.5, effective_mask(allowed, row_any)).to(cuda)
    e = _rel(out, ref)
    record(f"attention_tc masked {case} nmma={nmma}: rel err {e:.3e}")
    assert e < _tol(nmma)
    assert _rel(outp.float(), ref) < _tol(nmma) + 1e-2 * (nmma == 1)


# The plain bf16 mode (nmma 1) rounds q and k to 2^-9, so logits of magnitude |s| are off by ~2^-8 |s|: ~0.1 at the
# rising case's +-22, a 10 % error in P that belongs to that mode's precision, not to the online softmax.  It runs the
# peaked and dominant cases, whose large logits come from a few coordinates of moderate size.
@pytest.mark.parametrize("nmma,case", [(n, c) for n in (3, 1) for c in STRESS_CASES if n == 3 or c[0] != "rising"],
                         ids=lambda c: "-".join(map(str, c)) if isinstance(c, tuple) else str(c))
def test_attention_tc_online_softmax(cuda, record, nmma, case):
    """Hostile logits for the online softmax: peaked rows (std ~8), a running max that jumps in every key block (the
    accumulator and the row sum must be rescaled by alpha each time), and one key 30 units above the rest, alone in the
    ragged last block.  d = 160 runs the two-CTA (VPARTS = 2) path."""
    kind, B, heads, d, Tq, Tk = case
    q, k, v = stress_case(case)
    out, outp = _run(q, k, v, ceil8(Tk), nmma, cuda)
    ref = reference(q, k, v, d ** -0.5).to(cuda)
    e = _rel(out, ref)
    record(f"attention_tc stress {case} nmma={nmma}: rel err {e:.3e}")
    assert e < _tol(nmma)
    assert _rel(outp.float(), ref) < _tol(nmma) + 1e-2 * (nmma == 1)


def _fill_junk(t, g, lo=-4.0, hi=4.0):
    """distinct finite values, so that a wrong stride or offset reads a wrong value rather than a zero"""
    t.copy_(torch.rand(t.shape, generator=g) * (hi - lo) + lo)
    return t


@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("layout", ["unet_qk", "clip_qk", "decoder_slot", "maskclip_cache"])
def test_attention_tc_sliced_operands(cuda, record, nmma, layout):
    """Operands as the engines pass them: views into wider buffers whose other elements hold distinct junk.
    unet_qk / clip_qk: q and k are column slices of one [B*T, 2*Cp] projection output (unet.py:196-198, clip.py:53-59);
    decoder_slot: K and V^T are layer slot 1 of 3 of the level's [B*hw8, 3*CP] / [3*CP, B*hw8] planes (head.py:333-368);
    maskclip_cache: K and V^T are images 1..2 of a 3-image cache, K rows offset into a [3*TS, 2*Wd] buffer and V^T columns
    offset into a [Wd, 3*TS] one (clip.py:57-58, :87-92).  The output must be the fp64 attention of exactly the slices."""
    from odise_b200 import lib, ops
    g = torch.Generator().manual_seed(len(layout) * 31 + nmma)
    f16 = nmma == 3
    bits_d = row_any_d = None
    allowed = None
    if layout in ("unet_qk", "clip_qk"):
        B, heads, d, T, Tk = (2, 8, 40, 256, 256) if layout == "unet_qk" else (2, 16, 64, 584, 577)
        HS = ops.head_stride(d)
        Cp = heads * HS
        Tq = TkS = T
        buf = _fill_junk(torch.empty(B, T, 2, heads, HS), g)
        buf[..., d:] = 0.0                                    # head pad columns of q and k are zero
        q = buf[:, :, 0, :, :d].clone()
        k = buf[:, :Tk, 1, :, :d].clone()
        v = torch.randn(B, Tk, heads, d, generator=g)
        vt = _fill_junk(torch.empty(heads, HS, B, TkS), g, 100.0, 1000.0)
        vt[:, :d, :, :Tk] = v.permute(2, 3, 0, 1)
        qk = lib.split(buf.view(B * T, 2 * Cp).to(cuda))
        qP, kP = qk.col_slice(0, Cp), qk.col_slice(Cp, Cp)
        vP = lib.split(vt.view(Cp, B * TkS).to(cuda), f16=f16)
    elif layout == "decoder_slot":
        B, heads, d, Tq, Tk, TkS, nk, slot = 2, 8, 32, 100, 252, 256, 3, 1
        CP = heads * 64
        q = torch.randn(B, Tq, heads, d, generator=g)
        qp = torch.zeros(B * Tq, heads, 64)
        qp[:, :, :d] = q.view(B * Tq, heads, d)
        kbuf = _fill_junk(torch.empty(B, TkS, nk, heads, 64), g)
        kbuf[:, :, slot, :, d:] = 0.0
        k = kbuf[:, :Tk, slot, :, :d].clone()
        vbuf = _fill_junk(torch.empty(nk, heads, 64, B, TkS), g, 100.0, 1000.0)
        v = torch.randn(B, Tk, heads, d, generator=g)
        vbuf[slot, :, :d, :, :Tk] = v.permute(2, 3, 0, 1)
        allowed, row_any = _random_mask(B, Tq, Tk, g)
        bits_d, row_any_d = pack_bits(allowed).to(cuda), row_any.to(cuda)
        allowed = effective_mask(allowed, row_any)
        qP = lib.split(qp.view(B * Tq, CP).to(cuda))
        kP = lib.split(kbuf.view(B * TkS, nk * CP).to(cuda)).col_slice(slot * CP, CP)
        vP = lib.split(vbuf.view(nk * CP, B * TkS).to(cuda), f16=f16).row_slice(slot * CP, CP)
    else:
        B, heads, d, Tq, Tk, TkS, first = 2, 16, 64, 100, 577, 584, 1
        Wd = heads * d
        q = torch.randn(B, Tq, heads, d, generator=g)
        cache = _fill_junk(torch.empty(3, TkS, 2, heads, d), g)          # [3 images x TS rows, (q | k) x Wd]
        k = cache[first:first + B, :Tk, 1].clone()
        vbuf = _fill_junk(torch.empty(heads, d, 3, TkS), g, 100.0, 1000.0)
        v = torch.randn(B, Tk, heads, d, generator=g)
        vbuf[:, :, first:first + B, :Tk] = v.permute(2, 3, 0, 1)
        logits = maskclip_logits(B, Tq, 5).to(cuda)
        bits_d, row_any_d = ops.maskclip_bits(logits, B, Tq, 16, 16, 336, 14, Tq, 0)
        allowed = unpack_bits(bits_d, Tk).cpu()
        qP = lib.split(q.reshape(B * Tq, Wd).to(cuda))
        kP = lib.split(cache.view(3 * TkS, 2 * Wd).to(cuda)).col_slice(Wd, Wd).row_slice(first * TkS, B * TkS)
        vP = lib.split(vbuf.view(Wd, 3 * TkS).to(cuda), f16=f16).col_slice(first * TkS, B * TkS)
    out, _ = ops.attention_tc(qP, kP, vP, B, heads, d, Tq, Tk, d ** -0.5, nmma, want_f32=True, want_planes=False,
                              tk_stride=TkS, mask_bits=bits_d, row_any=row_any_d)
    torch.cuda.synchronize()
    ref = reference(q, k, v, d ** -0.5, allowed).to(cuda)
    e = _rel(out, ref)
    record(f"attention_tc sliced {layout} nmma={nmma}: rel err {e:.3e}")
    assert e < _tol(nmma)


def test_attention_tc_deterministic(cuda):
    """No atomics: the same inputs give the same bits, in the fp32 output and in the planes."""
    q, k, v, allowed, row_any, bits, _ = masked_case(("random", 2, 4, 64, 130, 577, 584))
    for kw in ({}, dict(bits=bits.to(cuda), row_any=row_any.to(cuda))):
        for nmma in (3, 1):
            o1, p1 = _run(q, k, v, 584, nmma, cuda, **kw)
            o2, p2 = _run(q, k, v, 584, nmma, cuda, **kw)
            assert torch.equal(o1, o2)
            assert torch.equal(p1.hi, p2.hi)
            assert (p1.lo is None) == (nmma == 1) and (p1.lo is None or torch.equal(p1.lo, p2.lo))


def test_softmax_split(cuda):
    from odise_b200 import ops
    x = torch.randn(300, 77, device=cuda) * 3
    p = ops.softmax_split(x, 300, 77, 80, 0.5)
    ref = (x.double() * 0.5).softmax(-1)
    got = p.float()
    assert _rel(got[:, :77], ref) < 2e-5 and got[:, 77:].abs().max() == 0


@pytest.mark.parametrize("cfg", [
    # (rows, cols, cols_pad, extra x columns, x offset in floats, score std); the kernel odise_softmax_split_f32 picks
    (64, 4096, 4096, 0, 0, 3.0),       # shared-memory kernel: the VAE mid-block's 4096-wide rows
    (301, 4096, 4096, 0, 0, 10.0),     # shared memory, rows not a multiple of its 4 rows per block, peaked scores
    (40, 1000, 1024, 0, 0, 3.0),       # shared memory, 24 pad columns
    (50, 1000, 1024, 20, 0, 3.0),      # shared memory, ldx = 1020 > cols
    (37, 510, 512, 0, 0, 3.0),         # cols < 512: warp-per-row kernel
    (9, 13000, 13000, 0, 0, 3.0),      # 4 rows of 13000 floats exceed 200 KB of shared memory: warp kernel
    (50, 1000, 1024, 20, 1, 3.0),      # x one float off 16-byte alignment: warp kernel
    (33, 3000, 3000, 0, 0, 10.0),      # shared memory, std 10
])
def test_softmax_split_kernels(cuda, record, cfg):
    from odise_b200 import ops
    rows, cols, cols_pad, extra, off, std = cfg
    g = torch.Generator().manual_seed(rows + cols + extra + off)
    ldx = cols + extra
    buf = (torch.randn(rows * ldx + off, generator=g) * std).to(cuda)
    x = buf[off:].view(rows, ldx)
    p = ops.softmax_split(x, rows, cols, cols_pad, 0.7)
    torch.cuda.synchronize()
    ref = (x[:, :cols].double() * 0.7).softmax(-1)
    got = p.float()
    e = _rel(got[:, :cols], ref)
    record(f"softmax_split {cfg}: rel err {e:.3e}")
    assert e < 2e-5
    pad = torch.cat([p.hi.view(rows, p.ld)[:, cols:], p.lo.view(rows, p.ld)[:, cols:]])
    assert (pad.float() == 0).all() and not torch.signbit(pad.float()).any()


@pytest.mark.parametrize("nmma", [3, 1])
@pytest.mark.parametrize("cfg", [(2, 100, 64, 64, 32, 32, None), (1, 100, 256, 256, 64, 64, None), (2, 37, 32, 32, 8, 8, None),
                                 # the decoder at a portrait 576 x 448 input: masks at H/4 x W/4 = 144 x 112 resized to its
                                 # H/32, H/16 and H/8 levels; the s5 level's 252 keys per image sit at a stride of 256
                                 (2, 100, 144, 112, 18, 14, 256), (2, 100, 144, 112, 36, 28, None),
                                 (1, 100, 144, 112, 72, 56, None),
                                 # landscape, 252 keys per image at a stride of 392 (140 pad rows per image)
                                 (2, 37, 112, 144, 14, 18, 392)])
def test_masked_attention_tc_d32(cuda, nmma, cfg):
    """Mask2Former masked cross-attention (odise.py:683-692, 760-774) on the wgmma kernel: head dim 32, mask bits from
    odise_attn_mask_bits_f32 (masks Hm x Wm resized to the key level Hl x Wl), fully-masked rows attend everywhere.
    TkS = rows per image in the key / value planes (None: Tk); its pad rows hold large finite junk that must be masked."""
    import torch.nn.functional as F
    from odise_b200 import lib, ops
    B, Tq, Hm, Wm, Hl, Wl, TkS = cfg
    Tk = Hl * Wl
    TkS = TkS or Tk
    heads, d, HS = 8, 32, 64
    g = torch.Generator().manual_seed(Tk + Tq)
    q = torch.randn(B, Tq, heads, d, generator=g).to(cuda)
    k = torch.randn(B, Tk, heads, d, generator=g).to(cuda)
    v = torch.randn(B, Tk, heads, d, generator=g).to(cuda)
    ml = (torch.randn(B, Tq, Hm, Wm, generator=g) * 3 - 2.0).to(cuda)
    ml[0, 3] = -5.0                      # fully masked row -> must attend everywhere
    ml[0, 5, : Hm // 2] = -9.0           # first key blocks fully masked for this row (exercises the -inf guards)
    bits, row_any = ops.attn_mask_bits(ml, B, Tq, Hm, Wm, Hl, Wl)
    qp = torch.zeros(B * Tq, heads, HS, device=cuda)
    qp[:, :, :d] = q.view(B * Tq, heads, d)
    kp = torch.zeros(B, TkS, heads, HS, device=cuda)
    kp[:, :Tk, :, :d] = k
    kp[:, Tk:] = 7.0                     # pad keys must be masked, not merely zero
    vt = torch.zeros(heads, HS, B, TkS, device=cuda)
    vt[:, :d, :, :Tk] = v.permute(2, 3, 0, 1)
    vt[:, :, :, Tk:] = 1e3               # finite: exp(-inf) = 0 must zero them, 0 * 1e3 stays 0
    scale = d ** -0.5
    out, _ = ops.attention_tc(lib.split(qp.view(B * Tq, -1)), lib.split(kp.view(B * TkS, -1)),
                              lib.split(vt.view(heads * HS, B * TkS), f16=nmma == 3), B, heads, d, Tq, Tk, scale, nmma,
                              want_f32=True, want_planes=False, tk_stride=TkS, mask_bits=bits, row_any=row_any)
    torch.cuda.synchronize()
    am = F.interpolate(ml, size=(Hl, Wl), mode="bilinear", align_corners=False).sigmoid().flatten(2) < 0.5
    am[torch.where(am.sum(-1) == am.shape[-1])] = False
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), k.double()) * scale
    s = s.masked_fill(am[:, None], float("-inf"))
    ref = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v.double()).reshape(B * Tq, heads * d)
    assert _rel(out, ref) < (TOL3 if nmma == 3 else 3e-2)          # fp64 masked attention: P rounding model (top of file)
