"""Every output-tile width of odise_gemm_bf16 gives the same bits.

The GEMM runs 64-, 128-, 160- or 256-wide output tiles (F16Q8 operands: 64 or 128) and a one-time per-shape autotune
picks the width by timing trial launches, so two processes may pick different widths for one shape.  That is harmless
only while every width computes the same arithmetic in the same k order and edge tiles (epilogue_quad, also the split-K
reduce) round the epilogue exactly like interior tiles.  Each case below runs the autotuned call first (which fills the
per-shape cache), then every width the operand mode can launch, forced through desc.force_bn, and checks

* the width actually launched (the `bn` column of the ODISE_PROFILE_CSV row written by odise_profile_end);
* bit identity with the autotuned call: fp32 outputs, (hi, lo) output planes and GroupNorm records, byte for byte,
  including the sentinel-filled columns around a column-slice output, which must stay untouched;
* accuracy against fp64 torch on the unrounded inputs (bf16x3 2e-5, bf16 2e-2, F16Q8 2e-4 and, against the exact F16Q8
  emulation, 2e-5), judged separately on the last partial row tile and on each width's N tail columns, each against its
  own max |ref|, so that a wrong edge tile cannot hide behind the scale of the interior.

Shapes are chosen so that the widths split N differently (320 = 256 + 64 = 2 x 160, 77 and 40 narrower than a tile,
1342 ragged) and every epilogue flag reaches both the interior path and epilogue_quad."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

PAD = 64                      # outputs are column slices [PAD, PAD + N) of wider sentinel-filled buffers
SENT_F32 = 7.0
SENT_PLANE = 0x3C01           # 1.0009765625 in fp16, 1.0078125 in bf16
TOL = {3: 2e-5, 1: 2e-2, 2: 2e-4}
TOL_GEGLU = {3: 3e-5, 1: 2e-2, 2: 3e-4}
TOL_EMUL = 2e-5               # F16Q8 against its exact emulation (fp32 accumulation level)
TOL_PLANES = {"bf16": 1e-4, "bf16_hi": 6e-3, "f16": 1e-4, "q8": 2e-4}   # one rounding of the output into the planes
MODES = {"bf16x3": 3, "bf16": 1, "q8": 2}


def _rup(x, m):
    return (x + m - 1) // m * m


def _launched_bn(csv):
    """output-tile width of the last GEMM launch recorded in the ODISE_PROFILE_CSV file"""
    with open(csv) as f:
        lines = [ln for ln in f.read().split("\n") if ln]
    head, last = lines[-2].split(","), lines[-1].split(",")
    assert head[5] == "bn", head
    return int(last[5])


def _q8_terms(x):
    """(hi, q_hi, q_lo) of an fp32 tensor as the F16Q8 planes store them, in fp64"""
    e5m2 = lambda t: t.clamp(-57344.0, 57344.0).to(torch.float8_e5m2).double()
    x = x.float()
    hi = x.clamp(-65504.0, 65504.0).half().float()
    return hi.double(), e5m2(x * 2.0 ** -6), e5m2((x - hi) * 2.0 ** 6)


def _emul(a, b):
    """a [.., M, K] x b [.., N, K]^T with the operands rounded as F16Q8 and the three products accumulated in fp64"""
    ah, aqh, aql = _q8_terms(a)
    bh, bqh, bql = _q8_terms(b)
    t = lambda x: x.transpose(-1, -2)
    return ah @ t(bh) + aqh @ t(bql) + aql @ t(bqh)


def _plane_words(P, rows, c0, n):
    """the stored words of columns [c0, c0 + n) of planes P as integer tensors [rows, n] (q8: fp16 hi, q_hi and q_lo bytes)"""
    out = [P.hi.view(torch.int16).view(rows, P.ld)[:, c0:c0 + n]]
    if P.lo is not None:
        if P.fmt == "q8":
            qb = P.lo.view(torch.uint8).view(rows, P.ld // 64, 2, 64)
            out += [qb[:, :, i, :].reshape(rows, P.ld)[:, c0:c0 + n] for i in (0, 1)]
        else:
            out.append(P.lo.view(torch.int16).view(rows, P.ld)[:, c0:c0 + n])
    return out


def _first_difference(a, b):
    """where two equally shaped integer tensors first differ, and how many elements do (for the failure message)"""
    bad = (a != b).nonzero()
    return f"{bad.shape[0]} of {a.numel()} words differ, first at {tuple(bad[0].tolist())}" if bad.shape[0] else "equal"


def _same_bytes(got, base, what):
    for key in base:
        for i, (x, y) in enumerate(zip(got[key], base[key])):
            assert torch.equal(x, y), f"{what}: {key}[{i}] differs from the autotuned call: {_first_difference(x, y)}"


class Problem:
    """One GEMM / implicit conv with its epilogue and outputs.  run(force_bn) launches it into fresh sentinel-filled outputs
    and returns them; check(outs) holds them against the fp64 reference."""

    def __init__(self, cuda, mode, M=None, N=None, K=None, *, batch=1, shared_b=False, conv=None, conv_mode=0, alpha=1.0,
                 bias=False, bias_m=False, groups=0, residual=False, act=0, geglu=False, gn=False, split_k=1,
                 outputs=("f32", "bf16"), seed=0):
        from odise_b200 import lib
        self.lib, self.cuda, self.nmma = lib, cuda, MODES[mode]
        lo = lib.Q8 if mode == "q8" else True
        g = torch.Generator().manual_seed(seed)
        rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(cuda)
        if conv is not None:
            Bc, H, W, C = conv
            stride, pad = (1, 1) if conv_mode == 0 else ((2, 1) if conv_mode == 1 else (2, 0))
            x = rnd(Bc, C, H, W)
            w = rnd(N, C, 3, 3, scale=1.0 / (3 * C ** 0.5))
            M, K, batch = Bc * (H // stride) * (W // stride), 9 * C, 1
            ap = lib.split(x.permute(0, 2, 3, 1).contiguous().view(Bc * H * W, C), lo=lo)
            bp = lib.split(w.permute(0, 2, 3, 1).contiguous().view(N, K), lo=lo)
            cols = F.unfold(F.pad(x, (0, 1, 0, 1)) if conv_mode == 2 else x, 3, padding=pad, stride=stride)
            A, Bw = cols.transpose(1, 2).reshape(1, M, K), w.reshape(1, N, K)      # k order (c, kh, kw): same products
            self.kw = dict(M=M, N=N, K=K, conv=(C, H, W), conv_mode=conv_mode)
        else:
            A = rnd(batch, M, K)
            Bw = rnd(1 if shared_b else batch, N, K, scale=K ** -0.5)
            ap, bp = lib.split(A.view(batch * M, K), lo=lo), lib.split(Bw.view(-1, K), lo=lo)
            self.kw = dict(M=M, N=N, K=K, batch=batch, a_bs=M * ap.ld if batch > 1 else 0,
                           b_bs=N * bp.ld if batch > 1 and not shared_b else 0)
        # GEGLU: quad-interleaved (a, gate) weight rows and bias, GEMM columns 8 j + (0..3) = a, 8 j + (4..7) = gate
        quads = lambda t: t.reshape(2, N // 8, 4, -1).transpose(0, 1).reshape(N, -1).contiguous()
        if geglu:
            bp = lib.split(quads(Bw.view(N, K)), lo=lo)
        self.M, self.N, self.batch, self.geglu = M, N, batch, geglu
        self.nout = N // 2 if geglu else N
        self.ap, self.bp, self.outputs = ap, bp, outputs
        self.kw.update(nmma=self.nmma, alpha=alpha, act=act, geglu=geglu)
        if split_k > 1:
            self.kw.update(split_k=split_k, workspace=torch.empty(split_k * batch * M * N, device=cuda))

        # fp64 reference of the final values [batch, M, nout]; for F16Q8 also on the emulated operand rounding
        def padded(rows, cols, scale=1.0):   # row stride a multiple of 8 floats: the vector epilogue stays on
            t = torch.zeros(rows, _rup(cols, 8), device=cuda)
            t[:, :cols] = rnd(rows, cols, scale=scale)
            return t[:, :cols]

        vb = rnd(N) if bias else None
        vbm = rnd(M) if bias_m else None
        rb = padded(-(-batch * M // groups), N) if groups else None
        res = padded(batch * M, N) if residual else None
        self.kw.update(bias=quads(vb).view(N) if geglu and bias else vb, bias_m=vbm)
        if groups:
            self.kw.update(rowbias=rb, rows_per_group=groups)
        if residual:
            self.kw.update(residual=res, ld_res=res.stride(0), res_bs=M * res.stride(0))

        def epi(prod):
            v = alpha * prod
            if bias:
                v = v + vb.double()
            if bias_m:
                v = v + vbm.double()[:, None]
            if geglu:
                return v[..., :N // 2] * F.gelu(v[..., N // 2:])
            if groups:
                v = v + rb.double().repeat_interleave(groups, 0)[:batch * M].view(batch, M, N)
            v = [lambda t: t, F.relu, F.silu, F.gelu, lambda t: t * torch.sigmoid(1.702 * t)][act](v)
            if residual:
                v = v + res.double().view(batch, M, N)
            return v

        self.ref = epi(A.double() @ Bw.double().transpose(1, 2))
        self.emul = epi(_emul(A, Bw)) if self.nmma == 2 else None
        self.gn = gn
        self.tol = (TOL_GEGLU if geglu else TOL)[self.nmma]

    def run(self, force_bn):
        lib, cuda, rows, n = self.lib, self.cuda, self.batch * self.M, self.nout
        kw = dict(self.kw, force_bn=force_bn)
        outs = {}
        if "f32" in self.outputs:
            ld = _rup(n + 2 * PAD, 8)
            buf = torch.full((rows, ld), SENT_F32, device=cuda)
            kw.update(out=buf[:, PAD:], ld_out=ld, out_bs=self.M * ld)
            outs["f32"] = buf
        fmt = next((o for o in self.outputs if o != "f32"), None)
        if fmt is not None:
            lo = {"bf16": True, "bf16_hi": False, "f16": True, "q8": lib.Q8}[fmt]
            P = lib.Planes.empty(rows, n + 2 * PAD, cuda, lo=lo, f16=fmt == "f16")
            for t in (P.hi, P.lo):
                if t is not None:
                    t.view(torch.int16).fill_(SENT_PLANE)
            kw.update(out_planes=P.col_slice(PAD, n), outp_bs=self.M * P.ld)
            outs["planes"], outs["fmt"] = P, fmt
        if self.gn:
            st = lib.GnStats(rows, n, cuda)
            st.t.fill_(float("nan"))
            kw.update(gn=st)
            outs["gn"] = st
        lib.gemm(self.ap, self.bp, **kw)
        torch.cuda.synchronize()
        if self.gn:
            assert not st.missing
        return outs

    @staticmethod
    def words(outs):
        """every byte the call may have written, as integer tensors"""
        w = {}
        if "f32" in outs:
            w["f32"] = [outs["f32"].view(torch.int32)]
        if "planes" in outs:
            P = outs["planes"]
            w["planes"] = [t.view(torch.int16) for t in (P.hi, P.lo) if t is not None]
        if "gn" in outs:
            w["gn"] = [outs["gn"].t.view(torch.int32)]
        return w

    def regions(self, widths):
        """(rows, cols) of the whole output, of the last partial 128-row tile and of each width's N tail columns"""
        M, n = self.M, self.nout
        rows = [slice(0, M)] + ([slice((M - 1) // 128 * 128, M)] if M % 128 else [])
        f = 2 if self.geglu else 1   # GEGLU: a tile of w GEMM columns writes w / 2 output columns
        cols = [slice(0, n)] + [slice((self.N - 1) // w * w // f, n) for w in sorted(set(widths)) if self.N % w]
        return [(r, c) for r in rows for c in cols]

    def check(self, outs, widths, what):
        rows, n, B, M = self.batch * self.M, self.nout, self.batch, self.M
        got = {}
        if "f32" in outs:
            buf = outs["f32"]
            assert (buf[:, :PAD] == SENT_F32).all() and (buf[:, PAD + n:] == SENT_F32).all(), f"{what}: fp32 outside the slice"
            got["f32"] = (buf[:, PAD:PAD + n].view(B, M, n), 0.0)
        if "planes" in outs:
            P, fmt = outs["planes"], outs["fmt"]
            for t, q in ((P.hi, False), (P.lo, fmt == "q8")):
                if t is not None:   # (q bytes: the slice's whole 64-column blocks)
                    t2 = t.view(torch.int16).view(rows, P.ld)
                    keep = torch.cat([t2[:, :PAD], t2[:, PAD + (_rup(n, 64) if q else n):]], 1)
                    assert (keep == SENT_PLANE).all(), f"{what}: planes written outside the slice"
            got["planes"] = (P.float()[:, PAD:PAD + n].view(B, M, n), TOL_PLANES[fmt])
            if "f32" in outs:
                # the epilogue writes the planes lib.split() makes of its own fp32 output, word for word (split takes
                # whole quads of columns: the sentinel columns after an N tail come along and are not compared)
                lo = {"bf16": True, "bf16_hi": False, "f16": True, "q8": self.lib.Q8}[fmt]
                ref_p = self.lib.split(outs["f32"][:, PAD:PAD + _rup(n, 4)], lo=lo, f16=fmt == "f16")
                for x, y in zip(_plane_words(P, rows, PAD, n), _plane_words(ref_p, rows, 0, n)):
                    assert torch.equal(x, y), f"{what}: planes != split(fp32 output): {_first_difference(x, y)}"
        regions = self.regions(widths)
        for key, (val, ptol) in got.items():
            refs = [(self.ref, max(self.tol, ptol))] + ([(self.emul, max(TOL_EMUL, ptol))] if self.emul is not None else [])
            for ref, tol in refs:
                for r, c in regions:
                    want = ref[:, r, c]
                    e = ((val[:, r, c].double() - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()
                    assert e < tol, f"{what}: {key} rel err {e:.3e} >= {tol:.0e} in rows {r.start}:{r.stop}, cols {c.start}:{c.stop}"
        if self.gn:
            # records (shift, S1, S2) per (32-row segment, column) of the fp32 output: shift = the segment's first row
            t = outs["gn"].t
            assert not t.isnan().any(), f"{what}: GroupNorm records missing"
            x = outs["f32"][:, PAD:PAD + n].view(rows // 32, 32, n)
            assert torch.equal(t[:, 0], x[:, 0]), f"{what}: GroupNorm shift"
            d = x.double() - x[:, :1].double()
            for i, s in ((1, d.sum(1)), (2, (d * d).sum(1))):
                bound = 1e-5 * (d.abs() ** i).sum(1) + 1e-30
                assert ((t[:, i].double() - s).abs() <= bound).all(), f"{what}: GroupNorm S{i}"


def _check_widths(prob, monkeypatch, tmp_path):
    """autotuned call, then every width of the operand mode: launched width, bit identity, accuracy"""
    from odise_b200 import lib
    csv = tmp_path / "gemm_profile.csv"
    monkeypatch.setenv("ODISE_PROFILE_CSV", str(csv))
    if prob.nmma == 2:
        widths = {64: 64, 128: 128, 160: 128, 256: 128}   # F16Q8 runs 64- and 128-wide tiles only
    else:
        widths = {64: 64, 128: 128, 160: 160, 256: 256}
    base = prob.run(0)                      # autotunes (or finds the shape in the cache) before any forced width
    lib.profile_begin()                     # the same call again, now on the cached width, which it reports
    again = prob.run(0)
    lib.profile_end()
    bn0 = _launched_bn(csv)
    assert bn0 in set(widths.values())
    base_w = Problem.words(base)
    _same_bytes(Problem.words(again), base_w, f"autotuned (bn {bn0}) twice")
    prob.check(base, widths.values(), f"autotuned (bn {bn0})")
    for req, want in widths.items():
        lib.profile_begin()
        outs = prob.run(req)
        lib.profile_end()
        assert _launched_bn(csv) == want, f"force_bn={req} launched bn {_launched_bn(csv)}"
        what = f"bn {want} (autotuned: bn {bn0})"
        prob.check(outs, widths.values(), what)
        _same_bytes(Problem.words(outs), base_w, what)


MODE_IDS = ["bf16x3", "bf16", "q8"]


# ---- plain products, no epilogue flags: any difference between widths here is the main loop itself
@pytest.mark.parametrize("mode", MODE_IDS)
@pytest.mark.parametrize("shape", [
    dict(M=1000, N=320, K=200),                         # ragged M, 320 = 256 + 64 = 2 x 160, partial k-block
    dict(M=512, N=77, K=64),                            # narrower than any tile, one k-block
    dict(M=4096, N=640, K=320),                         # UNet linear
    dict(M=288, N=40, K=64),                            # N <= 64
    dict(M=100, N=1342, K=256, batch=2, shared_b=True),   # batched over shared weights (b_bs = 0)
], ids=["1000x320x200", "512x77x64", "4096x640x320", "288x40x64", "2x100x1342x256"])
def test_widths_plain(cuda, monkeypatch, tmp_path, mode, shape):
    _check_widths(Problem(cuda, mode, seed=shape["M"] + shape["N"], **shape), monkeypatch, tmp_path)


# ---- every epilogue flag at N = 320 (an edge tile at 256, interior at 64 / 160) and N = 77 (edge tiles everywhere but 64)
EPILOGUES = {
    "bias": dict(bias=True),
    "alpha_bias": dict(alpha=0.37, bias=True),
    "bias_bias_m": dict(bias=True, bias_m=True),
    "alpha_bias_m": dict(alpha=0.37, bias_m=True),
    "rowbias": dict(groups=136),
    "residual": dict(residual=True),
    "relu": dict(bias=True, act=1),
    "silu": dict(bias=True, act=2),
    "gelu": dict(bias=True, act=3),
    "quickgelu": dict(bias=True, act=4),
    "geglu": dict(bias=True, geglu=True, outputs=("bf16",)),
    "gn_records": dict(bias=True, groups=272, residual=True, gn=True),
}


@pytest.mark.parametrize("mode", ["bf16x3", "q8"])
@pytest.mark.parametrize("N", [320, 77])
@pytest.mark.parametrize("epi", list(EPILOGUES))
def test_widths_epilogue(cuda, monkeypatch, tmp_path, mode, N, epi):
    kw = dict(EPILOGUES[epi])
    if kw.get("geglu"):
        N = _rup(N, 16)          # (a, gate) quads share a 16-column chunk
    if mode == "q8":            # F16Q8 operands -> F16Q8 output planes
        kw["outputs"] = tuple("q8" if o == "bf16" else o for o in kw.get("outputs", ("f32", "bf16")))
    _check_widths(Problem(cuda, mode, 544, N, 200, seed=N + len(epi), **kw), monkeypatch, tmp_path)


# ---- output kinds, as column slices of wider buffers: fp32 alone, fp32 + planes, planes alone in each format (F16Q8 output
# planes from bf16-pair operands: 160- and 256-wide tiles start in the middle of a 64-column q-byte block)
@pytest.mark.parametrize("N", [320, 77])
@pytest.mark.parametrize("outputs", [("f32",), ("f32", "bf16"), ("bf16",), ("bf16_hi",), ("f16",), ("q8",), ("f32", "q8")],
                         ids=lambda o: "+".join(o))
def test_widths_outputs(cuda, monkeypatch, tmp_path, N, outputs):
    _check_widths(Problem(cuda, "bf16x3", 1000, N, 200, alpha=0.37, bias=True, residual=True, outputs=outputs, seed=N + 3),
                  monkeypatch, tmp_path)


# ---- split-K: partial sums of every width through the reduce kernel's epilogue
@pytest.mark.parametrize("mode", ["bf16x3", "q8"])
@pytest.mark.parametrize("case", [
    dict(M=1024, N=1280, K=11520, split_k=2, bias=True),        # lib.auto_split's UNet 16 x 16 level
    dict(M=400, N=1024, K=4096, split_k=4, alpha=0.37, bias=True, groups=100, bias_m=True, residual=True),
], ids=["1024x1280x11520_split2", "400x1024x4096_split4_epilogue"])
def test_widths_split_k(cuda, monkeypatch, tmp_path, mode, case):
    kw = dict(case, outputs=("f32", "q8") if mode == "q8" else ("f32", "bf16"), seed=case["K"])
    _check_widths(Problem(cuda, mode, **kw), monkeypatch, tmp_path)


# ---- implicit 3x3 convs (input B, H, W, C -> N channels) with bias, per-image row bias, residual and GroupNorm records
@pytest.mark.parametrize("mode", ["bf16x3", "q8"])
@pytest.mark.parametrize("case", [
    dict(conv=(2, 64, 64, 64), N=320),                          # boxed: W = 64 divides the 128-pixel tile
    dict(conv=(2, 24, 160, 64), N=96),                          # segmented fetch: W = 160
    dict(conv=(2, 64, 64, 64), N=320, conv_mode=1),             # stride 2, pad (1, 1)
    dict(conv=(2, 64, 64, 64), N=320, conv_mode=2),             # stride 2, pad (0, 1)
    dict(conv=(16, 8, 8, 1280), N=1280, split_k=2),             # UNet 8 x 8 level, split-K (no records)
], ids=["boxed_w64", "segmented_w160", "stride2_mode1", "stride2_mode2", "8x8_c1280_split2"])
def test_widths_conv(cuda, monkeypatch, tmp_path, mode, case):
    kw = dict(case)
    Bc, H, W, C = kw["conv"]
    s = 1 if kw.get("conv_mode", 0) == 0 else 2
    split = kw.get("split_k", 1) > 1
    kw.update(bias=True, groups=(H // s) * (W // s), residual=True, gn=not split,
              outputs=("f32",), seed=H * W + C)
    _check_widths(Problem(cuda, mode, **kw), monkeypatch, tmp_path)
