"""Host-side logic of the operand-plane formats (odise_b200/lib.py::Planes, include/odise_b200.h ODISE_PLANES_*), no GPU:
geometry of F16Q8 planes (whole 64-wide k-blocks, zero pad), slicing rules, the byte layout Planes.float() decodes, and the
header / binding constants."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_constants_match_header():
    from odise_b200 import lib
    h = open(os.path.join(ROOT, "include", "odise_b200.h")).read()
    vals = {k: int(v) for k, v in re.findall(r"#define (ODISE_PLANES_[A-Z0-9]+) (\d+)", h)}
    assert vals == {"ODISE_PLANES_BF16": lib.PLANES_BF16, "ODISE_PLANES_F16": lib.PLANES_F16, "ODISE_PLANES_F16Q8": lib.PLANES_F16Q8}
    src = open(os.path.join(ROOT, "odise_b200", "csrc", "ptx.cuh")).read()
    assert int(re.search(r"constexpr int kQ8Shift = (\d+);", src).group(1)) == lib.Q8_SHIFT


def test_q8_plane_geometry_and_slices():
    from odise_b200.lib import Planes, Q8
    p = Planes.empty(10, 200, "cpu", lo=Q8)
    assert p.fmt == "q8" and p.ld == 256 and p.code == 2
    assert p.hi.numel() == 10 * 256 and p.lo.numel() == 10 * 256 and float(p.hi.float().abs().max()) == 0
    q = Planes.empty(10, 320, "cpu", lo=Q8)
    assert q.ld == 320                                    # whole k-blocks already
    s = q.col_slice(64, 128)
    assert s.fmt == "q8" and s.ld == 320 and s.hi.data_ptr() == q.hi.data_ptr() + 64 * 2
    with pytest.raises(AssertionError):
        q.col_slice(8, 64)                                # F16Q8 slices must start on a k-block
    r = q.row_slice(3, 4)
    assert r.rows == 4 and r.lo.data_ptr() == q.lo.data_ptr() + 3 * 320 * 2
    b = Planes.empty(10, 200, "cpu", lo=True)
    assert b.fmt == "bf16" and b.ld == 200 and b.col_slice(8, 64).fmt == "bf16"
    f = Planes.empty(10, 200, "cpu", lo=Q8, f16=True)     # fp16 pair wins over the engine-wide Q8 switch (attention V^T)
    assert f.fmt == "f16" and f.ld == 200
    assert Planes.empty(4, 64, "cpu", lo=False).lo is None


def test_q8_decode_matches_the_documented_byte_layout():
    """second plane = per 64-wide k-block: 64 bytes e5m2(x * 2^-6) then 64 bytes e5m2((x - fp16(x)) * 2^6)"""
    from odise_b200.lib import Planes, Q8, Q8_SHIFT
    g = torch.Generator().manual_seed(3)
    rows, cols = 5, 130
    x = (torch.randn(rows, cols, generator=g).abs() + 0.1) * torch.logspace(-1, 2, cols)   # inside the normal ranges
    p = Planes.empty(rows, cols, "cpu", lo=Q8)
    hi = x.half()
    p.hi.view(torch.float16).view(rows, p.ld)[:, :cols] = hi
    qb = p.lo.view(torch.uint8).view(rows, p.ld // 64, 2, 64)
    pad = torch.zeros(rows, p.ld)
    pad[:, :cols] = x
    padlo = torch.zeros(rows, p.ld)
    padlo[:, :cols] = x - hi.float()
    qb[:, :, 0, :] = (pad * 2.0 ** -Q8_SHIFT).to(torch.float8_e5m2).view(torch.uint8).view(rows, p.ld // 64, 64)
    qb[:, :, 1, :] = (padlo * 2.0 ** Q8_SHIFT).to(torch.float8_e5m2).view(torch.uint8).view(rows, p.ld // 64, 64)
    got = p.float()
    assert got.shape == (rows, cols)
    rel = ((got - x).abs() / x.abs().clamp_min(1e-30)).max().item()
    assert rel < 2.0 ** -13                                # fp16 hi (2^-11) refined by a 3-significant-bit correction


def test_producers_refuse_fp16_pairs_and_gemm_checks_formats():
    from odise_b200 import lib
    with pytest.raises(lib.OdiseError):
        lib.pargs(lib.Planes.empty(4, 64, "cpu", lo=True, f16=True))
    a, b = lib.Planes.empty(128, 64, "cpu", lo=lib.Q8), lib.Planes.empty(128, 64, "cpu", lo=True)
    with pytest.raises(lib.OdiseError):
        lib.gemm(a, b, out=torch.empty(128, 128))


def test_gemm_tile_policy_cost_model():
    """pick_tile() (csrc/gemm_tc.cu), the cost model behind the GEMM's tile choice under stream capture: the widest tile
    that keeps the waves full, 64-wide tiles where fewer output tiles than SMs would be left otherwise, at most 128 columns
    in the F16Q8 mode (two register accumulators), never CTA pairs."""
    import __graft_entry__ as ge
    ge.build()
    from odise_b200 import lib
    assert lib.gemm_tile_policy(65536, 512, 4608, conv=True, nmma=3) == (256, False)       # KL-VAE 64x64 conv
    assert lib.gemm_tile_policy(65536, 512, 4608, conv=True, nmma=2) == (128, False)
    assert lib.gemm_tile_policy(1048576, 256, 2304, conv=True, nmma=2) == (128, False)     # KL-VAE 256x256 level
    assert lib.gemm_tile_policy(65536, 320, 2880, conv=True, nmma=2) == (128, False)       # UNet 64x64 level: N = 320
    assert lib.gemm_tile_policy(4194304, 128, 1152, conv=True, nmma=2) == (128, False)     # N = 128
    assert lib.gemm_tile_policy(9344, 1024, 4096, nmma=2) == (128, False)                   # CLIP MLP projection
    assert lib.gemm_tile_policy(65536, 640, 320, nmma=3) == (160, False)                    # K < 1024: epilogue bound
    assert lib.gemm_tile_policy(400, 256, 256, nmma=3) == (64, False)                       # decoder linears: 4 M tiles
    assert lib.gemm_tile_policy(100, 256, 256, nmma=3) == (64, False)
    assert lib.gemm_tile_policy(65536, 512, 4608, nmma=1) == (256, False)
    for nmma in (1, 2, 3):
        for bn, pair in (lib.gemm_tile_policy(m, n, k, nmma=nmma) for m in (100, 4096, 65536) for n in (64, 320, 1342)
                         for k in (64, 640, 5760)):
            assert bn in ((64, 128) if nmma == 2 else (64, 128, 160, 256)) and pair is False
