"""CPU checks of the drop-in boundary: the shared library loads, exports every symbol include/odise_b200.h declares
and binds it in odise_b200/lib.py; argument validation returns error codes without touching a GPU."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


def _declared():
    h = open(os.path.join(ROOT, "include", "odise_b200.h")).read()
    return sorted(set(re.findall(r"\b(odise_[a-z0-9_]+)\s*\(", h)))


def test_every_declared_symbol_is_exported_and_bound_as_declared(built):
    from odise_b200 import lib
    dll = ctypes.CDLL(built)
    names = _declared()
    assert len(names) >= 30
    for n in names:
        assert hasattr(dll, n), f"{n} declared in the header but not exported"
    assert set(names) <= set(lib._PROTOS), set(names) - set(lib._PROTOS)     # no prototype skipped by the parser
    L = lib.load()
    for n, (restype, argtypes) in lib._PROTOS.items():
        fn = getattr(L, n)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, n
    assert L.odise_version() == 100


def test_argument_validation_without_gpu(built):
    from odise_b200 import lib
    L = lib.load()
    assert L.odise_msda_forward_f32(None, None, None, None, None, None, 1, 1, 1, 4, 1, 1, 1, None) == 10001
    d = lib.GemmDesc()
    assert L.odise_gemm_bf16(ctypes.byref(d), None) == 10001
    assert L.odise_attention_tc(None, None, 0, None, None, 0, None, None, 0, 0, None, None, None, 0, 1, 1, 40, 1, 1, 8,
                                1.0, 3, None, None, None) == 10001
    assert L.odise_split_f32(None, 0, None, None, 0, 1, 4, None) == 10001


def test_no_cpu_fallback():
    from odise_b200 import lib
    with pytest.raises(RuntimeError):
        lib.split(torch.zeros(4, 8))      # CPU tensor -> loud failure, never a silent eager path
    with pytest.raises(RuntimeError):
        lib.msda_forward(torch.zeros(1, 4, 1, 4), torch.tensor([[2, 2]]), torch.tensor([0]),
                         torch.zeros(1, 1, 1, 1, 1, 2), torch.zeros(1, 1, 1, 1, 1), 128)


def test_product_does_not_import_oracle():
    for f in os.listdir(os.path.join(ROOT, "odise_b200")):
        if f.endswith(".py"):
            src = open(os.path.join(ROOT, "odise_b200", f)).read()
            assert "import oracle" not in src and "from oracle" not in src, f


def test_crop_grid_matches_reference_rule():
    """slide_forward crop boxes (feature_extractor.py:197-218): 1024^2 -> 4 crops, 1280^2 -> 9 overlapping, 512^2 -> 1."""
    from odise_b200.backbone import BackboneEngine
    b, s = BackboneEngine.crop_grid(1024, 1024)
    assert s == 512 and b == [(0, 0), (0, 512), (512, 0), (512, 512)]
    b, s = BackboneEngine.crop_grid(1280, 1280)
    assert len(b) == 9 and b[-1] == (768, 768) and b[1] == (0, 512)
    b, s = BackboneEngine.crop_grid(512, 512)
    assert b == [(0, 0)]
    b, s = BackboneEngine.crop_grid(384, 640)
    assert s == 384 and b == [(0, 0), (0, 256)]


def test_t0_coefficients_and_spec_counts():
    from odise_b200 import spec
    from odise_b200.backbone import t0_coefficients
    c0, c1 = t0_coefficients()
    assert abs(c0 - 0.999575) < 1e-6 and abs(c1 - 0.029155) < 1e-6
    n_train = sum(torch.Size(s).numel() for _, s, _ in spec.backbone_params() + spec.head_params())
    # README.md:89 of the reference: 28.1 M trainable parameters (ours excludes null_embed / criterion-free params)
    assert 27.5e6 < n_train < 28.5e6, n_train


def test_auto_split_and_struct_layouts():
    """host heuristics / ctypes mirrors that never touch the device."""
    import ctypes
    import re
    from odise_b200 import lib
    # split K only where output tiles alone cannot fill 132 SMs and the partial-sum traffic pays for itself
    assert lib.auto_split(1024, 1280, 11520) == (160, 2)
    assert lib.auto_split(65536, 320, 2880) == (0, 1) and lib.auto_split(4096, 640, 5760) == (0, 1)
    assert lib.auto_split(256, 1280, 11520)[1] > 1
    assert lib.auto_split(128, 64, 512) == (0, 1)                       # too few k-blocks to split
    assert ctypes.sizeof(lib.GemmDesc) == 312 and ctypes.sizeof(lib.PostprocessGeom) == 16
    assert [n for n, _ in lib.PostprocessGeom._fields_] == ["pad_h", "pad_w", "img_h", "img_w"]
    # the GEMM descriptor mirrors the header field by field
    hdr = open(os.path.join(ROOT, "include", "odise_b200.h")).read()
    body = re.search(r"typedef struct odise_gemm_desc \{(.*?)\} odise_gemm_desc;", hdr, re.S)
    names = []
    for stmt in re.sub(r"/\*.*?\*/", "", body.group(1), flags=re.S).split(";"):
        names += [re.findall(r"\w+", d)[-1] for d in stmt.split(",") if re.findall(r"\w+", d)]
    assert names == [n for n, _ in lib.GemmDesc._fields_]


def test_signatures_bound_from_the_header():
    """a few entry points typed by hand, so that a wrong mapping rule of lib._parse_header fails here"""
    from ctypes import c_double, c_float, c_int, c_longlong, c_void_p, POINTER
    from odise_b200 import lib
    P = lib._PROTOS
    assert P["odise_split_f32"] == (c_int, [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_longlong, c_int,
                                            c_void_p])
    assert P["odise_gemm_bf16"] == (c_int, [POINTER(lib.GemmDesc), c_void_p])
    assert P["odise_postprocess_fused_f32"] == (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 8 + [c_double] +
                                                [c_void_p] * 7 + [c_int] * 9 + [POINTER(lib.PostprocessGeom), c_void_p])
    assert P["odise_mask_cost_f32"] == (c_int, [c_void_p] * 7 + [c_int] * 9 + [c_float] * 3 + [c_void_p])
    assert P["odise_msda_det_workspace_bytes"] == (c_longlong, [c_int] * 4)
    assert P["odise_version"] == (c_int, [])


def test_header_parser_refuses_unmapped_types():
    from ctypes import c_int, c_longlong, c_void_p, POINTER
    from odise_b200 import lib
    structs, protos = lib._parse_header("typedef struct { int a, b; size_t* p; } odise_s;  /* odise_y(size_t n); */\n"
                                        "long long odise_f(const odise_s* s, void* stream);")
    assert [(n, t) for n, t in structs["odise_s"]._fields_] == [("a", c_int), ("b", c_int), ("p", c_void_p)]
    assert protos == {"odise_f": (c_longlong, [POINTER(structs["odise_s"]), c_void_p])}
    with pytest.raises(lib.OdiseError, match="size_t n"):
        lib._parse_header("int odise_x(size_t n);")
    with pytest.raises(lib.OdiseError, match="size_t odise_x"):
        lib._parse_header("size_t odise_x(void);")
    with pytest.raises(lib.OdiseError, match="size_t b, c"):
        lib._parse_header("typedef struct { int a; size_t b, c; } odise_s;")


def test_constants_match_header_defines():
    """the ODISE_ACT_* / ODISE_PLANES_* / ODISE_MASK_MAX_* values lib.py spells out, and ODISE_ERR_UNSUPPORTED"""
    from odise_b200 import lib
    hdr = open(os.path.join(ROOT, "include", "odise_b200.h")).read()
    defines = {n: int(v) for n, v in re.findall(r"#define\s+ODISE_(\w+)\s+(\d+)", hdr)}
    pat = r"(ACT|PLANES|MASK_MAX)_[A-Z0-9_]+"
    assert {n: getattr(lib, n) for n in dir(lib) if re.fullmatch(pat, n)} == \
        {n: v for n, v in defines.items() if re.fullmatch(pat, n)}
    assert lib.ODISE_ERR_UNSUPPORTED == defines["ERR_UNSUPPORTED"]
