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


def test_every_declared_symbol_is_exported_and_bound(built):
    from odise_b200 import lib
    dll = ctypes.CDLL(built)
    names = _declared()
    assert len(names) >= 30
    for n in names:
        assert hasattr(dll, n), f"{n} declared in the header but not exported"
    bound = set(lib._SIGS) | {"odise_version", "odise_launch_count", "odise_groupnorm_ws_floats", "odise_mha_d32_ws_floats", "odise_panoptic_ws_bytes",
             "odise_instance_ws_bytes", "odise_postprocess_fused_ws_bytes"}
    assert set(names) <= bound, set(names) - bound
    assert lib.load().odise_version() == 100


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
    hdr = open(os.path.join(ROOT, "include", "odise_b200.h")).read()
    m = re.search(r"typedef struct \{([^}]*)\} odise_postprocess_geom;", hdr)
    fields = [f.strip(" ;") for f in m.group(1).replace("int", "").split(",")]
    assert fields == [n for n, _ in lib.PostprocessGeom._fields_] and ctypes.sizeof(lib.PostprocessGeom) == 16
    # the GEMM descriptor mirrors the header field by field
    body = re.search(r"typedef struct odise_gemm_desc \{(.*?)\} odise_gemm_desc;", hdr, re.S)
    names = []
    for stmt in re.sub(r"/\*.*?\*/", "", body.group(1), flags=re.S).split(";"):
        names += [re.findall(r"\w+", d)[-1] for d in stmt.split(",") if re.findall(r"\w+", d)]
    assert names == [n for n, _ in lib.GemmDesc._fields_]
