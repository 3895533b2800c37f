"""odise_b200.pixel_decoder on the CPU: the drop-in classes against Mask2Former's own (reached through oracle.refshim,
pinned in tests/golden/ref_pinned_pixel_decoder.pt where the reference tree is absent), the host-built geometry, the
FPN custom ops' schemas, fakes and errors, and the C ABI's argument checks."""
import ctypes
import inspect

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from odise_b200 import lib
from odise_b200 import pixel_decoder as pd
from oracle import refshim

FIX = "ref_pinned_pixel_decoder.pt"
CLASSES = ("MSDeformAttnPixelDecoder", "MSDeformAttnTransformerEncoderOnly", "MSDeformAttnTransformerEncoder",
           "MSDeformAttnTransformerEncoderLayer")
ODISE_SHAPES = [(32, 32), (64, 64), (128, 128)]     # s5, s4, s3 of a 1024^2 crop
ODD_SHAPES = [(5, 7), (10, 14), (19, 27)]


class Shape:
    def __init__(self, channels, stride):
        self.channels, self.stride = channels, stride


def _kw(shape_cls=Shape):
    return dict(input_shape={f"s{i}": shape_cls(channels=512, stride=2 ** i) for i in (2, 3, 4, 5)},
                transformer_dropout=0.0, transformer_nheads=8, transformer_dim_feedforward=1024,
                transformer_enc_layers=6, conv_dim=256, mask_dim=256, norm="GN",
                transformer_in_features=["s3", "s4", "s5"], common_stride=4)


def _ref_msd():
    refshim.modules()
    import importlib
    return importlib.import_module("mask2former.modeling.pixel_decoder.msdeformattn")


def _ref_build():
    R = refshim.modules()
    torch.manual_seed(0)
    return R.MSDeformAttnPixelDecoder(**_kw(R.ShapeSpec))


def _build():
    torch.manual_seed(0)
    return pd.MSDeformAttnPixelDecoder(**_kw())


def _signature(cls):
    """constructor keyword -> repr of its default ("<required>" for none)"""
    return {n: "<required>" if p.default is inspect.Parameter.empty else repr(p.default)
            for n, p in inspect.signature(cls.__init__).parameters.items() if n != "self"}


def _ref_surface():
    msd = _ref_msd()
    sd = _ref_build().state_dict()
    return dict(keys=list(sd), shapes=[list(v.shape) for v in sd.values()],
                params=refshim.sample(torch.cat([v.reshape(-1).float() for v in sd.values()]), k=8192),
                kwargs={c: _signature(getattr(msd, c)) for c in CLASSES})


def test_surface_matches_reference():
    """state-dict keys and shapes, parameters after torch.manual_seed (bit-equal), constructor keywords and their
    defaults"""
    ref = refshim.pinned("surface", _ref_surface, FIX)
    sd = _build().state_dict()
    assert list(sd) == ref["keys"]
    assert [list(v.shape) for v in sd.values()] == ref["shapes"]
    got, want = refshim.at_sample(torch.cat([v.reshape(-1).float() for v in sd.values()]), ref["params"])
    assert torch.equal(got, want)
    for c in CLASSES:
        assert _signature(getattr(pd, c)) == ref["kwargs"][c], c


def test_load_state_dict_both_ways():
    ref = refshim.pinned("surface", _ref_surface, FIX)
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(s, generator=g) for k, s in zip(ref["keys"], ref["shapes"])}
    m = _build()
    m.load_state_dict(sd)                 # strict: the reference's keys and shapes load into this module
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    if refshim.available():
        r = _ref_build()
        r.load_state_dict(m.state_dict())     # and this module's state dict loads into the reference's
        assert all(torch.equal(v, sd[k]) for k, v in r.state_dict().items())
    assert not any("geometry" in k for k in m.state_dict())


def _ref_geometry():
    msd = _ref_msd()
    res = {}
    for name, shapes in (("odise", ODISE_SHAPES), ("odd", ODD_SHAPES)):
        ss = torch.as_tensor(shapes, dtype=torch.long)
        lsi = torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1]))
        vr = torch.ones(2, len(shapes), 2)
        rp = msd.MSDeformAttnTransformerEncoder.get_reference_points(ss, vr, device="cpu")
        res[name] = dict(spatial_shapes=ss, level_start_index=lsi, reference_points=refshim.sample(rp, k=8192))
    return res


@pytest.mark.parametrize("name", ["odise", "odd"])
def test_host_geometry_matches_reference(name):
    """reference points from the levels' ints (the reference's linspace / division arithmetic) and the device-built
    spatial_shapes / level_start_index are bit-equal to the reference encoder's, at the ODISE level sizes and at a
    non-square set"""
    ref = refshim.pinned("geometry", _ref_geometry, FIX)[name]
    shapes = ODISE_SHAPES if name == "odise" else ODD_SHAPES
    rp = pd.MSDeformAttnTransformerEncoder.get_reference_points(shapes, torch.ones(2, len(shapes), 2), device="cpu")
    got, want = refshim.at_sample(rp, ref["reference_points"])
    assert torch.equal(got, want)
    enc = pd.MSDeformAttnTransformerEncoderOnly(d_model=64, nhead=2, num_encoder_layers=1, dim_feedforward=32,
                                                num_feature_levels=3)
    ss, lsi = enc.level_geometry(shapes, torch.device("cpu"))
    assert torch.equal(ss, ref["spatial_shapes"]) and torch.equal(lsi, ref["level_start_index"])
    assert enc.level_geometry(shapes, torch.device("cpu"))[0] is ss     # cached per (shapes, device)


def test_op_schemas():
    ops = torch.ops.odise_b200
    assert str(ops.fpn_upsample_add.default._schema) == \
        "odise_b200::fpn_upsample_add(Tensor z, Tensor cur, int h, int w) -> Tensor"
    assert str(ops.fpn_upsample_add_backward.default._schema) == \
        "odise_b200::fpn_upsample_add_backward(Tensor grad_y, int h, int w) -> Tensor"


def _message(fn, *a):
    with pytest.raises(lib.OdiseError) as e:
        fn(*a)
    return str(e.value)


def test_fakes_and_errors():
    ops = torch.ops.odise_b200
    with FakeTensorMode():
        mem = torch.empty(2, 40 * 30 + 99, 256, device="cuda")
        z = mem[:, 99:]                                     # a token slice: batch stride S*C, read in place
        cur = torch.empty(2, 256, 23, 17, device="cuda")
        y = ops.fpn_upsample_add(z, cur, 40, 30)
        assert y.shape == cur.shape and y.dtype == torch.float32 and y.stride() == cur.stride()
        gz = ops.fpn_upsample_add_backward(cur, 40, 30)
        assert gz.shape == (2, 1200, 256) and gz.is_contiguous()
        bad = [(z.double(), cur.double(), 40, 30),                                  # float64
               (z, cur.half(), 40, 30),                                             # mixed dtypes
               (z, cur, 30, 40 + 1),                                                # h*w disagrees with z
               (z.transpose(1, 2).contiguous().transpose(1, 2), cur, 40, 30),       # channel-major rows
               (z, cur.transpose(2, 3).contiguous().transpose(2, 3), 40, 30),       # non-contiguous cur
               (z[:, :, :200], cur[:, :200].contiguous(), 40, 30),                  # C = 200, not a multiple of 32
               (z[:1], cur, 40, 30)]                                                # batch disagrees
        for a in bad:
            msg = _message(ops.fpn_upsample_add, *a)
            assert msg == _message(lib.fpn_upsample_add, a[0], a[1], a[2:]), a
        for a in ((cur.transpose(2, 3), 40, 30), (cur[:, :200].contiguous(), 40, 30), (cur.double(), 40, 30),
                  (cur, 0, 30)):
            assert _message(ops.fpn_upsample_add_backward, *a) == _message(lib.fpn_upsample_add_backward, a[0], a[1:])
    # CPU tensors are refused before any launch
    _message(lib.fpn_upsample_add, torch.zeros(1, 4, 32), torch.zeros(1, 32, 4, 4), (2, 2))
    _message(lib.fpn_upsample_add_backward, torch.zeros(1, 32, 4, 4), (2, 2))


def test_cabi_exports_and_argument_checks():
    L = lib.load()
    ERR_ARG, ERR_UNSUP = 10001, 10006
    p = ctypes.c_void_p(16)
    f, b = L.odise_fpn_upsample_add_f32, L.odise_fpn_upsample_add_backward_f32
    assert f(None, 4096 * 256, p, p, 2, 256, 64, 64, 128, 128, None) == ERR_ARG
    assert f(p, 4096 * 256, p, None, 2, 256, 64, 64, 128, 128, None) == ERR_ARG
    assert f(p, 4096 * 256 - 1, p, p, 2, 256, 64, 64, 128, 128, None) == ERR_ARG         # batch stride below h*w*C
    assert f(p, 4096 * 200, p, p, 2, 200, 64, 64, 128, 128, None) == ERR_UNSUP          # C % 32
    assert f(p, 4096 * 256, p, p, 0, 256, 64, 64, 128, 128, None) == ERR_ARG
    assert f(p, 4096 * 256, p, p, 2, 256, 64, 64, 70000, 128, None) == ERR_UNSUP        # grid rows
    assert f(p, 1 << 31, p, p, 1, 256, 4096, 2048, 128, 128, None) == ERR_UNSUP         # h*w*C >= 2^31
    assert b(None, p, 4096 * 256, 2, 256, 64, 64, 128, 128, None) == ERR_ARG
    assert b(p, p, 100, 2, 256, 64, 64, 128, 128, None) == ERR_ARG
    assert b(p, p, 4096 * 96, 2, 96, 64, 64, 0, 128, None) == ERR_ARG
    assert b(p, p, 4096 * 48, 2, 48, 64, 64, 128, 128, None) == ERR_UNSUP
