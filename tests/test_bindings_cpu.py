"""The engine bindings against the C ABI header, without a GPU: every wrapper of odise_b200.ops, lib.split and lib.gemm,
HeadEngine's weight preparation and forward, and PostProcessor run against a stand-in for the library built from the
header's prototypes (lib._PROTOS).  ctypes does not check the argument count of a cdecl call, so without this a wrapper
that passes an argument too many or too few, or a pointer where the header takes a number, fails only on the GPU."""
import contextlib
import ctypes
import re

import pytest
import torch

from odise_b200 import lib, ops, spec
from odise_b200.head import HeadEngine
from odise_b200.postprocess import PostProcessor

STREAM = 0x5EED5EED0          # the stand-in's current stream
SIZE_QUERIES = ("_ws_floats", "_ws_bytes", "_workspace_bytes")


def _streamed():
    """the entry points whose last parameter is `void* stream`, read from the header's text"""
    with open(lib._HEADER) as f:
        text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    return {name for name, params in re.findall(r"\b(odise_\w+)\s*\(([^()]*)\)\s*;", text)
            if re.search(r"\bstream$", params.strip())}


STREAMED = _streamed()


class FakeLib:
    """Stands in for the loaded library.  Each header prototype becomes a function that checks the argument count,
    converts every argument with its declared ctypes type as a call through the real library would, checks that the
    stream is passed last to the entry points that take one and nowhere else, records the call and returns 0.  The
    size queries return a small positive count."""

    def __init__(self):
        self.calls = []
        for name, (_, argtypes) in lib._PROTOS.items():
            setattr(self, name, self._entry(name, argtypes))

    def _entry(self, name, argtypes):
        def call(*args):
            assert len(args) == len(argtypes), f"{name}: {len(args)} arguments, the header declares {len(argtypes)}"
            for i, (t, a) in enumerate(zip(argtypes, args)):
                try:
                    t.from_param(a)
                except (TypeError, ctypes.ArgumentError) as e:
                    raise AssertionError(f"{name}: argument {i} ({a!r}) is not a {t.__name__}: {e}") from None
                # ctypes takes any int as a pointer and truncates an int too wide for c_int: a pointer and a number
                # swapped pass the conversion above, so pointers must be None or an address, c_int fit 32 bits
                if t is ctypes.c_void_p:
                    assert a is None or a >= 1 << 16, f"{name}: argument {i} ({a!r}) is not an address"
                if t is ctypes.c_int:
                    assert -1 << 31 <= a < 1 << 31, f"{name}: argument {i} ({a!r}) does not fit a C int"
            at = [i for i, a in enumerate(args) if type(a) is int and a == STREAM]
            assert at == ([len(args) - 1] if name in STREAMED else []), f"{name}: the stream is at {at}"
            self.calls.append((name, args))
            return 64 if name.endswith(SIZE_QUERIES) else 0
        return call

    def launched(self):
        return {name for name, _ in self.calls if name in STREAMED}


@pytest.fixture
def fake(monkeypatch):
    f = FakeLib()
    monkeypatch.setattr(lib, "_lib", f)
    monkeypatch.setattr(lib, "_stream", lambda: STREAM)
    monkeypatch.setattr(lib, "nvtx", contextlib.nullcontext)
    monkeypatch.setattr(lib, "_FMT_STATE", [lib.PLANES_BF16])     # the stand-in's operand format, restored afterwards
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda t: True))    # lib._tensor's device check
    return f


def _r(*shape):
    return torch.randn(*shape)


def _i32(*shape):
    return torch.zeros(*shape, dtype=torch.int32)


def _bf16_pair(rows, cols, f16=False):
    return lib.Planes.empty(rows, cols, "cpu", f16=f16)


# wrapper call at a small shape -> the entry points it launches
Q8 = lib.Q8
CASES = {
    "group_norm": (lambda: ops.group_norm(_r(64, 32), 2, 32, _r(32), _r(32), 1e-5),
                   {"odise_groupnorm_stats_ws_f32", "odise_groupnorm_apply_bs_f32"}),
    "group_norm_records_f32_q8": (lambda: ops.group_norm(_r(64, 32), 2, 32, _r(32), _r(32), 1e-5, act=ops.ACT_SILU,
                                                         want_f32=True, lo=Q8, stats=lib.GnStats(64, 32, "cpu")),
                                  {"odise_groupnorm_finalize_seg_f32", "odise_groupnorm_apply_bs_f32"}),
    "group_norm_slice": (lambda: ops.group_norm(_r(64, 48)[:, 8:40], 2, 32, _r(32), _r(32), 1e-5, want_planes=False,
                                                y=_r(64, 96)[:, 32:], ldy=96, y_bs=32 * 96),
                         {"odise_groupnorm_stats_ws_f32", "odise_groupnorm_apply_bs_f32"}),
    "group_norm_res": (lambda: ops.group_norm_res(_r(64, 32), 2, 32, _r(32), _r(32), 1e-5, _r(64, 32), ops.ACT_RELU,
                                                  _r(64, 32), True),
                       {"odise_groupnorm_stats_ws_f32", "odise_groupnorm_apply_res_f32"}),
    "group_norm_res_records": (lambda: ops.group_norm_res(_r(64, 32), 2, 32, _r(32), _r(32), 1e-5, None, ops.ACT_NONE,
                                                          _r(64, 32), False, stats=lib.GnStats(64, 32, "cpu")),
                               {"odise_groupnorm_finalize_seg_f32", "odise_groupnorm_apply_res_f32"}),
    "layer_norm": (lambda: ops.layer_norm(_r(10, 32), _r(32), _r(32)), {"odise_layernorm_f32"}),
    "layer_norm_res_f32_q8": (lambda: ops.layer_norm(_r(10, 32), _r(32), _r(32), res=_r(10, 32), want_f32=True,
                                                     post_add=_r(10, 32), lo=Q8),
                              {"odise_layernorm_f32"}),
    "geglu": (lambda: ops.geglu(_r(10, 64)), {"odise_geglu_f32"}),
    "add_split": (lambda: ops.add_split(_r(20, 32), _r(10, 32), b_rows=10, want_f32=True), {"odise_add_split_f32"}),
    "add_split_q8": (lambda: ops.add_split(_r(20, 32), lo=Q8), {"odise_add_split_f32"}),
    "act_split": (lambda: ops.act_split(_r(10, 32), ops.ACT_GELU), {"odise_act_split_f32"}),
    "act_split_q8": (lambda: ops.act_split(_r(10, 32), ops.ACT_QUICKGELU, lo=Q8), {"odise_act_split_f32"}),
    "upsample2x_split": (lambda: ops.upsample2x_split(_r(24, 16), 2, 3, 4), {"odise_upsample2x_split_f32"}),
    "im2col3x3_split": (lambda: ops.im2col3x3_split(_r(24, 16), 2, 3, 4), {"odise_im2col3x3_split_f32"}),
    "im2col3x3_split_q8": (lambda: ops.im2col3x3_split(_r(24, 16), 2, 3, 4, stride=2, pad_lo=0, lo=Q8),
                           {"odise_im2col3x3_split_f32"}),
    "copy2d": (lambda: ops.copy2d(_r(10, 16), _r(10, 32)[:, 8:24], 0.5, accumulate=True), {"odise_copy2d_f32"}),
    "resize_nhwc": (lambda: ops.resize_nhwc(_r(24, 16), 2, 3, 4, 6, 8, True), {"odise_resize_nhwc_bs_f32"}),
    "resize_nhwc_into": (lambda: ops.resize_nhwc(_r(40, 16)[4:], 2, 3, 4, 6, 8, False, dst=_r(96, 16),
                                                 accumulate=True, src_bs=20 * 16),
                         {"odise_resize_nhwc_bs_f32"}),
    "nchw_to_nhwc": (lambda: ops.nchw_to_nhwc(_r(2, 16, 3, 4)), {"odise_nchw_to_nhwc_f32"}),
    "nhwc_to_nchw": (lambda: ops.nhwc_to_nchw(_r(24, 16), 2, 3, 4), {"odise_nhwc_to_nchw_f32"}),
    "attention_tc": (lambda: ops.attention_tc(_bf16_pair(16, 128), _bf16_pair(16, 128), _bf16_pair(128, 16, f16=True),
                                              1, 2, 32, 16, 16, 0.17, 3),
                     {"odise_attention_tc"}),
    "attention_tc_masked_f32_q8": (lambda: ops.attention_tc(_bf16_pair(16, 128), _bf16_pair(16, 128),
                                                            _bf16_pair(128, 16, f16=True), 1, 2, 32, 16, 12, 0.17, 2,
                                                            want_f32=True, tk_stride=16, mask_bits=_i32(16),
                                                            row_any=_i32(16), lo=Q8),
                                   {"odise_attention_tc"}),
    "softmax_split": (lambda: ops.softmax_split(_r(10, 32), 10, 30, 32, 0.5), {"odise_softmax_split_f32"}),
    "msda_fused": (lambda: ops.msda_fused(_r(16, 64), torch.tensor([[4, 4]]), torch.tensor([0]), _r(1, 16, 1, 2),
                                          _r(16, 16), _r(16, 8), 1, 16, 2, 32, 1, 16, 4),
                   {"odise_msda_fused_f32"}),
    "msda_fused_f32_q8": (lambda: ops.msda_fused(_r(16, 64), torch.tensor([[4, 4]]), torch.tensor([0]),
                                                 _r(1, 16, 1, 2), _r(16, 16), _r(16, 8), 1, 16, 2, 32, 1, 16, 4,
                                                 want_f32=True, lo=Q8),
                          {"odise_msda_fused_f32"}),
    "attn_mask_bits": (lambda: ops.attn_mask_bits(_r(1, 4, 8, 8), 1, 4, 8, 8, 4, 4), {"odise_attn_mask_bits_f32"}),
    "mha_d32": (lambda: ops.mha_d32(_r(4, 64), 64, _r(6, 64), _r(6, 64), 64, 1, 4, 6, 2, 0.17),
                {"odise_mha_d32_ws_f32"}),
    "mha_d32_masked_q8": (lambda: ops.mha_d32(_r(4, 64), 64, _r(6, 64), _r(6, 64), 64, 1, 4, 6, 2, 0.17, _i32(4),
                                              _i32(4), lo=Q8),
                          {"odise_mha_d32_ws_f32"}),
    "mask_binarize": (lambda: ops.mask_binarize(_r(2, 4, 64), 2, 4, 64), {"odise_mask_binarize_f32"}),
    "pool_normalize": (lambda: ops.pool_normalize(_r(8, 32), _r(8), 2, 4, 32), {"odise_pool_normalize_f32"}),
    "l2_normalize_split": (lambda: ops.l2_normalize_split(_r(10, 32)), {"odise_l2_normalize_split_f32"}),
    "l2_normalize_split_q8": (lambda: ops.l2_normalize_split(_r(10, 32), lo=Q8), {"odise_l2_normalize_split_f32"}),
    "class_max": (lambda: ops.class_max(_r(10, 7), torch.tensor([0, 2, 5, 7], dtype=torch.int32), _r(10, 1), 10, 3),
                  {"odise_class_max_f32"}),
    "bcast_fma": (lambda: ops.bcast_fma(_r(16), _r(2, 16), _r(6, 16), 2, 3, 16), {"odise_bcast_fma_f32"}),
    "rowscale": (lambda: ops.rowscale(_r(10, 32)[:, :16], _r(10)), {"odise_rowscale_f32"}),
    "image_crops_u8": (lambda: ops.image_crops(torch.zeros(1, 3, 8, 8, dtype=torch.uint8), _i32(2, 3), 2, 8, 8, 4, 4),
                       {"odise_image_crops_u8_f32"}),
    "image_crops_f32": (lambda: ops.image_crops(_r(1, 3, 8, 8), _i32(2, 3), 2, 8, 8, 4, 4),
                        {"odise_image_crops_f32"}),
    "clip_preprocess": (lambda: ops.clip_preprocess(torch.zeros(1, 3, 8, 8, dtype=torch.uint8), _i32(1, 3), 1, 8, 8,
                                                    8, 8, S=14),
                        {"odise_clip_preprocess"}),
    "clip_preprocess_f32": (lambda: ops.clip_preprocess(_r(1, 3, 8, 8), _i32(1, 3), 1, 8, 8, 8, 8, S=14),
                            {"odise_clip_preprocess"}),
    "crop_resize_bicubic": (lambda: ops.crop_resize_bicubic(_r(1, 3, 8, 8), _i32(1, 3), 1, 8, 8, 8, 8, S=16),
                            {"odise_crop_resize_bicubic"}),
    "maskclip_preprocess": (lambda: ops.maskclip_preprocess(torch.zeros(1, 3, 8, 8, dtype=torch.uint8), 1, 8, 8, S=14),
                            {"odise_maskclip_preprocess"}),
    "patchify_split": (lambda: ops.patchify_split(_r(2 * 28 * 28, 3), 2, 28, 14), {"odise_patchify_split_f32"}),
    "patchify_split_q8": (lambda: ops.patchify_split(_r(2 * 28 * 28, 3), 2, 28, 14, lo=Q8),
                          {"odise_patchify_split_f32"}),
    "maskclip_bits": (lambda: ops.maskclip_bits(_r(1, 4, 8, 8), 1, 4, 8, 8, 28, 14, 8, 4), {"odise_maskclip_bits_f32"}),
    "open_vocab_merge": (lambda: ops.open_vocab_merge(_r(10, 4), _r(10, 4), 4, torch.zeros(3, dtype=torch.uint8), 0.3,
                                                      0.7, 10, 3, want_open=True),
                         {"odise_open_vocab_merge_f32"}),
    "gather_rows": (lambda: ops.gather_rows(_r(10, 32), _i32(6)), {"odise_gather_rows_f32"}),
    "gather_rows_add": (lambda: ops.gather_rows(_r(10, 32), _i32(6), add=_r(3, 64)[:, :32], add_period=3),
                        {"odise_gather_rows_f32"}),
    "lib.split": (lambda: lib.split(_r(10, 32)), {"odise_split_f32"}),
    "lib.split_q8": (lambda: lib.split(_r(10, 32), lo=Q8), {"odise_split_f32"}),
    "lib.split_f16": (lambda: lib.split(_r(10, 32), f16=True), {"odise_split_f16_f32"}),
    "lib.gemm": (lambda: lib.gemm(_bf16_pair(10, 32), _bf16_pair(16, 32), out=_r(10, 16), bias=_r(16),
                                  act=ops.ACT_RELU),
                 {"odise_gemm_bf16"}),
}


@pytest.mark.parametrize("case", CASES)
def test_ops_wrapper(fake, case):
    """each wrapper launches the entry point it is named for, with arguments the header's prototype takes"""
    call, want = CASES[case]
    call()
    assert fake.launched() == want


@pytest.mark.parametrize("fn", [ops.image_crops, ops.clip_preprocess, ops.crop_resize_bicubic])
def test_image_dtype_refused(fake, fn):
    with pytest.raises(lib.OdiseError, match=f"^{fn.__name__}: uint8 or float32 image expected$"):
        fn(_r(1, 3, 8, 8).double(), _i32(1, 3), 1, 8, 8, 8, 8)
    assert not fake.calls


def test_maskclip_preprocess_dtype_refused(fake):
    with pytest.raises(lib.OdiseError, match="^maskclip_preprocess: uint8 or float32 image expected$"):
        ops.maskclip_preprocess(torch.zeros(1, 3, 8, 8, dtype=torch.int16), 1, 8, 8)
    assert not fake.calls


def test_head_engine(fake):
    """HeadEngine's weight preparation, one forward at B = 1 and 128 x 128, and the CLIP-text scoring"""
    eng = HeadEngine(spec.synth_state_dict(spec.head_params()), "cpu", nmma=3)
    assert fake.launched() == {"odise_split_f32"}
    g = torch.Generator().manual_seed(0)
    feats = {f"s{i}": (torch.randn((128 >> i) ** 2, 512, generator=g), 128 >> i, 128 >> i) for i in (2, 3, 4, 5)}
    eng.set_vocabulary("v", torch.randn(7, 768, generator=g), torch.randn(768, generator=g), [2, 1, 4])
    fake.calls.clear()
    eng.forward(feats, 1, vocab_key="v")
    assert fake.launched() == {
        "odise_split_f32", "odise_gemm_bf16", "odise_groupnorm_stats_ws_f32", "odise_groupnorm_finalize_seg_f32",
        "odise_groupnorm_apply_bs_f32", "odise_add_split_f32", "odise_msda_fused_f32", "odise_layernorm_f32",
        "odise_resize_nhwc_bs_f32", "odise_mask_binarize_f32", "odise_pool_normalize_f32", "odise_attn_mask_bits_f32",
        "odise_attention_tc", "odise_mha_d32_ws_f32", "odise_l2_normalize_split_f32", "odise_class_max_f32"}


def test_post_processor(fake):
    """all three heads at a padding geometry: the output is the un-padded image resized to (H, W)"""
    g = torch.Generator().manual_seed(0)
    pp = PostProcessor("cpu", 5, [0, 2])
    pp(torch.randn(2, 10, 6, generator=g), torch.randn(2, 10, 16, 16, generator=g), 48, 40, instance=True, topk=8,
       padded_size=(64, 64), image_size=(60, 50))
    assert fake.launched() == {"odise_query_scores_f32", "odise_postprocess_fused_f32", "odise_split_f32",
                               "odise_gemm_bf16"}
