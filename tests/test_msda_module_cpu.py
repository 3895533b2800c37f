"""CPU checks of the MSDeformAttn module drop-in (odise_b200.msda.MSDeformAttn): the fp64 module oracle
(oracle/msda_module.py::oracle_module_grads) is pinned against the reference's own MSDeformAttn module run on the CPU (its
ms_deform_attn_core_pytorch fallback); our module's state-dict keys, shapes and initialisation equal the reference's; the
new C entry point validates its arguments without a GPU; CPU tensors are refused (there is no CPU path)."""
import warnings

import pytest
import torch

FIXTURE = "ref_pinned_msda_module.pt"

# small encoder-style problems (queries = the pixels of all levels) at D = 32: 2-column reference points with a padding
# mask, and 4-column box reference points
PIN_CASES = {
    "grid_padding": dict(seed=1, N=2, d_model=64, n_heads=2, shapes=[(2, 2), (4, 4), (8, 8)], n_points=2, padding=True),
    "box": dict(seed=2, N=1, d_model=64, n_heads=2, shapes=[(4, 4), (8, 8)], n_points=3, box=True),
}
# constructor arguments whose state dicts are compared: the default, the ODISE pixel decoder's, and a tiny one whose
# whole seeded initialisation (xavier draws included) is stored
INIT_CONFIGS = {"default": (256, 4, 8, 4), "odise": (256, 3, 8, 4)}
SEEDED_CONFIG = (16, 2, 2, 2)
DETERMINISTIC = ("sampling_offsets.weight", "sampling_offsets.bias", "attention_weights.weight", "attention_weights.bias",
                 "value_proj.bias", "output_proj.bias")


def _reference_run(cfg):
    """output and gradients of the reference's MSDeformAttn module in fp64 on the CPU for module_problem(**cfg)"""
    from oracle import refshim
    from oracle.msda_module import MODULE_PARAMS, module_problem
    pr = module_problem(**cfg)
    m = refshim.modules().MSDeformAttn(cfg["d_model"], len(cfg["shapes"]), cfg["n_heads"], cfg["n_points"]).double()
    m.load_state_dict(pr["params"])
    q, x, r = (pr[k].clone().requires_grad_(True) for k in ("query", "input_flatten", "reference_points"))
    out = m(q, r, x, pr["spatial_shapes"], pr["level_start_index"], pr["padding_mask"])
    out.backward(pr["grad_output"])
    named = dict(m.named_parameters())
    grads = {k: named[k].grad for k in MODULE_PARAMS}
    grads.update(query=q.grad, input_flatten=x.grad, reference_points=r.grad)
    return dict(output=out.detach(), grads=grads)


def _store(v):
    from oracle import refshim
    return dict(output=refshim.sample(v["output"], k=1024),
                grads={k: refshim.sample(t, k=1024, seed=i) for i, (k, t) in enumerate(sorted(v["grads"].items()))})


@pytest.mark.parametrize("name", sorted(PIN_CASES))
def test_module_oracle_pinned_to_reference(name):
    """oracle_module_grads == the reference module's own forward and autograd backward (fp64), for the output and the
    gradients of all eight parameters, the query, the input and the reference points."""
    from oracle import refshim
    from oracle.msda_module import module_problem, oracle_module_grads, sample_margin
    cfg = PIN_CASES[name]
    pr = module_problem(**cfg)
    assert sample_margin(pr["params"], pr["query"], pr["reference_points"], pr["spatial_shapes"], cfg["n_heads"],
                         cfg["n_points"]) >= 0.02
    ref = refshim.pinned(name, lambda: _reference_run(cfg), fixture=FIXTURE, store=_store)
    out, grads = oracle_module_grads(pr["params"], pr["query"], pr["reference_points"], pr["input_flatten"],
                                     pr["spatial_shapes"], pr["level_start_index"], pr["padding_mask"],
                                     pr["grad_output"], cfg["n_heads"], cfg["n_points"], ref_grad=True)
    assert sorted(grads) == sorted(ref["grads"])
    for k, got in [("output", out)] + sorted(grads.items()):
        want = ref["output"] if k == "output" else ref["grads"][k]
        a, b = refshim.at_sample(got, want)
        scale = max(1.0, b.abs().max().item())
        assert (a - b).abs().max().item() < 1e-10 * scale, (name, k)


def _reference_init():
    from oracle import refshim
    Ref = refshim.modules().MSDeformAttn
    res = {}
    for key, args in INIT_CONFIGS.items():
        sd = Ref(*args).state_dict()
        res[key] = dict(keys=list(sd), shapes=[list(t.shape) for t in sd.values()],
                        bias=sd["sampling_offsets.bias"].clone(),
                        absmax={k: sd[k].abs().max() for k in DETERMINISTIC if k != "sampling_offsets.bias"})
    torch.manual_seed(0)
    res["seeded"] = {k: v.clone() for k, v in Ref(*SEEDED_CONFIG).state_dict().items()}
    return res


def test_module_state_dict_and_init_match_reference():
    """Same parameter names, order and shapes as the reference module (so state dicts load both ways), the same
    directional sampling_offsets bias, zeros where the reference puts zeros, and under one seed the same draws for the
    whole initial state (the four Linears are created and re-initialised in the reference's order)."""
    from oracle import refshim
    from odise_b200.msda import MSDeformAttn
    ref = refshim.pinned("init", _reference_init, fixture=FIXTURE)
    for key, args in INIT_CONFIGS.items():
        sd = MSDeformAttn(*args).state_dict()
        assert list(sd) == ref[key]["keys"], key
        assert [list(t.shape) for t in sd.values()] == ref[key]["shapes"], key
        assert torch.equal(sd["sampling_offsets.bias"], ref[key]["bias"]), key
        for k, v in ref[key]["absmax"].items():
            assert sd[k].abs().max() == v == 0, (key, k)
    torch.manual_seed(0)
    sd = MSDeformAttn(*SEEDED_CONFIG).state_dict()
    assert list(sd) == list(ref["seeded"])
    for k, v in ref["seeded"].items():
        assert torch.equal(sd[k], v), k


def test_module_loads_pixel_decoder_checkpoint_keys():
    """The self_attn entries of an ODISE checkpoint's pixel-decoder encoder layer (odise_b200/spec.py inventory) load
    into MSDeformAttn(256, 3, 8, 4) strictly, and the module's state dict goes back under the same keys."""
    from odise_b200 import spec
    from odise_b200.msda import MSDeformAttn
    prefix = "sem_seg_head.pixel_decoder.transformer.encoder.layers.0.self_attn."
    params = [p for p in spec.pixel_decoder_params() if p[0].startswith(prefix)]
    sd = spec.synth_state_dict(params, 0)
    m = MSDeformAttn(256, 3, 8, 4)
    m.load_state_dict({k[len(prefix):]: v for k, v in sd.items()}, strict=True)
    back = {prefix + k: v for k, v in m.state_dict().items()}
    assert sorted(back) == sorted(sd) and all(torch.equal(back[k], sd[k]) for k in sd)


def test_module_constructor_checks():
    from odise_b200.msda import MSDeformAttn
    with pytest.raises(ValueError):
        MSDeformAttn(d_model=100, n_heads=8)
    with pytest.warns(UserWarning):
        MSDeformAttn(d_model=240, n_heads=8)                 # D = 30
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        m = MSDeformAttn()
    assert m.im2col_step == 128 and (m.d_model, m.n_levels, m.n_heads, m.n_points) == (256, 4, 8, 4)


def test_module_has_no_cpu_path():
    from odise_b200 import lib
    from odise_b200.msda import MSDeformAttn, MSDeformAttnFusedFunction
    m = MSDeformAttn(64, 2, 2, 2)
    ss, lsi = torch.tensor([[2, 2], [1, 1]]), torch.tensor([0, 4])
    q, x, r = torch.zeros(1, 5, 64), torch.zeros(1, 5, 64), torch.zeros(1, 5, 2, 2)
    with pytest.raises(RuntimeError):
        m(q, r, x, ss, lsi)
    value, offs, logits = torch.zeros(1, 5, 2, 32), torch.zeros(1, 5, 2, 2, 2, 2), torch.zeros(1, 5, 2, 4)
    with pytest.raises(RuntimeError):
        lib.msda_fused_forward(value, ss, lsi, r, offs, logits)
    with pytest.raises(RuntimeError):
        lib.msda_fused_backward(value, ss, lsi, r, offs, logits, torch.zeros(1, 5, 64))
    with pytest.raises(RuntimeError):
        MSDeformAttnFusedFunction.apply(value.requires_grad_(), ss, lsi, r, offs, logits)


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    return ge.build()


def test_fused_backward_argument_validation_without_gpu(built):
    from odise_b200 import lib
    fn = lib.load().odise_msda_fused_backward_f32
    p = 16       # any non-null address: every call below fails its checks before anything is dereferenced or launched
    assert fn(*([None] * 10), 1, 1, 1, 32, 1, 1, 1, None) == 10001
    assert fn(*([p] * 9), None, 1, 1, 1, 32, 1, 1, 1, None) == 10001                      # grad_logits missing
    for bad in range(7):                                                                  # N S M D L Lq P
        dims = [1, 1, 1, 32, 1, 1, 1]
        dims[bad] = 0
        assert fn(*([p] * 10), *dims, None) == 10001
    assert fn(*([p] * 10), 1, 1, 1, 32, 9, 1, 1, None) == 10001                          # L > 8
    assert fn(*([p] * 10), 1, 1, 1, 64, 1, 1, 1, None) == lib.ODISE_ERR_UNSUPPORTED       # D != 32
    assert fn(*([p] * 10), 1, 1, 1, 32, 3, 1, 11, None) == lib.ODISE_ERR_UNSUPPORTED      # L * P = 33 > 32
    assert fn(*([p] * 10), 1, 1 << 26, 1, 32, 1, 1, 1, None) == lib.ODISE_ERR_UNSUPPORTED  # S * M * D >= 2^31
