"""Post-processing (odise_b200/postprocess.py, csrc/postprocess.cu) against the float64 reference tests/postprocess_ref.py
at the evaluation configurations.  At the identity geometry with hand-built logits every output is exact; under resampling
the panoptic map may differ only inside the decision bands the reference derives from the kernel's float32 arithmetic,
segments_info must be equal, and the semantic map and instance scores must be within bars derived the same way."""
import ctypes

import pytest
import torch

import postprocess_ref as pr
from odise_b200 import lib

pytestmark = pytest.mark.gpu

U = pr.U
SPLIT = 3 * 2.0 ** -18          # bf16x3: two split residuals and the dropped lo * lo product, relative per product


def _blobs(seed, B, Q, K, hs, ws, void=2.0):
    """float32 (cls [B, Q, K+1], masks [B, Q, hs, ws]): discs of random centre and radius, slope 1.5 per source pixel"""
    g = torch.Generator().manual_seed(seed)
    cls = torch.randn(B, Q, K + 1, generator=g) * 3
    cls[..., -1] -= void
    yy, xx = torch.meshgrid(torch.arange(hs).float(), torch.arange(ws).float(), indexing="ij")
    c = torch.rand(B, Q, 2, 1, 1, generator=g) * torch.tensor([hs, ws]).view(1, 1, 2, 1, 1).float()
    r = 1.5 + torch.rand(B, Q, 1, 1, generator=g) * min(hs, ws) / 4
    d = ((yy - c[:, :, 0]) ** 2 + (xx - c[:, :, 1]) ** 2).sqrt()
    return cls, (r - d) * 1.5 + torch.randn(B, Q, hs, ws, generator=g) * 0.15


def _is_thing(K, things, dev):
    t = torch.zeros(K, dtype=torch.uint8)
    t[list(things)] = 1
    return t.to(dev)


def _geom(geom):
    return None if geom is None else ctypes.byref(lib.PostprocessGeom(*geom))


def _query_scores(cls, thr=0.0):
    """the kernel's own float32 (probs [B*Q, K+1], scores, labels, keep) through odise_query_scores_f32"""
    B, Q, K1 = cls.shape
    dev = cls.device
    probs = torch.empty(B * Q, K1, device=dev)
    scores = torch.empty(B * Q, device=dev)
    labels, keep = (torch.empty(B * Q, dtype=torch.int32, device=dev) for _ in range(2))
    lib._launch("odise_query_scores_f32", cls.contiguous(), probs, None, scores, labels, keep, B, Q, (Q + 7) // 8 * 8,
                K1, thr)
    return probs, scores, labels, keep


def _run(cls, masks, K, things, H, W, geom=None, thr=0.0, nmma=3, **kw):
    from odise_b200.postprocess import PostProcessor
    dev = torch.device("cuda:0")
    pp = PostProcessor(dev, K, things, object_mask_threshold=thr, nmma=nmma)
    g = {} if geom is None else dict(padded_size=geom[:2], image_size=geom[2:])
    out = pp(cls.to(dev), masks.to(dev), H, W, **g, **kw)
    torch.cuda.synchronize()
    return pp, out


def _fused_depth(H, W):
    """additions behind one instance partial sum of post_fused_kernel + instance_finalize_kernel: the 5-level butterfly,
    the rows a warp walks, the 8 warps and the partials"""
    chunks = 16 if H >= 128 else 1
    rpc = ((H + chunks - 1) // chunks + 7) // 8 * 8
    return 5 + rpc // 8 + 8 + chunks * ((W + 31) // 32)


def _standalone_depth(H, W):
    """the same for instance_mask_partial_kernel: per-thread strided sums, butterfly, 8 warps, the chunks"""
    chunks = 16 if H >= 64 else 1
    rows = (H + chunks - 1) // chunks
    return (rows * W + 255) // 256 + 5 + 8 + chunks


def _check_semantic(got, cls_b, lg, err, Qp, record, tag):
    K = got.shape[0]
    P = torch.softmax(cls_b.double(), -1)[:, :K]
    s = torch.sigmoid(lg)
    ref = pr.semantic(cls_b, lg)
    # + Qp * 2^-126: a class probability below float32's normal range rounds to zero or a subnormal
    bound = (torch.einsum("qc,qhw->chw", P, s * err["rel_s"]) + ref * (err["eps_p"] + SPLIT + 6 * Qp * U)
             + Qp * 2.0 ** -126)
    d = (got.double() - ref).abs()
    assert bool((d <= 2 * bound).all()), (tag, (d / bound).max().item())
    record(f"postprocess parity {tag}: sem_seg max |err| / value {(d / ref.clamp_min(1e-300)).max().item():.2e}, "
           f"/ derived bound {(d / bound).max().item():.2f} of the allowed 2")


def _check_image(out, b, cls, masks, K, things, H, W, record, tag, geom=None, thr=0.0, exact=False, topk=None,
                 panoptic_on=True, depth=None):
    """one image of a PostProcessor output against the float64 reference; returns the reference's panoptic dict"""
    dev = torch.device("cuda:0")
    cls_b, masks_b = cls[b].to(dev), masks[b].to(dev)
    Q = cls_b.shape[0]
    is_thing = _is_thing(K, things, dev)
    lg = pr.resample(masks_b, H, W, geom)
    err = pr.errors(cls_b, masks_b, lg, geom)
    probs, scores, labels, keep = pr.query_scores(cls_b, K, thr)
    assert torch.equal(out["labels"][b].long(), labels) and torch.equal(out["keep"][b].bool(), keep), tag
    if exact:
        assert torch.equal(out["scores"][b].double(), scores), tag
    else:
        assert bool(((out["scores"][b].double() - scores).abs() <= err["eps_p"] * scores).all()), tag
        top2 = probs.topk(2, -1).values
        assert bool((top2[:, 0] - top2[:, 1] > 2 * err["eps_p"] * top2[:, 0]).all()), f"{tag}: a label is tied"
        assert bool(((scores - thr).abs() > 2 * err["eps_p"] * scores).all()), f"{tag}: a score is at the threshold"
    if "sem_seg" in out:
        _check_semantic(out["sem_seg"][b], cls_b, lg, err, (Q + 7) // 8 * 8, record, tag)
    ref = None
    if "panoptic_seg" in out:
        ref = pr.panoptic(scores, labels, keep, lg, is_thing, err=None if exact else err)
        from odise_b200.postprocess import PostProcessor
        info = PostProcessor.segments_info(out["seg_info"][b:b + 1], out["n_segments"][b:b + 1])[0]
        assert info == ref["info"], (tag, info, ref["info"])
        got = out["panoptic_seg"][b]
        if exact:
            assert torch.equal(got, ref["pan"]), (tag, (got != ref["pan"]).nonzero()[:8].tolist())
        else:
            assert not pr.unsure_queries(ref, keep), f"{tag}: an overlap decision lies within the bands"
            band = ref["band_fg"] | ref["band_arg"]
            frac = band.double().mean().item()
            record(f"postprocess parity {tag}: panoptic banded fraction {frac:.2e} ({int(band.sum())} of {band.numel()} px)")
            assert frac < 1e-4, (tag, frac)
            assert torch.equal(got[~band], ref["pan"][~band]), (tag, int((got != ref["pan"]).sum()))
    if "instances" in out:
        _check_instances(out["instances"], b, cls_b, probs, lg, err, K, is_thing, topk, panoptic_on, exact, depth, record, tag)
    return ref


def _check_instances(inst, b, cls_b, probs, lg, err, K, is_thing, topk, panoptic_on, exact, depth, record, tag):
    Q = probs.shape[0]
    k = min(topk, Q * K)
    sc, cl, qi, ok = (inst[n][b] for n in ("scores", "pred_classes", "query_index", "valid"))
    # the tail past min(topk, Q * K)
    assert bool((sc[k:] == 0).all() and (cl[k:] == -1).all() and (qi[k:] == 0).all() and (ok[k:] == 0).all()), tag
    sc, cl, qi, ok = sc[:k], cl[:k].long(), qi[:k].long(), ok[:k]
    flat = qi * K + cl
    # include/odise_b200.h's order: descending float32 class probability, ties towards the lower flat index
    p32 = _query_scores(cls_b[None])[0][:, :K]
    ps, order = torch.sort(p32.reshape(-1), descending=True, stable=True)
    assert torch.equal(flat, order[:k]), (tag, flat[:8].tolist(), order[:8].tolist())
    masks = inst["query_masks"][b] if inst["query_masks"] is not None else (lg > 0).to(torch.uint8)
    ref = pr.instance(probs, lg, K, is_thing, topk, panoptic_on, masks=masks, eps_p=err["eps_p"])
    if exact:
        assert torch.equal(flat, ref["flat"]), tag
    elif not ref["tied"]:
        assert set(flat.tolist()) == set(ref["flat"].tolist()), tag
    assert torch.equal(ok.bool(), is_thing.bool()[cl] if panoptic_on else torch.ones_like(ok, dtype=torch.bool)), tag
    if inst["query_masks"] is not None:
        want = lg > 0
        outside = torch.ones_like(want) if exact else lg.abs() > err["d1"]
        assert torch.equal(masks.bool()[outside], want[outside]), (tag, int((masks.bool() != want).sum()))
    # scores: float64 prob * mask score on the kernel's own binary masks, within the float32 bound
    m = masks.double()
    s = torch.sigmoid(lg)
    num = (s * m).flatten(1).sum(1)
    ms = num / (m.flatten(1).sum(1) + 1e-6)
    rel_ms = (s * m * err["rel_s"]).flatten(1).sum(1) / num.clamp_min(1e-300) + (depth + 3) * U
    want = probs[:, :K].reshape(-1)[flat] * ms[qi]
    bound = want * (err["eps_p"] + rel_ms[qi] + U) + 2.0 ** -126          # subnormal probabilities, as in the semantic bar
    d = (sc.double() - want).abs()
    assert bool((d <= 2 * bound).all()), (tag, (d / bound.clamp_min(1e-300)).max().item())
    record(f"postprocess parity {tag}: instance score max rel err {(d / want.clamp_min(1e-300)).max().item():.2e}")


# ---- a. exact bookkeeping at the identity geometry ----------------------------------------------------------------------
def _edge_batch():
    cls, masks = pr.edge_case()
    void, _ = pr.edge_case(void=True)
    return torch.stack([cls, void, cls]), torch.stack([masks, masks, masks])


def test_edge_cases_exact(cuda, record):
    """Every bookkeeping edge of postprocess_ref.EDGE_QUERIES (ratio exactly 0.8 kept, empty intersection, a dropped first
    stuff query followed by one that creates and one that merges, a thing twice, exact score * sigmoid ties, class tied
    with void, logits of exactly 0, the ragged last warp segment) and an image with no kept query between two full ones:
    panoptic map, segments_info, n_segments, scores, labels, keep, the instance selection and masks are exact."""
    cls, masks = _edge_batch()
    H, W = pr.EDGE_HW
    _, out = _run(cls, masks, pr.EDGE_K, pr.EDGE_THINGS, H, W, instance=True, topk=27)
    assert out["n_segments"].tolist() == [11, 0, 11]
    for b in range(3):
        _check_image(out, b, cls, masks, pr.EDGE_K, pr.EDGE_THINGS, H, W, record, f"edge b{b}", exact=True, topk=27,
                     depth=_fused_depth(H, W))
    # sigmoid(0) is exactly 0.5 on the device: the zero-logit pixels of query 11 are in its panoptic segment
    seg = out["panoptic_seg"][0]
    zeros = masks[0, 11].to(cuda) == 0
    assert bool((seg[zeros] == seg[zeros][0]).all()) and int(seg[zeros][0]) > 0
    assert not bool(out["instances"]["query_masks"][0, 11][zeros].any())


def test_edge_score_equal_to_threshold_is_dropped(cuda, record):
    cls, masks = _edge_batch()
    H, W = pr.EDGE_HW
    _, out = _run(cls, masks, pr.EDGE_K, pr.EDGE_THINGS, H, W)
    thr = float(out["scores"][0, 3])
    assert thr == 0.125                                    # Python's float of a float32 is exact: threshold == score
    _, out = _run(cls, masks, pr.EDGE_K, pr.EDGE_THINGS, H, W, thr=thr, instance=True, topk=27)
    assert not bool(out["keep"][0, [3, 4, 6]].any()) and bool(out["keep"][0, 5])
    for b in range(3):
        _check_image(out, b, cls, masks, pr.EDGE_K, pr.EDGE_THINGS, H, W, record, f"edge thr b{b}", thr=thr, exact=True,
                     topk=27, depth=_fused_depth(H, W))


# ---- b. resampled geometries ---------------------------------------------------------------------------------------
GEOMS = {
    "x4 256x320": dict(seed=10, hs=64, ws=80, H=256, W=320),
    "non-integer 293x215": dict(seed=19, hs=90, ws=66, H=293, W=215),
    "pad-crop-resize landscape": dict(seed=25, hs=80, ws=96, H=291, W=333, geom=(320, 384, 300, 342)),
    "pad-crop-resize portrait": dict(seed=1, hs=96, ws=80, H=333, W=291, geom=(384, 320, 342, 300)),
}


@pytest.mark.parametrize("name", list(GEOMS))
def test_resampled_geometries(cuda, record, name):
    g = GEOMS[name]
    Q, K = 50, 19
    things = range(0, K, 2)
    cls, masks = _blobs(g["seed"], 1, Q, K, g["hs"], g["ws"])
    _, out = _run(cls, masks, K, things, g["H"], g["W"], geom=g.get("geom"), instance=True, topk=100)
    ref = _check_image(out, 0, cls, masks, K, things, g["H"], g["W"], record, name, geom=g.get("geom"), topk=100,
                       depth=_fused_depth(g["H"], g["W"]))
    assert len(ref["info"]) > 0


@pytest.mark.parametrize("B", [1, 3, 8])
def test_batches_match_single_images(cuda, record, B):
    """A batch with an all-void image and an image whose every score is below the threshold: each image's outputs are
    bit-identical to that image alone at B = 1, so no per-image counter leaks between images."""
    Q, K, hs, ws, H, W, thr = 30, 19, 48, 40, 192, 160, 0.3
    things = range(0, K, 2)
    cls, masks = _blobs(100 + B, B, Q, K, hs, ws)
    if B > 1:
        cls[1, :, -1] += 50                                 # all void
        cls[-1] *= 0.05                                     # every score near 1 / (K + 1) < thr
    kw = dict(instance=True, topk=64, thr=thr)
    _, out = _run(cls, masks, K, things, H, W, **kw)
    for b in range(B):
        _, one = _run(cls[b:b + 1], masks[b:b + 1], K, things, H, W, **kw)
        for n in ("sem_seg", "panoptic_seg", "n_segments", "scores", "labels", "keep"):
            assert torch.equal(out[n][b], one[n][0]), (b, n)
        assert torch.equal(out["seg_info"][b], one["seg_info"][0])
        for n, v in out["instances"].items():
            assert torch.equal(v[b], one["instances"][n][0]), (b, n)
        _check_image(out, b, cls, masks, K, things, H, W, record, f"B={B} b{b}", thr=thr, topk=64,
                     depth=_fused_depth(H, W))
    if B > 1:
        assert out["n_segments"][1] == 0 and out["n_segments"][-1] == 0 and not bool(out["keep"][[1, B - 1]].any())


def test_four_1024_images(cuda, record):
    """4 x 1024^2 at Q = 100, K = 133 (COCO panoptic), ×4 from 256^2"""
    B, Q, K = 4, 100, 133
    things = range(80)
    cls, masks = _blobs(7, B, Q, K, 256, 256)
    _, out = _run(cls, masks, K, things, 1024, 1024, instance=True, topk=100)
    for b in range(B):
        _check_image(out, b, cls, masks, K, things, 1024, 1024, record, f"4x1024^2 b{b}", topk=100,
                     depth=_fused_depth(1024, 1024))
        torch.cuda.empty_cache()


# ---- c. sizes -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Q,K", [(100, 133), (250, 150), (646, 459), (100, 847)])
def test_query_and_vocabulary_sizes(cuda, record, Q, K):
    """Q up to 646, the most post_fused_kernel's 76 B of shared memory per query allows; K of COCO (133), ADE-150,
    PC-459 and ADE-full (847)"""
    things = range(0, K, 3)
    hs, ws, H, W = 80, 72, 320, 288
    cls, masks = _blobs(Q + K, 1, Q, K, hs, ws)
    _, out = _run(cls, masks, K, things, H, W, instance=True, topk=1024)
    _check_image(out, 0, cls, masks, K, things, H, W, record, f"Q={Q} K={K}", topk=1024, depth=_fused_depth(H, W))


def test_query_limit(cuda):
    from odise_b200.lib import OdiseError
    cls, masks = _blobs(0, 1, 647, 5, 8, 8)
    with pytest.raises(OdiseError):
        _run(cls, masks, 5, [0], 32, 32)


# ---- d. semantic ----------------------------------------------------------------------------------------------------
def test_semantic_bf16(cuda, record):
    """nmma = 1 (the plain-bf16 semantic GEMM of --precision bf16): within test_gpu_gemm.py's bf16 bar of the largest
    value, and the per-pixel argmax class; Q = 50 is not a multiple of 8, so the zero pad columns are on the path."""
    Q, K, H, W = 50, 133, 128, 96
    cls, masks = _blobs(11, 1, Q, K, 32, 24)
    _, out = _run(cls, masks, K, range(80), H, W, nmma=1, panoptic=False)
    lg = pr.resample(masks[0].to(cuda), H, W)
    ref = pr.semantic(cls[0].to(cuda), lg)
    got = out["sem_seg"][0].double()
    rel = ((got - ref).abs().max() / ref.abs().max()).item()
    agree = (got.argmax(0) == ref.argmax(0)).double().mean().item()
    record(f"postprocess parity semantic nmma=1: rel err {rel:.2e} of the max, argmax agreement {agree:.6f}")
    assert rel < 2e-2


# ---- e. instance ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("topk,Q,K", [(1, 45, 21), (100, 45, 21), (1024, 60, 21), (200, 10, 7)])
def test_instance_topk(cuda, record, topk, Q, K):
    """topk = 1, 100, 1024 (the kernel's limit) and topk > Q * K (the outputs past Q * K are the empty tail)"""
    things = range(0, K, 2)
    cls, masks = _blobs(topk, 2, Q, K, 20, 24)
    _, out = _run(cls, masks, K, things, 80, 96, semantic=False, panoptic=False, instance=True, topk=topk)
    for b in range(2):
        _check_image(out, b, cls, masks, K, things, 80, 96, record, f"instance topk={topk} Q*K={Q * K} b{b}", topk=topk,
                     depth=_fused_depth(80, 96))


def test_instance_options_and_duplicated_queries(cuda, record):
    """Duplicated query rows tie exactly and are ordered towards the lower flat index; panoptic_on = False marks every
    instance valid; instance_masks = False gives the same scores."""
    Q, K = 40, 9
    things = [0, 3, 6]
    cls, masks = _blobs(21, 1, Q, K, 24, 24)
    cls[0, 10:20] = cls[0, 0:10]
    masks[0, 10:20] = masks[0, 0:10]
    kw = dict(semantic=False, panoptic=False, instance=True, topk=200)
    _, on = _run(cls, masks, K, things, 96, 96, **kw)
    _, off = _run(cls, masks, K, things, 96, 96, panoptic_on=False, **kw)
    _, nom = _run(cls, masks, K, things, 96, 96, instance_masks=False, **kw)
    for o, p, tag in ((on, True, "dup panoptic_on"), (off, False, "dup panoptic_on=False")):
        _check_image(o, 0, cls, masks, K, things, 96, 96, record, tag, topk=200, panoptic_on=p,
                     depth=_fused_depth(96, 96))
    assert bool((off["instances"]["valid"][0] == 1).all())
    assert nom["instances"]["query_masks"] is None
    for n in ("scores", "pred_classes", "query_index", "valid"):
        assert torch.equal(nom["instances"][n], on["instances"][n]), n
    assert torch.equal(off["instances"]["scores"], on["instances"]["scores"])
    qi = on["instances"]["query_index"][0]
    assert bool(((qi >= 10) & (qi < 20)).any())             # the duplicates are among the selected


# ---- f. flag independence, h. determinism and synchronisation -----------------------------------------------------
def test_heads_do_not_depend_on_each_other(cuda):
    Q, K, H, W = 37, 19, 128, 72
    cls, masks = _blobs(31, 2, Q, K, 32, 18)
    things = range(0, K, 2)
    _, full = _run(cls, masks, K, things, H, W, instance=True, topk=100)
    _, again = _run(cls, masks, K, things, H, W, instance=True, topk=100)
    heads = {"semantic": ["sem_seg"], "panoptic": ["panoptic_seg", "seg_info", "n_segments"], "instance": ["instances"]}
    for mask in range(1, 8):
        on = {h: bool(mask >> i & 1) for i, h in enumerate(heads)}
        _, out = _run(cls, masks, K, things, H, W, topk=100, **on)
        for h, names in heads.items():
            for n in names:
                if not on[h]:
                    assert n not in out
                elif n == "instances":
                    for m, v in out[n].items():
                        assert torch.equal(v, full[n][m]) and torch.equal(v, again[n][m]), (on, m)
                else:
                    assert torch.equal(out[n], full[n]) and torch.equal(out[n], again[n]), (on, n)
        for n in ("scores", "labels", "keep"):
            assert torch.equal(out[n], full[n])


def test_no_host_synchronisation(cuda):
    from odise_b200.postprocess import PostProcessor
    cls, masks = _blobs(41, 2, 20, 7, 16, 16)
    pp = PostProcessor(cuda, 7, [0, 2])
    c, m = cls.to(cuda), masks.to(cuda)
    pp(c, m, 64, 64, instance=True)                         # warm: module load, GEMM plan
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = pp(c, m, 64, 64, instance=True, padded_size=(64, 64), image_size=(60, 57))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(pp.segments_info(out["seg_info"], out["n_segments"])) == 2


# ---- g. the standalone entry points -----------------------------------------------------------------------------
@pytest.mark.parametrize("geom", [None, (160, 192, 150, 171)])
def test_standalone_entry_points(cuda, record, geom):
    """odise_upsample_sigmoid_split_f32, odise_panoptic_inference_f32 and odise_instance_inference_f32 against the
    float64 reference and against the fused path"""
    B, Q, K, hs, ws = 2, 29, 11, 40, 48
    H, W = (96, 120) if geom is None else (97, 111)
    Qp = (Q + 7) // 8 * 8
    things = range(0, K, 2)
    cls, masks = _blobs(51, B, Q, K, hs, ws)
    _, fused = _run(cls, masks, K, things, H, W, geom=geom, instance=True, topk=100)
    c, m = cls.to(cuda), masks.to(cuda).contiguous()
    probs, scores, labels, keep = _query_scores(c)
    it = _is_thing(K, things, cuda)
    hi, lo = (torch.zeros(B * H * W, Qp, dtype=torch.bfloat16, device=cuda) for _ in range(2))
    up = torch.empty(B, Q, H, W, device=cuda)
    lib._launch("odise_upsample_sigmoid_split_f32", m, hi, lo, up, B, Q, Qp, hs, ws, H, W, _geom(geom))
    L = lib.load()
    pan = torch.empty(B, H, W, dtype=torch.int32, device=cuda)
    seg_info = torch.zeros(B, Q, 3, dtype=torch.int32, device=cuda)
    nseg = torch.empty(B, dtype=torch.int32, device=cuda)
    pws = torch.empty(int(L.odise_panoptic_ws_bytes(B, Q, H, W)), dtype=torch.uint8, device=cuda)
    lib._launch("odise_panoptic_inference_f32", m, scores, labels, keep, it, pan, seg_info, nseg, pws, B, Q, K, hs, ws, H,
                W, 0.8, _geom(geom))
    topk = 100
    isc = torch.empty(B, topk, device=cuda)
    icl, iq, iok = (torch.empty(B, topk, dtype=torch.int32, device=cuda) for _ in range(3))
    qm = torch.empty(B, Q, H, W, dtype=torch.uint8, device=cuda)
    iws = torch.empty(int(L.odise_instance_ws_bytes(B, Q, H, W)), dtype=torch.uint8, device=cuda)
    lib._launch("odise_instance_inference_f32", probs, m, it, isc, icl, iq, iok, qm, iws, B, Q, K, topk, hs, ws, H, W,
                _geom(geom))
    torch.cuda.synchronize()
    out = dict(panoptic_seg=pan, seg_info=seg_info, n_segments=nseg, scores=scores.view(B, Q), labels=labels.view(B, Q),
               keep=keep.view(B, Q), instances=dict(scores=isc, pred_classes=icl, query_index=iq, valid=iok,
                                                    query_masks=qm))
    tag = f"standalone geom={geom}"
    for b in range(B):
        lg = pr.resample(masks[b].to(cuda), H, W, geom)
        err = pr.errors(c[b], masks[b].to(cuda), lg, geom)
        samp = err["d1"] - pr.SIGMOID_BAND
        assert bool(((up[b].double() - lg).abs() <= samp).all()), (tag, ((up[b].double() - lg).abs() / samp).max())
        s = torch.sigmoid(lg)
        planes = (hi.float() + lo.float()).view(B, H, W, Qp)[b]
        d = (planes[..., :Q].permute(2, 0, 1).double() - s).abs()
        assert bool((d <= 2 * s * (err["rel_s"] + SPLIT)).all()), tag
        assert not bool(planes[..., Q:].any())
        _check_image(out, b, cls, masks, K, things, H, W, record, f"{tag} b{b}", geom=geom, topk=topk,
                     depth=_standalone_depth(H, W))
    # against the fused path: the same segments and selection; maps equal outside the bands checked above
    assert torch.equal(nseg, fused["n_segments"]) and torch.equal(seg_info, fused["seg_info"])
    for n in ("pred_classes", "query_index", "valid"):
        assert torch.equal(out["instances"][n], fused["instances"][n]), n
    diff = (pan != fused["panoptic_seg"]).double().mean().item()
    record(f"postprocess parity {tag}: standalone vs fused panoptic pixels differing {diff:.2e}")
    assert diff < 2e-4
