"""tests/postprocess_ref.py, the float64 reference of the GPU post-processing tests, against oracle/postprocess.py (which
tests/test_oracle_cpu.py pins to the reference's MaskFormer methods): on float64 inputs every output is equal."""
import pytest
import torch

from oracle import postprocess as opp
import postprocess_ref as pr


def _blobs(seed, Q, K, h, w):
    g = torch.Generator().manual_seed(seed)
    cls = torch.randn(Q, K + 1, generator=g, dtype=torch.float64) * 3
    cls[:, -1] -= 2
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    c = torch.rand(Q, 2, 1, 1, generator=g, dtype=torch.float64) * torch.tensor([h, w]).view(1, 2, 1, 1)
    r = 2 + torch.rand(Q, 1, 1, generator=g, dtype=torch.float64) * min(h, w) / 3
    d = ((yy - c[:, 0]) ** 2 + (xx - c[:, 1]) ** 2).sqrt()
    return cls, (r - d) * 2 + torch.randn(Q, h, w, generator=g, dtype=torch.float64) * 0.3


def _oracle_lg(masks, H, W, geom):
    up = opp.upsample_masks(masks[None], (H, W) if geom is None else geom[:2])[0]
    return up if geom is None else opp.sem_seg_postprocess(up, geom[2:], H, W)


def _check(cls, masks, K, things, H, W, geom=None, thr=0.0, topk=30, instance=True):
    is_thing = torch.zeros(K, dtype=torch.uint8)
    is_thing[list(things)] = 1
    lg = pr.resample(masks, H, W, geom)
    up = _oracle_lg(masks, H, W, geom)
    assert torch.equal(lg, up)
    assert torch.equal(pr.semantic(cls, lg), opp.semantic_inference(cls, up))
    probs, scores, labels, keep = pr.query_scores(cls, K, thr)
    ref = pr.panoptic(scores, labels, keep, lg, is_thing)
    pan, info = opp.panoptic_inference(cls, up, K, things, object_mask_threshold=thr)
    assert torch.equal(ref["pan"], pan) and ref["info"] == info
    for on in (True, False)[:2 if instance else 0]:
        got = pr.instance(probs, lg, K, is_thing, topk, panoptic_on=on)
        want = opp.instance_inference(cls, up, K, things, topk=got["k"], panoptic_on=on)
        v = got["valid"]
        assert bool((got["prob"][:-1] >= got["prob"][1:]).all())
        key = sorted(zip(got["classes"][v].tolist(), got["scores"][v].tolist()))
        assert key == sorted(zip(want["pred_classes"].tolist(), want["scores"].tolist()))
    return ref, info


@pytest.mark.parametrize("seed,Q,K,h,w,up", [(0, 20, 7, 24, 32, 2), (1, 50, 19, 40, 30, 2), (2, 9, 150, 16, 16, 1)])
def test_reference_equals_oracle_one_stage(seed, Q, K, h, w, up):
    cls, masks = _blobs(seed, Q, K, h, w)
    _, info = _check(cls, masks, K, range(0, K, 2), h * up, w * up)
    assert len(info) > 0


@pytest.mark.parametrize("geom,out", [((40, 48, 37, 43), (29, 31)), ((48, 40, 43, 37), (31, 29))])
def test_reference_equals_oracle_pad_crop_resize(geom, out):
    cls, masks = _blobs(3, 8, 11, geom[0] // 4, geom[1] // 4)
    _, info = _check(cls, masks, 11, range(0, 11, 2), *out, geom=geom)
    assert len(info) > 0


def test_reference_equals_oracle_with_threshold_and_void():
    cls, masks = _blobs(4, 30, 9, 12, 12)
    _check(cls, masks, 9, [0, 3], 48, 48, thr=0.6)
    cls[:, -1] += 100                                     # every query predicts void: an empty panoptic map
    ref, info = _check(cls, masks, 9, [0, 3], 48, 48)
    assert info == [] and not bool(ref["pan"].any())


def test_edge_case_equals_oracle_and_hits_every_edge():
    """The hand-built image of the GPU parity tests: every bookkeeping edge it is built for is really there."""
    cls, masks = pr.edge_case()
    H, W = pr.EDGE_HW
    ref, info = _check(cls.double(), masks.double(), pr.EDGE_K, pr.EDGE_THINGS, H, W, topk=27)
    a, o, i = (ref[k].tolist() for k in ("area", "orig", "inter"))
    assert (a[1], o[1]) == (8, 10) and ref["seg_of"][1] > 0                        # ratio exactly 0.8 is kept
    assert a[3] > 0 and o[3] > 0 and i[3] == 0 and ref["seg_of"][3] == 0           # empty intersection
    assert a[4] / o[4] < 0.8 and ref["seg_of"][4] == 0                             # stuff: first query dropped,
    assert ref["seg_of"][5] > 0 and ref["seg_of"][6] == ref["seg_of"][5]           # the next creates, the last merges
    assert len({int(ref["seg_of"][q]) for q in (1, 7, 8)}) == 3                    # thing 0 three times
    assert a[9] == 2 and a[10] == 10 and o[10] == 12 and ref["seg_of"][10] > 0     # exact score * sigmoid ties
    probs, scores, labels, keep = pr.query_scores(cls, pr.EDGE_K)
    assert labels[2] == 1 and labels[12] == 7 and bool(keep[2]) and bool(keep[12])   # class tied with void: kept
    assert not bool(keep[14])
    assert (ref["pan"] == ref["seg_of"][11]).sum() == 12                           # the exact zeros are foreground
    assert len(info) == 11 and ref["area"][13] == 8
    thr = float(scores[3])
    assert thr == 0.125
    ref_t, _ = _check(cls.double(), masks.double(), pr.EDGE_K, pr.EDGE_THINGS, H, W, thr=thr, topk=27)
    assert not bool(pr.query_scores(cls, pr.EDGE_K, thr)[3][[3, 4, 6]].any()) and ref_t["seg_of"][5] > 0
    void_cls, _ = pr.edge_case(void=True)
    assert _check(void_cls.double(), masks.double(), pr.EDGE_K, pr.EDGE_THINGS, H, W, instance=False)[1] == []


def test_bands_mark_only_decisions_near_a_threshold():
    """The float32 error bounds are small, an exact zero logit lies in the sigmoid band, a near-tie of score * sigmoid
    lies in the argmax band, and without bounds there are no bands."""
    cls, masks = _blobs(5, 12, 5, 10, 10)
    cls[:, -1] -= 10                                      # every query kept
    masks[1] = masks[0]
    cls[1] = cls[0]
    cls[1, 0] += 1e-9                                     # query 1: the same mask, a score larger by ~1e-10
    masks[0, 4, 4] = 0.0
    lg = pr.resample(masks, 10, 10)
    err = pr.errors(cls, masks, lg)
    _, scores, labels, keep = pr.query_scores(cls, 5)
    is_thing = torch.tensor([1, 0, 1, 0, 1], dtype=torch.uint8)
    ref = pr.panoptic(scores, labels, keep, lg, is_thing, err=err)
    assert bool((err["d1"] < 1e-4).all()) and bool((err["rel"] < 1e-4).all())
    assert bool((lg.abs() <= err["d1"])[0, 4, 4]) and bool(((lg.abs() <= err["d1"]) <= (lg.abs() < 1e-4)).all())
    won = ref["ids"] == 1
    assert bool(won.any()) and bool(ref["band_arg"][won].all()) and ref["n_unsure"][0] >= int(won.sum())
    far = (ref["ids"] != 0) & (ref["ids"] != 1)
    assert not bool(ref["band_arg"][far].any())
    plain = pr.panoptic(scores, labels, keep, lg, is_thing)
    assert not bool(plain["band_fg"].any() or plain["band_arg"].any()) and torch.equal(plain["pan"], ref["pan"])
