"""GPU parity of the device-side post-processing (odise_b200/postprocess.py) vs oracle/postprocess.py
(== the reference's MaskFormer.semantic_inference / panoptic_inference, tests/test_oracle_cpu.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _case(seed, B, Q, K, h, w):
    g = torch.Generator().manual_seed(seed)
    cls = torch.randn(B, Q, K + 1, generator=g) * 3
    cls[..., -1] -= 2.0                                    # most queries are "objects"
    # blobby masks so that segments survive the overlap test
    yy, xx = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")
    masks = torch.empty(B, Q, h, w)
    for b in range(B):
        for q in range(Q):
            cy, cx = torch.rand(2, generator=g) * torch.tensor([h, w])
            r = 2 + torch.rand(1, generator=g) * min(h, w) / 3
            masks[b, q] = (r - ((yy - cy) ** 2 + (xx - cx) ** 2).sqrt()) * 2 + torch.randn(h, w, generator=g) * 0.3
    return cls, masks


@pytest.mark.parametrize("cfg", [(1, 2, 20, 7, 24, 32, 4), (2, 1, 100, 150, 64, 64, 4), (3, 2, 50, 19, 32, 48, 2),
                                 (7, 2, 20, 7, 32, 24, 4), (8, 1, 50, 19, 36, 28, 4)])          # portrait: h > w
def test_postprocess(cuda, cfg):
    from odise_b200.postprocess import PostProcessor
    from oracle import postprocess as opp
    seed, B, Q, K, h, w, up = cfg
    H, W = h * up, w * up
    cls, masks = _case(seed, B, Q, K, h, w)
    things = list(range(0, K, 2))
    pp = PostProcessor(cuda, K, things)
    out = pp(cls.to(cuda), masks.to(cuda), H, W)
    torch.cuda.synchronize()
    infos = pp.segments_info(out["seg_info"], out["n_segments"])
    n_nonempty = 0
    for b in range(B):
        up_masks = opp.upsample_masks(masks[b:b + 1], (H, W))[0]
        sem = opp.semantic_inference(cls[b], up_masks)
        got = out["sem_seg"][b].cpu()
        rel = ((got.double() - sem.double()).abs().max() / sem.abs().max()).item()
        assert rel < 1e-4, rel
        pan, info = opp.panoptic_inference(cls[b], up_masks, K, things)
        assert info == infos[b], (info, infos[b])
        agree = (out["panoptic_seg"][b].cpu() == pan).float().mean().item()
        assert agree > 0.9995, agree          # ties at sigmoid == 0.5 / argmax rounding may flip isolated pixels
        n_nonempty += len(info) > 0
    assert n_nonempty > 0


@pytest.mark.parametrize("cfg", [(4, 2, 20, 7, 24, 32, 4, 50), (5, 1, 100, 150, 64, 64, 4, 100), (6, 1, 5, 3, 16, 16, 2, 100),
                                 (10, 2, 20, 7, 32, 24, 4, 50), (11, 1, 5, 3, 20, 12, 2, 100)])  # portrait: h > w
def test_instance_inference(cuda, cfg):
    """MaskFormer.instance_inference (maskformer_model.py:344-380): top-k (query, class) pairs, mask-weighted scores."""
    from odise_b200.postprocess import PostProcessor
    from oracle import postprocess as opp
    seed, B, Q, K, h, w, up, topk = cfg
    H, W = h * up, w * up
    cls, masks = _case(seed, B, Q, K, h, w)
    things = list(range(0, K, 2))
    pp = PostProcessor(cuda, K, things)
    out = pp(cls.to(cuda), masks.to(cuda), H, W, semantic=False, panoptic=False, instance=True, topk=topk)["instances"]
    torch.cuda.synchronize()
    k_eff = min(topk, Q * K)
    for b in range(B):
        up_masks = opp.upsample_masks(masks[b:b + 1], (H, W))[0]
        ref = opp.instance_inference(cls[b], up_masks, K, things, topk=k_eff, panoptic_on=True)
        ok = out["valid"][b].cpu().bool()
        assert int(out["valid"][b, k_eff:].sum()) == 0
        sc, pc, qi = out["scores"][b].cpu()[ok], out["pred_classes"][b].cpu()[ok], out["query_index"][b].cpu()[ok]
        assert sc.numel() == ref["scores"].numel()
        # the reference's top-k is unsorted: compare as sets ordered by (class, score)
        o1 = sorted(range(sc.numel()), key=lambda i: (int(pc[i]), float(sc[i])))
        o2 = sorted(range(sc.numel()), key=lambda i: (int(ref["pred_classes"][i]), float(ref["scores"][i])))
        assert [int(pc[i]) for i in o1] == [int(ref["pred_classes"][i]) for i in o2]
        assert torch.allclose(sc[o1], ref["scores"][o2], rtol=2e-4, atol=1e-6)
        gm = out["query_masks"][b].cpu()[qi.long()][o1].float()
        agree = (gm == ref["pred_masks"][o2]).float().mean().item()
        assert agree > 0.9999, agree
        assert torch.isin(pc, torch.tensor(things, dtype=pc.dtype)).all()


def test_postprocess_with_padding_and_resize(cuda):
    """odise.py:326-347: masks upsampled to the padded input, cropped to the image, resized to the dataset's original
    size (sem_seg_postprocess) BEFORE semantic / panoptic / instance inference."""
    _padding_and_resize(cuda, pad=(160, 192), img=(150, 171), outsz=(97, 111))


def test_postprocess_with_padding_and_resize_portrait(cuda):
    """the same in portrait: padded input 192 x 160, image 171 x 150, output 111 x 97"""
    _padding_and_resize(cuda, pad=(192, 160), img=(171, 150), outsz=(111, 97))


def _padding_and_resize(cuda, pad, img, outsz):
    from odise_b200.postprocess import PostProcessor
    from oracle import postprocess as opp
    B, Q, K, h, w = 1, 30, 11, pad[0] // 4, pad[1] // 4
    cls, masks = _case(9, B, Q, K, h, w)
    things = list(range(0, K, 2))
    pp = PostProcessor(cuda, K, things)
    out = pp(cls.to(cuda), masks.to(cuda), outsz[0], outsz[1], instance=True, topk=50, padded_size=pad, image_size=img)
    torch.cuda.synchronize()
    up = opp.sem_seg_postprocess(opp.upsample_masks(masks, pad)[0], img, *outsz)
    sem = opp.semantic_inference(cls[0], up)
    got = out["sem_seg"][0].cpu()
    assert got.shape == (K, *outsz)
    assert ((got.double() - sem.double()).abs().max() / sem.abs().max()).item() < 1e-4
    pan, info = opp.panoptic_inference(cls[0], up, K, things)
    assert info == pp.segments_info(out["seg_info"], out["n_segments"])[0] and len(info) > 0
    assert (out["panoptic_seg"][0].cpu() == pan).float().mean().item() > 0.999
    ref = opp.instance_inference(cls[0], up, K, things, topk=50, panoptic_on=True)
    ok = out["instances"]["valid"][0].cpu().bool()
    sc = out["instances"]["scores"][0].cpu()[ok]
    assert sc.numel() == ref["scores"].numel()
    assert torch.allclose(sc.sort().values, ref["scores"].sort().values, rtol=3e-4, atol=1e-6)
