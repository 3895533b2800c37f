"""Float64 reference of the inference post-processing (odise_b200/postprocess.py), per image, with the decisions a float32
kernel may legitimately take the other way marked per pixel.

The resample and the semantic einsum are oracle/postprocess.py's own functions (pinned to the reference by
tests/test_oracle_cpu.py) called on float64 tensors; the panoptic bookkeeping and the instance top-k are restated here so
that they also return their counters, the top-two argmax values and the kernel's documented output order.
tests/test_postprocess_ref_cpu.py checks that on float64 inputs everything equals the oracle.  All functions run on the
device of their inputs.

Decision bands.  u = 2^-24 is the float32 unit roundoff.  Per image, R = max (max - min) of a row of class logits and
m = ceil((K + 1) / 32).  Per (query, pixel), lg is the float64 logit, s its sigmoid and D a bound on the difference of
two neighbouring source logits near the pixel: the largest such difference in a 3 x 3 (two stages: 5 x 5) source window
max-pooled, then resampled like the logits; the window covers every source cell the pixel's neighbours touch, so each
of the convex weights multiplies a value at least as large as the differences the sampler meets.
  * Sampler (post_fused_kernel / bilerp, float32).  The source coordinate (o + 0.5) * fl(in / out) - 0.5 carries three
    roundings, so it is off by at most 3u * in source pixels (in = hs, ws; in a two-stage resize also img_h, img_w in
    padded pixels, where the first stage's field has slope <= D * hs / pad_h, D * ws / pad_w).  The fraction
    fy - floor(fy) is exact, and a coordinate error e moves the value by at most e * D.  The weights 1 - l and the
    three-level weighted sum round about six times per stage, each by at most u times the largest of the four
    neighbours, which is <= |lg| + 2D; that term is taken twice for slack.  So
        |lg_f32 - lg_f64| <= samp = 3u * D * (hs + ws [+ img_h * hs / pad_h + img_w * ws / pad_w])
                                    + 12u * (|lg| + 2D) * stages.
  * Sigmoid threshold (d1, absolute logit).  The kernel's sigmoid is __fdividef(1, 1 + __expf(-lg)).  __expf(x) is
    within 2 + |1.173 x| ulp and __fdividef within 2 ulp (CUDA C Programming Guide, intrinsic functions), so near
    lg = 0 the sigmoid is off by <= 2^-22 / 4 + 2^-23 < 2^-21.7, and sigmoid >= 0.5 can flip for |lg| < 2^-19.7:
        d1 = samp + 2^-19.
    The instance mask tests lg > 0 directly, inside the same band.
  * Argmax (relative).  The class probability expf(c - mx) / sum: the rounded argument costs u * R relative, expf
    2 ulp = 4u, the lane sums and the 5-level butterfly (m + 4) u, the IEEE division u:  eps_p = 2 (m + R + 9) u.  The
    sigmoid: a relative error r of 1 + e^-lg reaches s as r * (1 - s); r is (4 + 2.35 |lg|) u from __expf plus u from
    the add, and d lg moves s by (1 - s) d lg; __fdividef adds 4u:
        rel_s = ((5 + 2.35 |lg|) u + samp) (1 - s) + 4u.
    score * sigmoid rounds once more, so the kernel's value is within eps_p + rel_s + u of the float64 one, and the top
    two may trade places where they are closer than the sum of their two bounds.
"""
import math

import torch

from oracle import postprocess as opp

U = 2.0 ** -24
SIGMOID_BAND = 2.0 ** -19


def resample(masks, H, W, geom=None):
    """masks [Q, hs, ws] -> float64 logits [Q, H, W]: odise.py's one-stage resize to the padded input (geom None), or
    that resize to (pad_h, pad_w) followed by sem_seg_postprocess's crop to (img_h, img_w) and resize to (H, W)."""
    x = masks.double().unsqueeze(0)
    if geom is None:
        return opp.upsample_masks(x, (H, W))[0]
    ph, pw, ih, iw = geom
    return opp.sem_seg_postprocess(opp.upsample_masks(x, (ph, pw))[0], (ih, iw), H, W)


def semantic(cls, lg):
    """cls [Q, K+1], lg float64 [Q, H, W] -> sem_seg [K, H, W] (maskformer_model.py:280-284)"""
    return opp.semantic_inference(cls.double(), lg)


def errors(cls, masks, lg, geom=None):
    """The bounds of the module docstring for one image: dict(d1 [Q, H, W] absolute logit band, rel [Q, H, W] relative
    error of the kernel's score * sigmoid, rel_s [Q, H, W] of its sigmoid, eps_p of its class probabilities).
    cls [Q, K+1] and masks [Q, hs, ws] are the kernel's inputs, lg = resample(masks, ...)."""
    m = masks.double()
    g = torch.zeros_like(m)
    g[:, :-1] = (m[:, 1:] - m[:, :-1]).abs()
    g[:, :, :-1] = torch.maximum(g[:, :, :-1], (m[:, :, 1:] - m[:, :, :-1]).abs())
    g[:, 1:] = torch.maximum(g[:, 1:], g[:, :-1].clone())
    g[:, :, 1:] = torch.maximum(g[:, :, 1:], g[:, :, :-1].clone())
    k = 5 if geom is not None else 3
    D = resample(torch.nn.functional.max_pool2d(g.unsqueeze(0), k, 1, k // 2)[0], lg.shape[1], lg.shape[2], geom)
    c = cls.double()
    R = (c.max(-1).values - c.min(-1).values).max().item()
    stages = 2 if geom is not None else 1
    span = m.shape[1] + m.shape[2]
    if geom is not None:
        span += geom[2] * m.shape[1] / geom[0] + geom[3] * m.shape[2] / geom[1]
    a = lg.abs()
    samp = 3 * U * D * span + 12 * U * (a + 2 * D) * stages
    eps_p = 2 * (math.ceil(cls.shape[-1] / 32) + R + 9) * U
    rel_s = ((5 + 2.35 * a) * U + samp) * torch.sigmoid(-lg) + 4 * U
    return dict(d1=samp + SIGMOID_BAND, rel=eps_p + rel_s + U, rel_s=rel_s, eps_p=eps_p)


def query_scores(cls, K, threshold=0.0):
    """cls [Q, K+1] -> (probs [Q, K+1], scores, labels, keep) in float64: torch's max takes the first maximal index,
    so a class tied with void keeps the query; keep needs score > threshold"""
    probs = torch.softmax(cls.double(), -1)
    scores, labels = probs.max(-1)
    return probs, scores, labels, labels.ne(K) & (scores > threshold)


def panoptic(scores, labels, keep, lg, is_thing, overlap=0.8, err=None):
    """maskformer_model.py:286-342 on (scores, labels, keep) of query_scores and lg [Q, H, W].  Returns dict:
    pan int32 [H, W], info (segments_info list), ids [H, W] (argmax over kept queries, -1 without one), fg [H, W],
    area / orig / inter [Q] (the three counts of the overlap test), seg_of [Q] (segment id per query, 0 = none),
    and the bands of a float32 kernel under err (errors(); None: no bands): band_fg [H, W] (the winner's
    |lg| <= d1), band_arg [H, W] (the top two score * sigmoid closer than their two error bounds) and n_unsure [Q]: the
    pixels at which q's counts may differ (band_arg pixels where q is one of the top two, and pixels where |lg_q| <= d1)."""
    Q, H, W = lg.shape
    dev = lg.device
    s = torch.sigmoid(lg)
    pm = torch.where(keep.view(Q, 1, 1), scores.view(Q, 1, 1) * s, torch.full_like(s, -math.inf))
    z = torch.zeros(Q, dtype=torch.int64, device=dev)
    res = dict(pan=torch.zeros(H, W, dtype=torch.int32, device=dev), info=[], ids=torch.full((H, W), -1, device=dev),
               fg=torch.zeros(H, W, dtype=torch.bool, device=dev), area=z, orig=z, inter=z, seg_of=z,
               band_fg=torch.zeros(H, W, dtype=torch.bool, device=dev),
               band_arg=torch.zeros(H, W, dtype=torch.bool, device=dev), n_unsure=z)
    if not bool(keep.any()):
        return res
    ids = pm.argmax(0)                                        # first maximal index, as argmax over the kept subset
    wl = lg.gather(0, ids[None])[0]
    sfg = s >= 0.5
    fg = sfg.gather(0, ids[None])[0]
    area = torch.bincount(ids.flatten(), minlength=Q)
    orig = sfg.flatten(1).sum(1)
    inter = torch.bincount(ids[fg], minlength=Q)
    d1 = err["d1"] if err is not None else 0.0
    band_fg = wl.abs() <= (d1.gather(0, ids[None])[0] if err is not None else 0.0)
    band_lg = lg.abs() <= d1
    if err is not None and int(keep.sum()) > 1:
        top = pm.topk(2, dim=0)
        r = err["rel"].gather(0, top.indices)
        band_arg = (top.values[0] - top.values[1]) <= top.values[0] * r[0] + top.values[1] * r[1]
        hit = torch.zeros(Q, H, W, dtype=torch.bool, device=dev).scatter_(0, top.indices[:1], band_arg[None])
        hit |= torch.zeros_like(hit).scatter_(0, top.indices[1:2], band_arg[None])
    else:
        band_arg = torch.zeros(H, W, dtype=torch.bool, device=dev)
        hit = torch.zeros(Q, H, W, dtype=torch.bool, device=dev)
    n_unsure = (hit | band_lg).flatten(1).sum(1)
    # the sequential bookkeeping on host ints (the kernel: panoptic_assign_kernel)
    a_, o_, i_, kp, lb = (t.tolist() for t in (area, orig, inter, keep, labels))
    thing = [bool(v) for v in is_thing.tolist()]
    seg_of, info, stuff, cur = [0] * Q, [], {}, 0
    for q in range(Q):
        if not kp[q] or not (a_[q] > 0 and o_[q] > 0 and i_[q] > 0) or a_[q] / o_[q] < overlap:
            continue
        c = lb[q]
        if not thing[c]:
            if c in stuff:
                seg_of[q] = stuff[c]
                continue
            stuff[c] = cur + 1
        cur += 1
        seg_of[q] = cur
        info.append({"id": cur, "isthing": thing[c], "category_id": c})
    seg_of = torch.tensor(seg_of, dtype=torch.int64, device=dev)
    pan = torch.where(fg, seg_of[ids], 0).to(torch.int32)
    res.update(pan=pan, info=info, ids=ids, fg=fg, area=area, orig=orig, inter=inter, seg_of=seg_of, band_fg=band_fg,
               band_arg=band_arg, n_unsure=n_unsure)
    return res


def unsure_queries(ref, keep, overlap=0.8):
    """kept queries whose overlap-test outcome could change when each of its counts moves by n_unsure[q]"""
    out = []
    for q, (k, a, o, i, n) in enumerate(zip(*(t.tolist() for t in (keep, ref["area"], ref["orig"], ref["inter"],
                                                                    ref["n_unsure"])))):
        if not k or n == 0:
            continue
        kept = a - n > 0 and o - n > 0 and i - n > 0 and (a - n) / (o + n) >= overlap
        dropped = min(a, o, i) + n == 0 or (o - n > 0 and (a + n) / (o - n) < overlap)
        if not (kept or dropped):
            out.append(q)
    return out


def instance(probs, lg, K, is_thing, topk, panoptic_on=True, masks=None, eps_p=0.0):
    """maskformer_model.py:344-380 in the order include/odise_b200.h promises: descending class probability, ties towards
    the lower flat index q * K + c.  probs [Q, K+1] of query_scores, lg [Q, H, W]; masks: the binary masks to score with
    ([Q, H, W]; default lg > 0).  Returns dict(flat, query, classes, prob, mask_score, scores, valid [k], k, tied):
    valid = is_thing[class] under panoptic_on (the reference's filter), else all true; tied: the k-th and (k+1)-th
    probabilities are within eps_p relative, so the selected set is not determined at float32."""
    p = probs[:, :K].reshape(-1)
    k = min(topk, p.numel())
    ps, order = torch.sort(p, descending=True, stable=True)
    sel = order[:k]
    q, c = sel // K, sel % K
    mp = lg[q]
    pm = (mp > 0).float() if masks is None else masks[q].float()     # float32 0 / 1, so the count + 1e-6 is float32
    ms = (mp.sigmoid().flatten(1) * pm.flatten(1)).sum(1) / (pm.flatten(1).sum(1) + 1e-6)
    valid = is_thing.bool()[c] if panoptic_on else torch.ones(k, dtype=torch.bool, device=p.device)
    tied = k < p.numel() and bool(ps[k - 1] - ps[k] <= eps_p * ps[k - 1])
    return dict(flat=sel, query=q, classes=c, prob=ps[:k], mask_score=ms, scores=ps[:k] * ms, valid=valid, k=k,
                tied=tied)


# ---- a hand-built image for exact comparisons at the identity geometry (H = hs, W = ws) --------------------------------
EDGE_K, EDGE_THINGS, EDGE_HW = 14, (0, 1, 2, 3), (16, 40)
# (class-logit positions set to 0, all others -200) per query: n tied positions give the exact score 1/n in float32 and
# float64 alike, and the label is the first of them.  Mask logits are -8 except the listed (value, rows, cols) boxes.
EDGE_QUERIES = [
    ([13], [(8, (12, 16), (0, 40))]),                                  # 0 stuff, score 1: wins the background
    ([0, 11, 12, 14], [(8, (0, 2), (0, 5))]),                          # 1 area 8 / original 10 == 0.8: kept
    ([1, 14], [(8, (0, 1), (0, 2)), (8, (0, 1), (6, 9))]),             # 2 class tied with void: kept; covers 2 px of 1
    ([2, 3, 5, 6, 7, 8, 9, 10], [(8, (0, 1), (6, 8)), (-2, (3, 4), (20, 21))]),   # 3 area 1, original 2, intersection 0
    ([4, 5, 6, 7, 8, 9, 10, 11], [(8, (3, 5), (0, 5))]),               # 4 stuff 4, ratio 0.7: dropped
    ([4, 5, 6, 14], [(8, (3, 4), (0, 3)), (8, (5, 6), (0, 6))]),       # 5 stuff 4: creates the segment
    ([4, 5, 6, 7, 8, 9, 10, 11], [(8, (6, 7), (0, 4))]),               # 6 stuff 4: merges into it
    ([0, 5, 6, 7], [(8, (8, 10), (0, 3))]),                            # 7 thing 0 ...
    ([0, 8, 9, 10], [(8, (8, 10), (10, 13))]),                         # 8 ... predicted twice: two segments
    ([3, 12], [(8, (10, 11), (0, 2))]),                                # 9 tied with 10 on 2 px: the first query wins
    ([3, 12], [(8, (10, 11), (0, 2)), (8, (10, 11), (20, 30))]),       # 10 area 10 / original 12
    ([5, 6], [(0, (6, 8), (10, 15)), (8, (6, 7), (15, 17))]),          # 11 logits of exactly 0: foreground, not instance
    ([7, 14], [(8, (8, 10), (20, 25))]),                               # 12 another class tied with void
    ([2, 3, 4, 5], [(8, (0, 4), (38, 40))]),                           # 13 in the ragged last 32-wide segment of W = 40
    ([14], [(8, (10, 12), (30, 36))]),                                 # 14 void
]


def edge_case(void=False):
    """(cls [Q, K+1], masks [Q, H, W]) float32 of EDGE_QUERIES; void: every query predicts void"""
    H, W = EDGE_HW
    Q = len(EDGE_QUERIES)
    cls = torch.full((Q, EDGE_K + 1), -200.0)
    masks = torch.full((Q, H, W), -8.0)
    for q, (pos, boxes) in enumerate(EDGE_QUERIES):
        cls[q, [EDGE_K] if void else pos] = 0.0
        for v, (y0, y1), (x0, x1) in boxes:
            masks[q, y0:y1, x0:x1] = v
    return cls, masks
