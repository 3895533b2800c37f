"""Training drop-in for Mask2Former's SetCriterion and HungarianMatcher (third_party/Mask2Former/mask2former/modeling/
criterion.py and matcher.py), as the ODISE config builds them (configs/common/models/mask_generator_with_label.py:66-83).

    from odise_b200.criterion import SetCriterion, HungarianMatcher   # in place of the two mask2former imports

Both classes keep the reference's constructor signatures and defaults, weight_dict, the empty_weight buffer (state dicts
load both ways), forward results (matcher indices as CPU int64 tensor pairs; the criterion's loss_ce / loss_mask /
loss_dice with _i suffixes as 0-dim float32 tensors) and __repr__.

Random numbers: every torch.rand call of the reference is made with the same shape, dtype and device and in the same
order, per prediction set (the final one, then aux_outputs in order): rand(1, P, 2) per image for the matcher, then
rand(N, int(P * oversample_ratio), 2) and, if P - int(importance_sample_ratio * P) > 0, rand(N, that, 2) for the mask
losses, N = sum_b min(Q, T_b).  Row n of the loss draws belongs to the n-th matched pair in the reference's order (images
in order, scipy's row order within an image).  So with the same seed the points are the reference's points.

When SetCriterion.matcher is this module's HungarianMatcher, forward computes the cost matrices of every prediction set
and image into one [L, B, Q, Tmax] buffer, copies it to pinned host memory with one synchronisation, runs
scipy.optimize.linear_sum_assignment per (set, image), sends the pair tables back with one non-blocking copy and then
runs the losses of every set.  num_masks keeps the reference's all_reduce and .item() when torch.distributed is
initialised (and is computed on the host otherwise), so a forward makes at most 2 synchronising calls.  Any other matcher
object is called once per set, as the reference does.

With SetCriterion.match_on_device = True, every set on the fused path and max(Q, T_b) <= lib.MASK_MAX_ASSIGN, the
assignment runs on the device instead (lib.mask_assign: scipy's algorithm, fp64, scipy's indices ties included) and,
under torch.distributed, num_masks stays the all-reduced device tensor: forward and backward make no synchronising call.
Where the reference raises ValueError (a NaN or -inf cost, an infeasible problem) this path cannot, as raising needs a
synchronisation: SetCriterion.match_status [L, B] int32 holds 0, 1 (NaN / -inf) or 2 (infeasible) per (set, image).

The fused path (odise_mask_* kernels) runs a set when its tensors are on CUDA, pred_masks is float32 / float16 /
bfloat16 [B, Q, H, W], every target's "masks" is bool or uint8 of one [Hg, Wg] on that device, and the point counts are
within the kernels' limits (lib.MASK_MAX_*).  The target masks are read as bytes: no float copy of a target exists.  The
mask-loss gradient is summed in int64 fixed point, so it is bit-reproducible and the criterion runs under
torch.use_deterministic_algorithms(True).  Every other input, CPU tensors included, and any call with use_fused = False,
takes the composed path: the reference's algorithm in torch ops (F.grid_sample sampling, torch.topk selection)."""
import numpy as np
import torch
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib

_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def point_sample(input, point_coords, **kwargs):
    """detectron2's point_sample: F.grid_sample of input [N, C, H, W] at point_coords [N, P, 2] in [0, 1] x [0, 1]
    -> [N, C, P]."""
    return F.grid_sample(input, 2.0 * point_coords.unsqueeze(2) - 1.0, **kwargs).squeeze(3)


def _pairwise_sigmoid_ce(inputs, targets):
    """[n, P] logits x [m, P] labels -> [n, m] mean over points of BCE-with-logits"""
    pos = F.binary_cross_entropy_with_logits(inputs, torch.ones_like(inputs), reduction="none")
    neg = F.binary_cross_entropy_with_logits(inputs, torch.zeros_like(inputs), reduction="none")
    return (torch.einsum("nc,mc->nm", pos, targets) + torch.einsum("nc,mc->nm", neg, 1 - targets)) / inputs.shape[1]


def _pairwise_dice(inputs, targets):
    """[n, P] logits x [m, P] labels -> [n, m] dice loss 1 - (2 sum s t + 1) / (sum s + sum t + 1), s = sigmoid"""
    s = inputs.sigmoid().flatten(1)
    numerator = 2 * torch.einsum("nc,mc->nm", s, targets)
    denominator = s.sum(-1)[:, None] + targets.sum(-1)[None, :]
    return 1 - (numerator + 1) / (denominator + 1)


def _sigmoid_ce_loss(inputs, targets, num_masks):
    return F.binary_cross_entropy_with_logits(inputs, targets, reduction="none").mean(1).sum() / num_masks


def _dice_loss(inputs, targets, num_masks):
    s = inputs.sigmoid().flatten(1)
    numerator = 2 * (s * targets).sum(-1)
    denominator = s.sum(-1) + targets.sum(-1)
    return (1 - (numerator + 1) / (denominator + 1)).sum() / num_masks


def _point_counts(num_points, oversample_ratio, importance_sample_ratio):
    """(candidates, uncertain points) of detectron2's get_uncertain_point_coords_with_randomness"""
    assert oversample_ratio >= 1
    assert 0 <= importance_sample_ratio <= 1
    return int(num_points * oversample_ratio), int(importance_sample_ratio * num_points)


def _uncertain_points(coarse_logits, cand, rnd, k):
    """the k candidates of cand [N, S, 2] with the largest -|logit| (torch.topk), then the random points rnd"""
    logits = point_sample(coarse_logits, cand, align_corners=False)
    idx = torch.topk(-(torch.abs(logits[:, 0, :])), k=k, dim=1)[1]
    coords = torch.gather(cand, 1, idx[:, :, None].expand(-1, -1, 2))
    return coords if rnd is None else torch.cat([coords, rnd], dim=1)


class _Targets:
    """The targets of one forward: per-image counts, and (built once, on first use) the labels and the target masks as
    one [sum T, Hg, Wg] uint8 tensor."""

    def __init__(self, targets):
        self.targets = targets
        self.counts = [len(t["labels"]) for t in targets]
        self.Tmax = max(self.counts, default=0)
        self._labels = self._bytes = None

    def bytes_ok(self, device):
        ms = [t["masks"] for t in self.targets]
        if not ms or any(m.dim() != 3 or m.dtype not in (torch.bool, torch.uint8) or m.device != device for m in ms):
            return False
        if any(m.shape[0] != c for m, c in zip(ms, self.counts)):
            return False
        return len({tuple(m.shape[1:]) for m in ms}) == 1 and all(t["labels"].device == device for t in self.targets)

    def labels(self):
        if self._labels is None:
            self._labels = torch.cat([t["labels"].long() for t in self.targets])
        return self._labels

    def bytes(self):
        if self._bytes is None:
            self._bytes = torch.cat([t["masks"].view(torch.uint8) for t in self.targets]).contiguous()
        return self._bytes


def _fused_ok(pred_masks, pred_logits, tg, num_points, cand=0, k=0):
    return (pred_masks.is_cuda and pred_logits.is_cuda and pred_masks.dtype in _DTYPES and pred_masks.dim() == 4
            and pred_masks.shape[0] <= lib.MASK_MAX_IMAGES and 0 < num_points <= lib.MASK_MAX_POINTS
            and cand <= lib.MASK_MAX_CANDIDATES and k <= min(num_points, cand) and tg.bytes_ok(pred_masks.device))


def _assign(C, counts):
    """linear_sum_assignment of every [Q, T_b] slice of the cost buffer C [L, B, Q, Tmax]: one copy to the host (pinned,
    one synchronisation for a CUDA buffer) -> per set, per image (int64 i, int64 j) CPU tensors"""
    if C.is_cuda:
        host = torch.empty(C.shape, dtype=C.dtype, pin_memory=True)
        host.copy_(C, non_blocking=True)
        torch.cuda.current_stream(C.device).synchronize()
    else:
        host = C
    a = host.numpy()
    out = []
    for l in range(a.shape[0]):
        res = []
        for b, T in enumerate(counts):
            i, j = linear_sum_assignment(a[l, b, :, :T])
            res.append((torch.as_tensor(i, dtype=torch.int64), torch.as_tensor(j, dtype=torch.int64)))
        out.append(res)
    return out


class HungarianMatcher(nn.Module):
    """Mask2Former's HungarianMatcher: a one-to-one assignment of predictions to targets minimising
    cost_class * (-prob[label]) + cost_mask * sigmoid CE + cost_dice * dice over num_points random points shared by the
    masks of an image.  On CUDA with byte target masks the costs come from odise_mask_cost_* (one launch for the batch),
    and a call synchronises once for all its images; use_fused = False forces the composed path."""

    def __init__(self, cost_class: float = 1, cost_mask: float = 1, cost_dice: float = 1, num_points: int = 0):
        super().__init__()
        self.cost_class = cost_class
        self.cost_mask = cost_mask
        self.cost_dice = cost_dice
        assert cost_class != 0 or cost_mask != 0 or cost_dice != 0, "all costs cant be 0"
        self.num_points = num_points
        self.use_fused = True

    def _cost_composed(self, outputs, targets, b, coords):
        out_prob = outputs["pred_logits"][b].softmax(-1)
        cost_class = -out_prob[:, targets[b]["labels"]]
        out_mask = outputs["pred_masks"][b][:, None]
        tgt_mask = targets[b]["masks"].to(out_mask)[:, None]
        tgt_mask = point_sample(tgt_mask, coords.repeat(tgt_mask.shape[0], 1, 1), align_corners=False).squeeze(1)
        out_mask = point_sample(out_mask, coords.repeat(out_mask.shape[0], 1, 1), align_corners=False).squeeze(1)
        with torch.autocast("cuda", enabled=False):
            out_mask, tgt_mask = out_mask.float(), tgt_mask.float()
            cost_mask = _pairwise_sigmoid_ce(out_mask, tgt_mask)
            cost_dice = _pairwise_dice(out_mask, tgt_mask)
        C = self.cost_mask * cost_mask + self.cost_class * cost_class + self.cost_dice * cost_dice
        return C.reshape(out_mask.shape[0], -1)

    @torch.no_grad()
    def _costs(self, outputs, tg, points, out, fused=True):
        """cost matrices of one prediction set into out [B, Q, Tmax] (points: the B draws rand(1, P, 2))"""
        logits, pm = outputs["pred_logits"], outputs["pred_masks"]
        if fused and self.use_fused and _fused_ok(pm, logits, tg, self.num_points):
            prob = logits.float().softmax(-1).contiguous()
            lib.mask_cost(pm.contiguous(), prob, tg.labels(), tg.bytes(), torch.cat(points, 0), tg.counts,
                          self.cost_class, self.cost_mask, self.cost_dice, out=out)
            return
        for b, T in enumerate(tg.counts):
            out[b, :, :T] = self._cost_composed(outputs, tg.targets, b, points[b])

    def _draw(self, B, device):
        return [torch.rand(1, self.num_points, 2, device=device) for _ in range(B)]

    @torch.no_grad()
    def forward(self, outputs, targets):
        """-> [(index_i, index_j)] per image, int64 CPU tensors, len = min(num_queries, num_targets)"""
        tg = _Targets(targets)
        B, Q = outputs["pred_logits"].shape[:2]
        pm = outputs["pred_masks"]
        C = torch.empty(1, B, Q, tg.Tmax, dtype=torch.float32, device=pm.device)
        self._costs(outputs, tg, self._draw(B, pm.device), C[0])
        return _assign(C, tg.counts)[0]

    memory_efficient_forward = forward

    def __repr__(self, _repr_indent=4):
        head = "Matcher " + self.__class__.__name__
        body = ["cost_class: {}".format(self.cost_class), "cost_mask: {}".format(self.cost_mask),
                "cost_dice: {}".format(self.cost_dice)]
        return "\n".join([head] + [" " * _repr_indent + line for line in body])


class MaskLossFunction(Function):
    """(loss_mask, loss_dice) as one [2] float32 tensor, from odise_mask_loss_forward_*: pred [B, Q, H, W] (CUDA,
    float32 / float16 / bfloat16), target masks [sum T, Hg, Wg] uint8, pairs [N, 3] int64 (image, query, target row),
    pair_of [B*Q] int64, candidates [N, S, 2] and random points [N, P - k, 2].  Only the P loss points of each pair are
    saved for the backward, not the candidates.  The gradient of pred has pred's dtype, is zero on unmatched queries and
    is bit-reproducible."""

    @staticmethod
    def forward(ctx, pred, tgt, pairs, pair_of, cand, rnd, num_masks, num_points, k):
        losses, state = lib.mask_loss_forward(pred, tgt, pairs, cand, rnd, num_masks, num_points, k)
        ctx.save_for_backward(pred, tgt, pairs, pair_of, state)
        ctx.args = (num_masks, num_points)
        return losses

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_losses):
        pred, tgt, pairs, pair_of, state = ctx.saved_tensors
        num_masks, num_points = ctx.args
        grad = lib.mask_loss_backward(pred, tgt, pairs, pair_of, state, grad_losses.float().contiguous(), num_masks,
                                      num_points)
        return grad, None, None, None, None, None, None, None, None


class SetCriterion(nn.Module):
    """Mask2Former's SetCriterion: Hungarian matching, then the weighted class cross entropy ("labels") and the
    point-sampled sigmoid CE and dice mask losses ("masks") of every prediction set.  See the module docstring for the
    batched matching, the random-number contract and the fused path; use_fused = False forces the composed path."""

    def __init__(self, num_classes, matcher, class_weight, mask_weight, dice_weight, num_layers, eos_coef, losses,
                 num_points, oversample_ratio, importance_sample_ratio):
        super().__init__()
        self.num_classes = num_classes
        self.matcher = matcher
        weight_dict = {"loss_ce": class_weight, "loss_mask": mask_weight, "loss_dice": dice_weight}
        aux_weight_dict = {}
        for i in range(num_layers):
            aux_weight_dict.update({k + f"_{i}": v for k, v in weight_dict.items()})
        weight_dict.update(aux_weight_dict)
        self.weight_dict = weight_dict
        self.eos_coef = eos_coef
        self.losses = losses
        empty_weight = torch.ones(self.num_classes + 1)
        empty_weight[-1] = self.eos_coef
        self.register_buffer("empty_weight", empty_weight)
        self.num_points = num_points
        self.oversample_ratio = oversample_ratio
        self.importance_sample_ratio = importance_sample_ratio
        self.use_fused = True
        # match on the device (lib.mask_assign) when every set is fused: no synchronisation, and invalid costs are
        # reported in match_status [L, B] (1: NaN or -inf, 2: infeasible) instead of raising ValueError; match_status is
        # None after a forward that matched with scipy
        self.match_on_device = False
        self.match_status = None

    # ---- the composed path (the reference's algorithm; CPU indices) ----

    def loss_labels(self, outputs, targets, indices, num_masks):
        src_logits = outputs["pred_logits"].float()
        idx = self._get_src_permutation_idx(indices)
        target_classes_o = torch.cat([t["labels"][J] for t, (_, J) in zip(targets, indices)])
        target_classes = torch.full(src_logits.shape[:2], self.num_classes, dtype=torch.int64,
                                    device=src_logits.device)
        target_classes[idx] = target_classes_o
        return {"loss_ce": F.cross_entropy(src_logits.transpose(1, 2), target_classes, self.empty_weight)}

    def loss_masks(self, outputs, targets, indices, num_masks, points=None):
        """points: the (candidates, random points) draws for this call; None draws them here, as the reference does"""
        src_idx = self._get_src_permutation_idx(indices)
        tgt_idx = self._get_tgt_permutation_idx(indices)
        src_masks = outputs["pred_masks"][src_idx]
        masks = [t["masks"] for t in targets]
        # the targets padded to the batch's largest [T, H, W], as nested_tensor_from_tensor_list does
        size = [max(s) for s in zip(*[m.shape for m in masks])]
        padded = torch.zeros([len(masks)] + size, dtype=masks[0].dtype, device=masks[0].device)
        for m, p in zip(masks, padded):
            p[: m.shape[0], : m.shape[1], : m.shape[2]].copy_(m)
        target_masks = padded.to(src_masks)[tgt_idx]
        src_masks, target_masks = src_masks[:, None], target_masks[:, None]
        S, k = _point_counts(self.num_points, self.oversample_ratio, self.importance_sample_ratio)
        if points is None:
            points = self._draw_loss(src_masks.shape[0], src_masks.device)
        with torch.no_grad():
            point_coords = _uncertain_points(src_masks, points[0], points[1], k)
            point_labels = point_sample(target_masks, point_coords, align_corners=False).squeeze(1)
        point_logits = point_sample(src_masks, point_coords, align_corners=False).squeeze(1)
        return {"loss_mask": _sigmoid_ce_loss(point_logits, point_labels, num_masks),
                "loss_dice": _dice_loss(point_logits, point_labels, num_masks)}

    def _draw_loss(self, N, device):
        S, k = _point_counts(self.num_points, self.oversample_ratio, self.importance_sample_ratio)
        cand = torch.rand(N, S, 2, device=device)
        rnd = torch.rand(N, self.num_points - k, 2, device=device) if self.num_points - k > 0 else None
        return cand, rnd

    def _get_src_permutation_idx(self, indices):
        batch_idx = torch.cat([torch.full_like(src, i) for i, (src, _) in enumerate(indices)])
        src_idx = torch.cat([src for (src, _) in indices])
        return batch_idx, src_idx

    def _get_tgt_permutation_idx(self, indices):
        batch_idx = torch.cat([torch.full_like(tgt, i) for i, (_, tgt) in enumerate(indices)])
        tgt_idx = torch.cat([tgt for (_, tgt) in indices])
        return batch_idx, tgt_idx

    def get_loss(self, loss, outputs, targets, indices, num_masks):
        loss_map = {"labels": self.loss_labels, "masks": self.loss_masks}
        assert loss in loss_map, f"do you really want to compute {loss} loss?"
        return loss_map[loss](outputs, targets, indices, num_masks)

    # ---- the fused path (device pair tables; no CPU index reaches the device) ----

    def _labels_fused(self, outputs, tg, tab):
        src_logits = outputs["pred_logits"].float()
        B, Q, K1 = src_logits.shape
        if sum(tg.counts) == 0:
            tc = torch.full((B * Q,), self.num_classes, dtype=torch.int64, device=src_logits.device)
        else:
            lab = torch.index_select(tg.labels(), 0, tab["tg_of"].clamp(min=0))
            tc = torch.where(tab["tg_of"] >= 0, lab, self.num_classes)
        # the same weighted mean as the [B, K1, Q] form; the 2-D nll_loss has a deterministic CUDA forward
        return {"loss_ce": F.cross_entropy(src_logits.reshape(B * Q, K1), tc, self.empty_weight)}

    def _masks_fused(self, outputs, tg, tab, num_masks, points):
        S, k = _point_counts(self.num_points, self.oversample_ratio, self.importance_sample_ratio)
        cand, rnd = points()
        if rnd is None:
            rnd = cand.new_empty(cand.shape[0], 0, 2)
        # a num_masks device tensor divides the sums outside the op, which takes num_masks as a host float
        on_device = torch.is_tensor(num_masks)
        losses = MaskLossFunction.apply(outputs["pred_masks"].contiguous(), tg.bytes(), tab["pairs"], tab["pair_of"],
                                        cand, rnd, 1.0 if on_device else num_masks, self.num_points, k)
        if on_device:
            losses = losses / num_masks
        return {"loss_mask": losses[0], "loss_dice": losses[1]}

    @staticmethod
    def _tables(indices_sets, counts, Q, device):
        """per set: pairs [N, 3] (image, query, global target), pair_of and tg_of [B*Q] (pair / global target of each
        query, -1 if unmatched), all sent in one non-blocking copy from pinned memory"""
        B = len(counts)
        offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        parts, shapes = [], []
        for indices in indices_sets:
            pair_of = np.full(B * Q, -1, dtype=np.int64)
            tg_of = np.full(B * Q, -1, dtype=np.int64)
            pairs, n = [], 0
            for b, (i, j) in enumerate(indices):
                i, j = i.numpy(), j.numpy()
                rows = b * Q + i
                pair_of[rows] = n + np.arange(len(i))
                tg_of[rows] = offs[b] + j
                pairs.append(np.stack([np.full(len(i), b), i, offs[b] + j], 1).astype(np.int64).reshape(-1, 3))
                n += len(i)
            pairs = np.concatenate(pairs) if pairs else np.zeros((0, 3), np.int64)
            parts += [pairs.reshape(-1), pair_of, tg_of]
            shapes.append(n)
        host = torch.from_numpy(np.concatenate(parts) if parts else np.zeros(0, np.int64))
        return SetCriterion._split_tables(host.pin_memory().to(device, non_blocking=True), shapes, B, Q)

    @staticmethod
    def _split_tables(buf, shapes, B, Q):
        """the per-set views of one int64 table buffer laid out as _tables and lib.mask_assign write it: per set (n
        pairs) pairs [n, 3], then pair_of [B*Q], then tg_of [B*Q]"""
        out, o = [], 0
        for n in shapes:
            tab = {"pairs": buf[o:o + 3 * n].view(n, 3)}
            o += 3 * n
            tab["pair_of"] = buf[o:o + B * Q]
            tab["tg_of"] = buf[o + B * Q:o + 2 * B * Q]
            o += 2 * B * Q
            out.append(tab)
        return out

    # ---- forward ----

    def _num_masks(self, targets, device, keep_on_device=False):
        """the reference's num_masks as a float; keep_on_device: under torch.distributed, the all-reduced [1] device
        tensor itself, without the .item() synchronisation"""
        n = sum(len(t["labels"]) for t in targets)
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            num_masks = torch.as_tensor([n], dtype=torch.float)
            num_masks = num_masks.pin_memory().to(device, non_blocking=True) if device.type == "cuda" else \
                num_masks.to(device)
            torch.distributed.all_reduce(num_masks)
            num_masks = torch.clamp(num_masks / torch.distributed.get_world_size(), min=1)
            return num_masks if keep_on_device else num_masks.item()
        return torch.clamp(torch.as_tensor([n], dtype=torch.float), min=1).item()

    def forward(self, outputs, targets):
        outputs_without_aux = {k: v for k, v in outputs.items() if k != "aux_outputs"}
        sets = [outputs_without_aux] + list(outputs.get("aux_outputs", []))
        names = [""] + [f"_{i}" for i in range(len(sets) - 1)]
        device = next(iter(outputs.values())).device
        if not isinstance(self.matcher, HungarianMatcher):
            losses, num_masks = {}, None
            for out, sfx in zip(sets, names):
                indices = self.matcher(out, targets)
                if num_masks is None:
                    num_masks = self._num_masks(targets, device)
                for loss in self.losses:
                    losses.update({k + sfx: v for k, v in self.get_loss(loss, out, targets, indices,
                                                                         num_masks).items()})
            return losses
        return self._forward_batched(sets, names, targets, device)

    def _forward_batched(self, sets, names, targets, device):
        m, tg = self.matcher, _Targets(targets)
        for loss in self.losses:
            assert loss in ("labels", "masks"), f"do you really want to compute {loss} loss?"
        B, Q = sets[0]["pred_logits"].shape[:2]
        N = sum(min(Q, T) for T in tg.counts)
        masks = "masks" in self.losses
        S, k = _point_counts(self.num_points, self.oversample_ratio, self.importance_sample_ratio) if masks else (0, 0)
        fused = [self.use_fused and _fused_ok(out["pred_masks"], out["pred_logits"], tg, self.num_points if masks
                                              else 1, S if masks else 1, k) for out in sets]
        # every torch.rand call of the reference, in its order: per set, the matcher's per-image points, then the
        # loss's.  A fused set keeps the generator state before its loss draws instead of the draws (N x S x 2 floats
        # per set) and draws them again when its loss runs.
        draws = []
        for l, out in enumerate(sets):
            dev = out["pred_masks"].device
            mp = m._draw(B, dev)
            if not masks:
                draws.append((mp, None))
            elif fused[l]:
                state = torch.cuda.get_rng_state(dev)
                self._draw_loss(N, dev)
                draws.append((mp, state))
            else:
                draws.append((mp, self._draw_loss(N, dev)))
        rng_end = torch.cuda.get_rng_state(device) if any(fused) and masks else None
        on_device = self.match_on_device and all(fused) and max(Q, tg.Tmax) <= lib.MASK_MAX_ASSIGN
        num_masks = self._num_masks(targets, device, keep_on_device=on_device)
        C = torch.empty(len(sets), B, Q, tg.Tmax, dtype=torch.float32, device=sets[0]["pred_masks"].device)
        for l, out in enumerate(sets):
            m._costs(out, tg, draws[l][0], C[l], fused=self.use_fused)
        if on_device:
            buf, self.match_status = lib.mask_assign(C, tg.counts)
            indices, tabs = None, dict(enumerate(self._split_tables(buf, [N] * len(sets), B, Q)))
        else:
            indices, tabs, self.match_status = _assign(C, tg.counts), {}, None
            if any(fused):
                sel = [l for l, f in enumerate(fused) if f]
                tabs = dict(zip(sel, self._tables([indices[l] for l in sel], tg.counts, Q,
                                                  sets[0]["pred_masks"].device)))
        losses = {}
        for l, (out, sfx) in enumerate(zip(sets, names)):
            for loss in self.losses:
                if loss == "labels":
                    d = self._labels_fused(out, tg, tabs[l]) if fused[l] else \
                        self.loss_labels(out, targets, indices[l], num_masks)
                elif fused[l]:
                    dev = out["pred_masks"].device

                    def redraw(state=draws[l][1], dev=dev):
                        torch.cuda.set_rng_state(state, dev)
                        return self._draw_loss(N, dev)
                    d = self._masks_fused(out, tg, tabs[l], num_masks, redraw)
                else:
                    d = self.loss_masks(out, targets, indices[l], num_masks, points=draws[l][1])
                losses.update({k_ + sfx: v for k_, v in d.items()})
        if rng_end is not None:
            torch.cuda.set_rng_state(rng_end, device)
        return losses

    def __repr__(self):
        head = "Criterion " + self.__class__.__name__
        body = [
            "matcher: {}".format(self.matcher.__repr__(_repr_indent=8)),
            "losses: {}".format(self.losses),
            "weight_dict: {}".format(self.weight_dict),
            "num_classes: {}".format(self.num_classes),
            "eos_coef: {}".format(self.eos_coef),
            "num_points: {}".format(self.num_points),
            "oversample_ratio: {}".format(self.oversample_ratio),
            "importance_sample_ratio: {}".format(self.importance_sample_ratio),
        ]
        return "\n".join([head] + [" " * 4 + line for line in body])
