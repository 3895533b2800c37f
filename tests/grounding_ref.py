"""The grounding-loss oracle shared by the CPU and GPU tests: the reference's own MaskGroundingCriterion.get_loss run
rank by rank in one process.  For W > 1 emulated ranks comm.get_rank / get_world_size, get_world_batch_sizes and the
criterion's collect_func are patched: collect_func returns the torch.cat of every rank's tensor with the live local
one in its slot ("diff"), or the same without gradient ("concat").  Autograd of the sum of all ranks' losses then
gives each rank's "diff" gradients without collectives."""
from contextlib import contextmanager

import torch
import torch.nn.functional as F

from oracle import refshim


def inputs(sizes, S, Q, K, C, dtype=torch.float64, device="cpu", seed=0, valid=None):
    """per rank (masks [S, B_r, Q, C], words [B_r, K, C], valid bool [B_r, K]) and per set scales [S], from a seed;
    valid: None (a seeded pattern, every image with a valid word), or a bool [G, K] to use"""
    g = torch.Generator().manual_seed(seed)
    G = sum(sizes)
    m = torch.randn(S, G, Q, C, generator=g, dtype=torch.float64)
    w = torch.randn(G, K, C, generator=g, dtype=torch.float64)
    if valid is None:
        valid = torch.rand(G, K, generator=g) < 0.7
        valid[:, 0] = True
    scales = 10.0 + 5.0 * torch.rand(S, generator=g, dtype=torch.float64)
    out, r0 = [], 0
    for n in sizes:
        out.append((m[:, r0:r0 + n].to(device, dtype), w[r0:r0 + n].to(device, dtype), valid[r0:r0 + n].to(device)))
        r0 += n
    return out, scales.to(device, dtype if dtype == torch.float64 else torch.float32)


class _ValidMask(torch.Tensor):
    """the gathered valid mask, whose .float() (the reference's class weight of the cross entropy) is float64: the
    reference's float32 weight is refused by cross_entropy for float64 scores"""

    def float(self):
        return torch.Tensor.double(self).as_subclass(torch.Tensor)


@contextmanager
def _emulated(od, crit, rank, sizes, collect):
    saved = od.comm.get_rank, od.comm.get_world_size, od.get_world_batch_sizes
    od.comm.get_rank = lambda: rank
    od.comm.get_world_size = lambda: len(sizes)
    od.get_world_batch_sizes = lambda b, device: torch.tensor(sizes, dtype=torch.long, device=device)
    crit.collect_func = collect
    try:
        yield
    finally:
        od.comm.get_rank, od.comm.get_world_size, od.get_world_batch_sizes = saved


def reference_losses(ranks, scales, mode, loss_weight=1.0):
    """losses [W][S] of the reference criterion at every emulated rank for leaves `ranks` [(masks [S, B, Q, C], words,
    valid)] and scales [W][S] (each rank's own scale leaves); mode "diff", "concat" or None (W = 1 only)."""
    od = refshim.modules().odise_module
    crit = od.MaskGroundingCriterion(collect_mode=mode, loss_weight=loss_weight)
    sizes = [m.shape[1] for m, _, _ in ranks]
    S = ranks[0][0].shape[0]
    out = []
    for r, (m, w, v) in enumerate(ranks):
        targets = [{"word_valid_mask": v[b]} for b in range(v.shape[0])]
        losses = []
        for s in range(S):
            def collect(x, s=s, r=r):
                if x.dtype == torch.bool:
                    parts = [vv.any(dim=-1) for _, _, vv in ranks]
                    parts[r] = x
                    return torch.cat(parts).as_subclass(_ValidMask)
                if len(sizes) == 1:
                    return x
                elif x.shape[0] == sizes[r] * m.shape[2]:
                    parts = [F.normalize(mm[s], dim=-1).reshape(-1, x.shape[1]) for mm, _, _ in ranks]
                else:
                    parts = [F.normalize(ww, dim=-1).reshape(-1, x.shape[1]) for _, ww, _ in ranks]
                parts[r] = x
                y = torch.cat(parts)
                return y if mode == "diff" else y.detach()
            with _emulated(od, crit, r, sizes, collect):
                outputs = {"mask_embed": m[s], "word_embed": w, "logit_scale": scales[r][s]}
                losses.append(crit.get_loss(outputs, targets)["loss_mask_word"])
        out.append(losses)
    return out
