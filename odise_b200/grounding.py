"""Training drop-in for ODISE(caption)'s grounding loss: MaskGroundingCriterion (odise/modeling/meta_arch/odise.py:779-907)
with its collect modes "diff", "concat" and None.

    model.criterion.grounding_criterion = L(MaskGroundingCriterion)(collect_mode="diff", loss_weight=...)

with `from odise_b200.grounding import MaskGroundingCriterion` in the LazyConfig.  forward(outputs, targets) returns the
reference's dict: loss_mask_word for the final prediction set and loss_mask_word_{i} for outputs["aux_outputs"][i], all
`unbind` views of one [S] tensor of the S sets' losses.

All S sets run together.  Across W > 1 ranks (torch.distributed initialised and collect_mode not None) the batch sizes
are exchanged once per step (the step's one host read) and every set's masks, the words and the valid mask travel in
one padded all_gather (GatherFunction).  In "diff" mode its backward is one all_reduce of the packed gradient, of which
each rank keeps its own slot: the gradient of the sum of all ranks' losses, as diffdist's all_gather gives.  In
"concat" mode the gathered rows carry no gradient.  On one rank nothing is gathered and nothing is read on the host.

The losses come from GroundingFunction, three sm_90a kernels forward and three backward (grounding.cu), when the
tensors are on CUDA, the masks and words are float32 with autocast off or the masks are in the 16-bit autocast dtype
(the words in it or in float32), the shapes are within the kernels' limits (lib.GROUNDING_*), every set shares one
word_embed tensor and use_fused is True.  Every other input (CPU, float64, use_fused = False) runs the reference's
get_loss ops verbatim, set by set, on slices of the same gathered tensors, including its host-side isfinite fallback.
The kernels take the fallback on the device, round in 16 bits where autocast rounds, and sum every gradient in a fixed
order without atomics, so the fused path makes no host synchronisation and is bit-reproducible."""
import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib

# The kernels as torch custom ops (lib.custom_op).  lib's functions are looked up at call time, so that a test that
# patches them sees every call.
lib.custom_op("grounding(Tensor mask_embed, Tensor word_embed, Tensor word_valid, Tensor logit_scale, int batch, "
              "int offset, float loss_weight) -> (Tensor, Tensor)", lambda *args: lib.grounding_forward(*args))
lib.custom_op("grounding_backward(Tensor mask_embed, Tensor word_embed, Tensor logit_scale, Tensor state, "
              "Tensor grad_losses, int batch, int offset) -> (Tensor, Tensor, Tensor, Tensor, Tensor)",
              lambda *args: lib.grounding_backward(*args))


class GroundingFunction(Function):
    """losses float32 [S] of lib.grounding_forward.  mask_local [S, B, Q, C] and word_local [B, K, C] are this rank's
    rows, mask_global [S, G, Q, C], word_global [G, K, C] and valid_global bool [G, K] the gathered ones, which hold the
    local rows at offset .. offset + B - 1; logit_scale float32 [S].  The kernels read the gathered tensors only; the
    gradients of the uses of the local rows go to mask_local and word_local, those of the gathered rows to mask_global
    and word_global (on one rank the same tensors, whose two gradients autograd adds)."""

    @staticmethod
    def forward(ctx, mask_local, mask_global, word_local, word_global, valid_global, logit_scale, offset, loss_weight):
        batch = mask_local.shape[1]
        losses, state = torch.ops.odise_b200.grounding(mask_global, word_global, valid_global, logit_scale, batch,
                                                       offset, loss_weight)
        ctx.save_for_backward(mask_global, word_global, logit_scale, state)
        ctx.batch, ctx.offset = batch, offset
        return losses

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_losses):
        mask_global, word_global, logit_scale, state = ctx.saved_tensors
        gml, gmg, gwl, gwg, gs = torch.ops.odise_b200.grounding_backward(
            mask_global, word_global, logit_scale, state, grad_losses.float().contiguous(), ctx.batch, ctx.offset)
        return gml, gmg, gwl, gwg, None, gs, None, None


def _world():
    """(world size, rank) of torch.distributed, (1, 0) when it is not initialised"""
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def world_batch_sizes(batch, device):
    """every rank's batch size as Python ints: one all_gather and the step's one host read"""
    mine = torch.full((1,), batch, dtype=torch.long, device=device)
    sizes = [torch.empty_like(mine) for _ in range(dist.get_world_size())]
    dist.all_gather(sizes, mine)
    return torch.cat(sizes).tolist()


class GatherFunction(Function):
    """(mask_global [S, G, Q, C], word_global [G, K, C], valid_global bool [G, K]) of every rank's mask_local
    [S, B_r, Q, C], word_local [B_r, K, C] and valid_local [B_r, K] in rank order, for the ranks' batch sizes `sizes`:
    one all_gather of a buffer padded to the largest batch, in the wider of the two float dtypes.  Backward ("diff"):
    one all_reduce of the packed gradient, this rank's slot of which is the gradient of its inputs."""

    @staticmethod
    def forward(ctx, mask_local, word_local, valid_local, sizes, rank):
        S, B, Q, C = mask_local.shape
        K = word_local.shape[1]
        dt = torch.promote_types(mask_local.dtype, word_local.dtype)
        nm, nw = S * Q * C, K * C
        buf = mask_local.new_zeros(max(sizes), nm + nw + K, dtype=dt)
        buf[:B, :nm] = mask_local.transpose(0, 1).reshape(B, nm)
        buf[:B, nm:nm + nw] = word_local.reshape(B, nw)
        buf[:B, nm + nw:] = valid_local
        parts = [torch.empty_like(buf) for _ in sizes]
        dist.all_gather(parts, buf)
        rows = torch.cat([p[:n] for p, n in zip(parts, sizes)])
        G = rows.shape[0]
        mask_global = rows[:, :nm].reshape(G, S, Q, C).transpose(0, 1).to(mask_local.dtype).contiguous()
        word_global = rows[:, nm:nm + nw].reshape(G, K, C).to(word_local.dtype).contiguous()
        valid_global = rows[:, nm + nw:] != 0
        ctx.mark_non_differentiable(valid_global)
        ctx.sizes, ctx.rank, ctx.dtypes, ctx.dt = sizes, rank, (mask_local.dtype, word_local.dtype), dt
        return mask_global, word_global, valid_global

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_mask, grad_word, _grad_valid):
        sizes, rank, dt = ctx.sizes, ctx.rank, ctx.dt
        S, G, Q, C = grad_mask.shape if grad_mask is not None else (None,) * 4
        if grad_mask is None or grad_word is None:
            raise RuntimeError("GatherFunction: both gathered tensors need a gradient")
        K = grad_word.shape[1]
        nm, nw = S * Q * C, K * C
        buf = grad_mask.new_zeros(len(sizes), max(sizes), nm + nw, dtype=dt)
        r0 = 0
        for r, n in enumerate(sizes):
            buf[r, :n, :nm] = grad_mask[:, r0:r0 + n].transpose(0, 1).reshape(n, nm)
            buf[r, :n, nm:] = grad_word[r0:r0 + n].reshape(n, nw)
            r0 += n
        dist.all_reduce(buf)
        B = sizes[rank]
        own = buf[rank, :B]
        gm = own[:, :nm].reshape(B, S, Q, C).transpose(0, 1).to(ctx.dtypes[0]).contiguous()
        gw = own[:, nm:].reshape(B, K, C).to(ctx.dtypes[1])
        return gm, gw, None, None, None


def _fused_ok(mask_local, mask_global, word_local, valid, logit_scale):
    """whether the inputs take GroundingFunction"""
    if not all(t.is_cuda for t in (mask_local, word_local, valid, logit_scale)):
        return False
    if logit_scale.dtype != torch.float32 or valid.dtype != torch.bool:
        return False
    if torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
        if dt not in (torch.float16, torch.bfloat16) or mask_local.dtype != dt \
                or word_local.dtype not in (dt, torch.float32):
            return False
    elif not mask_local.dtype == word_local.dtype == torch.float32:
        return False
    S, B, Q, C = mask_local.shape
    return lib.grounding_supported(S, mask_global.shape[1], B, Q, word_local.shape[1], C)


def composed_loss(mask_local, mask_global, word_local, word_global, valid_global, logit_scale, offset, loss_weight,
                  local_in_global=True):
    """MaskGroundingCriterion.get_loss's ops in its order for one set, on the gathered rows.  With local_in_global the
    local rows are the gathered rows offset .. offset + B - 1 after the normalisation (one rank, or "diff": the
    gradient of the local uses reaches the inputs through the gather); otherwise ("concat": the gathered rows carry no
    gradient) the local inputs are normalised themselves."""
    batch_size, num_queries, embed_dim = mask_local.shape
    num_words = word_local.shape[1]
    global_batch_size = mask_global.shape[0]
    global_mask = F.normalize(mask_global, dim=-1)
    global_word = F.normalize(word_global, dim=-1)
    if local_in_global:
        mask_embed = global_mask[offset:offset + batch_size]
        word_embed = global_word[offset:offset + batch_size]
    else:
        mask_embed = F.normalize(mask_local, dim=-1)
        word_embed = F.normalize(word_local, dim=-1)
    mask_embed = mask_embed.reshape(batch_size * num_queries, embed_dim)
    word_embed = word_embed.reshape(batch_size * num_words, embed_dim)
    global_mask = global_mask.reshape(global_batch_size * num_queries, embed_dim)
    global_word = global_word.reshape(global_batch_size * num_words, embed_dim)

    sim_global_mask_word = global_mask @ word_embed.t() * logit_scale
    sim_global_mask_word = sim_global_mask_word.view(global_batch_size, num_queries, batch_size, num_words)
    sim_global_img_txt = (sim_global_mask_word.softmax(dim=1) * sim_global_mask_word).sum(dim=1).mean(dim=-1)

    sim_mask_global_word = mask_embed @ global_word.t() * logit_scale
    sim_mask_global_word = sim_mask_global_word.view(batch_size, num_queries, global_batch_size, num_words)
    sim_img_global_txt = (sim_mask_global_word.softmax(dim=1) * sim_mask_global_word).sum(dim=1).mean(dim=-1)

    labels = torch.arange(batch_size, dtype=torch.long, device=mask_local.device) + offset
    valid_mask = valid_global[offset:offset + batch_size].any(dim=-1)
    global_valid_mask = valid_global.any(dim=-1)

    loss_global_img_txt = F.cross_entropy(sim_global_img_txt.t(), labels, reduction="none")
    loss_global_img_txt = (loss_global_img_txt * valid_mask).mean()
    # .float() in the reference, which cross_entropy refuses for float64 scores
    loss_img_global_txt = F.cross_entropy(sim_img_global_txt, labels, weight=global_valid_mask.to(sim_img_global_txt.dtype))
    if not torch.isfinite(loss_img_global_txt).all():
        loss_img_global_txt = F.cross_entropy(sim_img_global_txt, labels)
    loss = 0.5 * (loss_global_img_txt + loss_img_global_txt)
    return loss * loss_weight


def grounding_losses(mask_local, mask_global, word_local, word_global, valid_global, logit_scale, offset,
                     loss_weight=1.0, *, local_in_global=True, use_fused=True):
    """losses [S] of S prediction sets from this rank's mask_local [S, B, Q, C] and word_local [B, K, C], the gathered
    mask_global [S, G, Q, C], word_global [G, K, C] and valid_global bool [G, K] (the local rows at offset ..
    offset + B - 1; on one rank the local tensors themselves) and logit_scale [S].  local_in_global = False when the
    gathered rows carry no gradient ("concat").  GroundingFunction where _fused_ok, composed_loss per set otherwise."""
    if use_fused and _fused_ok(mask_local, mask_global, word_local, valid_global, logit_scale):
        if not local_in_global:
            mask_global, word_global = mask_global.detach(), word_global.detach()
        return GroundingFunction.apply(mask_local.contiguous(), mask_global.contiguous(), word_local.contiguous(),
                                       word_global.contiguous(), valid_global.contiguous(), logit_scale, offset,
                                       float(loss_weight))
    return torch.stack([composed_loss(mask_local[s], mask_global[s], word_local, word_global, valid_global,
                                      logit_scale[s], offset, loss_weight, local_in_global)
                        for s in range(mask_local.shape[0])])


class MaskGroundingCriterion(nn.Module):
    """MaskGroundingCriterion(collect_mode="concat", loss_weight=1.0): the reference's constructor and losses, all
    prediction sets of a step at once; use_fused = False forces the reference's ops (for comparisons)."""

    def __init__(self, collect_mode="concat", loss_weight=1.0, *, use_fused=True):
        super().__init__()
        if collect_mode not in ("diff", "concat", None):
            raise ValueError(f"collect_mode {collect_mode} is not supported")
        self.collect_mode = collect_mode
        self.loss_weight = loss_weight
        self.use_fused = use_fused

    def extra_repr(self) -> str:
        return f"collect_mode={self.collect_mode}, \n" f"loss_weight={self.loss_weight} \n"

    def forward(self, outputs, targets):
        sets = [outputs] + list(outputs.get("aux_outputs", []))
        words = outputs["word_embed"]
        if any(s["word_embed"] is not words for s in sets[1:]):     # not the reference model's layout: set by set
            losses = torch.cat([self._losses([s], s["word_embed"], targets) for s in sets])
        else:
            losses = self._losses(sets, words, targets)
        losses = losses.unbind(0)
        out = {"loss_mask_word": losses[0]}
        out.update({f"loss_mask_word_{i}": l for i, l in enumerate(losses[1:])})
        return out

    def _losses(self, sets, words, targets):
        masks = torch.stack([s["mask_embed"] for s in sets])
        scales = torch.stack([s["logit_scale"] for s in sets])
        valid = torch.stack([t["word_valid_mask"] for t in targets], dim=0)
        world, rank = _world()
        if self.collect_mode is None or world == 1:
            return grounding_losses(masks, masks, words, words, valid, scales, 0, self.loss_weight,
                                    use_fused=self.use_fused)
        sizes = world_batch_sizes(masks.shape[1], masks.device)
        offset = sum(sizes[:rank])
        if self.collect_mode == "diff":
            mg, wg, vg = GatherFunction.apply(masks, words, valid, sizes, rank)
        else:
            with torch.no_grad():
                mg, wg, vg = GatherFunction.apply(masks, words, valid, sizes, rank)
        return grounding_losses(masks, mg, words, wg, vg, scales, offset, self.loss_weight,
                                local_in_global=self.collect_mode == "diff", use_fused=self.use_fused)
