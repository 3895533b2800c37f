"""Training drop-in for ODISE's category scoring: CategoryODISE.cal_pred_logits (odise/modeling/meta_arch/odise.py:181-207)
with ensemble_logits_with_labels(..., "max") (helper.py:79-109).

    from odise_b200.category import cal_pred_logits

    class FusedCategoryODISE(CategoryODISE):
        def cal_pred_logits(self, outputs):
            return cal_pred_logits(outputs)

cal_pred_logits(outputs) reads mask_embed [B, Q, C], text_embed [K', C], null_embed [1, C], labels (K lists of synonym
prompts, K' in all) and logit_scale from the outputs dict and returns pred_logits [B, Q, K + 1]: per class the max over
its prompts of logit_scale * cos(mask_embed, prompt), and the null column.  It runs CategoryLogitsFunction, one sm_90a
kernel forward and three backward (category_logits.cu), when the tensors are on CUDA, the product would be float32
(autocast off, float32 inputs) or 16 bits under torch.autocast (mask_embed in the autocast dtype, the bank in it or in
float32), the shapes are within the kernels' limits (lib.CATEGORY_*) and use_fused is True.  Every other input (CPU,
float64, a 16-bit module without autocast, use_fused = False) runs the reference's ops verbatim: the zeros tensor, the
per-class slice / max / assignment loop and the cat.

The kernels round in 16 bits where autocast rounds (the normalised operands, the matmul output and logit_scale before
the multiply), the lowest prompt index wins among equal stored values as in torch's max(dim), and the backward routes
each gradient to the prompt the forward chose, with fixed-order sums and no atomics: every gradient is
bit-reproducible.  The class offsets come from labels as Python ints and are written on the device by fill kernels
(a copy from pageable memory would synchronise), cached per (group sizes, device) outside any state dict, so forward
and backward make no host synchronisation and can be captured in a CUDA graph or traced by
torch.compile(fullgraph=True)."""
import torch
import torch.nn.functional as F
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib

# The kernels as torch custom ops (lib.custom_op).  lib's functions are looked up at call time, so that a test that
# patches them sees every call.
lib.custom_op("category_logits(Tensor mask_embed, Tensor text_embed, Tensor null_embed, Tensor logit_scale, "
              "Tensor group_start) -> (Tensor, Tensor, Tensor)", lambda *args: lib.category_logits_forward(*args))
lib.custom_op("category_logits_backward(Tensor mask_embed, Tensor text_embed, Tensor null_embed, Tensor logit_scale, "
              "Tensor group_start, Tensor winners, Tensor norms, Tensor grad_logits) -> (Tensor, Tensor, Tensor, Tensor)",
              lambda *args: lib.category_logits_backward(*args))


class CategoryLogitsFunction(Function):
    """(logits, winners, norms) of lib.category_logits_forward for contiguous CUDA mask_embed [B, Q, C], text_embed
    [K', C], null_embed [1, C], the float32 scalar logit_scale and the device table group_start [K + 1]; winners and
    norms are saved for the backward and not differentiable.  Gradients come back in each input's dtype."""

    @staticmethod
    def forward(ctx, mask_embed, text_embed, null_embed, logit_scale, group_start):
        out, win, norms = torch.ops.odise_b200.category_logits(mask_embed, text_embed, null_embed, logit_scale,
                                                               group_start)
        ctx.save_for_backward(mask_embed, text_embed, null_embed, logit_scale, group_start, win, norms)
        ctx.mark_non_differentiable(win, norms)
        ctx.set_materialize_grads(False)     # no zero-filled gradients for winners and norms: two launches per call
        return out, win, norms

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_logits, _grad_win, _grad_norms):
        mask_embed, text_embed, null_embed, logit_scale, group_start, win, norms = ctx.saved_tensors
        if grad_logits is None:
            grad_logits = mask_embed.new_zeros(win.shape)
        grad_logits = grad_logits.to(mask_embed.dtype).contiguous()
        gm, gt, gn, gs = torch.ops.odise_b200.category_logits_backward(mask_embed, text_embed, null_embed,
                                                                       logit_scale, group_start, win, norms,
                                                                       grad_logits)
        return gm, gt, gn, gs, None


_GROUPS = {}    # (group sizes, device) -> group_start int32 [K + 1]; not module state


def group_start(sizes, device):
    """The classes' prompt offsets [K + 1] int32 on `device` for their prompt counts, written by fill kernels rather
    than copied from the host; cached in eager mode, built in the graph when traced."""
    def build():
        vals = lib.category_group_start(list(sizes))
        return torch.stack([torch.full((), v, dtype=torch.int32, device=device) for v in vals])

    if torch.compiler.is_compiling():
        return build()
    key = (tuple(sizes), device)
    if key not in _GROUPS:
        _GROUPS[key] = build()
    return _GROUPS[key]


def _fused_ok(mask_embed, text_embed, null_embed, logit_scale, sizes):
    """whether the inputs take CategoryLogitsFunction"""
    ts = (mask_embed, text_embed, null_embed, logit_scale)
    if not all(isinstance(t, torch.Tensor) and t.is_cuda for t in ts):
        return False
    if logit_scale.dtype != torch.float32 or logit_scale.dim() != 0 or text_embed.dtype != null_embed.dtype:
        return False
    if torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
        if dt not in (torch.float16, torch.bfloat16) or mask_embed.dtype != dt \
                or text_embed.dtype not in (dt, torch.float32):
            return False
    elif not mask_embed.dtype == text_embed.dtype == torch.float32:
        return False
    if mask_embed.dim() != 3 or text_embed.dim() != 2 or tuple(null_embed.shape) != (1, text_embed.shape[1]):
        return False
    (B, Q, C), Kp, K = mask_embed.shape, text_embed.shape[0], len(sizes)
    return (C == text_embed.shape[1] and C % lib.CATEGORY_C_MULTIPLE == 0 and 0 < C <= lib.CATEGORY_MAX_C
            and B * Q > 0 and 1 <= K and sum(sizes) == Kp <= lib.CATEGORY_MAX_PROMPTS
            and 1 <= min(sizes) and max(sizes) <= lib.CATEGORY_MAX_GROUP and B * Q * max(K + 1, C) < 2 ** 31)


def ensemble_logits_with_labels(logits, labels, ensemble_method="max"):
    """helper.py:79-109 with its "max" ensemble: per class the max over its synonym columns, assigned into zeros"""
    len_list = [len(l) for l in labels]
    assert logits.shape[-1] == sum(len_list), f"{logits.shape[-1]} != {sum(len_list)}"
    assert ensemble_method == "max", ensemble_method
    ensemble_logits = torch.zeros(*logits.shape[:-1], len(labels), dtype=logits.dtype, device=logits.device)
    for i in range(len(labels)):
        ensemble_logits[..., i] = logits[..., sum(len_list[:i]): sum(len_list[: i + 1])].max(dim=-1).values
    return ensemble_logits


def composed_pred_logits(mask_embed, text_embed, null_embed, labels, logit_scale):
    """CategoryODISE.cal_pred_logits's ops in its order"""
    mask_embed = F.normalize(mask_embed, dim=-1)
    text_embed = F.normalize(text_embed, dim=-1)
    pred = logit_scale * (mask_embed @ text_embed.t())
    pred = ensemble_logits_with_labels(pred, labels, ensemble_method="max")
    null_embed = F.normalize(null_embed, dim=-1)
    null_pred = logit_scale * (mask_embed @ null_embed.t())
    return torch.cat([pred, null_pred], dim=-1)


def cal_pred_logits(outputs, *, use_fused=True):
    """CategoryODISE.cal_pred_logits(outputs) -> pred_logits [B, Q, K + 1]; see the module docstring for when the
    fused kernels run.  use_fused = False forces the reference's ops (for comparisons)."""
    mask_embed, text_embed, null_embed = outputs["mask_embed"], outputs["text_embed"], outputs["null_embed"]
    labels, logit_scale = outputs["labels"], outputs["logit_scale"]
    sizes = [len(l) for l in labels]
    if use_fused and _fused_ok(mask_embed, text_embed, null_embed, logit_scale, sizes):
        gs = group_start(sizes, mask_embed.device)
        return CategoryLogitsFunction.apply(mask_embed.contiguous(), text_embed.contiguous(), null_embed.contiguous(),
                                            logit_scale, gs)[0]
    return composed_pred_logits(mask_embed, text_embed, null_embed, labels, logit_scale)
