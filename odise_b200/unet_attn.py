"""Training drop-in for the attention of the SD-v1 UNet (ldm's CrossAttention, ldm/modules/attention.py; restated in
oracle/ldm.py:94-117), which ODISE backpropagates through in training.

    from odise_b200.unet_attn import replace_attention
    replace_attention(unet)          # before building the optimizer and the DDP wrap

CrossAttention keeps ldm's constructor keywords, submodules and state-dict keys (to_q, to_k, to_v, to_out.0, with
to_out.1 the Dropout).  On CUDA its attention core runs UNetAttnFunction: one sm_90a kernel pair
(odise_unet_attn_forward_* / _backward_*) that never writes the [B*h, Tq, Tk] score or probability tensors of the
einsum / softmax / einsum composition and saves only a per-row log-sum-exp for the backward.  Every gradient it returns
is bit-reproducible in default mode (fixed-order sums, no atomics), so torch.use_deterministic_algorithms changes
nothing here.  Every other input takes the composition itself, in ldm's op order.

The kernels are reached through two torch custom ops, torch.ops.odise_b200.unet_attn_forward and unet_attn_backward,
with fake implementations, so torch.compile (fullgraph=True included) traces the module without a graph break."""
import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib

_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def fused_faster(dtype, Tk):
    """whether the fused kernels beat the composed path at Tk keys (tools/unet_attn_bench.py at B = 8 on an H100, 16-bit
    arms under autocast; DESIGN.md §3 "UNet attention for training"): at every cross-attention (77 keys), at
    self-attention up to 256 keys and at 4096 keys, in every storage dtype.  At 1024 keys (the 32^2 latent) cuBLAS's
    products over the [B*h, Tq, Tk] scores are faster in every dtype, outside the run-to-run spread, so those layers take
    the composed path.  dtype is part of the rule's signature because the measurement is per dtype; the measured
    boundary is the same for all three."""
    return Tk <= 256 or Tk > 2048


# The kernels as torch custom ops (lib.custom_op).  lib's functions are looked up at call time, so that a test that
# patches them sees every call.
lib.custom_op("unet_attn_forward(Tensor q, Tensor k, Tensor v, int heads) -> (Tensor, Tensor)",
              lambda *args: lib.unet_attn_forward(*args))
lib.custom_op("unet_attn_backward(Tensor q, Tensor k, Tensor v, Tensor out, Tensor lse, Tensor grad_out, int heads) "
              "-> (Tensor, Tensor, Tensor)", lambda *args: lib.unet_attn_backward(*args))


class UNetAttnFunction(Function):
    """softmax(d^-1/2 q k^T) v per head on the projection outputs q [B, Tq, heads*d], k and v [B, Tk, heads*d] (CUDA,
    contiguous, one of float32 / float16 / bfloat16, d = 40, 80 or 160) -> [B, Tq, heads*d] in q's dtype.  Saves q, k,
    v, the output and lse [B*heads, Tq] float32; gradients for q, k and v in their dtype."""

    @staticmethod
    def forward(ctx, q, k, v, heads):
        out, lse = torch.ops.odise_b200.unet_attn_forward(q, k, v, heads)
        ctx.heads = heads
        ctx.save_for_backward(q, k, v, out, lse)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        q, k, v, out, lse = ctx.saved_tensors
        gq, gk, gv = torch.ops.odise_b200.unet_attn_backward(q, k, v, out, lse, grad_out.to(q.dtype).contiguous(),
                                                            ctx.heads)
        return gq, gk, gv, None


class CrossAttention(nn.Module):
    """ldm's CrossAttention: to_q, to_k, to_v (no bias), softmax(scale q k^T) v per head, to_out = Linear + Dropout.

    forward() runs the attention core as UNetAttnFunction when all of these hold: use_fused is True, the tensors are on
    CUDA, mask is None, the output dropout is not in effect (p = 0 or eval mode), scale is dim_head^-1/2 (what the kernels
    apply; ldm's value), lib.unet_attn_supported holds for the
    shapes, the projections return one dtype of float32 / float16 / bfloat16, and fused_faster(that dtype, Tk).  Every
    other input, CPU tensors included, takes ldm's einsum / softmax / einsum in ldm's op order (mask: a bool [B, ...] over the keys, False =
    blocked, filled with -finfo.max as ldm does)."""

    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.0):
        super().__init__()
        inner = dim_head * heads
        context_dim = context_dim or query_dim
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(dropout))
        self.use_fused = True          # False forces the composed path (for comparisons)

    def _dropout_active(self):
        return self.training and any(isinstance(m, nn.Dropout) and m.p > 0 for m in self.to_out)

    def _fused_ok(self, x, context, mask):
        if not self.use_fused or mask is not None or self._dropout_active():
            return False
        if not x.is_cuda or not context.is_cuda or x.dim() != 3 or context.dim() != 3 or x.shape[0] != context.shape[0]:
            return False
        inner = self.to_q.out_features
        if inner % self.heads or self.scale != (inner // self.heads) ** -0.5:     # the kernels scale by d^-1/2
            return False
        return lib.unet_attn_supported(x.shape[0], self.heads, inner // self.heads, x.shape[1], context.shape[1])

    def forward(self, x, context=None, mask=None):
        h = self.heads
        q = self.to_q(x)
        context = x if context is None else context
        k, v = self.to_k(context), self.to_v(context)
        if (self._fused_ok(x, context, mask) and q.dtype in _DTYPES and q.dtype == k.dtype == v.dtype
                and fused_faster(q.dtype, k.shape[1])):
            return self.to_out(UNetAttnFunction.apply(q.contiguous(), k.contiguous(), v.contiguous(), h))
        b, n, _ = q.shape
        q, k, v = (t.reshape(b, t.shape[1], h, -1).permute(0, 2, 1, 3) for t in (q, k, v))
        sim = torch.einsum("bhid,bhjd->bhij", q, k) * self.scale
        if mask is not None:
            sim.masked_fill_(~mask.reshape(b, -1)[:, None, None, :], -torch.finfo(sim.dtype).max)
        attn = sim.softmax(dim=-1)
        out = torch.einsum("bhij,bhjd->bhid", attn, v)
        out = out.permute(0, 2, 1, 3).reshape(b, n, -1)
        return self.to_out(out)

    @classmethod
    def adopt(cls, old):
        """A CrossAttention that owns old's to_q, to_k, to_v and to_out modules (the same Parameter objects) and takes
        its heads, scale and training mode"""
        heads = old.heads
        drop = next((m.p for m in old.to_out if isinstance(m, nn.Dropout)), 0.0)
        with torch.device("meta"):          # every submodule is replaced below: allocate nothing
            new = cls(old.to_q.in_features, old.to_k.in_features, heads, old.to_q.out_features // heads, drop)
        new.to_q, new.to_k, new.to_v, new.to_out = old.to_q, old.to_k, old.to_v, old.to_out
        new.scale = getattr(old, "scale", new.scale)
        new.train(old.training)
        return new


def _is_attention(m):
    return hasattr(m, "heads") and all(isinstance(getattr(m, c, None), nn.Module) for c in ("to_q", "to_k", "to_v",
                                                                                              "to_out"))


def replace_attention(model):
    """Swap every attention module of a UNet in place for a CrossAttention that owns the same submodules and
    Parameters, so an optimizer or DDP built afterwards sees the same parameters and the state dict keeps its keys.  The
    modules are found by structure: a `heads` attribute and to_q / to_k / to_v / to_out children.  -> the number
    swapped (32 for the SD-v1 UNet)."""
    names = [n for n, m in model.named_modules() if n and _is_attention(m) and not isinstance(m, CrossAttention)]
    for name in names:
        parent, _, child = name.rpartition(".")
        owner = model.get_submodule(parent)
        setattr(owner, child, CrossAttention.adopt(getattr(owner, child)))
    return len(names)
