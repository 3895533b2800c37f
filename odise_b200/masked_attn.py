"""Training drop-in for Mask2Former's masked cross-attention layer (CrossAttentionLayer of
third_party/Mask2Former/mask2former/modeling/transformer_decoder/mask2former_transformer_decoder.py:75-135).

    from odise_b200.masked_attn import CrossAttentionLayer   # in place of the class defined in that file

The layer keeps the reference's constructor, submodules (a real nn.MultiheadAttention, so state dicts load both ways),
initialisation and forward signatures.  On CUDA, with head dim 32 and a bool attn_mask (or none), its attention core runs
MaskedCrossAttnFunction: one sm_90a kernel pair (odise_masked_xattn_forward_* / _backward_*) that never writes the
[B*h, Q, S] score or probability tensors of nn.MultiheadAttention's math path and saves only a per-row log-sum-exp for the
backward.  Every gradient it returns is bit-reproducible in default mode (fixed-order sums, no atomics), so
torch.use_deterministic_algorithms changes nothing here.  Every other input takes nn.MultiheadAttention itself.

The kernels are reached through two torch custom ops, torch.ops.odise_b200.masked_xattn_forward and
masked_xattn_backward, with fake implementations, so torch.compile (fullgraph=True included) traces the layer without a
graph break."""
import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import lib

_DTYPES = (torch.float32, torch.float16, torch.bfloat16)

# The kernels as torch custom ops (lib.custom_op).  lib's functions are looked up at call time, so that a test that
# patches them sees every call.
lib.custom_op("masked_xattn_forward(Tensor q, Tensor k, Tensor v, Tensor? mask, int heads) -> (Tensor, Tensor)",
              lambda *args: lib.masked_xattn_forward(*args))
lib.custom_op("masked_xattn_backward(Tensor q, Tensor k, Tensor v, Tensor? mask, Tensor out, Tensor lse, "
              "Tensor grad_out, int heads) -> (Tensor, Tensor, Tensor)", lambda *args: lib.masked_xattn_backward(*args))


class MaskedCrossAttnFunction(Function):
    """softmax(s q k^T, blocked -> -inf) v per head, s = 1/sqrt(32), on the in-projection outputs q [Q, B, heads*32],
    k and v [S, B, heads*32] (CUDA, contiguous, one of float32 / float16 / bfloat16); mask None or bool [B*heads, Q, S] /
    [Q, S], True = blocked -> [Q, B, heads*32] in q's dtype.  Gradients for q, k and v in their dtype.  A row whose keys
    are all blocked gives NaN, as torch's softmax does: that output row, that row of the q gradient, and the k and v
    gradients of its (image, head)."""

    @staticmethod
    def forward(ctx, q, k, v, mask, heads):
        out, lse = torch.ops.odise_b200.masked_xattn_forward(q, k, v, mask, heads)
        ctx.heads = heads
        ctx.save_for_backward(q, k, v, mask, out, lse)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        q, k, v, mask, out, lse = ctx.saved_tensors
        gq, gk, gv = torch.ops.odise_b200.masked_xattn_backward(q, k, v, mask, out, lse,
                                                               grad_out.to(q.dtype).contiguous(), ctx.heads)
        return gq, gk, gv, None, None


def _activation(name):
    acts = {"relu": F.relu, "gelu": F.gelu, "glu": F.glu}
    if name not in acts:
        raise RuntimeError(f"activation should be relu/gelu, not {name}.")
    return acts[name]


class CrossAttentionLayer(nn.Module):
    """Mask2Former's CrossAttentionLayer: nn.MultiheadAttention(d_model, nhead, dropout) over (tgt + query_pos,
    memory + pos, memory), dropout, residual and LayerNorm, post-norm or (normalize_before) pre-norm.

    forward() runs the attention core as MaskedCrossAttnFunction when all of these hold: the tensors are on CUDA,
    d_model / nhead = 32, memory_mask is None or a bool tensor [B*nhead, Q, S] or [Q, S], memory_key_padding_mask is None,
    attention dropout is not in effect (p = 0 or eval mode), and the in-projections return float32, or float16 / bfloat16
    with at most fused_16bit_max_keys keys (4096 by default; None lifts the limit).
    The in-projection is F.linear with the three chunks of in_proj_weight / in_proj_bias, as
    F.multi_head_attention_forward does for distinct key and value; out_proj, dropout, residual and LayerNorm stay torch
    ops in the reference's order.  Every other input, CPU tensors included, and any call with use_fused = False, calls
    self.multihead_attn exactly as the reference does."""

    def __init__(self, d_model, nhead, dropout=0.0, activation="relu", normalize_before=False):
        super().__init__()
        self.multihead_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.norm = nn.LayerNorm(d_model)
        self.dropout = nn.Dropout(dropout)
        self.activation = _activation(activation)
        self.normalize_before = normalize_before
        self.use_fused = True          # False forces the composed path (for comparisons)
        # 16-bit projections with more keys than this take the composed path (None: fuse every length).  On an H100 the
        # 16-bit kernels are faster than nn.MultiheadAttention up to 64^2 keys and slower at 128^2, where they still
        # save most of the memory (DESIGN.md, "Masked cross-attention"): set None to trade that time for the memory.
        self.fused_16bit_max_keys = 4096
        self._reset_parameters()

    def _reset_parameters(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)

    def with_pos_embed(self, tensor, pos):
        return tensor if pos is None else tensor + pos

    def _fused_ok(self, query, key, value, attn_mask, key_padding_mask):
        mha = self.multihead_attn
        if not (self.use_fused and query.is_cuda and key.is_cuda and value.is_cuda):
            return False
        if key_padding_mask is not None or (mha.dropout > 0.0 and mha.training):
            return False
        if (not mha._qkv_same_embed_dim or mha.bias_k is not None or mha.add_zero_attn or mha.batch_first
                or mha.in_proj_bias is None or mha.head_dim != 32):
            return False
        if query.dim() != 3 or key.dim() != 3 or key.shape != value.shape or query.shape[1] != key.shape[1]:
            return False
        # the dtype the projections will return: autocast's, or the inputs'
        dtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else query.dtype
        cap = self.fused_16bit_max_keys
        if dtype in (torch.float16, torch.bfloat16) and cap is not None and key.shape[0] > cap:
            return False
        if attn_mask is not None:
            Q, B = query.shape[0], query.shape[1]
            S = key.shape[0]
            if attn_mask.dtype != torch.bool or not attn_mask.is_cuda:
                return False
            if tuple(attn_mask.shape) not in ((B * mha.num_heads, Q, S), (Q, S)):
                return False
        return True

    def _attention(self, query, key, value, attn_mask, key_padding_mask):
        mha = self.multihead_attn
        if self._fused_ok(query, key, value, attn_mask, key_padding_mask):
            w_q, w_k, w_v = mha.in_proj_weight.chunk(3)
            b_q, b_k, b_v = mha.in_proj_bias.chunk(3)
            q, k, v = F.linear(query, w_q, b_q), F.linear(key, w_k, b_k), F.linear(value, w_v, b_v)
            if q.dtype in _DTYPES and q.dtype == k.dtype == v.dtype:
                mask = None if attn_mask is None else attn_mask.contiguous()
                out = MaskedCrossAttnFunction.apply(q, k, v, mask, mha.num_heads)
                Q, B, E = out.shape
                return F.linear(out.view(Q * B, E), mha.out_proj.weight, mha.out_proj.bias).view(Q, B, E)
        return mha(query=query, key=key, value=value, attn_mask=attn_mask, key_padding_mask=key_padding_mask)[0]

    def forward_post(self, tgt, memory, memory_mask=None, memory_key_padding_mask=None, pos=None, query_pos=None):
        tgt2 = self._attention(self.with_pos_embed(tgt, query_pos), self.with_pos_embed(memory, pos), memory,
                               memory_mask, memory_key_padding_mask)
        tgt = tgt + self.dropout(tgt2)
        tgt = self.norm(tgt)
        return tgt

    def forward_pre(self, tgt, memory, memory_mask=None, memory_key_padding_mask=None, pos=None, query_pos=None):
        tgt2 = self.norm(tgt)
        tgt2 = self._attention(self.with_pos_embed(tgt2, query_pos), self.with_pos_embed(memory, pos), memory,
                               memory_mask, memory_key_padding_mask)
        tgt = tgt + self.dropout(tgt2)
        return tgt

    def forward(self, tgt, memory, memory_mask=None, memory_key_padding_mask=None, pos=None, query_pos=None):
        if self.normalize_before:
            return self.forward_pre(tgt, memory, memory_mask, memory_key_padding_mask, pos, query_pos)
        return self.forward_post(tgt, memory, memory_mask, memory_key_padding_mask, pos, query_pos)
