"""Attention.forward (alphafold2.py:125-190) in its general form: self- or cross-attention (`context`), a query mask and a
key mask (`context_mask`), an additive bias of any shape that broadcasts to [B, H, i, j] and tied queries.  With
context = context_mask = None it is evoformer_oracle.attention (tests/test_oracle_attention_forward.py pins both)."""
from __future__ import annotations

from typing import Optional

import torch

from oracle.evoformer_oracle import W, Tensor, _lin


def attention(w: W, p: str, x: Tensor, heads: int, mask: Optional[Tensor] = None, attn_bias: Optional[Tensor] = None,
              tie_dim: Optional[int] = None, context: Optional[Tensor] = None, context_mask: Optional[Tensor] = None) -> Tensor:
    """x: [B, i, d]; context: [B, j, d] or None (self); mask: [B, i] bool or None; context_mask: [B, j] bool or None.

    Masking happens only when mask is given (alphafold2.py:162): the key mask is then context_mask (context given; None:
    every key valid) or mask (self-attention), and masked logits are REPLACED by -finfo.max after the bias is added, so a
    masked query row attends uniformly to all j keys (quirk Q1).  tie_dim r: q (after scaling) is averaged over groups of r
    consecutive batch elements, each of which keeps its own keys (alphafold2.py:142-151)."""
    B, i, _ = x.shape
    c = x if context is None else context
    j = c.shape[1]
    q = _lin(w, p + "to_q", x)
    k, v = _lin(w, p + "to_kv", c).chunk(2, dim=-1)
    dh = q.shape[-1] // heads
    q = q.reshape(B, i, heads, dh).permute(0, 2, 1, 3) * dh ** -0.5
    k, v = (t.reshape(B, j, heads, dh).permute(0, 2, 1, 3) for t in (k, v))
    if tie_dim is not None:
        q = q.reshape(B // tie_dim, tie_dim, heads, i, dh).mean(dim=1)
        dots = torch.einsum("bhid,brhjd->brhij", q, k.reshape(B // tie_dim, tie_dim, heads, j, dh)).reshape(B, heads, i, j)
    else:
        dots = torch.einsum("bhid,bhjd->bhij", q, k)
    if attn_bias is not None:
        dots = dots + attn_bias.to(dots.dtype)
    if mask is not None:
        km = mask if context is None else (context_mask if context_mask is not None else torch.ones(B, j, dtype=torch.bool))
        pair = mask[:, None, :, None] & km.to(mask.device)[:, None, None, :]
        dots = dots.masked_fill(~pair, -torch.finfo(dots.dtype).max)
    out = torch.einsum("bhij,bhjd->bhid", dots.softmax(dim=-1), v)
    out = out.permute(0, 2, 1, 3).reshape(B, i, heads * dh)
    out = out * _lin(w, p + "gating", x).sigmoid()
    return _lin(w, p + "to_out", out)
