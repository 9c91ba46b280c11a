"""TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's template embedder (alphafold2.py:743-792).

Extends oracle/evoformer_oracle.py (same conventions: functional, dtype-generic, weights as a flat state dict with the
reference's key names) with
  * ``template_pointwise_attention``: ``Attention(x, context=..., mask=..., context_mask=...)`` (alphafold2.py:125-190),
  * ``alphafold2_distogram``: the distogram forward with the template branch (templates_feats / templates_mask /
    templates_angles) in the reference's order: glue -> templates -> angles -> (extra-MSA stack) -> trunk.
Pinned by tests/test_oracle_templates.py against fixtures written by oracle/make_golden_r3.py from the unmodified reference.
It must never be imported by ``alphafold2_b200``.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from oracle.evoformer_oracle import W, Tensor, _lin, _ln, evoformer, pairwise_attention_block


def template_pointwise_attention(w: W, p: str, x: Tensor, context: Tensor, heads: int, mask: Optional[Tensor] = None,
                                 context_mask: Optional[Tensor] = None) -> Tensor:
    """x [N, 1, d] queries, context [N, T, d]; mask [N, 1], context_mask [N, T] bool.  No LayerNorm on either side.
    As in the reference, masking only happens when `mask` is given (alphafold2.py:162): context_mask alone is ignored.  A
    query whose logits are all masked (-finfo.max) averages all T values uniformly."""
    N, i, _ = x.shape
    T = context.shape[1]
    q = _lin(w, p + "to_q", x)
    k, v = _lin(w, p + "to_kv", context).chunk(2, dim=-1)
    dh = q.shape[-1] // heads
    q = q.reshape(N, i, heads, dh).permute(0, 2, 1, 3) * dh ** -0.5
    k = k.reshape(N, T, heads, dh).permute(0, 2, 1, 3)
    v = v.reshape(N, T, heads, dh).permute(0, 2, 1, 3)
    dots = torch.einsum("bhid,bhjd->bhij", q, k)
    if mask is not None:
        cm = context_mask if context_mask is not None else torch.ones(1, T, dtype=torch.bool, device=x.device)
        pair = mask[:, None, :, None] & cm[:, None, None, :]
        dots = dots.masked_fill(~pair, -torch.finfo(dots.dtype).max)
    attn = dots.softmax(dim=-1)
    out = torch.einsum("bhij,bhjd->bhid", attn, v).permute(0, 2, 1, 3).reshape(N, i, heads * dh)
    out = out * _lin(w, p + "gating", x).sigmoid()
    return _lin(w, p + "to_out", out)


def template_pair_stack(w: W, feats: Tensor, templates_mask: Tensor, heads: int, layers: int):
    """alphafold2.py:751-760 -> (t [b, T, n, n, d], crossed mask [b, T, n, n])."""
    b, T, n = feats.shape[:3]
    t = _lin(w, "to_template_embed", feats)
    tm2 = templates_mask[:, :, :, None] & templates_mask[:, :, None, :]
    tf, mf = t.reshape(b * T, n, n, -1), tm2.reshape(b * T, n, n)
    for _ in range(layers):
        tf = pairwise_attention_block(w, "template_pairwise_embedder.", tf, heads, mf)
    return tf.reshape(b, T, n, n, -1), tm2


def embed_templates(w: W, x: Tensor, x_mask: Tensor, feats: Tensor, templates_mask: Tensor, heads: int, layers: int) -> Tensor:
    """alphafold2.py:743-785: x + pooled * pointwise attention over the templates (pooled = any template valid, NOT x_mask)."""
    b, n = x.shape[:2]
    T = feats.shape[1]
    t, tm2 = template_pair_stack(w, feats, templates_mask, heads, layers)
    x_point = x.reshape(b * n * n, 1, -1)
    t_point = t.permute(0, 2, 3, 1, 4).reshape(b * n * n, T, -1)
    x_mask_point = x_mask.reshape(b * n * n, 1)
    t_mask_point = tm2.permute(0, 2, 3, 1).reshape(b * n * n, T)
    pooled = template_pointwise_attention(w, "template_pointwise_attn.", x_point, t_point, heads, x_mask_point, t_mask_point)
    pooled = pooled * (t_mask_point.sum(dim=-1) > 0)[:, None, None].to(pooled.dtype)
    return x + pooled.reshape(b, n, n, -1)


def template_angle_features(w: W, angles: Tensor) -> Tensor:
    """template_angle_mlp (alphafold2.py:789): Linear -> exact-erf GELU -> Linear."""
    return _lin(w, "template_angle_mlp.2", F.gelu(_lin(w, "template_angle_mlp.0", angles)))


def alphafold2_distogram(w: W, seq: Tensor, msa: Optional[Tensor], mask: Optional[Tensor], msa_mask: Optional[Tensor], heads: int,
                         depth: int, templates_feats: Optional[Tensor] = None, templates_mask: Optional[Tensor] = None,
                         templates_angles: Optional[Tensor] = None, templates_embed_layers: int = 4, max_rel_dist: int = 32,
                         dtype=torch.float32, extra_msa_mask: Optional[Tensor] = None, extra_depth: int = 0) -> Tensor:
    """evoformer_oracle.alphafold2_distogram plus the template branch of alphafold2.py:743-792."""
    if msa is None:
        msa = seq[:, None, :]
        msa_mask = mask[:, None, :]
    b, n = seq.shape
    emb = w["token_emb.weight"].to(dtype)
    x1 = emb[seq]
    m = emb[msa] + x1[:, None]
    if msa_mask is None:
        msa_mask = torch.ones_like(msa).bool()
    xl, xr = _lin(w, "to_pairwise_repr", x1).chunk(2, dim=-1)
    x = xl[:, :, None, :] + xr[:, None, :, :]
    x_mask = (mask[:, :, None] & mask[:, None, :]) if mask is not None else None
    idx = torch.arange(n, device=seq.device)
    rel = (idx[:, None] - idx[None, :]).clamp(-max_rel_dist, max_rel_dist) + max_rel_dist
    x = x + w["pos_emb.weight"].to(dtype)[rel][None]
    if templates_feats is not None:
        x = embed_templates(w, x, x_mask, templates_feats.to(dtype), templates_mask, heads, templates_embed_layers)
    if templates_angles is not None:
        m = torch.cat((m, template_angle_features(w, templates_angles.to(dtype))), dim=1)
        msa_mask = torch.cat((msa_mask, templates_mask), dim=1)
    if extra_depth > 0:
        x, _ = evoformer(w, "extra_msa_evoformer.", x, emb[msa], heads, extra_depth, x_mask, extra_msa_mask, global_column_attn=True)
    x, m = evoformer(w, "net.", x, m, heads, depth, x_mask, msa_mask)
    te = (x + x.transpose(1, 2)) * 0.5
    return _lin(w, "to_distogram_logits.1", _ln(w, "to_distogram_logits.0", te))
