"""TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's recycling embedder (alphafold2.py:728-739).

Extends oracle/template_oracle.py (same conventions: functional, dtype-generic, weights as a flat state dict with the reference's
key names) with
  * ``recycle_embed``: the recyclables added to the pair tensor and to row 0 of the MSA tensor,
  * ``alphafold2_distogram``: template_oracle.alphafold2_distogram with an optional ``recyclables`` argument, in the reference's
    order: glue -> recycling -> templates -> angles -> (extra-MSA stack) -> trunk.
One deliberate difference from the literal reference: distances are the direct ones, |c_i - c_j| from coordinate differences in
fp64.  For n > 25 torch.cdist switches to |a|^2 + |b|^2 - 2 a.b, whose error reaches a few hundredths of an angstrom at
coordinates 40 A from the origin (DESIGN.md §2).  The bucket boundaries are the reference's own fp32 torch.linspace(2, 20, nb).
Pinned by tests/test_oracle_recycling.py against fixtures written by oracle/make_golden_r4.py from the unmodified reference.
It must never be imported by ``alphafold2_b200``.
"""
from __future__ import annotations

from typing import Optional

import torch

from oracle.evoformer_oracle import W, Tensor, _lin, _ln, evoformer
from oracle.template_oracle import embed_templates, template_angle_features


SHARED_PREFIX = "extra_msa_evoformer."


def fixture_state(state: W) -> W:
    """tests/golden/alphafold2_recycling.pt stores the trunk's weights once, under net.*: its extra-MSA stack has the same
    weights (oracle/make_golden_r4.py).  Returns the state with the extra_msa_evoformer.* keys restored."""
    out = dict(state)
    out.update({SHARED_PREFIX + k[len("net."):]: v.clone() for k, v in state.items() if k.startswith("net.")})
    return out


def recycling_boundaries(nb: int, device=None) -> Tensor:
    """alphafold2.py:736: the fp32 bucket edges; the reference searches the first nb - 1 of them."""
    return torch.linspace(2, 20, steps=nb, device=device)


def direct_distances(coords: Tensor) -> Tensor:
    """[b, n, c] -> [b, n, n] fp64, from coordinate differences (NaN coordinates give NaN distances)."""
    c = coords.double()
    return (c[:, :, None, :] - c[:, None, :, :]).pow(2).sum(-1).sqrt()


def distance_buckets(coords: Tensor, nb: int) -> Tensor:
    """torch.bucketize(dist, boundaries[:-1]) (right=False) with direct fp64 distances: NaN -> nb - 1."""
    dist = direct_distances(coords)
    return torch.bucketize(dist, recycling_boundaries(nb, coords.device)[:-1].double())


def recycle_embed(w: W, x: Tensor, m: Tensor, coords: Tensor, single_row: Tensor, pairwise_repr: Tensor):
    """alphafold2.py:730-739 -> (x, m): m[:, 0] += LN_msa(single_row); x = (x + LN_pair(pairwise_repr)) + E[bucket]."""
    dt = x.dtype
    m = m.clone()
    m[:, 0] = m[:, 0] + _ln(w, "recycling_msa_norm", single_row.to(dt))
    x = x + _ln(w, "recycling_pairwise_norm", pairwise_repr.to(dt))
    table = w["recycling_distance_embed.weight"].to(dt)
    return x + table[distance_buckets(coords, table.shape[0])], m


def alphafold2_distogram(w: W, seq: Tensor, msa: Optional[Tensor], mask: Optional[Tensor], msa_mask: Optional[Tensor], heads: int,
                         depth: int, recyclables=None, templates_feats: Optional[Tensor] = None,
                         templates_mask: Optional[Tensor] = None, templates_angles: Optional[Tensor] = None,
                         templates_embed_layers: int = 4, max_rel_dist: int = 32, dtype=torch.float32,
                         extra_msa_mask: Optional[Tensor] = None, extra_depth: int = 0) -> Tensor:
    """template_oracle.alphafold2_distogram plus the recycling embedder of alphafold2.py:728-739 (recyclables: any object with
    coords, single_msa_repr_row and pairwise_repr)."""
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
    if recyclables is not None:
        x, m = recycle_embed(w, x, m, recyclables.coords, recyclables.single_msa_repr_row, recyclables.pairwise_repr)
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
