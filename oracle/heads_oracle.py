"""CPU oracle of the angle heads of Alphafold2(predict_angles=True) (alphafold2.py:559-562, 813-836), plain torch, any dtype:

  * ``angle_heads``: (theta, phi, omega) logits from the trunk output x [b, n, n, d]; omega from (x + x^T) * 0.5 when
    symmetrize_omega (alphafold2.py:821, 833), else from x;
  * ``alphafold2_angles``: the whole forward (evoformer_oracle.alphafold2_distogram's trunk), returning distance and the three.
"""
from typing import Dict, Optional

import torch
from torch import Tensor

from oracle.evoformer_oracle import _lin, _ln, alphafold2_distogram

W = Dict[str, Tensor]


def angle_heads(w: W, x: Tensor, symmetrize_omega: bool):
    """x [b, n, n, d] -> (theta, phi, omega) in x's dtype, from the to_prob_theta / to_prob_phi / to_prob_omega weights in w."""
    theta = _lin(w, "to_prob_theta", x)
    phi = _lin(w, "to_prob_phi", x)
    s = (x + x.transpose(1, 2)) * 0.5 if symmetrize_omega else x
    return theta, phi, _lin(w, "to_prob_omega", s)


def alphafold2_angles(w: W, seq: Tensor, msa: Optional[Tensor], mask: Optional[Tensor], msa_mask: Optional[Tensor], heads: int,
                      depth: int, symmetrize_omega: bool, dtype=torch.float32):
    """Alphafold2.forward with predict_angles=True -> dict of distance, theta, phi, omega logits and the trunk output x."""
    x, _ = alphafold2_distogram(w, seq, msa, mask, msa_mask, heads, depth, dtype=dtype, return_trunk=True)
    distance = _lin(w, "to_distogram_logits.1", _ln(w, "to_distogram_logits.0", (x + x.transpose(1, 2)) * 0.5))
    theta, phi, omega = angle_heads(w, x, symmetrize_omega)
    return {"distance": distance, "theta": theta, "phi": phi, "omega": omega, "x": x}
