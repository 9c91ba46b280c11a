"""alphafold2_b200 — H100-native (sm_90a) drop-in for the Evoformer trunk hot path of lucidrains/alphafold2.

    from alphafold2_b200 import Alphafold2, Evoformer      # mirrors alphafold2_pytorch/__init__.py:1
"""
from .alphafold2 import (Alphafold2, Evoformer, EvoformerBlock, PairwiseAttentionBlock, MsaAttentionBlock,
                         AxialAttention, Attention, TriangleMultiplicativeModule, OuterMean, FeedForward,
                         ReturnValues, Recyclables, invalidate_packed, IPABlock, InvariantPointAttention,
                         attach_structure_module, recycle)
from .ops import set_precision
from .rotary import apply_rotary_pos_emb, rotate_every_two, FixedPositionalEmbedding, AxialRotaryEmbedding
from . import utils

__all__ = ["Alphafold2", "Evoformer", "EvoformerBlock", "PairwiseAttentionBlock", "MsaAttentionBlock",
           "AxialAttention", "Attention", "TriangleMultiplicativeModule", "OuterMean", "FeedForward",
           "ReturnValues", "Recyclables", "apply_rotary_pos_emb", "rotate_every_two",
           "FixedPositionalEmbedding", "AxialRotaryEmbedding", "invalidate_packed", "set_precision", "IPABlock",
           "InvariantPointAttention", "attach_structure_module", "recycle", "utils"]
