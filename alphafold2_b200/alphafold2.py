"""Host-side mirror of the reference module interface for the Evoformer trunk hot path.

Same class names, constructor signatures, forward signatures and ``state_dict`` keys as
``alphafold2_pytorch/alphafold2.py`` (reference @ 931466e), so reference checkpoints load unchanged and the
reference's own API smoke tests run against this package.  The forward bodies of every module on the hot
path (alphafold2.py:69-467) call hand-written sm_90a kernels through the C ABI in include/af2b200.h;
there is no PyTorch / CPU fallback for them.  Glue outside the trunk (embeddings, pair initialisation,
distogram head, alphafold2.py:676-726, 811-823) stays plain PyTorch on the device (SURVEY.md §8f n1).

Forward-only: the kernels are not differentiable (the reference trains through autograd; that is out of
scope of this path, see DESIGN.md).  The fp32 residual streams are updated in place on private copies.
"""
from __future__ import annotations

import math
import warnings
from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn

from . import banded, ops
from .stages import CudaStageOps

# constants of alphafold2_pytorch/constants.py:5-15 that the constructor defaults depend on
MAX_NUM_MSA = 20
MAX_NUM_TEMPLATES = 10
NUM_AMINO_ACIDS = 21
NUM_EMBEDDS_TR = 1280
DISTOGRAM_BUCKETS = 37
THETA_BUCKETS = 25
PHI_BUCKETS = 13
OMEGA_BUCKETS = 25


@dataclass
class Recyclables:                      # alphafold2.py:24-28
    coords: torch.Tensor
    single_msa_repr_row: torch.Tensor
    pairwise_repr: torch.Tensor


@dataclass
class ReturnValues:                     # alphafold2.py:30-37
    distance: torch.Tensor = None
    theta: torch.Tensor = None
    phi: torch.Tensor = None
    omega: torch.Tensor = None
    msa_mlm_loss: torch.Tensor = None
    recyclables: Recyclables = None


def exists(val):
    return val is not None


class _Packable(nn.Module):
    """Caches the bf16-packed weights of a module, re-packing when a parameter was modified.

    The cache key is (data_ptr, _version) of every parameter plus a global epoch: optimizer steps, ``copy_``,
    ``load_state_dict``, ``.to()/.cuda()`` and ``train()/eval()`` are all seen.  Writes through ``param.data``
    (``w.data.copy_()``, EMA ``p.data.mul_()``) change neither field in torch, so they need an explicit
    ``alphafold2_b200.invalidate_packed(model)`` -- or run with ``AF2_PACK_CHECK=1``, which adds a content
    fingerprint (one device sync per module and forward: a debugging aid, not the default)."""

    def _pack(self) -> ops.Packed:
        raise NotImplementedError

    def _pack_key(self):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters(recurse=True)) + (ops.pack_epoch(), ops.precision_of(self))
        if ops.PACK_CHECK:
            with torch.no_grad():
                key += tuple(float(p.detach().double().sum()) + float(p.detach().double().abs().sum()) for p in self.parameters(recurse=True))
        return key

    def packed(self) -> ops.Packed:
        key = self._pack_key()
        if self.__dict__.get("_pk_key") != key:
            with torch.no_grad():
                self.__dict__["_pk"] = self._pack()
            self.__dict__["_pk_key"] = key
        return self.__dict__["_pk"]

    def invalidate_packed(self):
        self.__dict__.pop("_pk", None)
        self.__dict__.pop("_pk_key", None)

    # the packed cache holds ctypes structs (device pointers): never copied / pickled with the module
    def __getstate__(self):
        st = dict(self.__dict__)
        st.pop("_pk", None)
        st.pop("_pk_key", None)
        return st

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k in ("_pk", "_pk_key"):
                continue
            new.__dict__[k] = copy.deepcopy(v, memo)
        return new

    def _load_from_state_dict(self, *args, **kwargs):
        self.invalidate_packed()
        return super()._load_from_state_dict(*args, **kwargs)

    def train(self, mode: bool = True):
        self.invalidate_packed()
        return super().train(mode)

    def _apply(self, fn, *args, **kwargs):
        self.invalidate_packed()
        return super()._apply(fn, *args, **kwargs)


def invalidate_packed(module: nn.Module) -> None:
    """Drop every cached packed-weight set under `module` (needed after in-place edits through ``param.data``)."""
    ops.bump_pack_epoch()
    for mod in module.modules():
        if isinstance(mod, _Packable):
            mod.invalidate_packed()


def _forward_only(*tensors):
    """SURVEY.md 8(b) error convention: the kernels are not differentiable.  Silently detaching would return wrong
    (zero) gradients, so a call that autograd would have to record raises instead."""
    if torch.is_grad_enabled() and any(t is not None and torch.is_tensor(t) and t.requires_grad for t in tensors):
        raise RuntimeError("alphafold2_b200 is forward-only (hand-written sm_90a kernels, no autograd): call it under "
                           "torch.no_grad() or pass tensors that do not require grad")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    """Private fp32 contiguous copy (the kernels update the residual stream in place)."""
    return t.detach().to(torch.float32).contiguous().clone()


# ------------------------------------------------------------------------------------------------------
# FeedForward (alphafold2.py:69-94)
# ------------------------------------------------------------------------------------------------------
class GEGLU(nn.Module):
    """Placeholder keeping nn.Sequential indices (and so state_dict keys) identical; fused into the kernel."""

    def forward(self, x):  # pragma: no cover - never called on the hot path
        a, g = x.chunk(2, dim=-1)
        return a * torch.nn.functional.gelu(g)


class FeedForward(_Packable):
    def __init__(self, dim, mult=4, dropout=0.):
        super().__init__()
        self.norm = nn.LayerNorm(dim)
        self.net = nn.Sequential(nn.Linear(dim, dim * mult * 2), GEGLU(), nn.Dropout(dropout), nn.Linear(dim * mult, dim))
        nn.init.zeros_(self.net[-1].weight)          # alphafold2.py:90
        nn.init.zeros_(self.net[-1].bias)

    def _pack(self):
        fn = ops.pack_feed_forward_strict if ops.precision_of(self) == "strict" else ops.pack_feed_forward
        return fn(self.norm.weight, self.norm.bias, self.net[0].weight, self.net[0].bias,
                                     self.net[3].weight, self.net[3].bias)

    def add_to_(self, x):
        """x <- x + FeedForward(x), in place."""
        return ops.feed_forward_(self.packed(), x)

    def forward(self, x, **kwargs):
        _forward_only(x)
        with torch.no_grad():
            res = _f32c(x)
            return (self.add_to_(res) - x).to(x.dtype)


# ------------------------------------------------------------------------------------------------------
# Attention / AxialAttention (alphafold2.py:98-255)
# ------------------------------------------------------------------------------------------------------
class Attention(_Packable):
    """Parameters with the reference's layout.  Inside the model, self-attention runs in AxialAttention's kernel call and the
    pointwise template attention through add_context_; forward() runs any standalone call (alphafold2.py:125-190)."""

    def __init__(self, dim, seq_len=None, heads=8, dim_head=64, dropout=0., gating=True):
        super().__init__()
        inner_dim = dim_head * heads
        self.seq_len = seq_len
        self.heads = heads
        self.dim_head = dim_head
        self.scale = dim_head ** -0.5
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim, inner_dim * 2, bias=False)
        self.to_out = nn.Linear(inner_dim, dim)
        self.gating = nn.Linear(dim, inner_dim)
        nn.init.constant_(self.gating.weight, 0.)    # alphafold2.py:119-120
        nn.init.constant_(self.gating.bias, 1.)
        self.dropout = nn.Dropout(dropout)
        nn.init.zeros_(self.to_out.weight)           # alphafold2.py:123
        nn.init.zeros_(self.to_out.bias)

    def _pack(self):
        fn = ops.pack_template_attention_strict if ops.precision_of(self) == "strict" else ops.pack_template_attention
        return fn(self.to_q.weight, self.to_kv.weight, self.gating.weight, self.gating.bias, self.to_out.weight, self.to_out.bias,
                  self.dim_head)

    def add_context_(self, x, t, x_mask, t_mask):
        """x [b, n, n, d] <- x + pooled * Attention(x, context=t, mask=x_mask, context_mask=t_mask) per pair position, in place:
        the pointwise template attention of alphafold2.py:764-785 (t [b * T, n, n, d], t_mask [b * T, n, n] crossed)."""
        return ops.template_pointwise_attention_(self.packed(), x, t, x_mask, t_mask, self.heads, self.dim_head)

    def forward(self, x, mask=None, attn_bias=None, context=None, context_mask=None, tie_dim=None):
        """alphafold2.py:125-190 on the GPU: gated self- or cross-attention (no LayerNorm, no residual), result in x.dtype.
        One query per batch element without a bias runs the pointwise template kernel; the rest the tensor-core attention
        (strict mode: the split-bf16 attention)."""
        _forward_only(x, context, attn_bias)
        with torch.no_grad():
            out = ops.attention_forward(self.packed(), x, self.heads, self.dim_head, mask=mask, attn_bias=attn_bias, context=context,
                                        context_mask=context_mask, tie_dim=tie_dim)
            return out.to(x.dtype)


class _TemplateEmbed(_Packable, nn.Linear):
    """to_template_embed (alphafold2.py:751): nn.Linear whose packed weight feeds af2_template_embed."""

    def _pack(self):
        return ops.pack_linear(self.weight, self.bias, strict=ops.precision_of(self) == "strict")

    def embed(self, feats):
        return ops.template_embed(self.packed(), feats)


class _TemplateAngleMLP(_Packable, nn.Sequential):
    """template_angle_mlp (alphafold2.py:789): Linear -> GELU -> Linear, one C-ABI call writing into rows of m."""

    def _pack(self):
        return ops.pack_template_angles(self[0].weight, self[0].bias, self[2].weight, self[2].bias,
                                        strict=ops.precision_of(self) == "strict")

    def write_(self, angles, m, row0):
        return ops.template_angle_features(self.packed(), angles, m, row0)


class _AngleHeads(_Packable):
    """Packed weights of the three angle heads for af2_angle_heads.  to_prob_theta / to_prob_phi / to_prob_omega stay the model's
    own nn.Linear modules (the reference's state_dict keys); this cache is kept outside the module tree and keys on their
    parameters."""

    def __init__(self, theta: nn.Linear, phi: nn.Linear, omega: nn.Linear):
        super().__init__()
        self.__dict__["heads"] = (theta, phi, omega)

    def parameters(self, recurse: bool = True):
        for h in self.heads:
            yield from h.parameters(recurse)

    def buckets(self):
        return tuple(h.out_features for h in self.heads)

    def _pack(self):
        t, p, o = self.heads
        return ops.pack_angle_heads(t.weight, t.bias, p.weight, p.bias, o.weight, o.bias)

    def run(self, x, symmetrize_omega: bool):
        return ops.angle_heads(self.packed(), x, symmetrize_omega)


class AxialAttention(_Packable):
    def __init__(self, dim, heads, row_attn=True, col_attn=True, accept_edges=False, global_query_attn=False, **kwargs):
        super().__init__()
        assert not (not row_attn and not col_attn), 'row or column attention must be turned on'
        self.row_attn = row_attn
        self.col_attn = col_attn
        self.global_query_attn = global_query_attn
        self.norm = nn.LayerNorm(dim)
        self.attn = Attention(dim=dim, heads=heads, **kwargs)
        # index 1 of the reference's Sequential is a parameter-free Rearrange('b i j h -> b h i j')
        self.edges_to_attn_bias = nn.Sequential(nn.Linear(dim, heads, bias=False), nn.Identity()) if accept_edges else None

    def _pack(self):
        a = self.attn
        we = self.edges_to_attn_bias[0].weight if self.edges_to_attn_bias is not None else None
        fn = ops.pack_attention_strict if ops.precision_of(self) == "strict" else ops.pack_attention
        return fn(self.norm.weight, self.norm.bias, a.to_q.weight, a.to_kv.weight, a.gating.weight,
                                  a.gating.bias, a.to_out.weight, a.to_out.bias, we, a.dim_head)

    def add_to_(self, x, edges=None, mask=None):
        assert self.row_attn ^ self.col_attn, 'has to be either row or column attention, but not both'
        return ops.axial_attention_(self.packed(), x, self.attn.heads, self.attn.dim_head, bool(self.row_attn), edges, mask,
                                    tied=bool(self.global_query_attn))

    def forward(self, x, edges=None, mask=None):
        _forward_only(x, edges)
        with torch.no_grad():
            res = _f32c(x)
            e = None
            if exists(edges) and self.edges_to_attn_bias is not None:
                e = res if edges is x else edges.detach().to(torch.float32).contiguous()
                if e is res:
                    e = e.clone()       # the bias must see the input, not the in-place result
            return (self.add_to_(res, e, mask) - x).to(x.dtype)


# ------------------------------------------------------------------------------------------------------
# TriangleMultiplicativeModule (alphafold2.py:257-317)
# ------------------------------------------------------------------------------------------------------
class TriangleMultiplicativeModule(_Packable):
    def __init__(self, *, dim, hidden_dim=None, mix='ingoing'):
        super().__init__()
        assert mix in {'ingoing', 'outgoing'}, 'mix must be either ingoing or outgoing'
        hidden_dim = hidden_dim if exists(hidden_dim) else dim
        if hidden_dim != dim:
            raise NotImplementedError("hidden_dim != dim is never used by the reference model (alphafold2.py:368-369)")
        self.mix = mix
        self.norm = nn.LayerNorm(dim)
        self.left_proj = nn.Linear(dim, hidden_dim)
        self.right_proj = nn.Linear(dim, hidden_dim)
        self.left_gate = nn.Linear(dim, hidden_dim)
        self.right_gate = nn.Linear(dim, hidden_dim)
        self.out_gate = nn.Linear(dim, hidden_dim)
        for gate in (self.left_gate, self.right_gate, self.out_gate):     # alphafold2.py:280-282
            nn.init.constant_(gate.weight, 0.)
            nn.init.constant_(gate.bias, 1.)
        self.to_out_norm = nn.LayerNorm(hidden_dim)
        self.to_out = nn.Linear(hidden_dim, dim)

    def _pack(self):
        fn = ops.pack_triangle_multiply_strict if ops.precision_of(self) == "strict" else ops.pack_triangle_multiply
        return fn(
            self.norm.weight, self.norm.bias, self.left_proj.weight, self.left_proj.bias, self.right_proj.weight,
            self.right_proj.bias, self.left_gate.weight, self.left_gate.bias, self.right_gate.weight,
            self.right_gate.bias, self.out_gate.weight, self.out_gate.bias, self.to_out_norm.weight,
            self.to_out_norm.bias, self.to_out.weight, self.to_out.bias)

    def add_to_(self, x, mask=None):
        return ops.triangle_multiply_(self.packed(), x, self.mix == 'ingoing', mask)

    def forward(self, x, mask=None):
        assert x.shape[1] == x.shape[2], 'feature map must be symmetrical'
        _forward_only(x)
        with torch.no_grad():
            res = _f32c(x)
            return (self.add_to_(res, mask) - x).to(x.dtype)


# ------------------------------------------------------------------------------------------------------
# OuterMean (alphafold2.py:321-351)
# ------------------------------------------------------------------------------------------------------
class OuterMean(_Packable):
    def __init__(self, dim, hidden_dim=None, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.norm = nn.LayerNorm(dim)
        hidden_dim = hidden_dim if exists(hidden_dim) else dim
        if hidden_dim != dim:
            raise NotImplementedError("hidden_dim != dim is never used by the reference model (alphafold2.py:364)")
        self.left_proj = nn.Linear(dim, hidden_dim)
        self.right_proj = nn.Linear(dim, hidden_dim)
        self.proj_out = nn.Linear(hidden_dim, dim)

    def _pack(self):
        fn = ops.pack_outer_mean_strict if ops.precision_of(self) == "strict" else ops.pack_outer_mean
        return fn(self.norm.weight, self.norm.bias, self.left_proj.weight, self.left_proj.bias,
                                   self.right_proj.weight, self.right_proj.bias, self.proj_out.weight, self.proj_out.bias)

    def add_to_(self, x, m, mask=None):
        """x <- x + OuterMean(m, mask)."""
        return ops.outer_mean_(self.packed(), x, m, mask, self.eps)

    def forward(self, x, mask=None):
        _forward_only(x)
        with torch.no_grad():
            m = x.detach().to(torch.float32).contiguous()
            b, _, n, d = m.shape
            out = torch.zeros(b, n, n, d, dtype=torch.float32, device=m.device)
            return self.add_to_(out, m, mask).to(x.dtype)


# ------------------------------------------------------------------------------------------------------
# Evoformer blocks (alphafold2.py:353-467)
# ------------------------------------------------------------------------------------------------------
def _pair_band(pair, x, S, band):
    """Pair rows per band for the pair track of `pair` (a PairwiseAttentionBlock) on x [B, N, N, d] with S MSA rows beside it:
    N (the whole-tensor calls) when they fit 85 % of what the device can still allocate (the template planner's headroom:
    the caching allocator cannot always reuse the blocks it frees), else ops.plan_pair_band's band.  `band` forces it (tests:
    a multiple of 8, which keeps every operand window 16-byte aligned for TMA; the planner's bands are multiples of
    ops.PAIR_BAND_ALIGN).  Strict mode is a parity mode and always runs whole.  Records pair.last_pair_band."""
    N = x.shape[1]
    ta = pair.triangle_attention_ingoing
    if not x.is_cuda or ops.precision_of(ta) == "strict":
        band = N
    elif band is None:
        shape = (x.shape[0], N, S, x.shape[3], ta.attn.heads, ta.attn.dim_head)
        if ops.workspace_holds(x.device, ops.pair_block_bytes(*shape, N)):
            band = N                      # the workspace already holds the whole-tensor calls: no device query per block
        else:
            band = ops.plan_pair_band(*shape, int(ops.device_budget(x.device) * 0.85))
    elif int(band) < N and (int(band) <= 0 or int(band) % 8):
        raise ValueError(f"pair band {band} must be a positive multiple of 8")
    band = min(int(band), N)
    if band < N and ta.global_query_attn:
        raise NotImplementedError(
            f"N_res {N} needs the pair track in bands of {band} rows, but tied-query column attention (global_query_attn, "
            "the extra-MSA stack) averages its queries over all columns and cannot run in column bands")
    pair.last_pair_band = band
    return band


def _block_bands(pair, x, S, band, msa_band):
    """(pair rows, MSA rows) per band of one Evoformer block whose pair block is `pair`, on x [B, N, N, d] and S MSA rows.
    Unforced: (N, S) when the workspace already holds the whole block, else ops.plan_block_bands, which keeps _pair_band's
    plan with the MSA track whole whenever that fits.  `band` forces the pair rows (as in _pair_band) and `msa_band` the MSA
    rows (any positive integer: row bands start at multiples of d * 4 bytes and column bands are compact copies).  Strict
    mode always runs whole."""
    N = x.shape[1]
    ta = pair.triangle_attention_ingoing
    if not x.is_cuda or ops.precision_of(ta) == "strict":
        return _pair_band(pair, x, S, band), S
    if msa_band is not None:
        if int(msa_band) <= 0:
            raise ValueError(f"MSA band {msa_band} must be a positive number of MSA rows")
        msa_band = min(int(msa_band), S)
    if band is None and msa_band is None:
        shape = (x.shape[0], N, S, x.shape[3], ta.attn.heads, ta.attn.dim_head)
        if not ops.workspace_holds(x.device, ops.pair_block_bytes(*shape, N)):
            band, msa_band = ops.plan_block_bands(*shape, int(ops.device_budget(x.device) * 0.85))
    return _pair_band(pair, x, S, band), S if msa_band is None else msa_band


class PairwiseAttentionBlock(nn.Module):
    def __init__(self, dim, seq_len, heads, dim_head, dropout=0., global_column_attn=False):
        super().__init__()
        self.outer_mean = OuterMean(dim)
        self.triangle_attention_outgoing = AxialAttention(dim=dim, heads=heads, dim_head=dim_head, row_attn=True, col_attn=False, accept_edges=True)
        self.triangle_attention_ingoing = AxialAttention(dim=dim, heads=heads, dim_head=dim_head, row_attn=False, col_attn=True, accept_edges=True, global_query_attn=global_column_attn)
        self.triangle_multiply_outgoing = TriangleMultiplicativeModule(dim=dim, mix='outgoing')
        self.triangle_multiply_ingoing = TriangleMultiplicativeModule(dim=dim, mix='ingoing')

    def update_(self, x, mask=None, msa_repr=None, msa_mask=None, band=None, msa_band=None):
        """In-place residual chain of alphafold2.py:378-385 on an fp32 pair tensor.

        Runs in bands of pair rows (banded.pair_block_, bitwise the same result) when the whole-tensor calls would not fit
        what the device can still allocate; `band` forces the rows per band (tests).  The band used is kept in
        self.last_pair_band (N: today's whole-tensor calls).  msa_band < S projects m for the outer mean in chunks of that many
        MSA rows (EvoformerBlock.update_ passes it when the MSA track runs in bands); with the pair rows whole the outer mean
        is then that projection and one contraction over all rows, and every other call stays whole."""
        S = msa_repr.shape[1] if exists(msa_repr) else 0
        band = _pair_band(self, x, S, band)
        msa_rows = int(msa_band) if msa_band is not None and int(msa_band) < S else None
        if not x.is_cuda or ops.precision_of(self.outer_mean) == "strict":
            msa_rows = None                       # strict mode (a parity mode) runs whole
        if band < x.shape[1] or msa_rows is not None:
            st = CudaStageOps()
            mask = mask.bool().contiguous() if exists(mask) else None
            msa_mask = msa_mask.bool().contiguous() if exists(msa_mask) else None
            pick = lambda t, b: None if t is None else t[b]  # noqa: E731
            if band < x.shape[1]:
                for b in range(x.shape[0]):
                    banded.pair_block_(self, x[b], pick(mask, b), pick(msa_repr, b), pick(msa_mask, b), band, st, msa_rows)
                return x
            for b in range(x.shape[0]):
                banded.outer_mean_(self.outer_mean, x[b], msa_repr[b], pick(msa_mask, b), msa_rows, st)
        elif exists(msa_repr):
            self.outer_mean.add_to_(x, msa_repr, msa_mask)
        self.triangle_multiply_outgoing.add_to_(x, mask)
        self.triangle_multiply_ingoing.add_to_(x, mask)
        self.triangle_attention_outgoing.add_to_(x, x, mask)
        self.triangle_attention_ingoing.add_to_(x, x, mask)
        return x

    def forward(self, x, mask=None, msa_repr=None, msa_mask=None):
        _forward_only(x, msa_repr)
        with torch.no_grad():
            mr = msa_repr.detach().to(torch.float32).contiguous() if exists(msa_repr) else None
            return self.update_(_f32c(x), mask, mr, msa_mask).to(x.dtype)


class MsaAttentionBlock(nn.Module):
    def __init__(self, dim, seq_len, heads, dim_head, dropout=0.):
        super().__init__()
        self.row_attn = AxialAttention(dim=dim, heads=heads, dim_head=dim_head, row_attn=True, col_attn=False, accept_edges=True)
        self.col_attn = AxialAttention(dim=dim, heads=heads, dim_head=dim_head, row_attn=False, col_attn=True)

    def update_(self, m, mask=None, pairwise_repr=None):
        self.row_attn.add_to_(m, pairwise_repr, mask)        # alphafold2.py:406
        self.col_attn.add_to_(m, None, mask)                 # alphafold2.py:407
        return m

    def forward(self, x, mask=None, pairwise_repr=None):
        _forward_only(x, pairwise_repr)
        with torch.no_grad():
            pr = pairwise_repr.detach().to(torch.float32).contiguous() if exists(pairwise_repr) else None
            return self.update_(_f32c(x), mask, pr).to(x.dtype)


class EvoformerBlock(nn.Module):
    def __init__(self, *, dim, seq_len, heads, dim_head, attn_dropout, ff_dropout, global_column_attn=False):
        super().__init__()
        self.layer = nn.ModuleList([
            PairwiseAttentionBlock(dim=dim, seq_len=seq_len, heads=heads, dim_head=dim_head, dropout=attn_dropout, global_column_attn=global_column_attn),
            FeedForward(dim=dim, dropout=ff_dropout),
            MsaAttentionBlock(dim=dim, seq_len=seq_len, heads=heads, dim_head=dim_head, dropout=attn_dropout),
            FeedForward(dim=dim, dropout=ff_dropout),
        ])

    def update_(self, x, m, mask, msa_mask, band=None, msa_band=None):
        """alphafold2.py:432-446 on private fp32 tensors, in place.  The pair track (pair block and transition) runs in bands
        of pair rows when the whole-tensor calls do not fit (PairwiseAttentionBlock.update_); `band` forces it (tests).
        When even the smallest pair bands do not fit beside the whole MSA track (deep MSAs), the MSA track runs in bands of
        MSA rows as well (banded.msa_track_, bitwise the same result); `msa_band` forces the MSA rows per band (tests: any
        positive integer).  The plan (ops.plan_block_bands) is made before any device work of the block; the bands used are
        kept in self.last_pair_band and self.last_msa_band (N and S: the whole-tensor calls)."""
        attn, ff, msa_attn, msa_ff = self.layer
        band, msa_band = _block_bands(attn, x, m.shape[1], band, msa_band)
        self.last_pair_band = band
        self.last_msa_band = msa_band
        if msa_band < m.shape[1]:
            mmk = msa_mask.bool().contiguous() if exists(msa_mask) else None
            for b in range(x.shape[0]):
                banded.msa_track_(msa_attn, msa_ff, m[b], None if mmk is None else mmk[b], x[b], msa_band, CudaStageOps())
        else:
            msa_attn.update_(m, msa_mask, x)
            msa_ff.add_to_(m)
        attn.update_(x, mask, m, msa_mask, band=band, msa_band=msa_band)
        if band < x.shape[1]:
            for b in range(x.shape[0]):
                banded.feed_forward_(ff, x[b], band, CudaStageOps())
        else:
            ff.add_to_(x)
        return x, m

    def forward(self, inputs):
        x, m, mask, msa_mask = inputs
        _forward_only(x, m)
        with torch.no_grad():
            xo, mo = self.update_(_f32c(x), _f32c(m), mask, msa_mask)
        return xo.to(x.dtype), mo.to(m.dtype), mask, msa_mask


class Evoformer(nn.Module):
    def __init__(self, *, depth, **kwargs):
        super().__init__()
        self.layers = nn.ModuleList([EvoformerBlock(**kwargs) for _ in range(depth)])

    def forward(self, x, m, mask=None, msa_mask=None):
        """x [b, N, N, d], m [b, S, N, d], mask [b, N, N] bool, msa_mask [b, S, N] bool -> (x, m).
        The reference's checkpoint_sequential(..., segments=1) is a plain sequential loop in forward."""
        _forward_only(x, m)
        with torch.no_grad():
            xo, mo = _f32c(x), _f32c(m)
            mk = mask.bool().contiguous() if exists(mask) else None
            mmk = msa_mask.bool().contiguous() if exists(msa_mask) else None
            for layer in self.layers:
                layer.update_(xo, mo, mk, mmk)
                self.last_pair_band = layer.last_pair_band
                self.last_msa_band = layer.last_msa_band
        return xo.to(x.dtype), mo.to(m.dtype)

    def run_(self, x, m, mask=None, msa_mask=None, band=None, msa_band=None):
        """Same as forward, for callers that own fp32 contiguous x / m and allow them to be updated in place (no private
        copies).  A sharded trunk (parallel.shard_evoformer replaces `forward`) goes through its schedule instead.
        `band` forces the pair rows and `msa_band` the MSA rows per band of every block (tests; see EvoformerBlock.update_);
        the bands the last block used are kept in self.last_pair_band and self.last_msa_band."""
        if "forward" in self.__dict__ or x.dtype != torch.float32 or m.dtype != torch.float32 or not (x.is_contiguous() and m.is_contiguous()):
            return self(x, m, mask=mask, msa_mask=msa_mask)
        with torch.no_grad():
            mk = mask.bool().contiguous() if exists(mask) else None
            mmk = msa_mask.bool().contiguous() if exists(msa_mask) else None
            for layer in self.layers:
                layer.update_(x, m, mk, mmk, band=band, msa_band=msa_band)
                self.last_pair_band = layer.last_pair_band
                self.last_msa_band = layer.last_msa_band
        return x, m


# ------------------------------------------------------------------------------------------------------
# Structure module (alphafold2.py:19, 608-615, 841-891): IPABlock of invariant-point-attention 0.2.x, attached explicitly
# ------------------------------------------------------------------------------------------------------
class InvariantPointAttention(nn.Module):
    """Parameters of invariant_point_attention.InvariantPointAttention(dim, heads): scalar keys / values of width 16, 4 point
    keys / values, the pair bias and to_out over [scalars | points (h p c) | point norms | pair aggregates].  It runs inside
    IPABlock's kernel calls (csrc/structure.cuh)."""

    def __init__(self, *, dim, heads=8, scalar_key_dim=16, scalar_value_dim=16, point_key_dim=4, point_value_dim=4, eps=1e-8):
        super().__init__()
        if (scalar_key_dim, scalar_value_dim, point_key_dim, point_value_dim, eps) != (16, 16, 4, 4, 1e-8):
            raise NotImplementedError("the kernels take the package defaults: scalar key / value width 16, 4 points, eps 1e-8")
        self.heads = heads
        self.to_scalar_q = nn.Linear(dim, scalar_key_dim * heads, bias=False)
        self.to_scalar_k = nn.Linear(dim, scalar_key_dim * heads, bias=False)
        self.to_scalar_v = nn.Linear(dim, scalar_value_dim * heads, bias=False)
        self.point_weights = nn.Parameter(torch.full((heads,), math.log(math.e - 1.)))     # softplus = 1 at init
        self.to_point_q = nn.Linear(dim, point_key_dim * heads * 3, bias=False)
        self.to_point_k = nn.Linear(dim, point_key_dim * heads * 3, bias=False)
        self.to_point_v = nn.Linear(dim, point_value_dim * heads * 3, bias=False)
        # index 1 of the package's Sequential is a parameter-free Rearrange('b ... h -> (b h) ...')
        self.to_pairwise_attn_bias = nn.Sequential(nn.Linear(dim, heads), nn.Identity())
        self.to_out = nn.Linear(heads * (scalar_value_dim + dim + point_value_dim * 4), dim)


class IPABlock(_Packable):
    """invariant_point_attention.IPABlock(dim, heads) in its post-norm form (the 0.2.x default):
    s = attn_norm(s + IPA(s, pair, R, t, mask)); s = ff_norm(s + ff(s)), ff = Linear -> ReLU -> Linear -> ReLU -> Linear.
    The package's parameter names and shapes, so a reference checkpoint with predict_coords=True loads strictly.  fp32 in both
    precision modes, as the reference runs it (alphafold2.py:854-859)."""

    def __init__(self, *, dim, ff_mult=1, ff_num_layers=3, post_norm=True, **kwargs):
        super().__init__()
        if (ff_mult, ff_num_layers, post_norm) != (1, 3, True):
            raise NotImplementedError("the kernels take the package defaults: ff_mult 1, 3 feed-forward layers, post-norm")
        self.attn_norm = nn.LayerNorm(dim)
        self.attn = InvariantPointAttention(dim=dim, **kwargs)
        self.ff_norm = nn.LayerNorm(dim)
        self.ff = nn.Sequential(nn.Linear(dim, dim), nn.ReLU(), nn.Linear(dim, dim), nn.ReLU(), nn.Linear(dim, dim))

    def _pack(self):
        return ops.pack_structure(self, None, None, None)

    def forward(self, x, *, pairwise_repr, rotations, translations, mask=None):
        """The package's call: x [b, n, d], pairwise_repr [b, n, n, d], rotations [b, n, 3, 3], translations [b, n, 3], mask [b, n]
        bool -> [b, n, d].  Alphafold2.forward runs the block through af2_structure_layer instead; this is the same kernels one
        call at a time."""
        _forward_only(x, pairwise_repr, rotations, translations)
        with torch.no_grad():
            t = self.packed().tensors
            heads = self.attn.heads
            s = _f32c(x)
            pair = pairwise_repr.detach().to(torch.float32).contiguous()
            rot = rotations.detach().to(torch.float32).contiguous()
            tr = translations.detach().to(torch.float32).contiguous()
            proj = ops.ipa_frames_(ops.structure_linear(s, t["w_proj"]), rot, tr, heads)
            feat = ops.ipa_attention(proj, pair, t["w_bias"], t["b_bias"], t["point_weights"], mask, rot, tr, heads)
            ops.structure_tail_(s, ops.structure_linear(feat, t["w_out"], t["b_out"]), t["attn_gamma"], t["attn_beta"],
                                self.attn_norm.eps)
            h = ops.structure_linear(ops.structure_linear(s, t["w_ff0"], t["b_ff0"], relu=True), t["w_ff2"], t["b_ff2"], relu=True)
            ops.structure_tail_(s, ops.structure_linear(h, t["w_ff4"], t["b_ff4"]), t["ff_gamma"], t["ff_beta"], self.ff_norm.eps)
            return s.to(x.dtype)


class _StructureWeights(_Packable):
    """Packed fp32 weights of af2_structure_layer: the attached ipa_block with the model's to_quaternion_update, to_points and
    lddt_linear.  Kept outside the module tree (like _AngleHeads), keyed on their parameters."""

    def __init__(self, block, qu, points, lddt):
        super().__init__()
        self.__dict__["mods"] = (block, qu, points, lddt)

    def parameters(self, recurse: bool = True):
        for mod in self.mods:
            yield from mod.parameters(recurse)

    def _pack(self):
        return ops.pack_structure(*self.mods)


class _PairProjection(_Packable):
    """trunk_to_pairwise_repr_dim packed for ops.pair_projection_: bf16, or split-bf16 when the model is in strict mode."""

    def __init__(self, lin):
        super().__init__()
        self.__dict__["lin"] = lin

    def parameters(self, recurse: bool = True):
        return self.lin.parameters(recurse)

    def _pack_key(self):
        return super()._pack_key() + (ops.precision_of(self.lin),)

    def _pack(self):
        return ops.pack_linear(self.lin.weight, self.lin.bias, strict=ops.precision_of(self.lin) == "strict")


NO_STRUCTURE_MODULE = (
    "predict_coords=True needs the structure module (IPABlock, alphafold2.py:19-20, 841-905), which the constructor leaves "
    "out because the reference's block is third-party: call alphafold2_b200.attach_structure_module(model) first")


def attach_structure_module(model: "Alphafold2") -> "Alphafold2":
    """Register model.ipa_block = IPABlock(dim=model.dim, heads=structure_module_heads) with ipa_block.attn.to_out zeroed
    (alphafold2.py:608-615), so that predict_coords=True runs and a reference predict_coords checkpoint loads strictly.  The
    constructor leaves it out because the reference's block is third-party.  A no-op when a block is attached.  Returns model."""
    if getattr(model, "ipa_block", None) is None:
        ref = next(model.parameters())
        block = IPABlock(dim=model.dim, heads=model.structure_module_heads).to(device=ref.device, dtype=ref.dtype)
        nn.init.zeros_(block.attn.to_out.weight)
        nn.init.zeros_(block.attn.to_out.bias)
        if "_af2_precision" in model.__dict__:
            ops.set_precision(block, model.__dict__["_af2_precision"])
        model.ipa_block = block
    return model



# ------------------------------------------------------------------------------------------------------
# Alphafold2 shell (alphafold2.py:469-905): constructor + distogram forward; trunk call at :802-807
# ------------------------------------------------------------------------------------------------------
class _MLMHead(nn.Module):
    """Parameter container for mlm.py:27-44 (``mlm.to_logits``); MLM noising/loss is training-only."""

    def __init__(self, dim, num_tokens):
        super().__init__()
        self.to_logits = nn.Linear(dim, num_tokens)


class Alphafold2(nn.Module):
    def __init__(
        self, *, dim, max_seq_len=2048, depth=6, heads=8, dim_head=64, max_rel_dist=32,
        num_tokens=NUM_AMINO_ACIDS, num_embedds=NUM_EMBEDDS_TR, max_num_msas=MAX_NUM_MSA,
        max_num_templates=MAX_NUM_TEMPLATES, extra_msa_evoformer_layers=4, attn_dropout=0., ff_dropout=0.,
        templates_dim=32, templates_embed_layers=4, templates_angles_feats_dim=55, predict_angles=False,
        symmetrize_omega=False, predict_coords=False, structure_module_depth=4, structure_module_heads=1,
        structure_module_dim_head=4, disable_token_embed=False, mlm_mask_prob=0.15,
        mlm_random_replace_token_prob=0.1, mlm_keep_token_same_prob=0.1, mlm_exclude_token_ids=(0,),
        recycling_distance_buckets=32
    ):
        super().__init__()
        self.dim = dim
        self.disable_token_embed = disable_token_embed
        self.token_emb = nn.Embedding(num_tokens + 1, dim) if not disable_token_embed else None
        self.to_pairwise_repr = nn.Linear(dim, dim * 2)
        self.max_rel_dist = max_rel_dist
        self.pos_emb = nn.Embedding(max_rel_dist * 2 + 1, dim)

        self.extra_msa_evoformer = Evoformer(dim=dim, depth=extra_msa_evoformer_layers, seq_len=max_seq_len, heads=heads,
                                             dim_head=dim_head, attn_dropout=attn_dropout, ff_dropout=ff_dropout,
                                             global_column_attn=True)
        self.to_template_embed = _TemplateEmbed(templates_dim, dim)
        self.templates_embed_layers = templates_embed_layers
        self.template_pairwise_embedder = PairwiseAttentionBlock(dim=dim, dim_head=dim_head, heads=heads, seq_len=max_seq_len)
        self.template_pointwise_attn = Attention(dim=dim, dim_head=dim_head, heads=heads, dropout=attn_dropout)
        self.template_angle_mlp = _TemplateAngleMLP(nn.Linear(templates_angles_feats_dim, dim), nn.GELU(), nn.Linear(dim, dim))

        self.predict_angles = predict_angles
        self.symmetrize_omega = symmetrize_omega
        if predict_angles:
            self.to_prob_theta = nn.Linear(dim, THETA_BUCKETS)
            self.to_prob_phi = nn.Linear(dim, PHI_BUCKETS)
            self.to_prob_omega = nn.Linear(dim, OMEGA_BUCKETS)

        self.embedd_project = nn.Linear(num_embedds, dim)
        self.net = Evoformer(dim=dim, depth=depth, seq_len=max_seq_len, heads=heads, dim_head=dim_head,
                             attn_dropout=attn_dropout, ff_dropout=ff_dropout)
        self.mlm = _MLMHead(dim, num_tokens)
        self.to_distogram_logits = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, DISTOGRAM_BUCKETS))

        self.predict_coords = predict_coords
        self.structure_module_depth = structure_module_depth
        self.structure_module_heads = structure_module_heads      # structure_module_dim_head: accepted, unused (as in the reference)
        self.msa_to_single_repr_dim = nn.Linear(dim, dim)
        self.trunk_to_pairwise_repr_dim = nn.Linear(dim, dim)
        # IPABlock (third-party invariant-point-attention, alphafold2.py:19,608-615) is not vendored by the reference, so the
        # default state_dict has no ipa_block.*: attach_structure_module(model) registers it (the package's layout).
        self.to_quaternion_update = nn.Linear(dim, 6)
        self.to_points = nn.Linear(dim, 3)
        self.lddt_linear = nn.Linear(dim, 1)
        self.recycling_msa_norm = nn.LayerNorm(dim)
        self.recycling_pairwise_norm = nn.LayerNorm(dim)
        self.recycling_distance_embed = nn.Embedding(recycling_distance_buckets, dim)
        self.recycling_distance_buckets = recycling_distance_buckets
        self._warned_training = False

    def angle_heads(self) -> _AngleHeads:
        """The packed-weight cache of to_prob_theta / to_prob_phi / to_prob_omega (predict_angles=True only)."""
        ah = self.__dict__.get("_angle_heads")
        if ah is None or ah.heads != (self.to_prob_theta, self.to_prob_phi, self.to_prob_omega):
            ah = _AngleHeads(self.to_prob_theta, self.to_prob_phi, self.to_prob_omega)
            self.__dict__["_angle_heads"] = ah
        return ah

    def _check_templates(self, seq, mask, templates_feats, templates_mask, templates_angles):
        """The template inputs the reference cannot handle crash it inside einops / torch.cat; here they raise ValueError up
        front, before any device work."""
        b, n = seq.shape[:2]
        if exists(templates_feats):
            if not exists(mask):
                raise ValueError("templates_feats needs `mask`: the pointwise template attention masks with the pair mask "
                                 "(alphafold2.py:767; the reference fails in einops without it)")
            if not exists(templates_mask):
                raise ValueError("templates_feats needs templates_mask [b, T, n] (alphafold2.py:752)")
            if templates_feats.dim() != 5 or templates_feats.shape[0] != b or tuple(templates_feats.shape[2:4]) != (n, n):
                raise ValueError(f"templates_feats must be [{b}, T, {n}, {n}, templates_dim], got {tuple(templates_feats.shape)}")
            if tuple(templates_mask.shape) != tuple(templates_feats.shape[:3]):
                raise ValueError(f"templates_mask must be {tuple(templates_feats.shape[:3])}, got {tuple(templates_mask.shape)}")
        if exists(templates_angles):
            if not exists(templates_mask):
                raise ValueError("templates_angles needs templates_mask [b, T, n]: it is appended to msa_mask (alphafold2.py:792)")
            if templates_angles.dim() != 4 or templates_angles.shape[0] != b or templates_angles.shape[2] != n:
                raise ValueError(f"templates_angles must be [{b}, T, {n}, angle_feats], got {tuple(templates_angles.shape)}")
            if tuple(templates_mask.shape) != tuple(templates_angles.shape[:3]):
                raise ValueError(f"templates_mask must be {tuple(templates_angles.shape[:3])}, got {tuple(templates_mask.shape)}")

    def template_pair_stack(self, templates_feats, templates_mask, band=None):
        """alphafold2.py:751-760: t = to_template_embed(feats) -> [b * T, n, n, d] fp32, then templates_embed_layers passes of
        the SAME template_pairwise_embedder (shared weights, no OuterMean) under the crossed mask.  Returns (t, crossed mask).
        `band` forces the pair rows per band of the pair blocks (PairwiseAttentionBlock.update_)."""
        b, T, n = templates_feats.shape[:3]
        tm = templates_mask.bool()
        tm2 = (tm[:, :, :, None] & tm[:, :, None, :]).reshape(b * T, n, n).contiguous()
        t = self.to_template_embed.embed(templates_feats.detach().float().contiguous()).reshape(b * T, n, n, -1)
        for _ in range(self.templates_embed_layers):
            self.template_pairwise_embedder.update_(t, tm2, band=band)
        return t, tm2

    def _template_plan(self, x, templates_feats, group, band):
        """(G, band) of embed_templates_; band = n is the whole-tensor path.  Strict mode (a parity mode) is never banded."""
        b, T = templates_feats.shape[:2]
        n, d = x.shape[1], x.shape[3]
        attn = self.template_pointwise_attn
        strict = ops.precision_of(attn) == "strict"
        if band is not None and not strict and int(band) < n and (int(band) <= 0 or int(band) % 8):
            raise ValueError(f"template band {band} must be a positive multiple of 8")
        forced = band is not None and not strict
        band = min(int(band), n) if forced else n
        if group is None and forced and band < n:
            group = 1                                    # forced bands: one template at a time, as the planner bands
        elif group is None:
            # 15 % headroom: the caching allocator cannot always reuse the blocks it frees (a growing workspace is allocated
            # before the old one is released); plans right at the limit ran out of memory at N_res 1024 and 2048 on an H100
            budget = int(ops.device_budget(x.device) * 0.85)
            plan = (b, T, n, d, attn.heads, attn.dim_head, ops.precision_of(attn), budget, templates_feats.shape[-1])
            if forced:
                group = ops.plan_template_groups(*plan)
            else:
                group, band = ops.plan_template_branch(*plan)
        return max(1, min(int(group), T)), band

    def embed_templates_(self, x, x_mask, templates_feats, templates_mask, group=None, band=None):
        """alphafold2.py:743-785 in place on the fp32 pair tensor x [b, n, n, d]: template pair stack, then the pointwise
        attention of every pair over its T templates, scaled by `any template valid` and added to x.  Under shard_evoformer
        every rank computes this whole (it runs before the sharded trunk); parallel.shard_alphafold2 shards it instead.

        The templates run in groups of G: each group's pair stack at batch b * G, then its step of the pointwise attention,
        whose online softmax carries over to the next group.  The result does not depend on G (bitwise), only the memory does:
        G = T when the whole branch fits what the device can still allocate (ops.plan_template_groups), fewer otherwise.
        `group` forces G (tests).  The G used is kept in self.last_template_group.

        When not even one template fits (bf16 mode), the pointwise attention runs in bands of pair rows as well
        (ops.plan_template_branch, ops.TemplateAttentionGroups with band): per group the pair stack, in the same bands, then
        per batch element and band q and gate of the band's rows of x, the group's k|v of those rows and the state-carrying kernel,
        and after the last group to_out into the band's rows of x.  Only the softmax state is kept for every pair; the result
        is bitwise the same.  `band` forces the rows per band (tests: a positive multiple of 8).  The band used is kept in
        self.last_template_band (n: the whole-tensor calls)."""
        T = templates_feats.shape[1]
        n = x.shape[1]
        attn = self.template_pointwise_attn
        G, band = self._template_plan(x, templates_feats, group, band)
        self.last_template_group = G
        self.last_template_band = band
        if G == T and band == n:
            t, tm2 = self.template_pair_stack(templates_feats, templates_mask)
            attn.add_context_(x, t, x_mask, tm2)
            return x
        if band < n:
            ops.release_workspace(x.device)          # the plan counted it as free: the softmax state may need its memory
        stack_band = band if band < n else None          # None: the pair stack keeps its own band planner
        acc = ops.TemplateAttentionGroups(attn.packed(), x, x_mask, attn.heads, attn.dim_head, stack_band)
        for t0 in range(0, T, G):
            t1 = min(t0 + G, T)
            t, tm2 = self.template_pair_stack(templates_feats[:, t0:t1], templates_mask[:, t0:t1], band=stack_band)
            acc.add(t, tm2, last=t1 == T)
            del t, tm2                                   # free this group's t before the next one is embedded
        return x

    def _embed_templates_reused_(self, x, x_mask, templates_feats, templates_mask, cache, stack_rows):
        """embed_templates_ for the iterations of recycle(), which share templates_feats and templates_mask.  The pair stack
        reads neither x nor the recyclables, so on the first iteration, when the branch runs whole (G = T, band = n) and
        ops.template_reuse_fits says that t and the crossed mask fit beside the whole-tensor plan of every later pair stack
        (stack_rows: their MSA rows), they are kept in `cache`; later iterations run only the pointwise attention on them,
        which only reads t.  Otherwise every iteration runs embed_templates_.  The decision is kept in self.last_template_reuse."""
        if "t" not in cache:
            b, T, n = templates_feats.shape[:3]
            G, band = self._template_plan(x, templates_feats, None, None)
            tri = self.template_pairwise_embedder.triangle_attention_ingoing.attn
            budget = int(ops.device_budget(x.device) * 0.85)         # the planners' headroom (_template_plan, _pair_band)
            keep = G == T and band == n and ops.template_reuse_fits(b, T, n, x.shape[3], tri.heads, tri.dim_head, stack_rows,
                                                                     budget)
            self.last_template_reuse = keep
            cache["t"] = self.template_pair_stack(templates_feats, templates_mask) if keep else None
            if keep:
                self.last_template_group, self.last_template_band = T, n
        if cache["t"] is None:
            return self.embed_templates_(x, x_mask, templates_feats, templates_mask)
        t, tm2 = cache["t"]
        return self.template_pointwise_attn.add_context_(x, t, x_mask, tm2)

    def _check_recyclables(self, b, n, device, recyclables, pair_rows=None):
        """Duck-typed like the reference (alphafold2.py:730-739 reads three attributes): its Recyclables and ours are both
        accepted.  Returns (coords, single_msa_repr_row, pairwise_repr); raises before any device work.  pair_rows: pairwise_repr
        may also be only a rank's pair rows [b, pair_rows, n, d] (parallel.shard_alphafold2(pair_rows=True))."""
        fields = ("coords", "single_msa_repr_row", "pairwise_repr")
        ts = tuple(getattr(recyclables, f, None) for f in fields)
        if not all(torch.is_tensor(t) for t in ts):
            raise NotImplementedError(f"recyclables must carry tensors {', '.join(fields)} (alphafold2.py:24-28); "
                                      f"got {type(recyclables).__name__}")
        coords, single, pair = ts
        pair_lead = (b, n, n, self.dim)
        if pair_rows is not None and pair.dim() == 4 and tuple(pair.shape) == (b, pair_rows, n, self.dim):
            pair_lead = tuple(pair.shape)
        expect = {"coords": (coords, 3, (b, n)), "single_msa_repr_row": (single, 3, (b, n, self.dim)),
                  "pairwise_repr": (pair, 4, pair_lead)}
        for name, (t, rank, lead) in expect.items():
            if t.dim() != rank or tuple(t.shape[:len(lead)]) != lead or (name == "coords" and t.shape[-1] < 1):
                want = f"[{b}, {n}, c]" if name == "coords" else str(list(lead))
                if name == "pairwise_repr" and pair_rows is not None:
                    want += f" or this rank's rows {[b, pair_rows, n, self.dim]}"
                raise ValueError(f"recyclables.{name} must be {want}, got {tuple(t.shape)}")
            if not torch.is_floating_point(t):
                raise ValueError(f"recyclables.{name} must be a floating tensor, got {t.dtype}")
            if t.device != device:
                raise ValueError(f"recyclables.{name} is on {t.device}, seq on {device}")
        return ts

    def embed_recyclables_(self, x, m, recyclables, row0=None):
        """alphafold2.py:730-739 in place on the fp32 pair tensor x [b, n, n, d] and row 0 of m [b, rows, n, d], one kernel:
        x += LN(pairwise_repr), then += recycling_distance_embed[bucket(|coords_i - coords_j|)]; m[:, 0] += LN(single_msa_repr_row).
        Masks do not gate it (as in the reference).  Under shard_evoformer every rank computes it whole (it runs before the trunk).
        row0: x holds only pair rows [row0, row0 + rows) ([b, rows, n, d]; parallel.shard_alphafold2(pair_rows=True)), and only
        those rows of pairwise_repr are read; pairwise_repr may then be the whole [b, n, n, d] or those rows [b, rows, n, d]."""
        n = x.shape[1] if row0 is None else x.shape[2]
        ts = self._check_recyclables(x.shape[0], n, x.device, recyclables, pair_rows=None if row0 is None else x.shape[1])
        if row0 is not None and ts[2].shape[1] != x.shape[1]:
            ts = (ts[0], ts[1], ts[2][:, row0:row0 + x.shape[1]])
        coords, single, pair = (t.detach().to(torch.float32).contiguous() for t in ts)
        args = (coords, single, pair, self.recycling_msa_norm.weight, self.recycling_msa_norm.bias, self.recycling_pairwise_norm.weight,
                self.recycling_pairwise_norm.bias, self.recycling_distance_embed.weight)
        if row0 is None:
            ops.recycle_embed_(x, m, *args, eps=self.recycling_pairwise_norm.eps)
        else:
            ops.recycle_embed_rows_(x, m, *args, row0, eps=self.recycling_pairwise_norm.eps)
        return x, m

    def _check_inputs(self, seq, mask, seq_embed, msa_embed, embedds, templates_feats, templates_mask, templates_angles, recyclables):
        """The checks forward makes before any device work."""
        assert not (self.disable_token_embed and not exists(seq_embed)), 'sequence embedding must be supplied if one has disabled token embedding'
        assert not (self.disable_token_embed and not exists(msa_embed)), 'msa embedding must be supplied if one has disabled token embedding'
        _forward_only(seq_embed, msa_embed, embedds, templates_feats, templates_angles)
        if exists(recyclables):
            _forward_only(*self._check_recyclables(seq.shape[0], seq.shape[1], seq.device, recyclables))
        self._check_templates(seq, mask, templates_feats, templates_mask, templates_angles)
        if self.training and not self._warned_training:
            warnings.warn("alphafold2_b200 is forward-only: running inference semantics (no MLM noising, no autograd)")
            self._warned_training = True

    def embed_template_angles_(self, m, msa_mask, templates_angles, templates_mask):
        """alphafold2.py:787-792: template_angle_mlp into the T rows of m after its S MSA rows; returns msa_mask with the
        templates' rows appended."""
        S = m.shape[1] - templates_angles.shape[1]
        self.template_angle_mlp.write_(templates_angles.detach().float().contiguous(), m, S)
        return torch.cat((msa_mask.bool(), templates_mask.bool()), dim=1)

    def extra_msa_inputs(self, msa, extra_msa_mask):
        """alphafold2.py:789-798, reproduced WITH its quirks (SURVEY.md Q11, do not "fix"): the extra-MSA stack embeds `msa`, not
        `extra_msa` (:790); only its pair output is kept; the default mask torch.ones_like(extra_m) has the embedding's rank and
        makes the reference fail in its first mask fold -- same here (ValueError).  Returns (extra_m, extra mask)."""
        extra_m = self.token_emb(msa).float().contiguous()
        em = extra_msa_mask if exists(extra_msa_mask) else torch.ones_like(extra_m).bool()
        if em.dim() != 3:
            raise ValueError("extra_msa_mask must be given with shape [b, n_msa, n] (the reference's default, "
                             "alphafold2.py:791, has the wrong rank and fails in einops too)")
        return extra_m, em

    def forward(
        self, seq, msa=None, mask=None, msa_mask=None, extra_msa=None, extra_msa_mask=None, seq_index=None,
        seq_embed=None, msa_embed=None, templates_feats=None, templates_mask=None, templates_angles=None,
        embedds=None, recyclables=None, return_trunk=False, return_confidence=False, return_recyclables=False,
        return_aux_logits=False
    ):
        return self._forward(seq, msa, mask, msa_mask, extra_msa, extra_msa_mask, seq_index, seq_embed, msa_embed, templates_feats,
                             templates_mask, templates_angles, embedds, recyclables, return_trunk, return_confidence,
                             return_recyclables, return_aux_logits)

    def _forward(
        self, seq, msa=None, mask=None, msa_mask=None, extra_msa=None, extra_msa_mask=None, seq_index=None,
        seq_embed=None, msa_embed=None, templates_feats=None, templates_mask=None, templates_angles=None,
        embedds=None, recyclables=None, return_trunk=False, return_confidence=False, return_recyclables=False,
        return_aux_logits=False, *, owned=None, template_cache=None
    ):
        """forward, with the two hooks of recycle() (both None in forward):
          owned: a one-element list [recyclables] given instead of `recyclables`, whose tensors the caller references nowhere
            else.  The list is emptied before this iteration's x and m exist, after a copy of single_msa_repr_row (a view of the
            previous MSA tensor, which is freed then); the pair tensor and coordinates are dropped once embed_recyclables_ has
            read them, before the templates, the extra-MSA stack and the trunk run.
          template_cache: a dict kept across the iterations of one prediction (_embed_templates_reused_)."""
        if owned is not None:
            recyclables = owned[0]
        self._check_inputs(seq, mask, seq_embed, msa_embed, embedds, templates_feats, templates_mask, templates_angles, recyclables)

        with torch.no_grad():
            if owned is not None and exists(recyclables):
                recyclables = Recyclables(recyclables.coords, recyclables.single_msa_repr_row.clone(), recyclables.pairwise_repr)
                owned.clear()
            if not exists(msa):                                        # alphafold2.py:656-658
                msa = seq[:, None, :]
                msa_mask = mask[:, None, :] if exists(mask) else None
            assert msa.shape[-1] == seq.shape[-1], 'sequence length of MSA and primary sequence must be the same'
            b, n = seq.shape[:2]
            device = seq.device

            fused_glue = seq.is_cuda and not self.disable_token_embed and exists(msa)
            if fused_glue:
                # alphafold2.py:676-726 as fused kernels (SURVEY.md 8f n1): embedding gather, m = emb[msa] + emb[seq], pair init
                if not exists(msa_mask):
                    msa_mask = torch.ones_like(msa).bool()
                # with template angles, m gets the T angle rows after the S MSA rows (alphafold2.py:789-790): allocated here at once
                m_rows = msa.shape[1] + (templates_angles.shape[1] if exists(templates_angles) else 0)
                x, m = ops.embed_pair_init(seq, msa, self.token_emb.weight, self.to_pairwise_repr.weight, self.to_pairwise_repr.bias,
                                           self.pos_emb.weight, self.max_rel_dist, seq_embed, msa_embed, seq_index, m_rows=m_rows)
            else:
                x = self.token_emb(seq) if not self.disable_token_embed else 0
                if exists(seq_embed):
                    x = x + seq_embed
                if exists(msa):
                    m = self.token_emb(msa) if not self.disable_token_embed else 0
                    if exists(msa_embed):
                        m = m + msa_embed
                    m = m + x[:, None]
                    if not exists(msa_mask):
                        msa_mask = torch.ones_like(msa).bool()
                elif exists(embedds):
                    m = self.embedd_project(embedds)
                    if not exists(msa_mask):
                        msa_mask = torch.ones_like(embedds[..., -1]).bool()

                x_left, x_right = self.to_pairwise_repr(x).chunk(2, dim=-1)
                x = x_left[:, :, None, :] + x_right[:, None, :, :]
                seq_index = seq_index if exists(seq_index) else torch.arange(n, device=device)
                rel = (seq_index[None, :, None] - seq_index[None, None, :]).clamp(-self.max_rel_dist, self.max_rel_dist) + self.max_rel_dist
                x = x + self.pos_emb(rel)
                x, m = x.float().contiguous(), m.float().contiguous()
                if exists(templates_angles):
                    m = torch.cat((m, m.new_empty(m.shape[0], templates_angles.shape[1], *m.shape[2:])), dim=1)
            x_mask = (mask[:, :, None] & mask[:, None, :]) if exists(mask) else None

            if exists(recyclables):                                    # alphafold2.py:730-739, before the templates read x
                self.embed_recyclables_(x, m, recyclables)
                if owned is not None:
                    recyclables = None
            if exists(templates_feats) and template_cache is not None:
                self._embed_templates_reused_(x, x_mask, templates_feats, templates_mask, template_cache,
                                              (m.shape[1],) + ((msa.shape[1],) if exists(extra_msa) else ()))
            elif exists(templates_feats):                              # alphafold2.py:743-785
                self.embed_templates_(x, x_mask, templates_feats, templates_mask)
            if exists(templates_angles):                               # alphafold2.py:787-792
                msa_mask = self.embed_template_angles_(m, msa_mask, templates_angles, templates_mask)

            if exists(extra_msa):                                      # alphafold2.py:789-798
                extra_m, em = self.extra_msa_inputs(msa, extra_msa_mask)
                x, _ = self.extra_msa_evoformer.run_(x.contiguous(), extra_m, mask=x_mask, msa_mask=em)

            x_trunk_in = x
            x, m = self.net.run_(x, m, mask=x_mask, msa_mask=msa_mask)     # alphafold2.py:802-807

            ret = ReturnValues()
            fused_angles = self.predict_angles and x.is_cuda and x.dtype == torch.float32 and \
                ops.angle_heads_ok(x.shape[-1], self.angle_heads().buckets())
            if self.predict_angles and not fused_angles:
                ret.theta_logits = self.to_prob_theta(x)
                ret.phi_logits = self.to_prob_phi(x)
            ln, lin = self.to_distogram_logits[0], self.to_distogram_logits[1]
            if x.is_cuda and x.dtype == torch.float32 and ops.distogram_head_ok(x.shape[-1], lin.weight.shape[0]):
                # alphafold2.py:821-823 in one kernel: symmetrise + LayerNorm + Linear(d -> 37)
                ret.distance = ops.distogram_head(x.contiguous(), ln.weight, ln.bias, lin.weight, lin.bias)
                trunk_embeds = None
            else:
                trunk_embeds = (x + x.transpose(1, 2)) * 0.5
                ret.distance = self.to_distogram_logits(trunk_embeds)
            if fused_angles:
                # alphafold2.py:813-836 in one kernel that reads x once: omega's (x + x^T) / 2 is formed on chip
                ret.theta_logits, ret.phi_logits, ret.omega_logits = self.angle_heads().run(x.contiguous(), self.symmetrize_omega)
            elif self.predict_angles:
                if self.symmetrize_omega and trunk_embeds is None:
                    trunk_embeds = (x + x.transpose(1, 2)) * 0.5
                ret.omega_logits = self.to_prob_omega(trunk_embeds if self.symmetrize_omega else x)
            if not self.predict_coords or return_trunk:
                return ret
            if getattr(self, "ipa_block", None) is not None:
                return self._structure_module(x, m, mask, ret, x_private=x is x_trunk_in, return_confidence=return_confidence,
                                              return_recyclables=return_recyclables, return_aux_logits=return_aux_logits)
        raise NotImplementedError(NO_STRUCTURE_MODULE)

    def structure_weights(self) -> _StructureWeights:
        """The packed-weight cache of the attached ipa_block with to_quaternion_update, to_points and lddt_linear."""
        sw = self.__dict__.get("_structure_weights")
        mods = (self.ipa_block, self.to_quaternion_update, self.to_points, self.lddt_linear)
        if sw is None or sw.mods != mods:
            sw = _StructureWeights(*mods)
            self.__dict__["_structure_weights"] = sw
        return sw

    def pair_projection(self) -> _PairProjection:
        pp = self.__dict__.get("_pair_projection")
        if pp is None or pp.lin is not self.trunk_to_pairwise_repr_dim:
            pp = _PairProjection(self.trunk_to_pairwise_repr_dim)
            self.__dict__["_pair_projection"] = pp
        return pp

    def _structure_module(self, x, m, mask, ret, x_private, return_confidence, return_recyclables, return_aux_logits):
        """alphafold2.py:841-905 on the trunk's x [b, n, n, d] and m [b, rows, n, d].  pairwise_repr is written over x when x is this
        forward's own buffer (the heads have read it; ops.pair_projection_ works in bands of pair rows through one scratch band),
        else into a fresh tensor.  Under shard_evoformer / shard_alphafold2 every rank holds the whole x and runs this whole."""
        b, n, _, d = x.shape
        heads = self.ipa_block.attn.heads
        ops._check_ipa_shape(b, n, heads, d)                                   # before any device work of the module
        single_msa_repr_row = m[:, 0]                                          # :845
        single = ops.structure_linear(single_msa_repr_row.contiguous(), self.msa_to_single_repr_dim.weight,
                                      self.msa_to_single_repr_dim.bias)        # :847
        x = x.contiguous()
        pair = ops.pair_projection_(self.pair_projection().packed(), x, out=x if x_private else torch.empty_like(x))   # :848
        quat, trans, rot, coords, confidence = structure_frames(b, n, x.device)
        mk = mask.bool() if exists(mask) else None
        depth = self.structure_module_depth
        pk = self.structure_weights().packed()
        for i in range(depth):                                                 # :872-885, the same ipa_block each layer
            last = i == depth - 1
            ops.structure_layer_(pk, single, pair, mk, quat, trans, rot, coords if last else None, confidence if last else None)
        if depth == 0:                                                         # :889-891 with q = (1, 0, 0, 0), t = 0
            ops.structure_linear(single, self.to_points.weight, self.to_points.bias, out=coords)
            ops.structure_linear(single, self.lddt_linear.weight, self.lddt_linear.bias, out=confidence)
        return structure_result(ret, coords, confidence, single_msa_repr_row, pair, return_confidence, return_recyclables,
                                return_aux_logits)


def structure_frames(b: int, n: int, device):
    """alphafold2.py:863-868: q = (1, 0, 0, 0), t = 0 per residue and R = quat_to_matrix(q) = I, with the coords [b, n, 3] and
    confidence [b, n, 1] buffers of the last layer: (quat, trans, rot, coords, confidence), fp32."""
    quat = torch.zeros(b, n, 4, dtype=torch.float32, device=device)
    quat[..., 0] = 1.
    trans = torch.zeros(b, n, 3, dtype=torch.float32, device=device)
    rot = torch.eye(3, dtype=torch.float32, device=device).repeat(b, n, 1, 1)
    coords = torch.empty(b, n, 3, dtype=torch.float32, device=device)
    confidence = torch.empty(b, n, 1, dtype=torch.float32, device=device)
    return quat, trans, rot, coords, confidence


def structure_result(ret, coords, confidence, single_msa_repr_row, pairwise_repr, return_confidence, return_recyclables,
                     return_aux_logits):
    """What Alphafold2.forward returns after the structure module (alphafold2.py:893-905), in the reference's precedence."""
    # :893 coords.type(original_dtype) is a no-op: coords stay fp32
    if return_recyclables:                                                     # :895-897
        ret.recyclables = Recyclables(coords, single_msa_repr_row, pairwise_repr)
    if return_aux_logits:                                                      # :899-900
        return coords, ret
    if return_confidence:                                                      # :902-903
        return coords, confidence
    return coords                                                              # :905 (return_recyclables alone: just coords)


def recycle(model: Alphafold2, seq, msa=None, *, num_recycles: int = 3, **forward_kwargs):
    """AlphaFold inference with recycling: what the last call of

        coords, ret = model(seq, msa, **kw, return_aux_logits=True, return_recyclables=True)
        for _ in range(num_recycles):
            coords, ret = model(seq, msa, **kw, recyclables=ret.recyclables, return_aux_logits=True, return_recyclables=True)

    returns, bitwise, where the caller's return_* flags in forward_kwargs (Alphafold2.forward's keyword arguments, an initial
    `recyclables` included) apply to the last call only.  num_recycles = 0 is one model(seq, msa, **forward_kwargs) call.

    On one GPU the loop does less than the one above, with the same bits:
      * the template pair stack runs once, when its output fits beside the later stages' whole-tensor plans
        (Alphafold2._embed_templates_reused_, ops.template_reuse_fits), and again on every iteration otherwise;
      * each iteration's recyclables (the pair tensor, the coordinates, the MSA tensor behind single_msa_repr_row) and heads'
        outputs are freed as soon as the next iteration's recycling embedder has read them, so the trunk of that iteration
        runs without a second pair tensor beside it.
    Sharded models do the same:
      * under parallel.shard_evoformer(model) the template branch runs whole on every rank, as on one GPU, and the reuse
        rule above applies on each rank;
      * under parallel.shard_alphafold2(model), default and pair_rows=True, each rank keeps its rows of every template's pair
        stack output (parallel.sharded_embed_templates_) when parallel.template_reuse_rows_fits allows it on every rank of the
        group (the ranks reduce their decisions, so they all take the same branch), and later iterations run only the
        pointwise attention over the kept rows; the recyclables (in pair_rows mode the rank's pair rows) are freed as above.
    The decision is kept in model.last_template_reuse.

    Refused before any device work: num_recycles < 0, and with num_recycles >= 1: predict_coords=False, return_trunk=True
    (no coordinates to recycle; ValueError) and an unattached structure module (NotImplementedError)."""
    if isinstance(num_recycles, bool) or not isinstance(num_recycles, int) or num_recycles < 0:
        raise ValueError(f"num_recycles must be a non-negative integer, got {num_recycles!r}")
    if num_recycles == 0:
        return model(seq, msa, **forward_kwargs)
    if not model.predict_coords:
        raise ValueError("recycling feeds back the structure module's coordinates: it needs Alphafold2(predict_coords=True)")
    if forward_kwargs.get("return_trunk", False):
        raise ValueError("return_trunk=True returns before the structure module, so there is nothing to recycle")
    if getattr(model, "ipa_block", None) is None:
        raise NotImplementedError(NO_STRUCTURE_MODULE)
    flags = ("return_confidence", "return_recyclables", "return_aux_logits")
    last_flags = {k: forward_kwargs.pop(k, False) for k in flags}
    inner = dict(return_recyclables=True, return_aux_logits=True)
    rec = forward_kwargs.pop("recyclables", None)
    held, cache = [rec], {}
    del rec
    # model._forward is Alphafold2._forward, or sharded_alphafold2_rows under shard_alphafold2(pair_rows=True)
    for _ in range(num_recycles):
        # only `held` references the recyclables: _forward empties it once they are read (the heads' outputs go with the tuple)
        held = [model._forward(seq, msa, owned=held, template_cache=cache, **inner, **forward_kwargs)[1].recyclables]
    return model._forward(seq, msa, owned=held, template_cache=cache, **last_flags, **forward_kwargs)
