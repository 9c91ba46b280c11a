"""The pair track of one Evoformer block in bands of pair rows, one band at a time on one GPU.

A block's whole-tensor calls each take one workspace for the whole [N, N, d] pair tensor; the largest (axial attention,
5.6 KB per pair token at d 256, 8 heads of 64) outgrows an 80 GB card near N_res 3,400.  Run band by band, a stage needs
its workspace for one band only, and the stages keep between bands just what the dependencies force:

  outer mean         m projected once (left | right, channel-major); per band its left operand's columns and
                     af2_outer_contract(row0, rows), which computes the band's normaliser rows itself
  triangle multiply  L, R and the output gate of EVERY band first (they all read the pre-update x), into whole-tensor
                     operands; then the contraction band by band.  Outgoing: the band's rows of L against all of R.
                     Ingoing: all of L against the column window R[c][k][i0:i1] (af2_triangle_contract_pitched)
  row attention      the pair bias of the whole x once, before any band updates x; then each row band
  column attention   the bias once; per column band a compact copy of x[:, j0:j1] (and its mask), attended and copied back
  pair transition    per row band (pointwise)

With band boundaries on multiples of ops.PAIR_BAND_ALIGN every band call picks the same GEMM tile and channel-to-token
kernel as the whole-tensor call, and every kernel computes an output element from the same inputs in the same order: the
result is bitwise that of the whole-tensor schedule.  No FLOP is added.

For deep MSAs the MSA track runs in bands of MSA rows as well (msa_track_): row attention per row band, column attention per
column band after the last row band, the transition per row band, and the outer mean's projection per chunk of MSA rows.

`ops` is the stage-op provider (parallel.CudaStageOps, the C ABI); tests/ drive the same schedule with oracle stage ops.
"""
from __future__ import annotations

from typing import Optional

import torch


def _bands(N: int, band: int):
    return [(i0, min(i0 + band, N)) for i0 in range(0, N, band)]


def _align8(n: int) -> int:
    return (n + 7) // 8 * 8


def _col_window(t: torch.Tensor, i0: int, i1: int) -> torch.Tensor:
    """t[..., i0:i1] as a contiguous operand with the zero-padded pitch align8(i1 - i0) the kernels read."""
    out = t.new_zeros(*t.shape[:-1], _align8(i1 - i0))
    out[..., :i1 - i0] = t[..., i0:i1]
    return out


def msa_column_band(S: int, N: int, rows: int) -> int:
    """Columns per band of the MSA column attention when the MSA track runs in bands of `rows` MSA rows: the same token budget
    as a row band (the largest multiple of 8 with S * C <= rows * N), at least 8 and at most N."""
    return min(N, max(8, rows * N // max(S, 1) // 8 * 8))


def msa_track_(msa_attn, msa_ff, m: torch.Tensor, msa_mask: Optional[torch.Tensor], x: torch.Tensor, rows: int, ops) -> torch.Tensor:
    """MsaAttentionBlock.update_ and the MSA transition (alphafold2.py:438-439) on ONE batch element in bands of `rows` MSA rows,
    in place.  m [S, N, d] fp32 contiguous, msa_mask [S, N] bool or None, x [N, N, d] the pair tensor (unchanged here).

      row attention      the pair bias of x once (x does not change during the MSA track); then each row band m[s0:s1]
      column attention   only after the last row band; per column band a compact copy of m[:, j0:j1] (and its mask), attended
                         without bias and copied back; C columns per band (msa_column_band)
      MSA transition     per row band (pointwise)

    Every band call picks the whole-tensor call's GEMM tiles (they depend on the output width only), so the result is bitwise
    that of the whole-tensor calls for any `rows`."""
    S, N, _ = m.shape
    ra, ca = msa_attn.row_attn, msa_attn.col_attn
    bias = ops.pair_bias(ra, x)
    for s0, s1 in _bands(S, rows):
        ops.axial_attention_(ra, m[s0:s1], bias, None if msa_mask is None else msa_mask[s0:s1], True)
    del bias
    for j0, j1 in _bands(N, msa_column_band(S, N, rows)):
        mc = m[:, j0:j1].contiguous()
        ops.axial_attention_(ca, mc, None, None if msa_mask is None else msa_mask[:, j0:j1].contiguous(), False)
        m[:, j0:j1] = mc
    return feed_forward_(msa_ff, m, rows, ops)


def outer_project_(om, m: torch.Tensor, msa_mask: Optional[torch.Tensor], rows: Optional[int], ops) -> torch.Tensor:
    """The outer mean's projected left | right operand of m [S, N, d]: [2d, S, pitch(N)] channel-major.  With rows < S it is
    projected in chunks of `rows` MSA rows, each into LR[:, s0:s1] with LR's channel stride: the projection's workspace then
    holds one chunk instead of all of m.  Projection is per token, so any chunking gives the same bits."""
    S, N, d = m.shape
    if rows is None or rows >= S:
        return ops.outer_project(om, m, msa_mask)
    LR = ops.outer_operand(S, N, d, m)
    for s0, s1 in _bands(S, rows):
        ops.outer_project(om, m[s0:s1], None if msa_mask is None else msa_mask[s0:s1], out=LR[:, s0:s1])
    return LR


def outer_mean_(om, x: torch.Tensor, m: torch.Tensor, msa_mask: Optional[torch.Tensor], rows: int, ops) -> torch.Tensor:
    """OuterMean.add_to_ on ONE batch element with the pair rows whole and m projected in chunks of `rows` MSA rows
    (outer_project_), then one contraction over all N pair rows."""
    d = x.shape[-1]
    LR = outer_project_(om, m, msa_mask, rows, ops)
    ops.outer_contract_(om, x, LR[:d], LR[d:], msa_mask, 0, 1)
    return x


def pair_block_(pair, x: torch.Tensor, mask: Optional[torch.Tensor], m: Optional[torch.Tensor], msa_mask: Optional[torch.Tensor],
                band: int, ops, msa_rows: Optional[int] = None) -> torch.Tensor:
    """PairwiseAttentionBlock.update_ (alphafold2.py:378-385) on ONE batch element in bands of `band` pair rows, in place.
    x [N, N, d] fp32 contiguous, mask [N, N] bool or None, m [S, N, d] / msa_mask [S, N] or None (no outer mean).
    msa_rows: project m for the outer mean in chunks of this many MSA rows (outer_project_); None: whole."""
    N, _, d = x.shape
    bands = _bands(N, band)
    rows_mask = (lambda i0, i1: None) if mask is None else (lambda i0, i1: mask[i0:i1])  # noqa: E731
    if m is not None:
        om = pair.outer_mean
        LR = outer_project_(om, m, msa_mask, msa_rows, ops)                      # [2d, S, pitch(N)]
        for i0, i1 in bands:
            ops.outer_contract_(om, x[i0:i1], _col_window(LR[:d], i0, i1), LR[d:], msa_mask, i0, 1)
        del LR
    L, R, G = ops.tri_operands(N, d, x)
    for ingoing in (False, True):
        tm = pair.triangle_multiply_ingoing if ingoing else pair.triangle_multiply_outgoing
        for i0, i1 in bands:                                                      # every projection before any update
            ops.tri_project(tm, x[i0:i1], rows_mask(i0, i1), out=(L[:, i0:i1], R[:, i0:i1], G[i0 * N:i1 * N]))
        for i0, i1 in bands:
            if ingoing:
                ops.tri_contract_window_(tm, x[i0:i1], L, R[:, :, i0:i1], G[i0 * N:i1 * N])
            else:
                ops.tri_contract_(tm, x[i0:i1], L[:, i0:i1], R, G[i0 * N:i1 * N], False, 1)
    del L, R, G
    ta = pair.triangle_attention_outgoing                                         # row attention
    bias = ops.pair_bias(ta, x)
    for i0, i1 in bands:
        ops.axial_attention_(ta, x[i0:i1], bias, rows_mask(i0, i1), True)
    ta = pair.triangle_attention_ingoing                                          # column attention
    bias = ops.pair_bias(ta, x)
    for j0, j1 in bands:
        xc = x[:, j0:j1].contiguous()
        ops.axial_attention_(ta, xc, bias, None if mask is None else mask[:, j0:j1].contiguous(), False)
        x[:, j0:j1] = xc
    return x


def feed_forward_(ff, x: torch.Tensor, band: int, ops) -> torch.Tensor:
    """The pair transition on x [N, N, d] in bands of `band` rows (pointwise: any split gives the same bits)."""
    for i0, i1 in _bands(x.shape[0], band):
        ops.feed_forward_(ff, x[i0:i1])
    return x
