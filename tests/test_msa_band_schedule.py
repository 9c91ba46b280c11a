"""CPU: the MSA track in bands of MSA rows (banded.msa_track_, banded.outer_mean_ and pair_block_'s chunked projection)
reproduces the oracle Evoformer when its stage ops are the oracle math in fp64.  Checks the row and column band slicing,
the projection chunks written into one operand with its channel stride, and that column attention starts only after the
last row band -- everything of the banded MSA path except the CUDA kernels (tests/test_gpu_msa_bands.py checks those,
bitwise against the whole-tensor calls)."""
import pytest
import torch

import alphafold2_b200 as A
from alphafold2_b200 import banded
from oracle import evoformer_oracle as O
from test_pair_band_schedule import BandOracleStageOps


def _align8(n):
    return (n + 7) // 8 * 8


class MsaBandOracleStageOps(BandOracleStageOps):
    """BandOracleStageOps with the outer mean's operand laid out as the kernels write it: [2d, S, align8(N)], filled chunk by
    chunk through outer_project(out=...).  Entries no chunk wrote stay NaN, so a missed chunk shows in the result."""

    def outer_operand(self, S, N, d, like):
        return like.new_full((2 * d, S, _align8(N)), float("nan"))

    def outer_project(self, om, m_cols, mask_cols, out=None):
        LR = super().outer_project(om, m_cols, mask_cols)
        if out is None:
            return LR
        out[..., :LR.shape[2]] = LR
        return out

    def outer_contract_(self, om, x_rows, L, Rg, msa_mask_full, row0, pieces):
        N = x_rows.shape[1]
        super().outer_contract_(om, x_rows, L, Rg[..., :N // pieces].contiguous(), msa_mask_full, row0, pieces)


def _msa_track_early_columns(msa_attn, msa_ff, m, msa_mask, x, rows, ops):
    """A wrong schedule: column attention after the FIRST row band instead of the last."""
    S, N, _ = m.shape
    bias = ops.pair_bias(msa_attn.row_attn, x)
    pick = lambda s0, s1: None if msa_mask is None else msa_mask[s0:s1]  # noqa: E731
    ops.axial_attention_(msa_attn.row_attn, m[:rows], bias, pick(0, rows), True)
    ops.axial_attention_(msa_attn.col_attn, m, None, msa_mask, False)
    for s0 in range(rows, S, rows):
        ops.axial_attention_(msa_attn.row_attn, m[s0:s0 + rows], bias, pick(s0, s0 + rows), True)
    return banded.feed_forward_(msa_ff, m, rows, ops)


def _banded_evoformer(evo, x, m, mask, msa_mask, band, msa_rows, ops, msa_track=banded.msa_track_):
    """EvoformerBlock.update_ with the MSA track in bands of msa_rows MSA rows and the pair track in bands of `band` pair rows
    (band >= N: the pair calls whole, the outer mean as chunked projection and one contraction, as the product runs it)."""
    x, m = x.clone(), m.clone()
    N = x.shape[1]
    for block in evo.layers:
        pair, ff, msa_attn, msa_ff = block.layer
        for b in range(x.shape[0]):
            mm = None if msa_mask is None else msa_mask[b]
            mk = None if mask is None else mask[b]
            msa_track(msa_attn, msa_ff, m[b], mm, x[b], msa_rows, ops)
            if band < N:
                banded.pair_block_(pair, x[b], mk, m[b], mm, band, ops, msa_rows)
            else:
                banded.outer_mean_(pair.outer_mean, x[b], m[b], mm, msa_rows, ops)
                banded.pair_block_(pair, x[b], mk, None, None, N, ops)
            banded.feed_forward_(ff, x[b], N, ops)
    return x, m


def _setup(B, N, S, seed, masked, d=16, H=2, dh=8, depth=2):
    torch.manual_seed(seed)
    evo = A.Evoformer(depth=depth, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
    st = O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.3)
    evo.load_state_dict(st)
    evo = evo.double()
    x = torch.randn(B, N, N, d, dtype=torch.float64)
    m = torch.randn(B, S, N, d, dtype=torch.float64)
    mask = msa_mask = None
    if masked:
        m1 = torch.ones(B, N, dtype=torch.bool)
        m1[:, -2:] = False
        m1[:, 1] = False
        mask = m1[:, :, None] & m1[:, None, :]
        msa_mask = torch.rand(B, S, N) > 0.2
        msa_mask[:, 0] = True
        msa_mask[:, 2] = False                            # a fully masked MSA row
        msa_mask[:, :, 3] = False                         # and a fully masked MSA column
    return evo, {k: v.double() for k, v in st.items()}, x, m, mask, msa_mask, H, depth


def _oracle(st64, x, m, mask, msa_mask, H, depth):
    outs = []
    for b in range(x.shape[0]):
        pick = lambda t: None if t is None else t[b:b + 1]  # noqa: E731
        outs.append(O.evoformer(st64, "", x[b:b + 1], m[b:b + 1], H, depth, pick(mask), pick(msa_mask)))
    return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("B,N,S,msa_rows,band", [
    (1, 9, 5, 1, 9), (1, 12, 5, 2, 12), (1, 13, 5, 3, 13), (1, 10, 5, 2, 10),     # pair rows whole
    (2, 11, 5, 3, 11),                                                           # batch 2
    (1, 12, 5, 2, 4), (1, 13, 5, 3, 8), (2, 10, 5, 1, 3),                         # with pair bands
    (1, 12, 5, 5, 12),                                                           # one band: the whole MSA track
])
def test_msa_banded_schedule_matches_oracle(B, N, S, msa_rows, band, masked):
    evo, st64, x, m, mask, msa_mask, H, depth = _setup(B, N, S, B * 1000 + N * 10 + msa_rows + band, masked)
    xo, mo = _banded_evoformer(evo, x, m, mask, msa_mask, band, msa_rows, MsaBandOracleStageOps())
    rx, rm = _oracle(st64, x, m, mask, msa_mask, H, depth)
    ex, em = (xo - rx).abs().max().item(), (mo - rm).abs().max().item()
    assert ex < 1e-4 and em < 1e-4, f"pair err {ex}, msa err {em}"
    assert not torch.equal(mo, m)


def test_early_column_attention_would_be_caught():
    """The check above can see the schedule error MSA row bands risk: column attention started before the last row band
    changes the result far beyond the tolerance."""
    evo, st64, x, m, mask, msa_mask, H, depth = _setup(1, 12, 5, 11, False, depth=1)
    ops = MsaBandOracleStageOps()
    good, gm = _banded_evoformer(evo, x, m, mask, msa_mask, 12, 2, ops)
    bad, bm = _banded_evoformer(evo, x, m, mask, msa_mask, 12, 2, ops, msa_track=_msa_track_early_columns)
    rx, rm = _oracle(st64, x, m, mask, msa_mask, H, depth)
    assert (gm - rm).abs().max().item() < 1e-4
    assert (bm - rm).abs().max().item() > 1e-3
