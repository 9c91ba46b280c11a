"""CPU: the banded pair-track schedule (alphafold2_b200/banded.py) reproduces the oracle Evoformer when its stage ops are the
oracle math in fp64.  Checks the slicing into row and column bands, the zero-padded operand pitches, which pair bias is taken
before which update, and that every triangle projection runs before any contraction -- everything of the banded path except
the CUDA kernels themselves (tests/test_gpu_pair_bands.py checks those, bitwise against the whole-tensor calls)."""
import pytest
import torch
import torch.nn.functional as F

import alphafold2_b200 as A
from alphafold2_b200 import banded
from oracle import evoformer_oracle as O
from stage_ops_oracle import OracleStageOps, _w


def _align8(n):
    return (n + 7) // 8 * 8


class BandOracleStageOps(OracleStageOps):
    """OracleStageOps with the banded schedule's calls, on operands laid out as the kernels read them: channel-major L / R
    with rows zero-padded to align8, windows of them, and zero-padded left operands of the outer mean."""

    def tri_operands(self, N, d, like):
        L = like.new_zeros(d, N, _align8(N))
        return L, torch.zeros_like(L), like.new_full((N * N, d), float("nan"))

    def tri_project(self, tm, x_loc, mask_loc, out=None):
        L, R, G = super().tri_project(tm, x_loc, mask_loc)
        if out is None:
            return L, R, G
        Lo, Ro, Go = out
        Lo[..., :L.shape[2]] = L
        Ro[..., :R.shape[2]] = R
        Go.copy_(G)
        return out

    def tri_contract_window_(self, tm, x_rows, L, R_win, gate):
        w = _w(tm, x_rows.dtype)
        d, N = L.shape[0], x_rows.shape[1]
        out = torch.einsum("cki,ckj->ijc", R_win, L[:, :, :N])
        out = F.layer_norm(out, (d,), w["to_out_norm.weight"], w["to_out_norm.bias"], 1e-5) * gate.view(out.shape)
        x_rows += F.linear(out, w["to_out.weight"], w["to_out.bias"])

    def outer_contract_(self, om, x_rows, L, Rg, msa_mask_full, row0, pieces):
        super().outer_contract_(om, x_rows, L[..., :x_rows.shape[0]], Rg, msa_mask_full, row0, pieces)


def _banded_evoformer(evo, x, m, mask, msa_mask, band, ops):
    """EvoformerBlock.update_ with the pair track in bands: the MSA track whole (as the product runs it), then per batch
    element the banded pair block and pair transition."""
    x, m = x.clone(), m.clone()
    for block in evo.layers:
        pair, ff, msa_attn, msa_ff = block.layer
        for b in range(x.shape[0]):
            mm = None if msa_mask is None else msa_mask[b]
            ops.axial_attention_(msa_attn.row_attn, m[b], ops.pair_bias(msa_attn.row_attn, x[b]), mm, True)
            ops.axial_attention_(msa_attn.col_attn, m[b], None, mm, False)
            ops.feed_forward_(msa_ff, m[b])
            banded.pair_block_(pair, x[b], None if mask is None else mask[b], m[b], mm, band, ops)
            banded.feed_forward_(ff, x[b], band, ops)
    return x, m


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("B,N,band", [(1, 12, 4), (1, 12, 6), (1, 10, 4), (1, 13, 8), (2, 10, 3), (2, 9, 9)])
def test_banded_schedule_matches_oracle(B, N, band, masked):
    torch.manual_seed(B * 100 + N * 10 + band)
    d, H, dh, S, depth = 16, 2, 8, 5, 2
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
        m1[:, 1] = False                                  # a fully masked row and column inside the first band
        mask = m1[:, :, None] & m1[:, None, :]
        msa_mask = torch.rand(B, S, N) > 0.2
        msa_mask[:, 0] = True
    xo, mo = _banded_evoformer(evo, x, m, mask, msa_mask, band, BandOracleStageOps())
    st64 = {k: v.double() for k, v in st.items()}
    for b in range(B):
        pick = lambda t: None if t is None else t[b:b + 1]  # noqa: E731
        rx, rm = O.evoformer(st64, "", x[b:b + 1], m[b:b + 1], H, depth, pick(mask), pick(msa_mask))
        ex = (xo[b:b + 1] - rx).abs().max().item()
        em = (mo[b:b + 1] - rm).abs().max().item()
        assert ex < 1e-4 and em < 1e-4, f"batch {b}: pair err {ex}, msa err {em}"
    assert not torch.equal(xo, x)


def test_stale_bias_would_be_caught():
    """The check above can see a schedule error of the kind banding risks: the column attention's bias taken from x before
    the row attention updated it changes the result far beyond the tolerance."""
    torch.manual_seed(3)
    d, H, dh, N, S = 16, 2, 8, 12, 4
    evo = A.Evoformer(depth=1, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
    st = O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.3)
    evo.load_state_dict(st)
    evo = evo.double()
    x = torch.randn(1, N, N, d, dtype=torch.float64)
    m = torch.randn(1, S, N, d, dtype=torch.float64)

    pair = evo.layers[0].layer[0]

    class StaleBias(BandOracleStageOps):
        def pair_bias(self, ax, x_rows):
            if ax is pair.triangle_attention_outgoing:         # the column attention's bias from x before the row attention
                self.stale = super().pair_bias(pair.triangle_attention_ingoing, x_rows)
            if ax is pair.triangle_attention_ingoing:
                return self.stale
            return super().pair_bias(ax, x_rows)

    good, _ = _banded_evoformer(evo, x, m, None, None, 4, BandOracleStageOps())
    bad, _ = _banded_evoformer(evo, x, m, None, None, 4, StaleBias())
    assert (good - bad).abs().max().item() > 1e-3
