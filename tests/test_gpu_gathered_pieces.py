"""The contractions the sharded schedule feeds with ALL-GATHERED operand pieces (alphafold2_b200/stages.py CudaStageOps),
checked on ONE GPU against the oracle stage ops: pieces whose width is not a multiple of 8 carry alignment padding, narrow
pieces are merged into one operand, wide ones are addressed in place through rank-4 tensor maps.  (The multi-GPU check in
tests/parallel_check_multi_gpu.py covers the same code with real collectives; this one runs in the single-GPU suite.)"""
import pytest
import torch

import alphafold2_b200 as A
from alphafold2_b200.parallel import _align8
from alphafold2_b200.stages import CudaStageOps
from oracle import evoformer_oracle as O
from stage_ops_oracle import OracleStageOps

pytestmark = pytest.mark.gpu
GARBAGE = 1.0e4          # what the padding columns hold: a result that read them is off by orders of magnitude


def _padded(t: torch.Tensor) -> torch.Tensor:
    """[..., w] fp32 -> bf16 [..., align8(w)] on the GPU, padding columns filled with GARBAGE."""
    out = torch.full(t.shape[:-1] + (_align8(t.shape[-1]),), GARBAGE, dtype=torch.bfloat16)
    out[..., :t.shape[-1]] = t.to(torch.bfloat16)
    return out.cuda()


def _rel(a: torch.Tensor, ref: torch.Tensor) -> float:
    return ((a.double().cpu() - ref).abs().max() / ref.pow(2).mean().sqrt()).item()


def _randomized(mod):
    st = O.randomize_zero_init_({k: v.clone() for k, v in mod.state_dict().items()}, std=0.05)
    mod.load_state_dict(st)
    return mod.eval()


@pytest.mark.parametrize("N,nl,P,d", [(48, 6, 8, 64), (40, 20, 2, 64), (64, 64, 8, 32), (256, 32, 8, 128), (512, 64, 8, 32), (384, 48, 2, 32)])
def test_triangle_ingoing_gathered_pieces(N, nl, P, d):
    """x_col [N, nl, d]: O[i][j] = sum_k R[k][i] L[k][j], the R operand gathered as P pieces of N/P columns each."""
    torch.manual_seed(N + P)
    tm = _randomized(A.TriangleMultiplicativeModule(dim=d, mix="ingoing"))
    K = N
    x = torch.randn(N, nl, d)
    bf = lambda t: t.to(torch.bfloat16).float()  # noqa: E731
    L, R, G = bf(torch.randn(d, K, nl)), bf(torch.randn(d, K, N)), bf(torch.rand(N * nl, d))
    pieces = [R[:, :, p * (N // P):(p + 1) * (N // P)] for p in range(P)]
    ref = x.double().clone()
    OracleStageOps().tri_contract_(tm, ref, L.double(), torch.cat(pieces, 0).double(), G.double(), True, P)
    xg = x.cuda()
    CudaStageOps().tri_contract_(tm.cuda(), xg, _padded(L), torch.cat([_padded(p) for p in pieces], 0), G.to(torch.bfloat16).cuda(), True, P)
    assert _rel(xg, ref) < 2e-2


@pytest.mark.parametrize("N,rows,P,d", [(48, 6, 8, 64), (40, 20, 2, 64), (256, 32, 8, 128), (384, 48, 2, 32)])
def test_triangle_outgoing_gathered_pieces(N, rows, P, d):
    """x_row [rows, N, d]: O[i][j] = sum_k L[i][k] R[j][k], the R operand gathered as P pieces of N/P rows each."""
    torch.manual_seed(N + P + 1)
    tm = _randomized(A.TriangleMultiplicativeModule(dim=d, mix="outgoing"))
    K = N
    x = torch.randn(rows, N, d)
    bf = lambda t: t.to(torch.bfloat16).float()  # noqa: E731
    L, R, G = bf(torch.randn(d, rows, K)), bf(torch.randn(d, N, K)), bf(torch.rand(rows * N, d))
    pieces = [R[:, p * (N // P):(p + 1) * (N // P)] for p in range(P)]
    ref = x.double().clone()
    OracleStageOps().tri_contract_(tm, ref, L.double(), torch.cat(pieces, 0).double(), G.double(), False, P)
    xg = x.cuda()
    CudaStageOps().tri_contract_(tm.cuda(), xg, _padded(L), torch.cat([_padded(p) for p in pieces], 0), G.to(torch.bfloat16).cuda(), False, P)
    assert _rel(xg, ref) < 2e-2


@pytest.mark.parametrize("N,rows,S,P,d,masked", [(48, 6, 8, 8, 64, True), (40, 20, 6, 2, 64, False), (256, 32, 128, 8, 32, True), (512, 64, 16, 8, 32, False)])
def test_outer_mean_gathered_pieces(N, rows, S, P, d, masked):
    """x_rows [rows, N, d] += OuterMean: L = this rank's columns of the MSA projection, R gathered as P pieces."""
    torch.manual_seed(N + S)
    om = _randomized(A.OuterMean(dim=d))
    row0 = rows * (P - 1)
    x = torch.randn(rows, N, d)
    bf = lambda t: t.to(torch.bfloat16).float()  # noqa: E731
    mm = (torch.rand(S, N) > 0.15) if masked else None
    if masked:
        mm[0] = True
    L, R = bf(torch.randn(d, S, rows)), bf(torch.randn(d, S, N))
    pieces = [R[:, :, p * (N // P):(p + 1) * (N // P)] for p in range(P)]
    ref = x.double().clone()
    OracleStageOps().outer_contract_(om, ref, L.double(), torch.cat(pieces, 0).double(), mm, row0, P)
    xg = x.cuda()
    CudaStageOps().outer_contract_(om.cuda(), xg, _padded(L), torch.cat([_padded(p) for p in pieces], 0), None if mm is None else mm.cuda(), row0, P)
    assert _rel(xg, ref) < 2e-2
