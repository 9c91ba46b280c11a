"""CPU: shard_alphafold2(pair_rows=True) without a GPU -- the per-rank memory estimate parallel.pair_rows_bytes, and the inputs the
rows forward refuses, which must raise before any device work or collective."""
import pytest
import torch
import torch.distributed as dist

import alphafold2_b200 as A
from alphafold2_b200 import parallel


def test_pair_rows_bytes_monotone_in_n():
    """Every length from P to 6000, even and uneven shards alike: the estimate never decreases with N, so the longest N_res that
    fits a budget bounds every shorter one."""
    for S, d, heads, dim_head in ((128, 256, 8, 64), (4, 128, 4, 32)):
        for P in range(1, 9):
            prev = 0
            for N in range(P, 6001):
                b = parallel.pair_rows_bytes(N, S, d, heads, dim_head, P)
                assert b >= prev, (S, d, P, N, prev, b)
                prev = b


def test_pair_rows_bytes_shrinks_with_p():
    """More ranks, fewer bytes per rank, at every length from 128 to 6000 (below that, shards of a few rows are dominated by the
    kernels' fixed tile padding)."""
    for S, d, heads, dim_head in ((128, 256, 8, 64), (4, 128, 4, 32)):
        for N in range(128, 6001):
            sizes = [parallel.pair_rows_bytes(N, S, d, heads, dim_head, P) for P in range(1, 9)]
            assert all(a > b for a, b in zip(sizes, sizes[1:])), (S, d, N, sizes)
    # at P = 1 the estimate holds at least the whole fp32 pair tensor
    assert parallel.pair_rows_bytes(512, 16, 128, 4, 32, 1) >= 4 * 512 * 512 * 128


@pytest.fixture
def four_ranks(monkeypatch):
    """dist as rank 0 of 4 ranks, with every collective raising."""
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 4)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)

    def collective(*args, **kwargs):
        raise AssertionError("a collective ran before the refusal")

    for name in ("all_gather_into_tensor", "all_to_all_single", "all_reduce", "barrier", "broadcast", "all_gather"):
        monkeypatch.setattr(dist, name, collective)


def _model(**kw):
    cfg = dict(dim=128, depth=1, heads=2, dim_head=32, max_seq_len=16, extra_msa_evoformer_layers=1, templates_embed_layers=1,
               predict_angles=True)
    cfg.update(kw)
    torch.manual_seed(0)
    return parallel.shard_alphafold2(A.Alphafold2(**cfg).eval(), use_graph=False, pair_rows=True)


def test_rows_forward_refusals_before_any_collective(four_ranks):
    seq = torch.randint(0, 21, (1, 12))
    msa = torch.randint(0, 21, (1, 3, 12))
    with pytest.raises(NotImplementedError, match="strict"):
        A.set_precision(_model(), "strict")(seq, msa)
    with pytest.raises(ValueError, match="batch 1"):
        _model()(seq.repeat(2, 1), msa.repeat(2, 1, 1))
    with pytest.raises(ValueError, match="smaller than the number of ranks"):
        _model()(seq[:, :3], msa[:, :, :3])
    with pytest.raises(ValueError, match="disable_token_embed"):
        _model(disable_token_embed=True)(seq, msa, seq_embed=torch.randn(1, 12, 128), msa_embed=torch.randn(1, 3, 12, 128))
    with pytest.raises(ValueError, match="distogram head"):
        _model(dim=64)(seq, msa)
    with pytest.raises(ValueError, match="extra_msa_mask"):
        _model()(seq, msa, extra_msa=msa)
    with pytest.raises(ValueError, match="CUDA"):
        _model()(seq, msa)


def test_pair_rows_mode_follows_the_last_call():
    model = A.Alphafold2(dim=32, depth=1, heads=2, dim_head=16, max_seq_len=8)
    parallel.shard_alphafold2(model, use_graph=False)
    assert "forward" not in model.__dict__
    parallel.shard_alphafold2(model, use_graph=False, pair_rows=True)
    assert "forward" in model.__dict__
    parallel.shard_alphafold2(model, use_graph=False)
    assert "forward" not in model.__dict__
