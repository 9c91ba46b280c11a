"""CPU: what shard_alphafold2(pair_rows=True) refuses before it runs the structure module -- an unattached structure module, a
structure head count invariant point attention does not take, and a recyclables.pairwise_repr that is neither the whole pair
tensor nor the rank's pair rows -- raised before any device work or collective."""
import pytest
import torch
import torch.distributed as dist

import alphafold2_b200 as A
from alphafold2_b200 import parallel


@pytest.fixture
def four_ranks(monkeypatch):
    """dist as rank 0 of 4 ranks, with every collective raising."""
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 4)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)

    def collective(*args, **kwargs):
        raise AssertionError("a collective ran before the refusal")

    for name in ("all_gather_into_tensor", "all_to_all_single", "all_reduce", "barrier", "broadcast", "all_gather"):
        monkeypatch.setattr(dist, name, collective)


def _model(attach=True, **kw):
    cfg = dict(dim=128, depth=1, heads=2, dim_head=32, max_seq_len=16, predict_angles=True, predict_coords=True)
    cfg.update(kw)
    torch.manual_seed(0)
    model = A.Alphafold2(**cfg).eval()
    if attach:
        A.attach_structure_module(model)
    return parallel.shard_alphafold2(model, use_graph=False, pair_rows=True)


def test_structure_refusals_before_any_collective(four_ranks):
    n = 14                                                        # pair shards 4/4/3/3: rank 0 holds rows [0, 4)
    seq = torch.randint(0, 21, (1, n))
    msa = torch.randint(0, 21, (1, 3, n))
    with pytest.raises(NotImplementedError, match="attach_structure_module"):
        _model(attach=False)(seq, msa)
    with pytest.raises(ValueError, match="invariant point attention"):
        _model(structure_module_heads=17)(seq, msa)

    def rec(rows):
        return A.Recyclables(torch.randn(1, n, 3), torch.randn(1, n, 128), torch.randn(1, rows, n, 128))

    for rows in (3, 5, n - 1):
        with pytest.raises(ValueError, match=r"pairwise_repr must be the whole \[1, 14, 14, 128\] or this rank's pair rows "
                                             r"\[1, 4, 14, 128\]"):
            _model()(seq, msa, recyclables=rec(rows))
    # the shapes it takes get as far as the CPU refusal; so does an unattached module with return_trunk=True
    for rows in (4, n):
        with pytest.raises(ValueError, match="CUDA"):
            _model()(seq, msa, recyclables=rec(rows))
    with pytest.raises(ValueError, match="CUDA"):
        _model(attach=False)(seq, msa, return_trunk=True)
