"""CPU: parallel.template_reuse_rows_fits, the rule by which alphafold2_b200.recycle lets a rank of shard_alphafold2 keep its rows
of the template pair stack's output across its iterations: T rows [rows, N, d] fp32 and their crossed mask rows [rows, N] bool
must fit beside parallel.pair_rows_bytes of every later sharded stack (the trunk and, with an extra MSA, the extra-MSA stack),
plus two whole pair tensors in the default mode.  Byte counts come from the library's workspace queries, which need no GPU."""
import pytest

from alphafold2_b200 import parallel

GB = 10 ** 9
H, DH = 8, 64
BUDGET_80 = int(0.85 * 80 * GB)


def _t_bytes(T, rows, N, d):
    return T * rows * N * d * 4 + T * rows * N                   # fp32 t rows, bool crossed mask rows


def _fits(T, rows, N, d, P, stack_rows, budget, whole_pair=False):
    return parallel.template_reuse_rows_fits(T, rows, N, d, H, DH, P, stack_rows, budget, whole_pair)


def _need(T, rows, N, d, P, stack_rows, whole_pair=False):
    held = 2 * N * N * d * 4 if whole_pair else 0
    return _t_bytes(T, rows, N, d) + held + max(parallel.pair_rows_bytes(N, S, d, H, DH, P) for S in stack_rows)


@pytest.mark.parametrize("T,N,d,P,stack_rows,whole_pair", [(4, 256, 256, 2, (132,), False), (4, 256, 256, 2, (132, 128), True),
                                                          (2, 43, 128, 3, (7, 5), False), (2, 43, 128, 3, (7, 5), True),
                                                          (1, 1000, 128, 8, (1,), False), (3, 2048, 256, 4, (516, 512), False)])
def test_boundary_is_t_rows_plus_the_largest_sharded_stack(T, N, d, P, stack_rows, whole_pair):
    rows = -(-N // P)
    need = _need(T, rows, N, d, P, stack_rows, whole_pair)
    assert _fits(T, rows, N, d, P, stack_rows, need, whole_pair)
    assert not _fits(T, rows, N, d, P, stack_rows, need - 1, whole_pair)


def test_uneven_shards_decide_per_rank():
    """N 43 over 3 ranks: shards 15 / 14 / 14.  A budget the smaller shards fit and the larger does not splits the ranks'
    answers; sharded_embed_templates_ reduces them (MIN over the group), so every rank then refuses."""
    T, N, d, P, rows = 2, 43, 128, 3, (7,)
    counts = parallel.shard_counts(N, P)
    assert counts == [15, 14, 14]
    budget = _need(T, 14, N, d, P, rows)
    assert budget < _need(T, 15, N, d, P, rows)
    answers = [_fits(T, c, N, d, P, rows, budget) for c in counts]
    assert answers == [False, True, True]
    assert min(answers) is False


def test_pair_rows_bytes_counts_the_largest_shard_for_every_rank():
    """The later stacks' share does not depend on the rank's own rows: only the kept rows do."""
    T, N, d, P, rows = 2, 43, 128, 3, (7,)
    assert _need(T, 15, N, d, P, rows) - _need(T, 14, N, d, P, rows) == _t_bytes(T, 1, N, d)


def test_extra_msa_stack_decides_when_it_is_the_larger():
    T, N, d, P = 4, 512, 256, 2
    trunk, extra = 8, 1024
    assert parallel.pair_rows_bytes(N, extra, d, H, DH, P) > parallel.pair_rows_bytes(N, trunk, d, H, DH, P)
    budget = _need(T, N // P, N, d, P, (trunk,))
    assert _fits(T, N // P, N, d, P, (trunk,), budget)
    assert not _fits(T, N // P, N, d, P, (trunk, extra), budget)


def test_default_mode_counts_two_whole_pair_tensors():
    T, N, d, P, rows = 2, 512, 128, 4, (16,)
    budget = _need(T, N // P, N, d, P, rows)
    assert _fits(T, N // P, N, d, P, rows, budget)
    assert not _fits(T, N // P, N, d, P, rows, budget, whole_pair=True)
    assert _fits(T, N // P, N, d, P, rows, budget + 2 * N * N * d * 4, whole_pair=True)


def test_c2_with_four_templates_reuses_on_an_80gb_card():
    for P in (2, 4, 8):
        assert _fits(4, -(-256 // P), 256, 256, P, (132,), BUDGET_80, whole_pair=True)


def test_long_proteins_on_eight_ranks():
    """C2's model (d 256, S 132) on 8 ranks in pair_rows mode, 85 % of 80 GB: at N_res 4096 the trunk takes 47 GB and 8 templates'
    rows (17.2 GB) still fit beside it; at 4608 (59.8 GB) 3 fit and 4 do not; at 4912, the longest N_res the trunk fits at all,
    not even one template's rows (3.1 GB) do."""
    P, d, S = 8, 256, (132,)
    for N, most in ((4096, 8), (4608, 3), (4912, 0)):
        rows = -(-N // P)
        assert [T for T in range(1, 9) if _fits(T, rows, N, d, P, S, BUDGET_80)] == list(range(1, most + 1)), N
