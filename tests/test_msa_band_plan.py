"""CPU: ops.msa_block_bytes / ops.plan_block_bands, the choice of how many pair rows and MSA rows one Evoformer block runs
at a time.

The byte counts come from the library's workspace queries, which need no GPU."""
import pytest

from alphafold2_b200 import banded, ops

GB = 10 ** 9
D, H, DH = 256, 8, 64
BUDGET_80 = int(0.85 * 80 * GB)


def _budget_80(N, S, d=D):
    """85 % of what an 80 GB card (79.1 GiB usable) has left beside x and m."""
    return int(0.85 * (79.1 * 2 ** 30 - (N * N + S * N) * d * 4))


def _bytes(N, S, R, RS, B=1, d=D):
    return ops.msa_block_bytes(B, N, S, d, H, DH, R, RS)


def _plan(N, S, budget, B=1, d=D):
    return ops.plan_block_bands(B, N, S, d, H, DH, budget)


@pytest.mark.parametrize("B,N,S,R", [(1, 256, 128, 256), (1, 1024, 64, 256), (2, 320, 16, 320), (1, 600, 0, 256),
                                     (1, 2048, 0, 2048), (1, 4096, 32, 1024)])
def test_whole_msa_track_is_the_pair_block(B, N, S, R):
    for RS in (S, S + 1, S + 1000):
        assert _bytes(N, S, R, RS, B) == ops.pair_block_bytes(B, N, S, D, H, DH, R)


@pytest.mark.parametrize("N,S", [(256, 128), (384, 512), (512, 1024)])      # bench.py's C2, C3, C4
def test_benchmark_workloads_keep_their_plan(N, S):
    assert _plan(N, S, BUDGET_80) == (ops.plan_pair_band(1, N, S, D, H, DH, BUDGET_80), S) == (N, S)


@pytest.mark.parametrize("N", [1024, 2048, 3072, 4096])
@pytest.mark.parametrize("S", [32, 128, 512, 1024])
def test_plan_is_the_pair_plan_wherever_that_fits(N, S):
    budget = _budget_80(N, S)
    try:
        R = ops.plan_pair_band(1, N, S, D, H, DH, budget)
    except MemoryError:
        pytest.skip("the pair plan does not fit here")
    assert _plan(N, S, budget) == (R, S)


@pytest.mark.parametrize("N,S", [(1024, 4096), (2048, 2048), (1024, 700)])
def test_plan_monotone_in_budget_and_fits(N, S):
    lo = _bytes(N, S, min(256, N), 64)
    hi = ops.pair_block_bytes(1, N, S, D, H, DH, N) * 2
    prev = (0, 0)
    for k in range(120):
        budget = lo + (hi - lo) * k // 119
        R, RS = _plan(N, S, budget)
        assert (R, RS) >= prev, f"budget {budget}: {(R, RS)} after {prev}"
        prev = (R, RS)
        assert R == N or (R % ops.PAIR_BAND_ALIGN == 0 and 0 < R < N)
        assert RS == S or (RS % ops.MSA_BAND_ALIGN == 0 and 0 < RS < S)
        assert _bytes(N, S, R, RS) <= budget
    assert prev == (N, S)


def test_tiny_budget_raises_memory_error():
    with pytest.raises(MemoryError, match="64 MSA rows"):
        _plan(2048, 8448, 1 << 30)
    with pytest.raises(MemoryError):
        _plan(200, 8, 0)


@pytest.mark.parametrize("N,S", [(2048, 8448), (1024, 16384)])
def test_deep_msas_are_banded_on_an_80gb_card(N, S):
    budget = _budget_80(N, S)
    with pytest.raises(MemoryError):
        ops.plan_pair_band(1, N, S, D, H, DH, budget)
    R, RS = _plan(N, S, budget)
    assert R == N, "the MSA bands alone should make these shapes fit with the pair rows whole"
    assert 0 < RS < S and RS % ops.MSA_BAND_ALIGN == 0
    assert _bytes(N, S, R, RS) <= budget < _bytes(N, S, R, RS + ops.MSA_BAND_ALIGN) or RS + ops.MSA_BAND_ALIGN >= S


def test_msa_bands_drop_the_whole_msa_workspaces():
    """What MSA bands are for: at N 2048 x S 8448 one band's workspaces and the whole LR are far below the whole MSA track."""
    N, S = 2048, 8448
    assert _bytes(N, S, N, 512) < 0.5 * ops.pair_block_bytes(1, N, S, D, H, DH, N)
    assert _bytes(N, S, N, 256) <= _bytes(N, S, N, 512) < _bytes(N, S, N, 2048) < _bytes(N, S, N, 4096)


@pytest.mark.parametrize("S,N,rows,want", [(5, 9, 1, 8), (5, 13, 2, 8), (5, 12, 3, 8), (64, 100, 64, 96), (8448, 2048, 512, 120),
                                           (4, 4, 100, 4)])
def test_column_band_width(S, N, rows, want):
    C = banded.msa_column_band(S, N, rows)
    assert C == want
    assert C == N or (C % 8 == 0 and (S * C <= rows * N or C == 8))
