"""CPU: ops.pair_block_bytes / ops.plan_pair_band, the choice of how many pair rows one Evoformer block runs at a time.

The byte counts come from the library's workspace queries, which need no GPU."""
import pytest

from alphafold2_b200 import _lib, ops

GB = 10 ** 9
D, H, DH = 256, 8, 64
BUDGET_80 = int(0.85 * 80 * GB)


def _bytes(N, S, R, B=1, d=D):
    return ops.pair_block_bytes(B, N, S, d, H, DH, R)


def _plan(N, S, budget, B=1, d=D):
    return ops.plan_pair_band(B, N, S, d, H, DH, budget)


@pytest.mark.parametrize("N,S", [(256, 128), (384, 512), (512, 1024)])      # bench.py's C2, C3, C4
def test_benchmark_workloads_run_whole(N, S):
    assert _plan(N, S, BUDGET_80) == N


@pytest.mark.parametrize("N,S,B", [(256, 128, 1), (1024, 64, 1), (2048, 32, 1), (600, 16, 2), (4096, 32, 1)])
def test_whole_whenever_it_fits(N, S, B):
    whole = _bytes(N, S, N, B)
    assert _plan(N, S, whole, B) == N
    assert _plan(N, S, whole + 1, B) == N


@pytest.mark.parametrize("N,S", [(1024, 64), (2048, 32), (4096, 128), (3001, 32)])
def test_plan_monotone_in_budget(N, S):
    lo, hi = _bytes(N, S, 256), _bytes(N, S, N) * 2
    prev = 0
    for k in range(200):
        R = _plan(N, S, lo + (hi - lo) * k // 199)
        assert R >= prev
        prev = R
    assert prev == N


@pytest.mark.parametrize("N,S", [(1024, 64), (2048, 32), (4096, 128), (3001, 32)])
def test_bands_are_aligned_and_fit(N, S):
    lo, hi = _bytes(N, S, 256), _bytes(N, S, N)
    for k in range(50):
        budget = lo + (hi - lo) * k // 49
        R = _plan(N, S, budget)
        assert R == N or (R % ops.PAIR_BAND_ALIGN == 0 and 0 < R < N)
        assert _bytes(N, S, R) <= budget


def test_n4096_is_banded_on_an_80gb_card():
    R = _plan(4096, 128, BUDGET_80)
    assert R < 4096 and R % 256 == 0
    assert _bytes(4096, 128, 4096) > BUDGET_80 >= _bytes(4096, 128, R)


def test_tiny_budget_raises_memory_error():
    with pytest.raises(MemoryError, match="bands of 256"):
        _plan(4096, 128, 1 << 30)
    with pytest.raises(MemoryError):
        _plan(200, 8, 0)                   # below one band: nothing smaller to fall back to


@pytest.mark.parametrize("B,N,S", [(1, 256, 128), (1, 1024, 64), (2, 320, 16), (1, 600, 0), (3, 136, 0)])
def test_whole_block_bytes_are_todays_workspaces(B, N, S):
    """At R = N the block is today's: the largest of its whole-tensor workspace queries, as the grow-only workspace
    allocates it (compare test_template_group_plan.py::test_whole_branch_bytes_are_todays_workspaces)."""
    lib = _lib.load()
    ax = lib.af2_axial_attention_workspace
    ws = [lib.af2_triangle_multiply_workspace(B, N, D), ax(B, N, N, D, H, DH, 1), ax(B, N, N, D, H, DH, 0),
          lib.af2_feed_forward_workspace(B * N * N, D, 4 * D)]
    if S:
        ws += [ax(B, S, N, D, H, DH, 1), ax(B, S, N, D, H, DH, 0), lib.af2_feed_forward_workspace(B * S * N, D, 4 * D),
               lib.af2_outer_mean_workspace(B, S, N, D)]
    assert _bytes(N, S, N, B) == int(max(ws) * 1.05) + 4096
    assert _bytes(N, S, N + 256, B) == _bytes(N, S, N, B)


def test_banded_bytes_do_not_hold_whole_tensor_workspaces():
    """What banding is for: at N 4096 one band's workspace plus the kept operands is far below the whole-tensor workspace,
    and smaller bands need less."""
    whole = _bytes(4096, 32, 4096)
    assert _bytes(4096, 32, 512) < 0.5 * whole
    assert _bytes(4096, 32, 256) < _bytes(4096, 32, 512) < _bytes(4096, 32, 1024)
