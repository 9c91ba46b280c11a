"""CPU: ops.plan_template_branch / template_branch_bytes(..., band), the choice of running the template branch in bands of
pair rows when not even one template fits whole.

The byte counts come from the library's workspace queries, which need no GPU."""
import pytest

from alphafold2_b200 import _lib, ops

GB = 10 ** 9
D, H, DH, K = 256, 8, 64, 32


def _bytes(n, G=1, T=4, b=1, band=None):
    return ops.template_branch_bytes(b, T, G, n, D, H, DH, "bf16", K, band=band)


def _plan(n, budget, T=4, b=1, precision="bf16"):
    return ops.plan_template_branch(b, T, n, D, H, DH, precision, budget, K)


@pytest.mark.parametrize("b,T,n", [(1, 4, 256), (1, 4, 1024), (1, 10, 1024), (1, 4, 2048), (2, 3, 136)])
def test_todays_plan_whenever_some_group_fits(b, T, n):
    for G in range(1, T + 1):
        budget = _bytes(n, G, T, b)
        want = ops.plan_template_groups(b, T, n, D, H, DH, "bf16", budget, K)
        assert _plan(n, budget, T, b) == (want, n)
    assert _plan(n, 1 << 50, T, b) == (T, n)


def test_band_none_is_todays_count():
    for G in (1, 2, 4):
        assert _bytes(1024, G, band=None) == ops.template_branch_bytes(1, 4, G, 1024, D, H, DH, "bf16", K)
        assert _bytes(1024, G, band=1024) == _bytes(1024, G)


@pytest.mark.parametrize("n", [1024, 2048, 3072, 3001])
def test_bands_only_when_no_group_fits(n):
    one = _bytes(n, 1)
    lo = _bytes(n, 1, band=256)
    for k in range(40):
        budget = lo + (one - lo) * k // 39
        G, R = _plan(n, budget)
        if budget >= one:
            assert R == n
        else:
            assert G == 1 and R < n and R % ops.PAIR_BAND_ALIGN == 0, (budget, G, R)
            assert _bytes(n, 1, band=R) <= budget
            if R + ops.PAIR_BAND_ALIGN < n:
                assert _bytes(n, 1, band=R + ops.PAIR_BAND_ALIGN) > budget, "not the largest band that fits"


@pytest.mark.parametrize("n", [1024, 2048, 3072])
def test_bytes_do_not_decrease_with_the_band(n):
    prev = 0
    for R in range(256, n, 256):
        cur = _bytes(n, 1, band=R)
        assert cur >= prev
        prev = cur
    assert _bytes(n, 1, band=256) < 0.65 * _bytes(n, 1), "bands of 256 rows must need far less than one whole template"


def test_banded_bytes_count_state_template_and_window_workspaces():
    """State of every pair, one template's t / crossed mask / templates_feats copy and one band's q | gate, plus the larger
    of the banded pair block and the band's workspace (as the grow-only workspace allocates it)."""
    lib = _lib.load()
    n, R, I = 2048, 512, H * DH
    P, rows, W = n * n, n * n, R * n
    ws = max(lib.af2_template_embed_workspace(rows, K), lib.af2_template_pointwise_begin_workspace(W, D),
             lib.af2_template_pointwise_group_workspace(1, 1, W, n * n, D, H, DH), lib.af2_template_pointwise_end_workspace(W, H, DH))
    persist = rows * D * 4 + rows + rows * K * 4 + P * (2 * H + I + 1) * 4 + W * 2 * I * 2
    got = _bytes(n, 1, band=R)
    assert got >= ops.pair_block_bytes(1, n, 0, D, H, DH, R) + persist
    assert got >= int(ws * 1.05) + 4096 + persist


def test_banded_bytes_do_not_depend_on_T():
    ref = _bytes(3072, 1, T=2, band=512)
    for T in (1, 4, 10):
        assert _bytes(3072, 1, T=T, band=512) == ref


def test_n3072_four_templates_are_banded_on_an_80gb_card():
    n = 3072
    x = n * n * D * 4
    budget = int(0.85 * (80 * GB - x))
    G, R = _plan(n, budget)
    assert G == 1 and R < n and R % 256 == 0
    assert _bytes(n, 1) > budget >= _bytes(n, 1, band=R)


def test_memory_error_below_one_band():
    n = 3072
    with pytest.raises(MemoryError, match="bands of 256"):
        _plan(n, _bytes(n, 1, band=256) - 1)
    with pytest.raises(MemoryError):
        _plan(200, 0)                      # n below one band: nothing smaller to fall back to


def test_strict_keeps_todays_plan():
    assert _plan(3072, 0, precision="strict") == (1, 3072)
    with pytest.raises(ValueError, match="strict"):
        ops.template_branch_bytes(1, 4, 1, 3072, D, H, DH, "strict", K, band=256)
