"""CPU: ops.plan_template_groups, the choice of how many templates the template branch runs at a time.

The byte counts come from the library's workspace queries, which need no GPU."""
import pytest

from alphafold2_b200 import _lib, ops

# C2-like model, N_res 512, 4 templates
SHAPE = dict(b=1, T=4, n=512, d=256, heads=8, dim_head=64)


def _bytes(G, precision, **kw):
    s = dict(SHAPE, **kw)
    return ops.template_branch_bytes(s["b"], s["T"], G, s["n"], s["d"], s["heads"], s["dim_head"], precision)


def _plan(budget, precision, **kw):
    s = dict(SHAPE, **kw)
    return ops.plan_template_groups(s["b"], s["T"], s["n"], s["d"], s["heads"], s["dim_head"], precision, budget)


@pytest.mark.parametrize("precision", ops.PRECISIONS)
def test_plan_fits_whole(precision):
    assert _plan(_bytes(4, precision), precision) == 4
    assert _plan(1 << 50, precision) == 4
    assert _plan(1 << 50, precision, T=10) == 10


@pytest.mark.parametrize("precision", ops.PRECISIONS)
def test_plan_tiny_budget_gives_one(precision):
    assert _plan(0, precision) == 1
    assert _plan(1 << 20, precision, T=10) == 1
    assert _plan(0, precision, T=1) == 1


@pytest.mark.parametrize("precision", ops.PRECISIONS)
@pytest.mark.parametrize("T", [2, 5, 10])
def test_plan_monotone_in_budget(precision, T):
    lo, hi = _bytes(1, precision, T=T) // 2, _bytes(T, precision, T=T) * 2
    prev = 0
    for k in range(200):
        G = _plan(lo + (hi - lo) * k // 199, precision, T=T)
        assert 1 <= G <= T and G >= prev
        prev = G
    assert prev == T


@pytest.mark.parametrize("precision", ops.PRECISIONS)
def test_plan_largest_group_that_fits(precision):
    T = 10
    for G in range(1, T + 1):
        budget = _bytes(G, precision, T=T)
        got = _plan(budget, precision, T=T)
        assert got >= G and _bytes(got, precision, T=T) <= budget


@pytest.mark.parametrize("precision", ops.PRECISIONS)
@pytest.mark.parametrize("b,T,n", [(1, 4, 512), (2, 3, 136), (1, 10, 2048)])
def test_whole_branch_bytes_are_todays_workspaces(precision, b, T, n):
    """At G = T the branch is today's: the largest of its workspace queries (as the grow-only workspace allocates it), plus t
    and the crossed template mask."""
    lib = _lib.load()
    d, h, dh, K = 256, 8, 64, 32
    rows = b * T * n * n
    if precision == "strict":
        ws = [lib.af2_template_embed_strict_workspace(rows, K), lib.af2_triangle_multiply_strict_workspace(b * T, n, d),
              lib.af2_axial_attention_strict_workspace(b * T, n, n, d, h, dh, 1),
              lib.af2_axial_attention_strict_workspace(b * T, n, n, d, h, dh, 0),
              lib.af2_template_pointwise_attention_strict_workspace(b, T, n, d, h, dh)]
    else:
        ws = [lib.af2_template_embed_workspace(rows, K), lib.af2_triangle_multiply_workspace(b * T, n, d),
              lib.af2_axial_attention_workspace(b * T, n, n, d, h, dh, 1), lib.af2_axial_attention_workspace(b * T, n, n, d, h, dh, 0),
              lib.af2_template_pointwise_attention_workspace(b, T, n, d, h, dh)]
    expect = int(max(ws) * 1.05) + 4096 + rows * d * 4 + rows
    assert ops.template_branch_bytes(b, T, T, n, d, h, dh, precision, K) == expect


def test_groups_do_not_depend_on_T():
    """With G fixed below T, the bytes are the same for every T: what the grouping is for."""
    ref = ops.template_branch_bytes(1, 2, 1, 1024, 256, 8, 64, "bf16")
    for T in (3, 4, 10, 100):
        assert ops.template_branch_bytes(1, T, 1, 1024, 256, 8, 64, "bf16") == ref
