"""CPU: ops.template_reuse_fits, the rule by which alphafold2_b200.recycle keeps the template pair stack's output across its
iterations: t [b * T, n, n, d] fp32 and the crossed mask [b * T, n, n] bool must fit beside the whole-tensor plan of the trunk
and, with an extra MSA, of the extra-MSA stack.  Byte counts come from the library's workspace queries, which need no GPU."""
import pytest

from alphafold2_b200 import _lib, ops

GB = 10 ** 9
H, DH = 8, 64
BUDGET_80 = int(0.85 * 80 * GB)


def _t_bytes(b, T, n, d):
    return b * T * n * n * d * 4 + b * T * n * n                 # fp32 t, bool crossed mask


def _whole(b, n, S, d):
    """The whole-tensor block of one pair stack with S MSA rows, restated from the workspace queries (the grow-only workspace
    takes 5 % and 4 KiB more than the largest request)."""
    lib = _lib.load()
    ax = lib.af2_axial_attention_workspace
    ws = [lib.af2_triangle_multiply_workspace(b, n, d), ax(b, n, n, d, H, DH, 1), ax(b, n, n, d, H, DH, 0),
          lib.af2_feed_forward_workspace(b * n * n, d, 4 * d)]
    if S:
        ws += [ax(b, S, n, d, H, DH, 1), ax(b, S, n, d, H, DH, 0), lib.af2_feed_forward_workspace(b * S * n, d, 4 * d),
               lib.af2_outer_mean_workspace(b, S, n, d)]
    return int(max(ws) * 1.05) + 4096


def _fits(b, T, n, d, rows, budget):
    return ops.template_reuse_fits(b, T, n, d, H, DH, rows, budget)


@pytest.mark.parametrize("b,T,n,d,rows", [(1, 4, 256, 256, (132,)), (1, 4, 256, 256, (132, 128)), (2, 2, 40, 64, (6, 4)),
                                          (1, 1, 600, 128, (1,)), (1, 3, 384, 256, (515, 512))])
def test_boundary_is_t_plus_the_largest_whole_stack(b, T, n, d, rows):
    need = _t_bytes(b, T, n, d) + max(_whole(b, n, S, d) for S in rows)
    assert _fits(b, T, n, d, rows, need)
    assert not _fits(b, T, n, d, rows, need - 1)


@pytest.mark.parametrize("b,T,n,d,rows", [(1, 4, 256, 256, (132, 128)), (1, 2, 1024, 128, (33,)), (2, 2, 320, 64, (20, 16)),
                                          (1, 4, 2048, 64, (1, 64))])
def test_refuses_exactly_when_a_stack_would_leave_its_whole_plan(b, T, n, d, rows):
    """For budgets around the boundary: reuse is allowed exactly when every later stack still plans whole (ops.plan_pair_band
    gives n) with t taken out of the budget."""
    t = _t_bytes(b, T, n, d)
    need = t + max(_whole(b, n, S, d) for S in rows)
    for budget in [need // 2, need - (1 << 20), need - 1, need, need + 1, need + (1 << 20), 2 * need]:
        whole = []
        for S in rows:
            try:
                whole.append(ops.plan_pair_band(b, n, S, d, H, DH, budget - t) == n)
            except MemoryError:
                whole.append(False)
        assert _fits(b, T, n, d, rows, budget) == all(whole), budget


def test_extra_msa_stack_decides_when_it_is_the_larger():
    """The extra-MSA stack's tied-query attention cannot run in bands: a budget the trunk fits but the deeper extra MSA does not
    refuses reuse."""
    b, T, n, d = 1, 4, 256, 256
    trunk, extra = 4, 1024
    assert _whole(b, n, extra, d) > _whole(b, n, trunk, d)
    budget = _t_bytes(b, T, n, d) + _whole(b, n, trunk, d)
    assert _fits(b, T, n, d, (trunk,), budget)
    assert not _fits(b, T, n, d, (trunk, extra), budget)


def test_c2_with_four_templates_reuses_on_an_80gb_card():
    assert _fits(1, 4, 256, 256, (128,), BUDGET_80)


def test_long_proteins_do_not_reuse_on_an_80gb_card():
    """At N_res 4096 and d 256 one template's t is 17.2 GB, beside a trunk that already runs in bands without it."""
    assert _t_bytes(1, 1, 4096, 256) > 17 * GB
    assert ops.plan_pair_band(1, 4096, 128, 256, H, DH, BUDGET_80) < 4096
    assert not _fits(1, 1, 4096, 256, (128,), BUDGET_80)
    assert _fits(1, 4, 2048, 256, (128,), BUDGET_80)                # 17.2 GB of t beside a whole trunk at N_res 2048
