"""-m gpu: the template branch run in groups of templates (Alphafold2.embed_templates_ with G < T).

The online softmax of the pointwise template attention carries its fp32 state (running max, running sum, accumulator, "any
template valid") from one group to the next, and every other step acts on each template alone, so the result must not depend
on G at all: bitwise equality against G = T, never a tolerance.
  * kernel: af2_template_pointwise_{bf16,f32}_state over groups == one af2_template_pointwise_{bf16,f32} launch, out and pooled;
  * model: embed_templates_ with G in {1, 2, T} == G = T, bf16 and strict, over batch, T, n and masks that leave pairs with
    every template masked (their templates then fall into different groups), a fully masked template and a partial x_mask;
  * Alphafold2.forward with G = 1 against the alphafold2_templates.pt fixture with the gates of test_alphafold2_templates_golden;
  * memory: the branch's peak at T = 8, G = 1 exceeds the peak at T = 1 by no more than the extra templates' inputs plus the
    state one group hands to the next, and does not grow from T = 2 to T = 8 beyond the extra inputs.
"""
import functools

import pytest
import torch

from gpu_util import check, check_strict
from oracle import evoformer_oracle as O
from test_gpu_templates import _templates_fixture

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("groups", [(1, 1, 1, 1, 1), (2, 2, 1), (1, 4), (3, 2)])
def test_state_carry_kernel_bitwise(dtype, groups):
    from alphafold2_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(sum(groups) * 10 + len(groups))
    B, T, n, heads, dh = 2, sum(groups), 37, 8, 32
    pairs, I = n * n, heads * dh
    P = B * pairs
    q = torch.randn(P, I, generator=g).to(dtype).cuda()
    gate = (torch.rand(P, I, generator=g) if dtype == torch.bfloat16 else torch.randn(P, I, generator=g)).to(dtype).cuda()
    kv = torch.randn(B, T, pairs, 2 * I, generator=g).to(dtype).cuda()
    xm = (torch.rand(P, generator=g) > 0.15).cuda()
    tm = torch.rand(B, T, pairs, generator=g) > 0.4
    tm[:, :, :200] = False                                # every template masked: uniform mean over all T, pooled 0
    tm[0, 1] = False                                      # one template fully masked
    tm[:, :, 200:260] = False
    tm[:, T - 1, 200:260] = True                          # valid only in the last group
    tm = tm.cuda()
    single = lib.af2_template_pointwise_bf16 if dtype == torch.bfloat16 else lib.af2_template_pointwise_f32
    state = lib.af2_template_pointwise_bf16_state if dtype == torch.bfloat16 else lib.af2_template_pointwise_f32_state
    stream = torch.cuda.current_stream().cuda_stream
    out1 = torch.full((P, I), float("nan"), dtype=dtype, device="cuda")
    pooled1 = torch.full((P,), float("nan"), device="cuda")
    _lib.check(single(q.data_ptr(), gate.data_ptr(), kv.data_ptr(), xm.data_ptr(), tm.data_ptr(), out1.data_ptr(), pooled1.data_ptr(),
                      B, T, pairs, heads, dh, stream))
    out2 = torch.full((P, I), float("nan"), dtype=dtype, device="cuda")
    pooled2 = torch.full((P,), float("nan"), device="cuda")
    run_max = torch.full((P, heads), float("nan"), device="cuda")
    run_sum = torch.full((P, heads), float("nan"), device="cuda")
    acc = torch.full((P, I), float("nan"), device="cuda")
    t0 = 0
    for k, G in enumerate(groups):
        kvg = kv[:, t0:t0 + G].contiguous()
        tmg = tm[:, t0:t0 + G].contiguous()
        _lib.check(state(q.data_ptr(), gate.data_ptr(), kvg.data_ptr(), xm.data_ptr(), tmg.data_ptr(), out2.data_ptr(),
                         pooled2.data_ptr(), run_max.data_ptr(), run_sum.data_ptr(), acc.data_ptr(), int(k == 0),
                         int(k == len(groups) - 1), B, G, pairs, heads, dh, stream))
        t0 += G
    torch.cuda.synchronize()
    assert torch.equal(_bits(out1), _bits(out2)), f"grouped {groups} output differs from one launch"
    assert torch.equal(pooled1, pooled2), f"grouped {groups} pooled differs from one launch"
    assert pooled1[:200].eq(0).all() and pooled1[200:260].eq(1).all()


def test_state_carry_out_in_place():
    """The grouped path writes the last group's output over q (bf16) / acc (fp32): same bits as a separate buffer."""
    from alphafold2_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(11)
    B, n, heads, dh, groups = 1, 29, 4, 64, (2, 1)
    pairs, I, T = n * n, heads * dh, sum(groups)
    P = B * pairs
    stream = torch.cuda.current_stream().cuda_stream
    for dtype, fn in ((torch.bfloat16, lib.af2_template_pointwise_bf16_state), (torch.float32, lib.af2_template_pointwise_f32_state)):
        q = torch.randn(P, I, generator=g).to(dtype).cuda()
        gate = torch.rand(P, I, generator=g).to(dtype).cuda()
        kv = torch.randn(B, T, pairs, 2 * I, generator=g).to(dtype).cuda()
        res = []
        for in_place in (False, True):
            qq = q.clone()
            pooled = torch.empty(P, device="cuda")
            run_max, run_sum, acc = (torch.empty(P, heads, device="cuda"), torch.empty(P, heads, device="cuda"),
                                     torch.empty(P, I, device="cuda"))
            out = (qq if dtype == torch.bfloat16 else acc) if in_place else torch.empty(P, I, dtype=dtype, device="cuda")
            t0 = 0
            for k, G in enumerate(groups):
                kvg = kv[:, t0:t0 + G].contiguous()
                _lib.check(fn(qq.data_ptr(), gate.data_ptr(), kvg.data_ptr(), None, None, out.data_ptr(), pooled.data_ptr(),
                              run_max.data_ptr(), run_sum.data_ptr(), acc.data_ptr(), int(k == 0), int(k == len(groups) - 1),
                              B, G, pairs, heads, dh, stream))
                t0 += G
            res.append(out.clone())
        assert torch.equal(_bits(res[0]), _bits(res[1])), f"{dtype}: in-place output differs"


def test_state_carry_rejects_missing_state():
    from alphafold2_b200 import _lib
    lib = _lib.load()
    z = torch.zeros(64, 64, dtype=torch.bfloat16, device="cuda")
    kv = torch.zeros(64, 128, dtype=torch.bfloat16, device="cuda")
    pooled = torch.zeros(64, device="cuda")
    rc = lib.af2_template_pointwise_bf16_state(z.data_ptr(), z.data_ptr(), kv.data_ptr(), None, None, z.data_ptr(), pooled.data_ptr(),
                                               None, None, None, 1, 0, 1, 1, 64, 1, 64, torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"state" in lib.af2_last_error()


# ------------------------------------------------------------------------------------------------------------------------
# model: embed_templates_
# ------------------------------------------------------------------------------------------------------------------------
D, HEADS, DH, K = 64, 2, 32, 32


@functools.lru_cache(maxsize=None)
def _model(precision):
    import alphafold2_b200 as A
    torch.manual_seed(21)
    model = A.Alphafold2(dim=D, depth=1, heads=HEADS, dim_head=DH, templates_dim=K, templates_embed_layers=2, max_seq_len=136)
    st = O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05)
    model.load_state_dict(st)
    return A.set_precision(model.cuda().eval(), precision)


def _inputs(b, T, n, masks, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, n, n, D, generator=g)
    feats = torch.randn(b, T, n, n, K, generator=g)
    tm = torch.ones(b, T, n, dtype=torch.bool)
    mask = torch.ones(b, n, dtype=torch.bool)
    if masks == "mixed":
        tm = torch.rand(b, T, n, generator=g) > 0.25
        tm[:, :, 3:6] = False                             # residues with every template masked: whole rows / columns of pairs
        if T > 1:
            tm[:, 0] = False                              # one template fully masked
            tm[:, :, 6] = False
            tm[:, T - 1, 6] = True                        # valid only in the last template
        mask[:, -max(2, n // 8):] = False                 # partial x_mask
    x_mask = mask[:, :, None] & mask[:, None, :]
    return x.cuda(), x_mask.cuda(), feats.cuda(), tm.cuda()


def _embed(model, x, x_mask, feats, tm, group):
    out = x.clone()
    with torch.no_grad():
        model.embed_templates_(out, x_mask, feats, tm, group=group)
    assert model.last_template_group == min(group, feats.shape[1])
    return out


@pytest.mark.parametrize("masks", ["ones", "mixed"])
@pytest.mark.parametrize("n", [24, 40, 136])
@pytest.mark.parametrize("T", [1, 3, 5])
@pytest.mark.parametrize("b", [1, 2])
@pytest.mark.parametrize("precision", ["bf16", "strict"])
def test_embed_templates_groups_bitwise(precision, b, T, n, masks):
    model = _model(precision)
    x, x_mask, feats, tm = _inputs(b, T, n, masks, seed=b * 1000 + T * 100 + n)
    ref = _embed(model, x, x_mask, feats, tm, T)
    assert not torch.equal(ref, x), "the template branch changed nothing: the test would prove nothing"
    for G in (1, 2):
        if G >= T:
            continue
        out = _embed(model, x, x_mask, feats, tm, G)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), ref.view(torch.int32)), \
            f"{precision} b{b} T{T} n{n} {masks}: G = {G} differs from G = T (max |diff| {(out - ref).abs().max().item():.3e})"


@pytest.mark.parametrize("precision", ["bf16", "strict"])
def test_alphafold2_templates_golden_one_template_at_a_time(precision):
    from test_gpu_templates import _af2
    fx = _templates_fixture()
    i = {k: v.cuda() for k, v in fx["inputs"].items()}
    model = _af2(fx["cfg"], fx["state"], precision)
    assert i["templates_feats"].shape[1] > 1
    model.embed_templates_ = functools.partial(type(model).embed_templates_, model, group=1)
    kw = {k: i[k] for k in fx["calls"]["feats_angles"]}
    ret = model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"], **kw)
    assert model.last_template_group == 1
    if precision == "strict":
        check_strict("strict/alphafold2_templates/feats_angles/golden/distance G=1", ret.distance, fx["out_fp32"]["feats_angles"])
    else:
        check("alphafold2_templates/feats_angles/golden/distance G=1", ret.distance, fx["out_fp64"]["feats_angles"],
              fx["out_autocast_bf16"]["feats_angles"])


# ------------------------------------------------------------------------------------------------------------------------
# memory
# ------------------------------------------------------------------------------------------------------------------------
def _peak(model, b, T, n, group):
    from alphafold2_b200 import ops
    x, x_mask, feats, tm = _inputs(b, T, n, "ones", seed=T)
    ops._WORKSPACE.clear()                                 # the grow-only workspace would carry the previous run's size
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        model.embed_templates_(x, x_mask, feats, tm, group=group)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    del x, x_mask, feats, tm
    ops._WORKSPACE.clear()
    return peak


def test_template_memory_does_not_grow_with_T():
    b, n = 1, 384
    model = _model("bf16")
    P, I = b * n * n, HEADS * DH
    per_template = b * n * n * K * 4 + b * n                # templates_feats and templates_mask of one more template
    # what one group hands to the next (q | gate bf16, run_max / run_sum / acc / pooled fp32) and the group's own crossed mask
    carry = P * 2 * I * 2 + P * (2 * HEADS + I + 1) * 4 + b * n * n
    slack = 4 << 20                                         # allocator rounding of the handful of tensors involved
    p1 = _peak(model, b, 1, n, 1)
    p2 = _peak(model, b, 2, n, 1)
    p8 = _peak(model, b, 8, n, 1)
    assert p8 - p2 <= 6 * per_template + slack, f"peak grows with T: T=2 {p2} B, T=8 {p8} B"
    assert p8 - p1 <= 7 * per_template + carry + slack, f"T=1 {p1} B, T=8 G=1 {p8} B, allowed {7 * per_template + carry + slack}"
    # and running all 8 at once does need more: the grouping is what keeps the peak flat
    p8_all = _peak(model, b, 8, n, 8)
    assert p8_all > p8
