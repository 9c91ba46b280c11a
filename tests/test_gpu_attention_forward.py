"""Attention.forward on the GPU (alphafold2.py:125-190): self- and cross-attention with masks, any broadcast bias and tied
queries, element-wise against the fp64 oracle (oracle/attention_oracle.py).  bf16 mode: the gates of tests/gpu_util.py
(max / mean error against rms(ref), and at most 1.15x the error of the oracle under CUDA autocast).  Strict mode:
allclose(rtol 1e-3, atol 1e-4) on every element.  Also the two call sites of the reference that reach a standalone
Attention: the template branch (alphafold2.py:767-775) and AxialAttention's call (:240-252)."""
import os

import pytest
import torch
import torch.nn.functional as F

import alphafold2_b200 as A
from oracle import attention_oracle as AO
from oracle import evoformer_oracle as O
from oracle import template_oracle as TO
from gpu_util import autocast_yardstick, check, check_strict, dev, to64

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "attention_forward.pt")


def _module(d, heads, dh, strict=False, seed=0):
    torch.manual_seed(seed)          # the default init of to_q / to_kv: the same weights whatever ran before
    a = A.Attention(d, heads=heads, dim_head=dh)
    st = O.randomize_zero_init_({k: v.clone() for k, v in a.state_dict().items()}, seed=seed)
    a.load_state_dict(st)
    a = a.cuda().eval()
    if strict:
        A.set_precision(a, "strict")
    return a, st


def _inputs(B, i, j, d, heads, seed, *, context=True, mask=True, context_mask=True, bias=None, masked_rows=False):
    g = torch.Generator().manual_seed(seed)
    kw = {"x": torch.randn(B, i, d, generator=g)}
    if context:
        kw["context"] = torch.randn(B, j, d, generator=g)
    if mask:
        kw["mask"] = torch.rand(B, i, generator=g) > 0.25
        if masked_rows:
            kw["mask"][0] = False
            kw["mask"][-1, : (i + 1) // 2] = False
    if context_mask:
        kw["context_mask"] = torch.rand(B, j, generator=g) > 0.25
    if bias is not None:
        shape = {"bhij": (B, heads, i, j), "1hij": (1, heads, i, j), "hij": (heads, i, j)}[bias]
        kw["attn_bias"] = torch.randn(*shape, generator=g)
    return kw


def _run(a, st, heads, kw, name, strict=False):
    cuda = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in kw.items()}
    before = {k: v.clone() for k, v in cuda.items() if torch.is_tensor(v)}
    with torch.no_grad():
        out = a(**cuda)
    torch.cuda.synchronize()
    for k, v in before.items():
        assert torch.equal(v, cuda[k]), f"{name}: input {k} modified"
    assert out.shape == kw["x"].shape and out.dtype == kw["x"].dtype
    k64 = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()}
    ref = AO.attention(to64(st), "", k64.pop("x"), heads, **k64)
    if strict:
        return check_strict(name, out, ref.float())
    w32 = dev(st, torch.float32)
    ac = autocast_yardstick(lambda: AO.attention(w32, "", cuda["x"], heads, **{k: v for k, v in cuda.items() if k != "x"}))
    return check(name, out, ref, ac)


# (name, dim_head, B, i, j, input options)
BF16_CASES = [
    ("self_dh16", 16, 2, 77, 77, dict(context=False, context_mask=False, bias="1hij")),
    ("self_dh32", 32, 2, 77, 77, dict(context=False, context_mask=False, bias="bhij")),
    ("self_dh64", 64, 2, 77, 77, dict(context=False, context_mask=False, bias="hij")),
    ("self_dh128", 128, 2, 77, 77, dict(context=False, context_mask=False, bias="1hij")),
    ("cross_i_gt_j", 32, 3, 200, 77, dict(bias="bhij")),
    ("cross_i_lt_j", 64, 2, 77, 300, dict(context_mask=False, bias="hij")),
    ("cross_j1", 32, 2, 33, 1, dict()),
    ("cross_context_mask_only", 64, 2, 45, 21, dict(mask=False)),
    ("self_no_mask_batch1", 32, 1, 130, 130, dict(context=False, mask=False, context_mask=False)),
    ("self_masked_rows", 64, 3, 50, 50, dict(context=False, context_mask=False, masked_rows=True, bias="1hij")),
    ("cross_masked_rows", 32, 3, 50, 19, dict(masked_rows=True)),
    ("one_query_bias", 32, 4, 1, 6, dict(bias="bhij")),
]


@pytest.mark.parametrize("name,dh,B,i,j,opts", BF16_CASES, ids=[c[0] for c in BF16_CASES])
def test_attention_forward_bf16(name, dh, B, i, j, opts):
    d, heads = 64, 4
    a, st = _module(d, heads, dh, seed=dh)
    _run(a, st, heads, _inputs(B, i, j, d, heads, seed=B * 1000 + i + j, **opts), name)


@pytest.mark.parametrize("T", list(range(1, 11)))
@pytest.mark.parametrize("B", [16, 64])
def test_attention_forward_one_query(T, B):
    """i = 1 over a short context: the pointwise template kernel.  Batch 1 at i = 1 is a strict case: with one query the
    bf16 gates would rest on the largest of d errors."""
    d, heads, dh = 128, 4, 32
    a, st = _module(d, heads, dh, seed=T)
    _run(a, st, heads, _inputs(B, 1, T, d, heads, seed=T, masked_rows=B > 1), f"one_query_T{T}_B{B}")


@pytest.mark.parametrize("context", [False, True])
def test_attention_forward_tied(context):
    d, heads, dh = 64, 4, 32
    a, st = _module(d, heads, dh, seed=7)
    kw = _inputs(6, 40, 40 if not context else 23, d, heads, seed=11, context=context, context_mask=context, bias="1hij")
    kw["tie_dim"] = 3
    _run(a, st, heads, kw, f"tied_context{int(context)}")


# strict: head widths the bf16 kernels do not take (12: also the general path for one query)
STRICT_CASES = [
    ("self", 32, 2, 45, 45, dict(context=False, context_mask=False, bias="1hij", masked_rows=True)),
    ("cross", 12, 3, 30, 13, dict(bias="bhij")),
    ("cross_context_mask_only", 32, 2, 20, 9, dict(mask=False, bias="hij")),
    ("one_query", 32, 5, 1, 4, dict(masked_rows=True)),
    ("one_query_dh12", 12, 5, 1, 4, dict()),
    ("one_query_batch1", 32, 1, 1, 7, dict()),
]


@pytest.mark.parametrize("name,dh,B,i,j,opts", STRICT_CASES, ids=[c[0] for c in STRICT_CASES])
def test_attention_forward_strict(name, dh, B, i, j, opts):
    d, heads = 40, 4
    a, st = _module(d, heads, dh, strict=True, seed=dh)
    _run(a, st, heads, _inputs(B, i, j, d, heads, seed=B + i + j, **opts), "strict_" + name, strict=True)


def test_attention_forward_strict_tied():
    d, heads, dh = 40, 4, 16
    a, st = _module(d, heads, dh, strict=True, seed=3)
    kw = _inputs(4, 21, 21, d, heads, seed=5, context=False, context_mask=False)
    kw["tie_dim"] = 2
    _run(a, st, heads, kw, "strict_tied", strict=True)


def _golden():
    return torch.load(GOLDEN, weights_only=False)


@pytest.mark.parametrize("strict", [False, True])
def test_attention_forward_golden(strict):
    """every case of the reference fixture: bf16 against the fp64 oracle, strict against the reference's fp32 output"""
    fx = _golden()
    cfg = fx["cfg"]
    a = A.Attention(cfg["dim"], heads=cfg["heads"], dim_head=cfg["dim_head"])
    a.load_state_dict(fx["state"])
    a = a.cuda().eval()
    if strict:
        A.set_precision(a, "strict")
    for name, case in fx["cases"].items():
        if strict:
            kw = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in case["inputs"].items()}
            with torch.no_grad():
                out = a(**kw)
            check_strict("golden_strict_" + name, out, case["out"])
        else:
            _run(a, fx["state"], cfg["heads"], case["inputs"], "golden_" + name)


def test_attention_forward_refusals():
    d, heads = 64, 4
    a, _ = _module(d, heads, 32)
    x = torch.randn(4, 9, d, device="cuda")
    c = torch.randn(4, 5, d, device="cuda")
    keep = (x.clone(), c.clone())
    with torch.no_grad():
        with pytest.raises(ValueError, match="tie_dim"):
            a(x, tie_dim=3)
        with pytest.raises(ValueError, match="broadcast"):
            a(x, context=c, attn_bias=torch.randn(4, heads, 9, 9, device="cuda"))
        with pytest.raises(ValueError, match="context_mask"):
            a(x, context=c, mask=torch.ones(4, 9, dtype=torch.bool, device="cuda"),
              context_mask=torch.ones(4, 9, dtype=torch.bool, device="cuda"))
        with pytest.raises(ValueError, match="dim_head 48 unsupported"):
            _module(d, heads, 48)[0](x)
        with pytest.raises(ValueError, match="too long"):
            _module(d, heads, 128)[0](x[:1], context=torch.randn(1, 20000, d, device="cuda"))
        with pytest.raises(ValueError, match="dim_head 6 unsupported"):
            _module(d, heads, 6, strict=True)[0](x)
    with pytest.raises(RuntimeError, match="forward-only"):
        a(x.clone().requires_grad_())
    torch.cuda.synchronize()
    assert torch.equal(x, keep[0]) and torch.equal(c, keep[1])


def test_template_call_site():
    """alphafold2.py:762-775 with this package's Attention as template_pointwise_attn: the pooled result matches the
    template oracle"""
    b, n, T, d, heads, dh = 2, 9, 4, 64, 4, 32
    g = torch.Generator().manual_seed(3)
    x = torch.randn(b, n, n, d, generator=g)
    t = torch.randn(b, T, n, n, d, generator=g)
    x_mask = torch.rand(b, n, n, generator=g) > 0.2
    t_mask = torch.rand(b, T, n, n, generator=g) > 0.4
    t_mask[:, :, 0, :] = False                  # pairs without any valid template: pooled 0
    a, st = _module(d, heads, dh, seed=4)
    x_point = x.reshape(b * n * n, 1, d)
    t_point = t.permute(0, 2, 3, 1, 4).reshape(b * n * n, T, d)
    x_mask_point = x_mask.reshape(b * n * n, 1)
    t_mask_point = t_mask.permute(0, 2, 3, 1).reshape(b * n * n, T)
    with torch.no_grad():
        pooled = a(x_point.cuda(), context=t_point.cuda(), mask=x_mask_point.cuda(), context_mask=t_mask_point.cuda())
    pooled_mask = (t_mask_point.sum(dim=-1) > 0)[:, None, None].cuda()
    out = (pooled * pooled_mask).reshape(b, n, n, d)
    ref = TO.template_pointwise_attention(to64(st), "", x_point.double(), t_point.double(), heads, x_mask_point, t_mask_point)
    ref = (ref * pooled_mask.cpu()).reshape(b, n, n, d)
    w32 = dev(st, torch.float32)
    ac = autocast_yardstick(lambda: TO.template_pointwise_attention(w32, "", x_point.cuda(), t_point.cuda(), heads, x_mask_point.cuda(),
                                                                    t_mask_point.cuda()) * pooled_mask).reshape(b, n, n, d)
    check("template_call_site", out, ref, ac)


@pytest.mark.parametrize("tied", [False, True])
def test_axial_call_site(tied):
    """alphafold2.py:222-252: AxialAttention(...).attn on the LayerNorm'd, folded rows with the repeated pair bias (and the
    tied queries of global_query_attn) matches oracle.axial_attention"""
    b, h, w, d, heads, dh = 1, 6, 21, 64, 4, 32
    torch.manual_seed(1)
    ax = A.AxialAttention(d, heads, row_attn=True, col_attn=False, accept_edges=True, global_query_attn=tied, dim_head=dh)
    st = O.randomize_zero_init_({k: v.clone() for k, v in ax.state_dict().items()}, seed=9)
    ax.load_state_dict(st)
    ax = ax.cuda().eval()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(b, h, w, d, generator=g)
    edges = torch.randn(b, w, w, d, generator=g)
    mask = torch.rand(b, h, w, generator=g) > 0.2
    xc, ec, mc = x.cuda(), edges.cuda(), mask.cuda()
    with torch.no_grad():
        xn = F.layer_norm(xc, (d,), ax.norm.weight, ax.norm.bias)
        xf = xn.reshape(b * h, w, d)
        mf = mc.reshape(b * h, w)
        bias = ax.edges_to_attn_bias[0](ec).permute(0, 3, 1, 2).repeat_interleave(h, dim=0)   # 'b h i j -> (b x) h i j'
        out = ax.attn(xf, mask=mf, attn_bias=bias, tie_dim=h if tied else None).reshape(b, h, w, d)
    ref = O.axial_attention(to64(st), "", x.double(), heads, True, edges.double(), mask, global_query_attn=tied)
    w32 = dev(st, torch.float32)
    ac = autocast_yardstick(lambda: O.axial_attention(w32, "", xc, heads, True, ec, mc, global_query_attn=tied))
    check(f"axial_call_site_tied{int(tied)}", out, ref, ac)
