"""-m gpu: the template embedder (alphafold2.py:743-792, SURVEY.md 8f n3).

Kernel alone (template_pointwise_kernel through af2_template_pointwise_{bf16,f32}_state, one launch over all templates) against
fp64 math on the exact operands the kernel was given, element-wise with `check_bound`.  For pair p, head h, templates t = 0..T-1 (s_t the logits in the kernel's
domain: log2 for the bf16 instantiation, natural log for the fp32 one; w_t = softmax weights of the valid templates, or 1/T
each when none is valid; o = sum_t w_t v_t; ref = gate * o):
  * each logit is an fp32 dot product of dh terms:              |ds_t| <= E_s = dh 2^-24 sum_e |q_e k_e|
  * a logit error ds changes weights by a factor 2^ds (e^ds):   relative weight error <= 2 c max_t E_s  (c = ln 2 for exp2, 1)
  * ex2.approx / expf of the new weight and of every running-max rescale (up to T of them), the final 1 / l:
                                                                relative weight error <= (T + 2) 2^-22
    so eps_w = 2 c max_t E_s + (T + 2) 2^-22;
  * the fp32 accumulations of l and of o over T terms:          (T + 4) 2^-23 sum_t w_t |v_t|
  * the gate product and the store: bf16 rounds once,           2^-8 |ref|;  fp32: sigmoid by expf and two roundings, 4 2^-23 |ref|
  |out - ref| <= store(|ref|) + |gate| (2 eps_w + (T + 4) 2^-23) sum_t w_t |v_t|
Weights below 2^-126 of the largest (logits more than 126 apart in the log2 domain) are flushed by ex2.approx.ftz; their true
contribution is below 2^-126 max|v| and is covered by the absolute floor 1e-30 * max|v|.  pooled must equal any_t t_mask exactly.
Output buffers start as NaN, a guard after them must stay NaN, and two identical launches must be bitwise equal.

Module (af2_template_pointwise_attention) against the fp64 oracle at a hot-path shape with `check()` and the autocast yardstick;
Alphafold2.forward with templates against fixtures of the unmodified reference (bf16: `check()`, strict: `check_strict()`), and
the reference's own test_templates configuration against the fp64 oracle.
"""
import math

import pytest
import torch

from conftest import load_golden
from gpu_util import autocast_yardstick, check, check_bound, check_strict, dev
from oracle import evoformer_oracle as O
from oracle import template_oracle as TO

pytestmark = pytest.mark.gpu


def _templates_fixture():
    """alphafold2_templates.pt with its bf16-stored (bf16-exact) weights and template inputs widened to fp32."""
    fx = load_golden("alphafold2_templates")
    for key in ("state", "inputs"):
        fx[key] = {k: (v.float() if torch.is_floating_point(v) else v) for k, v in fx[key].items()}
    return fx

U = 2.0 ** -24
GUARD = 64


def _masks(kind, B, T, pairs, g):
    xm = tm = None
    if kind in ("random", "all_t_masked", "x_masked", "wide_logits"):
        xm = torch.rand(B * pairs, generator=g) > 0.15
        tm = torch.rand(B * T * pairs, generator=g) > 0.3
    if kind == "all_t_masked":                       # every template masked at a third of the pairs: uniform mean, pooled 0
        sel = torch.rand(B, 1, pairs, generator=g) < 0.34
        tm = (tm.view(B, T, pairs) & ~sel).reshape(-1)
    if kind == "x_masked":                           # half the pairs masked by x_mask, their templates valid
        xm = torch.rand(B * pairs, generator=g) > 0.5
        tm = torch.ones(B * T * pairs, dtype=torch.bool)
    return xm, tm


def _reference(q, gate, kv, xm, tm, B, T, heads, dh, log2):
    P, I = q.shape
    pairs = P // B
    q64 = q.double().view(B, pairs, heads, dh)
    k64 = kv.double().view(B, T, pairs, 2 * I)[..., :I].reshape(B, T, pairs, heads, dh)
    v64 = kv.double().view(B, T, pairs, 2 * I)[..., I:].reshape(B, T, pairs, heads, dh)
    s = torch.einsum("bphe,btphe->bpht", q64, k64)
    es = dh * U * torch.einsum("bphe,btphe->bpht", q64.abs(), k64.abs())
    valid = torch.ones(B, pairs, T, dtype=torch.bool, device=q.device)
    if tm is not None:
        valid = tm.view(B, T, pairs).permute(0, 2, 1).clone()
    pooled = valid.any(-1).double().reshape(P)
    if xm is not None:
        valid = valid & xm.view(B, pairs, 1)
    valid = valid[:, :, None, :].expand(B, pairs, heads, T)
    none = ~valid.any(-1, keepdim=True)
    logit = s * (math.log(2.0) if log2 else 1.0)
    logit = torch.where(valid, logit, torch.full_like(logit, -float("inf")))
    w = torch.softmax(torch.where(none, torch.zeros_like(logit), logit), dim=-1)
    o = torch.einsum("bpht,btphe->bphe", w, v64)
    absv = torch.einsum("bpht,btphe->bphe", w, v64.abs())
    g64 = gate.double().view(B, pairs, heads, dh)
    if not log2:
        g64 = torch.sigmoid(g64)
    ref = (g64 * o).reshape(P, I)
    c = math.log(2.0) if log2 else 1.0
    eps_w = 2 * c * es.amax(-1, keepdim=True) + (T + 2) * 2.0 ** -22
    store = 2.0 ** -8 if log2 else 4 * 2.0 ** -23
    bound = store * ref.abs() + (g64.abs() * (2 * eps_w + (T + 4) * 2.0 ** -23) * absv).reshape(P, I)
    bound = bound + 1e-30 * v64.abs().max().item()
    return ref, pooled, bound


def _kernel_case(name, B, T, n, heads, dh, kind, dtype=torch.bfloat16, seed=0):
    from alphafold2_b200 import ops
    g = torch.Generator().manual_seed(seed)
    pairs, I = n * n, heads * dh
    P = B * pairs
    scale = 1.0
    if kind == "wide_logits":                        # logits spread over about +-200 (log2 domain)
        scale = (200.0 / 3.0 / math.sqrt(dh)) ** 0.5
    q = (torch.randn(P, I, generator=g) * scale).to(dtype)
    kv = (torch.randn(B * T * pairs, 2 * I, generator=g) * scale).to(dtype)
    kv[:, I:] = (torch.randn(B * T * pairs, I, generator=g)).to(dtype)
    gate = (torch.rand(P, I, generator=g) if dtype == torch.bfloat16 else torch.randn(P, I, generator=g) * 2).to(dtype)
    xm, tm = _masks(kind, B, T, pairs, g)
    cu = lambda t: None if t is None else t.cuda()  # noqa: E731
    q, kv, gate, xm, tm = cu(q), cu(kv), cu(gate), cu(xm), cu(tm)
    outs = []
    for _ in range(2):
        obuf = torch.full((P * I + GUARD,), float("nan"), dtype=dtype, device="cuda")
        pbuf = torch.full((P + GUARD,), float("nan"), dtype=torch.float32, device="cuda")
        ops.template_pointwise(q, gate, kv, B, T, heads, dh, x_mask=xm, t_mask=tm, out=obuf, pooled=pbuf)
        torch.cuda.synchronize()
        assert torch.isnan(obuf[P * I:].float()).all() and torch.isnan(pbuf[P:]).all(), f"{name}: guard written"
        outs.append((obuf, pbuf))
    assert torch.equal(outs[0][0].view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                       outs[1][0].view(torch.int16 if dtype == torch.bfloat16 else torch.int32)), f"{name}: launches differ"
    ref, pooled, bound = _reference(q, gate, kv, xm, tm, B, T, heads, dh, dtype == torch.bfloat16)
    assert torch.equal(outs[0][1][:P].double(), pooled), f"{name}: pooled != any_t t_mask"
    check_bound(name, outs[0][0][:P * I].view(P, I), ref, bound)


SHAPES = [(T, h, dh, B) for T in (1, 2, 3, 4, 10, 13) for (h, dh) in ((1, 32), (1, 64), (8, 32), (8, 64)) for B in (1, 2)]


@pytest.mark.parametrize("T,heads,dh,B", SHAPES)
def test_pointwise_kernel_shapes(T, heads, dh, B):
    _kernel_case(f"tpl_kernel T{T} h{heads} dh{dh} b{B} n37", B, T, 37, heads, dh, "random", seed=T * 100 + heads * 10 + dh + B)


@pytest.mark.parametrize("kind", ["none", "random", "all_t_masked", "x_masked", "wide_logits"])
@pytest.mark.parametrize("T,heads,dh", [(3, 8, 64), (10, 1, 32), (1, 8, 32)])
def test_pointwise_kernel_masks(kind, T, heads, dh):
    _kernel_case(f"tpl_kernel {kind} T{T} h{heads} dh{dh}", 2, T, 37, heads, dh, kind, seed=7 + T)


@pytest.mark.parametrize("n,B,T,heads,dh", [(1, 2, 1, 8, 64), (1, 1, 13, 1, 32), (257, 1, 4, 8, 64), (257, 1, 2, 1, 32)])
def test_pointwise_kernel_sizes(n, B, T, heads, dh):
    _kernel_case(f"tpl_kernel n{n} b{B} T{T} h{heads} dh{dh}", B, T, n, heads, dh, "random", seed=n + T)


@pytest.mark.parametrize("kind", ["random", "all_t_masked", "x_masked", "wide_logits"])
@pytest.mark.parametrize("T,heads,dh", [(4, 8, 64), (13, 2, 32)])
def test_pointwise_kernel_f32(kind, T, heads, dh):
    _kernel_case(f"tpl_kernel_f32 {kind} T{T} h{heads} dh{dh}", 2, T, 37, heads, dh, kind, dtype=torch.float32, seed=3 + T)


def test_pointwise_kernel_rejects_bad_shapes():
    from alphafold2_b200 import ops
    z = lambda *s: torch.zeros(*s, dtype=torch.bfloat16, device="cuda")  # noqa: E731
    with pytest.raises(ValueError, match="dim_head"):
        ops.template_pointwise(z(4, 48), z(4, 48), z(8, 96), 1, 2, 1, 48)
    with pytest.raises(ValueError, match="templates"):
        ops.template_pointwise(z(4, 64), z(4, 64), z(0, 128), 1, 0, 1, 64)


# ------------------------------------------------------------------------------------------------------------------------
# module and model
# ------------------------------------------------------------------------------------------------------------------------
def test_pointwise_module_hot_shape_vs_oracle():
    """d 256, H 8, dh 64, n 160, T 4: af2_template_pointwise_attention (GEMMs + kernel + to_out with the pooled row scale)."""
    import alphafold2_b200 as A
    torch.manual_seed(3)
    d, H, dh, n, T = 256, 8, 64, 160, 4
    att = A.Attention(dim=d, heads=H, dim_head=dh)
    st = O.randomize_zero_init_({k: v.clone() for k, v in att.state_dict().items()}, std=0.05)
    att.load_state_dict(st)
    att = att.cuda().eval()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, n, n, d, generator=g)
    t = torch.randn(T, n, n, d, generator=g)
    mask = torch.ones(1, n, dtype=torch.bool)
    mask[:, -20:] = False
    tm = torch.rand(1, T, n, generator=g) > 0.2
    tm[:, :, 7] = False
    tm[:, T - 1] = False
    xm = mask[:, :, None] & mask[:, None, :]
    tm2 = (tm[:, :, :, None] & tm[:, :, None, :]).reshape(T, n, n)
    with torch.no_grad():
        out = att.add_context_(x.cuda().clone(), t.cuda(), xm.cuda(), tm2.cuda())
    torch.cuda.synchronize()
    w64 = dev(st, torch.float64)

    def oracle(w, xx, tt):
        xp = xx.reshape(n * n, 1, d)
        tp = tt.permute(1, 2, 0, 3).reshape(n * n, T, d)
        tmp = tm2.cuda().permute(1, 2, 0).reshape(n * n, T)
        o = TO.template_pointwise_attention(w, "", xp, tp, H, xm.cuda().reshape(n * n, 1), tmp)
        return (o * tmp.any(-1)[:, None, None].to(o.dtype)).reshape(1, n, n, d)

    with torch.no_grad():
        ref = oracle(w64, x.double().cuda(), t.double().cuda())
        ac = autocast_yardstick(lambda: oracle(dev(st), x.cuda(), t.cuda())).float()
    check("template_pointwise/oracle/d256n160T4", out.double() - x.double().cuda(), ref, ac.double())


def _af2(fx_cfg, state, precision):
    import alphafold2_b200 as A
    model = A.Alphafold2(**fx_cfg)
    assert not model.load_state_dict(state, strict=False).unexpected_keys
    return A.set_precision(model.cuda().eval(), precision)


@pytest.mark.parametrize("precision", ["bf16", "strict"])
@pytest.mark.parametrize("call", ["feats_angles", "feats", "angles"])
def test_alphafold2_templates_golden(call, precision):
    fx = _templates_fixture()
    i = {k: v.cuda() for k, v in fx["inputs"].items()}
    model = _af2(fx["cfg"], fx["state"], precision)
    kw = {k: i[k] for k in fx["calls"][call]}
    ret = model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"], **kw)
    if precision == "strict":
        check_strict(f"strict/alphafold2_templates/{call}/golden/distance", ret.distance, fx["out_fp32"][call])
    else:
        check(f"alphafold2_templates/{call}/golden/distance", ret.distance, fx["out_fp64"][call], fx["out_autocast_bf16"][call])


def test_alphafold2_reference_test_templates_config():
    """tests/test_attention.py::test_templates of the reference (templates_angles_feats_dim = 32), through our Alphafold2,
    against the fp64 oracle."""
    import alphafold2_b200 as A
    torch.manual_seed(9)
    cfg = dict(dim=32, depth=2, heads=2, dim_head=32, templates_dim=32, templates_angles_feats_dim=32)
    model = A.Alphafold2(**cfg)
    st = O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()})
    model.load_state_dict(st)
    model = model.cuda().eval()
    seq, msa = torch.randint(0, 21, (2, 16)), torch.randint(0, 21, (2, 5, 16))
    mask, msa_mask = torch.ones(2, 16, dtype=torch.bool), torch.ones(2, 5, 16, dtype=torch.bool)
    feats, angles, tm = torch.randn(2, 3, 16, 16, 32), torch.randn(2, 3, 16, 32), torch.ones(2, 3, 16, dtype=torch.bool)
    ret = model(seq.cuda(), msa.cuda(), mask=mask.cuda(), msa_mask=msa_mask.cuda(), templates_feats=feats.cuda(),
                templates_angles=angles.cuda(), templates_mask=tm.cuda())
    args = dict(templates_feats=feats, templates_angles=angles, templates_mask=tm, templates_embed_layers=4)
    ref = TO.alphafold2_distogram({k: v.double() for k, v in st.items()}, seq, msa, mask, msa_mask, 2, 2, dtype=torch.float64, **args)
    ac = autocast_yardstick(lambda: TO.alphafold2_distogram(dev(st), seq.cuda(), msa.cuda(), mask.cuda(), msa_mask.cuda(), 2, 2,
                                                            **{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in args.items()}))
    check("alphafold2_reference_test_templates/oracle/distance", ret.distance, ref, ac.float().cpu())


def test_alphafold2_template_errors():
    import alphafold2_b200 as A
    model = A.Alphafold2(dim=32, depth=1, heads=2, dim_head=32, templates_embed_layers=1).cuda().eval()
    b, n, T = 1, 8, 2
    seq, msa = torch.randint(0, 21, (b, n)).cuda(), torch.randint(0, 21, (b, 2, n)).cuda()
    mask = torch.ones(b, n, dtype=torch.bool).cuda()
    feats, angles = torch.randn(b, T, n, n, 32).cuda(), torch.randn(b, T, n, 55).cuda()
    tm = torch.ones(b, T, n, dtype=torch.bool).cuda()
    with pytest.raises(ValueError, match="mask"):
        model(seq, msa, templates_feats=feats, templates_mask=tm)
    with pytest.raises(ValueError, match="templates_mask"):
        model(seq, msa, mask=mask, templates_feats=feats)
    with pytest.raises(ValueError, match="templates_mask"):
        model(seq, msa, mask=mask, templates_angles=angles)
    with pytest.raises(NotImplementedError, match="recyclables"):
        model(seq, msa, mask=mask, recyclables=object())
