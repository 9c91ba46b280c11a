"""-m gpu: every module of the hot path through the C ABI against (a) golden vectors generated from the
unmodified reference and (b) the fp64 oracle on seeded inputs at larger / ragged shapes."""
import pytest
import torch

from conftest import load_golden
from gpu_util import check, to64
from oracle import evoformer_oracle as O

pytestmark = pytest.mark.gpu


def _mod(cls, fx, **kw):
    import alphafold2_b200 as A
    m = getattr(A, cls)(**kw)
    m.load_state_dict(fx["state"])
    return m.cuda().eval()


def _cu(t):
    return None if t is None else t.cuda()


def test_feed_forward_golden():
    fx = load_golden("feed_forward")
    m = _mod("FeedForward", fx, dim=fx["cfg"]["dim"])
    out = m(fx["inputs"]["x"].cuda())
    check("feed_forward/golden", out, fx["out_fp64"], fx["out_autocast_bf16"])


@pytest.mark.parametrize("name,row,edges", [("axial_row_edges_masked", True, True), ("axial_col_masked", False, False),
                                            ("axial_col_edges_pair", False, True), ("axial_row_nomask", True, True)])
def test_axial_attention_golden(name, row, edges):
    fx = load_golden(name)
    c, i = fx["cfg"], fx["inputs"]
    m = _mod("AxialAttention", fx, dim=c["dim"], heads=c["heads"], dim_head=c["dim_head"], row_attn=row,
             col_attn=not row, accept_edges=edges)
    out = m(i["x"].cuda(), edges=_cu(i.get("edges")), mask=_cu(i.get("mask")))
    check(f"{name}/golden", out, fx["out_fp64"], fx["out_autocast_bf16"])


@pytest.mark.parametrize("mix", ["outgoing", "ingoing"])
def test_triangle_multiply_golden(mix):
    fx = load_golden(f"triangle_multiply_{mix}")
    i = fx["inputs"]
    m = _mod("TriangleMultiplicativeModule", fx, dim=fx["cfg"]["dim"], mix=mix)
    out = m(i["x"].cuda(), mask=i["mask"].cuda())
    check(f"triangle_multiply_{mix}/golden", out, fx["out_fp64"], fx["out_autocast_bf16"])


@pytest.mark.parametrize("name", ["outer_mean_masked", "outer_mean_nomask"])
def test_outer_mean_golden(name):
    fx = load_golden(name)
    i = fx["inputs"]
    m = _mod("OuterMean", fx, dim=fx["cfg"]["dim"])
    out = m(i["m"].cuda(), mask=_cu(i.get("mask")))
    check(f"{name}/golden", out, fx["out_fp64"], fx["out_autocast_bf16"])


def test_evoformer_block_golden():
    fx = load_golden("evoformer_block")
    c, i = fx["cfg"], fx["inputs"]
    m = _mod("EvoformerBlock", fx, dim=c["dim"], seq_len=c["N"], heads=c["heads"], dim_head=c["dim_head"],
             attn_dropout=0., ff_dropout=0.)
    x, mm, _, _ = m((i["x"].cuda(), i["m"].cuda(), i["mask"].cuda(), i["msa_mask"].cuda()))
    check("evoformer_block/golden/x", x, fx["out_fp64"][0], fx["out_autocast_bf16"][0])
    check("evoformer_block/golden/m", mm, fx["out_fp64"][1], fx["out_autocast_bf16"][1])


@pytest.mark.parametrize("name,depth", [("evoformer_depth2", 2), ("evoformer_nomask", 1)])
def test_evoformer_golden(name, depth):
    fx = load_golden(name)
    c, i = fx["cfg"], fx["inputs"]
    m = _mod("Evoformer", fx, depth=depth, dim=c["dim"], seq_len=c["N"], heads=c["heads"], dim_head=c["dim_head"],
             attn_dropout=0., ff_dropout=0.)
    x, mm = m(i["x"].cuda(), i["m"].cuda(), mask=_cu(i.get("mask")), msa_mask=_cu(i.get("msa_mask")))
    check(f"{name}/golden/x", x, fx["out_fp64"][0], fx["out_autocast_bf16"][0])
    check(f"{name}/golden/m", mm, fx["out_fp64"][1], fx["out_autocast_bf16"][1])


def test_alphafold2_distogram_golden():
    import alphafold2_b200 as A
    fx = load_golden("alphafold2_distogram")
    i = fx["inputs"]
    model = A.Alphafold2(**fx["cfg"])
    missing = model.load_state_dict(fx["state"], strict=False)
    assert not missing.unexpected_keys
    model = model.cuda().eval()
    ret = model(i["seq"].cuda(), i["msa"].cuda(), mask=i["mask"].cuda(), msa_mask=i["msa_mask"].cuda())
    assert tuple(ret.distance.shape) == tuple(fx["out_fp64"].shape)
    check("alphafold2/golden/distance", ret.distance, fx["out_fp64"])
    ret = model(i["seq"].cuda(), mask=i["mask"].cuda())
    check("alphafold2/golden/distance_no_msa", ret.distance, fx["out_fp32_no_msa"])


# ------------------------------- seeded inputs vs the fp64 oracle, bigger / ragged ------------------------------
def _rand_state(mod, seed):
    torch.manual_seed(seed)
    st = {k: v.clone() for k, v in mod.state_dict().items()}
    for k, v in st.items():
        if v.dim() >= 2:
            v.copy_(torch.randn_like(v) * (v.shape[-1] ** -0.5))
        elif k.endswith("norm.weight") or ".norm." in k and k.endswith("weight"):
            v.copy_(1 + 0.1 * torch.randn_like(v))
        else:
            v.copy_(0.1 * torch.randn_like(v))
    mod.load_state_dict(st)
    return st


@pytest.mark.parametrize("d,H,dh,N,S,B", [(128, 4, 32, 64, 4, 1), (256, 8, 64, 136, 40, 1), (64, 2, 64, 300, 130, 1),
                                          (32, 2, 32, 128, 5, 2)])
def test_evoformer_block_oracle(d, H, dh, N, S, B):
    import alphafold2_b200 as A
    blk = A.EvoformerBlock(dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
    st = _rand_state(blk, 5)
    blk = blk.cuda().eval()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, N, N, d, generator=g)
    m = torch.randn(B, S, N, d, generator=g)
    mask1 = torch.ones(B, N, dtype=torch.bool); mask1[:, -N // 8:] = False
    mask = mask1[:, :, None] & mask1[:, None, :]
    msa_mask = torch.rand(B, S, N, generator=g) > 0.1
    msa_mask[:, :, -N // 8:] = False
    msa_mask[:, 0, : N - N // 8] = True
    xo, mo, _, _ = blk((x.cuda(), m.cuda(), mask.cuda(), msa_mask.cuda()))
    rx, rm = O.evoformer_block(to64(st), "", x.double(), m.double(), H, mask, msa_mask, chunk=16)
    check(f"evoformer_block/oracle/d{d}N{N}S{S}/x", xo, rx)
    check(f"evoformer_block/oracle/d{d}N{N}S{S}/m", mo, rm)


# single modules at widths and lengths the shapes above miss: d = 192, 3 heads of 32, token counts that are no multiple of a
# 64-row tile, N = 70 / 72 / 136 (padded channel-major pitches) with masks
@pytest.mark.parametrize("d,T0,T1", [(256, 8, 250), (128, 3, 391), (192, 1, 128), (256, 300, 256)])
def test_feed_forward_oracle(d, T0, T1):
    import alphafold2_b200 as A
    ff = A.FeedForward(dim=d)
    st = _rand_state(ff, 1)
    ff = ff.cuda().eval()
    x = torch.randn(1, T0, T1, d, generator=torch.Generator().manual_seed(2))
    check(f"feed_forward/oracle/d{d}T{T0}x{T1}", ff(x.cuda()), O.feed_forward(to64(st), "", x.double()))


@pytest.mark.parametrize("d,H,dh,N,row", [(256, 8, 64, 72, True), (128, 4, 32, 64, False), (256, 3, 32, 40, True)])
def test_axial_attention_oracle(d, H, dh, N, row):
    import alphafold2_b200 as A
    ax = A.AxialAttention(dim=d, heads=H, dim_head=dh, row_attn=row, col_attn=not row, accept_edges=True)
    st = _rand_state(ax, 3)
    ax = ax.cuda().eval()
    x = torch.randn(1, N, N, d, generator=torch.Generator().manual_seed(4))
    m1 = torch.ones(1, N, dtype=torch.bool)
    m1[:, -5:] = False
    mask = m1[:, :, None] & m1[:, None, :]
    xc = x.cuda()
    out = ax(xc, edges=xc, mask=mask.cuda())
    ref = O.axial_attention(to64(st), "", x.double(), H, row, edges=x.double(), mask=mask)
    check(f"axial_attention/oracle/d{d}H{H}x{dh}N{N}", out, ref)


@pytest.mark.parametrize("d,N,mix", [(256, 72, "outgoing"), (128, 136, "ingoing"), (256, 128, "ingoing"), (256, 70, "outgoing")])
def test_triangle_multiply_oracle(d, N, mix):
    import alphafold2_b200 as A
    tm = A.TriangleMultiplicativeModule(dim=d, mix=mix)
    st = _rand_state(tm, 5)
    tm = tm.cuda().eval()
    x = torch.randn(1, N, N, d, generator=torch.Generator().manual_seed(6))
    m1 = torch.ones(1, N, dtype=torch.bool)
    m1[:, -7:] = False
    mask = m1[:, :, None] & m1[:, None, :]
    out = tm(x.cuda(), mask=mask.cuda())
    check(f"triangle_multiply/oracle/d{d}N{N}/{mix}", out, O.triangle_multiply(to64(st), "", x.double(), mix, mask))


@pytest.mark.parametrize("d,N,S", [(256, 72, 9), (128, 64, 33), (256, 50, 5)])
def test_outer_mean_oracle(d, N, S):
    import alphafold2_b200 as A
    om = A.OuterMean(dim=d)
    st = _rand_state(om, 7)
    om = om.cuda().eval()
    g = torch.Generator().manual_seed(8)
    m = torch.randn(1, S, N, d, generator=g)
    mask = torch.rand(1, S, N, generator=g) > 0.2
    out = om(m.cuda(), mask=mask.cuda())
    check(f"outer_mean/oracle/d{d}N{N}S{S}", out, O.outer_mean(to64(st), "", m.double(), mask))


def test_no_cpu_fallback():
    import alphafold2_b200 as A
    ff = A.FeedForward(dim=64)
    with pytest.raises(RuntimeError):
        ff(torch.randn(4, 64))
