"""-m gpu: the fused LayerNorm -> multi-segment projection kernel (csrc/proj_tc.cuh; af2_set_proj_mode 1 or 2) against
(a) the unfused LayerNorm + GEMM launches of the same library (mode 0) and (b) the fp64 oracle."""
import pytest
import torch

from gpu_util import check, to64
from oracle import evoformer_oracle as O

pytestmark = pytest.mark.gpu


def _rand_state(mod, seed):
    torch.manual_seed(seed)
    st = {k: v.clone() for k, v in mod.state_dict().items()}
    for k, v in st.items():
        if v.dim() >= 2:
            v.copy_(torch.randn_like(v) * (v.shape[-1] ** -0.5))
        elif "norm" in k and k.endswith("weight"):
            v.copy_(1 + 0.1 * torch.randn_like(v))
        else:
            v.copy_(0.1 * torch.randn_like(v))
    mod.load_state_dict(st)
    return st


def _set_mode(mode):
    from alphafold2_b200 import _lib
    _lib.load().af2_set_proj_mode(mode)


@pytest.fixture(autouse=True)
def _restore_mode():
    yield
    _set_mode(0)                                   # the library default


def _both(fn, mode):
    """run fn() under the fused mode `mode` and under the unfused launches; returns (fused, unfused)"""
    _set_mode(mode)
    a = fn()
    torch.cuda.synchronize()
    _set_mode(0)
    b = fn()
    torch.cuda.synchronize()
    return a, b


def _close(a, b, name):
    diff = (a.double() - b.double()).abs().max().item()
    rms = b.double().pow(2).mean().sqrt().item()
    print(f"{name}: fused vs unfused max diff {diff:.3e} (rms {rms:.3e})")
    assert torch.isfinite(a).all()
    assert diff <= 5e-2 * max(rms, 1e-6), f"{name}: fused/unfused differ by {diff}"


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("d,T0,T1", [(256, 8, 250), (128, 3, 391), (192, 1, 128), (256, 300, 256)])
def test_feed_forward_fused(mode, d, T0, T1):
    import alphafold2_b200 as A
    ff = A.FeedForward(dim=d)
    st = _rand_state(ff, 1)
    ff = ff.cuda().eval()
    x = torch.randn(1, T0, T1, d, generator=torch.Generator().manual_seed(2))
    a, b = _both(lambda: ff(x.cuda()), mode)
    _close(a, b, f"ff d{d}")
    check(f"proj/ff/mode{mode}/d{d}", a, O.feed_forward(to64(st), "", x.double()))


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("d,H,dh,N,row", [(256, 8, 64, 72, True), (128, 4, 32, 64, False), (256, 3, 32, 40, True)])
def test_axial_attention_fused(mode, d, H, dh, N, row):
    import alphafold2_b200 as A
    ax = A.AxialAttention(dim=d, heads=H, dim_head=dh, row_attn=row, col_attn=not row, accept_edges=True)
    st = _rand_state(ax, 3)
    ax = ax.cuda().eval()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, N, N, d, generator=g)
    m1 = torch.ones(1, N, dtype=torch.bool)
    m1[:, -5:] = False
    mask = m1[:, :, None] & m1[:, None, :]
    xc, mc = x.cuda(), mask.cuda()
    a, b = _both(lambda: ax(xc, edges=xc, mask=mc), mode)
    _close(a, b, f"axial d{d}")
    ref = O.axial_attention(to64(st), "", x.double(), H, row, edges=x.double(), mask=mask)
    check(f"proj/axial/mode{mode}/d{d}", a, ref)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("d,N,mix", [(256, 72, "outgoing"), (128, 136, "ingoing"), (256, 128, "ingoing"), (256, 70, "outgoing")])
def test_triangle_multiply_fused(mode, d, N, mix):
    import alphafold2_b200 as A
    tm = A.TriangleMultiplicativeModule(dim=d, mix=mix)
    st = _rand_state(tm, 5)
    tm = tm.cuda().eval()
    g = torch.Generator().manual_seed(6)
    x = torch.randn(1, N, N, d, generator=g)
    m1 = torch.ones(1, N, dtype=torch.bool)
    m1[:, -7:] = False
    mask = m1[:, :, None] & m1[:, None, :]
    xc, mc = x.cuda(), mask.cuda()
    a, b = _both(lambda: tm(xc, mask=mc), mode)
    _close(a, b, f"trimul d{d} {mix}")
    check(f"proj/trimul/mode{mode}/d{d}/{mix}", a, O.triangle_multiply(to64(st), "", x.double(), mix, mask))


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("d,N,S", [(256, 72, 9), (128, 64, 33), (256, 50, 5)])
def test_outer_mean_fused(mode, d, N, S):
    import alphafold2_b200 as A
    om = A.OuterMean(dim=d)
    st = _rand_state(om, 7)
    om = om.cuda().eval()
    g = torch.Generator().manual_seed(8)
    m = torch.randn(1, S, N, d, generator=g)
    mask = torch.rand(1, S, N, generator=g) > 0.2
    mc, kc = m.cuda(), mask.cuda()
    a, b = _both(lambda: om(mc, mask=kc), mode)
    _close(a, b, f"outer d{d}")
    check(f"proj/outer/mode{mode}/d{d}", a, O.outer_mean(to64(st), "", m.double(), mask))
