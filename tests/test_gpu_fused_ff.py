"""-m gpu: the fused GEGLU feed-forward kernel (csrc/ff_fused.cuh) against the two-GEMM composition it replaces, built from
the same packed tensors (LayerNorm, gated GELU GEMM, residual GEMM), bit for bit; that it is the kernel that runs; and the
fp64 oracle at the shapes it serves."""
import pytest
import torch

from gpu_util import check, to64
from oracle import evoformer_oracle as O

pytestmark = pytest.mark.gpu


def _ff(d, seed=1):
    import alphafold2_b200 as A
    ff = A.FeedForward(dim=d)
    torch.manual_seed(seed)
    st = {k: v.clone() for k, v in ff.state_dict().items()}
    for k, v in st.items():
        if v.dim() >= 2:
            v.copy_(torch.randn_like(v) * (v.shape[-1] ** -0.5))
        elif k == "norm.weight":
            v.copy_(1 + 0.1 * torch.randn_like(v))
        else:
            v.copy_(0.1 * torch.randn_like(v))
    ff.load_state_dict(st)
    return ff.cuda().eval(), st


def _two_gemm(pk, x):
    """x + FeedForward(x) through the separate kernels: LayerNorm -> gated GELU GEMM (h to memory) -> residual GEMM."""
    from alphafold2_b200 import ops
    t = pk.tensors
    d = x.shape[-1]
    hidden = t["w2"].shape[1]
    x2 = x.reshape(-1, d).clone()
    T = x2.shape[0]
    xn = ops.layernorm_bf16(x2, t["g"], t["b"])
    h = torch.empty(T, hidden, dtype=torch.bfloat16, device=x.device)
    ops.gemm_bf16_epilogue(xn.view(1, T, d), t["w1"].view(1, -1, d), h, bn=256, mode=ops.EPI_GATED_BF16,
                           act=ops.ACT_GELU, bias=t["b1"], ld_out=hidden, out_cols=hidden)
    ops.gemm_bf16_epilogue(h.view(1, T, hidden), t["w2"].view(1, d, hidden), x2, bn=256 if d > 128 else 128,
                           mode=ops.EPI_RESID_F32, bias=t["b2"], resid=x2, ld_resid=d, ld_out=d)
    return x2.view(x.shape)


@pytest.mark.parametrize("d,T", [(256, 65536), (256, 32768), (256, 1), (256, 65), (256, 127), (256, 129),
                                 (256, 2000), (256, 76800), (128, 391 * 3)])
def test_fused_equals_two_gemm(d, T):
    from alphafold2_b200 import ops
    ff, _ = _ff(d)
    pk = ff.packed()
    x = torch.randn(T, d, generator=torch.Generator().manual_seed(T), device="cpu").cuda()
    ref = _two_gemm(pk, x)
    out = ops.feed_forward_(pk, x.clone())
    torch.cuda.synchronize()
    diff = (out != ref).sum().item()
    assert torch.equal(out, ref), f"d={d} T={T}: {diff} elements differ, max |diff| {(out - ref).abs().max().item():.3e}"


@pytest.mark.parametrize("d,launches", [(256, 2), (128, 2), (192, 3)])
def test_fused_kernel_runs(d, launches):
    from alphafold2_b200 import _lib, ops
    ff, _ = _ff(d)
    pk = ff.packed()
    x = torch.randn(300, d, device="cuda")
    lib = _lib.load()
    ops.feed_forward_(pk, x)           # packs, allocates the workspace
    n0 = lib.af2_launch_count()
    ops.feed_forward_(pk, x)
    assert lib.af2_launch_count() - n0 == launches


@pytest.mark.parametrize("d,T0,T1", [(256, 256, 256), (256, 128, 256), (256, 8, 250), (128, 3, 391)])
def test_fused_oracle(d, T0, T1):
    ff, st = _ff(d)
    x = torch.randn(1, T0, T1, d, generator=torch.Generator().manual_seed(2))
    check(f"fused_ff/oracle/d{d}T{T0}x{T1}", ff(x.cuda()), O.feed_forward(to64(st), "", x.double()))
