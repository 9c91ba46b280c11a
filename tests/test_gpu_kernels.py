"""-m gpu: building-block kernels (wgmma GEMM in both operand layouts, LayerNorm, rotary) against fp64 math."""
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu


def _ops():
    from alphafold2_b200 import ops
    return ops


@pytest.mark.parametrize("M,N,K,batch", [(128, 64, 64, 1), (128, 128, 64, 1), (128, 256, 64, 1), (256, 256, 256, 1),
                                         (300, 200, 136, 1), (64, 24, 32, 1), (128, 128, 128, 3), (1000, 512, 1024, 1),
                                         (260, 260, 264, 5), (4096, 2048, 256, 1)])
def test_gemm_k_major(M, N, K, batch):
    ops = _ops()
    torch.manual_seed(M + N + K)
    a = torch.randn(batch, M, K, device="cuda").bfloat16()
    b = torch.randn(batch, N, K, device="cuda").bfloat16()
    c = ops.gemm_bf16(a, b)
    ref = torch.einsum("bmk,bnk->bmn", a.double(), b.double())
    err = (c.double() - ref).abs().max().item()
    assert torch.isfinite(c).all()
    assert err <= 2e-3 * (K ** 0.5), f"max err {err}"          # fp32 accumulation of exact bf16 products


@pytest.mark.parametrize("M,N,K,batch", [(128, 64, 64, 1), (128, 128, 64, 2), (256, 256, 128, 4), (64, 64, 8, 3),
                                         (264, 136, 72, 2), (384, 384, 512, 3), (24, 24, 4, 5)])
def test_gemm_mn_major(M, N, K, batch):
    ops = _ops()
    torch.manual_seed(M + N + K)
    a = torch.randn(batch, K, M, device="cuda").bfloat16()
    b = torch.randn(batch, K, N, device="cuda").bfloat16()
    c = ops.gemm_bf16(a, b, mn_major=True)
    ref = torch.einsum("bkm,bkn->bmn", a.double(), b.double())
    err = (c.double() - ref).abs().max().item()
    assert torch.isfinite(c).all()
    assert err <= 2e-3 * (K ** 0.5), f"max err {err}"


@pytest.mark.parametrize("T,d", [(1000, 256), (77, 64), (513, 128), (40, 32), (9, 512)])
def test_layernorm(T, d):
    ops = _ops()
    torch.manual_seed(T)
    x = torch.randn(T, d, device="cuda") * 3 + 1.5
    g = torch.randn(d, device="cuda")
    b = torch.randn(d, device="cuda")
    y = ops.layernorm_bf16(x, g, b)
    ref = torch.nn.functional.layer_norm(x.double(), (d,), g.double(), b.double(), 1e-5)
    err = (y.double() - ref).abs()
    assert (err <= 2 ** -8 * ref.abs() + 1e-5).all(), f"max err {err.max().item()}"   # one bf16 rounding


def test_rotary_bit_exact():
    from alphafold2_b200 import apply_rotary_pos_emb
    fx = load_golden("rotary")
    i = fx["inputs"]
    y = apply_rotary_pos_emb(i["x"].cuda(), (i["sin"].cuda(), i["cos"].cuda()))
    assert torch.equal(y.cpu(), fx["out_fp32"])                # integer/elementwise work: bit exact
    big = torch.randn(2, 8, 300, 64, device="cuda")
    from oracle.evoformer_oracle import apply_rotary_pos_emb as o_rot, fixed_positional_embedding
    s, c = fixed_positional_embedding(64, 300)
    assert torch.equal(apply_rotary_pos_emb(big, (s.cuda(), c.cuda())).cpu(), o_rot(big.cpu(), s, c))
