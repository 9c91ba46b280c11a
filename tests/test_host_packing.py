"""CPU tests of the host logic that prepares operands for the fused kernels (alphafold2_b200/ops.py) and of the
numerical claims DESIGN.md makes about the epilogue activations.  No GPU, no C-ABI compute calls."""
import math

import pytest
import torch

from alphafold2_b200 import ops


def test_cat_segments_folds_layernorm_affine():
    """W' = W diag(gamma), b' = W beta + b: (x_hat W'^T + b') == Linear(LayerNorm(x)) up to the bf16 rounding of W'."""
    g = torch.Generator().manual_seed(1)
    d = 64
    x = torch.randn(50, d, generator=g, dtype=torch.float64) * 2 + 0.5
    gamma, beta = torch.randn(d, generator=g), torch.randn(d, generator=g)
    w1, b1 = torch.randn(40, d, generator=g) * 0.1, torch.randn(40, generator=g)
    w2, b2 = torch.randn(300, d, generator=g) * 0.1, torch.randn(300, generator=g)
    wc, bc = ops._cat_segments([w1, w2], [b1, b2], gamma, beta)
    assert wc.shape == (256 + 512, d) and bc.shape == (256 + 512,)          # each segment starts on a 256-row tile
    xh = (x - x.mean(-1, keepdim=True)) / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-5)
    ln = xh * gamma.double() + beta.double()
    ref1 = ln @ w1.double().t() + b1.double()
    ref2 = ln @ w2.double().t() + b2.double()
    got = xh @ wc.double().t() + bc.double()
    scale = ref2.abs().max()
    assert (got[:, :40] - ref1).abs().max() < 2e-2 * scale                  # bf16 weights: 2^-9 relative per term
    assert (got[:, 256:556] - ref2).abs().max() < 2e-2 * scale
    assert torch.all(got[:, 40:256] == 0) and torch.all(got[:, 556:] == 0)  # padding rows: zero weights, zero bias


def test_pack_gated_interleaves_value_and_gate_rows():
    n_out, k, half = 200, 8, 128
    wv = torch.arange(n_out * k, dtype=torch.float32).reshape(n_out, k)
    wg = -wv
    bv, bg = torch.arange(n_out, dtype=torch.float32), -torch.arange(n_out, dtype=torch.float32)
    w, b = ops.pack_gated(wv, bv, wg, bg, half)
    assert w.shape == (2 * 2 * half, k)
    assert torch.equal(w[:128], wv[:128]) and torch.equal(w[128:256], wg[:128])       # tile 0: [value | gate]
    assert torch.equal(w[256:256 + 72], wv[128:]) and torch.equal(w[384:384 + 72], wg[128:])
    assert torch.all(w[256 + 72:384] == 0) and torch.all(w[384 + 72:] == 0)
    assert torch.equal(b[128:256], bg[:128]) and torch.equal(b[256:256 + 72], bv[128:])


def _gelu_fast(x: torch.Tensor) -> torch.Tensor:
    """The kernel's GELU (common.cuh gelu_fast2) restated in fp64: x / (1 + 2^(x Q(min(x^2, 49))))."""
    x2 = torch.clamp(x * x, max=49.0)
    q = x2 * 0.0009112266168574351 - 0.10617732324431346
    q = x2 * q - 2.3017271259199106
    return x / (1.0 + torch.exp2(x * q))


def test_gelu_fast_matches_erf_gelu():
    x = torch.linspace(-30, 30, 600001, dtype=torch.float64)
    ref = 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    err = (_gelu_fast(x) - ref).abs()
    assert err.max() < 5.5e-5                                               # DESIGN.md section 2
    assert torch.isfinite(_gelu_fast(torch.tensor([-1e4, 1e4, 0.0], dtype=torch.float64))).all()
    # the clamp on x^2 keeps the tails exact: gelu(-x) -> 0, gelu(x) -> x
    assert abs(float(_gelu_fast(torch.tensor([-20.0], dtype=torch.float64)))) < 1e-12
    assert abs(float(_gelu_fast(torch.tensor([20.0], dtype=torch.float64))) - 20.0) < 1e-9


def test_ops_refuse_cpu_tensors():
    with pytest.raises(RuntimeError):
        ops._require(torch.zeros(4), torch.float32, "x")
