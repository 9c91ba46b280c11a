"""CPU tests of the host logic that prepares operands for the fused kernels (alphafold2_b200/ops.py) and of the
numerical claims DESIGN.md makes about the epilogue activations.  No GPU, no C-ABI compute calls."""
import math

import pytest
import torch

from alphafold2_b200 import ops


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


def test_split_weight_planes_sum_exactly():
    """strict-mode weights: bf16 [rows, 3, align8(K)] planes p0 = bf16(w), p1 = bf16(w - p0), p2 = bf16(w - p0 - p1) sum to w
    exactly in fp64 (24 mantissa bits over three 8-bit planes, |w| >= 2^-110), ties and negatives included; pads are zero."""
    g = torch.Generator().manual_seed(3)
    rows, K = 41, 29
    mant = 1.0 + torch.randint(0, 1 << 23, (rows, K), generator=g).double() / (1 << 23)
    expo = torch.randint(-100, 100, (rows, K), generator=g).double()
    w = (torch.where(torch.rand(rows, K, generator=g) < 0.5, -1.0, 1.0) * mant * torch.exp2(expo)).float()
    w[0, :4] = torch.tensor([1 + 2.0 ** -8, -(1 + 2.0 ** -7 + 2.0 ** -8), 1 + 2.0 ** -8 + 2.0 ** -16 + 2.0 ** -17, 0.0])
    w[1, :3] = torch.tensor([-(2.0 ** -110) * (2 - 2.0 ** -23), 2.0 ** 127 * (2 - 2.0 ** -8 - 2.0 ** -23), -3.0])
    s = ops.split_weight(w)
    P = (K + 7) // 8 * 8
    assert s.dtype == torch.bfloat16 and tuple(s.shape) == (rows, ops.SPLIT_PLANES, P)
    p = s.double()
    assert torch.equal(p[..., 0, :] + p[..., 1, :] + p[..., 2, :], torch.nn.functional.pad(w.double(), (0, P - K)))
    assert torch.equal(s[..., 0, :K], w.to(torch.bfloat16))
    assert torch.all(s[..., K:] == 0)


def test_ops_refuse_cpu_tensors():
    with pytest.raises(RuntimeError):
        ops._require(torch.zeros(4), torch.float32, "x")
