"""CPU controls of the bounds in embed_bounds.py: each kernel of test_gpu_embed_heads.py is emulated on the CPU (bf16
operands by .bfloat16(), fp32 accumulation by float32 matmul, the bf16 store of the angle MLP's hidden activation), the
faithful emulation must pass every gate, and each plausible wrong variant must fail the gate named beside it:

  A  template embed   truncating fp32 -> bf16 conversion          bf16 GEMM bound (gemm_f32_bound)
                      dropped bias (bf16 and strict)              GEMM bound
  B  angle MLP        rows written at row0 - 1 / row0 + 1         row layout (outside rows unchanged, inside rows finite)
                      dropped b2 (bf16 and strict)                stage-2 bound
                      tanh-GELU (strict)                          stage-2 bound
                      K pad columns not zeroed                    stage-1 bound (non-finite; see below)
  C  pair init        rel = j - i instead of i - j                x bound
                      clamp at R - 1 instead of R                 x bound
  D  distogram        no symmetrisation                           distogram bound
                      unbiased variance                           distogram bound
                      eps 1e-6 instead of 1e-5                    distogram bound

Two mutants cannot be seen by an output bound, and the GPU test catches them another way.  The K pad columns of the bf16
weight are zero, so finite garbage in the pad columns of the converted activations multiplies to exactly 0; the GPU test
fills its workspace with NaN, which turns an unzeroed pad into NaN (NaN x 0 = NaN) -- emulated here with NaN garbage.  The
tanh-GELU differs from the erf-GELU by at most ~2e-4 absolute, below the 2^-8 |h| of the bf16 store, so only strict mode
sees it.
"""
import pytest
import torch

import embed_bounds as E

F = torch.float32


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bfr(x):
    return x.bfloat16().float()


def _trunc(x):
    """fp32 -> bf16 by truncation (dropping the low 16 bits) instead of rounding to nearest"""
    return (x.contiguous().view(torch.int32) & -65536).view(F)


# ------------------------------------------------------------------------------------------------------------------------
# A. to_template_embed
# ------------------------------------------------------------------------------------------------------------------------
def _emu_embed(feats, w, bias, strict, conv=_bfr, with_bias=True):
    a, ww = (feats, w) if strict else (conv(feats), _bfr(w))
    return a @ ww.T + (bias if with_bias else 0)


@pytest.mark.parametrize("K", [1, 32, 55, 200])
@pytest.mark.parametrize("strict", [False, True])
def test_template_embed_bound(K, strict):
    g = _gen(K)
    rows, d = 129, 36
    feats = torch.randn(rows, K, generator=g)
    w, bias = torch.randn(d, K, generator=g) * K ** -0.5, torch.randn(d, generator=g)
    ref, bound = E.template_embed_ref(feats, w, bias, strict)
    assert E.within(_emu_embed(feats, w, bias, strict), ref, bound)
    assert not E.within(_emu_embed(feats, w, bias, strict, with_bias=False), ref, bound), "dropped bias"
    if not strict:
        assert not E.within(_emu_embed(feats, w, bias, strict, conv=_trunc), ref, bound), "truncating conversion"


# ------------------------------------------------------------------------------------------------------------------------
# B. template angle MLP
# ------------------------------------------------------------------------------------------------------------------------
def _emu_angles(angles, w1, b1, w2, b2, m, row0, strict, shift=0, with_b2=True, gelu="none", pad=0.0):
    """-> (hidden activation as the kernel's workspace holds it, m with rows row0 + shift .. written)"""
    B, T, n, K = angles.shape
    Kp = E.a8(K)
    a = torch.full((B * T * n, Kp), pad)
    a[:, :K] = angles.reshape(-1, K)
    w1p = torch.zeros(w1.shape[0], Kp)
    w1p[:, :K] = w1
    if strict:
        h = a @ w1p.T + b1
        out = torch.nn.functional.gelu(h, approximate=gelu) @ w2.T
    else:
        h = torch.nn.functional.gelu(_bfr(a) @ _bfr(w1p).T + b1).bfloat16()
        out = h.float() @ _bfr(w2).T
    out = out + (b2 if with_b2 else 0)
    m = m.clone()
    m[:, row0 + shift:row0 + shift + T] = out.view(B, T, n, -1)
    return h, m


def _angle_gates(angles, w1, b1, w2, b2, m0, m1, h, row0, strict):
    B, T, n, K = angles.shape
    rows = m1[:, row0:row0 + T].reshape(B * T * n, -1)
    a = angles.reshape(-1, K)
    return dict(layout=E.angle_rows_layout(m0, m1, row0, T),
                stage1=E.within(h, *E.angles_stage1_ref(a, w1, b1, strict)),
                stage2=E.within(rows, *E.angles_stage2_ref(h, w2, b2, strict)),
                module=E.within(rows, *E.angles_module_ref(a, w1, b1, w2, b2, strict)))


@pytest.mark.parametrize("K", [3, 32, 55])
@pytest.mark.parametrize("strict", [False, True])
def test_template_angles_bound(K, strict):
    g = _gen(100 + K)
    B, T, n, d, S = 2, 3, 5, 64, 2
    m_rows, row0 = S + T + 1, S
    angles = torch.randn(B, T, n, K, generator=g)
    w1, b1 = torch.randn(d, K, generator=g) * K ** -0.5, torch.randn(d, generator=g)
    w2, b2 = torch.randn(d, d, generator=g) * d ** -0.5, torch.randn(d, generator=g)
    m0 = torch.full((B, m_rows, n, d), float("nan"))

    def gates(**mut):
        h, m1 = _emu_angles(angles, w1, b1, w2, b2, m0, row0, strict, **mut)
        return _angle_gates(angles, w1, b1, w2, b2, m0, m1, h, row0, strict)
    assert all(gates().values()), gates()
    assert not gates(shift=-1)["layout"], "rows written one template early"
    assert not gates(shift=1)["layout"], "rows written one template late"
    assert not gates(with_b2=False)["stage2"], "dropped b2"
    assert not gates(with_b2=False)["module"], "dropped b2"
    if K % 8:
        assert not gates(pad=float("nan"))["stage1"], "K pad columns not zeroed"
    if strict:
        assert not gates(gelu="tanh")["stage2"], "tanh-GELU"


# ------------------------------------------------------------------------------------------------------------------------
# C. pair init
# ------------------------------------------------------------------------------------------------------------------------
def _emu_pair_init(e, w_pair, b_pair, pos, R, si, flip=False, clamp=None):
    n, d = e.shape[1], e.shape[-1]
    lr = e @ w_pair.T + b_pair
    idx = torch.arange(n) if si is None else si
    rel = idx[:, None] - idx[None, :]
    c = R if clamp is None else clamp
    rel = (-rel if flip else rel).clamp(-c, c) + R
    return (lr[:, :, None, :d] + lr[:, None, :, d:]) + pos[rel][None]


@pytest.mark.parametrize("d,n,R,with_index", [(4, 9, 1, True), (36, 33, 1, False), (100, 70, 32, True), (256, 70, 32, False)])
def test_pair_init_bound(d, n, R, with_index):
    g = _gen(d + n)
    B, V = 2, 22
    emb = torch.randn(V, d, generator=g)
    w_pair, b_pair = torch.randn(2 * d, d, generator=g) * d ** -0.5, torch.randn(2 * d, generator=g)
    pos = torch.randn(2 * R + 1, d, generator=g)
    seq = torch.randint(0, V, (B, n), generator=g)
    msa = torch.randint(0, V, (B, 3, n), generator=g)
    se = torch.randn(B, n, d, generator=g)
    si = torch.randint(-4 * R - 5, 4 * R + 6, (n,), generator=g) if with_index else None
    e, m = E.token_embed(emb, seq, msa, se)
    assert torch.equal(m, (emb[msa] + (emb[seq] + se)[:, None])), "token_embed is not the kernels' order"
    ref, bound = E.pair_init_ref(e, w_pair, b_pair, pos, R, si)
    assert E.within(_emu_pair_init(e, w_pair, b_pair, pos, R, si), ref, bound)
    assert not E.within(_emu_pair_init(e, w_pair, b_pair, pos, R, si, flip=True), ref, bound), "j - i"
    assert not E.within(_emu_pair_init(e, w_pair, b_pair, pos, R, si, clamp=R - 1), ref, bound), "clamp at R - 1"


# ------------------------------------------------------------------------------------------------------------------------
# D. distogram head
# ------------------------------------------------------------------------------------------------------------------------
def _emu_distogram(x, gamma, beta, w, bias, sym=True, unbiased=False, eps=E.EPS):
    v = (x + x.transpose(1, 2)) * 0.5 if sym else x
    mean = v.mean(-1, keepdim=True)
    var = v.var(-1, unbiased=unbiased, keepdim=True)
    y = (v - mean) * torch.rsqrt(var + eps) * gamma + beta
    return y @ w.T + bias


@pytest.mark.parametrize("d", [128, 256, 384, 512])
def test_distogram_bound(d):
    g = _gen(d)
    x, gamma, beta, w, bias = E.distogram_inputs(2, 9, d, 37, g, "cpu")
    ref, bound = E.distogram_ref(x, gamma, beta, w, bias)
    assert E.within(_emu_distogram(x, gamma, beta, w, bias), ref, bound)
    assert not E.within(_emu_distogram(x, gamma, beta, w, bias, sym=False), ref, bound), "no symmetrisation"
    assert not E.within(_emu_distogram(x, gamma, beta, w, bias, unbiased=True), ref, bound), "unbiased variance"
    assert not E.within(_emu_distogram(x, gamma, beta, w, bias, eps=1e-6), ref, bound), "eps 1e-6"
