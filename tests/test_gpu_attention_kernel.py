"""-m gpu: the attention kernel alone (af2_attention_bf16 -> attention_tc.cuh), element-wise against fp64.

Reference.  The reference module's semantics, evaluated in fp64 on the GPU from the exact bf16 operands the kernel was
given: s = q k^T + bias (log2 domain), s.masked_fill(~(mask_q & mask_k), -max), p = softmax over all n keys (base 2),
out = (p v) * gate.  It does not follow the kernel's key codes: a fully masked query averages all n values, pad keys of the
last 128-key block do not exist.

Bound (per element).  The kernel computes the logits in fp32 from bf16 q / k (error ~dh 2^-24 sum|q k|, below 2^-12 in
probability at the +-200 log2 logits used here), rounds every probability p_j to bf16 for the PV product (unit roundoff
2^-8) but normalises by the fp32 sum of the unrounded ones, accumulates in fp32 and rounds the gated output to bf16 (2^-8):
    |out - ref| <= 2^-8 |ref| + C_ATTN * 2^-8 |g| sum_j p_j |v_j|
The second term is the bf16 rounding of P against the fp32 normaliser.  C_ATTN = 1 holds on an H100 80GB HBM3 (700 W power limit); the
worst err / bound of every case is written to the parity report (0.92 when this was written; the 2^-8 |ref| term alone
reaches ~0.5-1 wherever an output rounds by nearly half a bf16 ulp, so ratios close to 1 are expected).

Bias pad columns (j >= n of each align8(n) row) hold NaN here: they must never reach an output.
"""
import math

import pytest
import torch

from gpu_util import check_bound

pytestmark = pytest.mark.gpu

C_ATTN = 1.0
NEG = -torch.finfo(torch.float64).max


def _ops():
    from alphafold2_b200 import ops
    return ops


def _tok(nbatch, n, row):
    """token index of (b, i) and the strides: row attention folds contiguous rows, column attention strided columns"""
    tok_sb, tok_si = (n, 1) if row else (1, nbatch)
    b = torch.arange(nbatch, device="cuda")[:, None]
    i = torch.arange(n, device="cuda")[None, :]
    return b * tok_sb + i * tok_si, tok_sb, tok_si


def _mask(kind, nbatch, n, g):
    if kind == "none":
        return None
    m = torch.ones(nbatch, n, dtype=torch.bool)
    if kind == "suffix":
        m[:, n - max(1, n // 8):] = False
    elif kind == "holes":
        m = torch.rand(nbatch, n, generator=g) >= 0.3
    elif kind == "first_block":          # every key of block 0 masked, valid queries beyond it
        m[:, :128] = False
        m[:, 128:] = torch.rand(nbatch, n - 128, generator=g) >= 0.2
        m[:, -1] = True
    elif kind == "straddle":             # masked keys on both sides of key 128
        m[:, 121:136] = False
        m[:, 100:121] = torch.rand(nbatch, 21, generator=g) >= 0.5
    elif kind == "single":               # one valid key per folded row, in a different block per row
        m[:] = False
        pos = torch.randint(0, n, (nbatch,), generator=g)
        pos[0] = n - 1
        m[torch.arange(nbatch), pos] = True
    elif kind == "all_masked":           # even rows fully masked (uniform mean of all n values), odd rows with holes
        m = torch.rand(nbatch, n, generator=g) >= 0.3
        m[0::2] = False
    else:
        raise ValueError(kind)
    return m


def make_inputs(n, nbatch, heads, dh, bias, big, seed):
    g = torch.Generator().manual_seed(seed)
    I = heads * dh
    T = n * nbatch
    qkv = torch.randn(T, 3 * I, generator=g)
    if big:                              # logits spanning about +-200 in the log2 domain: exercises the max subtraction
        qkv[:, :I] *= 200.0 / (3.0 * math.sqrt(dh))
    qkv = qkv.to("cuda", torch.bfloat16)
    gate = torch.rand(T, I, generator=g).to("cuda", torch.bfloat16)
    bt = None
    if bias:
        npad = (n + 7) // 8 * 8
        bt = torch.full((heads, n, npad), float("nan"))
        bt[:, :, :n] = torch.randn(heads, n, n, generator=g) * (60.0 if big else 2.0)
        bt = bt.to("cuda", torch.bfloat16)
    return qkv, gate, bt, g


def attention_ref(qkv, gate, bias, mask_bn, n, nbatch, heads, dh, idx):
    """fp64 reference (module semantics) -> out [tokens, I] and the bound, both fp64 on the GPU"""
    I = heads * dh
    T = qkv.shape[0]
    out = torch.empty(T, I, dtype=torch.float64, device="cuda")
    bnd = torch.empty(T, I, dtype=torch.float64, device="cuda")
    chunk = max(1, (1 << 25) // (heads * n * n))            # folded rows per step: bounded fp64 temporaries
    for b0 in range(0, nbatch, chunk):
        ix = idx[b0:b0 + chunk]                               # [nb, n]
        nb = ix.shape[0]
        x = qkv[ix].double().view(nb, n, 3, heads, dh).permute(2, 0, 3, 1, 4)   # [3, nb, H, n, dh]
        q, k, v = x[0], x[1], x[2]
        s = q @ k.transpose(-1, -2)
        if bias is not None:
            s = s + bias[:, :, :n].double()[None]
        if mask_bn is not None:
            m = mask_bn[b0:b0 + nb].cuda()
            pair = m[:, None, :, None] & m[:, None, None, :]
            s = s.masked_fill(~pair, NEG)
        p = torch.softmax(s * math.log(2.0), dim=-1)
        o = (p @ v).permute(0, 2, 1, 3).reshape(nb, n, I)       # [nb, n, H*dh]
        pv = (p @ v.abs()).permute(0, 2, 1, 3).reshape(nb, n, I)
        gt = gate[ix].double()
        r = o * gt
        out[ix.flatten()] = r.reshape(-1, I)
        bnd[ix.flatten()] = (2.0 ** -8 * r.abs() + C_ATTN * 2.0 ** -8 * gt.abs() * pv).reshape(-1, I)
    return out, bnd


def run_case(name, n, nbatch, heads, dh, row, bias, mask_kind, big=False, seed=0):
    ops = _ops()
    qkv, gate, bt, g = make_inputs(n, nbatch, heads, dh, bias, big, seed)
    idx, tok_sb, tok_si = _tok(nbatch, n, row)
    m_bn = _mask(mask_kind, nbatch, n, g)
    mask_tok = None
    if m_bn is not None:
        mask_tok = torch.empty(n * nbatch, dtype=torch.bool, device="cuda")
        mask_tok[idx.flatten()] = m_bn.cuda().flatten()
    out = ops.attention_bf16(qkv, gate, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask_tok)
    ref, bnd = attention_ref(qkv, gate, bt, m_bn, n, nbatch, heads, dh, idx)
    check_bound(name, out, ref, bnd)
    return qkv, gate, bt, mask_tok, out


N_ALL = [1, 2, 7, 8, 127, 128, 129, 255, 256, 257, 384, 1000]
_BH = [(1, 1), (3, 3), (37, 8), (3, 1), (1, 8), (37, 3)]       # (nbatch, heads), cycled over the lengths


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("n", N_ALL)
def test_attention_lengths(n, bias, row, dh):
    """every 128-key block boundary, the odd-n bias pad column, folded batch 1 / 3 / 37 and 1 / 3 / 8 heads"""
    nbatch, heads = _BH[(N_ALL.index(n) + 2 * bias + row) % len(_BH)]
    if n >= 384:
        nbatch = min(nbatch, 3)
    mask = ["none", "holes", "suffix"][(N_ALL.index(n) + row) % 3]
    run_case(f"attn_len n{n} b{nbatch} h{heads} dh{dh} {'row' if row else 'col'} bias{int(bias)} {mask}",
             n, nbatch, heads, dh, row, bias, mask, seed=n * 7 + dh + bias)


MASK_KINDS = ["none", "suffix", "holes", "first_block", "straddle", "single", "all_masked"]


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("mask", MASK_KINDS)
@pytest.mark.parametrize("n,nbatch,heads,row", [(257, 3, 3, True), (384, 5, 8, False), (200, 37, 1, False)])
def test_attention_masks(n, nbatch, heads, row, mask, dh):
    run_case(f"attn_mask {mask} n{n} b{nbatch} h{heads} dh{dh} {'row' if row else 'col'}", n, nbatch, heads, dh, row,
             True, mask, seed=11 * n + dh)


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("mask", ["none", "holes", "first_block", "all_masked"])
@pytest.mark.parametrize("n", [129, 300])
def test_attention_large_logits(n, mask, dh):
    """bias and q scaled so that the logits span about +-200 (log2 domain)"""
    run_case(f"attn_big {mask} n{n} dh{dh}", n, 3, 3, dh, True, True, mask, big=True, seed=5 * n + dh)


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
def test_attention_slice_and_repeat_bitwise(row, dh):
    """CTAs are independent: one folded row computed alone has the bits it has inside an nbatch = 37 launch, and two identical
    launches give identical bits"""
    ops = _ops()
    n, nbatch, heads = 257, 37, 3
    qkv, gate, bt, mask, out = run_case(f"attn_slice n{n} b{nbatch} dh{dh} {'row' if row else 'col'}", n, nbatch, heads, dh,
                                        row, True, "holes", seed=3 + dh)
    idx, tok_sb, tok_si = _tok(nbatch, n, row)
    again = ops.attention_bf16(qkv, gate, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask)
    assert torch.equal(again.view(torch.int16), out.view(torch.int16))
    for b in (0, 17, 36):
        ix = idx[b]
        one = ops.attention_bf16(qkv[ix].contiguous(), gate[ix].contiguous(), n, 1, heads, dh, n, 1, bias=bt,
                                 mask=mask[ix].contiguous())
        assert torch.equal(one.view(torch.int16), out[ix].view(torch.int16)), f"folded row {b} differs when run alone"
