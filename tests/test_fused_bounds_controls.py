"""CPU controls of the bounds in fused_bounds.py: each fused kernel of test_gpu_fused_kernels.py is emulated on the CPU at
its rounding points (bf16 operands by .bfloat16(), fp32 accumulation by float32 matmul, the bf16 stores of h, the gate, the
tail, q / k / v and P), the faithful emulation must pass every gate, and each plausible wrong variant must fail the gate
named beside it:

  A  feed-forward      last 64-unit hidden chunk skipped                     ff bound
                       value and gate halves swapped                          ff bound
                       chunk c with the b1 of chunk c + 1 (256-row tile)      ff bound
                       b2 dropped                                             ff bound
                       residual not added                                     ff bound
  B  contraction tail  one-pass variance E[x^2] - mean^2 (channel mean 1e3)   tail bound (load, project)
                       b_ogate dropped                                        tail bound (project)
                       the gate / scale of token t + 1                        tail bound (load, scale)
                       LayerNorm statistics over one warpgroup's D/2 channels tail bound (load, project)
                       scale_const where a per-token scale is given           tail bound (scale)
  C  attention_proj    key codes of the previous folded row                   attention bound
                       K / V of the previous head                             attention bound
                       gate bias of head 0 for every head                     attention bound
                       last 64-channel chunk of d dropped (d = 96, 160)       attention bound
                       pad keys (>= n) left in the softmax (n % 128 != 0)     attention bound
                       fully masked query rows not uniform (zero instead)     attention bound

Every mutant here is visible to an output bound.  The GPU test adds what an output bound cannot see: writes outside the
output (NaN guards around it), and results that depend on the grid or the launch (bitwise against the unfused sequence and
against a second launch).
"""
import pytest
import torch

import fused_bounds as FB


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bfr(x):
    return x.bfloat16().float()


def _mm32(a, w):
    return a.float() @ w.float().T


# ------------------------------------------------------------------------------------------------------------------------
# A. feed-forward
# ------------------------------------------------------------------------------------------------------------------------
def _ff_inputs(D, hidden, T, g):
    x = torch.randn(T, D, generator=g)
    xn = torch.randn(T, D, generator=g).bfloat16()
    w1 = (torch.randn(2 * hidden, D, generator=g) * D ** -0.5).bfloat16()   # packed order: [128 value | 128 gate] per tile
    b1 = torch.randn(2 * hidden, generator=g) * 0.5
    w2 = (torch.randn(D, hidden, generator=g) * hidden ** -0.5).bfloat16()
    b2 = torch.randn(D, generator=g)
    return x, xn, w1, b1, w2, b2


def _emu_ff(x, xn, w1, b1, w2, b2, mutant=None):
    wu, wg, bu, bg = FB.unpack_w1(w1, b1)
    bu, bg = bu.clone(), bg.clone()
    if mutant == "swap":
        wu, wg, bu, bg = wg, wu, bg, bu
    if mutant == "b1_next_chunk":          # chunks 2t and 2t + 1 share a 256-row packed tile: chunk 2t takes 2t + 1's bias
        for c in range(0, bu.numel() // 64, 2):
            bu[64 * c:64 * c + 64] = bu[64 * c + 64:64 * c + 128]
            bg[64 * c:64 * c + 64] = bg[64 * c + 64:64 * c + 128]
    h = (_mm32(xn, wu) + bu) * torch.nn.functional.gelu(_mm32(xn, wg) + bg)
    h = _bfr(h)
    if mutant == "skip_last_chunk":
        h[:, -64:] = 0
    y = _mm32(h, w2)
    if mutant != "no_b2":
        y = y + b2
    return y if mutant == "no_resid" else x + y


@pytest.mark.parametrize("D,hidden", [(128, 128), (128, 384), (256, 512)])
def test_ff_bound(D, hidden):
    x, xn, w1, b1, w2, b2 = _ff_inputs(D, hidden, 70, _gen(D + hidden))
    ref, bound = FB.ff_ref(x, xn, w1, b1, w2, b2)
    assert FB.within(_emu_ff(x, xn, w1, b1, w2, b2), ref, bound)
    for mutant in ("skip_last_chunk", "swap", "b1_next_chunk", "no_b2", "no_resid"):
        assert not FB.within(_emu_ff(x, xn, w1, b1, w2, b2, mutant), ref, bound), mutant


# ------------------------------------------------------------------------------------------------------------------------
# B. contraction tail
# ------------------------------------------------------------------------------------------------------------------------
def _tail_inputs(D, T, g):
    w = lambda *s: (torch.randn(*s, generator=g) * D ** -0.5).bfloat16()   # noqa: E731
    return dict(O=torch.randn(T, D, generator=g) + 1e3, x=torch.randn(T, D, generator=g), w_out=w(D, D),
                b_out=torch.randn(D, generator=g), gamma=1 + 0.5 * torch.randn(D, generator=g),
                beta=torch.randn(D, generator=g), gate=torch.rand(T, D, generator=g).bfloat16(),
                xn=torch.randn(T, D, generator=g).bfloat16(), w_og=w(D, D), b_og=torch.randn(D, generator=g),
                scale=torch.rand(T, generator=g) + 0.5, scale_const=0.125)


def _emu_tail(c, kind, mutant=None):
    O, D = c["O"], c["O"].shape[1]
    if kind == "scale":
        s = c["scale"] if mutant != "scale_const" else torch.full_like(c["scale"], c["scale_const"])
        if mutant == "next_token":
            s = s.roll(-1)
        t = _bfr(O * s[:, None])
    else:
        if kind == "project":
            z = _mm32(c["xn"], c["w_og"]) + (0 if mutant == "no_b_og" else c["b_og"])
            gate = _bfr(torch.sigmoid(z))
        else:
            gate = c["gate"].float()
        if mutant == "next_token":
            gate = gate.roll(-1, 0)
        st = O[:, :D // 2] if mutant == "half_stats" else O
        mean = st.mean(1, keepdim=True)
        if mutant == "one_pass":
            var = (st * st).mean(1, keepdim=True) - mean * mean
        else:
            var = ((st - mean) ** 2).mean(1, keepdim=True)
        t = _bfr(((O - mean) * torch.rsqrt(var + FB.EPS) * c["gamma"] + c["beta"]) * gate)
    return c["x"] + (_mm32(t, c["w_out"]) + c["b_out"])


def _tail_ref(c, kind):
    kw = dict(scale=c["scale"]) if kind == "scale" else dict(gamma=c["gamma"], beta=c["beta"])
    if kind == "load":
        kw.update(gate=c["gate"])
    elif kind == "project":
        kw.update(xn=c["xn"], w_og=c["w_og"], b_og=c["b_og"])
    return FB.tail_ref(c["O"], c["x"], c["w_out"], c["b_out"], **kw)


TAIL_MUTANTS = {"scale": ["next_token", "scale_const"], "load": ["one_pass", "next_token", "half_stats"],
                "project": ["one_pass", "no_b_og", "half_stats"]}


@pytest.mark.parametrize("kind", list(TAIL_MUTANTS))
@pytest.mark.parametrize("D", [128, 256])
def test_tail_bound(D, kind):
    c = _tail_inputs(D, 70, _gen(D + len(kind)))
    ref, bound = _tail_ref(c, kind)
    assert FB.within(_emu_tail(c, kind), ref, bound)
    for mutant in TAIL_MUTANTS[kind]:
        assert not FB.within(_emu_tail(c, kind, mutant), ref, bound), mutant


def test_tail_scale_const_bound():
    """scale_const alone (no per-token scale): the reference takes fl(scale_const)"""
    c = _tail_inputs(128, 70, _gen(5))
    c["scale"] = torch.full((70,), c["scale_const"])
    ref, bound = FB.tail_ref(c["O"], c["x"], c["w_out"], c["b_out"], scale_const=c["scale_const"])
    assert FB.within(_emu_tail(c, "scale"), ref, bound)


# ------------------------------------------------------------------------------------------------------------------------
# C. projected attention
# ------------------------------------------------------------------------------------------------------------------------
def _attn_inputs(n, nbatch, heads, dh, d, bias, g):
    I = heads * dh
    xn = torch.randn(n * nbatch, d, generator=g).bfloat16()
    scale = dh ** -0.5 * 1.4426950408889634
    wqkv = torch.randn(3 * I, d, generator=g) * d ** -0.5
    wqkv[:I] *= scale * 4.0                                # logits of a few units: the softmax is far from uniform
    wqkv = wqkv.bfloat16()
    wg = (torch.randn(I, d, generator=g) * d ** -0.5).bfloat16()
    bg = torch.randn(I, generator=g)
    bt = None
    if bias:
        bt = torch.full((heads, n, (n + 7) // 8 * 8), float("nan"))
        bt[:, :, :n] = torch.randn(heads, n, n, generator=g) * 2.0
        bt = bt.bfloat16()
    m = torch.rand(nbatch, n, generator=g) >= 0.3          # different holes in every folded row
    m[1::3] = False                                        # fully masked rows
    m[2::3, : n // 2] = True
    idx = torch.arange(nbatch)[:, None] * n + torch.arange(n)[None, :]
    return xn, wqkv, wg, bg, bt, m, idx


def _emu_attn(xn, wqkv, wg, bg, bias, m, n, nbatch, heads, dh, mutant=None):
    """the kernel's arithmetic, row attention (folded row b = tokens b n .. b n + n - 1)"""
    I = heads * dh
    a = xn.float()
    if mutant == "drop_chunk":
        a = a.clone()
        a[:, (a.shape[1] - 1) // 64 * 64:] = 0
    bgm = bg[:dh].repeat(heads) if mutant == "gate_bias_head0" else bg
    qkv = _bfr(_mm32(a, wqkv)).view(nbatch, n, 3, heads, dh).permute(2, 0, 3, 1, 4)   # [3, nb, H, n, dh]
    gate = _bfr(torch.sigmoid(_mm32(a, wg) + bgm)).view(nbatch, n, heads, dh).permute(0, 2, 1, 3)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if mutant == "prev_head_kv":
        k, v = k.roll(1, 1), v.roll(1, 1)
        k[:, 0], v[:, 0] = qkv[1][:, 0], qkv[2][:, 0]
    mk = m.clone()
    if mutant == "stale_codes":
        mk[1:] = m[:-1]
    s = q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias[:, :, :n].float()[None]
    valid = m[:, None, :, None] & mk[:, None, None, :]
    s = s.masked_fill(~valid, float("-inf"))
    if mutant == "pad_keys":                               # kpad - n zero keys with logit 0 join every query's softmax
        npad = (n + 127) // 128 * 128 - n
        s = torch.cat([s, torch.zeros(*s.shape[:-1], npad)], -1)
        v = torch.cat([v, torch.zeros(*v.shape[:-2], npad, dh)], -2)
    any_valid = valid.any(-1, keepdim=True)
    if mutant != "masked_zero":                            # quirk Q1: no valid key -> uniform over the n keys
        s = torch.where(any_valid, s, torch.zeros_like(s))
    mx = s.amax(-1, keepdim=True)
    e = torch.exp2(s - torch.where(torch.isfinite(mx), mx, torch.zeros_like(mx)))
    o = (_bfr(e) @ v) / e.sum(-1, keepdim=True)
    if mutant == "masked_zero":
        o = torch.where(any_valid, o, torch.zeros_like(o))
    out = _bfr(o * gate)
    return out.permute(0, 2, 1, 3).reshape(nbatch * n, I)


@pytest.mark.parametrize("n,heads,dh,d,bias", [(130, 3, 32, 96, True), (70, 2, 64, 160, False), (129, 3, 64, 64, True)])
def test_attention_bound(n, heads, dh, d, bias):
    nbatch = 6
    xn, wqkv, wg, bg, bt, m, idx = _attn_inputs(n, nbatch, heads, dh, d, bias, _gen(n + d))
    ref, bound = FB.attention_proj_ref(xn, wqkv, wg, bg, bt, m, n, nbatch, heads, dh, idx)
    emu = lambda mut=None: _emu_attn(xn, wqkv, wg, bg, bt, m, n, nbatch, heads, dh, mut)   # noqa: E731
    assert FB.within(emu(), ref, bound)
    mutants = ["stale_codes", "prev_head_kv", "gate_bias_head0", "masked_zero"]
    if d % 64:
        mutants.append("drop_chunk")
    if bt is None:                                         # a bias pad column is NaN: a pad key would be NaN outright
        mutants.append("pad_keys")
    for mutant in mutants:
        assert not FB.within(emu(mutant), ref, bound), mutant
