"""-m gpu: Attention.forward (af2_attention_forward{,_strict}) kernel by kernel, element-wise against fp64: (A) the general
form of the attention kernel, attention_tc_kernel<DH, true>, (B) the bias copy attn_bias_log2_kernel and (C) the strict
kernels of attention_fwd.cuh, each through the C entry point that shares its launcher with the module (include/af2b200.h),
so grids and arguments are the module's; then (D) the module shapes test_gpu_attention_forward.py does not reach.

Kernel-level outputs start as NaN with a guard region after them: guards must stay NaN, and two identical launches must give
the same bits.  u = 2^-24.

A. attention_tc_kernel<DH, true>.  The fp64 reference of test_gpu_attention_kernel.py with a query length i and a key length
  j, from the exact bf16 q, k, v, gate and fp32 log2-domain bias the kernel received: s = q k^T + bias, logits where
  !(qmask[q] & kmask[k]) replaced by -max (a null mask counts as all valid, so a masked query averages all j values), p =
  softmax over the j keys in base 2, out = (p v) * gate.  Its per-element bound and C_ATTN are used unchanged:
      |out - ref| <= 2^-8 |ref| + C_ATTN 2^-8 |g| sum_k p_k |v_k|
  The fp32 bias adds one rounding of the logit sum, u relative to logits of at most a few hundred: far below the 2^-8 terms.
  Bias pad columns [j, align8(j)) hold NaN: they must never reach an output.
B. attn_bias_log2_kernel: bitwise fp32(bias) * fp32(log2 e) for every layout the module passes, pad columns exactly 0.
C. Strict kernels, with the bounds derived in test_gpu_strict_kernels.py: xqkv is a re-layout (exact, pads 0), xsoftmax
  meets the softmax bound of `_softmax_ref` (masked keys exactly 0, rows without a valid key exactly 1/j), xgate 5 u |ref|.
  Every case runs the chunk b0 > 0, nb < B that the module's chunk loop hands them.
"""
import math

import pytest
import torch

from gpu_util import check_bound, check_strict, to64
from oracle import attention_oracle as AO
from test_gpu_attention_forward import _inputs, _module, _run
from test_gpu_attention_kernel import C_ATTN, NEG, _mask
from test_gpu_strict_kernels import BF, GUARD, SPL, U, _al, _bits, _call, _nan, _p, _softmax_ref, _split_out, _twice

pytestmark = pytest.mark.gpu

NAN = float("nan")
DHS = [16, 32, 64, 128]


def _lib():
    from alphafold2_b200 import _lib as L
    return L.load()


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ------------------------------------------------------------------------------------------------------------------------
# A. attention_tc_kernel<DH, true>
# ------------------------------------------------------------------------------------------------------------------------
def _query_mask(B, i, g):
    """holes (masked queries average all j values), query 0 of batch element 0 valid, and with B > 1 the last batch element
    without any valid query"""
    m = torch.rand(B, i, generator=g) >= 0.3
    m[0, 0] = True
    if B > 1:
        m[B - 1] = False
    return m


def _key_mask(pattern, B, j, g):
    if pattern == "batch_keys":              # every key of batch element 0 masked, under its valid queries
        m = torch.rand(B, j, generator=g) >= 0.3
        m[0] = False
        return m
    return _mask(pattern, B, j, g)           # holes, first_block, straddle, single


def _x_masks(combo, pattern, B, i, j, g):
    """(qmask, kmask) bool on the GPU or None, as the module passes them: none; q (cross-attention without context_mask);
    qk (both); self (i == j, one buffer for both, holding the key pattern)"""
    if combo == "none":
        return None, None
    if combo == "self":
        assert i == j
        m = _key_mask(pattern, B, j, g).cuda()
        return m, m
    qm = _query_mask(B, i, g).cuda()
    return qm, (_key_mask(pattern, B, j, g).cuda() if combo == "qk" else None)


def _x_bias(kind, B, heads, i, j, g, scale):
    """fp32 log2-domain bias [Bb][heads][i][align8(j)] with NaN pad columns and its batch stride: none, batch (a slab per
    batch element) or shared (one slab, bias_sb = 0)"""
    if kind == "none":
        return None, 0
    Bb, npad = (B if kind == "batch" else 1), _al(j, 8)
    b = torch.full((Bb, heads, i, npad), NAN)
    b[..., :j] = torch.randn(Bb, heads, i, j, generator=g) * scale
    return b.cuda(), (heads * i * npad if kind == "batch" else 0)


def _x_inputs(B, i, j, heads, dh, g, big):
    """q pre-scaled like the module's to_q (logits of about +-3 in the log2 domain, or +-200 with big), gate in (0, 1)"""
    I = heads * dh
    q = torch.randn(B * i, I, generator=g) * ((200.0 / 3.0 if big else 1.0) / math.sqrt(dh))
    kv = torch.randn(B * j, 2 * I, generator=g)
    gate = torch.rand(B * i, I, generator=g)
    return q.to("cuda", BF), gate.to("cuda", BF), kv.to("cuda", BF)


def _x_launch(q, gate, kv, bias, bias_sb, qm, km, B, i, j, heads, dh):
    out = _nan(B * i * heads * dh, BF)
    _call("af2_attention_x_bf16", q.data_ptr(), gate.data_ptr(), kv.data_ptr(), _p(bias), bias_sb, _p(qm), _p(km), B, i, j, heads, dh,
          out.data_ptr())
    return out


def x_ref(q, gate, kv, bias, bias_sb, qm, km, B, i, j, heads, dh):
    """fp64 reference and bound (module docstring, A) -> ([B i, I], [B i, I])"""
    I = heads * dh
    out = torch.empty(B, i, I, dtype=torch.float64, device="cuda")
    bnd = torch.empty_like(out)
    chunk = max(1, (1 << 25) // (heads * i * j))
    for b0 in range(0, B, chunk):
        nb = min(chunk, B - b0)
        qq = q.view(B, i, heads, dh)[b0:b0 + nb].double().permute(0, 2, 1, 3)
        kk = kv.view(B, j, 2, heads, dh)[b0:b0 + nb].double()
        k, v = kk[:, :, 0].permute(0, 2, 1, 3), kk[:, :, 1].permute(0, 2, 1, 3)
        s = qq @ k.transpose(-1, -2)
        if bias is not None:
            s = s + (bias[b0:b0 + nb] if bias_sb else bias[:1])[..., :j].double()
        if qm is not None or km is not None:
            vq = qm[b0:b0 + nb] if qm is not None else torch.ones(nb, i, dtype=torch.bool, device="cuda")
            vk = km[b0:b0 + nb] if km is not None else torch.ones(nb, j, dtype=torch.bool, device="cuda")
            s = s.masked_fill(~(vq[:, None, :, None] & vk[:, None, None, :]), NEG)
        p = torch.softmax(s * math.log(2.0), dim=-1)
        o = (p @ v).permute(0, 2, 1, 3).reshape(nb, i, I)
        pv = (p @ v.abs()).permute(0, 2, 1, 3).reshape(nb, i, I)
        gt = gate.view(B, i, I)[b0:b0 + nb].double()
        out[b0:b0 + nb] = o * gt
        bnd[b0:b0 + nb] = 2.0 ** -8 * (o * gt).abs() + C_ATTN * 2.0 ** -8 * gt.abs() * pv
    return out.view(B * i, I), bnd.view(B * i, I)


def run_x(name, B, i, j, heads, dh, bias="none", combo="none", pattern="holes", big=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    q, gate, kv = _x_inputs(B, i, j, heads, dh, g, big)
    bt, bsb = _x_bias(bias, B, heads, i, j, g, 60.0 if big else 2.0)
    qm, km = _x_masks(combo, pattern, B, i, j, g)
    # some valid query must see a valid key: otherwise every output is gate * mean(v), which q, k and the bias never reach
    live = (qm if qm is not None else torch.ones(B, i, dtype=torch.bool, device="cuda")) & \
        (km.any(-1, keepdim=True) if km is not None else torch.ones(B, 1, dtype=torch.bool, device="cuda"))
    assert bool(live.any()), f"{name}: no valid query attends to a valid key"
    args = (q, gate, kv, bt, bsb, qm, km, B, i, j, heads, dh)
    out = _twice(lambda: _x_launch(*args))[: B * i * heads * dh].view(B * i, heads * dh)
    ref, bnd = x_ref(*args)
    check_bound(name, out, ref, bnd)
    return args, out


I_LEN = [1, 7, 127, 128, 129, 257, 384]
J_LEN = [1, 8, 127, 128, 129, 255, 256, 257, 1000]


@pytest.mark.parametrize("dh", DHS)
@pytest.mark.parametrize("j", J_LEN)
def test_x_lengths(j, dh):
    """the query lengths cycled against every key length (each 128-key block boundary, the odd bias pad), 1 / 3 / 8 heads"""
    jx, dx = J_LEN.index(j), DHS.index(dh)
    i = I_LEN[(jx + 3 * dx) % len(I_LEN)]
    heads = [1, 3, 8][(jx + dx) % 3]
    B = [2, 3, 1][(jx // 3 + dx) % 3]                               # every mask combination meets B = 1, 2 and 3 per dh
    bias = ["batch", "shared", "none"][(jx + 2 * dx) % 3]
    combo = ["none", "q", "qk"][jx % 3]
    run_x(f"attn_x_len i{i} j{j} dh{dh} h{heads} B{B} {bias} {combo}", B, i, j, heads, dh, bias, combo, "holes", seed=jx * 11 + dh)


KEY_PATTERNS = ["holes", "batch_keys", "first_block", "straddle", "single"]


@pytest.mark.parametrize("combo", ["qk", "self"])
@pytest.mark.parametrize("pattern", KEY_PATTERNS)
def test_x_masks(pattern, combo):
    """masked queries, masked batch elements and the key patterns of test_gpu_attention_kernel.py, per batch element"""
    dh = DHS[(KEY_PATTERNS.index(pattern) + (combo == "self")) % 4]
    i, j = (300, 300) if combo == "self" else (257, 300)
    run_x(f"attn_x_mask {pattern} {combo} dh{dh}", 3, i, j, 3, dh, "batch", combo, pattern, seed=7 * dh + len(pattern))


@pytest.mark.parametrize("big", [False, True], ids=["normal", "big"])
@pytest.mark.parametrize("bias", ["none", "batch", "shared"])
def test_x_bias(bias, big):
    """no bias, a slab per batch element, one shared slab with B > 1; big: logits of about +-200 (log2 domain)"""
    dh = DHS[(["none", "batch", "shared"].index(bias) + 2 * big) % 4]
    run_x(f"attn_x_bias {bias} {'big' if big else 'normal'} dh{dh}", 3, 129, 257, 3, dh, bias, "qk", "holes", big=big,
          seed=3 * dh + big)


@pytest.mark.parametrize("dh", DHS)
@pytest.mark.parametrize("count", ["1", "S-1", "S", "S+1", "3S"])
def test_x_work_items(count, dh):
    """item counts around the SM count S: from S + 1 items on, CTAs run a second item (other slot, flipped barrier phases,
    rewritten key codes) of another batch element, with its own bias slab and query-mask row"""
    S = _sms()
    heads, i = (1, 257) if count == "3S" else (1, 100)
    B = {"1": 1, "S-1": S - 1, "S": S, "S+1": S + 1, "3S": S}[count]
    items = (i + 127) // 128 * heads * B
    assert items == {"1": 1, "S-1": S - 1, "S": S, "S+1": S + 1, "3S": 3 * S}[count]
    run_x(f"attn_x_items {count} ({items}) dh{dh}", B, i, 200, heads, dh, "batch", "qk", "holes", seed=items + dh)


def _largest_j(dh):
    """the largest key length the workspace query accepts for the general kernel (i = 2, no bias)"""
    ws = _lib().af2_attention_forward_workspace
    lo, hi = 1, 1 << 20
    assert ws(2, 2, lo, 64, 1, dh, 0, 0) > 0 and ws(2, 2, hi, 64, 1, dh, 0, 0) < 0
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ws(2, 2, mid, 64, 1, dh, 0, 0) > 0 else (lo, mid)
    return lo


@pytest.mark.parametrize("dh", DHS)
def test_x_key_length_bound(dh):
    """the largest accepted key length runs correctly; one more is refused before anything launches, also for one query
    without a bias (the module's pointwise route, which this entry never takes)"""
    jmax = _largest_j(dh)
    run_x(f"attn_x_jmax j{jmax} dh{dh}", 2, 7, jmax, 2, dh, "batch", "qk", "straddle", seed=dh)
    lib = _lib()
    for i, bias in ((7, True), (1, False)):
        g = torch.Generator().manual_seed(1)
        q, gate, kv = _x_inputs(1, i, jmax + 1, 1, dh, g, False)
        bt, bsb = _x_bias("batch" if bias else "none", 1, 1, i, jmax + 1, g, 2.0)
        before = lib.af2_launch_count()
        with pytest.raises(ValueError, match="too long"):
            _x_launch(q, gate, kv, bt, bsb, None, None, 1, i, jmax + 1, 1, dh)
        assert lib.af2_launch_count() == before, "a refused call launched"


@pytest.mark.parametrize("dh", DHS)
def test_x_batch_independence(dh):
    """batch element b run alone, with its own slab and masks, has the bits of its rows inside a B = 37 launch"""
    B, i, j, heads = 37, 129, 257, 3
    args, out = run_x(f"attn_x_indep dh{dh}", B, i, j, heads, dh, "batch", "qk", "holes", seed=dh + 1)
    q, gate, kv, bt, bsb, qm, km = args[:7]
    for b in (0, 18, 36):
        rq, rk = slice(b * i, (b + 1) * i), slice(b * j, (b + 1) * j)
        one = _x_launch(q[rq].contiguous(), gate[rq].contiguous(), kv[rk].contiguous(), bt[b:b + 1].contiguous(), bsb,
                        qm[b:b + 1].contiguous(), km[b:b + 1].contiguous(), 1, i, j, heads, dh)
        assert torch.equal(_bits(one[: i * heads * dh]), _bits(out[rq].flatten())), f"batch element {b} differs when run alone"


# ------------------------------------------------------------------------------------------------------------------------
# B. attn_bias_log2_kernel
# ------------------------------------------------------------------------------------------------------------------------
BIAS_LAYOUTS = ["bhij", "1hij", "hij", "b1ij", "11ij", "ij", "b11j", "transposed", "expanded"]


def _bias_layout(kind, B, h, i, j, g, scale=1.0):
    """a bias tensor on the GPU in one of the layouts that broadcast to [B, h, i, j]"""
    if kind == "transposed":
        return (torch.randn(B, h, j, i, generator=g) * scale).cuda().transpose(-1, -2)
    if kind == "expanded":
        return (torch.randn(1, h, 1, j, generator=g) * scale).cuda().expand(B, h, i, j)
    shape = {"bhij": (B, h, i, j), "1hij": (1, h, i, j), "hij": (h, i, j), "b1ij": (B, 1, i, j), "11ij": (1, 1, i, j),
             "ij": (i, j), "b11j": (B, 1, 1, j)}[kind]
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _bias_strides(bias, B, h, i, j):
    """(Bb, (sb, sh, si, sj)) as ops.attention_forward passes them"""
    Bb = B if bias.dim() == 4 and bias.shape[0] == B and B > 1 else 1
    e = bias.expand(B, h, i, j)
    return Bb, (e.stride(0) if Bb > 1 else 0,) + tuple(e.stride()[1:])


@pytest.mark.parametrize("j", [1, 45, 48])
@pytest.mark.parametrize("layout", BIAS_LAYOUTS)
def test_bias_log2(layout, j):
    B, h, i = 3, 4, 37
    g = torch.Generator().manual_seed(len(layout) + j)
    bias = _bias_layout(layout, B, h, i, j, g, 30.0)
    Bb, st = _bias_strides(bias, B, h, i, j)
    npad = _al(j, 8)

    def run():
        out = _nan(Bb * h * i * npad)
        _call("af2_attn_bias_log2", bias.data_ptr(), *st, out.data_ptr(), Bb, h, i, j)
        return out
    out = _twice(run)[: Bb * h * i * npad].view(Bb, h, i, npad)
    exp = torch.zeros(Bb, h, i, npad, device="cuda")
    exp[..., :j] = bias.expand(B, h, i, j)[:Bb] * torch.tensor(1.4426950408889634, dtype=torch.float32, device="cuda")
    assert torch.equal(_bits(out), _bits(exp)), f"{layout}: log2-domain bias differs"


# ------------------------------------------------------------------------------------------------------------------------
# C. strict kernels, chunk b0 = 2, nb = 2 of B = 5
# ------------------------------------------------------------------------------------------------------------------------
H_S, B_S, B0, NB = 3, 5, 2, 2
IJ = [(7, 30), (30, 7)]


@pytest.mark.parametrize("dh", [12, 20])
@pytest.mark.parametrize("i,j", IJ)
def test_strict_xqkv_split(i, j, dh):
    g = torch.Generator(device="cuda").manual_seed(i + 3 * j + dh)
    I, Pd, Pn = H_S * dh, _al(dh, 8), _al(j, 8)
    qg = torch.randn(B_S * i, 2 * I, device="cuda", generator=g)
    kv = torch.randn(B_S * j, 2 * I, device="cuda", generator=g)
    sizes = [NB * H_S * i * SPL * Pd, NB * H_S * j * SPL * Pd, NB * H_S * dh * SPL * Pn]

    def run():
        q, k, vt = (_nan(n, BF) for n in sizes)
        _call("af2_strict_xqkv_split", qg.data_ptr(), kv.data_ptr(), q.data_ptr(), k.data_ptr(), vt.data_ptr(), B0, NB, H_S, i, j, dh)
        return torch.cat([q, k, vt])
    q, k, vt = torch.split(_twice(run), [n + GUARD for n in sizes])
    for t in (q, k, vt):
        assert torch.isnan(t[-GUARD:]).all(), "guard region written"
    qq = qg.view(B_S, i, 2, H_S, dh)[B0:B0 + NB, :, 0].double()
    kk = kv.view(B_S, j, 2, H_S, dh)[B0:B0 + NB].double()
    exp_q = qq.permute(0, 2, 1, 3).reshape(NB * H_S, i, dh)
    exp_k = kk[:, :, 0].permute(0, 2, 1, 3).reshape(NB * H_S, j, dh)
    exp_v = kk[:, :, 1].permute(0, 2, 3, 1).reshape(NB * H_S, dh, j)
    for name, buf, shape, cols, exp in (("q", q, (NB * H_S, i, Pd), dh, exp_q), ("k", k, (NB * H_S, j, Pd), dh, exp_k),
                                        ("vt", vt, (NB * H_S, dh, Pn), j, exp_v)):
        v = _split_out(f"strict/xqkv_split/{name}/i{i}j{j}dh{dh}", buf, shape, cols, exp, torch.zeros_like(exp))
        assert torch.equal(v, exp)


MASKINGS = ["none", "kmask_only", "q", "qk", "keys_all"]


def _strict_masks(masking, B, i, j, g):
    """(qmask [B, i], kmask [B, j]) on the GPU or None.  q: query holes, chunk element 0 without a valid query; keys_all:
    every query valid, every key of chunk element 1 masked"""
    qm = km = None
    if masking in ("q", "qk"):
        qm = torch.rand(B, i, generator=g) > 0.3
        qm[B0] = False
    if masking in ("kmask_only", "qk"):
        km = torch.rand(B, j, generator=g) > 0.3
    if masking == "keys_all":
        qm = torch.ones(B, i, dtype=torch.bool)
        km = torch.rand(B, j, generator=g) > 0.3
        km[B0 + 1] = False
    return (None if qm is None else qm.cuda()), (None if km is None else km.cuda())


@pytest.mark.parametrize("layout", ["none"] + BIAS_LAYOUTS)
@pytest.mark.parametrize("masking", MASKINGS)
@pytest.mark.parametrize("i,j", IJ)
def test_strict_xsoftmax_split(i, j, masking, layout):
    g = torch.Generator().manual_seed(i * 7 + j + len(masking) * 13 + len(layout))
    lds = _al(j, 4) + 4                                               # columns [j, lds) hold NaN
    S = torch.full((NB * H_S * i, lds), NAN)
    S[:, :j] = (torch.rand(NB * H_S * i, j, generator=g) * 2 - 1) * 80
    S = S.cuda()
    bias, st = None, (0, 0, 0, 0)
    if layout != "none":
        bias = _bias_layout(layout, B_S, H_S, i, j, g, 4.0)
        st = _bias_strides(bias, B_S, H_S, i, j)[1]
    qm, km = _strict_masks(masking, B_S, i, j, g)
    Pn = _al(j, 8)

    def run():
        P = _nan(NB * H_S * i * SPL * Pn, BF)
        _call("af2_strict_xsoftmax_split", S.data_ptr(), lds, _p(bias), *st, _p(qm), _p(km), P.data_ptr(), B0, NB, H_S, i, j)
        return P
    P = _twice(run)
    L = S[:, :j].double().view(NB, H_S, i, j)
    if bias is not None:
        L = L + bias.expand(B_S, H_S, i, j)[B0:B0 + NB].double()
    if qm is not None:                                               # the key mask counts only under a query mask
        kb = km[B0:B0 + NB] if km is not None else torch.ones(NB, j, dtype=torch.bool, device="cuda")
        valid = qm[B0:B0 + NB, :, None] & kb[:, None, :]
    else:
        valid = torch.ones(NB, i, j, dtype=torch.bool, device="cuda")
    ref, bound = _softmax_ref(L, None, valid)
    name = f"strict/xsoftmax_split/i{i}j{j}/{masking}/{layout}"
    v = _split_out(name, P, (NB * H_S * i, Pn), j, ref.reshape(-1, j), bound.reshape(-1, j)).view(NB, H_S, i, j)
    V = valid[:, None].expand_as(v)
    assert torch.all(v[~V & V.any(-1, keepdim=True)] == 0), f"{name}: a masked key got weight"
    full = ~valid.any(-1)                                             # [NB, i] query rows without a valid key
    assert bool(full.any()) == (masking in ("q", "qk", "keys_all"))
    if full.any():
        assert torch.all(v.permute(0, 2, 1, 3)[full] == float(torch.tensor(1.0 / j))), f"{name}: a row without keys is not uniform"


@pytest.mark.parametrize("dh", [12, 20])
@pytest.mark.parametrize("i", [7, 30])
def test_strict_xgate_split(i, dh):
    g = torch.Generator(device="cuda").manual_seed(i + dh)
    I, Pi = H_S * dh, _al(H_S * dh, 8)
    qg = torch.randn(B_S * i, 2 * I, device="cuda", generator=g)
    qg[:, I:] = (torch.rand(B_S * i, I, device="cuda", generator=g) * 2 - 1) * 20
    O = torch.randn(NB * H_S * i * dh, device="cuda", generator=g)

    def run():
        og = _nan(B_S * i * SPL * Pi, BF)
        _call("af2_strict_xgate_split", O.data_ptr(), qg.data_ptr(), og.data_ptr(), B0, NB, H_S, i, dh)
        return og
    og = _twice(run)
    pl = og[: B_S * i * SPL * Pi].view(B_S, i, SPL, Pi)
    others = torch.ones(B_S, dtype=torch.bool)
    others[B0:B0 + NB] = False
    assert torch.isnan(pl[others]).all(), "rows of batch elements outside the chunk written"
    ref = O.double().view(NB, H_S, i, dh).permute(0, 2, 1, 3).reshape(NB * i, I) * \
        torch.sigmoid(qg.view(B_S, i, 2 * I)[B0:B0 + NB, :, I:].double().reshape(NB * i, I))
    sel = pl[B0:B0 + NB].flatten()
    _split_out(f"strict/xgate_split/i{i}dh{dh}", sel, (NB * i, Pi), I, ref, 5 * U * ref.abs())


# ------------------------------------------------------------------------------------------------------------------------
# D. the module
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", BIAS_LAYOUTS)
@pytest.mark.parametrize("strict", [False, True], ids=["bf16", "strict"])
def test_module_bias_layouts(strict, layout):
    """a bias read through its strides gives the bits of the same values as a contiguous [B, h, i, j] tensor"""
    B, i, j, d, heads, dh = 3, 37, 45, 64, 4, 32
    a, _ = _module(d, heads, dh, strict=strict, seed=5)
    g = torch.Generator().manual_seed(len(layout))
    kw = {k: v.cuda() for k, v in _inputs(B, i, j, d, heads, seed=len(layout)).items()}
    bias = _bias_layout(layout, B, heads, i, j, g)
    with torch.no_grad():
        out = a(**kw, attn_bias=bias)
        dense = a(**kw, attn_bias=bias.expand(B, heads, i, j).contiguous())
    assert torch.equal(_bits(out), _bits(dense)), f"{layout}: differs from the contiguous bias"


@pytest.mark.parametrize("j", [129, 300])
@pytest.mark.parametrize("dh", [16, 128])
def test_module_cross_vs_oracle(dh, j):
    """cross-attention at dim_head 16 and 128 (the DH 128 epilogue reads the gate at the query token, i != j) with more work
    items than SMs"""
    d, heads, i = 64, 4, 257
    B = _sms() // (3 * heads) + 1
    assert 3 * heads * B > _sms()
    a, st = _module(d, heads, dh, seed=dh + j)
    _run(a, st, heads, _inputs(B, i, j, d, heads, seed=j + dh, bias="bhij" if j == 300 else "1hij"), f"cross_items_dh{dh}_j{j}")


def _strict_chunk(B, heads, i, j):
    """strict_xattn_chunk (attention_api.inl): batch elements per pass, logits below 1 GiB"""
    per = heads * i * _al(j, 4) * 4
    return min(max(1, (1 << 30) // per), B)


def test_module_strict_chunks():
    """B = ch + 1 takes one more pass of the strict chunk loop than B = ch, and batch elements 0, ch - 1 and ch (the first of
    the second pass) have the bits of B = 1 calls"""
    heads, dh, d, n = 1, 16, 32, 1024
    ch = _strict_chunk(1 << 20, heads, n, n)
    assert ch == 256
    B = ch + 1
    a, st = _module(d, heads, dh, strict=True, seed=13)
    g = torch.Generator().manual_seed(13)
    x, c = torch.randn(B, n, d, generator=g), torch.randn(B, n, d, generator=g)
    m, cm = torch.rand(B, n, generator=g) > 0.2, torch.rand(B, n, generator=g) > 0.2
    m[ch, : n // 2] = False
    cm[ch - 1] = False
    bias = torch.randn(B, 1, 1, n, generator=g) * 2                  # a key bias per batch element
    cuda = dict(x=x.cuda(), context=c.cuda(), mask=m.cuda(), context_mask=cm.cuda(), attn_bias=bias.cuda())
    lib = _lib()

    def call(sl):
        n0 = lib.af2_launch_count()
        with torch.no_grad():
            out = a(**{k: v[sl] for k, v in cuda.items()})
        return out, lib.af2_launch_count() - n0
    full, n_full = call(slice(0, B))
    _, n_ch = call(slice(0, ch))
    assert n_full - n_ch == 5, f"one more chunk pass took {n_full - n_ch} launches"
    for b in (0, ch - 1, ch):
        one, _ = call(slice(b, b + 1))
        assert torch.equal(_bits(one), _bits(full[b:b + 1])), f"batch element {b} differs from a B = 1 call"
    ref = AO.attention(to64(st), "", x[ch:ch + 1].double(), heads, mask=m[ch:ch + 1], attn_bias=bias[ch:ch + 1].double(),
                       context=c[ch:ch + 1].double(), context_mask=cm[ch:ch + 1])
    check_strict("strict_chunk_element_ch", full[ch:ch + 1], ref.float())


@pytest.mark.parametrize("strict", [False, True], ids=["bf16", "strict"])
def test_module_one_query_mask_without_context_mask(strict):
    """i = 1 without a bias (the pointwise template kernel) with a query mask and no context mask: a null key mask"""
    d, heads, dh = (40, 4, 32) if strict else (128, 4, 32)
    a, st = _module(d, heads, dh, strict=strict, seed=21)
    _run(a, st, heads, _inputs(16, 1, 5, d, heads, seed=21, context_mask=False, masked_rows=True), "one_query_no_context_mask",
         strict=strict)
