"""CPU controls of the bounds in structure_bounds.py: each structure-module kernel of test_gpu_structure_kernels.py is emulated
in fp32 in the kernel's own operation order (fmaf as one rounding of the exact product and sum, the per-lane chains and the
shuffle tree, the tile-wise online softmax with the kernel's TJ), the faithful emulation must pass every gate, and each plausible
wrong variant must fail the gate named beside it:

  IPA      point scale 1/sqrt 48 instead of 1/sqrt 54                      IPA bound
           pair bias without the 1/sqrt 3                                 IPA bound
           mask applied to keys only, not mask_i and mask_j                IPA bound (the fully masked query rows)
           -inf instead of -FLT_MAX for masked logits                      non-finite output
           online softmax without the alpha rescale                        IPA bound
           partial last tile read as TJ rows (the unused rows zero)        IPA bound
           (g - t) R instead of (g - t) R^T                                IPA bound (point columns)
  linear   ReLU before the bias; dropped bias                              GEMM bound
  tail     unbiased variance                                               tail bound (single)
           translation update with R_new instead of R_old                  tail bound (trans)
           coordinates with R_old                                          tail bound (coords)
           no sign normalisation of q                                      tail bound (sign-aware q check)

Every variant in the table is visible to an output bound; none needs another test to catch it.
"""
import math

import pytest
import torch

import structure_bounds as S

F = torch.float32
FLT_MAX = torch.finfo(F).max


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def fma(a, b, c):
    """fmaf: the exact a b + c rounded once to fp32 (the fp64 product of two fp32 values is exact)"""
    return (a.double() * b.double() + c.double()).float()


def f32(v):
    return torch.tensor(v, dtype=F)


def _warp_sum(x):
    """__shfl_xor tree over the last axis of 32 lanes (every lane ends with the same sum)"""
    for o in (16, 8, 4, 2, 1):
        x = x[..., :o] + x[..., o:2 * o]
    return x[..., 0]


def _lane_dot(y, w):
    """sum_c y[..., c] w[k, c] as the warp-per-row kernels form it: a per-lane fmaf chain over c = lane, lane + 32, .. and the
    shuffle tree -> [..., k]"""
    d = y.shape[-1]
    dp = (d + 31) // 32 * 32
    yl = torch.nn.functional.pad(y, (0, dp - d)).reshape(*y.shape[:-1], 1, dp // 32, 32)
    wl = torch.nn.functional.pad(w, (0, dp - d)).reshape(w.shape[0], dp // 32, 32)
    part = torch.zeros(*y.shape[:-1], w.shape[0], 32, dtype=F)
    for k in range(dp // 32):
        part = fma(yl[..., k, :], wl[:, k, :], part)
    return _warp_sum(part)


# ------------------------------------------------------------------------------------------------------------------------
# fp32 linear
# ------------------------------------------------------------------------------------------------------------------------
def _emu_linear(x, w, bias, relu, relu_first=False, drop_bias=False):
    acc = torch.zeros(x.shape[0], w.shape[0], dtype=F)
    for k in range(x.shape[1]):
        acc = fma(x[:, k:k + 1], w[None, :, k], acc)
    if relu and relu_first:
        acc = acc.clamp_min(0)
    if bias is not None and not drop_bias:
        acc = acc + bias
    return acc.clamp_min(0) if relu and not relu_first else acc


@pytest.mark.parametrize("M,N,K", [(1, 1, 1), (33, 3, 15), (31, 84, 17), (70, 36, 100)])
def test_linear_bound(M, N, K):
    g = _gen(M * 7 + N + K)
    x = torch.randn(M, K, generator=g)
    w, b = torch.randn(N, K, generator=g) * K ** -0.5, torch.randn(N, generator=g)
    for bias, relu in ((None, False), (b, False), (b, True), (None, True)):
        ref, bound = S.linear_ref(x, w, bias, relu)
        assert S.within(_emu_linear(x, w, bias, relu), ref, bound), (bias is not None, relu)
    ref, bound = S.linear_ref(x, w, b, True)
    assert not S.within(_emu_linear(x, w, b, True, relu_first=True), ref, bound), "ReLU before the bias"
    assert not S.within(_emu_linear(x, w, b, True, drop_bias=True), ref, bound), "dropped bias (ReLU)"
    ref, bound = S.linear_ref(x, w, b, False)
    assert not S.within(_emu_linear(x, w, b, False, drop_bias=True), ref, bound), "dropped bias"


# ------------------------------------------------------------------------------------------------------------------------
# frames
# ------------------------------------------------------------------------------------------------------------------------
def _emu_frames(proj, rot, trans, H):
    p = proj.clone().reshape(-1, 84 * H)
    R, t = rot.reshape(-1, 9), trans.reshape(-1, 3)
    X = p[:, 48 * H:].reshape(p.shape[0], -1, 3)
    G = torch.stack([fma(X[..., 0], R[:, None, c], fma(X[..., 1], R[:, None, 3 + c], fma(X[..., 2], R[:, None, 6 + c],
                                                                                         t[:, None, c]))) for c in range(3)], -1)
    p[:, 48 * H:] = G.reshape(p.shape[0], -1)
    return p.reshape(proj.shape)


@pytest.mark.parametrize("scale", [5.0, 500.0])
def test_frames_bound(scale):
    g = _gen(int(scale))
    rows, H = 23, 3
    proj = torch.randn(rows, 84 * H, generator=g)
    rot = S.quat_to_matrix(torch.randn(rows, 4, generator=g, dtype=torch.float64)).float()
    trans = torch.randn(rows, 3, generator=g) * scale
    ref, bound = S.frames_ref(proj, rot, trans, H)
    assert S.within(_emu_frames(proj, rot, trans, H), ref, bound)
    assert not S.within(_emu_frames(proj, rot.transpose(-1, -2).contiguous(), trans, H), ref, bound), "R^T"


# ------------------------------------------------------------------------------------------------------------------------
# invariant point attention
# ------------------------------------------------------------------------------------------------------------------------
def _emu_ipa(proj, pair, w_bias, b_bias, pw, mask, rot, trans, H, TJ, point_scale=54.0, pair_scale=True, keys_only=False,
             neg=-FLT_MAX, rescale=True, full_last_tile=False, transpose=True):
    """ipa_attention_kernel in fp32: logits of every (i, j, h) as the kernel forms them, then per tile of TJ keys the running
    max, the rescale alpha, the sum and the fmaf aggregates; the epilogue's division, (g - t) R^T and the norms"""
    B, n, _, d = pair.shape
    r3, r48 = f32(1 / math.sqrt(3)), f32(1 / math.sqrt(48))
    sp = torch.nn.functional.softplus(pw)
    coef = (f32(-0.5) * sp) * f32(1 / math.sqrt(point_scale))
    out = []
    for b in range(B):
        pr = proj[b]
        qs, ks, vs = (pr[:, k * 16 * H:(k + 1) * 16 * H].reshape(n, H, 16) for k in range(3))
        qp, kp, vp = (pr[:, 48 * H + k * 12 * H:48 * H + (k + 1) * 12 * H].reshape(n, H, 12) for k in range(3))
        P = pair[b]
        bias = _lane_dot(P, w_bias)                                           # [i, j, h]
        sdot = torch.zeros(n, n, H, dtype=F)
        for e in range(16):
            sdot = fma(qs[:, None, :, e], ks[None, :, :, e], sdot)
        df = qp[:, None] - kp[None]
        dist = torch.zeros(n, n, H, dtype=F)
        for e in range(12):
            dist = fma(df[..., e], df[..., e], dist)
        lb = (bias + b_bias) * r3 if pair_scale else bias + b_bias
        logit = (lb + sdot * r48) + coef * dist
        if mask is not None:
            ok = mask[b][None, :].expand(n, n) if keys_only else (mask[b][:, None] & mask[b][None, :])
            logit = torch.where(ok[..., None], logit, torch.full_like(logit, neg))
        # the logit of a zero key row (pair and projection 0): what a full read of a partial last tile adds
        zero_logit = b_bias * r3 + coef * (qp * qp).sum(-1)                  # [i, h]
        V = torch.cat((vs, vp), -1)                                           # [j, h, 28]
        m = torch.full((n, H), -math.inf, dtype=F)
        l = torch.zeros(n, H, dtype=F)
        acc = torch.zeros(n, H, d, dtype=F)
        accv = torch.zeros(n, H, 28, dtype=F)
        for j0 in range(0, n, TJ):
            rows = min(TJ, n - j0)
            L = logit[:, j0:j0 + rows]
            if full_last_tile and rows < TJ:
                L = torch.cat((L, zero_logit[:, None].expand(n, TJ - rows, H)), 1)
            m_new = torch.maximum(m, L.amax(1))
            p = torch.exp(L - m_new[:, None])
            alpha = torch.exp(m - m_new) if rescale else torch.ones_like(m)
            m = m_new
            l = l * alpha + p.sum(1)
            acc = acc * alpha[..., None]
            accv = accv * alpha[..., None]
            for jj in range(rows):
                acc = fma(p[:, jj, :, None], P[:, j0 + jj, None, :], acc)
                accv = fma(p[:, jj, :, None], V[None, j0 + jj], accv)
        o_pair = acc / l[..., None]
        o_s = accv[..., :16] / l[..., None]
        inv = 1 / l
        R, t = rot[b].reshape(n, 3, 3), trans[b].reshape(n, 3)
        gg = accv[..., 16:].reshape(n, H, 4, 3) * inv[..., None, None] - t[:, None, None, :]
        Rm = R if transpose else R.transpose(-1, -2)
        loc = torch.stack([fma(gg[..., 0], Rm[:, None, None, c, 0], fma(gg[..., 1], Rm[:, None, None, c, 1],
                                                                        gg[..., 2] * Rm[:, None, None, c, 2])) for c in range(3)], -1)
        sq = torch.zeros(n, H, 4, dtype=F)
        for c in range(3):
            sq = fma(loc[..., c], loc[..., c], sq)
        nrm = torch.sqrt(sq + f32(1e-8))
        out.append(torch.cat((o_s.reshape(n, -1), loc.reshape(n, -1), nrm.reshape(n, -1), o_pair.reshape(n, -1)), -1))
    return torch.stack(out)


def _ipa_inputs(n, H, d, TJ, g, scale=5.0):
    B = 2
    proj = torch.randn(B, n, 84 * H, generator=g)
    rot = S.quat_to_matrix(torch.randn(B, n, 4, generator=g, dtype=torch.float64)).float()
    trans = torch.randn(B, n, 3, generator=g) * scale
    proj = S.frames_ref(proj, rot, trans, H)[0].float()                       # points global, as af2_ipa_frames leaves them
    pair = torch.randn(B, n, n, d, generator=g)
    w_bias, b_bias = torch.randn(H, d, generator=g) * d ** -0.5, torch.randn(H, generator=g)
    pw = torch.randn(H, generator=g)
    pw[0] = 25.0                                                              # softplus's x > 20 branch, peaked logits
    pw[-1] = -30.0 if H > 1 else pw[-1]
    mask = torch.ones(B, n, dtype=torch.bool)
    mask[0, :TJ] = False                                                      # the whole first tile of keys ...
    mask[0, TJ + 2::4] = False                                                # ... and scattered fully masked query rows
    mask[1, S.mid_tile_length(n, TJ):] = False                                # padding that ends mid-tile
    return proj, pair, w_bias, b_bias, pw, mask, rot, trans


@pytest.mark.parametrize("n,H,d,TJ", [(37, 3, 36, 4), (29, 2, 8, 8), (9, 4, 4, 2)])
def test_ipa_bound(n, H, d, TJ):
    g = _gen(n * 10 + TJ)
    args = _ipa_inputs(n, H, d, TJ, g)
    ref, bound = S.ipa_attention_ref(*args, H, TJ, rows_per_chunk=7)
    OW = H * (32 + d)
    pts = torch.zeros(OW, dtype=torch.bool)
    pts[16 * H:32 * H] = True

    def gate(cols=None, **mut):
        out = _emu_ipa(*args, H, TJ, **mut)
        if cols is not None:
            return S.within(out[..., cols], ref[..., cols], bound[..., cols])
        return S.within(out, ref, bound)
    assert gate()
    assert not gate(point_scale=48.0), "point scale 1/sqrt 48"
    assert not gate(pair_scale=False), "pair bias without 1/sqrt 3"
    assert not gate(keys_only=True), "mask on keys only"
    assert not torch.isfinite(_emu_ipa(*args, H, TJ, neg=-math.inf)).all(), "-inf for masked logits"
    assert not gate(rescale=False), "no alpha rescale"
    assert not gate(full_last_tile=True), "partial last tile read as TJ rows"
    assert not gate(pts, transpose=False), "(g - t) R instead of R^T"


def test_ipa_bound_far_frames():
    """translations at 500: the bound must carry the |t| terms, and still see a transposed R"""
    g = _gen(500)
    n, H, d, TJ = 21, 2, 12, 4
    args = _ipa_inputs(n, H, d, TJ, g, scale=500.0)
    ref, bound = S.ipa_attention_ref(*args, H, TJ)
    assert S.within(_emu_ipa(*args, H, TJ), ref, bound)
    assert not S.within(_emu_ipa(*args, H, TJ, transpose=False), ref, bound), "(g - t) R"


# ------------------------------------------------------------------------------------------------------------------------
# tail
# ------------------------------------------------------------------------------------------------------------------------
def _emu_tail(s, o, gamma, beta, eps, w_qu=None, b_qu=None, quat=None, trans=None, rot=None, w_points=None, b_points=None,
              w_lddt=None, b_lddt=None, unbiased=False, t_with_new=False, coords_with_old=False, sign=True):
    d = s.shape[-1]
    v = s + o
    dp = (d + 31) // 32 * 32
    vl = torch.nn.functional.pad(v, (0, dp - d)).reshape(-1, dp // 32, 32)
    part = torch.zeros(v.shape[0], 32, dtype=F)
    for k in range(dp // 32):
        part = part + vl[:, k]
    mean = _warp_sum(part) / d
    c = torch.nn.functional.pad(v - mean[:, None], (0, dp - d)).reshape(-1, dp // 32, 32)
    part = torch.zeros(v.shape[0], 32, dtype=F)
    for k in range(dp // 32):
        part = fma(c[:, k], c[:, k], part)
    var = _warp_sum(part) / (d - 1 if unbiased else d)
    rstd = 1 / torch.sqrt(var + eps)
    y = fma((v - mean[:, None]) * rstd[:, None], gamma, beta)
    out = {"single": y}
    if w_qu is None:
        return out
    u = _lane_dot(y, w_qu) + b_qu
    a = quat
    b = torch.cat((torch.ones_like(u[:, :1]), u[:, :3]), -1)
    q = S._raw_qmul(a, b)
    if sign:
        q = torch.where(q[:, :1] < 0, -q, q)
    R_old = rot.reshape(-1, 3, 3)
    R_new = S.quat_to_matrix(q)
    Rt = R_new if t_with_new else R_old
    t = trans + torch.stack([fma(u[:, 3], Rt[:, 0, c], fma(u[:, 4], Rt[:, 1, c], u[:, 5] * Rt[:, 2, c])) for c in range(3)], -1)
    out.update(quat=q, trans=t, rot=R_new.reshape(-1, 9))
    if w_points is None:
        return out
    x = _lane_dot(y, w_points) + b_points
    Rc = R_old if coords_with_old else R_new
    out["coords"] = torch.stack([fma(x[:, 0], Rc[:, 0, c], fma(x[:, 1], Rc[:, 1, c], fma(x[:, 2], Rc[:, 2, c], t[:, c])))
                                 for c in range(3)], -1)
    out["confidence"] = _lane_dot(y, w_lddt) + b_lddt
    return out


def _tail_inputs(rows, d, g, t_scale=5.0):
    s, o = torch.randn(rows, d, generator=g) * 2, torch.randn(rows, d, generator=g)
    s[:5] += 300.0                                                            # a common offset the LayerNorm mean cancels
    gamma, beta = 1 + 0.3 * torch.randn(d, generator=g), 0.3 * torch.randn(d, generator=g)
    w_qu, b_qu = torch.randn(6, d, generator=g) * d ** -0.5, torch.randn(6, generator=g) * 0.3
    w_points, b_points = torch.randn(3, d, generator=g) * d ** -0.5, torch.randn(3, generator=g)
    w_lddt, b_lddt = torch.randn(1, d, generator=g) * d ** -0.5, torch.randn(1, generator=g)
    q = torch.randn(rows, 4, generator=g)
    q = q * torch.logspace(-2, 2, rows)[:, None] / q.norm(dim=-1, keepdim=True)   # norms 1e-2 .. 1e2
    q[: rows // 3, 0] *= 1e-4                                                 # real part near 0
    rot = S.quat_to_matrix(q.double()).float()
    trans = torch.randn(rows, 3, generator=g) * t_scale
    return dict(s=s, o=o, gamma=gamma, beta=beta, eps=1e-5, w_qu=w_qu, b_qu=b_qu, quat=q, trans=trans, rot=rot, w_points=w_points,
                b_points=b_points, w_lddt=w_lddt, b_lddt=b_lddt)


def _tail_gates(kw, out):
    ref = S.tail_ref(**kw)
    res = {}
    for name, got in out.items():
        r, bnd = ref[name]
        if name == "quat":
            r = S.align_quat_sign(got, r, ref["quat_ambiguous"])
        res[name] = S.within(got.reshape(r.shape), r, bnd)
    return res


@pytest.mark.parametrize("d", [4, 36, 260])
def test_tail_bound(d):
    g = _gen(d)
    kw = _tail_inputs(45, d, g, t_scale=500.0)
    for keep in ("single", "frames", "coords"):
        k = dict(kw)
        if keep != "coords":
            k.update(w_points=None, b_points=None, w_lddt=None, b_lddt=None)
        if keep == "single":
            k.update(w_qu=None, b_qu=None, quat=None, trans=None, rot=None)
        res = _tail_gates(k, _emu_tail(**k))
        assert all(res.values()), (keep, res)
    assert not _tail_gates(kw, _emu_tail(**kw, unbiased=True))["single"], "unbiased variance"
    assert not _tail_gates(kw, _emu_tail(**kw, t_with_new=True))["trans"], "translation with R_new"
    assert not _tail_gates(kw, _emu_tail(**kw, coords_with_old=True))["coords"], "coordinates with R_old"
    assert not _tail_gates(kw, _emu_tail(**kw, sign=False))["quat"], "no sign normalisation"


def test_tile_rule_tiers():
    """the restated rule reaches every tier the kernel has: TJ 32 / 16 / 8 at four CTAs per SM, 32 .. 1 at two, 8 and 4 at one"""
    tiers = {S.ipa_tile_rule(H, d)[:2] for H in range(1, 17) for d in range(4, 1025, 4)}
    assert tiers == {(4, 32), (4, 16), (4, 8), (2, 16), (2, 8), (2, 4), (2, 2), (2, 1), (1, 8), (1, 4)}
    assert S.ipa_tile_rule(16, 1024)[2] <= 227 * 1024
