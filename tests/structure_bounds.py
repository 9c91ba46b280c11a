"""fp64 references and per-element error bounds of the structure module's kernels (include/af2b200.h: af2_structure_linear,
af2_ipa_frames, af2_ipa_attention, af2_structure_tail), and a restatement of the attention kernel's tile rule.

Plain device-generic torch: test_gpu_structure_kernels.py gates the kernels with these bounds on the GPU, and
test_structure_bounds_controls.py checks on the CPU that a faithful fp32 emulation of each kernel passes them while plausible
wrong variants do not.  Every reference starts from the kernel's own fp32 inputs, so a kernel is judged alone.  u = 2^-24; a
k-term fmaf chain is off by at most k u sum|terms|; rsqrtf, expf and log1pf are within 2 ulp (4 u relative).

fp32 linear (csrc/structure.cuh: structure_linear_kernel).  Each output is one fmaf chain over K (slices of 16, in order), then
acc + bias, then the ReLU:  |y - ref| <= K u sum_k |x_k w_k| + 2 u |z|  (gemm_f32_bound, z the pre-ReLU value); the ReLU is
1-Lipschitz, so the bound of z holds for relu(z).

Frames (ipa_frames_kernel).  G_c = fmaf(x, R_0c, fmaf(y, R_1c, fmaf(z, R_2c, t_c))): three roundings, each of a partial sum:
|G_c - ref| <= 4 u (sum_k |X_k R_kc| + |t_c|).

Invariant point attention (ipa_attention_kernel), per query i, head h, key j:
  logit error delta_ij, each term with its own rounding:
    pair bias   (pair_ij . W_h + b_h) / sqrt 3: a ceil(d/32)-term fmaf chain per lane and 5 shuffle levels
                -> ((ceil(d/32) + 5) u sum|pair W| + u |pb|) / sqrt 3 + 6 u |l_b|   (rsqrtf and the product)
    scalar      q . k / sqrt 48: 16-term fmaf chain -> 16 u sum|q k| / sqrt 48 + 6 u |l_s|
    point       c_h |Q_i - K_j|^2, c_h = -softplus(w_h) / (2 sqrt 54): the 12 differences (u each, squared: 2 u), the chain
                (12 u) and c_h (softplus, rsqrtf, two products: 16 u) -> 32 u |l_p|      (all terms of dist are >= 0)
    sum         2 u (|l_b| + |l_s| + |l_p|)
  A masked pair (not mask_i and mask_j) is -FLT_MAX in the kernel and -DBL_MAX in the reference: both give exactly the weights
  0 (or 1 / n on a fully masked row), so delta = 0 there.
  Softmax.  The kernel's weight of key j is exp(l_j - m) up to the relative factor e^{rho_j}:
    rho_j = delta_j + u (m - l_j) + 4 u (ntiles + 1)
  (the roundings of l_j - m_t and of every later tile's m_old - m_new sum to u (m - l_j); one expf for p_j and one per later
  alpha).  Normalised, a_j -> a_j e^{eps_j} / S with |log S| <= rho_bar = log sum_j a_j e^{rho_j}, so
    |a^_j - a_j| <= a_j (e^{rho_j + rho_bar} - 1) =: w_j   and, as sum_j (a^_j - a_j) = 0,
    |o^ - o| <= sum_j w_j |v_j - o| + (n + ntiles) u sum_j a_j |v_j| + (7 ntiles + 2) u |o|
  (the accumulator: n fmafs and ntiles alpha products per output; the running sum: at most 5 shuffle levels, a product and an add
  per tile; the division).  The pair aggregates use the looser sum_j w_j (|v_j| + |o|).  (For the first-order steps: every
  exponent here is below 1e-3 wherever a_j is not 0.)
  Epilogue on the global o_point g: (g - t) carries u |g - t| more; l_c = sum_k (g - t)_k R_ck (a 3-term fmaf chain):
    |dl_c| <= sum_k |d(g - t)_k| |R_ck| + 3 u sum_k |(g - t)_k R_ck|
  so the translations enter through |g| ~ |t| in the softmax term and through u |g - t|.  The norm sqrt(|l|^2 + 1e-8) is
  1-Lipschitz in l; its own roundings add 4 u |norm|, and 1e-8f differs from 1e-8 by 6e-17.

Tail (structure_tail_kernel), warp per residue, VPL = ceil(d/32) values per lane:
  s <- LayerNorm(v), v = fl(s + o): _ln_ref's bound with k_d = VPL + 5, plus the shift u |v| of each input carried through the
  LayerNorm (as embed_bounds.distogram_ref does for its symmetrised input).
  dots (6 updates, 3 points, 1 confidence): |d| <= sum|W| dy + (VPL + 5) u sum (|y| + dy) |W| + u |ref|  (per-lane fmaf chain,
  shuffles, bias add).
  q' = q (x) (1, u_0, u_1, u_2): each component a 4-term sum:  |dq'| <= |q| (x) |du| + 5 u |q| (x) |(1, u)|  ((x): the product
  with every sign +).  Where |q'_0| <= its bound the sign flip may go either way, and both signs are right:
  quat_to_matrix(-q) = quat_to_matrix(q) and the next product re-normalises the sign -- so q is compared up to sign there.
  R' = quat_to_matrix(q') depends on q' / |q'| only: |dR| <= 8 sum|dq'| / |q'| (first order) + 24 u (its own roundings).
  t' = t + v R (R before the update): |dt'_c| <= sum_k |dv_k| |R_kc| + 3 u sum_k |v_k R_kc| + u |t'_c|.
  coords_c = sum_k x_k R'_kc + t'_c (fmaf chain): |d| <= sum_k (dx_k |R'_kc| + |x_k| dR'_kc) + dt'_c + 3 u (sum_k |x_k R'_kc| + |t'_c|).
"""
import math

import torch

from gpu_util import U32 as U, gemm_f32_bound
from test_gpu_strict_kernels import _ln_ref

IPA_SD, IPA_PT, IPA_PROJ = 16, 4, 84
IPA_VW = IPA_SD + 3 * IPA_PT
EPS_NORM = 1e-8
EPS_NORM_F32_GAP = abs(float(torch.tensor(EPS_NORM, dtype=torch.float32)) - EPS_NORM)
NEG_MAX64 = -torch.finfo(torch.float64).max

# (cap bytes, smallest TJ) of the three occupancy passes of ipa_tile_rows: 4, 2 and 1 CTAs per SM
IPA_PASSES = ((4, 56 * 1024, 8), (2, 113 * 1024, 1), (1, 227 * 1024, 1))


def _dot(a, w):
    """a [..., K] @ w [N, K]^T in fp64"""
    return a.double() @ w.double().transpose(0, 1)


# ------------------------------------------------------------------------------------------------------------------------
# tile rule (csrc/structure.cuh: IpaSmem; csrc/structure_api.inl: ipa_tile_rows)
# ------------------------------------------------------------------------------------------------------------------------
def ipa_smem_bytes(H, d, TJ):
    """dynamic shared memory of one attention CTA: two mbarriers, two pair tiles, two key-projection tiles, bias weights, the
    o_pair and value accumulators, the query, the tile's logits and four per-head statistics"""
    floats = 4 + 2 * TJ * d + 2 * TJ * IPA_PROJ * H + H * d + H * d + H * IPA_VW + H * (IPA_SD + 3 * IPA_PT) + H * TJ + 4 * H
    return 4 * floats


def ipa_tile_rule(H, d):
    """-> (CTAs per SM, TJ, bytes): the largest of 32, 16, 8 key rows that leaves room for four CTAs per SM, else the largest of
    32 .. 1 for two, else for one; (0, 0, 0) when nothing fits"""
    for ctas, cap, tj_min in IPA_PASSES:
        TJ = 32
        while TJ >= tj_min:
            b = ipa_smem_bytes(H, d, TJ)
            if b <= cap:
                return ctas, TJ, b
            TJ //= 2
    return 0, 0, 0


# ------------------------------------------------------------------------------------------------------------------------
# fp32 linear and frames
# ------------------------------------------------------------------------------------------------------------------------
def linear_ref(x, w, bias=None, relu=False):
    """(ref, bound) of act(x w^T + bias) for x [..., K], w [N, K]"""
    K = x.shape[-1]
    z = _dot(x, w)
    if bias is not None:
        z = z + bias.double()
    bound = gemm_f32_bound(_dot(x.abs(), w.abs()), K, z)
    return (z.clamp_min(0) if relu else z), bound


def frames_ref(proj, rot, trans, H):
    """(ref, bound) of af2_ipa_frames on proj [..., 84 H]: the point columns X R + t, the scalar columns unchanged (bound 0)"""
    lead = proj.shape[:-1]
    p = proj.double().reshape(-1, IPA_PROJ * H)
    R = rot.double().reshape(-1, 3, 3)
    t = trans.double().reshape(-1, 1, 3)
    X = p[:, 3 * IPA_SD * H:].reshape(p.shape[0], -1, 3)
    ref, bound = p.clone(), torch.zeros_like(p)
    ref[:, 3 * IPA_SD * H:] = (X @ R + t).reshape(p.shape[0], -1)
    bound[:, 3 * IPA_SD * H:] = (4 * U * (X.abs() @ R.abs() + t.abs())).reshape(p.shape[0], -1)
    return ref.reshape(*lead, -1), bound.reshape(*lead, -1)


# ------------------------------------------------------------------------------------------------------------------------
# invariant point attention
# ------------------------------------------------------------------------------------------------------------------------
def ipa_logits(P, qs, ks, qp, kp, w_bias, b_bias, point_weights, mm):
    """fp64 logits [H, r, n] and their bound delta of query rows with pair rows P [r, n, d], scalar q [r, H, 16] / k [n, H, 16],
    global points q [r, H, 12] / k [n, H, 12], mm [r, n] bool (True: attended) or None"""
    d = P.shape[-1]
    W = w_bias.double()
    pb = torch.einsum("ijd,hd->hij", P, W) + b_bias.double()[:, None, None]
    pb_abs = torch.einsum("ijd,hd->hij", P.abs(), W.abs())
    lb = pb / math.sqrt(3)
    ls = torch.einsum("ihe,jhe->hij", qs, ks) / math.sqrt(48)
    ls_abs = torch.einsum("ihe,jhe->hij", qs.abs(), ks.abs()) / math.sqrt(48)
    dist = (qp[:, None] - kp[None]).pow(2).sum(-1).permute(2, 0, 1)
    coef = -0.5 * torch.nn.functional.softplus(point_weights.double()) / math.sqrt(54)
    lp = coef[:, None, None] * dist
    logit = lb + ls + lp
    delta = (((d + 31) // 32 + 5) * U * pb_abs + U * pb.abs()) / math.sqrt(3) + 6 * U * lb.abs() + 16 * U * ls_abs \
        + 6 * U * ls.abs() + 32 * U * lp.abs() + 2 * U * (lb.abs() + ls.abs() + lp.abs())
    if mm is not None:
        logit = logit.masked_fill(~mm, NEG_MAX64)
        delta = delta.masked_fill(~mm, 0.0)
    return logit, delta


def _agg_bound(a, wgt, v, o, nterm, ocoef):
    """sum_j w_j |v_j - o| + nterm u sum_j a_j |v_j| + ocoef u |o| for v [n, H, k] (per-key values), a / wgt [H, r, n],
    o [r, H, k]"""
    diff = (v[None] - o[:, None]).abs()                                       # [r, n, H, k]
    return torch.einsum("hij,ijhk->ihk", wgt, diff) + nterm * U * torch.einsum("hij,jhk->ihk", a, v.abs()) + ocoef * U * o.abs()


def ipa_attention_ref(proj, pair, w_bias, b_bias, point_weights, mask, rot, trans, H, TJ, rows_per_chunk=None):
    """(ref, bound) of af2_ipa_attention's output [B, n, H (32 + d)] from its fp32 inputs: proj [B, n, 84 H] (points global),
    pair [B, n, n, d], mask [B, n] bool or None, rot [B, n, 3, 3], trans [B, n, 3]; TJ the kernel's key rows per tile.
    Query rows go in chunks so that the fp64 temporaries stay small."""
    B, n, _, d = pair.shape
    ntiles = (n + TJ - 1) // TJ
    OW = H * (2 * IPA_SD + d)
    ref = torch.empty(B, n, OW, dtype=torch.float64, device=pair.device)
    bound = torch.empty_like(ref)
    if rows_per_chunk is None:
        rows_per_chunk = max(1, min(n, (1 << 22) // max(1, n * max(d, H * IPA_VW))))
    for b in range(B):
        pr = proj[b].double()
        sq, sk, sv = (pr[:, k * IPA_SD * H:(k + 1) * IPA_SD * H].reshape(n, H, IPA_SD) for k in range(3))
        base = 3 * IPA_SD * H
        pq, pk, pv = (pr[:, base + k * 3 * IPA_PT * H:base + (k + 1) * 3 * IPA_PT * H].reshape(n, H, 3 * IPA_PT) for k in range(3))
        R = rot[b].double().reshape(n, 3, 3)
        t = trans[b].double().reshape(n, 3)
        for i0 in range(0, n, rows_per_chunk):
            i1 = min(n, i0 + rows_per_chunk)
            P = pair[b, i0:i1].double()
            mm = None if mask is None else (mask[b, i0:i1, None] & mask[b, None, :])
            logit, delta = ipa_logits(P, sq[i0:i1], sk, pq[i0:i1], pk, w_bias, b_bias, point_weights, mm)
            a = torch.softmax(logit, -1)
            m = logit.amax(-1, keepdim=True)
            rho = delta + U * (m - logit) + 4 * U * (ntiles + 1)
            if mm is not None:
                rho = rho.masked_fill(~mm, 0.0)
            rho_bar = torch.log((a * torch.exp(rho)).sum(-1, keepdim=True))
            wgt = a * torch.expm1(rho + rho_bar)
            nterm, ocoef = n + ntiles, 7 * ntiles + 2
            o_s = torch.einsum("hij,jhe->ihe", a, sv)
            o_g = torch.einsum("hij,jhe->ihe", a, pv)
            o_pair = torch.einsum("hij,ijd->ihd", a, P)
            e_s = _agg_bound(a, wgt, sv, o_s, nterm, ocoef)
            e_g = _agg_bound(a, wgt, pv, o_g, nterm, ocoef)
            e_pair = torch.einsum("hij,ijd->ihd", wgt, P.abs()) + wgt.sum(-1).transpose(0, 1)[..., None] * o_pair.abs() \
                + nterm * U * torch.einsum("hij,ijd->ihd", a, P.abs()) + ocoef * U * o_pair.abs()
            r = i1 - i0
            Ri, ti = R[i0:i1], t[i0:i1]
            gt = o_g.reshape(r, H, IPA_PT, 3) - ti[:, None, None, :]
            dgt = e_g.reshape(r, H, IPA_PT, 3) + U * gt.abs()
            loc = torch.einsum("ihpk,ick->ihpc", gt, Ri)
            dloc = torch.einsum("ihpk,ick->ihpc", dgt, Ri.abs()) + 3 * U * torch.einsum("ihpk,ick->ihpc", gt.abs(), Ri.abs())
            nrm = (loc.pow(2).sum(-1) + EPS_NORM).sqrt()
            dnrm = dloc.sum(-1) + 4 * U * nrm + EPS_NORM_F32_GAP / (2 * nrm)
            ref[b, i0:i1] = torch.cat((o_s.reshape(r, -1), loc.reshape(r, -1), nrm.reshape(r, -1), o_pair.reshape(r, -1)), -1)
            bound[b, i0:i1] = torch.cat((e_s.reshape(r, -1), dloc.reshape(r, -1), dnrm.reshape(r, -1), e_pair.reshape(r, -1)), -1)
    return ref, bound


# ------------------------------------------------------------------------------------------------------------------------
# layer tail
# ------------------------------------------------------------------------------------------------------------------------
def _abs_qmul(a, b):
    """the Hamilton product's component sums with every sign +: |a| (x) |b| for a, b >= 0"""
    a0, a1, a2, a3 = a.unbind(-1)
    b0, b1, b2, b3 = b.unbind(-1)
    return torch.stack((a0 * b0 + a1 * b1 + a2 * b2 + a3 * b3, a0 * b1 + a1 * b0 + a2 * b3 + a3 * b2,
                        a0 * b2 + a1 * b3 + a2 * b0 + a3 * b1, a0 * b3 + a1 * b2 + a2 * b1 + a3 * b0), -1)


def _raw_qmul(a, b):
    a0, a1, a2, a3 = a.unbind(-1)
    b0, b1, b2, b3 = b.unbind(-1)
    return torch.stack((a0 * b0 - a1 * b1 - a2 * b2 - a3 * b3, a0 * b1 + a1 * b0 + a2 * b3 - a3 * b2,
                        a0 * b2 - a1 * b3 + a2 * b0 + a3 * b1, a0 * b3 + a1 * b2 - a2 * b1 + a3 * b0), -1)


def quat_to_matrix(q):
    """pytorch3d quaternion_to_matrix (scale invariant): [..., 4] -> [..., 3, 3]"""
    r, i, j, k = q.unbind(-1)
    s = 2.0 / (q * q).sum(-1)
    o = torch.stack((1 - s * (j * j + k * k), s * (i * j - k * r), s * (i * k + j * r),
                     s * (i * j + k * r), 1 - s * (i * i + k * k), s * (j * k - i * r),
                     s * (i * k - j * r), s * (j * k + i * r), 1 - s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def _tail_dot(y, dy, w, b, vpl):
    aw = w.double().abs()
    ref = _dot(y, w) + b.double()
    return ref, _dot(dy, aw) + (vpl + 5) * U * _dot(y.abs() + dy, aw) + U * ref.abs()


def tail_ref(s, o, gamma, beta, eps, w_qu=None, b_qu=None, quat=None, trans=None, rot=None, w_points=None, b_points=None,
             w_lddt=None, b_lddt=None):
    """{name: (ref, bound)} of af2_structure_tail from its fp32 inputs (rows [rows, ...]): "single"; with w_qu "quat", "trans",
    "rot" (the updated frames; "quat_ambiguous" [rows] marks the rows whose sign may go either way); with w_points "coords" and
    "confidence" [rows, 1]"""
    d = s.shape[-1]
    vpl = (d + 31) // 32
    v = s.double() + o.double()
    g, be = gamma.double(), beta.double()
    y, dy = _ln_ref(v, g, be, vpl + 5, eps)
    mean = v.mean(-1, keepdim=True)
    xc = v - mean
    rstd = 1.0 / torch.sqrt((xc * xc).mean(-1, keepdim=True) + eps)
    va = v.abs()
    dy = dy + g.abs() * rstd * U * (va + va.mean(-1, keepdim=True) + (xc * rstd).abs() * rstd * (xc.abs() * va).mean(-1, keepdim=True))
    out = {"single": (y, dy)}
    if w_qu is None:
        return out
    upd, dupd = _tail_dot(y, dy, w_qu, b_qu, vpl)
    qa = quat.double().reshape(-1, 4)
    bq = torch.cat((torch.ones_like(upd[:, :1]), upd[:, :3]), -1)
    dbq = torch.cat((torch.zeros_like(dupd[:, :1]), dupd[:, :3]), -1)
    q2 = _raw_qmul(qa, bq)
    dq2 = _abs_qmul(qa.abs(), dbq) + 5 * U * _abs_qmul(qa.abs(), bq.abs())
    amb = q2[:, 0].abs() <= dq2[:, 0]
    qref = torch.where(q2[:, :1] < 0, -q2, q2)
    R0 = rot.double().reshape(-1, 3, 3)
    R2 = quat_to_matrix(q2)
    dR2 = (8 * dq2.sum(-1) / q2.norm(dim=-1))[:, None, None] + 24 * U
    vt, dvt = upd[:, 3:], dupd[:, 3:]
    t2 = trans.double().reshape(-1, 3) + torch.einsum("nk,nkc->nc", vt, R0)
    dt2 = torch.einsum("nk,nkc->nc", dvt, R0.abs()) + 3 * U * torch.einsum("nk,nkc->nc", vt.abs(), R0.abs()) + U * t2.abs()
    out.update(quat=(qref, dq2), trans=(t2, dt2), rot=(R2.reshape(-1, 9), dR2.expand(-1, 3, 3).reshape(-1, 9)), quat_ambiguous=amb)
    if w_points is None:
        return out
    x, dx = _tail_dot(y, dy, w_points, b_points, vpl)
    coords = torch.einsum("nk,nkc->nc", x, R2) + t2
    dcoords = torch.einsum("nk,nkc->nc", dx, R2.abs()) + torch.einsum("nk,nkc->nc", x.abs(), dR2.expand(-1, 3, 3)) + dt2 \
        + 3 * U * (torch.einsum("nk,nkc->nc", x.abs(), R2.abs()) + t2.abs())
    out.update(coords=(coords, dcoords), confidence=_tail_dot(y, dy, w_lddt, b_lddt, vpl))
    return out


def mid_tile_length(n, TJ):
    """a valid length for padding masks: about 3/4 of n, inside a tile of TJ keys when TJ > 1, at least 1"""
    L = max(1, n - max(1, n // 4))
    if TJ > 1 and L % TJ == 0 and L > 1:
        L -= 1
    return L


def align_quat_sign(q, ref, ambiguous):
    """ref with its sign flipped on the ambiguous rows where q points the other way (both signs are right there)"""
    flip = ambiguous & ((q.double() * ref).sum(-1) < 0)
    return torch.where(flip[:, None], -ref, ref)


def within(out, ref, bound):
    """the element-wise gate of gpu_util.check_bound as a predicate (finite and |out - ref| <= bound everywhere)"""
    return bool(torch.isfinite(out).all()) and bool(((out.double() - ref).abs() <= bound).all())
