"""TEST INFRASTRUCTURE ONLY -- plain-torch statement of the structure scores of alphafold2_pytorch/utils.py (kabsch_torch,
rmsd_torch, gdt_torch, tmscore_torch, lddt_ca_torch, distmat_loss_torch) and of alphafold2_b200.utils.score_coords, written
from the reference's behaviour, in any dtype, on CPU or GPU tensors.

Distances are the explicit expression sqrt((dx * dx + dy * dy) + dz * dz) with dx = a - b, one torch operation per step (no
FMA contraction), so in fp64 on fp32 inputs they are bitwise equal to the kernels' and the threshold decisions can be
compared exactly.  The reference's torch.cdist takes its matmul form above 25 points; inputs recorded in the fixture keep
every decision at least 1e-3 away from a threshold, so the two agree on all of them."""
import torch

LDDT_THRESHOLDS = (0.5, 1.0, 2.0, 4.0)
GDT_TS = (1.0, 2.0, 4.0, 8.0)
GDT_HA = (0.5, 1.0, 2.0, 4.0)
NEAR = 1e-9


def dist(a, b, dtype=torch.float64):
    """|a - b| over the last axis (3) of a, b [..., 3], evaluated in dtype in the kernels' order."""
    d = a.to(dtype) - b.to(dtype)
    return ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).sqrt()


def kabsch(X, Y, dtype=torch.float64):
    """X, Y [3, N] -> (U^T X_, Y_, U, S) with C = X_ Y_^T = V S W, V's last column negated when det V det W < 0, U = V W."""
    X, Y = X.to(dtype), Y.to(dtype)
    Xc = X - X.mean(dim=-1, keepdim=True)
    Yc = Y - Y.mean(dim=-1, keepdim=True)
    C = Xc @ Yc.t()
    V, S, W = torch.linalg.svd(C)
    if torch.det(V) * torch.det(W) < 0:
        V = V.clone()
        V[:, -1] = -V[:, -1]
    U = V @ W
    return (Xc.t() @ U).t(), Yc, U, S


def rmsd(X, Y, dtype=torch.float64):
    """[B, 3, N] -> [B]: sqrt of the mean over both the 3 and the N axes."""
    return ((X.to(dtype) - Y.to(dtype)) ** 2).mean(dim=(-1, -2)).sqrt()


def point_dist(X, Y, dtype=torch.float64):
    """[B, 3, N] -> [B, N]"""
    return dist(X.transpose(-1, -2), Y.transpose(-1, -2), dtype)


def gdt(X, Y, cutoffs, weights=None, dtype=torch.float64):
    """-> ([B] sum_k w_k GDT_k / K, counts [B, K]); a point counts when d <= cutoff"""
    d = point_dist(X, Y, dtype)
    counts = torch.stack([(d <= c).sum(-1) for c in cutoffs], -1)
    w = torch.ones(len(cutoffs), dtype=dtype) if weights is None else torch.tensor([float(v) for v in weights], dtype=dtype)
    g = counts.to(dtype) / d.shape[-1]
    return (g * w.to(g.device)).mean(-1), counts


def tm_d0(n):
    L = max(15, n)
    return 1.24 * (L - 15) ** (1 / 3) - 1.8


def tmscore(X, Y, dtype=torch.float64):
    d = point_dist(X, Y, dtype)
    return (1 / (1 + (d / tm_d0(X.shape[-1])) ** 2)).mean(-1)


def lddt_counts(true_ca, pred_ca, present, r0=15.0, chunk=None):
    """true_ca, pred_ca [b, N, 3], present [b, N] bool -> (count, score) int64 [b, N] over the CAs present (self included):
    count = #{j : d_true < r0}, score = sum over those j of #{t : |d_pred - d_true| <= t}.  chunk: rows per step."""
    b, n, _ = true_ca.shape
    chunk = chunk or n
    cnt = torch.zeros(b, n, dtype=torch.int64, device=true_ca.device)
    scr = torch.zeros_like(cnt)
    for r0_ in range(0, n, chunk):
        r1 = min(n, r0_ + chunk)
        dt = dist(true_ca[:, r0_:r1, None], true_ca[:, None])
        dp = dist(pred_ca[:, r0_:r1, None], pred_ca[:, None])
        pair = present[:, r0_:r1, None] & present[:, None, :]
        inr = (dt < r0) & pair
        diff = (dp - dt).abs()
        s = sum((diff <= t).to(torch.int64) for t in LDDT_THRESHOLDS)
        cnt[:, r0_:r1] = inr.sum(-1)
        scr[:, r0_:r1] = (s * inr).sum(-1)
        del dt, dp, diff, s
    return cnt * present, scr * present


def lddt_ratio(cnt, scr, present):
    """(score - 4) / (4 count - 4) in fp32, 0 where the CA is absent"""
    val = (scr.float() - 4.0) / (4.0 * cnt.float() - 4.0)
    return torch.where(present, val, torch.zeros_like(val))


def lddt_ca(true_coords, pred_coords, cloud_mask, r_0=15.0, chunk=None):
    """[b, L, C, 3] sidechainnet layout, CA = atom 1 -> (lddt [b, L] fp32, count, score)"""
    present = cloud_mask[..., 1].bool()
    cnt, scr = lddt_counts(true_coords[:, :, 1], pred_coords[:, :, 1], present, r_0, chunk)
    return lddt_ratio(cnt, scr, present), cnt, scr


def distmat_loss(X=None, Y=None, X_mat=None, Y_mat=None, q=2, distmat_mask=None, clamp=None, dtype=torch.float64):
    """the loss with the kernels' distances: mean over the mask of ((D_X - D_Y)^2)^(q / 2)"""
    def mat(c, m):
        if m is not None:
            return m.to(dtype)
        c = c.squeeze()
        if clamp is not None:
            c = torch.clamp(c, *clamp)
        return dist(c[..., :, None, :], c[..., None, :, :], dtype)
    d = (mat(X, X_mat) - mat(Y, Y_mat)) ** 2
    if q != 2:
        d = d ** (q / 2)
    if distmat_mask is None:
        return d.mean()
    return d[distmat_mask.expand(d.shape)].mean()


def score_coords(pred, true, mask=None):
    """score_coords as the composition of the mirrors in fp64 on each element's selected residues S.  Also returns the
    decisions that may differ from the kernels' because the last bits of U differ: points whose distance lies within 1e-9
    of a GDT cutoff (``gdt_near`` [b] counts)."""
    pred, true = pred.cpu(), true.cpu()
    b, n, _ = pred.shape
    mask = torch.ones(b, n, dtype=torch.bool) if mask is None else mask.bool().cpu()
    nan = float("nan")
    out = {k: torch.full((b,), nan, dtype=torch.float64) for k in ("rmsd", "gdt_ts", "gdt_ha", "tm_score", "lddt_mean")}
    out["aligned"] = torch.full((b, n, 3), nan, dtype=torch.float64)
    out["U"] = torch.full((b, 3, 3), nan, dtype=torch.float64)
    out["S"] = torch.full((b, 3), nan, dtype=torch.float64)
    out["gdt_near"] = torch.zeros(b, dtype=torch.int64)
    cnt, scr = lddt_counts(true, pred, mask)
    out["lddt"] = lddt_ratio(cnt, scr, mask)
    out["lddt_count"], out["lddt_score"] = cnt, scr
    for e in range(b):
        S = mask[e]
        if not S.any():
            continue
        P, T = pred[e][S].t().double().cpu(), true[e][S].t().double().cpu()
        A, B, U, sv = kabsch(P, T)
        A32, B32 = A.float()[None], B.float()[None]             # the mirrors' outputs are fp32
        out["rmsd"][e] = rmsd(A32, B32)[0]
        out["gdt_ts"][e] = gdt(A32, B32, GDT_TS)[0][0]
        out["gdt_ha"][e] = gdt(A32, B32, GDT_HA)[0][0]
        out["tm_score"][e] = tmscore(A32, B32)[0]
        d = point_dist(A, B)[0]
        out["gdt_near"][e] = sum(int(((d - c).abs() <= NEAR).sum()) for c in set(GDT_TS + GDT_HA))
        Pc = pred[e].t().double().cpu() - P.mean(-1, keepdim=True)
        out["aligned"][e] = ((Pc.t() @ U).t() + T.mean(-1, keepdim=True)).t()
        out["U"][e], out["S"][e] = U, sv
        l = out["lddt"][e][S]
        out["lddt_mean"][e] = l[torch.isfinite(l)].double().mean()
    return out
