"""TEST INFRASTRUCTURE ONLY -- round-10 fixture from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r10
  tests/golden/structure_metrics.pt  alphafold2_pytorch/utils.py run on the CPU in fp32:
    kabsch    Kabsch on a generic set, a reflected set (the determinant fix) and a planar set (rank-2 covariance)
    scores    RMSD, GDT TS and HA with and without weights [2, 1, 1, 1], and TMscore, batch 3, at N 10, 15, 16, 18, 19, 40; weighted GDT HA
              of a close pair (above 1)
    lddt      lddt_ca_torch at b 2, L 30 and L 40, C 14, with one missing CA and one isolated residue
    loss      distmat_loss_torch with coordinates, with matrices, with a bool mask, with clamp, with q = 1, and batched
  Every input is resampled until no fp64 decision lies within 1e-3 of a threshold (a GDT cutoff, r_0 or an lDDT threshold),
  so the reference's fp32 cdist and the oracle agree on every decision.  Under 500 KB."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402
from oracle import metrics_oracle as M  # noqa: E402

MARGIN = 1e-3
NS = (10, 15, 16, 18, 19, 40)


def near(x, thresholds):
    return any(bool(((x - t).abs() < MARGIN).any()) for t in thresholds)


def rotation(g):
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    return (q * torch.det(q)).float()


def pairs(b, n, g, spread):
    """[b, 3, N] X and Y = X + noise with point distances spread over the cutoffs, away from every cutoff"""
    while True:
        X = torch.randn(b, 3, n, generator=g) * 6
        Y = X + torch.randn(b, 3, n, generator=g) * spread
        if not near(M.point_dist(X, Y), M.GDT_TS + M.GDT_HA):
            return X, Y


def chain(L, C, g):
    """a sidechainnet-layout [L, C, 3] chain: CAs 3.8 A apart on a random walk, other atoms near their CA"""
    steps = torch.randn(L, 3, generator=g)
    ca = torch.cumsum(3.8 * steps / steps.norm(dim=-1, keepdim=True), 0)
    x = ca[:, None, :] + torch.randn(L, C, 3, generator=g)
    x[:, 1] = ca
    return x


def lddt_case(b, L, C, g):
    while True:
        true = torch.stack([chain(L, C, g) for _ in range(b)])
        pred = true + 0.8 * torch.randn(b, L, C, 3, generator=g)
        true[0, L - 1, 1] += 100.0                       # an isolated residue: no other CA within r_0
        pred[0, L - 1, 1] += 100.0
        mask = torch.ones(b, L, C, dtype=torch.bool)
        mask[1, 5, 1] = False                            # a missing CA
        mask[0, 3, 7:] = False
        ca_t, ca_p = true[:, :, 1], pred[:, :, 1]
        dt = M.dist(ca_t[:, :, None], ca_t[:, None])
        dp = M.dist(ca_p[:, :, None], ca_p[:, None])
        if not near(dt, (15.0,)) and not near((dp - dt).abs()[dt < 15.0], M.LDDT_THRESHOLDS):
            return true, pred, mask


def main():
    load_reference()
    import alphafold2_pytorch.utils as U
    g = torch.Generator().manual_seed(10)
    fx = {"kabsch": {}, "scores": {}, "lddt": {}, "loss": {}}

    X = torch.randn(3, 20, generator=g) * 5
    R = rotation(g)
    reflect = torch.diag(torch.tensor([1.0, 1.0, -1.0]))
    planar = X.clone()
    planar[2] = 0.0
    Rz = torch.tensor([[0.6, -0.8, 0.0], [0.8, 0.6, 0.0], [0.0, 0.0, 1.0]])
    sets = {"generic": (X, R @ X + 0.3 * torch.randn(3, 20, generator=g) + 2.0),
            "reflected": (X, R @ reflect @ X + 0.3 * torch.randn(3, 20, generator=g)),
            "planar": (planar, Rz @ planar + 1.0)}
    for name, (A, B) in sets.items():
        xa, yc = U.Kabsch(A, B)
        fx["kabsch"][name] = {"A": A, "B": B, "A_aligned": xa, "B_centred": yc}

    for n in NS:
        X, Y = pairs(3, n, g, 3.0)
        fx["scores"][n] = {"X": X, "Y": Y, "rmsd": U.RMSD(X, Y), "gdt_ts": U.GDT(X, Y), "gdt_ha": U.GDT(X, Y, mode="HA"),
                           "gdt_ts_w": U.GDT(X, Y, weights=[2, 1, 1, 1]), "gdt_ha_w": U.GDT(X, Y, mode="HA", weights=[2, 1, 1, 1]),
                           "tm": U.TMscore(X, Y)}
    X, Y = pairs(2, 40, g, 0.15)                         # nearly every point within 0.5 A: weighted HA above 1
    fx["close"] = {"X": X, "Y": Y, "gdt_ha_w": U.GDT(X, Y, mode="HA", weights=[2, 1, 1, 1])}
    for L in (30, 40):
        true, pred, mask = lddt_case(2, L, 14, g)
        fx["lddt"][L] = {"true": true, "pred": pred, "cloud_mask": mask, "lddt": U.lddt_ca_torch(true, pred, mask)}

    X, Y = torch.randn(30, 3, generator=g) * 4, torch.randn(30, 3, generator=g) * 4
    Xb, Yb = torch.randn(2, 30, 3, generator=g) * 4, torch.randn(2, 30, 3, generator=g) * 4
    Xm, Ym = torch.cdist(X, X), torch.cdist(Y, Y)
    bmask = torch.rand(30, 30, generator=g) > 0.3
    cases = {"coords": dict(X=X, Y=Y), "matrices": dict(X_mat=Xm, Y_mat=Ym), "coords_matrix": dict(X=X, Y_mat=Ym),
             "mask": dict(X=X, Y=Y, distmat_mask=bmask), "clamp": dict(X=X, Y=Y, clamp=(-2.0, 3.0)), "q1": dict(X=X, Y=Y, q=1),
             "batched": dict(X=Xb, Y=Yb), "batched_q3": dict(X=Xb, Y=Yb, q=3),
             "squeeze": dict(X=X[None], Y=Y[None])}
    for name, kw in cases.items():
        fx["loss"][name] = {"kwargs": kw, "loss": U.distmat_loss_torch(**kw)}
    path = os.path.join(OUT, "structure_metrics.pt")
    torch.save(fx, path)
    print(f"wrote structure_metrics ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
