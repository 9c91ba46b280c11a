"""TEST INFRASTRUCTURE ONLY -- plain-torch statement of the distogram-to-coordinates chain of alphafold2_pytorch/utils.py
(center_distogram_torch, mds_torch, mdscaling_torch and the phi mirror check), written from the reference's behaviour, in
any dtype.  Distances of the MDS loop are direct differences (the reference's torch.cdist takes its matmul form above 25
points; the two agree to rounding).  In fp32 under the same seed, mds_init draws exactly the reference's svd_lowrank init."""
import torch

DISTANCE_THRESHOLDS = torch.linspace(2, 20, steps=37)


def bin_centres(bins, dtype=torch.float32):
    """bins - half a bin width, first centre 1.5, last 1.33 * bins[-1] (computed in fp32 like the reference, then cast)."""
    c = bins.float() - 0.5 * (bins.float()[2] - bins.float()[1])
    c[0] = 1.5
    c[-1] = 1.33 * bins.float()[-1]
    return c.to(dtype)


def center_distogram(distogram, bins=DISTANCE_THRESHOLDS, center="mean", wide="std", softmax=False, mask=None, details=False,
                     row0=0):
    """-> (central, weights) [b, N, N] in distogram's dtype.  softmax: distogram holds logits.  mask [b, N]: pairs with a masked
    residue get weight 0 (coords_from_distogram).  details: also the median bin index and, per pair, the smallest
    |cumsum - half| over the bins relative to the total (a near-tie when tiny).  distogram may be the rows
    [row0, row0 + R) of a larger one, [b, R, N, bins] (without mask)."""
    p = distogram.softmax(-1) if softmax else distogram
    b, rows, n, nb = p.shape
    c = bin_centres(bins, p.dtype).to(p.device)
    mag = p.sum(-1)
    idx, margin = None, None
    if center == "median":
        cum = p.cumsum(-1)
        half = 0.5 * cum[..., -1:]
        idx = (cum < half).sum(-1).clamp(max=nb - 1)          # searchsorted side left, clamped to the last bin
        margin = ((cum - half).abs().min(-1).values / cum[..., -1].abs())
        central = c[idx]
    elif center == "mean":
        central = (p * c).sum(-1) / mag
    else:
        raise ValueError(center)
    keep = (central <= float(bins.float()[-2])).to(p.dtype)
    eye = (torch.arange(rows, device=p.device)[:, None] + row0) == torch.arange(n, device=p.device)[None, :]
    central = torch.where(eye, central * 0, central)           # *= 0: NaN stays NaN
    if wide in ("std", "var"):
        disp = (p * (c - central[..., None]) ** 2).sum(-1) / mag
        if wide == "std":
            disp = disp.sqrt()
    else:
        disp = torch.zeros_like(central)
    w = keep / (1 + disp)                                      # NaN stays NaN (the reference's w[w != w] *= 0)
    w = torch.where(eye, w * 0, w)
    if mask is not None:
        m = mask.bool()
        w = torch.where(m[:, :, None] & m[:, None, :], w, torch.zeros_like(w))
    if details:
        return central, w, idx, margin
    return central, w


def mds_init(pre):
    """u sqrt|s| of torch.svd_lowrank(M) per batch element, M = 0.5 (D[:, :1, :] + D[:, :, :1] - D), D = pre^2, first 3 columns
    (zero-padded below 3 points) -> [b, N, 3] in pre's dtype.  Draws from the RNG of pre's device, in the reference's order."""
    D = pre ** 2
    M = 0.5 * (D[:, :1, :] + D[:, :, :1] - D)
    outs = []
    for mi in M:
        u, s, _ = torch.svd_lowrank(mi)
        outs.append(u * s.abs().sqrt()[None, :])
    x = torch.stack(outs, 0)[..., :3]
    if x.shape[-1] < 3:
        x = torch.nn.functional.pad(x, (0, 3 - x.shape[-1]))
    return x


def mds(pre, weights=None, iters=10, tol=1e-5, eigen=False, init=None):
    """SMACOF as mds_torch runs it.  Returns dict(coords [b, 3, N], his [steps + 1, b], steps, stopped, stress [evaluated, b],
    vals [evaluated, b]); his[0] = inf.  The update is X <- (1 / N) B X even with weights; the loop stops at the first
    iteration with mean_b(his[-1] - stress / |X'|) <= tol and keeps the previous coords."""
    b, n, _ = pre.shape
    x = mds_init(pre) if init is None else init.to(pre.dtype)
    inf = torch.full((b,), float("inf"), dtype=pre.dtype, device=pre.device)
    empty = torch.zeros(0, b, dtype=pre.dtype, device=pre.device)
    if weights is None and eigen:
        return dict(coords=x.transpose(-1, -2), his=torch.zeros(1, b, dtype=pre.dtype, device=pre.device), steps=0, stopped=False,
                    stress=empty, vals=empty)
    w = torch.ones_like(pre) if weights is None else weights.to(pre.dtype)
    his, stresses, vals, stopped = [inf], [], [], False
    for _ in range(iters):
        diff = x[:, :, None, :] - x[:, None, :, :]
        dist = diff.pow(2).sum(-1).sqrt()
        stress = (w * (dist - pre) ** 2).sum(dim=(-1, -2)) * 0.5
        dist = torch.where(dist <= 0, dist + 1e-7, dist)
        r = w * (pre / dist)
        new = (r[..., None] * diff).sum(2) / n
        val = stress / new.pow(2).sum(dim=(-1, -2)).sqrt()
        stresses.append(stress)
        vals.append(val)
        if (his[-1] - val).mean() <= tol:
            stopped = True
            break
        x = new
        his.append(val)
    return dict(coords=x.transpose(-1, -2), his=torch.stack(his, 0), steps=len(his) - 1, stopped=stopped,
                stress=torch.stack(stresses, 0) if stresses else empty, vals=torch.stack(vals, 0) if vals else empty)


def dihedral(c1, c2, c3, c4):
    u1, u2, u3 = c2 - c1, c3 - c2, c4 - c3
    return torch.atan2((u2.norm(dim=-1, keepdim=True) * u1 * torch.cross(u2, u3, dim=-1)).sum(-1),
                       (torch.cross(u1, u2, dim=-1) * torch.cross(u2, u3, dim=-1)).sum(-1))


def phi_ratio(coords, N_mask, CA_mask, C_mask=None):
    """Fraction of negative backbone phi angles per element of coords [b, 3, N]; atoms picked by the [N] masks."""
    x = coords.transpose(-1, -2)
    N_mask, CA_mask = N_mask.bool(), CA_mask.bool()
    C_mask = ~(N_mask | CA_mask) if C_mask is None else C_mask.bool()
    n_t, ca_t, c_t = x[:, N_mask], x[:, CA_mask], x[:, C_mask]
    return (dihedral(c_t[:, :-1], n_t[:, 1:], ca_t[:, 1:], c_t[:, 1:]) < 0).to(coords.dtype).mean(-1)


def mdscaling(pre, weights=None, iters=10, tol=1e-5, fix_mirror=True, N_mask=None, CA_mask=None, C_mask=None, eigen=False,
              init=None):
    """mds, then with fix_mirror the z row negated where fewer than half the phi angles are negative; adds 'flipped' [b]."""
    out = mds(pre, weights, iters, tol, eigen, init)
    if fix_mirror:
        flip = phi_ratio(out["coords"], N_mask, CA_mask, C_mask) < 0.5
        c = out["coords"].clone()
        c[:, -1] = torch.where(flip[:, None], -c[:, -1], c[:, -1])
        out["coords"], out["flipped"] = c, flip
    return out


def backbone(n_res, generator=None, dtype=torch.float32, jitter=0.0):
    """An ideal-geometry backbone N, CA, C per residue (bond lengths 1.458 / 1.525 / 1.329 A, angles 111 / 117 / 122 deg) with
    helix-like torsions phi -60 and psi -45 (omega 180) plus optional jitter in degrees -> [3 n_res, 3].  Its phi angles are
    negative: the mirror image has them positive."""
    lengths = [1.458, 1.525, 1.329]                   # N-CA, CA-C, C-N
    angles = [121.7, 111.0, 117.2]                    # at N (C-N-CA), at CA (N-CA-C), at C (CA-C-N)
    torsions = [-60.0, -45.0, 180.0]                  # phi (C-N-CA-C), psi (N-CA-C-N), omega (CA-C-N-CA)
    pts = [torch.tensor([0.0, 0.0, 0.0], dtype=torch.float64), torch.tensor([1.458, 0.0, 0.0], dtype=torch.float64),
           torch.tensor([1.458 + 1.525 * 0.358, 1.525 * 0.934, 0.0], dtype=torch.float64)]
    for k in range(3, 3 * n_res):
        a, b, c = pts[-3], pts[-2], pts[-1]
        bond = lengths[(k - 1) % 3]
        ang = angles[(k - 1) % 3]
        tor = torsions[(k + 1) % 3]                   # atom k closes psi (N), omega (CA) or phi (C)
        if jitter:
            tor = tor + jitter * float(torch.randn((), generator=generator))
        ang_r, tor_r = torch.deg2rad(torch.tensor(ang, dtype=torch.float64)), torch.deg2rad(torch.tensor(tor, dtype=torch.float64))
        bc = (c - b) / (c - b).norm()
        nrm = torch.cross(b - a, bc, dim=0)
        nrm = nrm / nrm.norm()
        m = torch.stack([bc, torch.cross(nrm, bc, dim=0), nrm], 1)
        d2 = torch.stack([-bond * torch.cos(ang_r), bond * torch.sin(ang_r) * torch.cos(tor_r), bond * torch.sin(ang_r) * torch.sin(tor_r)])
        pts.append(c + m @ d2)
    return torch.stack(pts, 0).to(dtype)
