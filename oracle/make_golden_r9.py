"""TEST INFRASTRUCTURE ONLY -- round-9 fixture from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r9
  tests/golden/geometry_mds.pt  alphafold2_pytorch/utils.py run on the CPU in fp32:
    center    center_distogram_torch for center in (mean, median) x wide in (std, var, none) on three distograms: b 1 N 9,
              b 2 N 13 and b 1 N 30 (above cdist's 25-point switch), each with one pair whose bins sum to 0 (the NaN quirk)
    mds       MDScaling under torch.manual_seed(seed) right before the call (the svd_lowrank init draws from it):
              unweighted on quantised chain distances (runs many iterations), weighted from a centred distogram (stops at
              step 1), eigen=True, and fix_mirror with 3-point-per-residue N / CA masks.
  Inputs are built from ideal backbones (oracle.geometry_oracle.backbone), so distances are chain-like.  Under 500 KB."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402
from oracle import geometry_oracle as G  # noqa: E402

CENTERS = ("mean", "median")
WIDES = ("std", "var", "none")


def distogram_of(d, g, sharp=1.0):
    """A distogram [..., 37] peaked at the bin centres nearest the distances d, with noise: softmax of -sharp (d - c)^2 + noise."""
    c = G.bin_centres(G.DISTANCE_THRESHOLDS)
    logits = -sharp * (d[..., None] - c) ** 2 + 0.5 * torch.randn(*d.shape, c.shape[0], generator=g)
    return logits.softmax(-1)


def chain_distances(b, n_res, g, jitter=25.0):
    xs = torch.stack([G.backbone(n_res, generator=g, jitter=jitter) for _ in range(b)], 0)
    return xs, torch.cdist(xs, xs)


def main():
    load_reference()
    import alphafold2_pytorch.utils as U
    g = torch.Generator().manual_seed(9)
    fx = {"center": {}, "mds": {}}
    for name, (b, n) in {"b1_n9": (1, 9), "b2_n13": (2, 13), "b1_n30": (1, 30)}.items():
        _, d = chain_distances(b, max(n // 3, 2) + 1, g)
        dg = distogram_of(d[:, :n, :n], g)
        dg[0, 1, 4] = 0.0                                # a pair whose bins sum to 0
        dg[-1, n - 1, n - 1] = 0.0                        # and one on the diagonal
        outs = {}
        for center in CENTERS:
            for wide in WIDES:
                central, weights = U.center_distogram_torch(dg, center=center, wide=wide)
                outs[(center, wide)] = (central, weights)
        fx["center"][name] = {"distogram": dg, "out": outs}

    # MDS: 10 residues = 30 points (cdist's matmul form), batch 2
    xs, d = chain_distances(2, 10, g)
    quant = (d * 2).round() / 2 + 0.3 * (1 - torch.eye(30))          # non-Euclidean: many SMACOF iterations
    central, weights = U.center_distogram_torch(distogram_of(d, g, sharp=2.0))
    masker = torch.arange(30) % 3
    N_mask, CA_mask = masker == 0, masker == 1
    cases = {
        "unweighted": (dict(pre=quant), dict(iters=300, tol=1e-5, fix_mirror=False)),
        "unweighted_10": (dict(pre=quant), dict(iters=10, tol=1e-5, fix_mirror=False)),
        "weighted": (dict(pre=central, weights=weights), dict(iters=50, tol=1e-5, fix_mirror=False)),
        "eigen": (dict(pre=d), dict(iters=10, tol=1e-5, fix_mirror=False, eigen=True)),
        "mirror": (dict(pre=quant), dict(iters=20, tol=1e-5, fix_mirror=True, N_mask=N_mask, CA_mask=CA_mask, C_mask=None)),
        "mirror_weighted": (dict(pre=central, weights=weights),
                            dict(iters=20, tol=1e-5, fix_mirror=True, N_mask=N_mask, CA_mask=CA_mask, C_mask=None)),
    }
    for k, (name, (inp, kw)) in enumerate(cases.items()):
        seed = 100 + k
        torch.manual_seed(seed)
        coords, his = U.MDScaling(inp["pre"], weights=inp.get("weights"), verbose=0, **kw)
        fx["mds"][name] = {"inputs": inp, "kwargs": kw, "seed": seed, "coords": coords.clone(), "his": his.clone()}
        print(f"{name}: steps {his.shape[0] - 1}")
    fx["backbones"] = xs
    path = os.path.join(OUT, "geometry_mds.pt")
    torch.save(fx, path)
    print(f"wrote geometry_mds ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
