"""TEST INFRASTRUCTURE ONLY -- round-12 fixture from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r12
  tests/golden/angle_dihedrals.pt  alphafold2_pytorch/utils.py's get_dihedral_torch (utils.py:881-898) in fp64 on the CPU:
    random    2000 quadruples of random points (scale 5), the general case
    planar    quadruples in the z = 0 plane: cis (dihedral 0), trans (+-pi, by the sign of the zero the formula makes) and
              the same configurations rotated in the plane, so the sign convention of theta and omega and the ends of their
              range are pinned
    chiral    one right-handed quadruple (dihedral +pi/2 up to rounding) and its mirror image (-pi/2)
  Each case holds the four point sets c1..c4 [M, 3] fp64 and the reference's dihedrals [M] fp64.  A data fixture only."""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402


def main():
    load_reference()
    import alphafold2_pytorch.utils as U

    g = torch.Generator().manual_seed(12)

    def case(c1, c2, c3, c4):
        return {"c": [c1, c2, c3, c4], "dihedral": U.get_dihedral_torch(c1, c2, c3, c4)}

    fx = {}
    fx["random"] = case(*(torch.randn(2000, 3, generator=g, dtype=torch.float64) * 5 for _ in range(4)))
    # planar: c2 -> c3 along a direction in the plane, c1 and c4 on the same side (cis) or opposite sides (trans)
    pts = []
    for k in range(24):
        a = 2 * math.pi * k / 24
        d = torch.tensor([math.cos(a), math.sin(a), 0.0], dtype=torch.float64)
        p = torch.tensor([-math.sin(a), math.cos(a), 0.0], dtype=torch.float64)
        c2 = torch.tensor([1.0 + k, -2.0, 0.0], dtype=torch.float64)
        c3 = c2 + 1.5 * d
        for side in (1.0, -1.0):
            pts.append((c2 + 0.7 * p - 0.3 * d, c2, c3, c3 + side * 1.2 * p + 0.4 * d))
    fx["planar"] = case(*(torch.stack([q[i] for q in pts]) for i in range(4)))
    c1 = torch.tensor([[1.0, 0.0, 0.0]], dtype=torch.float64)
    c2 = torch.zeros(1, 3, dtype=torch.float64)
    c3 = torch.tensor([[0.0, 0.0, 1.0]], dtype=torch.float64)
    c4 = torch.tensor([[0.0, 1.0, 1.0]], dtype=torch.float64)
    mirror = torch.tensor([-1.0, 1.0, 1.0], dtype=torch.float64)
    fx["chiral"] = case(torch.cat([c1, c1 * mirror]), torch.cat([c2, c2 * mirror]), torch.cat([c3, c3 * mirror]),
                        torch.cat([c4, c4 * mirror]))
    path = os.path.join(OUT, "angle_dihedrals.pt")
    torch.save(fx, path)
    print(f"wrote angle_dihedrals ({os.path.getsize(path)} bytes)")
    for k, v in fx.items():
        print(f"  {k}: {v['dihedral'].shape[0]} dihedrals, range [{v['dihedral'].min().item():.4f}, {v['dihedral'].max().item():.4f}]")


if __name__ == "__main__":
    main()
