"""TEST INFRASTRUCTURE ONLY -- plain-torch statement of the angle heads' labels (the trRosetta inter-residue orientations, Yang
et al., PNAS 2020, DESIGN.md §4f) and of each head's cross-entropy against them, on CPU or GPU tensors.

Geometry is fp64 on the fp32 atoms, one torch operation per rounding in the kernels' order (csrc/angle_loss.cuh), so the
products, sums and square roots are the kernels' bit for bit; only atan2 may differ by an ulp between libraries, which moves
a label only for an angle within an ulp of a bin edge.  The dihedral is the reference's get_dihedral_torch (utils.py:881-898)
with its dot products summed from +0 (as torch's sum is) x, y, then z and its norm as sqrt((x^2 + y^2) + z^2);
tests/golden/angle_dihedrals.pt pins it against the unmodified reference.

The loss per head is distogram_loss_oracle's: loss64 in fp64 on the fp32 logits, loss_bound from the kernels' rounding points.
It must never be imported by ``alphafold2_b200``."""
import math

import torch

from oracle import distogram_loss_oracle as D

THETA_BUCKETS, PHI_BUCKETS, OMEGA_BUCKETS = 25, 13, 25
CONTACT = 20.0
CB_A, CB_B, CB_C = -0.58273431, 0.56802827, 0.54067466


def _sub(a, b):
    return [x - y for x, y in zip(a, b)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    """summed from +0 as torch's .sum(dim=-1) is, x, y, then z: a dot product of zeros is +0, never -0"""
    return ((0.0 + a[0] * b[0]) + a[1] * b[1]) + a[2] * b[2]


def _norm(a):
    return _dot(a, a).sqrt()


def _split(p: torch.Tensor):
    """[..., 3] -> its three fp64 components"""
    p = p.double()
    return [p[..., 0], p[..., 1], p[..., 2]]


def virtual_cb(backbone: torch.Tensor) -> torch.Tensor:
    """[..., A, 3] (atoms N, CA, C first) -> the virtual CB [..., 3] fp64: ((-0.58273431 a + 0.56802827 b) - 0.54067466 c) + CA
    with b = CA - N, c = C - CA, a = b x c"""
    n, ca, c = (_split(backbone[..., k, :]) for k in range(3))
    b, cc = _sub(ca, n), _sub(c, ca)
    a = _cross(b, cc)
    return torch.stack([((CB_A * a[k] + CB_B * b[k]) - CB_C * cc[k]) + ca[k] for k in range(3)], -1)


def dihedral(c1, c2, c3, c4) -> torch.Tensor:
    """get_dihedral_torch on [..., 3] points in fp64: atan2(((|u2| u1) . (u2 x u3)), ((u1 x u2) . (u2 x u3)))"""
    c1, c2, c3, c4 = (_split(t) for t in (c1, c2, c3, c4))
    u1, u2, u3 = _sub(c2, c1), _sub(c3, c2), _sub(c4, c3)
    c23 = _cross(u2, u3)
    n2 = _norm(u2)
    return torch.atan2(_dot([n2 * u for u in u1], c23), _dot(_cross(u1, u2), c23))


def planar_angle(a, b, c) -> torch.Tensor:
    """the angle at b of a-b-c in fp64: atan2(|v x w|, v . w), v = a - b, w = c - b"""
    a, b, c = (_split(t) for t in (a, b, c))
    v, w = _sub(a, b), _sub(c, b)
    return torch.atan2(_norm(_cross(v, w)), _dot(v, w))


def orientations(n: torch.Tensor, ca: torch.Tensor, cb: torch.Tensor):
    """N, CA, CB [b, N, 3] -> (theta, phi, omega, contact), each [b, N, N]: the angles in fp64 for every pair (contacts or
    not) and the contact mask i != j, |CB_i - CB_j| <= 20"""
    nn_ = n.shape[1]
    I = lambda t: t[:, :, None, :].expand(-1, -1, nn_, -1)  # noqa: E731 - residue i along rows
    J = lambda t: t[:, None, :, :].expand(-1, nn_, -1, -1)  # noqa: E731 - residue j along columns
    theta = dihedral(I(n), I(ca), I(cb), J(cb))
    omega = dihedral(I(ca), I(cb), J(cb), J(ca))
    phi = planar_angle(I(ca), I(cb), J(cb))
    d = _norm(_sub(_split(J(cb)), _split(I(cb))))
    contact = (d <= CONTACT) & ~torch.eye(nn_, dtype=torch.bool, device=d.device)[None]
    return theta, phi, omega, contact


def angles(backbone: torch.Tensor):
    """backbone [b, N, A, 3] -> orientations of its N, CA and virtual CB"""
    return orientations(backbone[:, :, 0].double(), backbone[:, :, 1].double(), virtual_cb(backbone))


def edges(nb: int, signed: bool, device=None) -> torch.Tensor:
    """the K = nb - 1 bin edges in fp64: -pi + (k + 1) (2 pi / K) when signed (theta, omega), (k + 1) (pi / K) otherwise (phi);
    the last edge is pi"""
    K = nb - 1
    e = [(-math.pi + (k + 1) * (2 * math.pi / K)) if signed else (k + 1) * (math.pi / K) for k in range(K)]
    e[-1] = math.pi
    return torch.tensor(e, dtype=torch.float64, device=device)


def bucket(v: torch.Tensor, contact: torch.Tensor, nb: int, signed: bool) -> torch.Tensor:
    """the label of angles v: the number of edges below (torch.bucketize, right=False), nb - 1 where there is no contact"""
    lab = torch.bucketize(v.contiguous(), edges(nb, signed, v.device))
    return lab.masked_fill(~contact, nb - 1)


def labels(backbone: torch.Tensor, mask, nb=(THETA_BUCKETS, PHI_BUCKETS, OMEGA_BUCKETS), ignore_index: int = -100):
    """get_bucketed_angle_matrices: (theta, phi, omega) int64 [b, N, N]; ignore_index where either residue is masked"""
    theta, phi, omega, contact = angles(backbone)
    out = [bucket(theta, contact, nb[0], True), bucket(phi, contact, nb[1], False), bucket(omega, contact, nb[2], True)]
    if mask is not None:
        keep = mask[..., None] & mask[..., None, :]
        out = [t.masked_fill(~keep, ignore_index) for t in out]
    return tuple(out)


def loss64(logits: torch.Tensor, lab: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    """one head's F.cross_entropy in fp64 (distogram_loss_oracle.loss64)"""
    return D.loss64(logits, lab, ignore_index)


def loss_bound(logits: torch.Tensor, lab: torch.Tensor, ignore_index: int = -100) -> float:
    """one head's bound on |kernel loss - loss64| (distogram_loss_oracle.loss_bound: the kernels' term is the same)"""
    return D.loss_bound(logits, lab, ignore_index)
