"""CPU: the angle-loss oracle (oracle/angle_loss_oracle.py) against the unmodified reference's get_dihedral_torch recorded in
tests/golden/angle_dihedrals.pt (oracle/make_golden_r12.py), its invariances, and controls for the loss bound it borrows from
the distogram-loss oracle: an fp32 emulation of the kernel at its rounding points must pass it, and plausible wrong label
definitions and a log-sum-exp without the max must fail it."""
import math

import pytest
import torch

from oracle import angle_loss_oracle as O
from oracle.ref_loader import reference_available

NB = (O.THETA_BUCKETS, O.PHI_BUCKETS, O.OMEGA_BUCKETS)


@pytest.fixture(scope="module")
def fx(golden):
    return golden("angle_dihedrals")


def backbone(b, n, g, scale=6.0):
    """[b, n, 3, 3] N, CA, C: CA on a random walk of 3.8 A steps in a box, N and C at bond lengths in random directions"""
    step = torch.randn(b, n, 3, generator=g, dtype=torch.float64)
    ca = (step / step.norm(dim=-1, keepdim=True) * 3.8).cumsum(1) * 0.5 + torch.randn(b, n, 3, generator=g, dtype=torch.float64) * scale
    d = torch.randn(b, n, 2, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True)
    return torch.stack([ca + 1.46 * d[:, :, 0], ca, ca + 1.52 * d[:, :, 1]], 2).float()


@pytest.mark.parametrize("name", ["random", "planar", "chiral"])
def test_dihedral_matches_reference(fx, name):
    c = fx[name]
    d = O.dihedral(*c["c"])
    ref = c["dihedral"]
    assert (d - ref).abs().max().item() <= 64 * 2 ** -52 * math.pi
    assert torch.equal(torch.signbit(d), torch.signbit(ref))
    if name == "planar":                          # cis exactly 0, trans exactly +pi (the formula's zero is +0)
        assert torch.equal(d, ref)
        assert set(d.tolist()) == {0.0, math.pi}


def test_edges_and_ends():
    for nb in (2, 3, 13, 25, 101):
        for signed in (True, False):
            e = O.edges(nb, signed)
            assert e.shape == (nb - 1,) and e[-1].item() == math.pi and bool((e[1:] > e[:-1]).all())
    contact = torch.ones(4, dtype=torch.bool)
    v = torch.tensor([-math.pi, math.pi, 0.0, math.nextafter(-math.pi, 0)], dtype=torch.float64)
    assert O.bucket(v, contact, 25, True).tolist() == [0, 23, 11, 0]            # 0 is the edge of bin 11 at K = 24
    assert O.bucket(torch.tensor([0.0, math.pi], dtype=torch.float64), contact[:2], 13, False).tolist() == [0, 11]
    assert O.bucket(v, ~contact, 25, True).tolist() == [24] * 4


def test_labels_cover_every_bin_and_no_contact():
    g = torch.Generator().manual_seed(1)
    bb = backbone(2, 300, g)
    mask = torch.rand(2, 300, generator=g) > 0.1
    th, ph, om = O.labels(bb, mask, NB, -7)
    for lab, nb in zip((th, ph, om), NB):
        keep = lab != -7
        assert set(lab[keep].unique().tolist()) == set(range(nb)), "every bin and the no-contact bucket occur"
        assert bool((lab.diagonal(dim1=1, dim2=2)[mask] == nb - 1).all()), "the diagonal is no contact"
        assert bool((lab[~(mask[..., None] & mask[..., None, :])] == -7).all())
    assert bool(((th == 24) == (om == 24)).all() & ((th == 24) == (ph == 12)).all())


def test_nan_atoms_are_no_contact():
    g = torch.Generator().manual_seed(2)
    bb = backbone(1, 40, g)
    bb[0, 5, 2, 1] = float("nan")                 # C of residue 5: its virtual CB is NaN
    th, ph, om = O.labels(bb, None)
    for lab, nb in zip((th, ph, om), NB):
        assert bool((lab[0, 5] == nb - 1).all()) and bool((lab[0, :, 5] == nb - 1).all())


def _far_from_edges(v, contact, nb, signed, tol):
    e = O.edges(nb, signed)
    return ~contact | ((v[..., None] - e).abs().min(-1).values > tol)


def test_rigid_motion_changes_no_angle():
    g = torch.Generator().manual_seed(3)
    bb = backbone(1, 200, g)
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    moved = (bb.double() @ q.T + torch.tensor([5.0, -3.0, 12.0], dtype=torch.float64)).float()
    a0, a1 = O.angles(bb), O.angles(moved)
    c0 = a0[3]
    near20 = ((O.virtual_cb(bb)[0][:, None] - O.virtual_cb(bb)[0][None]).norm(dim=-1) - 20).abs() < 1e-3
    assert torch.equal(c0[0] & ~near20, a1[3][0] & ~near20)
    for k in range(3):                            # theta, phi, omega: fp32 re-rounding of the atoms only
        diff = (a0[k] - a1[k])[c0]
        diff = torch.remainder(diff + math.pi, 2 * math.pi) - math.pi
        assert diff.abs().max().item() < 1e-3
    lab0, lab1 = O.labels(bb, None), O.labels(moved, None)
    for k, (nb, signed) in enumerate(zip(NB, (True, False, True))):
        ok = _far_from_edges(a0[k], c0, nb, signed, 1e-3) & _far_from_edges(a1[k], a1[3], nb, signed, 1e-3) & ~near20
        assert ok.float().mean() > 0.9
        assert torch.equal(lab0[k][ok], lab1[k][ok])


def test_mirror_negates_theta_and_omega():
    g = torch.Generator().manual_seed(4)
    bb = backbone(2, 150, g)
    n, ca, cb = bb[:, :, 0].double(), bb[:, :, 1].double(), O.virtual_cb(bb)
    m = torch.tensor([1.0, -1.0, 1.0], dtype=torch.float64)
    th, ph, om, c = O.orientations(n, ca, cb)
    th2, ph2, om2, c2 = O.orientations(n * m, ca * m, cb * m)
    assert torch.equal(c, c2)
    assert torch.equal(th2, -th) and torch.equal(om2, -om) and torch.equal(ph2, ph)


def test_omega_is_symmetric():
    g = torch.Generator().manual_seed(5)
    bb = backbone(1, 180, g)
    _, _, om, c = O.angles(bb)
    assert torch.equal(c, c.transpose(1, 2))
    assert (om - om.transpose(1, 2))[c].abs().max().item() <= 1e-12


# ---- the loss bound's controls: the kernel's fp32 arithmetic passes it, wrong label definitions fail it ----
def _wrong_labels(bb, mask, variant):
    if variant == "no_contact_first":
        return tuple(torch.where(t == nb - 1, 0, t + 1).masked_fill(t == -100, -100) for t, nb in zip(O.labels(bb, mask), NB))
    n, ca, cb = bb[:, :, 0].double(), bb[:, :, 1].double(), O.virtual_cb(bb)
    if variant == "ca_for_cb":
        th, ph, om, c = O.orientations(n, ca, ca + 1e-3 * (cb - ca))
    else:
        th, ph, om, c = O.orientations(n, ca, cb)
    if variant == "theta_swapped":
        th = th.transpose(1, 2)
    if variant == "dihedral_sign":
        th, om = -th, -om
    if variant == "diagonal_contact":
        c = c | torch.eye(c.shape[1], dtype=torch.bool)[None]
    out = (O.bucket(th, c, NB[0], True), O.bucket(ph, c, NB[1], False), O.bucket(om, c, NB[2], True))
    keep = mask[..., None] & mask[..., None, :]
    return tuple(t.masked_fill(~keep, -100) for t in out)


def _emulate(logits, lab, no_max=False):
    """the kernel's per-term fp32 arithmetic on the CPU, summed in fp64"""
    keep = lab != -100
    l, y = logits[keep], lab[keep]
    if no_max:
        t = torch.log(torch.exp(l).sum(-1)) - l.gather(-1, y[:, None])[:, 0]
    else:
        m = l.max(-1).values
        s = torch.zeros_like(m)
        for c in range(l.shape[-1]):
            s = s + torch.exp(l[:, c] - m)
        t = (m + torch.log(s)) - l.gather(-1, y[:, None])[:, 0]
    return (t.double().sum() / t.numel()).item()


@pytest.fixture(scope="module")
def scored():
    g = torch.Generator().manual_seed(6)
    b, n = 2, 90
    bb = backbone(b, n, g, scale=3.0)
    mask = torch.rand(b, n, generator=g) > 0.1
    lab = O.labels(bb, mask)
    # logits that favour the true labels, as a trained head's would: a wrong label costs far more than rounding
    logits = []
    for t, nb in zip(lab, NB):
        l = torch.randn(b, n, n, nb, generator=g)
        l.scatter_add_(-1, t.clamp(min=0)[..., None], torch.full((b, n, n, 1), 6.0))
        logits.append(l * 16.0)                   # past 88 in exp: overflows without the max
    return bb, mask, lab, logits


def test_kernel_emulation_passes_the_bound(scored):
    _, _, lab, logits = scored
    for l, t in zip(logits, lab):
        err = abs(_emulate(l, t) - O.loss64(l, t).item())
        assert err <= O.loss_bound(l, t), err


@pytest.mark.parametrize("variant", ["no_contact_first", "ca_for_cb", "theta_swapped", "dihedral_sign", "diagonal_contact", "no_max"])
def test_wrong_variants_fail_the_bound(scored, variant):
    bb, mask, lab, logits = scored
    wrong = lab if variant == "no_max" else _wrong_labels(bb, mask, variant)
    failed = []
    for l, t, w in zip(logits, lab, wrong):
        got = _emulate(l, w, no_max=variant == "no_max") if not torch.equal(t, w) or variant == "no_max" else None
        if got is not None:
            ref = O.loss64(l, t).item()
            failed.append(not abs(got - ref) <= O.loss_bound(l, t))
    assert failed and any(failed), f"{variant} passes the bound on every head"


@pytest.mark.skipif(not reference_available(), reason="the reference checkout is not present")
def test_oracle_vs_live_reference():
    """the unmodified reference's get_dihedral_torch on fresh points, fp64"""
    from oracle.ref_loader import load_reference
    load_reference()
    import alphafold2_pytorch.utils as U
    g = torch.Generator().manual_seed(7)
    c = [torch.randn(500, 3, generator=g, dtype=torch.float64) * 3 for _ in range(4)]
    ref = U.get_dihedral_torch(*c)
    assert (O.dihedral(*c) - ref).abs().max().item() <= 64 * 2 ** -52 * math.pi
