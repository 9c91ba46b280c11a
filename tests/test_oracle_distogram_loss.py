"""CPU: the distogram-loss oracle (oracle/distogram_loss_oracle.py) against the unmodified reference's
get_bucketed_distance_matrix and train_pre.py loss lines recorded in tests/golden/distogram_loss.pt (oracle/make_golden_r11.py),
the exact fp32 fma emulation the labels rest on, and controls for the loss bound (oracle.term_bound / loss_bound): an
emulation of the kernel at its fp32 rounding points must pass it, and plausible wrong variants must fail it.

A variant that swaps the IEEE expf for the MUFU ex2.approx form is not among them: its error is of the order of the rounding
of l - max, which the bound already allows for, so no bound derived from the rounding points can tell the two apart."""
import math
import struct

import pytest
import torch

from oracle import distogram_loss_oracle as O
from oracle.ref_loader import reference_available

CASES = ["small", "small_ignore3", "edges16", "masked", "large", "large16"]


@pytest.fixture(scope="module")
def fx(golden):
    return golden("distogram_loss")


@pytest.mark.parametrize("name", CASES)
def test_oracle_labels_and_loss_match_reference(fx, name):
    c = fx[name]
    lab = O.labels(c["coords"], c["mask"], c["nb"], c["ignore_index"])
    assert torch.equal(lab, c["labels"])
    ref = c["loss"].double().item()
    assert abs(O.loss64(c["logits"], lab, c["ignore_index"]).item() - ref) <= 64 * 2 ** -24 * abs(ref)


def test_fixture_covers_the_quirks(fx):
    s = fx["small"]
    nb = s["nb"]
    edges = O.boundaries(nb)
    d = O.direct_dist32(s["coords"])
    on_edge = (d[..., None] == edges[:-1]).any(-1) & (s["labels"] != -100)
    assert on_edge.sum() >= 20, "distances exactly on an edge"
    # a distance on an edge goes below it: label k for d == edges[k]
    k = (d[..., None] == edges[:-1]).float().argmax(-1)
    assert torch.equal(s["labels"][on_edge], k[on_edge])
    assert (s["labels"][1, 3][s["mask"][1]] == nb - 1).all(), "a NaN coordinate goes to the last bucket"
    assert (fx["small_ignore3"]["labels"] == 3).sum() > 0 and (fx["small"]["labels"] == 3).sum() > 0
    assert not fx["masked"]["mask"][1].any()
    assert fx["large"]["coords"].shape[1] > 25 and fx["large16"]["coords"].shape[1] > 25
    edges16 = O.boundaries(16)[:15]
    assert torch.equal(O.direct_dist32(fx["edges16"]["coords"])[:, 0, 1:16], edges16.expand(2, 15))


def test_fmaf32_is_one_rounding():
    """against math.fsum-exact rounding on random operands, and on constructed midpoints where double rounding would fail"""
    g = torch.Generator().manual_seed(3)
    a, b, c = (torch.randn(4000, generator=g) * s for s in (1.0, 3.0, 100.0))
    # midpoints: c with a low bit pattern such that a*b + c sits exactly between two fp32 values before the tail of a*b
    a2 = torch.tensor([1.0 + 2 ** -12, 1.0 + 2 ** -23], dtype=torch.float32)
    c2 = torch.tensor([2.0 ** 25, -1.0], dtype=torch.float32)
    a, b, c = torch.cat([a, a2]), torch.cat([b, a2]), torch.cat([c, c2])
    got = O.fmaf32(a, b, c)

    def exact(x, y, z):
        from fractions import Fraction
        v = Fraction(x) * Fraction(y) + Fraction(z)
        f = struct.unpack("f", struct.pack("f", float(v)))[0]       # nearest fp64, then fp32: fix the double rounding
        lo, hi = sorted((f, math.nextafter(f, math.inf if Fraction(f) < v else -math.inf)))
        lo = struct.unpack("f", struct.pack("f", lo))[0]
        cand = [lo, struct.unpack("f", struct.pack("f", hi))[0], f]
        return min(cand, key=lambda t: (abs(Fraction(t) - v), struct.unpack("I", struct.pack("f", t))[0] & 1))

    for i in range(0, len(a), 97):
        assert got[i].item() == exact(a[i].item(), b[i].item(), c[i].item()), i
    for i in range(len(a) - 2, len(a)):
        assert got[i].item() == exact(a[i].item(), b[i].item(), c[i].item()), i


def _emulate(logits, lab, ii, variant=None):
    """The kernel's per-term arithmetic in fp32 on the CPU, summed in fp64; variants are plausible mistakes."""
    keep = lab != ii
    if variant == "masked_counted":
        keep = torch.ones_like(keep)
        lab = lab.clamp(0, logits.shape[-1] - 1)
    if variant == "no_diagonal":
        keep = keep & ~torch.eye(lab.shape[1], dtype=torch.bool)[None]
    l = logits[keep]
    y = lab[keep]
    if variant == "label_plus_one":
        y = (y + 1).clamp(max=logits.shape[-1] - 1)
    m = l.max(-1).values
    if variant == "no_max":
        s = torch.exp(l).sum(-1)
        t = torch.log(s) - l.gather(-1, y[:, None])[:, 0]
    else:
        s = torch.zeros_like(m)
        for c in range(l.shape[-1]):
            s = s + torch.exp(l[:, c] - m)
        t = (m + torch.log(s)) - l.gather(-1, y[:, None])[:, 0]
    return (t.double().sum() / t.numel()).float()


@pytest.mark.parametrize("name", ["small", "edges16", "large16"])
@pytest.mark.parametrize("variant", [None, "label_plus_one", "no_diagonal", "masked_counted", "no_max"])
def test_loss_bound_controls(fx, name, variant):
    c = fx[name]
    logits = c["logits"] * (40.0 if variant in (None, "no_max") else 1.0)   # logits past 88: exp overflows without the max
    lab = O.labels(c["coords"], c["mask"], c["nb"], c["ignore_index"])
    ref = O.loss64(logits, lab, c["ignore_index"]).item()
    bound = O.loss_bound(logits, lab, c["ignore_index"])
    err = abs(_emulate(logits, lab, c["ignore_index"], variant).double().item() - ref)
    if variant is None:
        assert err <= bound, (err, bound)
    else:
        assert not err <= bound, f"{variant}: err {err} within the bound {bound}"


@pytest.mark.skipif(not reference_available(), reason="the reference checkout is not present")
def test_oracle_vs_live_reference():
    """the unmodified reference on fresh seeded inputs (the direct cdist range, N <= 25)"""
    from oracle.ref_loader import load_reference
    load_reference()
    import torch.nn.functional as F
    import alphafold2_pytorch.utils as U
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 16, 3, generator=g) * 4
    x[0, :8] = 0.0
    x[0, :8, 2] = torch.arange(8, dtype=torch.float32)
    mask = torch.rand(2, 16, generator=g) > 0.2
    logits = torch.randn(2, 16, 16, 37, generator=g)
    lab = U.get_bucketed_distance_matrix(x, mask, 37, -100)
    assert torch.equal(O.labels(x, mask, 37, -100), lab)
    ref = F.cross_entropy(logits.permute(0, 3, 1, 2), lab, ignore_index=-100).double().item()
    assert abs(O.loss64(logits, lab).item() - ref) <= 64 * 2 ** -24 * abs(ref)
