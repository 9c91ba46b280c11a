"""CPU: the plain-torch geometry oracle (oracle/geometry_oracle.py) against the unmodified reference's utils.py outputs recorded in
tests/golden/geometry_mds.pt (oracle/make_golden_r9.py): distogram centring in every mode, including the NaN of a pair whose bins
sum to 0, and MDScaling (unweighted, weighted, eigen, mirror fix) from the same seeded svd_lowrank init."""
import pytest
import torch

from oracle import geometry_oracle as G


@pytest.fixture(scope="module")
def fx(golden):
    return golden("geometry_mds")


def test_center_distogram_matches_reference(fx):
    for name, case in fx["center"].items():
        dg = case["distogram"]
        for (center, wide), (rc, rw) in case["out"].items():
            for dtype in (torch.float32, torch.float64):
                c, w = G.center_distogram(dg.to(dtype), center=center, wide=wide)
                assert c.shape == rc.shape and w.shape == rw.shape, (name, center, wide)
                assert torch.equal(torch.isnan(c), torch.isnan(rc)), (name, center, wide, "central NaN pattern")
                assert torch.equal(torch.isnan(w), torch.isnan(rw)), (name, center, wide, "weights NaN pattern")
                torch.testing.assert_close(c.float(), rc, rtol=1e-5, atol=1e-5, equal_nan=True)
                torch.testing.assert_close(w.float(), rw, rtol=1e-5, atol=1e-6, equal_nan=True)


def test_center_distogram_quirks(fx):
    """the zero-magnitude pair: NaN central and weight under the mean; the median puts it in bin 0 (centre 1.5, weight 1 with no
    dispersion); the diagonal is zero except where NaN"""
    case = fx["center"]["b2_n13"]
    rc, rw = case["out"][("mean", "std")]
    assert torch.isnan(rc[0, 1, 4]) and torch.isnan(rw[0, 1, 4])
    assert torch.isnan(rw[1, 12, 12]), "a NaN weight survives the diagonal's *= 0"
    mc, mw = case["out"][("median", "none")]
    assert mc[0, 1, 4] == 1.5 and mw[0, 1, 4] == 1.0
    d = torch.arange(13)
    assert (mc[:, d, d] == 0).all() and (mw[:, d, d] == 0).all()
    assert (G.bin_centres(G.DISTANCE_THRESHOLDS)[1:-1] == G.DISTANCE_THRESHOLDS[1:-1] - 0.25).all()


@pytest.mark.parametrize("name", ["unweighted", "unweighted_10", "weighted", "eigen", "mirror", "mirror_weighted"])
def test_mdscaling_matches_reference(fx, name):
    case = fx["mds"][name]
    kw, inp = case["kwargs"], case["inputs"]
    torch.manual_seed(case["seed"])
    out = G.mdscaling(inp["pre"], inp.get("weights"), kw["iters"], kw["tol"], kw["fix_mirror"], kw.get("N_mask"), kw.get("CA_mask"),
                      kw.get("C_mask"), kw.get("eigen", False))
    assert out["his"].shape == case["his"].shape, (name, out["steps"], case["his"].shape[0] - 1)
    torch.testing.assert_close(out["his"], case["his"], rtol=2e-4, atol=1e-5)
    scale = case["coords"].abs().max().item()
    torch.testing.assert_close(out["coords"], case["coords"], rtol=0, atol=2e-4 * scale)


def test_mds_init_draws_the_reference_init(fx):
    """eigen=True returns the init itself: the oracle's svd_lowrank lines reproduce it bitwise under the same seed"""
    case = fx["mds"]["eigen"]
    torch.manual_seed(case["seed"])
    x = G.mds_init(case["inputs"]["pre"])
    assert torch.equal(x.transpose(-1, -2), case["coords"])


def test_mirror_fix_and_stop_rule_in_fixture(fx):
    """the weighted loop stops at step 1 (the reference's unweighted update with realistic weights); after the mirror fix every
    element has at least half its phi angles negative; an unweighted chain runs many iterations"""
    assert fx["mds"]["weighted"]["his"].shape[0] == 2
    assert fx["mds"]["unweighted"]["his"].shape[0] > 20
    masker = torch.arange(30) % 3
    for name in ("mirror", "mirror_weighted"):
        ratio = G.phi_ratio(fx["mds"][name]["coords"], masker == 0, masker == 1)
        assert (ratio >= 0.5).all(), (name, ratio)
