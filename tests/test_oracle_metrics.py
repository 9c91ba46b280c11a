"""CPU: the plain-torch structure-score oracle (oracle/metrics_oracle.py) against the unmodified reference's utils.py outputs
recorded in tests/golden/structure_metrics.pt (oracle/make_golden_r10.py): Kabsch (generic, reflected, planar), RMSD, GDT TS
and HA with and without weights, TMscore at N 10 to 40, lddt_ca_torch and distmat_loss_torch, and the reference's quirks."""
import pytest
import torch

from oracle import metrics_oracle as M


@pytest.fixture(scope="module")
def fx(golden):
    return golden("structure_metrics")


def close(a, ref, rtol=1e-6):
    ref = ref.double()
    torch.testing.assert_close(a.double(), ref, rtol=rtol, atol=rtol * max(ref.abs().max().item(), 1e-30), equal_nan=True)


@pytest.mark.parametrize("name", ["generic", "reflected", "planar"])
def test_kabsch_matches_reference(fx, name):
    case = fx["kabsch"][name]
    xa, yc, U, _ = M.kabsch(case["A"], case["B"])
    close(xa, case["A_aligned"], 1e-5)
    close(yc, case["B_centred"])
    assert abs(torch.det(U).item() - 1.0) < 1e-12


def test_kabsch_determinant_fix(fx):
    """on the reflected set the fix is needed: the unfixed V W is a reflection, and the fixed one leaves an RMSD well above
    that of the generic set's noise"""
    case = fx["kabsch"]["reflected"]
    X, Y = case["A"].double(), case["B"].double()
    C = (X - X.mean(-1, keepdim=True)) @ (Y - Y.mean(-1, keepdim=True)).t()
    V, _, W = torch.linalg.svd(C)
    assert torch.det(V) * torch.det(W) < 0
    assert M.rmsd(case["A_aligned"][None], case["B_centred"][None]) > 1.0


@pytest.mark.parametrize("n", [10, 15, 16, 18, 19, 40])
def test_scores_match_reference(fx, n):
    case = fx["scores"][n]
    X, Y = case["X"], case["Y"]
    close(M.rmsd(X, Y), case["rmsd"])
    close(M.tmscore(X, Y), case["tm"])
    for key, cut, w in (("gdt_ts", M.GDT_TS, None), ("gdt_ha", M.GDT_HA, None), ("gdt_ts_w", M.GDT_TS, [2, 1, 1, 1]),
                        ("gdt_ha_w", M.GDT_HA, [2, 1, 1, 1])):
        g, counts = M.gdt(X, Y, cut, w)
        # the decisions: the reference's GDT_k are exact fractions of the counts
        wt = torch.tensor([1.0] * 4 if w is None else w, dtype=torch.float64)
        assert torch.equal(((counts.double() / n) * wt).mean(-1).float(), g.float())
        close(g, case[key])
        assert case[key].dtype == torch.float32


def test_score_quirks(fx):
    """TM d0 has no lower clamp (negative for N <= 18); weighted GDT is not normalised by the weights (can exceed 1)"""
    assert M.tm_d0(10) == M.tm_d0(15) == -1.8 and M.tm_d0(18) < 0 < M.tm_d0(19) < 0.2
    close_ = fx["close"]
    assert close_["gdt_ha_w"].max() > 1.0
    close(M.gdt(close_["X"], close_["Y"], M.GDT_HA, [2, 1, 1, 1])[0], close_["gdt_ha_w"])
    for n in (10, 15, 16, 18):
        X, Y = fx["scores"][n]["X"], fx["scores"][n]["Y"]
        d = M.point_dist(X, Y)
        d0 = M.tm_d0(n)
        close((1 / (1 + (d / d0) ** 2)).mean(-1), fx["scores"][n]["tm"])


@pytest.mark.parametrize("L", [30, 40])
def test_lddt_matches_reference(fx, L):
    case = fx["lddt"][L]
    ref = case["lddt"]
    l, cnt, scr = M.lddt_ca(case["true"], case["pred"], case["cloud_mask"])
    assert torch.equal(torch.isnan(l), torch.isnan(ref))
    torch.testing.assert_close(l, ref.float(), rtol=0, atol=0, equal_nan=True)   # exact counts, the same fp32 division
    assert ref[1, 5] == 0.0, "a residue without a CA scores 0"
    assert torch.isnan(ref[0, L - 1]) and cnt[0, L - 1] == 1, "a CA with no other CA within r_0 scores NaN"


@pytest.mark.parametrize("name", ["coords", "matrices", "coords_matrix", "mask", "clamp", "q1", "batched", "batched_q3",
                                  "squeeze"])
def test_distmat_loss_matches_reference(fx, name):
    case = fx["loss"][name]
    close(M.distmat_loss(**case["kwargs"]), case["loss"], 1e-5)


def test_loss_quirks(fx):
    """clamp acts on the coordinates; q = 1 is the mean absolute difference"""
    kw = fx["loss"]["clamp"]["kwargs"]
    X, Y = kw["X"].clamp(-2.0, 3.0), kw["Y"].clamp(-2.0, 3.0)
    close(M.distmat_loss(X=X, Y=Y), fx["loss"]["clamp"]["loss"], 1e-5)
    kw = fx["loss"]["q1"]["kwargs"]
    close((M.dist(kw["X"][:, None], kw["X"][None]) - M.dist(kw["Y"][:, None], kw["Y"][None])).abs().mean(),
          fx["loss"]["q1"]["loss"], 1e-5)
