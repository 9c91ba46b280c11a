"""GPU: the structure scores (alphafold2_b200.utils, csrc/metrics.cuh) against the fp64 oracle (oracle/metrics_oracle.py) and
the reference's recorded outputs (tests/golden/structure_metrics.pt): exact lDDT counts and threshold decisions, the
rotation, score_coords as the composition of the mirrors, degenerate inputs, reproducibility, launch counts, memory, shapes
past 2^31 elements and the refusals."""
import pytest
import torch

import alphafold2_b200 as A
from alphafold2_b200 import _lib, ops
from alphafold2_b200 import utils as U
from oracle import metrics_oracle as M

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _launches():
    return _lib.load().af2_launch_count()


def close(a, ref, rtol=1e-6):
    ref = ref.double().cpu()
    scale = ref.abs().nan_to_num().max().item() if ref.numel() else 0.0
    torch.testing.assert_close(a.double().cpu(), ref, rtol=rtol, atol=rtol * max(scale, 1e-30), equal_nan=True)


def _structures(b, n, seed, noise=1.5):
    """a chain-like true structure and a rotated, shifted, noisy prediction, [b, n, 3] fp32 (CPU)"""
    g = torch.Generator().manual_seed(seed)
    steps = torch.randn(b, n, 3, generator=g)
    true = torch.cumsum(3.8 * steps / steps.norm(dim=-1, keepdim=True), 1)
    q, _ = torch.linalg.qr(torch.randn(b, 3, 3, generator=g))
    pred = (true + noise * torch.randn(b, n, 3, generator=g)) @ q + 5.0
    return pred.float(), true.float()


def _kernel_rotation(pred, true, mask):
    b, n, _ = pred.shape
    rot = torch.empty(b, 3, 3, dtype=torch.float64, device=DEV)
    ops.superpose_scores(pred, true, b, n, mask=mask, mask_strides=(0, 0) if mask is None else mask.stride(), align=True,
                         rot=rot)
    return rot.cpu()


@pytest.mark.parametrize("n", [1, 2, 3, 17, 130, 1000])
@pytest.mark.parametrize("b", [1, 3])
@pytest.mark.parametrize("masked", [False, True])
def test_score_coords_against_fp64_oracle(n, b, masked):
    pred, true = _structures(b, n, seed=n * 7 + b)
    mask = None
    if masked:
        mask = torch.rand(b, n, generator=torch.Generator().manual_seed(n)) > 0.25
        mask[:, 0] = True
    out = U.score_coords(pred.to(DEV), true.to(DEV), None if mask is None else mask.to(DEV))
    ref = M.score_coords(pred, true, mask)
    # lDDT: exact counts give the exact fp32 ratio
    torch.testing.assert_close(out.lddt.cpu(), ref["lddt"], rtol=0, atol=0, equal_nan=True)
    close(out.lddt_mean, ref["lddt_mean"])
    rot = _kernel_rotation(pred.to(DEV), true.to(DEV), None if mask is None else mask.to(DEV))
    for e in range(b):
        R = rot[e]
        assert torch.allclose(R @ R.T, torch.eye(3, dtype=torch.float64), atol=1e-12) and abs(torch.det(R) - 1) < 1e-12
        S = ref["S"][e]
        separated = (S[0] > 0) and (S[2] / S[0] > 1e-3) and ((S[:2] - S[1:]).abs() >= 1e-3 * S[0]).all()
        if separated:
            assert (R - ref["U"][e]).abs().max() < 1e-9, (n, b, e)
        if ref["gdt_near"][e] == 0:
            close(out.gdt_ts[e], ref["gdt_ts"][e])
            close(out.gdt_ha[e], ref["gdt_ha"][e])
        # the aligned chain: unique when C has rank 2 or more; below that only the fitted points are determined
        sel = slice(None) if S[1] > 1e-3 * S[0] else (torch.ones(n, dtype=torch.bool) if mask is None else mask[e])
        close(out.aligned[e][sel], ref["aligned"][e][sel], 1e-6)
    close(out.rmsd, ref["rmsd"])
    close(out.tm_score, ref["tm_score"], 1e-5 if n <= 18 else 1e-6)


def test_score_coords_is_the_composition_of_the_mirrors():
    b, n = 3, 200
    pred, true = _structures(b, n, seed=5)
    mask = torch.rand(b, n, generator=torch.Generator().manual_seed(1)) > 0.3
    p, t, m = pred.to(DEV), true.to(DEV), mask.to(DEV)
    out = U.score_coords(p, t, m)
    for e in range(b):
        S = m[e]
        a, bb = U.Kabsch(p[e][S].T, t[e][S].T)
        assert torch.equal(out.rmsd[e:e + 1], U.RMSD(a, bb))
        assert torch.equal(out.gdt_ts[e:e + 1], U.GDT(a, bb))
        assert torch.equal(out.gdt_ha[e:e + 1], U.GDT(a, bb, mode="HA"))
        assert torch.equal(out.tm_score[e:e + 1], U.TMscore(a, bb))
        k = int(S.sum())
        tc = torch.zeros(1, k, 2, 3, device=DEV)
        pc = torch.zeros(1, k, 2, 3, device=DEV)
        tc[0, :, 1], pc[0, :, 1] = t[e][S], p[e][S]
        l = U.lddt_ca_torch(tc, pc, torch.ones(1, k, 2, dtype=torch.bool, device=DEV))
        torch.testing.assert_close(out.lddt[e][S], l[0], rtol=0, atol=0, equal_nan=True)
        assert (out.lddt[e][~S] == 0).all()
        # aligned: the fitted superposition applied to the whole chain, in the true frame
        moved = out.aligned[e][S] - t[e][S].mean(0)
        close(moved.T, a, 1e-5)


def test_grid_thresholds_inclusive_and_radius_strict():
    """distances and differences that hit 0.5, 1, 2, 4, 8 and r_0 = 15 exactly (all exact in fp32 and fp64)"""
    xs = torch.tensor([0.0, 0.5, 1.0, 2.0, 4.0, 8.0, 15.0, 16.0])
    n = xs.shape[0]
    true = torch.zeros(1, n, 2, 3)
    true[0, :, 1, 0] = xs
    pred = true.clone()
    pred[0, :, 1, 0] = xs * 2                                  # |d_pred - d_true| = |x_i - x_j| exactly
    cm = torch.ones(1, n, 2, dtype=torch.bool)
    l = U.lddt_ca_torch(true.to(DEV), pred.to(DEV), cm.to(DEV)).cpu()
    ref, cnt, scr = M.lddt_ca(true, pred, cm)
    torch.testing.assert_close(l, ref, rtol=0, atol=0, equal_nan=True)
    assert cnt[0, 0] == 6, "itself, 0.5, 1, 2, 4 and 8: d_true = 15 is outside r_0 (strict)"
    # residue 0 against 0.5, 1, 2, 4, 8: |d_pred - d_true| = d_true, each threshold counted when equal (inclusive)
    assert scr[0, 0] == 4 + 4 + 3 + 2 + 1 + 0
    # GDT: distances 0.5, 1, 2, 4, 8 exactly on the cutoffs count
    X = torch.zeros(1, 3, 6)
    Y = torch.zeros(1, 3, 6)
    Y[0, 0] = torch.tensor([0.5, 1.0, 2.0, 4.0, 8.0, 8.5])
    for k, c in enumerate((0.5, 1, 2, 4, 8)):
        g = U.gdt_torch(X.to(DEV), Y.to(DEV), [c]).cpu()
        assert torch.equal(g, torch.tensor([k + 1], dtype=torch.float32) / 6), (c, g)


@pytest.fixture(scope="module")
def fx(golden):
    return golden("structure_metrics")


def test_against_reference_fixture(fx):
    for name, case in fx["kabsch"].items():
        xa, yc = U.Kabsch(case["A"].to(DEV), case["B"].to(DEV))
        close(xa, case["A_aligned"], 1e-5)
        close(yc, case["B_centred"], 1e-6)
        xa2, _ = U.kabsch_torch(case["A"].to(DEV), case["B"].to(DEV), cpu=True)
        assert torch.equal(xa, xa2)
    for n, case in fx["scores"].items():
        X, Y = case["X"].to(DEV), case["Y"].to(DEV)
        close(U.RMSD(X, Y), case["rmsd"])
        close(U.TMscore(X, Y), case["tm"])
        for key, kw in (("gdt_ts", {}), ("gdt_ha", {"mode": "HA"}), ("gdt_ts_w", {"weights": [2, 1, 1, 1]}),
                        ("gdt_ha_w", {"mode": "ha", "weights": [2, 1, 1, 1]})):
            g = U.GDT(X, Y, **kw)
            assert g.dtype == torch.float32 and g.shape == (3,)
            close(g, case[key])
        assert torch.equal(U.GDT(X, Y, cutoffs=[3, 5, 7, 9]), U.GDT(X, Y)), "GDT's cutoffs argument is ignored"
    c = fx["close"]
    w = U.GDT(c["X"].to(DEV), c["Y"].to(DEV), mode="HA", weights=[2, 1, 1, 1])
    close(w, c["gdt_ha_w"])
    assert w.max() > 1.0
    for L, case in fx["lddt"].items():
        l = U.lddt_ca_torch(case["true"].to(DEV), case["pred"].to(DEV), case["cloud_mask"].to(DEV))
        torch.testing.assert_close(l.cpu(), case["lddt"], rtol=0, atol=0, equal_nan=True)
        assert l[1, 5] == 0 and torch.isnan(l[0, L - 1])
    for name, case in fx["loss"].items():
        kw = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in case["kwargs"].items()}
        close(U.distmat_loss_torch(**kw), case["loss"], 1e-5)


def test_rmsd_divides_by_3n_and_tm_d0():
    X = torch.zeros(2, 3, 16, device=DEV)
    Y = torch.zeros(2, 3, 16, device=DEV)
    Y[:, 0] = 3.0
    assert torch.allclose(U.RMSD(X, Y).cpu(), torch.full((2,), 3.0 / 3 ** 0.5))
    for n in (10, 15, 16, 18, 19, 40):
        X, Y = torch.randn(2, 3, n), torch.randn(2, 3, n)
        close(U.TMscore(X.to(DEV), Y.to(DEV)), M.tmscore(X, Y), 1e-5)
        close(U.tmscore_torch(X.to(DEV), Y.to(DEV)), M.tmscore(X, Y), 1e-5)
    X64 = torch.randn(2, 3, 20, dtype=torch.float64, device=DEV)
    assert U.rmsd_torch(X64, X64 + 1).dtype == torch.float64 and U.gdt_torch(X64, X64, [1]).dtype == torch.float32


def test_degenerate_inputs():
    # N = 1 and N = 2: the rotation is a proper rotation, the scores are finite; identical points: RMSD 0
    for n in (1, 2):
        pred, true = _structures(2, n, seed=n)
        out = U.score_coords(pred.to(DEV), true.to(DEV))
        assert torch.isfinite(out.rmsd).all() and torch.isfinite(out.aligned).all()
        ref = M.score_coords(pred, true)
        close(out.rmsd, ref["rmsd"], 1e-5)
    line = torch.zeros(1, 12, 3)
    line[0, :, 0] = torch.arange(12.0)
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(0)))
    out = U.score_coords((line @ q).to(DEV), line.to(DEV))
    assert out.rmsd.item() < 1e-5, "collinear points superpose exactly"
    same = torch.randn(1, 7, 3)
    same[:] = same[0, 0]
    out = U.score_coords(same.to(DEV), same.to(DEV))
    assert out.rmsd.item() == 0.0 and out.gdt_ts.item() == 1.0
    # an element with no selected residue: NaN; the other element is unaffected
    pred, true = _structures(2, 30, seed=3)
    mask = torch.ones(2, 30, dtype=torch.bool)
    mask[1] = False
    out = U.score_coords(pred.to(DEV), true.to(DEV), mask.to(DEV))
    for v in (out.rmsd, out.gdt_ts, out.gdt_ha, out.tm_score, out.lddt_mean):
        assert torch.isnan(v[1]) and torch.isfinite(v[0])
    assert (out.lddt[1] == 0).all() and torch.isnan(out.aligned[1]).all()
    # NaN coordinates propagate into the scores
    bad = pred.clone()
    bad[0, 4, 1] = float("nan")
    out = U.score_coords(bad.to(DEV), true.to(DEV))
    assert torch.isnan(out.rmsd[0]) and torch.isfinite(out.rmsd[1])


def test_reproducible_and_launch_counts():
    pred, true = (t.to(DEV) for t in _structures(4, 700, seed=9))
    mask = (torch.rand(4, 700, device=DEV) > 0.2)
    cm = torch.ones(4, 700, 3, dtype=torch.bool, device=DEV)
    tc = torch.stack([true, true, true], 2)
    pc = torch.stack([pred, pred, pred], 2)
    runs = [
        (lambda: U.score_coords(pred, true, mask), 3),
        (lambda: U.lddt_ca_torch(tc, pc, cm), 2),
        (lambda: U.distmat_loss_torch(X=pred, Y=true), 2),
        (lambda: U.distmat_loss_torch(X=pred, Y=true, distmat_mask=torch.ones(4, 700, 700, dtype=torch.bool, device=DEV)), 2),
        (lambda: U.RMSD(pred.transpose(1, 2), true.transpose(1, 2)), 1),
        (lambda: U.GDT(pred.transpose(1, 2), true.transpose(1, 2)), 1),
        (lambda: U.TMscore(pred.transpose(1, 2), true.transpose(1, 2)), 1),
        (lambda: U.Kabsch(pred[0].T, true[0].T), 1),
    ]
    for fn, budget in runs:
        n0 = _launches()
        a = fn()
        used = _launches() - n0
        assert used <= budget, (used, budget)
        b = fn()
        for x, y in zip(_tensors(a), _tensors(b)):
            assert torch.equal(x.nan_to_num(), y.nan_to_num()) and torch.equal(torch.isnan(x), torch.isnan(y))


def _tensors(v):
    if isinstance(v, tuple):
        return list(v)
    if isinstance(v, U.StructureScores):
        return list(vars(v).values())
    return [v]


def test_distmat_loss_operands_masks_and_q():
    g = torch.Generator().manual_seed(2)
    X, Y = torch.randn(2, 300, 3, generator=g) * 5, torch.randn(2, 300, 3, generator=g) * 5
    Xm = M.dist(X[:, :, None], X[:, None]).float()
    mask = torch.rand(2, 300, 300, generator=g) > 0.5
    cases = [dict(X=X, Y=Y), dict(X_mat=Xm, Y=Y), dict(X=X, Y_mat=Xm), dict(X_mat=Xm, Y_mat=Xm[:1]), dict(X=X, Y=Y, q=1),
             dict(X=X, Y=Y, q=3), dict(X=X, Y=Y, clamp=(-3.0, 4.0)), dict(X=X, Y=Y, distmat_mask=mask),
             dict(X=X[:1], Y=Y[0]), dict(X=X[0], Y=Y[0], distmat_mask=mask[0])]
    for kw in cases:
        dev = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
        close(U.distmat_loss_torch(**dev), M.distmat_loss(**kw), 1e-6)
    empty = torch.zeros(300, 300, dtype=torch.bool, device=DEV)
    assert torch.isnan(U.distmat_loss_torch(X=X[0].to(DEV), Y=Y[0].to(DEV), distmat_mask=empty))


def test_memory_at_n_8192():
    pred, true = (t.to(DEV) for t in _structures(1, 8192, seed=4))
    mask = torch.ones(1, 8192, dtype=torch.bool, device=DEV)
    tc = torch.stack([true, true], 2)
    pc = torch.stack([pred, pred], 2)
    cm = torch.ones(1, 8192, 2, dtype=torch.bool, device=DEV)
    for fn in (lambda: U.score_coords(pred, true, mask), lambda: U.lddt_ca_torch(tc, pc, cm),
               lambda: U.distmat_loss_torch(X=pred, Y=true)):
        fn()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() - base < 16 * 2 ** 20


def test_large_loss_matrix_path_past_2_31():
    """b 2, N 33,000 stored matrices: 2.18e9 entries per operand; the oracle sums in row chunks on the device"""
    b, n = 2, 33000
    gen = torch.Generator(device=DEV).manual_seed(3)
    Xm = torch.empty(b, n, n, device=DEV)
    Ym = torch.empty(b, n, n, device=DEV)
    for e in range(b):
        Xm[e].uniform_(0, 30, generator=gen)
        Ym[e].uniform_(0, 30, generator=gen)
    got = U.distmat_loss_torch(X_mat=Xm, Y_mat=Ym)
    total = torch.zeros((), dtype=torch.float64, device=DEV)
    for e in range(b):
        for r in range(0, n, 2048):
            total += ((Xm[e, r:r + 2048].double() - Ym[e, r:r + 2048].double()) ** 2).sum()
    close(got, total / (b * n * n), 1e-6)


def test_large_lddt_against_device_oracle():
    n = 16384
    pred, true = (t.to(DEV) for t in _structures(1, n, seed=6, noise=1.0))
    present = torch.ones(1, n, dtype=torch.bool, device=DEV)
    present[0, ::97] = False
    cm = torch.stack([present, present], 2)
    l = U.lddt_ca_torch(torch.stack([true, true], 2), torch.stack([pred, pred], 2), cm)
    cnt, scr = M.lddt_counts(true, pred, present, chunk=512)
    torch.testing.assert_close(l, M.lddt_ratio(cnt, scr, present), rtol=0, atol=0, equal_nan=True)


def test_refusals_before_device_work():
    x = torch.randn(2, 3, 10, device=DEV)
    c = torch.randn(1, 10, 4, 3, device=DEV)
    cm = torch.ones(1, 10, 4, dtype=torch.bool, device=DEV)
    p, t = torch.randn(2, 10, 3, device=DEV), torch.randn(2, 10, 3, device=DEV)
    n0 = _launches()
    bad = [
        (RuntimeError, lambda: U.RMSD(x.cpu(), x.cpu())),
        (RuntimeError, lambda: U.score_coords(p.cpu(), t.cpu())),
        (RuntimeError, lambda: U.distmat_loss_torch(X=p[0].cpu(), Y=t[0].cpu())),
        (RuntimeError, lambda: U.RMSD(x.clone().requires_grad_(), x)),
        (ValueError, lambda: U.RMSD(x, x[:, :, :9])),
        (ValueError, lambda: U.RMSD(x, x[0])),
        (ValueError, lambda: U.Kabsch(x, x)),
        (ValueError, lambda: U.kabsch_torch(x[0], x[0, :, :5])),
        (ValueError, lambda: U.score_coords(p, t[:, :9])),
        (ValueError, lambda: U.score_coords(p, t, torch.ones(2, 9, dtype=torch.bool, device=DEV))),
        (ValueError, lambda: U.score_coords(p[:, :0], t[:, :0])),
        (ValueError, lambda: U.RMSD(x[:, :, :0], x[:, :, :0])),
        (ValueError, lambda: U.distmat_loss_torch(X=p[0], Y=t[0], distmat_mask=torch.ones(10, 10, device=DEV))),
        (ValueError, lambda: U.distmat_loss_torch(X=p[0], Y=t[0], distmat_mask=torch.ones(9, 10, dtype=torch.bool))),
        (ValueError, lambda: U.distmat_loss_torch(X=p[0], Y=t[0, :9])),
        (ValueError, lambda: U.distmat_loss_torch(X=p[0])),
        (ValueError, lambda: U.lddt_ca_torch(c[:, :, :1], c[:, :, :1], cm[:, :, :1])),
        (ValueError, lambda: U.lddt_ca_torch(c, c[:, :9], cm)),
        (ValueError, lambda: U.lddt_ca_torch(c, c, cm[:, :9])),
        (ValueError, lambda: U.GDT(x, x, weights=[1, 2, 3])),
        (ValueError, lambda: U.gdt_torch(x, x, [1] * 9)),
        (NotImplementedError, lambda: U.distmat_loss_torch(X=p[0], Y=t[0], p=1)),
        (NotImplementedError, lambda: U.distmat_loss_torch(X=p[0], Y=t[0], custom=lambda a, b: (a - b).abs())),
        (NotImplementedError, lambda: U.RMSD(x, x, backend="numpy")),
        (NotImplementedError, lambda: U.Kabsch(x[0].cpu().numpy(), x[0].cpu().numpy())),
    ]
    for exc, fn in bad:
        with pytest.raises(exc):
            fn()
    assert _launches() == n0
    assert A.utils.score_coords is U.score_coords
