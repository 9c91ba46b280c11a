"""GPU: the distogram-to-coordinates chain (alphafold2_b200.utils, csrc/geometry.cuh) against the fp64 oracle
(oracle/geometry_oracle.py) and the reference's recorded outputs (tests/golden/geometry_mds.pt)."""
import pytest
import torch

import alphafold2_b200 as A
from alphafold2_b200 import _lib, ops
from alphafold2_b200 import utils as U
from oracle import geometry_oracle as G

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = [(c, w) for c in ("mean", "median") for w in ("std", "var", "none")]


def _launches():
    return _lib.load().af2_launch_count()


def _distogram(b, n, g, logits):
    x = torch.randn(b, n, n, 37, generator=g, dtype=torch.float64) * 3
    if logits:
        return x
    p = x.softmax(-1)
    if n > 1:
        p[0, 0, 1] = 0.0                                    # bins summing to 0: NaN under the mean
    p[-1, n - 1, n - 1] = 0.0
    return p


def _check_center(c, w, dg, center, wide, logits, row0=0):
    rc, rw, idx, margin = G.center_distogram(dg, center=center, wide=wide, softmax=logits, details=True, row0=row0)
    c, w = c.double().cpu(), w.double().cpu()
    assert torch.equal(torch.isnan(c), torch.isnan(rc)) and torch.equal(torch.isnan(w), torch.isnan(rw)), (center, wide, logits)
    if center == "median":
        sure = margin >= 1e-6                               # the oracle's |cumsum - half| at least 1e-6 of the total
        assert torch.equal(c[sure], rc[sure]), (wide, logits, "median bin differs away from a tie")
        sure_w = sure
    else:
        torch.testing.assert_close(c, rc, rtol=1e-5, atol=1e-5, equal_nan=True)
        sure_w = torch.ones_like(c, dtype=torch.bool)
    torch.testing.assert_close(w[sure_w], rw[sure_w], rtol=1e-4, atol=1e-5, equal_nan=True)


@pytest.mark.parametrize("logits", [False, True])
def test_center_distogram_against_fp64_oracle(logits):
    g = torch.Generator().manual_seed(1)
    for n in (1, 2, 37, 130, 257):
        for b in (1, 2):
            dg = _distogram(b, n, g, logits)
            x = dg.float().to(DEV)
            for center, wide in MODES:
                c, w = ops.center_distogram(x, U.DISTANCE_THRESHOLDS, center, wide, softmax=logits)
                assert c.shape == (b, n, n) and w.shape == (b, n, n)
                _check_center(c, w, dg.float().double(), center, wide, logits)


def test_center_distogram_torch_quirks():
    """the public call: NaN central and weight for a pair whose bins sum to 0 (also on the diagonal), the median puts it in bin 0;
    a 3-D distogram gets a batch dimension"""
    p = torch.rand(9, 9, 37).softmax(-1)
    p[1, 4] = 0.0
    p[3, 3] = 0.0
    c, w = U.center_distogram_torch(p.to(DEV))
    assert c.shape == (1, 9, 9) and torch.isnan(c[0, 1, 4]) and torch.isnan(w[0, 1, 4]) and torch.isnan(w[0, 3, 3])
    c, w = U.center_distogram_torch(p.to(DEV), center="median", wide="none")
    assert c[0, 1, 4].item() == 1.5 and w[0, 1, 4].item() == 1.0 and c[0, 3, 3].item() == 0.0


def _chain(b, n_res, seed, jitter=25.0):
    g = torch.Generator().manual_seed(seed)
    xs = torch.stack([G.backbone(n_res, generator=g, jitter=jitter, dtype=torch.float64) for _ in range(b)], 0)
    return xs, torch.cdist(xs, xs)


def _quantised(d):
    return (d * 2).round() / 2 + 0.3 * (1 - torch.eye(d.shape[-1], dtype=d.dtype))


def _run(pre, w, init, iters, tol):
    x = init.float().to(DEV).contiguous()
    k, stopped, his, stress = ops.mds_iterate_(pre.float().to(DEV).contiguous(), None if w is None else w.float().to(DEV).contiguous(),
                                               x, iters, tol)
    return x.double().cpu(), k, stopped, his.cpu(), stress.cpu()


def test_one_guttman_step_against_fp64_oracle():
    _, d = _chain(2, 30, 3)
    pre = _quantised(d)
    g = torch.Generator().manual_seed(4)
    init = torch.randn(2, 90, 3, generator=g, dtype=torch.float64) * 5
    init = init.float().double()
    w = torch.rand(2, 90, 90, generator=g, dtype=torch.float64).float().double()
    for weights in (None, w):
        x, k, stopped, his, stress = _run(pre, weights, init, 1, float("-inf"))
        ref = G.mds(pre.float().double(), weights, 1, float("-inf"), init=init)
        assert k == 1 and not stopped and ref["steps"] == 1
        torch.testing.assert_close(x, ref["coords"].transpose(-1, -2), rtol=0, atol=1e-4 * ref["coords"].abs().max().item())
        torch.testing.assert_close(stress, ref["stress"], rtol=1e-4, atol=0)
        torch.testing.assert_close(his[1:], ref["his"][1:], rtol=1e-4, atol=0)
        assert torch.isinf(his[0]).all()


@pytest.mark.parametrize("case", ["cap_unweighted", "never_stops", "weighted_step1", "true_distances"])
def test_loop_step_count_and_coords(case):
    xs, d = _chain(2, 40, 5)
    g = torch.Generator().manual_seed(6)
    w = None
    if case == "cap_unweighted":
        pre, iters, tol, init = _quantised(d), 12, 1e-5, G.mds_init(_quantised(d))
    elif case == "never_stops":
        pre, iters, tol, init = _quantised(d), 25, float("-inf"), torch.randn(2, 120, 3, generator=g, dtype=torch.float64) * 8
    elif case == "weighted_step1":
        peaked = (-(d[..., None] - G.bin_centres(G.DISTANCE_THRESHOLDS, torch.float64)) ** 2).softmax(-1)
        pre, w = G.center_distogram(peaked)
        w = w.float().double()
        iters, tol, init = 50, 1e-5, G.mds_init(pre)
    else:
        pre, iters, tol, init = d, 15, 1e-5, torch.randn(2, 120, 3, generator=g, dtype=torch.float64) * 8
    pre = pre.float().double()
    init = init.float().double()
    x, k, stopped, his, _ = _run(pre, w, init, iters, tol)
    ref = G.mds(pre, w, iters, tol, init=init)
    if case == "weighted_step1":
        assert ref["steps"] == 1 and ref["stopped"]
    else:
        assert ref["steps"] == iters and not ref["stopped"]
    assert (k, stopped) == (ref["steps"], ref["stopped"])
    torch.testing.assert_close(his[:k + 1], ref["his"], rtol=5e-4, atol=0)
    if stopped:                                             # the row of the iteration that stopped the loop
        torch.testing.assert_close(his[k + 1], ref["vals"][-1], rtol=5e-4, atol=0)
    scale = ref["coords"].abs().max().item()
    torch.testing.assert_close(x, ref["coords"].transpose(-1, -2), rtol=0, atol=1e-3 * scale)


def test_init_reconstructs_the_gram_matrix():
    """X X^T of the init matches the fp64 top-3 eigen-reconstruction of M on near-rank-3 inputs"""
    _, d = _chain(2, 60, 7, jitter=10.0)
    pre = (d + 1e-3 * torch.rand(d.shape, dtype=torch.float64)).float()
    torch.manual_seed(0)
    x = ops.mds_init(pre.to(DEV)).double().cpu()
    D = pre.double() ** 2
    M = 0.5 * (D[:, :1, :] + D[:, :, :1] - D)
    ev, V = torch.linalg.eigh(M)
    top = ev.abs().argsort(-1, descending=True)[:, :3]
    for e in range(2):
        Vt, lt = V[e][:, top[e]], ev[e][top[e]]
        recon = Vt @ torch.diag(lt) @ Vt.T
        err = (x[e] @ x[e].T - recon).abs().max() / recon.abs().max()
        assert err < 1e-3, err


@pytest.fixture(scope="module")
def fx(golden):
    return golden("geometry_mds")


@pytest.mark.parametrize("name", ["unweighted", "unweighted_10", "weighted", "eigen", "mirror", "mirror_weighted"])
def test_end_to_end_against_reference_fixture(fx, name):
    """the GPU draws a different init than the reference's CPU RNG, so compare what does not depend on the init's rotation:
    the pairwise distances of the coords, the history, and the chirality the mirror fix leaves"""
    case = fx["mds"][name]
    inp, kw = case["inputs"], dict(case["kwargs"])
    for k in ("N_mask", "CA_mask", "C_mask"):
        if kw.get(k) is not None:
            kw[k] = kw[k].to(DEV)
    torch.manual_seed(0)
    coords, his = U.MDScaling(inp["pre"].to(DEV), weights=None if inp.get("weights") is None else inp["weights"].to(DEV),
                              verbose=0, **kw)
    ref_c, ref_h = case["coords"].double(), case["his"].double()
    assert coords.shape == ref_c.shape and his.dtype == torch.float32
    c = coords.double().cpu()
    dist, ref_dist = torch.cdist(c.transpose(-1, -2), c.transpose(-1, -2)), torch.cdist(ref_c.transpose(-1, -2), ref_c.transpose(-1, -2))
    if name == "unweighted":                                # 52 steps to a 1e-5 plateau: the stop may land one step apart
        assert abs(his.shape[0] - ref_h.shape[0]) <= 1
        m = min(his.shape[0], ref_h.shape[0])
        torch.testing.assert_close(his[:m].double().cpu(), ref_h[:m], rtol=2e-3, atol=0)
    else:
        assert his.shape == ref_h.shape
        torch.testing.assert_close(his.double().cpu(), ref_h, rtol=2e-3, atol=1e-6)
    torch.testing.assert_close(dist, ref_dist, rtol=0, atol=5e-3 * ref_dist.max().item())
    if kw.get("fix_mirror"):
        masker = torch.arange(30) % 3
        mine = G.phi_ratio(c, masker == 0, masker == 1)
        ref = G.phi_ratio(ref_c, masker == 0, masker == 1)
        assert (mine >= 0.5).all() and torch.equal(mine, ref), (mine, ref)


def test_mirror_fix_flips_a_mirrored_backbone(monkeypatch):
    """from an exact init (true distances), element 0 starts as the mirror image and is flipped back; element 1 is not flipped"""
    xs, d = _chain(2, 12, 8, jitter=5.0)
    init = xs.float().clone()
    init[0, :, 2] = -init[0, :, 2]
    monkeypatch.setattr(ops, "mds_init", lambda pre: init.to(pre.device).contiguous())
    masker = torch.arange(36) % 3
    before = U.calc_phis_torch(init.transpose(-1, -2).to(DEV), masker == 0, masker == 1)
    assert before[0] < 0.5 <= before[1]
    coords, his = U.MDScaling(d.float().to(DEV), iters=5, fix_mirror=True, N_mask=masker == 0, CA_mask=masker == 1, verbose=0)
    after = U.calc_phis_torch(coords, masker == 0, masker == 1)
    assert (after == 1.0).all(), after
    ref = (xs - xs.mean(1, keepdim=True)).float().transpose(-1, -2)       # one Guttman step from the exact init centres it
    torch.testing.assert_close(coords.cpu(), ref, rtol=0, atol=1e-3)


def test_bitwise_reproducible_and_launch_count():
    _, d = _chain(2, 30, 9)
    pre = _quantised(d).float().to(DEV)
    outs = []
    for _ in range(2):
        torch.manual_seed(3)
        n0 = _launches()
        outs.append(U.mds_torch(pre, iters=200, tol=float("-inf"), verbose=0))
        assert _launches() - n0 == 1, "the whole loop is one launch"
    assert outs[0][1].shape == (201, 2)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    logits = torch.randn(2, 90, 90, 37, device=DEV)
    n0 = _launches()
    torch.manual_seed(3)
    a = U.coords_from_distogram(logits, iters=200)
    assert _launches() - n0 == 2
    torch.manual_seed(3)
    b = U.coords_from_distogram(logits, iters=200)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_eigen_and_verbose(capsys):
    _, d = _chain(1, 10, 10)
    pre = _quantised(d)[0].float().to(DEV)
    coords, his = U.mds_torch(pre, eigen=True)
    assert coords.shape == (1, 3, 30) and his.shape == (1, 1) and (his == 0).all()
    coords, his = U.mds_torch(pre, iters=300, verbose=2)
    lines = capsys.readouterr().out.splitlines()
    steps = his.shape[0] - 1
    assert sum(line.startswith("it: ") for line in lines) == steps + 1
    assert lines[-1].startswith(f"breaking at iteration {steps} with stress")


def test_coords_from_distogram_masks_and_memory():
    """masked residues get weight 0, and at N 2048 no [b, N, N, buckets] temporary is allocated"""
    n = 2048
    logits = torch.randn(1, n, n, 37, device=DEV)
    mask = torch.ones(1, n, dtype=torch.bool, device=DEV)
    mask[:, -100:] = False
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    coords, his = U.coords_from_distogram(logits, mask=mask, iters=3)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < logits.numel() * 4 // 2, f"{peak} B at peak"
    assert coords.shape == (1, n, 3) and torch.isfinite(coords).all() and his.shape[1] == 1
    c, w = ops.center_distogram(logits, torch.linspace(2, 20, 37), softmax=True, mask=mask)
    assert (w[:, -100:, :] == 0).all() and (w[:, :, -100:] == 0).all()
    rc, rw = G.center_distogram(logits[:, :64, :64].double().cpu(), torch.linspace(2, 20, 37), softmax=True)
    torch.testing.assert_close(w[:, :64, :64].double().cpu(), rw, rtol=2e-5, atol=2e-6)


def test_large_distogram_past_2_31_elements():
    """b 3, N 4800: 2.56e9 distogram elements; sampled rows match the oracle, and the whole chain runs"""
    b, n = 3, 4800
    logits = torch.empty(b, n, n, 37, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(11)
    for e in range(b):
        logits[e].normal_(generator=gen)
    for center, wide in (("mean", "std"), ("median", "var")):
        c, w = ops.center_distogram(logits, torch.linspace(2, 20, 37), center, wide, softmax=True)
        for e, r in ((0, 0), (1, 2399), (2, 4799)):
            dg = logits[e:e + 1, r:r + 1].double().cpu()
            _check_center(c[e:e + 1, r:r + 1], w[e:e + 1, r:r + 1], dg, center, wide, True, row0=r)
        del c, w
    coords, his = U.coords_from_distogram(logits, iters=3)
    assert coords.shape == (b, n, 3) and torch.isfinite(coords).all()


def test_refusals_before_device_work():
    pre = torch.rand(2, 12, 12, device=DEV)
    masker = torch.arange(12) % 3
    n0 = _launches()
    bad = [
        (ValueError, lambda: U.MDScaling(pre, fix_mirror=True, verbose=0)),
        (ValueError, lambda: U.MDScaling(pre, fix_mirror=True, N_mask=masker == 0, verbose=0)),
        (ValueError, lambda: U.MDScaling(pre, fix_mirror=True, N_mask=torch.arange(9) % 3 == 0, CA_mask=torch.arange(9) % 3 == 1,
                                         verbose=0)),
        (ValueError, lambda: U.mds_torch(pre, weights=torch.rand(2, 12, 11, device=DEV), verbose=0)),
        (ValueError, lambda: U.mds_torch(torch.rand(2, 12, 11, device=DEV), verbose=0)),
        (ValueError, lambda: U.center_distogram_torch(torch.rand(1, 5, 5, 2, device=DEV), bins=torch.linspace(2, 20, 2))),
        (ValueError, lambda: U.center_distogram_torch(torch.rand(1, 5, 5, 129, device=DEV), bins=torch.linspace(2, 20, 129))),
        (ValueError, lambda: U.center_distogram_torch(torch.rand(1, 5, 5, 36, device=DEV))),
        (ValueError, lambda: U.center_distogram_torch(torch.rand(1, 5, 5, 37, device=DEV), center="mode")),
        (ValueError, lambda: U.coords_from_distogram(torch.rand(1, 5, 5, 37, device=DEV), mask=torch.ones(1, 4, dtype=torch.bool))),
        (NotImplementedError, lambda: U.MDScaling(pre.cpu().numpy(), verbose=0)),
        (NotImplementedError, lambda: U.MDScaling(pre, backend="numpy", verbose=0)),
        (RuntimeError, lambda: U.mds_torch(pre.cpu(), verbose=0)),
        (RuntimeError, lambda: U.center_distogram_torch(torch.rand(1, 5, 5, 37))),
    ]
    for exc, fn in bad:
        with pytest.raises(exc):
            fn()
    assert _launches() == n0
    assert A.utils is U
