"""-m gpu: the distogram centring and the SMACOF loop (csrc/geometry.cuh) kernel by kernel against fp64.

Every case calls the C entry (af2_center_distogram, af2_mds_iterate) directly.  Outputs live in NaN-filled buffers with a
guard region after them that must stay untouched; the SMACOF workspace is owned by the test and filled with 0xff bytes (NaN as
fp32 and fp64), and the same call on a zero-filled workspace must give the same bits.  References are fp64 evaluated on the
exact fp32 operands the kernel received (oracle/geometry_oracle.py), and every element is gated by check_bound.  The build has
no --use_fast_math: expf and rsqrtf are within 2 ulp (<= 4u relative), IEEE sqrtf and division round once; u = 2^-24.

Centring, per pair of nb bins with bin centres c_k > 0 (both bin sets below have positive centres):
  * probabilities: the kernel reads p_k as given.  logits: v_k = expf(x_k - m) * (1 / s) with m the maximum and s the fp32
    sum; the common factor 1 / s cancels in every quantity below (each is a ratio to sum v), so v_k carries only a relative
    error delta_k <= (|x_k - m| + 5) u against the fp64 softmax: the rounded difference x_k - m, expf and the product with
    1 / s.  An e_k below the normal range also carries 2^-148 absolutely (s >= 1).  q_k = p_k / sum p.
  * mean: two fp32 sums of nb terms (sum v c, sum v) and one division:
      e_c = (2 nb + 4) u |c| + 1.01 sum_k q_k delta_k |c_k - c| + nb 2^-147 max_k |c_k - c|
  * median: the first k with cumsum >= half the total.  The kernel's cumsum carries at most nb u of the total, half the
    total (nb / 2) u, the softmax perturbation max_k delta_k: where the oracle's smallest |cumsum - half| / total (margin)
    exceeds (2 nb + 8) u + 2 max_k delta_k the bin must be the oracle's and the centre bitwise equal; closer pairs are ties and
    must only land on a bin centre.  With the centre exact, e_c = 0.
  * dispersion about the kernel's centre c^: sum_k v (c_k - c^)^2 / sum v, where (c_k - c^), its square and the product
    round once each, the sums take nb u each and the division u.  Moving the centre by e_c moves var by at most
    2 |mean - c| e_c + e_c^2 (zero to first order for the mean), and the weights' perturbation by sum q delta |(c_k - c)^2 - var|:
      e_var = (2 nb + 6) u var + 2 |mean - c| e_c + e_c^2 + 1.01 sum_k q_k delta_k |(c_k - c)^2 - var| + nb 2^-147 max (c_k - c)^2
      e_std = min(e_var / std, sqrt(e_var)) + u (std + sqrt(e_var))             (IEEE sqrtf, |sqrt a - sqrt b| bounds)
  * weight = keep / (1 + disp): 1 + disp and the division round once:  e_w = 1.01 (w^2 (e_disp + u (1 + disp)) + u w).
    keep = (c <= bins[-2]) must be the oracle's except where |c - bins[-2]| <= e_c; there the weight is either 0 or the
    oracle's 1 / (1 + disp).  Diagonal and masked weights are exactly 0; NaN (bins summing to 0, a pair of -inf logits) must
    be NaN in exactly the oracle's places.

One Guttman step, row i (N points, K = ceil(N / 32) + 5 terms per lane chain and shuffle levels):  the rounded differences
dx (u), dsq as three products and two sums of positive terms (5u), rsqrtf (4u + half of dsq's), d = dsq rs, r = w (delta rs)
and r dx (one rounding each): each term t_j = r_ij dx_ij carries at most 11 u relative; the fp32 row sum K u sum |t_j|; 1 / N
and the product two roundings:
      e_x = 1.01 ((K + 12) u sum_j |t_j| / N + 2 u |x'|)
A coincident pair (and the diagonal) has dx = 0 exactly: the kernel's d <= 0 branch and the oracle's 1e-7 both give 0.
The stress is an fp64 sum of fp32 terms w (d - delta)^2 with d = dsq rs within 7.5 u d:  per term 15 u d |d - delta| +
4 u (d - delta)^2, times w, halved, plus the fp64 chain (N + 64) 2^-52 stress.  his = stress / sqrt(sum x'^2) in fp64:
      e_his = 1.01 his (e_stress / stress + (sum 2 |x'| e_x + e_x^2) / (2 sum x'^2)) + 2^-50 his

The loop is checked bitwise instead where the arithmetic is the same: a batch element gives the same bits alone (B = 1) as
inside a batch whose work items outnumber the resident CTAs (every CTA then reloads X for a second element), and the
step-two result of N = MDS_MAX_N is held to the step bound from the kernel's own step-one coordinates.
"""
import math

import pytest
import torch

from gpu_util import check_bound
from oracle import geometry_oracle as G

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
GUARD = 4096
BAD_ARG, BAD_WS = -1, -4
MDS_MAX_N = 12288
MODES = [(c, w) for c in ("mean", "median") for w in ("std", "var", "none")]
CENTER = {"mean": 0, "median": 1}
WIDE = {"std": 0, "var": 1, "none": 2}


def _ops():
    from alphafold2_b200 import ops
    return ops


def _lib():
    from alphafold2_b200 import _lib
    return _lib.load()


def _rc(fn, *args):
    return getattr(_lib(), fn)(*args, _ops()._stream_ptr())


def _launches():
    return _lib().af2_launch_count()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _guarded(n, dtype=torch.float32, fill=float("nan")):
    return torch.full((n + GUARD,), fill, dtype=dtype, device=DEV)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else (t.view(torch.int64) if t.dtype == torch.float64 else t)


def _same_bits(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), what


# ------------------------------------------------------------------------------------------------------------------------
# centring
# ------------------------------------------------------------------------------------------------------------------------
def _bins(kind, nb):
    if kind == "thresholds":
        assert nb == 37
        return G.DISTANCE_THRESHOLDS.clone()
    return 2.5 + 0.75 * torch.arange(nb, dtype=torch.float32)        # uniform, spacing 0.75: centres 1.5, 2.875, ...


def _distogram(B, n, nb, logits, seed):
    """fp32 [B, n, n, nb] with the edges: logits of +-80, -inf in half the bins, a pair of -inf only; probabilities with a pair
    summing to 0, a one-hot pair and zeros in half the bins.  Every edge sits off the diagonal."""
    g = _gen(seed)
    x = torch.randn(B, n, n, nb, generator=g, device=DEV) * 3
    e = B - 1
    if logits:
        x[0, 0, 1] = torch.where(torch.arange(nb, device=DEV) % 2 == 0, 80.0, -80.0)
        x[0, 1, 2, ::2] = float("-inf")
        x[e, 2, 0] = float("-inf")
        x[e, 3, 1, 1:] = -80.0
        return x.contiguous()
    p = x.softmax(-1)
    p[0, 0, 1] = 0.0
    p[0, 1, 2] = 0.0
    p[0, 1, 2, nb // 2] = 1.0
    p[e, 2, 0, ::2] = 0.0
    return p.contiguous()


def _center_call(dist, centres, thr, mask, B, n, nb, center, wide, softmax):
    P = B * n * n
    c, w = _guarded(P), _guarded(P)
    rc = _rc("af2_center_distogram", dist.data_ptr(), centres.data_ptr(), thr, 0 if mask is None else mask.data_ptr(),
             c.data_ptr(), w.data_ptr(), B, n, nb, CENTER[center], WIDE[wide], int(softmax))
    assert rc == 0, _lib().af2_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(c[P:]).all() and torch.isnan(w[P:]).all(), "guard written"
    return c[:P].view(B, n, n), w[:P].view(B, n, n)


def _center_bounds(dist, bins, logits, center, wide, rc, margin):
    """the module docstring's bounds, evaluated in fp64 on the device; returns (e_c, e_w, sure_c, sure_keep, 1 / (1 + disp))"""
    nb = dist.shape[-1]
    x = dist.double()
    p = x.softmax(-1) if logits else x
    ck = G.bin_centres(bins, torch.float64).to(DEV)
    mag = p.sum(-1, keepdim=True)
    q = p / mag
    if logits:
        m = x.max(-1, keepdim=True).values
        gap = torch.where(torch.isfinite(x - m), (x - m).abs(), torch.zeros_like(x))
        delta = (gap + 5) * U
    else:
        delta = torch.zeros_like(x)
    tiny = nb * 2.0 ** -147
    mean = (q * ck).sum(-1)
    thr = float(bins.float()[-2])
    if center == "mean":
        dev_c = (ck - mean[..., None]).abs()
        e_c = (2 * nb + 4) * U * mean.abs() + 1.01 * (q * delta * dev_c).sum(-1) + tiny * dev_c.max(-1).values
        sure_c = torch.ones_like(mean, dtype=torch.bool)
        sure_keep = (mean - thr).abs() > e_c
        c = mean
    else:
        need = (2 * nb + 8) * U + 2 * delta.max(-1).values
        sure_c = (margin > need) | (mag[..., 0] == 0)
        e_c = torch.zeros_like(mean)
        sure_keep = sure_c
        c = rc
    eye = torch.eye(dist.shape[1], dtype=torch.bool, device=DEV)
    c = torch.where(eye, torch.zeros_like(c), c)                      # the kernel's dispersion uses the zeroed centre
    e_c_disp = torch.where(eye, torch.zeros_like(e_c), e_c)
    sq = (ck - c[..., None]) ** 2
    var = (q * sq).sum(-1)
    e_var = ((2 * nb + 6) * U * var + 2 * (mean - c).abs() * e_c_disp + e_c_disp ** 2
             + 1.01 * (q * delta * (sq - var[..., None]).abs()).sum(-1) + tiny * sq.max(-1).values)
    if wide == "var":
        disp, e_disp = var, e_var
    elif wide == "std":
        disp = var.sqrt()
        e_disp = torch.minimum(e_var / disp, e_var.sqrt()) + U * (disp + e_var.sqrt())
        e_disp = torch.where(disp == 0, e_var.sqrt(), e_disp)
    else:
        disp, e_disp = torch.zeros_like(var), torch.zeros_like(var)
    w1 = 1.0 / (1.0 + disp)
    e_w = 1.01 * (w1 ** 2 * (e_disp + U * (1 + disp)) + U * w1)
    return e_c, e_w, sure_c, sure_keep, w1


def _center_case(name, B, n, nb, bins_kind, logits, masked, seed):
    bins = _bins(bins_kind, nb)
    ops = _ops()
    centres = ops.bin_centres(bins, DEV)
    assert torch.equal(centres.cpu(), G.bin_centres(bins)), "the kernel's centres are the oracle's"
    thr = float(bins[-2])
    dist = _distogram(B, n, nb, logits, seed)
    mask = None
    if masked:                                                        # a different residue masked in each element
        mask = torch.ones(B, n, dtype=torch.uint8, device=DEV)
        for e in range(B):
            mask[e, (2 * e + 1) % n] = 0
            if e == B - 1 and B > 1:
                mask[e, (e + 3) % n] = 0
    for center, wide in MODES:
        c, w = _center_call(dist, centres, thr, mask, B, n, nb, center, wide, logits)
        rc, rw, idx, margin = G.center_distogram(dist.double(), bins, center, wide, softmax=logits,
                                                 mask=None if mask is None else mask.bool(), details=True)
        tag = f"geometry/center/{name}/nb{nb}_{bins_kind}_{'logits' if logits else 'probs'}/{center}_{wide}"
        assert torch.equal(torch.isnan(c), torch.isnan(rc)), f"{tag}: NaN centres differ"
        assert torch.equal(torch.isnan(w), torch.isnan(rw)), f"{tag}: NaN weights differ"
        e_c, e_w, sure_c, sure_keep, w1 = _center_bounds(dist, bins, logits, center, wide, rc, margin)
        fin = torch.isfinite(rc)
        eye = torch.eye(n, dtype=torch.bool, device=DEV).expand(B, n, n)
        assert (c[fin & eye] == 0).all(), f"{tag}: diagonal centre not 0"
        if center == "median":
            ties = fin & ~sure_c & ~eye
            on_centre = (c[ties].double()[:, None] == centres.double()[None, :]).any(-1)
            assert on_centre.all(), f"{tag}: a tied median is not a bin centre"
            sure = fin & (sure_c | eye)
            assert torch.equal(_bits(c[sure]), _bits(rc[sure].float())), f"{tag}: median bin differs"
        else:
            check_bound(f"{tag}/central", c[fin], rc[fin], e_c[fin])
        finw = torch.isfinite(rw)
        # where keep is a tie, the weight is 0 or the oracle's kept weight (masked and diagonal weights stay exactly 0)
        zeroed = eye if mask is None else (eye | ~(mask.bool()[:, :, None] & mask.bool()[:, None, :]))
        alt = torch.where(zeroed | (w == 0), torch.zeros_like(rw), w1)
        ref_w = torch.where(sure_keep, rw, alt)
        ok = finw & (sure_c | zeroed)
        assert (w[zeroed & finw] == 0).all(), f"{tag}: diagonal or masked weight not 0"
        check_bound(f"{tag}/weight", w[ok], ref_w[ok], torch.where(ref_w[ok] == 0, torch.zeros_like(e_w[ok]), e_w[ok]))


NBS = [3, 4, 37, 48, 49, 64, 127, 128]
SHAPES = {"P25": (1, 5, False), "P64": (1, 8, False), "P169": (1, 13, True), "B3_P147": (3, 7, True)}


@pytest.mark.parametrize("logits", [False, True])
@pytest.mark.parametrize("nb,bins_kind", [(nb, "uniform") for nb in NBS] + [(37, "thresholds")])
def test_center_distogram_vs_fp64(nb, bins_kind, logits):
    """P < 32, P a multiple of 32, a partial last run, and B 3 with n^2 = 49 (runs straddle elements) with a different mask per
    element; nb 48 is exactly 48 KB of shared memory per CTA, 49 the first count above it, 128 the largest (128 KB)"""
    for k, (name, (B, n, masked)) in enumerate(SHAPES.items()):
        _center_case(name, B, n, nb, bins_kind, logits, masked, seed=nb * 100 + k * 10 + int(logits))


@pytest.mark.parametrize("nb", [49, 128])
def test_center_distogram_grid_stride(nb):
    """45,000 pairs: more 32-pair runs than one wave of resident warps holds, so each warp takes several"""
    _center_case("B2_n150", 2, 150, nb, "uniform", True, True, seed=nb)


def test_center_distogram_refusals():
    """nb 2 and 129, and a dist 4 bytes past a 16-byte boundary: AF2_ERR_BAD_ARG, nothing launched, outputs untouched"""
    B, n = 1, 6
    buf = torch.rand(B * n * n * 129 + 4, device=DEV)
    centres = torch.linspace(1.5, 40, 129, device=DEV)
    c, w = _guarded(B * n * n), _guarded(B * n * n)
    cases = [(buf.data_ptr(), 2), (buf.data_ptr(), 129), (buf.data_ptr() + 4, 37)]
    for ptr, nb in cases:
        n0 = _launches()
        rc = _rc("af2_center_distogram", ptr, centres.data_ptr(), 19.5, None, c.data_ptr(), w.data_ptr(), B, n, nb, 0, 0, 1)
        torch.cuda.synchronize()
        assert rc == BAD_ARG, (nb, rc)
        assert _launches() == n0, "launched before refusing"
        assert torch.isnan(c).all() and torch.isnan(w).all(), "wrote before refusing"


# ------------------------------------------------------------------------------------------------------------------------
# SMACOF
# ------------------------------------------------------------------------------------------------------------------------
def _mds_call(delta, w, x0, iters, tol, fill=0xFF):
    """af2_mds_iterate on a copy of x0 inside a guarded buffer with a workspace filled with `fill` bytes -> (x, his, stress, steps)"""
    B, n, _ = x0.shape
    lib = _lib()
    need = lib.af2_mds_workspace(B, n, iters)
    assert need > 0
    ws = torch.full((need,), fill, dtype=torch.uint8, device=DEV)
    xb = _guarded(B * n * 3)
    xb[:B * n * 3] = x0.reshape(-1)
    his = _guarded((iters + 1) * B, torch.float64)
    stress = _guarded(max(iters, 1) * B, torch.float64)
    steps = _guarded(2, torch.int32, -7)
    rc = _rc("af2_mds_iterate", delta.data_ptr(), 0 if w is None else w.data_ptr(), xb.data_ptr(), his.data_ptr(),
             stress.data_ptr(), steps.data_ptr(), B, n, iters, float(tol), ws.data_ptr(), need)
    assert rc == 0, lib.af2_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(xb[B * n * 3:]).all() and torch.isnan(his[(iters + 1) * B:]).all(), "guard written"
    assert torch.isnan(stress[max(iters, 1) * B:]).all() and (steps[2:] == -7).all(), "guard written"
    return (xb[:B * n * 3].view(B, n, 3), his[:(iters + 1) * B].view(iters + 1, B), stress[:max(iters, 1) * B].view(-1, B),
            steps[:2].cpu().tolist())


def _mds_twice(delta, w, x0, iters, tol):
    """the poisoned workspace and a zero-filled one give the same bits"""
    a = _mds_call(delta, w, x0, iters, tol, 0xFF)
    b = _mds_call(delta, w, x0, iters, tol, 0x00)
    for u, v in zip(a[:3], b[:3]):
        _same_bits(u, v, "a poisoned workspace changed the result")
    assert a[3] == b[3]
    return a


def _step64(delta, w, x, chunk=256):
    """one Guttman step in fp64 in the oracle's difference form, row chunks at a time, with the bound's terms:
    -> (x' [B, N, 3], sum_j |t_j| / N [B, N, 3], stress [B], stress error bound [B])"""
    B, n, _ = x.shape
    x64 = x.double()
    new = torch.empty(B, n, 3, dtype=torch.float64, device=DEV)
    absn = torch.empty_like(new)
    stress = torch.zeros(B, dtype=torch.float64, device=DEV)
    e_st = torch.zeros_like(stress)
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        diff = x64[:, r0:r1, None, :] - x64[:, None, :, :]
        dist = diff.pow(2).sum(-1).sqrt()
        pre = delta[:, r0:r1].double()
        wt = torch.ones_like(pre) if w is None else w[:, r0:r1].double()
        res = dist - pre
        stress += (wt * res ** 2).sum((-1, -2)) * 0.5
        e_st += (wt * (15 * U * dist * res.abs() + 4 * U * res ** 2)).sum((-1, -2)) * 0.5
        d2 = torch.where(dist <= 0, dist + 1e-7, dist)
        t = (wt * (pre / d2))[..., None] * diff
        new[:, r0:r1] = t.sum(2) / n
        absn[:, r0:r1] = t.abs().sum(2) / n
        del diff, dist, pre, wt, res, d2, t
    e_st = 1.05 * e_st + (n + 64) * 2.0 ** -52 * stress
    return new, absn, stress, e_st


def _step_bounds(n, new, absn, stress, e_st):
    K = math.ceil(n / 32) + 5
    e_x = 1.01 * ((K + 12) * U * absn + 2 * U * new.abs())
    q = new.pow(2).sum((-1, -2))
    e_q = (2 * new.abs() * e_x + e_x ** 2).sum((-1, -2))
    his = stress / q.sqrt()
    e_his = 1.01 * his * (e_st / stress + e_q / (2 * q)) + 2.0 ** -50 * his
    return e_x, his, e_his


def _check_step(tag, x, stress_k, his_k, delta, w, x_in):
    n = x.shape[1]
    new, absn, st, e_st = _step64(delta, w, x_in)
    e_x, his, e_his = _step_bounds(n, new, absn, st, e_st)
    check_bound(f"{tag}/x", x, new, e_x)
    check_bound(f"{tag}/stress", stress_k, st, e_st)
    fin = torch.isfinite(his)
    assert torch.equal(torch.isnan(his_k), torch.isnan(his)), f"{tag}: NaN history differs"
    assert torch.equal(his_k[torch.isinf(his)], his[torch.isinf(his)]), f"{tag}: infinite history differs"
    check_bound(f"{tag}/his", his_k[fin], his[fin], e_his[fin])
    return new, st


def _mds_inputs(B, n, seed, weighted):
    g = _gen(seed)
    pts = torch.randn(B, n, 3, generator=g, device=DEV, dtype=torch.float64) * (2 * n) ** (1 / 3)
    delta = (torch.cdist(pts, pts) * (1 + 0.2 * torch.rand(B, n, n, generator=g, device=DEV, dtype=torch.float64))).float()
    delta = ((delta + delta.transpose(1, 2)) / 2).contiguous()
    w = torch.rand(B, n, n, generator=g, device=DEV).contiguous() if weighted else None
    x0 = (torch.randn(B, n, 3, generator=g, device=DEV) * 4).contiguous()
    return delta, w, x0


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("n", [1, 2, 15, 16, 17, 300])
def test_guttman_step_vs_fp64(n, weighted):
    """one step from a known init at B 2; element 0 has a delta with a non-zero diagonal and, from 3 points, two coincident points"""
    delta, w, x0 = _mds_inputs(2, n, seed=n * 2 + int(weighted), weighted=weighted)
    delta[0].diagonal().copy_(torch.rand(n, generator=_gen(n), device=DEV) * 3 + 0.5)
    if n >= 3:
        x0[0, n - 1] = x0[0, 0]
    x, his, stress, steps = _mds_twice(delta, w, x0, 1, float("-inf"))
    assert steps == [1, 0]
    assert torch.isinf(his[0]).all() and (his[0] > 0).all()
    ref = G.mds(delta.double(), None if w is None else w.double(), 1, float("-inf"), init=x0.double())
    new, st = _check_step(f"geometry/mds_step/n{n}_{'w' if weighted else 'unw'}", x, stress[0], his[1], delta, w, x0)
    # the chunked step is the oracle's mds step
    torch.testing.assert_close(new, ref["coords"].transpose(-1, -2), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(st, ref["stress"][0], rtol=1e-12, atol=0)


def _solo_vs_batch(B, n, iters, weighted, seed):
    delta, w, x0 = _mds_inputs(B, n, seed=seed, weighted=weighted)
    xb, hb, sb, kb = _mds_call(delta, w, x0, iters, float("-inf"))
    assert kb == [iters, 0]
    for e in range(B):
        xs, hs, ss, ks = _mds_call(delta[e:e + 1].contiguous(), None if w is None else w[e:e + 1].contiguous(),
                                   x0[e:e + 1].contiguous(), iters, float("-inf"))
        assert ks == kb
        _same_bits(xs[0], xb[e], f"n {n} element {e}: coords alone differ from the batch's")
        _same_bits(hs[:, 0].contiguous(), hb[:, e].contiguous(), f"n {n} element {e}: history differs")
        _same_bits(ss[:, 0].contiguous(), sb[:, e].contiguous(), f"n {n} element {e}: stress differs")
    return xb


@pytest.mark.parametrize("iters", [3, 4])
def test_mds_grid_independent_bitwise(iters):
    """B 12 x N 2048 is 1536 work items, more than the 1056 CTAs that can be resident (8 per SM): CTAs take items of two
    elements.  Alone each element is 128 items, at most one per CTA.  3 and 4 accepted steps: the result ends in the workspace
    buffer (copied out) or in the caller's."""
    _solo_vs_batch(12, 2048, iters, weighted=True, seed=iters)


def test_mds_grid_independent_bitwise_n4800():
    """N 4800: 76.8 KB of X per CTA, two CTAs per SM, 300 items per element, so at B 2 every CTA takes two or three items"""
    _solo_vs_batch(2, 4800, 3, weighted=False, seed=48)


def test_mds_max_n_vs_fp64():
    """N = MDS_MAX_N (192 KB of shared memory, one CTA per SM), B 2, weighted: step 1 against the fp64 step from the init, and
    step 2 against the fp64 step from the kernel's own step-1 coordinates (iters 1 ends in the workspace buffer, iters 2 in
    the caller's)"""
    n, B = MDS_MAX_N, 2
    delta, w, x0 = _mds_inputs(B, n, seed=12288, weighted=True)
    x1, h1, s1, k1 = _mds_call(delta, w, x0, 1, float("-inf"))
    assert k1 == [1, 0]
    _check_step("geometry/mds_max_n/step1", x1, s1[0], h1[1], delta, w, x0)
    x2, h2, s2, k2 = _mds_call(delta, w, x0, 2, float("-inf"))
    assert k2 == [2, 0]
    _same_bits(s2[0].contiguous(), s1[0].contiguous(), "the first iteration differs between iters 1 and 2")
    _same_bits(h2[:2].contiguous(), h1.contiguous(), "the first history rows differ between iters 1 and 2")
    _check_step("geometry/mds_max_n/step2", x2, s2[1], h2[2], delta, w, x1.clone())


def test_mds_refusals():
    """N = MDS_MAX_N + 1, negative iters (AF2_ERR_BAD_ARG) and a workspace one byte short (AF2_ERR_WORKSPACE): no launch,
    nothing written"""
    lib = _lib()
    n = MDS_MAX_N + 1
    assert lib.af2_mds_workspace(1, n, 1) < 0 and lib.af2_mds_workspace(1, 8, -1) < 0
    assert lib.af2_mds_workspace(1, MDS_MAX_N, 1) > 0
    big = torch.zeros(1, n, n, device=DEV)
    small, _, x0 = _mds_inputs(1, 8, seed=1, weighted=False)
    need = lib.af2_mds_workspace(1, 8, 2)
    ws = torch.full((need + 1024 + 4 * n * 3,), 0xFF, dtype=torch.uint8, device=DEV)
    cases = [(big, n, 1, ws.numel(), BAD_ARG), (small, 8, -1, ws.numel(), BAD_ARG), (small, 8, 2, need - 1, BAD_WS)]
    for delta, nn, iters, nws, code in cases:
        x = _guarded(3 * nn)
        his, stress = _guarded(8, torch.float64), _guarded(8, torch.float64)
        steps = _guarded(2, torch.int32, -7)
        n0 = _launches()
        rc = _rc("af2_mds_iterate", delta.data_ptr(), None, x.data_ptr(), his.data_ptr(), stress.data_ptr(), steps.data_ptr(),
                 1, nn, iters, float("-inf"), ws.data_ptr(), nws)
        torch.cuda.synchronize()
        assert rc == code, (nn, iters, nws, rc)
        assert _launches() == n0, "launched before refusing"
        assert torch.isnan(x).all() and torch.isnan(his).all() and torch.isnan(stress).all() and (steps == -7).all()
