"""-m gpu: the structure-score kernels (csrc/metrics.cuh) kernel by kernel against fp64.

Every case calls the C entry (af2_pair_distance_scores, af2_superpose_scores) directly with a workspace the test owns,
filled with 0xff bytes (NaN as fp32 / fp64, -1 as int32); the same call on a zero-filled workspace must give the same bits.
Outputs live in NaN-filled buffers (rot: zero-filled) with a guard region after them that must stay untouched.  References
are fp64 evaluated on the exact fp32 operands the kernel received (oracle/metrics_oracle.py); u = 2^-24.

Every threshold decision of the kernels uses dist64, the uncontracted fp64 expression the oracle's dist evaluates one torch
operation at a time, so decisions are compared exactly:
  * lDDT: the per-split int32 counters, summed over the splits, equal M.lddt_counts; the fp32 ratio is the oracle's bitwise;
    the mean is an fp64 sum of fp32 ratios in a fixed order, one division and one fp32 rounding:
      |mean - ref| <= u |ref| + (n + 64) 2^-52 mean |l|.
    Shapes are picked with a restatement of pd_split (_pd_split) so that each regime is reached on purpose: one split, 16
    splits, fewer than 32 columns per split, and a split longer than PD_TJ = 512 that ends in a partial tile.
  * Loss: each pair's term is the oracle's fp64 value (q 2 bitwise; q 1, 0.5, 3 through fabs / pow, a few ulp); the two fp64
    sums of M non-negative terms differ by at most (2 M + 70) 2^-53 of the total, the mean divides once and the result is
    rounded once to fp32:  |loss - ref| <= 1.01 (u + (2 M + 70) 2^-53) |ref|.
  * Superposition: the aligned points are fl32(U^T (x - cx)) (+ cy with shift) and fl32(y - cy), with the kernel's U (rot,
    compared with the oracle's on its own) and fp64 centroids, which differ from the oracle's by at most 2 (n_sel + 16)
    2^-53 max |x| per coordinate (two fixed-order fp64 sums):
      |xo - ref| <= u |ref| + 3 ecx + 8 2^-53 (sum_k |U_kc| |xc_k| + |cy|) + ecy,   |yo - ref| <= u |ref| + ecy + 2^-52 |ref|.
    The scores are checked on the kernel's own fp32 aligned points, where the kernel states that every threshold decision is
    the fp64 oracle's: the GDT counts exactly (through the fp32 GDT sum, restated bitwise with power-of-two weights), and
      |rmsd - ref| <= 1.01 (u + (n_sel + 40) 2^-53) ref                    (fp64 sum of n_sel squares, sqrt, fp32)
      |tm - ref|   <= u |ref| + (n_sel + 40) 2^-53 ref + mean_i (2 e_d0 + 4 2^-53) t_i,  e_d0 = 4 2^-53 (|d0| + 3.6) / |d0|
    (t_i = 1 / (1 + (d_i / d0)^2); d0 comes from pow in fp64 on both sides).
    The rotation is compared with the oracle's within 1e-9 where it is unique and well conditioned: C has rank 2 or more and
    the smallest denominator of the polar factor's sensitivity, s1 + s2 (s1 - s2 when the determinant fix applies), exceeds
    1e-4 s0.  Elsewhere it must be a proper rotation and the RMSD the oracle's minimum within 4 u max |coordinate| (each
    side's fp32 rounding of the aligned points) + 2^-40 max |coordinate|.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from gpu_util import check_bound
from oracle import metrics_oracle as M

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
E53 = 2.0 ** -53
GUARD = 4096
BAD_ARG = -1
PD_ROWS, PD_TJ, PD_MAX_SPLITS = 32, 512, 16
CUTS = (0.5, 1.0, 2.0, 4.0, 8.0)
GDT_SPECS = (((1, 2, 3, 4), (2.0, 1.0, 1.0, 0.5)), ((0, 1, 2, 3), (1.0, 1.0, 1.0, 1.0)))   # TS with weights, HA


def _L():
    from alphafold2_b200 import _lib as L
    return L


def _lib():
    return _L().load()


def _rc(fn, *args):
    from alphafold2_b200 import ops
    return getattr(_lib(), fn)(*args, ops._stream_ptr())


def _launches():
    return _lib().af2_launch_count()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _guarded(n, dtype=torch.float32, fill=float("nan")):
    return torch.full((n + GUARD,), fill, dtype=dtype, device=DEV)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else (t.view(torch.int64) if t.dtype == torch.float64 else t)


def _pts(t, off, sb, sn, sk):
    """af2_points at element offset `off` into t"""
    return C.byref(_L().Points(t.data_ptr() + off * t.element_size(), sb, sn, sk))


def _ws(B, n, fill):
    need = _lib().af2_metrics_workspace(B, n)
    assert need > 0
    return torch.full((need,), fill, dtype=torch.uint8, device=DEV)


def _pd_split(B, n):
    """restatement of metrics_api.inl pd_split: (splits, columns per split); used to pick shapes and name their regime"""
    ctas = (n + PD_ROWS - 1) // PD_ROWS * B
    s = max(1, min((264 + ctas - 1) // ctas, (n + 31) // 32, PD_MAX_SPLITS))
    cols = (n + s - 1) // s
    return (n + cols - 1) // cols, cols


def _structures(B, n, seed, noise=1.5):
    """a chain-like true structure [B, n, 3] and a rotated, shifted, noisy prediction, fp32 on the device"""
    g = _gen(seed)
    steps = torch.randn(B, n, 3, generator=g, device=DEV)
    true = torch.cumsum(3.8 * steps / steps.norm(dim=-1, keepdim=True), 1)
    q, _ = torch.linalg.qr(torch.randn(B, 3, 3, generator=g, device=DEV, dtype=torch.float64))
    pred = ((true.double() + noise * torch.randn(B, n, 3, generator=g, device=DEV, dtype=torch.float64)) @ q + 5.0).float()
    return pred.contiguous(), true.contiguous()


# ------------------------------------------------------------------------------------------------------------------------
# lDDT counters and finalisation
# ------------------------------------------------------------------------------------------------------------------------
LDDT_REGIMES = {"one_split": (9, 1000), "sixteen_splits": (1, 513), "narrow_splits": (2, 100), "long_split": (2, 3000)}
LDDT_LAYOUTS = [("bn3", None), ("b3n", "strided"), ("cloud", "strided"), ("shared_true", "shared"), ("bn3", "shared")]
CLOUD = 4                                                           # atoms per residue of the cloud layout; CA = atom 1


def test_pd_split_regimes():
    splits = {k: _pd_split(*v) for k, v in LDDT_REGIMES.items()}
    assert splits["one_split"] == (1, 1000)
    assert splits["sixteen_splits"][0] == PD_MAX_SPLITS
    assert splits["narrow_splits"][1] < 32
    s, cols = splits["long_split"]
    assert cols > PD_TJ and cols % PD_TJ and s > 1


def _lddt_operand(t, layout, which):
    """the [B, n, 3] structure t laid out as `layout` -> (buffer, element offset, sb, sn, sk)"""
    B, n, _ = t.shape
    if layout == "shared_true" and which == "true":
        return t[:1].contiguous(), 0, 0, 3, 1
    if layout == "b3n":
        return t.transpose(1, 2).contiguous(), 0, 3 * n, 1, n
    if layout == "cloud":
        c = torch.full((B, n, CLOUD, 3), float("nan"), device=DEV)
        c[:, :, 1] = t
        return c, 3, n * CLOUD * 3, CLOUD * 3, 1
    return t.contiguous(), 0, 3 * n, 3, 1


def _lddt_mask(B, n, kind, seed):
    """-> (buffer, element offset, mask_sb, mask_sn, present [B, n] bool) or None"""
    if kind is None:
        return None
    g = _gen(seed)
    if kind == "shared":
        present = (torch.rand(1, n, generator=g, device=DEV) > 0.2).expand(B, n)
        return present[:1].to(torch.uint8).contiguous(), 0, 0, 1, present
    present = torch.rand(B, n, generator=g, device=DEV) > 0.2
    cm = torch.zeros(B, n, CLOUD, dtype=torch.uint8, device=DEV)
    cm[:, :, 1] = present.to(torch.uint8)
    cm[:, :, 0] = 1 - cm[:, :, 1]                                     # the other atoms disagree with the CA
    return cm, 1, n * CLOUD, CLOUD, present


def _lddt_run(true, pred, layout, mk, B, n, fill):
    tb, toff, tsb, tsn, tsk = _lddt_operand(true, layout, "true")
    pb, poff, psb, psn, psk = _lddt_operand(pred, layout, "pred")
    ws = _ws(B, n, fill)
    lddt, mean = _guarded(B * n), _guarded(B)
    mptr, msb, msn = (0, 0, 0) if mk is None else (mk[0].data_ptr() + mk[1], mk[2], mk[3])
    rc = _rc("af2_pair_distance_scores", 0, _pts(tb, toff, tsb, tsn, tsk), 0, _pts(pb, poff, psb, psn, psk), 0, mptr, msb, msn,
             B, n, 15.0, float("-inf"), float("inf"), 2.0, None, ws.data_ptr(), ws.numel())
    assert rc == 0, _lib().af2_last_error()
    rc = _rc("af2_superpose_scores", None, None, mptr, msb, msn, B, n, 0, 0, None, None, None, None, None, 0, None, None, 1,
             lddt.data_ptr(), mean.data_ptr(), ws.data_ptr(), ws.numel())
    assert rc == 0, _lib().af2_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(lddt[B * n:]).all() and torch.isnan(mean[B:]).all(), "guard written"
    splits, _ = _pd_split(B, n)
    counts = ws.view(torch.int32)[:splits * B * n * 2].view(splits, B, n, 2)
    return counts.clone(), lddt[:B * n].view(B, n), mean[:B]


def _lddt_case(tag, true, pred, layout, mask_kind, seed):
    B, n, _ = true.shape
    mk = _lddt_mask(B, n, mask_kind, seed)
    present = torch.ones(B, n, dtype=torch.bool, device=DEV) if mk is None else mk[4]
    a = _lddt_run(true, pred, layout, mk, B, n, 0xFF)
    b = _lddt_run(true, pred, layout, mk, B, n, 0x00)
    for x, y in zip(a, b):
        assert torch.equal(_bits(x), _bits(y)), f"{tag}: a poisoned workspace changed the result"
    counts, lddt, mean = a
    t_ref = true[:1].expand(B, n, 3) if layout == "shared_true" else true
    cnt, scr = M.lddt_counts(t_ref, pred, present, chunk=512)
    got = counts.sum(0).long()
    assert torch.equal(got[..., 0], cnt), f"{tag}: in-radius counts differ"
    assert torch.equal(got[..., 1], scr), f"{tag}: score sums differ"
    ratio = M.lddt_ratio(cnt, scr, present)
    torch.testing.assert_close(lddt, ratio, rtol=0, atol=0, equal_nan=True)
    fin = torch.isfinite(ratio) & present
    l64 = torch.where(fin, ratio.double(), torch.zeros_like(ratio, dtype=torch.float64))
    ref = l64.sum(-1) / fin.sum(-1)
    assert torch.equal(torch.isnan(mean), torch.isnan(ref)), f"{tag}: NaN means differ"
    ok = ~torch.isnan(ref)
    bound = U * ref.abs() + (n + 64) * 2.0 ** -52 * (l64.abs().sum(-1) / fin.sum(-1).clamp_min(1))
    check_bound(f"{tag}/lddt_mean", mean[ok], ref[ok], bound[ok])
    return cnt


@pytest.mark.parametrize("layout,mask_kind", LDDT_LAYOUTS)
@pytest.mark.parametrize("regime", list(LDDT_REGIMES))
def test_lddt_counts_exact(regime, layout, mask_kind):
    B, n = LDDT_REGIMES[regime]
    pred, true = _structures(B, n, seed=B * 7 + n, noise=1.0)
    _lddt_case(f"metrics/lddt/{regime}/{layout}_{mask_kind}", true, pred, layout, mask_kind, seed=n)


def test_lddt_radius_and_thresholds_on_a_lattice():
    """integer coordinates: many true distances are exactly r0 = 15 (excluded: strict) and many differences exactly 0.5 .. 4
    (included); counts must still be exact"""
    B, n = 2, 400
    g = _gen(15)
    true = torch.randint(0, 17, (B, n, 3), generator=g, device=DEV).float()
    pred = true.clone()
    pred[:, ::3] += torch.randint(-2, 3, (B, (n + 2) // 3, 3), generator=g, device=DEV).float() * 0.5
    d = M.dist(true[:, :, None], true[:, None])
    assert int((d == 15.0).sum()) > 1000, "the lattice should put many pairs exactly on r0"
    for layout, mask_kind in (("bn3", None), ("b3n", "strided")):
        _lddt_case(f"metrics/lddt/lattice/{layout}_{mask_kind}", true, pred, layout, mask_kind, seed=3)


# ------------------------------------------------------------------------------------------------------------------------
# the distance-matrix loss
# ------------------------------------------------------------------------------------------------------------------------
LOSS_SHAPES = {"split": (2, 300), "unsplit": (8, 1100)}


def test_loss_shape_regimes():
    for name, (B, n) in LOSS_SHAPES.items():
        tiles = (n + PD_ROWS - 1) // PD_ROWS
        assert (tiles * B < 264) == (name == "split")
        if name == "split":
            assert _pd_split(B, n)[0] > 1


def _loss_run(a, a_mat, b, b_mat, mask, B, n, lo, hi, q, fill):
    def op(t, mat):
        sb = 0 if t.shape[0] == 1 else t.stride(0)
        return _pts(t, 0, sb, t.stride(1), 0 if mat else t.stride(2))
    ws = _ws(B, n, fill)
    out = _guarded(1)
    mptr, msb, msn = (0, 0, 0) if mask is None else (mask.data_ptr(), mask.stride(0), mask.stride(1))
    rc = _rc("af2_pair_distance_scores", 1, op(a, a_mat), int(a_mat), op(b, b_mat), int(b_mat), mptr, msb, msn, B, n, 15.0,
             float(lo), float(hi), float(q), out.data_ptr(), ws.data_ptr(), ws.numel())
    assert rc == 0, _lib().af2_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(out[1:]).all(), "guard written"
    return out[:1]


@pytest.mark.parametrize("shared", [None, "a", "b"])
@pytest.mark.parametrize("a_mat,b_mat", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("shape", list(LOSS_SHAPES))
def test_distmat_loss_vs_fp64(shape, a_mat, b_mat, shared):
    B, n = LOSS_SHAPES[shape]
    g = _gen(n + 2 * a_mat + b_mat)
    X, Y = (torch.randn(B, n, 3, generator=g, device=DEV) * 10 for _ in range(2))
    Xm, Ym = (M.dist(c[:, :, None], c[:, None]).float() for c in (torch.randn(B, n, 3, generator=g, device=DEV) * 8,
                                                                 torch.randn(B, n, 3, generator=g, device=DEV) * 8))
    if shared == "a":
        X, Xm = X[:1].contiguous(), Xm[:1].contiguous()
    elif shared == "b":
        Y, Ym = Y[:1].contiguous(), Ym[:1].contiguous()
    mbuf = torch.rand(B, n, n + 3, generator=g, device=DEV) > 0.4     # row stride n + 3
    mask = mbuf[:, :, :n]
    mask_u8 = mbuf.to(torch.uint8)[:, :, :n]
    a, b = (Xm if a_mat else X), (Ym if b_mat else Y)
    variants = [(2.0, None, None), (1.0, mask, None), (0.5, None, (-3.0, 4.0)), (3.0, mask, (-3.0, 4.0))]
    for q, m, clamp in variants:
        lo, hi = clamp if clamp else (float("-inf"), float("inf"))
        mk = None if m is None else mask_u8
        got = _loss_run(a, a_mat, b, b_mat, mk, B, n, lo, hi, q, 0xFF)
        again = _loss_run(a, a_mat, b, b_mat, mk, B, n, lo, hi, q, 0x00)
        assert torch.equal(_bits(got), _bits(again)), "a poisoned workspace changed the loss"
        kw = dict(X=None if a_mat else X.expand(B, n, 3), X_mat=Xm.expand(B, n, n) if a_mat else None,
                  Y=None if b_mat else Y.expand(B, n, 3), Y_mat=Ym.expand(B, n, n) if b_mat else None, q=q,
                  distmat_mask=m, clamp=clamp)
        ref = M.distmat_loss(**kw)                                    # B > 1 everywhere: the oracle's squeeze keeps [B, n, 3]
        terms = B * n * n if m is None else int(m.sum())
        bound = 1.01 * (U + (2 * terms + 70) * E53) * ref.abs()
        tag = f"metrics/loss/{shape}/{'mat' if a_mat else 'xyz'}_{'mat' if b_mat else 'xyz'}_shared{shared}/q{q}" \
              f"{'_mask' if m is not None else ''}{'_clamp' if clamp else ''}"
        check_bound(tag, got, ref.reshape(1), bound.reshape(1))
    empty = torch.zeros(B, n, n, dtype=torch.uint8, device=DEV)
    assert torch.isnan(_loss_run(a, a_mat, b, b_mat, empty, B, n, float("-inf"), float("inf"), 2.0, 0xFF)).all()


# ------------------------------------------------------------------------------------------------------------------------
# superposition and scores
# ------------------------------------------------------------------------------------------------------------------------
def _superpose_run(x, y, mask, align, shift, fill, rot_fill=0.0):
    """x, y [B, n, 3] fp32; x is passed in the [B, 3, n] layout.  mask [B, n] bool (passed with mask_sn 2) or None.  xo / yo are
    windows [:, 1:n + 1, 1:4] of NaN buffers [B, n + 3, 5]."""
    B, n, _ = x.shape
    xt = x.transpose(1, 2).contiguous()
    yc = y.contiguous()
    mptr, msb, msn = 0, 0, 0
    if mask is not None:
        mbuf = torch.zeros(B, n, 2, dtype=torch.uint8, device=DEV)
        mbuf[:, :, 0] = mask.to(torch.uint8)
        mbuf[:, :, 1] = 1 - mbuf[:, :, 0]
        mptr, msb, msn = mbuf.data_ptr(), 2 * n, 2
    xo = torch.full((B, n + 3, 5), float("nan"), device=DEV)
    yo = torch.full_like(xo, float("nan"))
    win = 5 + 1                                                       # element [0, 1, 1] of the buffer
    rot = _guarded(9 * B, torch.float64, rot_fill)
    rmsd, tm, g0, g1 = _guarded(B), _guarded(B), _guarded(B), _guarded(B)
    cut = (C.c_float * 8)(*CUTS)
    specs = (_L().GdtSpec * 2)()
    for k, (out, (idx, w)) in enumerate(zip((g0, g1), GDT_SPECS)):
        specs[k].out, specs[k].k = out.data_ptr(), len(idx)
        for j, (i, wj) in enumerate(zip(idx, w)):
            specs[k].idx[j], specs[k].w[j] = i, wj
    ws = _ws(B, n, fill)
    rc = _rc("af2_superpose_scores", _pts(xt, 0, 3 * n, 1, n), _pts(yc, 0, 3 * n, 3, 1), mptr, msb, msn, B, n, int(align),
             int(shift), _pts(xo, win, (n + 3) * 5, 5, 1), _pts(yo, win, (n + 3) * 5, 5, 1), rot.data_ptr() if align else None,
             rmsd.data_ptr(), tm.data_ptr(), len(CUTS), cut, specs, 0, None, None, ws.data_ptr(), ws.numel())
    assert rc == 0, _lib().af2_last_error()
    torch.cuda.synchronize()
    for t in (rmsd, tm, g0, g1):
        assert torch.isnan(t[B:]).all(), "guard written"
    assert (rot[9 * B:] == rot_fill).all(), "rot guard written"
    inside = torch.zeros(B, n + 3, 5, dtype=torch.bool, device=DEV)
    inside[:, 1:n + 1, 1:4] = True
    assert torch.isnan(xo[~inside]).all() and torch.isnan(yo[~inside]).all(), "xo / yo written outside their window"
    return dict(xo=xo[:, 1:n + 1, 1:4], yo=yo[:, 1:n + 1, 1:4], rot=rot[:9 * B].view(B, 3, 3), rmsd=rmsd[:B], tm=tm[:B],
                gdt=(g0[:B], g1[:B]))


def _gdt_fp32(counts, nsel):
    """the kernel's fp32 GDT sum, bitwise: s += fl(count_k / n_sel) * w_k (w a power of two: the product is exact), then s / K"""
    outs = []
    for idx, w in GDT_SPECS:
        s = np.float32(0.0)
        for i, wk in zip(idx, w):
            s = np.float32(s + np.float32(np.float32(counts[i]) / np.float32(nsel)) * np.float32(wk))
        outs.append(np.float32(s / np.float32(len(idx))))
    return outs


def _rotation_class(P, T):
    """oracle Kabsch in fp64 on the selected points -> (U, S, fixed, unique)"""
    Xc = P - P.mean(-1, keepdim=True)
    Yc = T - T.mean(-1, keepdim=True)
    V, S, W = torch.linalg.svd(Xc @ Yc.t())
    fixed = bool(torch.det(V) * torch.det(W) < 0)
    _, _, Uo, _ = M.kabsch(P, T)
    gap = (S[1] - S[2]) if fixed else (S[1] + S[2])
    unique = bool(S[0] > 0 and gap > 1e-4 * S[0])
    return Uo, S, fixed, unique


def _check_superpose(tag, x, y, mask, align, shift):
    """-> per element: "empty", "given" (align 0) or (unique or ambiguous, determinant fix applied)"""
    B, n, _ = x.shape
    out = _superpose_run(x, y, mask, align, shift, 0xFF)
    again = _superpose_run(x, y, mask, align, shift, 0x00)
    for k in ("xo", "yo", "rot", "rmsd", "tm"):
        assert torch.equal(_bits(out[k].contiguous()), _bits(again[k].contiguous())), f"{tag}: poisoned workspace changed {k}"
    for g, h in zip(out["gdt"], again["gdt"]):
        assert torch.equal(_bits(g), _bits(h)), f"{tag}: poisoned workspace changed gdt"
    # the scores on the fp32 points the kernel scored: with shift, xo holds them moved by cy, so take them from an unshifted run
    pts = out
    if shift:
        pts = _superpose_run(x, y, mask, align, False, 0xFF)
        for k in ("rmsd", "tm", "rot"):
            assert torch.equal(_bits(out[k].contiguous()), _bits(pts[k].contiguous())), f"{tag}: shift changed {k}"
    classes = []
    x64, y64 = x.double(), y.double()
    for e in range(B):
        sel = torch.ones(n, dtype=torch.bool, device=DEV) if mask is None else mask[e]
        nsel = int(sel.sum())
        et = f"{tag}/e{e}_nsel{nsel}"
        scores = [out["rmsd"][e], out["tm"][e], out["gdt"][0][e], out["gdt"][1][e]]
        if nsel == 0:
            assert all(torch.isnan(s) for s in scores), f"{et}: scores of an empty element are not NaN"
            if align:
                assert torch.isnan(out["rot"][e]).all(), f"{et}: rot of an empty element is not NaN"
                assert torch.isnan(out["xo"][e]).all(), f"{et}: aligned x of an empty element is not NaN"
            classes.append("empty")
            continue
        P, T = x64[e][sel].t(), y64[e][sel].t()
        if align:
            R = out["rot"][e]
            I3 = torch.eye(3, dtype=torch.float64, device=DEV)
            assert (R @ R.t() - I3).abs().max() <= 1e-12 and abs(float(torch.det(R)) - 1) <= 1e-12, f"{et}: not a rotation"
            Uo, S, fixed, unique = _rotation_class(P, T)
            classes.append(("unique" if unique else "ambiguous", fixed))
            if unique:
                err = float((R - Uo).abs().max())
                assert err <= 1e-9, f"{et}: rotation differs from the oracle's by {err:.3e}"
            cx, cy = P.mean(-1), T.mean(-1)
            ecx = 2 * (nsel + 16) * E53 * P.abs().max()
            ecy = 2 * (nsel + 16) * E53 * T.abs().max()
            xc = x64[e] - cx
            ax = xc @ R                                               # row i: U^T (x_i - cx)
            ref_x = ax + cy if shift else ax
            bx = (U * ref_x.abs() + 3 * ecx + 8 * E53 * ((xc.abs() @ R.abs()) + cy.abs()) + ecy)
            check_bound(f"{et}/xo", out["xo"][e], ref_x, bx)
            ref_y = y64[e] - cy
            check_bound(f"{et}/yo", out["yo"][e], ref_y, U * ref_y.abs() + ecy + 2.0 ** -52 * ref_y.abs())
        else:
            assert torch.equal(_bits(out["xo"][e].contiguous()), _bits(x[e])) and \
                torch.equal(_bits(out["yo"][e].contiguous()), _bits(y[e])), f"{et}: unaligned points not copied"
            classes.append("given")
        X32, Y32 = pts["xo"][e][sel], pts["yo"][e][sel]
        d = M.dist(X32, Y32)
        counts = [int((d <= c).sum()) for c in CUTS]
        for g, want in zip(out["gdt"], _gdt_fp32(counts, nsel)):
            assert g[e].item() == float(want), f"{et}: GDT {g[e].item()} != {float(want)}"
        rmsd_ref = (d * d).sum() / (3 * nsel)
        rmsd_ref = rmsd_ref.sqrt()
        check_bound(f"{et}/rmsd", out["rmsd"][e:e + 1], rmsd_ref.reshape(1),
                    (1.01 * (U + (nsel + 40) * E53) * rmsd_ref).reshape(1))
        d0 = M.tm_d0(nsel)
        t = 1.0 / (1.0 + (d / d0) ** 2)
        tm_ref = t.mean()
        e_d0 = 4 * E53 * (abs(d0) + 3.6) / abs(d0)
        btm = U * tm_ref.abs() + (nsel + 40) * E53 * tm_ref + ((2 * e_d0 + 4 * E53) * t).mean()
        check_bound(f"{et}/tm", out["tm"][e:e + 1], tm_ref.reshape(1), btm.reshape(1))
        if align and classes[-1][0] == "ambiguous":
            A, Bc, _, _ = M.kabsch(P, T)
            opt = M.rmsd(A.float()[None], Bc.float()[None])[0]
            scale = max(float(A.abs().max()), float(Bc.abs().max()), 1e-30)
            err = abs(out["rmsd"][e].item() - opt.item())
            assert err <= 4 * U * scale + 2.0 ** -40 * scale, f"{et}: RMSD {out['rmsd'][e].item()} is not the minimum {opt.item()}"
    return classes


def _selection(B_sizes, n, seed):
    g = _gen(seed)
    mask = torch.zeros(len(B_sizes), n, dtype=torch.bool, device=DEV)
    for e, k in enumerate(B_sizes):
        mask[e, torch.randperm(n, generator=g, device=DEV)[:k]] = True
    return mask


@pytest.mark.parametrize("align,shift,masked", [(1, 0, True), (1, 1, True), (0, 0, True), (1, 0, False)])
@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 1000])
def test_superpose_scores_vs_fp64(n, align, shift, masked):
    """elements with 0, 1, 2, 3 and all n points selected (a strided mask), or every point without a mask"""
    sizes = sorted({min(k, n) for k in (0, 1, 2, 3, n)}) if masked else [n, n]
    pred, true = _structures(len(sizes), n, seed=n * 3 + align + 2 * shift)
    mask = _selection(sizes, n, seed=n) if masked else None
    _check_superpose(f"metrics/superpose/n{n}/align{align}_shift{shift}_{'mask' if masked else 'nomask'}", pred, true, mask,
                     align, shift)


def test_kabsch_hard_cases():
    """a planar set (C of rank 2), a collinear one (rank 1), a rotated cube (three equal singular values: the polar factor is
    still unique) and an exact mirror image (the determinant fix applies), 8 points each"""
    g = _gen(8)
    n = 8
    Q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, device=DEV, dtype=torch.float64))
    if torch.det(Q) < 0:
        Q[:, 0] = -Q[:, 0]
    planar = torch.randn(n, 3, generator=g, device=DEV) * 5
    planar[:, 2] = 0
    line = torch.zeros(n, 3, device=DEV)
    line[:, 0] = torch.randn(n, generator=g, device=DEV) * 5
    cube = torch.tensor([[sx, sy, sz] for sx in (-1.0, 1.0) for sy in (-1.0, 1.0) for sz in (-1.0, 1.0)], device=DEV) * 3 + 1
    generic = torch.randn(n, 3, generator=g, device=DEV) * torch.tensor([6.0, 3.0, 1.5], device=DEV)
    true = torch.stack([planar, line, cube, generic], 0)
    pred = (true.double() @ Q).float()
    pred[3] = (true[3].double() * torch.tensor([1.0, 1.0, -1.0], device=DEV, dtype=torch.float64) @ Q).float()
    for shift in (0, 1):
        classes = _check_superpose(f"metrics/kabsch_hard/shift{shift}", pred + 2.0, true, None, 1, shift)
        assert [c[0] for c in classes] == ["unique", "ambiguous", "unique", "unique"], classes
        assert not classes[2][1] and classes[3][1], "the cube needs no determinant fix, the mirror image does"


def test_superpose_rot_refused_without_align():
    """rot with align = 0 has no rotation to receive: AF2_ERR_BAD_ARG before any launch, rot untouched"""
    B, n = 2, 10
    x, y = _structures(B, n, seed=1)
    rot = _guarded(9 * B, torch.float64, 0.0)
    rmsd = _guarded(B)
    ws = _ws(B, n, 0xFF)
    n0 = _launches()
    rc = _rc("af2_superpose_scores", _pts(x, 0, 3 * n, 3, 1), _pts(y, 0, 3 * n, 3, 1), None, 0, 0, B, n, 0, 0, None, None,
             rot.data_ptr(), rmsd.data_ptr(), None, 0, None, None, 0, None, None, ws.data_ptr(), ws.numel())
    torch.cuda.synchronize()
    assert rc == BAD_ARG, rc
    assert _launches() == n0, "launched before refusing"
    assert (rot == 0).all() and torch.isnan(rmsd).all(), "wrote before refusing"
