"""Mirror of the distogram-to-coordinates chain of alphafold2_pytorch/utils.py: center_distogram_torch (utils.py:718-764),
mds_torch / mdscaling_torch / MDScaling (utils.py:766-833, 1162-1181, 1256-1282) and the phi-angle mirror check
(calc_phis_torch, get_dihedral_torch, utils.py:881-957).

The centring runs as one kernel over the distogram and the SMACOF loop as one cooperative launch that keeps every iteration
on the device (csrc/geometry.cuh).  Return values, shapes and the reference's numerical quirks are kept (DESIGN.md §14).
Differences: per-iteration lines are printed after the loop from the recorded history, the mirror check stays on the
device, and inputs the reference would crash on raise ValueError before any device work.  ``coords_from_distogram`` is
one addition: distogram logits straight to coordinates.

The structure scores of utils.py:999-1247 (kabsch_torch / Kabsch, rmsd_torch / RMSD, gdt_torch / GDT, tmscore_torch /
TMscore, lddt_ca_torch, distmat_loss_torch) run as two kernels (csrc/metrics.cuh): a pass over the pairs for lDDT and the
loss, and one CTA per structure for the superposition and the per-point scores.  Names, layouts, return dtypes and the
reference's quirks are kept (DESIGN.md §4d); ``score_coords`` scores a batch of predictions in the model's layout.

The distogram loss of the reference's training script (train_pre.py:76-90) and its labels, get_bucketed_distance_matrix
(utils.py:45-50), run as one pass over the logits and a fixed-order finish (csrc/distogram_loss.cuh, DESIGN.md §4e).
The angle heads are scored the same way against the trRosetta orientations of the true backbone (csrc/angle_loss.cuh,
DESIGN.md §4f).
"""
import numbers
from dataclasses import dataclass

import torch

from . import ops
from .alphafold2 import DISTOGRAM_BUCKETS, OMEGA_BUCKETS, PHI_BUCKETS, THETA_BUCKETS, _forward_only

__all__ = ["DISTANCE_THRESHOLDS", "center_distogram_torch", "mds_torch", "mdscaling_torch", "get_dihedral_torch",
           "calc_phis_torch", "MDScaling", "coords_from_distogram", "kabsch_torch", "Kabsch", "rmsd_torch", "RMSD",
           "gdt_torch", "GDT", "tmscore_torch", "TMscore", "lddt_ca_torch", "distmat_loss_torch", "StructureScores",
           "score_coords", "get_bucketed_distance_matrix", "distogram_loss", "get_bucketed_angle_matrices", "AngleLoss",
           "angle_loss"]

DISTANCE_THRESHOLDS = torch.linspace(2, 20, steps=DISTOGRAM_BUCKETS)


def _batched(t: torch.Tensor, dims: int, name: str) -> torch.Tensor:
    """expand_dims_to (utils.py:63-66): one leading batch dimension added to a (dims - 1)-D tensor."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if t.dim() == dims - 1:
        t = t.reshape(1, *t.shape)
    if t.dim() != dims:
        raise ValueError(f"{name} must be {dims - 1}-D or {dims}-D, got shape {tuple(t.shape)}")
    return t


def _square(t: torch.Tensor, name: str) -> torch.Tensor:
    t = _batched(t, 3, name)
    if t.shape[1] != t.shape[2]:
        raise ValueError(f"{name} must be [b, N, N], got {tuple(t.shape)}")
    if not 1 <= t.shape[1] <= ops.MDS_MAX_N:
        raise ValueError(f"MDS takes 1 to {ops.MDS_MAX_N} points, got {t.shape[1]}")
    return t


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().float().contiguous()


def center_distogram_torch(distogram, bins=DISTANCE_THRESHOLDS, min_t=1., center="mean", wide="std"):
    """utils.py:718-764 -- (central, weights), each [b, N, N] fp32, from distogram [b, N, N, B] (or [N, N, B]) probabilities.
    center "mean" or "median"; wide "std", "var" or anything else for no dispersion.  min_t is unused, as in the reference."""
    distogram = _batched(distogram, 4, "distogram")
    return ops.center_distogram(_f32(distogram), bins, center=center, wide=wide)


def _smacof(pre, weights, iters, tol, verbose, init=None):
    """The init (unless given) and the on-device loop; prints the reference's per-iteration lines from the history."""
    x = ops.mds_init(pre) if init is None else init
    k, stopped, his, stress = ops.mds_iterate_(pre, weights, x, iters, tol)
    if verbose:
        for i in range(k + stopped):
            if verbose >= 2:
                print('it: %d, stress %s' % (i, stress[i].float()))
        if stopped:
            print('breaking at iteration %d with stress %s' % (k, his[k + 1].float()))
    return x, his[:k + 1].float()


def _check_mds_args(pre_dist_mat, weights):
    pre = _square(pre_dist_mat, "pre_dist_mat")
    if not pre.is_cuda:
        raise RuntimeError("pre_dist_mat must be a CUDA tensor (alphafold2_b200 has no CPU fallback)")
    if weights is not None:
        weights = _batched(weights, 3, "weights")
        if weights.shape != pre.shape:
            raise ValueError(f"weights must have the shape of pre_dist_mat {tuple(pre.shape)}, got {tuple(weights.shape)}")
    return pre, weights


def mds_torch(pre_dist_mat, weights=None, iters=10, tol=1e-5, eigen=False, verbose=2):
    """utils.py:766-833 -- weighted MDS of the distance matrix pre_dist_mat [b, N, N] (or [N, N]) -> (coords [b, 3, N],
    history [steps + 1, b]), his[0] = inf.  eigen without weights: the init and a zero history [1, b]."""
    pre, weights = _check_mds_args(pre_dist_mat, weights)
    pre = _f32(pre)
    if weights is None and eigen:
        x = ops.mds_init(pre)
        return x.transpose(-1, -2), torch.zeros(1, pre.shape[0], device=pre.device)
    if eigen and verbose:
        print("Can't use eigen flag if weights are active. Fallback to iterative")
    x, his = _smacof(pre, None if weights is None else _f32(weights), int(iters), tol, verbose)
    return x.transpose(-1, -2), his


def get_dihedral_torch(c1, c2, c3, c4):
    """utils.py:881-898 -- dihedral angle in radians of the points c1..c4 [..., 3] (atan2 form)."""
    u1 = c2 - c1
    u2 = c3 - c2
    u3 = c4 - c3
    return torch.atan2(((torch.norm(u2, dim=-1, keepdim=True) * u1) * torch.cross(u2, u3, dim=-1)).sum(dim=-1),
                       (torch.cross(u1, u2, dim=-1) * torch.cross(u2, u3, dim=-1)).sum(dim=-1))


def _backbone_index(N_mask, CA_mask, C_mask, n):
    """Point indices of the N, CA and C atoms from batch element 0's masks; C defaults to neither N nor CA."""
    if N_mask is None or CA_mask is None:
        raise ValueError("fix_mirror needs N_mask and CA_mask")
    masks = [_batched(torch.as_tensor(m), 2, name)[0].bool() for m, name in ((N_mask, "N_mask"), (CA_mask, "CA_mask"))]
    masks.append(~(masks[0] | masks[1]) if C_mask is None else _batched(torch.as_tensor(C_mask), 2, "C_mask")[0].bool())
    for m, name in zip(masks, ("N_mask", "CA_mask", "C_mask")):
        if m.shape[0] != n:
            raise ValueError(f"{name} must have {n} entries, one per point, got {m.shape[0]}")
    idx = [torch.nonzero(m).view(-1) for m in masks]
    counts = {int(i.numel()) for i in idx}
    if len(counts) != 1 or counts.pop() < 2:
        raise ValueError(f"the N, CA and C masks must select the same number (at least 2) of points, got "
                         f"{[int(i.numel()) for i in idx]}")
    return idx


def calc_phis_torch(pred_coords, N_mask, CA_mask, C_mask=None, prop=True, verbose=0):
    """utils.py:917-957 -- backbone phi angles of pred_coords [b, 3, N], the atoms picked by batch element 0's masks.
    prop: the fraction of negative phis per element [b]; otherwise a list of [residues - 1] angle tensors.  On the device."""
    x = pred_coords.detach().transpose(-1, -2)
    n_i, ca_i, c_i = (i.to(x.device) for i in _backbone_index(N_mask, CA_mask, C_mask, x.shape[1]))
    n_t, ca_t, c_t = x[:, n_i], x[:, ca_i], x[:, c_i]
    phis = get_dihedral_torch(c_t[:, :-1], n_t[:, 1:], ca_t[:, 1:], c_t[:, 1:])
    if prop:
        return (phis < 0).float().mean(dim=-1)
    return list(phis)


def mdscaling_torch(pre_dist_mat, weights=None, iters=10, tol=1e-5, fix_mirror=True, N_mask=None, CA_mask=None, C_mask=None,
                    eigen=False, verbose=2):
    """utils.py:1162-1181 -- mds_torch, then with fix_mirror the z row of every element with fewer than half its phi angles
    negative is negated (the mirror image of a backbone has the opposite phi signs)."""
    pre, _ = _check_mds_args(pre_dist_mat, weights)
    if fix_mirror:
        _backbone_index(N_mask, CA_mask, C_mask, pre.shape[-1])
    preds, stresses = mds_torch(pre, weights=weights, iters=iters, tol=tol, eigen=eigen, verbose=verbose)
    if not fix_mirror:
        return preds, stresses
    flip = calc_phis_torch(preds, N_mask, CA_mask, C_mask, prop=True) < 0.5
    preds[:, -1] = torch.where(flip[:, None], -preds[:, -1], preds[:, -1])
    if verbose == 2:
        print("Corrected mirror idxs:", torch.nonzero(flip).view(-1))
    return preds, stresses


def MDScaling(pre_dist_mat, **kwargs):
    """utils.py:1256-1282 -- mdscaling_torch on pre_dist_mat [b, N, N] or [N, N].  backend "torch" or "auto"; the numpy
    backend is not provided."""
    backend = kwargs.pop("backend", "auto")
    if backend == "auto":
        backend = "torch" if isinstance(pre_dist_mat, torch.Tensor) else "numpy"
    if backend != "torch":
        raise NotImplementedError(f"MDScaling: only the torch backend runs here (got {backend!r})")
    return mdscaling_torch(_batched(pre_dist_mat, 3, "pre_dist_mat"), **kwargs)


def coords_from_distogram(distance_logits, mask=None, iters=10, tol=1e-5, center="mean", wide="std"):
    """Coordinates straight from Alphafold2's distogram logits ``ret.distance`` [b, N, N, buckets] (or [N, N, buckets]): the
    centring with the softmax on chip (no softmaxed copy of the logits), the bins torch.linspace(2, 20, buckets), pairs with
    a masked residue (mask [b, N] bool) at weight 0, then weighted MDS.  Returns (coords [b, N, 3], history [steps + 1, b]).
    No mirror fix: a residue-level distogram has no backbone atoms."""
    logits = _batched(distance_logits, 4, "distance_logits")
    b, n, n2, nb = logits.shape
    if n != n2 or not 1 <= n <= ops.MDS_MAX_N:
        raise ValueError(f"distance_logits must be [b, N, N, buckets] with 1 <= N <= {ops.MDS_MAX_N}, got {tuple(logits.shape)}")
    if mask is not None:
        mask = _batched(torch.as_tensor(mask), 2, "mask")
    bins = torch.linspace(2, 20, steps=nb)
    central, weights = ops.center_distogram(_f32(logits), bins, center=center, wide=wide, softmax=True, mask=mask)
    return _smacof(central, weights, int(iters), tol, 0)


# --------------------------------------------------------------------------------------------------
# structure scores (utils.py:999-1247)
# --------------------------------------------------------------------------------------------------
GDT_TS_CUTOFFS = (1, 2, 4, 8)
GDT_HA_CUTOFFS = (0.5, 1, 2, 4)


def _scored(t, name: str) -> torch.Tensor:
    """The fp32 tensor the kernels read (a view when t is already fp32); CPU tensors and autograd inputs are refused."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (alphafold2_b200 has no CPU fallback)")
    if not t.is_floating_point():
        raise TypeError(f"{name} must be a floating tensor, got {t.dtype}")
    _forward_only(t)
    return t.detach() if t.dtype == torch.float32 else t.detach().float()


def _bdn(X, Y):
    """expand_arg_dims (utils.py:68-81): A, B of equal rank, [3, N] -> [1, 3, N]; then [B, 3, N] with N >= 1."""
    if not isinstance(X, torch.Tensor) or not isinstance(Y, torch.Tensor):
        raise TypeError("A and B must be torch.Tensors")
    if X.dim() != Y.dim():
        raise ValueError(f"Shapes of A and B must match: {tuple(X.shape)} and {tuple(Y.shape)}")
    if X.dim() == 2:
        X, Y = X[None], Y[None]
    if X.dim() != 3 or X.shape != Y.shape or X.shape[1] != 3:
        raise ValueError(f"A and B must both be [B, 3, N] or [3, N], got {tuple(X.shape)} and {tuple(Y.shape)}")
    if X.shape[-1] == 0:
        raise ValueError("A and B have no points")
    return X, Y


def _backend(A, backend):
    if backend == "auto":
        backend = "torch" if isinstance(A, torch.Tensor) else "numpy"
    if backend != "torch":
        raise NotImplementedError(f"only the torch backend runs here (got {backend!r})")


def kabsch_torch(X, Y, cpu=True):
    """utils.py:999-1029 -- Kabsch alignment of X into Y, both [3, N] -> (X centred and rotated, Y centred), each [3, N].
    C = X_ Y_^T = V S W; when det V det W < 0 the last column of V is negated; U = V W; X_aligned = U^T X_.  The covariance
    and the SVD are fp64 on the device; ``cpu`` is accepted and has no effect (nothing goes to the host)."""
    if not isinstance(X, torch.Tensor) or not isinstance(Y, torch.Tensor):
        raise TypeError("X and Y must be torch.Tensors")
    if X.dim() != 2 or X.shape != Y.shape or X.shape[0] != 3:
        raise ValueError(f"X and Y must both be [3, N], got {tuple(X.shape)} and {tuple(Y.shape)}")
    if X.shape[1] == 0:
        raise ValueError("X and Y have no points")
    x, y = _scored(X, "X"), _scored(Y, "Y")
    n = X.shape[1]
    ax = torch.empty(3, n, dtype=torch.float32, device=x.device)
    ay = torch.empty_like(ax)
    ops.superpose_scores(x.t()[None], y.t()[None], 1, n, align=True, out_x=ax.t()[None], out_y=ay.t()[None])
    return ax.to(X.dtype), ay.to(Y.dtype)


def Kabsch(A, B, backend="auto"):
    """utils.py:1281-1294 -- kabsch_torch on A, B [3, N].  Only 2-D input: any other rank raises ValueError."""
    _backend(A, backend)
    if not isinstance(B, torch.Tensor) or A.dim() != B.dim():
        raise ValueError("Shapes of A and B must match.")
    return kabsch_torch(A, B)


def _scores(X, Y, *, rmsd=False, tm=False, cutoffs=(), weights=None):
    """One superpose_scores launch over [B, 3, N] pairs as given (no alignment)."""
    X, Y = _bdn(X, Y)
    x, y = _scored(X, "X"), _scored(Y, "Y")
    b, n = X.shape[0], X.shape[2]
    new = lambda: torch.empty(b, dtype=torch.float32, device=x.device)  # noqa: E731
    out = {"rmsd": new() if rmsd else None, "tm": new() if tm else None, "gdt": new() if cutoffs else None}
    gdt = ()
    if cutoffs:
        gdt = ((out["gdt"], range(len(cutoffs)), [1.0] * len(cutoffs) if weights is None else weights),)
    ops.superpose_scores(x.transpose(1, 2), y.transpose(1, 2), b, n, rmsd=out["rmsd"], tm=out["tm"], cutoffs=cutoffs, gdt=gdt)
    return out


def rmsd_torch(X, Y):
    """utils.py:1098-1100 -- sqrt of the mean of (X - Y)^2 over both the 3 and the N axes (the usual RMSD over sqrt 3), for
    X, Y [B, 3, N] (or [3, N]) -> [B] in X's dtype."""
    return _scores(X, Y, rmsd=True)["rmsd"].to(X.dtype)


def RMSD(A, B, backend="auto"):
    """utils.py:1296-1308 -- rmsd_torch on [B, 3, N] or [3, N] -> [B]."""
    _backend(A, backend)
    return rmsd_torch(A, B)


def gdt_torch(X, Y, cutoffs, weights=None):
    """utils.py:1106-1123 -- sum_k w_k GDT_k / K with GDT_k the fraction of points with |X - Y| <= cutoffs[k] (not normalised
    by the weights: it can exceed 1), X, Y [B, 3, N] (or [3, N]) -> [B] fp32.  weights: K numbers or None for ones."""
    cutoffs = [float(c) for c in cutoffs]
    if not 1 <= len(cutoffs) <= ops.MAX_CUTOFFS:
        raise ValueError(f"GDT takes 1 to {ops.MAX_CUTOFFS} cutoffs, got {len(cutoffs)}")
    if weights is not None:
        weights = [float(w) for w in (weights.tolist() if isinstance(weights, torch.Tensor) else weights)]
        if len(weights) != len(cutoffs):
            raise ValueError(f"{len(weights)} GDT weights for {len(cutoffs)} cutoffs")
    return _scores(X, Y, cutoffs=cutoffs, weights=weights)["gdt"]


def GDT(A, B, *, mode="TS", cutoffs=[1, 2, 4, 8], weights=None, backend="auto"):  # noqa: B006 (the reference's signature)
    """utils.py:1310-1327 -- gdt_torch with the cutoffs of ``mode``: "HA" / "ha" 0.5, 1, 2, 4, anything else 1, 2, 4, 8.
    The ``cutoffs`` argument is ignored, as in the reference."""
    _backend(A, backend)
    return gdt_torch(A, B, GDT_HA_CUTOFFS if mode in ["HA", "ha"] else GDT_TS_CUTOFFS, weights=weights)


def tmscore_torch(X, Y):
    """utils.py:1143-1150 -- mean of 1 / (1 + (d / d0)^2), L = max(15, N), d0 = 1.24 (L - 15)^(1/3) - 1.8 without a lower
    clamp (negative for N <= 18), on the points as given (no superposition search), X, Y [B, 3, N] -> [B] in X's dtype."""
    return _scores(X, Y, tm=True)["tm"].to(X.dtype)


def TMscore(A, B, backend="auto"):
    """utils.py:1329-1344 -- tmscore_torch on [B, 3, N] or [3, N] -> [B]."""
    _backend(A, backend)
    return tmscore_torch(A, B)


def _bool_mask(mask, shape, name, device):
    if not isinstance(mask, torch.Tensor):
        mask = torch.as_tensor(mask)
    if mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"{name} must be a bool mask, got {mask.dtype}")
    if tuple(mask.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(mask.shape)}")
    return mask.to(device=device, dtype=torch.bool)


def lddt_ca_torch(true_coords, pred_coords, cloud_mask, r_0=15.):
    """utils.py:1204-1247 -- lDDT of each C-alpha (atom 1) of sidechainnet-layout coordinates [b, L, C, 3] with cloud_mask
    [b, L, C] -> [b, L] in true_coords' dtype.  Only CAs present in the mask take part.  Residue i: the pairs with a true
    distance < r_0 (itself included) each score #{t in 0.5, 1, 2, 4 : |d_pred - d_true| <= t}; lddt = (sum - 4) /
    (4 count - 4) in fp32.  A residue without a CA scores 0; one with no other CA within r_0 scores NaN."""
    for t, name in ((true_coords, "true_coords"), (pred_coords, "pred_coords")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
    if true_coords.dim() != 4 or true_coords.shape != pred_coords.shape or true_coords.shape[-1] != 3:
        raise ValueError(f"true_coords and pred_coords must both be [b, L, C, 3], got {tuple(true_coords.shape)} and "
                         f"{tuple(pred_coords.shape)}")
    b, n, c, _ = true_coords.shape
    if c < 2:
        raise ValueError(f"lddt_ca_torch reads the CA as atom 1: C must be at least 2, got {c}")
    if n == 0 or b == 0:
        raise ValueError("true_coords has no residues")
    t, p = _scored(true_coords, "true_coords"), _scored(pred_coords, "pred_coords")
    cm = _bool_mask(cloud_mask, (b, n, c), "cloud_mask", t.device)
    lddt = torch.empty(b, n, dtype=torch.float32, device=t.device)
    ca = cm[:, :, 1]
    ops.superpose_scores(None, None, b, n, mask=ca, mask_strides=ca.stride(), lddt=lddt,
                         lddt_points=(t[:, :, 1], p[:, :, 1]), r0=float(r_0))
    return lddt.to(true_coords.dtype)


def _loss_operand(coords, mat, name):
    """-> (fp32 view [Bx, N, 3] or [Bx, N, N], is_matrix, rank of the distance matrix the reference builds, dtype)."""
    if mat is None:
        if not isinstance(coords, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
        t = coords.squeeze()
        if t.dim() not in (2, 3) or t.shape[-1] != 3:
            raise ValueError(f"{name} must be [N, 3] or [B, N, 3] after squeeze(), got {tuple(coords.shape)}")
        return t if t.dim() == 3 else t[None], False, t.dim(), coords.dtype
    if not isinstance(mat, torch.Tensor):
        raise TypeError(f"{name}_mat must be a torch.Tensor")
    if mat.dim() not in (2, 3) or mat.shape[-1] != mat.shape[-2]:
        raise ValueError(f"{name}_mat must be [N, N] or [B, N, N], got {tuple(mat.shape)}")
    return mat if mat.dim() == 3 else mat[None], True, mat.dim(), mat.dtype


def distmat_loss_torch(X=None, Y=None, X_mat=None, Y_mat=None, p=2, q=2, custom=None, distmat_mask=None, clamp=None):
    """utils.py:1057-1096 -- mean over the True entries of distmat_mask (all of them by default, diagonal included, across
    the batch) of ((D_X - D_Y)^2)^(q / 2).  Each operand is coordinates X [N, 3] / [B, N, 3] (squeeze() applied, clamp
    clamping the coordinates) whose Euclidean distances are computed on the fly, or a distance matrix X_mat [N, N] /
    [B, N, N].  Returns a 0-d tensor.  No N x N matrix is built."""
    if (X is None and X_mat is None) or (Y is None and Y_mat is None):
        raise ValueError("The true and predicted coords or dist mats must be provided")
    if custom is not None:
        raise NotImplementedError("distmat_loss_torch: a custom loss is a Python callable, which cannot run inside the kernel")
    if (X_mat is None or Y_mat is None) and p != 2:
        raise NotImplementedError(f"distmat_loss_torch: only the Euclidean distance (p=2) is built, got p={p}")
    a, a_mat, a_rank, a_dtype = _loss_operand(X, X_mat, "X")
    b, b_mat, b_rank, b_dtype = _loss_operand(Y, Y_mat, "Y")
    n = a.shape[1]
    if b.shape[1] != n or n == 0:
        raise ValueError(f"the two operands must have the same N >= 1, got {tuple(a.shape)} and {tuple(b.shape)}")
    if a.shape[0] != b.shape[0] and 1 not in (a.shape[0], b.shape[0]):
        raise ValueError(f"batch sizes {a.shape[0]} and {b.shape[0]} do not broadcast")
    B = max(a.shape[0], b.shape[0])
    shape = (B, n, n) if max(a_rank, b_rank) == 3 else (n, n)
    va, vb = _scored(a, "X"), _scored(b, "Y")
    if a_mat and va.stride(-1) != 1:
        va = va.contiguous()
    if b_mat and vb.stride(-1) != 1:
        vb = vb.contiguous()
    mask = None
    if distmat_mask is not None:
        mask = _bool_mask(distmat_mask, shape, "distmat_mask", va.device).reshape(B, n, n)
    lo, hi = (float("-inf"), float("inf")) if clamp is None else clamp
    lo = float("-inf") if lo is None else float(lo)
    hi = float("inf") if hi is None else float(hi)
    out = ops.distmat_loss(va, a_mat, vb, b_mat, B, n, mask=mask, lo=lo, hi=hi, q=float(q))
    return out.to(torch.promote_types(a_dtype, b_dtype))


@dataclass
class StructureScores:
    """score_coords' result.  rmsd, gdt_ts, gdt_ha, tm_score, lddt_mean [b]; lddt [b, N]; aligned [b, N, 3]."""
    rmsd: torch.Tensor
    gdt_ts: torch.Tensor
    gdt_ha: torch.Tensor
    tm_score: torch.Tensor
    lddt: torch.Tensor
    lddt_mean: torch.Tensor
    aligned: torch.Tensor


def score_coords(pred, true, mask=None) -> StructureScores:
    """Score predicted coordinates against the true structure, per element of the batch: pred, true [b, N, 3] (or [N, 3]),
    mask [b, N] bool selecting the residues S to score (all when None).  The composition of the mirrors on S:
    ``A, B = Kabsch(pred[S].T, true[S].T)``; ``rmsd = RMSD(A, B)`` (the reference's: it divides by 3N, so it is the usual
    RMSD over sqrt 3); ``gdt_ts = GDT(A, B)``, ``gdt_ha = GDT(A, B, mode="HA")``; ``tm_score = TMscore(A, B)`` (the
    reference's formula on the RMSD-optimal superposition, not the TM-score program's search); ``lddt`` = lddt_ca_torch
    over S with 0 outside S; ``lddt_mean`` the mean of the finite lddt over S.  ``aligned`` is the whole predicted chain
    moved by the superposition fitted on S, in the true structure's frame.  An element with no selected residue gets NaN.
    Two kernel launches."""
    if not isinstance(pred, torch.Tensor) or not isinstance(true, torch.Tensor):
        raise TypeError("pred and true must be torch.Tensors")
    if pred.dim() == 2 and true.dim() == 2:
        pred, true = pred[None], true[None]
        if mask is not None and isinstance(mask, torch.Tensor) and mask.dim() == 1:
            mask = mask[None]
    if pred.dim() != 3 or pred.shape != true.shape or pred.shape[-1] != 3:
        raise ValueError(f"pred and true must both be [b, N, 3] or [N, 3], got {tuple(pred.shape)} and {tuple(true.shape)}")
    b, n, _ = pred.shape
    if n == 0 or b == 0:
        raise ValueError("pred has no residues")
    x, y = _scored(pred, "pred"), _scored(true, "true")
    m = None if mask is None else _bool_mask(mask, (b, n), "mask", x.device)
    dev = x.device
    new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
    rmsd, ts, ha, tm, lddt, mean, aligned = new(b), new(b), new(b), new(b), new(b, n), new(b), new(b, n, 3)
    ops.superpose_scores(x, y, b, n, mask=m, mask_strides=(0, 0) if m is None else m.stride(), align=True, shift=True,
                         out_x=aligned, rmsd=rmsd, tm=tm, cutoffs=GDT_TS_CUTOFFS + (0.5,),
                         gdt=((ts, (0, 1, 2, 3), (1.0,) * 4), (ha, (4, 0, 1, 2), (1.0,) * 4)), lddt=lddt, lddt_mean=mean,
                         lddt_points=(y, x))
    dt = pred.dtype
    return StructureScores(rmsd.to(dt), ts, ha, tm.to(dt), lddt.to(dt), mean.to(dt), aligned.to(dt))


# --------------------------------------------------------------------------------------------------
# distogram loss (train_pre.py:76-90 with get_bucketed_distance_matrix, utils.py:45-50)
# --------------------------------------------------------------------------------------------------
def _ignore_index(ignore_index) -> int:
    if isinstance(ignore_index, bool) or not isinstance(ignore_index, numbers.Integral):
        raise TypeError(f"ignore_index must be an integer, got {type(ignore_index).__name__}")
    if not -2 ** 63 <= int(ignore_index) < 2 ** 63:
        raise ValueError(f"ignore_index {int(ignore_index)} does not fit in int64")
    return int(ignore_index)


def _checked(t, name: str) -> torch.Tensor:
    """_scored's refusals (not a tensor, on the CPU, not floating, requires grad) without its conversion."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (alphafold2_b200 has no CPU fallback)")
    if not t.is_floating_point():
        raise TypeError(f"{name} must be a floating tensor, got {t.dtype}")
    _forward_only(t)
    return t


def _label_args(coords, mask, b=None, n=None, device=None):
    """Refusals of coords [b, N, c] and mask [b, N] bool (or None); nothing is converted or launched."""
    _checked(coords, "coords")
    if coords.dim() != 3 or coords.shape[-1] < 1:
        raise ValueError(f"coords must be [b, N, c] with c >= 1, got {tuple(coords.shape)}")
    if coords.shape[0] == 0 or coords.shape[1] == 0:
        raise ValueError(f"coords has no residues: {tuple(coords.shape)}")
    if b is not None and tuple(coords.shape[:2]) != (b, n):
        raise ValueError(f"coords must be [{b}, {n}, c] to match the distogram, got {tuple(coords.shape)}")
    if device is not None and coords.device != device:
        raise RuntimeError(f"coords are on {coords.device}, distance_logits on {device}")
    if mask is not None:
        if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool:
            raise TypeError(f"mask must be a bool tensor, got {getattr(mask, 'dtype', type(mask).__name__)}")
        if tuple(mask.shape) != tuple(coords.shape[:2]):
            raise ValueError(f"mask must have shape {tuple(coords.shape[:2])}, got {tuple(mask.shape)}")
        if mask.device != coords.device:
            raise RuntimeError(f"mask is on {mask.device}, coords on {coords.device}")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    return (t.detach() if t.dtype == torch.float32 else t.detach().float()).contiguous()


def get_bucketed_distance_matrix(coords, mask, num_buckets=DISTOGRAM_BUCKETS, ignore_index=-100):
    """utils.py:45-50 -- the distogram labels: int64 [b, N, N] for coords [b, N, c] and mask [b, N] bool (or [N, N] for [N, c]
    and [N]; mask None: every residue present).  Label = ignore_index where either residue is masked, otherwise the bucket of
    |coords_i - coords_j| under torch.linspace(2, 20, num_buckets)[:-1] (torch.bucketize, right=False: a distance on an edge
    goes below it, NaN to num_buckets - 1).  The distance is the direct one in fp32, as the recycling embedder takes it: above
    25 points the reference's torch.cdist uses |a|^2 + |b|^2 - 2 a.b, which can put a pair near an edge into the next bucket
    (DESIGN.md §2).  One kernel launch."""
    flat = isinstance(coords, torch.Tensor) and coords.dim() == 2
    if flat:
        coords = coords[None]
        mask = mask[None] if isinstance(mask, torch.Tensor) and mask.dim() == 1 else mask
    ii = _ignore_index(ignore_index)
    if isinstance(num_buckets, bool) or not isinstance(num_buckets, numbers.Integral) or num_buckets < 1:
        raise ValueError(f"num_buckets must be a positive integer, got {num_buckets!r}")
    _label_args(coords, mask)
    labels = ops.bucketed_distance(_f32c(coords), None if mask is None else mask.contiguous(), int(num_buckets), ii)
    return labels[0] if flat else labels


def _xent_args(distance_logits, coords, mask, ignore_index, rows=None):
    """The checks both loss entries share, all before any device work -> (logits, coords, mask, ignore_index) as the kernels
    read them.  rows: the number of pair rows distance_logits must hold (the whole N when None)."""
    ii = _ignore_index(ignore_index)
    _checked(distance_logits, "distance_logits")
    shape = tuple(distance_logits.shape)
    if len(shape) != 4 or shape[-1] < 1 or (rows is None and shape[1] != shape[2]):
        raise ValueError(f"distance_logits must be [b, N, N, buckets] with buckets >= 1, got {shape}")
    b, r, n, nb = shape
    if b == 0 or n == 0:
        raise ValueError(f"distance_logits has no pairs: {shape}")
    if rows is not None and r != rows:
        raise ValueError(f"distance_rows must hold this rank's {rows} pair rows of N = {n}, got {shape}")
    if nb > ops.XENT_MAX_BINS:
        raise ValueError(f"the distogram loss kernel takes at most {ops.XENT_MAX_BINS} buckets, got {nb}")
    _label_args(coords, mask, b, n, distance_logits.device)
    return _f32c(distance_logits), _f32c(coords), None if mask is None else mask.contiguous(), ii


def distogram_loss(distance_logits, coords, mask=None, ignore_index=-100):
    """The reference's distogram training loss (train_pre.py:76-90) in two kernel launches with no host synchronisation:
        labels = get_bucketed_distance_matrix(coords, mask, buckets, ignore_index)
        F.cross_entropy(rearrange(distance_logits, 'b i j c -> b c i j'), labels, ignore_index=ignore_index)
    for distance_logits [b, N, N, buckets] (Alphafold2's ret.distance), coords [b, N, c] (the C-alpha coordinates) and mask
    [b, N] bool or None (every residue counts).  The mean runs over every pair of the batch whose label is not ignore_index,
    diagonal included; an in-range ignore_index also drops the pairs in that bucket, and NaN is returned when nothing counts.
    No label matrix and no softmaxed copy of the logits is made: the extra device memory is 16 bytes per (element, row).
    Returns a 0-d fp32 tensor on the logits' device.  The labels are get_bucketed_distance_matrix's; each term is the fp32
    log-sum-exp minus the label's logit, summed in fp64 in a fixed order (DESIGN.md §4e), so the result is reproducible bit
    for bit and equal to parallel.distogram_loss_rows on the same distogram sharded by rows."""
    logits, x, m, ii = _xent_args(distance_logits, coords, mask, ignore_index)
    return ops.distogram_xent_finish(ops.distogram_xent_rows(logits, x, m, ii))


# --------------------------------------------------------------------------------------------------
# angle-head labels and loss (the trRosetta inter-residue orientations, DESIGN.md §4f)
# --------------------------------------------------------------------------------------------------
ANGLE_HEADS = ("theta", "phi", "omega")


@dataclass
class AngleLoss:
    """angle_loss's result: each head's mean cross-entropy over its counted pairs, a 0-d fp32 tensor on the logits' device."""
    theta: torch.Tensor
    phi: torch.Tensor
    omega: torch.Tensor


def _backbone_args(backbone, mask, b=None, n=None, device=None):
    """Refusals of backbone [b, N, A, 3] (A >= 3) and mask [b, N] bool (or None); nothing is converted or launched."""
    _checked(backbone, "backbone")
    if backbone.dim() != 4 or backbone.shape[-1] != 3 or backbone.shape[2] < 3:
        raise ValueError(f"backbone must be [b, N, A, 3] with A >= 3 (atoms N, CA, C first), got {tuple(backbone.shape)}")
    if backbone.shape[0] == 0 or backbone.shape[1] == 0:
        raise ValueError(f"backbone has no residues: {tuple(backbone.shape)}")
    if b is not None and tuple(backbone.shape[:2]) != (b, n):
        raise ValueError(f"backbone must be [{b}, {n}, A, 3] to match the angle logits, got {tuple(backbone.shape)}")
    if device is not None and backbone.device != device:
        raise RuntimeError(f"backbone is on {backbone.device}, the angle logits on {device}")
    if mask is not None:
        if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool:
            raise TypeError(f"mask must be a bool tensor, got {getattr(mask, 'dtype', type(mask).__name__)}")
        if tuple(mask.shape) != tuple(backbone.shape[:2]):
            raise ValueError(f"mask must have shape {tuple(backbone.shape[:2])}, got {tuple(mask.shape)}")
        if mask.device != backbone.device:
            raise RuntimeError(f"mask is on {mask.device}, backbone on {backbone.device}")


def _bucket_count(nb, name: str) -> int:
    if isinstance(nb, bool) or not isinstance(nb, numbers.Integral) or nb < 2:
        raise ValueError(f"{name} needs at least 2 buckets (one angular bin and no contact), got {nb!r}")
    return int(nb)


def get_bucketed_angle_matrices(backbone, mask, num_buckets=(THETA_BUCKETS, PHI_BUCKETS, OMEGA_BUCKETS), ignore_index=-100):
    """The angle heads' labels: the trRosetta orientations theta, phi and omega of every residue pair, bucketed, for backbone
    [b, N, A, 3] (A >= 3; atoms 0, 1, 2 are N, CA, C, sidechainnet's order, so the reference's 14-atom layout passes as it is)
    and mask [b, N] bool or None (every residue present); [N, A, 3] and [N] give [N, N].  Returns (theta, phi, omega), each
    int64 [b, N, N].  In fp64 on the fp32 atoms: the virtual CB of every residue, a contact is i != j with |CB_i - CB_j| <=
    20 A, and for a contact theta = dihedral(N_i, CA_i, CB_i, CB_j), omega = dihedral(CA_i, CB_i, CB_j, CA_j) in [-pi, pi] and
    phi = angle(CA_i, CB_i, CB_j) in [0, pi].  A head of nb buckets has nb - 1 bins of equal width (torch.bucketize, right=False:
    an angle on an edge goes below it) and puts no contact (the diagonal, farther pairs, missing atoms) in the last bucket,
    nb - 1; a pair with a masked residue gets ignore_index.  One kernel launch."""
    flat = isinstance(backbone, torch.Tensor) and backbone.dim() == 3
    if flat:
        backbone = backbone[None]
        mask = mask[None] if isinstance(mask, torch.Tensor) and mask.dim() == 1 else mask
    ii = _ignore_index(ignore_index)
    if not isinstance(num_buckets, (tuple, list)) or len(num_buckets) != 3:
        raise ValueError(f"num_buckets must be three bucket counts (theta, phi, omega), got {num_buckets!r}")
    nb = tuple(_bucket_count(v, h) for v, h in zip(num_buckets, ANGLE_HEADS))
    _backbone_args(backbone, mask)
    labels = ops.bucketed_angles(_f32c(backbone), None if mask is None else mask.contiguous(), nb, ii)
    return tuple(t[0] for t in labels) if flat else labels


def _angle_args(theta_logits, phi_logits, omega_logits, backbone, mask, ignore_index, rows=None):
    """The checks angle_loss and parallel.angle_loss_rows share, all before any device work -> (theta, phi, omega, backbone,
    mask, ignore_index) as the kernels read them.  rows: the number of pair rows the logits must hold (the whole N when None)."""
    ii = _ignore_index(ignore_index)
    heads = (theta_logits, phi_logits, omega_logits)
    for t, h in zip(heads, ANGLE_HEADS):
        _checked(t, f"{h}_logits")
    shape = tuple(theta_logits.shape)
    if len(shape) != 4 or (rows is None and shape[1] != shape[2]):
        raise ValueError(f"theta_logits must be [b, N, N, buckets], got {shape}")
    b, r, n, _ = shape
    if b == 0 or n == 0:
        raise ValueError(f"theta_logits has no pairs: {shape}")
    if rows is not None and r != rows:
        raise ValueError(f"the angle logits must hold this rank's {rows} pair rows of N = {n}, got {shape}")
    for t, h in zip(heads, ANGLE_HEADS):
        if t.dim() != 4 or tuple(t.shape[:3]) != (b, r, n):
            raise ValueError(f"{h}_logits must be [{b}, {r}, {n}, buckets] like theta_logits, got {tuple(t.shape)}")
        if t.device != theta_logits.device:
            raise RuntimeError(f"{h}_logits are on {t.device}, theta_logits on {theta_logits.device}")
        _bucket_count(t.shape[-1], f"{h}_logits")
    nbs = sum(t.shape[-1] for t in heads)
    if nbs > ops.XENT_MAX_BINS:
        raise ValueError(f"the angle loss kernel takes at most {ops.XENT_MAX_BINS} buckets over the three heads, got {nbs}")
    _backbone_args(backbone, mask, b, n, theta_logits.device)
    return (*(_f32c(t) for t in heads), _f32c(backbone), None if mask is None else mask.contiguous(), ii)


def _angle_result(losses: torch.Tensor) -> AngleLoss:
    return AngleLoss(losses[0], losses[1], losses[2])


def angle_loss(theta_logits, phi_logits, omega_logits, backbone, mask=None, ignore_index=-100) -> AngleLoss:
    """The angle heads scored against a true structure in two kernel launches with no host synchronisation: for each head,
        F.cross_entropy(rearrange(logits, 'b i j c -> b c i j'), labels, ignore_index=ignore_index)
    with (theta, phi, omega) labels = get_bucketed_angle_matrices(backbone, mask, (their bucket counts), ignore_index), for
    the logits [b, N, N, nb_h] of Alphafold2(predict_angles=True) (ret.theta_logits, ret.phi_logits, ret.omega_logits; each
    nb_h >= 2), backbone [b, N, A, 3] and mask [b, N] bool or None.  The F.cross_entropy conventions of distogram_loss hold:
    the diagonal counts (as no contact), an in-range ignore_index also drops that bucket, NaN when nothing counts.  No label
    matrix and no softmaxed copy is made: the extra device memory is 48 bytes per (element, row).  Returns an AngleLoss whose
    .theta, .phi and .omega are 0-d fp32 tensors on the logits' device, reproducible bit for bit and equal to
    parallel.angle_loss_rows on the same logits sharded by rows."""
    *heads, x, m, ii = _angle_args(theta_logits, phi_logits, omega_logits, backbone, mask, ignore_index)
    return _angle_result(ops.angle_xent_finish(ops.angle_xent_rows(*heads, x, m, ii)))
