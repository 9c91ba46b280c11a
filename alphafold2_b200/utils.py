"""Mirror of the distogram-to-coordinates chain of alphafold2_pytorch/utils.py: center_distogram_torch (utils.py:718-764),
mds_torch / mdscaling_torch / MDScaling (utils.py:766-833, 1162-1181, 1256-1282) and the phi-angle mirror check
(calc_phis_torch, get_dihedral_torch, utils.py:881-957).

The centring runs as one kernel over the distogram and the SMACOF loop as one cooperative launch that keeps every iteration
on the device (csrc/geometry.cuh).  Return values, shapes and the reference's numerical quirks are kept (DESIGN.md §14).
Differences: per-iteration lines are printed after the loop from the recorded history, the mirror check stays on the
device, and inputs the reference would crash on raise ValueError before any device work.  ``coords_from_distogram`` is
the one addition: distogram logits straight to coordinates.
"""
import torch

from . import ops
from .alphafold2 import DISTOGRAM_BUCKETS

__all__ = ["DISTANCE_THRESHOLDS", "center_distogram_torch", "mds_torch", "mdscaling_torch", "get_dihedral_torch",
           "calc_phis_torch", "MDScaling", "coords_from_distogram"]

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
