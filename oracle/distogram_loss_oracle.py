"""TEST INFRASTRUCTURE ONLY -- plain-torch statement of the reference's distogram loss (train_pre.py:76-90) and of its labels,
get_bucketed_distance_matrix (alphafold2_pytorch/utils.py:45-50), on CPU or GPU tensors.

The label of each pair is the kernels' fp32 decision emulated exactly: fp32 coordinate differences, squares summed by a
correctly rounded fp32 fma over the coordinates in order (``fmaf32``), a correctly rounded fp32 sqrt, then torch.bucketize
(right=False) over the first nb - 1 edges of the fp32 torch.linspace(2, 20, nb).  So oracle and kernels agree on every
label, edges and NaN included, and the loss below differs from the kernels' only by their fp32 arithmetic.  The reference's
torch.cdist is the same direct distance up to 25 points; above that it takes |a|^2 + |b|^2 - 2 a.b, and the fixture keeps
those distances 0.05 A from every edge (oracle/make_golden_r11.py).

``loss64`` is the cross-entropy in fp64 on the fp32 logits; ``term_bound`` is the worst-case error of the kernels' fp32
term, derived in its docstring (tests/test_oracle_distogram_loss.py holds its controls).
It must never be imported by ``alphafold2_b200``."""
import torch

U32 = 2.0 ** -24


def fmaf32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fp32 a * b + c with one rounding (IEEE fmaf), for fp32 tensors.  a * b is exact in fp64; the fp64 sum hi and its error
    lo (TwoSum) hold a * b + c exactly, and rounding hi to fp32 is the single rounding except when hi is an fp32 midpoint,
    where lo decides the direction."""
    p = a.double() * b.double()
    cd = c.double()
    hi = p + cd
    bb = hi - p
    lo = (p - (hi - bb)) + (cd - bb)
    r = hi.float()
    toward = torch.where(hi > r.double(), torch.full_like(r, float("inf")), torch.full_like(r, float("-inf")))
    other = torch.nextafter(r, toward)
    mid = (r.double() + other.double()) * 0.5
    tie = (hi == mid) & (lo != 0) & torch.isfinite(hi)
    # at a midpoint the exact value lies on lo's side of it
    up = torch.maximum(r, other)
    down = torch.minimum(r, other)
    return torch.where(tie, torch.where(lo > 0, up, down), r)


def boundaries(nb: int, device=None) -> torch.Tensor:
    """utils.py:47 -- the fp32 bucket edges; the first nb - 1 are searched."""
    return torch.linspace(2, 20, steps=nb, device=device)


def direct_dist32(coords: torch.Tensor) -> torch.Tensor:
    """[b, n, c] -> [b, n, n] fp32: differences in fp32, fmaf over c in order, sqrt (the kernels' distance, bit for bit)."""
    x = coords.float()
    s2 = torch.zeros(x.shape[0], x.shape[1], x.shape[1], dtype=torch.float32, device=x.device)
    for e in range(x.shape[-1]):
        d = x[:, :, None, e] - x[:, None, :, e]
        s2 = fmaf32(d, d, s2)
    return s2.sqrt()


def labels(coords: torch.Tensor, mask, nb: int, ignore_index: int = -100) -> torch.Tensor:
    """get_bucketed_distance_matrix with the kernels' distance: int64 [b, n, n]; ignore_index where either residue is masked."""
    lab = torch.bucketize(direct_dist32(coords), boundaries(nb, coords.device)[:-1])
    if mask is not None:
        lab = lab.masked_fill(~(mask[..., None] & mask[..., None, :]), ignore_index)
    return lab


def counted(lab: torch.Tensor, ignore_index: int) -> torch.Tensor:
    return lab != ignore_index


def terms64(logits: torch.Tensor, lab: torch.Tensor, ignore_index: int) -> torch.Tensor:
    """fp64 logsumexp(l) - l[label] of the fp32 logits [b, n, n, nb] at the counted pairs (a 1-D tensor, row-major order)."""
    keep = counted(lab, ignore_index)
    l = logits.double()[keep]
    y = lab[keep]
    return torch.logsumexp(l, -1) - l.gather(-1, y[:, None])[:, 0]


def loss64(logits: torch.Tensor, lab: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    """F.cross_entropy(logits.permute(0, 3, 1, 2), lab, ignore_index) in fp64: the mean of terms64, NaN when nothing counts."""
    t = terms64(logits, lab, ignore_index)
    return t.sum() / t.numel() if t.numel() else torch.tensor(float("nan"), dtype=torch.float64)


def term_bound(logits: torch.Tensor, lab: torch.Tensor, ignore_index: int) -> torch.Tensor:
    """Worst-case |fp32 kernel term - fp64 term| at each counted pair, from the kernel's rounding points (u = 2^-24):
      x_c = fl(l_c - m)             |dx_c| <= u |l_c - m|
      expf(x_c)                     <= 2 ulp: relative 4u
      s = sum_c in fp32             (nb - 1) u relative
        -> s = S (1 + rho),  |rho| <= sum_c p_c u |l_c - m| + 4u + (nb - 1) u  (p = softmax(l), to first order)
      logf(s)                       |ln(1 + rho)| plus 1 ulp, 2u |ln s|
      fl(m + ln s), fl(. - l_y)     u |m + ln s| + u |term|
    with a 1 % margin for the second-order terms."""
    keep = counted(lab, ignore_index)
    l = logits.double()[keep]
    y = lab[keep]
    nb = l.shape[-1]
    m = l.max(-1).values
    d = (l - m[:, None]).abs()
    p = torch.softmax(l, -1)
    rho = (p * d).nan_to_num(0.0).sum(-1) * U32 + (4 + nb - 1) * U32
    L = torch.logsumexp(l, -1) - m
    t = L + m - l.gather(-1, y[:, None])[:, 0]
    b = rho / (1 - rho) + 2 * U32 * L.abs() + U32 * (m + L).abs() + U32 * t.abs()
    return 1.01 * b


def loss_bound(logits: torch.Tensor, lab: torch.Tensor, ignore_index: int = -100) -> float:
    """Bound on |kernel loss - loss64|: the mean term bound, the fp64 sums (n 2^-52 of sum |t|), and the final fp32 rounding."""
    t = terms64(logits, lab, ignore_index)
    if t.numel() == 0:
        return 0.0
    b = term_bound(logits, lab, ignore_index)
    k = t.numel()
    mean = (t.sum() / k).abs().item()
    return (b.sum().item() + k * 2.0 ** -52 * t.abs().sum().item()) / k + 1.01 * U32 * mean + 1e-300
