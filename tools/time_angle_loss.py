"""Time utils.angle_loss against the eager lines it replaces (fp32 geometry, torch.bucketize and three F.cross_entropy calls)
at b 1, N 1024 / 2048 / 4096 and b 16, N 512.

    python tools/time_angle_loss.py [--sizes 1x1024,1x2048,1x4096,16x512] [--iters 20] [--cpu-dry-run]

Per size: the median time of each path from CUDA events, the GB/s of algorithmic traffic (the three heads' logits, 252 bytes
per pair, plus the backbone and mask, read once), the bandwidth floor at 3.35 TB/s (H100 SXM data sheet), and the peak
device memory above the inputs.  Prints the card name and power limit.  --cpu-dry-run builds the inputs at a tiny size and
runs the eager lines on the CPU, then stops: it checks the script without a device and measures nothing."""
import argparse
import math
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BW = 3.35e12
NB = (25, 13, 25)
A = 14


def _dihedral(c1, c2, c3, c4):
    u1, u2, u3 = c2 - c1, c3 - c2, c4 - c3
    c23 = torch.cross(u2, u3, dim=-1)
    return torch.atan2((u2.norm(dim=-1, keepdim=True) * u1 * c23).sum(-1), (torch.cross(u1, u2, dim=-1) * c23).sum(-1))


def eager(theta, phi, omega, bb, mask, ignore_index=-100):
    """the labels from the fp32 backbone as a user would write them, then one cross_entropy per head"""
    n_, ca, c = bb[:, :, 0], bb[:, :, 1], bb[:, :, 2]
    b, cc = ca - n_, c - ca
    cb = -0.58273431 * torch.cross(b, cc, dim=-1) + 0.56802827 * b - 0.54067466 * cc + ca
    N = bb.shape[1]
    I = lambda t: t[:, :, None].expand(-1, -1, N, -1)  # noqa: E731
    J = lambda t: t[:, None].expand(-1, N, -1, -1)  # noqa: E731
    contact = (torch.cdist(cb, cb) <= 20) & ~torch.eye(N, dtype=torch.bool, device=bb.device)
    v, w = I(ca) - I(cb), J(cb) - I(cb)
    ang = (_dihedral(I(n_), I(ca), I(cb), J(cb)),
           torch.atan2(torch.cross(v, w, dim=-1).norm(dim=-1), (v * w).sum(-1)),
           _dihedral(I(ca), I(cb), J(cb), J(ca)))
    keep = mask[..., None] & mask[..., None, :]
    out = []
    for a, lg, signed in zip(ang, (theta, phi, omega), (True, False, True)):
        K = lg.shape[-1] - 1
        edges = (torch.arange(1, K + 1, device=bb.device) * ((2 if signed else 1) * math.pi / K) - (math.pi if signed else 0)).float()
        lab = torch.bucketize(a, edges).masked_fill_(~contact, K).masked_fill_(~keep, ignore_index)
        out.append(F.cross_entropy(lg.permute(0, 3, 1, 2), lab, ignore_index=ignore_index))
    return out


def inputs(b, n, device):
    g = torch.Generator(device=device).manual_seed(n)
    logits = [torch.randn(b, n, n, k, device=device, generator=g) for k in NB]
    ca = torch.randn(b, n, 1, 3, device=device, generator=g) * 12
    bb = ca + torch.randn(b, n, A, 3, device=device, generator=g) * 1.5
    bb[:, :, 1:2] = ca
    mask = torch.rand(b, n, device=device, generator=g) > 0.05
    return logits, bb, mask


def traffic(b, n):
    return b * n * n * sum(NB) * 4 + b * n * 9 * 4 + b * n


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return sorted(ts)[len(ts) // 2]


def peak_above(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1x1024,1x2048,1x4096,16x512")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu-dry-run", action="store_true")
    a = ap.parse_args()
    sizes = [tuple(int(v) for v in s.split("x")) for s in a.sizes.split(",")]
    if a.cpu_dry_run:
        logits, bb, mask = inputs(2, 16, "cpu")
        print(f"dry run: eager losses {[round(t.item(), 6) for t in eager(*logits, bb, mask)]} at b 2, N 16; traffic at the "
              "timed sizes " + ", ".join(f"{b}x{n}: {traffic(b, n) / 1e9:.3f} GB" for b, n in sizes) + "; nothing measured")
        return
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure (use --cpu-dry-run to check the script)")
    from alphafold2_b200 import utils
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi: {q.stdout.strip() or q.stderr.strip()}")
    print(f"{'b x N':>9} {'kernel ms':>10} {'GB/s':>7} {'floor ms':>9} {'x floor':>8} {'peak MB':>8} | {'eager ms':>9} {'peak MB':>8} "
          f"{'speed-up':>8} {'max |diff|':>10}")
    for b, n in sizes:
        logits, bb, mask = inputs(b, n, "cuda")
        ours = lambda: utils.angle_loss(*logits, bb, mask)  # noqa: E731
        ref = lambda: eager(*logits, bb, mask)  # noqa: E731
        o, r = ours(), ref()
        diff = max(abs(x.item() - y.item()) for x, y in zip((o.theta, o.phi, o.omega), r))
        t_k, t_e = timed(ours, a.iters), timed(ref, max(3, a.iters // 4))
        m_k, m_e = peak_above(ours), peak_above(ref)
        byt = traffic(b, n)
        floor = byt / PEAK_BW * 1e3
        print(f"{b:>3} x {n:<4} {t_k:>10.3f} {byt / t_k / 1e6:>7.0f} {floor:>9.3f} {t_k / floor:>8.2f} {m_k / 2**20:>8.2f} | "
              f"{t_e:>9.3f} {m_e / 2**20:>8.1f} {t_e / t_k:>8.1f} {diff:>10.2e}")
        del logits, bb, mask, o, r
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
