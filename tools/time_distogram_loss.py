"""Time utils.distogram_loss against the reference's two eager lines (train_pre.py:76-90 with get_bucketed_distance_matrix,
utils.py:45-50, restated here on the device) at b 1, N 1024 / 2048 / 4096 and b 16, N 512.

    python tools/time_distogram_loss.py [--sizes 1x1024,1x2048,1x4096,16x512] [--iters 20] [--cpu-dry-run]

Per size: the median time of each path from CUDA events, the GB/s of algorithmic traffic (logits + coordinates + mask, read
once), the bandwidth floor at 3.35 TB/s (H100 SXM data sheet), and the peak device memory above the inputs.  Prints the card
name and power limit.  --cpu-dry-run builds the inputs at a tiny size and runs the eager lines on the CPU, then stops: it
checks the script without a device and measures nothing."""
import argparse
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BW = 3.35e12
NB = 37


def eager(logits, coords, mask, ignore_index=-100):
    """the reference's lines: cdist labels, masked_fill, then cross_entropy of the permuted distogram"""
    distances = torch.cdist(coords, coords, p=2)
    boundaries = torch.linspace(2, 20, steps=logits.shape[-1], device=coords.device)
    labels = torch.bucketize(distances, boundaries[:-1])
    labels.masked_fill_(~(mask[..., None] & mask[..., None, :]), ignore_index)
    return F.cross_entropy(logits.permute(0, 3, 1, 2), labels, ignore_index=ignore_index)


def inputs(b, n, device):
    g = torch.Generator(device=device).manual_seed(n)
    logits = torch.randn(b, n, n, NB, device=device, generator=g)
    coords = torch.randn(b, n, 3, device=device, generator=g) * 15
    mask = torch.rand(b, n, device=device, generator=g) > 0.05
    return logits, coords, mask


def traffic(b, n):
    return b * n * n * NB * 4 + b * n * 3 * 4 + b * n


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
        logits, coords, mask = inputs(2, 16, "cpu")
        print(f"dry run: eager loss {eager(logits, coords, mask).item():.6f} at b 2, N 16; traffic at the timed sizes "
              + ", ".join(f"{b}x{n}: {traffic(b, n) / 1e9:.3f} GB" for b, n in sizes) + "; nothing measured")
        return
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure (use --cpu-dry-run to check the script)")
    from alphafold2_b200 import utils
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi: {q.stdout.strip() or q.stderr.strip()}")
    print(f"{'b x N':>9} {'kernel ms':>10} {'GB/s':>7} {'floor ms':>9} {'x floor':>8} {'peak MB':>8} | {'eager ms':>9} {'peak MB':>8} "
          f"{'speed-up':>8} {'|diff|':>9}")
    for b, n in sizes:
        logits, coords, mask = inputs(b, n, "cuda")
        ours = lambda: utils.distogram_loss(logits, coords, mask)  # noqa: E731
        ref = lambda: eager(logits, coords, mask)  # noqa: E731
        diff = abs(ours().item() - ref().item())
        t_k, t_e = timed(ours, a.iters), timed(ref, max(3, a.iters // 4))
        m_k, m_e = peak_above(ours), peak_above(ref)
        byt = traffic(b, n)
        floor = byt / PEAK_BW * 1e3
        print(f"{b:>3} x {n:<4} {t_k:>10.3f} {byt / t_k / 1e6:>7.0f} {floor:>9.3f} {t_k / floor:>8.2f} {m_k / 2**20:>8.2f} | "
              f"{t_e:>9.3f} {m_e / 2**20:>8.1f} {t_e / t_k:>8.1f} {diff:>9.2e}")
        del logits, coords, mask
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
