"""Time the structure scores (alphafold2_b200.utils, csrc/metrics.cuh) against the eager torch lines they replace.

    python tools/time_metrics.py                     # b 1 x N 256 / 1024 / 4096 / 8192, and b 64 x N 512 (a decoy set)
    python tools/time_metrics.py --shapes 1x2048

One JSON line per measurement; the first names the card and its power limit (nvidia-smi), read in the same run.
  score_coords        all scores of a batch (two launches), ms per call (CUDA events around --reps calls after a warm-up).
                      eager: the reference's lines made runnable on the GPU (kabsch_torch with the covariance on the
                      device, gdt_torch with its weights on the device, tmscore_torch, rmsd_torch and lddt_ca_torch with
                      the cloud mask on the device), one element at a time as the reference's Kabsch takes one structure.
  lddt_ca_torch       C = 4 atoms per residue; pairs_per_s = b N^2 over the call time.  eager: the reference's loop.
  distmat_loss_torch  coordinates [b, N, 3]; pairs_per_s as above.  eager: the reference's two cdist matrices.
  kabsch_cpu          the reference's kabsch_torch with its default cpu=True host round trip, one element.
  peak_gb: peak memory allocated by the call beyond what was allocated before it.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, (torch.cuda.max_memory_allocated() - base) / 1e9


# ---- the reference's lines (alphafold2_pytorch/utils.py), with the host round trips and CPU tensors moved to the device ----
def eager_kabsch(X, Y, cpu=False):
    X_ = X - X.mean(dim=-1, keepdim=True)
    Y_ = Y - Y.mean(dim=-1, keepdim=True)
    C = torch.matmul(X_, Y_.t())
    if cpu:
        C = C.cpu()
    V, S, W = torch.linalg.svd(C)
    if (torch.det(V) * torch.det(W)) < 0.0:
        V[:, -1] = V[:, -1] * (-1)
    U = torch.matmul(V, W).to(X.device)
    return torch.matmul(X_.t(), U).t(), Y_


def eager_gdt(X, Y, cutoffs):
    weights = torch.ones(1, len(cutoffs), device=X.device)
    GDT = torch.zeros(X.shape[0], len(cutoffs), device=X.device)
    dist = ((X - Y) ** 2).sum(dim=1).sqrt()
    for i, cutoff in enumerate(cutoffs):
        GDT[:, i] = (dist <= cutoff).float().mean(dim=-1)
    return (GDT * weights).mean(-1)


def eager_tm(X, Y):
    L = max(15, X.shape[-1])
    d0 = 1.24 * (L - 15) ** (1 / 3) - 1.8
    dist = ((X - Y) ** 2).sum(dim=1).sqrt()
    return (1 / (1 + (dist / d0) ** 2)).mean(dim=-1)


def eager_lddt(true_coords, pred_coords, cloud_mask, r_0=15.):
    device, dtype = true_coords.device, true_coords.type()
    thresholds = torch.tensor([0.5, 1, 2, 4], device=device).type(dtype)
    cloud_mask = cloud_mask.bool()
    c_alpha_mask = torch.zeros(cloud_mask.shape[1:], device=device).bool()
    c_alpha_mask[..., 1] = True
    wrapper = torch.zeros(true_coords.shape[:2], device=device).type(dtype)
    for bi, seq in enumerate(true_coords):
        c_alphas = cloud_mask[bi] * c_alpha_mask
        selected_pred = pred_coords[bi, c_alphas, :]
        selected_target = true_coords[bi, c_alphas, :]
        dist_mat_pred = torch.cdist(selected_pred, selected_pred, p=2)
        dist_mat_target = torch.cdist(selected_target, selected_target, p=2)
        under_r0_target = dist_mat_target < r_0
        compare_dists = torch.abs(dist_mat_pred - dist_mat_target)[under_r0_target]
        score = torch.zeros_like(under_r0_target).float()
        max_score = torch.zeros_like(under_r0_target).float()
        max_score[under_r0_target] = 4.
        score[under_r0_target] = thresholds.shape[0] - torch.bucketize(compare_dists, boundaries=thresholds).float()
        l_mask = c_alphas.float().sum(dim=-1).bool()
        wrapper[bi, l_mask] = (score.sum(dim=-1) - thresholds.shape[0]) / (max_score.sum(dim=-1) - thresholds.shape[0])
    return wrapper


def eager_loss(X, Y):
    X_mat, Y_mat = torch.cdist(X, X, p=2), torch.cdist(Y, Y, p=2)
    mask = torch.ones_like(Y_mat).bool()
    return ((X_mat - Y_mat) ** 2)[mask].mean()


def eager_scores(pred, true, cloud_mask):
    for e in range(pred.shape[0]):
        A, B = eager_kabsch(pred[e].t(), true[e].t())
        A, B = A[None], B[None]
        torch.sqrt(torch.mean((A - B) ** 2, axis=(-1, -2)))
        eager_gdt(A, B, [1, 2, 4, 8])
        eager_gdt(A, B, [0.5, 1, 2, 4])
        eager_tm(A, B)
    tc = torch.stack([true] * 4, 2)
    eager_lddt(tc, torch.stack([pred] * 4, 2), cloud_mask)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["1x256", "1x1024", "1x4096", "1x8192", "64x512"])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_metrics.py measures on the GPU: no CUDA device found")
    from alphafold2_b200 import utils as U

    print(json.dumps({"card": _card(), "torch_name": torch.cuda.get_device_name()}), flush=True)
    for shape in args.shapes:
        b, n = (int(v) for v in shape.split("x"))
        torch.manual_seed(0)
        true = torch.cumsum(torch.nn.functional.normalize(torch.randn(b, n, 3, device="cuda"), dim=-1) * 3.8, 1)
        pred = true + torch.randn(b, n, 3, device="cuda")
        mask = torch.ones(b, n, dtype=torch.bool, device="cuda")
        tc, pc = torch.stack([true] * 4, 2), torch.stack([pred] * 4, 2)
        cm = torch.ones(b, n, 4, dtype=torch.bool, device="cuda")
        pairs = b * n * n
        runs = {
            "score_coords": (lambda: U.score_coords(pred, true, mask), lambda: eager_scores(pred, true, cm)),
            "lddt_ca_torch": (lambda: U.lddt_ca_torch(tc, pc, cm), lambda: eager_lddt(tc, pc, cm)),
            "distmat_loss_torch": (lambda: U.distmat_loss_torch(X=pred, Y=true), lambda: eager_loss(pred, true)),
        }
        for what, (kernel, eager) in runs.items():
            ms, peak = _timed(kernel, args.reps)
            rec = {"what": what, "path": "kernel", "b": b, "n": n, "ms": round(ms, 4), "peak_gb": round(peak, 4)}
            if what != "score_coords":
                rec["pairs_per_s"] = float(f"{pairs / ms * 1e3:.3e}")
            print(json.dumps(rec), flush=True)
            try:
                ms_e, peak_e = _timed(eager, max(1, args.reps // 10))
                print(json.dumps({"what": what, "path": "eager", "b": b, "n": n, "ms": round(ms_e, 4), "peak_gb": round(peak_e, 4),
                                  "speedup": round(ms_e / ms, 1)}), flush=True)
            except torch.OutOfMemoryError:
                print(json.dumps({"what": what, "path": "eager", "b": b, "n": n, "result": "out of memory"}), flush=True)
            torch.cuda.empty_cache()
        ms, _ = _timed(lambda: U.Kabsch(pred[0].t(), true[0].t()), args.reps)
        ms_c, _ = _timed(lambda: eager_kabsch(pred[0].t(), true[0].t(), cpu=True), args.reps)
        print(json.dumps({"what": "kabsch", "b": 1, "n": n, "kernel_ms": round(ms, 4), "eager_cpu_true_ms": round(ms_c, 4),
                          "speedup": round(ms_c / ms, 1)}), flush=True)


if __name__ == "__main__":
    main()
