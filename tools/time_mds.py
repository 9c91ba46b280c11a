"""Time the distogram-to-coordinates chain (alphafold2_b200.utils, csrc/geometry.cuh) against the eager torch lines it replaces.

    python tools/time_mds.py                       # N 256 / 1024 / 2048 / 4096, batch 1
    python tools/time_mds.py --n 2048 --iters 50

One JSON line per measurement; the first names the card and its power limit (nvidia-smi), read in the same run.
  center:  af2_center_distogram on [1, N, N, 37] fp32 logits (softmax on chip) and probabilities, ms per call (CUDA events
           around --reps calls after a warm-up), GB/s from the bytes the algorithm moves (N^2 (4 * 37 + 8): the distogram
           read once, central and weights written once), and floor_ms = those bytes at 3.35 TB/s (computed, not measured).
           eager: oracle.geometry_oracle.center_distogram run by torch on the same GPU.
  smacof:  the loop with tol=-inf so that exactly --iters iterations run, weighted and unweighted; ms per iteration
           (one call, CUDA events, minus nothing: the launch and the single step-count read are included) and GB/s from
           N^2 * 8 B (delta and w) or N^2 * 4 B per iteration.  eager: oracle.geometry_oracle.mds in fp32 on the GPU, which
           like the reference syncs the host once per iteration on the stop test.
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

HBM_TBS = 3.35            # H100 SXM data sheet, TB/s
NB = 37


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[256, 1024, 2048, 4096])
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--eager-iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_mds.py measures on the GPU: no CUDA device found")
    from alphafold2_b200 import ops
    from oracle import geometry_oracle as G

    print(json.dumps({"card": _card(), "torch_name": torch.cuda.get_device_name()}), flush=True)
    bins = torch.linspace(2, 20, NB)
    for n in args.n:
        torch.manual_seed(0)
        logits = torch.randn(1, n, n, NB, device="cuda")
        probs = logits.softmax(-1)
        nbytes = n * n * (4.0 * NB + 8.0)
        for label, x, sm in (("logits", logits, True), ("probs", probs, False)):
            ms, peak = _timed(lambda: ops.center_distogram(x, bins, softmax=sm), args.reps)
            print(json.dumps({"what": "center", "path": "kernel", "input": label, "n": n, "ms": round(ms, 4),
                              "gbs": round(nbytes / ms / 1e6, 1), "floor_ms": round(nbytes / HBM_TBS / 1e9, 4),
                              "peak_gb": round(peak, 3)}), flush=True)
        try:
            ms, peak = _timed(lambda: G.center_distogram(logits, bins, softmax=True), 3)
            print(json.dumps({"what": "center", "path": "eager", "input": "logits", "n": n, "ms": round(ms, 4),
                              "peak_gb": round(peak, 3)}), flush=True)
        except torch.OutOfMemoryError:
            print(json.dumps({"what": "center", "path": "eager", "n": n, "result": "out of memory"}), flush=True)
        del probs
        central, weights = ops.center_distogram(logits, bins, softmax=True)
        del logits
        central = torch.nan_to_num(central)
        init = ops.mds_init(central)
        for wl, w in (("weighted", weights), ("unweighted", None)):
            per_it = n * n * (8.0 if w is not None else 4.0)

            def kernel():
                x = init.clone()
                ops.mds_iterate_(central, w, x, args.iters, float("-inf"))
            ms, peak = _timed(kernel, 3)
            print(json.dumps({"what": "smacof", "path": "kernel", "weights": wl, "n": n, "iters": args.iters,
                              "ms_per_iter": round(ms / args.iters, 4), "gbs": round(per_it * args.iters / ms / 1e6, 1),
                              "floor_ms_per_iter": round(per_it / HBM_TBS / 1e9, 4), "peak_gb": round(peak, 3)}), flush=True)
            try:
                ms, peak = _timed(lambda: G.mds(central, w, args.eager_iters, float("-inf"), init=init), 1)
                print(json.dumps({"what": "smacof", "path": "eager", "weights": wl, "n": n, "iters": args.eager_iters,
                                  "ms_per_iter": round(ms / args.eager_iters, 4), "peak_gb": round(peak, 3)}), flush=True)
            except torch.OutOfMemoryError:
                print(json.dumps({"what": "smacof", "path": "eager", "weights": wl, "n": n, "result": "out of memory"}), flush=True)
        del central, weights, init
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
