"""Time Alphafold2.forward at a long N_res or a deep MSA on one GPU, whole or with the pair track in bands of pair rows and
the MSA track in bands of MSA rows.

    python tools/time_long.py --n-res 4096 --msa-rows 32 --depth 1
    python tools/time_long.py --n-res 2048 --band 2048 512 --repeat 5     # whole and 512-row bands, alternated
    python tools/time_long.py --n-res 2048 --msa-rows 8448                # the planner's MSA bands
    python tools/time_long.py --n-res 1024 --msa-rows 4096 --msa-band 4096 512 --repeat 3

--band lists the pair rows per band to run (0: the planner's choice, N_res or more: the whole-tensor calls) and --msa-band
the MSA rows per band (0: the planner's choice, msa-rows or more: the whole MSA track); every pair of the two lists runs,
alternating for --repeat rounds after one warm-up forward each.  One JSON line per forward:
  ms            forward time (CUDA events around the call, after a device synchronise)
  band          pair rows per band the trunk used (Evoformer.last_pair_band), msa_band the MSA rows (last_msa_band)
  peak_gb       peak memory allocated by the forward beyond what was allocated before it (fresh grow-only workspace)
  block_gb      ops.msa_block_bytes for those bands, and xm_gb the x and m it comes on top of
  copy_ms       time of the column-band copies of one block (x[:, j0:j1] -> compact buffer -> back, every band), timed
                alone on the same x; copy_share = depth * copy_ms / ms
  msa_copy_ms   the same for the MSA column bands (m[:, j0:j1] and its mask), msa_copy_share = depth * msa_copy_ms / ms
The first line names the card and its power limit (nvidia-smi).
"""
import argparse
import functools
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _copy_ms(N, d, band, mask, rows=None):
    """The column attention's band copies of one block, alone: per column band x[:, j0:j1] (and its mask) to a compact
    buffer and back.  rows: the same for m [rows, N, d] (MSA column bands)."""
    x = torch.empty(rows or N, N, d, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for it in range(2):                                   # the first pass warms the allocator
        ev[0].record()
        for j0 in range(0, N, band):
            j1 = min(j0 + band, N)
            xc = x[:, j0:j1].contiguous()
            mc = mask[:, j0:j1].contiguous()
            x[:, j0:j1] = xc
            del xc, mc
        ev[1].record()
    torch.cuda.synchronize()
    del x
    return ev[0].elapsed_time(ev[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-res", type=int, default=4096)
    ap.add_argument("--msa-rows", type=int, default=32)
    ap.add_argument("--depth", type=int, default=1)
    ap.add_argument("--band", type=int, nargs="+", default=[0])
    ap.add_argument("--msa-band", type=int, nargs="+", default=[0])
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--dim-head", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_long.py measures on the GPU; no CUDA device found")

    import alphafold2_b200 as A
    from alphafold2_b200 import banded, ops
    from oracle import evoformer_oracle as O

    N, S, d = a.n_res, a.msa_rows, a.dim
    print(json.dumps({"card": _card(), "n_res": N, "msa_rows": S, "depth": a.depth, "dim": d, "heads": a.heads, "dim_head": a.dim_head}),
          flush=True)
    torch.manual_seed(0)
    model = A.Alphafold2(dim=d, depth=a.depth, heads=a.heads, dim_head=a.dim_head, max_seq_len=N)
    model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}))
    model = model.cuda().eval()
    seq = torch.randint(0, 21, (1, N), device="cuda")
    msa = torch.randint(0, 21, (1, S, N), device="cuda")
    mask = torch.ones(1, N, dtype=torch.bool, device="cuda")
    msa_mask = torch.ones(1, S, N, dtype=torch.bool, device="cuda")
    run_ = type(model.net).run_
    xm = (N * N + S * N) * d * 4

    def forward(band, msa_band):
        kw = {k: v for k, v in (("band", band), ("msa_band", msa_band)) if v}
        model.net.run_ = functools.partial(run_, model.net, **kw)
        ops._WORKSPACE.clear()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        with torch.no_grad():
            ev[0].record()
            ret = model(seq, msa, mask=mask, msa_mask=msa_mask)
            ev[1].record()
        torch.cuda.synchronize()
        ok = bool(torch.isfinite(ret.distance).all())
        del ret
        return (ev[0].elapsed_time(ev[1]), torch.cuda.max_memory_allocated() - base, model.net.last_pair_band,
                model.net.last_msa_band, ok)

    runs = [(band, msa_band) for band in a.band for msa_band in a.msa_band]
    copies, msa_copies = {}, {}
    for band, msa_band in runs:
        forward(band, msa_band)                           # warm-up: module loads, weight packing, allocator
    for r in range(a.repeat):
        for band, msa_band in runs:
            ms, peak, used, used_msa, ok = forward(band, msa_band)
            if used < N and used not in copies:
                copies[used] = _copy_ms(N, d, used, mask[0, :, None] & mask[0, None, :])
            if used_msa < S and used_msa not in msa_copies:
                msa_copies[used_msa] = _copy_ms(N, d, banded.msa_column_band(S, N, used_msa), msa_mask[0], rows=S)
            cp, mcp = copies.get(used, 0.0), msa_copies.get(used_msa, 0.0)
            print(json.dumps({"round": r, "band_arg": band, "msa_band_arg": msa_band, "band": used, "msa_band": used_msa,
                              "ms": round(ms, 1), "peak_gb": round(peak / 1e9, 2),
                              "block_gb": round(ops.msa_block_bytes(1, N, S, d, a.heads, a.dim_head, used, used_msa) / 1e9, 2),
                              "xm_gb": round(xm / 1e9, 2), "copy_ms": round(cp, 1), "copy_share": round(a.depth * cp / ms, 4),
                              "msa_copy_ms": round(mcp, 1), "msa_copy_share": round(a.depth * mcp / ms, 4), "finite": ok}),
                  flush=True)


if __name__ == "__main__":
    main()
