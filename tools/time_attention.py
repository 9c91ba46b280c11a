"""Device time of the axial attention kernel (ops.attention_bf16) at the four call shapes of one Evoformer block:
   python tools/time_attention.py [--workload C2 C3 C4] [--launches 20]  -> one JSON line per call, then one summary line

Per workload (bench.py's WORKLOADS: N_res x MSA rows; heads 8, dim_head 64, all-ones masks) the calls are
  msa_row    n = N_res keys, folded batch S,     row folding,    pair bias
  msa_col    n = S keys,     folded batch N_res, column folding, no bias
  tri_start  n = N_res keys, folded batch N_res, row folding,    pair bias
  tri_end    n = N_res keys, folded batch N_res, column folding, pair bias
Each launch is timed by the library's per-launch CUDA events (the ones behind bench.py's kernel_classes) with L2 flushed
before it.  Algorithmic bytes are q, k, v, gate and output (tokens * heads * dim_head * 2 B * 5) plus the bias
(heads * n * n * 2 B), the figure the library's profile records; FLOPs are 4 * tokens * n * heads * dim_head.  The GB/s
fraction is of the H100 SXM data sheet's 3.35 TB/s, the TFLOP/s fraction of its 989 dense BF16 TFLOP/s.  The card name
and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from alphafold2_b200 import _lib, ops  # noqa: E402
from bench import CFG, WORKLOADS  # noqa: E402

HBM_DATASHEET = 3.35e12
BF16_DATASHEET = 989e12
KC_ATTENTION = 2


def calls(N, S):
    """(name, n, nbatch, row folding, bias) of the four attention launches of one block"""
    return [("msa_row", N, S, True, True), ("msa_col", S, N, False, False),
            ("tri_start", N, N, True, True), ("tri_end", N, N, False, True)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl = [v.strip() for v in q.split(",")]
        return dict(name=name, power_limit=pl)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(), error=str(e))


def time_call(lib, flush, n, nbatch, row, bias, launches, heads, dh):
    g = torch.Generator(device="cuda").manual_seed(n * 31 + nbatch)
    I = heads * dh
    T = n * nbatch
    qkv = torch.randn(T, 3 * I, device="cuda", generator=g).to(torch.bfloat16)
    gate = torch.rand(T, I, device="cuda", generator=g).to(torch.bfloat16)
    npad = (n + 7) // 8 * 8
    bt = torch.randn(heads, n, npad, device="cuda", generator=g).to(torch.bfloat16) if bias else None
    mask = torch.ones(T, dtype=torch.bool, device="cuda")
    tok_sb, tok_si = (n, 1) if row else (1, nbatch)

    def run():
        return ops.attention_bf16(qkv, gate, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask)

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    lib.af2_profile_enable(1)
    for _ in range(launches):
        flush.zero_()
        run()
    ms, fl, by = C.c_double(), C.c_double(), C.c_double()
    cnt = lib.af2_profile_read(KC_ATTENTION, C.byref(ms), C.byref(fl), C.byref(by))
    lib.af2_profile_enable(0)
    if cnt != launches:
        raise RuntimeError(f"expected {launches} attention launches, the profile recorded {cnt}")
    t = ms.value / launches
    b = by.value / launches
    f = fl.value / launches
    return dict(ms=t, algorithmic_bytes=b, gbs=b / (t * 1e-3) / 1e9, frac_of_hbm_datasheet=b / (t * 1e-3) / HBM_DATASHEET,
                flops=f, tflops=f / (t * 1e-3) / 1e12, frac_of_bf16_datasheet=f / (t * 1e-3) / BF16_DATASHEET)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["C2"], choices=list(WORKLOADS))
    ap.add_argument("--launches", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_attention.py needs a CUDA device")
    lib = _lib.load()
    heads, dh = CFG["heads"], CFG["dim_head"]
    flush = torch.empty(256 * 2 ** 20, dtype=torch.uint8, device="cuda")
    info = card()
    summary = {"card": info, "lib": _lib.LIB_PATH, "launches": args.launches, "ms_per_block": {}}
    for wl in args.workload:
        N, S = WORKLOADS[wl]
        total = 0.0
        for name, n, nbatch, row, bias in calls(N, S):
            r = time_call(lib, flush, n, nbatch, row, bias, args.launches, heads, dh)
            total += r["ms"]
            print(json.dumps(dict(workload=wl, call=name, n=n, nbatch=nbatch, heads=heads, dim_head=dh, bias=bias, **r)),
                  flush=True)
        summary["ms_per_block"][wl] = total
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
