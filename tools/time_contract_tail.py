"""Device time of one contraction tail per call, fused (contract_tail_kernel) against unfused ([out-gate GEMM,]
chan_to_token, to_out GEMM), at the pair shapes of C2 (N_res 256) and C3 (N_res 384), d = 256:
   python tools/time_contract_tail.py  -> one JSON line per (shape, variant, path)

Each timing is CUDA events around 20 launches of the call, with L2 flushed (a 256 MB write) before every launch and the
flush outside the events.  Bytes are algorithmic, computed from shapes: O fp32, the gate or xn bf16, x read and written, the
weights once, plus for the unfused path the bf16 intermediates (gate, tail) written and read back.  share_of_hbm is those
bytes over the time against 3.35 TB/s (H100 SXM data sheet).  The card name and power limit are read in the same run."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from alphafold2_b200 import ops  # noqa: E402

HBM = 3.35e12
REPS = 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl = [v.strip() for v in q.split(",")]
        return dict(name=name, power_limit=pl)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(), error=str(e))


def nbytes(kind, T, d, fused):
    w = (2 if kind == "project" else 1) * d * d * 2
    b = 4 * T * d + 8 * T * d + w + (2 * T * d if kind == "project" else 0) + (2 * T * d if kind == "load" else 0)
    if not fused:
        b += 4 * T * d                                  # the tail y written and read back
        if kind == "project":
            b += 4 * T * d                              # the gate written and read back
    return b


def main():
    torch.manual_seed(0)
    d = 256
    flush = torch.empty(256 * 2 ** 20, dtype=torch.uint8, device="cuda")
    out = []
    for label, N in (("C2", 256), ("C3", 384)):
        T = N * N
        src = torch.randn(d * T, device="cuda")
        x0 = torch.randn(T, d, device="cuda")
        xn = torch.randn(T, d, device="cuda").to(torch.bfloat16)
        gate = torch.rand(T, d, device="cuda").to(torch.bfloat16)
        y = torch.empty(T * d, dtype=torch.bfloat16, device="cuda")
        scale = torch.rand(T, device="cuda") + 0.5
        wo = (torch.randn(d, d, device="cuda") * d ** -0.5).to(torch.bfloat16)
        wog = (torch.randn(d, d, device="cuda") * d ** -0.5).to(torch.bfloat16)
        bo, bog = torch.randn(d, device="cuda"), torch.randn(d, device="cuda")
        gamma, beta = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
        for kind in ("project", "load", "scale"):
            kw = dict(chan_stride=T, pitch=N, rows=N, n=N, d=d)
            if kind == "scale":
                kw.update(mode=1, scale=scale, scale_const=1.0 / 128)
            else:
                kw.update(mode=0, gamma=gamma, beta=beta, gate=gate)
                if kind == "project":
                    kw.update(xn=xn, w_ogate=wog, b_ogate=bog)
            for path in (ops.CTAIL_FUSED, ops.CTAIL_UNFUSED):
                x = x0.clone()
                ops.contract_tail(src, x, wo, bo, y, variant=path, **kw)     # warm-up
                torch.cuda.synchronize()
                tot = 0.0
                for _ in range(REPS):
                    flush.zero_()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    ops.contract_tail(src, x, wo, bo, y, variant=path, **kw)
                    b.record()
                    b.synchronize()
                    tot += a.elapsed_time(b)
                ms = tot / REPS
                fused = path == ops.CTAIL_FUSED
                byts = nbytes(kind, T, d, fused)
                out.append(dict(shape=label, T=T, d=d, variant=kind, path="fused" if fused else "unfused", us_per_call=ms * 1e3,
                                bytes=byts, gbs=byts / (ms * 1e-3) / 1e9, share_of_hbm=byts / HBM / (ms * 1e-3)))
    c = card()
    for r in out:
        r["card"] = c
        print(json.dumps(r))


if __name__ == "__main__":
    main()
