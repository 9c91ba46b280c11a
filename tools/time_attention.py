"""Device time of the axial attention kernel (ops.attention_bf16) at the four call shapes of one Evoformer block:
   python tools/time_attention.py [--workload C2 C3 C4] [--launches 20] [--heads 8] [--dim-head 64]
   -> one JSON line per call, then one summary line

Per workload (bench.py's WORKLOADS: N_res x MSA rows; heads 8, dim_head 64 unless given, all-ones masks) the calls are
  msa_row    n = N_res keys, folded batch S,     row folding,    pair bias
  msa_col    n = S keys,     folded batch N_res, column folding, no bias
  tri_start  n = N_res keys, folded batch N_res, row folding,    pair bias
  tri_end    n = N_res keys, folded batch N_res, column folding, pair bias
Each launch is timed by the library's per-launch CUDA events (the ones behind bench.py's kernel_classes) with L2 flushed
before it.  Algorithmic bytes are q, k, v, gate and output (tokens * heads * dim_head * 2 B * 5) plus the bias
(heads * n * n * 2 B), the figure the library's profile records; FLOPs are 4 * tokens * n * heads * dim_head.  The GB/s
fraction is of the H100 SXM data sheet's 3.35 TB/s, the TFLOP/s fraction of its 989 dense BF16 TFLOP/s.  The card name
and power limit are read in the same run.

--projected times each call from the fp32 residual stream instead: LayerNorm -> the fused projection + attention kernel
against LayerNorm -> q|k|v GEMM -> gate GEMM -> attention kernel (time_projected), and reports both with the speedup; the
summary's ms_per_block is then the fused sequences' and unfused_ms_per_block the unfused ones'.  A call whose n is above
ops.attention_proj_max_n is refused by the fused kernel."""
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


def time_call(lib, flush, n, nbatch, row, bias, launches, heads, dh, eager=False):
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

    if eager:
        return time_eager(flush, qkv, gate, bt, mask, n, nbatch, row, launches, heads, dh)
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
    return rates(ms.value / launches, by.value / launches, fl.value / launches)


def time_eager(flush, qkv, gate, bt, mask, n, nbatch, row, launches, heads, dh):
    """The same call in eager PyTorch bf16, written as the reference's Attention.forward writes it (einsum, masked_fill,
    softmax, einsum, gate) on the token-layout q | k | v; timed with CUDA events around each call, L2 flushed before it.
    Bytes and FLOPs are the kernel's algorithmic figures, so the rates compare directly."""
    T, I = qkv.shape[0], heads * dh
    # [T, 3I] -> [3, b', heads, n, dh] in the folding's token order
    x = qkv.view(nbatch, n, 3, heads, dh) if row else qkv.view(n, nbatch, 3, heads, dh).transpose(0, 1)
    q, k, v = x.permute(2, 0, 3, 1, 4).unbind(0)
    g = (gate.view(nbatch, n, I) if row else gate.view(n, nbatch, I).transpose(0, 1))
    m = mask.view(nbatch, n) if row else mask.view(n, nbatch).transpose(0, 1)

    def run():
        dots = torch.einsum("bhid,bhjd->bhij", q, k)
        if bt is not None:
            dots = dots + bt[None, :, :, :n]
        pair = m[:, None, :, None] & m[:, None, None, :]
        dots = dots.masked_fill(~pair, -torch.finfo(dots.dtype).max)
        attn = dots.softmax(dim=-1)
        out = torch.einsum("bhij,bhjd->bhid", attn, v)
        return out.permute(0, 2, 1, 3).reshape(nbatch, n, I) * g

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(launches):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1)
    tokens = float(T)
    f = 4.0 * tokens * n * heads * dh
    b = tokens * heads * dh * 2.0 * 5 + (heads * n * n * 2.0 if bt is not None else 0.0)
    return rates(total / launches, b, f)


def time_projected(flush, n, nbatch, row, bias, launches, heads, dh, d):
    """LayerNorm -> fused projection + attention kernel (ops.attention_proj_bf16) against LayerNorm -> q|k|v GEMM -> gate GEMM
    -> attention kernel, the two sequences the module entries run; CUDA events around each sequence, L2 flushed before it.
    Algorithmic bytes: x read (fp32), xn written and read, the output written, the bias once, plus for the unfused sequence
    q|k|v and the gate written and read back.  FLOPs: the four projections plus QK^T and PV."""
    g = torch.Generator(device="cuda").manual_seed(n * 31 + nbatch)
    I = heads * dh
    T = n * nbatch
    x = torch.randn(T, d, device="cuda", generator=g)
    gamma, beta = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
    wqkv = (torch.randn(3 * I, d, device="cuda", generator=g) * d ** -0.5).to(torch.bfloat16)
    wg = (torch.randn(I, d, device="cuda", generator=g) * d ** -0.5).to(torch.bfloat16)
    bg = torch.randn(I, device="cuda", generator=g)
    npad = (n + 7) // 8 * 8
    bt = torch.randn(heads, n, npad, device="cuda", generator=g).to(torch.bfloat16) if bias else None
    mask = torch.ones(T, dtype=torch.bool, device="cuda")
    tok_sb, tok_si = (n, 1) if row else (1, nbatch)
    qkv = torch.empty(T, 3 * I, dtype=torch.bfloat16, device="cuda")
    gate = torch.empty(T, I, dtype=torch.bfloat16, device="cuda")
    bn = lambda c: 256 if c > 128 else (128 if c > 64 else 64)   # noqa: E731  (csrc/api.cu pick_bn)

    def fused():
        xn = ops.layernorm_bf16(x, gamma, beta)
        return ops.attention_proj_bf16(xn, wqkv, wg, bg, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask)

    def unfused():
        xn = ops.layernorm_bf16(x, gamma, beta)
        ops.gemm_bf16_epilogue(xn[None], wqkv[None], qkv, bn=bn(3 * I), mode=ops.EPI_STORE_BF16, ld_out=3 * I)
        ops.gemm_bf16_epilogue(xn[None], wg[None], gate, bn=bn(I), mode=ops.EPI_STORE_BF16, act=ops.ACT_SIGMOID, bias=bg, ld_out=I)
        return ops.attention_bf16(qkv, gate, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask)

    f = 2.0 * T * d * 4 * I + 4.0 * T * n * I
    b_f = 4.0 * T * d + 4.0 * T * d + 2.0 * T * I + 4.0 * I * d * 2 + (heads * n * n * 2.0 if bias else 0.0)
    b_u = b_f + 2.0 * T * 4 * I * 2
    out = {"fused": None}
    for name, run, b in (("fused", fused, b_f), ("unfused", unfused, b_u)):
        if name == "fused" and n > ops.attention_proj_max_n(dh):
            continue                     # the module entries run the unfused sequence for this call
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        total = 0.0
        for _ in range(launches):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            e1.synchronize()
            total += e0.elapsed_time(e1)
        out[name] = rates(total / launches, b, f)
    return out


def rates(t, b, f):
    return dict(ms=t, algorithmic_bytes=b, gbs=b / (t * 1e-3) / 1e9, frac_of_hbm_datasheet=b / (t * 1e-3) / HBM_DATASHEET,
                flops=f, tflops=f / (t * 1e-3) / 1e12, frac_of_bf16_datasheet=f / (t * 1e-3) / BF16_DATASHEET)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["C2"], choices=list(WORKLOADS))
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--heads", type=int, default=CFG["heads"])
    ap.add_argument("--dim-head", type=int, default=CFG["dim_head"], help="16, 32, 64 or 128")
    ap.add_argument("--eager", action="store_true", help="time the reference's eager PyTorch bf16 lines instead of the kernel")
    ap.add_argument("--projected", action="store_true",
                    help="time LayerNorm + the fused projection + attention kernel against LayerNorm + the q|k|v and gate GEMMs "
                         "+ the attention kernel, from the fp32 residual stream (dim 256)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_attention.py needs a CUDA device")
    lib = _lib.load()
    heads, dh = args.heads, args.dim_head
    flush = torch.empty(256 * 2 ** 20, dtype=torch.uint8, device="cuda")
    info = card()
    summary = {"card": info, "lib": _lib.LIB_PATH, "launches": args.launches, "ms_per_block": {}}
    for wl in args.workload:
        N, S = WORKLOADS[wl]
        total = 0.0
        for name, n, nbatch, row, bias in calls(N, S):
            if args.projected:
                r = time_projected(flush, n, nbatch, row, bias, args.launches, heads, dh, CFG["dim"])
                r["speedup"] = r["unfused"]["ms"] / r["fused"]["ms"] if r["fused"] else None
                total += (r["fused"] or r["unfused"])["ms"]
                summary.setdefault("unfused_ms_per_block", {}).setdefault(wl, 0.0)
                summary["unfused_ms_per_block"][wl] += r["unfused"]["ms"]
                print(json.dumps(dict(workload=wl, call=name, n=n, nbatch=nbatch, heads=heads, dim_head=dh, bias=bias, **r)),
                      flush=True)
                continue
            r = time_call(lib, flush, n, nbatch, row, bias, args.launches, heads, dh, args.eager)
            total += r["ms"]
            extra = {"impl": "eager_pytorch_bf16"} if args.eager else {}
            print(json.dumps(dict(workload=wl, call=name, n=n, nbatch=nbatch, heads=heads, dim_head=dh, bias=bias, **extra, **r)),
                  flush=True)
        summary["ms_per_block"][wl] = total
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
