"""Device time of one EvoformerBlock at a BASELINE shape (CUDA events, L2 flushed between iterations):
   AF2_N=384 AF2_S=512 python tools/time_block.py  -> one JSON line {N, S, ms_per_block, tflops}

AF2_PROFILE=1 adds a torch.profiler pass (CUDA activities, after the timed loop) that groups kernel time by name and, for
the linear GEMMs (K-major, BN 256), by epilogue kind: ms per block, us per 128 x 256 output tile on one SM (kernel time x
SM count / tiles), and TFLOP/s and GB/s from algorithmic FLOPs and bytes.  The fused feed-forward kernel has a row of its
own: ms per block, TFLOP/s, HBM GB/s and the L2->SM rate of its weight reads (W1 and W2 once per 128-row tile).  The card name, power limit and max SM clock are read in the same run.  AF2_PROFILE_OUT=path also
writes the result as JSON."""
import json
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alphafold2_b200 as A  # noqa: E402
from alphafold2_b200 import _lib  # noqa: E402
from bench import CFG, flops_per_block, randomize_zero_init_  # noqa: E402

N = int(os.environ.get("AF2_N", 256))
S = int(os.environ.get("AF2_S", 128))
it = int(os.environ.get("AF2_ITERS", 10))
torch.manual_seed(0)
blk = A.EvoformerBlock(dim=CFG["dim"], seq_len=N, heads=CFG["heads"], dim_head=CFG["dim_head"], attn_dropout=0., ff_dropout=0.)
randomize_zero_init_(blk)
blk = blk.cuda().eval()
if os.environ.get("AF2_PRECISION_BLOCK"):
    A.set_precision(blk, os.environ["AF2_PRECISION_BLOCK"])
x = torch.randn(1, N, N, CFG["dim"], device="cuda")
m = torch.randn(1, S, N, CFG["dim"], device="cuda")
mask = torch.ones(1, N, N, dtype=torch.bool, device="cuda")
msa_mask = torch.ones(1, S, N, dtype=torch.bool, device="cuda")
flush = torch.empty(256 * 2 ** 20, dtype=torch.uint8, device="cuda")
for _ in range(3):
    blk.update_(x.clone(), m.clone(), mask, msa_mask)
tot = 0.0
for _ in range(it):
    xx, mm = x.clone(), m.clone()
    flush.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    blk.update_(xx, mm, mask, msa_mask)
    b.record()
    b.synchronize()
    tot += a.elapsed_time(b)
ms = tot / it
fl = flops_per_block(N, S, CFG["dim"], CFG["heads"], CFG["dim_head"])
print(json.dumps({"N": N, "S": S, "ms_per_block": ms, "tflops": fl / (ms * 1e-3) / 1e12,
                  "env": {k: v for k, v in os.environ.items() if k.startswith("AF2_")}}))


# gemm_tc_kernel epilogue kinds (csrc/gemm_tc.cuh EpiKind)
EK_NAMES = {0: "GENERIC", 1: "STORE_TOK", 2: "STORE_TOK_SIG", 3: "STORE_CH", 4: "GATED_TOK_GELU", 5: "GATED_CH_SIG",
            6: "RESID_F32", 7: "STORE_F32", 8: "STORE_CH_SIG", 9: "RESID_F32_W"}


def linear_gemms(N, S, d, I):
    """(epilogue kind, M, accumulator columns, K) of every linear GEMM launch of one block (module path)."""
    Tm, Tx = S * N, N * N
    out = []
    for T in (Tm, Tm, Tx, Tx):        # MSA row / column attention, triangle attention start / end
        out += [(1, T, 3 * I, d), (2, T, I, d), (6, T, d, I)]
    out += [(3, Tm, 2 * d, d), (6, Tx, d, d)]                        # outer mean: left|right, out
    for _ in range(2):                # triangle multiply outgoing / ingoing: left, right, out gate, out
        out += [(5, Tx, 2 * d, d), (5, Tx, 2 * d, d), (2, Tx, d, d), (6, Tx, d, d)]
    return out


def ff_launches(N, S, d):
    """(T, d, hidden) of the fused feed-forward launches of one block (csrc/ff_fused.cuh): MSA and pair transitions."""
    return [(S * N, d, 4 * d), (N * N, d, 4 * d)]


def ff_cost(T, d, hidden):
    """Algorithmic FLOPs, HBM bytes (xn read, x read and written, the weights once) and L2->SM weight bytes (W1 and W2,
    3 d hidden bf16, once per 128-row tile) of one fused feed-forward launch."""
    wbytes = 3 * d * hidden * 2
    return 2.0 * T * 3 * d * hidden, float(2 * T * d + 8 * T * d + wbytes), float(-(-T // 128) * wbytes)


def gemm_cost(ek, M, Nacc, K):
    wout = Nacc // 2 if ek in (4, 5) else Nacc
    ebytes = 4 if ek in (6, 7, 9) else 2
    byts = 2 * M * K + 2 * Nacc * K + ebytes * M * wout + (4 * M * wout if ek in (6, 9) else 0)
    return 2.0 * M * Nacc * K, float(byts), M * Nacc / (128 * 256)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl, clk = [v.strip() for v in q.split(",")]
        return dict(name=name, power_limit=pl, clocks_max_sm=clk)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(), error=str(e))


if os.environ.get("AF2_PROFILE") == "1":
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(it):
            blk.update_(x.clone(), m.clone(), mask, msa_mask)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            k = kernels.setdefault(ev.key, [0.0, 0])
            k[0] += t / 1e3 / it
            k[1] += ev.count
    by_ek = {}
    for name, (ms_, cnt) in kernels.items():
        mt = re.search(r"gemm_tc_kernel<(\d+), (\d+), (true|false), (\d+)>", name)
        if mt and mt.group(3) == "false" and mt.group(1) == "256":
            by_ek.setdefault(int(mt.group(4)), [0.0, 0])
            by_ek[int(mt.group(4))][0] += ms_
            by_ek[int(mt.group(4))][1] += cnt // it
    cost = {}
    for ek, M, Nacc, K in linear_gemms(N, S, CFG["dim"], CFG["heads"] * CFG["dim_head"]):
        f, b_, tl = gemm_cost(ek, M, Nacc, K)
        c = cost.setdefault(ek, [0.0, 0.0, 0.0, 0])
        c[0] += f; c[1] += b_; c[2] += tl; c[3] += 1
    n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    rows = []
    for ek, (ms_, launches) in sorted(by_ek.items()):
        if ek not in cost:            # K-major EK_STORE_F32: the per-channel triangle contraction, not a Linear layer
            continue
        f, b_, tl, n_exp = cost[ek]
        rows.append(dict(epilogue=EK_NAMES.get(ek, str(ek)), launches=launches, launches_expected=n_exp,
                         ms_per_block=ms_, us_per_tile_128x256_per_sm=ms_ * 1e3 * n_sm / tl,
                         tflops=f / (ms_ * 1e-3) / 1e12, gbs=b_ / (ms_ * 1e-3) / 1e9))
    ff_ms, ff_n = 0.0, 0
    for name, (ms_, cnt) in kernels.items():
        if "ff_fused_kernel" in name:
            ff_ms += ms_
            ff_n += cnt // it
    f, hb, wb = (sum(v) for v in zip(*(ff_cost(*a) for a in ff_launches(N, S, CFG["dim"]))))
    ff_row = dict(kernel="ff_fused", launches=ff_n, launches_expected=len(ff_launches(N, S, CFG["dim"])), ms_per_block=ff_ms,
                  tflops=f / (ff_ms * 1e-3) / 1e12 if ff_ms else None, hbm_gbs=hb / (ff_ms * 1e-3) / 1e9 if ff_ms else None,
                  weight_l2_gbs=wb / (ff_ms * 1e-3) / 1e9 if ff_ms else None)
    res = dict(N=N, S=S, iters=it, card=card(), lib=_lib.LIB_PATH,
               linear_gemm_ms_per_block=sum(r["ms_per_block"] for r in rows) + ff_ms, linear_gemm_by_epilogue=rows,
               feed_forward=ff_row,
               kernels_ms_per_block=dict(sorted(((k, v[0]) for k, v in kernels.items()), key=lambda kv: -kv[1])[:25]))
    print(json.dumps(res))
    if os.environ.get("AF2_PROFILE_OUT"):
        with open(os.environ["AF2_PROFILE_OUT"], "w") as f:
            json.dump(res, f, indent=1)
