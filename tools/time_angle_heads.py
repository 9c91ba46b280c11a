"""Time the angle heads (alphafold2.py:813-836): af2_angle_heads against the eager heads it replaces (three nn.Linear on the fp32
pair tensor, plus (x + x^T) * 0.5 when symmetrize_omega), and Alphafold2.forward with predict_angles=True.

    python tools/time_angle_heads.py                                   # heads at N_res 256 / 1024 / 4096, d 256; C2 forward
    python tools/time_angle_heads.py --long 4096 5120                  # depth-1 forwards with symmetrized angles, both paths

One JSON line per measurement; the first names the card and its power limit (nvidia-smi).
  heads:   ms per call (CUDA events around each call, L2 flushed before it by writing 256 MB), kernel and eager alternated for
           --repeat rounds after a warm-up each; peak_gb = peak memory allocated by the call beyond what was allocated before it;
           bound_ms = the data sheet's bound for these bytes (x read once, outputs written once, at 3.35 TB/s): computed, not
           measured.  The outputs of both paths are compared on sampled rows (the last 8 included) against fp64 with the tests'
           gate: the kernel's max error <= 2 x eager fp32's.  An eager call that runs out of memory is reported as such.
  forward: Alphafold2.forward (C2 shape, or --long N_res at depth 1, MSA 32) with predict_angles=True, symmetrize_omega=True;
           path "kernel" or "eager" (ops.angle_heads_ok forced false: the eager heads); finished or out of memory, ms, peak.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35            # H100 SXM data sheet, TB/s
BUCKETS = (25, 13, 25)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


_FLUSH = None


def _flush_l2():
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    _FLUSH.fill_(1)


def _timed(fn, flush=True):
    """(ms, peak bytes beyond the allocation before the call, result) of one call, after an L2 flush unless flush is False"""
    if flush:
        _flush_l2()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    out = fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), torch.cuda.max_memory_allocated() - base, out


def _eager(w, x, sym):
    """the forward's eager heads (alphafold2.py:815-836 as nn.Linear calls on the fp32 pair tensor)"""
    theta = F.linear(x, w[0][0], w[0][1])
    phi = F.linear(x, w[1][0], w[1][1])
    omega = F.linear((x + x.transpose(1, 2)) * 0.5 if sym else x, w[2][0], w[2][1])
    return theta, phi, omega


def _compare(out_k, out_e, w, x, sym, rows):
    """max error of each path against fp64 on the sampled rows; gate of tests/test_gpu_angle_heads.py"""
    xr, xt = x[0, rows].double(), x[0, :, rows].transpose(0, 1).double()
    s = (xr + xt) * 0.5 if sym else xr
    ref = (F.linear(xr, w[0][0].double(), w[0][1].double()), F.linear(xr, w[1][0].double(), w[1][1].double()),
           F.linear(s, w[2][0].double(), w[2][1].double()))
    res = {}
    for name, k, e, r in zip(("theta", "phi", "omega"), out_k, out_e, ref):
        ek = (k[0, rows].double() - r).abs().max().item()
        ee = (e[0, rows].double() - r).abs().max().item()
        res[name] = {"kernel_err": ek, "eager_err": ee, "ok": ek <= 2 * ee}
    return res


def heads(N, d, sym, repeat):
    from alphafold2_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(N + sym)
    x = torch.randn(1, N, N, d, device="cuda", generator=g)
    w = [((torch.rand(nb, d, generator=g, device="cuda") * 2 - 1) * d ** -0.5, (torch.rand(nb, generator=g, device="cuda") * 2 - 1) * 0.1)
         for nb in BUCKETS]
    pk = ops.pack_angle_heads(w[0][0], w[0][1], w[1][0], w[1][1], w[2][0], w[2][1])
    rows = torch.tensor([0, 1, N // 2, N // 3] + list(range(N - 8, N)), device="cuda")
    out_bytes = N * N * sum(BUCKETS) * 4
    bound_ms = (N * N * d * 4 + out_bytes) / (HBM_TBS * 1e12) * 1e3
    paths = {"kernel": lambda: ops.angle_heads(pk, x, sym), "eager": lambda: _eager(w, x, sym)}
    outs, oom = {}, set()
    for name, fn in paths.items():                       # warm-up, and the outputs compared below
        try:
            outs[name] = _timed(fn)[2]
        except torch.OutOfMemoryError:
            oom.add(name)
            torch.cuda.empty_cache()
    if "kernel" in outs and "eager" in outs:
        cmp = _compare(outs["kernel"], outs["eager"], w, x, sym, rows)
        print(json.dumps({"what": "heads_compare", "n_res": N, "d": d, "sym": sym, "rows": len(rows), **cmp}), flush=True)
    outs.clear()
    for r in range(repeat):
        for name, fn in paths.items():
            if name in oom:
                print(json.dumps({"what": "heads", "path": name, "n_res": N, "d": d, "sym": sym, "round": r, "out_of_memory": True}), flush=True)
                continue
            try:
                ms, peak, out = _timed(fn)
                del out
            except torch.OutOfMemoryError:
                oom.add(name)
                torch.cuda.empty_cache()
                continue
            print(json.dumps({"what": "heads", "path": name, "n_res": N, "d": d, "sym": sym, "round": r, "ms": round(ms, 3),
                              "peak_gb": round(peak / 1e9, 3), "bound_ms": round(bound_ms, 3),
                              "gbs": round((N * N * d * 4 + out_bytes) / (ms * 1e6), 1)}), flush=True)
    del x
    torch.cuda.empty_cache()


def forward(N, S, depth, d, heads_, dim_head, repeat):
    import alphafold2_b200 as A
    from alphafold2_b200 import ops
    from oracle import evoformer_oracle as O
    torch.manual_seed(0)
    model = A.Alphafold2(dim=d, depth=depth, heads=heads_, dim_head=dim_head, max_seq_len=N, predict_angles=True, symmetrize_omega=True)
    model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}))
    model = model.cuda().eval()
    seq = torch.randint(0, 21, (1, N), device="cuda")
    msa = torch.randint(0, 21, (1, S, N), device="cuda")
    mask = torch.ones(1, N, dtype=torch.bool, device="cuda")
    msa_mask = torch.ones(1, S, N, dtype=torch.bool, device="cuda")
    ok_fn = ops.angle_heads_ok

    def run(path):
        ops.angle_heads_ok = ok_fn if path == "kernel" else (lambda d_, b_: False)
        try:
            ops._WORKSPACE.clear()
            torch.cuda.empty_cache()
            with torch.no_grad():
                ms, peak, ret = _timed(lambda: model(seq, msa, mask=mask, msa_mask=msa_mask), flush=False)
            fin = bool(torch.isfinite(ret.omega_logits).all())
            del ret
            return {"ms": round(ms, 1), "peak_gb": round(peak / 1e9, 2), "finished": True, "finite": fin}
        except (torch.OutOfMemoryError, MemoryError) as e:      # the allocator, or the pair-band planner before any device work
            torch.cuda.empty_cache()
            return {"finished": False, "out_of_memory": str(e).split(";")[0][:160]}
        finally:
            ops.angle_heads_ok = ok_fn

    for path in ("kernel", "eager"):
        run(path)                                        # warm-up
    for r in range(repeat):
        for path in ("kernel", "eager"):
            print(json.dumps({"what": "forward", "path": path, "n_res": N, "msa_rows": S, "depth": depth, "round": r, **run(path)}),
                  flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-res", type=int, nargs="+", default=[256, 1024, 4096])
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--long", type=int, nargs="*", default=None, help="N_res of depth-1 forwards (instead of the heads and C2)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_angle_heads.py measures on the GPU; no CUDA device found")
    print(json.dumps({"card": _card()}), flush=True)
    if a.long:
        global _FLUSH
        _FLUSH = None
        for N in a.long:
            forward(N, 32, 1, a.dim, 8, 64, 1)
        return
    for N in a.n_res:
        for sym in (False, True):
            heads(N, a.dim, sym, a.repeat)
    forward(256, 128, 12, 256, 8, 64, a.repeat)          # C2: dim 256, depth 12, heads 8 x 64, N_res 256, MSA 128


if __name__ == "__main__":
    main()
