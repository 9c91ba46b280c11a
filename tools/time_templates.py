"""Device time of Alphafold2.forward with templates at the C2 shape, split into its template parts (CUDA events):
   python tools/time_templates.py [--templates 4] [--steps 10] [--n-res 256] [--msa-rows 128] [--depth 12] [--group G]
                                  [--band R] [--precision bf16|strict] [--save-distance PATH]
   -> one JSON line

Model and inputs as bench.py's C2 step (dim 256, depth 12, heads 8, dim_head 64, N_res 256, MSA 128 x 256, batch 1, all-ones
masks) plus T templates: templates_feats, templates_angles and an all-ones templates_mask.  --n-res / --msa-rows / --depth
change the shape; --group forces the number of templates the branch runs at a time and --band the pair rows per band of
its pointwise attention (default: what ops.plan_template_branch picks from the free memory; template_group and
template_band report them, template_band = N_res when the branch runs whole, and planned_template_bytes is
ops.template_branch_bytes for that choice).  --save-distance writes the distogram of one forward (torch.save).  Reported in
ms per call:
  forward_ms / forward_without_templates_ms   Alphafold2.forward with and without the template inputs
  peak_alloc_*_bytes                          torch.cuda.max_memory_allocated over one such forward (from a fresh workspace)
  pair_stack_ms                               to_template_embed + templates_embed_layers pair blocks over b * T pair tensors
  pointwise_attention_ms                      bf16 copies, q / gate / k|v GEMMs, template_pointwise_kernel, to_out
  angle_mlp_ms                                template_angle_mlp into rows S..S+T-1 of m
and the pointwise kernel alone (the library's per-launch CUDA events, class "attention" of one call): ms, algorithmic bytes
(q, gate, T k|v rows, output, pooled scale, masks), GB/s and its share of the H100 SXM data sheet's 3.35 TB/s.  The card name
and power limit are read in the same run.  The part timings run all T templates at once; they are skipped (null) when the
forward ran them in groups.  --steps 1 skips the warm-up calls (long shapes)."""
import argparse
import ctypes as C
import functools
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alphafold2_b200 as A  # noqa: E402
from alphafold2_b200 import _lib, ops  # noqa: E402
from bench import CFG, N_RES, N_SEQ, randomize_zero_init_  # noqa: E402

HBM_DATASHEET = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--templates", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--n-res", type=int, default=N_RES)
    ap.add_argument("--msa-rows", type=int, default=N_SEQ)
    ap.add_argument("--depth", type=int, default=CFG["depth"])
    ap.add_argument("--group", type=int, default=None, help="templates per group (default: planned from free memory)")
    ap.add_argument("--band", type=int, default=None, help="pair rows per band of the template branch (default: planned)")
    ap.add_argument("--precision", choices=ops.PRECISIONS, default="bf16")
    ap.add_argument("--save-distance", default=None, help="torch.save the distogram of one forward to this path")
    args = ap.parse_args()
    T, n, S = args.templates, args.n_res, args.msa_rows
    cfg = dict(CFG, depth=args.depth)
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    torch.manual_seed(0)
    model = A.Alphafold2(**cfg)
    randomize_zero_init_(model)
    model = A.set_precision(model.to(dev).eval(), args.precision)
    if args.group is not None or args.band is not None:
        model.embed_templates_ = functools.partial(type(model).embed_templates_, model, group=args.group, band=args.band)
    seq = torch.randint(0, 21, (1, n), device=dev)
    msa = torch.randint(0, 21, (1, S, n), device=dev)
    mask = torch.ones(1, n, dtype=torch.bool, device=dev)
    msa_mask = torch.ones(1, S, n, dtype=torch.bool, device=dev)
    g = torch.Generator(device=dev).manual_seed(5)
    feats = torch.randn(1, T, n, n, model.to_template_embed.in_features, device=dev, generator=g)
    angles = torch.randn(1, T, n, model.template_angle_mlp[0].in_features, device=dev, generator=g)
    tm = torch.ones(1, T, n, dtype=torch.bool, device=dev)
    x_mask = mask[:, :, None] & mask[:, None, :]

    def timed(fn):
        with torch.no_grad():
            for _ in range(2 if args.steps > 1 else 0):
                fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                fn()
            b.record()
            b.synchronize()
        return a.elapsed_time(b) / args.steps

    def peak(fn):
        ops._WORKSPACE.clear()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        with torch.no_grad():
            fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated(dev)

    res = {"T": T, "steps": args.steps,
           "what": f"Alphafold2(dim={cfg['dim']}, depth={cfg['depth']}, heads={cfg['heads']}, dim_head={cfg['dim_head']}) "
                   f"N_res={n} MSA={S}x{n} batch=1, {T} templates; ms per call, CUDA events"}
    fwd = lambda: model(seq, msa, mask=mask, msa_mask=msa_mask, templates_feats=feats, templates_mask=tm,  # noqa: E731
                        templates_angles=angles)
    fwd_plain = lambda: model(seq, msa, mask=mask, msa_mask=msa_mask)  # noqa: E731
    try:
        res["peak_alloc_with_templates_bytes"] = peak(fwd)
    except MemoryError as ex:                      # the planner refuses before any device work of the branch
        res["memory_error"] = str(ex)
        print(json.dumps(dict(res, **_card(dev))))
        return
    res["template_group"] = model.last_template_group
    res["template_band"] = model.last_template_band
    res["planned_template_bytes"] = ops.template_branch_bytes(
        1, T, model.last_template_group, n, cfg["dim"], cfg["heads"], cfg["dim_head"], args.precision,
        model.to_template_embed.in_features, band=model.last_template_band)
    res["peak_alloc_without_templates_bytes"] = peak(fwd_plain)
    res["forward_ms"] = timed(fwd)
    res["forward_without_templates_ms"] = timed(fwd_plain)
    with torch.no_grad():
        dist = fwd().distance
    res["distance_checksum"] = float(dist.double().sum().item())
    if args.save_distance:
        torch.save(dist.cpu(), args.save_distance)
    if model.last_template_group < T or model.last_template_band < n:
        res["parts"] = "skipped: the forward ran the templates in groups or bands"
        print(json.dumps(dict(res, **_card(dev))))
        return
    with torch.no_grad():
        t, tm2 = model.template_pair_stack(feats, tm)
    xw = torch.randn(1, n, n, CFG["dim"], device=dev)
    mw = torch.empty(1, S + T, n, CFG["dim"], device=dev)
    res["pair_stack_ms"] = timed(lambda: model.template_pair_stack(feats, tm))
    res["pointwise_attention_ms"] = timed(lambda: model.template_pointwise_attn.add_context_(xw, t, x_mask, tm2))
    res["angle_mlp_ms"] = timed(lambda: model.template_angle_mlp.write_(angles, mw, S))
    lib.af2_profile_enable(1)
    with torch.no_grad():
        model.template_pointwise_attn.add_context_(xw, t, x_mask, tm2)
    ms, fl, by = C.c_double(), C.c_double(), C.c_double()
    n = lib.af2_profile_read(2, C.byref(ms), C.byref(fl), C.byref(by))
    lib.af2_profile_enable(0)
    rate = by.value / (ms.value * 1e-3) if ms.value > 0 else None
    res["pointwise_kernel"] = {"launches": int(n), "ms": ms.value, "algorithmic_bytes": by.value,
                               "gbs": rate / 1e9 if rate else None, "frac_of_hbm_datasheet": rate / HBM_DATASHEET if rate else None}
    print(json.dumps(dict(res, **_card(dev))))


def _card(dev):
    res = {"gpu": torch.cuda.get_device_name(dev)}
    try:
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        res["power_limit_w"] = f"unavailable: {ex}"
    return res


if __name__ == "__main__":
    main()
