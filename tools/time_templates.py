"""Device time of Alphafold2.forward with templates at the C2 shape, split into its template parts (CUDA events):
   python tools/time_templates.py [--templates 4] [--steps 10]  -> one JSON line

Model and inputs as bench.py's C2 step (dim 256, depth 12, heads 8, dim_head 64, N_res 256, MSA 128 x 256, batch 1, all-ones
masks) plus T templates: templates_feats, templates_angles and an all-ones templates_mask.  Reported in ms per call:
  forward_ms / forward_without_templates_ms   Alphafold2.forward with and without the template inputs
  pair_stack_ms                               to_template_embed + templates_embed_layers pair blocks over b * T pair tensors
  pointwise_attention_ms                      bf16 copies, q / gate / k|v GEMMs, template_pointwise_kernel, to_out
  angle_mlp_ms                                template_angle_mlp into rows S..S+T-1 of m
and the pointwise kernel alone (the library's per-launch CUDA events, class "attention" of one call): ms, algorithmic bytes
(q, gate, T k|v rows, output, pooled scale, masks), GB/s and its share of the H100 SXM data sheet's 3.35 TB/s.  The card name
and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alphafold2_b200 as A  # noqa: E402
from alphafold2_b200 import _lib  # noqa: E402
from bench import CFG, N_RES, N_SEQ, randomize_zero_init_  # noqa: E402

HBM_DATASHEET = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--templates", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    T = args.templates
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    torch.manual_seed(0)
    model = A.Alphafold2(**CFG)
    randomize_zero_init_(model)
    model = model.to(dev).eval()
    seq = torch.randint(0, 21, (1, N_RES), device=dev)
    msa = torch.randint(0, 21, (1, N_SEQ, N_RES), device=dev)
    mask = torch.ones(1, N_RES, dtype=torch.bool, device=dev)
    msa_mask = torch.ones(1, N_SEQ, N_RES, dtype=torch.bool, device=dev)
    g = torch.Generator(device=dev).manual_seed(5)
    feats = torch.randn(1, T, N_RES, N_RES, model.to_template_embed.in_features, device=dev, generator=g)
    angles = torch.randn(1, T, N_RES, model.template_angle_mlp[0].in_features, device=dev, generator=g)
    tm = torch.ones(1, T, N_RES, dtype=torch.bool, device=dev)
    x_mask = mask[:, :, None] & mask[:, None, :]
    with torch.no_grad():
        t, tm2 = model.template_pair_stack(feats, tm)
    xw = torch.randn(1, N_RES, N_RES, CFG["dim"], device=dev)
    mw = torch.empty(1, N_SEQ + T, N_RES, CFG["dim"], device=dev)

    def timed(fn):
        with torch.no_grad():
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                fn()
            b.record()
            b.synchronize()
        return a.elapsed_time(b) / args.steps

    res = {"T": T, "steps": args.steps,
           "what": f"Alphafold2(dim={CFG['dim']}, depth={CFG['depth']}, heads={CFG['heads']}, dim_head={CFG['dim_head']}) "
                   f"N_res={N_RES} MSA={N_SEQ}x{N_RES} batch=1, {T} templates; ms per call, CUDA events"}
    res["forward_ms"] = timed(lambda: model(seq, msa, mask=mask, msa_mask=msa_mask, templates_feats=feats, templates_mask=tm,
                                            templates_angles=angles))
    res["forward_without_templates_ms"] = timed(lambda: model(seq, msa, mask=mask, msa_mask=msa_mask))
    res["pair_stack_ms"] = timed(lambda: model.template_pair_stack(feats, tm))
    res["pointwise_attention_ms"] = timed(lambda: model.template_pointwise_attn.add_context_(xw, t, x_mask, tm2))
    res["angle_mlp_ms"] = timed(lambda: model.template_angle_mlp.write_(angles, mw, N_SEQ))
    lib.af2_profile_enable(1)
    with torch.no_grad():
        model.template_pointwise_attn.add_context_(xw, t, x_mask, tm2)
    ms, fl, by = C.c_double(), C.c_double(), C.c_double()
    n = lib.af2_profile_read(2, C.byref(ms), C.byref(fl), C.byref(by))
    lib.af2_profile_enable(0)
    rate = by.value / (ms.value * 1e-3) if ms.value > 0 else None
    res["pointwise_kernel"] = {"launches": int(n), "ms": ms.value, "algorithmic_bytes": by.value,
                               "gbs": rate / 1e9 if rate else None, "frac_of_hbm_datasheet": rate / HBM_DATASHEET if rate else None}
    res["gpu"] = torch.cuda.get_device_name(dev)
    try:
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        res["power_limit_w"] = f"unavailable: {ex}"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
