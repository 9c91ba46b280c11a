"""Device time and peak memory of alphafold2_b200.recycle against the caller's own recycling loop (CUDA events):
   python tools/time_recycle_loop.py [--steps 5] [--num-recycles 3] [--templates 0 4] [--n-res 256] [--msa-rows 128] [--depth 12]
   -> one JSON line per template count

Model and inputs as bench.py's C2 step (dim 256, depth 12, heads 8, dim_head 64, N_res 256, MSA 128 x 256, batch 1, all-ones
masks) with the structure module attached (predict_coords=True, structure depth 4) and T templates (templates_feats,
templates_angles, an all-ones templates_mask).  The manual loop is

    coords, ret = model(seq, msa, **kw, return_aux_logits=True, return_recyclables=True)
    for _ in range(num_recycles - 1):
        coords, ret = model(seq, msa, **kw, recyclables=ret.recyclables, return_aux_logits=True, return_recyclables=True)
    coords, confidence = model(seq, msa, **kw, recyclables=ret.recyclables, return_confidence=True)

and recycle(model, seq, msa, num_recycles=..., return_confidence=True, **kw) returns the same.  Reported:
  manual_ms / recycle_ms            per prediction (num_recycles + 1 forwards), median of --steps runs taken alternately, one
                                    of each per round after one warm-up of each, with min and max
  peak_alloc_manual / _recycle      torch.cuda.max_memory_allocated over one prediction, each from a released workspace
  template_reuse                    whether recycle kept the template pair stack (Alphafold2.last_template_reuse)
  outputs_equal                     coordinates and confidence of the two bitwise equal
--n-res / --msa-rows / --depth change the shape (e.g. --n-res 2048 --msa-rows 1 --depth 1 --templates 0 --steps 1 for the peaks
at a long length).  The card name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alphafold2_b200 as A  # noqa: E402
from alphafold2_b200 import ops  # noqa: E402
from bench import CFG, N_RES, N_SEQ, randomize_zero_init_  # noqa: E402


def manual_loop(model, seq, msa, num_recycles, **kw):
    coords, ret = model(seq, msa, **kw, return_aux_logits=True, return_recyclables=True)
    for _ in range(num_recycles - 1):
        coords, ret = model(seq, msa, **kw, recyclables=ret.recyclables, return_aux_logits=True, return_recyclables=True)
    return model(seq, msa, **kw, recyclables=ret.recyclables, return_confidence=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--num-recycles", type=int, default=3)
    ap.add_argument("--templates", type=int, nargs="+", default=[0, 4])
    ap.add_argument("--n-res", type=int, default=N_RES)
    ap.add_argument("--msa-rows", type=int, default=N_SEQ)
    ap.add_argument("--depth", type=int, default=CFG["depth"])
    args = ap.parse_args()
    n, S, R = args.n_res, args.msa_rows, args.num_recycles
    cfg = dict(CFG, depth=args.depth)
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = A.attach_structure_module(A.Alphafold2(**cfg, max_seq_len=max(n, 2048), predict_coords=True))
    randomize_zero_init_(model)
    model = model.to(dev).eval()
    seq = torch.randint(0, 21, (1, n), device=dev)
    msa = torch.randint(0, 21, (1, S, n), device=dev)
    card = _card(dev)
    for T in args.templates:
        kw = dict(mask=torch.ones(1, n, dtype=torch.bool, device=dev), msa_mask=torch.ones(1, S, n, dtype=torch.bool, device=dev))
        if T:
            g = torch.Generator(device=dev).manual_seed(5)
            kw.update(templates_feats=torch.randn(1, T, n, n, model.to_template_embed.in_features, device=dev, generator=g),
                      templates_angles=torch.randn(1, T, n, model.template_angle_mlp[0].in_features, device=dev, generator=g),
                      templates_mask=torch.ones(1, T, n, dtype=torch.bool, device=dev))
        runs = {"manual": lambda: manual_loop(model, seq, msa, R, **kw),
                "recycle": lambda: A.recycle(model, seq, msa, num_recycles=R, return_confidence=True, **kw)}
        res = {"T": T, "num_recycles": R, "steps": args.steps,
               "what": f"Alphafold2(dim={cfg['dim']}, depth={cfg['depth']}, heads={cfg['heads']}, dim_head={cfg['dim_head']}, "
                       f"predict_coords=True) N_res={n} MSA={S}x{n} batch=1, {T} templates, {R} recycles; ms per prediction, "
                       "CUDA events"}
        outs = {}
        for name in ("manual", "recycle"):
            ops.release_workspace(dev)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            with torch.no_grad():
                outs[name] = tuple(t.cpu() for t in runs[name]())
            torch.cuda.synchronize()
            res[f"peak_alloc_{name}_bytes"] = torch.cuda.max_memory_allocated(dev)
        res["outputs_equal"] = all(torch.equal(a, b) for a, b in zip(outs["manual"], outs["recycle"]))
        res["template_reuse"] = getattr(model, "last_template_reuse", None) if T else None
        times = {"manual": [], "recycle": []}
        with torch.no_grad():
            for rnd in range(args.steps + (1 if args.steps > 1 else 0)):
                for name in ("manual", "recycle"):
                    torch.cuda.synchronize()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    runs[name]()
                    b.record()
                    b.synchronize()
                    if rnd > 0 or args.steps == 1:
                        times[name].append(a.elapsed_time(b))
        for name, ts in times.items():
            res[f"{name}_ms"] = statistics.median(ts)
            res[f"{name}_ms_min_max"] = [min(ts), max(ts)]
        res["saving"] = 1 - res["recycle_ms"] / res["manual_ms"]
        print(json.dumps(dict(res, **card)), flush=True)


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
