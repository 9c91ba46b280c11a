"""Device time of the recycling embedder at the C2 shape (CUDA events):
   python tools/time_recycling.py [--steps 10]  -> one JSON line

Model and inputs as bench.py's C2 step (dim 256, depth 12, heads 8, dim_head 64, N_res 256, MSA 128 x 256, batch 1, all-ones
masks) plus recyclables (coordinates about 40 A from the origin, previous pair and MSA-row representations).  Reported:
  forward_ms / forward_without_recyclables_ms   Alphafold2.forward with and without recyclables, ms per call
  kernel                                        af2_recycle_embed alone: the library's per-launch CUDA events (class "misc" of
                                                one call), ms, algorithmic bytes (x and the previous pair read, x written, the
                                                same for row 0 of m, coordinates, table), GB/s and share of the H100 SXM data
                                                sheet's 3.35 TB/s
  eager_ms                                      alphafold2.py:730-739 restated in eager PyTorch on the same GPU (LayerNorms,
                                                cdist, bucketize, embedding gather, adds): a yardstick
The card name and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alphafold2_b200 as A  # noqa: E402
from alphafold2_b200 import _lib  # noqa: E402
from bench import CFG, N_RES, N_SEQ, randomize_zero_init_  # noqa: E402

HBM_DATASHEET = 3.35e12
KC_MISC = 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    torch.manual_seed(0)
    model = A.Alphafold2(**CFG)
    randomize_zero_init_(model)
    model = model.to(dev).eval()
    d = CFG["dim"]
    seq = torch.randint(0, 21, (1, N_RES), device=dev)
    msa = torch.randint(0, 21, (1, N_SEQ, N_RES), device=dev)
    mask = torch.ones(1, N_RES, dtype=torch.bool, device=dev)
    msa_mask = torch.ones(1, N_SEQ, N_RES, dtype=torch.bool, device=dev)
    g = torch.Generator(device=dev).manual_seed(5)
    rec = A.Recyclables(torch.randn(1, N_RES, 3, device=dev, generator=g) * 12.0 + 23.0,
                        torch.randn(1, N_RES, d, device=dev, generator=g), torch.randn(1, N_RES, N_RES, d, device=dev, generator=g))
    x = torch.randn(1, N_RES, N_RES, d, device=dev)
    m = torch.randn(1, N_SEQ, N_RES, d, device=dev)

    def eager(x, m):
        mn, pn, emb = model.recycling_msa_norm, model.recycling_pairwise_norm, model.recycling_distance_embed
        m[:, 0] = m[:, 0] + F.layer_norm(rec.single_msa_repr_row, (d,), mn.weight, mn.bias)
        x = x + F.layer_norm(rec.pairwise_repr, (d,), pn.weight, pn.bias)
        dist = torch.cdist(rec.coords, rec.coords, p=2)
        bnd = torch.linspace(2, 20, steps=model.recycling_distance_buckets, device=dev)
        return x + emb(torch.bucketize(dist, bnd[:-1])), m

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

    res = {"steps": args.steps,
           "what": f"Alphafold2(dim={d}, depth={CFG['depth']}, heads={CFG['heads']}, dim_head={CFG['dim_head']}) "
                   f"N_res={N_RES} MSA={N_SEQ}x{N_RES} batch=1, recyclables; ms per call, CUDA events"}
    res["forward_ms"] = timed(lambda: model(seq, msa, mask=mask, msa_mask=msa_mask, recyclables=rec))
    res["forward_without_recyclables_ms"] = timed(lambda: model(seq, msa, mask=mask, msa_mask=msa_mask))
    res["embed_recyclables_ms"] = timed(lambda: model.embed_recyclables_(x, m, rec))
    res["eager_ms"] = timed(lambda: eager(x, m))
    lib.af2_profile_enable(1)
    with torch.no_grad():
        for _ in range(args.steps):
            model.embed_recyclables_(x, m, rec)
    msd, fl, byd = C.c_double(), C.c_double(), C.c_double()
    launches = lib.af2_profile_read(KC_MISC, C.byref(msd), C.byref(fl), C.byref(byd))
    lib.af2_profile_enable(0)
    ms, by = msd.value / max(launches, 1), byd.value / max(launches, 1)
    rate = by / (ms * 1e-3) if ms > 0 else None
    res["kernel"] = {"launches": launches, "ms": ms, "algorithmic_bytes": by, "gbs": rate / 1e9 if rate else None,
                     "frac_of_hbm_datasheet": rate / HBM_DATASHEET if rate else None,
                     "datasheet_bound_ms": by / HBM_DATASHEET * 1e3}
    res["gpu"] = torch.cuda.get_device_name(dev)
    try:
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        res["power_limit_w"] = f"unavailable: {ex}"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
