"""Device time of the structure module on a shard of pair rows (CUDA events, one GPU):
   python tools/time_structure_rows.py [--steps 10] [--n-res 1024 2048 4096]  -> one JSON line

  layers     one structure layer at dim 256, heads 1 and 8, for each N_res: af2_structure_layer_rows_begin on the largest pair-row
             shard of P = 1, 2, 4, 8 ranks (ceil(N / P) rows, a [ceil(N / P), N, d] tensor) followed by _end on all N residues, and
             af2_structure_layer on the whole tensor: ms per layer, bytes of pair read (4 rows N d) and GB/s.  The all-gather of
             the to_out rows between the two halves is not in the time (it moves N d 4 bytes; with P processes it is a collective).
  forward    the C2 forward with coordinates (bench.py's model, structure_module_depth 4, heads 1) through
             shard_alphafold2(pair_rows=True) in a one-process NCCL group, against the unsharded Alphafold2.forward: the cost of
             the split, of the extra launches and of the one-rank collectives.  Eager schedule (use_graph=False) in both.
Speed on several GPUs is not measured here: it needs one GPU per rank.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import socket
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alphafold2_b200 as A  # noqa: E402
from alphafold2_b200 import ops  # noqa: E402
from time_structure import inputs, make_model, timed  # noqa: E402

D = 256


def layer_model(dev, heads):
    torch.manual_seed(0)
    model = A.attach_structure_module(A.Alphafold2(dim=D, depth=1, heads=8, dim_head=32, predict_coords=True,
                                                   structure_module_heads=heads))
    with torch.no_grad():
        for p in model.ipa_block.parameters():
            p.copy_(torch.randn_like(p) * p.shape[-1] ** -0.5)
    return model.to(dev).eval()


def layers(dev, n, heads, steps):
    pk = layer_model(dev, heads).structure_weights().packed()
    g = torch.Generator(device=dev).manual_seed(1)
    pair = torch.randn(1, n, n, D, device=dev, generator=g)
    single = torch.randn(1, n, D, device=dev, generator=g)
    quat = torch.zeros(1, n, 4, device=dev)
    quat[..., 0] = 1.
    trans, rot = torch.zeros(1, n, 3, device=dev), torch.eye(3, device=dev).repeat(1, n, 1, 1)
    o = torch.empty(1, n, D, device=dev)
    out = []
    for P in (1, 2, 4, 8):
        R = -(-n // P)
        rows = pair[:, :R]                                        # the leading rows: contiguous, the largest shard's size

        def step():
            ops.structure_layer_rows_begin_(pk, single, rows, None, quat, trans, rot, 0, out=o[:, :R])
            ops.structure_layer_rows_end_(pk, single, o, quat, trans, rot)

        ms = timed(step, steps)
        out.append(dict(n_res=n, heads=heads, dim=D, P=P, rows=R, ms=ms, pair_bytes=4 * R * n * D, gb_s=4 * R * n * D / ms / 1e6))
    ms = timed(lambda: ops.structure_layer_(pk, single, pair, None, quat, trans, rot), steps)
    out.append(dict(n_res=n, heads=heads, dim=D, P="whole", rows=n, ms=ms, pair_bytes=4 * n * n * D, gb_s=4 * n * n * D / ms / 1e6))
    return out


def forward(dev, steps):
    import torch.distributed as dist
    from alphafold2_b200 import parallel
    from bench import N_RES, N_SEQ
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
    try:
        model, rows = make_model(dev), parallel.shard_alphafold2(make_model(dev), use_graph=False, pair_rows=True)   # same weights
        seq, msa, mask, msa_mask = inputs(dev, N_RES, N_SEQ)
        with torch.no_grad():
            call = lambda m: m(seq, msa, mask=mask, msa_mask=msa_mask, return_confidence=True)  # noqa: E731
            res = {"unsharded_ms": [], "pair_rows_p1_ms": []}
            for _ in range(3):                                    # alternated: the spread is part of the result
                res["unsharded_ms"].append(timed(lambda: call(model), steps))
                res["pair_rows_p1_ms"].append(timed(lambda: call(rows), steps))
            res["coords_bitwise_equal"] = bool(torch.equal(call(model)[0], call(rows)[0]))
        return res
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--n-res", type=int, nargs="*", default=[1024, 2048, 4096])
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    out = {"layers": []}
    for n in args.n_res:
        for heads in (1, 8):
            out["layers"] += layers(dev, n, heads, args.steps)
            torch.cuda.empty_cache()
    out["forward_c2"] = forward(dev, args.steps)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out["gpu"] = gpu.stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
