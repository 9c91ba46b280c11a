"""torchrun --nproc-per-node P tests/parallel_check_multi_gpu_model.py : parallel.shard_alphafold2 on P GPUs vs the single-GPU
forward, with the trunk's and the extra-MSA stack's CUDA-graph replay equal to the eager schedule.

Covers what one GPU cannot: the peer-store exchange over CUDA IPC (the template pair stack reuses the arena the trunk holds
for the same N_res and dim; the first forward, which runs the templates before any arena exists, uses NCCL all-to-alls),
the NCCL all-gather of the tied queries' partial sums, and that gather as a node of the extra-MSA stack's captured graph.
Two forwards per case: the first creates the arenas and captures the graphs, the second replays them; both must give the
same distogram."""
import hashlib
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))   # repo root (this file lives in tests/)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import alphafold2_b200 as A  # noqa: E402
from alphafold2_b200 import parallel  # noqa: E402
from oracle import evoformer_oracle as O  # noqa: E402


def _cases(P):
    """(d, n, S, T): n a multiple of P and one that is not."""
    return [(64, 24 * P, 4, 2), (128, 24 * P + 1, 5, 3)]


def _digest_equal(t):
    h = hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()
    dig = torch.tensor([int(h[:15], 16)], dtype=torch.int64, device="cuda")
    lo, hi = dig.clone(), dig.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    return bool(lo.item() == hi.item())


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    ok = True
    for (d, n, S, T) in _cases(world):
        torch.manual_seed(0)
        model = A.Alphafold2(dim=d, depth=2, heads=2, dim_head=32, max_seq_len=n, extra_msa_evoformer_layers=2,
                             templates_embed_layers=2)
        model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05))
        model = model.cuda().eval()
        seq = torch.randint(0, 21, (1, n)).cuda()
        mask = torch.ones(1, n, dtype=torch.bool).cuda()
        mask[:, -n // 8:] = False
        tmask = torch.rand(1, T, n) > 0.1
        tmask[:, -1] = False
        kw = dict(msa=torch.randint(0, 21, (1, S, n)), msa_mask=torch.rand(1, S, n) > 0.1,
                  templates_feats=torch.randn(1, T, n, n, 32), templates_mask=tmask, templates_angles=torch.randn(1, T, n, 55),
                  extra_msa=torch.randint(0, 21, (1, S, n)), extra_msa_mask=torch.rand(1, S, n) > 0.1)
        kw = {k: v.cuda() for k, v in kw.items()}
        single = model(seq, mask=mask, **kw).distance
        parallel.shard_alphafold2(model)
        first = model(seq, mask=mask, **kw).distance
        second = model(seq, mask=mask, **kw).distance
        torch.cuda.synchronize()
        graphs = {name: ("eager-fallback: " + g.failed if g.failed else f"replayed, {g.launches_per_replay} launches")
                  for name, g in (("trunk", model.net._af2_graph), ("extra", model.extra_msa_evoformer._af2_graph))}
        res = {"rank": rank, "world": world, "cfg": [d, n, S, T], "graphs": graphs,
               "vs_single": (first - single).abs().max().item(), "scale": single.abs().max().item(),
               "replay_vs_first": (second - first).abs().max().item(), "ranks_bitwise_equal": _digest_equal(first)}
        good = (res["vs_single"] <= 2e-3 * res["scale"] and res["replay_vs_first"] == 0.0 and res["ranks_bitwise_equal"]
                and not any(v.startswith("eager") for v in graphs.values()))
        res["ok"] = bool(good)
        ok = ok and good
        print(json.dumps(res), flush=True)
        parallel.release_all_graphs()
    live = [ex for ex in parallel._PEER_ARENAS.values() if ex is not None]
    timeouts = any(ex.error() for ex in live)
    if rank == 0:
        print(json.dumps({"exchange": "peer-store kernel" if live else "nccl all_to_all", "arenas": len(parallel._PEER_ARENAS),
                          "barrier_timeouts": bool(timeouts)}), flush=True)
    ok = ok and not timeouts
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
