"""torchrun --nproc-per-node P tests/parallel_check_multi_gpu_uneven.py : the sharded trunk on P GPUs over uneven shards
(P does not divide N_res or the MSA depth) vs the single-GPU path, with CUDA-graph replay equal to the eager schedule.

With NCCL the row <-> column re-layouts run as the chunk-table peer-store kernel (af2_peer_exchange_chunks) over CUDA IPC
when every rank can map the others' arenas, else as NCCL all_to_all with split sizes.  Sizes are chosen per P so that
every case is uneven for it, including one without an MSA (S = 1: P - 1 empty MSA shards)."""
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
from alphafold2_b200.parallel import _GraphedTrunk, shard_offsets, sharded_evoformer_forward  # noqa: E402
from oracle import evoformer_oracle as O  # noqa: E402


def _cases(P):
    """(d, H, dh, N, S, masked), N and S not multiples of P (S = 1 is uneven for any P >= 2)."""
    up = lambda n: n + 1 if n % P == 0 else n  # noqa: E731
    return [(64, 2, 32, up(12 * P + 1), up(2 * P + 1), True), (64, 2, 32, up(16 * P + P // 2 + 1), 1, False),
            (256, 8, 64, up(32 * P + 1), up(4 * P + 3), True), (128, 4, 32, up(64 * P + 3), up(P + 2), False)]


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    ok = True
    for (d, H, dh, N, S, masked) in _cases(world):
        torch.manual_seed(0)
        evo = A.Evoformer(depth=2, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
        st = O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.05)
        evo.load_state_dict(st)
        evo = evo.cuda().eval()
        x, m = torch.randn(1, N, N, d), torch.randn(1, S, N, d)
        mask = msa_mask = None
        if masked:
            m1 = torch.ones(1, N, dtype=torch.bool); m1[:, -N // 8:] = False
            mask = m1[:, :, None] & m1[:, None, :]
            msa_mask = torch.rand(1, S, N) > 0.1
            msa_mask[:, 0] = True
        cu = lambda t: None if t is None else t.cuda()  # noqa: E731
        xs, ms = sharded_evoformer_forward(evo, x.cuda(), m.cuda(), cu(mask), cu(msa_mask))
        xr, mr = sharded_evoformer_forward(evo, x.cuda(), m.cuda(), cu(mask), cu(msa_mask), gather_output=False)
        on, os_ = shard_offsets(N, world), shard_offsets(S, world)
        shards = torch.equal(xr, xs[0, on[rank]:on[rank + 1]]) and torch.equal(mr, ms[0, os_[rank]:os_[rank + 1]])
        x1, m1_ = evo(x.cuda(), m.cuda(), mask=cu(mask), msa_mask=cu(msa_mask))
        gt = _GraphedTrunk(evo, None)
        xg, mg = gt(x.cuda(), m.cuda(), cu(mask), cu(msa_mask))
        xg2, mg2 = gt((x * 1.0).cuda(), (m * 1.0).cuda(), cu(mask), cu(msa_mask))
        torch.cuda.synchronize()
        gt.release()
        h = hashlib.sha256(xs.cpu().numpy().tobytes() + ms.cpu().numpy().tobytes()).hexdigest()
        dig = torch.tensor([int(h[:15], 16)], dtype=torch.int64, device="cuda")
        lo, hi = dig.clone(), dig.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        res = {"rank": rank, "world": world, "cfg": [d, H, dh, N, S, masked],
               "x_vs_single": (xs - x1).abs().max().item(), "m_vs_single": (ms - m1_).abs().max().item(),
               "x_scale": x1.abs().max().item(), "m_scale": m1_.abs().max().item(),
               "ranks_bitwise_equal": bool(lo.item() == hi.item()), "shards_equal": bool(shards),
               "graph": "eager-fallback: " + gt.failed if gt.failed else "replayed",
               "graph_vs_eager": max((xg - xs).abs().max().item(), (mg - ms).abs().max().item(),
                                     (xg2 - xs).abs().max().item(), (mg2 - ms).abs().max().item())}
        if N <= 128 and rank == 0:
            rx, rm = O.evoformer({k: v.double() for k, v in st.items()}, "", x.double(), m.double(), H, 2, mask, msa_mask, chunk=16)
            res["x_vs_oracle_rel"] = ((xs.double().cpu() - rx).abs().max() / rx.pow(2).mean().sqrt()).item()
            res["m_vs_oracle_rel"] = ((ms.double().cpu() - rm).abs().max() / rm.pow(2).mean().sqrt()).item()
        good = (res["x_vs_single"] <= 2e-3 * res["x_scale"] and res["m_vs_single"] <= 2e-3 * res["m_scale"]
                and res["graph_vs_eager"] == 0.0 and res["ranks_bitwise_equal"] and res["shards_equal"])
        res["ok"] = bool(good)
        ok = ok and good
        print(json.dumps(res), flush=True)
    from alphafold2_b200 import parallel as par
    live = [ex for ex in par._PEER_ARENAS.values() if ex is not None]
    timeouts = any(ex.error() for ex in live)
    if rank == 0:
        print(json.dumps({"exchange": "peer-store kernel" if live else "nccl all_to_all", "arenas": len(par._PEER_ARENAS),
                          "barrier_timeouts": bool(timeouts)}), flush=True)
    ok = ok and not timeouts
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
