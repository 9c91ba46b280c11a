"""-m gpu: parallel.shard_alphafold2(pair_rows=True) with P ranks on ONE GPU (the harness of tests/test_gpu_sharded_model_ranks.py:
P processes on cuda:0 in a gloo group, collectives staged through host memory), at P = 2, 3 and 4, even and uneven N_res, on an
Alphafold2 with templates (one of them fully masked), template angles, an extra MSA with its mask, recyclables and the angle
heads, in both omega modes.  Gates, on every rank:
  * ret.pair_rows is shard_offsets(N, P)[r:r + 2];
  * the rank's rows of distance / theta / phi / omega are bitwise those rows of the default shard_alphafold2 forward, and
    gather_pair_rows joins the distance shards into the default's whole distogram, bitwise;
  * the peak allocated memory of the rows forward is below the default forward's by at least what the replicated pair tensor
    costs beyond the rank's own rows, (1 - 1/P) 4 N^2 d bytes; both peaks are printed.  (At these sizes the grow-only
    workspace dominates both peaks, and the default mode's peak falls where it holds one whole pair tensor, not two.)
and on rank 0: the distogram within 2e-3 * max of the unsharded Alphafold2.forward and check() against the fp64 oracle.
Not covered here: the peer-store exchange, NCCL and graph replay (they need one GPU per rank)."""
import os
import types

import pytest
import torch

import test_gpu_sharded_model_ranks as H

pytestmark = pytest.mark.gpu

# P, n, S, T, symmetrize_omega   (d = 128: the distogram head kernel's smallest dim)
CASES = [
    (2, 40, 4, 1, False),      # even
    (3, 43, 5, 3, True),       # pair shards 15/14/14
    (4, 48, 4, 2, False),      # even
    (4, 50, 5, 2, True),       # pair shards 13/13/12/12
]
D = 128


def _peak(fn):
    from alphafold2_b200 import ops
    ops.release_workspace(torch.device("cuda", 0))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def _run_rows(rank, P, case):
    import torch.distributed as dist
    import alphafold2_b200 as A
    from alphafold2_b200 import parallel
    from gpu_util import check, to64
    from oracle import evoformer_oracle as O
    from oracle import recycling_oracle as RO
    n, S, T, sym = case
    torch.manual_seed(0)
    model = A.Alphafold2(dim=D, depth=2, heads=2, dim_head=32, max_seq_len=n, extra_msa_evoformer_layers=2, templates_embed_layers=2,
                         predict_angles=True, symmetrize_omega=sym)
    st = O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05)
    model.load_state_dict(st)
    model = model.cuda().eval()
    seq, mask, kw = H._model_inputs(D, n, S, T)
    names = ("distance", "theta_logits", "phi_logits", "omega_logits")
    single = model(seq, mask=mask, **kw).distance.cpu() if rank == 0 else None
    parallel.shard_alphafold2(model, use_graph=False)
    ref, mem_default = _peak(lambda: model(seq, mask=mask, **kw))
    ref = {k: getattr(ref, k).cpu() for k in names}
    parallel.shard_alphafold2(model, use_graph=False, pair_rows=True)
    ret, mem_rows = _peak(lambda: model(seq, mask=mask, **kw))
    on = parallel.shard_offsets(n, P)
    n0, n1 = on[rank], on[rank + 1]
    rows = {k: getattr(ret, k).cpu() for k in names}
    res = {"pair_rows_ok": tuple(ret.pair_rows) == (n0, n1), "mem": (mem_default, mem_rows), "pair_bytes": 4 * n * n * D}
    res["rows_equal"] = {k: rows[k].shape[1] == n1 - n0 and torch.equal(rows[k].view(torch.int32), ref[k][:, n0:n1].contiguous().view(torch.int32))
                         for k in names}
    whole = parallel.gather_pair_rows(ret.distance).cpu()
    res["gathered_equal"] = torch.equal(whole.view(torch.int32), ref["distance"].view(torch.int32))
    res["digest"] = tuple(float(v.double().sum()) for v in ref.values())
    if rank == 0:
        res.update(vs_single=(whole - single).abs().max().item(), scale=single.abs().max().item())
        rc = kw["recyclables"]
        rec = types.SimpleNamespace(coords=rc.coords.double().cpu(), single_msa_repr_row=rc.single_msa_repr_row.double().cpu(),
                                    pairwise_repr=rc.pairwise_repr.double().cpu())
        c = {k: v.cpu() for k, v in kw.items() if torch.is_tensor(v)}
        ref64 = RO.alphafold2_distogram(to64(st), seq.cpu(), c["msa"], mask.cpu(), c["msa_mask"], 2, 2, recyclables=rec,
                                        templates_feats=c["templates_feats"], templates_mask=c["templates_mask"],
                                        templates_angles=c["templates_angles"], templates_embed_layers=2, dtype=torch.float64,
                                        extra_msa_mask=c["extra_msa_mask"], extra_depth=2)
        res["vs_oracle"] = check(f"sharded_pair_rows_p{P}_one_gpu/n{n}S{S}T{T}sym{int(sym)}/distance", whole, ref64)["max_rel"]
    dist.barrier()
    return res


def _worker(rank, P, port, case, q):
    import datetime
    import sys
    import traceback
    import torch.distributed as dist
    sys.path[:0] = [H.ROOT, os.path.join(H.ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    res = {"rank": rank}
    try:
        from test_gpu_sharded_ranks_uneven import _stage_collectives_through_host
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=300))
        try:
            _stage_collectives_through_host()
            res.update(_run_rows(rank, P, case))
        finally:
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res["error"] = traceback.format_exc()
    q.put(res)


def _spawn(P, case):
    import queue
    import torch.multiprocessing as mp
    from test_gpu_sharded_ranks_uneven import _free_port
    if torch.cuda.is_initialized():
        import gc
        from alphafold2_b200 import ops
        gc.collect()
        ops.release_workspace(torch.device("cuda", 0))
        torch.cuda.empty_cache()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, P, port, case, q)) for r in range(P)]
    res = []
    try:
        for p in procs:
            p.start()
        while len(res) < P:
            try:
                res.append(q.get(timeout=600))
            except queue.Empty:
                break
            if "error" in res[-1]:
                break
    finally:
        for p in procs:
            p.join(timeout=60)
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    errors = [r for r in res if "error" in r]
    assert not errors, f"rank {errors[0]['rank']}:\n{errors[0]['error']}"
    assert len(res) == P, f"{P - len(res)} of {P} ranks did not report within the timeout"
    return sorted(res, key=lambda r: r["rank"])


@pytest.mark.parametrize("P,n,S,T,sym", CASES)
def test_shard_alphafold2_pair_rows_one_gpu(P, n, S, T, sym):
    res = _spawn(P, (n, S, T, sym))
    r0 = res[0]
    assert len({r["digest"] for r in res}) == 1, "the default mode's outputs differ between ranks"
    for r in res:
        print(f"  rank {r['rank']}: peak allocated {r['mem'][1] / 2**20:.2f} MiB pair_rows, {r['mem'][0] / 2**20:.2f} MiB default "
              f"(one fp32 pair tensor: {r['pair_bytes'] / 2**20:.2f} MiB; P={P} processes on one GPU)")
        assert r["pair_rows_ok"], r["rank"]
        assert all(r["rows_equal"].values()), (r["rank"], r["rows_equal"])
        assert r["gathered_equal"], r["rank"]
        assert r["mem"][0] - r["mem"][1] >= (1 - 1 / P) * r["pair_bytes"], (r["rank"], r["mem"], r["pair_bytes"])
    assert r0["vs_single"] <= 2e-3 * r0["scale"], r0
    print(f"pair_rows P={P} n={n} S={S} T={T} sym={sym}: distogram vs single {r0['vs_single'] / r0['scale']:.3e} max, "
          f"vs fp64 max_rel {r0['vs_oracle']:.3e}")
