"""-m gpu: all of an Alphafold2's pair-tensor work sharded over P ranks on ONE GPU (the harness of
tests/test_gpu_sharded_ranks_uneven.py: P processes on cuda:0 in a gloo group, collectives staged through host memory).

  * A tied-query Evoformer (global_column_attn=True, the extra-MSA stack) through sharded_evoformer_forward at P = 2, 3 and 4,
    even and uneven.  Gates: the gathered outputs bitwise equal on every rank; the gather_output=False shards equal to the
    gathered rows; the MSA return in line equal to the overlapped one; within 2e-3 * max of the single-GPU tied Evoformer;
    check() against the fp64 oracle.
  * parallel.shard_alphafold2 on an Alphafold2 with templates (one of them fully masked), template angles, an extra MSA with
    its mask and recyclables, at P = 2 and 3.  Gates: the distogram bitwise equal on every rank and within 2e-3 * max of the
    unsharded forward; x after the sharded template branch within 2e-3 * max|x| of the unsharded branch.  Each rank's peak
    allocated memory in the template branch is printed beside the unsharded branch's.
Not covered here: the peer-store exchange between processes, NCCL and graph replay (tests/parallel_check_multi_gpu_model.py)."""
import datetime
import os
import queue
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# P, d, H, dh, N, S, masked
TIED_CASES = [
    (2, 64, 2, 32, 48, 4, True),       # even
    (3, 64, 2, 32, 50, 7, True),       # pair shards 17/17/16, MSA shards 3/2/2
    (4, 128, 4, 32, 64, 8, False),     # even
    (4, 128, 4, 32, 66, 5, False),     # pair shards 17/17/16/16, MSA shards 2/1/1/1
]
# P, d, n, S, T (templates; the last one fully masked when T > 1)
MODEL_CASES = [
    (2, 64, 40, 4, 1),
    (3, 64, 43, 5, 3),
]


def _run_tied(rank, P, case):
    import alphafold2_b200 as A
    from alphafold2_b200 import parallel
    from gpu_util import check, to64
    from oracle import evoformer_oracle as O
    from test_gpu_sharded_ranks_uneven import _digest
    d, H, dh, N, S, masked = case
    torch.manual_seed(0)
    evo = A.Evoformer(depth=2, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0., global_column_attn=True)
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
    args = (evo, x.cuda(), m.cuda(), cu(mask), cu(msa_mask))
    xs, ms = (t.cpu() for t in parallel.sharded_evoformer_forward(*args))
    res = {"digest": _digest(xs, ms)}
    xr, mr = parallel.sharded_evoformer_forward(*args, gather_output=False)
    on, os_ = parallel.shard_offsets(N, P), parallel.shard_offsets(S, P)
    res["shards_equal"] = torch.equal(xr.cpu(), xs[0, on[rank]:on[rank + 1]]) and torch.equal(mr.cpu(), ms[0, os_[rank]:os_[rank + 1]])
    parallel.OVERLAP_MSA_RETURN = False
    try:
        xi, mi = (t.cpu() for t in parallel.sharded_evoformer_forward(*args))
    finally:
        parallel.OVERLAP_MSA_RETURN = True
    res["inline_return_equal"] = torch.equal(xi, xs) and torch.equal(mi, ms)
    if rank == 0:
        x1, m1_ = (t.cpu() for t in evo(x.cuda(), m.cuda(), mask=cu(mask), msa_mask=cu(msa_mask)))
        res.update(x_vs_single=(xs - x1).abs().max().item(), x_scale=x1.abs().max().item(),
                   m_vs_single=(ms - m1_).abs().max().item(), m_scale=m1_.abs().max().item())
        rx, rm = O.evoformer(to64(st), "", x.double(), m.double(), H, 2, mask, msa_mask, chunk=16, global_column_attn=True)
        res["x_vs_oracle"] = check(f"sharded_tied_p{P}_one_gpu/d{d}N{N}S{S}/x", xs, rx)["max_rel"]
        res["m_vs_oracle"] = check(f"sharded_tied_p{P}_one_gpu/d{d}N{N}S{S}/m", ms, rm)["max_rel"]
    return res


def _model_inputs(d, n, S, T):
    from alphafold2_b200 import Recyclables
    seq = torch.randint(0, 21, (1, n))
    mask = torch.ones(1, n, dtype=torch.bool)
    mask[:, -n // 8:] = False
    tmask = torch.rand(1, T, n) > 0.1
    if T > 1:
        tmask[:, -1] = False                                      # a template with no valid residue
    kw = dict(msa=torch.randint(0, 21, (1, S, n)), msa_mask=torch.rand(1, S, n) > 0.1,
              templates_feats=torch.randn(1, T, n, n, 32), templates_mask=tmask, templates_angles=torch.randn(1, T, n, 55),
              extra_msa=torch.randint(0, 21, (1, S, n)), extra_msa_mask=torch.rand(1, S, n) > 0.1)
    kw = {k: v.cuda() for k, v in kw.items()}
    kw["recyclables"] = Recyclables(coords=torch.randn(1, n, 3).cuda() * 5, single_msa_repr_row=torch.randn(1, n, d).cuda(),
                                    pairwise_repr=torch.randn(1, n, n, d).cuda())
    return seq.cuda(), mask.cuda(), kw


def _run_model(rank, P, case):
    import alphafold2_b200 as A
    from alphafold2_b200 import ops, parallel
    from oracle import evoformer_oracle as O
    from test_gpu_sharded_ranks_uneven import _digest
    d, n, S, T = case
    torch.manual_seed(0)
    model = A.Alphafold2(dim=d, depth=2, heads=2, dim_head=32, max_seq_len=n, extra_msa_evoformer_layers=2, templates_embed_layers=2)
    model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05))
    model = model.cuda().eval()
    seq, mask, kw = _model_inputs(d, n, S, T)
    # the template branch alone, on the same x
    x0 = torch.randn(1, n, n, d, device="cuda")
    x_mask = mask[:, :, None] & mask[:, None, :]
    dev = torch.device("cuda", 0)

    def branch(fn):
        x = x0.clone()
        ops.release_workspace(dev)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with torch.no_grad():
            fn(x, x_mask, kw["templates_feats"], kw["templates_mask"])
        torch.cuda.synchronize()
        return x.cpu(), torch.cuda.max_memory_allocated() - base

    x_single, mem_single = branch(model.embed_templates_)
    single = model(seq, mask=mask, **kw).distance.cpu()
    parallel.shard_alphafold2(model, use_graph=False)
    x_sharded, mem_sharded = branch(model.embed_templates_)
    dist_sharded = model(seq, mask=mask, **kw).distance.cpu()
    res = {"digest": _digest(dist_sharded), "shards_equal": True, "inline_return_equal": True,
           "mem": (mem_single, mem_sharded), "template_x_digest": _digest(x_sharded)}
    if rank == 0:
        res.update(x_vs_single=(dist_sharded - single).abs().max().item(), x_scale=single.abs().max().item(),
                   m_vs_single=(x_sharded - x_single).abs().max().item(), m_scale=x_single.abs().max().item())
    return res


def _worker(rank, P, port, kind, case, q):
    import sys
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    res = {"rank": rank}
    try:
        from test_gpu_sharded_ranks_uneven import _stage_collectives_through_host
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=300))
        try:
            _stage_collectives_through_host()
            res.update((_run_tied if kind == "tied" else _run_model)(rank, P, case))
        finally:
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res["error"] = traceback.format_exc()
    q.put(res)


def _spawn(P, kind, case):
    from test_gpu_sharded_ranks_uneven import _free_port
    if torch.cuda.is_initialized():          # the ranks share the GPU with this process: return what earlier tests left cached
        import gc
        from alphafold2_b200 import ops
        gc.collect()
        ops.release_workspace(torch.device("cuda", 0))
        torch.cuda.empty_cache()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, P, port, kind, case, q)) for r in range(P)]
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
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res.sort(key=lambda r: r["rank"])
    r0 = res[0]
    assert len({r["digest"] for r in res}) == 1, "the outputs differ between ranks"
    assert all(r["shards_equal"] for r in res), [r["rank"] for r in res if not r["shards_equal"]]
    assert all(r["inline_return_equal"] for r in res), [r["rank"] for r in res if not r["inline_return_equal"]]
    assert r0["x_vs_single"] <= 2e-3 * r0["x_scale"], r0
    assert r0["m_vs_single"] <= 2e-3 * r0["m_scale"], r0
    return res


@pytest.mark.parametrize("P,d,H,dh,N,S,masked", TIED_CASES)
def test_sharded_tied_evoformer_one_gpu(P, d, H, dh, N, S, masked):
    r0 = _spawn(P, "tied", (d, H, dh, N, S, masked))[0]
    print(f"sharded tied P={P} d={d} N={N} S={S}: x vs single {r0['x_vs_single'] / r0['x_scale']:.3e} max|x|, m vs single "
          f"{r0['m_vs_single'] / r0['m_scale']:.3e} max|m|; x vs fp64 {r0['x_vs_oracle']:.3e}, m vs fp64 {r0['m_vs_oracle']:.3e}")


@pytest.mark.parametrize("P,d,n,S,T", MODEL_CASES)
def test_shard_alphafold2_one_gpu(P, d, n, S, T):
    res = _spawn(P, "model", (d, n, S, T))
    r0 = res[0]
    assert len({r["template_x_digest"] for r in res}) == 1, "the template branch's x differs between ranks"
    print(f"shard_alphafold2 P={P} n={n} S={S} T={T}: distogram vs single {r0['x_vs_single'] / r0['x_scale']:.3e} max, "
          f"x after the template branch vs single {r0['m_vs_single'] / r0['m_scale']:.3e} max|x|")
    for r in res:
        print(f"  rank {r['rank']}: template branch peak allocated {r['mem'][1] / 2**20:.1f} MiB sharded, "
              f"{r['mem'][0] / 2**20:.1f} MiB unsharded (this process, P={P} processes on one GPU)")
