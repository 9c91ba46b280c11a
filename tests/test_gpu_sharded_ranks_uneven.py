"""-m gpu: the sharded trunk over uneven shards (P does not divide N_res or the MSA depth) at P ranks on ONE GPU, with
the real CudaStageOps; the harness of tests/test_gpu_sharded_ranks.py, its host-staged all-to-all extended to split sizes.

P processes on cuda:0 form a gloo group, so the schedule takes its collective path: every stage op is the sm_90a kernels,
the all-to-alls carry split sizes, the gathered pieces are padded to the largest shard, and every contraction reads the
pieces merged into one compact operand.  The collectives are staged through host memory (copy to the CPU, gloo on uint8
views, copy back), which moves every byte unchanged.  Gates per Evoformer case: the gathered (x, m) are bitwise equal on
every rank; they are within 2e-3 * max|x| (max|m|) of the unsharded Evoformer on the same GPU; rank 0 passes check()
against the fp64 oracle; with gather_output=False each rank's shards are its rows of the gathered output, bit for bit;
and the MSA return on the side stream gives the same bits as the return in line.  The Alphafold2.forward cases run the
whole model through shard_evoformer(model, use_graph=False): without an MSA (S = 1), and with template angle rows that
make S + T rows; gate: the distogram logits bitwise equal on every rank and within 2e-3 * max of the unsharded forward.
Not covered here: the peer-store exchange between processes, NCCL and the CUDA-graph replay
(tests/parallel_check_multi_gpu_uneven.py on several GPUs)."""
import datetime
import hashlib
import os
import queue
import socket
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# P, d, H, dh, N, S, masked
CASES = [
    (3, 64, 2, 32, 50, 7, True),       # pair shards 17/17/16, MSA shards 3/2/2
    (8, 64, 2, 32, 61, 1, False),      # S = 1: seven empty MSA shards
    (2, 256, 8, 64, 257, 5, True),     # pieces of 129 and 128 columns; the 128-column shard's ingoing contraction is padded
                                       # to 129 columns so that it runs the unsharded call's channel -> token kernel
    (4, 128, 4, 32, 259, 18, False),   # pieces of 65 and 64 columns
]
# P, d, n, S (0: no MSA), T (template angle rows)
MODEL_CASES = [
    (3, 64, 40, 0, 0),                 # model(seq, mask=mask): S = 1
    (4, 64, 45, 5, 2),                 # S + T = 7 MSA rows
]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _stage_collectives_through_host():
    """The two collectives of the schedule on CUDA tensors, carried by gloo on uint8 host copies (bit-exact transport);
    the all-to-all with or without split sizes."""
    all_gather, all_to_all = dist.all_gather_into_tensor, dist.all_to_all_single

    def host_bytes(t):
        return t.detach().contiguous().cpu().reshape(-1).view(torch.uint8)

    def all_gather_into_tensor(out, t, group=None, async_op=False):
        assert not async_op and out.is_contiguous()
        host = torch.empty(out.numel() * out.element_size(), dtype=torch.uint8)
        all_gather(host, host_bytes(t), group=group)
        out.copy_(host.view(out.dtype).view(out.shape))

    def all_to_all_single(out, t, output_split_sizes=None, input_split_sizes=None, group=None, async_op=False):
        assert not async_op and out.is_contiguous()
        host = torch.empty(out.numel() * out.element_size(), dtype=torch.uint8)
        if output_split_sizes is None and input_split_sizes is None:
            all_to_all(host, host_bytes(t), group=group)
        else:                                                  # split sizes count dim-0 slices: scale them to bytes
            unit_in = t.element_size() * (t[0].numel() if t.dim() > 1 else 1)
            unit_out = out.element_size() * (out[0].numel() if out.dim() > 1 else 1)
            all_to_all(host, host_bytes(t), output_split_sizes=[s * unit_out for s in output_split_sizes],
                       input_split_sizes=[s * unit_in for s in input_split_sizes], group=group)
        out.copy_(host.view(out.dtype).view(out.shape))

    dist.all_gather_into_tensor, dist.all_to_all_single = all_gather_into_tensor, all_to_all_single


def _digest(*ts):
    return hashlib.sha256(b"".join(t.contiguous().numpy().tobytes() for t in ts)).hexdigest()


def _run_evoformer(rank, P, case):
    import alphafold2_b200 as A
    from alphafold2_b200 import parallel
    from gpu_util import check, to64
    from oracle import evoformer_oracle as O
    d, H, dh, N, S, masked = case
    torch.manual_seed(0)                                   # every rank builds the same weights and inputs
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
    args = (evo, x.cuda(), m.cuda(), cu(mask), cu(msa_mask))
    assert parallel.OVERLAP_MSA_RETURN
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
        rx, rm = O.evoformer(to64(st), "", x.double(), m.double(), H, 2, mask, msa_mask, chunk=16)
        res["x_vs_oracle"] = check(f"sharded_uneven_p{P}_one_gpu/d{d}N{N}S{S}/x", xs, rx)["max_rel"]
        res["m_vs_oracle"] = check(f"sharded_uneven_p{P}_one_gpu/d{d}N{N}S{S}/m", ms, rm)["max_rel"]
    return res


def _run_model(rank, P, case):
    import alphafold2_b200 as A
    from alphafold2_b200 import parallel
    from oracle import evoformer_oracle as O
    d, n, S, T = case
    torch.manual_seed(0)
    model = A.Alphafold2(dim=d, depth=2, heads=2, dim_head=32, max_seq_len=n)
    model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05))
    model = model.cuda().eval()
    seq = torch.randint(0, 21, (1, n))
    mask = torch.ones(1, n, dtype=torch.bool)
    mask[:, -n // 8:] = False
    kw = {}
    if S:
        kw["msa"] = torch.randint(0, 21, (1, S, n))
        kw["msa_mask"] = torch.rand(1, S, n) > 0.1
    if T:
        kw["templates_angles"] = torch.randn(1, T, n, 55)
        kw["templates_mask"] = torch.ones(1, T, n, dtype=torch.bool)
    kw = {k: v.cuda() for k, v in kw.items()}
    res = {}
    if rank == 0:
        single = model(seq.cuda(), mask=mask.cuda(), **kw).distance.cpu()
    parallel.shard_evoformer(model, use_graph=False)
    dist_sharded = model(seq.cuda(), mask=mask.cuda(), **kw).distance.cpu()
    res["digest"] = _digest(dist_sharded)
    res["shards_equal"] = res["inline_return_equal"] = True
    if rank == 0:
        res.update(x_vs_single=(dist_sharded - single).abs().max().item(), x_scale=single.abs().max().item(),
                   m_vs_single=0.0, m_scale=1.0, x_vs_oracle=float("nan"), m_vs_oracle=float("nan"))
    return res


def _worker(rank, P, port, kind, case, q):
    import sys
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    res = {"rank": rank}
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=300))
        try:
            _stage_collectives_through_host()
            res.update((_run_evoformer if kind == "evoformer" else _run_model)(rank, P, case))
        finally:
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res["error"] = traceback.format_exc()
    q.put(res)


def _spawn(P, kind, case):
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
    assert len({r["digest"] for r in res}) == 1, "the gathered outputs differ between ranks"
    assert all(r["shards_equal"] for r in res), [r["rank"] for r in res if not r["shards_equal"]]
    assert all(r["inline_return_equal"] for r in res), [r["rank"] for r in res if not r["inline_return_equal"]]
    assert r0["x_vs_single"] <= 2e-3 * r0["x_scale"], r0
    assert r0["m_vs_single"] <= 2e-3 * r0["m_scale"], r0
    return r0


@pytest.mark.parametrize("P,d,H,dh,N,S,masked", CASES)
def test_sharded_uneven_one_gpu(P, d, H, dh, N, S, masked):
    r0 = _spawn(P, "evoformer", (d, H, dh, N, S, masked))
    print(f"sharded uneven P={P} d={d} N={N} S={S}: x vs single {r0['x_vs_single'] / r0['x_scale']:.3e} max|x|, m vs single "
          f"{r0['m_vs_single'] / r0['m_scale']:.3e} max|m|; x vs fp64 {r0['x_vs_oracle']:.3e}, m vs fp64 {r0['m_vs_oracle']:.3e}")


@pytest.mark.parametrize("P,d,n,S,T", MODEL_CASES)
def test_alphafold2_sharded_uneven_one_gpu(P, d, n, S, T):
    r0 = _spawn(P, "model", (d, n, S, T))
    print(f"Alphafold2 sharded P={P} n={n} S={S} T={T}: distogram vs single {r0['x_vs_single'] / r0['x_scale']:.3e} max")
