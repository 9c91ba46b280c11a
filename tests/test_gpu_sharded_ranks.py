"""-m gpu: the sharded trunk (alphafold2_b200/parallel.py) at P ranks on ONE GPU, with the real CudaStageOps.

P processes on cuda:0 form a gloo group, so peer_exchange_for returns None and the schedule takes its collective path:
every stage op is the sm_90a kernels, every contraction gets P gathered operand pieces, and the row <-> column re-layouts
are all-to-alls.  The collectives are staged through host memory (copy to the CPU, gloo on uint8 views, copy back), which
moves every byte unchanged.  Gates per case: the gathered (x, m) are bitwise equal on every rank; they are within
2e-3 * max|x| of the unsharded Evoformer on the same GPU (the gate of test_gpu_parallel.py and of
tests/parallel_check_multi_gpu.py); rank 0 passes check() against the fp64 oracle; with gather_output=False each rank's
shards are its rows of the gathered output, bit for bit; and the MSA return on the side stream (OVERLAP_MSA_RETURN)
gives the same bits as the return in line.  Not covered here: the peer-store exchange between processes, NCCL and the
CUDA-graph replay (tests/parallel_check_multi_gpu.py on several GPUs)."""
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

# P, d, H, dh, N, S, masked.  The contraction paths follow from the piece width N/P (api.cu: af2_triangle_contract,
# af2_outer_contract; parallel.py: CudaStageOps._merge_mn_pieces merges MN-major pieces narrower than 64 columns).
CASES = [
    (8, 64, 2, 32, 48, 8, True),      # 6 per piece: outer-mean and ingoing pieces merged into one operand (the padding bug
                                      # once seen at 8 GPUs), outgoing one launch per piece
    (2, 64, 2, 32, 40, 8, False),     # 20 per piece: pitches padded to 24, merged MN pieces, outgoing one launch per piece
    (4, 128, 4, 32, 256, 16, True),   # 64 per piece: rank-4 maps in all three contractions; the outgoing 256-column box
                                      # spans 4 pieces
    (3, 64, 2, 32, 192, 12, True),    # odd rank count, rank-4 maps; the outgoing 256-column box spans 3 pieces and runs past them
    (2, 256, 8, 64, 136, 40, True),   # 68 per piece: one launch per piece in all three contractions
    (2, 64, 2, 32, 384, 8, False),    # 192 per piece: MN rank-4 maps over 3 boxes per piece, outgoing one launch per piece
]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _stage_collectives_through_host():
    """The two collectives of the schedule on CUDA tensors, carried by gloo on uint8 host copies (bit-exact transport)."""
    all_gather, all_to_all = dist.all_gather_into_tensor, dist.all_to_all_single

    def host_bytes(t):
        return t.detach().contiguous().cpu().reshape(-1).view(torch.uint8)

    def all_gather_into_tensor(out, t, group=None, async_op=False):
        assert not async_op and out.is_contiguous()
        host = torch.empty(out.numel() * out.element_size(), dtype=torch.uint8)
        all_gather(host, host_bytes(t), group=group)
        out.copy_(host.view(out.dtype).view(out.shape))

    def all_to_all_single(out, t, output_split_sizes=None, input_split_sizes=None, group=None, async_op=False):
        assert output_split_sizes is None and input_split_sizes is None and not async_op and out.is_contiguous()
        host = torch.empty(out.numel() * out.element_size(), dtype=torch.uint8)
        all_to_all(host, host_bytes(t), group=group)
        out.copy_(host.view(out.dtype).view(out.shape))

    dist.all_gather_into_tensor, dist.all_to_all_single = all_gather_into_tensor, all_to_all_single


def _run(rank, P, case):
    import alphafold2_b200 as A
    from alphafold2_b200 import parallel
    from gpu_util import check, to64
    from oracle import evoformer_oracle as O
    _stage_collectives_through_host()
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
    res = {"digest": hashlib.sha256(xs.numpy().tobytes() + ms.numpy().tobytes()).hexdigest()}
    xr, mr = parallel.sharded_evoformer_forward(*args, gather_output=False)
    Rn, Rs = N // P, S // P
    res["shards_equal"] = torch.equal(xr.cpu(), xs[0, rank * Rn:(rank + 1) * Rn]) and torch.equal(mr.cpu(), ms[0, rank * Rs:(rank + 1) * Rs])
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
        res["x_vs_oracle"] = check(f"sharded_p{P}_one_gpu/d{d}N{N}/x", xs, rx)["max_rel"]
        res["m_vs_oracle"] = check(f"sharded_p{P}_one_gpu/d{d}N{N}/m", ms, rm)["max_rel"]
    return res


def _worker(rank, P, port, case, q):
    import sys
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    res = {"rank": rank}
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=300))
        try:
            res.update(_run(rank, P, case))
        finally:
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res["error"] = traceback.format_exc()
    q.put(res)


@pytest.mark.parametrize("P,d,H,dh,N,S,masked", CASES)
def test_sharded_ranks_one_gpu(P, d, H, dh, N, S, masked):
    if torch.cuda.is_initialized():          # the ranks share the GPU with this process: return what earlier tests left cached
        import gc
        from alphafold2_b200 import ops
        gc.collect()
        ops.release_workspace(torch.device("cuda", 0))
        torch.cuda.empty_cache()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, P, port, (d, H, dh, N, S, masked), q)) for r in range(P)]
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
    print(f"sharded P={P} d={d} N={N} S={S}: x vs single {r0['x_vs_single'] / r0['x_scale']:.3e} max|x|, m vs single "
          f"{r0['m_vs_single'] / r0['m_scale']:.3e} max|m|; x vs fp64 {r0['x_vs_oracle']:.3e} rms, m vs fp64 {r0['m_vs_oracle']:.3e} rms")
    assert len({r["digest"] for r in res}) == 1, "the gathered outputs differ between ranks"
    assert all(r["shards_equal"] for r in res), [r["rank"] for r in res if not r["shards_equal"]]
    assert all(r["inline_return_equal"] for r in res), [r["rank"] for r in res if not r["inline_return_equal"]]
    assert r0["x_vs_single"] <= 2e-3 * r0["x_scale"], r0
    assert r0["m_vs_single"] <= 2e-3 * r0["m_scale"], r0
