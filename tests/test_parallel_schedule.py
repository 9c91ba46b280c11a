"""CPU, world_size 2 and 4, gloo: the axis-sharded Evoformer schedule (alphafold2_b200/parallel.py) reproduces the
single-process oracle when its stage ops are the oracle math.  Checks slicing, all-to-all layouts, operand
gathers and the collective order -- everything of the N>1 path except the CUDA kernels themselves."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, masked, q):
    import sys
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import alphafold2_b200 as A
        from alphafold2_b200.parallel import sharded_evoformer_forward
        from oracle import evoformer_oracle as O
        from stage_ops_oracle import OracleStageOps
        torch.manual_seed(0)
        d, H, dh, N, S, depth = 16, 2, 8, 8, 4, 2
        evo = A.Evoformer(depth=depth, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
        st = O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.3)
        evo.load_state_dict(st)
        evo = evo.double()
        x = torch.randn(1, N, N, d, dtype=torch.float64)
        m = torch.randn(1, S, N, d, dtype=torch.float64)
        mask = msa_mask = None
        if masked:
            m1 = torch.ones(1, N, dtype=torch.bool); m1[:, -2:] = False
            mask = m1[:, :, None] & m1[:, None, :]
            msa_mask = torch.rand(1, S, N) > 0.2
            msa_mask[:, 0] = True
        xo, mo = sharded_evoformer_forward(evo, x, m, mask, msa_mask, group=None, stage_ops=OracleStageOps())
        rx, rm = O.evoformer({k: v.double() for k, v in st.items()}, "", x, m, H, depth, mask, msa_mask)
        # the sharded path works on fp32 shards (the product's residual-stream dtype): compare at fp32 accuracy
        ex = (xo.double() - rx).abs().max().item()
        em = (mo.double() - rm).abs().max().item()
        q.put((rank, ex, em))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("masked,world", [(False, 2), (True, 2), (True, 4)])
def test_sharded_schedule(masked, world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, masked, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, ex, em in res:
        assert ex < 1e-4 and em < 1e-4, f"rank {rank}: pair err {ex}, msa err {em}"


def test_merge_gathered_pieces_drops_alignment_padding():
    """CudaStageOps._merge_mn_pieces (host logic, no GPU): P gathered pieces [d, K, align8(w)] become one operand
    [d, K, align8(P*w)] whose column p*w + c is column c of piece p -- the padding columns of every piece are dropped
    (they were kept once: wrong pair rows at 8 GPUs whenever N/P is not a multiple of 8)."""
    import torch

    from alphafold2_b200.parallel import _align8
    from alphafold2_b200.stages import CudaStageOps
    for (n_total, P, d, K) in [(48, 8, 4, 3), (40, 2, 3, 5), (64, 8, 2, 2), (256, 8, 2, 4)]:
        w = n_total // P
        full = torch.arange(d * K * n_total, dtype=torch.float32).view(d, K, n_total)
        pieces = []
        for p in range(P):
            t = torch.full((d, K, _align8(w)), -1.0)
            t[..., :w] = full[..., p * w:(p + 1) * w]
            pieces.append(t)
        Rg = torch.cat(pieces, 0)
        merged, n_pieces = CudaStageOps._merge_mn_pieces(Rg, P, d, n_total)
        assert n_pieces == 1 and merged.shape == (d, K, _align8(n_total))
        assert torch.equal(merged[..., :n_total], full)
        assert (merged[..., n_total:] == 0).all()
    wide = torch.zeros(8 * 2, 3, 64)
    same, n_pieces = CudaStageOps._merge_mn_pieces(wide, 8, 2, 512)          # >= 64 columns per piece: addressed in place
    assert same is wide and n_pieces == 8


def _emulate_peer_exchange(src_bytes, plans, dst_nbytes):
    """What csrc/peer_api.inl's kernel does with the arguments of PeerExchange.plan_*: rank r copies, for every peer p,
    `rows` rows of `row_bytes` from src[r] + p*src_peer_stride + row*src_row_stride to dst[p] + dst_off + row*dst_row_stride."""
    import numpy as np
    P = len(src_bytes)
    dst = [np.zeros(dst_nbytes, dtype=np.uint8) for _ in range(P)]
    for r in range(P):
        pl = plans[r]
        for p in range(P):
            for row in range(pl["rows"]):
                so = p * pl["src_peer_stride"] + row * pl["src_row_stride"]
                do = pl["dst_off"] + row * pl["dst_row_stride"]
                dst[p][do:do + pl["row_bytes"]] = src_bytes[r][so:so + pl["row_bytes"]]
    return dst


def test_peer_exchange_plans_are_the_all_to_all_layouts():
    """Host arithmetic of the peer-store exchange (no GPU): emulating the kernel's copies with the planned strides and
    offsets on P simulated ranks gives exactly the column shards / row shards of the full tensor."""
    import numpy as np
    import torch

    from alphafold2_b200.parallel import PeerExchange
    for (N, C, d, P) in [(8, 8, 4, 2), (16, 16, 4, 4), (24, 24, 8, 8), (6, 12, 4, 2)]:
        full = torch.arange(N * C * d, dtype=torch.float32).view(N, C, d)
        R, Cl = N // P, C // P
        rows = [full[r * R:(r + 1) * R].contiguous() for r in range(P)]                       # [R, C, d]
        cols = [full[:, r * Cl:(r + 1) * Cl].contiguous() for r in range(P)]                  # [N, Cl, d]
        nbytes = R * C * d * 4
        as_bytes = lambda t: np.frombuffer(t.numpy().tobytes(), dtype=np.uint8)              # noqa: E731
        plans = [PeerExchange.plan_rows_to_cols(R, C, d, P, r) for r in range(P)]
        got = _emulate_peer_exchange([as_bytes(t) for t in rows], plans, nbytes)
        for r in range(P):
            assert np.array_equal(got[r], as_bytes(cols[r])), ("rows_to_cols", N, C, d, P, r)
        plans = [PeerExchange.plan_cols_to_rows(N, Cl, d, P, r) for r in range(P)]
        back = _emulate_peer_exchange(got, plans, nbytes)
        for r in range(P):
            assert np.array_equal(back[r], as_bytes(rows[r])), ("cols_to_rows", N, C, d, P, r)
