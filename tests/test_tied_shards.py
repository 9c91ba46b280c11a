"""CPU: the sharded schedule (alphafold2_b200/parallel.py) honours tied-query ("global") column attention, the ingoing
triangle attention of the extra-MSA stack (AxialAttention(global_query_attn=True), alphafold2.py:142-151, 250).

Its queries are averaged over all N columns, but a rank holds only its column shard.  The schedule gives the stage op a
`reduce` callable that all-gathers every rank's partial query sums; the fp64 oracle stage ops below sum their shard's
queries, reduce, and attend with the mean of all N columns.  Under gloo at 2 and 3 ranks, even and uneven, the schedule
reproduces the single-process oracle Evoformer with global_column_attn=True, and a trunk without tied attention never
calls the tied stage op."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = [(8, 3, False), (9, 4, True), (7, 1, True)]      # N, S, masked (N = 7 and 9 are uneven at 2 and 3 ranks)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _tied_oracle_stage_ops():
    """OracleStageOps (fp64) with the tied column-attention stage op, and the uneven gathered pieces merged into the
    compact operand of the unsharded call (as CudaStageOps does)."""
    from stage_ops_oracle import OracleStageOps, _w

    def merge(Rg, sizes, d, dim):          # [P*d, ...] with piece p's first sizes[p] rows (dim 1) or columns (dim 2)
        src = Rg.view(len(sizes), d, Rg.shape[1], Rg.shape[2])
        return torch.cat([src[p].narrow(dim, 0, n) for p, n in enumerate(sizes)], dim)

    class TiedOracleStageOps(OracleStageOps):
        tied_calls = 0

        def outer_contract_(self, om, x_rows, L, Rg, msa_mask_full, row0, pieces):
            if not isinstance(pieces, int):
                Rg, pieces = merge(Rg, pieces, L.shape[0], 2), 1
            super().outer_contract_(om, x_rows, L, Rg, msa_mask_full, row0, pieces)

        def tri_contract_(self, tm, x_loc, L, Rg, gate, ingoing, pieces):
            if not isinstance(pieces, int):
                Rg, pieces = merge(Rg, pieces, L.shape[0], 2 if ingoing else 1), 1
            super().tri_contract_(tm, x_loc, L, Rg, gate, ingoing, pieces)

        def tied_column_attention_(self, ax, x, bias, mask, reduce, ncols_total):
            """x [h, w, d]: column attention over the h rows of each of the w local columns, with the query of row i the mean of
            q[i, j] over all ncols_total columns of every rank."""
            self.tied_calls += 1
            w = _w(ax, x.dtype)
            h, wc, d = x.shape
            H = ax.attn.heads
            xf = F.layer_norm(x, (d,), w["norm.weight"], w["norm.bias"], 1e-5).transpose(0, 1)      # [w, h, d]
            q = F.linear(xf, w["attn.to_q.weight"])                                                  # [w, h, I]
            I = q.shape[-1]
            dh = I // H
            parts = reduce((q * dh ** -0.5).sum(0).contiguous())                                     # [nparts * h, I]
            qm = parts.view(-1, h, I).sum(0) / ncols_total                                           # [h, I]
            k, v = F.linear(xf, w["attn.to_kv.weight"]).chunk(2, dim=-1)
            k, v = (t.reshape(wc, h, H, dh).permute(0, 2, 1, 3) for t in (k, v))                     # [w, H, h, dh]
            dots = torch.einsum("hid,bhjd->bhij", qm.view(h, H, dh).permute(1, 0, 2), k)
            if bias is not None:
                dots = dots + bias[None, :, :, :h].to(dots.dtype)
            if mask is not None:
                mf = mask.transpose(0, 1)                                                            # [w, h]
                dots = dots.masked_fill(~(mf[:, None, :, None] & mf[:, None, None, :]), -torch.finfo(dots.dtype).max)
            out = torch.einsum("bhij,bhjd->bhid", dots.softmax(-1), v).permute(0, 2, 1, 3).reshape(wc, h, I)
            out = out * F.linear(xf, w["attn.gating.weight"], w["attn.gating.bias"]).sigmoid()
            x += F.linear(out, w["attn.to_out.weight"], w["attn.to_out.bias"]).transpose(0, 1)

    return TiedOracleStageOps()


def _worker(rank, world, port, q):
    import sys
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import alphafold2_b200 as A
        from alphafold2_b200.parallel import sharded_evoformer_forward
        from oracle import evoformer_oracle as O
        res = []
        for (N, S, masked) in SHAPES:
            for tied in (True, False):
                torch.manual_seed(N * 10 + S)
                d, H, dh, depth = 16, 2, 8, 2
                evo = A.Evoformer(depth=depth, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.,
                                  global_column_attn=tied)
                st = O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.3)
                evo.load_state_dict(st)
                evo = evo.double()
                x = torch.randn(1, N, N, d, dtype=torch.float64)
                m = torch.randn(1, S, N, d, dtype=torch.float64)
                mask = msa_mask = None
                if masked:
                    m1 = torch.ones(1, N, dtype=torch.bool)
                    m1[:, -2:] = False
                    mask = m1[:, :, None] & m1[:, None, :]
                    msa_mask = torch.rand(1, S, N) > 0.2
                    msa_mask[:, 0] = True
                ops = _tied_oracle_stage_ops()
                xo, mo = sharded_evoformer_forward(evo, x, m, mask, msa_mask, group=None, stage_ops=ops)
                st64 = {k: v.double() for k, v in st.items()}
                rx, rm = O.evoformer(st64, "", x, m, H, depth, mask, msa_mask, global_column_attn=tied)
                ux, _ = O.evoformer(st64, "", x, m, H, depth, mask, msa_mask, global_column_attn=not tied)
                res.append((N, S, masked, tied, (xo - rx).abs().max().item(), (mo - rm).abs().max().item(),
                            (ux - rx).abs().max().item(), ops.tied_calls))
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_tied_query_schedule(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, cases in res:
        for (N, S, masked, tied, ex, em, untied_gap, tied_calls) in cases:
            what = f"rank {rank}/{world} N={N} S={S} masked={masked} tied={tied}"
            assert ex < 1e-4 and em < 1e-4, f"{what}: pair err {ex}, msa err {em}"     # as tests/test_ragged_shards.py
            assert untied_gap > 1e-3, f"{what}: tied and untied attention agree to {untied_gap}: the case cannot tell them apart"
            assert tied_calls == (2 if tied else 0), f"{what}: {tied_calls} tied stage-op calls"
