"""CPU: the sharded trunk (alphafold2_b200/parallel.py) over uneven shards, when the rank count P does not divide N_res or
the MSA depth S.

  * shard_offsets is the balanced split (the first n % P ranks hold one row more);
  * the chunk-table plans of the peer-store exchange, emulated byte by byte, give exactly the column and row shards of
    the full tensor, also with empty MSA shards; for even shapes they and the arena layout are those of the equal-shard
    exchange;
  * the schedule under gloo at world 2, 3 and 4 with oracle stage ops that accept uneven gathered pieces reproduces the
    single-process oracle, and with gather_output=False each rank returns its own rows;
  * N_res < P is refused before any collective or arena."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shard_offsets_are_balanced():
    from alphafold2_b200.parallel import shard_counts, shard_offsets
    for n in range(0, 40):
        for P in (1, 2, 3, 4, 5, 8, 32):
            off = shard_offsets(n, P)
            assert off[0] == 0 and off[-1] == n and len(off) == P + 1
            assert off == [r * (n // P) + min(r, n % P) for r in range(P + 1)]
            c = shard_counts(n, P)
            assert max(c) - min(c) <= 1 and c == sorted(c, reverse=True)


# ------------------------------------------------------------------------------------------------------------
# chunk-table plans of the peer-store exchange, emulated
# ------------------------------------------------------------------------------------------------------------
def _emulate_chunks(src_bytes, plans, dst_nbytes):
    """What af2_peer_exchange_chunks does with the arguments of PeerExchange.plan_*_ragged: rank r copies, for every peer p,
    chunks[p]["rows"] rows of chunks[p]["row_bytes"] from src[r] + src_off + row*src_row_stride to
    dst[p] + dst_off + row*dst_row_stride."""
    P = len(src_bytes)
    dst = [np.zeros(n, dtype=np.uint8) for n in dst_nbytes]
    for r in range(P):
        pl = plans[r]
        for p in range(P):
            c = pl["chunks"][p]
            for row in range(c["rows"]):
                so = c["src_off"] + row * pl["src_row_stride"]
                do = c["dst_off"] + row * c["dst_row_stride"]
                dst[p][do:do + c["row_bytes"]] = src_bytes[r][so:so + c["row_bytes"]]
    return dst


RAGGED_SHAPES = [   # rows of the track (N for the pair track, S for the MSA track), N (the columns), d, P
    (5, 5, 4, 2), (3, 5, 4, 2), (1, 5, 4, 2),
    (7, 7, 4, 3), (1, 7, 4, 3), (2, 8, 8, 3),
    (10, 10, 4, 4), (3, 9, 4, 4), (1, 6, 4, 4), (6, 9, 4, 4),
    (13, 13, 4, 8), (1, 61, 4, 8), (5, 11, 4, 8), (9, 12, 4, 8), (17, 20, 4, 8),
]


@pytest.mark.parametrize("n,C,d,P", RAGGED_SHAPES)
def test_ragged_plans_are_the_all_to_all_layouts(n, C, d, P):
    from alphafold2_b200.parallel import PeerExchange, shard_offsets
    full = torch.arange(n * C * d, dtype=torch.float32).view(n, C, d)
    ro, co = shard_offsets(n, P), shard_offsets(C, P)
    rows = [full[ro[r]:ro[r + 1]].contiguous() for r in range(P)]           # [R_r, C, d]
    cols = [full[:, co[r]:co[r + 1]].contiguous() for r in range(P)]        # [n, C_r, d]
    as_bytes = lambda t: np.frombuffer(t.numpy().tobytes(), dtype=np.uint8)  # noqa: E731
    plans = [PeerExchange.plan_rows_to_cols_ragged(ro, co, d, r) for r in range(P)]
    for pl in plans:                                                       # what the kernel's argument checks demand
        assert pl["src_row_stride"] % 16 == 0
        for c in pl["chunks"]:
            assert all(c[k] % 16 == 0 for k in ("src_off", "dst_off", "dst_row_stride", "row_bytes"))
            assert c["rows"] == 0 or c["row_bytes"] >= 16
    got = _emulate_chunks([as_bytes(t) for t in rows], plans, [t.numel() * 4 for t in cols])
    for r in range(P):
        assert np.array_equal(got[r], as_bytes(cols[r])), ("rows_to_cols", n, C, P, r)
    plans = [PeerExchange.plan_cols_to_rows_ragged(ro, co, d, r) for r in range(P)]
    back = _emulate_chunks(got, plans, [t.numel() * 4 for t in rows])
    for r in range(P):
        assert np.array_equal(back[r], as_bytes(rows[r])), ("cols_to_rows", n, C, P, r)


@pytest.mark.parametrize("n,C,d,P", [(8, 8, 4, 2), (16, 16, 4, 4), (24, 24, 8, 8), (6, 12, 4, 2), (12, 48, 64, 3)])
def test_ragged_plans_of_even_shapes_are_the_equal_shard_plans(n, C, d, P):
    """For shapes P divides the chunk table holds the equal-shard exchange's arguments, chunk p at p * src_peer_stride."""
    from alphafold2_b200.parallel import PeerExchange, shard_offsets
    ro, co = shard_offsets(n, P), shard_offsets(C, P)
    for r in range(P):
        for even, ragged in ((PeerExchange.plan_rows_to_cols(n // P, C, d, P, r), PeerExchange.plan_rows_to_cols_ragged(ro, co, d, r)),
                             (PeerExchange.plan_cols_to_rows(n, C // P, d, P, r), PeerExchange.plan_cols_to_rows_ragged(ro, co, d, r))):
            assert ragged["src_row_stride"] == even["src_row_stride"]
            for p, c in enumerate(ragged["chunks"]):
                assert c == dict(src_off=p * even["src_peer_stride"], dst_off=even["dst_off"], dst_row_stride=even["dst_row_stride"],
                                 rows=even["rows"], row_bytes=even["row_bytes"])


@pytest.mark.parametrize("N,P,d,K", [(7, 2, 3, 5), (50, 3, 2, 4), (61, 8, 2, 3), (259, 4, 2, 2), (13, 8, 4, 1)])
def test_merge_uneven_pieces_is_the_concatenation_of_unpadded_pieces(N, P, d, K):
    """CudaStageOps._merge_mn_pieces / _merge_k_pieces with per-piece sizes (host logic, no GPU): pieces gathered the way
    the schedule gathers them (each padded with -1 to the widest piece's align8 width, or to the tallest piece's rows)
    become the concatenation of the unpadded pieces, and the MN result's alignment columns are zero."""
    from alphafold2_b200.parallel import _align8, shard_counts, shard_offsets
    from alphafold2_b200.stages import CudaStageOps
    widths, off = shard_counts(N, P), shard_offsets(N, P)
    full = torch.arange(d * K * N, dtype=torch.float32).view(d, K, N)
    W = _align8(max(widths))
    pieces = []
    for p in range(P):                                   # MN-major: piece p = columns off[p].. of the full operand
        t = torch.full((d, K, W), -1.0)
        t[..., :widths[p]] = full[..., off[p]:off[p + 1]]
        pieces.append(t)
    merged, n_pieces = CudaStageOps._merge_mn_pieces(torch.cat(pieces, 0), tuple(widths), d, N)
    assert n_pieces == 1 and merged.shape == (d, K, _align8(N))
    assert torch.equal(merged[..., :N], full) and (merged[..., N:] == 0).all()
    fullk = torch.arange(d * N * 8, dtype=torch.float32).view(d, N, 8)
    pieces = []
    for p in range(P):                                   # K-major: piece p = rows off[p].. of the full operand
        t = torch.full((d, max(widths), 8), -1.0)
        t[:, :widths[p]] = fullk[:, off[p]:off[p + 1]]
        pieces.append(t)
    merged, n_pieces = CudaStageOps._merge_k_pieces(torch.cat(pieces, 0), tuple(widths), d)
    assert n_pieces == 1 and torch.equal(merged, fullk)


def _equal_shard_layout(N, S, d, P, ctrl):
    """The arena layout of the equal-shard exchange (before uneven shards were supported)."""
    al = lambda n: (n + 255) // 256 * 256  # noqa: E731
    pair_b, msa_b = al(N // P * N * d * 4), al(S // P * N * d * 4)
    return dict(off={(0, "row"): ctrl, (0, "col"): ctrl + pair_b, (1, "row"): ctrl + 2 * pair_b, (1, "col"): ctrl + 2 * pair_b + msa_b},
                shapes={(0, "row"): (N // P, N, d), (0, "col"): (N, N // P, d), (1, "row"): (S // P, N, d), (1, "col"): (S, N // P, d)},
                total=ctrl + 2 * pair_b + 2 * msa_b)


def test_layout():
    """Even shapes: the layout of the equal-shard exchange on every rank.  Uneven: one offset table for all ranks (each
    buffer sized for the largest shard), every rank's own shapes, buffers apart and inside the arena."""
    from alphafold2_b200 import _lib
    from alphafold2_b200.parallel import PeerExchange, shard_counts
    ctrl = int(_lib.load().af2_peer_ctrl_bytes())
    for (N, S, d, P) in [(40, 8, 64, 1), (136, 8, 256, 2), (48, 12, 64, 3), (256, 16, 128, 4), (32, 32, 4, 32)]:
        want = _equal_shard_layout(N, S, d, P, ctrl)
        for r in range(P):
            lay = PeerExchange.layout(N, S, d, P, r)
            assert {k: lay[k] for k in ("off", "shapes", "total")} == want
    for (N, S, d, P) in [(7, 3, 16, 2), (7, 7, 4, 4), (61, 1, 64, 8), (257, 5, 256, 2), (259, 18, 128, 4), (50, 7, 64, 3)]:
        lays = [PeerExchange.layout(N, S, d, P, r) for r in range(P)]
        assert all(lay["off"] == lays[0]["off"] and lay["total"] == lays[0]["total"] for lay in lays)
        cn, cs = shard_counts(N, P), shard_counts(S, P)
        for r, lay in enumerate(lays):
            assert lay["shapes"] == {(0, "row"): (cn[r], N, d), (0, "col"): (N, cn[r], d), (1, "row"): (cs[r], N, d), (1, "col"): (S, cn[r], d)}
        spans = sorted((lays[0]["off"][k], lays[0]["off"][k] + max(int(np.prod(lay["shapes"][k])) for lay in lays) * 4)
                       for k in lays[0]["off"])
        assert spans[0][0] == ctrl and spans[-1][1] <= lays[0]["total"]
        assert all(a[1] <= b[0] and b[0] % 256 == 0 for a, b in zip(spans, spans[1:]))


# ------------------------------------------------------------------------------------------------------------
# the schedule under gloo
# ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


SCHEDULE_SHAPES = [(7, 3, False), (10, 1, False), (9, 5, True)]      # N, S, masked


def _ragged_oracle_stage_ops():
    """The oracle stage ops (tests/stage_ops_oracle.py) extended to the gathered operands of uneven shards: when P does
    not divide N_res the schedule pads every rank's piece to the largest shard and passes the contraction the pair shard
    sizes instead of a piece count; these ops keep each piece's rows or columns and contract the compact operand as one
    piece, as CudaStageOps does.  `ragged_calls` counts the contractions that saw uneven pieces."""
    from stage_ops_oracle import OracleStageOps

    def cols(Rg, widths, d):              # [P*d, K, W], piece p's columns first -> [d, K, sum(widths)]
        src = Rg.view(len(widths), d, Rg.shape[1], Rg.shape[2])
        return torch.cat([src[p, :, :, :w] for p, w in enumerate(widths)], 2)

    def rows(Rg, heights, d):             # [P*d, Rmax, K], piece p's rows first -> [d, sum(heights), K]
        src = Rg.view(len(heights), d, Rg.shape[1], Rg.shape[2])
        return torch.cat([src[p, :, :h] for p, h in enumerate(heights)], 1)

    class RaggedOracleStageOps(OracleStageOps):
        ragged_calls = 0

        def outer_contract_(self, om, x_rows, L, Rg, msa_mask_full, row0, pieces):
            if not isinstance(pieces, int):
                self.ragged_calls += 1
                Rg, pieces = cols(Rg, pieces, L.shape[0]), 1
            super().outer_contract_(om, x_rows, L, Rg, msa_mask_full, row0, pieces)

        def tri_contract_(self, tm, x_loc, L, Rg, gate, ingoing, pieces):
            if not isinstance(pieces, int):
                self.ragged_calls += 1
                Rg, pieces = (cols if ingoing else rows)(Rg, pieces, L.shape[0]), 1
            super().tri_contract_(tm, x_loc, L, Rg, gate, ingoing, pieces)

    return RaggedOracleStageOps()


def _worker(rank, world, port, q):
    import sys
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import alphafold2_b200 as A
        from alphafold2_b200.parallel import shard_offsets, sharded_evoformer_forward
        from oracle import evoformer_oracle as O
        res = []
        for (N, S, masked) in SCHEDULE_SHAPES:
            torch.manual_seed(N * 10 + S)
            d, H, dh, depth = 16, 2, 8, 2
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
            ops = _ragged_oracle_stage_ops()
            xo, mo = sharded_evoformer_forward(evo, x, m, mask, msa_mask, group=None, stage_ops=ops)
            xr, mr = sharded_evoformer_forward(evo, x, m, mask, msa_mask, group=None, stage_ops=ops, gather_output=False)
            on, os_ = shard_offsets(N, world), shard_offsets(S, world)
            shards = torch.equal(xr, xo[0, on[rank]:on[rank + 1]]) and torch.equal(mr, mo[0, os_[rank]:os_[rank + 1]])
            rx, rm = O.evoformer({k: v.double() for k, v in st.items()}, "", x, m, H, depth, mask, msa_mask)
            res.append((N, S, masked, (xo.double() - rx).abs().max().item(), (mo.double() - rm).abs().max().item(), shards,
                        tuple(xo.shape), tuple(mo.shape), ops.ragged_calls))
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_ragged_schedule(world):
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
        for (N, S, masked, ex, em, shards, xs, ms, ragged_calls) in cases:
            what = f"rank {rank}/{world} N={N} S={S} masked={masked}"
            assert xs == (1, N, N, 16) and ms == (1, S, N, 16), what
            assert ex < 1e-4 and em < 1e-4, f"{what}: pair err {ex}, msa err {em}"
            assert shards, f"{what}: the row shards are not the rows of the gathered output"
            assert (ragged_calls > 0) == (N % world != 0), f"{what}: {ragged_calls} contractions saw uneven pieces"


def test_fewer_residues_than_ranks_is_refused_before_any_collective(monkeypatch):
    """N_res < P: ValueError before any collective, peer arena or stage op (one process posing as rank 0 of 4)."""
    import alphafold2_b200 as A
    from alphafold2_b200 import parallel

    def forbidden(*a, **k):
        raise AssertionError("reached a collective, a peer arena or a stage op")
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 4)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    for name in ("all_gather_into_tensor", "all_to_all_single", "all_reduce", "barrier"):
        monkeypatch.setattr(dist, name, forbidden)
    monkeypatch.setattr(parallel, "peer_exchange_for", forbidden)
    monkeypatch.setattr(parallel.PeerExchange, "create", forbidden)

    class NoOps:
        def __getattr__(self, name):
            forbidden()
    evo = A.Evoformer(depth=1, dim=16, seq_len=3, heads=2, dim_head=8, attn_dropout=0., ff_dropout=0.)
    x, m = torch.randn(1, 3, 3, 16), torch.randn(1, 2, 3, 16)
    for stage_ops in (None, NoOps()):
        with pytest.raises(ValueError, match="smaller than the number of ranks"):
            parallel.sharded_evoformer_forward(evo, x, m, stage_ops=stage_ops)
