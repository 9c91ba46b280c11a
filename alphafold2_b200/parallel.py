"""Axis-sharded Evoformer trunk over the GPUs of one node (one process per GPU, torch.distributed / NCCL).

The reference has no multi-device path (SURVEY.md §2.2); this is the GPU-native addition named by the north
star: one sequence's forward is split over the MSA-row and pair-row axes (FastFold-DAP style).  At block entry
rank r owns pair rows x[r*N/P:(r+1)*N/P, :, :] and MSA rows m[r*S/P:(r+1)*S/P, :, :]; weights are replicated.
Every sub-op is embarrassingly parallel along ONE axis, so the schedule switches the sharded axis with
all-to-alls and all-gathers the one operand a contraction needs in full (SURVEY.md §8e):

  per block: 3 small all-gathers (pair bias, H*N*N bf16), 3 operand all-gathers (outer-mean right, triangle
  right x2; bf16 channel-major), 2 all-to-alls of m, 4 all-to-alls of x (fp32 residual stream).

"A single all-gather per block" (north star) is not dependency-feasible with exact semantics; the real count is
stated above and measured by bench.py --gpus N.  The compute between collectives is the same sm_90a kernels as
the single-GPU path (stage-level C ABI: af2_pair_bias / *_project / *_contract / af2_axial_attention_prebias).

`ops` is the stage-op provider: CudaStageOps (product, C ABI).  tests/ plug in a CPU oracle provider to check the
schedule itself (slicing, layouts, collectives) under gloo with world_size 2.
"""
from __future__ import annotations

import ctypes as C
import os
import weakref
from typing import Optional

import torch
import torch.distributed as dist

from . import _lib, ops as _ops


def _align8(n: int) -> int:
    return (n + 7) // 8 * 8


# ------------------------------------------------------------------------------------------------------------
# collectives (concatenate along dim 0 so that both NCCL and gloo accept them)
# ------------------------------------------------------------------------------------------------------------
def all_gather_cat0(t: torch.Tensor, group) -> torch.Tensor:
    P = dist.get_world_size(group)
    out = torch.empty((P * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t.contiguous(), group=group)
    return out


def rows_to_cols(t_row: torch.Tensor, group) -> torch.Tensor:
    """[R, C, d] (my R rows, all C columns) -> [P*R, C/P, d] (all rows, my columns)."""
    P = dist.get_world_size(group)
    R, Cc, d = t_row.shape
    send = t_row.view(R, P, Cc // P, d).permute(1, 0, 2, 3).contiguous()      # chunk p: my rows x columns of rank p
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)                           # chunk p: rows of rank p x my columns
    return recv.view(P * R, Cc // P, d)


def cols_to_rows(t_col: torch.Tensor, group) -> torch.Tensor:
    """[P*R, Cl, d] (all rows, my Cl columns) -> [R, P*Cl, d] (my rows, all columns)."""
    P = dist.get_world_size(group)
    RR, Cl, d = t_col.shape
    R = RR // P
    send = t_col.contiguous().view(P, R, Cl, d)                               # chunk p: rows of rank p x my columns
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)                           # chunk p: my rows x columns of rank p
    return recv.permute(1, 0, 2, 3).reshape(R, P * Cl, d)


class _Deferred:
    """cols_to_rows on a side stream: the MSA tensor goes back to row shards while the pair track of the same block runs
    (nothing reads it before the next block's row attention).  With NCCL the collective itself runs on the process
    group's stream either way and the side stream removes the main stream's wait for it; with the peer-memory exchange
    (ex) the exchange kernel itself runs on the side stream, on barrier channel 1.  `get()` joins."""

    def __init__(self, t_col: torch.Tensor, group, side, ex=None):
        cur = torch.cuda.current_stream()
        if ex is not None:
            ready = cur.record_event()
            with torch.cuda.stream(side):
                side.wait_event(ready)
                self.out = ex.cols_to_rows(t_col, PeerExchange.MSA, channel=1)
                self.done = side.record_event()
            self.keep = self.bufs = None
            return
        P = dist.get_world_size(group)
        RR, Cl, d = t_col.shape
        R = RR // P
        self.keep = t_col                                                     # source stays alive until the side stream is done
        send = t_col.contiguous().view(P, R, Cl, d)
        recv = torch.empty_like(send)                                         # allocated on the main stream: its pool, its ordering
        self.out = torch.empty(R, P * Cl, d, dtype=t_col.dtype, device=t_col.device)
        self.bufs = (send, recv)
        ready = cur.record_event()
        with torch.cuda.stream(side):
            side.wait_event(ready)
            dist.all_to_all_single(recv, send, group=group)
            self.out.view(R, P, Cl, d).copy_(recv.permute(1, 0, 2, 3))
            self.done = side.record_event()

    def get(self) -> torch.Tensor:
        torch.cuda.current_stream().wait_event(self.done)
        out, self.keep, self.bufs = self.out, None, None
        return out


# ------------------------------------------------------------------------------------------------------------
# peer-memory exchange: the row <-> column re-layouts as ONE kernel storing into the destination ranks' memory (NVLink)
# ------------------------------------------------------------------------------------------------------------
class _RawCuda:
    """A cudaMalloc'ed range presented to torch through the CUDA array interface (no copy, no ownership)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2, "strides": None}


PEER_EXCHANGE_ENABLED = os.environ.get("AF2_PEER_EXCHANGE", "1") not in ("", "0")
_PEER_ARENAS = {}           # (id(group), device index, N, S, d) -> PeerExchange | None (None: tried, not available)


class PeerExchange:
    """Row-shard <-> column-shard exchange of the pair and MSA tensors through peer memory (csrc/peer_api.inl).

    Every rank allocates one arena holding, for each of the two tracks, a row-layout buffer [R, C, d] and a column-layout
    buffer [P*R, C/P, d] (fp32), and maps the other ranks' arenas with CUDA IPC.  `rows_to_cols` / `cols_to_rows` launch one
    kernel that stores every chunk into its destination rank's buffer and joins a flag barrier; the returned tensor IS the
    local destination buffer.  The schedule strictly alternates the two layouts of a track, which is what makes one
    barrier per exchange sufficient: a rank starts writing a peer's buffer X only after that peer signalled the barrier
    of the exchange in which it last read X.  Single node only (IPC); `create` returns None when peer access, IPC or
    the array-interface wrapping is not available on every rank, and the schedule then uses NCCL all_to_all."""

    PAIR, MSA = 0, 1

    def __init__(self):
        self.base = None
        self.opened = []

    @classmethod
    def create(cls, group, device: torch.device, N: int, S: int, d: int):
        P, r = dist.get_world_size(group), dist.get_rank(group)
        lib = _lib.load()
        self = cls()
        self.group, self.P, self.rank, self.device = group, P, r, device
        ctrl = int(lib.af2_peer_ctrl_bytes())
        al = lambda n: (n + 255) // 256 * 256  # noqa: E731
        pair_b, msa_b = al(N // P * N * d * 4), al(S // P * N * d * 4)
        self.off = {(cls.PAIR, "row"): ctrl, (cls.PAIR, "col"): ctrl + pair_b,
                    (cls.MSA, "row"): ctrl + 2 * pair_b, (cls.MSA, "col"): ctrl + 2 * pair_b + msa_b}
        total = ctrl + 2 * pair_b + 2 * msa_b
        ok = P <= 32 and device.type == "cuda"
        handle = torch.zeros(72, dtype=torch.uint8)
        # 1. local arena + IPC handle (no collective inside: every rank reaches the all_gather below whatever happens here)
        try:
            if ok:
                base = C.c_void_p()
                _lib.check(lib.af2_peer_alloc(total, C.byref(base)))
                self.base = base.value
                hb = (C.c_ubyte * 64)()
                _lib.check(lib.af2_peer_export(self.base, hb))
                handle[:64] = torch.frombuffer(bytearray(hb), dtype=torch.uint8)
                handle[64] = 1
                handle[65] = device.index
                self.arena = torch.as_tensor(_RawCuda(self.base, total), device=device)
                if self.arena.data_ptr() != self.base:
                    raise RuntimeError("array-interface wrapping copied the arena")
        except Exception as e:  # noqa: BLE001
            ok = False
            self.why = f"{type(e).__name__}: {e}"
        if not ok:
            handle[64] = 0
        # 2. everyone's handle
        allh = torch.empty(P * 72, dtype=torch.uint8, device=device)
        dist.all_gather_into_tensor(allh, handle.to(device), group=group)
        allh = allh.cpu().view(P, 72)
        ok = ok and bool((allh[:, 64] == 1).all())
        # 3. map the peers
        bases = [0] * P
        if ok:
            try:
                for p in range(P):
                    if p == r:
                        bases[p] = self.base
                        continue
                    if not lib.af2_peer_can_access(device.index, int(allh[p, 65])):
                        raise RuntimeError(f"no peer access from device {device.index} to device {int(allh[p, 65])}")
                    hb = (C.c_ubyte * 64)(*allh[p, :64].tolist())
                    ptr = C.c_void_p()
                    _lib.check(lib.af2_peer_open(hb, C.byref(ptr)))
                    self.opened.append(ptr.value)
                    bases[p] = ptr.value
            except Exception as e:  # noqa: BLE001
                ok = False
                self.why = f"{type(e).__name__}: {e}"
        flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        if not int(flag.item()):
            why = getattr(self, "why", "another rank could not set it up")
            import sys
            print(f"[alphafold2_b200.parallel] rank {r}: peer-memory exchange not available ({why}); using NCCL all_to_all", file=sys.stderr)
            self._unmap_peers()
            dist.barrier(group=group)              # nobody frees an arena a peer still has mapped
            self._release_local()
            return None
        self.table = torch.tensor(bases, dtype=torch.int64, device=device)            # device array of the P arena bases
        self.shapes = {(cls.PAIR, "row"): (N // P, N, d), (cls.PAIR, "col"): (N, N // P, d),
                       (cls.MSA, "row"): (S // P, N, d), (cls.MSA, "col"): (S, N // P, d)}
        self.exchanges = 0
        return self

    def buffer(self, track: int, layout: str) -> torch.Tensor:
        shape = self.shapes[(track, layout)]
        n = shape[0] * shape[1] * shape[2] * 4
        o = self.off[(track, layout)]
        return self.arena[o:o + n].view(torch.float32).view(shape)

    def _exchange(self, src: torch.Tensor, src_peer_stride, src_row_stride, dst_off, dst_row_stride, rows, row_bytes, channel):
        _lib.check(_lib.load().af2_peer_exchange(src.data_ptr(), src_peer_stride, src_row_stride, self.table.data_ptr(), dst_off,
                                                  dst_row_stride, rows, row_bytes, channel, self.rank, self.P, _ops._stream_ptr()))
        self.exchanges += 1

    @staticmethod
    def plan_rows_to_cols(R: int, Cc: int, d: int, P: int, rank: int, itemsize: int = 4):
        """af2_peer_exchange arguments (bytes) that turn [R, Cc, d] row shards into [P*R, Cc/P, d] column shards:
        chunk p = my R rows x the Cc/P columns of rank p; it lands in rank p's column buffer at rows rank*R.. (contiguous).
        dst_off is relative to the destination buffer.  Pure arithmetic (tests/test_parallel_schedule.py emulates it)."""
        chunk = Cc // P * d * itemsize
        return dict(src_peer_stride=chunk, src_row_stride=Cc * d * itemsize, dst_off=rank * R * chunk, dst_row_stride=chunk,
                    rows=R, row_bytes=chunk)

    @staticmethod
    def plan_cols_to_rows(RR: int, Cl: int, d: int, P: int, rank: int, itemsize: int = 4):
        """The way back: [P*R, Cl, d] column shards -> [R, P*Cl, d] row shards.  Chunk p = the R rows of rank p x my Cl
        columns (contiguous at the source); it lands in rank p's row buffer at columns rank*Cl.. of every row."""
        R, chunk = RR // P, Cl * d * itemsize
        return dict(src_peer_stride=R * chunk, src_row_stride=chunk, dst_off=rank * chunk, dst_row_stride=P * chunk,
                    rows=R, row_bytes=chunk)

    def _run(self, src: torch.Tensor, plan: dict, dst_buffer_off: int, channel: int):
        self._exchange(src, plan["src_peer_stride"], plan["src_row_stride"], dst_buffer_off + plan["dst_off"], plan["dst_row_stride"],
                       plan["rows"], plan["row_bytes"], channel)

    def rows_to_cols(self, t_row: torch.Tensor, track: int, channel: int = 0) -> torch.Tensor:
        """[R, C, d] (my rows, all columns; the track's row buffer) -> the track's column buffer [P*R, C/P, d]."""
        R, Cc, d = t_row.shape
        assert t_row.data_ptr() == self.base + self.off[(track, "row")] and tuple(t_row.shape) == self.shapes[(track, "row")]
        self._run(t_row, self.plan_rows_to_cols(R, Cc, d, self.P, self.rank), self.off[(track, "col")], channel)
        return self.buffer(track, "col")

    def cols_to_rows(self, t_col: torch.Tensor, track: int, channel: int = 0) -> torch.Tensor:
        """[P*R, Cl, d] (all rows, my columns; the track's column buffer) -> the track's row buffer [R, P*Cl, d]."""
        RR, Cl, d = t_col.shape
        assert t_col.data_ptr() == self.base + self.off[(track, "col")] and tuple(t_col.shape) == self.shapes[(track, "col")]
        self._run(t_col, self.plan_cols_to_rows(RR, Cl, d, self.P, self.rank), self.off[(track, "row")], channel)
        return self.buffer(track, "row")

    def error(self) -> bool:
        return bool(self.base) and bool(_lib.load().af2_peer_error(self.base))

    def _unmap_peers(self):
        lib = _lib.load()
        for ptr in self.opened:
            lib.af2_peer_close(ptr)
        self.opened = []

    def _release_local(self):
        lib = _lib.load()
        self._unmap_peers()
        self.arena = None
        if self.base:
            lib.af2_peer_free(self.base)
            self.base = None

    def close(self):
        """Collective: unmap the peers, then free the arena (a rank frees only after everyone has unmapped it)."""
        if self.base is None:
            return
        torch.cuda.synchronize()
        self._unmap_peers()
        try:
            dist.barrier(group=self.group)
        except Exception:  # noqa: BLE001 - process group already gone: the driver reclaims the mappings at exit
            pass
        self._release_local()


def peer_exchange_for(group, device: torch.device, N: int, S: int, d: int):
    """The arena for this (group, shape), created on first use (collectively: every rank makes the same calls)."""
    if not PEER_EXCHANGE_ENABLED or device.type != "cuda" or dist.get_backend(group) != "nccl" or dist.get_world_size(group) < 2:
        return None
    key = (id(group), device.index, N, S, d)
    if key not in _PEER_ARENAS:
        if torch.cuda.is_current_stream_capturing():
            return None
        _PEER_ARENAS[key] = PeerExchange.create(group, device, N, S, d)
        _hook_teardown()
    return _PEER_ARENAS[key]


def release_peer_arenas() -> None:
    for key in list(_PEER_ARENAS):
        ex = _PEER_ARENAS.pop(key)
        if ex is not None:
            ex.close()


# ------------------------------------------------------------------------------------------------------------
# stage ops on the GPU (C ABI)
# ------------------------------------------------------------------------------------------------------------
class CudaStageOps:
    """Every method launches hand-written sm_90a kernels through libaf2b200.so; tensors are CUDA tensors."""

    def pair_bias(self, ax, x_rows: torch.Tensor) -> torch.Tensor:
        """bf16 [H, rows, align8(n)] = edges_to_attn_bias of a band of pair rows (raw, un-normalised x)."""
        pk = ax.packed()
        rows, n, d = x_rows.shape
        H = ax.attn.heads
        out = torch.zeros(H, rows, _align8(n), dtype=torch.bfloat16, device=x_rows.device)
        _lib.check(_lib.load().af2_pair_bias(x_rows.data_ptr(), pk.tensors["we"].data_ptr(), out.data_ptr(), rows, n, d, H,
                                             _ops._stream_ptr()))
        return out

    def axial_attention_(self, ax, x: torch.Tensor, bias: Optional[torch.Tensor], mask: Optional[torch.Tensor], row_attn: bool):
        """x [h, w, d] fp32 in place; bias bf16 [H, n, align8(n)] (n = attended length) or None."""
        pk = ax.packed()
        h, w, d = x.shape
        lib = _lib.load()
        nbytes = lib.af2_axial_attention_workspace(1, h, w, d, ax.attn.heads, ax.attn.dim_head, int(row_attn))
        ws = _ops.workspace(nbytes, x.device)
        m8 = None if mask is None else mask.contiguous()
        _lib.check(lib.af2_axial_attention_prebias(C.byref(pk.struct), x.data_ptr(), None if bias is None else bias.data_ptr(),
                                                   None if m8 is None else m8.data_ptr(), 1, h, w, d, ax.attn.heads,
                                                   ax.attn.dim_head, int(row_attn), ws.data_ptr(), ws.numel(), _ops._stream_ptr()))

    def feed_forward_(self, ff, x: torch.Tensor):
        _ops.feed_forward_(ff.packed(), x)

    def outer_project(self, om, m_cols: torch.Tensor, mask_cols: Optional[torch.Tensor]) -> torch.Tensor:
        """m [S, nl, d] -> bf16 [2d, S, align8(nl)] channel-major left | right."""
        pk = om.packed()
        S, nl, d = m_cols.shape
        out = torch.empty(2 * d, S, _align8(nl), dtype=torch.bfloat16, device=m_cols.device)
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_outer_project_workspace(S * nl, d), m_cols.device)
        mk = None if mask_cols is None else mask_cols.contiguous()
        _lib.check(lib.af2_outer_project(C.byref(pk.struct), m_cols.data_ptr(), None if mk is None else mk.data_ptr(), S * nl,
                                         nl, d, out.data_ptr(), S * _align8(nl), ws.data_ptr(), ws.numel(), _ops._stream_ptr()))
        return out

    @staticmethod
    def _merge_mn_pieces(Rg: torch.Tensor, pieces: int, d: int, n_total: int):
        """Gathered MN-major operand [pieces*d, K, align8(n_total/pieces)] with fewer than 64 columns per piece: the kernel's
        64-column TMA boxes cannot span pieces, so instead of `pieces` tiny launches the pieces are re-packed once into ONE
        operand [d, K, align8(n_total)] (a pass over the gathered tensor, ~10 us at C2) and contracted in a single launch.
        Each piece's alignment padding is dropped on the way: column p*(n_total/pieces)+c of the result is column c of piece p.
        Pieces of >= 64 columns are addressed in place."""
        K, w = Rg.shape[1], Rg.shape[2]
        if pieces == 1 or w >= 64:
            return Rg, pieces
        wt = n_total // pieces
        out = torch.zeros(d, K, _align8(n_total), dtype=Rg.dtype, device=Rg.device)
        out[:, :, :n_total].view(d, K, pieces, wt).copy_(Rg.view(pieces, d, K, w)[..., :wt].permute(1, 2, 0, 3))
        return out, 1

    def outer_contract_(self, om, x_rows: torch.Tensor, L: torch.Tensor, Rg: torch.Tensor, msa_mask_full, row0: int, pieces: int):
        """x_rows [rows, N, d] += OuterMean; L [d, S, align8(rows)], Rg [pieces*d, S, align8(N/pieces)]."""
        pk = om.packed()
        rows, N, d = x_rows.shape
        S = L.shape[1]
        Rg, pieces = self._merge_mn_pieces(Rg, pieces, d, N)
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_outer_contract_workspace(rows, N, d), x_rows.device)
        mk = None if msa_mask_full is None else msa_mask_full.contiguous()
        per_piece = Rg.numel() // pieces
        _lib.check(lib.af2_outer_contract(C.byref(pk.struct), x_rows.data_ptr(), L.data_ptr(), L.shape[1] * L.shape[2],
                                          Rg.data_ptr(), Rg.shape[1] * Rg.shape[2], per_piece, pieces,
                                          None if mk is None else mk.data_ptr(), row0, rows, N, S, d, float(om.eps),
                                          ws.data_ptr(), ws.numel(), _ops._stream_ptr()))

    def tri_project(self, tm, x_loc: torch.Tensor, mask_loc: Optional[torch.Tensor]):
        """x [rows, cols, d] -> (L, R) bf16 [d, rows, align8(cols)] channel-major, gate bf16 [rows*cols, d]."""
        pk = tm.packed()
        rows, cols, d = x_loc.shape
        L = torch.empty(d, rows, _align8(cols), dtype=torch.bfloat16, device=x_loc.device)
        R = torch.empty_like(L)
        gate = torch.empty(rows * cols, d, dtype=torch.bfloat16, device=x_loc.device)
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_triangle_project_workspace(rows * cols, d), x_loc.device)
        mk = None if mask_loc is None else mask_loc.contiguous()
        _lib.check(lib.af2_triangle_project(C.byref(pk.struct), x_loc.data_ptr(), None if mk is None else mk.data_ptr(),
                                            rows * cols, cols, d, L.data_ptr(), R.data_ptr(), rows * _align8(cols),
                                            gate.data_ptr(), ws.data_ptr(), ws.numel(), _ops._stream_ptr()))
        return L, R, gate

    def tri_contract_(self, tm, x_loc: torch.Tensor, L: torch.Tensor, Rg: torch.Tensor, gate: torch.Tensor, ingoing: bool, pieces: int):
        pk = tm.packed()
        rows, cols, d = x_loc.shape
        K = L.shape[1] if ingoing else cols
        if ingoing:
            Rg, pieces = self._merge_mn_pieces(Rg, pieces, d, rows)
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_triangle_contract_workspace(rows, cols, d), x_loc.device)
        per_piece = Rg.numel() // pieces
        _lib.check(lib.af2_triangle_contract(C.byref(pk.struct), x_loc.data_ptr(), L.data_ptr(), L.shape[1] * L.shape[2],
                                             Rg.data_ptr(), Rg.shape[1] * Rg.shape[2], per_piece, pieces, gate.data_ptr(),
                                             rows, cols, K, d, int(ingoing), ws.data_ptr(), ws.numel(), _ops._stream_ptr()))


# ------------------------------------------------------------------------------------------------------------
# the schedule
# ------------------------------------------------------------------------------------------------------------
def sharded_evoformer_forward(evo, x: torch.Tensor, m: torch.Tensor, mask: Optional[torch.Tensor] = None,
                              msa_mask: Optional[torch.Tensor] = None, group=None, stage_ops=None, gather_output: bool = True):
    """Evoformer.forward (alphafold2.py:458-467) for ONE sequence sharded over the ranks of `group`.

    x [1, N, N, d], m [1, S, N, d], mask [1, N, N] bool, msa_mask [1, S, N] bool are the full (replicated) inputs;
    returns the full (x, m) on every rank when gather_output, else this rank's row shards.
    """
    if stage_ops is None and _ops.precision_of(evo) == "strict":
        raise NotImplementedError("the strict precision mode runs on one GPU (it is a parity mode, not a throughput mode)")
    ops = stage_ops if stage_ops is not None else CudaStageOps()
    P = dist.get_world_size(group)
    r = dist.get_rank(group)
    if x.shape[0] != 1:
        raise ValueError("the sharded trunk handles one sequence per call (batch 1)")
    N, S = x.shape[1], m.shape[1]
    if N % P or S % P:
        raise ValueError(f"N_res={N} and N_seq={S} must be divisible by the number of ranks {P}")
    Rn, Rs = N // P, S // P
    with torch.no_grad():
        ex = peer_exchange_for(group, x.device, N, S, x.shape[-1]) if stage_ops is None else None
        if ex is not None:                                            # the shards live in the peer-mapped arena
            x_row, m_row = ex.buffer(PeerExchange.PAIR, "row"), ex.buffer(PeerExchange.MSA, "row")
            x_row.copy_(x[0, r * Rn:(r + 1) * Rn])
            m_row.copy_(m[0, r * Rs:(r + 1) * Rs])
            pair_to_cols = lambda t: ex.rows_to_cols(t, PeerExchange.PAIR)  # noqa: E731
            pair_to_rows = lambda t: ex.cols_to_rows(t, PeerExchange.PAIR)  # noqa: E731
            msa_to_cols = lambda t: ex.rows_to_cols(t, PeerExchange.MSA)  # noqa: E731
            msa_to_rows = lambda t: ex.cols_to_rows(t, PeerExchange.MSA)  # noqa: E731
        else:
            x_row = x[0, r * Rn:(r + 1) * Rn].detach().to(torch.float32).contiguous().clone()      # [N/P, N, d]
            m_row = m[0, r * Rs:(r + 1) * Rs].detach().to(torch.float32).contiguous().clone()      # [S/P, N, d]
            pair_to_cols = msa_to_cols = lambda t: rows_to_cols(t, group)  # noqa: E731
            pair_to_rows = msa_to_rows = lambda t: cols_to_rows(t, group)  # noqa: E731
        mask_full = None if mask is None else mask[0].bool()
        mm_full = None if msa_mask is None else msa_mask[0].bool().contiguous()
        mask_rows = None if mask_full is None else mask_full[r * Rn:(r + 1) * Rn].contiguous()
        mask_cols = None if mask_full is None else mask_full[:, r * Rn:(r + 1) * Rn].contiguous()
        mm_rows = None if mm_full is None else mm_full[r * Rs:(r + 1) * Rs].contiguous()
        mm_cols = None if mm_full is None else mm_full[:, r * Rn:(r + 1) * Rn].contiguous()

        def gathered_bias(ax, xr):
            b = ops.pair_bias(ax, xr)                                 # [H, Rn, npad]
            g = all_gather_cat0(b.transpose(0, 1).contiguous(), group)   # [N, H, npad] rows in global order
            return g.transpose(0, 1).contiguous()                    # [H, N, npad]

        overlap = OVERLAP_MSA_RETURN and x_row.is_cuda and P > 1
        side = torch.cuda.Stream() if overlap else None
        pending = None
        for block in evo.layers:
            pair, ff, msa_attn, msa_ff = block.layer
            d = x_row.shape[-1]
            # --- MSA track (alphafold2.py:438-439) ---
            bias_m = gathered_bias(msa_attn.row_attn, x_row)
            if pending is not None:
                m_row, pending = pending.get(), None
            ops.axial_attention_(msa_attn.row_attn, m_row, bias_m, mm_rows, True)
            m_col = msa_to_cols(m_row)                                                  # [S, N/P, d]
            ops.axial_attention_(msa_attn.col_attn, m_col, None, mm_cols, False)
            ops.feed_forward_(msa_ff, m_col)
            # --- outer mean into the pair rows (alphafold2.py:379) ---
            LR = ops.outer_project(pair.outer_mean, m_col, mm_cols)                      # [2d, S, pitch(N/P)]
            Rg = all_gather_cat0(LR[d:], group)                                          # [P*d, S, pitch]
            ops.outer_contract_(pair.outer_mean, x_row, LR[:d], Rg, mm_full, r * Rn, P)
            if overlap:
                pending = _Deferred(m_col, group, side, ex)                             # joins at the next block's row attention
            else:
                m_row = msa_to_rows(m_col)
            # --- triangle multiply outgoing on pair rows (alphafold2.py:381) ---
            tm = pair.triangle_multiply_outgoing
            L, R, G = ops.tri_project(tm, x_row, mask_rows)
            ops.tri_contract_(tm, x_row, L, all_gather_cat0(R, group), G, False, P)
            # --- triangle multiply ingoing on pair columns (alphafold2.py:382) ---
            x_col = pair_to_cols(x_row)                                                  # [N, N/P, d]
            tm = pair.triangle_multiply_ingoing
            L, R, G = ops.tri_project(tm, x_col, mask_cols)
            ops.tri_contract_(tm, x_col, L, all_gather_cat0(R, group), G, True, P)
            # --- triangle attention outgoing = row attention on pair rows (alphafold2.py:383) ---
            x_row = pair_to_rows(x_col)
            ta = pair.triangle_attention_outgoing
            ops.axial_attention_(ta, x_row, gathered_bias(ta, x_row), mask_rows, True)
            # --- triangle attention ingoing = column attention on pair columns (alphafold2.py:384) ---
            ta = pair.triangle_attention_ingoing
            bias = gathered_bias(ta, x_row)
            x_col = pair_to_cols(x_row)
            ops.axial_attention_(ta, x_col, bias, mask_cols, False)
            # --- pair transition (pointwise), back to rows (alphafold2.py:444) ---
            ops.feed_forward_(ff, x_col)
            x_row = pair_to_rows(x_col)

        if pending is not None:
            m_row, pending = pending.get(), None
        if not gather_output:
            return (x_row.clone(), m_row.clone()) if ex is not None else (x_row, m_row)   # arena buffers are reused by the next call
        xo = all_gather_cat0(x_row, group)[None]
        mo = all_gather_cat0(m_row, group)[None]
    return xo.to(x.dtype), mo.to(m.dtype)


COLLECTIVES_PER_BLOCK = {"all_gather_small_bias": 3, "all_gather_operand": 3, "all_to_all_msa": 2, "all_to_all_pair": 4}


OVERLAP_MSA_RETURN = True     # the MSA tensor's all-to-all back to row shards runs beside the pair track (side stream)
GRAPH_ENABLED = True     # module switch: set False to force the eager schedule (bench.py does, around its per-launch profiling pass)

_LIVE_GRAPHS = weakref.WeakSet()
_TEARDOWN_HOOKED = False


def graph_default() -> bool:
    """CUDA-graph replay of the sharded forward is the default (AF2_SHARD_GRAPH=0 or shard_evoformer(use_graph=False)
    selects the eager schedule).  With the sequence split over P ranks the eager schedule is host bound; the replay is
    bit-identical to it (tests/parallel_check_multi_gpu.py)."""
    import os
    return os.environ.get("AF2_SHARD_GRAPH", "1") not in ("", "0")


def release_all_graphs(peer_arenas: bool = True) -> None:
    """Drop every captured graph of this process.  A process that still owns a CUDA graph with NCCL nodes hangs when the
    communicator is torn down (torch 2.11 / NCCL 2.28.9), so this runs automatically before
    torch.distributed.destroy_process_group() and at interpreter exit (see _hook_teardown)."""
    for g in list(_LIVE_GRAPHS):
        g.release()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    if peer_arenas:
        release_peer_arenas()


def _hook_teardown() -> None:
    global _TEARDOWN_HOOKED
    if _TEARDOWN_HOOKED:
        return
    _TEARDOWN_HOOKED = True
    import atexit
    import functools
    atexit.register(release_all_graphs, False)      # at exit the driver reclaims the peer arenas; no collective there
    orig = dist.destroy_process_group

    @functools.wraps(orig)
    def destroy_process_group(*args, **kwargs):
        release_all_graphs()
        return orig(*args, **kwargs)

    dist.destroy_process_group = destroy_process_group
    try:
        import torch.distributed.distributed_c10d as c10d
        if getattr(c10d, "destroy_process_group", None) is orig:
            c10d.destroy_process_group = destroy_process_group
    except Exception:  # noqa: BLE001
        pass


def release_graphs(model) -> None:
    """Drop the captured graphs of a sharded model (kept for callers of round 1; teardown now does it on its own)."""
    evo = model.net if hasattr(model, "net") else model
    g = getattr(evo, "_af2_graph", None)
    if g is not None:
        g.release()
        torch.cuda.synchronize()


class _GraphedTrunk:
    """CUDA-graph replay of the sharded forward.

    With the sequence split over P ranks the device work per block shrinks by P while the host still walks ~60 C calls
    and ~12 NCCL enqueues per block, so from P = 2 on the eager schedule is bound by the host.  The whole forward
    (kernels, layout copies and NCCL collectives) is therefore captured once per signature and replayed; every rank
    captures the same sequence of collectives.

    What a captured graph bakes in, and how each is kept valid:
      * input tensors: read from the tensors seen at capture time (kept alive here); other tensors are copied into them;
      * packed weights: the Packed objects of every module are held here, and the signature contains the parameters'
        (data_ptr, _version) sum + the pack epoch, so load_state_dict / optimizer steps / invalidate_packed() recapture;
      * scratch: the capture runs inside a private workspace owned by this object (ops.private_workspace), so later eager
        ops that grow the shared workspace cannot free memory the graph points into.
    Outputs are returned as fresh tensors.  If capture is not possible the eager schedule is used and the reason is
    printed once."""

    def __init__(self, evo, group):
        self.evo, self.group = evo, group
        self.key = None
        self.graph = None
        self.inputs = None
        self.outputs = None
        self.failed = None
        self.launches_per_replay = 0
        self.ws = {}
        self.packed = None
        self._params = None
        _LIVE_GRAPHS.add(self)

    def release(self):
        self.graph, self.outputs, self.inputs, self.key, self.packed = None, None, None, None, None
        self.ws = {}
        import gc
        gc.collect()

    def _eager(self, x, m, mask, msa_mask):
        return sharded_evoformer_forward(self.evo, x, m, mask, msa_mask, self.group)

    def _weights_key(self):
        if self._params is None:
            self._params = list(self.evo.parameters())
        return (sum(p._version for p in self._params), sum(p.data_ptr() for p in self._params) & 0xffffffffffff,
                _ops.pack_epoch(), _ops.precision_of(self.evo))

    def __call__(self, x, m, mask=None, msa_mask=None):
        if not GRAPH_ENABLED or self.failed is not None or not x.is_cuda:
            return self._eager(x, m, mask, msa_mask)
        key = (tuple(x.shape), tuple(m.shape), x.dtype, m.dtype, None if mask is None else tuple(mask.shape),
               None if msa_mask is None else tuple(msa_mask.shape), x.device, self._weights_key())
        if key != self.key:
            try:
                self.release()
                self._capture(key, x, m, mask, msa_mask)
            except Exception as e:  # noqa: BLE001 - any capture failure falls back to the eager schedule
                self.failed = repr(e)
                self.release()
                import sys
                print(f"[alphafold2_b200.parallel] CUDA-graph capture failed, running eagerly: {self.failed}", file=sys.stderr)
                torch.cuda.synchronize()
                return self._eager(x, m, mask, msa_mask)
        for held, new in zip(self.inputs, (x, m, mask, msa_mask)):
            if held is not None and held.data_ptr() != new.data_ptr():
                held.copy_(new)
        self.graph.replay()
        return self.outputs[0].clone(), self.outputs[1].clone()

    def _capture(self, key, x, m, mask, msa_mask):
        from .alphafold2 import _Packable
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        self.ws = {}
        with torch.cuda.stream(side), _ops.private_workspace(self.ws, False):
            for _ in range(2):                      # packs weights, sizes the private workspace, initialises NCCL
                self._eager(x, m, mask, msa_mask)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        self.packed = [mod.packed() for mod in self.evo.modules() if isinstance(mod, _Packable)]
        n0 = _lib.load().af2_launch_count()
        g = torch.cuda.CUDAGraph()
        with _ops.private_workspace(self.ws, True), torch.cuda.graph(g):
            out = self._eager(x, m, mask, msa_mask)
        self.launches_per_replay = int(_lib.load().af2_launch_count() - n0)   # kernels of this library inside one replay
        self.graph, self.inputs, self.outputs, self.key = g, (x, m, mask, msa_mask), out, key


def shard_evoformer(model, group=None, use_graph: Optional[bool] = None):
    """Make `model.net(x, m, mask=, msa_mask=)` (an Alphafold2 or an Evoformer) run the sharded schedule.  Every rank
    must call forward with identical (replicated) inputs and gets the full outputs back.  use_graph: replay the schedule
    as one CUDA graph per input signature (see _GraphedTrunk and graph_default; default on, AF2_SHARD_GRAPH=0 disables)."""
    evo = model.net if hasattr(model, "net") else model
    if getattr(evo, "_af2_sharded", False):
        return model
    if use_graph is None:
        use_graph = graph_default()
    graphed = _GraphedTrunk(evo, group) if use_graph else None
    if graphed is not None:
        _hook_teardown()

    def fwd(x, m, mask=None, msa_mask=None, _evo=evo):
        if graphed is not None:
            return graphed(x, m, mask, msa_mask)
        return sharded_evoformer_forward(_evo, x, m, mask, msa_mask, group)

    evo.forward = fwd
    evo._af2_sharded = True
    evo._af2_graph = graphed
    return model
