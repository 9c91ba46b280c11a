"""Axis-sharded Evoformer trunk over the GPUs of one node (one process per GPU, torch.distributed / NCCL).

The reference has no multi-device path (SURVEY.md §2.2); this is the GPU-native addition named by the north
star: one sequence's forward is split over the MSA-row and pair-row axes (FastFold-DAP style).  At block entry
rank r owns pair rows x[r*N/P:(r+1)*N/P, :, :] and MSA rows m[r*S/P:(r+1)*S/P, :, :]; weights are replicated.  When P
does not divide N or S the shards are balanced instead (shard_offsets: the first N % P ranks hold one row more; MSA
shards may be empty), the all-to-alls take split sizes, gathered pieces are padded to the largest shard, and the
contractions read the gathered pieces merged into one compact operand.
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


def shard_offsets(n: int, P: int) -> list:
    """Balanced shards of n rows over P ranks: rank r owns rows [off[r], off[r+1]) with off[r] = r*(n//P) + min(r, n%P),
    so the first n % P ranks hold one row more.  A shard is empty when n < P."""
    q, rem = divmod(n, P)
    return [r * q + min(r, rem) for r in range(P + 1)]


def shard_counts(n: int, P: int) -> list:
    off = shard_offsets(n, P)
    return [b - a for a, b in zip(off, off[1:])]


def _pad_dim(t: torch.Tensor, dim: int, size: int) -> torch.Tensor:
    """t zero-padded along `dim` to `size` (the largest shard's extent, so that every rank contributes one shape)."""
    if t.shape[dim] == size:
        return t.contiguous()
    shape = list(t.shape)
    shape[dim] = size
    out = t.new_zeros(shape)
    out.narrow(dim, 0, t.shape[dim]).copy_(t)
    return out


# ------------------------------------------------------------------------------------------------------------
# collectives (concatenate along dim 0 so that both NCCL and gloo accept them).  counts / rows / cols: every rank's shard
# size along the split axes when the shards are uneven (shard_counts); None when every rank holds the same size.
# ------------------------------------------------------------------------------------------------------------
def all_gather_cat0(t: torch.Tensor, group, counts=None) -> torch.Tensor:
    """Every rank's t concatenated along dim 0 in rank order.  With counts, rank p holds counts[p] rows: each piece is padded
    to the largest and the receiver drops the padding."""
    if counts is not None:
        mx = max(counts)
        g = all_gather_cat0(_pad_dim(t, 0, mx), group)
        return torch.cat([g[p * mx:p * mx + c] for p, c in enumerate(counts)])
    P = dist.get_world_size(group)
    out = torch.empty((P * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t.contiguous(), group=group)
    return out


def _rows_to_cols_splits(t_row: torch.Tensor, rows, cols, r: int):
    """all_to_all_single operands of rows_to_cols over uneven shards: (send, recv, input splits, output splits)."""
    R, _, d = t_row.shape
    c0 = [0]
    for c in cols:
        c0.append(c0[-1] + c)
    send = torch.cat([t_row[:, c0[p]:c0[p + 1]].reshape(-1) for p in range(len(cols))])     # chunk p: my rows x columns of rank p
    recv = t_row.new_empty(sum(rows) * cols[r] * d)                                           # chunk p: rows of rank p x my columns
    return send, recv, [R * c * d for c in cols], [rp * cols[r] * d for rp in rows]


def rows_to_cols(t_row: torch.Tensor, group, rows=None, cols=None) -> torch.Tensor:
    """[R, C, d] (my R rows, all C columns) -> [P*R, C/P, d] (all rows, my columns).
    With rows / cols (every rank's row and column counts): [R_r, C, d] -> [sum(rows), cols[r], d]."""
    P = dist.get_world_size(group)
    R, Cc, d = t_row.shape
    if rows is not None:
        r = dist.get_rank(group)
        send, recv, isz, osz = _rows_to_cols_splits(t_row, rows, cols, r)
        dist.all_to_all_single(recv, send, output_split_sizes=osz, input_split_sizes=isz, group=group)
        return recv.view(sum(rows), cols[r], d)
    send = t_row.view(R, P, Cc // P, d).permute(1, 0, 2, 3).contiguous()      # chunk p: my rows x columns of rank p
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)                           # chunk p: rows of rank p x my columns
    return recv.view(P * R, Cc // P, d)


def _cols_to_rows_splits(t_col: torch.Tensor, rows, cols, r: int):
    """all_to_all_single operands of cols_to_rows over uneven shards: (send, recv, input splits, output splits)."""
    _, Cl, d = t_col.shape
    send = t_col.contiguous().view(-1)                                        # chunk p: rows of rank p x my columns
    recv = t_col.new_empty(rows[r] * sum(cols) * d)                           # chunk p: my rows x columns of rank p
    return send, recv, [rp * Cl * d for rp in rows], [rows[r] * c * d for c in cols]


def _place_row_chunks(out: torch.Tensor, recv: torch.Tensor, cols):
    """out [R, sum(cols), d] <- the received chunks (chunk p = my rows x the cols[p] columns of rank p)."""
    R, _, d = out.shape
    o = c0 = 0
    for c in cols:
        out[:, c0:c0 + c].copy_(recv[o:o + R * c * d].view(R, c, d))
        o, c0 = o + R * c * d, c0 + c


def cols_to_rows(t_col: torch.Tensor, group, rows=None, cols=None) -> torch.Tensor:
    """[P*R, Cl, d] (all rows, my Cl columns) -> [R, P*Cl, d] (my rows, all columns).
    With rows / cols (every rank's row and column counts): [sum(rows), cols[r], d] -> [rows[r], sum(cols), d]."""
    P = dist.get_world_size(group)
    RR, Cl, d = t_col.shape
    if rows is not None:
        r = dist.get_rank(group)
        send, recv, isz, osz = _cols_to_rows_splits(t_col, rows, cols, r)
        dist.all_to_all_single(recv, send, output_split_sizes=osz, input_split_sizes=isz, group=group)
        out = t_col.new_empty(rows[r], sum(cols), d)
        _place_row_chunks(out, recv, cols)
        return out
    R = RR // P
    send = t_col.contiguous().view(P, R, Cl, d)                               # chunk p: rows of rank p x my columns
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)                           # chunk p: my rows x columns of rank p
    return recv.permute(1, 0, 2, 3).reshape(R, P * Cl, d)


class _Deferred:
    """cols_to_rows on a side stream: the MSA tensor goes back to row shards while the pair track of the same block runs
    (nothing reads it before the next block's row attention).  With NCCL the collective itself runs on the process
    group's stream either way and the side stream removes the main stream's wait for it; with the peer-memory exchange
    (ex) the exchange kernel itself runs on the side stream, on barrier channel 1.  `get()` joins.
    rows / cols: as for cols_to_rows (uneven shards)."""

    def __init__(self, t_col: torch.Tensor, group, side, ex=None, rows=None, cols=None):
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
        self.keep = t_col                                                     # source stays alive until the side stream is done
        if rows is not None:
            r = dist.get_rank(group)
            send, recv, isz, osz = _cols_to_rows_splits(t_col, rows, cols, r)   # allocated on the main stream: its pool, its ordering
            self.out = torch.empty(rows[r], sum(cols), d, dtype=t_col.dtype, device=t_col.device)
            self.bufs = (send, recv)
            ready = cur.record_event()
            with torch.cuda.stream(side):
                side.wait_event(ready)
                dist.all_to_all_single(recv, send, output_split_sizes=osz, input_split_sizes=isz, group=group)
                _place_row_chunks(self.out, recv, cols)
                self.done = side.record_event()
            return
        R = RR // P
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

    @staticmethod
    def layout(N: int, S: int, d: int, P: int, rank: int = 0) -> dict:
        """Where the buffers of one rank's arena lie: off[(track, layout)] is a buffer's byte offset, shapes[(track, layout)]
        its fp32 shape on rank `rank`, total the arena's size in bytes, offsets[track] the shard_offsets of the track's rows
        (the columns of both tracks are the pair rows' shards).  The control block comes first; every buffer starts on 256 B
        and is sized for the largest shard (ceil(N/P), ceil(S/P)), so it starts at the same offset in every rank's arena."""
        ctrl = int(_lib.load().af2_peer_ctrl_bytes())
        al = lambda n: (n + 255) // 256 * 256  # noqa: E731
        Rn, Rs = -(-N // P), -(-S // P)
        pair_row, pair_col, msa_row, msa_col = al(Rn * N * d * 4), al(N * Rn * d * 4), al(Rs * N * d * 4), al(S * Rn * d * 4)
        on, os_ = shard_offsets(N, P), shard_offsets(S, P)
        nr, ns = on[rank + 1] - on[rank], os_[rank + 1] - os_[rank]
        PAIR, MSA = PeerExchange.PAIR, PeerExchange.MSA
        return dict(off={(PAIR, "row"): ctrl, (PAIR, "col"): ctrl + pair_row,
                         (MSA, "row"): ctrl + pair_row + pair_col, (MSA, "col"): ctrl + pair_row + pair_col + msa_row},
                    shapes={(PAIR, "row"): (nr, N, d), (PAIR, "col"): (N, nr, d),
                            (MSA, "row"): (ns, N, d), (MSA, "col"): (S, nr, d)},
                    total=ctrl + pair_row + pair_col + msa_row + msa_col, offsets={PAIR: on, MSA: os_})

    @classmethod
    def attach(cls, P: int, rank: int, base: int, table: torch.Tensor, device: torch.device, layout: dict, group=None):
        """Rank `rank` of an exchange over arenas that already exist: base is this rank's arena (laid out by `layout` for
        this rank), table the device int64 [P] of every rank's arena base as this process addresses it (its own included)."""
        self = cls()
        self.group, self.P, self.rank, self.device = group, P, rank, device
        self.base, self.table = base, table
        self.off, self.shapes, self.offsets = layout["off"], layout["shapes"], layout["offsets"]
        self.arena = torch.as_tensor(_RawCuda(base, layout["total"]), device=device)
        self.exchanges = 0
        return self

    @classmethod
    def create(cls, group, device: torch.device, N: int, S: int, d: int):
        P, r = dist.get_world_size(group), dist.get_rank(group)
        lib = _lib.load()
        self = cls()                   # holds the local arena and the peer mappings until every rank has them
        self.group, self.P, self.rank, self.device = group, P, r, device
        lay = cls.layout(N, S, d, P, r)
        total = lay["total"]
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
        ex = cls.attach(P, r, self.base, torch.tensor(bases, dtype=torch.int64, device=device), device, lay, group)
        ex.opened = self.opened                                                        # unmapped by close()
        return ex

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

    @staticmethod
    def plan_rows_to_cols_ragged(row_off, col_off, d: int, rank: int, itemsize: int = 4):
        """af2_peer_exchange_chunks arguments (bytes) for uneven shards (row_off / col_off: shard_offsets of the row and column
        axes): [R_rank, C, d] row shards -> [R_total, C_p, d] column shards.  chunks[p] = my rows x the columns of rank p; it
        lands in rank p's column buffer at row row_off[rank], whose rows are C_p columns wide.  For even shards the chunks are
        plan_rows_to_cols with src_off = p * src_peer_stride.  Pure arithmetic, like plan_rows_to_cols."""
        C, R = col_off[-1], row_off[rank + 1] - row_off[rank]
        chunks = []
        for p in range(len(col_off) - 1):
            w = (col_off[p + 1] - col_off[p]) * d * itemsize
            chunks.append(dict(src_off=col_off[p] * d * itemsize, dst_off=row_off[rank] * w, dst_row_stride=w, rows=R, row_bytes=w))
        return dict(src_row_stride=C * d * itemsize, chunks=chunks)

    @staticmethod
    def plan_cols_to_rows_ragged(row_off, col_off, d: int, rank: int, itemsize: int = 4):
        """The way back for uneven shards: [R_total, C_rank, d] -> [R_p, C, d].  chunks[p] = the rows of rank p x my columns
        (contiguous at the source; none when rank p has no rows); it lands in rank p's row buffer at columns col_off[rank]..
        of every row."""
        C = col_off[-1]
        w = (col_off[rank + 1] - col_off[rank]) * d * itemsize
        chunks = [dict(src_off=row_off[p] * w, dst_off=col_off[rank] * d * itemsize, dst_row_stride=C * d * itemsize,
                       rows=row_off[p + 1] - row_off[p], row_bytes=w) for p in range(len(col_off) - 1)]
        return dict(src_row_stride=w, chunks=chunks)

    def _run(self, src: torch.Tensor, plan: dict, dst_buffer_off: int, channel: int):
        self._exchange(src, plan["src_peer_stride"], plan["src_row_stride"], dst_buffer_off + plan["dst_off"], plan["dst_row_stride"],
                       plan["rows"], plan["row_bytes"], channel)

    def _run_chunks(self, src_ptr: int, plan: dict, dst_buffer_off: int, channel: int):
        table = (_lib.PeerChunk * self.P)(*[_lib.PeerChunk(c["src_off"], dst_buffer_off + c["dst_off"], c["dst_row_stride"],
                                                           c["row_bytes"], c["rows"], 0) for c in plan["chunks"]])
        _lib.check(_lib.load().af2_peer_exchange_chunks(src_ptr, plan["src_row_stride"], table, self.table.data_ptr(), channel,
                                                         self.rank, self.P, _ops._stream_ptr()))
        self.exchanges += 1

    def _even(self, track: int) -> bool:
        """Every rank holds the same rows of the track and the same columns: the single-shape exchange applies."""
        return all(o % self.P == 0 for o in (self.offsets[track][-1], self.offsets[self.PAIR][-1]))

    def _check_src(self, t: torch.Tensor, track: int, layout: str):
        assert tuple(t.shape) == self.shapes[(track, layout)]
        assert t.numel() == 0 or t.data_ptr() == self.base + self.off[(track, layout)]

    def rows_to_cols(self, t_row: torch.Tensor, track: int, channel: int = 0) -> torch.Tensor:
        """[R, C, d] (my rows, all columns; the track's row buffer) -> the track's column buffer [P*R, C/P, d]
        ([R_total, C_rank, d] for uneven shards)."""
        R, Cc, d = t_row.shape
        self._check_src(t_row, track, "row")
        if self._even(track):
            self._run(t_row, self.plan_rows_to_cols(R, Cc, d, self.P, self.rank), self.off[(track, "col")], channel)
        else:
            plan = self.plan_rows_to_cols_ragged(self.offsets[track], self.offsets[self.PAIR], d, self.rank)
            self._run_chunks(self.base + self.off[(track, "row")], plan, self.off[(track, "col")], channel)
        return self.buffer(track, "col")

    def cols_to_rows(self, t_col: torch.Tensor, track: int, channel: int = 0) -> torch.Tensor:
        """[P*R, Cl, d] (all rows, my columns; the track's column buffer) -> the track's row buffer [R, P*Cl, d]
        ([R_rank, C, d] for uneven shards)."""
        RR, Cl, d = t_col.shape
        self._check_src(t_col, track, "col")
        if self._even(track):
            self._run(t_col, self.plan_cols_to_rows(RR, Cl, d, self.P, self.rank), self.off[(track, "row")], channel)
        else:
            plan = self.plan_cols_to_rows_ragged(self.offsets[track], self.offsets[self.PAIR], d, self.rank)
            self._run_chunks(self.base + self.off[(track, "col")], plan, self.off[(track, "row")], channel)
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

    def tied_column_attention_(self, ax, x: torch.Tensor, bias: Optional[torch.Tensor], mask: Optional[torch.Tensor], reduce,
                               ncols_total: int):
        """Tied-query column attention (global_query_attn) of a column shard x [h, w, d] fp32 in place, whose queries average
        over ncols_total columns held by several ranks.  reduce: this shard's fp32 query sums [h, I] -> every shard's, in
        column-shard order [nparts * h, I] (the schedule: an all-gather).  bias as for axial_attention_."""
        pk = ax.packed()
        h, w, d = x.shape
        H, dh = ax.attn.heads, ax.attn.dim_head
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_axial_attention_workspace(1, h, w, d, H, dh, 0), x.device)
        m8 = None if mask is None else mask.contiguous()
        args = (C.byref(pk.struct), x.data_ptr(), None if bias is None else bias.data_ptr(), None if m8 is None else m8.data_ptr(),
                h, w, d, H, dh)
        qsum = torch.empty(h, H * dh, dtype=torch.float32, device=x.device)
        _lib.check(lib.af2_axial_attention_tied_begin(*args, qsum.data_ptr(), ws.data_ptr(), ws.numel(), _ops._stream_ptr()))
        parts = reduce(qsum).contiguous()              # the workspace keeps LN(x), q|k|v and the gate until the end call
        _lib.check(lib.af2_axial_attention_tied_end(*args, parts.data_ptr(), parts.shape[0] // h, ncols_total, ws.data_ptr(),
                                                    ws.numel(), _ops._stream_ptr()))

    def feed_forward_(self, ff, x: torch.Tensor):
        _ops.feed_forward_(ff.packed(), x)

    def outer_operand(self, S: int, N: int, d: int, like: torch.Tensor) -> torch.Tensor:
        """Whole outer-mean operand for the banded schedule: bf16 [2d, S, align8(N)]; outer_project(out=...) fills it in chunks
        of MSA rows (each chunk zeroes its own pad columns)."""
        return torch.empty(2 * d, S, _align8(N), dtype=torch.bfloat16, device=like.device)

    def outer_project(self, om, m_cols: torch.Tensor, mask_cols: Optional[torch.Tensor], out=None) -> torch.Tensor:
        """m [S, nl, d] -> bf16 [2d, S, align8(nl)] channel-major left | right.
        out: write into this instead, e.g. the MSA-row window [:, s0:s1] of outer_operand's tensor (its channel stride is kept)."""
        pk = om.packed()
        S, nl, d = m_cols.shape
        if out is None:
            out = torch.empty(2 * d, S, _align8(nl), dtype=torch.bfloat16, device=m_cols.device)
        elif tuple(out.shape) != (2 * d, S, _align8(nl)) or out.stride(1) != _align8(nl) or out.stride(2) != 1:
            raise ValueError("outer_project: out must be a [2d, rows, align8(cols)] window with one channel stride")
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_outer_project_workspace(S * nl, d), m_cols.device)
        mk = None if mask_cols is None else mask_cols.contiguous()
        _lib.check(lib.af2_outer_project(C.byref(pk.struct), m_cols.data_ptr(), None if mk is None else mk.data_ptr(), S * nl,
                                         nl, d, out.data_ptr(), out.stride(0), ws.data_ptr(), ws.numel(), _ops._stream_ptr()))
        return out

    @staticmethod
    def _merge_mn_pieces(Rg: torch.Tensor, pieces, d: int, n_total: int):
        """Gathered MN-major operand [pieces*d, K, align8(n_total/pieces)] with fewer than 64 columns per piece: the kernel's
        64-column TMA boxes cannot span pieces, so instead of `pieces` tiny launches the pieces are re-packed once into ONE
        operand [d, K, align8(n_total)] (a pass over the gathered tensor, ~10 us at C2) and contracted in a single launch.
        Each piece's alignment padding is dropped on the way: column p*(n_total/pieces)+c of the result is column c of piece p.
        Pieces of >= 64 columns are addressed in place.
        pieces may instead be the column count of every piece (uneven shards, [P*d, K, w] with piece p's columns in its
        first pieces[p]): those are always merged, column sum(pieces[:p])+c of the result being column c of piece p."""
        K, w = Rg.shape[1], Rg.shape[2]
        if not isinstance(pieces, int):
            assert sum(pieces) == n_total
            out = torch.zeros(d, K, _align8(n_total), dtype=Rg.dtype, device=Rg.device)
            src, c0 = Rg.view(len(pieces), d, K, w), 0
            for p, wp in enumerate(pieces):
                out[:, :, c0:c0 + wp].copy_(src[p, :, :, :wp])
                c0 += wp
            return out, 1
        if pieces == 1 or w >= 64:
            return Rg, pieces
        wt = n_total // pieces
        out = torch.zeros(d, K, _align8(n_total), dtype=Rg.dtype, device=Rg.device)
        out[:, :, :n_total].view(d, K, pieces, wt).copy_(Rg.view(pieces, d, K, w)[..., :wt].permute(1, 2, 0, 3))
        return out, 1

    @staticmethod
    def _merge_k_pieces(Rg: torch.Tensor, rows, d: int):
        """Gathered K-major operand of uneven shards [P*d, Rmax, K'] (piece p's rows in its first rows[p]) -> the compact
        [d, sum(rows), K'] of the unsharded call, rows in rank order."""
        src = Rg.view(len(rows), d, Rg.shape[1], Rg.shape[2])
        return torch.cat([src[p, :, :rp] for p, rp in enumerate(rows)], 1), 1

    def outer_contract_(self, om, x_rows: torch.Tensor, L: torch.Tensor, Rg: torch.Tensor, msa_mask_full, row0: int, pieces):
        """x_rows [rows, N, d] += OuterMean; L [d, S, align8(rows)], Rg [pieces*d, S, align8(N/pieces)].
        pieces: the number of equal pieces, or every piece's column count (uneven shards; see _merge_mn_pieces)."""
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

    def tri_operands(self, N: int, d: int, like: torch.Tensor):
        """Whole-tensor triangle-multiply operands for the banded schedule: L, R bf16 [d, N, align8(N)] (pad columns zero),
        gate bf16 [N*N, d]; tri_project(out=...) fills them band by band."""
        L = torch.zeros(d, N, _align8(N), dtype=torch.bfloat16, device=like.device)
        return L, torch.zeros_like(L), torch.empty(N * N, d, dtype=torch.bfloat16, device=like.device)

    def tri_project(self, tm, x_loc: torch.Tensor, mask_loc: Optional[torch.Tensor], out=None):
        """x [rows, cols, d] -> (L, R) bf16 [d, rows, align8(cols)] channel-major, gate bf16 [rows*cols, d].
        out = (L, R, gate): write into these instead, e.g. the row window [:, i0:i1] of tri_operands' L and R (their channel
        stride is kept) and rows [i0*cols, i1*cols) of its gate."""
        pk = tm.packed()
        rows, cols, d = x_loc.shape
        if out is None:
            L = torch.empty(d, rows, _align8(cols), dtype=torch.bfloat16, device=x_loc.device)
            R = torch.empty_like(L)
            gate = torch.empty(rows * cols, d, dtype=torch.bfloat16, device=x_loc.device)
        else:
            L, R, gate = out
            if L.stride() != R.stride() or tuple(L.shape) != (d, rows, _align8(cols)) or L.stride(1) != _align8(cols):
                raise ValueError("tri_project: out L / R must be [d, rows, align8(cols)] windows with one channel stride")
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_triangle_project_workspace(rows * cols, d), x_loc.device)
        mk = None if mask_loc is None else mask_loc.contiguous()
        _lib.check(lib.af2_triangle_project(C.byref(pk.struct), x_loc.data_ptr(), None if mk is None else mk.data_ptr(),
                                            rows * cols, cols, d, L.data_ptr(), R.data_ptr(), L.stride(0),
                                            gate.data_ptr(), ws.data_ptr(), ws.numel(), _ops._stream_ptr()))
        return L, R, gate

    def tri_contract_(self, tm, x_loc: torch.Tensor, L: torch.Tensor, Rg: torch.Tensor, gate: torch.Tensor, ingoing: bool, pieces):
        """L may be a row window of a larger channel-major operand (its channel stride is passed on).  pieces: the number of
        equal gathered pieces, or every piece's size along the gathered axis (uneven shards: merged into one operand)."""
        pk = tm.packed()
        rows, cols, d = x_loc.shape
        K = L.shape[1] if ingoing else cols
        if ingoing and not isinstance(pieces, int) and (cols % 4 == 0) != (rows % 4 == 0):
            return self._tri_contract_ingoing_padded_(tm, x_loc, L, Rg, gate, pieces)
        if ingoing:
            Rg, pieces = self._merge_mn_pieces(Rg, pieces, d, rows)
        elif not isinstance(pieces, int):
            Rg, pieces = self._merge_k_pieces(Rg, pieces, d)
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_triangle_contract_workspace(rows, cols, d), x_loc.device)
        per_piece = Rg.numel() // pieces
        _lib.check(lib.af2_triangle_contract(C.byref(pk.struct), x_loc.data_ptr(), L.data_ptr(), L.stride(0),
                                             Rg.data_ptr(), Rg.stride(0), per_piece, pieces, gate.data_ptr(),
                                             rows, cols, K, d, int(ingoing), ws.data_ptr(), ws.numel(), _ops._stream_ptr()))

    def _tri_contract_ingoing_padded_(self, tm, x_col: torch.Tensor, L: torch.Tensor, Rg: torch.Tensor, gate: torch.Tensor, pieces):
        """Ingoing contraction of an uneven column shard x_col [N, cols, d] whose width would make the contraction's
        channel -> token LayerNorm run another kernel than the unsharded call (N columns) runs: that kernel is picked by
        whether the output rows are dense, i.e. cols % 4 == 0 (api.cu c2t_select), and two kernels round differently.
        The shard is contracted padded with zero columns to a width that is dense exactly when N is (align4(cols) if
        N % 4 == 0, else cols + 1); the padding columns' outputs are dropped.  Every kept element is computed as in the
        unsharded call (the GEMM and the LayerNorm are per output element / per token)."""
        N, cols, d = x_col.shape
        cp = (cols + 3) // 4 * 4 if N % 4 == 0 else cols + 1
        x_pad = torch.zeros(N, cp, d, dtype=x_col.dtype, device=x_col.device)
        x_pad[:, :cols].copy_(x_col)
        L_pad = torch.zeros(d, L.shape[1], _align8(cp), dtype=L.dtype, device=L.device)
        L_pad[:, :, :cols].copy_(L[:, :, :cols])
        g_pad = torch.zeros(N, cp, d, dtype=gate.dtype, device=gate.device)
        g_pad[:, :cols].copy_(gate.view(N, cols, d))
        self.tri_contract_(tm, x_pad, L_pad, Rg, g_pad.view(N * cp, d), True, pieces)
        x_col.copy_(x_pad[:, :cols])

    def tri_contract_window_(self, tm, x_rows: torch.Tensor, L: torch.Tensor, R_win: torch.Tensor, gate: torch.Tensor):
        """Ingoing contraction of pair rows [i0, i1): x_rows [rows, N, d] += to_out(LN_c(O) * gate) with
        O[i][j] = sum_k R[k][i0 + i] L[k][j]; L bf16 [d, N, align8(N)], R_win = R[:, :, i0:i1] (a column window, read in
        place through af2_triangle_contract_pitched), gate [rows*N, d]."""
        pk = tm.packed()
        rows, cols, d = x_rows.shape
        K = L.shape[1]
        lib = _lib.load()
        ws = _ops.workspace(lib.af2_triangle_contract_workspace(rows, cols, d), x_rows.device)
        _lib.check(lib.af2_triangle_contract_pitched(C.byref(pk.struct), x_rows.data_ptr(), L.data_ptr(), L.stride(0), L.stride(1),
                                                     R_win.data_ptr(), R_win.stride(0), R_win.stride(1), gate.data_ptr(), rows, cols,
                                                     K, d, 1, ws.data_ptr(), ws.numel(), _ops._stream_ptr()))


# ------------------------------------------------------------------------------------------------------------
# the schedule
# ------------------------------------------------------------------------------------------------------------
class _PairShards:
    """A pair tensor [N, N, d] sharded over the ranks of `group` for the pair track: rank r owns pair rows (and columns)
    [n0, n1) = shard_offsets(N, P)[r:r + 2].  Holds the masks' row and column shards, the exchanges between the two layouts
    (to_cols: [Rn, N, d] -> [N, Rn, d], to_rows: back) and the gathers of the pair track."""

    def __init__(self, group, N: int, mask_full: Optional[torch.Tensor], to_cols, to_rows):
        self.group, self.N, self.P = group, N, dist.get_world_size(group)
        on = shard_offsets(N, self.P)
        r = dist.get_rank(group)
        self.n0, self.n1 = on[r], on[r + 1]
        self.counts = shard_counts(N, self.P) if N % self.P else None     # None: equal shards, the plain collectives
        self.Rn_max = -(-N // self.P)
        self.mask_rows = None if mask_full is None else mask_full[self.n0:self.n1].contiguous()
        self.mask_cols = None if mask_full is None else mask_full[:, self.n0:self.n1].contiguous()
        self.to_cols, self.to_rows = to_cols, to_rows

    def bias(self, ops, ax, x_row):
        b = ops.pair_bias(ax, x_row)                                  # [H, Rn, npad]
        g = all_gather_cat0(b.transpose(0, 1).contiguous(), self.group, self.counts)   # [N, H, npad] rows in global order
        return g.transpose(0, 1).contiguous()                        # [H, N, npad]

    def operand(self, t, dim):
        """A contraction's gathered operand and its `pieces`: P equal pieces, or with uneven shards each rank's piece padded
        along `dim` (dim 1: rows, K-major; dim 2: columns, MN-major, aligned to 8 like the kernels' pitch) and the pair shard
        sizes, which tell the stage op what to keep of each piece."""
        if self.counts is None:
            return all_gather_cat0(t, self.group), self.P
        return all_gather_cat0(_pad_dim(t, dim, self.Rn_max if dim == 1 else _align8(self.Rn_max)), self.group), tuple(self.counts)

    def query_sums(self, qsum):
        """The tied queries' partial sums [N, I] of every rank, in rank (= column-shard) order: [P * N, I].  Every rank's
        partial has the same shape, so even uneven shards need no padding."""
        return all_gather_cat0(qsum, self.group)


def sharded_pair_track(ops, pair, x_row: torch.Tensor, sh: _PairShards, outer=None, ff=None) -> torch.Tensor:
    """The pair track of one block (alphafold2.py:379-385, 444) on this rank's pair rows x_row [Rn, N, d]; returns the new row
    shard (with the peer-memory exchange, the arena's row buffer).  pair: a PairwiseAttentionBlock.
    outer: (L, Rg, msa_mask_full, pieces), the outer mean's operands (the trunk): contracted into x_row first.  ff: the pair
    transition, run on the column shard before the way back (the trunk).  The template pair stack passes neither.
    A pair block with tied-query ingoing attention (global_query_attn, the extra-MSA stack) gathers the queries' partial sums
    over the column shards (one all-gather more)."""
    if outer is not None:
        L, Rg, mm_full, pieces = outer
        ops.outer_contract_(pair.outer_mean, x_row, L, Rg, mm_full, sh.n0, pieces)
    # --- triangle multiply outgoing on pair rows (alphafold2.py:381) ---
    tm = pair.triangle_multiply_outgoing
    L, R, G = ops.tri_project(tm, x_row, sh.mask_rows)
    Rg, pieces = sh.operand(R, 1)
    ops.tri_contract_(tm, x_row, L, Rg, G, False, pieces)
    # --- triangle multiply ingoing on pair columns (alphafold2.py:382) ---
    x_col = sh.to_cols(x_row)                                                    # [N, N/P, d]
    tm = pair.triangle_multiply_ingoing
    L, R, G = ops.tri_project(tm, x_col, sh.mask_cols)
    Rg, pieces = sh.operand(R, 2)
    ops.tri_contract_(tm, x_col, L, Rg, G, True, pieces)
    # --- triangle attention outgoing = row attention on pair rows (alphafold2.py:383) ---
    x_row = sh.to_rows(x_col)
    ta = pair.triangle_attention_outgoing
    ops.axial_attention_(ta, x_row, sh.bias(ops, ta, x_row), sh.mask_rows, True)
    # --- triangle attention ingoing = column attention on pair columns (alphafold2.py:384) ---
    ta = pair.triangle_attention_ingoing
    bias = sh.bias(ops, ta, x_row)
    x_col = sh.to_cols(x_row)
    if ta.global_query_attn:
        ops.tied_column_attention_(ta, x_col, bias, sh.mask_cols, sh.query_sums, sh.N)
    else:
        ops.axial_attention_(ta, x_col, bias, sh.mask_cols, False)
    # --- pair transition (pointwise), back to rows (alphafold2.py:444) ---
    if ff is not None:
        ops.feed_forward_(ff, x_col)
    return sh.to_rows(x_col)


def sharded_evoformer_forward(evo, x: torch.Tensor, m: torch.Tensor, mask: Optional[torch.Tensor] = None,
                              msa_mask: Optional[torch.Tensor] = None, group=None, stage_ops=None, gather_output: bool = True,
                              rows_in: bool = False):
    """Evoformer.forward (alphafold2.py:458-467) for ONE sequence sharded over the ranks of `group`.

    x [1, N, N, d], m [1, S, N, d], mask [1, N, N] bool, msa_mask [1, S, N] bool are the full (replicated) inputs;
    returns the full (x, m) on every rank when gather_output, else this rank's row shards.
    rows_in: x is this rank's pair rows [1, n1 - n0, N, d] instead (no rank holds the whole pair tensor), and the outputs are
    the row shards whatever gather_output says.

    Any N >= P and S >= 1: rank r owns pair rows (and columns) [on[r], on[r+1]) and MSA rows [os[r], os[r+1]) with
    on = shard_offsets(N, P), os = shard_offsets(S, P); the first N % P (S % P) ranks hold one row more, and MSA shards
    are empty when S < P.  Shapes that P divides take the equal-shard path unchanged.  Tied-query ingoing attention
    (global_query_attn: the extra-MSA stack) averages its queries over all N columns through one more all-gather per block.
    """
    if stage_ops is None and _ops.precision_of(evo) == "strict":
        raise NotImplementedError("the strict precision mode runs on one GPU (it is a parity mode, not a throughput mode)")
    ops = stage_ops if stage_ops is not None else CudaStageOps()
    P = dist.get_world_size(group)
    r = dist.get_rank(group)
    if x.shape[0] != 1:
        raise ValueError("the sharded trunk handles one sequence per call (batch 1)")
    N, S = x.shape[2 if rows_in else 1], m.shape[1]
    if N < P:
        raise ValueError(f"N_res={N} is smaller than the number of ranks {P}: every rank needs at least one pair row")
    on, os_ = shard_offsets(N, P), shard_offsets(S, P)
    n0, n1, s0, s1 = on[r], on[r + 1], os_[r], os_[r + 1]
    if rows_in and x.shape[1] != n1 - n0:
        raise ValueError(f"rank {r} owns pair rows [{n0}, {n1}) of {N}; x holds {x.shape[1]} rows")
    x_src = x[0] if rows_in else x[0, n0:n1]
    # shard sizes of every rank for the collectives, None where P divides the axis (equal shards: the plain collectives)
    pair_counts = shard_counts(N, P) if N % P else None
    msa_counts = shard_counts(S, P) if S % P else None
    msa_ragged = pair_counts is not None or msa_counts is not None          # the MSA columns are the pair shards
    msa_splits = (shard_counts(S, P), shard_counts(N, P)) if msa_ragged else (None, None)
    with torch.no_grad():
        ex = peer_exchange_for(group, x.device, N, S, x.shape[-1]) if stage_ops is None else None
        if ex is not None:                                            # the shards live in the peer-mapped arena
            x_row, m_row = ex.buffer(PeerExchange.PAIR, "row"), ex.buffer(PeerExchange.MSA, "row")
            x_row.copy_(x_src)
            m_row.copy_(m[0, s0:s1])
            pair_to_cols = lambda t: ex.rows_to_cols(t, PeerExchange.PAIR)  # noqa: E731
            pair_to_rows = lambda t: ex.cols_to_rows(t, PeerExchange.PAIR)  # noqa: E731
            msa_to_cols = lambda t: ex.rows_to_cols(t, PeerExchange.MSA)  # noqa: E731
            msa_to_rows = lambda t: ex.cols_to_rows(t, PeerExchange.MSA)  # noqa: E731
        else:
            x_row = x_src.detach().to(torch.float32).contiguous().clone()            # [N/P, N, d]
            m_row = m[0, s0:s1].detach().to(torch.float32).contiguous().clone()      # [S/P, N, d]
            pair_to_cols = lambda t: rows_to_cols(t, group, pair_counts, pair_counts)  # noqa: E731
            pair_to_rows = lambda t: cols_to_rows(t, group, pair_counts, pair_counts)  # noqa: E731
            msa_to_cols = lambda t: rows_to_cols(t, group, *msa_splits)  # noqa: E731
            msa_to_rows = lambda t: cols_to_rows(t, group, *msa_splits)  # noqa: E731
        mask_full = None if mask is None else mask[0].bool()
        mm_full = None if msa_mask is None else msa_mask[0].bool().contiguous()
        sh = _PairShards(group, N, mask_full, pair_to_cols, pair_to_rows)
        mm_rows = None if mm_full is None else mm_full[s0:s1].contiguous()
        mm_cols = None if mm_full is None else mm_full[:, n0:n1].contiguous()

        overlap = OVERLAP_MSA_RETURN and x_row.is_cuda and P > 1
        side = torch.cuda.Stream() if overlap else None
        pending = None
        for block in evo.layers:
            pair, ff, msa_attn, msa_ff = block.layer
            d = x_row.shape[-1]
            # --- MSA track (alphafold2.py:438-439) ---
            bias_m = sh.bias(ops, msa_attn.row_attn, x_row)
            if pending is not None:
                m_row, pending = pending.get(), None
            if m_row.shape[0]:                                                          # an empty MSA shard has nothing to attend
                ops.axial_attention_(msa_attn.row_attn, m_row, bias_m, mm_rows, True)
            m_col = msa_to_cols(m_row)                                                  # [S, N/P, d]
            ops.axial_attention_(msa_attn.col_attn, m_col, None, mm_cols, False)
            ops.feed_forward_(msa_ff, m_col)
            # --- outer mean operands (alphafold2.py:379), contracted into the pair rows by the pair track ---
            LR = ops.outer_project(pair.outer_mean, m_col, mm_cols)                      # [2d, S, pitch(N/P)]
            Rg, pieces = sh.operand(LR[d:], 2)                                           # [P*d, S, pitch]
            # the MSA tensor goes back to row shards beside the pair track; nothing in it reads m
            if overlap:
                pending = _Deferred(m_col, group, side, ex, *msa_splits)                # joins at the next block's row attention
            else:
                m_row = msa_to_rows(m_col)
            x_row = sharded_pair_track(ops, pair, x_row, sh, outer=(LR[:d], Rg, mm_full, pieces), ff=ff)

        if pending is not None:
            m_row, pending = pending.get(), None
        if rows_in or not gather_output:
            return (x_row.clone(), m_row.clone()) if ex is not None else (x_row, m_row)   # arena buffers are reused by the next call
        xo = all_gather_cat0(x_row, group, pair_counts)[None]
        mo = all_gather_cat0(m_row, group, msa_counts)[None]
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

    def _eager(self, x, m, mask, msa_mask, rows_in=False):
        return sharded_evoformer_forward(self.evo, x, m, mask, msa_mask, self.group, rows_in=rows_in)

    def _weights_key(self):
        if self._params is None:
            self._params = list(self.evo.parameters())
        return (sum(p._version for p in self._params), sum(p.data_ptr() for p in self._params) & 0xffffffffffff,
                _ops.pack_epoch(), _ops.precision_of(self.evo))

    def __call__(self, x, m, mask=None, msa_mask=None, rows_in=False):
        if not GRAPH_ENABLED or self.failed is not None or not x.is_cuda:
            return self._eager(x, m, mask, msa_mask, rows_in)
        key = (tuple(x.shape), tuple(m.shape), x.dtype, m.dtype, None if mask is None else tuple(mask.shape),
               None if msa_mask is None else tuple(msa_mask.shape), x.device, self._weights_key(), rows_in)
        if key != self.key:
            try:
                self.release()
                self._capture(key, x, m, mask, msa_mask, rows_in)
            except Exception as e:  # noqa: BLE001 - any capture failure falls back to the eager schedule
                self.failed = repr(e)
                self.release()
                import sys
                print(f"[alphafold2_b200.parallel] CUDA-graph capture failed, running eagerly: {self.failed}", file=sys.stderr)
                torch.cuda.synchronize()
                return self._eager(x, m, mask, msa_mask, rows_in)
        for held, new in zip(self.inputs, (x, m, mask, msa_mask)):
            if held is not None and held.data_ptr() != new.data_ptr():
                held.copy_(new)
        self.graph.replay()
        return self.outputs[0].clone(), self.outputs[1].clone()

    def _capture(self, key, x, m, mask, msa_mask, rows_in=False):
        from .alphafold2 import _Packable
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        self.ws = {}
        with torch.cuda.stream(side), _ops.private_workspace(self.ws, False):
            for _ in range(2):                      # packs weights, sizes the private workspace, initialises NCCL
                self._eager(x, m, mask, msa_mask, rows_in)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        self.packed = [mod.packed() for mod in self.evo.modules() if isinstance(mod, _Packable)]
        n0 = _lib.load().af2_launch_count()
        g = torch.cuda.CUDAGraph()
        with _ops.private_workspace(self.ws, True), torch.cuda.graph(g):
            out = self._eager(x, m, mask, msa_mask, rows_in)
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

    def fwd(x, m, mask=None, msa_mask=None, _evo=evo, rows_in=False):
        if graphed is not None:
            return graphed(x, m, mask, msa_mask, rows_in)
        return sharded_evoformer_forward(_evo, x, m, mask, msa_mask, group, rows_in=rows_in)

    evo.forward = fwd
    evo._af2_sharded = True
    evo._af2_graph = graphed
    return model


def _pair_arena(group, device: torch.device, N: int, d: int):
    """A peer-memory arena this process already holds for pair tensors [N, N, d] over `group` (any MSA depth), or None."""
    for (g, dev, n, _, dd), ex in _PEER_ARENAS.items():
        if ex is not None and (g, dev, n, dd) == (id(group), device.index, N, d):
            return ex
    return None


def sharded_embed_templates_(model, x: torch.Tensor, x_mask: Optional[torch.Tensor], templates_feats: torch.Tensor,
                             templates_mask: torch.Tensor, group=None, rows_in: bool = False) -> torch.Tensor:
    """Alphafold2.embed_templates_ (alphafold2.py:743-785) with the pair work sharded over the ranks of `group`, in place on
    the full fp32 x [1, n, n, d] that every rank holds.  Rank r owns pair rows [n0, n1) = shard_offsets(n, P)[r:r + 2].

    The templates run one at a time, so a rank's memory does not grow with T.  For template k: to_template_embed of this
    rank's rows of templates_feats[0, k] (GEMM rows are independent: bitwise the rows of the whole call), the crossed mask's
    row and column shards, templates_embed_layers passes of sharded_pair_track (no outer mean, no transition), then one step
    of the state-carrying pointwise attention over this rank's pairs (af2_template_pointwise_rows_*, q and gate from
    x[0, n0:n1]).  After the last template to_out adds into those rows and an all-gather of the rows gives every rank the full
    x.  The row <-> column exchanges use the peer-memory arena the sharded trunk already holds for (n, d), when there is
    one (from the second forward on), and NCCL all-to-alls otherwise: both move the same bytes.  Runs eagerly.
    rows_in: x is this rank's pair rows [1, n1 - n0, n, d] (shard_alphafold2(pair_rows=True)); they are updated in place and
    nothing is gathered."""
    attn = model.template_pointwise_attn
    if _ops.precision_of(attn) == "strict":
        raise NotImplementedError("the strict precision mode runs on one GPU (it is a parity mode, not a throughput mode)")
    if x.shape[0] != 1:
        raise ValueError("the sharded template branch handles one sequence per call (batch 1)")
    if x.dtype != torch.float32 or not x.is_contiguous():
        raise ValueError("the sharded template branch updates a contiguous fp32 x in place")
    P = dist.get_world_size(group)
    T, n, d = templates_feats.shape[1], x.shape[2 if rows_in else 1], x.shape[3]
    if n < P:
        raise ValueError(f"N_res={n} is smaller than the number of ranks {P}: every rank needs at least one pair row")
    ops = CudaStageOps()
    lib = _lib.load()
    pair = model.template_pairwise_embedder
    H, dh = attn.heads, attn.dim_head
    I = H * dh
    with torch.no_grad():
        on = shard_offsets(n, P)
        r = dist.get_rank(group)
        n0, n1 = on[r], on[r + 1]
        counts = shard_counts(n, P) if n % P else None
        ex = _pair_arena(group, x.device, n, d)
        if ex is not None:
            to_cols = lambda t: ex.rows_to_cols(t, PeerExchange.PAIR)  # noqa: E731
            to_rows = lambda t: ex.cols_to_rows(t, PeerExchange.PAIR)  # noqa: E731
        else:
            to_cols = lambda t: rows_to_cols(t, group, counts, counts)  # noqa: E731
            to_rows = lambda t: cols_to_rows(t, group, counts, counts)  # noqa: E731
        Pn = (n1 - n0) * n                                                  # this rank's pairs
        x_rows = x[0] if rows_in else x[0, n0:n1]                           # a contiguous window of x
        xm = None if x_mask is None else x_mask[0, n0:n1].bool().contiguous()
        tm = templates_mask[0].bool()
        embed = model.to_template_embed.packed()
        w = C.byref(attn.packed().struct)
        s = _ops._stream_ptr()
        run_max = torch.empty(Pn, H, dtype=torch.float32, device=x.device)
        run_sum = torch.empty_like(run_max)
        acc = torch.empty(Pn, I, dtype=torch.float32, device=x.device)
        pooled = torch.empty(Pn, dtype=torch.float32, device=x.device)
        q = torch.empty(Pn, I, dtype=torch.bfloat16, device=x.device)      # the last template writes the gated output over q
        gate = torch.empty_like(q)
        ws = _ops.workspace(lib.af2_template_pointwise_rows_begin_workspace(Pn, d), x.device)
        _lib.check(lib.af2_template_pointwise_rows_begin(w, x_rows.data_ptr(), Pn, d, H, dh, q.data_ptr(), gate.data_ptr(),
                                                         ws.data_ptr(), ws.numel(), s))
        for k in range(T):
            t_row = _ops.template_embed(embed, templates_feats[0, k, n0:n1].detach().float().contiguous())   # [Rn, n, d]
            sh = _PairShards(group, n, tm[k][:, None] & tm[k][None, :], to_cols, to_rows)                     # crossed mask
            if ex is not None:
                t_row = ex.buffer(PeerExchange.PAIR, "row").copy_(t_row)
            for _ in range(model.templates_embed_layers):
                t_row = sharded_pair_track(ops, pair, t_row, sh)
            t_row = t_row.contiguous()
            ws = _ops.workspace(lib.af2_template_pointwise_rows_group_workspace(1, Pn, d, H, dh), x.device)
            _lib.check(lib.af2_template_pointwise_rows_group(
                w, t_row.data_ptr(), None if xm is None else xm.data_ptr(), sh.mask_rows.data_ptr(), 1, Pn, Pn, d, H, dh,
                q.data_ptr(), gate.data_ptr(), run_max.data_ptr(), run_sum.data_ptr(), acc.data_ptr(), pooled.data_ptr(),
                q.data_ptr(), int(k == 0), int(k == T - 1), ws.data_ptr(), ws.numel(), s))
            del t_row
        ws = _ops.workspace(lib.af2_template_pointwise_rows_end_workspace(Pn, H, dh), x.device)
        _lib.check(lib.af2_template_pointwise_rows_end(w, x_rows.data_ptr(), q.data_ptr(), pooled.data_ptr(), Pn, d, H, dh,
                                                       ws.data_ptr(), ws.numel(), s))
        if not rows_in:
            x[0].copy_(all_gather_cat0(x_rows, group, counts))
    return x


def shard_alphafold2(model, group=None, use_graph: Optional[bool] = None, pair_rows: bool = False):
    """Shard all of an Alphafold2's pair-tensor work over the ranks of `group`: the trunk (model.net) and the extra-MSA stack
    (model.extra_msa_evoformer, whose tied-query attention the schedule averages over all column shards) through
    shard_evoformer, each replayed as a CUDA graph when use_graph (see shard_evoformer), and the template branch
    (embed_templates_) through sharded_embed_templates_, eagerly.  Every rank must call forward with identical inputs (batch 1)
    and gets the full outputs back.  Returns `model`.

    pair_rows: model(...) runs sharded_alphafold2_rows instead, which keeps the pair tensor in row shards from the embedding
    to the heads and returns this rank's rows of the outputs (ret.pair_rows = (n0, n1); gather_pair_rows joins them)."""
    shard_evoformer(model.net, group, use_graph)
    shard_evoformer(model.extra_msa_evoformer, group, use_graph)

    def embed_templates_(x, x_mask, templates_feats, templates_mask):
        return sharded_embed_templates_(model, x, x_mask, templates_feats, templates_mask, group)

    model.embed_templates_ = embed_templates_
    if pair_rows:
        def forward(*args, **kwargs):
            return sharded_alphafold2_rows(model, group, *args, **kwargs)

        model.forward = forward
    else:
        model.__dict__.pop("forward", None)              # back to Alphafold2.forward, whatever an earlier call installed
    return model


def gather_pair_rows(t: torch.Tensor, group=None) -> torch.Tensor:
    """Every rank's pair rows t [1, n1 - n0, N, ...] (an output of shard_alphafold2(pair_rows=True): ret.distance,
    theta_logits, phi_logits, omega_logits) joined into the whole [1, N, N, ...] on every rank (one all-gather)."""
    N, P = t.shape[2], dist.get_world_size(group)
    return all_gather_cat0(t[0].contiguous(), group, shard_counts(N, P) if N % P else None)[None]


def _rows_refusals(model, group, seq, msa, extra_msa, extra_msa_mask, recyclables, return_trunk):
    """What sharded_alphafold2_rows cannot run, raised before any device work or collective."""
    from .alphafold2 import DISTOGRAM_BUCKETS
    if any(_ops.precision_of(mod) == "strict" for mod in (model.net, model.extra_msa_evoformer, model.template_pointwise_attn)):
        raise NotImplementedError("the strict precision mode runs on one GPU (it is a parity mode, not a throughput mode)")
    if model.predict_coords and not return_trunk:
        raise NotImplementedError("predict_coords=True needs the third-party structure module (see Alphafold2.forward)")
    if seq.dim() != 2 or seq.shape[0] != 1:
        raise ValueError(f"pair_rows mode handles one sequence per call (batch 1), got seq {tuple(seq.shape)}")
    P, N = dist.get_world_size(group), seq.shape[1]
    if N < P:
        raise ValueError(f"N_res={N} is smaller than the number of ranks {P}: every rank needs at least one pair row")
    if model.disable_token_embed:
        raise ValueError("pair_rows mode embeds tokens with the fused pair-init kernel: disable_token_embed is not supported")
    d = model.dim
    if not _ops.distogram_head_ok(d, DISTOGRAM_BUCKETS):
        raise ValueError(f"pair_rows mode: dim {d} is not taken by the distogram head kernel (a multiple of 128, <= 512)")
    if model.predict_angles and not _ops.angle_heads_ok(d, model.angle_heads().buckets()):
        raise ValueError(f"pair_rows mode: dim {d} and buckets {model.angle_heads().buckets()} are not taken by the angle heads kernel")
    if extra_msa is not None and (extra_msa_mask is None or extra_msa_mask.dim() != 3):
        raise ValueError("extra_msa_mask must be given with shape [b, n_msa, n] (the reference's default, alphafold2.py:791, has "
                         "the wrong rank and fails in einops too)")
    pair = getattr(recyclables, "pairwise_repr", None)
    if not seq.is_cuda or (msa is not None and not msa.is_cuda) or (torch.is_tensor(pair) and not pair.is_cuda):
        raise ValueError("pair_rows mode runs on CUDA tensors (seq, msa and recyclables on the GPU)")


def sharded_alphafold2_rows(model, group, seq, msa=None, mask=None, msa_mask=None, extra_msa=None, extra_msa_mask=None,
                            seq_index=None, seq_embed=None, msa_embed=None, templates_feats=None, templates_mask=None,
                            templates_angles=None, embedds=None, recyclables=None, return_trunk=False, return_confidence=False,
                            return_recyclables=False, return_aux_logits=False):
    """Alphafold2.forward of a model under shard_alphafold2(pair_rows=True): every pair-tensor stage runs on this rank's pair rows
    [n0, n1) = shard_offsets(N, P)[r:r + 2] and no rank holds the whole pair tensor.  Pair init rows -> recycling rows ->
    template branch on the rows -> template angles into m -> extra-MSA stack rows -> trunk rows -> one rows -> columns exchange
    of x -> distogram and angle heads on the rows.  Returns this rank's rows: ret.distance [1, n1 - n0, N, 37], theta / phi /
    omega_logits the same rows, ret.pair_rows = (n0, n1).  Each is bitwise those rows of the default shard_alphafold2 forward.
    The inputs stay replicated (every rank passes the same tensors and reads its rows of them); so does the MSA tensor m."""
    from .alphafold2 import ReturnValues
    _rows_refusals(model, group, seq, msa, extra_msa, extra_msa_mask, recyclables, return_trunk)
    model._check_inputs(seq, mask, seq_embed, msa_embed, embedds, templates_feats, templates_mask, templates_angles, recyclables)
    P, r, N = dist.get_world_size(group), dist.get_rank(group), seq.shape[1]
    on = shard_offsets(N, P)
    n0, n1 = on[r], on[r + 1]
    with torch.no_grad():
        if msa is None:                                                # alphafold2.py:656-658
            msa = seq[:, None, :]
            msa_mask = mask[:, None, :] if mask is not None else None
        if msa_mask is None:
            msa_mask = torch.ones_like(msa).bool()
        m_rows = msa.shape[1] + (templates_angles.shape[1] if templates_angles is not None else 0)
        x, m = _ops.embed_pair_init_rows(seq, msa, model.token_emb.weight, model.to_pairwise_repr.weight, model.to_pairwise_repr.bias,
                                         model.pos_emb.weight, model.max_rel_dist, n0, n1 - n0, seq_embed, msa_embed, seq_index,
                                         m_rows=m_rows)
        x_mask = (mask[:, :, None] & mask[:, None, :]) if mask is not None else None
        if recyclables is not None:
            model.embed_recyclables_(x, m, recyclables, row0=n0)
        if templates_feats is not None:
            sharded_embed_templates_(model, x, x_mask, templates_feats, templates_mask, group, rows_in=True)
        if templates_angles is not None:
            msa_mask = model.embed_template_angles_(m, msa_mask, templates_angles, templates_mask)
        if extra_msa is not None:
            extra_m, em = model.extra_msa_inputs(msa, extra_msa_mask)
            x, _ = model.extra_msa_evoformer(x, extra_m, mask=x_mask, msa_mask=em, rows_in=True)
            x = x[None]
        x_row, _ = model.net(x, m, mask=x_mask, msa_mask=msa_mask, rows_in=True)      # [n1 - n0, N, d]
        del x, m
        counts = shard_counts(N, P) if N % P else None
        x_col = rows_to_cols(x_row, group, counts, counts)                       # [N, n1 - n0, d]: the same rows as columns
        ret = ReturnValues()
        ln, lin = model.to_distogram_logits[0], model.to_distogram_logits[1]
        ret.distance = _ops.distogram_head_rows(x_row, x_col, ln.weight, ln.bias, lin.weight, lin.bias)
        if model.predict_angles:
            ret.theta_logits, ret.phi_logits, ret.omega_logits = _ops.angle_heads_rows(model.angle_heads().packed(), x_row, x_col,
                                                                                       model.symmetrize_omega)
        ret.pair_rows = (n0, n1)
    return ret


def pair_rows_bytes(N: int, S: int, d: int, heads: int, dim_head: int, P: int) -> int:
    """Device bytes one rank allocates in a shard_alphafold2(pair_rows=True) forward at its peak (the trunk's blocks), for the rank
    with the most pair rows, Rn = ceil(N / P), and an MSA of S rows (template angle rows included).  Not counted: the caller's
    replicated inputs (recyclables.pairwise_repr is a whole fp32 pair tensor, templates_feats T of them at templates_dim) and
    the weights.  Counted, from the library's workspace queries and the schedule's shapes:
      * the pair rows: the forward's x_rows, the trunk's working shard and its output, the peer arena's row and column buffers
        (4 fp32 [Rn, N, d] and one [N, Rn, d]), the replicated m and its arena buffers, the pair mask;
      * the operands a pair stage keeps: the gathered triangle operand (bf16 [d, N, align8(N)]) and the copy it is merged into
        (CudaStageOps merges the gathered pieces into one operand for uneven shards, and for even shards narrower than 64
        columns), the local L, R and gate, the gathered pair bias (twice: gathered and transposed); the outer mean's projected
        m and its gathered right operand, with its merged copy likewise;
      * the grow-only workspace sized for the largest stage call of a shard.
    The merged copies are counted at every P > 1, whether or not N % P makes the shards uneven: the estimate is then an upper
    bound that never decreases with N (an N that P divides needs at most what the next uneven N needs), so the longest N_res
    that fits a budget is a bound for every shorter length."""
    lib = _lib.load()
    Rn, Rs = -(-N // P), -(-S // P)
    N8 = _align8(N)
    ax = lib.af2_axial_attention_workspace
    ff = lambda tokens: lib.af2_feed_forward_workspace(tokens, d, 4 * d)  # noqa: E731
    ws = max(ax(1, Rn, N, d, heads, dim_head, 1), ax(1, N, Rn, d, heads, dim_head, 0), ax(1, max(Rs, 1), N, d, heads, dim_head, 1),
             ax(1, S, Rn, d, heads, dim_head, 0), ff(Rn * N), ff(S * Rn), lib.af2_triangle_project_workspace(Rn * N, d),
             lib.af2_triangle_contract_workspace(Rn, N, d), lib.af2_triangle_contract_workspace(N, Rn, d),
             lib.af2_outer_project_workspace(S * Rn, d), lib.af2_outer_contract_workspace(Rn, N, d))
    shard = Rn * N * d * 4
    resident = 6 * shard + S * N * d * 4 + 2 * (Rs * N * d * 4 + S * Rn * d * 4) + N * N
    merged = 2 if P > 1 else 1                                # gathered operand + the copy its pieces are merged into
    tri = merged * P * d * Rn * N8 * 2 + 2 * d * Rn * N8 * 2 + Rn * N * d * 2
    bias = 2 * heads * N * N8 * 2
    outer = 2 * d * S * _align8(Rn) * 2 + merged * P * d * S * _align8(Rn) * 2
    return int(resident + max(tri, outer) + bias + _ops._ws_alloc(ws))
