"""The stage ops on the GPU: each method is one stage of a pair or MSA module (pair bias, axial attention, a projection, a
contraction with its tail, the transition) on a band or shard of the tensors, launched through the stage-level C ABI.

The banded single-GPU schedule (banded.py) and the sharded multi-GPU schedule (parallel.py) both take their stage ops as a
provider object; CudaStageOps is the product's.  tests/ drive the same schedules with CPU oracle providers.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib, ops as _ops
from .ops import _align8


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
        """x_loc [rows, cols, d] += the triangle multiplication's contraction of L with the gathered Rg [pieces*d, ., .] and its
        tail.  Both operands are read in place with the pitches and channel strides of their strides, so a row window
        L[:, i0:i1] or a column window R[:, :, i0:i1] of a larger channel-major operand is just another operand.  pieces: the
        number of equal gathered pieces, or every piece's size along the gathered axis (uneven shards: merged into one operand)."""
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
        _lib.check(lib.af2_triangle_contract(C.byref(pk.struct), x_loc.data_ptr(), L.data_ptr(), L.stride(0), L.stride(1),
                                             Rg.data_ptr(), Rg.stride(0), Rg.stride(1), d * Rg.stride(0), pieces, gate.data_ptr(),
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
