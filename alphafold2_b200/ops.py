"""Tensor-level wrappers over the C ABI: argument validation, weight packing, workspace management.

PyTorch is used for device memory and streams only; every FLOP of the hot path runs inside libaf2b200.so.
"""
from __future__ import annotations

import ctypes as C
import functools
from typing import Dict, Optional

import torch

from . import _lib

_WORKSPACE: Dict[torch.device, torch.Tensor] = {}
_DEVICE_CHECKED = set()

# ---- packed-weight cache control (alphafold2._Packable) ----
import os as _os

PACK_CHECK = _os.environ.get("AF2_PACK_CHECK", "0") not in ("", "0")      # content fingerprint in the cache key (debug aid)
_PACK_EPOCH = 0
PRECISIONS = ("bf16", "strict")
_DEFAULT_PRECISION = _os.environ.get("AF2_PRECISION", "bf16")
if _DEFAULT_PRECISION not in PRECISIONS:
    raise ValueError(f"AF2_PRECISION must be one of {PRECISIONS}, got {_DEFAULT_PRECISION!r}")


def pack_epoch() -> int:
    return _PACK_EPOCH


def bump_pack_epoch() -> None:
    global _PACK_EPOCH
    _PACK_EPOCH += 1


def precision_of(module) -> str:
    """'bf16' (default: bf16 tensor-core operands, fp32 accumulate) or 'strict' (split-bf16 operands: 3 planes, 6 tensor-core passes; fp32-grade results
    inside the north star's rtol 1e-3 / atol 1e-4 band).  Set per model with alphafold2_b200.set_precision()."""
    return module.__dict__.get("_af2_precision", _DEFAULT_PRECISION)


def set_precision(module, mode: str):
    """Select the arithmetic of every hot-path module under `module`: 'bf16' or 'strict'.  Returns `module`."""
    if mode not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {mode!r}")
    for mod in module.modules():
        mod.__dict__["_af2_precision"] = mode
    return module



def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _require(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (alphafold2_b200 has no CPU fallback)")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    dev = t.device
    if dev not in _DEVICE_CHECKED:
        with torch.cuda.device(dev):
            _lib.check(_lib.load().af2_check_device())
        _DEVICE_CHECKED.add(dev)


_WS_PRIVATE = None        # (dict device -> tensor, locked) while a CUDA graph owner captures (parallel._GraphedTrunk)
_WS_CAPTURED: Dict[int, torch.Tensor] = {}     # shared workspaces handed out during a caller's CUDA-graph capture, by address


def workspace(nbytes: int, device) -> torch.Tensor:
    """Grow-only per-device scratch buffer, reused by every op (ops on one stream are serialised).  Inside a
    `private_workspace` scope the buffer belongs to the scope's owner (a captured CUDA graph keeps raw pointers into it).
    A shared buffer handed out while the current stream is capturing a CUDA graph is retained: growth and release_workspace
    drop it from the store but do not free it, since the graph replays into it; release_captured_workspaces() frees it."""
    device = torch.device(device)
    store, locked = (_WORKSPACE, False) if _WS_PRIVATE is None else _WS_PRIVATE
    buf = store.get(device)
    if buf is None or buf.numel() < nbytes:
        if locked:
            raise RuntimeError("workspace would have to grow during CUDA-graph capture (warm-up did not size it)")
        buf = None
        store.pop(device, None)
        buf = torch.empty(int(nbytes * 1.05) + 4096, dtype=torch.uint8, device=device)
        store[device] = buf
    if store is _WORKSPACE and torch.cuda.is_current_stream_capturing():
        _WS_CAPTURED[buf.data_ptr()] = buf
    return buf


def release_captured_workspaces() -> None:
    """Free the shared workspace buffers that ops used while a caller captured them in a CUDA graph (see workspace).  Call it
    once the graphs that captured ops are dropped; a graph replayed after this call reads and writes freed memory."""
    _WS_CAPTURED.clear()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


class private_workspace:
    """with private_workspace(store, locked): every op draws its scratch from `store` (dict owned by the caller)."""

    def __init__(self, store: dict, locked: bool):
        self.cfg = (store, locked)

    def __enter__(self):
        global _WS_PRIVATE
        self.prev = _WS_PRIVATE
        _WS_PRIVATE = self.cfg
        return self

    def __exit__(self, *exc):
        global _WS_PRIVATE
        _WS_PRIVATE = self.prev
        return False


def _mask_u8(mask: Optional[torch.Tensor], shape, name: str) -> Optional[torch.Tensor]:
    if mask is None:
        return None
    if mask.dtype != torch.bool:
        mask = mask.bool()
    if tuple(mask.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(mask.shape)}")
    return mask.contiguous()


# --------------------------------------------------------------------------------------------------
# weight packing (done once per parameter version; see alphafold2.py::_PackedCache)
# --------------------------------------------------------------------------------------------------
def _bf16(t):
    return t.detach().to(torch.bfloat16).contiguous()


def _f32(t):
    return t.detach().to(torch.float32).contiguous()


def gated_half(n_out: int) -> int:
    return 128 if n_out >= 128 else (64 if n_out >= 64 else 32)


def pack_gated(w_val, b_val, w_gate, b_gate, half: int):
    """Interleave value/gate rows per accumulator column tile: [half value rows | half gate rows] * tiles."""
    n_out, k = w_val.shape
    tiles = (n_out + half - 1) // half
    w = torch.zeros(tiles * 2 * half, k, dtype=torch.float32, device=w_val.device)
    b = torch.zeros(tiles * 2 * half, dtype=torch.float32, device=w_val.device)
    for t in range(tiles):
        lo, hi = t * half, min(n_out, (t + 1) * half)
        w[t * 2 * half: t * 2 * half + (hi - lo)] = w_val[lo:hi]
        w[t * 2 * half + half: t * 2 * half + half + (hi - lo)] = w_gate[lo:hi]
        b[t * 2 * half: t * 2 * half + (hi - lo)] = b_val[lo:hi]
        b[t * 2 * half + half: t * 2 * half + half + (hi - lo)] = b_gate[lo:hi]
    return w, b.contiguous()          # fp32; callers round to bf16


def _pad_rows(t: torch.Tensor, mult: int = 256) -> torch.Tensor:
    """Zero-pad dim 0 to a multiple of `mult`."""
    r = (-t.shape[0]) % mult
    if r == 0:
        return t
    return torch.cat([t, torch.zeros((r,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)], 0)


def _p(t):
    return None if t is None else t.data_ptr()


class Packed:
    """Keeps the packed tensors alive next to the ctypes struct that points at them."""

    def __init__(self, struct, tensors, kind: str = "bf16"):
        self.struct = struct
        self.tensors = tensors
        self.kind = kind          # "bf16" (default path) or "strict" (split-bf16 x3 operands)


def pack_feed_forward(norm_w, norm_b, w1, b1, w2, b2) -> Packed:
    hidden = w2.shape[1]
    half = gated_half(hidden)
    a_w, g_w = w1[:hidden].detach().float(), w1[hidden:].detach().float()
    a_b, g_b = b1[:hidden].detach().float(), b1[hidden:].detach().float()
    w1f, b1p = pack_gated(a_w, a_b, g_w, g_b, half)
    t = dict(g=_f32(norm_w), b=_f32(norm_b), w1=_bf16(w1f), b1=b1p, w2=_bf16(w2), b2=_f32(b2))
    s = _lib.FFWeights(t["g"].data_ptr(), t["b"].data_ptr(), t["w1"].data_ptr(), t["b1"].data_ptr(),
                       t["w2"].data_ptr(), t["b2"].data_ptr(), 2 * half)
    return Packed(s, t)


def pack_attention(norm_w, norm_b, wq, wkv, wg, bg, wo, bo, w_edge, dim_head: int) -> Packed:
    # alphafold2.py:112,138: q * dim_head^-0.5 is folded into to_q, together with log2(e) so that the kernel's
    # softmax works in the exp2 domain; the pair-bias projection gets the same log2(e).
    log2e = 1.4426950408889634
    scale = dim_head ** -0.5 * log2e
    wqkv = torch.cat([wq.detach().float() * scale, wkv.detach().float()], dim=0)
    t = dict(g=_f32(norm_w), b=_f32(norm_b), wqkv=_bf16(wqkv), wg=_bf16(wg), bg=_f32(bg), wo=_bf16(wo), bo=_f32(bo))
    if w_edge is not None:
        t["we"] = _f32(w_edge.detach().float() * log2e)
    s = _lib.AttnWeights(t["g"].data_ptr(), t["b"].data_ptr(), t["wqkv"].data_ptr(), t["wg"].data_ptr(),
                         t["bg"].data_ptr(), t["wo"].data_ptr(), t["bo"].data_ptr(),
                         t["we"].data_ptr() if w_edge is not None else None)
    return Packed(s, t)


def pack_triangle_multiply(norm_w, norm_b, wl, bl, wr, br, wlg, blg, wrg, brg, wog, bog, onw, onb, wo, bo) -> Packed:
    d = wl.shape[0]
    half = gated_half(d)
    f = lambda x: x.detach().float()  # noqa: E731
    wlp, blp = pack_gated(f(wl), f(bl), f(wlg), f(blg), half)
    wrp, brp = pack_gated(f(wr), f(br), f(wrg), f(brg), half)
    t = dict(g=_f32(norm_w), b=_f32(norm_b), wl=_bf16(wlp), bl=blp, wr=_bf16(wrp), br=brp, wog=_bf16(wog), bog=_f32(bog),
             ong=_f32(onw), onb=_f32(onb), wo=_bf16(wo), bo=_f32(bo))
    s = _lib.TriMulWeights(t["g"].data_ptr(), t["b"].data_ptr(), t["wl"].data_ptr(), t["bl"].data_ptr(),
                           t["wr"].data_ptr(), t["br"].data_ptr(), t["wog"].data_ptr(), t["bog"].data_ptr(),
                           t["ong"].data_ptr(), t["onb"].data_ptr(), t["wo"].data_ptr(), t["bo"].data_ptr(), 2 * half)
    return Packed(s, t)


def pack_outer_mean(norm_w, norm_b, wl, bl, wr, br, wo, bo) -> Packed:
    t = dict(g=_f32(norm_w), b=_f32(norm_b), wlr=_bf16(torch.cat([wl.detach(), wr.detach()], 0)),
             blr=_f32(torch.cat([bl.detach(), br.detach()], 0)), wo=_bf16(wo), bo=_f32(bo))
    s = _lib.OuterWeights(t["g"].data_ptr(), t["b"].data_ptr(), t["wlr"].data_ptr(), t["blr"].data_ptr(),
                          t["wo"].data_ptr(), t["bo"].data_ptr())
    return Packed(s, t)


# --------------------------------------------------------------------------------------------------
# strict precision mode: split-bf16 weights (v = hi + lo), fp32 biases / LayerNorm affine
# --------------------------------------------------------------------------------------------------
SPLIT_PLANES = 3       # bf16 planes per strict-mode operand (csrc/strict_kernels.cuh: SPL)


def split_weight(w: torch.Tensor) -> torch.Tensor:
    """fp32 [rows, K] -> bf16 [rows, 3, align8(K)]: plane 0 = bf16(w), plane 1 = bf16(w - p0), plane 2 = bf16(w - p0 - p1)
    (24 mantissa bits in total; the subtractions are exact in fp32); pad columns zero."""
    w = w.detach().to(torch.float32)
    rows, K = w.shape
    P = (K + 7) // 8 * 8
    out = torch.zeros(rows, SPLIT_PLANES, P, dtype=torch.bfloat16, device=w.device)
    r = w
    for pl in range(SPLIT_PLANES):
        h = r.to(torch.bfloat16)
        out[:, pl, :K] = h
        r = r - h.float()
    return out.contiguous()


def _bias_pad(b: torch.Tensor) -> torch.Tensor:
    """fp32 bias zero-padded to a multiple of 256 entries: the GEMM epilogue loads biases per 32-column chunk of a 256-column tile."""
    return _pad_rows(b.detach().to(torch.float32).reshape(-1)).contiguous()


def pack_feed_forward_strict(norm_w, norm_b, w1, b1, w2, b2) -> Packed:
    t = dict(g=_f32(norm_w), b=_f32(norm_b), w1=split_weight(w1), b1=_bias_pad(b1), w2=split_weight(w2), b2=_bias_pad(b2))
    s = _lib.FFWeightsStrict(*(t[k].data_ptr() for k in ("g", "b", "w1", "b1", "w2", "b2")))
    pk = Packed(s, t, "strict")
    pk.hidden = int(w2.shape[1])
    return pk


def pack_attention_strict(norm_w, norm_b, wq, wkv, wg, bg, wo, bo, w_edge, dim_head: int) -> Packed:
    wcat = torch.cat([wq.detach().float() * dim_head ** -0.5, wkv.detach().float(), wg.detach().float()], 0)   # alphafold2.py:138
    bcat = torch.cat([torch.zeros(wq.shape[0] + wkv.shape[0], device=wq.device), bg.detach().float()], 0)
    t = dict(g=_f32(norm_w), b=_f32(norm_b), w=split_weight(wcat), bias=_bias_pad(bcat), wo=split_weight(wo), bo=_bias_pad(bo))
    if w_edge is not None:
        t["we"] = _f32(w_edge)
    s = _lib.AttnWeightsStrict(t["g"].data_ptr(), t["b"].data_ptr(), t["w"].data_ptr(), t["bias"].data_ptr(), t["wo"].data_ptr(),
                               t["bo"].data_ptr(), _p(t.get("we")))
    return Packed(s, t, "strict")


def pack_triangle_multiply_strict(norm_w, norm_b, wl, bl, wr, br, wlg, blg, wrg, brg, wog, bog, onw, onb, wo, bo) -> Packed:
    f = lambda x: x.detach().float()  # noqa: E731
    w5 = torch.cat([f(wl), f(wr), f(wlg), f(wrg), f(wog)], 0)
    b5 = torch.cat([f(bl), f(br), f(blg), f(brg), f(bog)], 0)
    t = dict(g=_f32(norm_w), b=_f32(norm_b), w5=split_weight(w5), b5=_bias_pad(b5), ong=_f32(onw), onb=_f32(onb), wo=split_weight(wo), bo=_bias_pad(bo))
    s = _lib.TriMulWeightsStrict(*(t[k].data_ptr() for k in ("g", "b", "w5", "b5", "ong", "onb", "wo", "bo")))
    return Packed(s, t, "strict")


def pack_outer_mean_strict(norm_w, norm_b, wl, bl, wr, br, wo, bo) -> Packed:
    t = dict(g=_f32(norm_w), b=_f32(norm_b), wlr=split_weight(torch.cat([wl.detach().float(), wr.detach().float()], 0)),
             blr=_bias_pad(torch.cat([bl.detach(), br.detach()], 0)), wo=split_weight(wo), bo=_bias_pad(bo))
    s = _lib.OuterWeightsStrict(*(t[k].data_ptr() for k in ("g", "b", "wlr", "blr", "wo", "bo")))
    return Packed(s, t, "strict")


# --------------------------------------------------------------------------------------------------
# ops (all in place on the fp32 residual stream)
# --------------------------------------------------------------------------------------------------
def feed_forward_(pk: Packed, x: torch.Tensor) -> torch.Tensor:
    """x [..., d] fp32  <-  x + FeedForward(x)   (alphafold2.py:74-94, 439, 444)."""
    _require(x, torch.float32, "x")
    lib = _lib.load()
    d = x.shape[-1]
    tokens = x.numel() // d
    if pk.kind == "strict":
        hidden = pk.hidden
        ws = workspace(lib.af2_feed_forward_strict_workspace(tokens, d, hidden), x.device)
        _lib.check(lib.af2_feed_forward_strict(C.byref(pk.struct), x.data_ptr(), tokens, d, hidden, ws.data_ptr(), ws.numel(),
                                               _stream_ptr()))
        return x
    hidden = pk.tensors["w2"].shape[1]
    nbytes = lib.af2_feed_forward_workspace(tokens, d, hidden)
    ws = workspace(nbytes, x.device)
    _lib.check(lib.af2_feed_forward(C.byref(pk.struct), x.data_ptr(), tokens, d, hidden, ws.data_ptr(), ws.numel(),
                                    _stream_ptr()))
    return x


def axial_attention_(pk: Packed, x: torch.Tensor, heads: int, dim_head: int, row_attn: bool,
                     edges: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None, tied: bool = False) -> torch.Tensor:
    """x [b, h, w, d] fp32  <-  x + AxialAttention(x, edges, mask)   (alphafold2.py:192-255, 98-190).
    tied: global_query_attn -- queries averaged over the folded axis (alphafold2.py:142-151, 250)."""
    _require(x, torch.float32, "x")
    if x.dim() != 4:
        raise ValueError("x must be [b, h, w, d]")
    B, h, w, d = x.shape
    n = w if row_attn else h
    if edges is not None:
        _require(edges, torch.float32, "edges")
        if tuple(edges.shape) != (B, n, n, d):
            raise ValueError(f"edges must be [{B}, {n}, {n}, {d}], got {tuple(edges.shape)}")
        if "we" not in pk.tensors:
            edges = None                      # module built without accept_edges: the reference ignores edges
    mask = _mask_u8(mask, (B, h, w), "mask")
    lib = _lib.load()
    if pk.kind == "strict":
        ws = workspace(lib.af2_axial_attention_strict_workspace(B, h, w, d, heads, dim_head, int(row_attn)), x.device)
        _lib.check(lib.af2_axial_attention_strict(C.byref(pk.struct), x.data_ptr(), _ptr(edges), _ptr(mask), B, h, w, d, heads,
                                                  dim_head, int(row_attn), int(tied), ws.data_ptr(), ws.numel(), _stream_ptr()))
        return x
    nbytes = lib.af2_axial_attention_workspace(B, h, w, d, heads, dim_head, int(row_attn))
    ws = workspace(nbytes, x.device)
    _lib.check(lib.af2_axial_attention_ex(C.byref(pk.struct), x.data_ptr(), _ptr(edges), _ptr(mask), B, h, w, d, heads,
                                          dim_head, int(row_attn), int(tied), ws.data_ptr(), ws.numel(), _stream_ptr()))
    return x


def triangle_multiply_(pk: Packed, x: torch.Tensor, ingoing: bool, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [b, N, N, d] fp32  <-  x + TriangleMultiplicativeModule(x, mask)   (alphafold2.py:257-317)."""
    _require(x, torch.float32, "x")
    assert x.dim() == 4 and x.shape[1] == x.shape[2], "feature map must be symmetrical"   # alphafold2.py:293
    B, N, _, d = x.shape
    mask = _mask_u8(mask, (B, N, N), "mask")
    lib = _lib.load()
    if pk.kind == "strict":
        ws = workspace(lib.af2_triangle_multiply_strict_workspace(B, N, d), x.device)
        _lib.check(lib.af2_triangle_multiply_strict(C.byref(pk.struct), x.data_ptr(), _ptr(mask), B, N, d, int(ingoing),
                                                    ws.data_ptr(), ws.numel(), _stream_ptr()))
        return x
    nbytes = lib.af2_triangle_multiply_workspace(B, N, d)
    ws = workspace(nbytes, x.device)
    _lib.check(lib.af2_triangle_multiply(C.byref(pk.struct), x.data_ptr(), _ptr(mask), B, N, d, int(ingoing),
                                         ws.data_ptr(), ws.numel(), _stream_ptr()))
    return x


def outer_mean_(pk: Packed, x: torch.Tensor, m: torch.Tensor, msa_mask: Optional[torch.Tensor] = None,
                eps: float = 1e-5) -> torch.Tensor:
    """x [b, N, N, d] fp32  <-  x + OuterMean(m, msa_mask)   (alphafold2.py:321-351, 379)."""
    _require(x, torch.float32, "x")
    _require(m, torch.float32, "m")
    B, S, N, d = m.shape
    if tuple(x.shape) != (B, N, N, d):
        raise ValueError(f"x must be [{B}, {N}, {N}, {d}], got {tuple(x.shape)}")
    msa_mask = _mask_u8(msa_mask, (B, S, N), "msa_mask")
    lib = _lib.load()
    if pk.kind == "strict":
        ws = workspace(lib.af2_outer_mean_strict_workspace(B, S, N, d), x.device)
        _lib.check(lib.af2_outer_mean_strict(C.byref(pk.struct), x.data_ptr(), m.data_ptr(), _ptr(msa_mask), B, S, N, d,
                                             float(eps), ws.data_ptr(), ws.numel(), _stream_ptr()))
        return x
    nbytes = lib.af2_outer_mean_workspace(B, S, N, d)
    ws = workspace(nbytes, x.device)
    _lib.check(lib.af2_outer_mean(C.byref(pk.struct), x.data_ptr(), m.data_ptr(), _ptr(msa_mask), B, S, N, d,
                                  float(eps), ws.data_ptr(), ws.numel(), _stream_ptr()))
    return x


def apply_rotary_pos_emb(x: torch.Tensor, sinu_pos) -> torch.Tensor:
    """rotary.py:15-20.  x [b, h, n, dh] fp32, sinu_pos = (sin, cos) each [1 or b, n, rot]."""
    sin, cos = sinu_pos
    _require(x, torch.float32, "x")
    sin, cos = sin.contiguous().float(), cos.contiguous().float()
    b, h, n, dh = x.shape
    y = torch.empty_like(x)
    _lib.check(_lib.load().af2_rotary(x.data_ptr(), sin.data_ptr(), cos.data_ptr(), y.data_ptr(), b, h, n, dh,
                                      sin.shape[-1], sin.shape[0], _stream_ptr()))
    return y


# --------------------------------------------------------------------------------------------------
# pre- / post-trunk glue (SURVEY.md 8f n1)
# --------------------------------------------------------------------------------------------------
def _w32(t: torch.Tensor) -> torch.Tensor:
    t = t.detach()
    return t if (t.dtype == torch.float32 and t.is_contiguous()) else t.to(torch.float32).contiguous()


def embed_pair_init(seq, msa, token_emb, w_pair, b_pair, pos_emb, max_rel_dist: int, seq_embed=None, msa_embed=None, seq_index=None,
                    m_rows: Optional[int] = None):
    """alphafold2.py:676-726 in three fused kernels: returns (x [b,n,n,d], m [b,m_rows,n,d]) fp32.  m_rows > s leaves rows s..
    m_rows - 1 of m unwritten (the template angle features go there)."""
    return _embed_pair_init(seq, msa, token_emb, w_pair, b_pair, pos_emb, max_rel_dist, seq_embed, msa_embed, seq_index, m_rows, None)


def embed_pair_init_rows(seq, msa, token_emb, w_pair, b_pair, pos_emb, max_rel_dist: int, row0: int, rows: int, seq_embed=None,
                         msa_embed=None, seq_index=None, m_rows: Optional[int] = None):
    """embed_pair_init writing only pair rows [row0, row0 + rows): returns (x_rows [b,rows,n,d], m [b,m_rows,n,d] whole), bitwise
    those rows of embed_pair_init's x and its m (af2_embed_pair_init_rows)."""
    return _embed_pair_init(seq, msa, token_emb, w_pair, b_pair, pos_emb, max_rel_dist, seq_embed, msa_embed, seq_index, m_rows,
                            (int(row0), int(rows)))


def _embed_pair_init(seq, msa, token_emb, w_pair, b_pair, pos_emb, max_rel_dist, seq_embed, msa_embed, seq_index, m_rows, window):
    if not seq.is_cuda:
        raise RuntimeError("seq must be a CUDA tensor (alphafold2_b200 has no CPU fallback)")
    emb = _w32(token_emb)
    _require(emb, torch.float32, "token_emb.weight")
    B, n = seq.shape
    S = msa.shape[1]
    d = emb.shape[1]
    seq = seq.to(torch.int64).contiguous()
    msa = msa.to(torch.int64).contiguous()
    x = torch.empty(B, n if window is None else max(window[1], 0), n, d, dtype=torch.float32, device=seq.device)
    R = S if m_rows is None else int(m_rows)
    if R < S:
        raise ValueError(f"m_rows {R} < {S} MSA rows")
    m = torch.empty(B, R, n, d, dtype=torch.float32, device=seq.device)
    se = None if seq_embed is None else _w32(seq_embed)
    me = None if msa_embed is None else _w32(msa_embed)
    si = None if seq_index is None else seq_index.to(device=seq.device, dtype=torch.int64).contiguous()
    lib = _lib.load()
    ws = workspace(lib.af2_embed_pair_init_workspace(B, n, d), seq.device)
    wp, bp, pe = _w32(w_pair), _w32(b_pair), _w32(pos_emb)

    def call(sq, ms, s_e, m_e, xo, mo, nb):
        head = (sq.data_ptr(), ms.data_ptr(), emb.data_ptr(), emb.shape[0], _ptr(s_e), _ptr(m_e), wp.data_ptr(), bp.data_ptr(),
                pe.data_ptr(), int(max_rel_dist), _ptr(si), xo.data_ptr(), mo.data_ptr(), nb, S, n, d)
        tail = (ws.data_ptr(), ws.numel(), _stream_ptr())
        if window is None:
            _lib.check(lib.af2_embed_pair_init(*head, *tail))
        else:
            _lib.check(lib.af2_embed_pair_init_rows(*head, *window, *tail))

    if R != S and B > 1:
        # the kernels write S contiguous rows per batch element: one call per element into its slice of m
        for b in range(B):
            pick = lambda t: None if t is None else t[b]  # noqa: E731
            call(seq[b], msa[b], pick(se), pick(me), x[b], m[b], 1)
        return x, m
    call(seq, msa, se, me, x, m, B)
    return x, m


def distogram_head_ok(d: int, buckets: int) -> bool:
    return d % 128 == 0 and d <= 512 and (buckets * d + buckets) * 4 <= 200 * 1024


def distogram_head(x, ln_w, ln_b, w, b) -> torch.Tensor:
    """alphafold2.py:821-823: Linear(LayerNorm((x + x^T) / 2)) -> [b, n, n, buckets] fp32, one fused kernel."""
    _require(x, torch.float32, "x")
    B, n, _, d = x.shape
    buckets = w.shape[0]
    out = torch.empty(B, n, n, buckets, dtype=torch.float32, device=x.device)
    g, be, ww, bb = _w32(ln_w), _w32(ln_b), _w32(w), _w32(b)
    _lib.check(_lib.load().af2_distogram_head(x.data_ptr(), g.data_ptr(), be.data_ptr(), ww.data_ptr(), bb.data_ptr(), out.data_ptr(),
                                              B, n, d, buckets, _stream_ptr()))
    return out


def _rows_cols(x_rows: torch.Tensor, x_cols: Optional[torch.Tensor]):
    """(rows, n, d) of a row shard x_rows [rows, n, d] and its column shard x_cols [n, rows, d] (None: not needed)."""
    _require(x_rows, torch.float32, "x_rows")
    if x_rows.dim() != 3:
        raise ValueError(f"x_rows must be [rows, n, d], got {tuple(x_rows.shape)}")
    rows, n, d = x_rows.shape
    if x_cols is not None:
        _require(x_cols, torch.float32, "x_cols")
        if tuple(x_cols.shape) != (n, rows, d):
            raise ValueError(f"x_cols must be [{n}, {rows}, {d}], got {tuple(x_cols.shape)}")
    return rows, n, d


def distogram_head_rows(x_rows, x_cols, ln_w, ln_b, w, b) -> torch.Tensor:
    """distogram_head on pair rows [row0, row0 + rows): x_rows [rows, n, d] and the same rows as columns, x_cols [n, rows, d]
    (x_cols[j][i - row0] = x[j][i]) -> [1, rows, n, buckets] fp32, bitwise those rows of distogram_head(x)."""
    rows, n, d = _rows_cols(x_rows, x_cols)
    buckets = w.shape[0]
    out = torch.empty(1, rows, n, buckets, dtype=torch.float32, device=x_rows.device)
    g, be, ww, bb = _w32(ln_w), _w32(ln_b), _w32(w), _w32(b)
    _lib.check(_lib.load().af2_distogram_head_rows(x_rows.data_ptr(), x_cols.data_ptr(), g.data_ptr(), be.data_ptr(), ww.data_ptr(),
                                                   bb.data_ptr(), out.data_ptr(), rows, n, d, buckets, _stream_ptr()))
    return out


ANGLE_COLS = 64          # output columns of af2_angle_heads' tile (csrc/heads.cuh: AH_COLS)


def angle_heads_ok(d: int, buckets) -> bool:
    """Whether af2_angle_heads takes dim d and buckets (n_theta, n_phi, n_omega) in both omega modes (include/af2b200.h)."""
    nt, np_, no = (int(v) for v in buckets)
    row0 = min((nt + np_) // 8 * 8, 32)      # the symmetrised pass's 32-row weight window (csrc/heads_api.inl)
    return (d % 32 == 0 and 0 < d <= 320 and min(nt, np_, no) >= 1 and nt + np_ + no <= ANGLE_COLS
            and nt + np_ - row0 + no <= 32)


def pack_angle_heads(w_theta, b_theta, w_phi, b_phi, w_omega, b_omega) -> Packed:
    """The three heads as one 64-row weight [W_t; W_p; W_o; 0] in split-bf16 planes, bf16 [d / 32][3][64][32], and its bias [64]."""
    ws = [w.detach().float() for w in (w_theta, w_phi, w_omega)]
    d = ws[0].shape[1]
    rows = sum(w.shape[0] for w in ws)
    w = torch.zeros(ANGLE_COLS, d, dtype=torch.float32, device=ws[0].device)
    w[:rows] = torch.cat(ws, 0)
    bias = torch.zeros(ANGLE_COLS, dtype=torch.float32, device=w.device)
    bias[:rows] = torch.cat([b.detach().float() for b in (b_theta, b_phi, b_omega)])
    planes = split_weight(w).reshape(ANGLE_COLS, SPLIT_PLANES, d // 32, 32).permute(2, 1, 0, 3).contiguous()
    pk = Packed(None, dict(planes=planes, bias=bias), "split")
    pk.buckets = tuple(int(t.shape[0]) for t in ws)
    return pk


def angle_heads(pk: Packed, x: torch.Tensor, symmetrize_omega: bool):
    """alphafold2.py:813-836: (theta, phi, omega) logits [b, n, n, buckets] fp32 from the trunk output x [b, n, n, d] in one kernel
    that reads x once; omega from (x + x^T) / 2 when symmetrize_omega, formed in shared memory (no temporary of x's size)."""
    _require(x, torch.float32, "x")
    B, n, n2, d = x.shape
    if n != n2:
        raise ValueError(f"x must be [b, n, n, d], got {tuple(x.shape)}")
    nt, np_, no = pk.buckets
    theta = torch.empty(B, n, n, nt, dtype=torch.float32, device=x.device)
    phi = torch.empty(B, n, n, np_, dtype=torch.float32, device=x.device)
    omega = torch.empty(B, n, n, no, dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().af2_angle_heads(x.data_ptr(), pk.tensors["planes"].data_ptr(), pk.tensors["bias"].data_ptr(),
                                           theta.data_ptr(), phi.data_ptr(), omega.data_ptr(), B, n, d, nt, np_, no,
                                           int(bool(symmetrize_omega)), _stream_ptr()))
    return theta, phi, omega


def angle_heads_rows(pk: Packed, x_rows: torch.Tensor, x_cols: Optional[torch.Tensor], symmetrize_omega: bool):
    """angle_heads on pair rows [row0, row0 + rows): (theta, phi, omega) [1, rows, n, buckets] fp32 from x_rows [rows, n, d], and
    with symmetrize_omega from the same rows as columns x_cols [n, rows, d] (x_cols[j][i - row0] = x[j][i]; unused otherwise).
    Bitwise those rows of angle_heads(x)."""
    rows, n, d = _rows_cols(x_rows, x_cols if symmetrize_omega else None)
    nt, np_, no = pk.buckets
    theta = torch.empty(1, rows, n, nt, dtype=torch.float32, device=x_rows.device)
    phi = torch.empty(1, rows, n, np_, dtype=torch.float32, device=x_rows.device)
    omega = torch.empty(1, rows, n, no, dtype=torch.float32, device=x_rows.device)
    _lib.check(_lib.load().af2_angle_heads_rows(x_rows.data_ptr(), _ptr(x_cols) if symmetrize_omega else None,
                                                pk.tensors["planes"].data_ptr(), pk.tensors["bias"].data_ptr(), theta.data_ptr(),
                                                phi.data_ptr(), omega.data_ptr(), rows, n, d, nt, np_, no,
                                                int(bool(symmetrize_omega)), _stream_ptr()))
    return theta, phi, omega


_RECYCLE_BOUNDARIES: Dict[tuple, torch.Tensor] = {}


def recycling_boundaries(nb: int, device) -> torch.Tensor:
    """torch.linspace(2, 20, steps=nb) on `device` (alphafold2.py:736), cached per (nb, device): built by the same torch call as
    the reference's, so the bucket edges are bitwise its own.  The kernel searches the first nb - 1 of them."""
    device = torch.device(device)
    key = (int(nb), device)
    t = _RECYCLE_BOUNDARIES.get(key)
    if t is None:
        t = torch.linspace(2, 20, steps=int(nb), device=device, dtype=torch.float32)
        _RECYCLE_BOUNDARIES[key] = t
    return t


def recycle_embed_(x, m, coords, single_row, prev_pair, msa_gamma, msa_beta, pair_gamma, pair_beta, table, eps: float = 1e-5,
                   boundaries: Optional[torch.Tensor] = None):
    """alphafold2.py:730-739 in one kernel, in place: x [b,n,n,d] += LN_pair(prev_pair), then += table[bucket(dist)]; row 0 of
    m [b,rows,n,d] += LN_msa(single_row).  coords [b,n,c], single_row [b,n,d], prev_pair [b,n,n,d]; every tensor fp32 on x's
    device.  `boundaries` defaults to recycling_boundaries(table rows)."""
    return _recycle_embed(x, m, coords, single_row, prev_pair, msa_gamma, msa_beta, pair_gamma, pair_beta, table, eps, boundaries,
                          None)


def recycle_embed_rows_(x_rows, m, coords, single_row, prev_pair_rows, msa_gamma, msa_beta, pair_gamma, pair_beta, table, row0: int,
                        eps: float = 1e-5, boundaries: Optional[torch.Tensor] = None):
    """recycle_embed_ on pair rows [row0, row0 + rows): x_rows and prev_pair_rows [b,rows,n,d] (those rows of x and of the previous
    pair tensor), coords whole; row 0 of m is updated whole.  Bitwise those rows of recycle_embed_ and the same m."""
    return _recycle_embed(x_rows, m, coords, single_row, prev_pair_rows, msa_gamma, msa_beta, pair_gamma, pair_beta, table, eps,
                          boundaries, int(row0))


def _recycle_embed(x, m, coords, single_row, prev_pair, msa_gamma, msa_beta, pair_gamma, pair_beta, table, eps, boundaries, row0):
    _require(x, torch.float32, "x")
    _require(m, torch.float32, "m")
    B, rows, n, d = x.shape
    if row0 is None and rows != n:
        raise ValueError(f"x must be [b, n, n, d], got {tuple(x.shape)}")
    if m.dim() != 4 or m.shape[0] != B or m.shape[2] != n or m.shape[3] != d or m.shape[1] < 1:
        raise ValueError(f"m must be [{B}, rows, {n}, {d}], got {tuple(m.shape)}")
    nb = table.shape[0]
    bnd = recycling_boundaries(nb, x.device) if boundaries is None else boundaries
    ts = {"coords": coords, "single_row": single_row, "prev_pair": prev_pair, "msa_gamma": msa_gamma, "msa_beta": msa_beta,
          "pair_gamma": pair_gamma, "pair_beta": pair_beta, "table": table, "boundaries": bnd}
    ts = {k: _w32(v) for k, v in ts.items()}
    for k, v in ts.items():
        _require(v, torch.float32, k)
        if v.device != x.device:
            raise ValueError(f"{k} is on {v.device}, x on {x.device}")
    if ts["boundaries"].numel() < nb:
        raise ValueError(f"boundaries must hold {nb} values, got {ts['boundaries'].numel()}")
    c = ts["coords"].shape[-1]
    want = {"coords": (B, n, c), "single_row": (B, n, d), "prev_pair": (B, rows, n, d), "msa_gamma": (d,), "msa_beta": (d,),
            "pair_gamma": (d,), "pair_beta": (d,), "table": (nb, d)}
    for k, shape in want.items():
        if tuple(ts[k].shape) != shape:
            raise ValueError(f"{k} must be {shape}, got {tuple(ts[k].shape)}")
    args = (ts["coords"].data_ptr(), c, ts["single_row"].data_ptr(), ts["prev_pair"].data_ptr(), ts["msa_gamma"].data_ptr(),
            ts["msa_beta"].data_ptr(), ts["pair_gamma"].data_ptr(), ts["pair_beta"].data_ptr(), ts["table"].data_ptr(),
            ts["boundaries"].data_ptr(), nb, x.data_ptr(), m.data_ptr(), m.stride(0), B, n, d, float(eps))
    if row0 is None:
        _lib.check(_lib.load().af2_recycle_embed(*args, _stream_ptr()))
    else:
        _lib.check(_lib.load().af2_recycle_embed_rows(*args, row0, rows, _stream_ptr()))
    return x, m


# --------------------------------------------------------------------------------------------------
# building blocks exported for the parity tests
# --------------------------------------------------------------------------------------------------
def layernorm_bf16(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    _require(x, torch.float32, "x")
    d = x.shape[-1]
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _lib.check(_lib.load().af2_layernorm_bf16(x.data_ptr(), _f32(gamma).data_ptr(), _f32(beta).data_ptr(), y.data_ptr(),
                                              x.numel() // d, d, float(eps), _stream_ptr()))
    return y


def gemm_split(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Strict-mode building block: a [batch, M, K] x b [batch, N, K] fp32 -> [batch, M, N] fp32 through split-bf16 operands
    (three bf16 planes per operand, six tensor-core passes, fp32 accumulate)."""
    _require(a, torch.float32, "a")
    _require(b, torch.float32, "b")
    batch, M, K = a.shape
    N = b.shape[1]
    P = (K + 7) // 8 * 8
    lib = _lib.load()
    a_s = torch.empty(batch * M, SPLIT_PLANES, P, dtype=torch.bfloat16, device=a.device)
    b_s = torch.empty(batch * N, SPLIT_PLANES, P, dtype=torch.bfloat16, device=a.device)
    _lib.check(lib.af2_split_bf16(a.data_ptr(), a_s.data_ptr(), batch * M, K, _stream_ptr()))
    _lib.check(lib.af2_split_bf16(b.data_ptr(), b_s.data_ptr(), batch * N, K, _stream_ptr()))
    ldc = (N + 3) // 4 * 4
    c = torch.empty(batch, M, ldc, dtype=torch.float32, device=a.device)
    _lib.check(lib.af2_gemm_split_f32(a_s.data_ptr(), b_s.data_ptr(), c.data_ptr(), ldc, M, N, K, batch, _stream_ptr()))
    return c[:, :, :N]


def gemm_bf16(a: torch.Tensor, b: torch.Tensor, mn_major: bool = False) -> torch.Tensor:
    """a [batch, M, K] x b [batch, N, K] -> [batch, M, N]  (mn_major: a [batch, K, M], b [batch, K, N])."""
    _require(a, torch.bfloat16, "a")
    _require(b, torch.bfloat16, "b")
    if mn_major:
        batch, K, M = a.shape
        N = b.shape[2]
        lda, ldb = M, N
    else:
        batch, M, K = a.shape
        N = b.shape[1]
        lda, ldb = K, K
    ldc = (N + 3) // 4 * 4
    c = torch.empty(batch, M, ldc, dtype=torch.float32, device=a.device)
    _lib.check(_lib.load().af2_gemm_bf16_f32(a.data_ptr(), lda, a.shape[1] * a.shape[2], b.data_ptr(), ldb,
                                             b.shape[1] * b.shape[2], c.data_ptr(), ldc, M * ldc, M, N, K, batch,
                                             int(mn_major), _stream_ptr()))
    return c[:, :, :N]


# epilogue of af2_gemm_bf16_epilogue (include/af2b200.h)
EPI_STORE_BF16, EPI_GATED_BF16, EPI_RESID_F32, EPI_STORE_F32 = 0, 1, 2, 3
ACT_NONE, ACT_SIGMOID, ACT_GELU = 0, 1, 2
LAYOUT_TOKEN, LAYOUT_CHANNEL = 0, 1


def gemm_bf16_epilogue(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, bn: int, mode: int, act: int = ACT_NONE,
                       layout: int = LAYOUT_TOKEN, mn_major: bool = False, bias: Optional[torch.Tensor] = None,
                       rowscale: Optional[torch.Tensor] = None, resid: Optional[torch.Tensor] = None, ld_resid: int = 0,
                       ld_out: int, out_batch: int = 0, cm_inner: int = 0, cm_pitch: int = 0,
                       out_cols: int = 0) -> torch.Tensor:
    """a [batch, M, K] x b [batch, N, K] (mn_major: a [batch, K, M], b [batch, K, N]) through the GEMM epilogue `mode` / `act` /
    `layout` with an accumulator column tile of `bn`; the output is written into the flat buffer `out` (bf16 or fp32 by
    mode) with the pitches given (include/af2b200.h, af2_gemm_epilogue).  `resid` (mode EPI_RESID_F32) may be `out` itself.
    Returns `out`."""
    _require(a, torch.bfloat16, "a")
    _require(b, torch.bfloat16, "b")
    _require(out, torch.float32 if mode in (EPI_RESID_F32, EPI_STORE_F32) else torch.bfloat16, "out")
    if mn_major:
        batch, K, M = a.shape
        N = b.shape[2]
        lda, ldb = M, N
    else:
        batch, M, K = a.shape
        N = b.shape[1]
        lda, ldb = K, K
    for t, name in ((bias, "bias"), (rowscale, "rowscale"), (resid, "resid")):
        if t is not None:
            _require(t, torch.float32, name)
    e = _lib.GemmEpilogue(bn=bn, mode=mode, act=act, layout=layout, use_rowscale=int(rowscale is not None), bias=_ptr(bias),
                          rowscale=_ptr(rowscale), resid=_ptr(resid), ld_resid=ld_resid,
                          out=out.data_ptr(), ld_out=ld_out, out_batch=out_batch,
                          cm_inner=cm_inner, cm_pitch=cm_pitch, out_cols=out_cols)
    _lib.check(_lib.load().af2_gemm_bf16_epilogue(a.data_ptr(), lda, a.shape[1] * a.shape[2], b.data_ptr(), ldb,
                                                  b.shape[1] * b.shape[2], M, N, K, batch, int(mn_major), C.byref(e),
                                                  _stream_ptr()))
    return out


def attention_bf16(qkv: torch.Tensor, gate: torch.Tensor, n: int, nbatch: int, heads: int, dim_head: int, tok_sb: int,
                   tok_si: int, bias: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The attention kernel alone: qkv bf16 [tokens, 3 * heads * dim_head], gate bf16 [tokens, heads * dim_head] (sigmoid
    applied), bias bf16 [heads, n, align8(n)] in the log2 domain, mask bool [tokens]; token (b, i) = b * tok_sb + i * tok_si.
    Returns bf16 [tokens, heads * dim_head]."""
    _require(qkv, torch.bfloat16, "qkv")
    _require(gate, torch.bfloat16, "gate")
    I = heads * dim_head
    if qkv.dim() != 2 or qkv.shape[1] != 3 * I or tuple(gate.shape) != (qkv.shape[0], I):
        raise ValueError(f"qkv must be [tokens, {3 * I}] and gate [tokens, {I}]")
    if bias is not None:
        _require(bias, torch.bfloat16, "bias")
        if tuple(bias.shape) != (heads, n, (n + 7) // 8 * 8):
            raise ValueError(f"bias must have shape {(heads, n, (n + 7) // 8 * 8)}, got {tuple(bias.shape)}")
    mask = _mask_u8(mask, (qkv.shape[0],), "mask")
    out = torch.empty(qkv.shape[0], I, dtype=torch.bfloat16, device=qkv.device)
    _lib.check(_lib.load().af2_attention_bf16(qkv.data_ptr(), gate.data_ptr(), _ptr(bias), _ptr(mask), out.data_ptr(), n,
                                              nbatch, heads, dim_head, tok_sb, tok_si, _stream_ptr()))
    return out


def attention_proj_bf16(xn: torch.Tensor, w_qkv: torch.Tensor, w_gate: torch.Tensor, b_gate: Optional[torch.Tensor], n: int,
                        nbatch: int, heads: int, dim_head: int, tok_sb: int, tok_si: int, bias: Optional[torch.Tensor] = None,
                        mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """attention_bf16 with the projections inside the kernel: xn bf16 [tokens, d], w_qkv bf16 [3 * heads * dim_head, d],
    w_gate bf16 [heads * dim_head, d], b_gate fp32 [heads * dim_head] or None; bias and mask as attention_bf16.  Returns bf16
    [tokens, heads * dim_head]."""
    _require(xn, torch.bfloat16, "xn")
    _require(w_qkv, torch.bfloat16, "w_qkv")
    _require(w_gate, torch.bfloat16, "w_gate")
    I = heads * dim_head
    d = xn.shape[-1]
    if tuple(w_qkv.shape) != (3 * I, d) or tuple(w_gate.shape) != (I, d):
        raise ValueError(f"w_qkv must be [{3 * I}, {d}] and w_gate [{I}, {d}]")
    if b_gate is not None:
        _require(b_gate, torch.float32, "b_gate")
    if bias is not None:
        _require(bias, torch.bfloat16, "bias")
        if tuple(bias.shape) != (heads, n, (n + 7) // 8 * 8):
            raise ValueError(f"bias must have shape {(heads, n, (n + 7) // 8 * 8)}, got {tuple(bias.shape)}")
    T = xn.numel() // d
    mask = _mask_u8(mask, (T,), "mask")
    out = torch.empty(T, I, dtype=torch.bfloat16, device=xn.device)
    _lib.check(_lib.load().af2_attention_proj_bf16(xn.data_ptr(), d, w_qkv.data_ptr(), w_gate.data_ptr(), _ptr(b_gate), _ptr(bias),
                                                   _ptr(mask), out.data_ptr(), n, nbatch, heads, dim_head, tok_sb, tok_si,
                                                   _stream_ptr()))
    return out


def attention_proj_max_n(dim_head: int) -> int:
    """the longest sequence the fused projection + attention kernel keeps in shared memory (0: no kernel at this dim_head)"""
    return int(_lib.load().af2_attention_proj_max_n(dim_head))


def _addr(t: torch.Tensor, offset: int = 0) -> int:
    """device address of element `offset` of the flat buffer t"""
    return t.data_ptr() + offset * t.element_size()


def gemm_bf16_f32_strided(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, *, M: int, N: int, K: int, batch: int,
                          mn_major: bool, bn: int, lda: int, a_batch: int, ldb: int, b_batch: int, ldc: int, c_batch: int,
                          a_off: int = 0, b_off: int = 0, c_off: int = 0, a_pr: int = 0, a_piece: int = 0, b_pr: int = 0,
                          b_piece: int = 0) -> torch.Tensor:
    """af2_gemm_bf16_f32_gathered on flat buffers with explicit strides, as the contractions issue it: operand A (B) starts
    at element a_off (b_off) of a (b), C at element c_off of the fp32 buffer c.  a_pr / b_pr > 0 address the operand as
    gathered pieces a_piece / b_piece elements apart (include/af2b200.h).  Returns c."""
    _require(a, torch.bfloat16, "a")
    _require(b, torch.bfloat16, "b")
    _require(c, torch.float32, "c")
    _lib.check(_lib.load().af2_gemm_bf16_f32_gathered(_addr(a, a_off), lda, a_batch, _addr(b, b_off), ldb, b_batch,
                                                      _addr(c, c_off), ldc, c_batch, M, N, K, batch, int(mn_major), bn,
                                                      a_pr, a_piece, b_pr, b_piece, _stream_ptr()))
    return c


C2T_AUTO, C2T_SIMT, C2T_TILE, C2T_TMA = 0, 1, 2, 3


def _c2t_args(src, chan_stride, pitch, rows, n, d, mode, gamma, beta, gate, scale, scale_const, eps, y, src_off, gate_off, y_off):
    _require(src, torch.float32, "src")
    _require(y, torch.bfloat16, "y")
    if mode == 0:
        _require(gate, torch.bfloat16, "gate")
    for t, name in ((gamma, "gamma"), (beta, "beta"), (scale, "scale")):
        if t is not None:
            _require(t, torch.float32, name)
    return (_addr(src, src_off), chan_stride, pitch, rows, n, d, mode, _ptr(gamma), _ptr(beta),
            None if gate is None else _addr(gate, gate_off), _ptr(scale), float(scale_const), float(eps), _addr(y, y_off))


def chan_to_token(src: torch.Tensor, y: torch.Tensor, *, chan_stride: int, pitch: int, rows: int, n: int, d: int, mode: int,
                  gamma: Optional[torch.Tensor] = None, beta: Optional[torch.Tensor] = None,
                  gate: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None, scale_const: float = 1.0,
                  eps: float = 1e-5, variant: int = C2T_AUTO, src_off: int = 0, gate_off: int = 0, y_off: int = 0) -> int:
    """af2_chan_to_token on flat buffers (src fp32, gate / y bf16; *_off in elements): channel-major src -> token-major y,
    mode 0 LayerNorm over channels * gate, mode 1 * scale.  Returns the kernel variant that ran (C2T_*)."""
    ran = C.c_int(0)
    args = _c2t_args(src, chan_stride, pitch, rows, n, d, mode, gamma, beta, gate, scale, scale_const, eps, y, src_off,
                     gate_off, y_off)
    _lib.check(_lib.load().af2_chan_to_token(*args, variant, C.byref(ran), _stream_ptr()))
    return ran.value


CTAIL_AUTO, CTAIL_UNFUSED, CTAIL_FUSED = 0, 1, 2


def contract_tail(src: torch.Tensor, x: torch.Tensor, w_out: torch.Tensor, b_out: Optional[torch.Tensor], y: torch.Tensor, *,
                  chan_stride: int, pitch: int, rows: int, n: int, d: int, mode: int,
                  gamma: Optional[torch.Tensor] = None, beta: Optional[torch.Tensor] = None,
                  gate: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None, scale_const: float = 1.0,
                  eps: float = 1e-5, xn: Optional[torch.Tensor] = None, w_ogate: Optional[torch.Tensor] = None,
                  b_ogate: Optional[torch.Tensor] = None, variant: int = CTAIL_AUTO, src_off: int = 0, gate_off: int = 0,
                  x_off: int = 0) -> int:
    """af2_contract_tail: x[t] (fp32 [tokens][d] at x_off, in place) += tail(src)[t] w_out^T + b_out with the tail of
    chan_to_token (mode 0 LayerNorm over channels * gate, mode 1 * scale); with xn / w_ogate the gate is projected first,
    gate = sigmoid(xn w_ogate^T + b_ogate).  y: bf16 workspace of the unfused path.  Returns the path that ran
    (CTAIL_UNFUSED or CTAIL_FUSED)."""
    for t, name in ((x, "x"), (w_out, "w_out")):
        if not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"contract_tail: {name} must be a contiguous CUDA tensor")
    ran = C.c_int(0)
    args = _c2t_args(src, chan_stride, pitch, rows, n, d, mode, gamma, beta, gate, scale, scale_const, eps, y, src_off,
                     gate_off, 0)
    _lib.check(_lib.load().af2_contract_tail(*args[:13], _ptr(xn), _ptr(w_ogate), _ptr(b_ogate), w_out.data_ptr(),
                                             _ptr(b_out), _addr(x, x_off), args[13], variant, C.byref(ran), _stream_ptr()))
    return ran.value


def chan_to_token_select(src: torch.Tensor, y: torch.Tensor, *, chan_stride: int, pitch: int, rows: int, n: int, d: int,
                         mode: int, gamma: Optional[torch.Tensor] = None, beta: Optional[torch.Tensor] = None,
                         gate: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None, scale_const: float = 1.0,
                         eps: float = 1e-5, src_off: int = 0, gate_off: int = 0, y_off: int = 0) -> int:
    """the kernel variant chan_to_token(variant=C2T_AUTO) would run for these arguments; launches nothing"""
    args = _c2t_args(src, chan_stride, pitch, rows, n, d, mode, gamma, beta, gate, scale, scale_const, eps, y, src_off,
                     gate_off, y_off)
    v = _lib.load().af2_chan_to_token_select(*args)
    if v < 0:
        _lib.check(v)
    return v


OUTER_SCALE_AUTO, OUTER_SCALE_BYTES, OUTER_SCALE_BITS = 0, 1, 2


def outer_scale(mask: torch.Tensor, scale: torch.Tensor, *, row0: int, rows: int, eps: float, variant: int = OUTER_SCALE_AUTO,
                words: Optional[torch.Tensor] = None) -> int:
    """af2_outer_scale: scale fp32 [rows * N] (flat) <- 1 / (S (count_ij + eps)) for pair rows [row0, row0 + rows) of the bool
    mask [S, N]; words: uint32-sized workspace of ceil(S / 32) * N elements or None.  Returns the variant that ran."""
    S, N = mask.shape
    m = _mask_u8(mask, (S, N), "mask")
    _require(scale, torch.float32, "scale")
    if words is not None and words.numel() * words.element_size() < (S + 31) // 32 * N * 4:
        raise ValueError("outer_scale: words workspace too small")
    ran = C.c_int(0)
    _lib.check(_lib.load().af2_outer_scale(m.data_ptr(), scale.data_ptr(), _ptr(words), row0, rows, S, N, float(eps), variant,
                                           C.byref(ran), _stream_ptr()))
    return ran.value


# --------------------------------------------------------------------------------------------------
# template embedder (alphafold2.py:743-792, SURVEY.md 8f n3)
# --------------------------------------------------------------------------------------------------
def _pad_cols(w: torch.Tensor) -> torch.Tensor:
    """fp32 [rows, K] zero-padded to align8(K) columns: bf16 operand rows must be 16-byte multiples for TMA."""
    w = w.detach().float()
    r = (-w.shape[1]) % 8
    return w if r == 0 else torch.cat([w, torch.zeros(w.shape[0], r, dtype=w.dtype, device=w.device)], 1)


def pack_template_attention(wq, wkv, wg, bg, wo, bo, dim_head: int) -> Packed:
    """Attention(context=...) weights of the pointwise template attention; dim_head^-0.5 * log2(e) folded into to_q."""
    scale = dim_head ** -0.5 * 1.4426950408889634
    t = dict(wq=_bf16(wq.detach().float() * scale), wg=_bf16(wg), bg=_f32(bg), wkv=_bf16(wkv), wo=_bf16(wo), bo=_f32(bo))
    s = _lib.TemplateAttnWeights(*(t[k].data_ptr() for k in ("wq", "wg", "bg", "wkv", "wo", "bo")))
    return Packed(s, t)


def pack_template_attention_strict(wq, wkv, wg, bg, wo, bo, dim_head: int) -> Packed:
    wqg = torch.cat([wq.detach().float() * dim_head ** -0.5, wg.detach().float()], 0)
    bqg = torch.cat([torch.zeros(wq.shape[0], device=wq.device), bg.detach().float()], 0)
    t = dict(wqg=split_weight(wqg), bqg=_f32(bqg), wkv=split_weight(wkv), wo=split_weight(wo), bo=_f32(bo))
    s = _lib.TemplateAttnWeightsStrict(*(t[k].data_ptr() for k in ("wqg", "bqg", "wkv", "wo", "bo")))
    return Packed(s, t, "strict")


def pack_linear(w, b, strict: bool = False) -> Packed:
    """nn.Linear for af2_template_embed: bf16 [out, align8(in)] (zero pad columns), or split-bf16 in strict mode."""
    t = dict(w=split_weight(w) if strict else _bf16(_pad_cols(w)), b=_f32(b))
    pk = Packed(None, t, "strict" if strict else "bf16")
    pk.k_in = int(w.shape[1])
    return pk


def pack_template_angles(w1, b1, w2, b2, strict: bool = False) -> Packed:
    """template_angle_mlp = Linear(K, d) -> GELU -> Linear(d, d); K zero-padded to a multiple of 8."""
    if strict:
        t = dict(w1=split_weight(w1), b1=_f32(b1), w2=split_weight(w2), b2=_f32(b2))
    else:
        t = dict(w1=_bf16(_pad_cols(w1)), b1=_f32(b1), w2=_bf16(w2), b2=_f32(b2))
    cls = _lib.TemplateAngleWeightsStrict if strict else _lib.TemplateAngleWeights
    pk = Packed(cls(*(t[k].data_ptr() for k in ("w1", "b1", "w2", "b2"))), t, "strict" if strict else "bf16")
    pk.k_in = int(w1.shape[1])
    return pk


def template_embed(pk: Packed, feats: torch.Tensor) -> torch.Tensor:
    """to_template_embed (alphafold2.py:751): feats [..., K] fp32 -> t [..., d] fp32."""
    _require(feats, torch.float32, "templates_feats")
    K = feats.shape[-1]
    if K != pk.k_in:
        raise ValueError(f"templates_feats has {K} features, to_template_embed expects {pk.k_in}")
    d = pk.tensors["w"].shape[0]
    rows = feats.numel() // K
    t = torch.empty(*feats.shape[:-1], d, dtype=torch.float32, device=feats.device)
    lib = _lib.load()
    if pk.kind == "strict":
        ws = workspace(lib.af2_template_embed_strict_workspace(rows, K), feats.device)
        fn = lib.af2_template_embed_strict
    else:
        ws = workspace(lib.af2_template_embed_workspace(rows, K), feats.device)
        fn = lib.af2_template_embed
    _lib.check(fn(pk.tensors["w"].data_ptr(), pk.tensors["b"].data_ptr(), feats.data_ptr(), t.data_ptr(), rows, K, d, ws.data_ptr(),
                  ws.numel(), _stream_ptr()))
    return t


def template_pointwise_attention_(pk: Packed, x: torch.Tensor, t: torch.Tensor, x_mask: Optional[torch.Tensor],
                                  t_mask: Optional[torch.Tensor], heads: int, dim_head: int) -> torch.Tensor:
    """x [B, n, n, d] fp32 <- x + pooled * Attention(x, context=t, mask=x_mask, context_mask=t_mask) at every pair position
    (alphafold2.py:764-785).  t [B * T, n, n, d] fp32 (template-major: row b * T + t), t_mask [B * T, n, n] (the crossed
    template mask), x_mask [B, n, n] or None; pooled = any template valid at the pair."""
    _require(x, torch.float32, "x")
    _require(t, torch.float32, "t")
    if x.dim() != 4 or x.shape[1] != x.shape[2]:
        raise ValueError(f"x must be [B, n, n, d], got {tuple(x.shape)}")
    B, n, _, d = x.shape
    if t.dim() != 4 or B == 0 or t.shape[0] % B or tuple(t.shape[1:]) != (n, n, d):
        raise ValueError(f"t must be [B * T, {n}, {n}, {d}], got {tuple(t.shape)}")
    T = t.shape[0] // B
    xm = _mask_u8(x_mask, (B, n, n), "x_mask")
    tm = _mask_u8(t_mask, (B * T, n, n), "t_mask")
    lib = _lib.load()
    if pk.kind == "strict":
        ws = workspace(lib.af2_template_pointwise_attention_strict_workspace(B, T, n, d, heads, dim_head), x.device)
        fn = lib.af2_template_pointwise_attention_strict
    else:
        ws = workspace(lib.af2_template_pointwise_attention_workspace(B, T, n, d, heads, dim_head), x.device)
        fn = lib.af2_template_pointwise_attention
    _lib.check(fn(C.byref(pk.struct), x.data_ptr(), t.data_ptr(), _ptr(xm), _ptr(tm), B, T, n, d, heads, dim_head, ws.data_ptr(),
                  ws.numel(), _stream_ptr()))
    return x


def attention_forward(pk: Packed, x: torch.Tensor, heads: int, dim_head: int, mask: Optional[torch.Tensor] = None,
                      attn_bias: Optional[torch.Tensor] = None, context: Optional[torch.Tensor] = None,
                      context_mask: Optional[torch.Tensor] = None, tie_dim: Optional[int] = None) -> torch.Tensor:
    """Attention.forward (alphafold2.py:125-190) with the packed weights of pack_template_attention{,_strict}: x [B, i, d],
    context [B, j, d] or None (self-attention), mask [B, i] and context_mask [B, j] bool or None, attn_bias any float tensor
    that broadcasts to [B, heads, i, j], tie_dim r (queries averaged over groups of r batch elements) or None.  Masking
    happens only when mask is given.  Returns fp32 [B, i, d].  Every shape rule is checked before anything runs on the
    device (ValueError)."""
    if not torch.is_tensor(x) or x.dim() != 3 or not x.is_floating_point():
        raise ValueError(f"x must be a float tensor [B, i, d], got {tuple(x.shape) if torch.is_tensor(x) else type(x)}")
    B, i, d = x.shape
    j = i
    if context is not None:
        if not torch.is_tensor(context) or context.dim() != 3 or not context.is_floating_point() or context.shape[0] != B \
                or context.shape[2] != d or context.device != x.device:
            raise ValueError(f"context must be a float tensor [{B}, j, {d}] on {x.device}, got {tuple(context.shape)}")
        j = context.shape[1]
    if tie_dim is not None and (int(tie_dim) != tie_dim or tie_dim < 1 or B % tie_dim):
        raise ValueError(f"tie_dim {tie_dim} must be a positive divisor of the batch {B}")
    for name, m, n in (("mask", mask, i), ("context_mask", context_mask, j)):
        if m is not None and (not torch.is_tensor(m) or tuple(m.shape) != (B, n) or m.device != x.device):
            raise ValueError(f"{name} must be [{B}, {n}] on {x.device}, got {tuple(m.shape) if torch.is_tensor(m) else type(m)}")
    strides, bias_batch = (0, 0, 0, 0), 0
    if attn_bias is not None:
        if not torch.is_tensor(attn_bias) or not attn_bias.is_floating_point() or attn_bias.device != x.device:
            raise ValueError(f"attn_bias must be a float tensor on {x.device}")
        try:
            ok = torch.broadcast_shapes(attn_bias.shape, (B, heads, i, j)) == (B, heads, i, j)
        except RuntimeError:
            ok = False
        if not ok:
            raise ValueError(f"attn_bias of shape {tuple(attn_bias.shape)} does not broadcast to {(B, heads, i, j)}")
        # one bias slab per batch element, or one for all of them (batch stride 0)
        bias_batch = B if attn_bias.dim() == 4 and attn_bias.shape[0] == B and B > 1 else 1
    strict = pk.kind == "strict"
    lib = _lib.load()
    wsfn = lib.af2_attention_forward_strict_workspace if strict else lib.af2_attention_forward_workspace
    tie = int(tie_dim) if tie_dim is not None else 0
    # the workspace query checks every shape rule of the C entry point (negative: refused, nothing launched)
    nbytes = wsfn(B, i, j, d, heads, dim_head, tie, bias_batch)
    if nbytes < 0:
        _lib.check(int(nbytes))
    if not x.is_cuda:
        raise RuntimeError("x must be a CUDA tensor (alphafold2_b200 has no CPU fallback)")
    xf = x.detach().to(torch.float32).contiguous()
    _require(xf, torch.float32, "x")
    cf = None if context is None else context.detach().to(torch.float32).contiguous()
    bias = None
    if attn_bias is not None:
        bias = attn_bias.detach().to(torch.float32).expand(B, heads, i, j)
        strides = (bias.stride(0) if bias_batch > 1 else 0,) + tuple(bias.stride()[1:])
    xm = _mask_u8(mask, (B, i), "mask")
    cm = _mask_u8(context_mask, (B, j), "context_mask")
    out = torch.empty(B, i, d, dtype=torch.float32, device=x.device)
    ws = workspace(nbytes, x.device)
    fn = lib.af2_attention_forward_strict if strict else lib.af2_attention_forward
    _lib.check(fn(C.byref(pk.struct), xf.data_ptr(), _ptr(cf), _ptr(xm), _ptr(cm), _ptr(bias), *strides, B, i, j, d, heads, dim_head, tie,
                  out.data_ptr(), ws.data_ptr(), ws.numel(), _stream_ptr()))
    return out


class TemplateAttentionGroups:
    """template_pointwise_attention_ over the templates one group at a time (af2_template_pointwise_begin / _group / _end):
        g = TemplateAttentionGroups(pk, x, x_mask, heads, dim_head, band=None)
        g.add(t, t_mask, last=False) ...; g.add(t, t_mask, last=True)     # t [B * G, R, C, d], t_mask [B * G, R, C] per group
    x [B, R, C, d] is R rows of C pairs per batch element (the pair tensor, or a rank's rows of it).  Adds to x exactly what
    one template_pointwise_attention_ over the concatenated groups adds (bitwise).  Between the calls it holds the fp32
    online-softmax state of every pair; a group's t may be freed as soon as its add() returns.
      band None or >= R: one window of all B * R * C pairs.  q and gate of x are made here, each add() is one group step and
        the last one adds to_out to x.
      band < R (bf16 only): each add() runs, per batch element and band of `band` pair rows, q and gate of the band's rows of
        x, the group step on those rows and, on the last add(), to_out into them, so q, gate and k|v exist for one band at a
        time.  x changes only in the last add(), band by band, after the band's own q and gate are made."""

    def __init__(self, pk: Packed, x: torch.Tensor, x_mask: Optional[torch.Tensor], heads: int, dim_head: int,
                 band: Optional[int] = None):
        _require(x, torch.float32, "x")
        if x.dim() != 4:
            raise ValueError(f"x must be [B, R, C, d], got {tuple(x.shape)}")
        B, R, Cn, d = x.shape
        self.strict = pk.kind == "strict"
        if band is not None and int(band) < R:
            if self.strict:
                raise NotImplementedError("the pointwise template attention runs in bands of pair rows in bf16 mode only")
            if int(band) <= 0 or int(band) % 8:
                raise ValueError(f"template band {band} must be a positive multiple of 8")
        self.pk, self.x, self.heads, self.dim_head = pk, x, heads, dim_head
        self.band = R if band is None else min(int(band), R)
        self.xm = _mask_u8(x_mask, (B, R, Cn), "x_mask")
        self.first, self.done = True, False
        P, I, dev = B * R * Cn, heads * dim_head, x.device
        W = P if self.band == R else self.band * Cn              # pairs of one window
        self.run_max = torch.empty(P, heads, dtype=torch.float32, device=dev)
        self.run_sum = torch.empty(P, heads, dtype=torch.float32, device=dev)
        self.acc = torch.empty(P, I, dtype=torch.float32, device=dev)
        self.pooled = torch.empty(P, dtype=torch.float32, device=dev)
        # the last group writes the gated output of a window from the start of q (one window's rows), or of the accumulator in
        # strict mode, which runs as one window
        if self.strict:
            qg = torch.empty(W, 2 * I, dtype=torch.float32, device=dev)
            self.qgate, self.out = (qg,), self.acc
        else:
            q = torch.empty(W, I, dtype=torch.bfloat16, device=dev)
            self.qgate, self.out = (q, torch.empty(W, I, dtype=torch.bfloat16, device=dev)), q
        lib, sfx = _lib.load(), "_strict" if self.strict else ""
        self.fn = {s: getattr(lib, f"af2_template_pointwise_{s}{sfx}") for s in ("begin", "group", "end")}
        self.ws_fn = {s: getattr(lib, f"af2_template_pointwise_{s}{sfx}_workspace") for s in ("begin", "group", "end")}
        self.w, self.qgate_ptrs = C.byref(pk.struct), [v.data_ptr() for v in self.qgate]
        if self.band == R:
            self._begin(_stream_ptr(), workspace(self.ws_fn["begin"](P, d), dev), 0, P)

    def _begin(self, s, ws, o, P):
        d = self.x.shape[3]
        _lib.check(self.fn["begin"](self.w, _addr(self.x, o * d), P, d, self.heads, self.dim_head, *self.qgate_ptrs, ws.data_ptr(),
                                    ws.numel(), s))

    def _group(self, s, ws, t, tm, o, ot, B, G, pairs, t_stride, last):
        d, h, I = self.x.shape[3], self.heads, self.heads * self.dim_head
        _lib.check(self.fn["group"](
            self.w, _addr(t, ot * d), None if self.xm is None else _addr(self.xm, o), None if tm is None else _addr(tm, ot), B, G,
            pairs, t_stride, d, h, self.dim_head, *self.qgate_ptrs, _addr(self.run_max, o * h), _addr(self.run_sum, o * h),
            _addr(self.acc, o * I), _addr(self.pooled, o), self.out.data_ptr(), int(self.first), int(last), ws.data_ptr(),
            ws.numel(), s))

    def _end(self, s, ws, o, P):
        d = self.x.shape[3]
        _lib.check(self.fn["end"](self.w, _addr(self.x, o * d), self.out.data_ptr(), _addr(self.pooled, o), P, d, self.heads,
                                  self.dim_head, ws.data_ptr(), ws.numel(), s))

    def add(self, t: torch.Tensor, t_mask: Optional[torch.Tensor], last: bool) -> None:
        """One group of templates; on the last one (last=True) x gets the attention output."""
        if self.done:
            raise RuntimeError("TemplateAttentionGroups: the last group has already been added")
        _require(t, torch.float32, "t")
        B, R, Cn, d = self.x.shape
        if t.dim() != 4 or t.shape[0] % B or t.shape[0] == 0 or tuple(t.shape[1:]) != (R, Cn, d):
            raise ValueError(f"t must be [B * G, {R}, {Cn}, {d}], got {tuple(t.shape)}")
        G = t.shape[0] // B
        tm = _mask_u8(t_mask, (B * G, R, Cn), "t_mask")
        h, dh, RC, s = self.heads, self.dim_head, R * Cn, _stream_ptr()
        if self.band == R:
            self._group(s, workspace(self.ws_fn["group"](B, G, RC, RC, d, h, dh), t.device), t, tm, 0, 0, B, G, RC, RC, last)
            if last:
                self._end(s, workspace(self.ws_fn["end"](B * RC, h, dh), t.device), 0, B * RC)
        else:
            W = self.band * Cn
            ws = workspace(max(self.ws_fn["begin"](W, d), self.ws_fn["group"](1, G, W, RC, d, h, dh), self.ws_fn["end"](W, h, dh)),
                           t.device)
            for b in range(B):
                for i0 in range(0, R, self.band):
                    P, o = (min(i0 + self.band, R) - i0) * Cn, b * RC + i0 * Cn
                    self._begin(s, ws, o, P)
                    self._group(s, ws, t, tm, o, b * G * RC + i0 * Cn, 1, G, P, RC, last)
                    if last:
                        self._end(s, ws, o, P)
        self.first = False
        self.done = last


def _ws_alloc(nbytes: int) -> int:
    return int(nbytes * 1.05) + 4096                # what workspace() allocates for a request of nbytes


def template_branch_bytes(b: int, T: int, G: int, n: int, d: int, heads: int, dim_head: int, precision: str,
                          templates_dim: int = 32, band: Optional[int] = None) -> int:
    """Device bytes the template branch (Alphafold2.embed_templates_) allocates beyond x and its own inputs when it runs the T
    templates in groups of G: the grow-only workspace sized for the largest call (to_template_embed, the pair-stack modules at
    batch b * G, the pointwise attention), plus what lives beside it: t and the crossed mask of one group and, with more than
    one group, that group's copy of templates_feats, q and gate of x and the fp32 softmax state.  Computed from the library's
    workspace queries: no GPU needed.

    band < n (bf16 only): the branch in bands of `band` pair rows (TemplateAttentionGroups with band, the pair stack in the
    same bands):
    the fp32 softmax state of every pair, one group's t, crossed mask and templates_feats copy, one band's q and gate, plus
    the larger of the banded pair block (pair_block_bytes with S = 0) and one band's begin / group / end workspace."""
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")
    lib = _lib.load()
    strict = precision == "strict"
    sfx = "_strict" if strict else ""
    begin, group, end = (getattr(lib, f"af2_template_pointwise_{step}{sfx}_workspace") for step in ("begin", "group", "end"))
    G = max(1, min(G, T))
    bg, P, I, nn = b * G, b * n * n, heads * dim_head, n * n
    rows = bg * n * n
    if band is not None and band < n:
        if strict:
            raise ValueError("strict mode runs the template branch whole: no band")
        W = band * n
        ws = [lib.af2_template_embed_workspace(rows, templates_dim), begin(W, d), group(1, G, W, nn, d, heads, dim_head),
              end(W, heads, dim_head)]
        persist = rows * d * 4 + rows + rows * templates_dim * 4               # t, crossed mask, templates_feats copy
        persist += P * (2 * heads + I + 1) * 4 + W * 2 * I * 2                 # whole-tensor state, one band's q | gate
        # the workspace is grow-only: a band's window workspace larger than the pair block's stays beside the block's operands
        pair_ws, keep = _pair_block_parts(bg, n, 0, d, heads, dim_head, band)
        return _ws_alloc(max(pair_ws, *ws)) + keep + persist
    ax = lib.af2_axial_attention_strict_workspace if strict else lib.af2_axial_attention_workspace
    ws = [getattr(lib, f"af2_template_embed{sfx}_workspace")(rows, templates_dim),
          getattr(lib, f"af2_triangle_multiply{sfx}_workspace")(bg, n, d),
          ax(bg, n, n, d, heads, dim_head, 1), ax(bg, n, n, d, heads, dim_head, 0)]
    persist = rows * d * 4 + rows                                          # t, crossed mask
    if G == T:
        ws.append(getattr(lib, f"af2_template_pointwise_attention{sfx}_workspace")(b, T, n, d, heads, dim_head))
    else:
        ws += [begin(P, d), group(b, G, nn, nn, d, heads, dim_head), end(P, heads, dim_head)]
        persist += rows * templates_dim * 4                                # the group's contiguous templates_feats
        persist += P * 2 * I * (4 if strict else 2)                        # q | gate
        persist += P * (2 * heads + I + 1) * 4                             # run_max, run_sum, acc, pooled
    return _ws_alloc(max(ws)) + persist


def plan_template_groups(b: int, T: int, n: int, d: int, heads: int, dim_head: int, precision: str, budget: int,
                         templates_dim: int = 32) -> int:
    """How many templates the template branch runs at a time: T whenever template_branch_bytes fits `budget` (bytes), else the
    largest G that fits (the last group may be smaller), and 1 when nothing fits (the allocation then fails as it would)."""
    if T <= 1 or template_branch_bytes(b, T, T, n, d, heads, dim_head, precision, templates_dim) <= budget:
        return max(T, 1)
    for G in range(T - 1, 1, -1):
        if template_branch_bytes(b, T, G, n, d, heads, dim_head, precision, templates_dim) <= budget:
            return G
    return 1


def plan_template_branch(b: int, T: int, n: int, d: int, heads: int, dim_head: int, precision: str, budget: int,
                         templates_dim: int = 32):
    """(G, band) of the template branch: plan_template_groups' G and band = n (the whole-tensor calls) whenever some G fits
    `budget` (bytes), and always in strict mode (whole-tensor only); else G = 1 and the largest multiple of PAIR_BAND_ALIGN
    pair rows below n that fits (template_branch_bytes with band).  Raises MemoryError when not even one band of
    PAIR_BAND_ALIGN rows fits, before any device work."""
    G = plan_template_groups(b, T, n, d, heads, dim_head, precision, budget, templates_dim)
    if precision == "strict" or template_branch_bytes(b, T, G, n, d, heads, dim_head, precision, templates_dim) <= budget:
        return G, n
    R = (n - 1) // PAIR_BAND_ALIGN * PAIR_BAND_ALIGN
    while R >= PAIR_BAND_ALIGN:
        if template_branch_bytes(b, T, 1, n, d, heads, dim_head, precision, templates_dim, band=R) <= budget:
            return 1, R
        R -= PAIR_BAND_ALIGN
    least = template_branch_bytes(b, T, 1, n, d, heads, dim_head, precision, templates_dim,
                                  band=PAIR_BAND_ALIGN if n > PAIR_BAND_ALIGN else None)
    raise MemoryError(f"the template branch at N_res {n} (batch {b}, {T} templates, dim {d}) needs {least / 2**30:.2f} GiB beyond x "
                      f"and its inputs even one template at a time in bands of {PAIR_BAND_ALIGN} pair rows; "
                      f"{budget / 2**30:.2f} GiB can be allocated")


def template_reuse_fits(b: int, T: int, n: int, d: int, heads: int, dim_head: int, stack_rows, budget: int) -> bool:
    """Whether a recycling loop may keep the template pair stack's output t [b * T, n, n, d] fp32 and its crossed mask
    [b * T, n, n] bool across its iterations: they must fit `budget` (bytes) beside the whole-tensor plan of every pair stack
    that runs after the templates, one per entry of stack_rows (its MSA rows: the trunk's, and the extra-MSA stack's when
    there is one), so that keeping t moves none of them into bands.  That is a matter of correctness as well as speed: the
    extra-MSA stack's tied-query column attention cannot run in pair bands at all."""
    t_bytes = b * T * n * n * (d * 4 + 1)
    return all(t_bytes + pair_block_bytes(b, n, S, d, heads, dim_head, n) <= budget for S in stack_rows)


PAIR_BAND_ALIGN = 256      # band boundaries: every band call then picks the whole-tensor call's GEMM tile and chan_to_token kernel


def _align8(n: int) -> int:
    return (n + 7) // 8 * 8


@functools.lru_cache(maxsize=256)
def pair_block_bytes(B: int, N: int, S: int, d: int, heads: int, dim_head: int, R: int) -> int:
    """Device bytes one Evoformer block (bf16 path) allocates beyond x [B, N, N, d] and m [B, S, N, d] when its pair track runs
    in bands of R pair rows (EvoformerBlock.update_; S = 0: a pair block without the MSA track, as in the template stack).
    R >= N is today's whole-tensor schedule: the grow-only workspace sized for its largest call.  R < N: the workspace sized
    for the MSA track and one band's calls, plus the largest set of operands one pair stage keeps for the whole tensor
    (triangle multiply: L, R and gate of all rows; column attention: the pair bias and one column band's copy of x and of
    the mask; outer mean: the projected m and one band's left operand).  Computed from the library's workspace queries."""
    ws, keep = _pair_block_parts(B, N, S, d, heads, dim_head, R)
    return _ws_alloc(ws) + keep


@functools.lru_cache(maxsize=256)
def _pair_block_parts(B: int, N: int, S: int, d: int, heads: int, dim_head: int, R: int):
    """pair_block_bytes in its two parts: (largest workspace request, bytes of the operands kept beside the workspace)."""
    lib = _lib.load()
    ax = lib.af2_axial_attention_workspace
    ff = lambda tokens: lib.af2_feed_forward_workspace(tokens, d, 4 * d)  # noqa: E731
    ws = [ax(B, S, N, d, heads, dim_head, 1), ax(B, S, N, d, heads, dim_head, 0), ff(B * S * N)] if S > 0 else []
    if R >= N:
        if S > 0:
            ws.append(lib.af2_outer_mean_workspace(B, S, N, d))
        ws += [lib.af2_triangle_multiply_workspace(B, N, d), ax(B, N, N, d, heads, dim_head, 1), ax(B, N, N, d, heads, dim_head, 0),
               ff(B * N * N)]
        return max(ws), 0
    np8 = _align8(N)
    ws += [lib.af2_triangle_project_workspace(R * N, d), lib.af2_triangle_contract_workspace(R, N, d),
           ax(1, R, N, d, heads, dim_head, 1), ax(1, N, R, d, heads, dim_head, 0), ff(R * N)]
    keep = [2 * d * N * np8 * 2 + N * N * d * 2,                               # triangle multiply: L, R, gate
            heads * N * np8 * 2 + N * R * (d * 4 + 1)]                         # column attention: bias, band of x and mask
    if S > 0:
        ws += [lib.af2_outer_project_workspace(S * N, d), lib.af2_outer_contract_workspace(R, N, d)]
        keep.append(2 * d * S * np8 * 2 + d * S * _align8(R) * 2)             # outer mean: projected m, band's left operand
    return max(ws), max(keep)


def plan_pair_band(B: int, N: int, S: int, d: int, heads: int, dim_head: int, budget: int) -> int:
    """Pair rows per band of one Evoformer block: N (today's whole-tensor calls) whenever pair_block_bytes(..., N) fits `budget`
    (bytes), else the largest multiple of PAIR_BAND_ALIGN below N that fits.  Raises MemoryError when not even one band of
    PAIR_BAND_ALIGN rows fits."""
    if pair_block_bytes(B, N, S, d, heads, dim_head, N) <= budget:
        return N
    R = (N - 1) // PAIR_BAND_ALIGN * PAIR_BAND_ALIGN
    while R >= PAIR_BAND_ALIGN:
        if pair_block_bytes(B, N, S, d, heads, dim_head, R) <= budget:
            return R
        R -= PAIR_BAND_ALIGN
    least = pair_block_bytes(B, N, S, d, heads, dim_head, min(PAIR_BAND_ALIGN, N))
    raise MemoryError(f"one Evoformer block at N_res {N} (batch {B}, {S} MSA rows, dim {d}) needs {least / 2**30:.2f} GiB beyond "
                      f"x and m even in bands of {PAIR_BAND_ALIGN} pair rows; {budget / 2**30:.2f} GiB can be allocated")


MSA_BAND_ALIGN = 64       # the planner's MSA bands: multiples of 64 rows (any band gives the same bits; this bounds the search)


@functools.lru_cache(maxsize=4096)
def msa_block_bytes(B: int, N: int, S: int, d: int, heads: int, dim_head: int, R: int, RS: int) -> int:
    """Device bytes one Evoformer block (bf16 path) allocates beyond x and m with the pair track in bands of R pair rows and the
    MSA track in bands of RS MSA rows (banded.msa_track_, one batch element at a time).  RS >= S is pair_block_bytes(..., R).
    RS < S: the workspace sized for the largest of one MSA row band's attention and transition, one column band's attention
    (banded.msa_column_band columns), one projection chunk, the outer contraction (R rows, or N when the pair rows are whole) and
    the pair track's calls at R (whole at batch B when R >= N); beside it the largest set of operands kept at one time: the
    row attention's pair bias, one column band's copy of m and of its mask, the whole projected m (LR) and one band's left
    operand, or the pair track's operands at R."""
    if RS >= S:
        return pair_block_bytes(B, N, S, d, heads, dim_head, R)
    from .banded import msa_column_band
    lib = _lib.load()
    ax = lib.af2_axial_attention_workspace
    np8 = _align8(N)
    Cb = msa_column_band(S, N, RS)
    pair_ws, pair_keep = _pair_block_parts(B, N, 0, d, heads, dim_head, R)
    ws = [pair_ws, ax(1, RS, N, d, heads, dim_head, 1), ax(1, S, Cb, d, heads, dim_head, 0),
          lib.af2_feed_forward_workspace(RS * N, d, 4 * d), lib.af2_outer_project_workspace(RS * N, d),
          lib.af2_outer_contract_workspace(min(R, N), N, d)]
    keep = [pair_keep,
            heads * N * np8 * 2,                                                  # row attention: the pair bias of x
            _pt_round(S * Cb * d * 4) + _pt_round(S * Cb),                        # column attention: band of m and mask
            _pt_round(2 * d * S * np8 * 2) + (_pt_round(d * S * _align8(R) * 2) if R < N else 0)]   # outer mean: LR, left window
    return _pt_round(_ws_alloc(max(ws))) + max(keep)


def _pt_round(nbytes: int) -> int:
    """What PyTorch's caching allocator takes for a large request: a multiple of 2 MiB (at these sizes the rounding is no
    longer lost in the planner's other margins)."""
    return (nbytes + (1 << 21) - 1) >> 21 << 21


def plan_block_bands(B: int, N: int, S: int, d: int, heads: int, dim_head: int, budget: int):
    """(R, RS): pair rows and MSA rows per band of one Evoformer block.  (plan_pair_band(...), S) whenever that fits `budget`
    (bytes), so every shape that runs with the MSA track whole keeps its plan.  Otherwise the largest R (N, or a multiple of
    PAIR_BAND_ALIGN) for which some RS fits, then the largest RS (a multiple of MSA_BAND_ALIGN below S) that fits with it: pair
    bands copy and cost time, MSA row bands do not.  Raises MemoryError, before any device work, when not even
    R = PAIR_BAND_ALIGN with RS = MSA_BAND_ALIGN fits."""
    try:
        return plan_pair_band(B, N, S, d, heads, dim_head, budget), S
    except MemoryError:
        pass
    least = min(PAIR_BAND_ALIGN, N)
    if S > MSA_BAND_ALIGN:
        fits = lambda R, RS: msa_block_bytes(B, N, S, d, heads, dim_head, R, RS) <= budget  # noqa: E731
        for R in [N] + list(range((N - 1) // PAIR_BAND_ALIGN * PAIR_BAND_ALIGN, PAIR_BAND_ALIGN - 1, -PAIR_BAND_ALIGN)):
            if fits(R, MSA_BAND_ALIGN):
                RS = (S - 1) // MSA_BAND_ALIGN * MSA_BAND_ALIGN
                while not fits(R, RS):
                    RS -= MSA_BAND_ALIGN
                return R, RS
        need = msa_block_bytes(B, N, S, d, heads, dim_head, least, MSA_BAND_ALIGN)
    else:
        need = pair_block_bytes(B, N, S, d, heads, dim_head, least)
    raise MemoryError(f"one Evoformer block at N_res {N} (batch {B}, {S} MSA rows, dim {d}) needs {need / 2**30:.2f} GiB beyond "
                      f"x and m even in bands of {least} pair rows and {min(MSA_BAND_ALIGN, S)} MSA rows; "
                      f"{budget / 2**30:.2f} GiB can be allocated")


def workspace_holds(device, nbytes: int) -> bool:
    """Whether the current grow-only workspace of `device` is already at least `nbytes` (a call needing no more allocates
    nothing)."""
    store = _WORKSPACE if _WS_PRIVATE is None else _WS_PRIVATE[0]
    ws = store.get(torch.device(device))
    return ws is not None and ws.numel() >= nbytes


def release_workspace(device) -> None:
    """Drop the grow-only workspace of `device` and return its memory to the driver, so that tensors which outlive single ops
    can use it; the next op allocates a workspace of the size it needs.  device_budget counts the workspace as available,
    which holds only once it is released (a workspace left at the trunk's whole-tensor size by an earlier forward would
    otherwise stay beside them).  A no-op inside a locked private_workspace scope.  A buffer that a CUDA-graph capture used
    stays allocated (workspace); while the current stream is capturing, nothing is returned to the driver."""
    store, locked = (_WORKSPACE, False) if _WS_PRIVATE is None else _WS_PRIVATE
    if not locked and store.pop(torch.device(device), None) is not None and not torch.cuda.is_current_stream_capturing():
        torch.cuda.empty_cache()


def device_budget(device) -> int:
    """Bytes the template branch or a pair block can still allocate on `device`: what the driver reports free, plus what
    PyTorch's caching allocator holds unused, plus the current grow-only workspace (which every op reuses)."""
    device = torch.device(device)
    free, _ = torch.cuda.mem_get_info(device)
    cached = torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)
    store = _WORKSPACE if _WS_PRIVATE is None else _WS_PRIVATE[0]
    ws = store.get(device)
    return int(free + cached + (ws.numel() if ws is not None else 0))


def template_angle_features(pk: Packed, angles: torch.Tensor, m: torch.Tensor, row0: int) -> torch.Tensor:
    """template_angle_mlp (alphafold2.py:789-790): angles [B, T, n, K] fp32 -> rows row0 .. row0 + T - 1 of m [B, R, n, d] fp32
    (the reference concatenates them after the S MSA rows: row0 = S).  Returns m."""
    _require(angles, torch.float32, "templates_angles")
    _require(m, torch.float32, "m")
    B, T, n, K = angles.shape
    if K != pk.k_in:
        raise ValueError(f"templates_angles has {K} features, template_angle_mlp expects {pk.k_in}")
    if m.dim() != 4 or m.shape[0] != B or m.shape[2] != n:
        raise ValueError(f"m must be [{B}, rows, {n}, d], got {tuple(m.shape)}")
    d, R = m.shape[3], m.shape[1]
    lib = _lib.load()
    if pk.kind == "strict":
        ws = workspace(lib.af2_template_angles_strict_workspace(B, T, n, K, d), m.device)
        fn = lib.af2_template_angles_strict
    else:
        ws = workspace(lib.af2_template_angles_workspace(B, T, n, K, d), m.device)
        fn = lib.af2_template_angles
    _lib.check(fn(C.byref(pk.struct), angles.data_ptr(), m.data_ptr(), B, T, n, K, d, R, int(row0), ws.data_ptr(), ws.numel(),
                  _stream_ptr()))
    return m


def template_pointwise(q: torch.Tensor, gate: torch.Tensor, kv: torch.Tensor, B: int, T: int, heads: int, dim_head: int,
                       x_mask: Optional[torch.Tensor] = None, t_mask: Optional[torch.Tensor] = None,
                       out: Optional[torch.Tensor] = None, pooled: Optional[torch.Tensor] = None):
    """The pointwise template-attention kernel alone, one launch over all T templates (include/af2b200.h,
    af2_template_pointwise_bf16_state / _f32_state with first = last = 1 and no state): q, gate [P, I],
    kv [B * T * pairs, 2I] with P = B * pairs; bf16 operands (q in the log2 domain, gate after the sigmoid) or fp32 operands
    (the strict instantiation: natural-log domain, gate logits).  x_mask bool [P], t_mask bool [B * T * pairs].
    out / pooled: caller-given output buffers (flat views of at least P * I / P elements) or None.
    Returns (out [P, I] in the operand dtype, pooled fp32 [P])."""
    dt = q.dtype
    if dt not in (torch.bfloat16, torch.float32):
        raise TypeError(f"q must be bfloat16 or float32, got {dt}")
    for t, name in ((q, "q"), (gate, "gate"), (kv, "kv")):
        _require(t, dt, name)
    I = heads * dim_head
    P = q.shape[0]
    if B <= 0 or P % B or tuple(q.shape) != (P, I) or tuple(gate.shape) != (P, I) or tuple(kv.shape) != (P * T, 2 * I):
        raise ValueError(f"q / gate must be [P, {I}] and kv [P * T, {2 * I}] with P a multiple of B")
    xm = _mask_u8(x_mask, (P,), "x_mask")
    tm = _mask_u8(t_mask, (P * T,), "t_mask")
    out = torch.empty(P, I, dtype=dt, device=q.device) if out is None else out
    pooled = torch.empty(P, dtype=torch.float32, device=q.device) if pooled is None else pooled
    _require(out, dt, "out")
    _require(pooled, torch.float32, "pooled")
    if out.numel() < P * I or pooled.numel() < P:
        raise ValueError("out / pooled too small")
    fn = _lib.load().af2_template_pointwise_bf16_state if dt == torch.bfloat16 else _lib.load().af2_template_pointwise_f32_state
    _lib.check(fn(q.data_ptr(), gate.data_ptr(), kv.data_ptr(), _ptr(xm), _ptr(tm), out.data_ptr(), pooled.data_ptr(), None, None,
                  None, 1, 1, B, T, P // B, heads, dim_head, _stream_ptr()))
    return out, pooled


# --------------------------------------------------------------------------------------------------
# structure module (alphafold2.py:841-891): fp32 in both precision modes, except the pair projection (pair_projection_)
# --------------------------------------------------------------------------------------------------
IPA_MAX_HEADS = 16        # csrc/structure.cuh: IPA_MAX_HEADS
IPA_MAX_BATCH = 65535     # csrc/structure.cuh: IPA_MAX_BATCH (the attention grid's y dimension)
IPA_PROJ = 84             # projection floats per head: q|k|v scalars (3 x 16) and q|k|v points (3 x 4 x 3)
PAIR_PROJECTION_BAND_BYTES = 16 << 20     # scratch band of pair_projection_: pair rows of at most this many bytes


def ipa_shape_ok(B: int, n: int, heads: int, d: int) -> bool:
    """The shapes af2_ipa_attention and af2_structure_layer take (the C side rejects the others with ValueError, unlaunched)."""
    return 1 <= B <= IPA_MAX_BATCH and n >= 1 and 1 <= heads <= IPA_MAX_HEADS and d >= 4 and d % 4 == 0 and d <= 1024


def _check_ipa_shape(B: int, n: int, heads: int, d: int):
    if not ipa_shape_ok(B, n, heads, d):
        raise ValueError(f"invariant point attention takes 1 <= batch <= {IPA_MAX_BATCH}, n >= 1, 1 <= heads <= {IPA_MAX_HEADS} and dim "
                         f"a multiple of 4 up to 1024; got batch {B}, n {n}, heads {heads}, dim {d}")


def ipa_tile_rows(heads: int, d: int):
    """(key rows per tile, dynamic shared memory bytes) of af2_ipa_attention's CTA for (heads, d) (af2_ipa_tile_rows); (0, 0) for
    a shape it does not take."""
    smem = C.c_int(0)
    tj = _lib.load().af2_ipa_tile_rows(int(heads), int(d), C.byref(smem))
    return int(tj), int(smem.value)


def pack_structure(block, to_quaternion_update, to_points, lddt_linear) -> Packed:
    """fp32 weights of one structure layer (af2_structure_weights): the IPABlock `block` (the package's parameter names) and the
    model's to_quaternion_update / to_points / lddt_linear (None: the block alone, which af2_structure_layer refuses)."""
    a = block.attn
    t = dict(
        w_proj=torch.cat([_f32(l.weight) for l in (a.to_scalar_q, a.to_scalar_k, a.to_scalar_v, a.to_point_q, a.to_point_k,
                                                   a.to_point_v)], 0).contiguous(),
        w_bias=_f32(a.to_pairwise_attn_bias[0].weight), b_bias=_f32(a.to_pairwise_attn_bias[0].bias),
        point_weights=_f32(a.point_weights), w_out=_f32(a.to_out.weight), b_out=_f32(a.to_out.bias),
        attn_gamma=_f32(block.attn_norm.weight), attn_beta=_f32(block.attn_norm.bias),
        w_ff0=_f32(block.ff[0].weight), b_ff0=_f32(block.ff[0].bias), w_ff2=_f32(block.ff[2].weight), b_ff2=_f32(block.ff[2].bias),
        w_ff4=_f32(block.ff[4].weight), b_ff4=_f32(block.ff[4].bias), ff_gamma=_f32(block.ff_norm.weight),
        ff_beta=_f32(block.ff_norm.bias))
    for name, lin in (("qu", to_quaternion_update), ("points", to_points), ("lddt", lddt_linear)):
        if lin is not None:
            t["w_" + name], t["b_" + name] = _f32(lin.weight), _f32(lin.bias)
    s = _lib.StructureWeights(*(_p(t.get(k)) for k, _ in _lib.StructureWeights._fields_))
    pk = Packed(s, t, "f32")
    pk.heads = int(a.heads)
    pk.eps = (float(block.attn_norm.eps), float(block.ff_norm.eps))
    return pk


def structure_linear(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor] = None, relu: bool = False,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 nn.Linear over the rows of x [..., K] (af2_structure_linear): [..., N]; ReLU after the bias when `relu`."""
    _require(x, torch.float32, "x")
    w = _w32(w)
    _require(w, torch.float32, "w")
    N, K = w.shape
    if x.shape[-1] != K:
        raise ValueError(f"x has {x.shape[-1]} features, the weight takes {K}")
    b = _w32(b) if b is not None else None
    if b is not None and tuple(b.shape) != (N,):
        raise ValueError(f"bias must be [{N}], got {tuple(b.shape)}")
    out = torch.empty(*x.shape[:-1], N, dtype=torch.float32, device=x.device) if out is None else out
    _require(out, torch.float32, "out")
    rows = x.numel() // K
    if out.numel() != rows * N:
        raise ValueError(f"out must hold {rows} x {N} values")
    _lib.check(_lib.load().af2_structure_linear(x.data_ptr(), w.data_ptr(), _ptr(b), out.data_ptr(), rows, N, K, int(relu),
                                                _stream_ptr()))
    return out


def _frame_args(rot: torch.Tensor, trans: torch.Tensor, rows: int):
    _require(rot, torch.float32, "rot")
    _require(trans, torch.float32, "trans")
    if rot.numel() != rows * 9 or trans.numel() != rows * 3:
        raise ValueError(f"rot must be [..., 3, 3] and trans [..., 3] over {rows} residues")


def ipa_frames_(proj: torch.Tensor, rot: torch.Tensor, trans: torch.Tensor, heads: int) -> torch.Tensor:
    """The point columns of proj [..., 84 heads] taken to the global frame in place: X R + t per residue."""
    _require(proj, torch.float32, "proj")
    if not 1 <= heads <= IPA_MAX_HEADS or proj.shape[-1] != IPA_PROJ * heads:
        raise ValueError(f"proj must be [..., {IPA_PROJ} * heads] with 1 <= heads <= {IPA_MAX_HEADS}")
    rows = proj.numel() // proj.shape[-1]
    _frame_args(rot, trans, rows)
    _lib.check(_lib.load().af2_ipa_frames(proj.data_ptr(), rot.data_ptr(), trans.data_ptr(), rows, heads, _stream_ptr()))
    return proj


def ipa_attention(proj: torch.Tensor, pair: torch.Tensor, w_bias, b_bias, point_weights, mask: Optional[torch.Tensor],
                  rot: torch.Tensor, trans: torch.Tensor, heads: int) -> torch.Tensor:
    """The invariant point attention kernel alone (af2_ipa_attention): proj [B, n, 84 heads] (points global), pair [B, n, n, d],
    mask [B, n] bool or None, rot [B, n, 3, 3], trans [B, n, 3] -> the to_out input [B, n, heads (32 + d)] fp32."""
    _require(pair, torch.float32, "pair")
    if pair.dim() != 4 or pair.shape[1] != pair.shape[2]:
        raise ValueError(f"pair must be [B, n, n, d], got {tuple(pair.shape)}")
    B, n, _, d = pair.shape
    _check_ipa_shape(B, n, heads, d)
    _require(proj, torch.float32, "proj")
    if tuple(proj.shape) != (B, n, IPA_PROJ * heads):
        raise ValueError(f"proj must be [{B}, {n}, {IPA_PROJ * heads}], got {tuple(proj.shape)}")
    _frame_args(rot, trans, B * n)
    wb, bb, pw = _w32(w_bias), _w32(b_bias), _w32(point_weights)
    if tuple(wb.shape) != (heads, d) or tuple(bb.shape) != (heads,) or tuple(pw.shape) != (heads,):
        raise ValueError(f"w_bias must be [{heads}, {d}], b_bias and point_weights [{heads}]")
    mk = _mask_u8(mask, (B, n), "mask")
    out = torch.empty(B, n, heads * (32 + d), dtype=torch.float32, device=pair.device)
    _lib.check(_lib.load().af2_ipa_attention(proj.data_ptr(), pair.data_ptr(), wb.data_ptr(), bb.data_ptr(), pw.data_ptr(), _ptr(mk),
                                             rot.data_ptr(), trans.data_ptr(), out.data_ptr(), B, n, heads, d, _stream_ptr()))
    return out


def ipa_attention_rows(proj: torch.Tensor, pair_rows: torch.Tensor, w_bias, b_bias, point_weights, mask: Optional[torch.Tensor],
                       rot: torch.Tensor, trans: torch.Tensor, heads: int, row0: int) -> torch.Tensor:
    """ipa_attention of the query rows [row0, row0 + R) at batch 1 (af2_ipa_attention_rows): pair_rows [1, R, n, d] holds those
    pair rows; proj [1, n, 84 heads] (points global), mask [1, n], rot [1, n, 3, 3] and trans [1, n, 3] cover every residue ->
    the to_out input [1, R, heads (32 + d)] fp32, bitwise those rows of ipa_attention."""
    _require(pair_rows, torch.float32, "pair_rows")
    if pair_rows.dim() != 4 or pair_rows.shape[0] != 1:
        raise ValueError(f"pair_rows must be [1, R, n, d], got {tuple(pair_rows.shape)}")
    _, R, n, d = pair_rows.shape
    _check_ipa_shape(1, n, heads, d)
    if row0 < 0 or row0 + R > n:
        raise ValueError(f"query rows [{row0}, {row0 + R}) are not inside [0, {n})")
    _require(proj, torch.float32, "proj")
    if tuple(proj.shape) != (1, n, IPA_PROJ * heads):
        raise ValueError(f"proj must be [1, {n}, {IPA_PROJ * heads}], got {tuple(proj.shape)}")
    _frame_args(rot, trans, n)
    wb, bb, pw = _w32(w_bias), _w32(b_bias), _w32(point_weights)
    if tuple(wb.shape) != (heads, d) or tuple(bb.shape) != (heads,) or tuple(pw.shape) != (heads,):
        raise ValueError(f"w_bias must be [{heads}, {d}], b_bias and point_weights [{heads}]")
    mk = _mask_u8(mask, (1, n), "mask")
    out = torch.empty(1, R, heads * (32 + d), dtype=torch.float32, device=pair_rows.device)
    _lib.check(_lib.load().af2_ipa_attention_rows(proj.data_ptr(), pair_rows.data_ptr(), wb.data_ptr(), bb.data_ptr(), pw.data_ptr(),
                                                  _ptr(mk), rot.data_ptr(), trans.data_ptr(), out.data_ptr(), n, row0, R, heads, d,
                                                  _stream_ptr()))
    return out


def structure_tail_(single: torch.Tensor, o: torch.Tensor, gamma, beta, eps: float = 1e-5, w_qu=None, b_qu=None, quat=None,
                    trans=None, rot=None, w_points=None, b_points=None, w_lddt=None, b_lddt=None, coords=None, confidence=None):
    """af2_structure_tail on single [..., d] in place: LayerNorm(single + o); with w_qu the frame update of quat / trans / rot;
    with coords (and confidence) the coordinates and confidence of the updated frames.  Returns single."""
    _require(single, torch.float32, "single")
    _require(o, torch.float32, "o")
    d = single.shape[-1]
    rows = single.numel() // d
    if o.shape != single.shape:
        raise ValueError("o must have single's shape")
    ws = {k: (_w32(v) if v is not None else None) for k, v in dict(gamma=gamma, beta=beta, w_qu=w_qu, b_qu=b_qu, w_points=w_points,
                                                                   b_points=b_points, w_lddt=w_lddt, b_lddt=b_lddt).items()}
    for t, name, size in ((quat, "quat", 4), (trans, "trans", 3), (rot, "rot", 9), (coords, "coords", 3), (confidence, "confidence", 1)):
        if t is not None:
            _require(t, torch.float32, name)
            if t.numel() != rows * size:
                raise ValueError(f"{name} must hold {size} values per residue")
    _lib.check(_lib.load().af2_structure_tail(
        single.data_ptr(), o.data_ptr(), ws["gamma"].data_ptr(), ws["beta"].data_ptr(), float(eps), _ptr(ws["w_qu"]), _ptr(ws["b_qu"]),
        _ptr(quat), _ptr(trans), _ptr(rot), _ptr(ws["w_points"]), _ptr(ws["b_points"]), _ptr(ws["w_lddt"]), _ptr(ws["b_lddt"]),
        _ptr(coords), _ptr(confidence), rows, d, _stream_ptr()))
    return single


def _structure_layer_args(pk: Packed, single: torch.Tensor, quat, trans, rot, coords, confidence):
    """The per-residue operands of a structure layer, checked: (B, n, d) of single [B, n, d]."""
    _require(single, torch.float32, "single")
    B, n, d = single.shape
    _check_ipa_shape(B, n, pk.heads, d)
    for t, name, size in ((quat, "quat", 4), (trans, "trans", 3), (rot, "rot", 9), (coords, "coords", 3), (confidence, "confidence", 1)):
        if t is not None:
            _require(t, torch.float32, name)
            if t.numel() != B * n * size:
                raise ValueError(f"{name} must hold {size} values per residue")
    if (coords is None) != (confidence is None):
        raise ValueError("coords and confidence are written together")
    if pk.eps[0] != pk.eps[1]:
        raise ValueError("attn_norm and ff_norm must share one eps")
    return B, n, d


def structure_layer_(pk: Packed, single: torch.Tensor, pair: torch.Tensor, mask: Optional[torch.Tensor], quat: torch.Tensor,
                     trans: torch.Tensor, rot: torch.Tensor, coords: Optional[torch.Tensor] = None,
                     confidence: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One layer of alphafold2.py:863-885 (af2_structure_layer) on single [B, n, d] in place, with the frames quat [B, n, 4],
    trans [B, n, 3] and rot [B, n, 3, 3] updated; on the last layer coords [B, n, 3] and confidence [B, n, 1] are written."""
    _require(pair, torch.float32, "pair")
    B, n, d = _structure_layer_args(pk, single, quat, trans, rot, coords, confidence)
    if tuple(pair.shape) != (B, n, n, d):
        raise ValueError(f"pair must be [{B}, {n}, {n}, {d}], got {tuple(pair.shape)}")
    mk = _mask_u8(mask, (B, n), "mask")
    lib = _lib.load()
    ws = workspace(lib.af2_structure_layer_workspace(B, n, d, pk.heads), single.device)
    _lib.check(lib.af2_structure_layer(C.byref(pk.struct), single.data_ptr(), pair.data_ptr(), _ptr(mk), quat.data_ptr(), trans.data_ptr(),
                                       rot.data_ptr(), _ptr(coords), _ptr(confidence), B, n, d, pk.heads, pk.eps[0], ws.data_ptr(),
                                       ws.numel(), _stream_ptr()))
    return single


def structure_layer_rows_begin_(pk: Packed, single: torch.Tensor, pair_rows: torch.Tensor, mask: Optional[torch.Tensor],
                                quat: torch.Tensor, trans: torch.Tensor, rot: torch.Tensor, row0: int,
                                out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The first half of structure_layer_ at batch 1 for the pair rows [row0, row0 + R) that pair_rows [1, R, n, d] holds
    (af2_structure_layer_rows_begin): the projections and frames of all n residues of single [1, n, d], the attention of the R
    query rows and their to_out, written into out [1, R, d] (default: a new tensor), which is returned.  single and the frames
    are read, not written.  The rows of every shard, gathered in row order, are what structure_layer_rows_end_ takes."""
    _require(pair_rows, torch.float32, "pair_rows")
    B, n, d = _structure_layer_args(pk, single, quat, trans, rot, None, None)
    if pair_rows.dim() != 4 or pair_rows.shape[0] != B or tuple(pair_rows.shape[2:]) != (n, d) or B != 1:
        raise ValueError(f"pair_rows must be [1, R, {n}, {d}] with single [1, {n}, {d}], got {tuple(pair_rows.shape)} and "
                         f"{tuple(single.shape)}")
    R = pair_rows.shape[1]
    if row0 < 0 or row0 + R > n:
        raise ValueError(f"query rows [{row0}, {row0 + R}) are not inside [0, {n})")
    out = torch.empty(1, R, d, dtype=torch.float32, device=single.device) if out is None else out
    _require(out, torch.float32, "out")
    if tuple(out.shape) != (1, R, d):
        raise ValueError(f"out must be [1, {R}, {d}], got {tuple(out.shape)}")
    mk = _mask_u8(mask, (1, n), "mask")
    lib = _lib.load()
    ws = workspace(lib.af2_structure_layer_rows_workspace(n, R, d, pk.heads), single.device)
    _lib.check(lib.af2_structure_layer_rows_begin(C.byref(pk.struct), single.data_ptr(), pair_rows.data_ptr(), _ptr(mk), quat.data_ptr(),
                                                  trans.data_ptr(), rot.data_ptr(), out.data_ptr(), n, row0, R, d, pk.heads,
                                                  ws.data_ptr(), ws.numel(), _stream_ptr()))
    return out


def structure_layer_rows_end_(pk: Packed, single: torch.Tensor, o: torch.Tensor, quat: torch.Tensor, trans: torch.Tensor,
                              rot: torch.Tensor, coords: Optional[torch.Tensor] = None,
                              confidence: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The second half of structure_layer_ at batch 1 (af2_structure_layer_rows_end): single [1, n, d] <- attn_norm(single + o)
    with o [1, n, d] the gathered structure_layer_rows_begin_ rows, then the feed-forward, ff_norm and the frame update, in place;
    on the last layer coords [1, n, 3] and confidence [1, n, 1] are written.  Returns single."""
    _require(o, torch.float32, "o")
    B, n, d = _structure_layer_args(pk, single, quat, trans, rot, coords, confidence)
    if B != 1 or o.shape != single.shape:
        raise ValueError(f"single and o must both be [1, n, d], got {tuple(single.shape)} and {tuple(o.shape)}")
    lib = _lib.load()
    ws = workspace(lib.af2_structure_layer_rows_workspace(n, n, d, pk.heads), single.device)
    _lib.check(lib.af2_structure_layer_rows_end(C.byref(pk.struct), single.data_ptr(), o.data_ptr(), quat.data_ptr(), trans.data_ptr(),
                                                rot.data_ptr(), _ptr(coords), _ptr(confidence), n, d, pk.heads, pk.eps[0],
                                                ws.data_ptr(), ws.numel(), _stream_ptr()))
    return single


def plan_pair_projection_band(rows: int, n: int, d: int, precision: str, budget: int) -> int:
    """Pair rows per band of pair_projection_: at most PAIR_PROJECTION_BAND_BYTES of scratch, fewer when the scratch band and the
    GEMM's operand copy (bf16, or three bf16 planes in strict mode) exceed `budget` bytes, at least one row."""
    row_bytes = n * d * 4
    per_row = row_bytes + n * d * 2 * (SPLIT_PLANES if precision == "strict" else 1)
    band = min(rows, max(1, PAIR_PROJECTION_BAND_BYTES // row_bytes), max(1, budget // per_row))
    return max(1, int(band))


def pair_projection_(pk: Packed, x: torch.Tensor, out: Optional[torch.Tensor] = None, band: Optional[int] = None) -> torch.Tensor:
    """trunk_to_pairwise_repr_dim (alphafold2.py:850) over x [B, n, n, d] fp32, written into `out` (default: into x itself) in bands
    of pair rows through one scratch band: each output row depends on its own input row only, so no second pair tensor is
    needed.  The GEMM is af2_template_embed's (bf16 operands, or split-bf16 in strict mode: pk from pack_linear).  `band` forces
    the pair rows per band (tests); by default plan_pair_projection_band under 85 % of device_budget.  Returns out."""
    _require(x, torch.float32, "x")
    B, n, n2, d = x.shape
    if n != n2 or pk.k_in != d or pk.tensors["w"].shape[0] != d:
        raise ValueError(f"x must be [B, n, n, {pk.k_in}] and the projection square, got {tuple(x.shape)}")
    out = x if out is None else out
    _require(out, torch.float32, "out")
    if out.shape != x.shape:
        raise ValueError("out must have x's shape")
    return _pair_projection(pk, x, out, band)


def pair_projection_rows_(pk: Packed, x: torch.Tensor, band: Optional[int] = None) -> torch.Tensor:
    """pair_projection_ in place over pair rows x [B, R, n, d] (a rank's rows under shard_alphafold2(pair_rows=True)), through
    the same scratch band: bitwise those rows of pair_projection_ of the whole tensor.  Returns x."""
    _require(x, torch.float32, "x")
    if x.dim() != 4 or pk.k_in != x.shape[-1] or pk.tensors["w"].shape[0] != x.shape[-1]:
        raise ValueError(f"x must be [B, R, n, {pk.k_in}] and the projection square, got {tuple(x.shape)}")
    return _pair_projection(pk, x, x, band)


def _pair_projection(pk: Packed, x: torch.Tensor, out: torch.Tensor, band: Optional[int]) -> torch.Tensor:
    B, R, n, d = x.shape
    rows = B * R
    strict = pk.kind == "strict"
    if band is None:
        band = plan_pair_projection_band(rows, n, d, pk.kind, int(device_budget(x.device) * 0.85))
    band = max(1, min(int(band), rows))
    lib = _lib.load()
    qfn, fn = ((lib.af2_template_embed_strict_workspace, lib.af2_template_embed_strict) if strict else
               (lib.af2_template_embed_workspace, lib.af2_template_embed))
    ws = workspace(qfn(band * n, d), x.device)
    xs, os_ = x.view(rows, n * d), out.view(rows, n * d)
    scratch = torch.empty(band, n * d, dtype=torch.float32, device=x.device) if out.data_ptr() == x.data_ptr() else None
    for r0 in range(0, rows, band):
        r1 = min(rows, r0 + band)
        dst = os_[r0:r1] if scratch is None else scratch[:r1 - r0]
        _lib.check(fn(pk.tensors["w"].data_ptr(), pk.tensors["b"].data_ptr(), xs[r0:r1].data_ptr(), dst.data_ptr(), (r1 - r0) * n, d, d,
                      ws.data_ptr(), ws.numel(), _stream_ptr()))
        if scratch is not None:
            os_[r0:r1].copy_(dst)
    return out


# --------------------------------------------------------------------------------------------------
# distogram to coordinates (alphafold2_pytorch/utils.py:718-833)
# --------------------------------------------------------------------------------------------------
CENTER_MODES = {"mean": 0, "median": 1}
MAX_BINS = 128           # csrc/geometry.cuh: CD_MAX_BINS
MDS_MAX_N = 12288        # csrc/geometry.cuh: MDS_MAX_N


def wide_mode(wide) -> int:
    """0 std, 1 var, 2 none: like the reference, any other value means no dispersion (utils.py:751-756)."""
    return {"std": 0, "var": 1}.get(wide, 2) if isinstance(wide, str) else 2


def bin_centres(bins: torch.Tensor, device) -> torch.Tensor:
    """utils.py:733-735, the same torch lines: bins - half a bin width, the first centre 1.5 and the last 1.33 * bins[-1]."""
    c = (bins - 0.5 * (bins[2] - bins[1])).to(device)
    c[0] = 1.5
    c[-1] = 1.33 * bins[-1]
    return c.float().contiguous()


def check_bins(bins: torch.Tensor, nb: int):
    if bins.dim() != 1 or bins.shape[0] != nb:
        raise ValueError(f"bins must be a 1-D tensor of the distogram's {nb} buckets, got {tuple(bins.shape)}")
    if not 3 <= nb <= MAX_BINS:
        raise ValueError(f"the distogram kernel takes 3 to {MAX_BINS} bins, got {nb}")


def center_distogram(dist: torch.Tensor, bins: torch.Tensor, center: str = "mean", wide="std", softmax: bool = False,
                     mask: Optional[torch.Tensor] = None):
    """center_distogram_torch (utils.py:718-764) in one pass over dist [B, N, N, nb] fp32 -> (central, weights) [B, N, N] fp32.
    softmax: dist holds logits, normalised on chip.  mask [B, N]: a pair with a masked residue gets weight 0."""
    if dist.dim() != 4 or dist.shape[1] != dist.shape[2]:
        raise ValueError(f"distogram must be [b, N, N, bins], got {tuple(dist.shape)}")
    B, n, _, nb = dist.shape
    check_bins(bins, nb)
    if center not in CENTER_MODES:
        raise ValueError(f"center must be one of {tuple(CENTER_MODES)}, got {center!r}")
    mask = _mask_u8(mask, (B, n), "mask")
    _require(dist, torch.float32, "distogram")
    thr = float(bins[-2])
    centres = bin_centres(bins, dist.device)
    if mask is not None:
        mask = mask.to(dist.device)
    central = torch.empty(B, n, n, dtype=torch.float32, device=dist.device)
    weights = torch.empty_like(central)
    _lib.check(_lib.load().af2_center_distogram(dist.data_ptr(), centres.data_ptr(), thr, _ptr(mask), central.data_ptr(),
                                                weights.data_ptr(), B, n, nb, CENTER_MODES[center], wide_mode(wide), int(bool(softmax)),
                                                _stream_ptr()))
    return central, weights


def mds_init(pre_dist_mat: torch.Tensor) -> torch.Tensor:
    """mds_torch's initialisation (utils.py:789-798), the same torch lines on the device: the top singular vectors of
    M = 0.5 (D[:, :1, :] + D[:, :, :1] - D), D = pre_dist_mat^2, by torch.svd_lowrank (randomised: it draws from the RNG of
    the tensor's device), scaled by sqrt|s| -> [B, N, 3] fp32.  Below 3 points svd_lowrank gives fewer columns: the rest are 0."""
    D = pre_dist_mat ** 2
    M = 0.5 * (D[:, :1, :] + D[:, :, :1] - D)
    svds = [torch.svd_lowrank(mi) for mi in M]
    u = torch.stack([s[0] for s in svds], dim=0)
    s = torch.stack([s[1] for s in svds], dim=0)
    x = torch.bmm(u, torch.diag_embed(s).abs().sqrt())[..., :3]
    if x.shape[-1] < 3:
        x = torch.nn.functional.pad(x, (0, 3 - x.shape[-1]))
    return x.float().contiguous()


def mds_iterate_(delta: torch.Tensor, weights: Optional[torch.Tensor], x: torch.Tensor, iters: int, tol: float):
    """The SMACOF loop of mds_torch (utils.py:805-831) in one cooperative launch with no host synchronisation inside: delta and
    weights [B, N, N] fp32 (weights None: all ones), x [B, N, 3] fp32 in: the init, out (in place): the coords the reference
    returns.  Reads the step count once at the end and returns (steps, stopped, his [steps + 1 + stopped, B] fp64,
    stress [steps + stopped, B] fp64): his[0] = inf, his[k + 1] = stress_k / |X_k'|; the last row is that of the iteration
    that stopped the loop when stopped."""
    _require(delta, torch.float32, "pre_dist_mat")
    _require(x, torch.float32, "x")
    if weights is not None:
        _require(weights, torch.float32, "weights")
    B, n, _ = delta.shape
    lib = _lib.load()
    need = lib.af2_mds_workspace(B, n, int(iters))
    if need < 0:
        _lib.check(-1)
    dev = delta.device
    his = torch.empty(int(iters) + 1, B, dtype=torch.float64, device=dev)
    stress = torch.empty(max(int(iters), 1), B, dtype=torch.float64, device=dev)
    steps = torch.empty(2, dtype=torch.int32, device=dev)
    ws = workspace(need, dev)
    _lib.check(lib.af2_mds_iterate(delta.data_ptr(), _ptr(weights), x.data_ptr(), his.data_ptr(), stress.data_ptr(), steps.data_ptr(),
                                   B, n, int(iters), float(tol), ws.data_ptr(), ws.numel(), _stream_ptr()))
    k, stopped = (int(v) for v in steps.tolist())
    return k, bool(stopped), his[:k + 1 + stopped], stress[:k + stopped]


# --------------------------------------------------------------------------------------------------
# structure scores (alphafold2_pytorch/utils.py:999-1247)
# --------------------------------------------------------------------------------------------------
MAX_CUTOFFS = 8          # csrc/metrics.cuh: SS_MAX_CUT


def _points(t: Optional[torch.Tensor], strides=None):
    """af2_points of a [B, n, 3]-like view: strides (sb, sn, sk) in elements, default the view's own."""
    if t is None:
        return None
    sb, sn, sk = t.stride() if strides is None else strides
    return _lib.Points(t.data_ptr(), sb, sn, sk)


def _byref(s):
    return None if s is None else C.byref(s)


def _f32_view(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (alphafold2_b200 has no CPU fallback)")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")


def metrics_workspace(B: int, n: int, device) -> torch.Tensor:
    need = _lib.load().af2_metrics_workspace(int(B), int(n))
    if need < 0:
        _lib.check(-1)
    return workspace(need, device)


def superpose_scores(x, y, B: int, n: int, *, mask=None, mask_strides=(0, 0), align=False, shift=False, out_x=None, out_y=None,
                     rot=None, rmsd=None, tm=None, cutoffs=(), gdt=(), lddt=None, lddt_mean=None, lddt_points=None, r0=15.0):
    """af2_superpose_scores, preceded by the lDDT pair pass when lddt_points = (true, predicted) is given, on one workspace.
    x, y: fp32 CUDA views [B, n, 3] (any strides; the [B, 3, n] layouts are passed as their transposes), or None for lDDT
    alone.  mask: uint8/bool [B, n]-strided selection (mask_strides in elements) or None.  Outputs are preallocated
    tensors written in place: out_x / out_y [B, n, 3] views, rot [B, 3, 3] fp64, rmsd / tm / lddt_mean [B] fp32,
    lddt [B, n] fp32.  gdt: up to two (out [B] fp32, cutoff indices, weights)."""
    for t, name in ((x, "x"), (y, "y")):
        if t is not None:
            _f32_view(t, name)
    outs = [t for t in (rmsd, tm, lddt, lddt_mean) if t is not None] + [g[0] for g in gdt]
    for t in outs:
        _require(t, torch.float32, "output")
    dev = (x if x is not None else lddt_points[0]).device
    lib = _lib.load()
    ws = metrics_workspace(B, n, dev)
    mptr = _ptr(mask)
    if lddt_points is not None:
        tp, pp = lddt_points
        _f32_view(tp, "true_coords")
        _f32_view(pp, "pred_coords")
        _lib.check(lib.af2_pair_distance_scores(0, C.byref(_points(tp)), 0, C.byref(_points(pp)), 0, mptr, mask_strides[0],
                                                mask_strides[1], B, n, float(r0), float("-inf"), float("inf"), 2.0, None,
                                                ws.data_ptr(), ws.numel(), _stream_ptr()))
    cut = (C.c_float * MAX_CUTOFFS)(*[float(c) for c in cutoffs])
    specs = (_lib.GdtSpec * 2)()
    for g, (out, idx, w) in enumerate(gdt):
        specs[g].out = out.data_ptr()
        specs[g].k = len(idx)
        for k, (i, wk) in enumerate(zip(idx, w)):
            specs[g].idx[k] = int(i)
            specs[g].w[k] = float(wk)
    _lib.check(lib.af2_superpose_scores(_byref(_points(x)), _byref(_points(y)), mptr, mask_strides[0], mask_strides[1], B, n,
                                        int(bool(align)), int(bool(shift)), _byref(_points(out_x)), _byref(_points(out_y)),
                                        _ptr(rot), _ptr(rmsd), _ptr(tm), len(cutoffs), cut, specs, int(lddt is not None),
                                        _ptr(lddt), _ptr(lddt_mean), ws.data_ptr(), ws.numel(), _stream_ptr()))


def distmat_loss(a, a_matrix: bool, b, b_matrix: bool, B: int, n: int, mask=None, lo=float("-inf"), hi=float("inf"), q=2.0):
    """af2_pair_distance_scores in loss mode: a, b are fp32 CUDA views, coordinates [Bx, n, 3] or matrices [Bx, n, n] with
    Bx 1 (shared by the batch) or B; mask bool [B, n, n] contiguous or None -> the mean loss, a 0-d fp32 tensor."""
    _f32_view(a, "X")
    _f32_view(b, "Y")
    out = torch.empty((), dtype=torch.float32, device=a.device)
    _require(out, torch.float32, "loss")
    if mask is not None and not mask.is_contiguous():
        mask = mask.contiguous()

    def pts(t, mat):
        sb = 0 if t.shape[0] == 1 else t.stride(0)
        return _lib.Points(t.data_ptr(), sb, t.stride(1), 0 if mat else t.stride(2))
    ws = metrics_workspace(B, n, a.device)
    _lib.check(_lib.load().af2_pair_distance_scores(1, C.byref(pts(a, a_matrix)), int(a_matrix), C.byref(pts(b, b_matrix)),
                                                    int(b_matrix), _ptr(mask), n * n, n, B, n, 15.0, float(lo), float(hi),
                                                    float(q), out.data_ptr(), ws.data_ptr(), ws.numel(), _stream_ptr()))
    return out


# --------------------------------------------------------------------------------------------------
# distogram loss (train_pre.py:76-90 with get_bucketed_distance_matrix, alphafold2_pytorch/utils.py:45-50)
# --------------------------------------------------------------------------------------------------
XENT_MAX_BINS = 4096     # csrc/distogram_loss.cuh: DX_MAX_BINS


def _label_inputs(coords: torch.Tensor, mask: Optional[torch.Tensor], nb: int):
    """coords fp32 [B, n, c] contiguous on a CUDA device, mask bool [B, n] contiguous on it or None, and the bucket edges."""
    _require(coords, torch.float32, "coords")
    if mask is not None:
        _require(mask, torch.bool, "mask")
    return recycling_boundaries(nb, coords.device)


def distogram_xent_rows(logits: torch.Tensor, coords: torch.Tensor, mask: Optional[torch.Tensor], ignore_index: int,
                        row0: int = 0) -> torch.Tensor:
    """af2_distogram_xent_rows: logits [B, rows, n, nb] fp32 contiguous (the distogram rows [row0, row0 + rows)), coords
    [B, n, c] fp32, mask [B, n] bool or None -> the per-row partials [B, rows, 2] int64: column 0 holds the fp64 bits of the
    row's sum (.view(torch.float64)), column 1 the number of counted pairs.  One launch; no other device memory."""
    _require(logits, torch.float32, "distance_logits")
    B, rows, n, nb = logits.shape
    bnd = _label_inputs(coords, mask, nb)
    part = torch.empty(B, rows, 2, dtype=torch.int64, device=logits.device)
    if rows == 0:
        return part
    _lib.check(_lib.load().af2_distogram_xent_rows(logits.data_ptr(), coords.data_ptr(), coords.shape[-1], _ptr(mask), bnd.data_ptr(), B,
                                                   n, nb, int(row0), rows, int(ignore_index), part.data_ptr(), _stream_ptr()))
    return part


def distogram_xent_finish(part: torch.Tensor) -> torch.Tensor:
    """af2_distogram_xent_finish over partials [B, n, 2] int64 in row order (distogram_xent_rows of every row, joined along the
    rows) -> the mean, a 0-d fp32 tensor on their device.  One launch."""
    _require(part, torch.int64, "partials")
    out = torch.empty((), dtype=torch.float32, device=part.device)
    _lib.check(_lib.load().af2_distogram_xent_finish(part.data_ptr(), part.numel() // 2, out.data_ptr(), _stream_ptr()))
    return out


def bucketed_distance(coords: torch.Tensor, mask: Optional[torch.Tensor], nb: int, ignore_index: int) -> torch.Tensor:
    """af2_bucketed_distance: coords [B, n, c] fp32, mask [B, n] bool or None -> labels [B, n, n] int64.  One launch."""
    bnd = _label_inputs(coords, mask, nb)
    B, n, c = coords.shape
    labels = torch.empty(B, n, n, dtype=torch.int64, device=coords.device)
    _lib.check(_lib.load().af2_bucketed_distance(coords.data_ptr(), c, _ptr(mask), bnd.data_ptr(), B, n, int(nb), int(ignore_index),
                                                 labels.data_ptr(), _stream_ptr()))
    return labels


# --------------------------------------------------------------------------------------------------
# angle-head labels and loss (the trRosetta orientations from the backbone, DESIGN.md §4f)
# --------------------------------------------------------------------------------------------------
def _angle_nb(nb) -> C.Array:
    return (C.c_int * 3)(*(int(v) for v in nb))


def angle_xent_rows(theta: torch.Tensor, phi: torch.Tensor, omega: torch.Tensor, backbone: torch.Tensor,
                    mask: Optional[torch.Tensor], ignore_index: int, row0: int = 0) -> torch.Tensor:
    """af2_angle_xent_rows: theta / phi / omega [B, rows, n, nb_h] fp32 contiguous (the heads' rows [row0, row0 + rows)),
    backbone [B, n, A, 3] fp32 contiguous, mask [B, n] bool or None -> the per-row partials [B, rows, 3, 2] int64: per head
    (theta, phi, omega) column 0 holds the fp64 bits of the row's sum (.view(torch.float64)), column 1 the number of counted
    pairs.  One launch; no other device memory."""
    for t, name in ((theta, "theta_logits"), (phi, "phi_logits"), (omega, "omega_logits")):
        _require(t, torch.float32, name)
    _require(backbone, torch.float32, "backbone")
    if mask is not None:
        _require(mask, torch.bool, "mask")
    B, rows, n = theta.shape[:3]
    part = torch.empty(B, rows, 3, 2, dtype=torch.int64, device=theta.device)
    if rows == 0:
        return part
    nb = _angle_nb((theta.shape[-1], phi.shape[-1], omega.shape[-1]))
    _lib.check(_lib.load().af2_angle_xent_rows(theta.data_ptr(), phi.data_ptr(), omega.data_ptr(), backbone.data_ptr(),
                                               backbone.shape[2], _ptr(mask), nb, B, n, int(row0), rows, int(ignore_index),
                                               part.data_ptr(), _stream_ptr()))
    return part


def angle_xent_finish(part: torch.Tensor) -> torch.Tensor:
    """af2_angle_xent_finish over partials [B, n, 3, 2] int64 in row order (angle_xent_rows of every row, joined along the
    rows) -> the three heads' mean terms, fp32 [3] (theta, phi, omega) on their device.  One launch."""
    _require(part, torch.int64, "partials")
    out = torch.empty(3, dtype=torch.float32, device=part.device)
    _lib.check(_lib.load().af2_angle_xent_finish(part.data_ptr(), part.numel() // 6, out.data_ptr(), _stream_ptr()))
    return out


def bucketed_angles(backbone: torch.Tensor, mask: Optional[torch.Tensor], nb, ignore_index: int):
    """af2_bucketed_angles: backbone [B, n, A, 3] fp32, mask [B, n] bool or None, nb the three bucket counts -> the labels
    (theta, phi, omega), each [B, n, n] int64.  One launch."""
    _require(backbone, torch.float32, "backbone")
    if mask is not None:
        _require(mask, torch.bool, "mask")
    B, n, A = backbone.shape[:3]
    out = [torch.empty(B, n, n, dtype=torch.int64, device=backbone.device) for _ in range(3)]
    _lib.check(_lib.load().af2_bucketed_angles(backbone.data_ptr(), A, _ptr(mask), _angle_nb(nb), B, n, int(ignore_index),
                                               out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), _stream_ptr()))
    return tuple(out)
