"""Tensor-level wrappers over the C ABI: argument validation, weight packing, workspace management.

PyTorch is used for device memory and streams only; every FLOP of the hot path runs inside libaf2b200.so.
"""
from __future__ import annotations

import ctypes as C
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


def workspace(nbytes: int, device) -> torch.Tensor:
    """Grow-only per-device scratch buffer, reused by every op (ops on one stream are serialised).  Inside a
    `private_workspace` scope the buffer belongs to the scope's owner (a captured CUDA graph keeps raw pointers into it)."""
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
    return buf


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
    return w, b.contiguous()          # fp32; callers round to bf16 (after folding the LayerNorm affine where needed)


def _pad_rows(t: torch.Tensor, mult: int = 256) -> torch.Tensor:
    """Zero-pad dim 0 to a multiple of `mult` (segments of the fused projection kernel start on 256-column tiles)."""
    r = (-t.shape[0]) % mult
    if r == 0:
        return t
    return torch.cat([t, torch.zeros((r,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)], 0)


def _cat_segments(ws, bs, gamma, beta):
    """Operands of the fused LayerNorm -> projection kernel (proj_tc.cuh): every segment zero-padded to 256-row tiles and
    the LayerNorm affine folded in, W' = W diag(gamma) (bf16), b' = W beta + b (fp32, accumulator-column order); the
    kernel's producer then only computes (x - mean) * rstd."""
    w = torch.cat([_pad_rows(x.detach().float()) for x in ws], 0)
    b = torch.cat([_pad_rows(x.detach().float()) for x in bs], 0)
    g, be = gamma.detach().float(), beta.detach().float()
    return _bf16(w * g[None, :]), (b + w @ be).contiguous()


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
    if half == 128:                                         # the fused kernel works on 256-column accumulator tiles
        t["wcat"], t["bcat"] = _cat_segments([w1f], [b1p], norm_w, norm_b)
    s = _lib.FFWeights(t["g"].data_ptr(), t["b"].data_ptr(), t["w1"].data_ptr(), t["b1"].data_ptr(),
                       t["w2"].data_ptr(), t["b2"].data_ptr(), 2 * half, _p(t.get("wcat")), _p(t.get("bcat")), None)
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
    t["wcat"], t["bcat"] = _cat_segments([wqkv, wg], [torch.zeros(wqkv.shape[0], device=wqkv.device), bg], norm_w, norm_b)
    s = _lib.AttnWeights(t["g"].data_ptr(), t["b"].data_ptr(), t["wqkv"].data_ptr(), t["wg"].data_ptr(),
                         t["bg"].data_ptr(), t["wo"].data_ptr(), t["bo"].data_ptr(),
                         t["we"].data_ptr() if w_edge is not None else None, t["wcat"].data_ptr(), t["bcat"].data_ptr(), None)
    return Packed(s, t)


def pack_triangle_multiply(norm_w, norm_b, wl, bl, wr, br, wlg, blg, wrg, brg, wog, bog, onw, onb, wo, bo) -> Packed:
    d = wl.shape[0]
    half = gated_half(d)
    f = lambda x: x.detach().float()  # noqa: E731
    wlp, blp = pack_gated(f(wl), f(bl), f(wlg), f(blg), half)
    wrp, brp = pack_gated(f(wr), f(br), f(wrg), f(brg), half)
    t = dict(g=_f32(norm_w), b=_f32(norm_b), wl=_bf16(wlp), bl=blp, wr=_bf16(wrp), br=brp, wog=_bf16(wog), bog=_f32(bog),
             ong=_f32(onw), onb=_f32(onb), wo=_bf16(wo), bo=_f32(bo))
    if half == 128:
        t["wcat"], t["bcat"] = _cat_segments([wlp, wrp, wog], [blp, brp, bog], norm_w, norm_b)
    s = _lib.TriMulWeights(t["g"].data_ptr(), t["b"].data_ptr(), t["wl"].data_ptr(), t["bl"].data_ptr(),
                           t["wr"].data_ptr(), t["br"].data_ptr(), t["wog"].data_ptr(), t["bog"].data_ptr(),
                           t["ong"].data_ptr(), t["onb"].data_ptr(), t["wo"].data_ptr(), t["bo"].data_ptr(), 2 * half,
                           _p(t.get("wcat")), _p(t.get("bcat")), None, None)
    return Packed(s, t)


def pack_outer_mean(norm_w, norm_b, wl, bl, wr, br, wo, bo) -> Packed:
    t = dict(g=_f32(norm_w), b=_f32(norm_b), wlr=_bf16(torch.cat([wl.detach(), wr.detach()], 0)),
             blr=_f32(torch.cat([bl.detach(), br.detach()], 0)), wo=_bf16(wo), bo=_f32(bo))
    t["wcat"], t["bcat"] = _cat_segments([torch.cat([wl.detach(), wr.detach()], 0)], [t["blr"]], norm_w, norm_b)
    s = _lib.OuterWeights(t["g"].data_ptr(), t["b"].data_ptr(), t["wlr"].data_ptr(), t["blr"].data_ptr(),
                          t["wo"].data_ptr(), t["bo"].data_ptr(), t["wcat"].data_ptr(), t["bcat"].data_ptr(),
                          None, None)
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
# L2 residency of the pair stream (AF2_L2_PERSIST, default off until measured -- see DESIGN.md)
# --------------------------------------------------------------------------------------------------
L2_PERSIST = float(_os.environ.get("AF2_L2_PERSIST", "0") or 0)     # 0: off; (0, 1]: hit ratio of the window over x


class l2_resident:
    """with l2_resident(x): kernels launched on the current stream keep x's address range persisting in L2."""

    def __init__(self, t: Optional[torch.Tensor]):
        self.t = t if (L2_PERSIST > 0 and t is not None and t.is_cuda) else None

    def __enter__(self):
        if self.t is not None:
            try:
                _lib.check(_lib.load().af2_l2_persist(self.t.data_ptr(), self.t.numel() * self.t.element_size(), float(L2_PERSIST), _stream_ptr()))
            except RuntimeError as e:
                import sys
                print(f"[alphafold2_b200] L2 persistence not applied: {e}", file=sys.stderr)
                self.t = None
        return self

    def __exit__(self, *exc):
        if self.t is not None:
            _lib.check(_lib.load().af2_l2_persist(None, 0, 0.0, _stream_ptr()))
        return False


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
    if not seq.is_cuda:
        raise RuntimeError("seq must be a CUDA tensor (alphafold2_b200 has no CPU fallback)")
    emb = _w32(token_emb)
    _require(emb, torch.float32, "token_emb.weight")
    B, n = seq.shape
    S = msa.shape[1]
    d = emb.shape[1]
    seq = seq.to(torch.int64).contiguous()
    msa = msa.to(torch.int64).contiguous()
    x = torch.empty(B, n, n, d, dtype=torch.float32, device=seq.device)
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
    if R != S and B > 1:
        # the kernels write S contiguous rows per batch element: one call per element into its slice of m
        for b in range(B):
            pick = lambda t: None if t is None else t[b]  # noqa: E731
            _lib.check(lib.af2_embed_pair_init(seq[b].data_ptr(), msa[b].data_ptr(), emb.data_ptr(), emb.shape[0], _ptr(pick(se)),
                                               _ptr(pick(me)), wp.data_ptr(), bp.data_ptr(), pe.data_ptr(), int(max_rel_dist), _ptr(si),
                                               x[b].data_ptr(), m[b].data_ptr(), 1, S, n, d, ws.data_ptr(), ws.numel(), _stream_ptr()))
        return x, m
    _lib.check(lib.af2_embed_pair_init(seq.data_ptr(), msa.data_ptr(), emb.data_ptr(), emb.shape[0], _ptr(se), _ptr(me), wp.data_ptr(),
                                       bp.data_ptr(), pe.data_ptr(), int(max_rel_dist), _ptr(si), x.data_ptr(), m.data_ptr(), B, S, n, d,
                                       ws.data_ptr(), ws.numel(), _stream_ptr()))
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
    _require(x, torch.float32, "x")
    _require(m, torch.float32, "m")
    B, n, _, d = x.shape
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
    want = {"coords": (B, n, c), "single_row": (B, n, d), "prev_pair": (B, n, n, d), "msa_gamma": (d,), "msa_beta": (d,),
            "pair_gamma": (d,), "pair_beta": (d,), "table": (nb, d)}
    for k, shape in want.items():
        if tuple(ts[k].shape) != shape:
            raise ValueError(f"{k} must be {shape}, got {tuple(ts[k].shape)}")
    _lib.check(_lib.load().af2_recycle_embed(
        ts["coords"].data_ptr(), c, ts["single_row"].data_ptr(), ts["prev_pair"].data_ptr(), ts["msa_gamma"].data_ptr(),
        ts["msa_beta"].data_ptr(), ts["pair_gamma"].data_ptr(), ts["pair_beta"].data_ptr(), ts["table"].data_ptr(),
        ts["boundaries"].data_ptr(), nb, x.data_ptr(), m.data_ptr(), m.stride(0), B, n, d, float(eps), _stream_ptr()))
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
    """The pointwise template-attention kernel alone (include/af2b200.h, af2_template_pointwise_bf16 / _f32): q, gate [P, I],
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
    fn = _lib.load().af2_template_pointwise_bf16 if dt == torch.bfloat16 else _lib.load().af2_template_pointwise_f32
    _lib.check(fn(q.data_ptr(), gate.data_ptr(), kv.data_ptr(), _ptr(xm), _ptr(tm), out.data_ptr(), pooled.data_ptr(), B, T, P // B,
                  heads, dim_head, _stream_ptr()))
    return out, pooled
