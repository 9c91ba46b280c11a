"""-m gpu: the three fused persistent kernels element-wise against fp64, across their persistent schedules: the GEGLU
feed-forward (ff_fused_kernel<D, 64>), the contraction tail (contract_tail_kernel<D, V>, all three variants) and axial
attention with in-kernel projections (attention_proj_kernel<DH>).

Each kernel launches min(work items, SMs) CTAs; a CTA walks its items with a stride of the grid, and its TMA producer runs
ahead across items through a ring of mbarrier-tracked slots whose slot index and phase carry from one item to the next.
The cases therefore take their item (tile) counts from the device's SM count: below the grid, equal to it, one above it
and 2 SMs + 5, each ending in a partial last tile; they include rings whose depth does not divide the stages an item uses
(attention_proj at n <= 128 with 2 or 6 stages per item on 4 slots, DH 32 at n = 1000 with 16 stages on 3; the tail's
weight ring at D = 256, 3 slots against 4 or 8 chunks per tile, and at D = 128 with a loaded gate, 2 chunks on 8 slots),
consecutive attention items with different masks, the zero-filled last channel chunk (d = 32, 96, 160) and the C2 / C3
calls.

Every case checks four things:
  (a) the fused kernel ran: the library's launch count, or the path ops.contract_tail reports;
  (b) every element is within the fp64 bound of fused_bounds.py (derived there; worst err / bound to the parity report);
  (c) the output is bitwise the unfused sequence the kernel replaces (test_gpu_fused_ff._two_gemm,
      test_gpu_contract_tail's CTAIL_UNFUSED path, test_gpu_attention_proj._unfused);
  (d) a second identical launch gives the same bits.
Outputs go to caller-owned buffers with NaN guards before and after them, which must stay NaN: x is a view inside a larger
buffer for the feed-forward and the tail, and af2_attention_proj_bf16 is called through the C ABI with a guarded output.
"""
import pytest
import torch

import fused_bounds as FB
from gpu_util import check_bound
from test_gpu_attention_kernel import _mask, _tok
from test_gpu_attention_persistent import _mixed_mask, _ragged_suffix, _sms

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 64
GRID = {"half": lambda sm: sm // 2, "equal": lambda sm: sm, "one_above": lambda sm: sm + 1, "many": lambda sm: 2 * sm + 5}


def _ops():
    from alphafold2_b200 import ops
    return ops


def _lib():
    from alphafold2_b200 import _lib
    return _lib


def _launches():
    return _lib().load().af2_launch_count()


def _guarded(n, dtype):
    """(buffer of n elements with GUARD NaN elements on both sides, the inner view)"""
    buf = torch.full((n + 2 * GUARD,), NAN, dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + n]


def _guards_intact(buf, n, name):
    assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[GUARD + n:].float()).all(), f"{name}: write outside"


def _same(a, b, what):
    ia = a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32)
    ib = b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32)
    diff = (ia != ib).sum().item()
    assert diff == 0, f"{what}: {diff} of {a.numel()} elements differ"


# ------------------------------------------------------------------------------------------------------------------------
# A. feed-forward: x += W2 h + b2 over 128-row tiles (ops.feed_forward_: LayerNorm launch + ff_fused_kernel)
# ------------------------------------------------------------------------------------------------------------------------
def ff_case(name, D, hidden, T, seed):
    from test_gpu_fused_ff import _two_gemm
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).cuda()   # noqa: E731
    pk = ops.pack_feed_forward(1 + 0.1 * r(D), 0.1 * r(D), r(2 * hidden, D) * D ** -0.5, 0.5 * r(2 * hidden),
                               r(D, hidden) * hidden ** -0.5, r(D))
    t = pk.tensors
    x0 = r(T, D)
    buf, xv = _guarded(T * D, torch.float32)
    xv.copy_(x0.flatten())
    x = xv.view(T, D)
    torch.cuda.synchronize()
    before = _launches()
    ops.feed_forward_(pk, x)
    torch.cuda.synchronize()
    assert _launches() - before == 2, "the LayerNorm and ff_fused_kernel"                                  # (a)
    _guards_intact(buf, T * D, name)
    xn = ops.layernorm_bf16(x0, t["g"], t["b"])               # the LayerNorm launch of feed_forward_, its input to the kernel
    ref, bound = FB.ff_ref(x0, xn, t["w1"], t["b1"], t["w2"], t["b2"])
    check_bound(name, x, ref, bound)                                                                       # (b)
    _same(x, _two_gemm(pk, x0), f"{name} against the two-GEMM path")                                       # (c)
    buf2, xv2 = _guarded(T * D, torch.float32)
    xv2.copy_(x0.flatten())
    ops.feed_forward_(pk, xv2.view(T, D))
    torch.cuda.synchronize()
    _same(xv2, xv, f"{name} second launch")                                                                # (d)


FF_RES = [1, 64, 65]


@pytest.mark.parametrize("count", list(GRID))
@pytest.mark.parametrize("hidden", [128, 384, "4d"])
@pytest.mark.parametrize("D", [128, 256])
def test_ff_tile_counts(D, hidden, count):
    """128-row tiles below, at, one above and 2 SMs + 5 times the grid; the last tile holds 1, 64 or 65 rows"""
    hidden = 4 * D if hidden == "4d" else hidden
    tiles = GRID[count](_sms())
    res = FF_RES[(list(GRID).index(count) + hidden // 128) % 3]
    T = (tiles - 1) * 128 + res
    ff_case(f"fused ff D{D} hidden{hidden} {count} T{T}", D, hidden, T, seed=T + hidden)


@pytest.mark.parametrize("T", [256 * 256, 128 * 256], ids=["pair", "msa"])
def test_ff_c2(T):
    """the C2 feed-forwards: dim 256, hidden 1024, the pair (256 x 256) and MSA (128 x 256) tokens"""
    ff_case(f"fused ff C2 T{T}", 256, 1024, T, seed=T)


# ------------------------------------------------------------------------------------------------------------------------
# B. contraction tail: x += tail(O) W_out^T + b_out over 64-token tiles (ops.contract_tail, CTAIL_FUSED)
# ------------------------------------------------------------------------------------------------------------------------
def tail_case(name, D, kind, rows, n, seed, use_scale=True):
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    T = rows * n
    cs = (T + 3) // 4 * 4                                     # the TMA tensor map needs a 16-byte channel stride
    f = lambda *s: torch.randn(*s, generator=g).cuda()   # noqa: E731
    w = lambda *s: (torch.randn(*s, generator=g) * D ** -0.5).to("cuda", torch.bfloat16)   # noqa: E731
    O = f(T, D) + 1e3 if kind != "scale" else 3 * f(T, D) + 0.5
    src = torch.full((D * cs,), NAN, device="cuda")           # pad columns t >= T of every channel: never read
    src.view(D, cs)[:, :T] = O.t()
    x0 = f(T, D)
    w_out, b_out = w(D, D), f(D)
    gamma, beta = 1 + 0.5 * f(D), f(D)
    gate = torch.rand(T, D, generator=g).to("cuda", torch.bfloat16)
    xn, w_og, b_og = f(T, D).bfloat16(), w(D, D), f(D)
    scale = (torch.rand(T, generator=g) + 0.5).cuda()
    kw = dict(chan_stride=cs, pitch=n, rows=rows, n=n, d=D)
    if kind == "scale":
        kw.update(mode=1, scale=scale if use_scale else None, scale_const=0.125)
        rkw = dict(scale=scale) if use_scale else dict(scale_const=0.125)
    else:
        kw.update(mode=0, gamma=gamma, beta=beta, gate=gate)
        rkw = dict(gamma=gamma, beta=beta, gate=gate)
        if kind == "project":
            kw.update(gate=torch.empty_like(gate), xn=xn, w_ogate=w_og, b_ogate=b_og)    # gate: the unfused path's output
            rkw = dict(gamma=gamma, beta=beta, xn=xn, w_og=w_og, b_og=b_og)
    y = torch.empty(T * D, dtype=torch.bfloat16, device="cuda")

    def run(variant):
        buf, xv = _guarded(T * D, torch.float32)
        xv.copy_(x0.flatten())
        torch.cuda.synchronize()
        before = _launches()
        ran = ops.contract_tail(src, buf, w_out, b_out, y, variant=variant, x_off=GUARD, **kw)
        torch.cuda.synchronize()
        _guards_intact(buf, T * D, name)
        return xv.view(T, D), ran, _launches() - before

    x, ran, launches = run(ops.CTAIL_FUSED)
    assert ran == ops.CTAIL_FUSED and launches == 1                                                        # (a)
    ref, bound = FB.tail_ref(O, x0, w_out, b_out, **rkw)
    check_bound(name, x, ref, bound)                                                                       # (b)
    xu, ran_u, _ = run(ops.CTAIL_UNFUSED)
    assert ran_u == ops.CTAIL_UNFUSED
    _same(x, xu, f"{name} against the unfused tail")                                                       # (c)
    _same(run(ops.CTAIL_FUSED)[0], x, f"{name} second launch")                                             # (d)


TAIL_RES = [1, 63]


@pytest.mark.parametrize("count", list(GRID))
@pytest.mark.parametrize("kind", ["project", "load", "scale"])
@pytest.mark.parametrize("D", [128, 256])
def test_tail_tile_counts(D, kind, count):
    """64-token tiles below, at, one above and 2 SMs + 5 times the grid; the last tile holds 1 or 63 tokens.  At D = 256 the
    3-slot weight ring drifts against the 4 (8 with the projected gate) chunks of every tile; at D = 128 a loaded gate or a
    scale uses 2 chunks of 8 slots"""
    tiles = GRID[count](_sms())
    T = (tiles - 1) * 64 + TAIL_RES[(list(GRID).index(count) + D // 128) % 2]
    tail_case(f"fused tail D{D} {kind} {count} T{T}", D, kind, 1, T, seed=T + D + len(kind))


@pytest.mark.parametrize("D", [128, 256])
def test_tail_scale_const(D):
    """the outer mean without a mask: O * scale_const for every token"""
    T = (2 * _sms() + 5 - 1) * 64 + 63
    tail_case(f"fused tail D{D} scale_const T{T}", D, "scale", 1, T, seed=D, use_scale=False)


@pytest.mark.parametrize("kind", ["project", "load", "scale"])
def test_tail_c2(kind):
    """the C2 tail: B 1, N 256, D 256 (rows 256 x n 256)"""
    tail_case(f"fused tail C2 {kind}", 256, kind, 256, 256, seed=len(kind))


# ------------------------------------------------------------------------------------------------------------------------
# C. attention with in-kernel projections (af2_attention_proj_bf16): one item per (folded row, head)
# ------------------------------------------------------------------------------------------------------------------------
def _attn_weights(heads, dh, d, g):
    """w_qkv with the q rows scaled by dim_head^-0.5 log2 e, as pack_attention folds them; w_gate, b_gate"""
    I = heads * dh
    wqkv = torch.randn(3 * I, d, generator=g) * d ** -0.5
    wqkv[:I] *= dh ** -0.5 * 1.4426950408889634
    wg = torch.randn(I, d, generator=g) * d ** -0.5
    return wqkv.to("cuda", torch.bfloat16), wg.to("cuda", torch.bfloat16), torch.randn(I, generator=g).cuda()


def _mask_bn(kind, nbatch, n, g):
    if kind == "mixed":
        return _mixed_mask(nbatch, n, g)
    if kind == "ragged":
        return _ragged_suffix(nbatch, n, g)
    return _mask(kind, nbatch, n, g)


def _proj_call(xn, d, wqkv, wg, bg, bias, mask_tok, n, nbatch, heads, dh, tok_sb, tok_si):
    """af2_attention_proj_bf16 into a NaN-guarded output; returns (guarded buffer, output view, launches)"""
    L, ops = _lib(), _ops()
    lib = L.load()
    T, I = xn.shape[0], heads * dh
    buf, out = _guarded(T * I, torch.bfloat16)
    m = None if mask_tok is None else mask_tok.to(torch.uint8).contiguous()
    torch.cuda.synchronize()
    before = lib.af2_launch_count()
    L.check(lib.af2_attention_proj_bf16(xn.data_ptr(), d, wqkv.data_ptr(), wg.data_ptr(), bg.data_ptr(),
                                        None if bias is None else bias.data_ptr(), None if m is None else m.data_ptr(),
                                        out.data_ptr(), n, nbatch, heads, dh, tok_sb, tok_si, ops._stream_ptr()))
    torch.cuda.synchronize()
    return buf, out.view(T, I), lib.af2_launch_count() - before


def attn_case(name, n, nbatch, heads, dh, d, row, bias, mask, seed):
    """mask: a test_gpu_attention_kernel mask kind, "mixed", "ragged" or "none" """
    from test_gpu_attention_proj import _unfused
    g = torch.Generator().manual_seed(seed)
    T, I = n * nbatch, heads * dh
    xn = torch.randn(T, d, generator=g).to("cuda", torch.bfloat16)
    wqkv, wg, bg = _attn_weights(heads, dh, d, g)
    bt = None
    if bias:
        bt = torch.full((heads, n, (n + 7) // 8 * 8), NAN)    # pad columns must never reach an output
        bt[:, :, :n] = torch.randn(heads, n, n, generator=g) * 2.0
        bt = bt.to("cuda", torch.bfloat16)
    idx, tok_sb, tok_si = _tok(nbatch, n, row)
    m_bn = _mask_bn(mask, nbatch, n, g)
    mask_tok = None
    if m_bn is not None:
        mask_tok = torch.empty(T, dtype=torch.bool, device="cuda")
        mask_tok[idx.flatten()] = m_bn.cuda().flatten()
    buf, out, launches = _proj_call(xn, d, wqkv, wg, bg, bt, mask_tok, n, nbatch, heads, dh, tok_sb, tok_si)
    assert launches == 1, "one attention_proj_kernel launch"                                              # (a)
    _guards_intact(buf, T * I, name)
    ref, bound = FB.attention_proj_ref(xn, wqkv, wg, bg, bt, m_bn, n, nbatch, heads, dh, idx)
    check_bound(name, out, ref, bound)                                                                     # (b)
    del ref, bound
    _same(out, _unfused(xn, wqkv, wg, bg, n, nbatch, heads, dh, tok_sb, tok_si, bt, mask_tok),
          f"{name} against the unfused sequence")                                                          # (c)
    _same(_proj_call(xn, d, wqkv, wg, bg, bt, mask_tok, n, nbatch, heads, dh, tok_sb, tok_si)[1], out,
          f"{name} second launch")                                                                         # (d)


def _rc(row):
    return "row" if row else "col"


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
@pytest.mark.parametrize("count", list(GRID))
def test_attn_item_counts(count, row, dh):
    """items (folded row, head) below, at, one above and 2 SMs + 5 times the grid; n ends mid key block (100: 4 stages,
    257: 3 stages at dim_head 64) and neighbouring rows carry different masks"""
    items = GRID[count](_sms())
    n = 257 if count == "many" else 100
    attn_case(f"fused attn items {count} n{n} b{items} dh{dh} {_rc(row)}", n, items, 1, dh, 128, row, True, "mixed",
              seed=items + dh + row)


@pytest.mark.parametrize("n,d", [(100, 64), (128, 192), (37, 192)])
def test_attn_ring_drift(n, d):
    """dim_head 64, n <= 128: each item consumes 2 ceil(d / 64) = 2 or 6 stages of the 4-stage ring, so the ring position
    shifts from item to item; 2 SMs + 5 items and more"""
    heads = 3
    nbatch = (2 * _sms() + 5 + heads - 1) // heads
    attn_case(f"fused attn drift n{n} d{d} b{nbatch}", n, nbatch, heads, 64, d, n != 128, True, "mixed", seed=n + d)


def test_attn_ring_drift_dh32():
    """dim_head 32 with 896 < n <= 1024 runs on 3 stages; an item consumes 2 * 8 stages at d = 64 (16 = 1 mod 3)"""
    n = min(1000, _ops().attention_proj_max_n(32))
    assert n > 896
    attn_case(f"fused attn drift dh32 n{n}", n, 2 * _sms() + 5, 1, 32, 64, True, True, "ragged", seed=n)


@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
@pytest.mark.parametrize("mask", ["mixed", "ragged", "all_masked", "single"])
def test_attn_masks_per_item(mask, row):
    """consecutive items of one CTA on folded rows with different masks, fully masked rows (row attention) or columns
    (column attention) among them: the key codes of one item must not leak into the next"""
    nbatch = 2 * _sms() + 5
    attn_case(f"fused attn mask {mask} n129 b{nbatch} {_rc(row)}", 129, nbatch, 1, 64, 128, row, True, mask,
              seed=len(mask) + row)


@pytest.mark.parametrize("d", [32, 96, 160])
def test_attn_partial_channel_chunk(d):
    """d not a multiple of 64: the last 64-channel chunk is zero-filled past d"""
    attn_case(f"fused attn d{d}", 129, 2 * _sms() // 3 + 1, 3, 64, d, False, True, "holes", seed=d)


@pytest.mark.parametrize("heads", [1, 3, 8])
def test_attn_heads(heads):
    attn_case(f"fused attn heads{heads}", 200, (2 * _sms() + 5 + heads - 1) // heads, heads, 64, 128, True, True, "mixed",
              seed=heads)


@pytest.mark.parametrize("n", [1, 127, 129, 255, 256, 257, 383, 384])
def test_attn_lengths(n):
    """lengths at the key-block edges; 257 .. 384 run on the 3-stage ring"""
    nbatch = max(1, (2 * _sms() + 5) // 8 + 1)
    attn_case(f"fused attn n{n} b{nbatch}", n, nbatch, 8, 64, 256, n % 2 == 1, True, "mixed", seed=n)


def test_attn_no_bias():
    attn_case("fused attn nobias", 129, 2 * _sms() + 5, 1, 64, 128, True, False, "mixed", seed=5)


# the four attention calls of one Evoformer block at C2 (N_res 256, MSA 128 x 256, heads 8, dim_head 64, dim 256), and the
# C3 pair-row call (N_res 384: 3 stages)
HOT = {"msa_row": (256, 128, True, True), "msa_col": (128, 256, False, False), "tri_start": (256, 256, True, True),
       "tri_end": (256, 256, False, True), "c3_pair_row": (384, 384, True, True)}


@pytest.mark.parametrize("call", list(HOT))
def test_attn_hot_shapes(call):
    n, nbatch, row, bias = HOT[call]
    attn_case(f"fused attn {call}", n, nbatch, 8, 64, 256, row, bias, "ragged", seed=len(call))
