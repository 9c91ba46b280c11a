"""-m gpu: axial attention with the q, k, v and gate projections inside the kernel (attention_proj.cuh), bitwise against the
unfused sequence it replaces.

The fused kernel accumulates every projected element in the projection GEMM's k order and rounds it to bf16 where the GEMM
epilogue does, then runs the attention kernel's softmax and PV code, so its output must equal, bit for bit:
    qkv  = af2_gemm_bf16_epilogue(xn, w_qkv)                       (bf16 store)
    gate = af2_gemm_bf16_epilogue(xn, w_gate, bias b_gate, sigmoid)  (bf16 store)
    og   = af2_attention_bf16(qkv, gate, bias, mask)
The module entries (af2_axial_attention{,_ex}) take the fused kernel whenever a call fits it; the calls that do not (tied
queries, dim_head 16 / 128, n above the bound) keep the unfused launches.  Both are checked bitwise against the same
sequence run through the exported building blocks, and by their launch counts.
"""
import pytest
import torch

from test_gpu_attention_kernel import _mask, _tok

pytestmark = pytest.mark.gpu


def _ops():
    from alphafold2_b200 import ops
    return ops


def _pick_bn(n):
    return 256 if n > 128 else (128 if n > 64 else 64)


def _weights(heads, dh, d, g):
    I = heads * dh
    wqkv = (torch.randn(3 * I, d, generator=g) * d ** -0.5).to("cuda", torch.bfloat16)
    wg = (torch.randn(I, d, generator=g) * d ** -0.5).to("cuda", torch.bfloat16)
    bg = torch.randn(I, generator=g).to("cuda")
    return wqkv, wg, bg


def _unfused(xn, wqkv, wg, bg, n, nbatch, heads, dh, tok_sb, tok_si, bias, mask):
    ops = _ops()
    T = xn.shape[0]
    I = heads * dh
    qkv = torch.empty(T, 3 * I, dtype=torch.bfloat16, device="cuda")
    ops.gemm_bf16_epilogue(xn[None], wqkv[None], qkv, bn=_pick_bn(3 * I), mode=ops.EPI_STORE_BF16, ld_out=3 * I)
    gate = torch.empty(T, I, dtype=torch.bfloat16, device="cuda")
    ops.gemm_bf16_epilogue(xn[None], wg[None], gate, bn=_pick_bn(I), mode=ops.EPI_STORE_BF16, act=ops.ACT_SIGMOID, bias=bg,
                           ld_out=I)
    return ops.attention_bf16(qkv, gate, n, nbatch, heads, dh, tok_sb, tok_si, bias=bias, mask=mask)


def _mask_tok(kind, nbatch, n, idx, g):
    """token-indexed bool mask of a test_gpu_attention_kernel mask kind; "mixed" = holes with every third row fully masked"""
    if kind == "mixed":
        m = torch.rand(nbatch, n, generator=g) >= 0.3
        m[0::3] = False
    elif kind == "ones":
        m = torch.ones(nbatch, n, dtype=torch.bool)
    else:
        m = _mask(kind, nbatch, n, g)
    if m is None:
        return None
    out = torch.empty(n * nbatch, dtype=torch.bool, device="cuda")
    out[idx.flatten()] = m.cuda().flatten()
    return out


def check_fused(n, nbatch, heads, dh, d, row, bias, mask_kind, seed):
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    T = n * nbatch
    xn = torch.randn(T, d, generator=g).to("cuda", torch.bfloat16)
    wqkv, wg, bg = _weights(heads, dh, d, g)
    bt = None
    if bias:
        npad = (n + 7) // 8 * 8
        bt = torch.full((heads, n, npad), float("nan"))   # pad columns must never reach an output
        bt[:, :, :n] = torch.randn(heads, n, n, generator=g) * 2.0
        bt = bt.to("cuda", torch.bfloat16)
    idx, tok_sb, tok_si = _tok(nbatch, n, row)
    mask = _mask_tok(mask_kind, nbatch, n, idx, g)
    out = ops.attention_proj_bf16(xn, wqkv, wg, bg, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask)
    ref = _unfused(xn, wqkv, wg, bg, n, nbatch, heads, dh, tok_sb, tok_si, bt, mask)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    diff = (out.view(torch.int16) != ref.view(torch.int16)).sum().item()
    assert diff == 0, f"n{n} b{nbatch} h{heads} dh{dh} d{d} {'row' if row else 'col'}: {diff} of {out.numel()} elements differ"


def _bound(dh):
    return _ops().attention_proj_max_n(dh)


def test_bound():
    """K and V of every key stay in shared memory: n <= 384 at dim_head 64 (all four C2 calls: n = 256 and 128)"""
    assert _bound(64) == 384
    assert _bound(32) >= 768
    assert _bound(16) == 0 and _bound(128) == 0


@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
@pytest.mark.parametrize("n", [1, 7, 63, 64, 65, 127, 128, 129, 255, 256, "bound"])
def test_fused_lengths(n, row):
    n = _bound(64) if n == "bound" else n
    check_fused(n, 3 if n <= 256 else 2, 8, 64, 256, row, True, "mixed", seed=n + 7 * row)


@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("d", [64, 128, 256])
@pytest.mark.parametrize("heads", [1, 3, 8])
def test_fused_heads_dims(heads, d, bias):
    check_fused(129, 2, heads, 64, d, False, bias, "holes", seed=heads * 1000 + d + bias)


@pytest.mark.parametrize("mask", ["none", "ones", "holes", "all_masked", "single", "first_block", "straddle"])
def test_fused_masks(mask):
    check_fused(256, 4, 8, 64, 256, False, True, mask, seed=len(mask))


@pytest.mark.parametrize("n", [65, 256, "bound"])
def test_fused_dim_head_32(n):
    n = _bound(32) if n == "bound" else n
    check_fused(n, 2, 3, 32, 128, True, True, "mixed", seed=n)


@pytest.mark.parametrize("dh,n", [(64, "above"), (16, 64), (128, 64)])
def test_fused_refuses(dh, n):
    """n above the bound and dim_head 16 / 128 are refused (the module entries keep the unfused path for them)"""
    ops = _ops()
    n = _bound(64) + 1 if n == "above" else n
    g = torch.Generator().manual_seed(1)
    xn = torch.randn(n, 64, generator=g).to("cuda", torch.bfloat16)
    wqkv, wg, bg = _weights(2, dh, 64, g)
    with pytest.raises(Exception):
        ops.attention_proj_bf16(xn, wqkv, wg, bg, n, 1, 2, dh, n, 1)


# ----------------------------------------------------------------------------------------------------------------------
# module entries: the fused path where it applies, the unfused one elsewhere, both bitwise the unfused sequence
# ----------------------------------------------------------------------------------------------------------------------
def _module_ref(pk, x, mask, heads, dh, row):
    """af2_axial_attention without edges through the exported building blocks: LayerNorm, the two projection GEMMs, the
    attention kernel per batch element and to_out + bias + residual"""
    ops = _ops()
    t = pk.tensors
    B, h, w, d = x.shape
    I = heads * dh
    T = B * h * w
    n, nb = (w, h) if row else (h, w)
    tok_sb, tok_si = (w, 1) if row else (1, w)
    xn = ops.layernorm_bf16(x.reshape(T, d), t["g"], t["b"]).reshape(T, d)
    og = torch.empty(T, I, dtype=torch.bfloat16, device="cuda")
    for b in range(B):
        sl = slice(b * h * w, (b + 1) * h * w)
        mb = mask.reshape(T)[sl] if mask is not None else None
        og[sl] = _unfused(xn[sl].contiguous(), t["wqkv"], t["wg"], t["bg"], n, nb, heads, dh, tok_sb, tok_si, None, mb)
    y = x.clone().reshape(T, d)
    ops.gemm_bf16_epilogue(og[None], t["wo"][None], y, bn=_pick_bn(d), mode=ops.EPI_RESID_F32, bias=t["bo"], resid=y, ld_resid=d,
                           ld_out=d)
    return y.reshape(B, h, w, d)


def _pack(heads, dh, d, g):
    ops = _ops()
    I = heads * dh
    r = lambda *s: torch.randn(*s, generator=g).cuda()   # noqa: E731
    return ops.pack_attention(1.0 + 0.1 * r(d), 0.1 * r(d), r(I, d) * d ** -0.5, r(2 * I, d) * d ** -0.5, r(I, d) * d ** -0.5,
                              r(I), r(d, I) * I ** -0.5, r(d), None, dh)


@pytest.mark.parametrize("case", ["fused", "fused_b2", "col", "above_bound", "dh16", "dh128", "tied"])
def test_module_paths(case):
    """the module entry's output is bitwise the unfused sequence's, and it launches the fused kernel exactly where it fits:
    LayerNorm, one fused attention per batch element and to_out, against LayerNorm, the two projection GEMMs, (the query
    tying and) one attention per batch element and to_out"""
    from alphafold2_b200 import _lib
    ops = _ops()
    lib = _lib.load()
    B, heads, dh, d, row, tied = 1, 4, 64, 128, True, False
    n, nb = 200, 5
    if case == "fused_b2":
        B = 2
    elif case == "col":
        row = False
    elif case == "above_bound":
        n = _bound(64) + 1
    elif case == "dh16":
        dh = 16
    elif case == "dh128":
        dh = 128
    elif case == "tied":
        tied = True
        row = False
    fused = case in ("fused", "fused_b2", "col")
    g = torch.Generator().manual_seed(len(case) * 31 + ord(case[-1]))
    pk = _pack(heads, dh, d, g)
    shape = (B, nb, n, d) if row else (B, n, nb, d)
    x = torch.randn(*shape, generator=g).cuda()
    mask = torch.rand(*shape[:3], generator=g) >= 0.2
    mask[:, 0] = False                                   # fully masked rows (row attention) or columns' first query
    mask = mask.cuda()
    y = x.clone()
    torch.cuda.synchronize()
    before = lib.af2_launch_count()
    ops.axial_attention_(pk, y, heads, dh, row, mask=mask, tied=tied)
    launches = lib.af2_launch_count() - before
    assert launches == (2 + B if fused else 4 + B + (B if tied else 0)), (case, launches)
    if tied:
        return   # tied queries: the unfused path (launch count above); tests/test_gpu_tied_attention_parts.py checks its bits
    ref = _module_ref(pk, x, mask, heads, dh, row)
    torch.cuda.synchronize()
    diff = (y.view(torch.int32) != ref.view(torch.int32)).sum().item()
    assert diff == 0, f"{case}: {diff} of {y.numel()} elements differ"
