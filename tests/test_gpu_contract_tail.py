"""-m gpu: the fused tail of the triangle multiplications and the outer mean (contract_tail.cuh), bitwise against the
launches it replaces.

contract_tail_kernel computes x += tail(O) w_out^T + b_out in one launch, where the unfused path runs
    [gate = bf16(sigmoid(xn w_ogate^T + b_ogate))    out-gate GEMM, EK_STORE_TOK_SIG]
    y = chan_to_token(O, gate | scale)                chan_to_token_tma_kernel
    x = (y w_out^T + b_out) + x                       to_out GEMM, EK_RESID_F32
It accumulates each projected element in the GEMM's k order, rounds where the GEMM epilogues and chan_to_token round, and
takes chan_to_token's LayerNorm arithmetic, so x must come out bit for bit the same.  Checked per variant (projected gate,
loaded gate, scale) through af2_contract_tail, per module (af2_triangle_multiply, af2_outer_mean) against the same module
run from its stage entries with the unfused tail, and by launch counts where the fused path must and must not run.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops():
    from alphafold2_b200 import ops
    return ops


def _lib():
    from alphafold2_b200 import _lib
    return _lib


def _pick_bn(n):
    return 256 if n > 128 else (128 if n > 64 else 64)


def _a(n, m):
    return (n + m - 1) // m * m


def _weights(d, g):
    w = lambda *s: (torch.randn(*s, generator=g) * d ** -0.5).to("cuda", torch.bfloat16)   # noqa: E731
    f = lambda *s: torch.randn(*s, generator=g).to("cuda")                                 # noqa: E731
    return dict(wog=w(d, d), bog=f(d), wo=w(d, d), bo=f(d), gamma=1 + 0.1 * f(d), beta=0.1 * f(d))


def _case(rows, n, d, g, *, chan_stride=None, pitch=None, src_off=0):
    pitch = n if pitch is None else pitch
    cs = rows * pitch if chan_stride is None else chan_stride
    src = torch.randn(src_off + d * cs, generator=g).mul_(3.0).add_(0.5).to("cuda")
    T = rows * n
    xn = torch.randn(T, d, generator=g).to("cuda", torch.bfloat16)
    gate = torch.rand(T, d, generator=g).to("cuda", torch.bfloat16)
    x = torch.randn(T, d, generator=g).to("cuda")
    scale = (torch.rand(T, generator=g) + 0.5).to("cuda")
    return dict(src=src, cs=cs, pitch=pitch, xn=xn, gate=gate, x=x, scale=scale, T=T)


def _run(c, w, rows, n, d, variant, kind, *, src_off=0, x=None, x_off=0, use_scale=True, bias=True):
    """one af2_contract_tail call on a copy of x; returns (x, path that ran, launches)"""
    ops = _ops()
    x = (c["x"] if x is None else x).clone()
    y = torch.empty(c["T"] * d, dtype=torch.bfloat16, device="cuda")
    kw = dict(chan_stride=c["cs"], pitch=c["pitch"], rows=rows, n=n, d=d, variant=variant, src_off=src_off, x_off=x_off)
    if kind == "scale":
        kw.update(mode=1, scale=c["scale"] if use_scale else None, scale_const=0.125)
    else:
        kw.update(mode=0, gamma=w["gamma"], beta=w["beta"], gate=c["gate"].clone())
        if kind == "project":
            kw.update(xn=c["xn"], w_ogate=w["wog"], b_ogate=w["bog"] if bias else None)
    lib = _lib().load()
    before = lib.af2_launch_count()
    ran = ops.contract_tail(c["src"], x, w["wo"], w["bo"] if bias else None, y, **kw)
    torch.cuda.synchronize()
    return x, ran, lib.af2_launch_count() - before


def _same(a, b):
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"max |diff| {(a - b).abs().max().item():.3e}"


@pytest.mark.parametrize("d", [128, 256])
@pytest.mark.parametrize("kind", ["project", "load", "scale"])
@pytest.mark.parametrize("rows,n", [(2, 32), (1, 100), (2, 96), (3, 44), (128, 64)])
def test_fused_equals_unfused(d, kind, rows, n):
    """tile edges (64 tokens, 64 exactly, 200, 192, a partial last tile of 4) and a many-tile grid; batch 2 folds as rows"""
    ops = _ops()
    g = torch.Generator().manual_seed(rows * 1000 + n + d)
    w = _weights(d, g)
    c = _case(rows, n, d, g)
    xf, rf, lf = _run(c, w, rows, n, d, ops.CTAIL_FUSED, kind)
    xu, ru, lu = _run(c, w, rows, n, d, ops.CTAIL_UNFUSED, kind)
    xa, ra, _ = _run(c, w, rows, n, d, ops.CTAIL_AUTO, kind)
    assert (rf, ru, ra) == (ops.CTAIL_FUSED, ops.CTAIL_UNFUSED, ops.CTAIL_FUSED)
    assert lf == 1 and lu == (3 if kind == "project" else 2)
    _same(xf, xu)
    _same(xa, xu)
    assert not torch.equal(xf, c["x"])


@pytest.mark.parametrize("d", [128, 256])
def test_scale_const_and_no_bias(d):
    ops = _ops()
    g = torch.Generator().manual_seed(7 + d)
    w = _weights(d, g)
    c = _case(3, 40, d, g)
    for kind, kw in (("scale", dict(use_scale=False)), ("project", dict(bias=False)), ("load", dict(bias=False))):
        xf, _, _ = _run(c, w, 3, 40, d, ops.CTAIL_FUSED, kind, **kw)
        xu, _, _ = _run(c, w, 3, 40, d, ops.CTAIL_UNFUSED, kind, **kw)
        _same(xf, xu)


@pytest.mark.parametrize("kind", ["load", "scale"])
def test_band_window(kind):
    """a band of rows [row0, row0 + rows) of a larger tensor: O with a longer channel stride, src and x at offsets"""
    ops = _ops()
    d, N, row0, rows = 256, 72, 24, 20
    g = torch.Generator().manual_seed(11)
    w = _weights(d, g)
    c = _case(rows, N, d, g, chan_stride=N * N + 8, src_off=row0 * N)
    big = torch.randn(N * N * d, generator=g).to("cuda")
    c["x"] = big
    kw = dict(src_off=row0 * N, x_off=row0 * N * d)
    xf, rf, _ = _run(c, w, rows, N, d, ops.CTAIL_FUSED, kind, **kw)
    xu, ru, _ = _run(c, w, rows, N, d, ops.CTAIL_UNFUSED, kind, **kw)
    assert (rf, ru) == (ops.CTAIL_FUSED, ops.CTAIL_UNFUSED)
    _same(xf, xu)
    _same(xf[: row0 * N * d], big[: row0 * N * d])
    _same(xf[(row0 + rows) * N * d:], big[(row0 + rows) * N * d:])


@pytest.mark.parametrize("case", ["misaligned_x", "padded_cols", "d64"])
def test_unfused_where_fused_cannot_run(case):
    ops = _ops()
    g = torch.Generator().manual_seed(3)
    if case == "d64":
        d, rows, n, pitch = 64, 2, 40, None
    elif case == "padded_cols":
        d, rows, n, pitch = 128, 3, 42, 44
    else:
        d, rows, n, pitch = 128, 2, 40, None
    w = _weights(d, g)
    c = _case(rows, n, d, g, pitch=pitch)
    x_off = 1 if case == "misaligned_x" else 0
    xbig = torch.randn(c["T"] * d + x_off, generator=g).to("cuda")
    xa, ra, la = _run(c, w, rows, n, d, ops.CTAIL_AUTO, "load", x=xbig, x_off=x_off)
    xu, ru, _ = _run(c, w, rows, n, d, ops.CTAIL_UNFUSED, "load", x=xbig, x_off=x_off)
    assert ra == ops.CTAIL_UNFUSED and la == 2
    _same(xa, xu)
    with pytest.raises(ValueError):
        _run(c, w, rows, n, d, ops.CTAIL_FUSED, "load", x=xbig, x_off=x_off)


# ---------------------------------------------------------------------------------------------------------------------
# module level: the whole-module entries (fused tail, projected gate) against the module rebuilt from its stage entries
# with the unfused tail
# ---------------------------------------------------------------------------------------------------------------------
def _trimul_pack(d, g):
    ops = _ops()
    r = lambda *s: (torch.randn(*s, generator=g) * d ** -0.5).to("cuda")   # noqa: E731
    v = lambda *s: (0.1 * torch.randn(*s, generator=g)).to("cuda")         # noqa: E731
    return ops.pack_triangle_multiply(1 + v(d), v(d), r(d, d), v(d), r(d, d), v(d), r(d, d), v(d), r(d, d), v(d), r(d, d),
                                      v(d), 1 + v(d), v(d), r(d, d), v(d))


def _trimul_unfused(pk, x, mask, ingoing):
    ops, L = _ops(), _lib()
    lib = L.load()
    B, N, _, d = x.shape
    T, np8, np4 = B * N * N, _a(N, 8), _a(N, 4)
    cs_lr, cs_o = B * N * np8, B * N * np4
    Lc = torch.zeros(d * cs_lr, dtype=torch.bfloat16, device="cuda")
    Rc = torch.zeros_like(Lc)
    gate = torch.empty(T * d, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(lib.af2_triangle_project_workspace(T, d), dtype=torch.uint8, device="cuda")
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    L.check(lib.af2_triangle_project(C.byref(pk.struct), x.data_ptr(), None if m is None else m.data_ptr(), T, N, d,
                                     Lc.data_ptr(), Rc.data_ptr(), cs_lr, gate.data_ptr(), ws.data_ptr(), ws.numel(), None))
    Oc = torch.empty(d * cs_o, dtype=torch.float32, device="cuda")
    for b in range(B):
        a, bb = (Rc, Lc) if ingoing else (Lc, Rc)
        ops.gemm_bf16_f32_strided(a, bb, Oc, M=N, N=N, K=N, batch=d, mn_major=bool(ingoing), bn=_pick_bn(N), lda=np8,
                                  a_batch=cs_lr, ldb=np8, b_batch=cs_lr, ldc=np4, c_batch=cs_o, a_off=b * N * np8,
                                  b_off=b * N * np8, c_off=b * N * np4)
    y = torch.empty(T * d, dtype=torch.bfloat16, device="cuda")
    t = pk.tensors
    ran = ops.contract_tail(Oc, x, t["wo"], t["bo"], y, chan_stride=cs_o, pitch=np4, rows=B * N, n=N, d=d, mode=0,
                            gamma=t["ong"], beta=t["onb"], gate=gate, variant=ops.CTAIL_UNFUSED)
    assert ran == ops.CTAIL_UNFUSED
    return x


@pytest.mark.parametrize("B,N,d", [(1, 256, 256), (2, 72, 128)])
@pytest.mark.parametrize("ingoing", [0, 1])
@pytest.mark.parametrize("masked", [False, True])
def test_triangle_multiply_module(B, N, d, ingoing, masked):
    ops = _ops()
    g = torch.Generator().manual_seed(B * 100 + N + ingoing)
    pk = _trimul_pack(d, g)
    x = torch.randn(B, N, N, d, generator=g).to("cuda")
    mask = (torch.rand(B, N, N, generator=g) > 0.2).to("cuda") if masked else None
    lib = _lib().load()
    before = lib.af2_launch_count()
    xf = ops.triangle_multiply_(pk, x.clone(), bool(ingoing), mask)
    torch.cuda.synchronize()
    launches = lib.af2_launch_count() - before
    # LayerNorm, [mask to float], left / right GEMMs, one contraction per batch element, the fused tail
    assert launches == 1 + int(masked) + 2 + B + 1
    xu = _trimul_unfused(pk, x.clone(), mask, ingoing)
    torch.cuda.synchronize()
    _same(xf, xu)


def _outer_pack(d, g):
    ops = _ops()
    r = lambda *s: (torch.randn(*s, generator=g) * d ** -0.5).to("cuda")   # noqa: E731
    v = lambda *s: (0.1 * torch.randn(*s, generator=g)).to("cuda")         # noqa: E731
    return ops.pack_outer_mean(1 + v(d), v(d), r(d, d), v(d), r(d, d), v(d), r(d, d), v(d))


def _outer_unfused(pk, x, m, msa_mask, eps):
    ops, L = _ops(), _lib()
    lib = L.load()
    B, S, N, d = m.shape
    Tm, np8, np4 = B * S * N, _a(N, 8), _a(N, 4)
    cs_lr, cs_o = B * S * np8, B * N * np4
    scale = torch.empty(B * N * N, dtype=torch.float32, device="cuda")
    words = torch.empty((S + 31) // 32 * N, dtype=torch.int32, device="cuda")
    if msa_mask is not None:
        for b in range(B):
            ops.outer_scale(msa_mask[b], scale[b * N * N:(b + 1) * N * N], row0=0, rows=N, eps=eps, words=words)
    LRc = torch.zeros(2 * d * cs_lr, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(lib.af2_outer_project_workspace(Tm, d), dtype=torch.uint8, device="cuda")
    mm = None if msa_mask is None else msa_mask.to(torch.uint8).contiguous()
    L.check(lib.af2_outer_project(C.byref(pk.struct), m.data_ptr(), None if mm is None else mm.data_ptr(), Tm, N, d,
                                  LRc.data_ptr(), cs_lr, ws.data_ptr(), ws.numel(), None))
    Oc = torch.empty(d * cs_o, dtype=torch.float32, device="cuda")
    for b in range(B):
        ops.gemm_bf16_f32_strided(LRc, LRc, Oc, M=N, N=N, K=S, batch=d, mn_major=True, bn=_pick_bn(N), lda=np8,
                                  a_batch=cs_lr, ldb=np8, b_batch=cs_lr, ldc=np4, c_batch=cs_o, a_off=b * S * np8,
                                  b_off=d * cs_lr + b * S * np8, c_off=b * N * np4)
    y = torch.empty(B * N * N * d, dtype=torch.bfloat16, device="cuda")
    t = pk.tensors
    ran = ops.contract_tail(Oc, x, t["wo"], t["bo"], y, chan_stride=cs_o, pitch=np4, rows=B * N, n=N, d=d, mode=1,
                            scale=scale if msa_mask is not None else None, scale_const=1.0 / S, variant=ops.CTAIL_UNFUSED)
    assert ran == ops.CTAIL_UNFUSED
    return x


@pytest.mark.parametrize("B,S,N,d", [(1, 128, 256, 256), (2, 12, 68, 128)])
@pytest.mark.parametrize("masked", [False, True])
def test_outer_mean_module(B, S, N, d, masked):
    ops = _ops()
    g = torch.Generator().manual_seed(S + N + int(masked))
    pk = _outer_pack(d, g)
    x = torch.randn(B, N, N, d, generator=g).to("cuda")
    m = torch.randn(B, S, N, d, generator=g).to("cuda")
    msa_mask = (torch.rand(B, S, N, generator=g) > 0.2).to("cuda") if masked else None
    xf = ops.outer_mean_(pk, x.clone(), m, msa_mask, 1e-5)
    xu = _outer_unfused(pk, x.clone(), m, msa_mask, 1e-5)
    torch.cuda.synchronize()
    _same(xf, xu)
