"""-m gpu: the second half of the triangle-multiply and outer-mean modules, kernel by kernel, element-wise against fp64:
(A) the per-channel contractions laid out as the modules issue them, (B) the same contractions over gathered operand
pieces (the sharded schedule's rank-4 tensor maps), (C) the channel-major -> token-major kernels (SIMT, tile, TMA) and
(D) the OuterMean normaliser (byte loop, bit-packed).

References are fp64, evaluated on the GPU with plain torch from the exact bf16 / fp32 operands the kernel was given.  Every
element is gated by a bound derived from the kernel's rounding (below); the worst err / bound of each case goes to the
parity report.  Output buffers start as NaN, and every element outside the valid output must still be NaN afterwards.
u = 2^-24 is the fp32 unit roundoff, 2^-8 the bf16 one.

A / B. Contractions (bf16 operands, fp32 accumulation over K terms, fp32 store): gpu_util.gemm_f32_bound,
    |out - ref| <= C_GEMM K u sum_k |a_k b_k| + 2 u |ref|
  Lc / Rc are channel-major [d][B * rows][align8(cols)] with B = 2 (a batch offset inside the channel and a channel stride
  far larger than M K), Oc is [d][B * N][align4(N)].  The pad columns of Lc / Rc hold NaN: the tensor maps stop at the
  logical extent, so the contractions never read them (any read would make an output NaN).  The modules' memsets of the
  pads are therefore not needed by the contractions.  Gathered pieces sit further apart than their size, and the gap holds
  NaN, so reading past a piece shows up; the gathered launch must also match, bit for bit, the same GEMM with the same tile
  width over the concatenated operand, since only the addressing differs.

C. Channel -> token.  Mode 1: y = bf16(fl(x * s)):  |y - ref| <= 2^-8 |ref| + 2 u |ref|.
  Mode 0: y = bf16(((x_c - mean) rstd w_c + b_c) g_c) with fp32 two-pass moments.  Each kernel sums the d channels in a
  tree of depth at most k_d = max(d/32 + 5 (SIMT: d/32 per lane + 5 shuffle levels), d/8 + 8 (tile: d/8 per thread + 8
  partials), 32 + d/32 (TMA: 32 per thread + d/32 partials)), then scales by 1/d (two roundings where 1/d is inexact):
    |dmean|  <= (k_d + 2) u mean_c |x_c|
    |dxhat_c| <= rstd (|dmean| + u |x_c - mean|) + |xhat_c| (k_d + 3) u + |xhat_c| (rstd dmean)^2 / 2
  The (k_d + 3) u term bounds the variance sum of squares (depth k_d, one rounding per square), the 1/d and + eps
  roundings, the rsqrtf error (2 ulp) and the product (x - mean) rstd; the relative variance error is halved by the square
  root.  The last term is the variance bias of a shifted mean (sum (x - mean')^2 = sum (x - mean)^2 + d dmean^2).  Then
  three fp32 roundings (* w, + b, * g) and the bf16 store:
    |y - ref| <= 2^-8 |ref| + |g_c| (|w_c| |dxhat_c| + 3 u (|xhat_c w_c| + |b_c|))
  Channel values have mean 1e3 and unit spread, so a one-pass E[x^2] - mean^2 variance fails by orders of magnitude.  A
  token whose channels are all equal (1024: its fp32 sum and mean are exact in every kernel) must give exactly
  bf16(fl(b_c g_c)).  Gates hold exact zeros and negative values.

D. OuterMean normaliser: scale = 1 / fl(S fl(cnt + eps)) with cnt exact: three fp32 roundings,
    |scale - ref| <= 4 u |ref|       (IEEE division: the library is built without fast math)
  The byte-loop and bit-packed kernels count the same integers, so they must agree bit for bit.

Every test that forces a kernel first lets the host decide whether it may run: a forced kernel whose preconditions the call
does not meet raises ValueError and launches nothing (the output stays NaN).
"""
import pytest
import torch

from gpu_util import U32 as U, check_bound, gemm_f32_bound

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 64


def _ops():
    from alphafold2_b200 import ops
    return ops


def _al(v, a):
    return (v + a - 1) // a * a


def _pick_bn(n):
    """the tile width the modules use for n output columns (api.cu pick_bn)"""
    return 256 if n > 128 else (128 if n > 64 else 64)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _gemm_ref(a, b, K):
    """a [batch, M, K], b [batch, N, K] fp64 -> (a b^T, gemm_f32_bound)"""
    ref = a @ b.transpose(1, 2)
    return ref, gemm_f32_bound(a.abs() @ b.abs().transpose(1, 2), K, ref)


# ------------------------------------------------------------------------------------------------------------------------
# A. per-channel contractions as af2_triangle_multiply / af2_outer_mean issue them
# ------------------------------------------------------------------------------------------------------------------------
def _contraction(kind, N, d, S=None, B=2, seed=0):
    ops = _ops()
    g = _gen(seed)
    np8, np4 = _al(N, 8), _al(N, 4)
    inner = S if kind == "outer" else N                 # rows per batch element of Lc / Rc: k (outgoing) / the MSA depth
    cs_lr, cs_o = B * inner * np8, B * N * np4

    def operand():
        t = torch.randn(d, B * inner, np8, generator=g, device="cuda").bfloat16()
        t[:, :, N:] = NAN
        return t

    Lc, Rc = operand(), operand()
    Oc = torch.full((d * cs_o,), NAN, device="cuda")
    K = S if kind == "outer" else N
    refs, bounds = [], []
    for b in range(B):
        off = b * inner * np8
        if kind == "outgoing":     # O_c = L_c R_c^T, both K-major
            A, Bm, mn = Lc, Rc, False
        elif kind == "ingoing":    # O_c = R_c^T L_c, both MN-major
            A, Bm, mn = Rc, Lc, True
        else:                      # O_c = L_c^T R_c over the S sequences, both MN-major
            A, Bm, mn = Lc, Rc, True
        ops.gemm_bf16_f32_strided(A, Bm, Oc, M=N, N=N, K=K, batch=d, mn_major=mn, bn=_pick_bn(N), lda=np8, a_batch=cs_lr,
                                  ldb=np8, b_batch=cs_lr, ldc=np4, c_batch=cs_o, a_off=off, b_off=off, c_off=b * N * np4)
        a64 = A[:, b * inner:(b + 1) * inner, :N].double()
        b64 = Bm[:, b * inner:(b + 1) * inner, :N].double()
        if mn:
            a64, b64 = a64.transpose(1, 2), b64.transpose(1, 2)
        r, bd = _gemm_ref(a64, b64, K)
        refs.append(r)
        bounds.append(bd)
    torch.cuda.synchronize()
    O = Oc.view(d, B, N, np4)
    check_bound(f"contraction {kind} N{N} d{d}" + (f" S{S}" if S else ""), O[..., :N],
                torch.stack(refs, 1), torch.stack(bounds, 1))
    assert torch.isnan(O[..., N:]).all(), "write into the pad columns of Oc"


@pytest.mark.parametrize("d", [128, 256])
@pytest.mark.parametrize("N", [37, 44, 64, 136, 300, 384])
@pytest.mark.parametrize("kind", ["outgoing", "ingoing"])
def test_triangle_contraction(kind, N, d):
    _contraction(kind, N, d, seed=N * 7 + d + (kind == "ingoing"))


@pytest.mark.parametrize("kind", ["outgoing", "ingoing"])
def test_triangle_contraction_d32(kind):
    _contraction(kind, 44, 32, seed=3)


OUTER_SHAPES = ([(128, N, S) for N in (37, 44, 64, 136, 300, 384) for S in (1, 5, 33, 128)] +
                [(128, 37, 1030), (128, 136, 1030), (128, 300, 1030),
                 (256, 44, 5), (256, 64, 33), (256, 300, 1), (256, 384, 128), (256, 136, 1030), (32, 37, 33)])


@pytest.mark.parametrize("d,N,S", OUTER_SHAPES)
def test_outer_contraction(d, N, S):
    _contraction("outer", N, d, S=S, seed=N + S + d)


# ------------------------------------------------------------------------------------------------------------------------
# B. gathered operand pieces (af2_triangle_contract / af2_outer_contract with pieces > 1)
# ------------------------------------------------------------------------------------------------------------------------
def _piece_buffer(parts, gap):
    """pieces [d][r][w] bf16, each stored with channel stride r * w + 8 and followed by `gap` NaN elements
    -> (flat buffer, channel stride, piece stride)"""
    d, r, w = parts[0].shape
    cs = r * w + 8
    piece = d * cs + gap
    buf = torch.full((len(parts) * piece,), NAN, dtype=torch.bfloat16, device="cuda")
    for p, t in enumerate(parts):
        buf[p * piece:p * piece + d * cs].view(d, cs)[:, :r * w] = t.reshape(d, r * w)
    return buf, cs, piece


def _nan_pad(t, width):
    """[..., w] -> [..., width] with NaN columns past w"""
    out = torch.full(t.shape[:-1] + (width,), NAN, dtype=t.dtype, device=t.device)
    out[..., :t.shape[-1]] = t
    return out.contiguous()


def _gathered(case, pc, M, N, K, d, bn, seed):
    """case: 'outgoing' (K-major, B pieces of pc rows), 'ingoing' (MN-major, A pieces of pc columns), 'outer' (MN-major,
    B pieces of pc columns), 'kmajor_a' (K-major, A pieces of pc rows)"""
    ops = _ops()
    g = _gen(seed)
    mn = case in ("ingoing", "outer")
    a_log = torch.randn(d, M, K, generator=g, device="cuda").bfloat16()       # logical A [c][m][k], B [c][n][k]
    b_log = torch.randn(d, N, K, generator=g, device="cuda").bfloat16()
    ldc = _al(N, 4)

    def stored(t):                      # the contiguous operand as the kernel reads it: [c][rows][align8(K)] or [c][K][align8(rows)]
        t = t.transpose(1, 2) if mn else t
        return _nan_pad(t, _al(t.shape[-1], 8))

    def piece_buf(t, pr):               # the same operand split along rows / columns: piece p = [c][pr][align8(K)] or [c][K][align8(pr)]
        parts = [t[:, p * pr:(p + 1) * pr] for p in range(t.shape[1] // pr)]
        parts = [_nan_pad(q.transpose(1, 2), _al(pr, 8)) if mn else _nan_pad(q, _al(K, 8)) for q in parts]
        buf, cs, piece = _piece_buffer(parts, 8 * (3 if mn else 5))
        return buf, parts[0].shape[-1], cs, piece

    A_c, B_c = stored(a_log), stored(b_log)
    plain = dict(M=M, N=N, K=K, batch=d, mn_major=mn, bn=bn, ldc=ldc, c_batch=M * ldc + 4)
    pa = dict(lda=A_c.shape[-1], a_batch=A_c.shape[1] * A_c.shape[2])
    pb = dict(ldb=B_c.shape[-1], b_batch=B_c.shape[1] * B_c.shape[2])
    a_src, b_src = A_c, B_c
    if case in ("ingoing", "kmajor_a"):
        a_src, lda, cs, piece = piece_buf(a_log, pc)
        pa = dict(lda=lda, a_batch=cs, a_pr=pc, a_piece=piece)
    else:
        b_src, ldb, cs, piece = piece_buf(b_log, pc)
        pb = dict(ldb=ldb, b_batch=cs, b_pr=pc, b_piece=piece)
    size = d * plain["c_batch"] + GUARD
    out = torch.full((size,), NAN, device="cuda")
    ops.gemm_bf16_f32_strided(a_src, b_src, out, **plain, **pa, **pb)
    cat = torch.full((size,), NAN, device="cuda")
    ops.gemm_bf16_f32_strided(A_c, B_c, cat, **plain, lda=A_c.shape[-1], a_batch=A_c.shape[1] * A_c.shape[2],
                              ldb=B_c.shape[-1], b_batch=B_c.shape[1] * B_c.shape[2])
    torch.cuda.synchronize()
    O = out[:d * plain["c_batch"]].view(d, -1)[:, :M * ldc].view(d, M, ldc)
    ref, bound = _gemm_ref(a_log.double(), b_log.double(), K)
    check_bound(f"gathered {case} pc{pc} M{M} N{N} K{K} d{d} bn{bn}", O[..., :N], ref, bound)
    valid = torch.zeros(size, dtype=torch.bool, device="cuda")
    valid[:d * plain["c_batch"]].view(d, -1)[:, :M * ldc].view(d, M, ldc)[..., :N] = True
    assert torch.isnan(out[~valid]).all(), "write outside the output"
    assert torch.equal(out[valid].view(torch.int32), cat[valid].view(torch.int32)), \
        "gathered launch differs from the same GEMM over the concatenated operand"


@pytest.mark.parametrize("pc,cols,bn", [(32, 512, None), (64, 512, None), (128, 512, None), (256, 512, None),
                                        (512, 1024, None), (256, 512, 128), (128, 256, 64), (64, 128, None)])
def test_gathered_outgoing_b_pieces(pc, cols, bn):
    """O_c = L_c R_c^T with R gathered as cols / pc pieces of pc rows; bn None = the module's pick_bn(cols).  pc < bn,
    pc == bn and pc > bn (the box spans several pieces / one piece holds several boxes)"""
    _gathered("outgoing", pc, M=200, N=cols, K=100, d=24, bn=bn or _pick_bn(cols), seed=pc + cols)


@pytest.mark.parametrize("pr", [64, 128, 192])
def test_gathered_ingoing_a_pieces(pr):
    """O_c = R_c^T L_c with R (MN-major) gathered as 3 pieces of pr columns"""
    _gathered("ingoing", pr, M=3 * pr, N=100, K=77, d=24, bn=_pick_bn(100), seed=pr)


@pytest.mark.parametrize("pc", [64, 128])
def test_gathered_outer_b_pieces(pc):
    """O_c = L_c^T R_c over S = 33 sequences, R (MN-major) gathered as 4 pieces of pc columns"""
    _gathered("outer", pc, M=50, N=4 * pc, K=33, d=24, bn=_pick_bn(4 * pc), seed=pc + 1)


def test_gathered_kmajor_a_pieces():
    _gathered("kmajor_a", 128, M=256, N=72, K=100, d=8, bn=128, seed=5)


def test_gathered_rejections():
    """documented limits of the rank-4 maps: no launch, ValueError"""
    ops = _ops()
    a = torch.zeros(1 << 16, dtype=torch.bfloat16, device="cuda")
    c = torch.full((1 << 16,), NAN, device="cuda")
    kw = dict(K=64, batch=2, ldc=128, c_batch=128 * 128)
    with pytest.raises(ValueError, match="multiple of 128"):      # K-major A pieces: whole 128-row tiles
        ops.gemm_bf16_f32_strided(a, a, c, M=128, N=128, mn_major=False, bn=128, lda=64, a_batch=8192, ldb=64, b_batch=8192,
                                  a_pr=64, a_piece=4096, **kw)
    with pytest.raises(ValueError, match="multiple of 64"):       # MN-major A pieces: whole 64-column boxes
        ops.gemm_bf16_f32_strided(a, a, c, M=96, N=128, mn_major=True, bn=128, lda=96, a_batch=8192, ldb=128, b_batch=8192,
                                  a_pr=96, a_piece=8192, **kw)
    with pytest.raises(ValueError, match="do not tile BN"):       # K-major B pieces must divide or be divided by bn
        ops.gemm_bf16_f32_strided(a, a, c, M=128, N=192, mn_major=False, bn=256, lda=64, a_batch=8192, ldb=64, b_batch=8192,
                                  b_pr=96, b_piece=8192, **kw)
    with pytest.raises(ValueError, match="do not tile BN"):       # ... in groups of 8 rows
        ops.gemm_bf16_f32_strided(a, a, c, M=128, N=48, mn_major=False, bn=64, lda=64, a_batch=8192, ldb=64, b_batch=8192,
                                  b_pr=4, b_piece=1024, **kw)
    with pytest.raises(ValueError, match="multiple of 64"):       # MN-major B pieces: whole 64-column boxes
        ops.gemm_bf16_f32_strided(a, a, c, M=128, N=128, mn_major=True, bn=128, lda=128, a_batch=8192, ldb=32, b_batch=2048,
                                  b_pr=32, b_piece=4096, **kw)
    torch.cuda.synchronize()
    assert torch.isnan(c).all()


# ------------------------------------------------------------------------------------------------------------------------
# C. channel -> token (af2_chan_to_token)
# ------------------------------------------------------------------------------------------------------------------------
VNAME = {1: "simt", 2: "tile", 3: "tma"}
CONST = 1024.0


def _k_d(d):
    return max(d / 32 + 5, d / 8 + 8, 32 + d / 32)


def _legal(d, N):
    """the kernels the host accepts for a dense (N % 4 == 0) or padded token grid with aligned pointers"""
    v = {1}
    if N % 4 == 0 and d % 64 == 0 and d <= 256:
        v.add(2)
    if N % 4 == 0 and d in (128, 256):
        v.add(3)
    return v


def _c2t_inputs(d, N, B, mode, seed, gate_off=0):
    g = _gen(seed)
    rows, T = B * N, B * N * N
    pitch = _al(N, 4)                                  # the modules' Oc pitch
    cs = rows * pitch + 12
    x = torch.randn(d, T, generator=g, device="cuda") + 1e3
    const = torch.arange(T, device="cuda") % 7 == 3
    x[:, const] = CONST
    src = torch.full((d * cs,), NAN, device="cuda")
    src.view(d, cs)[:, :rows * pitch].view(d, rows, pitch)[:, :, :N] = x.view(d, rows, N)
    args = dict(chan_stride=cs, pitch=pitch, rows=rows, n=N, d=d, eps=1e-5)
    inp = dict(x=x, const=const, T=T)
    if mode == "ln":
        gamma = torch.randn(d, generator=g, device="cuda")
        beta = torch.randn(d, generator=g, device="cuda")
        gate = torch.randn(T, d, generator=g, device="cuda")
        gate[torch.rand(T, d, generator=g, device="cuda") < 0.1] = 0.0
        gbuf = torch.full((gate_off + T * d + GUARD,), NAN, dtype=torch.bfloat16, device="cuda")
        gbuf[gate_off:gate_off + T * d] = gate.flatten().bfloat16()
        args.update(mode=0, gamma=gamma, beta=beta, gate=gbuf, gate_off=gate_off)
        inp.update(gamma=gamma, beta=beta, gate=gbuf[gate_off:gate_off + T * d].view(T, d))
    elif mode == "scale_const":
        S = 37
        args.update(mode=1, scale_const=1.0 / S)
        inp.update(scale=torch.full((T,), 1.0 / S, dtype=torch.float32, device="cuda"))
    else:
        S, eps = 8, 1e-5
        cnt = torch.randint(0, S + 1, (T,), generator=g, device="cuda").float()
        scale = (1.0 / (S * (cnt + eps))).float()
        scale[torch.rand(T, generator=g, device="cuda") < 0.1] = 0.0
        args.update(mode=1, scale=scale)
        inp.update(scale=scale)
    return src, args, inp


def _c2t_ref(d, mode, inp):
    x = inp["x"].double().t()                          # [T][d]
    if mode != "ln":
        ref = x * inp["scale"].double()[:, None]
        return ref, 2.0 ** -8 * ref.abs() + 2 * U * ref.abs()
    w, b, g = inp["gamma"].double(), inp["beta"].double(), inp["gate"].double()
    mean = x.mean(1, keepdim=True)
    var = ((x - mean) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + float(torch.tensor(1e-5, dtype=torch.float32)))
    xh = (x - mean) * rstd
    ref = (xh * w + b) * g
    k = _k_d(d)
    dmean = (k + 2) * U * x.abs().mean(1, keepdim=True)
    dxh = rstd * (dmean + U * (x - mean).abs()) + xh.abs() * (k + 3) * U + xh.abs() * (rstd * dmean) ** 2 / 2
    bound = 2.0 ** -8 * ref.abs() + g.abs() * (w.abs() * dxh + 3 * U * ((xh * w).abs() + b.abs()))
    return ref, bound


def _c2t_run(d, N, B, mode, variant, seed, gate_off=0, y_off=0):
    """forced variant (or 0 = auto) on one layout; returns the variant that ran (0: rejected)"""
    ops = _ops()
    src, args, inp = _c2t_inputs(d, N, B, mode, seed, gate_off)
    T = inp["T"]
    y = torch.full((y_off + T * d + GUARD,), NAN, dtype=torch.bfloat16, device="cuda")
    auto = ops.chan_to_token_select(src, y, y_off=y_off, **args)
    if variant and variant not in _legal(d, N) or (variant in (2, 3) and (gate_off or y_off)):
        with pytest.raises(ValueError, match="cannot run"):
            ops.chan_to_token(src, y, variant=variant, y_off=y_off, **args)
        torch.cuda.synchronize()
        assert torch.isnan(y.float()).all(), "a rejected variant wrote output"
        return 0
    ran = ops.chan_to_token(src, y, variant=variant, y_off=y_off, **args)
    torch.cuda.synchronize()
    assert ran == (variant or auto)
    out = y[y_off:y_off + T * d].view(T, d)
    ref, bound = _c2t_ref(d, mode, inp)
    check_bound(f"c2t {VNAME[ran]} {mode} d{d} N{N} B{B} gate+{gate_off} y+{y_off}", out, ref, bound)
    assert torch.isnan(y[:y_off].float()).all() and torch.isnan(y[y_off + T * d:].float()).all(), "write outside y"
    if mode == "ln":                                   # constant tokens: exactly beta * gate, rounded once to bf16
        c = inp["const"]
        exact = (inp["beta"][None, :] * inp["gate"][c].float()).bfloat16()
        assert torch.equal(out[c].view(torch.int16), exact.view(torch.int16)), "constant token is not beta * gate"
    return ran


C2T_DIMS = [32, 64, 96, 128, 192, 224, 256]
# (N, B): partial last TMA tile (T = N^2 = 16 mod 32), N % 4 != 0 (padded pitch), batch offset inside `rows`, T = 16
C2T_SHAPES = [(44, 1), (37, 1), (40, 2), (4, 1)]


@pytest.mark.parametrize("variant", [0, 1, 2, 3], ids=["auto", "simt", "tile", "tma"])
@pytest.mark.parametrize("mode", ["ln", "scale_const", "scale_tok"])
@pytest.mark.parametrize("N,B", C2T_SHAPES)
@pytest.mark.parametrize("d", C2T_DIMS)
def test_chan_to_token(d, N, B, mode, variant):
    ran = _c2t_run(d, N, B, mode, variant, seed=d + 13 * N + B)
    if variant == 0:                                   # the modules' choice: TMA > tile > SIMT where legal
        assert ran == max(_legal(d, N)), f"auto picked {VNAME[ran]}"


@pytest.mark.parametrize("variant", [1, 2, 3], ids=["simt", "tile", "tma"])
@pytest.mark.parametrize("mode", ["ln", "scale_tok"])
@pytest.mark.parametrize("d", [128, 256])
def test_chan_to_token_many_tiles(d, mode, variant):
    """67 600 tokens (partial last tile): 2113 TMA tiles over at most 132 CTAs wrap the 4-stage rings several times"""
    assert _c2t_run(d, 260, 1, mode, variant, seed=d + variant) == variant


@pytest.mark.parametrize("mode,gate_off,y_off", [("ln", 1, 0), ("ln", 0, 1), ("scale_tok", 0, 1)])
def test_chan_to_token_misaligned(mode, gate_off, y_off):
    """gate or y based one element off a 16-byte boundary: the host must route the call to the SIMT kernel"""
    ops = _ops()
    d, N = 128, 44
    src, args, _ = _c2t_inputs(d, N, 1, mode, 11, gate_off)
    y = torch.full((y_off + N * N * d + GUARD,), NAN, dtype=torch.bfloat16, device="cuda")
    assert ops.chan_to_token_select(src, y, y_off=y_off, **args) == ops.C2T_SIMT
    for v in (2, 3):
        assert _c2t_run(d, N, 1, mode, v, seed=11, gate_off=gate_off, y_off=y_off) == 0
    assert _c2t_run(d, N, 1, mode, 0, seed=11, gate_off=gate_off, y_off=y_off) == ops.C2T_SIMT


# ------------------------------------------------------------------------------------------------------------------------
# D. OuterMean normaliser (af2_outer_scale)
# ------------------------------------------------------------------------------------------------------------------------
def _bits_fit(S, N):
    return (S + 31) // 32 * N * 4 <= 160 * 1024


@pytest.mark.parametrize("kind", ["holes", "ones"])
@pytest.mark.parametrize("third", [False, True], ids=["row0", "row0_third"])
@pytest.mark.parametrize("N", [1, 37, 256, 520])
@pytest.mark.parametrize("S", [1, 31, 32, 33, 100, 1024, 4096])
def test_outer_scale(S, N, third, kind):
    ops = _ops()
    g = _gen(S * 1000 + N)
    eps = 1e-5
    row0 = N // 3 if third else 0
    rows = N - row0
    if kind == "ones":
        mask = torch.ones(S, N, dtype=torch.bool, device="cuda")
    else:
        mask = torch.rand(S, N, generator=g, device="cuda") >= 0.3
        mask[:, torch.arange(N, device="cuda") % 7 == 3] = False          # fully masked residues: scale = 1 / (S eps)
        if N == 1:
            mask[:] = False
    words = torch.empty((S + 31) // 32 * N, dtype=torch.int32, device="cuda")
    m64 = mask.double()
    cnt = m64[:, row0:].t() @ m64
    ref = 1.0 / (S * (cnt + float(torch.tensor(eps, dtype=torch.float32))))
    outs = {}
    for v in (ops.OUTER_SCALE_BYTES, ops.OUTER_SCALE_BITS):
        out = torch.full((rows * N + GUARD,), NAN, device="cuda")
        if v == ops.OUTER_SCALE_BITS and not _bits_fit(S, N):
            with pytest.raises(ValueError, match="shared memory"):
                ops.outer_scale(mask, out, row0=row0, rows=rows, eps=eps, variant=v, words=words)
            torch.cuda.synchronize()
            assert torch.isnan(out).all()
            continue
        assert ops.outer_scale(mask, out, row0=row0, rows=rows, eps=eps, variant=v, words=words) == v
        torch.cuda.synchronize()
        name = "bits" if v == ops.OUTER_SCALE_BITS else "bytes"
        check_bound(f"outer_scale {name} S{S} N{N} row0 {row0} {kind}", out[:rows * N].view(rows, N), ref, 4 * U * ref.abs())
        assert torch.isnan(out[rows * N:]).all(), "write past the scale rows"
        outs[v] = out[:rows * N]
    if len(outs) == 2:
        assert torch.equal(outs[1].view(torch.int32), outs[2].view(torch.int32)), "bit-packed and byte-loop kernels differ"
    out = torch.full((rows * N,), NAN, device="cuda")
    auto = ops.outer_scale(mask, out, row0=row0, rows=rows, eps=eps, words=words)
    assert auto == (ops.OUTER_SCALE_BITS if _bits_fit(S, N) else ops.OUTER_SCALE_BYTES)
    if S == 4096 and N == 520:
        assert auto == ops.OUTER_SCALE_BYTES
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), outs[auto].view(torch.int32))
