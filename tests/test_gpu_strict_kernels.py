"""-m gpu: the strict precision mode kernel by kernel, element-wise against fp64: (A) the split encoding, (B) the split-bf16
GEMM in both operand layouts and (C) every SIMT kernel that feeds or follows it.  Each kernel runs through the C entry
point that shares its launcher with the strict modules (include/af2b200.h), so the grid and arguments are the modules'.

References are fp64, evaluated on the GPU with plain torch from the exact fp32 / bf16 operands the kernel received.  Output
buffers start as NaN with a guard region after them; guards must stay NaN, and two identical launches must be bitwise equal.
u = 2^-24 is the fp32 unit roundoff.

Split planes.  Every kernel that writes split operands stores p0 = bf16(v), p1 = bf16(v - p0), p2 = bf16(v - p0 - p1) of its
fp32 value v.  For each element the test forms v^ = p0 + p1 + p2 in fp64 (exact: three bf16 values whose span is below 53
bits) and requires: v^ is an fp32 value, p0 == bf16(v^) and p1 == bf16(v^ - p0) (so p2 == v^ - p0 - p1) wherever v^ = 0 or
|v^| >= 2^-110 (the exact range derived in A); then v^ meets the kernel's fp64 bound plus 2^-134 (the split below that range;
softmax weights reach it).  Pad columns [cols, align8(cols)) must be exactly 0 where the kernel owns them; the token -> channel
kernel writes none, so its pads must stay NaN.

A. Split encoding.  With round-to-nearest, |v - p0| <= 2^-8 2^e for 2^e <= |v| < 2^(e+1), so p1 carries the next 8 bits and
  p2 = v - p0 - p1 has its lowest bit at ulp(v) = 2^(e-23); p2 is a bf16 value as long as that bit is not below the smallest
  bf16 subnormal 2^-133, i.e. |v| >= 2^-110.  At the top, p0 = bf16(v) overflows to inf once |v| >= 2^128 - 2^119 (bf16 max
  (2 - 2^-7) 2^127 plus half its ulp).  So the planes sum to v EXACTLY for v = 0 and 2^-110 <= |v| < 2^128 - 2^119; below
  2^-110 (fp32 subnormals included) the last plane is rounded to the bf16 subnormal grid: |v^ - v| <= 2^-134.  Strict-mode
  activations never reach either end.  The device split must equal the host ops.split_weight of the same matrix bit for
  bit: weights are split on the host, activations on the device, and the GEMM assumes one encoding.

B. Split GEMM, C = A B^T on planes: the six passes (A plane, B plane) = (0,2) (2,0) (1,1) (0,1) (1,0) (0,0), small ones first,
  all into one fp32 accumulator.  Every bf16 x bf16 product is exact in fp32, so what remains is
  * the accumulation: gpu_util's C_GEMM K u sum |terms| for the last pass, which dominates: the five earlier passes sum terms
    below 2^-7 |a_k b_k| each, and add at most 6 2^-7 K u sum |a_k b_k| to it:  C_GEMM K u (1 + 2^-4) sum_k |a_k b_k|
  * the dropped pairs (1,2) (2,1) (2,2): |p1| <= 2^-8 (1 + 2^-8) |v| and |p2| <= 2^-16 |v|:  <= 1.01 2^-23 sum_k |a_k b_k|
  * the epilogue roundings of acc + bias and of + residual:  2 u (|ref| + |resid|)
  (gpu_util.gemm_split_bound).  That worst case is larger than what a missing pass does to random data, so two exact tests
  pin the wiring:
  * plane wiring: only plane i of A and plane j of B hold values.  The six pairs the kernel uses must give the fp32 GEMM of
    those planes (gemm_f32_bound); the three it drops must give exactly the bias (+ residual).
  * exact gather: B rows one-hot with +-2^s entries and A random fp32 with all 24 mantissa bits in use, then A one-hot and B
    random.  Every output must equal +-2^s a bitwise: it goes through passes (2,0) (1,0) (0,0) (or (0,2) (0,1) (0,0)), whose
    partial sums are all fp32 values.  This assumes the tensor cores' fp32 accumulation returns a sum exactly whenever it is
    representable (all other terms are exact zeros); a failure here is a finding about the hardware, not a tolerance.
  NaN fills the pad columns [K, P) of K-major operands, [M or N, P) of MN-major ones and a gap after every batch: the tensor
  maps stop at the logical extent, so no launch reads them (any read would make an output NaN).

C. SIMT kernels.  fp32 arithmetic is IEEE (no fast math); expf and erff are within 2 ulp, rsqrtf within 2 ulp.
  * LayerNorm split (one warp per row: ceil(d/32) terms per lane, 5 shuffle levels, k_d = ceil(d/32) + 5):
      |dmean| <= (k_d + 2) u mean|x|;  rstd relative ((k_d + 5) / 2 + 4) u (variance sum, squares, / d, + eps, halved by the
      square root, rsqrtf's 2 ulp); xhat = (x - mean) rstd one more rounding:
      |dxhat| <= rstd (|dmean| + u |x - mean|) + |xhat| ((k_d + 5) / 2 + 5) u + |xhat| (rstd dmean)^2 / 2
      |dy| <= |gamma| |dxhat| + 2 u (|xhat gamma| + |beta|).   A constant row must give exactly beta.
  * GELU: g = 0.5 x (1 + erff(x c)), c = fl(1/sqrt 2): the argument carries 2 u |x| / sqrt 2 (c and the product), erff 2 ulp
    <= 2^-23 absolute, then (1 + erf), * (1 + erf) one rounding each:
      |dg| <= |x| / 2 (2^-23 + 2 / sqrt(pi) exp(-x^2 / 2) 2 u |x| / sqrt 2 + u |1 + erf|) + u |g|;  GEGLU: |a| |dg| + u |v|.
    Near x = -5, 1 + erf cancels to ~1e-6 and the absolute erff term dominates.
  * sigmoid 1 / (1 + expf(-x)): relative 2^-22 (expf) + 2 u (add, IEEE divide) <= 4 u;  gate split O s: 5 u |ref|.  Below
    x = -88.7, expf(-x) overflows and the kernel's sigmoid is exactly 0 (true value < 2^-127): an absolute 2^-126 term.
  * q/k/v split and token -> channel without gate: a re-layout, v^ must equal the fp32 input bitwise (and 0 in owned pads).
  * pair bias: fmaf chains of ceil(d/32) terms per lane + 5 shuffle adds:  (ceil(d/32) + 6) u sum_c |x_c w_c|.
  * softmax: the logit l = s + b carries u |L|, the max u |L_max|, l - max u |L - L_max|: together 2 u (|L| + |L_max|) in the
    exponent;  expf 2^-22 relative (also inside the sum), the n-term sum (ceil(n/32) + 5) u, 1 / sum and the product 2 u:
      |dp| <= p (2 u (|L| + |L_max|) + 2 u max_k (|L_k| + |L_max|) + 2^-21 + (ceil(n/32) + 7) u) + 2^-147
    (the last term covers results in the fp32 subnormal range).  Masked entries must be exactly 0, a fully masked query row
    exactly uniform 1/n over all n keys (quirk Q1).
  * channel -> token mode 0: the LayerNorm bound above over the d channels (same warp tree), then * sigmoid(gate):
      |dv| <= s |dy| + 5 u |y s| + 2^-126 |y|;  a constant token must give exactly fl(beta s) (gates chosen so that s is 0, 1/2 or 1).
    Mode 1: one rounding, u |ref|.
  * tie_queries: a sequential fp32 sum of nbatch terms and one division:  (nbatch + 1) u mean|q|; bf16 adds the store,
    2^-8 |ref|.  Columns outside the q block must stay bitwise unchanged.
"""
import ctypes as C

import pytest
import torch

from gpu_util import U32 as U, check_bound, gemm_f32_bound, gemm_split_bound

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 64
SPL = 3
BF = torch.bfloat16
EPI_RESID_F32, EPI_STORE_F32 = 2, 3
USED_PAIRS = ((0, 2), (2, 0), (1, 1), (0, 1), (1, 0), (0, 0))


def _lib():
    from alphafold2_b200 import _lib as L
    return L


def _call(fn, *args):
    from alphafold2_b200 import ops
    L = _lib()
    L.check(getattr(L.load(), fn)(*args, ops._stream_ptr()))


def _p(t):
    return None if t is None else t.data_ptr()


def _al(v, a):
    return (v + a - 1) // a * a


def _pick_bn(n):
    """the tile width the modules use for n output columns (api.cu pick_bn)"""
    return 256 if n > 128 else (128 if n > 64 else 64)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _nan(n, dtype=torch.float32):
    return torch.full((n + GUARD,), NAN, dtype=dtype, device="cuda")


def _bits(t):
    return t.view(torch.int16 if t.dtype == BF else torch.int32)


def _twice(run):
    """run() -> output buffer; runs it twice and requires bitwise-equal buffers (guards included)"""
    a, b = run(), run()
    assert torch.equal(_bits(a), _bits(b)), "two identical launches differ"
    assert torch.isnan(a[-GUARD:]).all(), "guard region written"
    return a


TINY = 2.0 ** -110      # below it the last plane is rounded to the bf16 subnormal grid (A): |v^ - v| <= 2^-134


def _valid_split(pl):
    """pl bf16 [..., 3, W] -> v^ = p0 + p1 + p2 in fp64; asserts that the planes are the split of v^ (as values: +-0 alike)
    wherever v^ lies in the exact range of the split (0 or |v^| >= 2^-110)"""
    p = pl.double()
    v = p[..., 0, :] + p[..., 1, :] + p[..., 2, :]
    assert torch.isfinite(v).all(), "non-finite split plane"
    ex = (v == 0) | (v.abs() >= TINY)
    assert torch.equal(v.float().double()[ex], v[ex]), "planes sum to a value fp32 cannot hold"
    assert torch.equal(p[..., 0, :][ex], v.float().to(BF).double()[ex]), "p0 != bf16(v)"
    assert torch.equal(p[..., 1, :][ex], (v - p[..., 0, :]).float().to(BF).double()[ex]), "p1 != bf16(v - p0)"
    assert torch.equal(p[..., 2, :][ex], (v - p[..., 0, :] - p[..., 1, :])[ex])
    return v


def _split_out(name, buf, shape, cols, ref, bound, pads="zero", valid=True):
    """buf: flat bf16 split buffer [*shape, 3, P] (+ guard); checks planes, accuracy on [:cols] (bound + 2^-134, the split of
    values below 2^-110) and the pads; returns v^.  valid = False only sums the planes."""
    P = shape[-1]
    n = 1
    for s in shape[:-1]:
        n *= s
    pl = buf[: n * SPL * P].view(*shape[:-1], SPL, P)
    summed = _valid_split if valid else (lambda t: t.double().sum(-2))
    if pads == "zero":
        v = summed(pl)
        assert torch.all(v[..., cols:] == 0), f"{name}: pad columns not zero"
    else:
        v = summed(pl[..., :cols])
        assert torch.isnan(pl[..., cols:]).all(), f"{name}: pad columns written"
    check_bound(name, v[..., :cols], ref, bound + 2.0 ** -134)
    return v[..., :cols]


def _planes(x):
    """fp32 [..., K] -> fp32 [..., 3, K]: the three bf16 planes, computed in torch like ops.split_weight"""
    r, out = x.float(), []
    for _ in range(SPL):
        h = r.to(BF).float()
        out.append(h)
        r = r - h
    return torch.stack(out, -2)


# ------------------------------------------------------------------------------------------------------------------------
# A. split encoding
# ------------------------------------------------------------------------------------------------------------------------
def _device_split(x):
    rows, K = x.shape
    P = _al(K, 8)
    y = _nan(rows * SPL * P, BF)
    _call("af2_split_bf16", x.data_ptr(), y.data_ptr(), rows, K)
    return y


@pytest.mark.parametrize("K", [1, 13, 64, 100])
def test_split_encoding_exact(K):
    g = _gen(K)
    rows = 97
    mant = 1.0 + torch.randint(0, 1 << 23, (rows, K), device="cuda", generator=g).double() / (1 << 23)   # all 24 bits
    expo = torch.randint(-110, 128, (rows, K), device="cuda", generator=g).double()
    sign = torch.where(torch.rand(rows, K, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    x = (sign * mant * torch.exp2(expo)).float()
    top = 2.0 ** 128 - 2.0 ** 119                                  # p0 overflows from here on
    x = torch.where(x.abs() >= top, torch.sign(x) * 1.5 * 2.0 ** 127, x)
    # ties at each plane boundary: bit 8 (p0 / p1) and bit 16 (p1 / p2) below the leading one exactly half, odd / even
    e = torch.exp2(torch.randint(-40, 40, (rows,), device="cuda", generator=g).double())
    x[:, 0] = (e * (1 + 2.0 ** -8)).float()                       # p0 tie to even (down)
    if K > 1:
        x[:, 1] = (-e * (1 + 2.0 ** -7 + 2.0 ** -8)).float()      # p0 tie to even (up), negative
    if K > 2:
        x[:, 2] = (e * (1 + 2.0 ** -8 + 2.0 ** -16 + 2.0 ** -17)).float()
    if K > 3:
        x[:, 3] = 0.0
    if K > 4:
        x[:, 4] = -0.0
    if K > 5:
        x[:, 5] = (2.0 ** -110 * (2 - 2.0 ** -23))
    if K > 6:
        x[:, 6] = float(top - 2.0 ** 104)                          # the largest fp32 below the overflow threshold
    P = _al(K, 8)
    y = _twice(lambda: _device_split(x))
    v = _split_out(f"strict/split/K{K}", y, (rows, P), K, x.double(), torch.zeros_like(x, dtype=torch.float64))
    assert torch.equal(v, x.double())


def test_split_encoding_tiny():
    """below 2^-110 (fp32 subnormals included) the last plane is rounded to the bf16 subnormal grid: |v^ - v| <= 2^-134"""
    g = _gen(7)
    x = torch.cat([torch.exp2(-torch.linspace(110.0, 149.0, 400, device="cuda", dtype=torch.float64)),
                   torch.rand(400, device="cuda", generator=g, dtype=torch.float64) * 2.0 ** -110]).float()
    x = torch.cat([x, -x]).view(8, 200)
    y = _twice(lambda: _device_split(x))
    _split_out("strict/split/tiny", y, (8, 200), 200, x.double(), torch.zeros_like(x, dtype=torch.float64), valid=False)  # + 2^-134


@pytest.mark.parametrize("rows,K", [(37, 29), (64, 256), (5, 1)])
def test_device_split_matches_host_split_weight(rows, K):
    from alphafold2_b200 import ops
    g = _gen(rows * K)
    x = torch.randn(rows, K, device="cuda", generator=g) * torch.exp2(torch.randint(-30, 30, (rows, K), device="cuda", generator=g).float())
    P = _al(K, 8)
    dev = _device_split(x)[: rows * SPL * P].view(rows, SPL, P)
    for host in (ops.split_weight(x), ops.split_weight(x.cpu()).cuda()):
        assert torch.equal(_bits(dev), _bits(host))


# ------------------------------------------------------------------------------------------------------------------------
# B. split GEMM
# ------------------------------------------------------------------------------------------------------------------------
def _operand(planes, mn_major, gap=8):
    """planes fp32 [batch, R, 3, K] (bf16 values) -> (flat bf16 buffer, ld, plane stride, batch stride).  K-major: [batch][R][3][P],
    P = align8(K);  MN-major: [batch][3][K][Pr], Pr = align8(R).  NaN in the pads and in a gap after every batch."""
    batch, R, _, K = planes.shape
    if not mn_major:
        P = _al(K, 8)
        bs = R * SPL * P + gap
        buf = torch.full((batch, bs), NAN, dtype=BF, device="cuda")
        buf[:, : R * SPL * P].view(batch, R, SPL, P)[..., :K] = planes.to(BF)
        return buf.flatten(), SPL * P, P, bs
    Pr = _al(R, 8)
    bs = SPL * K * Pr + gap
    buf = torch.full((batch, bs), NAN, dtype=BF, device="cuda")
    buf[:, : SPL * K * Pr].view(batch, SPL, K, Pr)[..., :R] = planes.permute(0, 2, 3, 1).to(BF)
    return buf.flatten(), Pr, K * Pr, bs


def _gemm(A, B, M, N, K, batch, mn_major, bn, mode=EPI_STORE_F32, bias=None, out=None, ld_out=None, resid=None):
    """af2_gemm_split_epilogue; returns the flat fp32 output (a new NaN buffer [batch][M][ld_out] + guard unless `out`)"""
    L = _lib()
    ld_out = ld_out or _al(N, 4)
    if out is None:
        out = _nan(batch * M * ld_out)
    e = L.GemmEpilogue(bn=bn, mode=mode, act=0, layout=0, use_rowscale=0, bias=_p(bias), rowscale=None, resid=_p(resid),
                       ld_resid=ld_out if resid is not None else 0, out=out.data_ptr(), ld_out=ld_out,
                       out_batch=M * ld_out, cm_inner=0, cm_pitch=0, out_cols=0)
    (a, lda, ah, ab), (b, ldb, bh, bb) = A, B
    _call("af2_gemm_split_epilogue", a.data_ptr(), lda, ah, ab, b.data_ptr(), ldb, bh, bb, M, N, K, batch, int(mn_major), C.byref(e))
    return out


def _out_view(out, batch, M, N, ld):
    o = out[: batch * M * ld].view(batch, M, ld)
    assert torch.isnan(o[..., N:]).all(), "output pad columns written"
    return o[..., :N]


def _bias(N, g):
    b = torch.zeros(_al(N, 256), device="cuda")
    b[:N] = torch.randn(N, device="cuda", generator=g)
    return b


@pytest.mark.parametrize("mn_major", [False, True])
@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("K", [40, 64, 200])
def test_gemm_split_plane_wiring(mn_major, bn, batch, K):
    """plane i of A x plane j of B alone: the six used pairs give their fp32 GEMM, the three dropped ones exactly the bias"""
    g = _gen(bn + K + batch)
    M, N = 130, bn + 24
    bias = _bias(N, g)
    for i in range(SPL):
        for j in range(SPL):
            pa = torch.zeros(batch, M, SPL, K, device="cuda")
            pb = torch.zeros(batch, N, SPL, K, device="cuda")
            pa[:, :, i] = torch.randn(batch, M, K, device="cuda", generator=g).to(BF).float()
            pb[:, :, j] = torch.randn(batch, N, K, device="cuda", generator=g).to(BF).float()
            A, B = _operand(pa, mn_major), _operand(pb, mn_major)
            out = _twice(lambda: _gemm(A, B, M, N, K, batch, mn_major, bn, bias=bias))
            o = _out_view(out, batch, M, N, _al(N, 4))
            name = f"strict/gemm_wiring/{'mn' if mn_major else 'k'}/bn{bn}/b{batch}/K{K}/A{i}B{j}"
            if (i, j) in USED_PAIRS:
                a64, b64 = pa[:, :, i].double(), pb[:, :, j].double()
                ref = a64 @ b64.transpose(1, 2) + bias[:N].double()
                check_bound(name, o, ref, gemm_f32_bound(a64.abs() @ b64.abs().transpose(1, 2), K, ref))
            else:
                assert torch.equal(o, bias[:N].expand(batch, M, N)), f"{name}: a dropped plane pair reached the output"


def _one_hot(batch, R, K, g):
    """[batch, R, K] fp32 rows with a single +-2^s entry (column idx[r]); returns (rows, idx, value)"""
    idx = torch.randint(0, K, (batch, R), device="cuda", generator=g)
    val = torch.exp2(torch.randint(-20, 21, (batch, R), device="cuda", generator=g).float())
    val = torch.where(torch.rand(batch, R, device="cuda", generator=g) < 0.5, -val, val)
    x = torch.zeros(batch, R, K, device="cuda")
    x.scatter_(2, idx[..., None], val[..., None])
    return x, idx, val


def _full_mantissa(shape, g):
    m = 1.0 + torch.randint(1, 1 << 23, shape, device="cuda", generator=g).double() / (1 << 23)
    m = m + (m * (1 << 23)).remainder(2).eq(0).double() * 2.0 ** -23      # odd last bit: all 24 bits in use
    s = torch.where(torch.rand(shape, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    return (s * m * torch.exp2(torch.randint(-8, 9, shape, device="cuda", generator=g).double())).float()


def _tok2chan_operand(x, mn_major, gap=8):
    """the token -> channel split kernel builds operand A[c] of x [C, M, K] (no gate, no mask), as the contractions use it"""
    Cc, M, K = x.shape
    if not mn_major:      # K-major [c][M][3][P]: rows = M, inner = K
        P = _al(K, 8)
        cs = M * SPL * P + gap
        src = x.permute(1, 2, 0).contiguous()                     # token (m, k) = m * K + k, channel c
        out = torch.full((Cc * cs,), NAN, dtype=BF, device="cuda")
        _call("af2_strict_tok2chan_split", src.data_ptr(), Cc, 0, -1, None, out.data_ptr(), Cc, M, K, cs, P, SPL * P)
        return out, SPL * P, P, cs
    P = _al(M, 8)          # MN-major [c][3][K][P]: rows = K, inner = M
    cs = SPL * K * P + gap
    src = x.permute(2, 1, 0).contiguous()                         # token (k, m) = k * M + m
    out = torch.full((Cc * cs,), NAN, dtype=BF, device="cuda")
    _call("af2_strict_tok2chan_split", src.data_ptr(), Cc, 0, -1, None, out.data_ptr(), Cc, K, M, cs, K * P, P)
    return out, P, K * P, cs


@pytest.mark.parametrize("mn_major", [False, True])
@pytest.mark.parametrize("K", [24, 200])
@pytest.mark.parametrize("source", ["host", "split_kernel", "tok2chan"])
def test_gemm_split_exact_gather(mn_major, K, source):
    """one-hot +-2^s operand against a random full-mantissa one: every output is +-2^s a, bit for bit"""
    if source == "split_kernel" and mn_major:
        pytest.skip("af2_split_bf16 writes token-major (K-major) rows only")
    g = _gen(K + 31 * mn_major)
    batch, M, N = 3, 150, 72
    bn = _pick_bn(N)
    a = _full_mantissa((batch, M, K), g)
    b = _full_mantissa((batch, N, K), g)
    bh, bidx, bval = _one_hot(batch, N, K, g)
    ah, aidx, aval = _one_hot(batch, M, K, g)
    # B one-hot: C[m][n] = bval[n] a[m][bidx[n]];  A one-hot: C[m][n] = aval[m] b[n][aidx[m]]
    for name, ra, rb, exp in (
            ("Bonehot", a, bh, bval[:, None, :] * torch.gather(a, 2, bidx[:, None, :].expand(batch, M, N))),
            ("Aonehot", ah, b, aval[:, :, None] * torch.gather(b, 2, aidx[:, None, :].expand(batch, N, M)).transpose(1, 2))):
        if source == "host":
            A = _operand(_planes(ra), mn_major)
        elif source == "split_kernel":
            y = _device_split(ra.reshape(batch * M, K))
            A = (y, SPL * _al(K, 8), _al(K, 8), M * SPL * _al(K, 8))
        else:
            A = _tok2chan_operand(ra, mn_major)
        B = _operand(_planes(rb), mn_major)
        out = _twice(lambda: _gemm(A, B, M, N, K, batch, mn_major, bn))
        o = _out_view(out, batch, M, N, _al(N, 4))
        bad = o != exp
        assert not bad.any(), (f"{source}/{name}/{'mn' if mn_major else 'k'}/K{K}: {int(bad.sum())} outputs differ from +-2^s a, "
                               f"first {o[bad][0].item()!r} vs {exp[bad][0].item()!r}")


def _random_gemm(name, M, N, K, batch, mn_major, g, bn=None, mode=EPI_STORE_F32, with_bias=True, a_pos=False, ld_out=None):
    bn = bn or _pick_bn(N)
    a = torch.randn(batch, M, K, device="cuda", generator=g)
    if a_pos:
        a = torch.rand(batch, M, K, device="cuda", generator=g) / K            # probabilities (P V)
    b = torch.randn(batch, N, K, device="cuda", generator=g)
    bias = _bias(N, g) if with_bias else None
    A, B = _operand(_planes(a), mn_major), _operand(_planes(b), mn_major)
    ld = ld_out or _al(N, 4)
    if mode == EPI_RESID_F32:
        x0 = torch.randn(M * ld + GUARD, device="cuda", generator=g)
        x0.view(-1)[M * ld:] = NAN
        x0[: M * ld].view(M, ld)[:, N:] = NAN

        def run():
            x = x0.clone()
            return _gemm(A, B, M, N, K, batch, mn_major, bn, mode, bias, out=x, ld_out=ld, resid=x)
        out = _twice(run)
        resid = x0[: M * ld].view(1, M, ld)[..., :N].double()
    else:
        out = _twice(lambda: _gemm(A, B, M, N, K, batch, mn_major, bn, mode, bias, ld_out=ld))
        resid = torch.zeros(1, device="cuda", dtype=torch.float64)
    o = _out_view(out, batch, M, N, ld)
    a64, b64 = a.double(), b.double()
    ref = a64 @ b64.transpose(1, 2) + resid + (bias[:N].double() if bias is not None else 0)
    check_bound(name, o, ref, gemm_split_bound(a64.abs() @ b64.abs().transpose(1, 2), K, ref, resid))


@pytest.mark.parametrize("d,N", [(32, 4 * 64), (64, 5 * 64), (128, 2 * 512), (256, 4 * 512), (256, 5 * 256), (100, 5 * 100)])
def test_gemm_split_projection(d, N):
    _random_gemm(f"strict/gemm/proj/d{d}N{N}", 300, N, d, 1, False, _gen(d + N))


@pytest.mark.parametrize("K,N,ld,bn", [(256, 256, 256, 256), (256, 256, 260, 256), (256, 256, 258, 256), (1024, 256, 256, 256),
                                       (128, 128, 128, 128), (64, 100, 100, 128), (512, 64, 66, 64)])
def test_gemm_split_residual_in_place(K, N, ld, bn):
    """output projections x += A W^T + b in place: ld 256 / 260 take the TMA epilogue at bn 256, ld 258 and bn < 256 do not"""
    _random_gemm(f"strict/gemm/resid/K{K}N{N}ld{ld}bn{bn}", 333, N, K, 1, False, _gen(K + ld), bn=bn, mode=EPI_RESID_F32, ld_out=ld)


@pytest.mark.parametrize("dh,n,bh", [(32, 33, 6), (32, 130, 4), (64, 256, 3), (64, 384, 2)])
def test_gemm_split_logits(dh, n, bh):
    """S = Q K^T per (b', head), K = dim_head, ld_out = align4(n)"""
    _random_gemm(f"strict/gemm/qk/dh{dh}n{n}", n, n, dh, bh, False, _gen(dh + n), with_bias=False)


@pytest.mark.parametrize("dh,n,bh", [(32, 33, 6), (32, 130, 4), (64, 384, 2)])
def test_gemm_split_pv(dh, n, bh):
    """O = P V per (b', head), K = n, B = V^T"""
    _random_gemm(f"strict/gemm/pv/dh{dh}n{n}", n, dh, n, bh, False, _gen(dh * n), with_bias=False, a_pos=True)


@pytest.mark.parametrize("kind,N,K,d", [("outgoing", 37, 37, 16), ("outgoing", 130, 130, 8), ("ingoing", 37, 37, 16),
                                        ("ingoing", 130, 130, 8), ("outer", 70, 1, 16), ("outer", 70, 5, 16), ("outer", 70, 130, 8)])
def test_gemm_split_contractions(kind, N, K, d):
    """the per-channel contractions: batch = channels, triangle K = N (outgoing K-major, ingoing MN-major), outer mean K = S"""
    _random_gemm(f"strict/gemm/{kind}/N{N}K{K}", N, N, K, d, kind != "outgoing", _gen(N + K), with_bias=False)


def test_gemm_split_rejects_other_epilogues():
    L = _lib()
    g = _gen(1)
    A = _operand(_planes(torch.randn(1, 64, 32, device="cuda", generator=g)), False)
    out = _nan(64 * 64)
    for mode, act, layout, bn in ((0, 0, 0, 64), (1, 0, 0, 64), (3, 1, 0, 64), (3, 0, 1, 64), (3, 0, 0, 96)):
        e = L.GemmEpilogue(bn=bn, mode=mode, act=act, layout=layout, out=out.data_ptr(), ld_out=64)
        with pytest.raises(ValueError):
            _call("af2_gemm_split_epilogue", A[0].data_ptr(), A[1], A[2], A[3], A[0].data_ptr(), A[1], A[2], A[3], 64, 64, 32, 1, 0, C.byref(e))
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


# ------------------------------------------------------------------------------------------------------------------------
# C. SIMT kernels
# ------------------------------------------------------------------------------------------------------------------------
def _ln_ref(x, gamma, beta, k_d, eps=1e-5):
    """fp64 LayerNorm over the last axis and the bound of the module docstring"""
    mean = x.mean(-1, keepdim=True)
    xc = x - mean
    rstd = 1.0 / torch.sqrt((xc * xc).mean(-1, keepdim=True) + eps)
    xh = xc * rstd
    dmean = (k_d + 2) * U * x.abs().mean(-1, keepdim=True)
    dxh = rstd * (dmean + U * xc.abs()) + xh.abs() * ((k_d + 5) / 2 + 5) * U + xh.abs() * (rstd * dmean) ** 2 / 2
    y = xh * gamma + beta
    return y, gamma.abs() * dxh + 2 * U * ((xh * gamma).abs() + beta.abs())


@pytest.mark.parametrize("d", [32, 100, 128, 256])
def test_strict_layernorm_split(d):
    g = _gen(d)
    T = 203                                                           # not a multiple of the 8 rows per block
    x = torch.randn(T, d, device="cuda", generator=g) * 3 + 0.5
    x[:40] = 1e3 + torch.randn(40, d, device="cuda", generator=g)    # mean 1e3, unit spread
    x[40:44] = torch.tensor([1024.0, -3.5, 0.0, 7.0], device="cuda")[:, None]   # constant rows: exactly beta
    gamma = torch.randn(d, device="cuda", generator=g)
    beta = torch.randn(d, device="cuda", generator=g)
    P = _al(d, 8)

    def run():
        y = _nan(T * SPL * P, BF)
        _call("af2_strict_ln_split", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), T, d)
        return y
    y = _twice(run)
    ref, bound = _ln_ref(x.double(), gamma.double(), beta.double(), (d + 31) // 32 + 5)
    v = _split_out(f"strict/ln_split/d{d}", y, (T, P), d, ref, bound)
    assert torch.equal(v[40:44], beta.double().expand(4, d)), "a constant row must give exactly beta"


def _gelu_ref(x):
    c = 0.7071067811865476
    e = torch.erf(x * c)
    gl = 0.5 * x * (1 + e)
    dg = x.abs() / 2 * (2.0 ** -23 + 2 / torch.pi ** 0.5 * torch.exp(-x * x / 2) * 2 * U * x.abs() * c + U * (1 + e).abs()) + U * gl.abs()
    return gl, dg


def _gelu_inputs(rows, d, g):
    x = (torch.rand(rows, d, device="cuda", generator=g) * 20 - 10)
    x.view(-1)[:401] = torch.linspace(-6, -4, 401, device="cuda")    # 1 + erf(x / sqrt 2) cancels
    return x


@pytest.mark.parametrize("hid", [36, 128, 257])
def test_strict_geglu_split(hid):
    g = _gen(hid)
    T = 77
    h = torch.empty(T, 2 * hid, device="cuda")
    h[:, :hid] = torch.randn(T, hid, device="cuda", generator=g)
    h[:, hid:] = _gelu_inputs(T, hid, g)
    P = _al(hid, 8)

    def run():
        y = _nan(T * SPL * P, BF)
        _call("af2_strict_geglu_split", h.data_ptr(), y.data_ptr(), T, hid)
        return y
    y = _twice(run)
    a = h[:, :hid].double()
    gl, dg = _gelu_ref(h[:, hid:].double())
    ref = a * gl
    _split_out(f"strict/geglu_split/h{hid}", y, (T, P), hid, ref, a.abs() * dg + U * ref.abs())


@pytest.mark.parametrize("d", [36, 128, 257])
def test_strict_gelu_split(d):
    g = _gen(d + 1)
    rows = 77
    h = _gelu_inputs(rows, d, g).contiguous()
    P = _al(d, 8)

    def run():
        y = _nan(rows * SPL * P, BF)
        _call("af2_strict_gelu_split", h.data_ptr(), y.data_ptr(), rows, d)
        return y
    y = _twice(run)
    ref, dg = _gelu_ref(h.double())
    _split_out(f"strict/gelu_split/d{d}", y, (rows, P), d, ref, dg)


def _tokens(b0, nb, n, sb, si):
    """token index [nb, n] of folded batch element b0 + b', position i"""
    return (b0 + torch.arange(nb, device="cuda"))[:, None] * sb + torch.arange(n, device="cuda")[None, :] * si


@pytest.mark.parametrize("dh", [20, 32, 64])
@pytest.mark.parametrize("n", [1, 7, 33, 130])
@pytest.mark.parametrize("row", [True, False])
def test_strict_qkv_split(dh, n, row):
    g = _gen(dh * n + row)
    H, nbt, b0, nb = 2, 5, 2, 3                                       # a chunk: b0 > 0, nb < the folded batch
    I = H * dh
    p1 = torch.randn(nbt * n, 4 * I, device="cuda", generator=g)
    sb, si = (n, 1) if row else (1, nbt)
    Pd, Pn = _al(dh, 8), _al(n, 8)

    def run():
        q, k, vt = _nan(nb * H * n * SPL * Pd, BF), _nan(nb * H * n * SPL * Pd, BF), _nan(nb * H * dh * SPL * Pn, BF)
        _call("af2_strict_qkv_split", p1.data_ptr(), q.data_ptr(), k.data_ptr(), vt.data_ptr(), b0, nb, H, n, dh, sb, si)
        return torch.cat([q, k, vt])
    out = _twice(run)
    q, k, vt = torch.split(out, [nb * H * n * SPL * Pd + GUARD, nb * H * n * SPL * Pd + GUARD, nb * H * dh * SPL * Pn + GUARD])
    for t in (q, k, vt):
        assert torch.isnan(t[-GUARD:]).all()
    rows = p1[_tokens(b0, nb, n, sb, si)].double()                   # [nb, n, 4I]
    exp_q = rows[..., :I].view(nb, n, H, dh).permute(0, 2, 1, 3).reshape(nb * H, n, dh)
    exp_k = rows[..., I:2 * I].view(nb, n, H, dh).permute(0, 2, 1, 3).reshape(nb * H, n, dh)
    exp_v = rows[..., 2 * I:3 * I].view(nb, n, H, dh).permute(0, 2, 3, 1).reshape(nb * H, dh, n)
    for name, buf, shape, cols, exp in (("q", q, (nb * H, n, Pd), dh, exp_q), ("k", k, (nb * H, n, Pd), dh, exp_k),
                                        ("vt", vt, (nb * H, dh, Pn), n, exp_v)):
        v = _split_out(f"strict/qkv_split/{name}/dh{dh}n{n}{'row' if row else 'col'}", buf, shape, cols, exp, torch.zeros_like(exp))
        assert torch.equal(v, exp)


@pytest.mark.parametrize("d,H", [(32, 1), (100, 3), (128, 4), (256, 8)])
def test_strict_pair_bias(d, H):
    g = _gen(d + H)
    T = 37 * 37
    x = torch.randn(T, d, device="cuda", generator=g)
    w = torch.randn(H, d, device="cuda", generator=g)

    def run():
        b = _nan(H * T)
        _call("af2_strict_pair_bias", x.data_ptr(), w.data_ptr(), b.data_ptr(), T, d, H)
        return b
    b = _twice(run)
    ref = w.double() @ x.double().t()
    check_bound(f"strict/pair_bias/d{d}H{H}", b[: H * T].view(H, T), ref,
                ((d + 31) // 32 + 6) * U * (w.double().abs() @ x.double().abs().t()))


def _softmax_ref(S, bias, valid):
    """S [nb, H, n, n] fp64 logits (bias added), valid [nb, n, n] bool -> (p, bound) of the module docstring"""
    n = S.shape[-1]
    v = valid[:, None].expand_as(S)
    Lm = torch.where(v, S, torch.tensor(-torch.inf, dtype=S.dtype, device=S.device))
    full = ~v.any(-1, keepdim=True)                                   # fully masked row: uniform over all n keys
    p = torch.where(full, torch.full_like(S, 1.0 / n), torch.softmax(torch.where(full, torch.zeros_like(Lm), Lm), -1))
    Lmax = torch.where(full, torch.zeros_like(S[..., :1]), Lm.amax(-1, keepdim=True)).abs()
    eps_j = torch.where(v, 2 * U * (S.abs() + Lmax), torch.zeros_like(S))
    rel = eps_j + eps_j.amax(-1, keepdim=True) + 2.0 ** -21 + ((n + 31) // 32 + 7) * U
    return p, p * rel + 2.0 ** -147


@pytest.mark.parametrize("n", [1, 31, 32, 33, 130, 384])
@pytest.mark.parametrize("masking", ["none", "suffix", "holes", "single", "query"])
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("row", [True, False])
def test_strict_softmax_split(n, masking, with_bias, row):
    if n == 384 and (masking in ("suffix", "single") or not with_bias):
        pytest.skip("n = 384 runs the hole and query masks with bias")
    g = _gen(n * 7 + len(masking) + with_bias + 2 * row)
    H, nbt, b0, nb = 2, 4, 1, 2
    lds = _al(n, 4) + 4                                               # lds > n: the columns [n, lds) hold NaN
    S = torch.full((nb * H * n, lds), NAN, device="cuda")
    S[:, :n] = (torch.rand(nb * H * n, n, device="cuda", generator=g) * 2 - 1) * 80
    bias = torch.randn(H, n, n, device="cuda", generator=g) * 4 if with_bias else None
    keep = torch.ones(nbt, n, dtype=torch.bool, device="cuda")
    if masking == "suffix":
        keep[:, n - n // 4:] = False
    elif masking == "holes":
        keep = torch.rand(nbt, n, device="cuda", generator=g) > 0.3
        keep[:, 0] = True
    elif masking == "single":
        keep[:] = False
        keep[:, n // 2] = True
    elif masking == "query":                                          # some fully masked query rows
        keep = torch.rand(nbt, n, device="cuda", generator=g) > 0.5
    mask = None if masking == "none" else (keep if row else keep.t().contiguous()).to(torch.uint8)
    msb, msi = (n, 1) if row else (1, nbt)
    Pn = _al(n, 8)

    def run():
        P = _nan(nb * H * n * SPL * Pn, BF)
        _call("af2_strict_softmax_split", S.data_ptr(), lds, _p(bias), _p(mask), P.data_ptr(), b0, nb, H, n, msb, msi)
        return P
    P = _twice(run)
    L = S[:, :n].double().view(nb, H, n, n) + (bias.double() if with_bias else 0)
    kb = keep[b0:b0 + nb]
    valid = kb[:, :, None] & kb[:, None, :] if mask is not None else torch.ones(nb, n, n, dtype=torch.bool, device="cuda")
    ref, bound = _softmax_ref(L, bias, valid)
    name = f"strict/softmax_split/n{n}/{masking}/{'bias' if with_bias else 'nobias'}/{'row' if row else 'col'}"
    v = _split_out(name, P, (nb * H * n, Pn), n, ref.reshape(nb * H * n, n), bound.reshape(nb * H * n, n))
    v = v.view(nb, H, n, n)
    V = valid[:, None].expand_as(v)
    assert torch.all(v[~V & V.any(-1, keepdim=True)] == 0), f"{name}: a masked key got weight"
    full = ~valid.any(-1)                                             # [nb, n] query rows without a valid key
    if full.any():
        assert torch.all(v.permute(0, 2, 1, 3)[full] == float(torch.tensor(1.0 / n))), f"{name}: a fully masked row is not uniform"


@pytest.mark.parametrize("dh,H,n", [(32, 2, 33), (20, 3, 7), (64, 1, 130)])
@pytest.mark.parametrize("row", [True, False])
def test_strict_gate_split(dh, H, n, row):
    g = _gen(dh + H + n + row)
    nbt, b0, nb = 5, 2, 2
    I = H * dh
    Pi = _al(I, 8)
    T = nbt * n
    p1 = torch.randn(T, 4 * I, device="cuda", generator=g)
    p1[:, 3 * I:] = (torch.rand(T, I, device="cuda", generator=g) * 2 - 1) * 20
    ldo = dh + 3
    O = torch.full((nb * H * n, ldo), NAN, device="cuda")
    O[:, :dh] = torch.randn(nb * H * n, dh, device="cuda", generator=g)
    sb, si = (n, 1) if row else (1, nbt)

    def run():
        og = _nan(T * SPL * Pi, BF)
        _call("af2_strict_gate_split", O.data_ptr(), ldo, p1.data_ptr(), og.data_ptr(), b0, nb, H, n, dh, sb, si)
        return og
    og = _twice(run)
    tok = _tokens(b0, nb, n, sb, si).flatten()                        # [nb * n] tokens of the chunk, b'-major
    o = O[:, :dh].double().view(nb, H, n, dh).permute(0, 2, 1, 3).reshape(nb * n, I)
    ref = o * torch.sigmoid(p1[tok, 3 * I:].double())
    pl = og[: T * SPL * Pi].view(T, SPL, Pi)
    others = torch.ones(T, dtype=torch.bool, device="cuda")
    others[tok] = False
    assert torch.isnan(pl[others]).all(), "rows of tokens outside the chunk written"
    sel = pl[tok].contiguous().flatten()
    _split_out(f"strict/gate_split/dh{dh}H{H}n{n}{'row' if row else 'col'}", torch.cat([sel, _nan(0, BF)]), (nb * n, Pi), I,
               ref, 5 * U * ref.abs())


@pytest.mark.parametrize("mn_major", [False, True])
@pytest.mark.parametrize("gate", [False, True])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("rows,inner,Cc", [(5, 37, 40), (33, 70, 17)])
def test_strict_tok2chan_split(mn_major, gate, masked, rows, inner, Cc):
    g = _gen(rows + inner + Cc + 2 * gate + masked + 4 * mn_major)
    T = rows * inner
    ld = 3 * Cc + 5
    src = torch.randn(T, ld, device="cuda", generator=g)
    src[:, 2 * Cc:3 * Cc] = (torch.rand(T, Cc, device="cuda", generator=g) * 2 - 1) * 20
    mask = (torch.rand(T, device="cuda", generator=g) > 0.3).to(torch.uint8) if masked else None
    P = _al(inner, 8)
    if mn_major:
        cs, hs, rs = SPL * rows * P + 8, rows * P, P
    else:
        cs, hs, rs = rows * SPL * P + 8, P, SPL * P

    def run():
        out = _nan(Cc * cs, BF)
        _call("af2_strict_tok2chan_split", src.data_ptr(), ld, Cc, 2 * Cc if gate else -1, _p(mask), out.data_ptr(), Cc, rows,
              inner, cs, hs, rs)
        return out
    out = _twice(run)
    val = src[:, Cc:2 * Cc].double()
    if gate:
        val = val * torch.sigmoid(src[:, 2 * Cc:3 * Cc].double())
    if masked:
        val = val * mask.double()[:, None]
    ref = val.view(rows, inner, Cc).permute(2, 0, 1)                  # [c][r][k]
    body = out[: Cc * cs].view(Cc, cs)
    assert torch.isnan(body[:, cs - 8:]).all(), "gap after a channel written"
    if mn_major:
        pl = body[:, : cs - 8].view(Cc, SPL, rows, P).permute(0, 2, 1, 3)
    else:
        pl = body[:, : cs - 8].view(Cc, rows, SPL, P)
    flat = torch.cat([pl.contiguous().flatten(), _nan(0, BF)])
    name = f"strict/tok2chan/{'mn' if mn_major else 'k'}/{'gate' if gate else 'nogate'}/{'mask' if masked else 'nomask'}/r{rows}i{inner}C{Cc}"
    v = _split_out(name, flat, (Cc, rows, P), inner, ref, 5 * U * ref.abs(), pads="nan")
    if not gate:
        assert torch.equal(v, ref)


@pytest.mark.parametrize("d", [32, 128, 256, 384])
@pytest.mark.parametrize("n,rows", [(37, 3), (64, 2)])
def test_strict_chan_to_token_layernorm(d, n, rows):
    """mode 0; d 384 takes the opt-in shared-memory path (d * 33 floats > 48 KB)"""
    g = _gen(d + n)
    pitch = _al(n, 4)
    chan_stride = rows * pitch + 4
    src = torch.full((d, chan_stride), NAN, device="cuda")
    body = torch.randn(d, rows, n, device="cuda", generator=g) * 2 + 0.3
    body[:, 0, :5] = 1e3 + torch.randn(d, 5, device="cuda", generator=g)          # mean 1e3 over channels
    body[:, 0, 5] = 1024.0                                                         # constant tokens
    body[:, 0, 6] = -3.5
    src[:, : rows * pitch].view(d, rows, pitch)[..., :n] = body
    gamma = torch.randn(d, device="cuda", generator=g)
    beta = torch.randn(d, device="cuda", generator=g)
    T = rows * n
    gate_ld, gate_off = 2 * d + 3, d + 1
    gsrc = torch.randn(T, gate_ld, device="cuda", generator=g) * 4
    gsrc[5:7, gate_off:gate_off + d] = torch.tensor([0.0, 30.0, -200.0], device="cuda")[torch.arange(d, device="cuda") % 3]
    P = _al(d, 8)

    def run():
        y = _nan(T * SPL * P, BF)
        _call("af2_strict_chan_to_token", src.data_ptr(), chan_stride, pitch, rows, n, d, 0, gamma.data_ptr(), beta.data_ptr(),
              gsrc.data_ptr(), gate_ld, gate_off, None, C.c_float(0.0), C.c_float(1e-5), y.data_ptr())
        return y
    y = _twice(run)
    x = body.double().permute(1, 2, 0).reshape(T, d)
    yl, dy = _ln_ref(x, gamma.double(), beta.double(), (d + 31) // 32 + 5)
    s = torch.sigmoid(gsrc[:, gate_off:gate_off + d].double())
    ref = yl * s
    v = _split_out(f"strict/c2t/ln/d{d}n{n}", y, (T, P), d, ref, s * dy + 5 * U * ref.abs() + 2.0 ** -126 * yl.abs())
    sx = torch.tensor([0.5, 1.0, 0.0], dtype=torch.float64, device="cuda")[torch.arange(d, device="cuda") % 3]
    exact = (beta * sx.float()).double()
    assert torch.equal(v[5:7], exact.expand(2, d)), "a constant token must give exactly beta * gate"


@pytest.mark.parametrize("d", [32, 100, 384])
@pytest.mark.parametrize("with_scale", [False, True])
def test_strict_chan_to_token_scale(d, with_scale):
    g = _gen(d + with_scale)
    n, rows = 45, 3
    pitch = _al(n, 4) + 4
    chan_stride = rows * pitch
    src = torch.full((d, chan_stride), NAN, device="cuda")
    body = torch.randn(d, rows, n, device="cuda", generator=g) * 10
    src.view(d, rows, pitch)[..., :n] = body
    T = rows * n
    scale = torch.rand(T, device="cuda", generator=g) if with_scale else None
    if with_scale:
        scale[::7] = 0.0
    sc = C.c_float(1.0 / 130)
    P = _al(d, 8)

    def run():
        y = _nan(T * SPL * P, BF)
        _call("af2_strict_chan_to_token", src.data_ptr(), chan_stride, pitch, rows, n, d, 1, None, None, None, 0, 0, _p(scale),
              sc, C.c_float(1e-5), y.data_ptr())
        return y
    y = _twice(run)
    x = body.double().permute(1, 2, 0).reshape(T, d)
    s = scale.double()[:, None] if with_scale else torch.tensor(sc.value, dtype=torch.float64, device="cuda")
    ref = x * s
    v = _split_out(f"strict/c2t/scale/d{d}/{'vec' if with_scale else 'const'}", y, (T, P), d, ref, U * ref.abs())
    if with_scale:
        assert torch.all(v[::7] == 0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("nbatch", [1, 5, 130])
@pytest.mark.parametrize("row", [True, False])
def test_tie_queries(dtype, nbatch, row):
    g = _gen(nbatch + row + (dtype == BF))
    n, cols, ld = 37, 40, 3 * 40 + 4
    T = n * nbatch
    buf0 = (torch.randn(T, ld, device="cuda", generator=g) * 2 + 0.5).to(dtype)
    sb, si = (n, 1) if row else (1, nbatch)
    fn = "af2_tie_queries_f32" if dtype == torch.float32 else "af2_tie_queries_bf16"

    def run():
        b = torch.cat([buf0.flatten(), torch.full((GUARD,), NAN, dtype=dtype, device="cuda")])
        _call(fn, b.data_ptr(), ld, cols, n, nbatch, sb, si)
        return b
    out = _twice(run)
    o = out[: T * ld].view(T, ld)
    assert torch.equal(_bits(o[:, cols:]), _bits(buf0[:, cols:])), "columns outside the q block changed"
    tok = _tokens(0, nbatch, n, sb, si)                               # [nbatch, n]
    q = buf0[tok, :cols].double()                                     # [nbatch, n, cols]
    mean = q.mean(0)
    bound = (nbatch + 1) * U * q.abs().mean(0) + (2.0 ** -8 * mean.abs() if dtype == BF else 0)
    got = o[tok, :cols].double()
    assert torch.equal(got, got[:1].expand_as(got)), "tied queries differ across the folded batch"
    check_bound(f"strict/tie_queries/{'f32' if dtype == torch.float32 else 'bf16'}/nb{nbatch}/{'row' if row else 'col'}",
                got[0], mean, bound)
