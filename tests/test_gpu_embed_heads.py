"""-m gpu: the template input projections, the pair-init glue and the distogram head, element-wise against fp64.

  A  af2_template_embed[_strict]    to_template_embed: fp32 feats -> bf16 (or split) -> GEMM + bias      (alphafold2.py:751)
  B  af2_template_angles[_strict]   template_angle_mlp into rows row0 .. row0 + T - 1 of m              (alphafold2.py:789-790)
  C  af2_embed_pair_init            token embedding, MSA init, pair init with relative positions        (alphafold2.py:676-726)
  D  af2_distogram_head             Linear(LayerNorm((x + x^T) / 2))                                     (alphafold2.py:821-823)

Every case calls the C entry with a workspace this test owns, filled with NaN (bytes 0xff are NaN as bf16 and as fp32): an
unzeroed pad column or a read of stale workspace turns into NaN in the output.  Output buffers start as NaN with a guard
region after them that must stay NaN, and two identical launches must be bitwise equal.  References are fp64 from the exact
operands the kernel was given (tests/embed_bounds.py, which test_embed_bounds_controls.py checks on the CPU against
emulated kernels and wrong variants of them).  u = 2^-24, b = 2^-8 (bf16 round-to-nearest), C_GEMM and the GEMM bounds as
in gpu_util.py.

A. bf16: the conversion kernels (f32_to_bf16_vec_kernel when K == align8(K), K % 4 == 0 and feats are 16-byte aligned,
   f32_to_bf16_pad_kernel otherwise) round to nearest and zero the pad columns, so the GEMM sees exactly bf16(feats) and the
   packed bf16(w):  |t - ref| <= gemm_f32_bound over align8(K) terms, ref = bf16(feats) bf16(w)^T + bias in fp64.  A
   truncating conversion leaves up to 2^-8 relative error per operand, orders of magnitude above that bound.  strict: the
   three split planes carry the fp32 operands exactly, gemm_split_bound against fp32 feats w^T + bias.
B. The workspace holds the hidden activation h where the entry takes it (template_api.inl: after align_up(R Kp 2, 256)
   bytes of converted angles, R Kp 2 3 in strict mode), so each stage is gated on its own:
   bf16   stage 1  h = bf16(gelu(z)), z = bf16(a) bf16(w1)^T + b1:  |h - gelu(z)| <= b |h| + 1.13 E1 + eps_gelu(z),
                   E1 = C_GEMM Kp u sum|a w1| (the bf16-store bound of test_gpu_kernels.py; 1.13 >= max |gelu'|)
          stage 2  rows of m against h_kernel bf16(w2)^T + b2: gemm_f32_bound over d terms
   strict stage 1  h = a w1^T + b1 in fp32: gemm_split_bound
          stage 2  the split GELU kernel feeds gelu(h_kernel) with error dg (test_gpu_strict_kernels.py _gelu_ref):
                   gemm_split_bound over d terms + sum_j |w2_ij| dg_j
   and end to end against the module's fp64 output from its fp32 weights (embed_bounds.angles_module_ref):
          |out - ref| <= sum_j |w2_ij| dh_j + C d u sum_j (|h_j| + dh_j) |w2_ij| + 2 u |ref|
   with dh the hidden activation's error from the fp32 operands (in bf16 mode it includes the operand roundings of a, w1,
   and the packed bf16(w2) adds b sum |h w2|).  Biases are N(0, 1), so a dropped bias exceeds every bound.  m is NaN
   before the call: rows [row0, row0 + T) of every batch element must come out finite, every other row bitwise unchanged.
C. m: the kernels evaluate (emb[msa] (+ msa_embed)) + (emb[seq] (+ seq_embed)) with IEEE fp32 adds, so it must equal the
   same fp32 torch expression bitwise.  x: lr = e W^T + b is a per-lane fmaf chain of ceil(d/32) terms, 5 shuffle levels
   and the bias add, dlr <= (ceil(d/32) + 5) u sum|e w| + u |lr|; x = (l_i + r_j) + pos[clamp(idx_i - idx_j, -R, R) + R]
   adds two roundings:  |x - ref| <= (1 + 2u) (dl_i + dr_j) + u |l_i + r_j| + u |ref|.  Token ids cover the whole vocabulary
   (the last row included); seq_index is non-monotonic with gaps beyond +-R on both sides.
D. v = (x_ij + x_ji) * 0.5 carries u |v|.  LayerNorm (one warp per token, VPL = d / 32 values per lane): _ln_ref of
   test_gpu_strict_kernels.py with k_d = VPL + 5, plus what the rounded v does to it, |gamma| rstd u (|v| + mean|v| +
   |xhat| rstd mean(|v - mean| |v|)) (the shift of v, of its mean, and the first-order change of the variance).  The Linear
   is a per-lane fmaf chain + 5 shuffle levels + the bias add:  |out - ref| <= sum|w| dy + (VPL + 5) u sum(|y| + dy)|w| +
   u |out|.  Inputs include tokens with a common offset of ~150 (the mean cancels) and tokens of variance ~1e-4 (eps
   matters).  out[b, i, j] must equal out[b, j, i] bitwise: the kernel forms the same v for both orders.

Rejections: every rejected call gets buffers sized for the call as given plus slack (spare rows, a wider d), must return
AF2_ERR_BAD_ARG, launch nothing (af2_launch_count unchanged) and leave its NaN outputs untouched.
"""
import ctypes as C

import pytest
import torch

import embed_bounds as E
from gpu_util import check_bound

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 4096
BAD_ARG = -1


def _ops():
    from alphafold2_b200 import ops
    return ops


def _lib():
    from alphafold2_b200 import _lib
    return _lib.load()


def _rc(fn, *args):
    return getattr(_lib(), fn)(*args, _ops()._stream_ptr())


def _ok(fn, *args):
    from alphafold2_b200 import _lib as L
    L.check(_rc(fn, *args))


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _nan(n):
    return torch.full((n + GUARD,), NAN, device="cuda")


def _ws(nbytes):
    return torch.full((int(nbytes),), 0xFF, dtype=torch.uint8, device="cuda")


def _p(t):
    return 0 if t is None else t.data_ptr()


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _twice(run):
    """run() -> tuple of buffers, the first a NaN-guarded output; two runs must agree bitwise and leave the guard NaN"""
    a, b = run(), run()
    for x, y in zip(a, b):
        assert torch.equal(_bits(x), _bits(y)), "two identical launches differ"
    assert torch.isnan(a[0][-GUARD:]).all(), "guard region written"
    return a


def _rejected(fn, args, bufs):
    """the call returns AF2_ERR_BAD_ARG, launches nothing and leaves the NaN buffers untouched"""
    n0 = _lib().af2_launch_count()
    rc = _rc(fn, *args)
    torch.cuda.synchronize()
    assert rc == BAD_ARG, f"{fn}: rc {rc}"
    assert _lib().af2_launch_count() == n0, f"{fn}: launched a kernel before rejecting"
    for b in bufs:
        assert torch.isnan(b).all(), f"{fn}: wrote before rejecting"


# ------------------------------------------------------------------------------------------------------------------------
# A. to_template_embed
# ------------------------------------------------------------------------------------------------------------------------
EMBED_K = {"vec32": (32, 0), "pad32_offset4": (32, 1), "k1": (1, 0), "k55": (55, 0), "k200": (200, 0)}


def _embed_case(kcase, d, rows, strict):
    ops = _ops()
    K, off = EMBED_K[kcase]
    g = _gen(K * 7 + d + rows)
    fbuf = torch.randn(rows * K + off, generator=g, device="cuda")
    feats = fbuf[off:].view(rows, K)                         # off = 1: based 4 bytes past an aligned address
    w, bias = torch.randn(d, K, generator=g, device="cuda") * K ** -0.5, torch.randn(d, generator=g, device="cuda")
    pk = ops.pack_linear(w, bias, strict)
    fn = "af2_template_embed_strict" if strict else "af2_template_embed"
    nws = getattr(_lib(), fn + "_workspace")(rows, K)

    def run():
        out, ws = _nan(rows * d), _ws(nws)
        _ok(fn, pk.tensors["w"].data_ptr(), pk.tensors["b"].data_ptr(), feats.data_ptr(), out.data_ptr(), rows, K, d,
            ws.data_ptr(), nws)
        return (out,)
    out, = _twice(run)
    ref, bound = E.template_embed_ref(feats, w, bias, strict)
    mode = "strict" if strict else "bf16"
    check_bound(f"{mode}/template_embed/{kcase}/d{d}/rows{rows}", out[:rows * d].view(rows, d), ref, bound)


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("d", [32, 36, 128, 256])
@pytest.mark.parametrize("kcase", list(EMBED_K))
def test_template_embed_against_fp64(kcase, d, strict):
    _embed_case(kcase, d, 129, strict)


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("rows", [1, 127, 2 * 3 * 37 ** 2, 70001])
@pytest.mark.parametrize("kcase,d", [("k55", 128), ("vec32", 256)])
def test_template_embed_rows(kcase, d, rows, strict):
    _embed_case(kcase, d, rows, strict)


@pytest.mark.parametrize("strict", [False, True])
def test_template_embed_rejects(strict):
    """d % 4 and each null pointer; buffers sized for d = 40"""
    ops = _ops()
    rows, K, D = 9, 32, 40
    feats = torch.randn(rows, K, device="cuda")
    pk = ops.pack_linear(torch.randn(D, K, device="cuda"), torch.randn(D, device="cuda"), strict)
    fn = "af2_template_embed_strict" if strict else "af2_template_embed"
    ws = _ws(getattr(_lib(), fn + "_workspace")(rows, K))
    w, b = pk.tensors["w"].data_ptr(), pk.tensors["b"].data_ptr()
    for d, wp, fp, null_out in ((34, w, feats.data_ptr(), False), (36, 0, feats.data_ptr(), False), (36, w, 0, False),
                                (36, w, feats.data_ptr(), True)):
        out = _nan(rows * D)
        _rejected(fn, (wp, b, fp, 0 if null_out else out.data_ptr(), rows, K, d, ws.data_ptr(), ws.numel()), [out])


# ------------------------------------------------------------------------------------------------------------------------
# B. template angle MLP
# ------------------------------------------------------------------------------------------------------------------------
S_MSA = 3


def _angle_weights(K, d, g):
    w1, b1 = torch.randn(d, K, generator=g, device="cuda") * K ** -0.5, torch.randn(d, generator=g, device="cuda")
    w2, b2 = torch.randn(d, d, generator=g, device="cuda") * d ** -0.5, torch.randn(d, generator=g, device="cuda")
    return w1, b1, w2, b2


def _angles_case(B, T, n, K, d, where, strict):
    ops = _ops()
    m_rows = S_MSA + T + 2
    row0 = {"first": 0, "after_msa": S_MSA, "last": m_rows - T}[where]
    g = _gen(B * 1000 + T * 100 + n + K + d)
    angles = torch.randn(B, T, n, K, generator=g, device="cuda")
    w1, b1, w2, b2 = _angle_weights(K, d, g)
    pk = ops.pack_template_angles(w1, b1, w2, b2, strict)
    fn = "af2_template_angles_strict" if strict else "af2_template_angles"
    nws = getattr(_lib(), fn + "_workspace")(B, T, n, K, d)
    R, Kp = B * T * n, E.a8(K)
    off_h = (R * Kp * 2 * (3 if strict else 1) + 255) // 256 * 256
    size = B * m_rows * n * d

    def run():
        mb, ws = _nan(size), _ws(nws)
        _ok(fn, C.byref(pk.struct), angles.data_ptr(), mb.data_ptr(), B, T, n, K, d, m_rows, row0, ws.data_ptr(), nws)
        return mb, ws
    mb, ws = _twice(run)
    if strict:
        h = ws[off_h:off_h + R * d * 4].view(torch.float32).view(R, d)
    else:
        h = ws[off_h:off_h + R * d * 2].view(torch.bfloat16).view(R, d)
    m = mb[:size].view(B, m_rows, n, d)
    assert E.angle_rows_layout(torch.full_like(m, NAN), m, row0, T), "rows outside [row0, row0 + T) written, or rows inside not"
    rows = m[:, row0:row0 + T].reshape(R, d)
    a = angles.view(R, K)
    name = f"{'strict' if strict else 'bf16'}/template_angles/B{B}T{T}n{n}K{K}d{d}/{where}"
    check_bound(name + "/stage1", h, *E.angles_stage1_ref(a, w1, b1, strict))
    check_bound(name + "/stage2", rows, *E.angles_stage2_ref(h, w2, b2, strict))
    check_bound(name + "/module", rows, *E.angles_module_ref(a, w1, b1, w2, b2, strict))


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("d", [32, 64, 256, 264])
@pytest.mark.parametrize("K", [3, 8, 32, 55])
def test_template_angles_against_fp64(K, d, strict):
    _angles_case(3, 4, 37, K, d, "after_msa", strict)


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("where", ["first", "after_msa", "last"])
@pytest.mark.parametrize("n", [1, 37, 130])
@pytest.mark.parametrize("B,T", [(1, 1), (1, 4), (3, 1), (3, 4)])
def test_template_angles_layout(B, T, n, where, strict):
    _angles_case(B, T, n, 55, 264, where, strict)


@pytest.mark.parametrize("strict", [False, True])
def test_template_angles_rejects(strict):
    """d % 8, row0 < 0 and row0 + T > m_rows are rejected; T = 0 and n = 0 return OK and write nothing.  m has T spare rows
    and room for d = 40."""
    ops = _ops()
    B, T, n, K, D = 2, 2, 5, 55, 40
    m_rows = S_MSA + T
    pk = ops.pack_template_angles(*_angle_weights(K, D, _gen(5)), strict)
    fn = "af2_template_angles_strict" if strict else "af2_template_angles"
    angles = torch.randn(B, T, n, K, device="cuda")
    ws = _ws(getattr(_lib(), fn + "_workspace")(B, T, n, K, D))
    for d, row0 in ((36, S_MSA), (40, -1), (40, m_rows - T + 1)):
        mb = _nan(B * (m_rows + T) * n * D)
        _rejected(fn, (C.byref(pk.struct), angles.data_ptr(), mb.data_ptr(), B, T, n, K, d, m_rows, row0, ws.data_ptr(),
                       ws.numel()), [mb])
    for t_, n_ in ((0, n), (T, 0)):
        mb = _nan(B * (m_rows + T) * n * D)
        n0 = _lib().af2_launch_count()
        _ok(fn, C.byref(pk.struct), angles.data_ptr(), mb.data_ptr(), B, t_, n_, K, D, m_rows, S_MSA, ws.data_ptr(), ws.numel())
        torch.cuda.synchronize()
        assert _lib().af2_launch_count() == n0 and torch.isnan(mb).all(), f"T {t_} n {n_}: launched or wrote"


# ------------------------------------------------------------------------------------------------------------------------
# C. pair init
# ------------------------------------------------------------------------------------------------------------------------
VOCAB = 22


def _pair_inputs(B, S, n, d, R, embeds, index, g):
    dev = "cuda"
    emb = torch.randn(VOCAB, d, generator=g, device=dev)
    wp, bp = torch.randn(2 * d, d, generator=g, device=dev) * d ** -0.5, torch.randn(2 * d, generator=g, device=dev)
    pos = torch.randn(2 * R + 1, d, generator=g, device=dev)
    seq = torch.randint(0, VOCAB, (B, n), generator=g, device=dev)
    msa = torch.randint(0, VOCAB, (B, S, n), generator=g, device=dev)
    seq.view(-1)[0] = VOCAB - 1                              # the last embedding row is read
    msa.view(-1)[-1] = VOCAB - 1
    se = torch.randn(B, n, d, generator=g, device=dev) if embeds else None
    me = torch.randn(B, S, n, d, generator=g, device=dev) if embeds else None
    # non-monotonic, gaps beyond +-R on both sides and many inside
    si = torch.randint(-4 * R - 5, 4 * R + 6, (n,), generator=g, device=dev) if index else None
    return emb, wp, bp, pos, seq, msa, se, me, si


def _pair_call(inp, B, S, n, d, R):
    emb, wp, bp, pos, seq, msa, se, me, si = inp
    nws = _lib().af2_embed_pair_init_workspace(B, n, d)

    def run():
        xb, mb, ws = _nan(B * n * n * d), _nan(B * S * n * d), _ws(nws)
        _ok("af2_embed_pair_init", seq.data_ptr(), msa.data_ptr(), emb.data_ptr(), VOCAB, _p(se), _p(me), wp.data_ptr(),
            bp.data_ptr(), pos.data_ptr(), R, _p(si), xb.data_ptr(), mb.data_ptr(), B, S, n, d, ws.data_ptr(), nws)
        return xb, mb
    xb, mb = _twice(run)
    assert torch.isnan(mb[-GUARD:]).all(), "guard after m written"
    return xb[:B * n * n * d].view(B, n, n, d), mb[:B * S * n * d].view(B, S, n, d)


# (d, n, B, S, R, embeds, index): d at the vector widths' edges (4 channels: one lane; 1024: the limit), n > 2R + 1 where
# the clamp must bite, and the shapes of the earlier tolerance test (256 256 1 128, 128 70 2 5, 32 24 2 3)
PAIR_CASES = ([(d, 33, 3, 5, 1, True, True) for d in (4, 36, 100, 256, 1024)]
              + [(d, 200, 1, 1, 32, False, True) for d in (4, 36, 100, 256, 1024)]
              + [(d, 2, 3, 1, 1, False, False) for d in (4, 100)]
              + [(36, 1, 1, 5, 1, True, False), (1024, 1, 3, 1, 32, True, True), (100, 70, 1, 5, 32, True, False),
                 (256, 256, 1, 128, 32, False, False), (128, 70, 2, 5, 32, True, True), (32, 24, 2, 3, 32, False, False)])


@pytest.mark.parametrize("d,n,B,S,R,embeds,index", PAIR_CASES)
def test_pair_init_against_fp64(d, n, B, S, R, embeds, index):
    inp = _pair_inputs(B, S, n, d, R, embeds, index, _gen(d * 7 + n + B + S))
    emb, wp, bp, pos, seq, msa, se, me, si = inp
    x, m = _pair_call(inp, B, S, n, d, R)
    e, mref = E.token_embed(emb, seq, msa, se, me)
    assert torch.equal(m.view(torch.int32), mref.view(torch.int32)), \
        f"MSA init not bitwise: max |err| {(m - mref).abs().max().item():.3e}"
    ref, bound = E.pair_init_ref(e, wp, bp, pos, R, si)
    check_bound(f"pair_init/d{d}n{n}B{B}S{S}R{R}{'/embeds' if embeds else ''}{'/index' if index else ''}", x, ref, bound)


def test_pair_init_host_loop_with_spare_rows():
    """ops.embed_pair_init with m_rows > S and B = 2 runs one call per batch element into its slice of m: the same bits as one
    whole-batch call"""
    B, S, n, d, R = 2, 5, 70, 128, 32
    inp = _pair_inputs(B, S, n, d, R, True, True, _gen(11))
    emb, wp, bp, pos, seq, msa, se, me, si = inp
    x0, m0 = _pair_call(inp, B, S, n, d, R)
    x, m = _ops().embed_pair_init(seq, msa, emb, wp, bp, pos, R, se, me, si, m_rows=S + 3)
    assert tuple(m.shape) == (B, S + 3, n, d)
    assert torch.equal(x.view(torch.int32), x0.view(torch.int32))
    assert torch.equal(m[:, :S].contiguous().view(torch.int32), m0.view(torch.int32))


def test_pair_init_rejects():
    """d % 4 and d > 1024; buffers sized for d = 1032"""
    B, S, n, D, R = 1, 2, 3, 1032, 1
    emb, wp, bp, pos, seq, msa, _, _, _ = _pair_inputs(B, S, n, D, R, False, False, _gen(3))
    ws = _ws(_lib().af2_embed_pair_init_workspace(B, n, D))
    for d in (6, 1028):
        xb, mb = _nan(B * n * n * D), _nan(B * S * n * D)
        _rejected("af2_embed_pair_init", (seq.data_ptr(), msa.data_ptr(), emb.data_ptr(), VOCAB, 0, 0, wp.data_ptr(),
                                          bp.data_ptr(), pos.data_ptr(), R, 0, xb.data_ptr(), mb.data_ptr(), B, S, n, d,
                                          ws.data_ptr(), ws.numel()), [xb, mb])


# ------------------------------------------------------------------------------------------------------------------------
# D. distogram head
# ------------------------------------------------------------------------------------------------------------------------
def _distogram_case(B, n, d, nb):
    x, gamma, beta, w, bias = E.distogram_inputs(B, n, d, nb, _gen(B * 10000 + n * 10 + d + nb), "cuda")
    size = B * n * n * nb

    def run():
        ob = _nan(size)
        _ok("af2_distogram_head", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), w.data_ptr(), bias.data_ptr(), ob.data_ptr(),
            B, n, d, nb)
        return (ob,)
    ob, = _twice(run)
    out = ob[:size].view(B, n, n, nb)
    assert torch.equal(out.view(torch.int32), out.transpose(1, 2).contiguous().view(torch.int32)), "out[b, i, j] != out[b, j, i]"
    via_ops = _ops().distogram_head(x, gamma, beta, w, bias)
    assert torch.equal(via_ops.view(torch.int32), out.view(torch.int32)), "ops.distogram_head differs from the C entry"
    step = max(1, (1 << 23) // (n * d))                       # the fp64 reference in bands of pair rows
    parts = [E.distogram_ref(x, gamma, beta, w, bias, slice(i, min(n, i + step))) for i in range(0, n, step)]
    ref, bound = torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1)
    check_bound(f"distogram/B{B}n{n}d{d}nb{nb}", out, ref, bound)


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("n", [1, 2, 9, 33, 130])
@pytest.mark.parametrize("d", [128, 256, 384, 512])
def test_distogram_against_fp64(d, n, B):
    _distogram_case(B, n, d, 37)


@pytest.mark.parametrize("d,n,B,nb", [(d, 33, 2, nb) for d in (128, 256) for nb in (1, 33, 64)]
                         + [(512, 700, 1, 37), (256, 256, 1, 37), (128, 70, 2, 37), (512, 9, 1, 99)])
def test_distogram_buckets_and_rounds(d, n, B, nb):
    """outputs across two 32-output chunks, many grid-stride rounds per warp at n 700, the largest bucket count that fits
    at d 512"""
    _distogram_case(B, n, d, nb)


@pytest.mark.parametrize("d,nb", [(128, 37), (512, 37), (96, 37), (640, 37), (512, 99), (512, 100), (512, 101), (384, 132),
                                  (384, 133)])
def test_distogram_shape_rule_matches_the_c_entry(d, nb):
    """ops.distogram_head_ok and af2_distogram_head accept and reject the same (d, buckets); a rejected call launches nothing.
    x and w are sized for max(d, 512) channels, so an accepted call never reads past them."""
    B, n = 1, 9
    D = max(d, 512)
    x = torch.randn(B * n * n * D, device="cuda")
    gamma, beta = torch.ones(D, device="cuda"), torch.zeros(D, device="cuda")
    w, bias = torch.randn(nb * D, device="cuda"), torch.zeros(nb, device="cuda")
    out = _nan(B * n * n * nb)
    args = (x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), B, n, d, nb)
    if _ops().distogram_head_ok(d, nb):
        _ok("af2_distogram_head", *args)
        torch.cuda.synchronize()
        assert torch.isfinite(out[:B * n * n * nb]).all() and torch.isnan(out[-GUARD:]).all()
    else:
        _rejected("af2_distogram_head", args, [out])
