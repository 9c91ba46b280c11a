"""-m gpu: building-block kernels against fp64 math: the wgmma GEMM with every epilogue (gemm_tc.cuh), the pair-bias kernels,
LayerNorm and rotary.

References are fp64, evaluated on the GPU with plain torch from the exact bf16 / fp32 operands the kernel was given, and
every element is gated by a bound derived from the kernel's documented rounding (worst err / bound per case goes to the
parity report):

GEMM (bf16 operands, fp32 accumulation in the tensor cores, K-term accumulation error):
    E = C_GEMM * K * 2^-24 * sum_k |a_k b_k|                         (accumulator error of one column)
  bf16 stores:   |out - ref| <= 2^-8 |ref| + |rs| * (A' E + eps_act(x))
    x = acc + bias, ref = act(x) * rs; A' bounds |act'| (1 none, 1/4 sigmoid, 1.13 erf-GELU); eps_act is the documented
    error of the kernel's approximations (common.cuh): sigmoid ~1e-6 relative, erf-GELU 1.5e-7 absolute on erf, i.e.
    eps_gelu(x) = 1.5e-7 |x| + 1e-6 |gelu(x)|.
  gated:         |out - ref| <= 2^-8 |ref| + |rs| * (|act(g)| E_u + |u| (A' E_g + eps_act(g))),  ref = u act(g) rs
  fp32 stores:   |out - ref| <= E + 2^-23 |ref| + 2^-24 |resid|  (two fp32 roundings: + bias, + residual; E + 2^-23 |ref| is
                 gpu_util.gemm_f32_bound, shared with test_gpu_contractions.py)
  Activations and gates are applied in fp64 in the reference; 2^-8 is the unit roundoff of the bf16 store.  Rows whose row
  scale is 0 must come out exactly 0.  C_GEMM = 1 holds on an H100 80GB HBM3 (700 W power limit): worst err / bound 0.28 on the fp32
  outputs, 0.99 on the bf16 ones, where the rounding term alone reaches ~1 for outputs that round by nearly half an ulp.

Pair bias (fp32 x, w):  |out - ref| <= 2^-8 |ref| + 2^-14 sum_k |x_k w_k|; the tensor-core kernel carries ~16 bits per
operand (hi + lo bf16 splits, three products), the SIMT and LayerNorm-kernel paths are fp32 FMA chains.

Output buffers are filled with NaN first: every element outside the valid output (pitch padding, columns past out_cols,
rows past M, the element before an offset base) must still be NaN afterwards.
"""
import pytest
import torch

from conftest import load_golden
from gpu_util import C_GEMM, U32 as U, check_bound, gemm_f32_bound

pytestmark = pytest.mark.gpu


def _ops():
    from alphafold2_b200 import ops
    return ops


# ------------------------------------------------------------------------------------------------------------------------
# GEMM epilogues
# ------------------------------------------------------------------------------------------------------------------------
ACT_D = {0: 1.0, 1: 0.25, 2: 1.13}


def _act(x, act):
    if act == 1:
        return torch.sigmoid(x)
    if act == 2:
        return torch.nn.functional.gelu(x)
    return x


def _act_eps(x, act):
    if act == 1:
        return 1e-6 * torch.sigmoid(x)
    if act == 2:
        return 1.5e-7 * x.abs() + 1e-6 * torch.nn.functional.gelu(x).abs()
    return torch.zeros_like(x)


def _operand(logical, mn_major):
    """logical [batch, rows, K] -> the stored operand (K-major as is, MN-major [batch, K, rows])"""
    return (logical.transpose(1, 2) if mn_major else logical).contiguous()


def _out_index(batch, M, ncols, layout, store, dev):
    """flat element index of (b, row, col) in the output buffer, plus the epilogue pitch arguments"""
    b = torch.arange(batch, device=dev)[:, None, None]
    r = torch.arange(M, device=dev)[None, :, None]
    c = torch.arange(ncols, device=dev)[None, None, :]
    off = 1 if store == "scalar" else 0                      # odd base: no paired stores
    if layout == 0:
        ld = ncols + (1 if ncols % 2 == 0 else 0) if store == "scalar" else ncols + (ncols % 2) + 2
        ob = M * ld + (3 if store == "scalar" else 4)
        idx = off + b * ob + r * ld + c
        kw = dict(ld_out=ld, out_batch=ob)
    else:
        inner, pitch = 13, 16                                # cm_inner not a multiple of 8
        ld = (M + inner - 1) // inner * pitch + 3
        ob = ld * ncols + 5
        idx = off + b * ob + c * ld + (r // inner) * pitch + r % inner
        kw = dict(ld_out=ld, out_batch=ob, cm_inner=inner, cm_pitch=pitch)
    size = off + batch * kw["out_batch"] + 16
    return idx, size, off, kw


def gemm_case(name, *, M, K, nout, batch, bn, mn_major, mode, act, layout, rowscale, store, seed, bias=True):
    ops = _ops()
    dev = "cuda"
    g = torch.Generator().manual_seed(seed)
    gated = mode == ops.EPI_GATED_BF16
    half = bn // 2
    a = torch.randn(batch, M, K, generator=g).bfloat16()
    if gated:
        tiles = (nout + half - 1) // half
        wv = torch.randn(batch, nout, K, generator=g).bfloat16().float()
        wg = torch.randn(batch, nout, K, generator=g).bfloat16().float()
        bv, bg = torch.randn(nout, generator=g), torch.randn(nout, generator=g)
        packed = [ops.pack_gated(wv[i], bv, wg[i], bg, half) for i in range(batch)]
        w = torch.stack([p[0] for p in packed]).bfloat16()
        bvec = packed[0][1]
        nacc = tiles * bn
    else:
        nacc = (nout + 7) // 8 * 8 if mn_major else nout     # MN-major operand pitches must be 16-byte multiples
        w = torch.randn(batch, nacc, K, generator=g).bfloat16()
        bvec = torch.randn((nacc + bn - 1) // bn * bn, generator=g)
    bvec = bvec if bias else None
    rs = None
    if rowscale:
        rs = torch.rand(batch * M, generator=g) * 1.5 + 0.5
        rs[torch.rand(batch * M, generator=g) < 0.25] = 0.0
    a, w = a.to(dev), w.to(dev)
    idx, size, off, kw = _out_index(batch, M, nout, layout, store, dev)
    f32 = mode in (ops.EPI_RESID_F32, ops.EPI_STORE_F32)
    buf = torch.full((size,), float("nan"), dtype=torch.float32 if f32 else torch.bfloat16, device=dev)
    resid = None
    if mode == ops.EPI_RESID_F32:                            # in place: out == resid
        resid = torch.randn(batch, M, nout, generator=g).to(dev)
        buf[idx] = resid
    out = ops.gemm_bf16_epilogue(_operand(a, mn_major), _operand(w, mn_major), buf[off:], bn=bn, mode=mode, act=act,
                                 layout=layout, mn_major=mn_major, bias=None if bvec is None else bvec.to(dev),
                                 rowscale=None if rs is None else rs.to(dev),
                                 resid=buf[off:] if resid is not None else None, ld_resid=kw["ld_out"],
                                 out_cols=nout, **kw)
    torch.cuda.synchronize()
    # ---- fp64 reference ----
    a64 = a.double()
    rs64 = torch.ones(batch, M, 1, dtype=torch.float64, device=dev) if rs is None else rs.to(dev).double().view(batch, M, 1)
    if gated:
        wv64, wg64 = wv.to(dev).double(), wg.to(dev).double()
        u = a64 @ wv64.transpose(1, 2)
        gg = a64 @ wg64.transpose(1, 2)
        eu = C_GEMM * K * U * (a64.abs() @ wv64.abs().transpose(1, 2))
        eg = C_GEMM * K * U * (a64.abs() @ wg64.abs().transpose(1, 2))
        if bias:
            u, gg = u + bv.to(dev).double(), gg + bg.to(dev).double()
        ref = u * _act(gg, act) * rs64
        bound = 2.0 ** -8 * ref.abs() + rs64.abs() * (_act(gg, act).abs() * eu + u.abs() * (ACT_D[act] * eg + _act_eps(gg, act)))
    else:
        w64 = w.double()[:, :nout]
        x = a64 @ w64.transpose(1, 2)
        absdot = a64.abs() @ w64.abs().transpose(1, 2)
        e = C_GEMM * K * U * absdot
        if bias:
            x = x + bvec[:nout].to(dev).double()
        if mode == ops.EPI_RESID_F32:
            ref = x + resid.double()
            bound = gemm_f32_bound(absdot, K, ref) + U * resid.double().abs()
        elif mode == ops.EPI_STORE_F32:
            ref = x
            bound = gemm_f32_bound(absdot, K, ref)
        else:
            ref = _act(x, act) * rs64
            bound = 2.0 ** -8 * ref.abs() + rs64.abs() * (ACT_D[act] * e + _act_eps(x, act))
    got = out[idx - off]
    check_bound(name, got, ref, bound)
    written = torch.zeros(size, dtype=torch.bool, device=dev)
    written[idx.flatten()] = True
    stray = ~torch.isnan(buf[~written].float())
    assert not stray.any(), f"{name}: {int(stray.sum())} elements written outside the output"
    return a, w, bvec, rs, out, idx - off, kw


# (mode, act, layout, rowscale): every combination launch_gemm maps to an EK_* kind at BN = 256, plus generic-only ones
KINDS = {
    "store_tok": (0, 0, 0, False),            # EK_STORE_TOK
    "store_tok_sig": (0, 1, 0, False),        # EK_STORE_TOK_SIG
    "store_ch": (0, 0, 1, False),             # EK_STORE_CH
    "store_ch_rs": (0, 0, 1, True),           # EK_STORE_CH with the row scale
    "gated_tok_gelu": (1, 2, 0, False),       # EK_GATED_TOK_GELU
    "gated_ch_sig": (1, 1, 1, False),         # EK_GATED_CH_SIG
    "gated_ch_sig_rs": (1, 1, 1, True),       # EK_GATED_CH_SIG with the row scale
    "resid_f32": (2, 0, 0, False),            # EK_RESID_F32, in place
    "store_f32": (3, 0, 0, False),            # EK_STORE_F32
    "store_tok_gelu_rs": (0, 2, 0, True),     # EK_GENERIC at every BN
    "gated_tok_sig_rs": (1, 1, 0, True),      # EK_GENERIC
    "store_ch_sig": (0, 1, 1, False),         # EK_GENERIC
}


def _nout(kind, bn):
    """odd output column count whose last column tile is partial"""
    W = bn // 2 if KINDS[kind][0] == 1 else bn
    return W + W // 2 + 1


def _run_kind(kind, bn, mn_major, store, M, K, batch, seed, nout=None, tag=""):
    mode, act, layout, rs = KINDS[kind]
    if mode == 2:
        batch = 1
    nout = nout or _nout(kind, bn)
    name = f"gemm {kind}{tag} bn{bn} {'mn' if mn_major else 'k'} {store} M{M} N{nout} K{K} b{batch}"
    return gemm_case(name, M=M, K=K, nout=nout, batch=batch, bn=bn, mn_major=mn_major, mode=mode, act=act, layout=layout,
                     rowscale=rs, store=store, seed=seed, bias=mode != 3)


@pytest.mark.parametrize("store", ["vec", "scalar"])
@pytest.mark.parametrize("mn_major", [False, True], ids=["kmajor", "mnmajor"])
@pytest.mark.parametrize("bn", [256, 128, 64])
@pytest.mark.parametrize("kind", list(KINDS))
def test_gemm_epilogue(kind, bn, mn_major, store):
    _run_kind(kind, bn, mn_major, store, M=296, K=200, batch=2,
              seed=100 * list(KINDS).index(kind) + bn + 7 * mn_major + 3 * (store == "scalar"))


@pytest.mark.parametrize("K", [8, 40, 584])
@pytest.mark.parametrize("mn_major", [False, True], ids=["kmajor", "mnmajor"])
@pytest.mark.parametrize("bn", [256, 128, 64])
@pytest.mark.parametrize("kind", ["store_f32", "gated_tok_gelu"])
def test_gemm_k_depth(kind, bn, mn_major, K):
    """fewer k-blocks than pipeline stages (3 / 4 / 6 for BN 256 / 128 / 64) and many more"""
    _run_kind(kind, bn, mn_major, "vec", M=136, K=K, batch=1, seed=K + bn)


@pytest.mark.parametrize("mn_major", [False, True], ids=["kmajor", "mnmajor"])
@pytest.mark.parametrize("bn", [256, 128, 64])
@pytest.mark.parametrize("kind", ["store_f32", "gated_ch_sig_rs"])
def test_gemm_many_tiles(kind, bn, mn_major):
    """65 x 5 = 325 output tiles > 2 x 132 SMs: the persistent producer wraps its stage / phase across tiles many times"""
    W = bn // 2 if KINDS[kind][0] == 1 else bn
    _run_kind(kind, bn, mn_major, "vec", M=8200, K=136, batch=1, seed=bn + 1, nout=5 * W - 3)


@pytest.mark.parametrize("kind,bn,mn_major", [("gated_tok_gelu", 256, False), ("store_f32", 128, True),
                                              ("store_ch_rs", 64, False)])
def test_gemm_tile_alone_bitwise(kind, bn, mn_major):
    """a 128-row tile computed alone has the bits it has inside a 325-tile launch; two identical launches agree bit for bit"""
    ops = _ops()
    mode, act, layout, _ = KINDS[kind]
    W = bn // 2 if mode == 1 else bn
    nout = 5 * W - 3
    a, w, bvec, rs, out, idx, kw = _run_kind(kind, bn, mn_major, "vec", M=8200, K=136, batch=1, seed=7, nout=nout)
    bits = torch.int16 if out.dtype == torch.bfloat16 else torch.int32
    again = torch.full_like(out, float("nan"))
    ops.gemm_bf16_epilogue(_operand(a, mn_major), _operand(w, mn_major), again, bn=bn, mode=mode, act=act, layout=layout,
                           mn_major=mn_major, bias=None if bvec is None else bvec.cuda(), rowscale=None if rs is None else rs.cuda(),
                           out_cols=nout, **kw)
    assert torch.equal(again[idx].view(bits), out[idx].view(bits))
    for mt in (0, 37, 64):
        r0, r1 = mt * 128, min(8200, mt * 128 + 128)
        _, size, _, kw1 = _out_index(1, r1 - r0, nout, layout, "vec", "cuda")
        one = torch.full((size,), float("nan"), dtype=out.dtype, device="cuda")
        ops.gemm_bf16_epilogue(_operand(a[:, r0:r1], mn_major), _operand(w, mn_major), one, bn=bn, mode=mode, act=act,
                               layout=layout, mn_major=mn_major, bias=None if bvec is None else bvec.cuda(),
                               rowscale=None if rs is None else rs[r0:r1].contiguous().cuda(), out_cols=nout, **kw1)
        idx1, _, _, _ = _out_index(1, r1 - r0, nout, layout, "vec", "cuda")
        assert torch.equal(one[idx1].view(bits), out[idx[:, r0:r1]].view(bits)), f"tile {mt} differs when run alone"


# the public fp32 entry point (af2_gemm_bf16_f32, tile width picked from N) under the same element-wise bound
def _gemm_store_f32(mn_major, M, N, K, batch):
    ops = _ops()
    torch.manual_seed(M + N + K)
    a = torch.randn(batch, M, K, device="cuda").bfloat16()
    b = torch.randn(batch, N, K, device="cuda").bfloat16()
    c = ops.gemm_bf16(_operand(a, mn_major), _operand(b, mn_major), mn_major=mn_major)
    ref = a.double() @ b.double().transpose(1, 2)
    bound = gemm_f32_bound(a.double().abs() @ b.double().abs().transpose(1, 2), K, ref)
    check_bound(f"gemm_f32 {'mn' if mn_major else 'k'} M{M} N{N} K{K} b{batch}", c, ref, bound)


@pytest.mark.parametrize("M,N,K,batch", [(128, 64, 64, 1), (128, 128, 64, 1), (128, 256, 64, 1), (256, 256, 256, 1),
                                         (300, 200, 136, 1), (64, 24, 32, 1), (128, 128, 128, 3), (1000, 512, 1024, 1),
                                         (260, 260, 264, 5), (4096, 2048, 256, 1)])
def test_gemm_k_major(M, N, K, batch):
    _gemm_store_f32(False, M, N, K, batch)


@pytest.mark.parametrize("M,N,K,batch", [(128, 64, 64, 1), (128, 128, 64, 2), (256, 256, 128, 4), (64, 64, 8, 3),
                                         (264, 136, 72, 2), (384, 384, 512, 3), (24, 24, 4, 5)])
def test_gemm_mn_major(M, N, K, batch):
    _gemm_store_f32(True, M, N, K, batch)


def test_gemm_epilogue_rejects_bad_arguments():
    ops = _ops()
    a = torch.randn(1, 128, 64, device="cuda").bfloat16()
    w = torch.randn(1, 64, 64, device="cuda").bfloat16()
    out = torch.zeros(128 * 64, device="cuda")
    with pytest.raises(ValueError, match="bn"):
        ops.gemm_bf16_epilogue(a, w, out, bn=96, mode=ops.EPI_STORE_F32, ld_out=64)
    a2, w2 = a.expand(2, -1, -1).contiguous(), w.expand(2, -1, -1).contiguous()
    with pytest.raises(ValueError, match="residual"):       # the residual is not batched: batch 1 only
        ops.gemm_bf16_epilogue(a2, w2, out, bn=64, mode=ops.EPI_RESID_F32, resid=out, ld_resid=64, ld_out=64)


# ------------------------------------------------------------------------------------------------------------------------
# pair bias: af2_pair_bias (tensor-core kernel for d in {128, 256}, SIMT kernel for other d % 32 == 0 <= 256 with <= 8
# heads, LayerNorm-kernel bias path otherwise)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,heads", [(128, 1), (128, 3), (128, 8), (256, 1), (256, 3), (256, 8),      # mma kernel
                                     (32, 3), (96, 8), (224, 1), (224, 5),                            # SIMT kernel
                                     (128, 12), (136, 4)])                                            # LayerNorm kernel
@pytest.mark.parametrize("rows,n", [(7, 37), (33, 257)])
def test_pair_bias(d, heads, rows, n):
    from alphafold2_b200 import _lib, ops
    g = torch.Generator().manual_seed(d * heads + n)
    x = (torch.randn(rows, n, d, generator=g) * 2 + 0.5).cuda()
    w = torch.randn(heads, d, generator=g).cuda()
    npad = (n + 7) // 8 * 8
    guard = 64
    out = torch.zeros(heads * rows * npad + guard, dtype=torch.bfloat16, device="cuda")
    out[-guard:] = float("nan")                            # the caller zero-fills [H][rows][npad]; nothing past it is touched
    _lib.check(_lib.load().af2_pair_bias(x.data_ptr(), w.data_ptr(), out.data_ptr(), rows, n, d, heads, ops._stream_ptr()))
    torch.cuda.synchronize()
    o = out[:-guard].view(heads, rows, npad)
    x64, w64 = x.double(), w.double()
    ref = torch.einsum("rjk,hk->hrj", x64, w64)
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -14 * torch.einsum("rjk,hk->hrj", x64.abs(), w64.abs())
    check_bound(f"pair_bias d{d} h{heads} rows{rows} n{n}", o[:, :, :n], ref, bound)
    assert (o[:, :, n:].float() == 0).all(), "pad columns must keep the caller's zeros"
    assert torch.isnan(out[-guard:].float()).all(), "write past the bias buffer"


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,d", [(1000, 256), (77, 64), (513, 128), (40, 32), (9, 512)])
def test_layernorm(T, d):
    ops = _ops()
    torch.manual_seed(T)
    x = torch.randn(T, d, device="cuda") * 3 + 1.5
    g = torch.randn(d, device="cuda")
    b = torch.randn(d, device="cuda")
    y = ops.layernorm_bf16(x, g, b)
    ref = torch.nn.functional.layer_norm(x.double(), (d,), g.double(), b.double(), 1e-5)
    err = (y.double() - ref).abs()
    assert (err <= 2 ** -8 * ref.abs() + 1e-5).all(), f"max err {err.max().item()}"   # one bf16 rounding


def test_rotary_bit_exact():
    from alphafold2_b200 import apply_rotary_pos_emb
    fx = load_golden("rotary")
    i = fx["inputs"]
    y = apply_rotary_pos_emb(i["x"].cuda(), (i["sin"].cuda(), i["cos"].cuda()))
    assert torch.equal(y.cpu(), fx["out_fp32"])                # integer/elementwise work: bit exact
    big = torch.randn(2, 8, 300, 64, device="cuda")
    from oracle.evoformer_oracle import apply_rotary_pos_emb as o_rot, fixed_positional_embedding
    s, c = fixed_positional_embedding(64, 300)
    assert torch.equal(apply_rotary_pos_emb(big, (s.cuda(), c.cuda())).cpu(), o_rot(big.cpu(), s, c))
