"""-m gpu: the structure module kernel by kernel against fp64 (bounds and their derivation: structure_bounds.py; CPU controls of
those bounds: test_structure_bounds_controls.py).

  * invariant point attention at one (heads, dim) per shared-memory tier of the tile rule (4, 2 or 1 CTAs per SM, 32 .. 1 key
    rows per tile), at n = 1, TJ - 1, TJ, TJ + 1 and k TJ + 1 (k >= 10), with no mask, padding that ends inside a tile, a fully
    masked first tile of keys, scattered fully masked query rows, translations at 5 and 500, and point weights at +25 and -30;
  * the tile rule itself against its restatement, the device's shared memory and the cases above;
  * the fp32 linear at ragged M, N, K with the bias and the ReLU on and off, and at 2^21 + 1 rows;
  * the frame and tail kernels at dims that are not multiples of 32, quaternions of norm 1e-2 .. 1e2 and real part near 0, and
    translations up to 500;
  * the refusals of shapes the grids cannot hold (batch > 65535, more than 65535 column tiles), before any launch.

The layer and the stack compose LayerNorms, where bounds are not worth deriving; they are gated by an fp32 yardstick instead:
the oracle (oracle/structure_oracle.py) in fp32 on the GPU with TF32 off.  Against the fp64 oracle the kernels' max error must
be <= YARD_F x the yardstick's max error + YARD_FLOOR x rms(ref).  Measured on an H100 80GB HBM3 (700 W power limit), the
kernels' max error over the yardstick's: one layer 4.59 (rot at (1, 65, 1024, 16)), 4.52 (its single), 3.89 (single at (1, 257,
384, 12)), <= 3.5 elsewhere; the 8-layer stacks <= 1.73 (strict and bf16); IPABlock.forward 1.51; depth
0 1.60.  The ratio grows with the layer's widest contraction: the fp32 linear sums K terms in one fmaf chain (to_out: K = H (32 +
d) = 16 896 at (16, 1024)), within its own bound K u sum|x w| (test_structure_linear_vs_fp64), where cuBLAS's fp32 GEMM sums
in blocks.  YARD_F = 8 leaves 1.7x margin over the worst.
"""
from contextlib import contextmanager

import pytest
import torch

import alphafold2_b200 as A
from alphafold2_b200 import _lib, ops
from oracle import structure_oracle as SO
from oracle.evoformer_oracle import _lin
import structure_bounds as S
from gpu_util import check_bound
from test_structure_bounds_controls import _tail_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
YARD_F = 8.0
YARD_FLOOR = 1e-6


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------------
# the tile rule
# ------------------------------------------------------------------------------------------------------------------------
# one (heads, dim) per tier (CTAs per SM, TJ): the AlphaFold-like (12, 384) and the largest shape (16, 1024) among them
TIERS = {
    (4, 32): (1, 32), (4, 16): (2, 168), (4, 8): (4, 100),
    (2, 16): (5, 288), (2, 8): (7, 432), (2, 4): (12, 384), (2, 2): (16, 616), (2, 1): (16, 736),
    (1, 8): (15, 800), (1, 4): (16, 1024),
}
EXTRA_TJ4 = [(16, 256), (4, 1024)]                      # two more shapes of the (2, 4) tier


def test_tile_rule_matches_restatement():
    opt = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    for H in range(1, 17):
        for d in range(4, 1025, 4):
            ctas, tj, nbytes = S.ipa_tile_rule(H, d)
            assert ops.ipa_tile_rows(H, d) == (tj, nbytes), (H, d)
            assert 0 < nbytes <= opt, (H, d, nbytes, opt)
    for H, d in ((0, 32), (17, 32), (4, 30), (4, 1028), (4, 0)):
        assert ops.ipa_tile_rows(H, d) == (0, 0)
    for tier, (H, d) in TIERS.items():
        assert S.ipa_tile_rule(H, d)[:2] == tier, (H, d)
    for H, d in EXTRA_TJ4:
        assert S.ipa_tile_rule(H, d)[:2] == (2, 4)


# ------------------------------------------------------------------------------------------------------------------------
# invariant point attention
# ------------------------------------------------------------------------------------------------------------------------
def _ipa_inputs(B, n, H, d, TJ, masked, scale, seed):
    """fp32 kernel inputs on the GPU.  Point weights per head cycle through +25 (softplus' x > 20 branch, peaked logits), -30
    (point term ~1e-13) and N(0, 1).  masked: batch 0 has its whole first tile of keys masked and every fourth residue after
    it (fully masked query rows), batch 1 padding that ends inside a tile."""
    g = _gen(seed)
    proj = torch.randn(B, n, 84 * H, device=DEV, generator=g)
    rot = SO.quaternion_to_matrix(torch.randn(B, n, 4, device=DEV, generator=g, dtype=torch.float64)).float().contiguous()
    trans = torch.randn(B, n, 3, device=DEV, generator=g) * scale
    ops.ipa_frames_(proj, rot, trans, H)                                     # points global: the kernel's own input
    pair = torch.randn(B, n, n, d, device=DEV, generator=g)
    w_bias = torch.randn(H, d, device=DEV, generator=g) * d ** -0.5
    b_bias = torch.randn(H, device=DEV, generator=g)
    pw = torch.randn(H, device=DEV, generator=g)
    pw[0::3] = 25.0
    pw[1::3] = -30.0
    mask = None
    if masked:
        mask = torch.ones(B, n, dtype=torch.bool, device=DEV)
        mask[0, :TJ] = False
        mask[0, TJ + 2::4] = False
        if B > 1:
            mask[1, S.mid_tile_length(n, TJ):] = False
    return proj, pair, w_bias, b_bias, pw, mask, rot, trans


def _ns(TJ):
    big = TJ * max(10, -(-200 // TJ)) + 1
    return sorted({max(1, TJ - 1), TJ, TJ + 1, big})


IPA_CASES = [(tier, H, d, n) for tier, (H, d) in TIERS.items() for n in sorted({1, *_ns(tier[1])})] + \
            [((2, 4), H, d, n) for H, d in EXTRA_TJ4 for n in (3, 41)]


@pytest.mark.parametrize("B,masked,scale", [(1, False, 500.0), (2, True, 5.0), (2, True, 500.0)])
@pytest.mark.parametrize("tier,H,d,n", IPA_CASES)
def test_ipa_attention_vs_fp64(tier, H, d, n, B, masked, scale):
    ctas, TJ = tier
    assert ops.ipa_tile_rows(H, d)[0] == TJ                                  # the case is in the tier it claims
    args = _ipa_inputs(B, n, H, d, TJ, masked, scale, seed=H * 100003 + d * 101 + n * 7 + B + int(scale))
    out = ops.ipa_attention(*args, H)
    ref, bound = S.ipa_attention_ref(*args, H, TJ)
    check_bound(f"structure/ipa/{ctas}cta_tj{TJ}/H{H}_d{d}/n{n}_B{B}_{'mask' if masked else 'nomask'}_t{int(scale)}",
                out, ref, bound)


def test_ipa_rows_window_bitwise_one_cta():
    """ipa_attention_rows on an uneven window of query rows is bitwise those rows of ipa_attention (1-CTA tier)"""
    H, d = TIERS[(1, 8)]
    n, row0, R = 45, 7, 19
    proj, pair, w_bias, b_bias, pw, mask, rot, trans = _ipa_inputs(2, n, H, d, 8, True, 500.0, seed=3)
    proj, pair, mask, rot, trans = proj[:1].contiguous(), pair[:1].contiguous(), mask[:1], rot[:1].contiguous(), trans[:1].contiguous()
    whole = ops.ipa_attention(proj, pair, w_bias, b_bias, pw, mask, rot, trans, H)
    rows = ops.ipa_attention_rows(proj, pair[:, row0:row0 + R].contiguous(), w_bias, b_bias, pw, mask, rot, trans, H, row0)
    assert torch.equal(rows.view(torch.int32), whole[:, row0:row0 + R].view(torch.int32))


def test_ipa_batch_limit_refused():
    """batch is the grid's y dimension: 65536 is refused with ValueError, by the Python check and by the C entry, unlaunched"""
    B, n, H, d = 65536, 1, 1, 4
    assert not ops.ipa_shape_ok(B, n, H, d) and ops.ipa_shape_ok(B - 1, n, H, d)
    proj = torch.zeros(B, n, 84 * H, device=DEV)
    pair = torch.zeros(B, n, n, d, device=DEV)
    rot = torch.eye(3, device=DEV).repeat(B, n, 1, 1)
    trans = torch.zeros(B, n, 3, device=DEV)
    w = torch.zeros(H, d, device=DEV)
    z = torch.zeros(H, device=DEV)
    with pytest.raises(ValueError):
        ops.ipa_attention(proj, pair, w, z, z, None, rot, trans, H)
    out = torch.empty(B, n, H * (32 + d), device=DEV)
    before = _lib.load().af2_launch_count()
    with pytest.raises(ValueError, match="batch"):
        _lib.check(_lib.load().af2_ipa_attention(proj.data_ptr(), pair.data_ptr(), w.data_ptr(), z.data_ptr(), z.data_ptr(), None,
                                                 rot.data_ptr(), trans.data_ptr(), out.data_ptr(), B, n, H, d, None))
    assert _lib.load().af2_launch_count() == before


# ------------------------------------------------------------------------------------------------------------------------
# fp32 linear
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 15, 17, 12 * 416])
@pytest.mark.parametrize("N", [1, 3, 6, 33, 84 * 12])
@pytest.mark.parametrize("M", [1, 31, 33, 4097])
def test_structure_linear_vs_fp64(M, N, K):
    g = _gen(M * 31 + N * 7 + K)
    x = torch.randn(M, K, device=DEV, generator=g)
    w = torch.randn(N, K, device=DEV, generator=g) * K ** -0.5
    b = torch.randn(N, device=DEV, generator=g)
    for bias, relu in ((None, False), (b, False), (b, True), (None, True)):
        out = ops.structure_linear(x, w, bias, relu=relu)
        ref, bound = S.linear_ref(x, w, bias, relu)
        check_bound(f"structure/linear/M{M}_N{N}_K{K}_{'bias' if bias is not None else 'nobias'}_{'relu' if relu else 'id'}",
                    out, ref, bound)


def test_structure_linear_rows_beyond_grid_y():
    """2^21 + 1 rows: more row tiles than a grid's y dimension holds"""
    M, N, K = 2 ** 21 + 1, 3, 4
    g = _gen(21)
    x = torch.randn(M, K, device=DEV, generator=g)
    w, b = torch.randn(N, K, device=DEV, generator=g), torch.randn(N, device=DEV, generator=g)
    out = ops.structure_linear(x, w, b, relu=True)
    ref, bound = S.linear_ref(x, w, b, True)
    check_bound("structure/linear/M2097153_N3_K4_bias_relu", out, ref, bound)


def test_structure_linear_columns_beyond_grid_y_refused():
    N = 65535 * 32 + 1
    x = torch.zeros(1, 1, device=DEV)
    w = torch.zeros(N, 1, device=DEV)
    before = _lib.load().af2_launch_count()
    with pytest.raises(ValueError):
        ops.structure_linear(x, w)
    assert _lib.load().af2_launch_count() == before


# ------------------------------------------------------------------------------------------------------------------------
# frames and tail
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [5.0, 500.0])
@pytest.mark.parametrize("H", [1, 5, 16])
def test_ipa_frames_vs_fp64(H, scale):
    g = _gen(H * 10 + int(scale))
    rows = 203
    proj = torch.randn(rows, 84 * H, device=DEV, generator=g)
    rot = SO.quaternion_to_matrix(torch.randn(rows, 4, device=DEV, generator=g, dtype=torch.float64)).float().contiguous()
    trans = torch.randn(rows, 3, device=DEV, generator=g) * scale
    ref, bound = S.frames_ref(proj, rot, trans, H)
    out = ops.ipa_frames_(proj.clone(), rot, trans, H)
    check_bound(f"structure/frames/H{H}_t{int(scale)}", out, ref, bound)


@pytest.mark.parametrize("part", ["single", "frames", "coords"])
@pytest.mark.parametrize("d", [4, 36, 260, 1024])
def test_structure_tail_vs_fp64(d, part):
    rows = 203
    kw = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in _tail_inputs(rows, d, torch.Generator().manual_seed(d), 500.0).items()}
    if part != "coords":
        kw.update(w_points=None, b_points=None, w_lddt=None, b_lddt=None)
    if part == "single":
        kw.update(w_qu=None, b_qu=None, quat=None, trans=None, rot=None)
    ref = S.tail_ref(**kw)
    got = {k: (v.clone() if torch.is_tensor(v) and k in ("s", "quat", "trans", "rot") else v) for k, v in kw.items()}
    coords = torch.empty(rows, 3, device=DEV) if part == "coords" else None
    conf = torch.empty(rows, 1, device=DEV) if part == "coords" else None
    ops.structure_tail_(got["s"], got["o"], got["gamma"], got["beta"], got["eps"], got["w_qu"], got["b_qu"], got["quat"], got["trans"],
                        got["rot"], got["w_points"], got["b_points"], got["w_lddt"], got["b_lddt"], coords, conf)
    outs = {"single": got["s"]}
    if part != "single":
        outs.update(quat=got["quat"], trans=got["trans"], rot=got["rot"].reshape(rows, 9))
    if part == "coords":
        outs.update(coords=coords, confidence=conf)
    for name, out in outs.items():
        r, bound = ref[name]
        if name == "quat":
            r = S.align_quat_sign(out, r, ref["quat_ambiguous"])
        check_bound(f"structure/tail/d{d}_{part}/{name}", out, r, bound)


# ------------------------------------------------------------------------------------------------------------------------
# layer, block and stack against the fp32 yardstick
# ------------------------------------------------------------------------------------------------------------------------
@contextmanager
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def yard_check(name, out, ref64, yard):
    """max |out - ref| <= YARD_F max |yard - ref| + YARD_FLOOR rms(ref), through check_bound (a uniform bound); prints the
    measured ratio of the two max errors"""
    ref64 = ref64.double()
    y_err = (yard.double() - ref64).abs().max().item()
    k_err = (out.double() - ref64).abs().max().item()
    rms = ref64.pow(2).mean().sqrt().item()
    print(f"yardstick {name}: kernel max err {k_err:.3e}, fp32 oracle {y_err:.3e}, ratio {k_err / max(y_err, 1e-300):.3f}")
    check_bound(f"{name}/yardstick", out, ref64, torch.full_like(ref64, YARD_F * y_err + YARD_FLOOR * rms))


def _block_state(d, H, g):
    """random weights of one IPABlock (the package's names), to_out non-zero, LayerNorms off identity"""
    sd = {}
    for k, v in SO.IPABlock(dim=d, heads=H).state_dict().items():
        if k.endswith("norm.weight"):
            sd[k] = 1 + 0.2 * torch.randn(v.shape, generator=g)
        elif v.dim() == 1:
            sd[k] = 0.2 * torch.randn(v.shape, generator=g)
        else:
            sd[k] = torch.randn(v.shape, generator=g) * v.shape[-1] ** -0.5
    sd["attn.point_weights"] = torch.randn(H, generator=g)
    return sd


def _frames(b, n, g, t_scale):
    q = torch.randn(b, n, 4, generator=g, dtype=torch.float64)
    q = torch.where(q[..., :1] < 0, -q, q).float()
    R = SO.quaternion_to_matrix(q.double()).float()
    t = torch.randn(b, n, 3, generator=g) * t_scale
    return q, R, t


def _pad_mask(b, n):
    mask = torch.ones(b, n, dtype=torch.bool)
    mask[0, n - max(1, n // 5):] = False
    return mask


def _oracle_layer(w, s, pair, q, R, t, H, mask):
    s = SO.ipa_block(w, "ipa_block.", s, pair, R, t, H, mask)
    u, v = _lin(w, "to_quaternion_update", s).chunk(2, dim=-1)
    q2 = SO.quaternion_multiply(q, torch.nn.functional.pad(u, (1, 0), value=1.0))
    t2 = t + torch.einsum("bnc,bncr->bnr", v, R)
    R2 = SO.quaternion_to_matrix(q2)
    coords = torch.einsum("bnc,bncd->bnd", _lin(w, "to_points", s), R2) + t2
    return dict(single=s, quat=q2, trans=t2, rot=R2, coords=coords, confidence=_lin(w, "lddt_linear", s))


@pytest.mark.parametrize("b,n,d,H", [(2, 37, 36, 3), (1, 257, 384, 12), (1, 65, 1024, 16)])
def test_structure_layer_vs_yardstick(b, n, d, H):
    g = torch.Generator().manual_seed(n + d)
    blk = A.IPABlock(dim=d, heads=H)
    sd = _block_state(d, H, g)
    blk.load_state_dict(sd)
    qu, pts, lddt = torch.nn.Linear(d, 6), torch.nn.Linear(d, 3), torch.nn.Linear(d, 1)
    blk, qu, pts, lddt = (m.to(DEV) for m in (blk, qu, pts, lddt))
    pk = ops.pack_structure(blk, qu, pts, lddt)
    s = torch.randn(b, n, d, generator=g)
    pair = torch.randn(b, n, n, d, generator=g)
    q, R, t = _frames(b, n, g, 20.0)
    mask = _pad_mask(b, n)
    w = {"ipa_block." + k: v for k, v in sd.items()}
    for name, lin in (("to_quaternion_update", qu), ("to_points", pts), ("lddt_linear", lddt)):
        w[name + ".weight"], w[name + ".bias"] = lin.weight.detach().cpu(), lin.bias.detach().cpu()

    single, quat, trans, rot = (v.to(DEV).contiguous() for v in (s, q, t, R))
    coords, conf = torch.empty(b, n, 3, device=DEV), torch.empty(b, n, 1, device=DEV)
    ops.structure_layer_(pk, single, pair.to(DEV), mask.to(DEV), quat, trans, rot, coords, conf)
    got = dict(single=single, quat=quat, trans=trans, rot=rot, coords=coords, confidence=conf)

    def run(dtype):
        with _no_tf32():
            wd = {k: v.to(DEV, dtype) for k, v in w.items()}
            return _oracle_layer(wd, *(v.to(DEV, dtype) for v in (s, pair, q, R, t)), H, mask.to(DEV))
    ref = run(torch.float64)
    yard = run(torch.float32)
    for k in got:
        yard_check(f"structure/layer/b{b}_n{n}_d{d}_H{H}/{k}", got[k], ref[k], yard[k])


@pytest.mark.parametrize("precision", ["strict", "bf16"])
@pytest.mark.parametrize("b,n,d,H", [(1, 256, 256, 8), (2, 96, 128, 12)])
def test_structure_stack_vs_yardstick(b, n, d, H, precision):
    """eight layers through Alphafold2._structure_module (the forward's structure module on the trunk's x and m) against the
    oracle's structure_module fed the same x and m_0; bf16 mode: the reference's trunk_to_pairwise_repr_dim takes bf16-rounded x
    and W, as the kernel's GEMM operands are"""
    g = torch.Generator().manual_seed(n * 3 + d + H)
    torch.manual_seed(n + d)
    model = A.attach_structure_module(A.Alphafold2(dim=d, depth=1, heads=2, dim_head=16, predict_coords=True,
                                                   structure_module_depth=8, structure_module_heads=H))
    sd = model.state_dict()
    for k, v in _block_state(d, H, g).items():
        sd["ipa_block." + k] = v
    model.load_state_dict(sd)
    model = A.set_precision(model.to(DEV).eval(), precision)
    x = torch.randn(b, n, n, d, generator=g)
    m = torch.randn(b, 1, n, d, generator=g)
    mask = _pad_mask(b, n)
    ret = A.ReturnValues()
    with torch.no_grad():
        coords, conf = model._structure_module(x.to(DEV), m.to(DEV), mask.to(DEV), ret, x_private=False, return_confidence=True,
                                               return_recyclables=True, return_aux_logits=False)
    got = dict(coords=coords, confidence=conf, pair=ret.recyclables.pairwise_repr)
    w = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    x_in = x
    if precision == "bf16":
        x_in = x.bfloat16().float()
        w["trunk_to_pairwise_repr_dim.weight"] = w["trunk_to_pairwise_repr_dim.weight"].bfloat16().float()

    def run(dtype):
        with _no_tf32():
            wd = {k: (v.to(DEV, dtype) if torch.is_floating_point(v) else v.to(DEV)) for k, v in w.items()}
            c, single, pair = SO.structure_module(wd, x_in.to(DEV, dtype), m[:, 0].to(DEV, dtype), H, 8, mask.to(DEV))
            return dict(coords=c, confidence=_lin(wd, "lddt_linear", single), pair=pair)
    ref = run(torch.float64)
    yard = run(torch.float32)
    for k in got:
        yard_check(f"structure/stack8_{precision}/b{b}_n{n}_d{d}_H{H}/{k}", got[k], ref[k], yard[k])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ipa_block_forward_vs_yardstick(dtype):
    """IPABlock.forward (the package's call, one kernel at a time) against the oracle's ipa_block; x is left unchanged and a bf16
    x comes back bf16, the fp32 path's output rounded"""
    b, n, d, H = 2, 53, 64, 6
    g = torch.Generator().manual_seed(53)
    sd = _block_state(d, H, g)
    blk = A.IPABlock(dim=d, heads=H)
    blk.load_state_dict(sd)
    blk = blk.to(DEV).eval()
    x = torch.randn(b, n, d, generator=g).to(DEV, dtype)
    pair = torch.randn(b, n, n, d, generator=g)
    _, R, t = _frames(b, n, g, 20.0)
    mask = _pad_mask(b, n).to(DEV)
    x0 = x.clone()
    out = blk(x, pairwise_repr=pair.to(DEV), rotations=R.to(DEV), translations=t.to(DEV), mask=mask)
    assert torch.equal(x, x0), "the caller's x was written"
    assert out.dtype == dtype and out.shape == x.shape
    if dtype == torch.bfloat16:
        out32 = blk(x.float(), pairwise_repr=pair.to(DEV), rotations=R.to(DEV), translations=t.to(DEV), mask=mask)
        assert torch.equal(out, out32.bfloat16())
        return

    def run(dt):
        with _no_tf32():
            wd = {k: v.to(DEV, dt) for k, v in sd.items()}
            return SO.ipa_block(wd, "", x.to(dt), pair.to(DEV, dt), R.to(DEV, dt), t.to(DEV, dt), H, mask)
    yard_check("structure/ipa_block_forward/b2_n53_d64_H6", out, run(torch.float64), run(torch.float32))


def test_structure_depth_zero_vs_yardstick():
    """structure_module_depth = 0: coords = to_points(single) with q = (1, 0, 0, 0), t = 0, and the confidence of single"""
    b, n, d, H = 2, 40, 64, 4
    g = torch.Generator().manual_seed(40)
    torch.manual_seed(40)
    model = A.attach_structure_module(A.Alphafold2(dim=d, depth=1, heads=2, dim_head=16, predict_coords=True,
                                                   structure_module_depth=0, structure_module_heads=H)).to(DEV).eval()
    x, m = torch.randn(b, n, n, d, generator=g), torch.randn(b, 1, n, d, generator=g)
    mask = _pad_mask(b, n)
    with torch.no_grad():
        coords, conf = model._structure_module(x.to(DEV), m.to(DEV), mask.to(DEV), A.ReturnValues(), x_private=False,
                                               return_confidence=True, return_recyclables=False, return_aux_logits=False)
    w = {k: v.detach() for k, v in model.state_dict().items()}

    def run(dt):
        with _no_tf32():
            wd = {k: (v.to(dt) if torch.is_floating_point(v) else v) for k, v in w.items()}
            c, single, _ = SO.structure_module(wd, x.to(DEV, dt), m[:, 0].to(DEV, dt), H, 0, mask.to(DEV))
            return dict(coords=c, confidence=_lin(wd, "lddt_linear", single))
    ref, yard = run(torch.float64), run(torch.float32)
    for k, out in (("coords", coords), ("confidence", conf)):
        yard_check(f"structure/depth0/{k}", out, ref[k], yard[k])
