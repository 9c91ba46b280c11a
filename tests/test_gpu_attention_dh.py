"""-m gpu: the tensor-core attention kernel at head widths 16 and 128 (attention_tc_kernel<16> / <128>), alone and through
every layer that reaches it.

  * the kernel alone against the fp64 reference of test_gpu_attention_kernel.py (same inputs, mask kinds and per-element
    bound, C_ATTN included): every 128-key block boundary, 1 / 2 / 4 / 16 heads, row and column folding, with and without
    bias (NaN in the bias pad columns), large logits, every mask kind, fewer work items than SMs and many times more;
  * one call at n = 16,384 keys per width (the DH 128 shared-memory layout keeps two 128-key stages in flight there);
  * two identical launches give identical bits, and a folded row run alone has the bits it has inside a larger launch;
  * AxialAttention (row, column, with edges, with tied queries) and EvoformerBlock against the fp64 oracle with the gates of
    gpu_util.py, including the autocast yardstick; the reference fixtures of oracle/make_golden_r6.py;
  * Alphafold2.forward at dim_head 128 with templates, recyclables and predict_angles against the oracle;
  * forced pair bands of 8 and 16 rows and forced MSA bands give the whole-tensor bits;
  * dim_head 8, 24, 48, 96 and 256 are refused with a ValueError that names the supported widths.
"""
import functools

import pytest
import torch

from conftest import load_golden
from gpu_util import autocast_yardstick, check, dev, to64
from oracle import evoformer_oracle as O
from oracle import recycling_oracle as RO
from oracle.make_golden_r6 import fixture_state
from test_gpu_attention_kernel import MASK_KINDS, _tok, make_inputs, run_case
from test_gpu_modules import _rand_state

pytestmark = pytest.mark.gpu

WIDTHS = [16, 128]
N_ALL = [1, 5, 127, 128, 129, 255, 300, 384, 1000]
HEADS = [1, 2, 4, 16]


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


# ------------------------------------------------ the kernel alone ------------------------------------------------
@pytest.mark.parametrize("dh", WIDTHS)
@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("n", N_ALL)
def test_attention_dh_lengths(n, bias, row, dh):
    k = N_ALL.index(n)
    heads = HEADS[(k + bias + 2 * row) % len(HEADS)]
    nbatch = [1, 3, 7][(k + row) % 3] if n < 384 else 2
    mask = ["none", "holes", "suffix"][(k + row + bias) % 3]
    run_case(f"attn_dh len n{n} b{nbatch} h{heads} dh{dh} {'row' if row else 'col'} bias{int(bias)} {mask}",
             n, nbatch, heads, dh, row, bias, mask, seed=n * 7 + dh + bias)


@pytest.mark.parametrize("dh", WIDTHS)
@pytest.mark.parametrize("mask", MASK_KINDS)
@pytest.mark.parametrize("n,nbatch,heads,row", [(257, 3, 4, True), (384, 5, 2, False), (200, 37, 1, False), (130, 2, 16, True)])
def test_attention_dh_masks(n, nbatch, heads, row, mask, dh):
    run_case(f"attn_dh mask {mask} n{n} b{nbatch} h{heads} dh{dh} {'row' if row else 'col'}", n, nbatch, heads, dh, row,
             True, mask, seed=11 * n + dh)


@pytest.mark.parametrize("dh", WIDTHS)
@pytest.mark.parametrize("mask", ["none", "holes", "first_block", "all_masked"])
@pytest.mark.parametrize("n", [129, 300])
def test_attention_dh_large_logits(n, mask, dh):
    """q and the bias scaled so that the logits span about +-200 (log2 domain)"""
    run_case(f"attn_dh big {mask} n{n} dh{dh}", n, 3, 4, dh, True, True, mask, big=True, seed=5 * n + dh)


@pytest.mark.parametrize("dh", WIDTHS)
@pytest.mark.parametrize("n,nbatch,heads,row", [(129, 1, 1, True),       # 2 work items on a 132-SM card
                                                (256, 150, 16, False),   # 4800 items: ~36 per CTA
                                                (1000, 40, 4, True)])    # 1280 items of 8 key blocks
def test_attention_dh_item_counts(n, nbatch, heads, row, dh):
    run_case(f"attn_dh items n{n} b{nbatch} h{heads} dh{dh}", n, nbatch, heads, dh, row, True, "holes", seed=n + nbatch + dh)


@pytest.mark.parametrize("dh", WIDTHS)
def test_attention_dh_long_sequence(dh):
    """n = 16,384 keys, the MSA column attention at the deepest MSA the README reports: every query row checked"""
    run_case(f"attn_dh long n16384 dh{dh}", 16384, 1, 1, dh, True, True, "holes", seed=dh)


@pytest.mark.parametrize("dh", WIDTHS)
@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
def test_attention_dh_repeat_and_slice_bitwise(row, dh):
    from alphafold2_b200 import ops
    n, nbatch, heads = 257, 37, 4
    qkv, gate, bt, mask, out = run_case(f"attn_dh slice n{n} b{nbatch} dh{dh} {'row' if row else 'col'}", n, nbatch, heads,
                                        dh, row, True, "holes", seed=3 + dh)
    idx, tok_sb, tok_si = _tok(nbatch, n, row)
    again = ops.attention_bf16(qkv, gate, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask)
    assert torch.equal(_bits(again), _bits(out)), "two identical launches differ"
    for b in (0, 17, 36):
        ix = idx[b]
        one = ops.attention_bf16(qkv[ix].contiguous(), gate[ix].contiguous(), n, 1, heads, dh, n, 1, bias=bt,
                                 mask=mask[ix].contiguous())
        assert torch.equal(_bits(one), _bits(out[ix])), f"folded row {b} differs when run alone"


# ------------------------------------------------ modules vs the fp64 oracle ------------------------------------------------
# inner width I = heads * dim_head of 256 or 512, as the gates of gpu_util.py were set on (C2: 8 x 64)
@pytest.mark.parametrize("d,H,dh,N,row,tied", [(256, 32, 16, 72, True, False), (256, 16, 16, 70, False, False),
                                               (256, 4, 128, 72, True, False), (256, 4, 128, 136, False, False),
                                               (256, 32, 16, 64, False, True), (256, 4, 128, 40, False, True)])
def test_axial_attention_dh_oracle(d, H, dh, N, row, tied):
    import alphafold2_b200 as A
    ax = A.AxialAttention(dim=d, heads=H, dim_head=dh, row_attn=row, col_attn=not row, accept_edges=True,
                          global_query_attn=tied)
    st = _rand_state(ax, 3 + dh)
    ax = ax.cuda().eval()
    x = torch.randn(1, N, N, d, generator=torch.Generator().manual_seed(4))
    m1 = torch.ones(1, N, dtype=torch.bool)
    m1[:, -5:] = False
    mask = m1[:, :, None] & m1[:, None, :]
    xc, mc = x.cuda(), mask.cuda()
    out = ax(xc, edges=xc, mask=mc)
    with torch.no_grad():
        ref = O.axial_attention(to64(st), "", x.double(), H, row, edges=x.double(), mask=mask, global_query_attn=tied)
        ac = autocast_yardstick(lambda: O.axial_attention(dev(st), "", xc, H, row, edges=xc, mask=mc,
                                                          global_query_attn=tied)).float().cpu()
    check(f"axial_attention_dh/oracle/d{d}H{H}x{dh}N{N}{'row' if row else 'col'}{'_tied' if tied else ''}", out, ref, ac)


@pytest.mark.parametrize("d,H,dh,N,S", [(256, 16, 16, 72, 12), (256, 4, 128, 72, 12)])
def test_evoformer_block_dh_oracle(d, H, dh, N, S):
    import alphafold2_b200 as A
    blk = A.EvoformerBlock(dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
    st = _rand_state(blk, 5)
    blk = blk.cuda().eval()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, N, N, d, generator=g)
    m = torch.randn(1, S, N, d, generator=g)
    mask1 = torch.ones(1, N, dtype=torch.bool)
    mask1[:, -N // 8:] = False
    mask = mask1[:, :, None] & mask1[:, None, :]
    msa_mask = torch.rand(1, S, N, generator=g) > 0.1
    msa_mask[:, :, -N // 8:] = False
    msa_mask[:, 0, : N - N // 8] = True
    cu = [t.cuda() for t in (x, m, mask, msa_mask)]
    xo, mo, _, _ = blk(tuple(cu))
    with torch.no_grad():
        rx, rm = O.evoformer_block(to64(st), "", x.double(), m.double(), H, mask, msa_mask, chunk=16)
        ax_, am_ = autocast_yardstick(lambda: O.evoformer_block(dev(st), "", cu[0], cu[1], H, cu[2], cu[3], chunk=16))
    check(f"evoformer_block_dh/oracle/d{d}H{H}x{dh}N{N}S{S}/x", xo, rx, ax_.float().cpu())
    check(f"evoformer_block_dh/oracle/d{d}H{H}x{dh}N{N}S{S}/m", mo, rm, am_.float().cpu())


@pytest.mark.parametrize("name", ["evoformer_dh16", "evoformer_dh128"])
def test_evoformer_block_dh_golden(name):
    import alphafold2_b200 as A
    fx = load_golden(name)
    c, i = fx["cfg"], fx["inputs"]
    blk = A.EvoformerBlock(dim=c["dim"], seq_len=c["N"], heads=c["heads"], dim_head=c["dim_head"], attn_dropout=0., ff_dropout=0.)
    blk.load_state_dict(fixture_state(fx))
    blk = blk.cuda().eval()
    x, m, _, _ = blk((i["x"].float().cuda(), i["m"].float().cuda(), i["mask"].cuda(), i["msa_mask"].cuda()))
    check(f"{name}/golden/x", x, fx["out_fp64"][0], fx["out_autocast_bf16"][0])
    check(f"{name}/golden/m", m, fx["out_fp64"][1], fx["out_autocast_bf16"][1])


def test_alphafold2_dh128_golden():
    import alphafold2_b200 as A
    fx = load_golden("alphafold2_dh128")
    i = {k: v.cuda() for k, v in fx["inputs"].items()}
    model = A.Alphafold2(**fx["cfg"])
    missing = model.load_state_dict(fixture_state(fx), strict=False)
    assert not missing.unexpected_keys
    model = model.cuda().eval()
    ret = model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"], templates_feats=i["templates_feats"].float(),
                templates_angles=i["templates_angles"].float(), templates_mask=i["templates_mask"])
    check("alphafold2_dh128/golden/distance", ret.distance, fx["out_fp64"], fx["out_autocast_bf16"])


def test_alphafold2_dh128_templates_recyclables_angles_oracle():
    import alphafold2_b200 as A
    torch.manual_seed(51)
    b, n, S, T, d, H = 1, 40, 6, 2, 64, 2
    cfg = dict(dim=d, depth=1, heads=H, dim_head=128, templates_embed_layers=1)
    model = A.Alphafold2(**cfg, predict_angles=True)
    st = O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(52)
    for k in ("recycling_msa_norm", "recycling_pairwise_norm"):
        st[k + ".weight"] = 1.0 + 0.3 * torch.randn(d, generator=g)
        st[k + ".bias"] = 0.3 * torch.randn(d, generator=g)
    model.load_state_dict(st)
    model = model.cuda().eval()
    seq, msa = torch.randint(0, 21, (b, n), generator=g), torch.randint(0, 21, (b, S, n), generator=g)
    mask = torch.ones(b, n, dtype=torch.bool)
    mask[:, -4:] = False
    msa_mask = torch.rand(b, S, n, generator=g) > 0.1
    tm = torch.rand(b, T, n, generator=g) > 0.15
    feats, angles = torch.randn(b, T, n, n, 32, generator=g), torch.randn(b, T, n, 55, generator=g)
    coords = torch.randn(b, n, 3, generator=g) * 10.0
    rec = A.Recyclables(coords.cuda(), torch.randn(b, n, d, generator=g).cuda(), torch.randn(b, n, n, d, generator=g).cuda())
    cu = [t.cuda() for t in (seq, msa, mask, msa_mask)]
    tk = dict(templates_feats=feats.cuda(), templates_angles=angles.cuda(), templates_mask=tm.cuda())
    ret = model(*cu[:2], mask=cu[2], msa_mask=cu[3], recyclables=rec, **tk)
    torch.cuda.synchronize()
    kw = dict(recyclables=rec, templates_embed_layers=1, **tk)
    with torch.no_grad():
        ref = RO.alphafold2_distogram(dev(st, torch.float64), *cu, H, 1, dtype=torch.float64, **kw).cpu()
        ac = autocast_yardstick(lambda: RO.alphafold2_distogram(dev(st), *cu, H, 1, **kw)).float().cpu()
    check("alphafold2_dh128/templates_recyclables_angles/oracle/distance", ret.distance, ref, ac)
    for name in ("theta_logits", "phi_logits", "omega_logits"):
        t = getattr(ret, name)
        assert t is not None and t.shape[:3] == (b, n, n) and torch.isfinite(t).all(), name


# ------------------------------------------------ bands: whole-tensor bits ------------------------------------------------
@functools.lru_cache(maxsize=None)
def _evo(d, H, dh):
    import alphafold2_b200 as A
    evo = A.Evoformer(depth=1, dim=d, seq_len=64, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
    evo.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.05, seed=dh))
    return evo.cuda().eval()


def _band_inputs(N, S, d, seed):
    g = torch.Generator().manual_seed(seed)
    x, m = torch.randn(1, N, N, d, generator=g), torch.randn(1, S, N, d, generator=g)
    res = torch.rand(1, N, generator=g) > 0.1
    res[:, N - 3:] = False
    msa_mask = torch.rand(1, S, N, generator=g) > 0.2
    msa_mask[:, 0] = True
    msa_mask[:, 2] = False
    return x.cuda(), m.cuda(), (res[:, :, None] & res[:, None, :]).cuda(), msa_mask.cuda()


def _run(evo, x, m, mask, msa_mask, **kw):
    xo, mo = x.clone(), m.clone()
    evo.run_(xo, mo, mask, msa_mask, **kw)
    torch.cuda.synchronize()
    return xo, mo


@pytest.mark.parametrize("d,H,dh", [(128, 8, 16), (128, 2, 128)])
@pytest.mark.parametrize("bands", [dict(band=8), dict(band=16), dict(msa_band=2), dict(msa_band=3, band=16)],
                         ids=["pair8", "pair16", "msa2", "msa3_pair16"])
def test_dh_bands_bitwise(d, H, dh, bands):
    N, S = 44, 9
    evo = _evo(d, H, dh)
    x, m, mask, msa_mask = _band_inputs(N, S, d, seed=dh)
    rx, rm = _run(evo, x, m, mask, msa_mask)
    assert (evo.last_pair_band, evo.last_msa_band) == (N, S), "the whole-tensor reference should fit"
    bx, bm = _run(evo, x, m, mask, msa_mask, **bands)
    assert (evo.last_pair_band, evo.last_msa_band) == (bands.get("band", N), bands.get("msa_band", S))
    for name, a, r in (("x", bx, rx), ("m", bm, rm)):
        assert torch.equal(_bits(a), _bits(r)), f"{name}, {bands}: max |diff| {(a - r).abs().max().item():.3e}"


# ------------------------------------------------ rejections ------------------------------------------------
@pytest.mark.parametrize("dh", [8, 24, 48, 96, 256])
def test_unsupported_dim_head_is_refused(dh):
    import alphafold2_b200 as A
    from alphafold2_b200 import ops
    ax = A.AxialAttention(dim=64, heads=2, dim_head=dh, row_attn=True, col_attn=False).cuda().eval()
    x = torch.randn(1, 8, 8, 64, device="cuda")
    before = x.clone()
    with pytest.raises(ValueError, match=r"dim_head %d unsupported \(16, 32, 64 or 128 in bf16 mode; strict mode takes any "
                                         r"multiple of 4\)" % dh):
        ax(x)
    torch.cuda.synchronize()
    assert torch.equal(x, before)
    qkv, gate, _, _ = make_inputs(8, 1, 2, dh, False, False, 0)
    with pytest.raises(ValueError, match="16, 32, 64 or 128"):
        ops.attention_bf16(qkv, gate, 8, 1, 2, dh, 8, 1)
