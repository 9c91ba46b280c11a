"""-m gpu: the MSA track run in bands of MSA rows (banded.msa_track_ and the chunked outer-mean projection, through
EvoformerBlock.update_).

Every band call computes each output element from the same inputs, in the same order and with the same kernel as the
whole-tensor call, so the banded trunk must give the whole-tensor trunk's bits: torch.equal on the bit patterns, never a
tolerance.
  * Evoformer.run_ with forced MSA bands against the whole-tensor calls: d 256 and 128, S not a multiple of 8, ragged bands,
    masks with fully masked MSA rows and columns, batch 2, pair rows whole and in bands, and the extra-MSA stack's tied-query
    column attention with the pair rows whole;
  * Alphafold2.forward with MSA bands of 1 and 2 rows on the distogram, templates (angle rows in m), extra-MSA and angles
    fixtures;
  * memory: at N_res 512 x S 4096 the peak with MSA bands is below the whole-tensor peak by what the planner computes;
  * N_res 2048 x S 8448, where m has 4.4e9 elements: the kernels that still touch all of m on sampled MSA rows, a depth-1
    forward that the planner bands, and one block with two MSA band sizes giving equal bits.
"""
import functools

import pytest
import torch

import embed_bounds as E
from conftest import load_golden
from gpu_util import check_bound
from oracle import evoformer_oracle as O

pytestmark = pytest.mark.gpu

GB = 10 ** 9


def _bits(t):
    return t.contiguous().view(torch.int32)


@functools.lru_cache(maxsize=None)
def _evo(d, H, dh, depth, seed, tied=False):
    import alphafold2_b200 as A
    torch.manual_seed(seed)
    evo = A.Evoformer(depth=depth, dim=d, seq_len=64, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0., global_column_attn=tied)
    evo.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.05, seed=seed))
    return evo.cuda().eval()


def _inputs(B, N, S, d, masked, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, N, d, generator=g)
    m = torch.randn(B, S, N, d, generator=g)
    mask = msa_mask = None
    if masked:
        res = torch.rand(B, N, generator=g) > 0.1
        res[:, 5] = False
        res[:, N - 3:] = False
        mask = (res[:, :, None] & res[:, None, :]).cuda()
        msa_mask = torch.rand(B, S, N, generator=g) > 0.2
        msa_mask[:, 0] = True
        msa_mask[:, 2] = False                              # a fully masked MSA row
        msa_mask[:, :, 7] = False                           # and a fully masked MSA column
        msa_mask = msa_mask.cuda()
    return x.cuda(), m.cuda(), mask, msa_mask


def _run(evo, x, m, mask, msa_mask, **kw):
    xo, mo = x.clone(), m.clone()
    evo.run_(xo, mo, mask, msa_mask, **kw)
    torch.cuda.synchronize()
    return xo, mo


def _same(a, r, what):
    assert torch.equal(_bits(a), _bits(r)), f"{what}: max |diff| {(a - r).abs().max().item():.3e}"


@pytest.mark.parametrize("d,H,dh,N,S,B,depth,masked,band,msa_band", [
    (256, 8, 64, 256, 37, 1, 2, True, None, 5),            # S not a multiple of 8, ragged bands: 7 x 5 + 2
    (256, 8, 64, 300, 24, 1, 1, False, None, 24 // 3),     # bands that divide S, N_res not a multiple of 8
    (128, 4, 32, 200, 21, 2, 1, True, None, 4),            # batch 2
    (128, 4, 32, 136, 9, 1, 1, True, None, 1),             # one MSA row per band: 8-column column bands
    (128, 4, 32, 300, 19, 1, 1, True, 256, 3),             # with pair bands (256 + 44)
    (256, 8, 64, 512, 13, 2, 1, True, 256, 6),             # with pair bands, batch 2
])
def test_msa_banded_trunk_bitwise(d, H, dh, N, S, B, depth, masked, band, msa_band):
    evo = _evo(d, H, dh, depth, 7)
    x, m, mask, msa_mask = _inputs(B, N, S, d, masked, seed=N + S + msa_band)
    rx, rm = _run(evo, x, m, mask, msa_mask)
    assert (evo.last_pair_band, evo.last_msa_band) == (N, S), "the whole-tensor reference should fit"
    assert not torch.equal(rm, m)
    bx, bm = _run(evo, x, m, mask, msa_mask, band=band, msa_band=msa_band)
    assert (evo.last_pair_band, evo.last_msa_band) == (band or N, msa_band)
    _same(bx, rx, f"x, MSA bands of {msa_band}, pair bands of {band}")
    _same(bm, rm, f"m, MSA bands of {msa_band}, pair bands of {band}")


@pytest.mark.parametrize("msa_band", [2, 5])
def test_tied_query_stack_with_msa_bands(msa_band):
    """The extra-MSA stack's tied-query pair column attention stays the whole-tensor call when only the MSA track is banded."""
    evo = _evo(128, 4, 32, 1, 8, tied=True)
    x, m, mask, msa_mask = _inputs(1, 136, 11, 128, True, seed=msa_band)
    rx, rm = _run(evo, x, m, mask, msa_mask)
    bx, bm = _run(evo, x, m, mask, msa_mask, msa_band=msa_band)
    assert (evo.last_pair_band, evo.last_msa_band) == (136, msa_band)
    _same(bx, rx, "x")
    _same(bm, rm, "m")


def test_msa_band_must_be_positive():
    evo = _evo(128, 4, 32, 1, 7)
    x, m, _, _ = _inputs(1, 64, 4, 128, False, seed=1)
    with pytest.raises(ValueError, match="positive"):
        evo.run_(x, m, msa_band=0)


# ------------------------------------------------------------------------------------------------------------------------
# Alphafold2.forward on the fixtures
# ------------------------------------------------------------------------------------------------------------------------
def _fixture_model(name):
    import alphafold2_b200 as A
    fx = load_golden(name)
    fx["inputs"] = {k: (v.float() if torch.is_floating_point(v) else v).cuda() for k, v in fx["inputs"].items()}
    model = A.Alphafold2(**fx["cfg"])
    model.load_state_dict({k: (v.float() if torch.is_floating_point(v) else v) for k, v in fx["state"].items()}, strict=False)
    return model.cuda().eval(), fx["inputs"]


def _forward(model, i, msa_band, **kw):
    for evo in (model.net, model.extra_msa_evoformer):
        evo.run_ = functools.partial(type(evo).run_, evo, msa_band=msa_band)
    try:
        with torch.no_grad():
            return model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"], **kw)
    finally:
        del model.net.run_, model.extra_msa_evoformer.run_


@pytest.mark.parametrize("msa_band", [1, 2])
@pytest.mark.parametrize("name", ["alphafold2_distogram", "alphafold2_templates", "alphafold2_extra_msa", "alphafold2_angles"])
def test_alphafold2_forward_fixture_bitwise(name, msa_band):
    model, i = _fixture_model(name)
    kw = {}
    if name == "alphafold2_templates":
        kw = {k: i[k] for k in ("templates_feats", "templates_angles", "templates_mask")}
    elif name == "alphafold2_extra_msa":
        kw = {k: i[k] for k in ("extra_msa", "extra_msa_mask")}
    ref = _forward(model, i, None, **kw)
    rows = i["msa"].shape[1] + (i["templates_angles"].shape[1] if "templates_angles" in kw else 0)
    assert model.net.last_msa_band == rows
    out = _forward(model, i, msa_band, **kw)
    assert model.net.last_msa_band == msa_band < rows
    for key in ("distance", "theta_logits", "phi_logits", "omega_logits"):
        a, r = getattr(out, key, None), getattr(ref, key, None)
        if r is not None:
            _same(a, r, f"{name} {key}, MSA bands of {msa_band}")


# ------------------------------------------------------------------------------------------------------------------------
# memory
# ------------------------------------------------------------------------------------------------------------------------
def _peak(evo, x, m, **kw):
    from alphafold2_b200 import ops
    ops._WORKSPACE.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    evo.run_(x, m, **kw)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ops._WORKSPACE.clear()
    return peak


def test_msa_bands_lower_the_peak_by_what_the_planner_computes():
    from alphafold2_b200 import ops
    d, H, dh, N, S, RS = 256, 8, 64, 512, 4096, 512
    evo = _evo(d, H, dh, 1, 7)
    x, m, _, _ = _inputs(1, N, S, d, False, seed=3)
    whole = _peak(evo, x.clone(), m.clone())
    assert (evo.last_pair_band, evo.last_msa_band) == (N, S)
    banded = _peak(evo, x.clone(), m.clone(), msa_band=RS)
    assert evo.last_msa_band == RS
    planned_whole, planned = ops.pair_block_bytes(1, N, S, d, H, dh, N), ops.msa_block_bytes(1, N, S, d, H, dh, N, RS)
    print(f"N {N} S {S}: peak whole {whole / GB:.3f} GB, MSA bands of {RS} {banded / GB:.3f} GB; planned "
          f"{planned_whole / GB:.3f} / {planned / GB:.3f} GB")
    # the whole-tensor figure includes the grow-only workspace's 5 % growth margin, which one block need not allocate
    assert whole - banded >= planned_whole / 1.05 - planned, f"saved {(whole - banded) / GB:.3f} GB"
    assert banded <= planned, "the planner under-counts the MSA-banded block"


# ------------------------------------------------------------------------------------------------------------------------
# N_res 2048 x S 8448: m has 4.43e9 elements
# ------------------------------------------------------------------------------------------------------------------------
N_BIG, S_BIG = 2048, 8448


def _need(gb):
    from alphafold2_b200 import ops
    ops._WORKSPACE.clear()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < gb * GB:
        pytest.skip(f"needs {gb} GB free on the device, {free / GB:.1f} GB of {total / GB:.1f} GB are")


def test_deep_msa_whole_m_kernels_against_torch():
    """MSA init, the template angle rows after row S, the recycling row and the outer-mean normaliser, on the first, a middle
    and the last 8 MSA rows, where a wrapped 32-bit offset into m would show."""
    from alphafold2_b200 import ops
    _need(40)
    N, S, d, T, R = N_BIG, S_BIG, 256, 2, 32
    assert S * N * d > 2 ** 32
    g = torch.Generator().manual_seed(4)
    emb = torch.randn(22, d, generator=g).cuda()
    w_pair, b_pair = (torch.randn(2 * d, d, generator=g) * d ** -0.5).cuda(), torch.randn(2 * d, generator=g).cuda()
    pos = torch.randn(2 * R + 1, d, generator=g).cuda()
    seq = torch.randint(0, 21, (1, N), generator=g).cuda()
    msa = torch.randint(0, 21, (1, S, N), generator=g).cuda()
    x, m = ops.embed_pair_init(seq, msa, emb, w_pair, b_pair, pos, R, m_rows=S + T)
    rows = torch.tensor([0, 1, S // 2] + list(range(S - 8, S)), device="cuda")
    _, want = E.token_embed(emb, seq, msa[:, rows])             # (emb[msa] + emb[seq]) in fp32, the kernel's order
    assert torch.equal(m[0, rows], want[0]), f"MSA init not bitwise on MSA rows {rows.tolist()}"
    want = m[0, rows].clone()
    # template angle rows S .. S + T - 1, against the module's fp64 output (the end-to-end bound of test_gpu_embed_heads.py)
    K = 55
    w1, b1 = (torch.randn(d, K, generator=g) * K ** -0.5).cuda(), torch.randn(d, generator=g).cuda()
    w2, b2 = (torch.randn(d, d, generator=g) * d ** -0.5).cuda(), torch.randn(d, generator=g).cuda()
    angles = torch.randn(1, T, N, K, generator=g).cuda()
    ops.template_angle_features(ops.pack_template_angles(w1, b1, w2, b2), angles, m, S)
    ref, bound = E.angles_module_ref(angles.view(-1, K), w1, b1, w2, b2, strict=False)
    check_bound(f"bf16/template_angles/deep_msa/N{N}S{S}/module", m[0, S:].reshape(T * N, d), ref, bound)
    assert torch.equal(m[0, rows], want), "the angle rows wrote into the MSA rows"
    # recycling: row 0 of m += LN(single row) (m's batch stride is (S + T) * N * d elements); x += LN(0) + table[bucket] = 0
    row0 = m[0, 0].clone()
    single = torch.randn(1, N, d, generator=g).cuda()
    ones, zeros = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
    ops.recycle_embed_(x, m, torch.zeros(1, N, 3, device="cuda"), single, torch.zeros_like(x), ones, zeros, ones, zeros,
                       torch.zeros(32, d, device="cuda"))
    want_r = row0.double() + torch.nn.functional.layer_norm(single[0].double(), (d,), eps=1e-5)
    err = (m[0, 0].double() - want_r).abs().max().item()
    assert err < 1e-4, f"recycling row 0: max |err| {err:.3e}"
    assert torch.equal(m[0, rows[1:]], want[1:]), "recycling wrote outside row 0"
    del x, row0, single
    # outer-mean normaliser over msa_mask [S][N] on sampled pair rows
    mk = torch.rand(S, N, generator=g) > 0.3
    mk[S - 1] = True
    mkc = mk.cuda()
    for r0 in (0, N - 8):
        scale = torch.empty(8 * N, device="cuda")
        ops.outer_scale(mkc, scale, row0=r0, rows=8, eps=1e-5)
        mf = mk.double()
        cnt = mf[:, r0:r0 + 8].T @ mf
        want_s = 1.0 / (S * (cnt + 1e-5))
        err = (scale.view(8, N).double().cpu() - want_s).abs().max().item()
        assert err <= 1e-6 * want_s.abs().max().item(), f"outer normaliser rows {r0}..: max |err| {err:.3e}"


def test_deep_msa_forward_is_banded_and_symmetric():
    import alphafold2_b200 as A
    _need(70)
    N, S, d = N_BIG, S_BIG, 256
    torch.manual_seed(5)
    model = A.Alphafold2(dim=d, depth=1, heads=8, dim_head=64, max_seq_len=N)
    model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}))
    model = model.cuda().eval()
    seq = torch.randint(0, 21, (1, N), device="cuda")
    msa = torch.randint(0, 21, (1, S, N), device="cuda")
    mask = torch.ones(1, N, dtype=torch.bool, device="cuda")
    mask[:, -5:] = False
    msa_mask = torch.rand(1, S, N, device="cuda") > 0.1
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        dist = model(seq, msa, mask=mask, msa_mask=msa_mask).distance
    torch.cuda.synchronize()
    print(f"N {N} S {S}: bands of {model.net.last_pair_band} pair rows and {model.net.last_msa_band} MSA rows, "
          f"peak {torch.cuda.max_memory_allocated() / GB:.1f} GB")
    assert model.net.last_msa_band < S
    assert bool(torch.isfinite(dist).all())
    assert torch.equal(_bits(dist), _bits(dist.transpose(1, 2)))


def test_deep_msa_block_two_band_sizes_equal():
    _need(70)
    N, S, d = N_BIG, S_BIG, 256
    evo = _evo(d, 8, 64, 1, 9)
    first = None
    for rows in (1024, 2816):
        g = torch.Generator(device="cuda").manual_seed(6)
        x = torch.randn(1, N, N, d, device="cuda", generator=g)
        m = torch.randn(1, S, N, d, device="cuda", generator=g)
        evo.run_(x, m, band=N, msa_band=rows)
        torch.cuda.synchronize()
        assert (evo.last_pair_band, evo.last_msa_band) == (N, rows)
        assert torch.isfinite(x).all()
        if first is None:
            first = (x.cpu(), m.cpu())                 # the device cannot hold two copies beside the block's workspace
            del x, m
            continue
        assert torch.equal(_bits(x.cpu()), _bits(first[0])), "x differs between MSA bands of 1024 and 2816"
        for s0 in range(0, S, 1024):
            assert torch.equal(_bits(m[:, s0:s0 + 1024].cpu()), _bits(first[1][:, s0:s0 + 1024])), f"m rows {s0}.. differ"
