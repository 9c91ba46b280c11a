"""-m gpu: the pair track run in bands of pair rows (alphafold2_b200/banded.py through PairwiseAttentionBlock.update_).

Every band call computes each output element from the same inputs, in the same order and with the same kernel as the
whole-tensor call, so the banded trunk must give the whole-tensor trunk's bits: torch.equal on the bit patterns, never a
tolerance.
  * Evoformer.run_ with forced bands against the whole-tensor calls: divisible and ragged bands, masks with fully masked rows
    and columns, N_res not a multiple of 8, batch 2; Alphafold2.forward on the alphafold2_distogram.pt inputs;
  * memory: at N_res 1024 the peak with 256-row bands is below the whole-tensor peak by at least what pair_block_bytes says;
  * N_res 4096, where x has 2^32 elements: the kernels that still read the whole pair tensor against PyTorch on sampled rows
    (the last 8 included, where a wrapped 32-bit offset shows), a depth-1 Alphafold2.forward that the planner bands, and one
    block with bands of 256 and 512 rows giving equal bits.
"""
import functools

import pytest
import torch

from conftest import load_golden
from oracle import evoformer_oracle as O

pytestmark = pytest.mark.gpu

GB = 10 ** 9


def _bits(t):
    return t.contiguous().view(torch.int32)


@functools.lru_cache(maxsize=None)
def _evo(d, H, dh, depth, seed):
    import alphafold2_b200 as A
    torch.manual_seed(seed)
    evo = A.Evoformer(depth=depth, dim=d, seq_len=64, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
    evo.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.05, seed=seed))
    return evo.cuda().eval()


def _inputs(B, N, S, d, masked, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, N, d, generator=g)
    m = torch.randn(B, S, N, d, generator=g)
    mask = msa_mask = None
    if masked:
        res = torch.rand(B, N, generator=g) > 0.1
        res[:, 5] = False                                   # fully masked row and column in the first band
        res[:, N - 3:] = False                              # ... and in the last one
        res[:, 300 % N] = False
        mask = res[:, :, None] & res[:, None, :]
        msa_mask = torch.rand(B, S, N, generator=g) > 0.2
        msa_mask[:, 0] = True
        msa_mask = msa_mask.cuda()
        mask = mask.cuda()
    return x.cuda(), m.cuda(), mask, msa_mask


def _run(evo, x, m, mask, msa_mask, band):
    xo, mo = x.clone(), m.clone()
    evo.run_(xo, mo, mask, msa_mask, band=band)
    torch.cuda.synchronize()
    return xo, mo


@pytest.mark.parametrize("d,H,dh,N,S,B,depth,masked,band", [
    (256, 8, 64, 512, 32, 1, 2, False, 256),               # bands that divide N
    (256, 8, 64, 600, 32, 1, 1, True, 256),                # 256 + 256 + 88
    (128, 4, 32, 320, 16, 2, 1, True, 256),                # batch 2: 256 + 64
    (128, 4, 32, 300, 8, 1, 1, True, 256),                 # N_res not a multiple of 8: padded operand rows
    (128, 4, 32, 300, 8, 1, 1, False, 64),                 # many small bands
])
def test_banded_trunk_bitwise(d, H, dh, N, S, B, depth, masked, band):
    evo = _evo(d, H, dh, depth, 7)
    x, m, mask, msa_mask = _inputs(B, N, S, d, masked, seed=N + band)
    rx, rm = _run(evo, x, m, mask, msa_mask, None)
    assert evo.last_pair_band == N, "the whole-tensor reference should fit"
    assert not torch.equal(rx, x)
    bx, bm = _run(evo, x, m, mask, msa_mask, band)
    assert evo.last_pair_band == band
    for name, a, r in (("x", bx, rx), ("m", bm, rm)):
        assert torch.equal(_bits(a), _bits(r)), \
            f"{name}: bands of {band} differ from the whole-tensor calls (max |diff| {(a - r).abs().max().item():.3e})"


@pytest.mark.parametrize("band", [8, 16])
def test_alphafold2_forward_fixture_bitwise(band):
    import alphafold2_b200 as A
    fx = load_golden("alphafold2_distogram")
    i = {k: v.cuda() for k, v in fx["inputs"].items()}
    model = A.Alphafold2(**fx["cfg"])
    model.load_state_dict(fx["state"], strict=False)
    model = model.cuda().eval()
    ref = model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"]).distance
    assert model.net.last_pair_band == i["seq"].shape[1]
    model.net.run_ = functools.partial(type(model.net).run_, model.net, band=band)
    out = model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"]).distance
    assert model.net.last_pair_band == band
    assert torch.equal(_bits(out), _bits(ref)), f"bands of {band}: max |diff| {(out - ref).abs().max().item():.3e}"


def test_forced_band_must_keep_tma_alignment():
    evo = _evo(128, 4, 32, 1, 7)
    x, m, _, _ = _inputs(1, 64, 4, 128, False, seed=1)
    with pytest.raises(ValueError, match="multiple of 8"):
        evo.run_(x, m, band=20)


def test_tied_query_stack_refuses_bands():
    import alphafold2_b200 as A
    evo = A.Evoformer(depth=1, dim=128, seq_len=64, heads=4, dim_head=32, attn_dropout=0., ff_dropout=0.,
                      global_column_attn=True).cuda().eval()
    x, m, _, _ = _inputs(1, 64, 4, 128, False, seed=2)
    x0 = x.clone()
    with pytest.raises(NotImplementedError, match="global_query_attn"):
        evo.run_(x, m, band=32)
    assert torch.equal(x, x0), "the refusal came after device work"


# ------------------------------------------------------------------------------------------------------------------------
# memory
# ------------------------------------------------------------------------------------------------------------------------
def _peak(evo, x, m, band):
    from alphafold2_b200 import ops
    ops._WORKSPACE.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    evo.run_(x, m, band=band)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ops._WORKSPACE.clear()
    return peak


def test_bands_lower_the_peak_by_what_the_planner_computes():
    from alphafold2_b200 import ops
    d, H, dh, N, S = 256, 8, 64, 1024, 32
    evo = _evo(d, H, dh, 1, 7)
    x, m, _, _ = _inputs(1, N, S, d, False, seed=3)
    whole = _peak(evo, x.clone(), m.clone(), None)
    assert evo.last_pair_band == N
    banded = _peak(evo, x.clone(), m.clone(), 256)
    want = ops.pair_block_bytes(1, N, S, d, H, dh, N) - ops.pair_block_bytes(1, N, S, d, H, dh, 256)
    print(f"N {N}: peak whole {whole / GB:.3f} GB, bands of 256 {banded / GB:.3f} GB; planned "
          f"{ops.pair_block_bytes(1, N, S, d, H, dh, N) / GB:.3f} / {ops.pair_block_bytes(1, N, S, d, H, dh, 256) / GB:.3f} GB")
    assert whole - banded >= want, f"saved {(whole - banded) / GB:.3f} GB, planned {want / GB:.3f} GB"
    assert banded <= ops.pair_block_bytes(1, N, S, d, H, dh, 256), "the planner under-counts the banded block"


# ------------------------------------------------------------------------------------------------------------------------
# N_res 4096: x has 2^32 elements
# ------------------------------------------------------------------------------------------------------------------------
N_BIG = 4096
ROWS = [0, 1, 1000, 2047, 2048, 3001] + list(range(N_BIG - 8, N_BIG))


def _need(gb):
    from alphafold2_b200 import ops
    ops._WORKSPACE.clear()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < gb * GB:
        pytest.skip(f"needs {gb} GB free on the device, {free / GB:.1f} GB of {total / GB:.1f} GB are")


def test_n4096_whole_tensor_kernels_against_torch():
    from alphafold2_b200 import _lib, ops
    _need(45)
    N, d, H, S, R = N_BIG, 256, 8, 1, 32
    assert N * N * d == 2 ** 32
    g = torch.Generator().manual_seed(4)
    emb = torch.randn(22, d, generator=g).cuda()
    w_pair, b_pair = (torch.randn(2 * d, d, generator=g) * d ** -0.5).cuda(), torch.randn(2 * d, generator=g).cuda()
    pos = torch.randn(2 * R + 1, d, generator=g).cuda()
    seq = torch.randint(0, 21, (1, N), generator=g).cuda()
    msa = torch.randint(0, 21, (1, S, N), generator=g).cuda()
    x, _ = ops.embed_pair_init(seq, msa, emb, w_pair, b_pair, pos, R)
    rows = torch.tensor(ROWS, device="cuda")
    j = torch.arange(N, device="cuda")
    # pair init: x[i][j] = left[i] + right[j] + pos_emb[clamp(i - j)]
    e = emb[seq[0]].double()
    lr = e @ w_pair.double().T + b_pair.double()
    want = lr[rows, None, :d] + lr[None, :, d:] + pos.double()[(rows[:, None] - j[None]).clamp(-R, R) + R]
    err = (x[0, rows].double() - want).abs().max().item()
    assert err < 1e-4, f"pair init: max |err| {err:.3e} on rows {ROWS}"
    # pair bias of the whole x (the triangle attentions' bias, and the MSA row attention's from x)
    we = (torch.randn(H, d, generator=g) * d ** -0.5).cuda()
    bias = torch.zeros(H, N, N, dtype=torch.bfloat16, device="cuda")
    _lib.check(_lib.load().af2_pair_bias(x.data_ptr(), we.data_ptr(), bias.data_ptr(), N, N, d, H, ops._stream_ptr()))
    want = torch.einsum("rjd,hd->hrj", x[0, rows].double(), we.double())
    err = (bias[:, rows].double() - want).abs().max().item()
    assert err <= 2e-2 * want.abs().max().item(), f"pair bias: max |err| {err:.3e} (bf16 output) on rows {ROWS}"
    del bias
    # distogram head: Linear(LayerNorm((x + x^T) / 2))
    ln_w, ln_b = torch.randn(d, generator=g).cuda(), torch.randn(d, generator=g).cuda()
    w, b = (torch.randn(37, d, generator=g) * d ** -0.5).cuda(), torch.randn(37, generator=g).cuda()
    dist = ops.distogram_head(x, ln_w, ln_b, w, b)
    sym = (x[0, rows].double() + x[0, :, rows].transpose(0, 1).double()) * 0.5
    want = torch.nn.functional.layer_norm(sym, (d,), ln_w.double(), ln_b.double(), 1e-5) @ w.double().T + b.double()
    err = (dist[0, rows].double() - want).abs().max().item()
    assert err < 1e-3, f"distogram: max |err| {err:.3e} on rows {ROWS}"
    del dist
    # recycling embedder: x += LN(previous pair) + table[bucket(|c_i - c_j|)]
    prev = x.clone()
    x_rows = x[0, rows].clone()
    coords = (torch.randn(1, N, 3, generator=g) * 10).cuda()
    single = torch.randn(1, N, d, generator=g).cuda()
    m1 = torch.zeros(1, 1, N, d, device="cuda")
    table = torch.randn(32, d, generator=g).cuda()
    ones, zeros = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
    ops.recycle_embed_(x, m1, coords, single, prev, ones, zeros, ln_w, ln_b, table)
    dd = (coords[0, rows, None] - coords[0, None]).pow(2).sum(-1).sqrt()
    bucket = torch.bucketize(dd, ops.recycling_boundaries(32, "cuda")[:31])
    want = (x_rows.double() + torch.nn.functional.layer_norm(prev[0, rows].double(), (d,), ln_w.double(), ln_b.double(), 1e-5)
            + table.double()[bucket])
    err = (x[0, rows].double() - want).abs().max().item()
    assert err < 1e-3, f"recycling: max |err| {err:.3e} on rows {ROWS}"


def test_n4096_forward_is_banded_and_symmetric():
    import alphafold2_b200 as A
    _need(60)
    N, S, d = N_BIG, 32, 256
    torch.manual_seed(5)
    model = A.Alphafold2(dim=d, depth=1, heads=8, dim_head=64, max_seq_len=N)
    model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}))
    model = model.cuda().eval()
    seq = torch.randint(0, 21, (1, N), device="cuda")
    msa = torch.randint(0, 21, (1, S, N), device="cuda")
    mask = torch.ones(1, N, dtype=torch.bool, device="cuda")
    mask[:, -5:] = False
    with torch.no_grad():
        dist = model(seq, msa, mask=mask, msa_mask=torch.ones(1, S, N, dtype=torch.bool, device="cuda")).distance
    torch.cuda.synchronize()
    print(f"N {N}: bands of {model.net.last_pair_band} rows, peak {torch.cuda.max_memory_allocated() / GB:.1f} GB")
    assert model.net.last_pair_band < N
    assert bool(torch.isfinite(dist).all())
    assert torch.equal(_bits(dist), _bits(dist.transpose(1, 2)))


def test_n4096_block_bands_256_and_512_equal():
    _need(70)
    N, S, d = N_BIG, 8, 256
    evo = _evo(d, 8, 64, 1, 9)
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(1, N, N, d, device="cuda", generator=g)
    m = torch.randn(1, S, N, d, device="cuda", generator=g)
    x2, m2 = x.clone(), m.clone()
    evo.run_(x, m, band=256)
    evo.run_(x2, m2, band=512)
    torch.cuda.synchronize()
    assert torch.isfinite(x).all()
    assert torch.equal(_bits(x), _bits(x2)), f"max |diff| {(x - x2).abs().max().item():.3e}"
    assert torch.equal(_bits(m), _bits(m2))
