"""-m gpu: the recycling embedder (alphafold2.py:728-739).

Kernel alone (glue_recycle_kernel through af2_recycle_embed) against fp64 math on the exact operands the kernel was given,
element-wise with `check_bound`.  u = 2^-24.  For a row p of d values (mean mu, rstd = 1 / sqrt(var + eps), z = (p - mu) rstd,
y = gamma z + beta) the kernel computes, in fp32:
  * the mean as a sum of d terms and one division:          |dmu| <= u (sum |p| + |mu|)
  * the centred values p - mu^ (one rounding each), the biased variance as a sum of d squares, + eps, sqrtf and 1 / x
    (IEEE, one rounding each):                               rstd^ = rstd (1 + r), |r| <= ((d + 1) / 2 + 3) u, to first order
                                                             (the variance about mu^ exceeds the one about mu by d dmu^2 only)
  * z^ = (p - mu^) rstd^ (one rounding):                     |z^ - z| <= rstd |dmu| + |z| ((d + 1) / 2 + 5) u
  * y^ = fmaf(z^, gamma, beta) (one rounding):               |y^ - y| <= |gamma| |z^ - z| + u |y^|
  * the two fp32 adds (x + y^) + E[k] on the pair, m + y^ on row 0 of m, one rounding each.
The test bound doubles the dmu term (it also reaches the variance) and counts u (|gamma z| + |beta|) for the fma:
  e_y   = 2 |gamma| rstd dmu + |gamma| |z| (d / 2 + 8) u + 2 u (|gamma z| + |beta|)
  pair: |out - ref| <= e_y + u (|x + y| + |ref|);   row 0 of m: |out - ref| <= e_y + u |ref|.
The bucket k of the pair is compared exactly (the table row must be the one the fp64 distance selects), except where the fp64
distance lies within max(4, (c + 4) / 2) u dist of a boundary: there either neighbour is accepted (the kernel's fp32 distance,
c squared differences summed by fmaf then sqrtf, has a relative error below that).  Rows of m other than row 0 (the template
angle rows among them) must stay bitwise equal, guard regions after x and m must stay untouched, and two identical launches
must be bitwise equal.

Buckets alone: with gamma = beta = 0 and x = 0 every output row is bitwise one table row (channel 0 of row k holds k), so the
kernel's bucket is read back and compared with torch.bucketize of the fp64 distance; a distance equal to boundaries[k] (the
points (0, 0, 0) and (b_k, 0, 0)) must land in k, NaN coordinates in nb - 1, coincident points in 0.

Module: Alphafold2.forward with recyclables against the fixture of the unmodified reference (bf16: `check()` with its autocast
yardstick; strict: `check_strict()` against the reference's fp64 output, which the fixture stores rounded to fp32), the C2
shape (d 256, n 256, S 128, one block) against the fp64 oracle, the disable_token_embed glue path, and the error cases.
"""
import pytest
import torch

from conftest import load_golden
from gpu_util import autocast_yardstick, check, check_bound, check_strict, dev
from oracle import evoformer_oracle as O
from oracle import recycling_oracle as RO

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GUARD = 4096
EPS = 1e-5


def _ln64(p, g, b):
    p = p.double()
    mu = p.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt((p - mu).pow(2).mean(-1, keepdim=True) + EPS)
    z = (p - mu) * rstd
    y = z * g.double() + b.double()
    d = p.shape[-1]
    dmu = U * (p.abs().sum(-1, keepdim=True) + mu.abs())
    ey = 2 * g.double().abs() * rstd * dmu + g.double().abs() * z.abs() * (d / 2 + 8) * U + 2 * U * ((g.double() * z).abs() + b.double().abs())
    return y, ey


def _launch(x0, m0, coords, s, p, mg, mb, pg, pb, table, bnd):
    """One af2_recycle_embed on fresh copies of x0 / m0 inside NaN-guarded buffers; returns (x, m)."""
    from alphafold2_b200 import ops
    nx, nm = x0.numel(), m0.numel()
    xb = torch.full((nx + GUARD,), float("nan"), device="cuda")
    mb_ = torch.full((nm + GUARD,), float("nan"), device="cuda")
    xb[:nx] = x0.flatten()
    mb_[:nm] = m0.flatten()
    x, m = xb[:nx].view(x0.shape), mb_[:nm].view(m0.shape)
    ops.recycle_embed_(x, m, coords, s, p, mg, mb, pg, pb, table, eps=EPS, boundaries=bnd)
    torch.cuda.synchronize()
    assert torch.isnan(xb[nx:]).all() and torch.isnan(mb_[nm:]).all(), "guard written"
    return x, m


def _kernel_case(name, B, n, d, nb, c, rows=3, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *sh, s=1.0, o=0.0: torch.randn(*sh, generator=g, device="cuda") * s + o  # noqa: E731
    x0 = rn(B, n, n, d)
    m0 = rn(B, rows, n, d)
    p = rn(B, n, n, d, s=2.0, o=3.0)
    s = rn(B, n, d, s=1.5, o=-2.0)
    pg, pb, mg, mb = rn(d, s=0.5, o=1.0), rn(d, s=0.5), rn(d, s=0.5, o=1.0), rn(d, s=0.5)
    table = rn(nb, d)
    coords = rn(B, n, c, s=9.0, o=5.0)
    if n > 3:
        coords[0, 1] = coords[0, 2]                          # coincident residues
        coords[-1, 3] = float("nan")                         # a residue with NaN coordinates
    from alphafold2_b200 import ops
    bnd = ops.recycling_boundaries(nb, "cuda")
    outs = [_launch(x0, m0, coords, s, p, mg, mb, pg, pb, table, bnd) for _ in range(2)]
    (x1, m1), (x2, m2) = outs
    assert torch.equal(x1.view(torch.int32), x2.view(torch.int32)) and torch.equal(m1.view(torch.int32), m2.view(torch.int32)), \
        f"{name}: launches differ"
    assert torch.equal(m1[:, 1:].view(torch.int32), m0[:, 1:].view(torch.int32)), f"{name}: rows of m other than row 0 changed"

    dist = RO.direct_distances(coords)
    tol = max(4.0, (c + 4) / 2) * U * dist.nan_to_num(0.0)
    b64 = bnd[:-1].double()
    k_lo = torch.bucketize(dist - tol, b64)
    k_hi = torch.bucketize(dist + tol, b64)
    k_mid = torch.bucketize(dist, b64)
    y, ey = _ln64(p, pg, pb)
    base = x0.double() + y
    t64 = table.double()
    ref = base + t64[k_mid]
    amb = k_lo != k_hi
    if amb.any():                                            # a boundary within the distance's rounding: accept either neighbour
        alt_lo, alt_hi = base + t64[k_lo], base + t64[k_hi]
        x64 = x1.double()
        pick_lo = (x64 - alt_lo).abs().amax(-1) <= (x64 - alt_hi).abs().amax(-1)
        ref = torch.where(amb[..., None], torch.where(pick_lo[..., None], alt_lo, alt_hi), ref)
    bound = ey + U * (base.abs() + ref.abs())
    check_bound(f"{name}/pair", x1, ref, bound)
    ym, eym = _ln64(s, mg, mb)
    refm = m0[:, 0].double() + ym
    check_bound(f"{name}/msa_row0", m1[:, 0], refm, eym + U * refm.abs())


SMALL = [(B, n, d, nb, c) for n in (1, 7, 37) for d in (32, 128, 256, 384) for nb in (1, 2, 32, 64)
         for (B, c) in [((n + d + nb) % 2 + 1, 3 if (d // 32 + nb) % 2 else 5)]]
LARGE = [(1, n, d, 32, 3) for n in (256, 300) for d in (32, 128, 256, 384)] + [(2, 300, 256, 64, 5), (2, 256, 128, 1, 3)]


@pytest.mark.parametrize("B,n,d,nb,c", SMALL + LARGE)
def test_recycle_kernel_vs_fp64(B, n, d, nb, c):
    _kernel_case(f"recycle_kernel b{B} n{n} d{d} nb{nb} c{c}", B, n, d, nb, c, seed=B * 7 + n * 3 + d + nb * 11 + c)


def _bucket_case(name, coords, nb, d=32):
    """gamma = beta = 0, x = 0: every output row is bitwise table[k]; returns the kernel's buckets [B, n, n]."""
    from alphafold2_b200 import ops
    B, n, _ = coords.shape
    g = torch.Generator(device="cuda").manual_seed(nb)
    table = torch.randn(nb, d, generator=g, device="cuda")
    table[:, 0] = torch.arange(nb, device="cuda", dtype=torch.float32)
    z = torch.zeros(d, device="cuda")
    p = torch.randn(B, n, n, d, generator=g, device="cuda")
    x = torch.zeros(B, n, n, d, device="cuda")
    m = torch.zeros(B, 1, n, d, device="cuda")
    ops.recycle_embed_(x, m, coords, torch.randn(B, n, d, device="cuda"), p, z, z, z, z, table, eps=EPS)
    torch.cuda.synchronize()
    k = x[..., 0].long()
    assert ((k >= 0) & (k < nb)).all(), f"{name}: bucket out of range"
    assert torch.equal(x.view(torch.int32), table[k].view(torch.int32)), f"{name}: output row is not a table row"
    assert (m == 0).all()
    return k


@pytest.mark.parametrize("nb", [1, 2, 32, 64])
@pytest.mark.parametrize("n,c,center", [(37, 3, 0.0), (300, 3, 40.0 / 3 ** 0.5), (64, 5, 10.0)])
def test_recycle_buckets_match_bucketize(nb, n, c, center):
    from alphafold2_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n + nb)
    coords = torch.randn(1, n, c, generator=g, device="cuda") * 7.0 + center
    coords[0, 5] = coords[0, 4]
    coords[0, 9] = float("nan")
    coords[0, 11, 1] = float("nan")                          # one NaN coordinate is enough
    k = _bucket_case(f"buckets n{n} c{c} nb{nb}", coords, nb)
    dist = RO.direct_distances(coords)
    b64 = ops.recycling_boundaries(nb, "cuda")[:-1].double()
    tol = 4.0 * U * dist.nan_to_num(0.0) * max(1.0, (c + 4) / 8)
    k_lo, k_hi = torch.bucketize(dist - tol, b64), torch.bucketize(dist + tol, b64)
    ok = (k == k_lo) | (k == k_hi)
    amb = int((k_lo != k_hi).sum())
    print(f"buckets n{n} c{c} nb{nb}: {amb} pairs within rounding of a boundary")
    assert ok.all(), f"bucket mismatch at {ok.logical_not().nonzero()[:5].tolist()}"
    assert (k[0, 9] == nb - 1).all() and (k[0, :, 9] == nb - 1).all() and (k[0, 11] == nb - 1).all()
    assert k[0, 4, 5] == 0 and k[0, 5, 4] == 0 and (torch.diagonal(k[0])[torch.isfinite(coords[0]).all(-1)] == 0).all()


@pytest.mark.parametrize("nb", [2, 7, 32, 64])
def test_recycle_distance_on_a_boundary(nb):
    """coords (0, 0, 0) and (b_k, 0, 0) for k = 0 .. nb-2: the distance is exactly boundaries[k] and must land in k."""
    from alphafold2_b200 import ops
    bnd = ops.recycling_boundaries(nb, "cuda")
    coords = torch.zeros(1, nb, 3, device="cuda")
    coords[0, 1:, 0] = bnd[:-1]
    k = _bucket_case(f"boundary nb{nb}", coords, nb)
    want = torch.arange(nb - 1, device="cuda")
    assert torch.equal(k[0, 0, 1:], want) and torch.equal(k[0, 1:, 0], want)


def test_recycle_kernel_rejects_bad_args():
    from alphafold2_b200 import ops
    f = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
    B, n, d, nb = 1, 4, 32, 8
    args = lambda dd=d, c=3: (f(B, n, n, dd), f(B, 2, n, dd), f(B, n, c), f(B, n, dd), f(B, n, n, dd), f(dd), f(dd), f(dd), f(dd),  # noqa: E731
                              f(nb, dd))
    with pytest.raises(ValueError, match="dim"):
        ops.recycle_embed_(*args(dd=30))
    with pytest.raises(ValueError, match="dim"):
        ops.recycle_embed_(*args(dd=1028))
    with pytest.raises(ValueError):
        ops.recycle_embed_(*args(c=0))
    a = list(args())
    a[4] = torch.zeros(B * n * n * d + 1, device="cuda")[1:].view(B, n, n, d)     # previous pair 4 bytes off 16-byte alignment
    with pytest.raises(ValueError, match="aligned"):
        ops.recycle_embed_(*a)
    with pytest.raises(ValueError, match="boundaries"):
        ops.recycle_embed_(*args(), boundaries=torch.zeros(nb - 1, device="cuda"))


# ------------------------------------------------------------------------------------------------------------------------
# module and model
# ------------------------------------------------------------------------------------------------------------------------
def _fixture():
    fx = load_golden("alphafold2_recycling")
    for key in ("state", "inputs"):
        fx[key] = {k: (v.float() if torch.is_floating_point(v) else v) for k, v in fx[key].items()}
    fx["state"] = RO.fixture_state(fx["state"])                # the extra-MSA stack shares the trunk's stored weights
    return fx


def _af2(cfg, state, precision):
    import alphafold2_b200 as A
    model = A.Alphafold2(**cfg)
    assert not model.load_state_dict(state, strict=False).unexpected_keys
    return A.set_precision(model.cuda().eval(), precision)


@pytest.mark.parametrize("precision", ["bf16", "strict"])
@pytest.mark.parametrize("call", ["recycling", "recycling_templates", "recycling_extra_msa", "recycling_no_msa"])
def test_alphafold2_recycling_golden(call, precision):
    import alphafold2_b200 as A
    fx = _fixture()
    i = {k: v.cuda() for k, v in fx["inputs"].items()}
    spec = fx["calls"][call]
    model = _af2(fx["cfg"], fx["state"], precision)
    rec = A.Recyclables(i["coords"], i["single_msa_repr_row"], i["pairwise_repr"])
    kw = {k: i[k] for k in spec["kwargs"]}
    if spec["msa"]:
        ret = model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"], recyclables=rec, return_recyclables=True, **kw)
    else:
        ret = model(i["seq"], mask=i["mask"], recyclables=rec, **kw)
    if precision == "strict":
        # the literal band against the reference's fp64 output (stored rounded to fp32): no looser than against its fp32 run
        check_strict(f"strict/alphafold2_recycling/{call}/golden/distance", ret.distance, fx["out_fp64"][call])
    else:
        check(f"alphafold2_recycling/{call}/golden/distance", ret.distance, fx["out_fp64"][call], fx["out_autocast_bf16"][call])
    assert ret.recyclables is None


def test_alphafold2_recycling_c2_vs_oracle():
    """d 256, heads 8, dim_head 64, n 256, S 128, one block, coordinates about 40 A from the origin: against the fp64 oracle."""
    import alphafold2_b200 as A
    torch.manual_seed(31)
    n, S, d = 256, 128, 256
    model = A.Alphafold2(dim=d, depth=1, heads=8, dim_head=64)
    st = O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(32)
    for k in ("recycling_msa_norm", "recycling_pairwise_norm"):
        st[k + ".weight"] = 1.0 + 0.3 * torch.randn(d, generator=g)
        st[k + ".bias"] = 0.3 * torch.randn(d, generator=g)
    model.load_state_dict(st)
    model = model.cuda().eval()
    seq, msa = torch.randint(0, 21, (1, n)), torch.randint(0, 21, (1, S, n))
    mask = torch.ones(1, n, dtype=torch.bool)
    mask[:, -16:] = False
    msa_mask = torch.rand(1, S, n, generator=g) > 0.1
    coords = torch.randn(1, n, 3, generator=g) * 12.0 + 23.0
    coords[0, 17] = float("nan")
    rec = A.Recyclables(coords.cuda(), torch.randn(1, n, d, generator=g).cuda(), torch.randn(1, n, n, d, generator=g).cuda())
    cu = [t.cuda() for t in (seq, msa, mask, msa_mask)]
    ret = model(*cu[:2], mask=cu[2], msa_mask=cu[3], recyclables=rec)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = RO.alphafold2_distogram(dev(st, torch.float64), *cu, 8, 1, recyclables=rec, dtype=torch.float64).cpu()
        ac = autocast_yardstick(lambda: RO.alphafold2_distogram(dev(st), *cu, 8, 1, recyclables=rec)).float().cpu()
    check("alphafold2_recycling/c2_d256_n256_s128/oracle/distance", ret.distance, ref, ac)


def test_alphafold2_recycling_disable_token_embed():
    """The eager glue path (disable_token_embed): seq_embed = W[seq], msa_embed = W[msa] equals the oracle's token embedding W."""
    import alphafold2_b200 as A
    torch.manual_seed(41)
    n, S, d = 24, 3, 64
    model = A.Alphafold2(dim=d, depth=1, heads=2, dim_head=32, disable_token_embed=True)
    st = O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(42)
    for k in ("recycling_msa_norm", "recycling_pairwise_norm"):
        st[k + ".weight"] = 1.0 + 0.3 * torch.randn(d, generator=g)
        st[k + ".bias"] = 0.3 * torch.randn(d, generator=g)
    model.load_state_dict(st)
    model = model.cuda().eval()
    W = torch.randn(22, d, generator=g)
    seq, msa = torch.randint(0, 21, (1, n)), torch.randint(0, 21, (1, S, n))
    mask, msa_mask = torch.ones(1, n, dtype=torch.bool), torch.ones(1, S, n, dtype=torch.bool)
    mask[:, -3:] = False
    coords = torch.randn(1, n, 3, generator=g) * 8.0
    rec = A.Recyclables(coords.cuda(), torch.randn(1, n, d, generator=g).cuda(), torch.randn(1, n, n, d, generator=g).cuda())
    ret = model(seq.cuda(), msa.cuda(), mask=mask.cuda(), msa_mask=msa_mask.cuda(), seq_embed=W[seq].cuda(), msa_embed=W[msa].cuda(),
                recyclables=rec)
    st["token_emb.weight"] = W
    cu = [t.cuda() for t in (seq, msa, mask, msa_mask)]
    with torch.no_grad():
        ref = RO.alphafold2_distogram(dev(st, torch.float64), *cu, 2, 1, recyclables=rec, dtype=torch.float64).cpu()
        ac = autocast_yardstick(lambda: RO.alphafold2_distogram(dev(st), *cu, 2, 1, recyclables=rec)).float().cpu()
    check("alphafold2_recycling/disable_token_embed/oracle/distance", ret.distance, ref, ac)


def test_alphafold2_recycling_errors_and_dtypes():
    import alphafold2_b200 as A
    torch.manual_seed(5)
    model = A.Alphafold2(dim=32, depth=1, heads=2, dim_head=32).cuda().eval()
    b, n = 2, 8
    seq, msa = torch.randint(0, 21, (b, n)).cuda(), torch.randint(0, 21, (b, 2, n)).cuda()
    mask = torch.ones(b, n, dtype=torch.bool).cuda()
    rec = A.Recyclables((torch.randn(b, n, 3) * 8).cuda(), torch.randn(b, n, 32).bfloat16().cuda(),
                        torch.randn(b, n, n, 32).bfloat16().cuda())
    with pytest.raises(NotImplementedError, match="recyclables"):
        model(seq, msa, mask=mask, recyclables=object())
    with pytest.raises(ValueError, match="single_msa_repr_row"):
        model(seq, msa, mask=mask, recyclables=A.Recyclables(rec.coords, rec.single_msa_repr_row.cpu(), rec.pairwise_repr))
    with pytest.raises(ValueError, match="pairwise_repr"):
        model(seq, msa, mask=mask, recyclables=A.Recyclables(rec.coords, rec.single_msa_repr_row, rec.pairwise_repr[:, :-1]))
    # any floating dtype is widened to fp32: bf16 / fp64 recyclables give the same result as their fp32 values
    r_lo = model(seq, msa, mask=mask, recyclables=rec, return_recyclables=True)
    r32 = model(seq, msa, mask=mask, recyclables=A.Recyclables(rec.coords.double(), rec.single_msa_repr_row.float(),
                                                               rec.pairwise_repr.float()))
    assert r_lo.recyclables is None
    assert torch.equal(r_lo.distance, r32.distance)
    r0 = model(seq, msa, mask=mask)
    assert not torch.equal(r0.distance, r32.distance)
    coords_model = A.Alphafold2(dim=32, depth=1, heads=2, dim_head=32, predict_coords=True).cuda().eval()
    with pytest.raises(NotImplementedError):
        coords_model(seq, msa, mask=mask, recyclables=rec)
