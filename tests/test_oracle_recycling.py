"""-m "not gpu": the recycling oracle (oracle/recycling_oracle.py) against the fixture of the UNMODIFIED reference
(oracle/make_golden_r4.py) and, when the reference is present, against the live reference, including an n > 25 case that
documents how far torch.cdist's distances are off there; plus the argument checks of Alphafold2.forward's recycling input, which
run before any device work."""
import pytest
import torch

from conftest import load_golden
from oracle import recycling_oracle as RO
from oracle.ref_loader import reference_available


def _fixture():
    """alphafold2_recycling.pt with its bf16-stored (bf16-exact) weights and inputs widened to fp32, the extra-MSA stack's
    weights restored from the trunk's."""
    fx = load_golden("alphafold2_recycling")
    for key in ("state", "inputs"):
        fx[key] = {k: (v.float() if torch.is_floating_point(v) else v) for k, v in fx[key].items()}
    fx["state"] = RO.fixture_state(fx["state"])                # the extra-MSA stack shares the trunk's stored weights
    return fx


def _to(w, dt):
    return {k: (v.to(dt) if torch.is_floating_point(v) else v) for k, v in w.items()}


class _Rec:
    def __init__(self, coords, single_msa_repr_row, pairwise_repr):
        self.coords, self.single_msa_repr_row, self.pairwise_repr = coords, single_msa_repr_row, pairwise_repr


def _oracle(fx, call, dtype):
    i, cfg, spec = fx["inputs"], fx["cfg"], fx["calls"][call]
    st = _to(fx["state"], dtype)
    rec = _Rec(i["coords"], i["single_msa_repr_row"].to(dtype), i["pairwise_repr"].to(dtype))
    kw = {k: i[k] for k in spec["kwargs"] if k != "extra_msa"}
    if "extra_msa" in spec["kwargs"]:
        kw["extra_depth"] = cfg["extra_msa_evoformer_layers"]
    msa, msa_mask = (i["msa"], i["msa_mask"]) if spec["msa"] else (None, None)
    return RO.alphafold2_distogram(st, i["seq"], msa, i["mask"], msa_mask, cfg["heads"], cfg["depth"], recyclables=rec,
                                   templates_embed_layers=cfg["templates_embed_layers"], dtype=dtype, **kw)


CALLS = ["recycling", "recycling_templates", "recycling_extra_msa", "recycling_no_msa"]


@pytest.mark.parametrize("call", CALLS)
def test_alphafold2_recycling_golden(call):
    fx = _fixture()
    assert sorted(fx["calls"]) == sorted(CALLS)
    ref = fx["out_fp64"][call]                                 # the reference's fp64 output, stored rounded to fp32
    torch.testing.assert_close(_oracle(fx, call, torch.float32), ref, rtol=5e-4, atol=5e-5)
    torch.testing.assert_close(_oracle(fx, call, torch.float64), ref.double(), rtol=1e-6, atol=1e-7)


def test_recycling_fixture_coordinates_cover_the_cases():
    c = _fixture()["inputs"]["coords"]
    assert c.dtype == torch.float32
    dist = RO.direct_distances(c)
    k = RO.distance_buckets(c, 32)
    assert set(k.flatten().tolist()) == set(range(32))                      # every bucket occurs
    assert torch.isnan(c).any() and (k[torch.isnan(dist)] == 31).all()        # NaN coordinates -> the last bucket
    off = ~torch.eye(c.shape[1], dtype=torch.bool)
    assert ((dist == 0) & off).any()                                         # two coincident residues
    fin = dist[torch.isfinite(dist)]
    assert (fin > 20).any()
    bnd = RO.recycling_boundaries(32)[:-1].double()
    assert (fin[:, None] - bnd[None, :]).abs().min() >= 1e-3                  # no distance near a boundary


def test_bucketize_edges():
    """torch.bucketize(right=False) on the reference's boundaries: exactly 2.0 -> 0, 20.0 and inf -> nb - 1, NaN -> nb - 1;
    nb = 1 (an empty boundary list) -> 0 everywhere."""
    for nb in (1, 2, 32, 64):
        bnd = RO.recycling_boundaries(nb)[:-1]
        v = torch.tensor([2.0, 20.0, float("inf"), float("nan"), 0.0])
        k = torch.bucketize(v, bnd)
        assert k.tolist() == ([0, nb - 1, nb - 1, nb - 1, 0] if nb > 1 else [0] * 5)
        for j in range(nb - 1):
            assert torch.bucketize(bnd[j:j + 1], bnd).item() == j                # a value equal to boundaries[j] lands in j


@pytest.mark.skipif(not reference_available(), reason="needs the reference source tree")
@pytest.mark.parametrize("n", [12, 64])
def test_recycling_oracle_matches_live_reference(n):
    """For n <= 25 torch.cdist is direct and the oracle matches the reference.  For n > 25 cdist computes |a|^2 + |b|^2 - 2 a.b;
    at coordinates about 40 A from the origin its error reaches hundredths of an angstrom (including on the diagonal), so the
    reference's buckets change near boundaries.  The oracle then matches the reference run with the direct distances."""
    from oracle.evoformer_oracle import randomize_zero_init_
    from oracle.make_golden import _masks
    from oracle.ref_loader import load_reference
    ref = load_reference()
    torch.manual_seed(23)
    cfg = dict(dim=32, depth=1, heads=2, dim_head=32)
    model = ref.Alphafold2(**cfg).eval()
    st = randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, seed=24)
    g = torch.Generator().manual_seed(25)
    for k in ("recycling_msa_norm", "recycling_pairwise_norm"):
        st[k + ".weight"] = 1.0 + 0.5 * torch.randn(32, generator=g)
        st[k + ".bias"] = 0.5 * torch.randn(32, generator=g)
    model.load_state_dict(st)
    b, s = 2, 3
    seq, msa = torch.randint(0, 21, (b, n)), torch.randint(0, 21, (b, s, n))
    mk, mmk = _masks(b, s, n, 26)
    coords = torch.randn(b, n, 3, generator=g) * 3.0 + 23.0                  # about 40 A from the origin
    rec = ref.Recyclables(coords=coords, single_msa_repr_row=torch.randn(b, n, 32, generator=g),
                          pairwise_repr=torch.randn(b, n, n, 32, generator=g))
    with torch.no_grad():
        r = model(seq, msa, mask=mk, msa_mask=mmk, recyclables=rec).distance
    o = RO.alphafold2_distogram(st, seq, msa, mk, mmk, 2, 1, recyclables=rec)
    cd = torch.cdist(coords, coords, p=2).double()
    err = (cd - RO.direct_distances(coords)).abs().max().item()
    print(f"n {n}: max |cdist - direct| = {err:.3e} A")
    if n <= 25:
        assert err < 1e-4
        torch.testing.assert_close(o, r, rtol=5e-4, atol=5e-5)
        return
    assert err > 1e-3                                          # the switch to the |a|^2 + |b|^2 - 2 a.b formula is visible
    real = torch.cdist
    try:
        torch.cdist = lambda a, b_, p=2.0, **kw: (a[:, :, None] - b_[:, None]).pow(2).sum(-1).sqrt()
        with torch.no_grad():
            r_direct = model(seq, msa, mask=mk, msa_mask=mmk, recyclables=rec).distance
    finally:
        torch.cdist = real
    torch.testing.assert_close(o, r_direct, rtol=5e-4, atol=5e-5)


def _model_and_inputs():
    import alphafold2_b200 as A
    model = A.Alphafold2(dim=32, depth=1, heads=2, dim_head=32).eval()
    b, n = 2, 8
    seq, msa = torch.randint(0, 21, (b, n)), torch.randint(0, 21, (b, 2, n))
    mask = torch.ones(b, n, dtype=torch.bool)
    return model, seq, msa, mask, A.Recyclables(torch.randn(b, n, 3), torch.randn(b, n, 32), torch.randn(b, n, n, 32))


def test_recycling_argument_errors():
    """Recyclables the kernel cannot take raise before any device work: these run on CPU tensors."""
    import alphafold2_b200 as A
    model, seq, msa, mask, rec = _model_and_inputs()
    b, n = seq.shape
    with pytest.raises(NotImplementedError, match="recyclables"):
        model(seq, msa, mask=mask, recyclables=object())
    with pytest.raises(NotImplementedError, match="recyclables"):
        model(seq, msa, mask=mask, recyclables=_Rec(rec.coords, rec.single_msa_repr_row, None))
    bad = {"coords": [torch.randn(b, n), torch.randn(b, n + 1, 3), torch.randn(b, n, 0)],
           "single_msa_repr_row": [torch.randn(b, n, 16), torch.randn(b, 1, n, 32)],
           "pairwise_repr": [torch.randn(b, n, n + 1, 32), torch.randn(b, n, 32)]}
    for field, values in bad.items():
        for v in values:
            kw = {"coords": rec.coords, "single_msa_repr_row": rec.single_msa_repr_row, "pairwise_repr": rec.pairwise_repr, field: v}
            with pytest.raises(ValueError, match=field):
                model(seq, msa, mask=mask, recyclables=A.Recyclables(**kw))
    with pytest.raises(ValueError, match="pairwise_repr"):
        model(seq, msa, mask=mask, recyclables=_Rec(rec.coords, rec.single_msa_repr_row,
                                                    torch.zeros(b, n, n, 32, dtype=torch.int32)))
    with pytest.raises(ValueError, match="coords"):
        model(seq, msa, mask=mask, recyclables=_Rec(torch.empty(b, n, 3, device="meta"), rec.single_msa_repr_row,
                                                    rec.pairwise_repr))
    grad = torch.randn(b, n, n, 32, requires_grad=True)
    with pytest.raises(RuntimeError, match="forward-only"):
        model(seq, msa, mask=mask, recyclables=A.Recyclables(rec.coords, rec.single_msa_repr_row, grad))


def test_recycling_keeps_state_keys():
    import alphafold2_b200 as A
    keys = set(A.Alphafold2(dim=32, depth=1, heads=2, dim_head=32, recycling_distance_buckets=7).state_dict())
    for k in ("recycling_msa_norm.weight", "recycling_msa_norm.bias", "recycling_pairwise_norm.weight",
              "recycling_pairwise_norm.bias", "recycling_distance_embed.weight"):
        assert k in keys
