"""-m "not gpu": the template-embedder oracle (oracle/template_oracle.py) against fixtures of the UNMODIFIED reference
(oracle/make_golden_r3.py) and, when the reference is present, against the live reference; plus the argument checks of
Alphafold2.forward's template branch, which run before any device work."""
import pytest
import torch

from conftest import load_golden
from oracle import template_oracle as TO
from oracle.ref_loader import reference_available


def _templates_fixture():
    """alphafold2_templates.pt with its bf16-stored (bf16-exact) weights and template inputs widened to fp32."""
    fx = load_golden("alphafold2_templates")
    for key in ("state", "inputs"):
        fx[key] = {k: (v.float() if torch.is_floating_point(v) else v) for k, v in fx[key].items()}
    return fx


def _to(w, dt):
    return {k: (v.to(dt) if torch.is_floating_point(v) else v) for k, v in w.items()}


def test_template_pointwise_attention_golden():
    fx = load_golden("template_pointwise")
    i, c = fx["inputs"], fx["cfg"]
    out = TO.template_pointwise_attention(fx["state"], "", i["x"], i["context"], c["heads"], i["mask"], i["context_mask"])
    torch.testing.assert_close(out, fx["out_fp32"], rtol=1e-5, atol=1e-6)
    out = TO.template_pointwise_attention(_to(fx["state"], torch.float64), "", i["x"].double(), i["context"].double(), c["heads"],
                                          i["mask"], i["context_mask"])
    torch.testing.assert_close(out, fx["out_fp64"], rtol=1e-10, atol=1e-12)
    # quirk: a masked query, or one whose context is all masked, averages all T values uniformly
    w = _to(fx["state"], torch.float64)
    v = torch.nn.functional.linear(i["context"].double(), w["to_kv.weight"])[..., c["heads"] * c["dim_head"]:]
    uni = (~i["mask"][:, 0]) | (~i["context_mask"]).all(-1)
    assert uni.any()
    gate = torch.sigmoid(torch.nn.functional.linear(i["x"].double(), w["gating.weight"], w["gating.bias"]))
    expect = torch.nn.functional.linear(v.mean(1, keepdim=True) * gate, w["to_out.weight"], w["to_out.bias"])
    torch.testing.assert_close(out[uni], expect[uni], rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("call", ["feats_angles", "feats", "angles"])
def test_alphafold2_templates_golden(call):
    fx = _templates_fixture()
    i, cfg = fx["inputs"], fx["cfg"]
    kw = {k: i[k] for k in fx["calls"][call]}
    out = TO.alphafold2_distogram(fx["state"], i["seq"], i["msa"], i["mask"], i["msa_mask"], cfg["heads"], cfg["depth"],
                                  templates_embed_layers=cfg["templates_embed_layers"], **kw)
    torch.testing.assert_close(out, fx["out_fp32"][call], rtol=5e-4, atol=5e-5)
    out = TO.alphafold2_distogram(_to(fx["state"], torch.float64), i["seq"], i["msa"], i["mask"], i["msa_mask"], cfg["heads"],
                                  cfg["depth"], templates_embed_layers=cfg["templates_embed_layers"], dtype=torch.float64, **kw)
    torch.testing.assert_close(out, fx["out_fp64"][call], rtol=1e-6, atol=1e-7)


def test_template_fixture_masks_cover_the_quirks():
    i = _templates_fixture()["inputs"]
    tm, mask = i["templates_mask"], i["mask"]
    assert (~tm).all(-1).any()                                   # a template fully masked
    assert (~tm).all(1).any()                                    # a residue where every template is masked
    assert (~mask).any()                                         # a masked residue suffix ...
    tm2 = tm[:, :, :, None] & tm[:, :, None, :]
    xm = mask[:, :, None] & mask[:, None, :]
    assert (tm2.any(1) & ~xm).any()                              # ... whose pairs still have a valid template


def test_pooled_is_not_x_mask():
    """alphafold2.py:779: a pair masked by x_mask that has a valid template still receives the (uniform-mean) update."""
    fx = _templates_fixture()
    st, i = _to(fx["state"], torch.float64), fx["inputs"]
    b, n = i["seq"].shape
    x = torch.randn(b, n, n, 32, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    xm = i["mask"][:, :, None] & i["mask"][:, None, :]
    out = TO.embed_templates(st, x, xm, i["templates_feats"].double(), i["templates_mask"], 2, 1)
    tm = i["templates_mask"]
    pooled = (tm[:, :, :, None] & tm[:, :, None, :]).any(1)
    assert ((out - x).abs().amax(-1)[~xm & pooled] > 0).all()
    assert ((out - x)[~pooled] == 0).all()


@pytest.mark.skipif(not reference_available(), reason="needs the reference source tree")
def test_template_oracle_matches_live_reference():
    from oracle.evoformer_oracle import randomize_zero_init_
    from oracle.make_golden import _masks
    from oracle.make_golden_r3 import template_masks
    from oracle.ref_loader import load_reference
    ref = load_reference()
    torch.manual_seed(11)
    cfg = dict(dim=32, depth=1, heads=2, dim_head=32, templates_embed_layers=1, templates_angles_feats_dim=13)
    model = ref.Alphafold2(**cfg).eval()
    st = randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, seed=12)
    model.load_state_dict(st)
    b, n, s, T = 1, 17, 2, 2
    seq, msa = torch.randint(0, 21, (b, n)), torch.randint(0, 21, (b, s, n))
    mk, mmk = _masks(b, s, n, 21)
    tm = template_masks(b, T, n, 22)
    feats, angles = torch.randn(b, T, n, n, 32), torch.randn(b, T, n, 13)
    with torch.no_grad():
        r = model(seq, msa, mask=mk, msa_mask=mmk, templates_feats=feats, templates_mask=tm, templates_angles=angles).distance
    o = TO.alphafold2_distogram(st, seq, msa, mk, mmk, 2, 1, templates_feats=feats, templates_mask=tm, templates_angles=angles,
                                templates_embed_layers=1)
    torch.testing.assert_close(o, r, rtol=5e-4, atol=5e-5)


def _model_and_inputs():
    import alphafold2_b200 as A
    model = A.Alphafold2(dim=32, depth=1, heads=2, dim_head=32, templates_embed_layers=1).eval()
    b, n, T = 1, 8, 2
    seq, msa = torch.randint(0, 21, (b, n)), torch.randint(0, 21, (b, 2, n))
    mask = torch.ones(b, n, dtype=torch.bool)
    return model, seq, msa, mask, torch.randn(b, T, n, n, 32), torch.randn(b, T, n, 55), torch.ones(b, T, n, dtype=torch.bool)


def test_template_argument_errors():
    """Inputs the reference cannot handle (it fails inside einops / torch.cat) raise ValueError naming the missing argument,
    before any device work: these run on CPU tensors."""
    model, seq, msa, mask, feats, angles, tm = _model_and_inputs()
    with pytest.raises(ValueError, match="mask"):
        model(seq, msa, templates_feats=feats, templates_mask=tm)
    with pytest.raises(ValueError, match="templates_mask"):
        model(seq, msa, mask=mask, templates_feats=feats)
    with pytest.raises(ValueError, match="templates_mask"):
        model(seq, msa, mask=mask, templates_angles=angles)
    with pytest.raises(NotImplementedError, match="recyclables"):
        model(seq, msa, mask=mask, recyclables=object())


def test_template_modules_keep_state_keys():
    import alphafold2_b200 as A
    model = A.Alphafold2(dim=32, depth=1, heads=2, dim_head=32)
    keys = set(model.state_dict())
    for k in ("to_template_embed.weight", "to_template_embed.bias", "template_angle_mlp.0.weight", "template_angle_mlp.2.bias",
              "template_pointwise_attn.to_q.weight", "template_pointwise_attn.to_out.bias"):
        assert k in keys
