"""The fp64 oracle at head widths 16 and 128 against fixtures of the UNMODIFIED reference (oracle/make_golden_r6.py): an
EvoformerBlock with 4 heads x 16 and one with 2 heads x 128, and Alphafold2.forward at dim_head 128 with two templates."""
import pytest
import torch

from conftest import load_golden
from oracle import evoformer_oracle as O
from oracle import template_oracle as TO
from oracle.make_golden_r6 import fixture_state


def _f64(st):
    return {k: (v.double() if torch.is_floating_point(v) else v) for k, v in st.items()}


@pytest.mark.parametrize("name,dh", [("evoformer_dh16", 16), ("evoformer_dh128", 128)])
def test_evoformer_block_dim_head_golden(name, dh):
    fx = load_golden(name)
    c, i = fx["cfg"], fx["inputs"]
    assert c["dim_head"] == dh
    st = _f64(fixture_state(fx))
    assert st["layer.2.row_attn.attn.to_q.weight"].shape[0] == c["heads"] * dh
    x, m = O.evoformer_block(st, "", i["x"].double(), i["m"].double(), c["heads"], i["mask"], i["msa_mask"])
    for o, ref in zip((x, m), fx["out_fp64"]):
        # the fixture holds the fp64 run rounded to fp32
        assert torch.allclose(o, ref.double(), rtol=1e-6, atol=1e-6), f"{name}: {(o - ref.double()).abs().max().item():.3e}"
    assert (~i["mask"]).any() and (~i["msa_mask"]).any(), "the fixture should carry partial masks"


def test_alphafold2_dim_head_128_golden():
    fx = load_golden("alphafold2_dh128")
    c, i = fx["cfg"], fx["inputs"]
    st = _f64(fixture_state(fx))
    out = TO.alphafold2_distogram(st, i["seq"], i["msa"], i["mask"], i["msa_mask"], c["heads"], c["depth"],
                                  templates_feats=i["templates_feats"].double(), templates_mask=i["templates_mask"],
                                  templates_angles=i["templates_angles"].double(),
                                  templates_embed_layers=c["templates_embed_layers"], dtype=torch.float64)
    ref = fx["out_fp64"].double()
    assert torch.allclose(out, ref, rtol=1e-6, atol=1e-6), f"{(out - ref).abs().max().item():.3e}"
    assert i["templates_feats"].shape[1] == 2 and i["templates_mask"].any(-1).all()


def test_dim_head_fixture_weights_are_the_seeded_ones():
    """a fixture's weights are regenerated from its seed; a different seed must not pass the digest check"""
    fx = dict(load_golden("alphafold2_dh128"))
    fixture_state(fx)
    fx["seed"] += 1
    with pytest.raises(AssertionError, match="no longer reproduces"):
        fixture_state(fx)
