"""The general Attention.forward oracle (oracle/attention_oracle.py) against the unmodified reference's Attention
(tests/golden/attention_forward.pt, oracle/make_golden_r8.py), and against evoformer_oracle.attention where both apply."""
import os

import pytest
import torch

from oracle import attention_oracle as AO
from oracle import evoformer_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "attention_forward.pt")


def _fixture():
    return torch.load(GOLDEN, weights_only=False)


def _names():
    return sorted(_fixture()["cases"])


@pytest.mark.parametrize("name", _names())
def test_oracle_matches_reference(name):
    fx = _fixture()
    case = fx["cases"][name]
    st64 = {k: v.double() for k, v in fx["state"].items()}
    kw = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in case["inputs"].items()}
    out = AO.attention(st64, "", kw.pop("x"), fx["cfg"]["heads"], **kw)
    ref = case["out"].double()
    assert out.shape == ref.shape
    assert torch.allclose(out, ref, rtol=1e-5, atol=1e-6), (out - ref).abs().max().item()


def test_defaults_are_self_attention_oracle():
    fx = _fixture()
    st64 = {k: v.double() for k, v in fx["state"].items()}
    for name in ("self", "self_mask", "self_bias_bhij", "self_bias_1hij", "tied_self"):
        kw = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in fx["cases"][name]["inputs"].items()}
        x = kw.pop("x")
        a = AO.attention(st64, "", x, fx["cfg"]["heads"], **kw)
        b = O.attention(st64, "", x, fx["cfg"]["heads"], **kw)
        assert torch.equal(a, b), name
