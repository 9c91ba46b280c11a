"""The angle-heads oracle (oracle/heads_oracle.py) against tests/golden/alphafold2_angles.pt, which the unmodified reference
generated (oracle/make_golden_r5.py): from the stored trunk output and end to end, with symmetrize_omega off and on."""
import pytest
import torch

from conftest import load_golden
from oracle import heads_oracle as HO

CALLS = ("sym0", "sym1")
NAMES = {"theta": "theta_logits", "phi": "phi_logits", "omega": "omega_logits", "distance": "distance"}


def _outs(fx, call, kind="out_fp64"):
    """the call's outputs: distance, theta and phi are stored once (symmetrize_omega does not change them), omega per call"""
    return {**fx[kind], **fx["calls"][call][kind]}


def _f64(st):
    return {k: (v.double() if torch.is_floating_point(v) else v) for k, v in st.items()}


@pytest.mark.parametrize("call", CALLS)
def test_angle_heads_from_trunk_output(call):
    fx = load_golden("alphafold2_angles")
    c = fx["calls"][call]
    out = HO.angle_heads(_f64(fx["state"]), fx["x_fp64"].double(), c["symmetrize_omega"])
    for name, o in zip(("theta", "phi", "omega"), out):
        ref = _outs(fx, call)[NAMES[name]].double()
        assert o.shape == ref.shape
        # the fixture holds the fp64 run rounded to fp32, and x the same way: 1e-6 covers both roundings
        assert torch.allclose(o, ref, rtol=1e-6, atol=1e-6), f"{call}/{name}: {(o - ref).abs().max().item():.3e}"


@pytest.mark.parametrize("call", CALLS)
def test_alphafold2_angles_end_to_end(call):
    fx = load_golden("alphafold2_angles")
    c, cfg, i = fx["calls"][call], fx["cfg"], fx["inputs"]
    out = HO.alphafold2_angles(_f64(fx["state"]), i["seq"], i["msa"], i["mask"], i["msa_mask"], cfg["heads"], cfg["depth"],
                               c["symmetrize_omega"], dtype=torch.float64)
    assert torch.allclose(out["x"], fx["x_fp64"].double(), rtol=1e-6, atol=1e-6)
    for name, key in NAMES.items():
        ref = _outs(fx, call)[key].double()
        assert torch.allclose(out[name], ref, rtol=1e-6, atol=1e-6), f"{call}/{name}: {(out[name] - ref).abs().max().item():.3e}"
    # fp32 oracle: the reference's fp32 class
    out32 = HO.alphafold2_angles(fx["state"], i["seq"], i["msa"], i["mask"], i["msa_mask"], cfg["heads"], cfg["depth"],
                                 c["symmetrize_omega"], dtype=torch.float32)
    for name, key in NAMES.items():
        assert torch.allclose(out32[name].double(), _outs(fx, call)[key].double(), rtol=1e-3, atol=1e-4), f"{call}/{name} fp32"


def test_fixture_omega_symmetric_exactly_when_symmetrized():
    fx = load_golden("alphafold2_angles")
    for call in CALLS:
        c = fx["calls"][call]
        om = c["out_fp64"]["omega_logits"]
        assert torch.equal(om, om.transpose(1, 2)) == c["symmetrize_omega"], call
        ac = c["out_autocast_bf16"]["omega_logits"]
        assert torch.equal(ac, ac.transpose(1, 2)) == c["symmetrize_omega"], call
    assert fx["x_fp64"].shape[1] % 8 != 0, "the fixture should end in a partial 8-token tile"
