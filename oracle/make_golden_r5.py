"""TEST INFRASTRUCTURE ONLY — round-5 fixture from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r5
  tests/golden/alphafold2_angles.pt  Alphafold2(dim=32, depth=1, heads=2, dim_head=32, predict_angles=True).forward, b 2, n 20
                                     (two whole 8-token tiles and a partial one), S 4, partial masks; two calls sharing the weights:
                                     symmetrize_omega False, then True (the flag is a plain attribute, alphafold2.py:550).  Stored:
                                     distance, theta_logits and phi_logits once (the flag does not change them: asserted), omega_logits
                                     per call; and the trunk output x, captured by a forward hook on the reference's `net`, so that the
                                     heads can be pinned without the trunk.
Weights and inputs are bf16-exact (stored as bf16); outputs and trunk output of the fp64 run are stored rounded once to fp32
(relative error <= 2^-24, far inside every tolerance that reads them) and serve as the fp32 reference too; the bf16-autocast
run's outputs (bf16 already: its Linear layers run in bf16) are stored as bf16 for the bf16-mode gates.  Under 1 MB.
Same conventions as oracle/make_golden_r4.py otherwise."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.evoformer_oracle import randomize_zero_init_  # noqa: E402
from oracle.make_golden import _masks, OUT  # noqa: E402

OUTPUTS = ("distance", "theta_logits", "phi_logits", "omega_logits")


def main():
    ref = load_reference()
    torch.manual_seed(23)
    mcfg = dict(dim=32, depth=1, heads=2, dim_head=32, predict_angles=True)
    model = ref.Alphafold2(**mcfg).eval()
    full = randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()})
    full = {k: (v.bfloat16().float() if torch.is_floating_point(v) else v) for k, v in full.items()}
    model.load_state_dict(full)
    used = ("token_emb.", "to_pairwise_repr.", "pos_emb.", "net.", "to_distogram_logits.", "to_prob_")
    state = {k: (v.bfloat16() if torch.is_floating_point(v) else v) for k, v in full.items() if k.startswith(used)}

    bb, n, s = 2, 20, 4
    seq = torch.randint(0, 21, (bb, n))
    msa = torch.randint(0, 21, (bb, s, n))
    mk, mmk = _masks(bb, s, n, 29)
    inputs = {"seq": seq, "msa": msa, "mask": mk, "msa_mask": mmk}
    fx = {"cfg": mcfg, "state": state, "inputs": inputs, "out_fp64": {}, "out_autocast_bf16": {}, "calls": {}}

    trunk = {}
    hook = model.net.register_forward_hook(lambda mod, args, out: trunk.__setitem__("x", out[0].detach().clone()))

    def run(autocast=False):
        with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16, enabled=autocast):
            ret = model(seq, msa, mask=mk, msa_mask=mmk)
        return {k: getattr(ret, k) for k in OUTPUTS}, trunk["x"].float()

    for sym in (False, True):
        model.symmetrize_omega = sym
        model.double()
        out64, x64 = run()
        model.float()
        outac, _ = run(autocast=True)
        assert all(v.dtype == torch.bfloat16 for v in outac.values())
        fx["calls"][f"sym{int(sym)}"] = {"symmetrize_omega": sym, "out_fp64": {k: v.float() for k, v in out64.items()},
                                         "out_autocast_bf16": outac, "x_fp64": x64}
    hook.remove()
    # the trunk, the distance, theta and phi do not depend on the flag: stored once
    c0, c1 = fx["calls"]["sym0"], fx["calls"]["sym1"]
    assert torch.equal(c0["x_fp64"], c1["x_fp64"])
    fx["x_fp64"] = c0.pop("x_fp64")
    c1.pop("x_fp64")
    for kind in ("out_fp64", "out_autocast_bf16"):
        for k in ("distance", "theta_logits", "phi_logits"):
            assert torch.equal(c0[kind][k], c1[kind][k]), (kind, k)
            fx[kind][k] = c0[kind].pop(k)
            c1[kind].pop(k)
    path = os.path.join(OUT, "alphafold2_angles.pt")
    torch.save(fx, path)
    print(f"wrote alphafold2_angles ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
