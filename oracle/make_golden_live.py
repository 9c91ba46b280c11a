"""TEST INFRASTRUCTURE ONLY — generate tests/golden/live_reference_*.pt from the UNMODIFIED reference.

Run where the reference is installed (see oracle/ref_loader.py):   python -m oracle.make_golden_live
tests/test_oracle_vs_reference.py compares the oracle against these stored reference outputs, so it runs anywhere.
Each fixture: {"cfg", "seed", "inputs", "ref_out"}.  The weights are not stored: seeded_state() rebuilds them from the seed
over the state-dict keys of this package's drop-in module (the same keys as the reference's, tests/test_cabi_loads.py).
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
EVO_CASES = [(24, 5, 32, 2, 16, 2, True), (17, 3, 64, 4, 16, 1, False)]


def seeded_state(module, seed):
    """fp32 weights for every entry of module.state_dict(): N(0, fan_in^-1/2) matrices, 1 + N(0, 0.1) norm scales,
    N(0, 0.1) vectors; integer buffers are kept.  Drawn in sorted key order, so the values depend on the key names and
    shapes only, not on the order in which the module registers its submodules."""
    g = torch.Generator().manual_seed(seed)
    st = {}
    for k, v in sorted(module.state_dict().items()):
        if not v.is_floating_point():
            st[k] = v.clone()
        elif v.dim() >= 2:
            st[k] = torch.randn(v.shape, generator=g) * (v.shape[-1] ** -0.5)
        elif "norm" in k and k.endswith("weight"):
            st[k] = 1 + 0.1 * torch.randn(v.shape, generator=g)
        else:
            st[k] = 0.1 * torch.randn(v.shape, generator=g)
    return st


def evoformer_case(ref, N, S, d, H, dh, depth, masked):
    import alphafold2_b200 as A
    torch.manual_seed(11 + N)
    evo = ref.Evoformer(depth=depth, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.).eval()
    st = seeded_state(A.Evoformer(depth=depth, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.), seed=N)
    evo.load_state_dict(st)
    x, m = torch.randn(1, N, N, d), torch.randn(1, S, N, d)
    mask = msa_mask = None
    if masked:
        m1 = torch.ones(1, N, dtype=torch.bool)
        m1[:, -3:] = False
        mask = m1[:, :, None] & m1[:, None, :]
        msa_mask = torch.rand(1, S, N) > 0.15
        msa_mask[:, :, -3:] = False
        msa_mask[:, 0, :N - 3] = True
    with torch.no_grad():
        rx, rm = evo.double()(x.double(), m.double(), mask=mask, msa_mask=msa_mask)
    return {"cfg": dict(N=N, S=S, d=d, H=H, dh=dh, depth=depth), "seed": N,
            "inputs": {"x": x, "m": m, "mask": mask, "msa_mask": msa_mask}, "ref_out": (rx, rm)}


def distogram_case(ref):
    import alphafold2_b200 as A
    torch.manual_seed(5)
    cfg = dict(dim=32, depth=1, heads=2, dim_head=16)
    model = ref.Alphafold2(**cfg).eval()
    st = seeded_state(A.Alphafold2(**cfg), seed=3)
    model.load_state_dict(st)
    seq = torch.randint(0, 21, (1, 20))
    msa = torch.randint(0, 21, (1, 3, 20))
    mask = torch.ones(1, 20, dtype=torch.bool)
    mask[:, -2:] = False
    msa_mask = torch.ones(1, 3, 20, dtype=torch.bool)
    msa_mask[:, :, -2:] = False
    with torch.no_grad():
        r = model(seq, msa, mask=mask, msa_mask=msa_mask).distance
    return {"cfg": cfg, "seed": 3, "inputs": {"seq": seq, "msa": msa, "mask": mask, "msa_mask": msa_mask}, "ref_out": r}


def main():
    from oracle.ref_loader import load_reference
    ref = load_reference()
    for case in EVO_CASES:
        N, S, d, H, dh, depth, masked = case
        torch.save(evoformer_case(ref, *case), os.path.join(OUT, f"live_reference_evoformer_N{N}_d{d}.pt"))
    torch.save(distogram_case(ref), os.path.join(OUT, "live_reference_distogram.pt"))


if __name__ == "__main__":
    main()
