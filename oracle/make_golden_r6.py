"""TEST INFRASTRUCTURE ONLY — round-6 fixtures from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r6
Head widths other than 32 / 64:
  tests/golden/evoformer_dh16.pt        EvoformerBlock(dim=64, heads=4, dim_head=16), b 1, N 24, S 5, partial masks
  tests/golden/evoformer_dh128.pt       EvoformerBlock(dim=128, heads=2, dim_head=128), b 1, N 20, S 4, partial masks
  tests/golden/alphafold2_dh128.pt      Alphafold2(dim=32, depth=1, heads=2, dim_head=128, templates_embed_layers=1).forward,
                                        b 1, n 12, S 3, two templates (feats + angles), partial masks
Weights.  The d 128 block alone has 1.25 M parameters (2.5 MB in bf16), so the weights are not stored: each fixture stores the
seed, the key -> shape list and the SHA-256 of the bf16 weights, and `seeded_state` regenerates them (CPU torch.randn from a
seeded Generator, rounded to bf16).  Readers assert the digest, so a change in the generator fails loudly instead of
comparing against other weights.  Matrices are N(0, 1 / fan_in), LayerNorm weights 1 + N(0, 0.01), other vectors N(0, 0.01).
Inputs are bf16-exact (stored as bf16); outputs of the fp64 run are stored rounded once to fp32 (relative error <= 2^-24);
the bf16-autocast run's outputs are stored as the reference returns them (the blocks' fp32 residual streams, the distogram's
bf16 logits).  Each file is under 1 MB."""
import hashlib
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.make_golden import _masks, OUT  # noqa: E402


def seeded_state(shapes: dict, seed: int) -> dict:
    """bf16-exact fp32 weights for {key: shape}, drawn in sorted key order from one seeded CPU generator"""
    g = torch.Generator().manual_seed(seed)
    st = {}
    for k in sorted(shapes):
        shape = tuple(shapes[k])
        r = torch.randn(shape, generator=g, dtype=torch.float32)
        if len(shape) >= 2:
            v = r * shape[-1] ** -0.5
        elif "norm" in k and k.endswith("weight"):
            v = 1 + 0.1 * r
        else:
            v = 0.1 * r
        st[k] = v.bfloat16().float()
    return st


def state_digest(state: dict) -> str:
    h = hashlib.sha256()
    for k in sorted(state):
        h.update(k.encode())
        h.update(state[k].detach().bfloat16().contiguous().view(torch.int16).numpy().tobytes())
    return h.hexdigest()


def fixture_state(fx: dict) -> dict:
    """the fixture's weights (fp32, bf16-exact), regenerated and checked against the stored digest"""
    st = seeded_state(fx["shapes"], fx["seed"])
    assert state_digest(st) == fx["sha256"], "seeded_state no longer reproduces the fixture's weights"
    return st


def _shapes(state, used=None):
    return {k: list(v.shape) for k, v in state.items() if torch.is_floating_point(v) and (used is None or k.startswith(used))}


def evoformer_case(ref, name, d, H, dh, N, S, seed):
    blk = ref.EvoformerBlock(dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.).eval()
    shapes = _shapes(blk.state_dict())
    st = seeded_state(shapes, seed)
    blk.load_state_dict(st)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(1, N, N, d, generator=g).bfloat16()
    m = torch.randn(1, S, N, d, generator=g).bfloat16()
    mask1, msa_mask = _masks(1, S, N, seed + 2)
    mask = mask1[:, :, None] & mask1[:, None, :]

    def run(dt, autocast=False):
        blk.to(dt)
        with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16, enabled=autocast):
            out = blk((x.to(dt), m.to(dt), mask, msa_mask))[:2]
        blk.float()
        return out

    o64 = run(torch.float64)
    oac = run(torch.float32, autocast=True)
    fx = {"cfg": dict(dim=d, heads=H, dim_head=dh, N=N, S=S, b=1), "seed": seed, "shapes": shapes, "sha256": state_digest(st),
          "inputs": {"x": x, "m": m, "mask": mask, "msa_mask": msa_mask},
          "out_fp64": [o.float() for o in o64], "out_autocast_bf16": list(oac)}
    path = os.path.join(OUT, name + ".pt")
    torch.save(fx, path)
    print(f"wrote {name} ({os.path.getsize(path)} bytes)")


def alphafold2_case(ref, seed):
    from oracle.make_golden_r3 import template_masks
    mcfg = dict(dim=32, depth=1, heads=2, dim_head=128, templates_embed_layers=1)
    model = ref.Alphafold2(**mcfg).eval()
    used = ("token_emb.", "to_pairwise_repr.", "pos_emb.", "net.", "to_distogram_logits.", "to_template_embed.",
            "template_pairwise_embedder.", "template_pointwise_attn.", "template_angle_mlp.")
    full = model.state_dict()
    shapes = {k: s for k, s in _shapes(full, used).items() if not k.startswith("template_pairwise_embedder.outer_mean.")}
    st = seeded_state(shapes, seed)
    model.load_state_dict({**full, **st})
    b, n, s, T = 1, 12, 3, 2
    g = torch.Generator().manual_seed(seed + 1)
    seq = torch.randint(0, 21, (b, n), generator=g)
    msa = torch.randint(0, 21, (b, s, n), generator=g)
    mk, mmk = _masks(b, s, n, seed + 2)
    tm = template_masks(b, T, n, seed + 3)
    tm[0, T - 1, :n // 2] = True                          # the second template keeps valid residues
    feats = torch.randn(b, T, n, n, 32, generator=g).bfloat16()
    angles = torch.randn(b, T, n, 55, generator=g).bfloat16()
    inputs = {"seq": seq, "msa": msa, "mask": mk, "msa_mask": mmk, "templates_feats": feats, "templates_angles": angles,
              "templates_mask": tm}

    def run(dt, autocast=False):
        model.to(dt)
        with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16, enabled=autocast):
            out = model(seq, msa, mask=mk, msa_mask=mmk, templates_feats=feats.to(dt), templates_angles=angles.to(dt),
                        templates_mask=tm).distance
        model.float()
        return out

    fx = {"cfg": mcfg, "seed": seed, "shapes": shapes, "sha256": state_digest(st), "inputs": inputs,
          "out_fp64": run(torch.float64).float(), "out_autocast_bf16": run(torch.float32, autocast=True).bfloat16()}
    path = os.path.join(OUT, "alphafold2_dh128.pt")
    torch.save(fx, path)
    print(f"wrote alphafold2_dh128 ({os.path.getsize(path)} bytes)")


def main():
    from oracle.ref_loader import load_reference
    ref = load_reference()
    evoformer_case(ref, "evoformer_dh16", 64, 4, 16, 24, 5, 61)
    evoformer_case(ref, "evoformer_dh128", 128, 2, 128, 20, 4, 62)
    alphafold2_case(ref, 63)


if __name__ == "__main__":
    main()
