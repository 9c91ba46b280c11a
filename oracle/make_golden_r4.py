"""TEST INFRASTRUCTURE ONLY — round-4 fixture from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r4
  tests/golden/alphafold2_recycling.pt  Alphafold2(dim=32, depth=1, heads=2, dim_head=32, templates_embed_layers=1,
                                        extra_msa_evoformer_layers=1).forward with recyclables, b 2, n 12, S 3, four calls:
                                        recyclables alone; with templates_feats + templates_angles; with extra_msa /
                                        extra_msa_mask (the reference's test_recycling shape); msa=None
n = 12 <= 25, so the reference's torch.cdist is the direct formula and its buckets are the intended ones.  The coordinates hold
one residue with NaN coordinates, two coincident residues and pairs beyond 20 A; every bucket 0..31 occurs, and no finite
distance lies within 1e-3 A of a boundary (seeds are tried until both hold), so the fixture does not depend on how a distance
is rounded.  Weights (both recycling LayerNorms' gamma and beta randomised, so that a gamma / beta swap shows) and
representations are rounded to bf16-exact values and stored as bf16; coordinates are stored in fp32.
Kept small (a fixture this size belongs in the repository only below 1 MB):
  * the extra-MSA stack is given the trunk's weights and they are stored once, under net.*; recycling_oracle.fixture_state()
    restores the extra_msa_evoformer.* keys.  The call with extra_msa pins where recycling sits relative to that stack; the
    stack's own weights are pinned by alphafold2_extra_msa.pt (oracle/make_golden_r2.py);
  * the fp64 outputs are stored rounded once to fp32 (relative error <= 2^-24, far inside every tolerance that reads them), and
    serve as the fp32 reference too: no separate fp32 run is stored.
Same conventions as oracle/make_golden.py and oracle/make_golden_r3.py otherwise."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.evoformer_oracle import randomize_zero_init_  # noqa: E402
from oracle.make_golden import _masks, OUT  # noqa: E402
from oracle.make_golden_r3 import template_masks  # noqa: E402
from oracle.recycling_oracle import SHARED_PREFIX, direct_distances, fixture_state, recycling_boundaries  # noqa: E402

NB = 32
MARGIN = 1e-3
CALLS = {"recycling": dict(kwargs=[], msa=True),
         "recycling_templates": dict(kwargs=["templates_feats", "templates_angles", "templates_mask"], msa=True),
         "recycling_extra_msa": dict(kwargs=["extra_msa", "extra_msa_mask"], msa=True),
         "recycling_no_msa": dict(kwargs=[], msa=False)}


def fixture_coords(b, n, seed):
    """Residues on a jittered line in each batch element, batch 1 with a NaN residue (4) and two coincident ones (7, 8)."""
    g = torch.Generator().manual_seed(seed)
    pos = torch.rand(b, n, generator=g) * 26.0
    c = torch.stack((pos, torch.randn(b, n, generator=g) * 0.4, torch.randn(b, n, generator=g) * 0.4), -1)
    c = c + torch.tensor([7.0, -3.0, 12.0])
    c[1, 8] = c[1, 7]
    c[1, 4] = float("nan")
    return c.float()


def coords_ok(c):
    dist = direct_distances(c)
    bnd = recycling_boundaries(NB)[:-1].double()
    k = torch.bucketize(dist, bnd)
    fin = dist[torch.isfinite(dist)]
    near = (fin[:, None] - bnd[None, :]).abs().min().item() < MARGIN
    return (not near) and set(k.flatten().tolist()) == set(range(NB)) and bool((fin > 20).any())


def main():
    ref = load_reference()
    torch.manual_seed(17)
    mcfg = dict(dim=32, depth=1, heads=2, dim_head=32, templates_embed_layers=1, extra_msa_evoformer_layers=1,
                recycling_distance_buckets=NB)
    model = ref.Alphafold2(**mcfg).eval()
    full = randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()})
    g = torch.Generator().manual_seed(18)
    for k in ("recycling_msa_norm", "recycling_pairwise_norm"):
        full[k + ".weight"] = 1.0 + 0.5 * torch.randn(32, generator=g)
        full[k + ".bias"] = 0.5 * torch.randn(32, generator=g)
    full = {k: (v.bfloat16().float() if torch.is_floating_point(v) else v) for k, v in full.items()}
    for k in [k for k in full if k.startswith(SHARED_PREFIX)]:
        del full[k]
    full = fixture_state(full)
    model.load_state_dict(full)
    used = ("token_emb.", "to_pairwise_repr.", "pos_emb.", "net.", "to_distogram_logits.", "to_template_embed.",
            "template_pairwise_embedder.", "template_pointwise_attn.", "template_angle_mlp.", "recycling_")
    state = {k: (v.bfloat16() if torch.is_floating_point(v) else v) for k, v in full.items()
             if k.startswith(used) and not k.startswith("template_pairwise_embedder.outer_mean.")}

    bb, n, s, T = 2, 12, 3, 2
    seed = 100
    while not coords_ok(fixture_coords(bb, n, seed)):
        seed += 1
    coords = fixture_coords(bb, n, seed)
    seq = torch.randint(0, 21, (bb, n))
    msa = torch.randint(0, 21, (bb, s, n))
    mk, mmk = _masks(bb, s, n, 19)
    _, emk = _masks(bb, s, n, 20)                          # extra_msa_mask has the MSA's shape (the stack embeds `msa`)
    single = (torch.randn(bb, n, 32, generator=g) * 1.5 + 0.3).bfloat16()
    pair = (torch.randn(bb, n, n, 32, generator=g) * 2.0 - 0.4).bfloat16()
    inputs = {"seq": seq, "msa": msa, "mask": mk, "msa_mask": mmk, "coords": coords, "single_msa_repr_row": single,
              "pairwise_repr": pair, "templates_feats": torch.randn(bb, T, n, n, 32, generator=g).bfloat16(),
              "templates_angles": torch.randn(bb, T, n, 55, generator=g).bfloat16(), "templates_mask": template_masks(bb, T, n, 21),
              "extra_msa": torch.randint(0, 21, (bb, 5, n)), "extra_msa_mask": emk}
    fx = {"cfg": mcfg, "state": state, "inputs": inputs, "coords_seed": seed, "calls": CALLS,
          "out_fp64": {}, "out_autocast_bf16": {}}

    def run(call, dt):
        cv = lambda v: v.to(dt) if torch.is_floating_point(v) else v  # noqa: E731
        rec = ref.Recyclables(coords=cv(coords), single_msa_repr_row=cv(single), pairwise_repr=cv(pair))
        kw = {k: cv(inputs[k]) for k in CALLS[call]["kwargs"]}
        if CALLS[call]["msa"]:
            return model(seq, msa, mask=mk, msa_mask=mmk, recyclables=rec, **kw).distance
        return model(seq, mask=mk, recyclables=rec, **kw).distance

    with torch.no_grad():
        for call in CALLS:
            model.double()
            fx["out_fp64"][call] = run(call, torch.float64).float()
            model.float()
            with torch.autocast("cpu", dtype=torch.bfloat16):
                fx["out_autocast_bf16"][call] = run(call, torch.float32)
    torch.save(fx, os.path.join(OUT, "alphafold2_recycling.pt"))
    print(f"wrote alphafold2_recycling (coordinate seed {seed})")


if __name__ == "__main__":
    main()
