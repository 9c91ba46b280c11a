"""TEST INFRASTRUCTURE ONLY — round-3 fixtures from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r3
  tests/golden/template_pointwise.pt    Attention(x, context=..., mask=..., context_mask=...): the pointwise template attention
                                        (alphafold2.py:125-190 with context, called as at :769-774)
  tests/golden/alphafold2_templates.pt  Alphafold2(dim=32, depth=1, heads=2, dim_head=32, templates_embed_layers=2).forward
                                        with templates, b 2, n 12, S 3, T 3, three calls: feats + angles, feats only, angles only;
                                        bf16-exact weights and template inputs, stored as bf16
Masks produce every quirk of the template branch: a masked residue suffix in `mask` (pairs masked by x_mask that still have
valid templates), one template fully masked, one residue where every template is masked (pooled = 0), random holes.
Same conventions as oracle/make_golden.py."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.evoformer_oracle import randomize_zero_init_  # noqa: E402
from oracle.make_golden import _masks, _run, _autocast, OUT  # noqa: E402


def template_masks(b, T, n, seed):
    g = torch.Generator().manual_seed(seed)
    tm = torch.rand(b, T, n, generator=g) > 0.15          # random holes
    tm[0, T - 1] = False                                  # one template fully masked
    tm[:, :, 5] = False                                   # a residue where every template is masked
    tm[:, 0, -3:] = True                                  # the residues masked in `mask` keep a valid template
    return tm


CALLS = ("feats_angles", "feats", "angles")


def main():
    ref = load_reference()

    # ---------------- Attention with context, alone -----------------
    torch.manual_seed(5)
    d, H, dh, Np, T = 32, 2, 32, 300, 4
    mod = ref.Attention(dim=d, heads=H, dim_head=dh)
    state = randomize_zero_init_({k: v.clone() for k, v in mod.state_dict().items()})
    mod.load_state_dict(state)
    mod.eval()
    g = torch.Generator().manual_seed(6)
    x, ctx = torch.randn(Np, 1, d, generator=g) * 2, torch.randn(Np, T, d, generator=g) * 2
    mask = torch.rand(Np, 1, generator=g) > 0.2
    cmask = torch.rand(Np, T, generator=g) > 0.3
    cmask[:, 1] = False                                   # one context slot never valid
    cmask[:20] = False                                    # rows with every context slot masked
    fn = lambda md, dt: md(x.to(dt), mask=mask, context=ctx.to(dt), context_mask=cmask)  # noqa: E731
    fx = {"cfg": dict(dim=d, heads=H, dim_head=dh, N=Np, T=T), "state": state,
          "inputs": {"x": x, "context": ctx, "mask": mask, "context_mask": cmask},
          "out_fp32": _run(mod, torch.float32, fn), "out_fp64": _run(mod, torch.float64, fn), "out_autocast_bf16": _autocast(mod, fn)}
    torch.save(fx, os.path.join(OUT, "template_pointwise.pt"))
    print("wrote template_pointwise")

    # ---------------- Alphafold2.forward with templates -----------------
    # Kept small: the weights (the reference's init, Q8-randomised) and the template inputs are rounded to bf16-exact values
    # and stored as bf16, only the weights the forward reads are stored, and tests widen them to fp32 losslessly.
    torch.manual_seed(7)
    mcfg = dict(dim=32, depth=1, heads=2, dim_head=32, templates_embed_layers=2)
    model = ref.Alphafold2(**mcfg).eval()
    full = randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()})
    full = {k: (v.bfloat16().float() if torch.is_floating_point(v) else v) for k, v in full.items()}
    model.load_state_dict(full)
    used = ("token_emb.", "to_pairwise_repr.", "pos_emb.", "net.", "to_distogram_logits.", "to_template_embed.",
            "template_pairwise_embedder.", "template_pointwise_attn.", "template_angle_mlp.")
    state = {k: (v.bfloat16() if torch.is_floating_point(v) else v) for k, v in full.items()
             if k.startswith(used) and not k.startswith("template_pairwise_embedder.outer_mean.")}
    bb, n, s, T = 2, 12, 3, 3
    seq = torch.randint(0, 21, (bb, n))
    msa = torch.randint(0, 21, (bb, s, n))
    mk, mmk = _masks(bb, s, n, 15)
    tm = template_masks(bb, T, n, 16)
    feats = torch.randn(bb, T, n, n, 32).bfloat16()
    angles = torch.randn(bb, T, n, 55).bfloat16()
    args = {"feats_angles": dict(templates_feats=feats, templates_angles=angles, templates_mask=tm),
            "feats": dict(templates_feats=feats, templates_mask=tm),
            "angles": dict(templates_angles=angles, templates_mask=tm)}
    fx = {"cfg": mcfg, "state": state, "inputs": {"seq": seq, "msa": msa, "mask": mk, "msa_mask": mmk, "templates_feats": feats,
                                                "templates_angles": angles, "templates_mask": tm},
          "calls": {c: sorted(args[c]) for c in CALLS}, "out_fp32": {}, "out_fp64": {}, "out_autocast_bf16": {}}
    with torch.no_grad():
        for c in CALLS:
            a32 = {k: (v.float() if torch.is_floating_point(v) else v) for k, v in args[c].items()}
            a64 = {k: (v.double() if torch.is_floating_point(v) else v) for k, v in args[c].items()}
            fx["out_fp32"][c] = model(seq, msa, mask=mk, msa_mask=mmk, **a32).distance
            model.double()
            fx["out_fp64"][c] = model(seq, msa, mask=mk, msa_mask=mmk, **a64).distance
            model.float()
            with torch.autocast("cpu", dtype=torch.bfloat16):
                fx["out_autocast_bf16"][c] = model(seq, msa, mask=mk, msa_mask=mmk, **a32).distance
    torch.save(fx, os.path.join(OUT, "alphafold2_templates.pt"))
    print("wrote alphafold2_templates")


if __name__ == "__main__":
    main()
