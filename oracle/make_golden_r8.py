"""TEST INFRASTRUCTURE ONLY — round-8 fixture from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r8
  tests/golden/attention_forward.pt  the reference's Attention(dim=32, heads=2, dim_head=16) called on its own, fp32 on CPU:
                                     self-attention, cross-attention (i > j and i < j), the three bias shapes [B, h, i, j],
                                     [1, h, i, j] and [h, i, j], mask without context_mask, context_mask without mask (ignored),
                                     fully masked query rows, one query over a short context (the template call site) and tied
                                     queries with and without a context.  Lengths are not multiples of 8.
Weights and inputs are bf16-exact fp32; outputs are the fp32 results.  Under 200 KB."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.evoformer_oracle import randomize_zero_init_  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402

CFG = dict(dim=32, heads=2, dim_head=16)


def _bf(t):
    return t.bfloat16().float()


def cases(B=4, i=11, jc=6, d=32, h=2, seed=5):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: _bf(torch.randn(*s, generator=g))  # noqa: E731
    x, xl, c, cl = r(B, i, d), r(B, 3, d), r(B, jc, d), r(B, 19, d)
    m = torch.rand(B, i, generator=g) > 0.3
    m[1] = False                                           # a batch element with every query masked: uniform rows
    cm, cml = torch.rand(B, jc, generator=g) > 0.3, torch.rand(B, 19, generator=g) > 0.3
    x1, t1 = r(B, 1, d), r(B, 4, d)
    m1, tm1 = torch.rand(B, 1, generator=g) > 0.3, torch.rand(B, 4, generator=g) > 0.3
    tm1[0] = False
    return {
        "self": dict(x=x),
        "self_mask": dict(x=x, mask=m),
        "self_bias_bhij": dict(x=x, mask=m, attn_bias=r(B, h, i, i)),
        "self_bias_1hij": dict(x=x, attn_bias=r(1, h, i, i)),
        "self_bias_hij": dict(x=x, mask=m, attn_bias=r(h, i, i)),
        "cross_i_gt_j": dict(x=x, context=c, mask=m, context_mask=cm),
        "cross_i_lt_j": dict(x=xl, context=cl, mask=m[:, :3], context_mask=cml, attn_bias=r(B, h, 3, 19)),
        "cross_no_context_mask": dict(x=x, context=c, mask=m),
        "cross_context_mask_only": dict(x=x, context=c, context_mask=cm),
        "cross_j1": dict(x=x, context=c[:, :1], mask=m, context_mask=cm[:, :1]),
        "template": dict(x=x1, context=t1, mask=m1, context_mask=tm1),
        "tied_self": dict(x=x, mask=m, tie_dim=2),
        "tied_cross": dict(x=x, context=c, mask=m, context_mask=cm, tie_dim=2, attn_bias=r(B, h, i, jc)),
    }


def main():
    ref = load_reference()
    torch.manual_seed(31)
    attn = ref.Attention(**CFG).eval()
    st = randomize_zero_init_({k: v.clone() for k, v in attn.state_dict().items()})
    st = {k: _bf(v) for k, v in st.items()}
    attn.load_state_dict(st)
    fx = {"cfg": CFG, "state": st, "cases": {}}
    with torch.no_grad():
        for name, kw in cases().items():
            fx["cases"][name] = {"inputs": kw, "out": attn(**kw)}
    path = os.path.join(OUT, "attention_forward.pt")
    torch.save(fx, path)
    print(f"wrote attention_forward ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
