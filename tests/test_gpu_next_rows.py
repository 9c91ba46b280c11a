"""-m gpu: the extra-MSA stack (SURVEY.md 8(f) row n2): tied-query ("global") ingoing triangle attention
(alphafold2.py:142-151, 250, 367) and Alphafold2.forward(extra_msa=...) (alphafold2.py:789-798 incl. quirk Q11) -- against
fixtures from the unmodified reference.  The pre- / post-trunk glue kernels of row n1 (pair init, distogram head) are tested
element-wise in test_gpu_embed_heads.py."""
import pytest
import torch

from conftest import load_golden
from gpu_util import check, check_strict
from oracle import evoformer_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision", ["bf16", "strict"])
def test_evoformer_global_column_attn_golden(precision):
    import alphafold2_b200 as A
    fx = load_golden("evoformer_global_col")
    c, i = fx["cfg"], fx["inputs"]
    evo = A.Evoformer(depth=1, dim=c["dim"], seq_len=c["N"], heads=c["heads"], dim_head=c["dim_head"], attn_dropout=0.,
                      ff_dropout=0., global_column_attn=True)
    evo.load_state_dict(fx["state"])
    evo = A.set_precision(evo.cuda().eval(), precision)
    x, m = evo(i["x"].cuda(), i["m"].cuda(), mask=i["mask"].cuda(), msa_mask=i["msa_mask"].cuda())
    if precision == "strict":
        check_strict("strict/evoformer_global_col/golden/x", x, fx["out_fp32"][0])
        check_strict("strict/evoformer_global_col/golden/m", m, fx["out_fp32"][1])
    else:
        check("evoformer_global_col/golden/x", x, fx["out_fp64"][0], fx["out_autocast_bf16"][0])
        check("evoformer_global_col/golden/m", m, fx["out_fp64"][1], fx["out_autocast_bf16"][1])


@pytest.mark.parametrize("precision", ["bf16", "strict"])
def test_alphafold2_extra_msa_golden(precision):
    import alphafold2_b200 as A
    fx = load_golden("alphafold2_extra_msa")
    i = fx["inputs"]
    model = A.Alphafold2(**fx["cfg"])
    assert not model.load_state_dict(fx["state"], strict=False).unexpected_keys
    model = A.set_precision(model.cuda().eval(), precision)
    cu = {k: v.cuda() for k, v in i.items()}
    ret = model(cu["seq"], cu["msa"], mask=cu["mask"], msa_mask=cu["msa_mask"], extra_msa=cu["extra_msa"], extra_msa_mask=cu["extra_msa_mask"])
    if precision == "strict":
        check_strict("strict/alphafold2_extra_msa/golden/distance", ret.distance, fx["out_fp32"])
    else:
        check("alphafold2_extra_msa/golden/distance", ret.distance, fx["out_fp64"], fx["out_autocast_bf16"])
    with pytest.raises(ValueError):                       # the reference's default extra_msa_mask has the wrong rank (quirk Q11)
        model(cu["seq"], cu["msa"], mask=cu["mask"], msa_mask=cu["msa_mask"], extra_msa=cu["extra_msa"])


def test_tied_attention_big_shape_vs_oracle():
    """tied queries at a hot-path shape (d 256, H 8, dh 64, N 160): bf16 path vs the fp64 oracle."""
    import alphafold2_b200 as A
    from gpu_util import dev
    torch.manual_seed(2)
    d, H, dh, N = 256, 8, 64, 160
    ax = A.AxialAttention(dim=d, heads=H, dim_head=dh, row_attn=False, col_attn=True, accept_edges=True, global_query_attn=True)
    st = O.randomize_zero_init_({k: v.clone() for k, v in ax.state_dict().items()})
    ax.load_state_dict(st)
    ax = ax.cuda().eval()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, N, N, d, generator=g)
    mask1 = torch.ones(1, N, dtype=torch.bool); mask1[:, -20:] = False
    mask = mask1[:, :, None] & mask1[:, None, :]
    out = ax(x.cuda(), edges=x.cuda(), mask=mask.cuda())
    with torch.no_grad():
        ref = O.axial_attention(dev(st, torch.float64), "", x.double().cuda(), H, False, x.double().cuda(), mask.cuda(), global_query_attn=True)
    check("tied_attention/oracle/d256N160", out, ref)
