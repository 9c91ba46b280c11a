"""-m gpu: the persistent attention kernel's scheduling, element-wise against fp64.

The kernel launches min(items, SMs) CTAs, and each CTA walks the work items (b', 128 queries, head) with a stride of the
grid, fetching the next item's Q, gate and key codes while it computes the current one.  These tests cover what that
schedule can get wrong: item counts around the grid size, consecutive items of one CTA with different masks (the key codes
are double-buffered per item), and results that must not depend on the grid.  The reference and the per-element bound are
those of test_gpu_attention_kernel.py.
"""
import pytest
import torch

from gpu_util import check_bound
from test_gpu_attention_kernel import MASK_KINDS, _mask, _ops, _tok, attention_ref, make_inputs

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _mixed_mask(nbatch, n, g):
    """folded row b takes the mask of kind kinds[b % len(kinds)]: neighbouring rows differ, fully masked ones included"""
    kinds = MASK_KINDS if n > 128 else [k for k in MASK_KINDS if k not in ("first_block", "straddle")]   # those need n > 128
    m = torch.ones(nbatch, n, dtype=torch.bool)
    for k, kind in enumerate(kinds):
        part = _mask(kind, nbatch, n, g)
        if part is not None:
            m[k::len(kinds)] = part[k::len(kinds)]
    return m


def _ragged_suffix(nbatch, n, g):
    """folded row b is valid on a prefix of random length 1..n"""
    keep = torch.randint(1, n + 1, (nbatch,), generator=g)
    return torch.arange(n)[None, :] < keep[:, None]


def check_case(name, n, nbatch, heads, dh, row, bias, mask, seed, big=False):
    """mask: a kind of test_gpu_attention_kernel._mask, "mixed", "ragged" or None; returns the inputs and the output"""
    ops = _ops()
    qkv, gate, bt, g = make_inputs(n, nbatch, heads, dh, bias, big, seed)
    idx, tok_sb, tok_si = _tok(nbatch, n, row)
    if mask == "mixed":
        m_bn = _mixed_mask(nbatch, n, g)
    elif mask == "ragged":
        m_bn = _ragged_suffix(nbatch, n, g)
    elif mask is None:
        m_bn = torch.ones(nbatch, n, dtype=torch.bool)
    else:
        m_bn = _mask(mask, nbatch, n, g)
    mask_tok = None
    if m_bn is not None:
        mask_tok = torch.empty(n * nbatch, dtype=torch.bool, device="cuda")
        mask_tok[idx.flatten()] = m_bn.cuda().flatten()
    out = ops.attention_bf16(qkv, gate, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask_tok)
    ref, bnd = attention_ref(qkv, gate, bt, m_bn, n, nbatch, heads, dh, idx)
    check_bound(name, out, ref, bnd)
    return qkv, gate, bt, mask_tok, out


# items = nbatch * heads * ceil(n / 128), relative to the grid of one CTA per SM
GRID_CASES = {"half": lambda sm: (100, sm // 2, 1), "equal": lambda sm: (100, sm, 1), "one_above": lambda sm: (100, sm + 1, 1),
              "many": lambda sm: (257, 2 * sm + 5, 3)}


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
@pytest.mark.parametrize("items", list(GRID_CASES))
def test_persistent_item_counts(items, row, dh):
    """item counts below, equal to, one above and many times the persistent grid"""
    n, nbatch, heads = GRID_CASES[items](_sms())
    check_case(f"persist_items {items} n{n} b{nbatch} h{heads} dh{dh} {'row' if row else 'col'}", n, nbatch, heads, dh, row,
               True, "mixed", seed=13 * nbatch + dh)


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("mask", MASK_KINDS + ["mixed"])
@pytest.mark.parametrize("n,nbatch,heads,row", [(129, 45, 8, True), (257, 23, 8, False), (1024, 5, 8, True)])
def test_persistent_masks_per_item(n, nbatch, heads, row, mask, dh):
    """several items per CTA whose folded rows carry different masks; n ending mid key block and n = 1024"""
    check_case(f"persist_mask {mask} n{n} b{nbatch} h{heads} dh{dh} {'row' if row else 'col'}", n, nbatch, heads, dh, row,
               True, mask, seed=7 * n + dh)


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("row", [True, False], ids=["row", "col"])
def test_persistent_rows_alone_bitwise(row, dh):
    """every folded row of a launch of many items per CTA has the bits it has when launched alone (one CTA per item then),
    and two identical launches are bitwise identical"""
    ops = _ops()
    n, nbatch, heads = 257, 64, 8
    qkv, gate, bt, mask, out = check_case(f"persist_bitwise n{n} b{nbatch} dh{dh} {'row' if row else 'col'}", n, nbatch, heads,
                                          dh, row, True, "mixed", seed=29 + dh)
    idx, tok_sb, tok_si = _tok(nbatch, n, row)
    again = ops.attention_bf16(qkv, gate, n, nbatch, heads, dh, tok_sb, tok_si, bias=bt, mask=mask)
    assert torch.equal(again.view(torch.int16), out.view(torch.int16))
    for b in range(nbatch):
        ix = idx[b]
        one = ops.attention_bf16(qkv[ix].contiguous(), gate[ix].contiguous(), n, 1, heads, dh, n, 1, bias=bt,
                                 mask=mask[ix].contiguous())
        assert torch.equal(one.view(torch.int16), out[ix].view(torch.int16)), f"folded row {b} differs when run alone"


# the four attention calls of one Evoformer block at the C2 shape (N_res 256, MSA 128 x 256, heads 8, dim_head 64)
C2_CALLS = {"msa_row": (256, 128, True, True), "msa_col": (128, 256, False, False), "tri_start": (256, 256, True, True),
            "tri_end": (256, 256, False, True)}


@pytest.mark.parametrize("mask", [None, "ragged"], ids=["ones", "ragged_suffix"])
@pytest.mark.parametrize("call", list(C2_CALLS))
def test_persistent_c2_shapes(call, mask):
    n, nbatch, row, bias = C2_CALLS[call]
    check_case(f"persist_c2 {call} {mask or 'ones'}", n, nbatch, 8, 64, row, bias, mask, seed=len(call) + (mask is None))
